"""What the lossless encode costs, in one call, on three workloads:

  BASELINE config 2/3   44.1 kHz stereo, 10 minutes, seed 1: 12 919 frames (nothing to repair)
  config-4-shaped file  48 kHz, 8 channels, 10 minutes, seed 2: 14 062 frames, two subframes to repair
  worst case            4 096 frames of 8 channels, every frame one of the two golden lossy frames

For each: DeviceCodec.encode against DeviceCodec.encode_lossless (CUDA events), and selab200_encode_container
against selab200_encode_container_lossless (pinned buffers), alternated so that drift on a shared host hits both
alike.  The card's name and power limit are read in the same call.
Usage: python tools/lossless_timing.py [reps] [out.json]   (prints one JSON line; also writes it to out.json if named)"""
import ctypes as C
import json
import os
import pathlib
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sela_b200 import _lib, synth  # noqa: E402
from sela_b200.device import DeviceCodec  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
OUT = sys.argv[2] if len(sys.argv) > 2 else None
GOLD = pathlib.Path(ROOT) / "tests" / "golden" / "golden_frames.npz"


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        out["power_limit_and_max_sm_clock"] = r.stdout.strip()
    except OSError as e:
        out["power_limit_and_max_sm_clock"] = "nvidia-smi unavailable: %s" % e
    return out


def event_ms(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def wall_ms(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(t)


def measure(name, pcm, ch, rate):
    L = _lib.lib()
    n_frames = pcm.shape[0] // 2048
    pcm = np.ascontiguousarray(pcm[:n_frames * 2048], np.int16).reshape(-1)
    out = {"workload": name, "frames": n_frames, "channels": ch}

    codec = DeviceCodec(n_frames, ch, device=0)
    t = torch.from_numpy(pcm).to(torch.device("cuda", 0))
    codec.encode_lossless(t)
    codec.check_status()
    out["recoded_subframes"] = int(codec.lossless_report().size)
    dev = []
    for _ in range(3):  # alternated
        dev.append((event_ms(lambda: codec.encode(t), REPS), event_ms(lambda: codec.encode_lossless(t), REPS)))
    codec.check_status()
    enc, ll = min(r[0] for r in dev), min(r[1] for r in dev)
    out["device_encode_ms"] = round(enc, 3)
    out["device_encode_lossless_ms"] = round(ll, 3)
    out["device_overhead"] = round(ll / enc - 1, 4)
    # where the difference goes: device time per kernel and call (torch.profiler, a pass of its own)
    for key, fn in (("kernels_encode_ms", codec.encode), ("kernels_encode_lossless_ms", codec.encode_lossless)):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(REPS):
                fn(t)
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            if us:
                name = e.key.split("(")[0].split("<")[0].replace("void ", "").replace("selab200::", "")
                per[name] = round(per.get(name, 0) + us / 1e3 / REPS, 4)
        out[key] = per
    del codec, t
    torch.cuda.empty_cache()

    cap = L.selab200_container_bound(n_frames, ch)
    h_pcm = L.selab200_host_alloc(pcm.size * 2)
    h_blob = L.selab200_host_alloc(cap)
    h_rep = L.selab200_host_alloc(n_frames * ch * 16)
    C.memmove(h_pcm, pcm.ctypes.data, pcm.size * 2)
    used, n_rep = C.c_size_t(0), C.c_size_t(0)

    def plain():
        _lib.check(L.selab200_encode_container(h_pcm, n_frames, ch, rate, 16, h_blob, cap, C.addressof(used)))

    def lossless():
        _lib.check(L.selab200_encode_container_lossless(h_pcm, n_frames, ch, rate, 16, h_blob, cap, C.addressof(used),
                                                        h_rep, n_frames * ch, C.addressof(n_rep)))

    host = [(wall_ms(plain, REPS), wall_ms(lossless, REPS)) for _ in range(3)]
    p, q = min(r[0] for r in host), min(r[1] for r in host)
    out["encode_container_ms"] = round(p, 3)
    out["encode_container_lossless_ms"] = round(q, 3)
    out["host_overhead"] = round(q / p - 1, 4)
    assert n_rep.value == out["recoded_subframes"]
    for h in (h_pcm, h_blob, h_rep):
        L.selab200_host_free(h)
    return out


def main():
    _lib.init(0)
    lossy = np.load(GOLD)["pcm_oct_reference_lossy"].reshape(2, 2048, 8)
    result = {"card": card(), "reps": REPS, "results": [
        measure("BASELINE config 2/3", synth.sine_noise(44100, 2, n_frames=12919, seed=1), 2, 44100),
        measure("config-4-shaped 10 min 8 ch, seed 2", synth.sine_noise(48000, 8, 600, seed=2), 8, 48000),
        measure("worst case: 4096 golden lossy frames", np.concatenate([lossy] * 2048).reshape(-1, 8), 8, 48000),
    ]}
    line = json.dumps(result)
    if OUT:
        with open(OUT, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
