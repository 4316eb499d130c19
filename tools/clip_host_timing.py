"""What host-resident containers (DESIGN.md 7.10) cost against device-resident ones, and against opening the files a
call touches, on three workloads:

  many files      256 stereo 30 s files (synth.sine_noise, seed k for file k), 2 048 one-second clips, every channel
  one long file   BASELINE config 2/3 (44.1 kHz stereo, 10 minutes, seed 1), 64 one-second clips, every channel
  8 channels      8 config-4-shaped files (48 kHz, 8 channels, 60 s, seeds 0..7), 512 one-second clips of channel 0

For each, the medians of alternated runs of device time (CUDA events around a call that synchronises before it
returns) and wall time of:
  (a) ClipDecoder.decode_device on device-resident containers;
  (b) the same on host-resident containers (ClipDecoder(host_resident=True));
  (c) per call, ClipDecoder over just the files the clips touch (each opened from host bytes: its whole image
      uploaded), decode_device, close.
Every output is compared with (a)'s.  Also: bytes_fetched against the bytes (c) uploads, checked against the runs
of the fetch rule computed here; in a pass of its own (torch.profiler) the device time per kernel of (b), with
k_clip_fetch's bytes over its time; the same runs copied by torch, one copy_ per run from pinned tensors into one
device buffer; the device memory each way of opening the files takes (torch.cuda.mem_get_info before and after:
other processes share the card, so this is approximate); and the open time per GB of both opens.  The pinned host-to-device
rate of tools/pcie_probe.py is measured in the same call, and the card's name and power limit are read with it.
Usage: python tools/clip_host_timing.py [reps] [out.json]   (prints one JSON line; also writes it to out.json)"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sela_b200 import ClipDecoder, codec, synth  # noqa: E402
from pairing_timing import card, kernels_ms  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
OUT = sys.argv[2] if len(sys.argv) > 2 else None
FRAME = 2048
DEV = torch.device("cuda", 0)


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b), (time.perf_counter() - t0) * 1e3


def subframe_ranges(blob):
    """Per frame, per position: the byte range [at, end) the unpack reads (the walk of the file's frame headers)."""
    ch, n_frames = blob[10], int.from_bytes(bytes(blob[11:15]), "little")
    at, out = 15, []
    for _ in range(n_frames):
        at += 4
        frame = []
        for _ in range(ch):
            rn = int.from_bytes(bytes(blob[at + 4:at + 6]), "little")
            n = int.from_bytes(bytes(blob[at + 7 + 4 * rn + 1:at + 7 + 4 * rn + 3]), "little")
            frame.append((at + 7, at + 7 + 4 * rn + 5 + 4 * n + 3))
            at += 7 + 4 * rn + 5 + 4 * n
        out.append(frame)
    return out


def fetch_runs(ranges, ks, starts, length, positions):
    """The fetch rule's runs (k, lo, hi) for the default group sizes; positions(k, f): the positions decoded (None:
    every one, in groups of whole frames)."""
    keys = sorted({(k, f) for k, s in zip(ks, starts) for f in range(s // FRAME, (s + length - 1) // FRAME + 1)})
    runs, rows = [], 0
    ch0 = len(ranges[keys[0][0]][0])
    for i, (k, f) in enumerate(keys):
        pos = range(len(ranges[k][f])) if positions is None else positions(k, f)
        cut = i % max(1, 32768 // ch0) == 0 if positions is None else (i == 0 or rows + len(pos) > 32768)
        rows = 0 if cut else rows
        rows += len(pos)
        for j, p in enumerate(pos):
            a, b = ranges[k][f][p]
            lo, hi = a & ~15, (b + 15) & ~15
            if runs and not (cut and j == 0) and runs[-1][0] == k and lo <= runs[-1][2]:
                runs[-1] = (k, runs[-1][1], max(runs[-1][2], hi))
            else:
                runs.append((k, lo, hi))
    return runs


def measure(name, blobs, ks, starts, length, channels):
    out = {"workload": name, "files": len(blobs), "clips": len(ks), "clip_samples": length, "channels": channels,
           "file_bytes": sum(len(b) for b in blobs)}
    free0 = torch.cuda.mem_get_info(DEV)[0]
    _, _, t_open = timed(lambda: ClipDecoder(blobs).close())          # warm: the first open pays for the pool
    dev, _, t_open = timed(lambda: ClipDecoder(blobs))
    free_dev = torch.cuda.mem_get_info(DEV)[0]
    host, _, t_open_host = timed(lambda: ClipDecoder(blobs, host_resident=True))
    free_host = torch.cuda.mem_get_info(DEV)[0]
    gb = out["file_bytes"] / 1e9
    out["open_ms_per_GB"] = round(t_open / gb, 1)
    out["open_host_ms_per_GB"] = round(t_open_host / gb, 1)
    out["device_MB_taken_by_open"] = {"device_resident": (free0 - free_dev) >> 20,
                                      "host_resident": (free_dev - free_host) >> 20}
    kw = dict(channels=channels)

    def a():
        return dev.decode_device(ks, starts, length, **kw)

    def b():
        return host.decode_device(ks, starts, length, **kw)

    touched = sorted(set(ks))
    index = {k: i for i, k in enumerate(touched)}

    def c():
        with ClipDecoder([blobs[k] for k in touched]) as d:
            return d.decode_device([index[k] for k in ks], starts, length, **kw)

    ref = a()
    assert torch.equal(b(), ref) and torch.equal(c(), ref)
    out["frames_decoded"], out["subframes_decoded"] = host.frames_decoded, host.subframes_decoded
    assert (dev.frames_decoded, dev.subframes_decoded) == (host.frames_decoded, host.subframes_decoded)
    out["bytes_fetched"] = host.bytes_fetched
    out["bytes_uploaded_c"] = sum(len(blobs[k]) for k in touched)

    # the runs of the fetch rule, checked against the decoder's count, and the same runs copied by torch
    ranges = [subframe_ranges(bl) for bl in blobs]
    positions = None if channels is None else (lambda k, f: [0])     # channel 0 of an independent-channel encode
    runs = fetch_runs(ranges, ks, starts, length, positions)
    assert sum(hi - lo for _, lo, hi in runs) == host.bytes_fetched
    out["runs"] = len(runs)
    pinned = [torch.frombuffer(bytearray(bytes(bl) + bytes(64)), dtype=torch.uint8).pin_memory() for bl in blobs]
    stage = torch.empty(host.bytes_fetched, dtype=torch.uint8, device=DEV)

    def torch_copy():
        at = 0
        for k, lo, hi in runs:
            stage[at:at + hi - lo].copy_(pinned[k][lo:hi], non_blocking=True)
            at += hi - lo

    timing = {"a_device_resident": [], "b_host_resident": [], "c_open_per_call": [], "torch_copy_runs": []}
    for _ in range(REPS):  # alternated
        for key, fn in zip(timing, (a, b, c, torch_copy)):
            timing[key].append(timed(fn)[1:])
    for key, v in timing.items():
        out[key + "_device_ms"] = round(float(np.median([x[0] for x in v])), 3)
        out[key + "_wall_ms"] = round(float(np.median([x[1] for x in v])), 3)
    per = kernels_ms(b, REPS)
    out["b_kernels_ms"] = per
    fetch = per.get("k_clip_fetch", 0)
    if fetch:
        out["k_clip_fetch_GBps"] = round(host.bytes_fetched / (fetch * 1e-3) / 1e9, 2)
    dev.close()
    host.close()
    return out


def pcie_h2d():
    """The host-to-device lines of tools/pcie_probe.py, run in this call."""
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "pcie_probe.py")], capture_output=True, text=True,
                       timeout=600)
    return [line for line in p.stdout.splitlines() if "H2D" in line]


def main():
    rng = np.random.default_rng(7)
    results = {"card": card(), "workloads": []}
    blobs = [codec.encode_container(synth.sine_noise(44100, 2, seconds=30, seed=k), 2, 44100) for k in range(256)]
    total = codec.container_info(blobs[0])["n_frames"] * FRAME
    ks = rng.integers(0, 256, 2048).tolist()
    starts = rng.integers(0, total - 44100 + 1, 2048).tolist()
    results["workloads"].append(measure("256 stereo 30 s files, 2048 one-second clips", blobs, ks, starts, 44100, None))
    blob = codec.encode_container(synth.sine_noise(44100, 2, seconds=600, seed=1), 2, 44100)
    total = codec.container_info(blob)["n_frames"] * FRAME
    starts = rng.integers(0, total - 44100 + 1, 64).tolist()
    results["workloads"].append(measure("BASELINE config 2/3, 64 one-second clips", [blob], [0] * 64, starts, 44100,
                                        None))
    rng = np.random.default_rng(11)
    blobs = [codec.encode_container(synth.sine_noise(48000, 8, seconds=60, seed=k), 8, 48000) for k in range(8)]
    total = codec.container_info(blobs[0])["n_frames"] * FRAME
    ks = rng.integers(0, 8, 512).tolist()
    starts = rng.integers(0, total - 48000 + 1, 512).tolist()
    results["workloads"].append(measure("8 config-4-shaped 60 s files, 512 one-second clips of channel 0", blobs, ks,
                                        starts, 48000, [0]))
    results["pcie_probe_h2d"] = pcie_h2d()
    line = json.dumps(results)
    print(line)
    if OUT:
        with open(OUT, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
