"""What the channel pairing (DESIGN.md 7.4) and the search + pairing (7.5) cost and save, on three workloads:

  BASELINE config 2/3     44.1 kHz stereo, 10 minutes, seed 1: 12 919 frames
  config-4-shaped file    48 kHz, 8 channels of independent sine + noise, 10 minutes, seed 2: 14 062 frames
                          (the cost where nothing is gained)
  correlated 8 channels   one source in every channel with a gain per channel and small independent noise
                          (tests/exact_pairing.common_source), 2 000 frames: cost and gain

For each: device time of DeviceCodec.encode, encode_lossless, encode_search, encode_pairing and encode_search_pairing
(CUDA events, runs alternated in one process so that drift on a shared card hits all alike), device time per kernel
(torch.profiler, a pass of its own), and the words each writes.  The card's name and power limit are read in the same call.
Usage: python tools/pairing_timing.py [reps] [out.json]   (prints one JSON line; also writes it to out.json if named)"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sela_b200 import _lib, synth  # noqa: E402
from sela_b200.device import DeviceCodec  # noqa: E402
import exact_pairing  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
OUT = sys.argv[2] if len(sys.argv) > 2 else None


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        out["power_limit_max_sm_clock_sm_clock"] = r.stdout.strip()
    except OSError as e:
        out["power_limit_max_sm_clock_sm_clock"] = "nvidia-smi unavailable: %s" % e
    return out


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernels_ms(fn, reps):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if us:
            name = e.key.split("(")[0].split("<")[0].replace("void ", "").replace("selab200::", "")
            per[name] = round(per.get(name, 0) + us / 1e3 / reps, 4)
    return per


def measure(name, pcm, ch):
    n_frames = pcm.shape[0] // 2048
    pcm = np.ascontiguousarray(pcm[:n_frames * 2048], np.int16).reshape(-1)
    out = {"workload": name, "frames": n_frames, "channels": ch}
    codec = DeviceCodec(n_frames, ch, device=0)
    t = torch.from_numpy(pcm).to(torch.device("cuda", 0))
    codec.encode(t)
    codec.check_status()
    out["words_default"] = int(codec.words_used.item())
    codec.encode_lossless(t)
    codec.check_status()
    words_lossless = int(codec.words_used.item())
    codec.encode_pairing(t)
    codec.check_status()
    words_pairing, base_words = int(codec.words_used.item()), int(codec.base_words.item())
    assert base_words == words_lossless
    out["words_lossless"] = words_lossless
    out["words_pairing"] = words_pairing
    out["difference_subframes"] = int(codec.n_difference.item())
    out["saving"] = round(1 - words_pairing / words_lossless, 5)
    codec.encode_search(t)
    codec.check_status()
    words_search = int(codec.words_used.item())
    codec.encode_search_pairing(t)
    codec.check_status()
    words_sp, base_words = int(codec.words_used.item()), int(codec.base_words.item())
    assert base_words == words_search and words_sp <= words_search
    out["words_search"] = words_search
    out["words_search_pairing"] = words_sp
    out["search_pairing_difference_subframes"] = int(codec.n_difference.item())
    out["search_pairing_saving_vs_search"] = round(1 - words_sp / words_search, 5)
    out["search_pairing_saving_vs_default"] = round(1 - words_sp / out["words_default"], 5)
    forms = (("encode", codec.encode), ("encode_lossless", codec.encode_lossless), ("encode_search", codec.encode_search),
             ("encode_pairing", codec.encode_pairing), ("encode_search_pairing", codec.encode_search_pairing))
    runs = [[event_ms(lambda: fn(t), REPS) for _, fn in forms] for _ in range(3)]  # alternated
    codec.check_status()
    for i, (name_, fn) in enumerate(forms):
        out["device_%s_ms" % name_] = round(min(r[i] for r in runs), 3)
    out["runs_ms"] = [[round(v, 3) for v in r] for r in runs]
    for name_, fn in forms[1:]:
        out["kernels_%s_ms" % name_] = kernels_ms(lambda: fn(t), REPS)
    del codec, t
    torch.cuda.empty_cache()
    return out


def main():
    _lib.init(0)
    result = {"card": card(), "reps": REPS, "results": [
        measure("BASELINE config 2/3", synth.sine_noise(44100, 2, n_frames=12919, seed=1), 2),
        measure("config-4-shaped 10 min 8 ch, seed 2", synth.sine_noise(48000, 8, 600, seed=2), 8),
        measure("correlated 8 ch, 2000 frames, seed 7", exact_pairing.common_source(2000, 8, 7), 8),
    ]}
    result["card_after"] = card()
    line = json.dumps(result)
    if OUT:
        with open(OUT, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
