"""What the guided order search (DESIGN.md 7.7) costs and saves against the default encode and the order search (-S),
on three workloads:

  BASELINE config 2/3     44.1 kHz stereo, 10 minutes, seed 1: 12 919 frames
  config-4-shaped file    48 kHz, 8 channels of independent sine + noise, 10 minutes, seed 2: 14 062 frames
  music-like stereo       tests/exact_window.music_like(40, 2, 11) (decaying harmonics + AR(8)-coloured noise),
                          tiled 50 times: 2 000 frames

For each: device time of DeviceCodec.encode, encode_search and encode_search_guided with K = 1, 2, 4, 8 (CUDA events,
runs alternated in one process so that drift on a shared card hits all alike), the words each writes and the share
of -S's saving over the default encode each keeps, and in a pass of its own the device time per kernel
(torch.profiler).  The card's name and power limit are read in the same call.
Usage: python tools/search_guided_timing.py [reps] [out.json]   (prints one JSON line; also writes it to out.json if
named)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sela_b200 import _lib, synth  # noqa: E402
from sela_b200.device import DeviceCodec  # noqa: E402
import exact_window  # noqa: E402
from pairing_timing import card, event_ms, kernels_ms  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
OUT = sys.argv[2] if len(sys.argv) > 2 else None
KS = (1, 2, 4, 8)


def measure(name, pcm, ch):
    n_frames = pcm.shape[0] // 2048
    pcm = np.ascontiguousarray(pcm[:n_frames * 2048], np.int16).reshape(-1)
    out = {"workload": name, "frames": n_frames, "channels": ch}
    dc = DeviceCodec(n_frames, ch, device=0)
    t = torch.from_numpy(pcm).to(torch.device("cuda", 0))
    dc.encode(t)
    dc.check_status()
    out["words_default"] = words_default = int(dc.words_used.item())
    dc.encode_search(t)
    dc.check_status()
    out["words_search"] = words_search = int(dc.words_used.item())
    for K in KS:
        dc.encode_search_guided(t, K)
        dc.check_status()
        words = int(dc.words_used.item())
        assert int(dc.ref_words.item()) == words_default and words_search <= words <= words_default
        out["words_guided_%d" % K] = words
        out["share_of_search_saving_%d" % K] = round((words_default - words) / max(words_default - words_search, 1), 4)
    out["search_saving_vs_default"] = round(1 - words_search / words_default, 5)
    forms = [("encode", dc.encode), ("encode_search", dc.encode_search)] + \
        [("encode_search_guided_%d" % K, lambda x, K=K: dc.encode_search_guided(x, K)) for K in KS]
    runs = [[event_ms(lambda: fn(t), REPS) for _, fn in forms] for _ in range(3)]  # alternated
    dc.check_status()
    for i, (name_, _) in enumerate(forms):
        out["device_%s_ms" % name_] = round(min(r[i] for r in runs), 3)
    out["runs_ms"] = [[round(v, 3) for v in r] for r in runs]
    for name_, fn in forms[1:]:
        out["kernels_%s_ms" % name_] = kernels_ms(lambda: fn(t), 1)
    del dc, t
    torch.cuda.empty_cache()
    return out


def main():
    _lib.init(0)
    music = exact_window.music_like(40, 2, 11)
    result = {"card": card(), "reps": REPS, "results": [
        measure("BASELINE config 2/3", synth.sine_noise(44100, 2, n_frames=12919, seed=1), 2),
        measure("config-4-shaped 10 min 8 ch, seed 2", synth.sine_noise(48000, 8, 600, seed=2), 8),
        measure("music-like stereo, 40 frames x 50", np.tile(music, (50, 1)), 2),
    ]}
    result["card_after"] = card()
    line = json.dumps(result)
    if OUT:
        with open(OUT, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
