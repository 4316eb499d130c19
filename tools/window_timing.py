"""What the window search (DESIGN.md 7.6) costs and saves against the default encode and the order search (-S), on
three workloads:

  BASELINE config 2/3     44.1 kHz stereo, 10 minutes, seed 1: 12 919 frames
  config-4-shaped file    48 kHz, 8 channels of independent sine + noise, 10 minutes, seed 2: 14 062 frames
  music-like stereo       tests/exact_window.music_like(40, 2, 11) (decaying harmonics + AR(8)-coloured noise),
                          tiled 50 times: 2 000 frames

For each: device time of DeviceCodec.encode, encode_search and encode_search_windows with masks 1 (Tukey(0.5)) and 31
(all five windows) (CUDA events, runs alternated in one process so that drift on a shared card hits all alike), device
time per kernel (torch.profiler, a pass of its own), and the words each writes.  On the music-like family the device's
words for both masks are also checked against the CPU model (tests/exact_window.py) on the 40 distinct frames.  The
card's name and power limit are read in the same call.
Usage: python tools/window_timing.py [reps] [out.json]   (prints one JSON line; also writes it to out.json if named)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sela_b200 import _lib, codec, synth  # noqa: E402
from sela_b200.device import DeviceCodec  # noqa: E402
import exact_window  # noqa: E402
from pairing_timing import card, event_ms, kernels_ms  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
OUT = sys.argv[2] if len(sys.argv) > 2 else None
MASKS = (1, 31)


def measure(name, pcm, ch):
    n_frames = pcm.shape[0] // 2048
    pcm = np.ascontiguousarray(pcm[:n_frames * 2048], np.int16).reshape(-1)
    out = {"workload": name, "frames": n_frames, "channels": ch}
    dc = DeviceCodec(n_frames, ch, device=0)
    t = torch.from_numpy(pcm).to(torch.device("cuda", 0))
    dc.encode(t)
    dc.check_status()
    out["words_default"] = int(dc.words_used.item())
    dc.encode_search(t)
    dc.check_status()
    out["words_search"] = words_search = int(dc.words_used.item())
    for mask in MASKS:
        dc.encode_search_windows(t, mask)
        dc.check_status()
        words, base = int(dc.words_used.item()), int(dc.base_words.item())
        assert base == words_search and words <= words_search
        out["words_windows_%d" % mask] = words
        out["window_units_%d" % mask] = int(dc.n_window.item())
        out["saving_vs_search_%d" % mask] = round(1 - words / words_search, 5)
        out["saving_vs_default_%d" % mask] = round(1 - words / out["words_default"], 5)
    forms = [("encode", dc.encode), ("encode_search", dc.encode_search)] + \
        [("encode_search_windows_%d" % m, lambda x, m=m: dc.encode_search_windows(x, m)) for m in MASKS]
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


def model_check(pcm, ch):
    """The device's words on `pcm` against the CPU model, for every mask."""
    out = {}
    for mask in MASKS:
        _, words, _, n_window = codec.encode_frames_search_windows(pcm, ch, mask)
        tables = [codec.analysis_window(i) for i in exact_window.mask_rows(mask)]
        model, _, _, _, chosen = exact_window.model_batch(pcm, ch, tables)
        want = sum(sum(c.words for c, _ in em) for em in model.values())
        out["mask_%d" % mask] = {"device_words": int(words.size), "model_words": int(want),
                                 "device_window_units": int(n_window), "model_window_units": int((chosen >= 0).sum())}
        assert words.size == want and n_window == (chosen >= 0).sum(), out
    return out


def main():
    _lib.init(0)
    music = exact_window.music_like(40, 2, 11)
    result = {"card": card(), "reps": REPS, "music_like_model_check": model_check(music, 2), "results": [
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
