"""What choosing channels in the clip decode (DESIGN.md 7.9) saves against decoding every channel and picking after:

  8 channels   8 config-4-shaped files (48 kHz, 8 channels of independent sine + noise, 60 s, seeds 0..7),
               512 one-second clips at seeded random (file, start): channel 0 alone, as int16
  stereo       256 stereo 30 s files (44.1 kHz, synth.sine_noise, seed k for file k), 2 048 one-second clips:
               channel 0 alone, channel 1 alone, and the float32 mean of both

Against, in each case, ClipDecoder.decode_device over every channel as int16 followed by the torch slice (or the
torch convert-and-mean).  Runs are alternated in one process; their medians are reported as device time (CUDA events
around a call that synchronises before it returns) and wall time.  Every output is checked against the full decode
first.  Also frames_decoded and subframes_decoded, and, in passes of their own, the device time per kernel of both
(torch.profiler), with k_clip_gather_select's bytes over its time: each selected row's samples read once (the parent
rows of difference-coded channels are not counted) and the output written once.  The card's name and power limit are
read in the same call.
Usage: python tools/clip_select_timing.py [reps] [out.json]   (prints one JSON line; also writes it to out.json)"""
import json
import os
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


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), (time.perf_counter() - t0) * 1e3


def measure(name, dec, ks, starts, length, sel, mean):
    dtype = torch.float32 if mean else torch.int16

    def chosen():
        return dec.decode_device(ks, starts, length, channels=sel, dtype=dtype, mean=mean)

    def full_then_torch():
        x = dec.decode_device(ks, starts, length)
        if mean:
            return x.to(torch.int32).sum(-1, keepdim=True).float() / float(32768 * x.shape[-1])
        return x[..., sel].contiguous()

    ref = full_then_torch()
    full_frames, full_subframes = dec.frames_decoded, dec.subframes_decoded
    assert torch.equal(chosen(), ref)
    out = {"workload": name, "clips": len(ks), "clip_samples": length, "channels": sel, "mean": mean,
           "frames_decoded": dec.frames_decoded, "subframes_decoded": dec.subframes_decoded,
           "full_subframes_decoded": full_subframes}
    assert dec.frames_decoded == full_frames
    runs = {"chosen": [], "full_then_torch": []}
    for _ in range(REPS):  # alternated
        runs["chosen"].append(timed(chosen))
        runs["full_then_torch"].append(timed(full_then_torch))
    for key, v in runs.items():
        out[key + "_device_ms"] = round(float(np.median([x[0] for x in v])), 3)
        out[key + "_wall_ms"] = round(float(np.median([x[1] for x in v])), 3)
    per = kernels_ms(chosen, REPS)
    out["chosen_kernels_ms"] = per
    out["full_kernels_ms"] = kernels_ms(full_then_torch, REPS)
    gather = per.get("k_clip_gather_select", 0)
    n_sel = dec.channels if sel is None else len(sel)
    moved = len(ks) * length * (2 * n_sel + (4 if mean else 2 * len(sel)))
    if gather:
        out["k_clip_gather_select_GBps"] = round(moved / (gather * 1e-3) / 1e9, 1)
        out["k_clip_gather_select_share_of_3_35_TBps"] = round(moved / (gather * 1e-3) / 3.35e12, 3)
    return out


def main():
    rng = np.random.default_rng(11)
    results = {"card": card(), "workloads": []}
    blobs = [codec.encode_container(synth.sine_noise(48000, 8, seconds=60, seed=k), 8, 48000) for k in range(8)]
    total = codec.container_info(blobs[0])["n_frames"] * FRAME
    ks = rng.integers(0, 8, 512).tolist()
    starts = rng.integers(0, total - 48000 + 1, 512).tolist()
    with ClipDecoder(blobs) as dec:
        results["workloads"].append(measure("8 config-4-shaped 60 s files, 512 one-second clips", dec, ks, starts,
                                            48000, [0], False))
    blobs = [codec.encode_container(synth.sine_noise(44100, 2, seconds=30, seed=k), 2, 44100) for k in range(256)]
    total = codec.container_info(blobs[0])["n_frames"] * FRAME
    ks = rng.integers(0, 256, 2048).tolist()
    starts = rng.integers(0, total - 44100 + 1, 2048).tolist()
    name = "256 stereo 30 s files, 2048 one-second clips"
    with ClipDecoder(blobs) as dec:
        for sel, mean in (([0], False), ([1], False), (None, True)):
            results["workloads"].append(measure(name, dec, ks, starts, 44100, sel, mean))
    line = json.dumps(results)
    print(line)
    if OUT:
        with open(OUT, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
