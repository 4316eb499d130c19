"""What random access (DESIGN.md 7.8) costs against the two ways a loader reads clips without it, on two workloads:

  many files      256 stereo 30 s files (synth.sine_noise, seed k for file k), 2 048 one-second clips at seeded random
                  (file, start)
  one long file   BASELINE config 2/3 (44.1 kHz stereo, 10 minutes, seed 1), 64 one-second clips

For each, the device time (CUDA events on the current stream around a call that synchronises before it returns) and
the wall time of:
  (a) ClipDecoder.decode_device: one call, every covered frame decoded once, clips cut out on the device;
  (b) the host workaround: per clip, the covered frames' bytes behind a hand-made 15-byte header, decode_container,
      slice, upload;
  (c) decode_container of every file, then slice and upload.
Runs are alternated in one process; every output is compared with (c)'s.  Also frames_decoded against the frames the
clips cover, and, in a pass of its own, the device time per kernel of (a) (torch.profiler) with k_clip_gather's bytes
(read + written) over its time against 3.35 TB/s.  The card's name and power limit are read in the same call.
Usage: python tools/clip_timing.py [reps] [out.json]   (prints one JSON line; also writes it to out.json if named)"""
import json
import os
import struct
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sela_b200 import ClipDecoder, codec, synth  # noqa: E402
from pairing_timing import card, kernels_ms  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
OUT = sys.argv[2] if len(sys.argv) > 2 else None
FRAME, SECOND = 2048, 44100
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


def measure(name, blobs, ks, starts):
    length = SECOND
    offsets = [codec.container_frame_offsets(b)[1] for b in blobs]
    dec = ClipDecoder(blobs)

    def a():
        return dec.decode_device(ks, starts, length)

    def b():
        clips = []
        for k, s in zip(ks, starts):
            blob, off = blobs[k], offsets[k]
            f0, f1 = s // FRAME, (s + length - 1) // FRAME + 1
            head = bytes(blob[:11]) + struct.pack("<I", f1 - f0)
            _, pcm = codec.decode_container(np.frombuffer(head + bytes(blob[off[f0]:off[f1]]), np.uint8))
            at = s - f0 * FRAME
            clips.append(pcm.reshape(-1, 2)[at:at + length])
        return torch.from_numpy(np.stack(clips)).to(DEV)

    def c():
        whole = [codec.decode_container(blob)[1].reshape(-1, 2) for blob in blobs]
        return torch.from_numpy(np.stack([whole[k][s:s + length] for k, s in zip(ks, starts)])).to(DEV)

    ref = c()
    assert torch.equal(a(), ref) and torch.equal(b(), ref)
    covered = len({(k, f) for k, s in zip(ks, starts) for f in range(s // FRAME, (s + length - 1) // FRAME + 1)})
    out = {"workload": name, "files": len(blobs), "clips": len(ks), "clip_samples": length,
           "frames_decoded": dec.frames_decoded, "frames_covered": covered,
           "frames_in_files": sum(len(o) - 1 for o in offsets)}
    runs = {"a_clip_decoder": [], "b_host_workaround": [], "c_whole_files": []}
    for _ in range(REPS):  # alternated
        for key, fn in zip(runs, (a, b, c)):
            runs[key].append(timed(fn)[1:])
    for key, v in runs.items():
        out[key + "_device_ms"] = round(float(np.median([x[0] for x in v])), 3)
        out[key + "_wall_ms"] = round(float(np.median([x[1] for x in v])), 3)
    per = kernels_ms(a, REPS)
    out["a_kernels_ms"] = per
    gather = per.get("k_clip_gather", 0)
    moved = 2 * len(ks) * length * 2 * 2  # every output byte read once and written once
    if gather:
        out["k_clip_gather_GBps"] = round(moved / (gather * 1e-3) / 1e9, 1)
        out["k_clip_gather_share_of_3_35_TBps"] = round(moved / (gather * 1e-3) / 3.35e12, 3)
    dec.close()
    return out


def main():
    rng = np.random.default_rng(7)
    blobs = [codec.encode_container(synth.sine_noise(SECOND, 2, seconds=30, seed=k), 2, SECOND) for k in range(256)]
    total = codec.container_info(blobs[0])["n_frames"] * FRAME
    ks = rng.integers(0, 256, 2048).tolist()
    starts = rng.integers(0, total - SECOND + 1, 2048).tolist()
    results = {"card": card(), "workloads": [measure("256 stereo 30 s files, 2048 one-second clips", blobs, ks, starts)]}
    blob = codec.encode_container(synth.sine_noise(SECOND, 2, seconds=600, seed=1), 2, SECOND)
    total = codec.container_info(blob)["n_frames"] * FRAME
    starts = rng.integers(0, total - SECOND + 1, 64).tolist()
    results["workloads"].append(measure("BASELINE config 2/3, 64 one-second clips", [blob], [0] * 64, starts))
    line = json.dumps(results)
    print(line)
    if OUT:
        with open(OUT, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
