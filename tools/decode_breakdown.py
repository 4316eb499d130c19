"""Where the decoder's time goes, launch by launch, on bench.py's workload.

    python tools/decode_breakdown.py [--reps 30] [--out FILE.json]

Encodes the 10-minute seed-1 stereo synthetic of bench.py once (12 919 frames), then
  * times the whole decode call (selab200_decode_frames_device) with CUDA events over --reps calls;
  * times every kernel and memset of the same calls from the CUDA activity records of torch.profiler
    (a run of its own, so that tracing does not slow the event-timed run), summed per launch name and
    divided by the number of calls;
  * prints the card's name, power limit and SM clocks next to the numbers;
  * counts, on the CPU from the descriptors, how many of the multiply slots the synthesis kernel issues are
    taps of a predictor: useful taps (sum of the orders) over issued slots (lanes x taps per lane x 2 048
    samples, the same factor everywhere), for the former three-class plan (four subframes per warp, 8 lanes
    of 4 / 8 / 16 taps) and for the segment plan of k_decode_plan (kernels.cuh), restated in segment_plan below.
Needs a CUDA device; there is no CPU path for the timings.
"""
import argparse
import collections
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from sela_b200 import _lib, synth  # noqa: E402

FRAME = 2048
TAPS_PER_LANE = 8       # kTapsPerLane (kernels.cuh)


def segment_width(order):
    """Lanes of a subframe's segment: ceil(order / TAPS_PER_LANE), at least one."""
    return np.maximum(1, -(-np.asarray(order) // TAPS_PER_LANE))


def segment_plan(orders):
    """The warp templates k_decode_plan computes from the width counts: the widest width left starts a warp,
    which is then filled greedily with the widest segments that still fit; the template is repeated as often as
    the counts allow.  Returns [(repeats, {width: copies})] and the number of warps."""
    counts = np.bincount(segment_width(orders), minlength=32).tolist()
    templates, warps = [], 0
    while any(counts):
        room, take = 32, {}
        for w in range(len(counts) - 1, 0, -1):
            k = min(counts[w], room // w)
            if k:
                take[w] = k
                room -= k * w
        n = min(counts[w] // k for w, k in take.items())
        for w, k in take.items():
            counts[w] -= n * k
        templates.append((n, take))
        warps += n
    return templates, warps


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or "nvidia-smi unavailable"


def class_plan_slots(orders):
    """Issued tap slots per sample of the three-class plan: classes <= 28 / <= 56 / <= 112 (4 / 8 / 16 taps per
    lane), each class padded to whole warps of four subframes, 32 lanes per warp."""
    cls = np.where(orders <= 28, 0, np.where(orders <= 56, 1, 2))
    slots = 0
    for c, tpl in enumerate((4, 8, 16)):
        warps = (int((cls == c).sum()) + 3) // 4
        slots += warps * 32 * tpl
    return slots


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", help="also write the numbers as JSON to this file")
    args = ap.parse_args()
    assert args.reps >= 20, "at least 20 repetitions"

    import torch
    from torch.profiler import ProfilerActivity, profile
    from sela_b200.device import DeviceCodec

    if not torch.cuda.is_available():
        raise SystemExit("decode_breakdown.py: no CUDA device")
    pcm_np = synth.sine_noise(44100, 2, seconds=600, seed=1)
    n_frames = pcm_np.shape[0] // FRAME
    pcm = torch.from_numpy(pcm_np.reshape(-1)).cuda()
    out = torch.empty_like(pcm)
    codec = DeviceCodec(n_frames, 2)
    codec.encode(pcm)
    torch.cuda.synchronize()
    codec.check_status()
    n_words = int(codec.words_used.item())

    def decode():
        codec.decode(out, n_words)

    for _ in range(5):
        decode()
    torch.cuda.synchronize()
    codec.check_status()
    assert torch.equal(out, pcm), "round trip"

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.reps + 1)]
    ev[0].record()
    for i in range(args.reps):
        decode()
        ev[i + 1].record()
    torch.cuda.synchronize()
    per_call = [ev[i].elapsed_time(ev[i + 1]) for i in range(args.reps)]

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            decode()
        torch.cuda.synchronize()
    launches = collections.defaultdict(lambda: [0, 0.0])
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        name = e.name.split("(")[0].replace("void ", "").replace("selab200::", "")
        launches[name][0] += 1
        launches[name][1] += e.device_time_total / 1e3   # us -> ms
    stages = {k: {"launches_per_call": n / args.reps, "ms_per_call": t / args.reps} for k, (n, t) in launches.items()}

    descs = codec.descs.cpu().numpy().view(_lib.DESC_DTYPE)
    orders = descs["lpc_order"].astype(np.int64)
    useful = int(orders.sum())
    cls_slots = class_plan_slots(orders)
    templates, seg_warps = segment_plan(orders)
    seg_slots = seg_warps * 32 * TAPS_PER_LANE
    result = {
        "card": card(),
        "workload": "bench.py's: 44.1 kHz stereo, 10 min sine+noise, seed 1, %d frames, %d subframes" % (n_frames, orders.size),
        "reps": args.reps,
        "decode_ms": {"mean": float(np.mean(per_call)), "min": float(np.min(per_call)), "max": float(np.max(per_call))},
        "launches": stages,
        "tap_slots": {
            "useful_taps_per_sample": useful,
            "three_classes": {"issued_slots_per_sample": cls_slots, "fill": useful / cls_slots},
            "segments": {"taps_per_lane": TAPS_PER_LANE, "warps": seg_warps, "templates": len(templates),
                         "issued_slots_per_sample": seg_slots, "fill": useful / seg_slots,
                         "lane_fill": int(segment_width(orders).sum()) / (seg_warps * 32)},
        },
    }
    print("card: %s" % result["card"])
    print("decode call: %.3f ms mean (min %.3f, max %.3f) over %d calls" % (
        result["decode_ms"]["mean"], result["decode_ms"]["min"], result["decode_ms"]["max"], args.reps))
    total = sum(s["ms_per_call"] for s in stages.values())
    for k, s in sorted(stages.items(), key=lambda kv: -kv[1]["ms_per_call"]):
        print("  %-48s %5.1f launches  %8.4f ms  %5.1f %%" % (k[:48], s["launches_per_call"], s["ms_per_call"],
                                                           100 * s["ms_per_call"] / total))
    print("  %-48s %14s %8.4f ms (sum of kernel times)" % ("", "", total))
    ts = result["tap_slots"]
    print("tap slots: useful %d per sample; three classes %d issued (%.1f %%); segments of %d taps per lane: "
          "%d warps, %d issued (%.1f %%), lanes used %.1f %%" % (
              useful, cls_slots, 100 * ts["three_classes"]["fill"], TAPS_PER_LANE, seg_warps,
              ts["segments"]["issued_slots_per_sample"], 100 * ts["segments"]["fill"], 100 * ts["segments"]["lane_fill"]))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
