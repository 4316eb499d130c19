"""Instructions the synthesis recurrence issues per decoded sample, read from the SASS of the built library.

    python tools/synthesis_sass.py [--lib sela_b200/libsela_b200.so] [--out FILE.json]

For k_synthesise_segments and k_lpc_samples (kernels.cuh), runs `cuobjdump -sass` on the library and finds the
steady-state block of the recurrence (segment_block<false>, lpc.cuh): the straight-line run that holds kSegBlock (16)
SHFL.IDX, one broadcast of a finished sample each.  A run ends at a branch, a convergence barrier (BSSY / BSYNC) or
an exit; BRA.DIV is not an end, since it leaves only for the compiler's divergent fallback, which a converged warp
never takes.  Reports the instructions from one SHFL.IDX to the next (the SHFL.IDX counted once per sample), their
mean over the 15 gaps, the whole run over 16 samples, and the opcode mix per sample.  Needs the CUDA toolkit's
cuobjdump, no GPU.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
KERNELS = {
    "k_synthesise_segments": "_ZN8selab20021k_synthesise_segmentsENS_12DecodeParamsE",
    "k_lpc_samples": "_ZN8selab20013k_lpc_samplesEPKijPKhS1_Pi",
}
SAMPLES_PER_BLOCK = 16  # kSegBlock (lpc.cuh)
INSN = re.compile(r"/\*([0-9a-f]+)\*/\s+(.*?)\s*;")
ENDS_RUN = ("BRA", "BSSY", "BSYNC", "EXIT", "RET", "CALL", "JMP", "BREAK", "WARPSYNC")


def sass(lib, mangled):
    cmd = ["cuobjdump", "-sass", "-fun", mangled, lib]
    text = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
    out = []
    for line in text.splitlines():
        m = INSN.search(line)
        if not m:
            continue
        body = m.group(2)
        words = body.split()
        op = words[1] if words[0].startswith("@") else words[0]
        out.append((int(m.group(1), 16), op, body))
    if not out:
        raise SystemExit("synthesis_sass.py: %s not found in %s" % (mangled, lib))
    return out


def runs(insns):
    """Straight-line runs: split after every instruction that ends one (BRA.DIV excepted)."""
    cur = []
    for ins in insns:
        cur.append(ins)
        op = ins[1]
        if op.split(".")[0] in ENDS_RUN and not op.startswith("BRA.DIV"):
            yield cur
            cur = []
    if cur:
        yield cur


def steady_block(insns):
    """The run with exactly SAMPLES_PER_BLOCK SHFL.IDX (the first block, whose sample 0 is its residue, has one
    fewer).  Exactly one such run is expected."""
    found = [r for r in runs(insns) if sum(op == "SHFL.IDX" for _, op, _ in r) == SAMPLES_PER_BLOCK]
    if len(found) != 1:
        raise SystemExit("synthesis_sass.py: expected one run with %d SHFL.IDX, found %d"
                         % (SAMPLES_PER_BLOCK, len(found)))
    return found[0]


def analyse(lib, mangled):
    run = steady_block(sass(lib, mangled))
    idx = [i for i, (_, op, _) in enumerate(run) if op == "SHFL.IDX"]
    gaps = [b - a for a, b in zip(idx, idx[1:])]
    mix = collections.Counter(op for _, op, _ in run[idx[0] + 1:idx[-1] + 1])
    n = len(gaps)
    return {
        "block": "0x%x-0x%x" % (run[0][0], run[-1][0]),
        "per_sample_between_shfl_idx": sum(gaps) / n,
        "gaps": gaps,
        "whole_run_per_sample": len(run) / SAMPLES_PER_BLOCK,
        "opcode_mix_per_sample": {op: round(c / n, 2) for op, c in mix.most_common()},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "sela_b200", "libsela_b200.so"))
    ap.add_argument("--out", help="also write the numbers as JSON to this file")
    args = ap.parse_args()
    if not os.path.exists(args.lib):
        raise SystemExit("synthesis_sass.py: %s not built (python -m sela_b200.build)" % args.lib)
    result = {name: analyse(args.lib, mangled) for name, mangled in KERNELS.items()}
    for name, r in result.items():
        print("%s: steady-state block %s, %.2f instructions per sample between SHFL.IDX (whole run %.2f)"
              % (name, r["block"], r["per_sample_between_shfl_idx"], r["whole_run_per_sample"]))
        print("  gaps: %s" % " ".join(map(str, r["gaps"])))
        print("  " + ", ".join("%s %.2f" % kv for kv in r["opcode_mix_per_sample"].items()))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    sys.exit(main())
