#!/usr/bin/env python3
"""Generate the golden vectors under tests/golden/ from the UNMODIFIED reference.

Run in the build container (needs /root/reference; builds oracle/_ref via oracle/Makefile):

    python tests/golden/make_golden.py

The reference ships no golden files (SURVEY.md 4), so these are outputs of the reference's own
classes (frame::FrameEncoder / FrameDecoder through oracle/ref_shim.cpp) on seeded inputs.
They travel to the GPU box, where /root/reference does not exist.

  golden_frames.npz
    pcm_<case>      int16 [n_frames*2048, channels]   input
    descs_<case>    structured (32-byte descriptor)   reference encoder output
    words_<case>    uint32                            reference encoder output (arena)
    decoded_<case>  int16                             reference DECODER output for (descs, words)

  lpc_first_order.npy   float64 [128]   the reference's firstOrderCoefficients table (src/include/lpc.hpp),
                                         written when the reference tree is named: make_golden.py REFERENCE_TREE
"""
import pathlib
import re
import sys

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import oracle_lib as ol  # noqa: E402
import signals  # noqa: E402
from sela_b200 import synth  # noqa: E402


def cases():
    out = {}
    st = synth.sine_noise(44100, 2, n_frames=6, seed=1)                       # BASELINE config 2/3 shape
    st[2048 * 2:2048 * 4, 1] = st[2048 * 2:2048 * 4, 0] - (st[2048 * 2:2048 * 4, 1] >> 5)
    st[2048 * 4:2048 * 5, 1] = st[2048 * 4:2048 * 5, 0]
    out["stereo"] = st
    out["mono_config1"] = synth.config1_frame().astype(np.int16).reshape(-1, 1)  # BASELINE config 1
    out["oct"] = synth.sine_noise(48000, 8, n_frames=2, seed=2)                # config 4 shape
    fam = signals.families()
    names = sorted(fam)
    out["edge_mono"] = np.concatenate([fam[n] for n in names]).astype(np.int16).reshape(-1, 1)
    out["edge_stereo"] = np.concatenate(
        [np.stack([fam[n], fam[names[(i * 5 + 2) % len(names)]]], axis=1) for i, n in enumerate(names)]).astype(np.int16)
    out["three"] = synth.sine_noise(32000, 3, n_frames=2, seed=9)
    # Two frames of the config-4-shaped 10-minute file (48 kHz, 8 channels, seed 2) on which the REFERENCE is
    # not lossless: its decoder departs from the source at sample 1 of one channel (frame 8975 channel 1,
    # frame 13577 channel 4; encoder and decoder round the prediction differently when the Q35 sum lands
    # exactly on a half, SURVEY.md 7.3).  The decoded_* array pins what the reference decoder returns.
    big = synth.sine_noise(48000, 8, 600, seed=2)
    out["oct_reference_lossy"] = np.concatenate([big[8975 * 2048:8976 * 2048], big[13577 * 2048:13578 * 2048]])
    return out


def write_lpc_table(ref_tree):
    text = (pathlib.Path(ref_tree) / "src" / "include" / "lpc.hpp").read_text()
    m = re.search(r"firstOrderCoefficients\[128\]\s*=\s*\{([^}]*)\}", text)
    vals = np.array([float(t) for t in m.group(1).replace("\n", " ").split(",") if t.strip()], np.float64)
    assert vals.size == 128
    np.save(pathlib.Path(__file__).parent / "lpc_first_order.npy", vals)


def main():
    if len(sys.argv) > 1:
        write_lpc_table(sys.argv[1])
    assert ol.have_ref() or pathlib.Path("/root/reference").exists(), "needs the reference tree"
    R = ol.load("ref")
    assert R.kind == "reference"
    blob = {}
    for name, pcm in cases().items():
        ch = pcm.shape[1]
        descs, words = R.encode_frames(pcm, ch)
        blob["pcm_" + name] = pcm
        blob["descs_" + name] = descs
        blob["words_" + name] = words
        blob["decoded_" + name] = R.decode_frames(descs, words, ch)
        print("%-14s ch=%d frames=%d words=%d lossless=%s" % (
            name, ch, pcm.shape[0] // 2048, words.size, np.array_equal(blob["decoded_" + name], pcm.reshape(-1))))
    np.savez_compressed(pathlib.Path(__file__).parent / "golden_frames.npz", **blob)


if __name__ == "__main__":
    main()
