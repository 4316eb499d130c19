"""GPU parity of the second-generation Rice decoder (sela_b200/csrc/rice_vs.cuh): streams cut into S parts
by k_rice_split_index and decoded by k_rice_decode_vc, for every S, against the reference's decoder
(rice::RiceDecoder, src/rice/rice_decoder.cpp:11-52) -- including the streams it must hand back to the
general parser (periodic streams that never resynchronise, long unary runs, streams with more symbols per part than it keeps checkpoints for)."""
import numpy as np
import pytest

import oracle_lib as ol
import sela_b200
from exact_rice import pack_stream, zigzag
from rice_families import synthetic_streams
from sela_b200 import _lib, synth
from sela_b200.device import rice_decode_frames

pytestmark = pytest.mark.gpu
FRAME = 2048
SPLITS = ["0", "1", "2", "4", "8", "16"]


@pytest.fixture(scope="module")
def O():
    return ol.best()


def build_batch(streams, channels=1, gap_words=(0, 1, 2, 3, 5)):
    """streams: list of (k, words). Returns descriptors + arena with the streams at every 16-byte phase."""
    n = len(streams)
    assert n % channels == 0
    descs = np.zeros(n, _lib.DESC_DTYPE)
    arena = []
    at = 0
    for i, (k, w) in enumerate(streams):
        pad = gap_words[i % len(gap_words)]
        arena.append(np.full(pad, 0xFFFFFFFF, np.uint32))     # all-ones filler: must never be parsed
        at += pad
        d = descs[i]
        d["channel"] = i % channels
        d["parent_channel"] = i % channels
        d["lpc_order"] = 1
        d["refl_rice_param"] = 0
        d["refl_words"] = 1
        d["refl_offset"] = at
        arena.append(np.zeros(1, np.uint32))
        at += 1
        d["res_rice_param"] = k
        d["res_words"] = w.size
        d["samples"] = FRAME
        d["res_offset"] = at
        arena.append(w)
        at += w.size
    return descs, np.concatenate(arena)


@pytest.mark.parametrize("split", SPLITS)
def test_split_decoder_synthetic_streams(O, monkeypatch, split):
    monkeypatch.setenv("SELAB200_RICE_SPLIT", split)
    rng = np.random.default_rng(11)
    streams = synthetic_streams(rng) * 3                      # > one warp of streams at every S
    descs, arena = build_batch([(k, w) for k, w, _ in streams])
    res, flagged = rice_decode_frames(descs, arena, 1)
    for i, (k, w, us) in enumerate(streams):
        want = O.rice_decode(w, k, FRAME)
        assert np.array_equal(res[i], want), (split, i, k)
    u = np.asarray(streams[0][2], np.uint64)
    assert np.array_equal(res[0], ((u >> np.uint64(1)).astype(np.int64) ^ -(u & np.uint64(1)).astype(np.int64)).astype(np.int32))
    if split not in ("0",):
        assert flagged < len(streams)                          # the fast decoder did most of the work


@pytest.mark.parametrize("split", SPLITS)
def test_split_decoder_encoded_batch(O, monkeypatch, split):
    """Streams produced by the encoder (stereo, difference coding, all order classes)."""
    monkeypatch.setenv("SELAB200_RICE_SPLIT", split)
    pcm = synth.sine_noise(44100, 2, n_frames=150, seed=3)
    pcm[FRAME * 20:FRAME * 40] //= 64                          # a quiet passage: small k
    pcm[FRAME * 60:FRAME * 70] = 0                             # silence: k = 0, 64-word streams
    pcm[FRAME * 80:FRAME * 90, 1] = pcm[FRAME * 80:FRAME * 90, 0] + 3   # difference-coded frames
    d, w = O.encode_frames(pcm, 2)
    res, flagged = rice_decode_frames(d, w, 2)
    for i in range(0, d.size, 7):
        want = O.rice_decode(w[int(d[i]["res_offset"]):int(d[i]["res_offset"]) + int(d[i]["res_words"])],
                             int(d[i]["res_rice_param"]), FRAME)
        assert np.array_equal(res[i], want), (split, i)
    out = sela_b200.decode_frames(d, w, 2)                     # and the whole decode chain on top of it
    assert np.array_equal(out, O.decode_frames(d, w, 2))
    if split not in ("0",):
        assert flagged <= d.size // 4, flagged


def test_split_decoder_truncated_stream_is_rejected(O, monkeypatch):
    for split in ("1", "8"):
        monkeypatch.setenv("SELAB200_RICE_SPLIT", split)
        rng = np.random.default_rng(4)
        us = zigzag(np.round(rng.laplace(0, 900, FRAME)).astype(np.int64))
        w = pack_stream(us, 11)
        descs, arena = build_batch([(11, w[:w.size // 2])] * 4)
        with pytest.raises(_lib.SelaB200Error) as e:
            rice_decode_frames(descs, arena, 1)
        assert e.value.status == -6
