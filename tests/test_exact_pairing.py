"""Pins the CPU model of the channel pairing (exact_pairing.py, DESIGN.md 7.4) without a GPU: its candidates against
the existing models and the compiled reference, its choice against a brute force over every parent vector, and its
streams against the port's and the reference's decoders."""
import numpy as np
import pytest

import exact_lossless as xl
import exact_pairing as xp
import oracle_lib as ol
from sela_b200 import synth

FRAME = 2048


@pytest.fixture(scope="module")
def O():
    return ol.load("port")


def _planes(pcm, ch):
    return np.asarray(pcm, np.int64).reshape(-1, FRAME, ch).transpose(0, 2, 1)


def test_stereo_candidate_is_the_stereo_difference_unit(O):
    """Candidate (0, 1) of a stereo frame is the base's difference unit, which is what the lossless model and the
    reference encoder code: same words, same residues."""
    pcm = xp.common_source(2, 2, 5)
    for f, planes in enumerate(_planes(pcm, 2)):
        m = xp.model_frame(O, planes)
        u = m["cands"][0, 1]
        d = xl.analyse(O, planes[0] - planes[1])
        assert not d.tie and u.words == d.words and np.array_equal(u.res, d.res) and u.order == d.order
        for D in [O] + ([ol.load("ref")] if ol.have_ref() else []):
            descs, words = D.encode_frames(pcm[f * FRAME:(f + 1) * FRAME].reshape(-1), 2)
            if int(descs[1]["subframe_type"]) == 1:
                assert int(descs[1]["refl_words"]) + int(descs[1]["res_words"]) == u.words
                assert int(descs[1]["lpc_order"]) == u.order
                kr, wr = O.rice_encode(u.res)
                at = int(descs[1]["res_offset"])
                assert np.array_equal(words[at:at + wr.size], wr)


@pytest.mark.parametrize("name", [f[0] for f in xp.families()])
def test_model_streams_decode_back(O, name):
    """2, 3, 4, 6 and 8 channels: the model's stream decodes back under the port and the compiled reference, is never
    larger than the base, and the families pair as they are built to."""
    _, pcm, ch = next(f for f in xp.families() if f[0] == name)
    model = xp.model_batch(O, pcm, ch)
    descs, words = xp.pack(O, model, ch)
    for D in [O] + ([ol.load("ref")] if ol.have_ref() else []):
        assert np.array_equal(D.decode_frames(descs, words, ch), pcm.reshape(-1))
    for m in model.values():
        assert m["words"] <= m["base_words"]
        for c, p in enumerate(m["par"]):
            assert p == c or (m["par"][p] == p and (p, c) not in m["tied"])
    pars = [m["par"] for m in model.values()]
    if name == "common_source_8":   # several children on one parent
        assert all(sum(p != c for c, p in enumerate(par)) >= 4 for par in pars)
        assert any(max(par.count(p) for p in set(par)) >= 3 for par in pars)
        assert sum(m["words"] for m in model.values()) < 0.9 * sum(m["base_words"] for m in model.values())
    if name == "dual_mono_in_six":
        assert all(par[4] == 2 or par[2] == 4 for par in pars)
    if name == "equal_and_negated":
        assert all(par[:2] == (0, 0) and par[2:] == (2, 3) for par in pars)
        assert all(not m["emitted"][1][0].res.any() for m in model.values())


def test_independent_noise_keeps_the_lossless_stream(O):
    pcm = synth.sine_noise(48000, 8, n_frames=2, seed=4).astype(np.int16)
    model = xp.model_batch(O, pcm, 8)
    assert all(m["par"] == tuple(range(8)) and m["words"] == m["base_words"] for m in model.values())
    base = xl.model_batch(O, pcm, 8, every=True)
    for f, m in model.items():
        for (u, t, _), (v, tv) in zip(m["emitted"], base[f][0]):
            assert (t, u.order, u.words) == (tv, v.order, v.words) and np.array_equal(u.res, v.res)


def test_choice_equals_brute_force():
    """Random cost tables with equal entries and invalid ones, C <= 4: rule 3 and every tie-break of rule 4."""
    rng = np.random.default_rng(7)
    hit_diff_break = hit_lex_break = 0
    for trial in range(1500):
        C = int(rng.integers(2, 5))
        I = [int(v) for v in rng.integers(3, 7, C)]
        D = [[None if p == c or rng.random() < 0.2 else int(rng.integers(1, 6)) for c in range(C)] for p in range(C)]
        for c in range(C):
            if rng.random() < 0.1:
                I[c] = None
        if all(v is None for v in I):
            continue
        got, want = xp.assign(I, D), xp.assign_brute(I, D)
        assert got == want, (I, D)
        if got is None:     # no valid assignment: cannot happen in the encoder, whose base is one
            continue
        par, total = got
        alone = sum(v for v in I if v is not None) if all(v is not None for v in I) else None
        hit_diff_break += alone == total and par == tuple(range(C))
        hit_lex_break += sum(p != c for c, p in enumerate(par)) > 0
    assert hit_diff_break > 20 and hit_lex_break > 200


def test_tie_break_examples():
    assert xp.assign([5, 5], [[None, 5], [5, None]]) == ((0, 1), 10)          # equal words: fewest differences
    assert xp.assign([5, 5], [[None, 4], [4, None]]) == ((0, 0), 9)           # equal words and count: lexicographic
    assert xp.assign([5, 5], [[None, 4], [3, None]]) == ((1, 1), 8)           # ch0 against ch1 wins
    assert xp.assign([5, None], [[None, 9], [1, None]]) == ((0, 0), 14)       # a tied channel cannot be a parent
    assert xp.assign([5, 5, 5], [[None, 1, 1], [1, None, 1], [1, 1, None]]) == ((0, 0, 0), 7)
    assert xp.assign([5, 5, 5], [[None, None, 1], [1, None, 2], [1, 1, None]]) == ((2, 2, 2), 7)


def test_pairing_entry_points_have_no_cpu_fallback():
    import ctypes as C
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from sela_b200 import _lib
    import sela_b200
    L = _lib.lib()
    assert L.selab200_init(0) == -1
    pcm = np.zeros(2 * 2048, np.int16)
    descs = np.zeros(2, _lib.DESC_DTYPE)
    words = np.zeros(8192, np.uint32)
    used, base, nd = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    blob = np.zeros(1 << 16, np.uint8)
    assert L.selab200_encode_frames_pairing(pcm.ctypes.data, 1, 2, descs.ctypes.data, words.ctypes.data, words.size,
                                            C.addressof(used), C.addressof(base), C.addressof(nd)) == -7
    assert L.selab200_encode_container_pairing(pcm.ctypes.data, 1, 2, 44100, 16, blob.ctypes.data, blob.size,
                                               C.addressof(used), C.addressof(base), C.addressof(nd)) == -7
    assert L.selab200_encode_pairing_workspace_bytes(10, 8) > L.selab200_encode_lossless_workspace_bytes(10, 8)
    with pytest.raises(sela_b200.SelaB200Error):
        sela_b200.encode_frames_pairing(pcm, 2)
