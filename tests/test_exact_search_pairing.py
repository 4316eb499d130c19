"""Pins the CPU model of the search + pairing (exact_search_pairing.py, DESIGN.md 7.5) without a GPU: its choice
against a brute force over every parent vector, its candidates against the per-unit search model, its bounds against
the search and pairing models, its streams against the port's and the compiled reference's decoders, and the size of
its workspace."""
import numpy as np
import pytest

import analysis_corpus
import exact_lossless as xl
import exact_pairing as xp
import exact_search as xs
import exact_search_pairing as xsp
import oracle_lib as ol
import test_encode_workspace
from sela_b200 import _lib, synth

FRAME = 2048


@pytest.fixture(scope="module")
def O():
    return ol.load("port")


@pytest.fixture(scope="module")
def family_models():
    return {name: (pcm, ch, xsp.model_batch(pcm, ch)) for name, pcm, ch in xp.families()}


def test_choice_on_searched_tables_equals_brute_force(family_models):
    n = 0
    for name, (pcm, ch, (model, _, _, _, _)) in family_models.items():
        if ch > 4:
            continue
        for v in model.values():
            assert xp.assign(v["I"], v["D"]) == xp.assign_brute(v["I"], v["D"]) == (v["par"], v["words"]), name
            n += 1
    assert n >= 9


def test_mono_is_the_search_model():
    pcm = synth.sine_noise(44100, 1, n_frames=3, seed=5).astype(np.int16)
    model = xsp.model_batch(pcm, 1)[0]
    want, _ = xs.model_batch(ol.load("port"), pcm, 1)
    for f, v in model.items():
        (u, t, parent), = v["emitted"]
        (w, tw), = want[f]
        assert (t, parent, u.order, u.words) == (tw, 0, w.order, w.words) and np.array_equal(u.res, w.res)
        assert v["words"] == v["base_words"] == w.words


@pytest.mark.parametrize("name", [f[0] for f in xp.families()])
def test_model_streams_decode_back_and_are_never_larger_than_the_search(O, family_models, name):
    """2, 3, 4, 6 and 8 channels: the stream decodes back under the port and the compiled reference, and no frame is
    larger than the search model's."""
    pcm, ch, (model, _, _, _, _) = family_models[name]
    descs, words = xsp.pack(O, model, ch)
    for D in [O] + ([ol.load("ref")] if ol.have_ref() else []):
        assert np.array_equal(D.decode_frames(descs, words, ch), pcm.reshape(-1))
    search, _ = xs.model_batch(O, pcm, ch)
    for f, v in model.items():
        assert v["base_words"] == sum(u.words for u, _ in search[f])
        assert v["words"] <= v["base_words"]
        for c, p in enumerate(v["par"]):
            assert p == c or v["par"][p] == p


def _never_larger_than_the_pairing(O, pcm, ch, model):
    pairing = xp.model_batch(O, pcm, ch)
    recoded = xl.model_batch(O, pcm, ch)
    n = 0
    for f, v in model.items():
        if f not in recoded:
            assert v["words"] <= pairing[f]["words"], f
            n += 1
    return n


@pytest.mark.parametrize("name", [f[0] for f in xp.families()])
def test_never_larger_than_the_pairing_where_nothing_is_repaired_families(O, family_models, name):
    pcm, ch, (model, _, _, _, _) = family_models[name]
    assert _never_larger_than_the_pairing(O, pcm, ch, model) >= 1


@pytest.mark.parametrize("batch", ["three_channels", "stereo_pairs"])
def test_never_larger_than_the_pairing_where_nothing_is_repaired_corpus(O, batch):
    _, pcm, ch = next(b for b in analysis_corpus.batches() if b[0] == batch)
    pcm = np.asarray(pcm).reshape(-1, FRAME, ch)[::7].reshape(-1, ch)
    model = xsp.model_batch(pcm, ch)[0]
    assert _never_larger_than_the_pairing(O, pcm, ch, model) >= 3


def test_candidate_winners_equal_the_per_unit_search(O, family_models):
    for name in ("common_source_3", "equal_and_negated", "full_scale_opposite_3", "common_source_stereo"):
        pcm, ch, (model, m, index, Qc, refc) = family_models[name]
        planes = np.asarray(pcm, np.int64).reshape(-1, FRAME, ch).transpose(0, 2, 1)
        for (f, p, c), row in index.items():
            win, ref, words, tie = xs.search_unit(O, planes[f, p] - planes[f, c], Qc[row], refc[row])
            u = model[f]["cands"][p, c]
            assert (u.order, u.words) == (win.order, win.words) and np.array_equal(u.res, win.res), (name, f, p, c)
            assert np.array_equal(m["words"][row], words) and np.array_equal(m["tie"][row], tie)


def test_workspace_bytes_follow_the_layout():
    """The search layout with every region padded, the pairing tables, and a 416-byte SearchUnit per (frame, p, c)."""
    L = _lib.lib()
    a = lambda n: (n + 255) // 256 * 256
    for (n_frames, ch), (plain, lossless, search, pairing) in test_encode_workspace.SIZES.items():
        n_units = n_frames * (3 if ch == 2 else ch)
        n_pairs = n_frames * ch * ch
        want = plain + a(416 * n_units) + (pairing - lossless) + a(416 * n_pairs)
        assert L.selab200_encode_search_pairing_workspace_bytes(n_frames, ch) == want, (n_frames, ch)
        assert want >= max(search, pairing - lossless + plain)
