"""Pins the CPU model of the window search (exact_window.py, DESIGN.md 7.6) without a GPU: the window table against
its formulas, the windowed analysis against exact_analysis with a window of all ones, the choice against a brute force
over every (analysis, order), the bound against the order search, its streams against the port's and the compiled
reference's decoders, and the size of its workspace."""
import numpy as np
import pytest

import analysis_corpus
import exact_analysis as xa
import exact_search as xs
import exact_window as xw
import oracle_lib as ol
import signals
import test_encode_workspace
from sela_b200 import _lib, codec, synth

FRAME = 2048


@pytest.fixture(scope="module")
def O():
    return ol.load("port")


def _tukey(n, p):
    w = np.ones(n)
    L = int(np.floor(p * (n - 1) / 2))
    i = np.arange(L)
    v = 0.5 * (1.0 - np.cos(np.pi * i / L))
    w[:L] = v
    w[n - L:] = v[::-1]
    return w


def test_window_table_equals_its_formulas():
    n = np.arange(FRAME)
    half = np.zeros(FRAME)
    want = [_tukey(FRAME, 0.5), _tukey(FRAME, 0.25), 0.5 - 0.5 * np.cos(2 * np.pi * n / (FRAME - 1)),
            np.concatenate([_tukey(FRAME // 2, 0.5), half[:FRAME // 2]]),
            np.concatenate([half[:FRAME // 2], _tukey(FRAME // 2, 0.5)])]
    for i, w in enumerate(want):
        got = codec.analysis_window(i)
        ulps = np.abs(got.view(np.int64) - w.view(np.int64))
        assert ulps.max() <= 1, (i, int(ulps.argmax()))
        assert got[0] == 0.0 and (got >= 0).all() and (got <= 1).all()
    assert (codec.analysis_window(0)[511:1537] == 1.0).all() and codec.analysis_window(0)[510] < 1.0
    for bad in (-1, 5):
        with pytest.raises(_lib.SelaB200Error) as e:
            codec.analysis_window(bad)
        assert e.value.status == -3


def test_all_ones_window_is_the_reference_analysis():
    S = np.array([v for v in signals.families().values()] + list(signals.random_frames(12, 3)), np.int64)
    S = np.concatenate([S, analysis_corpus.units(xw.music_like(2, 2, 4), 2)])
    a = xa.analyse(S)
    b = xw.analyse_windowed(S, np.ones(FRAME))
    for f in ("mean", "ac", "k"):
        assert np.all(xa.same_bits(a[f], b[f])), f
    q, _ = xs.all_q(S)
    assert np.array_equal(q, b["q"])


def test_silent_window_quantises_to_zero():
    """A window that sees only silence: ac[0] = 0, NaN through the recursion, every q 0."""
    s = np.zeros((1, FRAME), np.int64)
    for i in range(5):
        b = xw.analyse_windowed(s, codec.analysis_window(i))
        assert b["ac"][0, 0] == 1.0 and np.isnan(b["ac"][0, 1:]).all() and (b["q"] == 0).all()


def test_window_q_is_clamped_to_the_decoders_range():
    """Frame 3 of random_frames(12, 5) is near-singular under every window: its windowed Schur recursion rounds to
    |k| > 1, and the record keeps q clamped to [-64, 63]."""
    S = signals.random_frames(12, 5)[3:4].astype(np.int64)
    for i in range(5):
        raw = xw.analyse_windowed(S, codec.analysis_window(i))["q"]
        assert ((raw < -64) | (raw > 63)).any(), i
        assert np.array_equal(xw.window_q(S, codec.analysis_window(i)), np.clip(raw, -64, 63))


def test_quantiser_clamps_before_narrowing():
    """An infinite or huge k clamps to the end of the range, as the device's saturating conversion and clamp give;
    NaN quantises to 0."""
    k = np.zeros((5, 100))
    k[:, 2] = [np.inf, -np.inf, 1e12, -1e12, np.nan]
    k[:, 0] = [5.0, -5.0, np.inf, 0.0, np.nan]   # coefficient 0: sqrt(k + 1), NaN below -1
    k[:, 1] = [-5.0, 5.0, -np.inf, 0.0, np.nan]
    q = xw.quantise_clamped(k)
    assert q[:, 2].tolist() == [63, -64, 63, -64, 0]
    assert q[:, 0].tolist() == [63, 0, 63, 26, 0] and q[:, 1].tolist() == [63, 0, 63, 26, 0]
    assert q.dtype == np.int32 and (q[:, 3:] == 0).all()


def test_orders_outside_the_domain_are_never_chosen():
    """Frame 9 of random_frames(12, 5) under the Hann window: its q drive the step-up past the int64 conversion's
    domain.  Such orders count as tied, and the record's winner is none of them."""
    S = signals.random_frames(12, 5)[9:10].astype(np.int64)
    mw = xw._search_records(S, xw.window_q(S, codec.analysis_window(2)))
    assert (~mw["domain"]).any()
    assert mw["tie"][~mw["domain"]].all()
    assert mw["domain"][0, mw["order"][0] - 1]


def _brute(m, mw, u, n):
    """The rule of 7.6 by enumeration: every tie-free (window, order) of the unit against its order search words."""
    S = min(int(m["words"][u, o]) for o in range(xs.MAX_ORDER) if not m["tie"][u, o])
    best = None
    for w in range(n):
        r = u * n + w
        for o in range(xs.MAX_ORDER):
            if not mw["tie"][r, o] and (best is None or (int(mw["words"][r, o]), w, o + 1) < best):
                best = (int(mw["words"][r, o]), w, o + 1)
    return (best[1], best[2], best[0]) if best[0] < S else (None, None, S)


@pytest.fixture(scope="module")
def music():
    pcm = xw.music_like(3, 2, 11)
    tables = [codec.analysis_window(i) for i in range(5)]
    return pcm, xw.model_batch(pcm, 2, tables)


def test_choice_equals_brute_force(music):
    pcm, (model, base_words, mw, Qw, chosen) = music
    _, _, m, _, _ = xs.model_batch_all(pcm, 2)
    n = Qw.shape[1]
    for u in range(chosen.size):
        w, o, words = _brute(m, mw, u, n)
        assert (-1 if w is None else w) == chosen[u], u
    assert (chosen >= 0).sum() >= 3


def test_never_more_than_the_order_search_and_equal_where_no_window_wins(music):
    pcm, (model, base_words, mw, Qw, chosen) = music
    base, _, m, _, _ = xs.model_batch_all(pcm, 2)
    per = 3
    for f, em in model.items():
        assert sum(c.words for c, _ in em) <= base_words[f]
        if (chosen[f * per:(f + 1) * per] < 0).all():
            assert [(c.order, c.words, t) for c, t in em] == [(c.order, c.words, t) for c, t in base[f]]
    saved = sum(base_words.values()) - sum(sum(c.words for c, _ in em) for em in model.values())
    assert saved > 0


def test_no_window_better_is_the_order_search(O):
    """Every window all ones: each record equals the order search of the plain analysis, which is never strictly
    better than its own winner, so the model is the order search's."""
    pcm = synth.sine_noise(44100, 2, n_frames=2, seed=8)
    model, base_words, mw, _, chosen = xw.model_batch(pcm, 2, np.ones((1, FRAME)))
    base, _ = xs.model_batch(O, pcm, 2)
    assert (chosen < 0).all()
    for f, em in model.items():
        assert [(c.order, c.words, t) for c, t in em] == [(c.order, c.words, t) for c, t in base[f]]


@pytest.mark.parametrize("ch", [1, 2, 3, 8])
def test_model_streams_decode_back(O, ch):
    pcm = xw.music_like(2 if ch <= 3 else 1, ch, 20 + ch)
    tables = [codec.analysis_window(i) for i in (0, 3)]
    model, base_words, _, _, chosen = xw.model_batch(pcm, ch, tables)
    descs, words = xw.pack(O, model, ch)
    for D in [O] + ([ol.load("ref")] if ol.have_ref() else []):
        assert np.array_equal(D.decode_frames(descs, words, ch), pcm.reshape(-1))
    xw.check_frames(O, descs, words, pcm, ch, model)
    assert words.size <= sum(base_words.values())


def test_workspace_bytes_follow_the_layout():
    """The search layout with every region padded, a 416-byte SearchUnit per (unit, window) and an 8-byte key per
    unit."""
    L = _lib.lib()
    a = lambda n: (n + 255) // 256 * 256
    for (n_frames, ch), (plain, _, search, _) in test_encode_workspace.SIZES.items():
        n_units = n_frames * (3 if ch == 2 else ch)
        for mask in (1, 2, 5, 31):
            n = bin(mask).count("1")
            want = plain + a(416 * n_units) + a(416 * n_units * n) + a(8 * n_units)
            assert L.selab200_encode_search_windows_workspace_bytes(n_frames, ch, mask) == want, (n_frames, ch, mask)
            assert want >= search
