"""The CPU model of the guided order search (exact_search_guided.py) pinned on its own: the estimates against the
definition written out in scalar Python, k = -1 and equal estimates, K = 100 against the order search's model, the
bounds against the order search and the default encoder, decoding of 1, 2, 3 and 8 channels, and the size of the
workspace."""
import numpy as np

import analysis_corpus
import exact_search as xs
import exact_search_guided as xg
import oracle_lib as ol
import signals
import test_encode_workspace
from sela_b200 import _lib, synth

FRAME = 2048


def _corpus_units(per_batch=6):
    out = []
    for name, pcm, ch in analysis_corpus.batches():
        u = analysis_corpus.units(pcm, ch)
        out.append(u[np.linspace(0, u.shape[0] - 1, per_batch).astype(int)])
    return np.concatenate(out)


def test_estimates_are_the_scalar_definition_bit_for_bit():
    S = analysis_corpus.all_units()
    Q, _ = xs.all_q(S[::7])
    E = xg.estimates(Q)
    for n, q in enumerate(Q):
        assert np.array_equal(E[n].view(np.uint64), xg.estimates_scalar(q).view(np.uint64)), n
    # np.cumprod along the orders gives the same doubles: the products run left to right
    A = 1.0 - xs.dequantised(Q) * xs.dequantised(Q)
    P = np.cumprod(np.concatenate([np.ones((len(Q), 1)), (A[:, 0] * A[:, 1])[:, None], A[:, 2:]], axis=1), axis=1)
    Rs = np.cumprod(np.full(100, xg.R))
    assert np.array_equal((P * Rs).view(np.uint64), E.view(np.uint64))
    assert (E >= 0).all() and (E[:, 0] == xg.R).all()


def test_coefficient_minus_one_gives_zero_estimates_and_the_lower_order_first():
    """q = -64 at index i >= 2 dequantises to k = -1: E is 0 from order i + 1 on, and among those equal estimates the
    lower order ranks first."""
    q = np.full(100, 5, np.int32)
    q[[0, 1]] = [20, -10]
    for i in (2, 39, 40, 63, 64, 98, 99):
        qi = q.copy()
        qi[i] = -64
        E = xg.estimates(qi[None])
        assert (E[0, i:] == 0).all() and (E[0, :i] > 0).all()
        r = xg.ranks(E)[0]
        assert list(r[i:]) == list(range(100 - i))
        for K in (1, 2, 4):
            L = set(np.nonzero(xg.listed(E, [3], K)[0])[0] + 1)
            zero = set(range(i + 1, min(i + 1 + K, 101)))
            assert {1, 3} | zero <= L, (i, K)
            if len(zero) == K:
                assert L == {1, 3} | zero, (i, K)


def test_equal_estimates_list_the_lower_order():
    """Equal estimates at two orders rank by order between them."""
    E = np.array([[0.5, 0.25, 0.25, 0.75] + [1.0] * 96])
    r = xg.ranks(E)[0]
    assert (r[1], r[2], r[0], r[3]) == (0, 1, 2, 3)
    assert list(np.nonzero(xg.listed(E, [4], 1)[0])[0] + 1) == [1, 2, 4]


def _batches():
    return [("random", signals.random_frames(6, 3).astype(np.int16).reshape(-1), 1),
            ("baseline", synth.sine_noise(44100, 2, n_frames=6, seed=1).reshape(-1), 2),
            ("three", synth.sine_noise(48000, 3, n_frames=3, seed=4).reshape(-1), 3),
            ("eight", synth.sine_noise(48000, 8, n_frames=2, seed=2).reshape(-1), 8)]


def test_k100_is_the_order_search_and_every_k_lies_between_it_and_the_default():
    for name, pcm, ch in _batches():
        S, Q, refs = xg.unit_inputs(pcm, ch)
        table = (S, Q, refs, xs.search_units(S, Q, refs))
        m = table[3]
        full, full_ref = xs.model_batch_all(pcm, ch)[:2]
        prev = None
        for K in (1, 2, 4, 8, 100):
            model, ref_words, g = xg.model_batch(pcm, ch, K, table=table)
            assert ref_words == full_ref
            u = np.arange(len(refs))
            w = m["words"][u, g["order"] - 1]
            assert (w >= m["words"][u, m["order"] - 1]).all(), (name, K)
            assert (m["tie"][u, refs - 1] | (w <= m["ref_words"])).all(), (name, K)
            assert not (m["tie"][u, g["order"] - 1]).any()
            if prev is not None:
                assert (w <= prev).all()   # the listed sets grow with K
            prev = w
        for f in full:
            for (a, ta), (b, tb) in zip(model[f], full[f]):
                assert (a.order, a.words, ta) == (b.order, b.words, tb), (name, f)
                assert np.array_equal(a.q, b.q) and np.array_equal(a.res, b.res), (name, f)


def test_model_output_decodes_back():
    O = ol.load("port")
    decoders = [O] + ([ol.load("ref")] if ol.have_ref() else [])
    for name, pcm, ch in _batches():
        for K in (1, 4):
            model, ref_words, _ = xg.model_batch(pcm, ch, K)
            descs, words = xs.pack(O, model, ch)
            assert words.size <= sum(ref_words.values()), name
            for D in decoders:
                assert np.array_equal(D.decode_frames(descs, words, ch), np.asarray(pcm, np.int16).reshape(-1)), name


def test_workspace_bytes_follow_the_layout():
    """The search layout with every region padded and a 16-byte order mask per unit."""
    L = _lib.lib()
    a = lambda n: (n + 255) // 256 * 256
    for (n_frames, ch), (plain, _, search, _) in test_encode_workspace.SIZES.items():
        n_units = n_frames * (3 if ch == 2 else ch)
        want = plain + a(416 * n_units) + a(16 * n_units)
        assert L.selab200_encode_search_guided_workspace_bytes(n_frames, ch) == want, (n_frames, ch)
        assert want >= search
