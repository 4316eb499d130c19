"""The CPU model of the order search (exact_search.py) pinned on its own: its predictors against the compiled
reference at every order, order 1's zero predictor, its all-order FIR against exact_lossless.Unit, its words at the
reference order against the default encoder, and its output decoding back to the source."""
import numpy as np

import analysis_corpus
import exact_lossless as xl
import exact_search as xs
import oracle_lib as ol
import signals


def _corpus_units():
    """A few units of every corpus batch: channels, 17-bit differences, DC, silence."""
    out = []
    for name, pcm, ch in analysis_corpus.batches():
        u = analysis_corpus.units(pcm, ch)
        out.append(u[np.linspace(0, u.shape[0] - 1, 6).astype(int)])
    return np.concatenate(out)


def test_predictor_of_every_order_is_the_reference_one():
    """Row o of exact_search.predictors (the port's lpc_coefficients at order o, from every quantised coefficient)
    equals what the compiled reference's LinearPredictor builds with optimalLpcOrder = o."""
    O = ol.load("port")
    units = _corpus_units()
    qs, _ = xs.all_q(units)
    R = ol.load("ref") if ol.have_ref() else None
    for q in qs[::3]:
        C = xs.predictors(O, q)
        assert not C[1].any()
        if R is not None:
            for o in range(1, 101):
                assert np.array_equal(C[o, 1:o + 1], R.lpc_coefficients(q, o)[1:]), o


def test_order_one_predicts_nothing():
    """Order 1: the predictor is zero whatever q[0] is (not row 0 of the step-up), the residues are the samples and
    the unit never ties."""
    O = ol.load("port")
    s = signals.families()["sine_noise"].astype(np.int64)
    for q0 in (-64, -20, 0, 17, 63):
        q = np.zeros(100, np.int32)
        q[:3] = [q0, 5, -3]
        C = xs.predictors(O, q)
        assert not C[1].any() and C[2, 1] != 0
        res, tie = xs.fir_all(s, C)
        assert np.array_equal(res[0], s) and not tie[0]
        u = xl.Unit(O, s, 1, q)
        assert not u.c[1:].any() and np.array_equal(u.res, s)


def test_all_order_fir_is_the_lossless_model_at_every_order():
    O = ol.load("port")
    units = _corpus_units()
    qs, refs = xs.all_q(units)
    for s, q in list(zip(units, qs))[::7]:
        C = xs.predictors(O, q)
        res, tie = xs.fir_all(s, C)
        for o in range(1, 101):
            u = xl.Unit(O, s, o, np.where(np.arange(100) < o, q, 0))
            assert np.array_equal(u.c[1:], C[o, 1:o + 1])
            assert np.array_equal(u.res, res[o - 1]) and u.tie == tie[o - 1], o


def test_quantisation_and_reference_order_are_the_analysis_ones():
    """The first `order` coefficients of all_q are the port's quantised coefficients, and the order is its order."""
    O = ol.load("port")
    units = _corpus_units()
    qs, refs = xs.all_q(units)
    for s, q, o in zip(units, qs, refs):
        a = O.lpc_analyse(s.astype(np.int32))
        assert a["order"] == o and np.array_equal(a["q"], q[:o])


def test_reference_words_are_the_default_encoders():
    """Per frame, the model's words at the reference orders (with the reference's stereo decision) are the default
    encoder's words; a unit whose reference order has no tie never gets more words."""
    O = ol.load("port")
    for name, pcm, ch in analysis_corpus.batches():
        n = pcm.size // (2048 * ch)
        frames = sorted(set(np.linspace(0, n - 1, min(n, 6)).astype(int).tolist()))
        sub = np.asarray(pcm, np.int16).reshape(n, -1)[frames].reshape(-1)
        model, ref_words = xs.model_batch(O, sub, ch)
        d, w = O.encode_frames(sub, ch)
        for f in range(len(frames)):
            fd = d[f * ch:(f + 1) * ch]
            assert ref_words[f] == int(fd["refl_words"].sum()) + int(fd["res_words"].sum()), (name, f)
        units = analysis_corpus.units(sub, ch)
        qs, refs = xs.all_q(units)
        for s, q, o in zip(units, qs, refs):
            win, ref, _, _ = xs.search_unit(O, s, q, o)
            assert ref.tie or win.words <= ref.words


def test_model_output_decodes_back():
    O = ol.load("port")
    decoders = [O] + ([ol.load("ref")] if ol.have_ref() else [])
    cases = [(signals.random_frames(6, 3).astype(np.int16).reshape(-1), 1),
             (np.stack([v for v in signals.families().values()]).astype(np.int16).reshape(-1), 1),
             (analysis_corpus.batches()[1][1][:2048 * 6], 2)]
    for pcm, ch in cases:
        model, ref_words = xs.model_batch(O, pcm, ch)
        descs, words = xs.pack(O, model, ch)
        assert words.size <= sum(ref_words.values())
        for D in decoders:
            assert np.array_equal(D.decode_frames(descs, words, ch), np.asarray(pcm, np.int16).reshape(-1))


def test_equal_words_prefer_the_reference_order_then_the_lowest():
    """q = [10, 5, 0, ...] on two_tone: orders 2..8 cost the same words (zero taps leave the predictor as it is and
    add one bit each to the reflection stream), order 9 one word more."""
    O = ol.load("port")
    s = signals.families()["two_tone"].astype(np.int64)
    q = np.zeros(100, np.int32)
    q[:2] = [10, 5]
    for ref, want in ((5, 5), (2, 2), (8, 8), (20, 2), (1, 2)):
        win, refc, words, tie = xs.search_unit(O, s, q, ref)
        assert list(words[1:8]) == [984] * 7 and words[8] == 985 and not tie.any()
        assert win.order == want and win.words == 984
