"""The CPU model of the order search (exact_search.py) pinned on its own: its predictors against the compiled
reference at every order, order 1's zero predictor, its all-order FIR against exact_lossless.Unit, its words at the
reference order against the default encoder, and its output decoding back to the source; then the batched model
(exact_search.search_units) pinned to the per-unit one part by part: predictors and their domain on every corpus
unit, the limb FIR, the vectorised Rice sizes and the winners."""
import ctypes as C

import numpy as np

import analysis_corpus
import exact_lossless as xl
import exact_search as xs
import oracle_lib as ol
import rice_encode_families as ref
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


# ---- the batched model (exact_search.search_units), pinned to the per-unit one ----

def test_batched_predictors_are_the_ports_at_every_order_on_every_corpus_unit():
    """Every corpus unit at every order 1..100: the float64 step-up across units gives, bit for bit, the port's
    lpc_coefficients (order 1: zero), and every one of them is inside the int64 domain of the conversion."""
    O = ol.load("port")
    S = analysis_corpus.all_units()
    qs, _ = xs.all_q(S)
    outside = 0
    for a in range(0, len(qs), 256):
        C, dom = xs.predictors_all(qs[a:a + 256])
        outside += int((~dom[:, 1:]).sum())
        assert not C[:, 1].any()
        for n, q in enumerate(qs[a:a + 256]):
            assert np.array_equal(C[n], xs.predictors(O, q)), a + n
    print("%d units x 100 orders, %d outside the domain" % (len(qs), outside))
    assert outside == 0


def _planted_units(O, n):
    """Corpus units with a tie planted (exact_lossless.place_tie) at one order each, its FIR row tied."""
    rng = np.random.default_rng(7)
    S = analysis_corpus.all_units()
    qs, _ = xs.all_q(S)
    out = []
    for u in rng.permutation(len(S)):
        o = int(rng.integers(2, 101))
        c = xs.predictors(O, qs[u])[o, :o + 1]
        s = S[u].copy()
        lim = 65535 if np.abs(s).max() > 32767 else 32767
        if xl.place_tie(s, c, int(rng.integers(200, 2000)), lo=-lim, hi=lim, rng=rng):
            out.append((s, qs[u], o))
        if len(out) == n:
            return out
    raise AssertionError("too few ties placed")


def test_limb_fir_is_fir_all_and_the_lossless_model():
    """The four-limb float64 FIR equals fir_all (residues and tie flags, every order) on 300 corpus units, among them
    every 17-bit difference unit of stereo_pairs' full-scale pairs, and on units with a planted tie; on every 10th
    unit each order is also checked against exact_lossless.Unit."""
    O = ol.load("port")
    name, pcm, ch = analysis_corpus.batches()[1]
    pairs = analysis_corpus.units(pcm, ch)
    wide = pairs[np.abs(pairs).max(axis=1) > 32767]
    assert len(wide) >= 8
    S = analysis_corpus.all_units()
    S = np.concatenate([wide, S[np.linspace(0, len(S) - 1, 300 - len(wide)).astype(int)]])
    qs, _ = xs.all_q(S)
    planted = _planted_units(O, 24)
    S = np.concatenate([S, np.stack([p[0] for p in planted])])
    qs = np.concatenate([qs, np.stack([p[1] for p in planted])])
    C, _ = xs.predictors_all(qs)
    res, tie = xs.fir_limbs(S, C)
    for n in range(len(S)):
        r, t = xs.fir_all(S[n], C[n])
        assert np.array_equal(res[n], r) and np.array_equal(tie[n], t), n
        if n % 10 == 0:
            for o in range(1, 101):
                u = xl.Unit(O, S[n], o, np.where(np.arange(100) < o, qs[n], 0))
                assert np.array_equal(u.res, res[n, o - 1]) and u.tie == tie[n, o - 1], (n, o)
    for n, (_, _, o) in enumerate(planted):
        assert tie[len(S) - len(planted) + n, o - 1], n


def _port_rice(O, x):
    k, bits = C.c_uint32(0), C.c_uint64(0)
    x = np.ascontiguousarray(x, np.int32)
    words = int(O.lib.sela_oracle_rice_size(x.ctypes.data, x.size, C.byref(k), C.byref(bits)))
    return k.value, bits.value, words


def test_vectorised_rice_is_the_ports():
    """rice_choose (k, bits, words) equals sela_oracle_rice_size on both streams at every order of sampled corpus
    units and on every row of the Rice encoder's value families inside the reference's zig-zag domain."""
    O = ol.load("port")
    S = analysis_corpus.all_units()
    S = S[np.linspace(0, len(S) - 1, 12).astype(int)]
    qs, _ = xs.all_q(S)
    C_, _ = xs.predictors_all(qs)
    res, _ = xs.fir_limbs(S, C_)
    orders = np.arange(1, 101)
    kq, bq, wq = xs.rice_choose(np.broadcast_to(qs[:, None, :], (len(S), 100, 100)), orders[None, :])
    kr, br, wr = xs.rice_choose(res)
    for n in range(len(S)):
        for o in orders:
            assert (kq[n, o - 1], bq[n, o - 1], wq[n, o - 1]) == _port_rice(O, qs[n, :o]), (n, o)
            assert (kr[n, o - 1], br[n, o - 1], wr[n, o - 1]) == _port_rice(O, res[n, o - 1]), (n, o)
    checked = 0
    for name in ref.NAMES:
        for b in ref.family(name):
            rows = ref.in_reference_domain(b)
            if not rows:
                continue
            k, bits, words = xs.rice_choose(b.values[rows], b.counts[rows])
            for i, r in enumerate(rows):
                c = int(b.counts[r])
                if c:
                    assert (k[i], bits[i], words[i]) == _port_rice(O, b.values[r, :c]), (name, r)
                    checked += 1
    assert checked > 5000


def _gpu_test_frames():
    """The unforced batches test_encode_search.py compares with the per-unit model (the families, 16 random frames,
    the 12-frame BASELINE slice and the golden oct_reference_lossy frames), and 6 frames of every corpus batch, whose
    whole batches test_encode_search.py compares with the batched model."""
    import pathlib
    from sela_b200 import synth
    gold = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
    out = [("families", np.stack([v for v in signals.families().values()]).astype(np.int16).reshape(-1), 1),
           ("random", signals.random_frames(16, 3).astype(np.int16).reshape(-1), 1),
           ("baseline", synth.sine_noise(44100, 2, n_frames=12, seed=1).reshape(-1), 2),
           ("oct_reference_lossy", gold["pcm_oct_reference_lossy"].reshape(-1), 8)]
    for name, pcm, ch in analysis_corpus.batches():
        n = pcm.size // (2048 * ch)
        frames = sorted(set(np.linspace(0, n - 1, min(n, 6)).astype(int).tolist()))
        out.append((name, np.asarray(pcm, np.int16).reshape(n, -1)[frames].reshape(-1), ch))
    return out


def test_batched_winners_are_model_batchs():
    """model_batch_all (the batched model) and model_batch (the per-unit one) agree on the frames of _gpu_test_frames:
    winners, their residues and words, the stereo decision and the reference words."""
    O = ol.load("port")
    for name, pcm, ch in _gpu_test_frames():
        fast, fast_ref, _, _, _ = xs.model_batch_all(pcm, ch)
        slow, slow_ref = xs.model_batch(O, pcm, ch)
        assert fast_ref == slow_ref, name
        for f in slow:
            for (a, ta), (b, tb) in zip(fast[f], slow[f]):
                assert (a.order, a.words, ta) == (b.order, b.words, tb), (name, f)
                assert np.array_equal(a.q, b.q) and np.array_equal(a.res, b.res), (name, f)
        da, wa = xs.pack(O, fast, ch)
        db, wb = xs.pack(O, slow, ch)
        assert da.tobytes() == db.tobytes() and np.array_equal(wa, wb), name
