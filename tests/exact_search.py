"""The exact CPU model of the order search (DESIGN.md 7.3).

For every analysis unit: all 100 quantised reflection coefficients from the exact analysis model (exact_analysis:
quantise_reflection of every k, not only the first `order`), the reference encoder's order, and then every candidate
order 1..100 -- the predictor the port's lpc_coefficients builds at that order (order 1: zero), the FIR with the tie
test of every output and the Rice words of both streams, as exact_lossless.Unit computes them for one order.  The
winner is the tie-free order with the fewest words; between equal words the reference order if it is among them, else
the lowest.  The stereo decision (difference iff strictly fewer words) then runs on the winners.

Two forms compute the same thing:
  - per unit (search_unit): the port's predictors, one wrapping uint64 matrix product for the FIR of all 100 orders
    (fir_all) and the port's Rice sizes.  It is the reference, pinned order by order to exact_lossless.Unit, and
    costs about 30 ms per unit (numpy runs the uint64 product without BLAS);
  - batched (search_units / model_batch_all): the step-up in float64 across units, the FIR as four exact float64
    GEMMs on 16-bit limbs of the coefficients, the Rice sizes vectorised over every row, and per (unit, order) the
    fields of the device's search trace (DESIGN.md 7.3).  tests/test_exact_search.py pins it to the per-unit form.
    It costs about 15 ms per unit, so the GPU tests compare whole batches with it."""
import numpy as np

import analysis_corpus
import exact_analysis as xa
import exact_decode as xd
import exact_lossless as xl

FRAME = 2048
MAX_ORDER = 100
MAX_RICE = 20
U64 = np.uint64
SCALE = 34359738368.0   # 2^35
DOMAIN = float(1 << 62)
DIGEST_K = U64(0x9E3779B97F4A7C15)   # the search trace's digests (include/sela_b200.h)
DIGEST_K2 = U64(0xD6E8FEB86659FD93)


def all_q(units):
    """units: int [F, 2048] -> (q int32 [F, 100]: every quantised reflection coefficient, order [F]: the reference
    encoder's order)."""
    a = xa.analyse(units)
    q0, q1, qr = xa.quantise(a["k"])
    q = qr.copy()
    q[:, 0] = q0[:, 0]
    q[:, 1] = q1[:, 1]
    return q.astype(np.int32), a["order"].astype(int)


def predictors(O, q):
    """int64 [101, 101]: row o (1..100) is c[0..o] of the predictor LinearPredictor builds at order o from q[0..o),
    zero past o; c[0] (unused) is zero.  Row 1 is zero: order 1 has the single reflection coefficient 0."""
    C = np.zeros((MAX_ORDER + 1, MAX_ORDER + 1), np.int64)
    q = np.ascontiguousarray(q, np.int32)
    for o in range(1, MAX_ORDER + 1):
        C[o, 1:o + 1] = O.lpc_coefficients(q, o)[1:]
    return C


def fir_all(s, C):
    """The FIR of every order at once: (res int32 [100, 2048], tie bool [100]), row o - 1 for order o, each as
    exact_lossless.fir(s, C[o], o) computes it."""
    s = np.asarray(s, np.int64)
    pad = np.concatenate([np.zeros(MAX_ORDER, np.int64), s])
    T = np.lib.stride_tricks.sliding_window_view(pad, MAX_ORDER + 1)[:, ::-1]   # T[i, j] = s[i - j]
    P = T.astype(U64) @ C[1:].T.astype(U64)                                      # [2048, 100], mod 2^64
    total = P + U64(1 << 34)
    enc = total.view(np.int64) >> 35
    dec = (U64(1 << 35) - total).view(np.int64) >> 35
    tie = (((enc + dec) & 0xFFFFFFFF) != 0).any(axis=0)
    return (s[:, None] - enc).astype(np.int32).T, tie


class Coded:
    """One unit coded at one order: what exact_lossless.check_against_model reads (order, q, res) and its words."""

    def __init__(self, order, q, res, words):
        self.order, self.q, self.res, self.words = order, q, res, words


def search_unit(O, s, q, ref_order):
    """-> (winner: Coded, reference: Coded, words int [100] by order - 1, tie bool [100])."""
    q = np.asarray(q, np.int32)
    res, tie = fir_all(s, predictors(O, q))
    words = np.array([xl.rice_words(O, q[:o]) + xl.rice_words(O, res[o - 1]) for o in range(1, MAX_ORDER + 1)])
    orders = np.arange(1, MAX_ORDER + 1)
    key = np.where(tie, np.iinfo(np.int64).max, words * 256 + np.where(orders == ref_order, 0, orders))
    o = int(orders[np.argmin(key)])
    qz = lambda o: np.where(np.arange(MAX_ORDER) < o, q, 0).astype(np.int32)
    win = Coded(o, qz(o), res[o - 1], int(words[o - 1]))
    ref = Coded(ref_order, qz(ref_order), res[ref_order - 1], int(words[ref_order - 1]))
    ref.tie = bool(tie[ref_order - 1])
    return win, ref, words, tie


def emitted(units, channels):
    """(unit index, subframe type) per channel: the stereo decision (difference iff strictly fewer words)."""
    return xl.emitted(units, channels)


def model_batch(O, pcm, channels, frames=None, preds=None):
    """The search of a batch -> ({frame: [(Coded, type) per channel]}, {frame: reference words}) over `frames` (all by
    default).  preds: one (order, q[100]) per analysis unit in encoder order, as selab200_encode_search_forced takes
    them, or None to analyse the units."""
    units = analysis_corpus.units(pcm, channels)
    per = 3 if channels == 2 else channels
    n_frames = units.shape[0] // per
    frames = range(n_frames) if frames is None else frames
    idx = np.array([f * per + k for f in frames for k in range(per)], int)
    if preds is None:
        qs, refs = all_q(units[idx]) if idx.size else (np.zeros((0, MAX_ORDER), np.int32), np.zeros(0, int))
    else:
        qs = np.array([np.asarray(preds[i][1], np.int32)[:MAX_ORDER] for i in idx]).reshape(-1, MAX_ORDER)
        refs = np.array([int(preds[i][0]) for i in idx], int)
    model, ref_words = {}, {}
    for n, f in enumerate(frames):
        found = [search_unit(O, units[f * per + k], qs[n * per + k], refs[n * per + k]) for k in range(per)]
        wins, ref = [w for w, _, _, _ in found], [r for _, r, _, _ in found]
        model[f] = [(wins[k], t) for k, t in emitted(wins, channels)]
        ref_words[f] = sum(ref[k].words for k, _ in emitted(ref, channels))
    return model, ref_words


def pack(O, model, channels):
    """The model's frames (all of a batch, in order) as (descs, words), the way the encoder lays them out."""
    descs = np.zeros(len(model) * channels, xl.ol.DESC_DTYPE)
    words = []
    at = 0
    for f in sorted(model):
        for ch, (u, t) in enumerate(model[f]):
            kq, wq = O.rice_encode(u.q[:u.order])
            kr, wr = O.rice_encode(u.res)
            d = descs[f * channels + ch]
            d["channel"], d["subframe_type"], d["parent_channel"] = ch, t, 0 if t else ch
            d["refl_rice_param"], d["refl_words"], d["lpc_order"] = kq, wq.size, u.order
            d["res_rice_param"], d["res_words"], d["samples"] = kr, wr.size, FRAME
            d["refl_offset"], d["res_offset"] = at, at + wq.size
            words += [wq, wr]
            at += wq.size + wr.size
    return descs, np.concatenate(words).astype(np.uint32) if words else np.zeros(0, np.uint32)


def check_frames(O, descs, words, pcm, channels, model):
    """The subframes of every frame in `model` equal the model's, field for field and word for word, and the whole
    batch decodes back to its source under the port (and the compiled reference, where built)."""
    xl.check_against_model(O, descs, words, pcm, channels, {f: (em, []) for f, em in model.items()})


# ---------------------------------------------------------------- batched --

def dequantised(Q):
    """Q int [U, 100] -> the reflection coefficients LinearPredictor dequantises at any order >= 2 (q[0] through the
    first-order table, q[1] through the second-order one, the rest q / 64), float64 [U, 100]."""
    Q = np.asarray(Q, np.int64)
    K = Q / 64.0
    K[:, 0] = xd.FIRST[Q[:, 0] + 64]
    K[:, 1] = xd.SECOND[Q[:, 1] + 64]
    return K


def predictors_all(Q):
    """The predictor of every order of every unit -> (C int64 [U, 101, 101], domain bool [U, 101]).

    C[u, o] is row o of predictors(): c[0..o] of the predictor LinearPredictor builds at order o, zero past o; row 1
    (and row 0) is zero.  The step-up (linear_predictor.cpp:30-61) runs once per unit in float64 with the reference's
    operations in its order: the predictor of order o is the row after iteration o - 1.  domain[u, o]: every
    2^35 * t[m] of order o is below 2^62, where the conversion to int64 is defined (order 1: true)."""
    K = dequantised(Q)
    U = K.shape[0]
    t = np.zeros((U, MAX_ORDER))
    C = np.zeros((U, MAX_ORDER + 1, MAX_ORDER + 1), np.int64)
    dom = np.ones((U, MAX_ORDER + 1), bool)
    for i in range(MAX_ORDER):
        k = K[:, i:i + 1]
        half = i >> 1
        if half:
            lo = np.arange(half)
            a, b = t[:, lo], t[:, i - 1 - lo]
            t[:, lo] = a + k * b
            t[:, i - 1 - lo] = b + k * a
        if i & 1:
            t[:, half] = t[:, half] + t[:, half] * K[:, i]
        t[:, i] = K[:, i]
        o = i + 1
        if o >= 2:
            v = SCALE * -t[:, :o]
            ok = (np.abs(v) < DOMAIN).all(axis=1)
            dom[:, o] = ok
            C[:, o, 1:o + 1] = np.where(ok[:, None], v, 0.0).astype(np.int64)
    return C, dom


def fir_limbs(S, C):
    """The FIR of every order of every unit: (res int32 [U, 100, 2048], tie bool [U, 100]), [u, o - 1] as fir_all
    computes row o - 1 for unit u.  S int [U, 2048] (|s| < 2^16), C int64 [U, 101, 101].

    The coefficients mod 2^64 are split into four 16-bit limbs; each limb's Toeplitz product is a float64 GEMM whose
    every partial sum is below 100 * 2^16 * 2^16 < 2^39, so exact; the four are recombined with wrapping uint64
    shifts and adds into the prediction sum mod 2^64."""
    S = np.asarray(S, np.int64)
    U = S.shape[0]
    assert np.abs(S).max(initial=0) < 1 << 16
    pad = np.concatenate([np.zeros((U, MAX_ORDER), np.int64), S], axis=1)
    T = np.lib.stride_tricks.sliding_window_view(pad, MAX_ORDER + 1, axis=1)[:, :, ::-1][:, :, 1:]   # s[i - j]
    T = T.astype(np.float64)                                                    # [U, 2048, 100], j = 1..100
    Cu = C[:, 1:, 1:].view(U64).transpose(0, 2, 1)                              # [U, j, o]
    P = np.zeros((U, FRAME, MAX_ORDER), np.int64)                               # int64 arrays wrap like uint64
    for p in range(4):
        limb = ((Cu >> U64(16 * p)) & U64(0xFFFF)).astype(np.float64)
        P += np.matmul(T, limb).astype(np.int64) << (16 * p)
    total = P + (1 << 34)
    enc = total >> 35
    dec = ((1 << 35) - total) >> 35
    tie = (((enc + dec) & 0xFFFFFFFF) != 0).any(axis=1)
    return (S[:, :, None] - enc).astype(np.int32).transpose(0, 2, 1), tie


def rice_choose(X, n=None):
    """calculateOptimumRiceParam on every row of X (int32 [..., N]), of its first n[...] values where n is given ->
    (k, bits, words): the first arg-min over k in [0, 20) of sum(zigzag >> k) + n * (1 + k), and the bits rounded
    up to 32."""
    X = np.asarray(X, np.int64)
    u = (((X << 1) ^ (X >> 63)) & 0xFFFFFFFF).astype(np.uint32)    # zigzag of int32, as uint32
    N = X.shape[-1]
    if n is None:
        n = np.full(X.shape[:-1], N, np.int64)
    else:
        n = np.asarray(n, np.int64)
        u = np.where(np.arange(N) < n[..., None], u, np.uint32(0))
    best = bestk = None
    for k in range(MAX_RICE):
        bits = np.add.reduce(u >> np.uint32(k), axis=-1, dtype=np.int64) + n * (1 + k)
        if best is None:
            best, bestk = bits, np.zeros(bits.shape, np.int64)
        else:
            better = bits < best
            best, bestk = np.where(better, bits, best), np.where(better, k, bestk)
    return bestk, best, (best + 31) // 32


def pred_digest(C):
    """C int64 [..., 101, 101] -> sum_{j=1..100} (c[j] + j * K2) * K mod 2^64 of every row, uint64 [..., 101]."""
    j = np.arange(1, MAX_ORDER + 1, dtype=U64)
    with np.errstate(over="ignore"):
        return ((C[..., 1:].view(U64) + j * DIGEST_K2) * DIGEST_K).sum(axis=-1, dtype=U64)


def res_digest(R):
    """R int32 [..., 2048] -> sum_i ((i << 32) | (uint32)r[i]) * K mod 2^64, uint64 [...]."""
    i = np.arange(FRAME, dtype=U64) << U64(32)
    with np.errstate(over="ignore"):
        return ((i | R.view(np.uint32).astype(U64)) * DIGEST_K).sum(axis=-1, dtype=U64)


TRACE_FIELDS = ("tie", "refl_k", "refl_words", "res_k", "res_words", "pred_digest", "res_digest")


def search_units(S, Q, refs, chunk=16):
    """The batched model of the search of units S (int [U, 2048]) with all 100 q (Q int [U, 100]) and reference orders
    refs [U] -> dict of arrays:
      per (unit, order), [U, 100] at order - 1: the fields of the search trace (TRACE_FIELDS) and `domain`;
      per unit: `order` (the winner), `best` (its key, words << 8 | (order == ref ? 0 : order)), `ref_words`, and
      `res` (int32 [U, 2048], the winner's residues)."""
    S = np.asarray(S, np.int64)
    Q = np.asarray(Q, np.int32)
    refs = np.asarray(refs, np.int64)
    U = S.shape[0]
    out = {f: np.zeros((U, MAX_ORDER), np.uint64 if "digest" in f else np.int64) for f in TRACE_FIELDS}
    out["tie"] = np.zeros((U, MAX_ORDER), bool)
    out["domain"] = np.zeros((U, MAX_ORDER), bool)
    out["res"] = np.zeros((U, FRAME), np.int32)
    orders = np.arange(1, MAX_ORDER + 1)
    kq, _, wq = rice_choose(np.broadcast_to(Q[:, None, :], (U, MAX_ORDER, MAX_ORDER)), orders[None, :])
    out["refl_k"][:], out["refl_words"][:] = kq, wq
    for a in range(0, U, chunk):
        b = min(U, a + chunk)
        C, dom = predictors_all(Q[a:b])
        res, tie = fir_limbs(S[a:b], C)
        kr, _, wr = rice_choose(res)
        out["domain"][a:b], out["tie"][a:b] = dom[:, 1:], tie
        out["res_k"][a:b], out["res_words"][a:b] = kr, wr
        out["pred_digest"][a:b] = pred_digest(C)[:, 1:]
        out["res_digest"][a:b] = res_digest(res)
        words = wq[a:b] + wr
        key = np.where(tie, np.iinfo(np.int64).max, words * 256 + np.where(orders == refs[a:b, None], 0, orders))
        w = np.argmin(key, axis=1)
        out.setdefault("best", np.zeros(U, np.int64))[a:b] = key[np.arange(b - a), w]
        out.setdefault("order", np.zeros(U, np.int64))[a:b] = w + 1
        out["res"][a:b] = res[np.arange(b - a), w]
    out["words"] = out["refl_words"] + out["res_words"]
    out["ref_words"] = out["words"][np.arange(U), refs - 1]
    return out


def model_batch_all(pcm, channels, preds=None):
    """model_batch over every frame of a batch through the batched model -> (model, ref_words, units, Q, refs):
    model and ref_words as model_batch's, units the dict of search_units, Q and refs the units' q and reference
    orders (analysed, or from preds as model_batch takes them)."""
    S = analysis_corpus.units(pcm, channels)
    per = 3 if channels == 2 else channels
    if preds is None:
        Q, refs = all_q(S)
    else:
        Q = np.array([np.asarray(p[1], np.int32)[:MAX_ORDER] for p in preds]).reshape(-1, MAX_ORDER)
        refs = np.array([int(p[0]) for p in preds], int)
    m = search_units(S, Q, refs)
    qz = lambda u, o: np.where(np.arange(MAX_ORDER) < o, Q[u], 0).astype(np.int32)
    model, ref_words = {}, {}
    for f in range(S.shape[0] // per):
        us = range(f * per, (f + 1) * per)
        wins = [Coded(int(m["order"][u]), qz(u, m["order"][u]), m["res"][u], int(m["words"][u, m["order"][u] - 1]))
                for u in us]
        refc = [Coded(int(refs[u]), None, None, int(m["ref_words"][u])) for u in us]
        model[f] = [(wins[k], t) for k, t in emitted(wins, channels)]
        ref_words[f] = sum(refc[k].words for k, _ in emitted(refc, channels))
    return model, ref_words, m, Q, refs
