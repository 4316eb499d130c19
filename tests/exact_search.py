"""The exact CPU model of the order search (DESIGN.md 7.3).

For every analysis unit: all 100 quantised reflection coefficients from the exact analysis model (exact_analysis:
quantise_reflection of every k, not only the first `order`), the reference encoder's order, and then every candidate
order 1..100 -- the predictor the port's lpc_coefficients builds at that order (order 1: zero), the FIR with the tie
test of every output and the Rice words of both streams, as exact_lossless.Unit computes them for one order.  The
winner is the tie-free order with the fewest words; between equal words the reference order if it is among them, else
the lowest.  The stereo decision (difference iff strictly fewer words) then runs on the winners.

The FIR of all 100 orders is one wrapping uint64 matrix product (fir_all); tests/test_exact_search.py pins it, order
by order, to exact_lossless.Unit.  A unit costs about 30 ms, so the GPU tests compare chosen slices of each batch."""
import numpy as np

import analysis_corpus
import exact_analysis as xa
import exact_lossless as xl

FRAME = 2048
MAX_ORDER = 100
U64 = np.uint64


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
