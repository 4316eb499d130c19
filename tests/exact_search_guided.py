"""The exact CPU model of the guided order search (DESIGN.md 7.7).

Per analysis unit, from its 100 quantised reflection coefficients q and reference order (exact_search.all_q):
  - the estimate E_o = P_o * R_o of every order 1..100: k_i the doubles the step-up dequantises
    (exact_search.dequantised), a_i = 1 - k_i * k_i, P_1 = 1, P_2 = a_0 * a_1, P_o = P_{o-1} * a_{o-1}, R_1 = r,
    R_o = R_{o-1} * r with r = 2^(1/256) rounded to a double; every product rounded as written, sequentially in o;
  - the rank of every order by (E_o, o), and the listed orders: rank < K, order 1 and the reference order;
  - the winner: exact_search.search_units' per-order table restricted to the listed orders, with the order search's
    key (words << 8 | (order == ref ? 0 : order), tied orders excluded).
The batch layout, the stereo decision and the packing are exact_search's."""
import numpy as np

import analysis_corpus
import exact_search as xs

MAX_ORDER = 100
R = float.fromhex("0x1.00b1afa5abcbfp+0")
NO_KEY = np.iinfo(np.int64).max


def estimates(Q):
    """Q int [U, 100] -> E float64 [U, 100], E[u, o - 1] the estimate of order o."""
    K = xs.dequantised(Q)
    A = 1.0 - K * K
    U = A.shape[0]
    P = np.empty((U, MAX_ORDER))
    Rs = np.empty(MAX_ORDER)
    P[:, 0] = 1.0
    Rs[0] = R
    for o in range(2, MAX_ORDER + 1):
        P[:, o - 1] = (A[:, 0] if o == 2 else P[:, o - 2]) * A[:, o - 1]
        Rs[o - 1] = Rs[o - 2] * R
    return P * Rs


def estimates_scalar(q):
    """estimates() of one unit in plain Python floats, the definition written out."""
    k = xs.dequantised(np.asarray(q).reshape(1, MAX_ORDER))[0]
    a = [1.0 - float(x) * float(x) for x in k]
    out, p, r = [], 1.0, R
    for o in range(1, MAX_ORDER + 1):
        if o == 2:
            p = a[0] * a[1]
        elif o > 2:
            p = p * a[o - 1]
        if o > 1:
            r = r * R
        out.append(p * r)
    return np.array(out)


def ranks(E):
    """E [U, 100] -> int [U, 100]: the number of orders before each by (E, order)."""
    e = E[:, None, :]                 # [u, o, m]: order m + 1 against order o + 1
    eo = E[:, :, None]
    before = (e < eo) | ((e == eo) & (np.arange(MAX_ORDER)[None, None, :] < np.arange(MAX_ORDER)[None, :, None]))
    return before.sum(axis=2)


def listed(E, refs, K):
    """bool [U, 100]: the orders the guided search sizes or has sized (rank < K, order 1, the reference order)."""
    L = ranks(E) < K
    L[:, 0] = True
    L[np.arange(E.shape[0]), np.asarray(refs) - 1] = True
    return L


def winners(m, refs, L):
    """The winners among the listed orders of the per-order table m (exact_search.search_units) -> (order [U],
    best [U]: the winner's key)."""
    orders = np.arange(1, MAX_ORDER + 1)
    key = np.where(m["tie"] | ~L, NO_KEY, m["words"] * 256 + np.where(orders == np.asarray(refs)[:, None], 0, orders))
    w = np.argmin(key, axis=1)
    return w + 1, key[np.arange(len(w)), w]


def residues(S, Q, units, orders, chunk=16):
    """The residues of units[i] at orders[i], through the batched model's predictors and FIR."""
    out = np.zeros((len(units), xs.FRAME), np.int32)
    for a in range(0, len(units), chunk):
        idx = units[a:a + chunk]
        C, _ = xs.predictors_all(Q[idx])
        res, _ = xs.fir_limbs(S[idx], C)
        out[a:a + len(idx)] = res[np.arange(len(idx)), np.asarray(orders[a:a + chunk]) - 1]
    return out


def unit_inputs(pcm, channels, preds=None):
    """(S, Q, refs): the batch's analysis units, their q and reference orders (analysed, or from preds as
    exact_search.model_batch_all takes them)."""
    S = analysis_corpus.units(pcm, channels)
    if preds is None:
        Q, refs = xs.all_q(S)
    else:
        Q = np.array([np.asarray(p[1], np.int32)[:MAX_ORDER] for p in preds]).reshape(-1, MAX_ORDER)
        refs = np.array([int(p[0]) for p in preds], int)
    return S, Q, refs


def model_batch(pcm, channels, K, preds=None, table=None):
    """The guided search of a whole batch -> (model, ref_words, g): model and ref_words as
    exact_search.model_batch_all's; g a dict with the per-order table `m` (exact_search.search_units), `E`, `listed`,
    `order` and `best` per unit, and S, Q, refs.  table: (S, Q, refs, m) of an earlier call on the same batch."""
    if table is None:
        S, Q, refs = unit_inputs(pcm, channels, preds)
        m = xs.search_units(S, Q, refs)
    else:
        S, Q, refs, m = table
    per = 3 if channels == 2 else channels
    E = estimates(Q)
    L = listed(E, refs, K)
    order, best = winners(m, refs, L)
    res = m["res"].copy()
    moved = np.nonzero(order != m["order"])[0]
    if moved.size:
        res[moved] = residues(S, Q, moved, order[moved])
    qz = lambda u, o: np.where(np.arange(MAX_ORDER) < o, Q[u], 0).astype(np.int32)
    model, ref_words = {}, {}
    for f in range(S.shape[0] // per):
        us = range(f * per, (f + 1) * per)
        wins = [xs.Coded(int(order[u]), qz(u, order[u]), res[u], int(m["words"][u, order[u] - 1])) for u in us]
        refc = [xs.Coded(int(refs[u]), None, None, int(m["ref_words"][u])) for u in us]
        model[f] = [(wins[k], t) for k, t in xs.emitted(wins, channels)]
        ref_words[f] = sum(refc[k].words for k, _ in xs.emitted(refc, channels))
    g = dict(m=m, E=E, listed=L, order=order, best=best, S=S, Q=Q, refs=refs)
    return model, ref_words, g
