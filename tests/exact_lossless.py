"""The exact CPU model of the lossless encode (DESIGN.md 7.2), and a tie placer.

The model is built on the plain-C port (oracle/liboracle.so): the tie criterion in NumPy (int64 wrap), and the
repair rule -- candidates, rounds, fewest words, first candidate on a tie -- over the port's lpc_coefficients and
rice_size.  A unit is either analysed as the encoder analyses it, or coded with a given predictor (order, q), as
selab200_encode_lossless_forced codes it.

place_tie plants a tie at a chosen output of a chosen predictor by setting two or three samples just before it.
Inside the domain (every partial prediction sum below 2^62) output i ties iff P = sum_j c[j] s[i-j] is 2^34 mod
2^35; the placer solves that congruence for the sample under the tap with the lowest 2-adic valuation and sweeps
one or two other samples until the solution lies inside the row's range."""
import ctypes as C

import numpy as np

import analysis_corpus
import oracle_lib as ol

FRAME = 2048
U64 = np.uint64
Q = 35
M35 = 1 << Q
TIE = 1 << (Q - 1)
DOMAIN = 1 << 62
PLACER_TAPS = 8  # place_tie only writes samples i-8 .. i-1


# ------------------------------------------------------------------ model --

def fir(s, c, order):
    """The encoder's residual and the tie test of every output: (res int32[2048], tie bool[2048])."""
    s = np.asarray(s, np.int64)
    su = s.astype(U64)
    cu = np.asarray(c, np.int64).astype(U64)
    P = np.zeros(s.size, U64)
    for j in range(1, order + 1):
        P[j:] += cu[j] * su[:-j]
    total = P + U64(1 << 34)
    enc = total.view(np.int64) >> 35                   # (2^34 + P) >> 35
    dec = (U64(1 << 35) - total).view(np.int64) >> 35  # (2^34 - P) >> 35
    tie = ((enc + dec) & 0xFFFFFFFF) != 0              # as int32: enc + dec != 0
    return (s - enc).astype(np.int32), tie


def rice_words(O, x):
    x = np.ascontiguousarray(x, np.int32)
    k, bits = C.c_uint32(0), C.c_uint64(0)
    O.lib.sela_oracle_rice_size.restype = C.c_size_t
    return int(O.lib.sela_oracle_rice_size(x.ctypes.data, x.size, C.byref(k), C.byref(bits)))


def repair_edit(o, c):
    """Candidate c of a unit of order o (kernels.cuh repair_edit): (order, j, delta)."""
    n1 = 5 if o == 2 else 7
    if c < n1:
        if c == n1 - 1:
            return o - 1, 0, 0
        return o, (c >> 1) if (c >> 1) < 2 else o - 1, 1 if c & 1 else -1
    c -= n1
    n_edits = 2 * (o - 3) if o > 3 else 0
    if c < n_edits:
        return o, 2 + (c >> 1), 1 if c & 1 else -1
    return o - 2 - (c - n_edits), 0, 0


def round1(o):
    return 5 if o == 2 else 7


class Unit:
    def __init__(self, O, s, order, q):
        self.s, self.order = s, order
        self.q = np.zeros(100, np.int32)
        self.q[:order] = np.asarray(q, np.int32)[:order]
        self.c = O.lpc_coefficients(self.q, order)
        self.res, ties = fir(s, self.c, order)
        self.ties = ties
        self.tie = bool(ties.any())
        self.words = rice_words(O, self.q[:order]) + rice_words(O, self.res)


def analyse(O, s):
    a = O.lpc_analyse(np.asarray(s, np.int32))
    q = np.zeros(100, np.int32)
    q[:a["order"]] = a["q"]
    return Unit(O, s, a["order"], q)


def candidate_predictor(u, cand):
    """(order, q) of candidate `cand` of unit u, or None for an edit that leaves [-64, 63]."""
    order, j, delta = repair_edit(u.order, cand)
    q = u.q.copy()
    q[order:] = 0
    if delta:
        q[j] += delta
        if not -64 <= q[j] <= 63:
            return None
    return order, q


def candidate(O, u, cand):
    """Candidate `cand` of unit u as a Unit (+ .cand), or None where it is no candidate."""
    p = candidate_predictor(u, cand)
    if p is None:
        return None
    v = Unit(O, u.s, *p)
    v.cand = cand
    return v


def repair(O, u):
    """The winner of the repair of a unit with a tie, as a Unit (+ .cand)."""
    o = u.order
    n1 = round1(o)
    for cands in (range(n1), range(n1, 3 * o - 1)):
        best = None
        for cand in cands:
            v = candidate(O, u, cand)
            if v is not None and not v.tie and (best is None or v.words < best.words):
                best = v
        if best is not None:
            return best
    raise AssertionError("order 1 is always a candidate")


def emitted(units, channels):
    """(unit index, subframe type) per channel: the encoder's stereo decision (difference iff strictly smaller)."""
    if channels != 2:
        return [(k, 0) for k in range(channels)]
    return [(0, 0), (2, 1) if units[2].words < units[1].words else (1, 0)]


def model_frame(O, planes, channels, preds=None):
    """planes: the frame's unit signals in encoder order; preds: their predictors (order, q), or None to analyse
    them -> (emitted units per channel with their type, report entries (channel, ref_order, ref_words, order,
    words))."""
    if preds is None:
        units = [analyse(O, s) for s in planes]
    else:
        units = [Unit(O, s, o, q) for s, (o, q) in zip(planes, preds)]
    ref = emitted(units, channels)
    if not any(units[k].tie for k, _ in ref):
        return [(units[k], t) for k, t in ref], []
    now_units = [repair(O, u) if u.tie else u for u in units]
    now = emitted(now_units, channels)
    report = []
    for ch in range(channels):
        (ka, _), (kb, _) = ref[ch], now[ch]
        if ka != kb or units[kb].tie:
            report.append((ch, units[ka].order, units[ka].words, now_units[kb].order, now_units[kb].words))
    return [(now_units[k], t) for k, t in now], report


def model_batch(O, pcm, channels, preds=None, every=False):
    """-> {frame: (emitted, report)} for the frames the model re-codes, or with `every` for every frame.  preds:
    one predictor (order, q) per analysis unit in encoder order, or None to analyse the units."""
    out = {}
    units = analysis_corpus.units(pcm, channels)
    per = 3 if channels == 2 else channels
    for f in range(units.shape[0] // per):
        p = None if preds is None else preds[f * per:(f + 1) * per]
        em, rep = model_frame(O, units[f * per:(f + 1) * per], channels, p)
        if rep or every:
            out[f] = (em, rep)
    return out


# ----------------------------------------------------------- comparisons --

def as_tuples(report):
    return [(int(e["frame"]), int(e["channel"]), int(e["ref_order"]), int(e["ref_words"]), int(e["order"]),
             int(e["words"])) for e in report]


def expected_report(model):
    return [(f, ch, ro, rw, o, w) for f in sorted(model) for ch, ro, rw, o, w in model[f][1]]


def check_against_model(O, descs, words, pcm, channels, model):
    """The subframes of every frame in `model` equal the model's, field for field and word for word, and the whole
    batch decodes back to its source under the port (and the compiled reference, where built)."""
    d = descs.reshape(-1, channels)
    for f, (em, _) in model.items():
        for ch, (u, t) in enumerate(em):
            s = d[f][ch]
            assert (int(s["lpc_order"]), int(s["subframe_type"])) == (u.order, t), (f, ch)
            kq, wq = O.rice_encode(u.q[:u.order])
            kr, wr = O.rice_encode(u.res)
            assert (int(s["refl_rice_param"]), int(s["res_rice_param"])) == (kq, kr), (f, ch)
            got_q = words[int(s["refl_offset"]):int(s["refl_offset"]) + int(s["refl_words"])]
            got_r = words[int(s["res_offset"]):int(s["res_offset"]) + int(s["res_words"])]
            assert np.array_equal(got_q, wq) and np.array_equal(got_r, wr), (f, ch)
    src = np.asarray(pcm, np.int16).reshape(-1)
    for D in [O] + ([ol.load("ref")] if ol.have_ref() else []):
        assert np.array_equal(D.decode_frames(descs, words, channels), src)


# ------------------------------------------------------------ tie placer --

def valuation(x):
    """2-adic valuation of x mod 2^35 (35 for 0)."""
    x %= M35
    return Q if x == 0 else (x & -x).bit_length() - 1


def prediction(s, c, i):
    """P = sum_j c[j] s[i-j] mod 2^35 (Python integers)."""
    return sum(int(c[j]) * int(s[i - j]) for j in range(1, min(len(c) - 1, i) + 1)) % M35


def place_tie(s, c, i, lo=-32768, hi=32767, target=TIE, rng=None, near=True):
    """Set two or three of s[i-8 .. i-1] (int64, in place) so that P at output i is `target` mod 2^35 -- a tie for
    the default target.  c: the predictor c[0..order] (c[0] unused).  lo, hi: the samples' range, scalars or arrays
    over the positions.  near: the solution closest to the samples there (in windows that double), so that a tie
    does not plant a spike in the signal; else the first one found.  Samples before i-8 are left alone, so ties
    placed at increasing positions at least 9 apart stay ties.  -> False (s unchanged) where none was found."""
    rng = np.random.default_rng(i) if rng is None else rng
    order = len(c) - 1
    lo_at = (lambda k: int(lo[k])) if np.ndim(lo) else (lambda k: int(lo))
    hi_at = (lambda k: int(hi[k])) if np.ndim(hi) else (lambda k: int(hi))
    taps = [j for j in range(1, min(order, PLACER_TAPS, i) + 1) if int(c[j]) % M35]
    if not taps:
        return False
    j1 = min(taps, key=lambda j: (valuation(int(c[j])), j))
    others = [j for j in taps if j != j1][:2]
    v = valuation(int(c[j1]))
    m = 1 << (Q - v)
    inv = pow((int(c[j1]) % M35) >> v, -1, m)
    free = [j1] + others
    x0, lo1, hi1 = int(s[i - j1]), lo_at(i - j1), hi_at(i - j1)
    rest = (prediction(s, c, i) - sum(int(c[j]) * int(s[i - j]) for j in free)) % M35
    R0 = (target - rest) % M35
    c2 = U64(int(c[others[0]]) % (1 << 64)) if others else U64(0)
    c3 = int(c[others[1]]) if len(others) > 1 else 0
    y0 = int(s[i - others[0]]) if others else 0
    z0 = int(s[i - others[1]]) if len(others) > 1 else 0

    def solve(ys, z):
        """x for every y at this z: (ok, x), x the representative of the solution nearest x0 (or >= lo)."""
        R = (U64(R0) - c2 * ys.astype(U64) - U64(c3 * z % M35)) & U64(M35 - 1)
        ok = (R & U64((1 << v) - 1)) == 0
        x = (((R >> U64(v)) * U64(inv)) & U64(m - 1)).astype(np.int64)   # the solution mod 2^(35-v)
        base = x0 - m // 2 if near else lo1
        x = base + (x - base) % m
        x = np.where(x < lo1, x + m, np.where(x > hi1, x - m, x))
        return ok & (x >= lo1) & (x <= hi1), x

    for w in ([32 << k for k in range(12)] if near else [1 << 17]):
        if others:
            j2 = others[0]
            ys = np.arange(max(lo_at(i - j2), y0 - w), min(hi_at(i - j2), y0 + w) + 1, dtype=np.int64)
        else:
            ys = np.zeros(1, np.int64)
        if len(others) > 1:
            j3 = others[1]
            zs = np.arange(max(lo_at(i - j3), z0 - w), min(hi_at(i - j3), z0 + w) + 1)
            zs = zs[np.argsort(np.abs(zs - z0), kind="stable")] if near else rng.permutation(zs)
            zs = zs[:4096]
        else:
            zs = [z0]
        best = None
        for z in zs:
            if best is not None and (not near or abs(int(z) - z0) >= best[0]):
                break
            ok, x = solve(ys, int(z))
            if near:
                ok &= np.abs(x - x0) <= w
            if ok.any():
                cost = np.abs(x - x0) + np.abs(ys - y0) + abs(int(z) - z0)
                k = int(np.argmin(np.where(ok, cost, np.iinfo(np.int64).max))) if near else \
                    int(rng.choice(np.nonzero(ok)[0]))
                if best is None or cost[k] < best[0]:
                    best = (int(cost[k]), int(x[k]), int(ys[k]), int(z))
        if best is not None:
            s[i - j1] = best[1]
            if others:
                s[i - others[0]] = best[2]
            if len(others) > 1:
                s[i - others[1]] = best[3]
            assert prediction(s, c, i) == target % M35
            return True
    return False


def place_tie_difference(ch0, ch1, c, i, target=TIE, rng=None, near=True):
    """place_tie on the difference ch0 - ch1 of a stereo frame, moving ch0 only, so that both channels stay
    inside int16."""
    d = ch0 - ch1
    if not place_tie(d, c, i, lo=-32768 - ch1, hi=32767 - ch1, target=target, rng=rng, near=near):
        return False
    ch0[:] = d + ch1
    return True


def partial_sum_bound(c, lim):
    """A bound on every partial sum of the prediction of a signal with |s| <= lim."""
    return sum(abs(int(x)) for x in c[1:]) * lim


def assert_in_domain(O, u, lim):
    """Unit u and every candidate of its repair have coefficients and partial sums below 2^62 on |s| <= lim, so
    that the reference decoder is defined on all of them (DESIGN.md 7)."""
    cs = [u.c]
    for cand in range(3 * u.order - 1 if u.order >= 2 else 0):
        p = candidate_predictor(u, cand)
        if p is not None:
            cs.append(O.lpc_coefficients(p[1], p[0]))
    for c in cs:
        assert partial_sum_bound(c, lim) < DOMAIN, "a predictor outside the reference decoder's domain"
