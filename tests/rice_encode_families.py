"""Value streams for the Rice encoder tests (TEST INFRASTRUCTURE): families of input the encoder's parameter search
and packer (warp_rice_choose, warp_rice_pack in sela_b200/csrc/rice.cuh) must code exactly, most of which real
audio never produces.

Every family returns a list of Batch: int32 values [n, stride], the count of each row that is coded, and the exact
model's answer (exact_rice.encode_batch).  Values behind a row's count are random and large: they are never coded.
Each builder asserts through the model that its streams have the property the family is named for.

    lengths    every n from 0 to 2048 at three value scales: every lane split (4 to 64 values per lane), empty
               trailing lanes, n mod 4 != 0
    winner     for every k in 0..19, streams whose unique arg-min is k, at n = 2048 and at short n
    ties       total_k == total_{k+1} for every k in 0..18 (the lowest k must win), three-way plateaus, and
               near-ties one bit either way
    planes     in every lane, every value with the same bit p set (p = 0..31): a lane count of exactly 64 at
               n = 2048, a partial last lane at n = 1985..2047; all 19 low bits set; values >= 2^19
    long       symbols of 31-k, 32-k, 32, 33, 63, 64, 65 and about 1000 ones as a lane's first or last value,
               with lanes starting at every bit phase of a word
    sharing    k = 0 streams of 0s and 1s at n <= 128 (up to eight lanes in one word), and streams whose every
               lane codes to a whole number of words, so that lane boundaries fall on word boundaries
    extremes   INT32_MIN, INT32_MAX, +-2^30 and +-(2^30 - 1) at n = 1, 64 and 2048 (the 2048-value INT32_MIN stream
               takes 525 504 words)
    stride     row strides 1..7 and 2047 with counts < stride, the values behind the count chosen so that coding
               them would change k

The lane split mirrors rice_lane_range: `per` = ceil(n / 32) rounded up to a multiple of 4 values per lane.
"""
import functools
from dataclasses import dataclass

import numpy as np

import exact_rice as XR

FRAME = 2048
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
KS = range(XR.MAX_RICE)


@dataclass
class Batch:
    values: np.ndarray   # int32 [n, stride]
    counts: np.ndarray   # int64 [n]
    enc: XR.Encoded      # the model on values[i, :counts[i]]


def lane_ranges(n):
    """rice_lane_range: (per, lo [32], hi [32])."""
    per = (((n + 31) >> 5) + 3) & ~3
    lo = np.minimum(np.arange(32) * per, n)
    return per, lo, np.minimum(lo + per, n)


def from_u(u):
    """int32 values whose zig-zag is u (any uint32)."""
    return XR.unzigzag(np.asarray(u, np.uint64)).astype(np.int64)


def symbol_starts(u, k):
    """First bit of each symbol of one stream at k."""
    lens = (np.asarray(u, np.uint64) >> np.uint64(k)).astype(np.int64) + 1 + k
    return np.concatenate([[0], np.cumsum(lens)[:-1]])


def lane_starts(u, k):
    """First bit of each non-empty lane of one stream of len(u) values at k."""
    _, lo, hi = lane_ranges(len(u))
    starts = np.append(symbol_starts(u, k), int(((np.asarray(u, np.uint64) >> np.uint64(k)).astype(np.int64) + 1 + k).sum()))
    return starts[lo[hi > lo]]


def make_batch(rng, rows, stride=FRAME, counts=None):
    """rows: 1-D int value arrays; each goes into a row of `stride` values, random values of up to 2^29 behind it."""
    counts = np.array([len(r) for r in rows] if counts is None else counts, np.int64)
    values = rng.integers(-(1 << 29), 1 << 29, (len(rows), stride))
    for i, r in enumerate(rows):
        values[i, :len(r)] = r
    return Batch(values.astype(np.int32), counts, XR.encode_batch(values, counts))


def _u_rows(b):
    return [XR.zigzag(b.values[i, :c]) for i, c in enumerate(b.counts)]


# -------------------------------------------------------------------------------------------- families --

def lengths(rng):
    out = []
    for scale in (3, 1000, 1 << 21):
        out.append(make_batch(rng, [rng.integers(-scale, scale + 1, n) for n in range(FRAME + 1)]))
    pers = {lane_ranges(n)[0] for n in range(1, FRAME + 1)}
    assert pers == set(range(4, 65, 4)), pers
    assert any((lambda p, lo, hi: (hi == lo).any())(*lane_ranges(n)) for n in range(1, FRAME + 1))
    assert [np.array_equal(b.counts, np.arange(FRAME + 1)) for b in out] == [True] * 3
    ks = [int(b.enc.k[-1]) for b in out]
    assert ks[0] <= 2 and 7 <= ks[1] <= 10 and ks[2] == 19, ks              # three regimes of k
    assert (np.abs(out[2].values[-1]) >= 1 << 18).any()                    # u >= 2^19 reaches `top`
    return out


def winner(rng):
    rows = []
    for k in KS:
        for n in (FRAME, 5, 33, 100):
            m = 64 if n == FRAME else 512
            t = rng.uniform(0.2, 3.0, (m, 1))
            u = np.minimum(np.floor(rng.exponential(1.0, (m, n)) * t * (1 << k)), (1 << 31) - 1).astype(np.uint64)
            e = XR.encode_batch(from_u(u))
            unique = (np.sort(e.totals, axis=1)[:, 1] > e.totals.min(axis=1)) & (e.k == k)
            pick = np.flatnonzero(unique)[:2]
            assert pick.size == 2, ("no unique winner", k, n)
            rows += [from_u(u[i]) for i in pick]
    b = make_batch(rng, rows)
    srt = np.sort(b.enc.totals, axis=1)
    assert (srt[:, 1] > srt[:, 0]).all()                                    # every arg-min is unique
    assert set(b.enc.k.tolist()) == set(KS)
    return [b]


def ties(rng):
    rows, want = [], []        # want: (lowest arg-min, the set of k at the minimum, margin to the runner-up)

    def band(k, n):
        u = rng.integers(1 << k, 1 << (k + 1), n).astype(np.uint64)
        if k:
            u[:8] |= np.uint64(1 << (k - 1))                                # f(k-1) stays above f(k)
        return u
    for k in range(XR.MAX_RICE - 1):
        for n in (FRAME, 64, 7, 1985):
            rows.append(from_u(band(k, n)))                                 # every u >> k == 1
            want.append((k, {k, k + 1}, None))
        for n in (FRAME, 64):
            lo = rng.integers(0, 1 << k, n // 2) if k else np.zeros(n // 2, np.int64)
            hi = rng.integers(3 << k, 4 << k, n // 2)
            rows.append(from_u(rng.permutation(np.concatenate([lo, hi]).astype(np.uint64))))   # u >> k in {0, 3}
            want.append((k, {k, k + 1}, None))
        for n in (FRAME, 100):                                             # near-ties: one symbol moved by one bit
            u = band(k, n)
            u[-1] = rng.integers(0, 1 << k) if k else 0                     # sum of ceil((u >> k) / 2) = n - 1
            rows.append(from_u(u))
            want.append((k, {k}, 1))
            u = band(k, n)
            u[-1] = rng.integers(3 << k, 4 << k)                            # n + 1
            rows.append(from_u(u))
            want.append((k + 1, {k + 1}, 1))
    for k in range(1, XR.MAX_RICE - 1):
        for n in (FRAME, 100, 3):                                          # u in [2^k, 1.5 * 2^k): k-1, k, k+1 tie
            rows.append(from_u(rng.integers(1 << k, (1 << k) + (1 << (k - 1)), n).astype(np.uint64)))
            want.append((k - 1, {k - 1, k, k + 1}, None))
    b = make_batch(rng, rows)
    t = b.enc.totals
    for i, (k, at_min, margin) in enumerate(want):
        assert b.enc.k[i] == k and set(np.flatnonzero(t[i] == t[i].min()).tolist()) == at_min, (i, k, t[i])
        if margin:
            assert np.sort(t[i])[1] - t[i].min() == margin, (i, t[i])
    two = {min(s) for _, s, _ in want if len(s) == 2}
    assert two == set(range(XR.MAX_RICE - 1))                               # every (k, k+1) ties
    assert {min(s) for _, s, _ in want if len(s) == 3} == set(range(XR.MAX_RICE - 2))
    return [b]


def planes(rng):
    rows, bits = [], []
    for p in range(32):        # above bit 19 only `top` sees the bit, and the streams grow to 2^(p - 19) ones a value
        for n in range(1985, FRAME + 1) if p < 20 else (1985, 2000, 2016, 2047, FRAME):
            u = (np.uint64(1 << p) | (rng.integers(0, 1 << 32, n, dtype=np.uint64) & np.uint64((1 << p) - 1)))
            rows.append(from_u(u))
            bits.append(p)
    low = (1 << 19) - 1
    for n in (FRAME, 1985, 2000, 64):
        rows.append(from_u(np.full(n, low, np.uint64)))                                      # 19 planes full
        rows.append(from_u(np.uint64(low) | (rng.integers(1, 1 << 13, n).astype(np.uint64) << np.uint64(19))))
    b = make_batch(rng, rows)
    us = _u_rows(b)
    for i, p in enumerate(bits):
        assert ((us[i] >> np.uint64(p)) & np.uint64(1)).all()
        assert b.enc.k[i] == min(p, XR.MAX_RICE - 1), (p, b.enc.k[i])
    _, lo, hi = lane_ranges(FRAME)
    assert (hi - lo == 64).all() and sorted(p for p, c in zip(bits, b.counts) if c == FRAME) == list(range(32))
    last = {int(c) - 31 * 64 for c in b.counts[:len(bits)]}
    assert last == set(range(1, 65))                                        # every size of the last lane
    assert all((u & np.uint64(low) == low).all() for u in us[len(bits):])   # all 19 planes count every value
    assert {int(u.max()) >> 19 > 0 for u in us[len(bits):]} == {False, True}
    return [b]


def _background(rng, k, n):
    """Values whose arg-min is k with a margin of about n/10 below and n/2 above (k = 0: 0.6 n)."""
    if k == 0:
        return (rng.random(n) < 0.4).astype(np.uint64)
    hi = rng.random(n) < 0.55
    return np.where(hi, rng.integers(3 << (k - 1), 2 << k, n), rng.integers(0, 1 << (k - 1), n)).astype(np.uint64)


def long(rng):
    rows, marks = [], []
    for k in (0, 1, 5, 11, 18, 19):
        for q in (31 - k, 32 - k, 32, 33, 63, 64, 65, int(rng.integers(1000, 1100))):
            big = q > 65
            for n, lanes in ((FRAME, (0, 5, 13, 31)), (1000, (2, 31))):
                if big and n != FRAME:
                    continue
                _, lo, hi = lane_ranges(n)
                for side in ("first", "last"):
                    for _ in range(2):
                        u = _background(rng, k, n)
                        at = np.array([lo[l] if side == "first" else hi[l] - 1 for l in lanes])
                        at = at[:1] if big else at
                        u[at] = (np.uint64(q) << np.uint64(k)) | (rng.integers(0, 1 << k, at.size).astype(np.uint64)
                                                                  if k else np.uint64(0))
                        rows.append(from_u(u))
                        marks.append((k, q, side, at))
    b = make_batch(rng, rows)
    us = _u_rows(b)
    phases = set()
    for i, (k, q, side, at) in enumerate(marks):
        assert b.enc.k[i] == k, (i, k, q, b.enc.k[i])
        assert ((us[i][at] >> np.uint64(k)) == q).all()
        if side == "first":
            phases |= set((symbol_starts(us[i], k)[at] % 32).tolist())
    assert phases == set(range(32))                                         # a lane's first bit at every phase
    assert {(k, q, s) for k, q, s, _ in marks} == {(k, q, s) for k, q, _, _ in marks for s in ("first", "last")}
    return [b]


def sharing(rng):
    rows = []
    for n in range(1, 129):
        rows += [from_u(rng.integers(0, 2, n)), from_u(rng.integers(0, 2, n))]
    for n in (1, 8, 31, 64, 127, 128):
        rows += [np.full(n, -1), np.zeros(n, np.int64)]                    # u = 1 everywhere, u = 0 everywhere
    small = make_batch(rng, rows)
    assert (small.enc.k == 0).all()
    assert max(lane_ranges(int(n))[0] for n in small.counts) == 4
    most = 0
    for u in _u_rows(small):
        w = lane_starts(u, 0) // 32
        most = max(most, int(np.bincount(w).max()) if w.size else 0)
    assert most >= 7, most                                                  # up to 8 lanes start in one word

    rows, ks = [], []
    for k in (0, 1, 3, 11, 19):
        for n in (FRAME, 1000):
            for _ in range(2):
                u = _background(rng, k, n)
                _, lo, hi = lane_ranges(n)
                for a, z in zip(lo, hi):
                    if z > a:
                        d = -int(((u[a:z] >> np.uint64(k)).astype(np.int64) + 1 + k).sum()) % 32
                        inc = d // (z - a) + (np.arange(z - a) < d % (z - a))
                        u[a:z] += inc.astype(np.uint64) << np.uint64(k)
                rows.append(from_u(u))
                ks.append(k)
    aligned = make_batch(rng, rows)
    for i, u in enumerate(_u_rows(aligned)):
        assert aligned.enc.k[i] == ks[i], (i, ks[i], aligned.enc.k[i])
        assert (lane_starts(u, ks[i]) % 32 == 0).all() and aligned.enc.bits[i] % 32 == 0
    return [small, aligned]


EXTREMES = (I32_MIN, I32_MAX, 1 << 30, -(1 << 30), (1 << 30) - 1, -((1 << 30) - 1))


def extremes(rng):
    rows = []
    for n in (1, 64, FRAME):
        rows += [np.full(n, v) for v in EXTREMES]
        rows.append(rng.choice(EXTREMES, n))
        rows.append(np.where(rng.random(n) < 0.5, rng.choice(EXTREMES, n), rng.integers(-9, 10, n)))
    b = make_batch(rng, rows)
    big = b.enc.n_words[(b.counts == FRAME) & (b.values == I32_MIN).all(axis=1)]
    assert big.tolist() == [FRAME * ((((1 << 32) - 1) >> 19) + 20) // 32]  # 525 504 words
    return [b]


def stride(rng):
    out = []
    for s in (1, 2, 3, 4, 5, 6, 7, 2047):
        counts = list(range(s)) * 3 if s < 8 else [0, 1, 4, 63, 64, 65, 1000, 1985, 2000, 2046] * 2
        rows = [rng.integers(-3, 4, c) for c in counts]
        b = make_batch(rng, rows, stride=s)
        b.values[:, :] = np.where(np.arange(s)[None, :] < b.counts[:, None], b.values,
                                  rng.choice([-(1 << 20), 1 << 20], b.values.shape))
        b = Batch(b.values, b.counts, XR.encode_batch(b.values, b.counts))
        whole = XR.encode_batch(b.values)
        coded = b.counts > 0
        assert (whole.k[coded] != b.enc.k[coded]).all()                     # the values behind would change k
        assert (b.counts < s).all()
        out.append(b)
    return out


FAMILIES = {"lengths": lengths, "winner": winner, "ties": ties, "planes": planes, "long": long,
            "sharing": sharing, "extremes": extremes, "stride": stride}
NAMES = sorted(FAMILIES)


@functools.lru_cache(maxsize=None)
def family(name, seed=0):
    """The batches of one family (cached: callers must not modify them)."""
    return FAMILIES[name](np.random.default_rng([seed, NAMES.index(name)]))


def in_reference_domain(b):
    """Rows of a batch whose coded values all have |x| < 2^30 (where the reference's zig-zag is defined)."""
    return [i for i, c in enumerate(b.counts) if c == 0 or np.abs(b.values[i, :c].astype(np.int64)).max() < (1 << 30)]
