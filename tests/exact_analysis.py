"""Exact model of the encoder's floating-point analysis (lpc::ResidueGenerator), in numpy float64.

Restates, operation for operation, what src/lpc/residue_generator.cpp computes before the integer stages:
quantizeSamples (x = s / 32767), the mean chain and generateAutoCorrelation (mean-removed lags 0..100, then
normalised by lag 0), generateReflectionCoefficients (the Schur recursion, always all 100 coefficients),
generateoptimalLpcOrder and quantizeReflectionCoefficients.  Every sum is ONE sequential chain, as in the
reference; the model is vectorised across frames and across lags/elements, never across the terms of a sum.
numpy's float64 operations are IEEE-rounded and never fused, so the model is bitwise exact wherever the
reference is.  It is pinned against the compiled reference in tests/test_exact_analysis.py.

Two switches restate plausible edits that break the reference's rounding without changing its maths:
lag_chains=2 sums each lag as two interleaved chains (even j, odd j) added at the end, and
schur_reciprocal=True takes k = -g * (1/err) instead of -g / err.  Tests use them to show that a corpus can
see such an edit.
"""
import numpy as np

SQRT2 = 1.4142135623730950488016887242096  # src/include/lpc.hpp:9
MAX_ORDER = 100                            # src/include/lpc.hpp:7
LAGS = MAX_ORDER + 1
THRESHOLD = 0.05                           # residue_generator.cpp:73


def quantise(k):
    """q of every k as coefficient 0, as coefficient 1 and as any later one (residue_generator.cpp:80-96).
    A NaN (k outside [-1, 1] under the square root, or a NaN k) quantises to 0.  -> three int64 arrays."""
    k = np.asarray(k, np.float64)
    with np.errstate(invalid="ignore"):
        v0 = np.floor(64.0 * (-1.0 + SQRT2 * np.sqrt(k + 1.0)))
        v1 = np.floor(64.0 * (-1.0 + SQRT2 * np.sqrt(-k + 1.0)))
        vr = np.floor(64.0 * k)
    return tuple(np.where(np.isnan(v), 0.0, v).astype(np.int64) for v in (v0, v1, vr))


def significant(k):
    """Whether k counts for the order (residue_generator.cpp:73); NaN does not."""
    with np.errstate(invalid="ignore"):
        return np.abs(np.asarray(k, np.float64)) > THRESHOLD


def analyse(s, lag_chains=1, schur_reciprocal=False):
    """s: int [F, N] signals -> dict of mean[F], ac[F, 101], k[F, 100], order[F], q[F, 100] (zero past the order)."""
    s = np.atleast_2d(np.asarray(s, np.int64))
    F, N = s.shape
    x = s.astype(np.float64) / 32767.0                       # quantizeSamples: one correctly rounded division
    total = np.zeros(F)
    for j in range(N):
        total = total + x[:, j]
    mean = total / N
    d = x - mean[:, None]                                    # the reference recomputes the same value per use

    chains = [np.zeros((F, LAGS)) for _ in range(lag_chains)]
    for j in range(N):
        m = min(j, LAGS - 1)                                 # lags 0..m have a term at j
        a = chains[j % lag_chains]
        a[:, :m + 1] = a[:, :m + 1] + d[:, j:j + 1] * d[:, j - m:j + 1][:, ::-1]   # ac[i] += d[j] * d[j - i]
    ac = chains[0]
    for extra in chains[1:]:
        ac = ac + extra

    with np.errstate(invalid="ignore", divide="ignore"):
        ac[:, 1:] = ac[:, 1:] / ac[:, :1]                    # silence: 0 / 0 = NaN, which runs through to q = 0
        ac[:, 0] = 1.0

        g0 = ac[:, 1:].copy()
        g1 = g0.copy()
        err = ac[:, 0].copy()
        k = np.zeros((F, MAX_ORDER))
        for i in range(MAX_ORDER):
            if i:
                kp = k[:, i - 1:i]
                n = MAX_ORDER - i
                up = g1[:, 1:n + 1].copy()                   # both updates read the old g1[j + 1]
                g1[:, :n] = up + kp * g0[:, :n]
                g0[:, :n] = up * kp + g0[:, :n]
            head = g1[:, 0]
            k[:, i] = -head * (1.0 / err) if schur_reciprocal else -head / err
            err = err + head * k[:, i]

    big = significant(k)
    order = np.where(big.any(axis=1), MAX_ORDER - np.argmax(big[:, ::-1], axis=1), 1)   # default 1 (lpc.hpp:76)
    q0, q1, qr = quantise(k)
    q = qr.copy()
    q[:, 0] = q0[:, 0]
    q[:, 1] = q1[:, 1]
    q[np.arange(MAX_ORDER)[None, :] >= order[:, None]] = 0
    return dict(mean=mean, ac=ac, k=k, order=order, q=q)


def _from_key(key):
    """Inverse of the order-preserving map double -> int64 (the bit pattern, negated for negative doubles)."""
    key = np.asarray(key, np.int64)
    mag = np.abs(key).view(np.float64)
    return np.where(key < 0, -mag, mag)


def _to_key(x):
    bits = np.abs(np.asarray(x, np.float64)).view(np.int64)
    return np.where(np.signbit(x), -bits, bits)


def first_reaching(f, levels, lo=-1.0, hi=1.0):
    """For a non-decreasing f on the doubles of [lo, hi]: the smallest double k with f(k) >= L, per level L.
    Bisects on the ordered integer keys of the doubles, all levels at once."""
    levels = np.asarray(levels, np.int64)
    a = np.full(levels.shape, _to_key(lo))   # f(from_key(a)) < L  (checked below)
    b = np.full(levels.shape, _to_key(hi))   # f(from_key(b)) >= L
    assert (f(_from_key(a)) < levels).all() and (f(_from_key(b)) >= levels).all()
    while (b - a > 1).any():
        mid = a + (b - a) // 2
        up = f(_from_key(mid)) >= levels
        b = np.where(up, mid, b)
        a = np.where(up, a, mid)
    return _from_key(b)


def quantiser_probes():
    """Inputs where the quantiser or the order threshold can go wrong: for every level of q[0] and of q[1] the
    double where its floor steps (found by bisection on this model), the steps of the linear quantiser at
    L/64, each with its neighbours within +-2 ulps; then +-1, +-0, the doubles just outside [-1, 1] and
    beyond (NaN under the square root), NaN, and the 0.05 threshold +-1 ulp.  (Not the infinities: 64 * inf
    does not convert to int32, in C or on the device.)"""
    q0 = lambda k: quantise(k)[0]
    neg_q1 = lambda k: -quantise(k)[1]          # q[1] falls as k rises
    steps = [first_reaching(q0, np.arange(-63, 65)), first_reaching(neg_q1, np.arange(-63, 65)),
             np.arange(-64, 65) / 64.0]
    out = []
    for b in np.concatenate(steps):
        x = [b]
        for direction in (np.inf, -np.inf):
            y = b
            for _ in range(2):
                y = np.nextafter(y, direction)
                x.append(y)
        out += x
    t = THRESHOLD
    out += [1.0, -1.0, 0.0, -0.0, np.nextafter(1.0, 2.0), np.nextafter(-1.0, -2.0), 1.5, -1.5, 2.0, -2.0, np.nan,
            t, np.nextafter(t, 1.0), np.nextafter(t, 0.0), -t, np.nextafter(-t, -1.0), np.nextafter(-t, 0.0)]
    return np.array(out, np.float64)


def quantiser_expected(k):
    """quantiser_probes' layout of the answers: int32 [n, 4] = q as coefficient 0, 1, any later one, |k| > 0.05."""
    q0, q1, qr = quantise(k)
    return np.stack([q0, q1, qr, significant(k)], axis=1).astype(np.int32)


def same_bits(a, b):
    """Elementwise: the same 64-bit pattern (so +0 and -0 differ), except that NaN equals NaN whatever its
    payload (x86 and CUDA produce different NaN payloads)."""
    a = np.ascontiguousarray(a, np.float64)
    b = np.ascontiguousarray(b, np.float64)
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))
