"""An exact integer model of the reference decoder (TEST INFRASTRUCTURE), with the reference's domain.

    synthesise   SampleGenerator::generateSamples (src/lpc/sample_generator.cpp:11-30):
                   s[0] = r[0];  s[i] = r[i] - (int32)((2^34 - sum_{j=1..order} c[j]*s[i-j]) >> 35)
                 run in numpy int64, one step per sample, batched over subframes.
    decode       FrameDecoder::process (src/frame/frame_decoder.cpp:11-72): independent subframes first,
                 then dependent ones as parent - difference, each into the slot its `channel` field names;
                 interleaved with the (int16)(uint16) cast of the WAV writer (src/file/wav_file.cpp:249-251).

The predictor c[] comes from the CPU oracle (lpc_coefficients, pinned against the reference elsewhere).

The reference is written in int64/int32 C++ and is only defined while nothing overflows.  A subframe is
IN THE DOMAIN when
  - its q index the dequantisation tables inside [-64, 63] (linear_predictor.cpp:23-27, no bound check);
  - every 2^35 * coefficient of the float step-up is below 2^62 in magnitude, so the (int64_t) conversion
    (linear_predictor.cpp:59) is defined;
  - at every step 2^34 + sum_j |c[j]| * |s[i-j]| < 2^62, which bounds every partial sum of `temp`;
  - r[i] - (temp >> 35) stays inside int32 (and for a dependent subframe, parent - difference as well).
The bounds are evaluated in float64: 2^62 leaves a factor of two to int64's limit, far more than float64
rounding can take.  Outside the domain the reference's result is undefined and the tests assert nothing
about it.
"""
import pathlib
import struct

import numpy as np

import oracle_lib as ol

FRAME = 2048
Q = 35
HALF = 1 << (Q - 1)
LIMIT = float(1 << 62)
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1

# the reference's dequantisation tables (src/include/lpc.hpp): the first-order table is stored as a golden
# vector; the second-order one is its negation except for index 0; higher orders are q / 64
FIRST = np.load(pathlib.Path(__file__).resolve().parent / "golden" / "lpc_first_order.npy")
SECOND = -FIRST
SECOND[0] = struct.unpack("<d", struct.pack("<Q", 0xBFE0000000000001))[0]   # -0.5 - 2^-53


def _port():
    return ol.load("port")


def reflection(order, q):
    """LinearPredictor::dequantizeReflectionCoefficients; None if a q indexes outside the tables."""
    if order <= 1:
        return [0.0]
    q = [int(v) for v in q[:order]]
    if min(q) < -64 or max(q) > 63:
        return None
    return [float(FIRST[q[0] + 64]), float(SECOND[q[1] + 64])] + [float(v) / 64.0 for v in q[2:]]


def coefficients_in_domain(cases):
    """cases: iterable of (order, q).  True where the reference's step-up (linear_predictor.cpp:30-61, redone
    here in float64 in the same operation order) keeps every 2^35 * coefficient below 2^62."""
    out = []
    for order, q in cases:
        k = reflection(order, q)
        if k is None:
            out.append(False)
            continue
        t = [0.0] * max(order, 1)
        for i in range(order):
            t[i] = k[i]
            half = i >> 1
            for j in range(half):
                a, b = t[j], t[i - 1 - j]
                t[j] = a + k[i] * b
                t[i - 1 - j] = b + k[i] * a
            if i & 1:
                t[half] = t[half] + t[half] * k[i]
        out.append(all(abs(34359738368.0 * v) < LIMIT for v in t[:order]))
    return np.array(out, bool)


def prediction(S, C):
    """Non-recursive half of the recurrence for KNOWN samples: p[i] = (2^34 - sum_j C[:, j-1] * S[:, i-j]) >> 35
    with S[:, <0] = 0, plus the per-row domain bound.  S int64 [n, FRAME], C int64 [n, W] = c[1..W]."""
    S = np.asarray(S, np.int64)
    C = np.asarray(C, np.int64)
    n, W = C.shape
    acc = np.full(S.shape, HALF, np.int64)
    bound = np.full(S.shape, float(HALF))
    aS = np.abs(S.astype(np.float64))
    for j in range(1, W + 1):
        cj = C[:, j - 1:j]
        if not cj.any():
            continue
        acc[:, j:] -= cj * S[:, :-j]                   # wraps outside the domain; flagged below
        bound[:, j:] += np.abs(cj.astype(np.float64)) * aS[:, :-j]
    return acc >> Q, (bound < LIMIT).all(axis=1)


def coefficients(orders, qs, O=None):
    """c[1..W] per subframe from the oracle, zero padded to the largest order (W >= 1)."""
    O = O or _port()
    W = max(1, max(int(o) for o in orders))
    C = np.zeros((len(orders), W), np.int64)
    for i, (o, q) in enumerate(zip(orders, qs)):
        o = int(o)
        c = O.lpc_coefficients(np.asarray(q[:o], np.int32), o)
        C[i, :c.size - 1] = c[1:]
    return C


def synthesise(res, orders, qs, O=None):
    """res int32 [n, 2048], orders [n], qs [n][>= order] -> (samples int32 [n, 2048], in_domain bool [n])."""
    res = np.asarray(res, np.int64).reshape(-1, FRAME)
    n = res.shape[0]
    C = coefficients(orders, qs, O)
    W = C.shape[1]
    Crev = C[:, ::-1].copy()                            # Crev[:, m] = c[W - m]
    S = np.zeros((n, W + FRAME), np.int64)              # W zero samples of history in front
    fits = np.ones(n, bool)
    for i in range(FRAME):
        temp = HALF - (S[:, i:i + W] * Crev).sum(axis=1)
        v = res[:, i] - (temp >> Q)
        fits &= (v >= I32_MIN) & (v <= I32_MAX)
        S[:, W + i] = ((v - I32_MIN) & 0xFFFFFFFF) + I32_MIN
    out = S[:, W:]
    _, bounded = prediction(out, C)
    ok = fits & bounded & coefficients_in_domain(zip(orders, qs))
    return out.astype(np.int32), ok


def decode(subs, channels, O=None):
    """Crafted subframes (tests/crafted.Sub, file order, `channels` per frame) -> (interleaved int16 PCM,
    int32 planes [n_frames, channels, 2048] indexed by channel field, in_domain bool per subframe)."""
    n = len(subs)
    assert n % channels == 0
    syn, ok = synthesise(np.stack([s.res for s in subs]), [s.order for s in subs], [s.q for s in subs], O)
    n_frames = n // channels
    planes = np.zeros((n_frames, channels, FRAME), np.int64)
    dom = ok.copy()
    for f in range(n_frames):
        idx = range(f * channels, (f + 1) * channels)
        for i in idx:
            if subs[i].type == 0:
                planes[f, subs[i].channel] = syn[i]
        for i in idx:
            if subs[i].type == 1:
                p = next(k for k in idx if subs[k].type == 0 and subs[k].channel == subs[i].parent)
                v = planes[f, subs[i].parent] - syn[i].astype(np.int64)
                dom[i] = dom[i] and dom[p] and v.min() >= I32_MIN and v.max() <= I32_MAX
                planes[f, subs[i].channel] = v
    pcm = (planes.transpose(0, 2, 1).reshape(-1) & 0xFFFF).astype(np.uint16).view(np.int16)
    return pcm, planes.astype(np.int32), dom
