"""Crafted decoder input (TEST INFRASTRUCTURE): subframes with chosen channel fields, types, parents,
predictor orders, quantised reflection coefficients and residues, Rice-coded and laid out as a
descriptor table + word arena the way a .sela file carries them (src/file/sela_file.cpp:105-137).

The decoder accepts anything the descriptors allow -- any order 0..100, any q, any int32 residue -- while
the encoder only ever produces a narrow slice of that.  These builders reach the rest: samples chosen
first (any int32) and residues derived from them through the decoder's own prediction, so the decoded
signal is known exactly (tests/exact_decode.py) and can be steered into every sample range.
"""
from dataclasses import dataclass

import numpy as np

import exact_decode as X
import exact_rice as XR
from oracle_lib import DESC_DTYPE

FRAME = 2048
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1


def rice_code(O, x):
    """(k, words) as the reference's RiceEncoder writes them.  Its signed-to-unsigned step shifts in int32
    (rice_encoder.cpp:12-18), which is only defined for |x| < 2^30; beyond that the exact encoder model
    (exact_rice.encode) extends it the way the device does, and the reference's DEcoder reads that back
    correctly for every int32."""
    x = np.asarray(x, np.int64)
    if x.size == 0 or np.abs(x).max() < (1 << 30):
        return O.rice_encode(x.astype(np.int32))
    return XR.encode(x)


@dataclass
class Sub:
    """One subframe: descriptor fields plus the decoded values of its two Rice streams."""
    channel: int
    type: int
    parent: int
    order: int
    q: np.ndarray          # int32 [order]
    res: np.ndarray        # int32 [2048]
    samples: np.ndarray = None   # what the reference decodes from them, where the builder knows it


def build(O, subs, gap_words=(0, 1, 2, 3, 5)):
    """subs in file order -> (descs, words).  All-ones filler words between streams put every stream at
    every 16-byte phase of the arena (and must never be parsed)."""
    descs = np.zeros(len(subs), DESC_DTYPE)
    arena, at = [], 0
    for i, s in enumerate(subs):
        kq, wq = rice_code(O, np.asarray(s.q[:s.order], np.int64))
        kr, wr = rice_code(O, np.asarray(s.res, np.int64))
        assert wq.size <= 0xFFFF and wr.size <= 0xFFFF, (i, wq.size, wr.size)
        d = descs[i]
        d["channel"], d["subframe_type"], d["parent_channel"] = s.channel, s.type, s.parent
        d["lpc_order"], d["samples"] = s.order, FRAME
        for name, k, w in (("refl", kq, wq), ("res", kr, wr)):
            pad = gap_words[(2 * i + (name == "res")) % len(gap_words)]
            arena.append(np.full(pad, 0xFFFFFFFF, np.uint32))
            at += pad
            d[name + "_rice_param"], d[name + "_words"], d[name + "_offset"] = k, w.size, at
            arena.append(np.asarray(w, np.uint32))
            at += w.size
    arena.append(np.full(4, 0xFFFFFFFF, np.uint32))
    return descs, np.concatenate(arena)


# ---------------------------------------------------------------------------------- subframe content --

def draw_q(rng, order, low=(-64, 63), high=8):
    """q[0], q[1] anywhere in [-64, 63] (q[1] = -64 is the SECOND0 table entry), higher q in [-high, high]."""
    q = np.zeros(order, np.int32)
    q[:2] = rng.integers(low[0], low[1] + 1, min(order, 2))
    if order > 2:
        q[2:] = rng.integers(-high, high + 1, order - 2)
    return q


def residues_for(O, samples, order, q):
    """The residues from which the reference decoder reproduces `samples` exactly (None when a residue would
    leave int32 or the prediction leaves the reference's domain)."""
    s = np.asarray(samples, np.int64)
    c = np.asarray(O.lpc_coefficients(np.asarray(q, np.int32), order), np.int64)
    if not X.coefficients_in_domain([(order, q)])[0]:
        return None
    pred, ok = X.prediction(s[None, :], c[None, 1:])
    r = s + pred[0]
    if not ok[0] or r.min() < I32_MIN or r.max() > I32_MAX:
        return None
    return r.astype(np.int32)


def signal(rng, amp, n=FRAME):
    """A band-limited random walk scaled to about +-amp, plus white noise: content every predictor order sees."""
    w = np.cumsum(rng.normal(0, 1, n))
    w = w - np.linspace(w[0], w[-1], n)
    w = w / max(np.abs(w).max(), 1e-9)
    x = amp * (0.8 * w + 0.2 * rng.uniform(-1, 1, n))
    return np.clip(np.round(x), I32_MIN, I32_MAX).astype(np.int64)


def edge_q(rng, order):
    """The only predictors that can take int32-limit samples inside the domain are tiny: q = 26 / 27 are the
    first-order entries closest to a zero reflection coefficient, higher q = 0 is exactly zero."""
    q = np.zeros(order, np.int32)
    q[:2] = rng.choice([26, 27], min(order, 2))
    return q


def edge_spikes(O, rng, base, order, q, n_spikes=16, margin=256):
    """`base` with n_spikes samples placed within `margin` of INT32_MAX or INT32_MIN, further apart than the
    predictor is long.  The side is picked per spike so that the residue s + prediction stays inside int32."""
    s = np.asarray(base, np.int64).copy()
    c = [int(v) for v in O.lpc_coefficients(np.asarray(q, np.int32), order)]
    gap = max(order + 1, FRAME // (n_spikes + 1))
    pos = np.arange(1, n_spikes + 1) * gap + rng.integers(-3, 4, n_spikes)
    for i in pos[pos < FRAME]:
        t = (1 << 34) - sum(c[j] * int(s[i - j]) for j in range(1, order + 1) if i - j >= 0)
        p = t >> 35
        u = int(rng.integers(0, margin))
        s[i] = I32_MAX - u if p <= 0 else I32_MIN + u
    return s


def crafted_subframe(O, rng, order, kind, channel=0, sub_type=0, parent=None, tries=40):
    """A subframe whose decoded samples fall in range `kind`:
         "small"  |s| <= 65535
         "wide"   beyond 16 bits (the int16 output wraps), in [-2^17, 2^22)
         "neg17"  below -2^17 in front of non-zero taps (outside the biased IIR's old window)
         "edge"   within 2^8 of the int32 limits
    Predictors are redrawn until the case is inside the reference's domain."""
    parent = channel if parent is None else parent
    for _ in range(tries):
        if kind == "edge":
            q = edge_q(rng, order)
            base = signal(rng, 3000)
            s = edge_spikes(O, rng, base, order, q)
        else:
            q = draw_q(rng, order, high=8 if kind == "small" else 4)
            amp = {"small": 30000, "wide": 1 << 20, "neg17": 1 << 19}[kind]
            s = signal(rng, amp)
            if kind == "small":
                s = np.clip(s, -65535, 65535)
            if kind == "wide":                                 # kept apart from "neg17": nothing below -2^17
                s = s - s.min() - (1 << 17)
            if kind == "neg17":
                s[rng.integers(0, FRAME, 64)] = -int(rng.integers(131073, 1 << 21))
        r = residues_for(O, s, order, q)
        if r is not None:
            return Sub(channel, sub_type, parent, order, q, r, s.astype(np.int32))
    raise AssertionError("no in-domain %s subframe of order %d" % (kind, order))


def difference_subframe(O, rng, order, parent, channel, kind="small", tries=40):
    """A difference-coded subframe (type 1) on `parent` (a Sub with known samples) whose parent - difference
    stays inside int32: small values, of the parent's sign wherever the parent is large.  kind "edge": within
    2^8 of INT32_MIN wherever the parent is, so that both operands of parent - difference are near INT32_MIN."""
    big = np.abs(parent.samples.astype(np.int64)) > (1 << 30)
    low = parent.samples.astype(np.int64) <= I32_MIN + 255
    for _ in range(tries):
        q = edge_q(rng, order) if kind == "edge" else draw_q(rng, order)
        d = signal(rng, 3000)
        d[big] = np.sign(parent.samples[big]) * np.abs(d[big])
        if kind == "edge":
            d[low] = I32_MIN + rng.integers(0, 256, int(low.sum()))
        r = residues_for(O, d, order, q)
        if r is not None:
            return Sub(channel, 1, parent.channel, order, q, r, d.astype(np.int32))
    raise AssertionError("no in-domain difference subframe of order %d" % order)


def sample_ranges(samples):
    """Which of the four ranges a set of int32 samples reaches."""
    s = np.asarray(samples, np.int64)
    return {
        "small": bool((np.abs(s) <= 65535).any()),
        "wide": bool((np.abs(s) > 65535).any()),
        "neg17": bool((s < -(1 << 17)).any()),
        "edge": bool(((s >= I32_MAX - 255) | (s <= I32_MIN + 255)).any()),
    }
