"""The encoder's FIR residual (lpc.cuh, warp_fir_residual: mma.sync on byte limbs) against an exact integer model.

    fir_residues   r[i] = s[i] - (int32)((2^34 + sum_{j=1..order} c[j] * s[i-j]) >> 35),  s[<0] = 0,
                   the sum taken mod 2^64 (numpy int64 wraps), as generateResidues
                   (src/lpc/residue_generator.cpp:98-119) computes it wherever its int64 sum does not overflow.

The model is pinned to the C port's residues (CPU); the device function runs through selab200_fir_probe, for both
row forms: the int16 row of a channel unit and the row + parity bits of a 17-bit unit.
"""
import functools

import numpy as np
import pytest

import oracle_lib as ol
import signals
from sela_b200 import _lib

FRAME = 2048
MAX_ORDER = 100
Q = 35
HALF = 1 << (Q - 1)


def fir_residues(S, C, orders):
    """S int [n, 2048], C int64 [n, 101] (c[:, 0] unused), orders [n] -> int32 [n, 2048]."""
    S = np.asarray(S, np.int64)
    C = np.asarray(C, np.int64)
    orders = np.asarray(orders)
    acc = np.full(S.shape, HALF, np.int64)
    for j in range(1, MAX_ORDER + 1):
        cj = np.where(orders >= j, C[:, j], 0)[:, None]
        if cj.any():
            acc[:, j:] += cj * S[:, :-j]                 # wraps mod 2^64
    return (S - (acc >> Q)).astype(np.int32)


def signed_digits(c):
    """How many signed base-256 digits the device splits c into: the bytes of (c + H) ^ H, H = 0x8080...80."""
    H = 0x8080808080808080
    v = ((int(c) + H) % (1 << 64)) ^ H
    return (v.bit_length() + 7) // 8


def _with_digits(rng, L, size):
    """int64 values of at most L signed digits, the first one of exactly L."""
    e = rng.integers(-128, 128, size=(size, L)).astype(object)
    e[0, L - 1] = rng.choice([-128, -1, 1, 127])
    v = [sum(int(d) << (8 * p) for p, d in enumerate(row)) % (1 << 64) for row in e]
    out = np.array([x - (1 << 64) if x >= 1 << 63 else x for x in v], np.int64)
    assert signed_digits(out[0]) == L and max(signed_digits(x) for x in out) == L
    return out


def _natural():
    fam = signals.families()
    return np.stack([fam[n] for n in sorted(fam)]).astype(np.int32)


def test_model_matches_the_port():
    """The model on the port's own (order, c) gives the port's residues, for 16- and 17-bit signals."""
    O = ol.load("port")
    x = _natural()
    rng = np.random.default_rng(5)
    x = np.concatenate([x, rng.integers(-65535, 65536, size=(4, FRAME), dtype=np.int32)])
    for s in x:
        a = O.lpc_analyse(s)
        C = np.zeros((1, MAX_ORDER + 1), np.int64)
        C[0, :a["c"].size] = a["c"]
        assert np.array_equal(fir_residues(s[None], C, [a["order"]])[0], a["res"])


def test_signed_digit_count():
    assert [signed_digits(v) for v in (0, 1, -1, 127, 128, -128, -129, 2 ** 63 - 1, -2 ** 63)] == \
        [0, 1, 1, 1, 2, 1, 2, 8, 8]


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = _lib.lib()
    assert L.selab200_init(0) == -1
    s = np.zeros(FRAME, np.int32)
    orders = np.zeros(1, np.int32)
    c = np.zeros(MAX_ORDER + 1, np.int64)
    res = np.zeros(FRAME, np.int32)
    assert L.selab200_fir_probe(s.ctypes.data, orders.ctypes.data, c.ctypes.data, 1, 0, res.ctypes.data) == -7
    ties = np.zeros(1, np.uint8)
    assert L.selab200_fir_tie_probe(s.ctypes.data, orders.ctypes.data, c.ctypes.data, 1, 0, res.ctypes.data,
                                    ties.ctypes.data) == -7
    from sela_b200 import SelaB200Error, codec
    with pytest.raises(SelaB200Error):
        codec.fir_tie_probe(s, orders, c, False)


# ----------------------------------------------------------------------------------------------------- GPU --

def _probe_both(S, C, orders, wide):
    from sela_b200 import codec
    got = codec.fir_probe(S, orders, C, wide)
    want = fir_residues(S, C, orders)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, "signals %s differ (first at order %d)" % (bad[:8].tolist(), np.asarray(orders)[bad[0]])


@pytest.mark.gpu
@pytest.mark.parametrize("wide", [False, True])
def test_every_order(wide):
    """Orders 0..100, k-step edges 24/25, 56/57, 88/89 included, full-width random coefficients."""
    rng = np.random.default_rng(11 + wide)
    orders = np.arange(MAX_ORDER + 1)
    lim = 65535 if wide else 32767
    S = rng.integers(-lim - (not wide), lim + 1, size=(orders.size, FRAME), dtype=np.int32)
    C = rng.integers(-2 ** 63, 2 ** 63 - 1, size=(orders.size, MAX_ORDER + 1), dtype=np.int64, endpoint=True)
    _probe_both(S, C, orders, wide)


@pytest.mark.gpu
@pytest.mark.parametrize("wide", [False, True])
def test_every_digit_count(wide):
    """Predictors whose largest coefficient needs 1..8 signed digits, the saturated +-2^63 ends included, on
    samples at the extremes of the row form."""
    rng = np.random.default_rng(23 + wide)
    rows_C, rows_o = [], []
    for L in range(1, 9):
        for order in (1, 24, 25, 57, 100):
            C = np.zeros(MAX_ORDER + 1, np.int64)
            C[1:order + 1] = rng.permutation(_with_digits(rng, L, order))
            rows_C.append(C)
            rows_o.append(order)
    for v in (-2 ** 63, 2 ** 63 - 1):
        for order in (1, 57, 100):
            C = np.full(MAX_ORDER + 1, v, np.int64)
            C[0] = 0
            rows_C.append(C)
            rows_o.append(order)
    n = len(rows_o)
    if wide:
        ext = np.array([-65535, 65535, -65534, 65534, -1, 1, 0], np.int32)
    else:
        ext = np.array([-32768, 32767, -32767, 32766, -1, 1, 0], np.int32)
    S = ext[rng.integers(0, ext.size, size=(n, FRAME))]
    S[: n // 2] = np.where(rng.random((n // 2, FRAME)) < 0.5, S[: n // 2], ext[0])   # long runs of the minimum
    _probe_both(S, np.stack(rows_C), rows_o, wide)


@pytest.mark.gpu
def test_alternating_parity():
    """17-bit rows whose parity alternates (and its complement), at the ends of the range and at random."""
    rng = np.random.default_rng(31)
    t = np.arange(FRAME)
    rows = [np.where(t % 2 == 0, 65535, -65535), np.where(t % 2 == 0, -65534, 65533),
            np.where(t % 2 == 0, 1, 0), (rng.integers(-32767, 32768, FRAME) * 2 + (t % 2))]
    S = np.stack([r.astype(np.int32) for r in rows] * 3)
    C = np.zeros((S.shape[0], MAX_ORDER + 1), np.int64)
    orders = np.array([1, 25, 57, 100] * 3)
    for i in range(S.shape[0]):
        C[i, 1:] = _with_digits(rng, 1 + i % 8, MAX_ORDER)
    _probe_both(S, C, orders, True)


# ------------------------------------------------------------------------------ the tie flag (CHECK) --

@functools.lru_cache(maxsize=None)
def _planted_rows(wide, offset, seed):
    """A signal per output position i = 1 .. 2047 with random full-range c and random samples, whose prediction at
    i is set to 2^34 + offset mod 2^35 by the placer (offset 0: a tie; +-1: a near miss).  Where the placer finds no
    solution the low taps are drawn again; at the first outputs, which see one or two samples, c[1] is solved for
    instead (its low 35 bits; the high ones stay random)."""
    from exact_lossless import M35, place_tie, prediction
    rng = np.random.default_rng(seed)
    lim = 65535 if wide else 32767
    lo = -lim - (not wide)
    S = rng.integers(lo, lim + 1, size=(FRAME - 1, FRAME)).astype(np.int64)
    C = rng.integers(-2 ** 63, 2 ** 63 - 1, size=(FRAME - 1, MAX_ORDER + 1), dtype=np.int64, endpoint=True)
    C[:, 0] = 0
    orders = rng.integers(8, MAX_ORDER + 1, FRAME - 1)
    C[np.arange(MAX_ORDER + 1)[None, :] > orders[:, None]] = 0   # the taps the placer sees are the FIR's
    for r, i in enumerate(range(1, FRAME)):
        if i <= 2:
            S[r, i - 1] |= 1
            rest = (prediction(S[r], C[r], i) - int(C[r, 1]) * int(S[r, i - 1])) % M35
            low = (HALF + offset - rest) * pow(int(S[r, i - 1]) % M35, -1, M35) % M35
            v = (int(C[r, 1]) >> Q << Q | low) % (1 << 64)
            C[r, 1] = v - (1 << 64) if v >= 1 << 63 else v
            assert prediction(S[r], C[r], i) == (HALF + offset) % M35
            continue
        for attempt in range(16):
            if attempt:
                C[r, 1:9] = rng.integers(-2 ** 63, 2 ** 63 - 1, 8, dtype=np.int64, endpoint=True)
            if place_tie(S[r], C[r], i, lo, lim, target=HALF + offset, rng=rng, near=False):
                break
        else:
            raise AssertionError("nothing placed at %d" % i)
    return S, C, orders


def _tie_model(S, C, orders):
    from exact_lossless import fir
    res, first = [], []
    for s, c, o in zip(S, C, orders):
        r, tie = fir(s, c, int(o))
        res.append(r)
        first.append(int(np.argmax(tie)) if tie.any() else -1)
    return np.stack(res), np.array(first)


def _tie_probe(S, C, orders, wide):
    from sela_b200 import codec
    res, ties = codec.fir_tie_probe(S, orders, C, wide)
    want_res, first = _tie_model(S, C, orders)
    assert np.array_equal(res, want_res)
    assert np.array_equal(res, fir_residues(S, C, orders))
    bad = np.nonzero(ties != (first >= 0))[0]
    assert bad.size == 0, "signals %s: device %s, model first tie %s" % (bad[:8], ties[bad[:8]], first[bad[:8]])
    return ties, first


def test_placer_on_full_range_predictors():
    """The planted rows (CPU): one tie, at the planted output, and none for a near miss."""
    for wide in (False, True):
        S, C, orders = _planted_rows(wide, 0, 40 + wide)
        _, first = _tie_model(S[::97], C[::97], orders[::97])
        assert np.array_equal(first, np.arange(1, FRAME)[::97])
        S, C, orders = _planted_rows(wide, 1, 44 + wide)
        _, first = _tie_model(S[::97], C[::97], orders[::97])
        assert (first == -1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("wide", [False, True])
def test_tie_at_every_output(wide):
    """One planted tie per signal at every output position 1 .. 2047: every slot of the mma epilogue."""
    S, C, orders = _planted_rows(wide, 0, 40 + wide)
    ties, first = _tie_probe(S, C, orders, wide)
    assert ties.all() and np.array_equal(first, np.arange(1, FRAME))


@pytest.mark.gpu
@pytest.mark.parametrize("wide", [False, True])
def test_near_misses_do_not_tie(wide):
    """P = 2^34 +- 1 mod 2^35 at every output position, and rows with no tie anywhere: the flag stays clear."""
    S1, C1, o1 = _planted_rows(wide, 1, 44 + wide)
    S2, C2, o2 = _planted_rows(wide, -1, 46 + wide)
    rng = np.random.default_rng(48 + wide)
    lim = 65535 if wide else 32767
    S3 = rng.integers(-lim, lim + 1, size=(64, FRAME))
    C3 = rng.integers(-2 ** 40, 2 ** 40, size=(64, MAX_ORDER + 1))
    o3 = np.arange(64) % 3   # orders 0 .. 2
    S = np.concatenate([S1, S2, S3])
    ties, first = _tie_probe(S, np.concatenate([C1, C2, C3]), np.concatenate([o1, o2, o3]), wide)
    assert not ties.any()


@pytest.mark.gpu
@pytest.mark.parametrize("wide", [False, True])
def test_wrap_territory(wide):
    """Saturated +-2^63 coefficients and sums at and near +-2^63, where the 64-bit wrap decides: the sum of the two
    roundings is then -2^29 or 1 - 2^29 instead of 0 or 1, and the device must follow the formula bit for bit."""
    rng = np.random.default_rng(50 + wide)
    lim = 65535 if wide else 32767
    rows_S, rows_C, rows_o = [], [], []
    for c1 in (-2 ** 63, 2 ** 63 - 1, 2 ** 62, -2 ** 62, 3 * 2 ** 61, -(2 ** 63) + 2 ** 34, 2 ** 63 - 2 ** 34):
        for order in (1, 2, 100):
            for odd_at in (None, 0, 1, 7, 1000, FRAME - 2):
                s = 2 * rng.integers(-(lim // 2), lim // 2 + 1, FRAME)
                if odd_at is not None:
                    s[odd_at] += 1
                c = np.zeros(MAX_ORDER + 1, np.int64)
                c[1:order + 1] = c1
                if order == 100:
                    c[2:101:2] = -c1 if c1 != -2 ** 63 else c1
                rows_S.append(s)
                rows_C.append(c)
                rows_o.append(order)
    S, C, o = np.stack(rows_S), np.stack(rows_C), np.array(rows_o)
    ties, first = _tie_probe(S, C, o, wide)
    assert ties.any() and not ties.all()


@pytest.mark.gpu
def test_natural_signals_against_the_port():
    """The port's (order, c) of each natural signal: the device's residues equal the port's, in every row form
    that holds the signal."""
    from sela_b200 import codec
    O = ol.load("port")
    x = _natural()
    C = np.zeros((x.shape[0], MAX_ORDER + 1), np.int64)
    orders = np.zeros(x.shape[0], np.int32)
    want = np.zeros_like(x)
    for i, s in enumerate(x):
        a = O.lpc_analyse(s)
        orders[i] = a["order"]
        C[i, :a["c"].size] = a["c"]
        want[i] = a["res"]
    assert np.array_equal(codec.fir_probe(x, orders, C, True), want)
    narrow = (x >= -32768).all(axis=1) & (x <= 32767).all(axis=1)
    assert narrow.any()
    assert np.array_equal(codec.fir_probe(x[narrow], orders[narrow], C[narrow], False), want[narrow])
