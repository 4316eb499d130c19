"""The exact decoder model (tests/exact_decode.py) and the crafted streams (tests/crafted.py) against the CPU
oracle and the compiled reference (marker `ref`).  CPU only: this pins the yardstick the GPU synthesis
tests (tests/test_synthesis.py) measure the kernels with."""
import numpy as np
import pytest

import crafted as CR
import exact_decode as X
import exact_rice as XR
import oracle_lib as ol

FRAME = 2048
WHICH = ["port", pytest.param("ref", marks=pytest.mark.ref)]
ORDERS = [0, 1, 2, 3, 27, 28, 29, 56, 57, 100]


@pytest.fixture(scope="module")
def P():
    return ol.load("port")


@pytest.fixture(scope="module")
def range_set(P):
    """Subframes in all four sample ranges at orders on both sides of every class edge, plus the table ends:
    q = -64 (k = -1 exactly, and the SECOND0 entry of the second-order table) and q = 63."""
    rng = np.random.default_rng(2026)
    subs = [CR.crafted_subframe(P, rng, o, kind) for kind in ("small", "wide", "neg17", "edge") for o in ORDERS]
    for q01 in ([-64, 0], [0, -64], [-64, -64], [63, 63], [63, -64], [-64, 63]):
        for order, kind in ((2, "small"), (3, "neg17"), (2, "wide")):
            q = np.array(q01 + [0] * (order - 2), np.int32)
            s = CR.signal(rng, 20000 if kind == "small" else 1 << 19)
            if kind == "neg17":
                s[rng.integers(0, FRAME, 32)] = -(1 << 18)
            r = CR.residues_for(P, s, order, q)
            if r is not None:
                subs.append(CR.Sub(0, 0, 0, order, q, r))
    return subs


def test_crafted_set_covers_every_sample_range(P, range_set):
    s, ok = X.synthesise(np.stack([c.res for c in range_set]), [c.order for c in range_set],
                         [c.q for c in range_set], P)
    assert ok.all()
    reached = CR.sample_ranges(s)
    assert reached == {"small": True, "wide": True, "neg17": True, "edge": True}, reached
    # every range also occurs in front of non-zero taps, which is where the arithmetic is stressed
    C = X.coefficients([c.order for c in range_set], [c.q for c in range_set], P)
    taps = np.abs(C).sum(axis=1) > 0
    assert CR.sample_ranges(s[taps]) == reached
    # and the extremes of q occur where the guard admits them
    q01 = {tuple(c.q[:2]) for c in range_set if c.order >= 2}
    assert {(-64, 0), (0, -64), (-64, -64), (63, 63)} <= q01, q01


@pytest.mark.parametrize("which", WHICH)
def test_model_equals_sample_generator(P, range_set, which):
    """Exact model == oracle port == compiled reference, per subframe (SampleGenerator::process)."""
    O = ol.load(which)
    s, ok = X.synthesise(np.stack([c.res for c in range_set]), [c.order for c in range_set],
                         [c.q for c in range_set], P)
    assert ok.all()
    for i, c in enumerate(range_set):
        assert np.array_equal(O.lpc_synthesise(c.res, c.order, c.q[:c.order]), s[i]), (i, c.order, list(c.q[:2]))


def _frames(P, rng):
    """Three-channel frames with permuted channel fields and a difference subframe whose parent sits at a higher
    position, and stereo frames with the difference first; samples in every range."""
    kinds = ("small", "wide", "neg17", "edge")
    subs = []
    for f, kind in enumerate(kinds):
        orders = [[2, 57, 29], [100, 0, 28], [3, 56, 1], [27, 2, 100]][f]
        a = CR.crafted_subframe(P, rng, orders[0], kind, channel=2)
        b = CR.difference_subframe(P, rng, orders[1], a, channel=0)
        c = CR.crafted_subframe(P, rng, orders[2], kind, channel=1)
        subs += [b, c, a]
    stereo = []
    for f, kind in enumerate(kinds):
        p = CR.crafted_subframe(P, rng, [29, 2, 100, 56][f], kind, channel=f % 2)
        d = CR.difference_subframe(P, rng, [28, 57, 1, 100][f], p, channel=1 - f % 2)
        stereo += [d, p]
    return subs, stereo


@pytest.mark.parametrize("which", WHICH)
def test_model_equals_frame_decoder(P, which):
    """decode_frames on crafted streams: the Rice coding, the channel-field indexing and parent - difference of
    the model against FrameDecoder::process."""
    O = ol.load(which)
    rng = np.random.default_rng(7)
    three, stereo = _frames(P, rng)
    for subs, ch in ((three, 3), (stereo, 2)):
        pcm, planes, dom = X.decode(subs, ch, P)
        assert dom.all()
        descs, words = CR.build(P, subs)
        assert np.array_equal(O.decode_frames(descs, words, ch, threads=1), pcm), ch
    assert CR.sample_ranges(X.decode(three, 3, P)[1]) == {"small": True, "wide": True, "neg17": True, "edge": True}


def test_rice_code_matches_reference_encoder_and_decodes_every_int32(P):
    rng = np.random.default_rng(3)
    x = rng.integers(-(1 << 20), 1 << 20, FRAME)
    k, w = CR.rice_code(P, x)
    assert np.array_equal(XR.pack_stream(XR.zigzag(x), k), w)          # both paths lay out the same bits
    x[[0, 5, 700, 2047]] = [X.I32_MIN, X.I32_MAX, X.I32_MIN + 1, -(1 << 30)]
    k, w = CR.rice_code(P, x)
    assert np.array_equal(P.rice_decode(w, k, FRAME), x)


def test_domain_guard():
    P = ol.load("port")
    # outside the tables
    assert list(X.coefficients_in_domain([(2, [64, 0]), (3, [0, 0, -65]), (1, [500]), (2, [-64, -64])])) == \
        [False, False, True, True]
    # k = -1 at every order: the step-up coefficients grow like binomials and leave 2^62 / 2^35
    assert not X.coefficients_in_domain([(40, [-64] * 40)])[0]
    # the order-2 predictor q = [20, -10] on a residue of -140000: in the domain, and the sample is < -2^17
    r = np.zeros(FRAME, np.int32)
    r[3] = -140000
    s, ok = X.synthesise(r[None], [2], [np.array([20, -10], np.int32)], P)
    assert ok[0] and s[0].min() < -(1 << 17)
    assert np.array_equal(s[0], P.lpc_synthesise(r, 2, np.array([20, -10], np.int32)))
    # int32-limit samples behind a full-size coefficient: the int64 products overflow
    r[3] = X.I32_MIN
    assert not X.synthesise(r[None], [2], [np.array([20, -10], np.int32)], P)[1][0]
    # a residue that pushes the sample past int32
    r[3] = X.I32_MAX
    r[4] = X.I32_MAX
    assert X.synthesise(r[None], [0], [np.zeros(0, np.int32)], P)[1][0]      # no predictor: s = r
    assert not X.synthesise(r[None], [2], [np.array([26, 27], np.int32)], P)[1][0]
