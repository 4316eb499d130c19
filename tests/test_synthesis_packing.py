"""The segment packing of the batch synthesis kernel (k_decode_plan + k_synthesise_segments) on crafted streams,
against the reference decoder and the exact integer model of tests/exact_decode.py.

A subframe of order o runs on max(1, ceil(o / 8)) lanes of a warp; warps are filled from warp templates made from
the width counts, widest first, subframes of one width in file order.  These batches reach: every segment width
1..13 (orders 0 and 1 included) on both sides of each width edge, warps packed to exactly 32 lanes next to a partly
empty last warp, difference subframes at every segment position of a warp, and samples at the int32 limits."""
import numpy as np
import pytest

import crafted as CR
from test_synthesis import EDGES, check_decode, width

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def O():
    import oracle_lib as ol
    return ol.best()


@pytest.fixture(scope="module")
def P():
    import oracle_lib as ol
    return ol.load("port")


def test_every_segment_width():
    assert sorted({width(o) for o in EDGES}) == list(range(1, 14))


@pytest.mark.parametrize("kind", ["small", "wide", "edge"])
def test_every_width(O, P, kind):
    rng = np.random.default_rng(600 + len(kind))
    subs = [CR.crafted_subframe(P, rng, o, kind) for o in EDGES]
    check_decode(O, P, subs, 1)


def test_full_warps_and_a_partial_last_warp(O, P):
    """Eight width-8 subframes fill two warps of 4 x 8 = 32 lanes; two order-100 subframes (13 lanes each) and
    one of width 6 fill a third; one width-4 subframe is alone in the last warp, 28 lanes empty."""
    rng = np.random.default_rng(610)
    orders = [57, 64, 60, 63, 58, 61, 62, 59] + [100, 41, 100] + [32]
    assert sum(width(o) for o in orders[:8]) == 64 and sum(width(o) for o in orders[8:11]) == 32
    subs = [CR.crafted_subframe(P, rng, o, "wide" if i % 3 == 0 else "small") for i, o in enumerate(orders)]
    check_decode(O, P, subs, 1)


def test_difference_at_every_segment_position(O, P):
    """Stereo frames whose subframes all have width 4: a warp holds eight of them in file order, so frames 0-3
    (difference first) and 4-7 (difference second) put a difference subframe on every segment of a warp; frames
    8-13 mix widths, so parents and differences land in different warps."""
    rng = np.random.default_rng(620)
    subs = []
    for f in range(14):
        if f < 8:
            op, od = 25 + f, 32 - f
        else:
            op, od = [(100, 3), (1, 97), (0, 64), (48, 9), (17, 88), (72, 72)][f - 8]
        par_ch, diff_ch = (1, 0) if f % 3 else (0, 1)
        par = CR.crafted_subframe(P, rng, op, "small", channel=par_ch)
        child = CR.difference_subframe(P, rng, od, par, channel=diff_ch)
        subs += [child, par] if (f < 4 or (f >= 8 and f % 2)) else [par, child]
    check_decode(O, P, subs, 2)


def test_int32_extremes_across_widths(O, P):
    """Samples within 2^8 of the int32 limits on segments of every width, several warps."""
    rng = np.random.default_rng(630)
    subs = [CR.crafted_subframe(P, rng, o, "edge") for o in EDGES + EDGES[::-1]]
    assert CR.sample_ranges(np.stack([s.samples for s in subs]))["edge"]
    check_decode(O, P, subs, 1)
