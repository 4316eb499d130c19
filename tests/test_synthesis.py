"""GPU synthesis (the LPC IIR of decode) on crafted streams: sela_b200.decode_frames and sela_b200.lpc_samples
against the reference decoder and the exact integer model of tests/exact_decode.py.

The encoder only produces 16/17-bit signals and the orders its analysis picks; the decoder must reproduce
the reference for every stream the descriptors admit.  These batches reach what encoder output does not:
orders 0-3 and around 28, 56 and 100 (segments of 1, 4, 7, 8 and 13 lanes), subframes of several segment widths
side by side, ragged width counts and a width change across the 1024-subframe tile of the packing plan, samples
beyond 16 bits, below -2^17 and at the int32 limits, permuted channel fields, difference subframes at every
position and channel count 1-16, with parent and difference both near INT32_MIN (k_diff_fixup)."""
import numpy as np
import pytest

import crafted as CR
import exact_decode as X
import oracle_lib as ol
import sela_b200

pytestmark = pytest.mark.gpu
FRAME = 2048
ORDERS = [0, 1, 2, 3, 27, 28, 29, 30, 31, 55, 56, 57, 60, 61, 99, 100]
KINDS = ["small", "wide", "neg17", "edge"]
TAPS = 8                                                            # kTapsPerLane (lpc.cuh)


def width(order):
    """Lanes of the synthesis segment of a subframe of this order (segment_width, lpc.cuh)."""
    return max(1, -(-order // TAPS))


# every width 1..13: orders 0, 1, both ends of each width and the largest order
EDGES = sorted({0, 1, 100} | {o for w in range(1, 13) for o in (TAPS * w, TAPS * w + 1)})


@pytest.fixture(scope="module")
def O():
    return ol.best()


@pytest.fixture(scope="module")
def P():
    return ol.load("port")


def check_decode(O, P, subs, channels):
    """decode_frames on the crafted batch == reference decoder == exact model.  Returns (descs, words, pcm)."""
    want, _, dom = X.decode(subs, channels, P)
    assert dom.all()                                               # every case is inside the reference's domain
    descs, words = CR.build(P, subs)
    assert np.array_equal(O.decode_frames(descs, words, channels), want)
    got = sela_b200.decode_frames(descs, words, channels)
    if not np.array_equal(got, want):
        bad = (got != want).reshape(-1, FRAME, channels).any(axis=1)     # [frame, channel field]
        wrong = [i for i, s in enumerate(subs) if bad[i // channels, s.channel]]
        pytest.fail("%d of %d subframes differ, first: %s" % (
            len(wrong), len(subs), [(i, subs[i].order, subs[i].type) for i in wrong[:8]]))
    return descs, words, want


def content(P, rng, order, i, **kw):
    return CR.crafted_subframe(P, rng, order, "wide" if i % 2 else "small", **kw)


# ------------------------------------------------------------------------------------- orders --

def test_order_classes_alone_and_mixed(O, P):
    """Every order of ORDERS four times, then groups of four orders of two segment widths each: the plan packs
    segments of different widths into one warp, each stepping its own order up."""
    rng = np.random.default_rng(100)
    orders = [o for o in ORDERS for _ in range(4)]
    mixed = [[0, 1, 2, 28], [27, 3, 28, 0], [29, 30, 55, 56], [56, 31, 29, 55], [57, 60, 99, 100], [100, 61, 57, 99]]
    for g in mixed:
        assert len({width(o) for o in g}) == 2, g
        orders += g
    subs = [content(P, rng, o, i) for i, o in enumerate(orders)]
    check_decode(O, P, subs, 1)


# ------------------------------------------------------------------------------- packing plan --

def _mono(P, rng, orders):
    return [CR.crafted_subframe(P, rng, int(o), "small") for o in orders]


def test_class_layout_ragged_segments_across_classify_tiles(O, P):
    """>= 1100 subframes drawn from three order ranges: the packing plan runs two CTAs, width counts are ragged,
    and the segment width changes across subframe 1024 (the first subframe of the plan's second CTA)."""
    rng = np.random.default_rng(101)
    counts = {0: 401, 1: 350, 2: 351}
    pool = {0: [0, 1, 2, 3, 17, 27, 28], 1: [29, 30, 31, 40, 55, 56], 2: [57, 60, 61, 80, 99, 100]}
    cls = np.concatenate([np.full(n, c) for c, n in counts.items()])
    rng.shuffle(cls)
    j = int(np.flatnonzero(cls != cls[1023])[0])
    cls[[1024, j]] = cls[[j, 1024]]                                # subframes 1023 and 1024 from different ranges
    orders = [int(rng.choice(pool[int(c)])) for c in cls]
    assert width(orders[1023]) != width(orders[1024])
    check_decode(O, P, _mono(P, rng, orders), 1)


@pytest.mark.parametrize("orders", [
    [0, 5, 28, 17, 1, 2, 3, 28, 11],                               # all orders <= 28
    [1, 70, 100, 2, 28, 57, 99, 0, 61],                            # none in 29..56
    [100], [29, 3], [57, 0, 56], [28, 29, 56, 57, 100],            # 1, 2, 3 and 5 subframes
], ids=["class0_only", "no_class1", "n1", "n2", "n3", "n5"])
def test_class_layout_small_batches(O, P, orders):
    check_decode(O, P, _mono(P, np.random.default_rng(len(orders) + sum(orders)), orders), 1)


# -------------------------------------------------------------------------------- sample range --

def _range_batch(P, kind, seed, orders=ORDERS):
    rng = np.random.default_rng(seed)
    return [CR.crafted_subframe(P, rng, o, kind) for o in orders]


@pytest.mark.parametrize("kind", KINDS)
def test_sample_range_decode(O, P, kind):
    """|s| <= 65535; beyond 16 bits (the int16 output wraps); below -2^17; within 2^8 of the int32 limits."""
    subs = _range_batch(P, kind, 200 + KINDS.index(kind))
    assert CR.sample_ranges(np.stack([s.samples for s in subs]))[kind]
    check_decode(O, P, subs, 1)


@pytest.mark.parametrize("kind", KINDS)
def test_sample_range_lpc_samples(O, P, kind):
    """The same subframes, then every segment width (EDGES), through the stage-level entry point (k_lpc_samples:
    the decoder's segment recurrence, one subframe per warp)."""
    subs = _range_batch(P, kind, 200 + KINDS.index(kind), ORDERS + EDGES)
    res = np.stack([s.res for s in subs])
    orders = np.array([s.order for s in subs], np.uint8)
    q = np.zeros((len(subs), 100), np.int32)
    for i, s in enumerate(subs):
        q[i, :s.order] = s.q
    want, dom = X.synthesise(res, orders, q, P)
    assert dom.all() and np.array_equal(want, np.stack([s.samples for s in subs]))
    for i, s in enumerate(subs):
        assert np.array_equal(O.lpc_synthesise(s.res, s.order, s.q), want[i]), i
    got = sela_b200.lpc_samples(res, orders, q)
    wrong = [(i, int(orders[i])) for i in range(len(subs)) if not np.array_equal(got[i], want[i])]
    assert not wrong, wrong


# ------------------------------------------------------------------------------------- stereo --

def _stereo(P, rng):
    """Difference subframe at position 0 and at position 1, with the channel fields in and out of position
    order; parent and difference always of different segment widths."""
    subs = []
    layouts = [  # (position 0, position 1): (channel, type) -- parent channel is the other one
        ((0, 0), (1, 1)), ((0, 1), (1, 0)), ((1, 0), (0, 1)), ((1, 1), (0, 0)), ((1, 0), (0, 0)), ((0, 0), (1, 0))]
    pairs = [(2, 57), (100, 28), (29, 0), (56, 99), (1, 61), (30, 3)]
    for f, (lay, (op, od)) in enumerate(zip(layouts, pairs)):
        assert width(op) != width(od)
        (c0, t0), (c1, t1) = lay
        par = content(P, rng, op, f, channel=c0 if t0 == 0 else c1)
        if t0 or t1:
            child = CR.difference_subframe(P, rng, od, par, channel=c0 if t0 else c1)
        else:
            child = content(P, rng, od, f + 1, channel=c1)
        subs += [child, par] if t0 else [par, child]
    return subs


def test_stereo_difference_positions_and_classes(O, P):
    check_decode(O, P, _stereo(P, np.random.default_rng(300)), 2)


# ------------------------------------------------------------------------------- channel count --

def _frames(P, rng, ch, n_frames=2):
    """Frame 0: independent subframes, channel fields a random permutation of the positions.  Further frames
    (ch >= 2): difference subframes.  From 3 channels: two of them share one parent, which sits at a higher
    channel index than its children; positions permuted as well.  From 2 channels a last frame: _edge_frame."""
    subs = []
    for f in range(n_frames):
        chans = rng.permutation(ch)
        orders = rng.choice(ORDERS, ch)
        frame = [None] * ch
        if f == 0 or ch == 1:
            for pos in range(ch):
                frame[pos] = content(P, rng, int(orders[pos]), pos + f, channel=int(chans[pos]))
        else:
            parent_ch = ch - 1
            kids = [0, 1] if ch >= 3 else [0]
            pos_of = {int(c): p for p, c in enumerate(chans)}
            par = content(P, rng, int(orders[pos_of[parent_ch]]), f, channel=parent_ch)
            frame[pos_of[parent_ch]] = par
            for c in range(ch - 1):
                o = int(orders[pos_of[c]])
                frame[pos_of[c]] = (CR.difference_subframe(P, rng, o, par, channel=c) if c in kids
                                    else content(P, rng, o, c, channel=c))
        subs += frame
    if ch >= 2:
        subs += _edge_frame(P, rng, ch)
    return subs


def _edge_frame(P, rng, ch):
    """Channel 0 is the difference to channel ch - 1, and both are within 2^8 of INT32_MIN at the same sample
    positions: parent - difference is small there, though in int32 arithmetic the int16 output of the parent
    minus the difference would overflow.  Other channels independent, positions permuted."""
    par = CR.crafted_subframe(P, rng, int(rng.choice(ORDERS[2:])), "edge", channel=ch - 1)
    kid = CR.difference_subframe(P, rng, int(rng.choice(ORDERS)), par, channel=0, kind="edge")
    assert ((par.samples <= CR.I32_MIN + 255) & (kid.samples <= CR.I32_MIN + 255)).any()
    by_channel = {0: kid, ch - 1: par}
    for c in range(1, ch - 1):
        by_channel[c] = content(P, rng, int(rng.choice(ORDERS)), c, channel=c)
    return [by_channel[int(c)] for c in rng.permutation(ch)]


@pytest.mark.parametrize("ch", range(1, 17))
def test_every_channel_count(O, P, ch):
    subs = _frames(P, np.random.default_rng(400 + ch), ch)
    check_decode(O, P, subs, ch)


# ------------------------------------------------------------------------------ chunked decode --

@pytest.mark.parametrize("ch", [2, 5])
def test_chunked_decode(O, P, monkeypatch, ch):
    """The pipelined host call cuts the batch into chunks of SELAB200_CHUNK_FRAMES frames: the packing plan and
    the difference fix-up per chunk must give the same output."""
    rng = np.random.default_rng(500 + ch)
    subs = _stereo(P, rng) if ch == 2 else _frames(P, rng, ch, n_frames=5)
    descs, words, want = check_decode(O, P, subs, ch)
    for cf in ("1", "3"):
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", cf)
        assert np.array_equal(sela_b200.decode_frames(descs, words, ch), want), cf
