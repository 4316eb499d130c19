"""GPU synthesis (the LPC IIR of decode) on crafted streams: sela_b200.decode_frames and sela_b200.lpc_samples
against the reference decoder and the exact integer model of tests/exact_decode.py.

The encoder only produces 16/17-bit signals and the orders its analysis picks; the decoder must reproduce
the reference for every stream the descriptors admit.  These batches reach what encoder output does not:
orders on both sides of every predictor-order class edge, four subframes of different orders in one warp,
class segments with ragged ends and a class change across the 1024-subframe classify tile, samples beyond
16 bits, below -2^17 and at the int32 limits, permuted channel fields, difference subframes at every
position and channel count 1-16 (the general kernel k_synthesise)."""
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


@pytest.fixture(scope="module")
def O():
    return ol.best()


@pytest.fixture(scope="module")
def P():
    return ol.load("port")


def order_class(order):
    return 0 if order <= 28 else 1 if order <= 56 else 2          # kernels.cuh order_class()


def warps(orders):
    """Subframe ids per warp of k_synthesise_quad, as k_decode_classify lays them out for a mono batch: a stable
    counting sort by order class, widest class first, every class segment padded to a multiple of four
    (None = an empty slot)."""
    slots = []
    for c in (2, 1, 0):
        ids = [i for i, o in enumerate(orders) if order_class(o) == c]
        slots += ids + [None] * (-len(ids) % 4)
    return [slots[i:i + 4] for i in range(0, len(slots), 4)]


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


# ------------------------------------------------------------------------------- order classes --

def test_order_classes_alone_and_mixed(O, P):
    rng = np.random.default_rng(100)
    orders = [o for o in ORDERS for _ in range(4)]                 # every order alone in a warp
    mixed = [[0, 1, 2, 28], [27, 3, 28, 0], [29, 30, 55, 56], [56, 31, 29, 55], [57, 60, 99, 100], [100, 61, 57, 99]]
    for g in mixed:
        orders += g
    # Each class count is a multiple of four here and k_decode_classify keeps file order inside a class, so
    # every listed group of four lands in one warp of the batch kernel:
    groups = [tuple(w) for w in warps(orders)]
    base = 4 * len(ORDERS)
    for j, g in enumerate(mixed):
        assert tuple(range(base + 4 * j, base + 4 * j + 4)) in groups, g
    subs = [content(P, rng, o, i) for i, o in enumerate(orders)]
    check_decode(O, P, subs, 1)


# -------------------------------------------------------------------------------- class layout --

def _mono(P, rng, orders):
    return [CR.crafted_subframe(P, rng, int(o), "small") for o in orders]


def test_class_layout_ragged_segments_across_classify_tiles(O, P):
    """>= 1100 subframes: classify runs two CTAs; every class count is 1, 2 or 3 mod 4, and class membership
    changes across subframe 1024 (the first subframe of the second classify tile)."""
    rng = np.random.default_rng(101)
    counts = {0: 401, 1: 350, 2: 351}                              # = 1, 2, 3 (mod 4)
    pool = {0: [0, 1, 2, 3, 17, 27, 28], 1: [29, 30, 31, 40, 55, 56], 2: [57, 60, 61, 80, 99, 100]}
    cls = np.concatenate([np.full(n, c) for c, n in counts.items()])
    rng.shuffle(cls)
    j = int(np.flatnonzero(cls != cls[1023])[0])
    cls[[1024, j]] = cls[[j, 1024]]                                # subframes 1023 and 1024 in different classes
    orders = [int(rng.choice(pool[int(c)])) for c in cls]
    assert order_class(orders[1023]) != order_class(orders[1024])
    assert sorted(np.bincount([order_class(o) for o in orders]) % 4) == [1, 2, 3]
    check_decode(O, P, _mono(P, rng, orders), 1)


@pytest.mark.parametrize("orders", [
    [0, 5, 28, 17, 1, 2, 3, 28, 11],                               # all class 0
    [1, 70, 100, 2, 28, 57, 99, 0, 61],                            # class 1 empty
    [100], [29, 3], [57, 0, 56], [28, 29, 56, 57, 100],            # 1, 2, 3 and 5 subframes
], ids=["class0_only", "no_class1", "n1", "n2", "n3", "n5"])
def test_class_layout_small_batches(O, P, orders):
    check_decode(O, P, _mono(P, np.random.default_rng(len(orders) + sum(orders)), orders), 1)


# -------------------------------------------------------------------------------- sample range --

def _range_batch(P, kind, seed):
    rng = np.random.default_rng(seed)
    return [CR.crafted_subframe(P, rng, o, kind) for o in ORDERS]


@pytest.mark.parametrize("kind", KINDS)
def test_sample_range_decode(O, P, kind):
    """|s| <= 65535; beyond 16 bits (the int16 output wraps); below -2^17; within 2^8 of the int32 limits."""
    subs = _range_batch(P, kind, 200 + KINDS.index(kind))
    assert CR.sample_ranges(np.stack([s.samples for s in subs]))[kind]
    check_decode(O, P, subs, 1)


@pytest.mark.parametrize("kind", KINDS)
def test_sample_range_lpc_samples(O, P, kind):
    """The same subframes through the stage-level entry point (k_lpc_samples: warp_iir_pair, classes 30 / 60)."""
    subs = _range_batch(P, kind, 200 + KINDS.index(kind))
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
    order; parent and difference always in different order classes."""
    subs = []
    layouts = [  # (position 0, position 1): (channel, type) -- parent channel is the other one
        ((0, 0), (1, 1)), ((0, 1), (1, 0)), ((1, 0), (0, 1)), ((1, 1), (0, 0)), ((1, 0), (0, 0)), ((0, 0), (1, 0))]
    pairs = [(2, 57), (100, 28), (29, 0), (56, 99), (1, 61), (30, 3)]
    for f, (lay, (op, od)) in enumerate(zip(layouts, pairs)):
        assert order_class(op) != order_class(od)
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
    channel index than its children; positions permuted as well."""
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
    return subs


@pytest.mark.parametrize("ch", range(1, 17))
def test_every_channel_count(O, P, ch):
    subs = _frames(P, np.random.default_rng(400 + ch), ch)
    check_decode(O, P, subs, ch)


# ------------------------------------------------------------------------------ chunked decode --

@pytest.mark.parametrize("ch", [2, 5])
def test_chunked_decode(O, P, monkeypatch, ch):
    """The pipelined host call cuts the batch into chunks of SELAB200_CHUNK_FRAMES frames: order classes and the
    general kernel per chunk must give the same output."""
    rng = np.random.default_rng(500 + ch)
    subs = _stereo(P, rng) if ch == 2 else _frames(P, rng, ch, n_frames=5)
    descs, words, want = check_decode(O, P, subs, ch)
    for cf in ("1", "3"):
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", cf)
        assert np.array_equal(sela_b200.decode_frames(descs, words, ch), want), cf
