"""The lossless repair (lossless.cuh) on crafted units against the exact model of exact_lossless.py.

Ties cannot be reached through PCM alone: the analysis picks the predictor.  Here every unit is coded with a chosen
predictor (codec.encode_lossless_forced) and its samples carry ties planted by exact_lossless.place_tie in the base
predictor and in chosen repair candidates, at increasing positions.  Each scenario asserts on the model that it
reaches what it is named for (a round-2 winner, a cut, two candidates with the same words, a stereo decision that
flips, ...), so that a change in the generator cannot quietly void it; the CPU tests run exactly these assertions.
The GPU tests then compare the device with the model: the report, and every frame's subframes word for word --
re-coded frames against the model's repair, every other frame against the model's coding of its chosen
predictors -- and decode the batch under the port and, where built, the compiled reference."""
import functools

import numpy as np
import pytest

import oracle_lib as ol
from exact_lossless import (PLACER_TAPS, Unit, as_tuples, assert_in_domain, candidate, candidate_predictor,
                            check_against_model, expected_report, fir, model_batch, place_tie, place_tie_difference,
                            repair, repair_edit, round1)

FRAME = 2048
I16 = (-32768, 32767)


def _O():
    return ol.load("port")


def random_q(rng, order, small=6):
    """A stable predictor (every reflection coefficient inside (-1, 1)) with a strong first two coefficients."""
    q = np.zeros(100, np.int32)
    q[0] = rng.integers(20, 46)
    if order > 1:
        q[1] = rng.integers(-45, -19)
    if order > 2:
        q[2:order] = rng.integers(-small, small + 1, order - 2)
    return q


def ar_signal(rng, order, q, amp):
    """A signal the predictor (order, q) fits: the decoder's recurrence on small noise, clipped to int16."""
    r = rng.integers(-amp, amp + 1, FRAME).astype(np.int32)
    return np.clip(_O().lpc_synthesise(r, order, q[:order]).astype(np.int64), *I16)


class Planter:
    """Plants ties in a unit's signal at increasing positions, each at least PLACER_TAPS + 1 after the last."""

    def __init__(self, s, rng, lo=I16[0], hi=I16[1], pos=12, ch1=None):
        self.s, self.rng, self.lo, self.hi, self.pos, self.ch1 = s, rng, lo, hi, pos, ch1

    def tie(self, order, q):
        c = _O().lpc_coefficients(np.asarray(q, np.int32), order)
        while True:
            assert self.pos < FRAME, "no room left for another tie"
            if self.ch1 is not None:
                ok = place_tie_difference(self.s, self.ch1, c, self.pos, rng=self.rng)
            else:
                ok = place_tie(self.s, c, self.pos, self.lo, self.hi, rng=self.rng)
            self.pos += PLACER_TAPS + 1 if ok else 1
            if ok:
                return

    def signal(self):
        return self.s - self.ch1 if self.ch1 is not None else self.s


def steer(p, order, q, goal, tie_first=(), limit=60):
    """A tie in the base predictor (order, q), then in the candidates `tie_first`, then in the model's winner
    until goal(unit, winner) holds -> (unit, winner)."""
    O = _O()
    p.tie(order, q)
    u = Unit(O, p.signal(), order, q)
    for cand in tie_first:
        cp = candidate_predictor(u, cand)
        if cp is not None:
            p.tie(*cp)
    for _ in range(limit):
        u = Unit(O, p.signal(), order, q)
        assert u.tie
        w = repair(O, u)
        if goal(u, w):
            return u, w
        if w.order == 1 or p.pos > FRAME - 64:  # order 1 cannot be given a tie
            break
        p.tie(w.order, w.q)
    raise Unreachable()


class Unreachable(Exception):
    pass


def mono_unit(seed, order, goal, tie_first=(), q=None, amp=1500, small=6, tries=40):
    """A unit of the given order whose repair reaches `goal`, from the first of `tries` seeds that gets there (low
    orders with coefficients that end in many zero bits tie on their own, and a candidate that already ties
    cannot be made to win)."""
    for k in range(tries):
        rng = np.random.default_rng(seed + 1000 * k)
        qk = random_q(rng, order, small) if q is None else q
        s = ar_signal(rng, order, qk, amp)
        try:
            u, w = steer(Planter(s, rng), order, qk, goal, tie_first)
        except Unreachable:
            continue
        assert_in_domain(_O(), u, 32768)
        return u, w
    raise AssertionError("no seed reaches the goal")


def is_edit(o, cand):
    return repair_edit(o, cand)[2] != 0


# ------------------------------------------------------------ scenarios --
# Each returns (pcm int16 [n * 2048, channels], channels, predictors per unit, model units/winners for the claims).

def _mono_batch(units):
    pcm = np.stack([u.s for u in units])[:, :, None].reshape(-1, 1)
    return pcm.astype(np.int16), 1, [(u.order, u.q) for u in units]


@functools.lru_cache(maxsize=None)
def round1_kinds():
    """A round-1 winner of each kind: q[0] -+ 1, q[1] -+ 1, q[o-1] -+ 1 and order o-1, at orders 8 and 2."""
    out = []
    for target in range(7):
        out.append(mono_unit(100 + target, 8, lambda u, w, t=target: w.cand == t))
    for target in range(5):
        out.append(mono_unit(120 + target, 2, lambda u, w, t=target: w.cand == t))
    for (u, w), t in zip(out, list(range(7)) + list(range(5))):
        assert w.cand == t and w.words >= 0
    return out


@functools.lru_cache(maxsize=None)
def round2_cases():
    out = {}
    # every round-1 candidate ties: an edit of a middle coefficient wins
    out["edit"] = mono_unit(200, 8, lambda u, w: w.cand >= 7 and is_edit(8, w.cand), tie_first=range(7))
    # every edit ties: a cut to order o-2 .. 2 wins
    o = 7
    edits = [c for c in range(3 * o - 1) if is_edit(o, c) or c == 6]
    out["cut"] = mono_unit(201, o, lambda u, w: w.cand >= 7 and not is_edit(o, w.cand) and w.order >= 2,
                           tie_first=edits)
    # everything but order 1 ties: the last candidate, 3o-2, wins
    o = 4
    out["order1"] = mono_unit(202, o, lambda u, w: w.cand == 3 * o - 2, tie_first=range(3 * o - 2))
    # order 100: round 2 runs with its full stride of 292 candidates
    out["order100"] = mono_unit(203, 100, lambda u, w: w.cand >= 7, tie_first=range(7), small=3)
    # order 3 with every round-1 candidate tied: order 1 is the only round-2 candidate
    out["order3"] = mono_unit(204, 3, lambda u, w: w.cand == 7, tie_first=range(7))
    out["order3_round1"] = mono_unit(205, 3, lambda u, w: w.cand < 7)
    assert out["order100"][0].order == 100 and 3 * 100 - 1 - 7 == 292
    assert out["order3"][1].order == 1 and 3 * 3 - 1 == 8
    for k in ("edit", "cut", "order1", "order100", "order3"):
        u, w = out[k]
        assert all(candidate(_O(), u, c) is None or candidate(_O(), u, c).tie for c in range(round1(u.order))), k
    return out


@functools.lru_cache(maxsize=None)
def bounds_cases():
    """q[j] at -64 and 63 for j = 0, 1, o-1 and a round-2 j: the edit that leaves [-64, 63] is no candidate."""
    out = []
    o = 8
    for n, (j, v) in enumerate([(0, -64), (0, 63), (1, -64), (1, 63), (o - 1, -64), (o - 1, 63), (3, -64), (3, 63)]):
        rng = np.random.default_rng(300 + n)
        q = random_q(rng, o)
        q[j] = v
        tie_first = range(7) if j == 3 else ()
        goal = (lambda u, w: w.cand >= 7) if j == 3 else (lambda u, w: True)
        u, w = mono_unit(300 + n, o, goal, tie_first, q=q, amp=600)
        dropped = [c for c in range(3 * o - 1) if candidate_predictor(u, c) is None]
        assert dropped == [{0: 0, 1: 2, o - 1: 4, 3: 7 + 2 * (3 - 2)}[j] + (v == 63)], (j, v, dropped)
        out.append((u, w))
    return out


@functools.lru_cache(maxsize=None)
def equal_words_case():
    """Two tie-free candidates of the winning round with the same, fewest words: the earlier one wins."""
    O = _O()
    for seed in range(400, 520):
        rng = np.random.default_rng(seed)
        o = 8
        q = random_q(rng, o)
        p = Planter(ar_signal(rng, o, q, 1500), rng)
        p.tie(o, q)
        for _ in range(6):
            u = Unit(O, p.signal(), o, q)
            cands = [v for v in (candidate(O, u, c) for c in range(7)) if v is not None and not v.tie]
            if len(cands) < 2:
                break
            best = min(v.words for v in cands)
            equal = [v.cand for v in cands if v.words == best]
            if len(equal) > 1:
                w = repair(O, u)
                assert w.cand == equal[0] < equal[1]
                assert_in_domain(O, u, 32768)
                return u, w, equal
            p.tie(o, min(cands, key=lambda v: (v.words, v.cand)).q)
    raise AssertionError("no unit with two equal best candidates")


def mono_scenario(name):
    if name == "round1":
        units = [u for u, _ in round1_kinds()]
    elif name == "round2":
        units = [u for u, _ in round2_cases().values()]
    elif name == "bounds":
        units = [u for u, _ in bounds_cases()]
    elif name == "equal_words":
        units = [equal_words_case()[0]]
    else:
        raise ValueError(name)
    # a clean unit in front: a frame that is not re-coded and keeps the coding of its predictor
    rng = np.random.default_rng(7)
    q = random_q(rng, 5)
    clean = Unit(_O(), ar_signal(rng, 5, q, 300), 5, q)
    assert not clean.tie
    return _mono_batch([clean] + units)


@functools.lru_cache(maxsize=None)
def large_batch():
    """Every distinct unit above, tiled over 8 channels and enough frames that the units outnumber the warps of the
    repair grids (min(units, SMs * 32) <= 4224 on an H100): every grid-stride loop wraps."""
    units = ([u for u, _ in round1_kinds()] + [u for u, _ in round2_cases().values()] +
             [u for u, _ in bounds_cases()] + [equal_words_case()[0]])
    n_frames = 640
    idx = np.arange(n_frames * 8) % len(units)
    assert idx.size > 132 * 32 and any(repair(_O(), units[k]).cand >= 7 for k in set(idx))
    planes = np.stack([units[k].s for k in idx]).reshape(n_frames, 8, FRAME)
    pcm = planes.transpose(0, 2, 1).reshape(-1, 8).astype(np.int16)
    return pcm, 8, [(units[k].order, units[k].q) for k in idx], (units, idx)


def _stereo(ch0, ch1, preds):
    for ch in (ch0, ch1):
        assert ch.min() >= -32768 and ch.max() <= 32767
    return np.stack([ch0, ch1], axis=1).astype(np.int16), 2, preds


def _units(O, pcm, channels, preds):
    import analysis_corpus
    return [Unit(O, s, o, q) for s, (o, q) in zip(analysis_corpus.units(pcm, channels), preds)]


@functools.lru_cache(maxsize=None)
def stereo_case(kind):
    O = _O()
    rng = np.random.default_rng({"ch0": 600, "ch1_loses": 601, "diff_wins": 602, "diff_loses": 603}.get(kind, 604))
    o = 8
    q1, qd = random_q(rng, o), random_q(rng, o)
    if kind == "ch0":            # ch0 flagged; ch0 is always emitted
        ch1 = ar_signal(rng, o, q1, 1500)
        ch0 = np.clip(ch1 + ar_signal(rng, o, qd, 200), *I16)
        Planter(ch0, rng).tie(o, q1)
        preds = [(o, q1), (o, q1), (o, qd)]
    elif kind == "ch1_loses":    # ch1 flagged, the clean difference has fewer words: nothing is re-coded
        ch1 = ar_signal(rng, o, q1, 3000)
        ch0 = np.clip(ch1 + ar_signal(rng, o, qd, 100), *I16)
        Planter(ch1, rng).tie(o, q1)
        preds = [(o, q1), (o, q1), (o, qd)]
    elif kind in ("diff_wins", "diff_loses"):  # the 17-bit difference flagged (the WIDE tie test)
        big, small = (3000, 100) if kind == "diff_wins" else (100, 3000)
        ch1 = ar_signal(rng, o, q1, big)
        ch0 = np.clip(ch1 + ar_signal(rng, o, qd, small), *I16)
        Planter(ch0, rng, ch1=ch1).tie(o, qd)
        preds = [(o, q1), (o, q1), (o, qd)]
    elif kind == "flip":         # both side candidates flagged; the decision flips after the repair
        for seed in range(700, 760):
            rng = np.random.default_rng(seed)
            q1 = random_q(rng, o)
            ch1 = ar_signal(rng, o, q1, 1500)
            ch0 = np.clip(ch1 + ar_signal(rng, o, q1, 1400), *I16)
            Planter(ch1, rng, pos=12).tie(o, q1)
            pd = Planter(ch0, rng, ch1=ch1, pos=12)
            pd.tie(o, q1)
            preds = [(o, q1), (o, q1), (o, q1)]
            for _ in range(12):
                pcm, _, _ = _stereo(ch0, ch1, preds)
                u = _units(O, pcm, 2, preds)
                if not (u[1].tie and u[2].tie) or u[2].words >= u[1].words:
                    break
                w1, w2 = repair(O, u[1]), repair(O, u[2])
                if w2.words >= w1.words:
                    return _stereo(ch0, ch1, preds)
                pd.tie(w2.order, w2.q)  # the difference's best repair ties too: its next one costs more
        raise AssertionError("no flipping stereo frame")
    else:
        raise ValueError(kind)
    return _stereo(ch0, ch1, preds)


@functools.lru_cache(maxsize=None)
def multichannel_case(channels):
    """Two frames of `channels` channels: the first with several flagged channels, the second clean."""
    rng = np.random.default_rng(800 + channels)
    flagged = {3: (0, 2), 8: (1, 4, 5, 7)}[channels]
    planes, preds = [], []
    for f in range(2):
        for ch in range(channels):
            o = int(rng.integers(2, 12))
            q = random_q(rng, o)
            s = ar_signal(rng, o, q, 1500)
            if f == 0 and ch in flagged:
                Planter(s, rng, pos=int(rng.integers(1, 200))).tie(o, q)
            planes.append(s)
            preds.append((o, q))
    pcm = np.stack(planes).reshape(2, channels, FRAME).transpose(0, 2, 1).reshape(-1, channels)
    return pcm.astype(np.int16), channels, preds


def stereo_claims(kind):
    """What each stereo scenario is named for, on the model."""
    O = _O()
    pcm, ch, preds = stereo_case(kind)
    u = _units(O, pcm, ch, preds)
    m = model_batch(O, pcm, ch, preds, every=True)
    em, rep = m[0]
    if kind == "ch0":
        assert u[0].tie and not u[1].tie and not u[2].tie and [r[0] for r in rep] == [0]
    elif kind == "ch1_loses":
        assert u[1].tie and not u[2].tie and u[2].words < u[1].words and rep == []
    elif kind == "diff_wins":
        assert u[2].tie and not u[1].tie and u[2].words < u[1].words
        assert [r[0] for r in rep] == [1] and em[1][1] == 1
    elif kind == "diff_loses":
        assert u[2].tie and not u[1].tie and u[2].words >= u[1].words and rep == []
    elif kind == "flip":
        assert u[1].tie and u[2].tie and u[2].words < u[1].words       # the reference emits the difference
        assert em[1][1] == 0 and rep == [(1, u[2].order, u[2].words, em[1][0].order, em[1][0].words)]  # now ch1
    for k in range(3):
        assert_in_domain(O, u[k], 65535 if k == 2 else 32768)
    return m


# ------------------------------------------------------------------- CPU --

def test_round1_winners_of_every_kind():
    assert [w.cand for _, w in round1_kinds()] == list(range(7)) + list(range(5))
    assert [u.order for u, _ in round1_kinds()] == [8] * 7 + [2] * 5


def test_round2_and_small_orders():
    c = round2_cases()
    o = 8
    assert c["edit"][1].cand >= 7 and 2 <= repair_edit(o, c["edit"][1].cand)[1] <= o - 2
    u, w = c["cut"]
    assert w.cand >= 7 + 2 * (u.order - 3) and 2 <= w.order <= u.order - 2
    u, w = c["order1"]
    assert w.cand == 3 * u.order - 2 and w.order == 1
    assert c["order100"][0].order == 100 and c["order100"][1].cand >= 7
    assert c["order3"][1].cand == 7 and c["order3"][1].order == 1
    assert c["order3_round1"][1].cand < 7


def test_bounds_drop_edits():
    assert len(bounds_cases()) == 8


def test_equal_words_earlier_candidate_wins():
    u, w, equal = equal_words_case()
    assert w.cand == min(equal) and len(equal) >= 2


def test_large_batch_wraps_every_loop():
    pcm, ch, preds, (units, idx) = large_batch()
    assert len(preds) == pcm.shape[0] // FRAME * ch > 132 * 32
    assert all(u.tie for u in units)


@pytest.mark.parametrize("kind", ["ch0", "ch1_loses", "diff_wins", "diff_loses", "flip"])
def test_stereo_claims(kind):
    stereo_claims(kind)


@pytest.mark.parametrize("channels", [3, 8])
def test_multichannel_claims(channels):
    O = _O()
    pcm, ch, preds = multichannel_case(channels)
    m = model_batch(O, pcm, ch, preds, every=True)
    assert [r[0] for r in m[0][1]] == list({3: (0, 2), 8: (1, 4, 5, 7)}[channels]) and m[1][1] == []


@pytest.mark.parametrize("wide", [False, True])
def test_placer_and_criterion_against_the_decoders(wide):
    """Crafted units, 16- and 17-bit, ties planted at early positions and at order 100: the tie test fires iff the
    decode differs from the source, and the first tie is the first wrong sample, under the port and the compiled
    reference where built."""
    O = _O()
    decoders = [O] + ([ol.load("ref")] if ol.have_ref() else [])
    lim = 65535 if wide else 32767
    n = 0
    for seed, order, first in [(900, 1, None), (901, 2, 1), (902, 3, 2), (903, 8, 1), (904, 8, 3), (905, 30, 5),
                               (906, 100, 1), (907, 100, 9), (908, 100, None), (909, 12, 2040)]:
        rng = np.random.default_rng(seed + 50 * wide)
        q = random_q(rng, order, small=3)
        s = np.clip(ar_signal(rng, order, q, 300) * (2 if wide else 1), -lim, lim)
        c = O.lpc_coefficients(q, order)
        if first is not None:
            pos = first
            while not place_tie(s, c, pos, -lim, lim, rng=rng):
                pos += 1
            assert pos < first + 8
            if pos + 200 < FRAME:
                assert place_tie(s, c, pos + 100, -lim, lim, rng=rng)
        u = Unit(O, s, order, q)
        assert_in_domain(O, u, lim)
        res, tie = fir(s, u.c, order)
        assert tie.any() == (first is not None)
        if first is not None:
            assert np.argmax(tie) == pos
        for D in decoders:
            wrong = D.lpc_synthesise(res, order, q[:order]) != s
            assert wrong.any() == tie.any()
            if tie.any():
                assert np.argmax(wrong) == np.argmax(tie)
                n += 1
    assert n == 8 * len(decoders)


def test_placer_near_miss_leaves_no_tie():
    O = _O()
    rng = np.random.default_rng(950)
    q = random_q(rng, 10)
    c = O.lpc_coefficients(q, 10)
    s = ar_signal(rng, 10, q, 200)
    for i, d in zip(range(20, 2000, 40), [1, -1] * 100):
        assert place_tie(s, c, i, target=(1 << 34) + d, rng=rng)
    res, tie = fir(s, c, 10)
    assert not tie.any()
    assert np.array_equal(O.lpc_synthesise(res, 10, q[:10]), s)


# ------------------------------------------------------------------- GPU --

def _run(pcm, channels, preds, model=None):
    from sela_b200 import codec
    O = _O()
    descs, words, rep = codec.encode_lossless_forced(pcm, channels, preds)
    if model is None:
        model = model_batch(O, pcm, channels, preds, every=True)
    assert as_tuples(rep) == expected_report(model)
    check_against_model(O, descs, words, pcm, channels, model)
    return model


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["round1", "round2", "bounds", "equal_words"])
def test_mono_scenarios(name):
    pcm, ch, preds = mono_scenario(name)
    m = _run(pcm, ch, preds)
    assert m[0][1] == [] and all(m[f][1] for f in range(1, len(m)))


@pytest.mark.gpu
def test_large_batch():
    O = _O()
    pcm, ch, preds, (units, idx) = large_batch()
    per_unit = []
    for u in units:   # the model of each distinct unit once; every frame is eight independent units
        w = repair(O, u)
        per_unit.append(((w, 0), (u.order, u.words, w.order, w.words)))
    model = {}
    for f in range(idx.size // 8):
        ks = idx[f * 8:(f + 1) * 8]
        model[f] = ([per_unit[k][0] for k in ks], [(c,) + per_unit[k][1] for c, k in enumerate(ks)])
    _run(pcm, ch, preds, model)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ch0", "ch1_loses", "diff_wins", "diff_loses", "flip"])
def test_stereo(kind):
    m = stereo_claims(kind)
    _run(*stereo_case(kind), model=m)


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [3, 8])
def test_multichannel(channels):
    _run(*multichannel_case(channels))


@pytest.mark.gpu
def test_forced_predictor_domain():
    """An order outside 0..100, a q outside [-64, 63] and a non-zero q past the order are refused."""
    from sela_b200 import SelaB200Error, _lib, codec
    pcm = np.zeros((FRAME, 1), np.int16)
    for order, j, v in [(101, 0, 0), (-1, 0, 0), (2, 0, 64), (2, 1, -65), (2, 2, 1), (100, 99, -65)]:
        pred = np.zeros(1, _lib.PREDICTOR_DTYPE)
        pred["order"] = order
        pred["q"][0, j] = v
        with pytest.raises(SelaB200Error) as e:
            codec.encode_lossless_forced(pcm, 1, pred)
        assert e.value.status == -5
    pred = np.zeros(1, _lib.PREDICTOR_DTYPE)
    pred["order"], pred["q"][0, :2] = 2, (-64, 63)
    codec.encode_lossless_forced(pcm, 1, pred)
