"""The Rice residue decoder on arbitrary bit content against the exact parse model (tests/exact_rice.py): the split
index, the virtual-stream decoder and the first-generation parser (sela_b200/csrc/rice_vs.cuh, rice.cuh) through
every entry point that reaches them, at every k, every split S and every 16-byte phase of the arena.

Positions are checked by the kernels themselves (each part must end where the next begins); these tests check the
values, which that argument does not cover, and the acceptance boundary: a stream that ends on its last bit is
accepted, trailing words are accepted, one word short is SELAB200_ERR_BITSTREAM."""
import numpy as np
import pytest
import torch

import crafted as CR
import exact_decode as X
import exact_rice as XR
import oracle_lib as ol
import rice_families as RF
import sela_b200
from gpu_calls import decode_frames_device
from sela_b200 import _lib, wavio
from sela_b200.device import rice_decode_frames

pytestmark = pytest.mark.gpu
FRAME = 2048
SPLITS = ["0", "1", "2", "4", "8", "16", None]          # None: the default policy
GOOD = ("random", "trailing", "runs", "wrap", "long", "periodic")

# Streams the general parser decoded again, out of each family's batch, per split S (measured on an H100 80GB HBM3).
# The flags depend on the bits alone, not on timing, so the measured counts are the bounds: a kernel change that
# hands more streams to the fall-back fails here, and one that hands fewer passes.  What the bounds prove is that
# the split and virtual-stream kernels decode the arbitrary streams themselves, so that the values test tests
# them and not only the general parser.  Some streams are the fall-back's by design:
#   trailing, S = 2  the 32 streams with trailing words about as long as the stream put all 2048 symbols into lane
#                    0's half of the words: more symbols than its kCpMax checkpoints reach;
#   runs             runs of 31 - k ones or more at low k: symbols longer than the windows;
#   wrap             q * 2^k >= 2^32 needs q >= 2^(32-k) ones: at most k >= 22 fit the decoder's ring, so this
#                    family mostly tests the general parser (the `random` family at k = 29..31 holds wrapping
#                    symbols the virtual-stream kernel decodes itself);
#   long             more than 65 535 bits in a lane's chunk: the 16-bit checkpoints run out.
# S = 0 runs the general parser alone; nothing is flagged.
FAMILY_SIZES = {"random": 64, "trailing": 64, "runs": 1120, "wrap": 20, "long": 64, "periodic": 96}
FLAGGED = {  # S: random, trailing, runs, wrap, long, periodic
    1: (0, 0, 169, 13, 64, 0),
    2: (0, 32, 284, 13, 64, 3),
    4: (0, 0, 534, 15, 64, 25),
    8: (0, 0, 643, 15, 64, 24),
    16: (10, 6, 733, 17, 64, 25),
}
# Streams of exact_end_streams() (64) flagged, per S, measured as above.  Ending on the last bit of the last word
# does not send a stream to the fall-back: the few flagged at S > 1 are the split index's (a kernel that flagged
# every exact end would flag all 64 at every S).
EXACT_END_FLAGGED = {1: 0, 2: 2, 4: 0, 8: 2, 16: 8}


def _policy_S(split, n_sub):
    """The split S that decodes a batch of n_sub streams: SELAB200_RICE_SPLIT, or else the default policy of
    rice_split_log2 (c_abi.cu), which scales with the device's SM count.  0 (the general parser alone) -> 0."""
    if split is not None:
        return int(split)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if n_sub >= 81 * sms:
        return 1
    log2s = 0
    while log2s < 4 and (n_sub << log2s) < 270 * sms:
        log2s += 1
    return 1 << log2s


def _split(monkeypatch, split):
    if split is None:
        monkeypatch.delenv("SELAB200_RICE_SPLIT", raising=False)
    else:
        monkeypatch.setenv("SELAB200_RICE_SPLIT", split)


@pytest.fixture(scope="module")
def model():
    """Per family: its streams in a shuffled order (flagged and fast-path streams share warps), their values and
    the bits their parse needs."""
    out = {}
    for i, name in enumerate(GOOD):
        s = RF.family(name)
        perm = np.random.default_rng(i).permutation(len(s))
        s = [s[j] for j in perm]
        v, b = XR.parse_batch(s, FRAME)
        out[name] = (s, v, b)
    return out


def _res(streams, **kw):
    return [dict(res=s, **kw) for s in streams]


@pytest.mark.parametrize("split", SPLITS)
def test_values_every_family(model, monkeypatch, split):
    _split(monkeypatch, split)
    flagged, S = {}, {}
    for name in GOOD:
        s, v, _ = model[name]
        descs, arena = RF.layout(_res(s))
        res, flagged[name] = rice_decode_frames(descs, arena, 1)
        S[name] = _policy_S(split, len(s))
        bad = np.flatnonzero((res != v).any(axis=1))
        assert bad.size == 0, (name, split, bad[:8].tolist(), [s[i][0] for i in bad[:8]])
    # every family in one batch, interleaved, an odd number of streams
    mixed = [(name, i) for name in GOOD for i in range(len(model[name][0]))]
    perm = np.random.default_rng(3).permutation(len(mixed))
    pick = [mixed[j] for j in perm[:len(mixed) - 1 + len(mixed) % 2]]
    descs, arena = RF.layout(_res([model[n][0][i] for n, i in pick]))
    res, _ = rice_decode_frames(descs, arena, 1)
    want = np.stack([model[n][1][i] for n, i in pick])
    assert np.array_equal(res, want), split
    for i, name in enumerate(GOOD):
        assert len(model[name][0]) == FAMILY_SIZES[name]
        bound = FLAGGED[S[name]][i] if S[name] else 0
        assert flagged[name] <= bound, (name, split, S[name], flagged)


def test_general_parser_alone_flags_nothing(model, monkeypatch):
    """With the general parser alone (S = 0) no stream is flagged, whatever the scratch the flags live in held
    before: a stage-level encode of 1 024 streams first leaves its non-zero counts there (the flag count once
    reported them)."""
    vals = np.random.default_rng(1).integers(1, 1 << 20, (1024, FRAME)).astype(np.int32)
    sela_b200.rice_encode(vals)
    _split(monkeypatch, "0")
    s, v, _ = model["random"]
    res, flagged = rice_decode_frames(*RF.layout(_res(s)), 1)
    assert flagged == 0 and np.array_equal(res, v)


def exact_end_streams(rng):
    """Random symbols at every k, the last one lengthened so that the stream ends on the last bit of its last word."""
    out = []
    for k in range(32):
        qs, pays = rng.geometric(0.5, FRAME) - 1, rng.integers(0, 1 << 32, FRAME, dtype=np.uint64)
        qs[-1] += -XR.code_bits(qs.astype(np.uint64) << np.uint64(k), k) % 32
        out.append((k, RF.symbols(qs, pays, k)))
    return out


@pytest.mark.parametrize("split", ["1", "2", "4", "8", "16", None])
def test_exact_end_takes_the_fast_path(monkeypatch, split):
    """A stream that ends exactly on its last bit is decoded by the virtual-stream kernel itself: its last part's
    end check accepts pos == 32 * words.  (Were it to flag such streams, the general parser would still decode
    them correctly: only the flagged count shows it.)"""
    _split(monkeypatch, split)
    streams = exact_end_streams(np.random.default_rng(9)) * 2
    values, bits = XR.parse_batch(streams, FRAME)
    assert (bits == 32 * np.array([w.size for _, w in streams])).all()
    descs, arena = RF.layout(_res(streams))
    res, flagged = rice_decode_frames(descs, arena, 1)
    assert np.array_equal(res, values)
    assert flagged <= EXACT_END_FLAGGED[_policy_S(split, len(streams))], (split, flagged)


def _sample(model, rng, per_family=3):
    out = []
    for name in GOOD:
        s, v, b = model[name]
        for i in rng.choice(len(s), per_family, replace=False):
            out.append((name, s[i][0], s[i][1], int(-(-b[i] // 32)), v[i]))
    return out


@pytest.mark.parametrize("split", SPLITS)
def test_acceptance_boundary(model, monkeypatch, split):
    """need words: accepted; need + t: accepted, same values; need - 1 and the `short` family (0 words, fewer than
    4 * S words, fewer than the parse needs): -6, wherever the stream sits in a batch of good ones -- first, in the
    middle of a warp, on a warp's last lane, in a later CTA -- and at every 16-byte phase."""
    _split(monkeypatch, split)
    rng = np.random.default_rng(int(split or 99) + 1)
    sample = _sample(model, rng)
    subs, want = [], []
    for j, (_, k, w, need, v) in enumerate(sample):
        more = np.concatenate([w[:need], rng.integers(0, 1 << 32, 1 + j % 7, dtype=np.uint64).astype(np.uint32)])
        subs += [dict(res=(k, w[:need]), phase=j), dict(res=(k, more), phase=j + 2)]
        want += [v, v]
    descs, arena = RF.layout(subs)
    assert XR.accepts(descs, arena, 1, frames=False)
    res, _ = rice_decode_frames(descs, arena, 1)
    assert np.array_equal(res, np.stack(want)), split
    good = _res(model["random"][0] + model["periodic"][0])[:128 + 9]
    S = max(1, _policy_S(split, len(good) + 1))
    per_warp, per_cta = 32 // S, 128 // S
    # one word short of the need, and short streams: none at all, below 4 * S words (unsplittable), at 4 * S - 1
    short = [(k, w[:need - 1]) for _, k, w, need, _ in sample]
    fam = RF.family("short")
    sizes = np.array([w.size for _, w in fam])
    pick = [int(np.flatnonzero(sizes == 0)[0])] + list(np.flatnonzero(sizes == 4 * S - 1)[:1])
    pick += list(rng.choice(np.flatnonzero(sizes < 4 * S), 14 - len(pick), replace=False))
    short += [fam[i] for i in pick]
    _, bits = XR.parse_batch(short, FRAME)
    assert (bits > 32 * np.array([w.size for _, w in short])).all()     # the model rejects every one
    at = [0, per_warp // 2, per_warp - 1, per_cta + 1]
    for j, (k, w) in enumerate(short):
        subs = list(good)
        subs.insert(at[j % 4], dict(res=(k, w), phase=j // 4))           # every position at every phase
        descs, arena = RF.layout(subs)
        assert int(descs["res_offset"][at[j % 4]]) % 4 == j // 4 % 4
        with pytest.raises(_lib.SelaB200Error) as e:
            rice_decode_frames(descs, arena, 1)
        assert e.value.status == XR.ERR_BITSTREAM, (k, w.size, split, at[j % 4])


def _entry_points(descs, words, channels, pcm):
    """Status and output of every frame-level entry point: None where all raised -6, else the one output."""
    outs, errs = [], []
    calls = [lambda: sela_b200.decode_frames(descs, words, channels),
             lambda: decode_frames_device(descs, words, channels),
             lambda: sela_b200.decode_container(
                 np.frombuffer(wavio.pack_container(descs, words, 44100, channels), np.uint8))[1]]
    for call in calls:
        try:
            outs.append(call())
        except _lib.SelaB200Error as e:
            errs.append(e.status)
    try:
        rep = sela_b200.verify_frames(descs, words, channels, pcm)
    except _lib.SelaB200Error as e:
        errs.append(e.status)
        rep = None
    assert not (outs and errs), errs
    if errs:
        assert set(errs) == {XR.ERR_BITSTREAM}
        return None, None
    for o in outs[1:]:
        assert np.array_equal(o, outs[0])
    return outs[0], rep


@pytest.mark.parametrize("channels", [1, 2])
def test_entry_points_agree(model, channels):
    """Order-0 subframes (no predictor: the PCM is the residue's low 16 bits) through decode_frames, verify_frames,
    decode_frames_device and decode_container: the same status and the same output."""
    rng = np.random.default_rng(channels)
    picked = [(s, v) for name in GOOD for s, v in zip(model[name][0][:10], model[name][1][:10])]
    picked = picked[:len(picked) // channels * channels]
    subs = _res([s for s, _ in picked], order=0, refl=(0, np.zeros(0, np.uint32)))
    descs, arena = RF.layout(subs, channels)
    vals = np.stack([v for _, v in picked]).reshape(-1, channels, FRAME)
    pcm = (vals.transpose(0, 2, 1).reshape(-1) & 0xFFFF).astype(np.uint16).view(np.int16)
    out, rep = _entry_points(descs, arena, channels, pcm)
    assert out is not None and np.array_equal(out, pcm)
    assert rep.size == 0
    assert np.array_equal(ol.best().decode_frames(descs, arena, channels), pcm)
    flip = pcm.copy()
    at = int(rng.integers(0, flip.size))
    flip[at] ^= 1
    rep = sela_b200.verify_frames(descs, arena, channels, flip)
    assert rep.size == 1
    f, c, t = at // (FRAME * channels), at % channels, at % (FRAME * channels) // channels
    assert (rep[0]["frame"], rep[0]["channel"], rep[0]["first_sample"], rep[0]["n_differing"]) == (f, c, t, 1)
    # one residue stream one word short: every entry point reports it, none decodes anything
    short = descs.copy()
    i = int(rng.integers(0, 10))                                # a `random` stream: no trailing words
    short["res_words"][i] -= 1
    assert not XR.accepts(short, arena, channels)
    assert _entry_points(short, arena, channels, pcm) == (None, None)
    # a residue stream of the `short` family in place of one of them: 0 words, a few, fewer than 64
    fam = RF.family("short")
    for j, n in enumerate((0, 3, 63)):
        stream = next(s for s in fam if s[1].size == n)
        i = (7 * j + channels) % len(subs)
        descs_s, arena_s = RF.layout(subs[:i] + [dict(subs[i], res=stream)] + subs[i + 1:], channels)
        assert not XR.accepts(descs_s, arena_s, channels)
        assert _entry_points(descs_s, arena_s, channels, pcm) == (None, None), n


def test_reflection_streams():
    """k_rice_decode on the reflection streams (which = 0): count = order 1..100 at every k, exact and with
    trailing words, through decode_frames against the exact decoder model; one word short is -6."""
    P = ol.load("port")
    rng = np.random.default_rng(8)
    subs, crafted = [], []
    for order in range(1, 101):
        for k in {order % 32, (order + 11) % 32, (order + 22) % 32}:
            q = CR.draw_q(rng, order)
            r = rng.integers(-300, 301, FRAME).astype(np.int32)
            w = XR.pack_stream(XR.zigzag(q), k)
            if len(subs) % 2:
                w = np.concatenate([w, rng.integers(0, 1 << 32, 1 + len(subs) % 5, dtype=np.uint64).astype(np.uint32)])
            subs.append(dict(order=order, refl=(k, w), res=(9, XR.pack_stream(XR.zigzag(r), 9))))
            crafted.append(CR.Sub(0, 0, 0, order, q, r))
    assert {s["refl"][0] for s in subs} == set(range(32))
    descs, arena = RF.layout(subs)
    pcm, _, dom = X.decode(crafted, 1, P)
    assert dom.mean() > 0.5
    out = sela_b200.decode_frames(descs, arena, 1).reshape(-1, FRAME)
    want = pcm.reshape(-1, FRAME)
    assert np.array_equal(out[dom], want[dom])
    by_k = {}
    for i, s in enumerate(subs):
        by_k.setdefault(s["refl"][0], i)
    for k, i in sorted(by_k.items()):
        kk, w = subs[i]["refl"]
        need = -(-XR.code_bits(XR.zigzag(crafted[i].q), kk) // 32)
        bad = list(subs[:130])
        bad.insert(k * 4 % 130, dict(subs[i], refl=(kk, w[:need - 1])))
        descs, arena = RF.layout(bad)
        assert not XR.accepts(descs, arena, 1)
        with pytest.raises(_lib.SelaB200Error) as e:
            sela_b200.decode_frames(descs, arena, 1)
        assert e.value.status == XR.ERR_BITSTREAM, k


def test_stage_rice_decode_zero_extends(model):
    """selab200_rice_decode reads zeros past n_words and never fails on length: overrunning streams decode to the
    model's zero-extended values with status 0."""
    rng = np.random.default_rng(6)
    streams = list(RF.family("short"))
    for _, k, w, need, _ in _sample(model, rng, 4):
        streams += [(k, w[:need - 1]), (k, w[:need])]
    stride = max(w.size for _, w in streams) + 3
    W = np.full((len(streams), stride), 0xFFFFFFFF, np.uint32)     # behind n_words: ones, which must not be read
    for i, (_, w) in enumerate(streams):
        W[i, :w.size] = w
    out = sela_b200.rice_decode(W, [w.size for _, w in streams], [k for k, _ in streams], [FRAME] * len(streams))
    values, bits = XR.parse_batch(streams, FRAME)
    assert (bits > 32 * np.array([w.size for _, w in streams])).sum() >= len(streams) // 2
    assert np.array_equal(out, values)
