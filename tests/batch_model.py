"""Whole-batch model (TEST INFRASTRUCTURE): what a batch of any size must code and decode to, built from a small
bank of frames whose outputs are known exactly.

Frames are coded independently, so a batch's correct output is its frames' outputs laid end to end: descriptor i
is the bank descriptor of its frame, with offsets moved to the exclusive prefix sum of the words before it; the
arena is the concatenation of the frames' words; the PCM and the verify report are those of the frames, the report
at batch-global frame numbers.  A batch is `bank[idx]` for a seeded index sequence, and its expected output is
index arithmetic: no CPU coder runs at batch size.

  encode_bank(channels)   ol.best()'s encoding of 100-200 distinct frames (signal families, random frames, sine +
                          noise, silence, DC, identical and inverted channels, full-scale noise; stereo: ties of the
                          stereo decision; 8 channels: the golden frames the reference decoder does not reproduce)
  tile(bank, idx)         the expected descriptors, words, words_used, source PCM, decoded PCM and verify report
  decode_bank()           crafted mono subframes of every synthesis segment width 1..13 in every sample range
  frames16_bank()         crafted 16-channel frames with difference subframes (test_synthesis._frames)
  segment_templates       the decode packing plan (k_decode_plan, kernels.cuh), restated
  plan_chunks             the host calls' chunk plan (c_abi.cu), restated

The restatements choose cases and state what a case reaches; the device is judged on its outputs alone."""
import functools
from dataclasses import dataclass, field

import numpy as np

import crafted as CR
import exact_decode as X
import oracle_lib as ol
import signals
from sela_b200 import synth
from sela_b200._lib import VERIFY_DTYPE

FRAME = 2048
SCAN_TILE = 1024                 # kScanTile: subframes per CTA of the encode scan and the decode plan
MAX_WIDTH = 13                   # kMaxWidth: synthesis segment lanes of an order-100 subframe
MAX_TEMPLATES = 2 * MAX_WIDTH    # kMaxTemplates: the shared template array of k_decode_plan
TAPS = 8                         # kTapsPerLane
MAX_CHUNKS = 72                  # kMaxChunks
I16 = 16383


def width(order):
    """Synthesis segment lanes of a subframe of this order (segment_width, lpc.cuh)."""
    return max(1, -(-int(order) // TAPS))


def synthesis_warps(n_sub):
    """The seg_index allocation of a decode, in warps (synthesis_warps, kernels.cuh)."""
    return n_sub // 2 + 1


# ----------------------------------------------------------------------------------------- banks --

@dataclass
class Bank:
    """Frames coded one by one.  descs: DESC_DTYPE [n, channels] with offsets into `words` (the frames' words in
    bank order); pcm / decoded: int16 [n, 2048, channels]; records: per-frame report entries (a structured array
    with a "frame" field holding the bank frame)."""
    channels: int
    names: list
    pcm: np.ndarray
    descs: np.ndarray
    words: np.ndarray
    decoded: np.ndarray
    records: np.ndarray
    frame_start: np.ndarray = field(init=False)
    frame_words: np.ndarray = field(init=False)

    def __post_init__(self):
        d = self.descs
        self.frame_start = d[:, 0]["refl_offset"].astype(np.int64)
        end = (d[:, -1]["res_offset"] + d[:, -1]["res_words"]).astype(np.int64)
        self.frame_words = end - self.frame_start
        assert np.array_equal(self.frame_start[1:], end[:-1]), "bank frames are not laid out end to end"
        self.arenas = [self.words[a:b] for a, b in zip(self.frame_start, end)]

    def __len__(self):
        return len(self.names)

    def index(self, name):
        return self.names.index(name)


@dataclass
class Batch:
    descs: np.ndarray       # DESC_DTYPE [n_frames * channels]
    words: np.ndarray       # uint32 [used]
    used: int
    pcm: np.ndarray         # int16 interleaved source
    decoded: np.ndarray     # int16 interleaved, what the reference decoder makes of (descs, words)
    report: np.ndarray      # records at batch-global frame numbers


def report_records(decoded, source, channels):
    """VERIFY_DTYPE entries, one per (frame, channel) whose decoded samples differ from the source, in order."""
    d = np.asarray(decoded, np.int16).reshape(-1, FRAME, channels).astype(np.int32)
    s = np.asarray(source, np.int16).reshape(-1, FRAME, channels).astype(np.int32)
    diff = d != s
    out = []
    for f, c in zip(*np.nonzero(diff.any(axis=1))):
        first = int(np.argmax(diff[f, :, c]))
        out.append((int(f), int(c), first, int(diff[f, :, c].sum()), int(d[f, first, c] - s[f, first, c])))
    return np.array(out, VERIFY_DTYPE)


def tile_records(records, idx, frame_base=0):
    """A bank's per-frame records, repeated wherever idx uses their frame, in (batch frame, bank order) order."""
    idx = np.asarray(idx)
    pos, which = [], []
    for r, b in enumerate(records["frame"]):
        p = np.flatnonzero(idx == b)
        pos.append(p)
        which.append(np.full(p.size, r))
    if not pos:
        return records[:0].copy()
    pos, which = np.concatenate(pos), np.concatenate(which)
    order = np.lexsort((which, pos))
    out = records[which[order]].copy()
    out["frame"] = pos[order] + frame_base
    return out


def tile(bank, idx, frame_base=0):
    """The batch bank[idx] as the encoder must code it (the frames of `idx` in turn)."""
    idx = np.asarray(idx, np.int64)
    ch = bank.channels
    fw = bank.frame_words[idx]
    start = np.zeros(idx.size + 1, np.int64)
    np.cumsum(fw, out=start[1:])
    descs = bank.descs[idx].copy()
    shift = (start[:-1] - bank.frame_start[idx])[:, None]
    for name in ("refl_offset", "res_offset"):
        descs[name] = (descs[name].astype(np.int64) + shift).astype(np.uint64)
    words = np.concatenate([bank.arenas[i] for i in idx]) if idx.size else np.zeros(0, np.uint32)
    return Batch(descs.reshape(-1), words, int(start[-1]), bank.pcm[idx].reshape(-1), bank.decoded[idx].reshape(-1),
                 tile_records(bank.records, idx, frame_base))


def unit_words(O, x):
    """(refl_words + res_words, the two streams' words) of one analysis unit as the reference codes it."""
    a = O.lpc_analyse(np.asarray(x, np.int32))
    _, wq = O.rice_encode(a["q"][:a["order"]])
    _, wr = O.rice_encode(a["res"])
    return wq.size + wr.size, np.concatenate([wq, wr])


def _half_signal(rng):
    """A stereo right channel R with |R| <= 16383, so that L = 2R fits 16 bits and L - R = R."""
    return np.clip(CR.signal(rng, 12000), -I16, I16).astype(np.int32)


def stereo_tie(O, rng, delta, same=False, tries=2000):
    """(L, R) whose difference unit L - R codes to exactly `delta` words more than R (delta = 0: equal totals;
    `same`: identical streams too, L = 2R).  Found by perturbing a few samples of L = 2R."""
    for _ in range(tries):
        r = _half_signal(rng)
        n_r, w_r = unit_words(O, r)
        if same:
            return 2 * r, r
        for _ in range(tries // 20):
            lft = 2 * r
            pos = rng.integers(0, FRAME, int(rng.integers(1, 6)))
            lft[pos] += rng.integers(-4, 5, pos.size)
            n_d, w_d = unit_words(O, lft - r)
            if n_d - n_r == delta and (delta != 0 or not np.array_equal(w_d, w_r)):
                return lft, r
    raise AssertionError("no stereo frame with a difference of %d words" % delta)


# stereo tie frames: name -> (words of L - R minus words of R, the subframe_type the decision gives channel 1)
TIES = {"tie_same": (0, 0), "tie_different": (0, 0), "diff_one_less": (-1, 1), "diff_one_more": (1, 0)}


def _stereo_frames(O, rng):
    fam = signals.families()
    names = list(fam)
    out = {}
    for i, n in enumerate(names):                                        # every family against the next one
        out["fam_" + n] = np.stack([fam[n], fam[names[(i + 5) % len(names)]]], 1)
    rand = signals.random_frames(100, seed=11)
    for i in range(50):
        out["random_%d" % i] = np.stack([rand[2 * i], rand[2 * i + 1]], 1)
    sn = synth.sine_noise(44100, 2, n_frames=12, seed=5).reshape(12, FRAME, 2)
    for i in range(12):
        out["sine_noise_%d" % i] = sn[i]
    out["silence"] = np.zeros((FRAME, 2), np.int32)
    out["dc"] = np.tile([[1234, -20000]], (FRAME, 1))
    for i in range(4):
        x = rand[90 + i].astype(np.int64)
        out["identical_%d" % i] = np.stack([x, x], 1)
        out["inverted_%d" % i] = np.stack([x, np.clip(-x, -32768, 32767)], 1)
        out["full_noise_%d" % i] = rng.integers(-32768, 32768, (FRAME, 2))
    for name, (delta, _) in TIES.items():
        lft, r = stereo_tie(O, rng, delta, same=name == "tie_same")
        out[name] = np.stack([lft, r], 1)
    return out


def _oct_frames(O, rng):
    fam = signals.families()
    names = list(fam)
    out = {}
    for i in range(len(names)):
        out["fam_%d" % i] = np.stack([fam[names[(i + 3 * c) % len(names)]] for c in range(8)], 1)
    rand = signals.random_frames(8 * 40, seed=12).reshape(40, 8, FRAME)
    for i in range(40):
        out["random_%d" % i] = rand[i].T
    sn = synth.sine_noise(48000, 8, n_frames=16, seed=6).reshape(16, FRAME, 8)
    for i in range(16):
        out["sine_noise_%d" % i] = sn[i]
    out["silence"] = np.zeros((FRAME, 8), np.int32)
    out["dc"] = np.tile(np.arange(-4, 4) * 4000, (FRAME, 1))
    for i in range(3):
        x = rand[i, 0].astype(np.int64)
        out["identical_%d" % i] = np.tile(x[:, None], (1, 8))
        out["inverted_%d" % i] = np.stack([x if c % 2 == 0 else np.clip(-x, -32768, 32767) for c in range(8)], 1)
        out["full_noise_%d" % i] = rng.integers(-32768, 32768, (FRAME, 8))
    lossy = LOSSY_OCT.reshape(2, FRAME, 8)
    out["lossy_a"], out["lossy_b"] = lossy[0], lossy[1]
    return out


def _golden_lossy():
    import pathlib
    return np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")["pcm_oct_reference_lossy"]


LOSSY_OCT = _golden_lossy()   # frame 8975 / 13577 of synth.sine_noise(48000, 8, 600, seed=2): not reproduced


@functools.lru_cache(maxsize=None)
def encode_bank(channels):
    """The bank of `channels` (2 or 8), coded by ol.best().  Built once per session."""
    O = ol.best()
    rng = np.random.default_rng(1000 + channels)
    frames = _stereo_frames(O, rng) if channels == 2 else _oct_frames(O, rng)
    names = list(frames)
    pcm = np.stack([np.asarray(frames[n]) for n in names]).astype(np.int16)
    assert pcm.shape == (len(names), FRAME, channels)
    descs, words = O.encode_frames(pcm.reshape(-1), channels)
    decoded = O.decode_frames(descs, words, channels).reshape(pcm.shape)
    return Bank(channels, names, pcm, descs.reshape(-1, channels), words, decoded,
                report_records(decoded, pcm, channels))


def lossless_bank(bank, encode_lossless):
    """`bank` coded by `encode_lossless(pcm, channels) -> (descs, words, report)` (the library's lossless encode,
    run on the bank alone): a Bank whose records are the lossless report."""
    descs, words, report = encode_lossless(bank.pcm.reshape(-1), bank.channels)
    return Bank(bank.channels, bank.names, bank.pcm, descs.reshape(-1, bank.channels), words, bank.pcm,
                np.asarray(report))


# ---------------------------------------------------------------------------------- decode banks --

KINDS = ["small", "wide", "neg17", "edge"]


def orders_of_width(w):
    return list(range(0, TAPS + 1)) if w == 1 else list(range(TAPS * (w - 1) + 1, min(TAPS * w, 100) + 1))


@dataclass
class DecodeBank:
    """Crafted subframes (channels each per frame) coded into one arena.  descs: DESC_DTYPE [n, channels]; pcm:
    int16 [n, 2048, channels], their exact decode; widths: [n, channels] segment widths."""
    channels: int
    descs: np.ndarray
    words: np.ndarray
    pcm: np.ndarray
    widths: np.ndarray

    def tile(self, idx):
        """(descs, words, pcm) of the batch self[idx]: every descriptor points into the one bank arena."""
        idx = np.asarray(idx, np.int64)
        return self.descs[idx].reshape(-1), self.words, self.pcm[idx].reshape(-1)


def _decode_bank(P, subs, channels):
    want, _, dom = X.decode(subs, channels, P)
    assert dom.all()
    descs, words = CR.build(P, subs)
    n = len(subs) // channels
    return DecodeBank(channels, descs.reshape(n, channels), words, want.reshape(n, FRAME, channels),
                      np.array([width(s.order) for s in subs]).reshape(n, channels))


@functools.lru_cache(maxsize=None)
def decode_bank(per_width=8):
    """Mono subframes, per_width of each segment width 1..13, the sample ranges of crafted.KINDS in turn and
    orders spread over the width (both of its ends included)."""
    P = ol.load("port")
    rng = np.random.default_rng(77)
    subs = []
    for w in range(1, MAX_WIDTH + 1):
        orders = orders_of_width(w)
        pick = [orders[0], orders[-1]] + list(rng.choice(orders, per_width - 2))
        for j, o in enumerate(pick):
            subs.append(CR.crafted_subframe(P, rng, int(o), KINDS[j % len(KINDS)]))
    return _decode_bank(P, subs, 1)


@functools.lru_cache(maxsize=None)
def frames16_bank():
    """16-channel crafted frames: independent subframes, difference subframes (two children of one parent) and
    parent and difference both near INT32_MIN (test_synthesis._frames)."""
    import test_synthesis as TS
    P = ol.load("port")
    subs = TS._frames(P, np.random.default_rng(416), 16, n_frames=3)
    return _decode_bank(P, subs, 16)


def by_width(bank, counts, rng):
    """Bank subframe indices for a batch with counts[w - 1] subframes of width w, shuffled."""
    w = bank.widths[:, 0]
    idx = np.concatenate([rng.choice(np.flatnonzero(w == v), int(c)) for v, c in enumerate(counts, 1) if c])
    rng.shuffle(idx)
    return idx


# ------------------------------------------------------------------------------- packing plan --

def segment_templates(counts):
    """counts[w - 1] subframes of width w (w = 1..13) -> templates [(repeats, first_warp, copies by width)],
    as k_decode_plan makes them: the widest width left opens a warp, which is filled greedily, widest first."""
    c = [0] + [int(x) for x in counts] + [0] * (15 - len(counts))
    out, warp = [], 0
    while True:
        room, rep, copies = 32, None, [0] * 16
        for v in range(15, 0, -1):
            k = 0 if v > MAX_WIDTH else min(c[v], room // v)
            copies[v] = k
            room -= k * v
            if k:
                rep = c[v] // k if rep is None else min(rep, c[v] // k)
        if room == 32:
            return out
        for v in range(1, 16):
            c[v] -= rep * copies[v]
        out.append((rep, warp, copies))
        warp += rep


def plan_warps(templates):
    return sum(t[0] for t in templates)


# 26 templates (the bound, MAX_TEMPLATES) at 93 259 subframes: counts by width 1..13
TEMPLATES_26 = [4863, 5706, 9165, 6285, 8311, 9268, 9653, 10634, 6995, 6584, 1212, 8760, 5823]


# --------------------------------------------------------------------------------- chunk plan --

def chunk_frames(n_frames, forced=None):
    """chunk_frames_for (c_abi.cu); `forced`: SELAB200_CHUNK_FRAMES."""
    if forced is not None and forced > 0:
        c = forced
    else:
        c = min(max(-(-n_frames // 8), 512), 16384)
    while -(-n_frames // c) > MAX_CHUNKS:
        c *= 2
    return c


def plan_chunks(n_frames, forced=None):
    """plan_chunks (c_abi.cu) -> (chunk boundaries, what the plan reached: chunk size, whether it was doubled to
    stay within MAX_CHUNKS, and whether the first / last base chunk was cut into tapering pieces)."""
    cf = chunk_frames(n_frames, forced)
    n_base = -(-n_frames // cf)
    taper = forced is None and n_base >= 4 and n_base + 6 <= MAX_CHUNKS
    start, cut_first, cut_last = [0], False, False
    for c in range(n_base):
        f0 = c * cf
        f1 = min(f0 + cf, n_frames)
        n = f1 - f0
        if taper and c == 0 and n >= 512:
            start += [f0 + n // 8, f0 + n // 2]
            cut_first = True
        elif taper and c == n_base - 1 and n >= 512:
            start += [f0 + n // 2, f0 + n // 2 + n // 4, f0 + n // 2 + n // 4 + n // 8]
            cut_last = True
        start.append(f1)
    base = forced if forced is not None and forced > 0 else min(max(-(-n_frames // 8), 512), 16384)
    return start, dict(chunk=cf, base_chunks=n_base, doubled=cf != base, taper=taper,
                       cut_first=cut_first, cut_last=cut_last, chunks=len(start) - 1)


# ------------------------------------------------------------------------------- suite shapes --

# one-call device batches: (channels, frames) -> scan CTAs = ceil(frames * channels / SCAN_TILE)
DEVICE_BATCHES = [(2, 12919), (2, 33000), (8, 8200)]
# frames of a one-call batch that hold the stereo ties / lossy frames: both sides of the CTA edges at subframes
# 1024 and 32768 (the scan's 33rd CTA), and the last frame
EDGE_FRAMES = [511, 512, 16383, 16384]

# decode-plan batches (mono unless said otherwise): counts by width 1..13
PLAN_26 = TEMPLATES_26                               # the template bound, 92 CTAs
PLAN_ODD13 = [0] * 12 + [65537]                      # odd count of width 13: the warp bound, 65 CTAs
PLAN_WIDTH1 = [66017] + [0] * 12                     # 32 segments per warp, a partial last warp, 65 CTAs
FRAMES16 = 4200                                      # 16-channel frames: 67 200 subframes, 66 CTAs

# host calls: (frames, SELAB200_CHUNK_FRAMES or None) and the plan each reaches
HOST_PLANS = [
    (1, None), (511, None), (512, None),             # one chunk
    (513, None), (1536, None),                       # untapered
    (1537, None), (2047, None),                      # first chunk tapered, short last chunk not cut
    (2048, None), (4096, None), (5000, None),        # both ends tapered
    (4097, None),                                    # chunk size 513
    (72, 1), (500, 7), (73, 1), (505, 7),            # exactly 72 chunks; then doubled to 37
]


def host_idx(bank, n_frames, forced, special, seed):
    """A seeded batch of bank frames with `special` bank frames (ties, lossy frames) in turn at both sides of every
    chunk boundary and at both ends."""
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, len(bank), n_frames)
    start, _ = plan_chunks(n_frames, forced)
    at = sorted({p for s in start for p in (s - 1, s) if 0 <= p < n_frames})
    for j, p in enumerate(at):
        idx[p] = special[j % len(special)]
    return idx
