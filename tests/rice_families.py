"""Residue streams for the Rice decoder tests (TEST INFRASTRUCTURE): families of bit content the encoder never
writes, at every k from 0 to 31, and a layout that puts them behind descriptors.

Every family returns a list of (k, words): `words` is the whole stream, res_words = words.size.  What the streams
decode to, and how many of their bits the parse needs, comes from the exact model (tests/exact_rice.py).

    random     uniformly random words cut to what the parse needs: arbitrary bit content, the resync and
               merge of the split index on input the encoder never writes
    trailing   the same with 1-7 random words behind the last symbol, or up to twice the stream's length
    runs       runs of exactly 31-k, 32-k, 33-k, 63, 64, 65 and ~1000 ones at symbols t*2048/S and t*2048/S +- 1
               (every S), also starting at a word boundary and ending on a word's last bit
    wrap       symbols with q * 2^k >= 2^32 (k >= 12; below that a single symbol needs more than 65 535 words)
    long       40 000-65 535 words: the split index's 16-bit checkpoints run out
    periodic   a long periodic stretch, then random bits: wrong-phase parses that stay out of step
    short      0 words, and fewer than 64 (= 4 * 16) words: unsplittable, and every such stream of 2048 symbols
               overruns
"""
import functools

import numpy as np

import exact_rice as XR
from exact_rice import pack_stream, zigzag
from oracle_lib import DESC_DTYPE

FRAME = 2048
KS = range(32)
ONES = np.uint32(0xFFFFFFFF)
BOUNDARIES = np.arange(1, 16) * (FRAME // 16)   # symbol t*2048/S for every S = 2..16


def symbols(qs, pays, k):
    """Words of the symbols (q ones, a zero, the low k bits of pay MSB first), any q."""
    qs = np.asarray(qs, np.uint64)
    pays = np.asarray(pays, np.uint64) & np.uint64((1 << k) - 1)
    return pack_stream((qs << np.uint64(k)) | pays, k)


def _random_symbols(rng, k, n=FRAME):
    return rng.geometric(0.5, n) - 1, rng.integers(0, 1 << 32, n, dtype=np.uint64)


def _cut_to_need(streams):
    """Cut every stream to the words its 2048-symbol parse needs (the rest of its last word stays as it is)."""
    _, bits = XR.parse_batch(streams, FRAME)
    out = []
    for (k, w), b in zip(streams, bits):
        need = int(-(-b // 32))
        assert need <= w.size, (k, need, w.size)
        out.append((k, w[:need].copy()))
    return out


def random_streams(rng, per_k=2):
    raw = []
    for k in KS:
        for _ in range(per_k):
            n = FRAME * (k + 2) // 32 * 2 + 64
            raw.append((k, rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)))
    return _cut_to_need(raw)


def trailing_streams(rng, per_k=2):
    out = []
    for i, (k, w) in enumerate(random_streams(rng, per_k)):
        extra = 1 + i % 7 if i % 2 == 0 else w.size if i % 4 == 1 else int(rng.integers(w.size // 2, w.size))
        extra = min(extra, 0xFFFF - w.size)
        out.append((k, np.concatenate([w, rng.integers(0, 1 << 32, extra, dtype=np.uint64).astype(np.uint32)])))
    return out


def _align(qs, pays, k, at, end_on_word):
    """Lengthen the run of symbol at-1 so that symbol `at` starts on a word boundary (end_on_word: so that its
    terminator is the last bit of a word)."""
    lens = qs.astype(np.int64) + 1 + k
    start = int(lens[:at].sum())
    target = 31 - int(qs[at]) if end_on_word else 0
    qs[at - 1] += (target - start) % 32


def run_streams(rng):
    out = []
    for k in KS:
        for run in (31 - k, 32 - k, 33 - k, 63, 64, 65, int(rng.integers(990, 1010))):
            for shift, align in ((-1, None), (0, None), (1, None), (0, "start"), (0, "end")):
                qs, pays = _random_symbols(rng, k)
                at = BOUNDARIES + shift
                qs[at] = run
                if align:
                    for a in at:
                        _align(qs, pays, k, a, align == "end")
                out.append((k, symbols(qs, pays, k)))
    return out


def wrap_streams(rng):
    out = []
    for k in range(12, 32):
        qmin = 1 << (32 - k)
        n_wrap = int(max(1, min(12, 40000 * 32 // (qmin * 3))))
        qs, pays = _random_symbols(rng, k)
        at = np.concatenate([BOUNDARIES, rng.integers(0, FRAME, 16)])[:n_wrap]
        at[-1] = FRAME - 1                           # and the last symbol
        qs[at] = qmin + rng.integers(0, 4, at.size)
        out.append((k, symbols(qs, pays, k)))
    return out


def long_streams(rng):
    out = []
    for k in KS:
        for lumpy in (False, True):
            qs, pays = _random_symbols(rng, k)
            target = int(rng.integers(40100, 0xFFFF + 1)) * 32
            extra = target - XR.code_bits((qs.astype(np.uint64) << np.uint64(k)), k) - 31
            at = rng.choice(FRAME, 16, replace=False) if lumpy else np.arange(FRAME)
            qs[at] += extra // at.size
            w = symbols(qs, pays, k)
            assert 40000 <= w.size <= 0xFFFF, w.size
            out.append((k, w))
    return out


def periodic_streams(rng):
    raw = []
    for k in KS:
        for q, pay in ((0, 0), (1, (1 << k) - 1), (2, 0x55555555)):
            m = int(rng.integers(1000, 2000))
            head = symbols(np.full(m, q), np.full(m, pay, np.uint64), k)
            tail = rng.integers(0, 1 << 32, FRAME * (k + 2) // 32 * 2 + 64, dtype=np.uint64).astype(np.uint32)
            raw.append((k, np.concatenate([head, tail])))
    return _cut_to_need(raw)


def short_streams(rng):
    return [(k, rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32))
            for k in KS for n in (0, 1 + k % 4, 4 * (1 + k % 16) - 1)]


def synthetic_streams(rng):
    """Streams of chosen values (tests/test_rice_split.py): (k, words, u)."""
    out = []
    lap = lambda scale: np.round(rng.laplace(0, scale, FRAME)).astype(np.int64)
    # the BASELINE regime (k ~ 11) and its neighbours, chosen k around the optimum and away from it
    for scale, k in [(900, 10), (900, 11), (900, 12), (60, 5), (60, 7), (3, 1), (3, 2), (0.3, 0), (20000, 15), (20000, 13)]:
        out.append((k, zigzag(lap(scale))))
    # silence and constants: periodic streams in which a wrong-phase parse may never resynchronise
    out.append((0, zigzag(np.zeros(FRAME))))
    out.append((10, zigzag(np.full(FRAME, 1234))))
    out.append((3, zigzag(np.full(FRAME, -5))))
    out.append((6, zigzag(np.tile([37, -37], FRAME // 2))))
    out.append((11, zigzag(np.tile([1000, 1001, -999], FRAME // 3 + 1)[:FRAME])))
    # outliers: a few symbols longer than one 32-bit window, and very long runs
    v = lap(500); v[[5, 700, 701, 2047]] = [40000, -60000, 90000, -120000]; out.append((9, zigzag(v)))
    v = lap(30); v[::97] = 5000; out.append((4, zigzag(v)))
    v = lap(2); v[1000] = 3000; out.append((0, zigzag(v)))
    v = lap(800); v[256 * np.arange(1, 8)] = 70000; out.append((10, zigzag(v)))   # long symbols AT the part boundaries
    v = lap(800); v[256 * np.arange(1, 8) - 1] = -70000; out.append((10, zigzag(v)))
    # loud then quiet: parts with very different bit densities
    v = np.concatenate([lap(8000)[:300], lap(3)[:FRAME - 300]]); out.append((4, zigzag(v)))
    v = np.concatenate([lap(2)[:1800], lap(6000)[:248]]); out.append((3, zigzag(v)))
    # k extremes
    out.append((19, zigzag(rng.integers(-(1 << 19), 1 << 19, FRAME))))
    out.append((24, zigzag(rng.integers(-(1 << 23), 1 << 23, FRAME))))
    out.append((31, rng.integers(0, 1 << 31, FRAME).astype(np.uint64)))
    # full-scale noise: the longest streams 16-bit audio produces
    out.append((16, zigzag(rng.integers(-65535, 65536, FRAME))))
    return [(k, pack_stream(us, k), us) for k, us in out]


FAMILIES = {"random": random_streams, "trailing": trailing_streams, "runs": run_streams, "wrap": wrap_streams,
            "long": long_streams, "periodic": periodic_streams, "short": short_streams}


@functools.lru_cache(maxsize=None)
def family(name, seed=0):
    """The streams of one family (cached: callers must not modify them)."""
    return FAMILIES[name](np.random.default_rng([seed, sorted(FAMILIES).index(name)]))


# ---------------------------------------------------------------------------------------------- layout --

def layout(subs, channels=1):
    """subs: list of dicts with `res` = (k, words) and optionally `refl` = (k, words), `order`, `channel`, `type`,
    `parent`, `phase`.  Returns (descs, arena): each stream behind 1-4 all-ones filler words chosen so that residue
    stream i starts at 16-byte phase `phase` (default i % 4) of the arena, and all-ones behind the last one --
    words a parser must never read.  Defaults: channel i % channels, independent, order 1 with a one-word zero reflection
    stream (one symbol: 0)."""
    descs = np.zeros(len(subs), DESC_DTYPE)
    arena, at = [], 0
    for i, s in enumerate(subs):
        d = descs[i]
        d["channel"] = s.get("channel", i % channels)
        d["subframe_type"] = s.get("type", 0)
        d["parent_channel"] = s.get("parent", d["channel"])
        d["lpc_order"] = s.get("order", 1)
        d["samples"] = FRAME
        for name in ("refl", "res"):
            k, w = s.get(name, (0, np.zeros(1, np.uint32))) if name == "refl" else s["res"]
            pad = 1 + (s.get("phase", i) - at - 1) % 4 if name == "res" else 1 + i % 3
            arena.append(np.full(pad, ONES, np.uint32))
            at += pad
            d[name + "_rice_param"], d[name + "_words"], d[name + "_offset"] = k, w.size, at
            arena.append(np.asarray(w, np.uint32))
            at += w.size
    arena.append(np.full(4, ONES, np.uint32))
    return descs, np.concatenate(arena)

