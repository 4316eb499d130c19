"""An exact model of Rice coding and of the decoder's acceptance rule (TEST INFRASTRUCTURE).

    encode       rice::RiceEncoder (src/rice/rice_encoder.cpp:12-81) on any int32 input: the zig-zag, the k
                 search and the bit layout, with every total an exact integer.
    encode_batch the same over many rows at once, vectorised (see encode_batch for the domain and the
                 device's extension of it).
    pack_stream  the packer alone, at a chosen k (also for streams the search would never choose).
    parse        rice::RiceDecoder (src/rice/rice_decoder.cpp:21-52) on any bit content: a run of ones, a
                 zero, then k payload bits MSB first; the value is (ones << k) | payload in uint32 (line 37 shifts
                 a uint32_t, so q << k wraps), then unzigzagged as convertUnsignedToSigned does.  Bits past
                 n_words read as zero; bits_needed is where the last symbol ends, so a parse that went past the
                 stream's words has bits_needed > 32 * n_words.
    parse_batch  the same over many streams at once, one step per symbol for the whole batch.  A run of ones
                 is found without a loop: the rest of the current word, else the first word behind it that is
                 not all ones (a table over the batch's words), so streams with runs of thousands of ones and
                 tens of thousands of words take no longer than any other.
    accepts      whether the decoder returns SELAB200_ERR_BITSTREAM (-6) for a batch of descriptors and words:
                 desc_ok / frame_check of sela_b200/csrc, and, for the frame-level decoders, both streams of every
                 subframe ending inside their words (bits_needed <= 32 * words).  The stage-level
                 selab200_rice_decode zero-extends instead and never fails on length.

Plain NumPy, no device and no oracle inside: tests/test_exact_rice_model.py pins it against the reference's
encoder and decoder.
"""
from dataclasses import dataclass

import numpy as np

FRAME = 2048
MAX_ORDER = 100
MAX_RICE = 20                # k in 0..19 (rice_encoder.cpp:20-33)
ERR_BITSTREAM = -6

_REV8 = np.array([int("{:08b}".format(i)[::-1], 2) for i in range(256)], np.uint64)
_ALL_ONES = np.uint64(0xFFFFFFFF)
_M32 = np.uint64(0xFFFFFFFF)


def _rev32(x):
    x = np.asarray(x, np.uint64)
    b = lambda s: _REV8[((x >> np.uint64(s)) & np.uint64(255)).astype(np.intp)]
    return (b(0) << np.uint64(24)) | (b(8) << np.uint64(16)) | (b(16) << np.uint64(8)) | b(24)


def _ctz32(v):
    """Trailing zeros of 32-bit values (as uint64); 32 for zero."""
    v = np.asarray(v, np.uint64)
    low = v & (~v + np.uint64(1))
    return np.where(v == 0, 32, np.frexp(low.astype(np.float64))[1] - 1).astype(np.int64)


def unzigzag(u):
    """convertUnsignedToSigned (rice_decoder.cpp:46-52) of uint32 values."""
    u = np.asarray(u, np.uint64) & _M32
    v = (u >> np.uint64(1)).astype(np.int64) ^ -(u & np.uint64(1)).astype(np.int64)
    return v.astype(np.int32)


# ---------------------------------------------------------------------------------------------- encoder --

def zigzag(x):
    """Zig-zag of int32 values in the 32-bit domain with uint32 wrap, ((uint32)x << 1) ^ (x >> 31), as the
    device's `zigzag` computes it -> uint64 holding the uint32.  That is 2x for x >= 0 and -2x - 1 below.
    For |x| < 2^30 it equals convertSignedToUnsigned (rice_encoder.cpp:12-18); beyond that the reference's
    int32 shift overflows (undefined behaviour), and this, a bijection of int32 onto uint32, is the device's
    extension of it."""
    x = np.asarray(x, np.int64)
    assert x.size == 0 or (x.min() >= -(1 << 31) and x.max() < (1 << 31)), "not int32"
    return np.where(x >= 0, 2 * x, -2 * x - 1).astype(np.uint64)


def _pack_rows(us, counts, ks):
    """generateEncodedBits + writeInts (rice_encoder.cpp:35-71) for many rows at once.  us: uint64 [n, width],
    row i coding its first counts[i] values at k = ks[i]; q = u >> k may be any size.  Each symbol is q ones, a
    zero, then the k low bits of u MSB first; bit b of a row goes to word b / 32, bit b % 32, and the rest of
    the last word is zero.  -> list of n uint32 arrays, ceil(bits / 32) words each."""
    us = np.asarray(us, np.uint64)
    n = us.shape[0]
    counts = np.asarray(counts, np.int64).reshape(n)
    ks = np.asarray(ks, np.int64).reshape(n)
    live = np.arange(us.shape[1])[None, :] < counts[:, None]
    u = us[live]                                                   # row after row
    row = np.repeat(np.arange(n), counts)
    k = ks[row]
    q = (u >> k.astype(np.uint64)).astype(np.int64)
    lens = q + 1 + k
    ends = np.cumsum(lens)
    first = np.concatenate([[0], np.cumsum(counts)])               # each row's first symbol
    before = np.concatenate([[0], ends])[first]                    # bits of the rows in front of each row
    row_bits = before[1:] - before[:-1]
    n_words = (row_bits + 31) // 32
    base = np.concatenate([[0], np.cumsum(n_words)]) * 32          # every row starts on a word boundary
    start = base[row] + (ends - lens - before[row])                # first bit of each symbol
    total = int(base[-1])
    # the runs of ones as +1 at their first bit and -1 behind their last: runs never touch, so one pass of
    # plain stores and a running sum lay them all out
    edge = np.zeros(total + 1, np.int8)
    run = q > 0
    edge[start[run]] = 1
    edge[start[run] + q[run]] = -1
    bits = np.cumsum(edge[:total], dtype=np.int8).astype(np.uint8)
    for j in range(int(ks.max()) if n else 0):                    # payload bit j: bit k - 1 - j of u
        s = np.flatnonzero(k > j)
        bits[start[s] + q[s] + 1 + j] = ((u[s] >> (k[s] - 1 - j).astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
    flat = np.packbits(bits, bitorder="little").view("<u4").astype(np.uint32)
    return [flat[base[i] // 32:base[i + 1] // 32] for i in range(n)]


def pack_stream(us, k):
    """One stream of symbols u (uint64, any q = u >> k) at a chosen k -> its uint32 words."""
    us = np.asarray(us, np.uint64).reshape(-1)
    return _pack_rows(us[None, :], [us.size], [k])[0]


@dataclass
class Encoded:
    k: np.ndarray        # int64 [n]: the first arg-min of the totals
    bits: np.ndarray     # int64 [n]: requiredBits, the minimum total
    n_words: np.ndarray  # int64 [n]
    words: list          # n uint32 arrays, n_words[i] words each
    totals: np.ndarray   # int64 [n, 20]: the code length at every k


def encode_batch(rows, counts=None, chunk=1024):
    """rice::RiceEncoder::process (rice_encoder.cpp:73-81) of many streams.  rows: int32 values [n, width],
    row i coding its first counts[i] (default: all) -> Encoded.

    u is `zigzag` (exact for |x| < 2^30, the device's extension beyond).  total_k = sum(u >> k) + n * (1 + k)
    for k in 0..19 as exact integers, and k is the first arg-min (calculateOptimumRiceParam scans k upward and
    keeps a total only if it is strictly smaller).  words = ceil(bits / 32), computed exactly: the reference
    computes ceil((float)bits / 32), which is exact below 2^24 bits, and its domain never exceeds
    2048 * (4095 + 20) bits."""
    rows = np.asarray(rows, np.int64)
    if rows.ndim == 1:
        rows = rows[None, :]
    n, width = rows.shape
    counts = np.full(n, width, np.int64) if counts is None else np.asarray(counts, np.int64).reshape(n)
    assert ((counts >= 0) & (counts <= width)).all()
    ks = np.arange(MAX_RICE, dtype=np.int64)
    totals = np.zeros((n, MAX_RICE), np.int64)
    for a in range(0, n, chunk):                                   # in slices: [n, 2048] uint64 per pass
        u = zigzag(rows[a:a + chunk])
        u[np.arange(width)[None, :] >= counts[a:a + chunk, None]] = 0
        for k in ks:
            totals[a:a + chunk, k] = (u >> np.uint64(k)).sum(axis=1).astype(np.int64)
    totals += counts[:, None] * (1 + ks[None, :])
    k = np.argmin(totals, axis=1)                                  # the first of equal minima
    bits = totals[np.arange(n), k]
    words, a, ends = [], 0, np.cumsum(bits)
    while a < n:                                                   # in slices of about 2^26 bits
        z = max(a + 1, int(np.searchsorted(ends, ends[a] - bits[a] + (1 << 26), side="right")))
        words += _pack_rows(zigzag(rows[a:z]), counts[a:z], k[a:z])
        a = z
    return Encoded(k=k, bits=bits, n_words=(bits + 31) // 32, words=words, totals=totals)


def encode(values):
    """One stream of int32 values -> (k, words)."""
    e = encode_batch(np.asarray(values, np.int64).reshape(1, -1))
    return int(e.k[0]), e.words[0]


def parse_batch(streams, counts):
    """streams: list of (k, words), every word of `words` belonging to the stream; counts: one symbol count for all
    or one per stream.  Returns (values int32 [n, max count], zero past a stream's count; bits_needed int64 [n])."""
    n = len(streams)
    counts = np.broadcast_to(np.asarray(counts, np.int64), (n,)).copy()
    width = int(counts.max()) if n else 0
    values = np.zeros((n, width), np.int32)
    if n == 0:
        return values, np.zeros(0, np.int64)
    ks = np.array([int(k) for k, _ in streams], np.int64)
    assert ((ks >= 0) & (ks < 32)).all()
    # one flat array of 32-bit words: each stream's words, then enough zero words for every symbol that runs past
    # them (at most count * (k + 1) bits) and two more for the window's look-ahead
    sizes = np.array([np.asarray(w).size for _, w in streams], np.int64)
    pads = (counts * (ks + 1) + 31) // 32 + 2
    base = np.concatenate([[0], np.cumsum(sizes + pads)])
    flat = np.zeros(int(base[-1]) + 2, np.uint64)
    for i, (_, w) in enumerate(streams):
        flat[base[i]:base[i] + sizes[i]] = np.asarray(w, np.uint32)
    not_ones = np.flatnonzero(flat != _ALL_ONES)   # every stream's zero padding ends any run
    pos = base[:-1] * 32                           # global bit position of each stream's parse
    ku = ks.astype(np.uint64)
    for t in range(width):
        live = np.flatnonzero(counts > t)
        p = pos[live]
        w, sh = p >> 5, (p & 31).astype(np.uint64)
        rest = flat[w] >> sh                                          # the 32 - sh bits left in this word
        c = _ctz32(~rest & _M32)                                      # trailing ones, at most 32 - sh
        term = p + c
        run_on = c >= 32 - (p & 31)                                   # the rest of the word is all ones
        if run_on.any():
            w2 = not_ones[np.searchsorted(not_ones, w[run_on] + 1)]
            term[run_on] = w2 * 32 + _ctz32(~flat[w2] & _M32)
        ones = (term - p).astype(np.uint64)
        b = term + 1                                                  # first payload bit
        bw, bs = b >> 5, (b & 31).astype(np.uint64)
        win = ((flat[bw] | (flat[bw + 1] << np.uint64(32))) >> bs) & _M32
        k = ku[live]
        pay = np.where(k > 0, _rev32(win) >> ((np.uint64(32) - k) & np.uint64(31)), np.uint64(0))
        u = ((ones << k) & _M32) | pay                                # uint32 shift, rice_decoder.cpp:37
        values[live, t] = unzigzag(u)
        pos[live] = b + k.astype(np.int64)
    return values, pos - base[:-1] * 32


def parse(words, n_words, k, count):
    """One stream: the first n_words of `words` -> (values int32[count], bits_needed)."""
    v, bits = parse_batch([(k, np.asarray(words, np.uint32)[:n_words])], [count])
    return v[0, :count], int(bits[0])


def code_bits(us, k):
    """Bits the symbols u (uint64, any q = u >> k) take: q ones, a zero and k payload bits each."""
    us = np.asarray(us, np.uint64)
    return int(((us >> np.uint64(k)).astype(np.int64) + 1 + k).sum())


# ------------------------------------------------------------------------------------------ acceptance --

def in_arena(offset, words, n_words):
    """A stream of `words` words at word `offset` lies in an arena of n_words words (no sum that could wrap)."""
    offset, words, n_words = int(offset), int(words), int(n_words)
    return words <= n_words and offset <= n_words - words


def desc_ok(d, channels, n_words):
    """desc_ok (sela_b200/csrc/common.cuh): the fields of one descriptor."""
    return (int(d["channel"]) < channels and int(d["parent_channel"]) < channels and int(d["subframe_type"]) <= 1
            and int(d["lpc_order"]) <= MAX_ORDER and int(d["refl_rice_param"]) < 32
            and int(d["res_rice_param"]) < 32 and int(d["samples"]) == FRAME
            and in_arena(d["refl_offset"], d["refl_words"], n_words)
            and in_arena(d["res_offset"], d["res_words"], n_words)
            and not (int(d["subframe_type"]) == 1 and int(d["parent_channel"]) == int(d["channel"])))


def frame_ok(fd, channels, n_words):
    """frame_check (sela_b200/csrc/kernels.cuh): every descriptor passes desc_ok, the channel fields are a
    permutation and no difference subframe has a difference subframe for parent."""
    if not all(desc_ok(d, channels, n_words) for d in fd):
        return False
    if len({int(d["channel"]) for d in fd}) != len(fd):
        return False
    diff = {int(d["channel"]) for d in fd if int(d["subframe_type"]) == 1}
    return not any(int(d["parent_channel"]) in diff for d in fd if int(d["subframe_type"]) == 1)


def _stream(words, d, name):
    at, n = int(d[name + "_offset"]), int(d[name + "_words"])
    return int(d[name + "_rice_param"]), np.asarray(words[at:at + n], np.uint32)


def accepts(descs, words, channels, frames=True):
    """Whether a decoder returns status 0 (True) or SELAB200_ERR_BITSTREAM (False) for the batch.
    frames=True: decode_frames, verify_frames, their *_device forms and the container decode -- frame_check on
    every frame, and both streams of every subframe must end inside their words.
    frames=False: selab200_rice_decode_frames_device -- desc_ok on every descriptor, and the residue stream must
    end inside its words (the reflection streams are not decoded there)."""
    n_words = len(words)
    n_frames = len(descs) // channels
    if frames:
        if not all(frame_ok(descs[f * channels:(f + 1) * channels], channels, n_words) for f in range(n_frames)):
            return False
    elif not all(desc_ok(d, channels, n_words) for d in descs):
        return False
    streams, counts, limits = [], [], []
    for d in descs:
        for name in (("refl", "res") if frames else ("res",)):
            streams.append(_stream(words, d, name))
            counts.append(int(d["lpc_order"]) if name == "refl" else FRAME)
            limits.append(32 * int(d[name + "_words"]))
    if not streams:
        return True
    _, bits = parse_batch(streams, counts)
    return bool((bits <= np.array(limits)).all())
