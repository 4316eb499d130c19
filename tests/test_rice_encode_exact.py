"""The Rice encoder's compiled kernels against the exact encoder model (tests/exact_rice.py): the parameter search
warp_rice_choose and the packer warp_rice_pack (sela_b200/csrc/rice.cuh), through the stage operator
selab200_rice_encode on every family of tests/rice_encode_families.py, and through the batch encoder on the frames
of tests/analysis_corpus.py.  Every bit of every word the encoder defines is compared; nothing here rests on the
reference being built."""
import numpy as np
import pytest

import analysis_corpus
import exact_rice as XR
import rice_encode_families as REF
from sela_b200 import _lib, codec
from test_fir_probe import fir_residues

pytestmark = pytest.mark.gpu
FRAME = 2048
ONES = 0xFFFFFFFF
ERR_CAPACITY = -4
CHUNK_WORDS = 1 << 24          # rows x words_stride of one call: 64 MB of words


def _raw_encode(values, counts, words_stride):
    """selab200_rice_encode as it is (codec.rice_encode raises on a status) -> (status, k, n_words, words)."""
    _lib.init(0)
    values = np.ascontiguousarray(values, np.int32)
    n, stride = values.shape
    counts = np.ascontiguousarray(counts, np.uint32)
    k, nw = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    words = np.zeros((n, words_stride), np.uint32)
    rc = _lib.lib().selab200_rice_encode(values.ctypes.data, counts.ctypes.data, n, stride, k.ctypes.data,
                                         nw.ctypes.data, words.ctypes.data, words_stride)
    return rc, k, nw, words


def _fill_pool(n, words_stride, value):
    """Leave the device's word pool holding `value` in every word an encode of n rows of words_stride words uses:
    selab200_rice_decode uploads its words into that pool (a decode of no symbols does nothing else)."""
    z = np.zeros(n, np.uint32)
    codec.rice_decode(np.full((n, words_stride), value, np.uint32), z, z, z, out_stride=1)


def _chunks(b):
    """Row subsets of a batch, each with a words_stride of its own largest n_words, small enough to transfer."""
    order = np.argsort(b.enc.n_words, kind="stable")
    out, cur = [], []
    for i in order:
        ws = max(1, int(b.enc.n_words[i]))
        if cur and (len(cur) + 1) * ws > CHUNK_WORDS:
            out.append(np.array(cur))
            cur = []
        cur.append(i)
    if cur:
        out.append(np.array(cur))
    return [(rows, max(1, int(b.enc.n_words[rows].max()))) for rows in out]


def _model_words(b, rows, ws):
    m = np.zeros((len(rows), ws), np.uint32)
    for j, i in enumerate(rows):
        m[j, :b.enc.n_words[i]] = b.enc.words[i]
    return m


def _defined(nw, ws):
    return np.arange(ws)[None, :] < np.asarray(nw, np.int64)[:, None]


def _check_rows(b, rows, k, nw, words, ws, what):
    assert np.array_equal(k, b.enc.k[rows]), (what, rows[np.flatnonzero(k != b.enc.k[rows])[:5]])
    assert np.array_equal(nw, b.enc.n_words[rows]), (what, rows[np.flatnonzero(nw != b.enc.n_words[rows])[:5]])
    mask = _defined(nw, ws)
    bad = np.flatnonzero(((words != _model_words(b, rows, ws)) & mask).any(axis=1))
    assert bad.size == 0, (what, "rows differ", rows[bad[:5]])
    # the padding bits of the last word are zero
    bits = b.enc.bits[rows]
    last = np.flatnonzero(bits % 32)
    tail = words[last, nw[last].astype(np.int64) - 1] >> (bits[last] % 32).astype(np.uint32)
    assert not tail.any(), (what, rows[last[np.flatnonzero(tail)[:5]]])


@pytest.mark.parametrize("fill", [0, ONES], ids=["pool_zeros", "pool_ones"])
@pytest.mark.parametrize("name", REF.NAMES)
def test_family_equals_model(name, fill):
    """rice_param, n_words and words [0, n_words) equal the model whatever the word pool held before: once after
    a call that left zeros there, once after one that left all-ones words."""
    reached = False
    for b in REF.family(name):
        for rows, ws in _chunks(b):
            _fill_pool(len(rows), ws, fill)
            rc, k, nw, words = _raw_encode(b.values[rows], b.counts[rows], ws)
            assert rc == 0, _lib.lib().selab200_last_error()
            _check_rows(b, rows, k, nw, words, ws, name)
            reached |= bool((words[~_defined(nw, ws)] == fill).any())
    assert reached, "no word behind n_words showed the pool's contents: the fill did not reach the pool"


@pytest.mark.parametrize("name", REF.NAMES)
def test_family_round_trip(name):
    """The words the encoder wrote decode back to the input values, by selab200_rice_decode and by the parse
    model, in the uint32 wrap domain (int32 in, int32 out)."""
    for b in REF.family(name):
        for rows, ws in _chunks(b):
            vals, counts = b.values[rows], b.counts[rows]
            k, nw, words = codec.rice_encode(vals, counts, words_stride=ws)
            out = codec.rice_decode(words, nw, k, counts, out_stride=vals.shape[1])
            parsed, bits = XR.parse_batch([(int(k[j]), words[j, :nw[j]]) for j in range(len(rows))], counts)
            want = np.where(_defined(counts, vals.shape[1]), vals, 0)
            assert np.array_equal(out[:, :vals.shape[1]], want), name      # zero past each count
            got = np.zeros_like(want)
            got[:, :parsed.shape[1]] = parsed
            assert np.array_equal(got, want), name
            assert np.array_equal(bits, b.enc.bits[rows]), name


@pytest.mark.parametrize("name", ["lengths", "winner", "long"])
def test_capacity_contract(name):
    """words_stride equal to the largest n_words succeeds; one word less returns SELAB200_ERR_CAPACITY with
    n_words and rice_param set for every stream, and every stream that fits has its words."""
    for b in REF.family(name):
        for rows, ws in _chunks(b):
            vals, counts = b.values[rows], b.counts[rows]
            rc, k, nw, words = _raw_encode(vals, counts, ws)
            assert rc == 0
            _check_rows(b, rows, k, nw, words, ws, name)
            small = ws - 1
            fits = b.enc.n_words[rows] <= small
            assert not fits.all()
            _fill_pool(len(rows), small, ONES)
            rc, k, nw, words = _raw_encode(vals, counts, small)
            assert rc == ERR_CAPACITY, rc
            assert np.array_equal(k, b.enc.k[rows]) and np.array_equal(nw, b.enc.n_words[rows])
            f = np.flatnonzero(fits)
            _check_rows(b, rows[f], k[f], nw[f], words[f], small, name + " after CAPACITY")
    rc, k, nw, words = _raw_encode(np.zeros((1, 4), np.int32), np.array([4]), 1)    # the library carries on
    assert rc == 0 and (k[0], nw[0], words[0, 0]) == (0, 1, 0)


def _encoder_runs():
    for name, pcm, channels in analysis_corpus.batches():
        descs, words, trace = codec.encode_trace(pcm, channels)
        yield name, channels, descs, words, trace, analysis_corpus.units(pcm, channels)


def test_batch_encoder_streams_equal_model():
    """Every subframe the batch encoder emits for the analysis corpus (mono, stereo with its 17-bit difference
    unit, 3 and 8 channels): its reflection stream equals the model's encode(q[:order]) of the analysis unit it
    came from -- the reflection streams are the encoder's only streams of n = order values -- and its residue
    stream the model's encode of the unit's FIR residues."""
    seen_orders, seen_diff = set(), False
    for name, channels, descs, words, trace, units in _encoder_runs():
        n_frames = len(descs) // channels
        f, c = np.divmod(np.arange(len(descs)), channels)
        if channels == 2:
            unit = 3 * f + np.where(c == 0, 0, np.where(descs["subframe_type"] == 1, 2, 1))
            seen_diff |= bool((descs["subframe_type"] == 1).any())
        else:
            unit = f * channels + c
        assert unit.max() < len(trace) and len(descs) == n_frames * channels
        order = trace["order"][unit].astype(np.int64)
        assert np.array_equal(descs["lpc_order"], order), name
        seen_orders |= set(order.tolist())
        refl = XR.encode_batch(trace["q"][unit], order)
        res = XR.encode_batch(fir_residues(units[unit], trace["c"][unit], order))
        for field, e in (("refl", refl), ("res", res)):
            assert np.array_equal(descs[field + "_rice_param"], e.k), (name, field)
            assert np.array_equal(descs[field + "_words"], e.n_words), (name, field)
            for i, d in enumerate(descs):
                at = int(d[field + "_offset"])
                assert np.array_equal(words[at:at + int(e.n_words[i])], e.words[i]), (name, field, i)
    assert seen_diff and len(seen_orders) >= 20, (seen_diff, sorted(seen_orders))
