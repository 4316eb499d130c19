"""The exact Rice parse model (tests/exact_rice.py) and the stream families (tests/rice_families.py) against the
CPU oracle and the compiled reference (marker `ref`).  CPU only: this pins the yardstick the GPU Rice tests
(tests/test_rice_exact.py) measure the kernels with."""
import numpy as np
import pytest

import exact_rice as XR
import oracle_lib as ol
import rice_encode_families as REF
import rice_families as RF
from exact_rice import pack_stream

FRAME = 2048
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
WHICH = ["port", pytest.param("ref", marks=pytest.mark.ref)]


@pytest.fixture(scope="module")
def in_bounds():
    """A sample of every family but `short`, each stream with the bits its parse needs."""
    out = []
    for name in ("random", "trailing", "runs", "wrap", "long", "periodic"):
        s = RF.family(name)
        out += s[::max(1, len(s) // 48)]
    return out


@pytest.mark.parametrize("which", WHICH)
def test_model_equals_reference_decoder(in_bounds, which):
    O = ol.load(which)
    values, bits = XR.parse_batch(in_bounds, FRAME)
    for i, (k, w) in enumerate(in_bounds):
        assert bits[i] <= 32 * w.size, (i, k)
        assert np.array_equal(values[i], O.rice_decode(w, k, FRAME)), (i, k)


def test_model_zero_extends_like_the_padded_port():
    """Streams cut one word short: the port reads the zero words its wrapper puts behind them (the reference's
    own decoder would read past its vector)."""
    O = ol.load("port")
    rng = np.random.default_rng(5)
    for k in (0, 1, 7, 19, 31):
        us = rng.integers(0, 1 << min(k + 3, 32), FRAME, dtype=np.uint64)
        w = pack_stream(us, k)[:-1]
        v, bits = XR.parse(w, w.size, k, FRAME)
        assert bits > 32 * w.size
        assert np.array_equal(v, O.rice_decode(w, k, FRAME)), k


def test_model_inverts_pack_stream():
    rng = np.random.default_rng(1)
    cases = []
    for k in range(32):
        us = rng.integers(0, 1 << min(k + 9, 32), FRAME, dtype=np.uint64)
        us[:4] = [0, (1 << 32) - 1, (1 << 31) - 1, 1 << 31]                 # the int32 extremes
        us[:4] &= np.uint64((1 << min(k + 9, 32)) - 1)
        cases.append((k, us, pack_stream(us, k)))
    # each stream as it is, and with trailing words behind it
    streams = [(k, w) for k, _, w in cases] + [(k, np.concatenate([w, np.full(3, 0xFFFFFFFF, np.uint32)]))
                                                for k, _, w in cases]
    values, bits = XR.parse_batch(streams, FRAME)
    for i, (k, us, w) in enumerate(cases * 2):
        assert np.array_equal(values[i], XR.unzigzag(us)), (i, k)
        assert bits[i] == XR.code_bits(us, k), (i, k)
    assert XR.parse(cases[5][2], cases[5][2].size, 5, FRAME)[1] == bits[5]


def test_model_wraps_q_shift_in_uint32():
    for k, q, pay in ((31, 2, 5), (31, 3, 0), (20, 4096, 77), (12, 1 << 20, 1), (16, (1 << 17) + 3, 0xFFFF)):
        w = RF.symbols([q, 0], [pay, 0], k)
        v, bits = XR.parse(w, w.size, k, 2)
        u = ((q << k) & 0xFFFFFFFF) | pay
        assert v[0] == XR.unzigzag(np.uint64(u)), (k, q)
        assert bits == q + 1 + k + 1 + k


def test_model_equals_synthetic_streams():
    streams = RF.synthetic_streams(np.random.default_rng(11))
    values, bits = XR.parse_batch([(k, w) for k, w, _ in streams], FRAME)
    for i, (k, w, us) in enumerate(streams):
        assert np.array_equal(values[i], XR.unzigzag(np.asarray(us, np.uint64))), (i, k)
        assert bits[i] == XR.code_bits(us, k)


def test_families_reach_what_they_claim():
    ks = lambda s: {k for k, _ in s}
    for name in ("random", "trailing", "runs", "long", "periodic", "short"):
        assert ks(RF.family(name)) == set(range(32)), name
    assert ks(RF.family("wrap")) == set(range(12, 32))
    for name in ("random", "trailing", "runs", "wrap", "long", "periodic"):
        s = RF.family(name)
        _, bits = XR.parse_batch(s, FRAME)
        words = np.array([w.size for _, w in s])
        assert (bits <= 32 * words).all(), name
        need = -(-bits // 32)
        if name in ("random", "periodic"):
            assert (need == words).all(), name
        if name == "trailing":
            assert (words > need).all() and (words == 2 * need).any()
    assert all(40000 <= w.size <= 0xFFFF for _, w in RF.family("long"))
    _, bits = XR.parse_batch(RF.family("short"), FRAME)
    assert (bits > 32 * np.array([w.size for _, w in RF.family("short")])).all()


# ------------------------------------------------------------------------------------------- encoder --

@pytest.mark.parametrize("which", WHICH)
@pytest.mark.parametrize("name", REF.NAMES)
def test_encoder_model_equals_reference_encoder(name, which):
    """(k, words) of the encoder model on every stream of every family that lies in the reference's domain
    (|x| < 2^30), against rice::RiceEncoder."""
    O = ol.load(which)
    n = 0
    for b in REF.family(name):
        for i in REF.in_reference_domain(b):
            k, w = O.rice_encode(b.values[i, :b.counts[i]])
            assert (k, w.size) == (b.enc.k[i], b.enc.n_words[i]), (name, i)
            assert np.array_equal(w, b.enc.words[i]), (name, i)
            n += 1
    assert n >= (6 if name == "extremes" else 20), n                      # extremes: the +-(2^30 - 1) streams


@pytest.mark.parametrize("name", REF.NAMES)
def test_encoder_model_round_trips(name):
    """Every family (each builder asserts its own property through the model) parses back to its values with the
    parse model, ending on the encoder's last bit; the totals are the textbook sums."""
    for b in REF.family(name):
        values, bits = XR.parse_batch(list(zip(b.enc.k, b.enc.words)), b.counts)
        for i, c in enumerate(b.counts):
            assert np.array_equal(values[i, :c], b.values[i, :c]), (name, i)
        assert np.array_equal(bits, b.enc.bits)
        assert np.array_equal(b.enc.n_words, [w.size for w in b.enc.words])
        for i in range(0, len(b.counts), 97):
            us = [int(u) for u in XR.zigzag(b.values[i, :b.counts[i]])]
            assert [sum(u >> k for u in us) + len(us) * (1 + k) for k in range(20)] == b.enc.totals[i].tolist()


def test_encoder_model_search_and_layout():
    """The first arg-min wins a tie; zig-zag in the uint32 domain; the layout, bit by bit."""
    assert XR.encode([1, 1])[0] == 0                                      # u = 2: totals 6, 6, 8, ...
    assert XR.encode([])[0] == 0 and XR.encode([])[1].size == 0
    assert XR.zigzag([0, -1, 1, I32_MIN, I32_MAX]).tolist() == [0, 1, 2, (1 << 32) - 1, (1 << 32) - 2]
    k, w = XR.encode([3, -2, 0])                                         # u = 6, 3, 0: totals 12, 10, 10, 12
    assert k == 1
    bits = "111" "0" "0" + "1" "0" "1" + "0" "0"                         # q ones, a zero, the payload bit
    assert w.tolist() == [int(bits[::-1], 2)]


def test_acceptance_predicate():
    assert XR.in_arena(0, 0, 0) and XR.in_arena(5, 5, 10) and not XR.in_arena(6, 5, 10)
    assert not XR.in_arena((1 << 64) - 3, 3, 10)                   # 2^64 - w + w wraps to 0 in uint64
    assert not XR.in_arena(0, 11, 10)
    streams = RF.family("random")[:4]
    descs, arena = RF.layout([{"res": s} for s in streams], channels=2)
    assert XR.accepts(descs, arena, 2) and XR.accepts(descs, arena, 2, frames=False)
    bad = descs.copy()
    bad["res_words"][2] -= 1                                        # one word short
    assert not XR.accepts(bad, arena, 2) and not XR.accepts(bad, arena, 2, frames=False)
    dup = descs.copy()
    dup["channel"][1] = 0                                           # a frame rule: only the frame decoders apply it
    assert not XR.accepts(dup, arena, 2) and XR.accepts(dup, arena, 2, frames=False)
    wrapped = descs.copy()
    wrapped["res_offset"][3] = (1 << 64) - int(wrapped["res_words"][3])
    assert not XR.accepts(wrapped, arena, 2) and not XR.accepts(wrapped, arena, 2, frames=False)
