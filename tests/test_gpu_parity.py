"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle, bit for bit.
Run on the H100:  python -m pytest tests -m gpu -x -q
"""
import numpy as np
import pytest

import exact_rice as XR
import oracle_lib as ol
import signals
import sela_b200
from sela_b200 import synth

pytestmark = pytest.mark.gpu

FRAME = 2048


@pytest.fixture(scope="module")
def O():
    return ol.best()


def test_device_selftest_scaling():
    import ctypes as C
    from sela_b200 import _lib
    _lib.init(0)
    bad = C.c_uint32(123)
    _lib.check(_lib.lib().selab200_selftest(C.addressof(bad)))
    assert bad.value == 0


def test_lpc_residues_families(O):
    fam = signals.families()
    names = sorted(fam)
    x = np.stack([fam[n] for n in names])
    order, q, res = sela_b200.lpc_residues(x)
    for i, n in enumerate(names):
        a = O.lpc_analyse(x[i])
        assert order[i] == a["order"], (n, order[i], a["order"])
        assert np.array_equal(q[i, :a["order"]], a["q"]), n
        assert not q[i, a["order"]:].any(), n
        assert np.array_equal(res[i], a["res"]), n


def test_lpc_residues_random(O):
    x = signals.random_frames(192, seed=21)
    order, q, res = sela_b200.lpc_residues(x)
    for i in range(x.shape[0]):
        a = O.lpc_analyse(x[i])
        assert order[i] == a["order"], i
        assert np.array_equal(q[i, :a["order"]], a["q"]), i
        assert np.array_equal(res[i], a["res"]), i


def test_lpc_residues_dc_levels(O):
    """x - mean is rounding noise on constant frames: summation order decides q[0] (SURVEY 7.3-H1)."""
    levels = np.array(list(range(-32768, 32768, 131)) + [-1, 1, 32767], np.int32)
    x = np.repeat(levels[:, None], FRAME, axis=1)
    order, q, res = sela_b200.lpc_residues(x)
    for i, lv in enumerate(levels):
        a = O.lpc_analyse(x[i])
        assert (order[i], list(q[i, :a["order"]])) == (a["order"], list(a["q"])), lv
        assert np.array_equal(res[i], a["res"]), lv


def test_lpc_difference_domain(O):
    """17-bit inputs (L-R of two 16-bit channels)."""
    rng = np.random.default_rng(3)
    a = rng.integers(-32768, 32768, (16, FRAME))
    b = rng.integers(-32768, 32768, (16, FRAME))
    x = (a - b).astype(np.int32)
    x[0] = 65535
    x[1] = -65535
    order, q, res = sela_b200.lpc_residues(x)
    for i in range(x.shape[0]):
        r = O.lpc_analyse(x[i])
        assert order[i] == r["order"] and np.array_equal(q[i, :r["order"]], r["q"])
        assert np.array_equal(res[i], r["res"])


def test_lpc_samples_roundtrip_and_oracle(O):
    x = np.concatenate([np.stack(list(signals.families().values())), signals.random_frames(64, seed=5)])
    order, q, res = sela_b200.lpc_residues(x)
    back = sela_b200.lpc_samples(res, order, q)
    lossless = 0
    for i in range(x.shape[0]):
        # the reference decoder is the contract: encoder rounds (c+P)>>35, decoder -((c-P)>>35),
        # which differ when P mod 2^35 == 2^34 (SURVEY.md 7.3-H5i) -- e.g. the sparse-spike frame here
        want = O.lpc_synthesise(res[i], int(order[i]), q[i, :order[i]])
        assert np.array_equal(back[i], want), i
        lossless += bool(np.array_equal(want, x[i]))
    assert lossless >= x.shape[0] - 2
    # arbitrary (not encoder-produced) residues/coefficients against the oracle's synthesiser
    rng = np.random.default_rng(9)
    n = 48
    res2 = rng.integers(-300, 300, (n, FRAME)).astype(np.int32)
    order2 = rng.integers(0, 101, n).astype(np.uint8)
    order2[:4] = [0, 1, 2, 100]
    q2 = rng.integers(-20, 20, (n, 100)).astype(np.int32)
    q2[:, 0] = rng.integers(-64, 64, n)
    q2[:, 1] = rng.integers(-64, 64, n)
    got = sela_b200.lpc_samples(res2, order2, q2)
    for i in range(n):
        want = O.lpc_synthesise(res2[i], int(order2[i]), q2[i, :order2[i]])
        assert np.array_equal(got[i], want), (i, order2[i])


def test_rice_encode_decode(O):
    rng = np.random.default_rng(13)
    cases = []
    for n, scale in [(100, 400), (1, 5), (2048, 3), (2048, 70000), (333, 1 << 20), (17, 0), (2048, 1),
                     (2047, 900), (31, 100000), (64, 12), (2048, 1 << 17)]:
        cases.append(rng.integers(-scale, scale + 1, n).astype(np.int32))
    cases.append((200 + rng.integers(0, 201, 100)).astype(np.int32))      # test/ricetests.cpp:11-13
    spike = np.zeros(2048, np.int32); spike[5] = 1 << 22; spike[1999] = -(1 << 21)   # long unary runs
    cases.append(spike)
    stride = 2048
    vals = np.zeros((len(cases), stride), np.int32)
    counts = np.array([c.size for c in cases], np.uint32)
    for i, c in enumerate(cases):
        vals[i, :c.size] = c
    k, nw, words = sela_b200.rice_encode(vals, counts, words_stride=8192)
    for i, c in enumerate(cases):
        ko, wo = O.rice_encode(c)
        assert k[i] == ko, (i, k[i], ko)
        assert nw[i] == wo.size, (i, nw[i], wo.size)
        assert np.array_equal(words[i, :nw[i]], wo), i
    out = sela_b200.rice_decode(words, nw, k, counts, out_stride=stride)
    for i, c in enumerate(cases):
        assert np.array_equal(out[i, :c.size], c), i


KAT = {
    "sine_deg": (17, 4, 3, 7, 552, 0xFF6EFF00, 0x00000010, 0x0BC50C3B, 0xFAF0DFE3),
    "zeros": (1, 0, 1, 0, 64, 0, 0, 0x4B95F515, 0xE6A1D1C5),
    "dc_1234": (1, 6, 1, 10, 832, 0xCC9664B3, 0x25992CC9, 0x1DAF5698, 0xFF0C5DC5),
    "cosine_deg": (16, 4, 3, 7, 585, 0xFFFFFFFF, 0x00000019, 0x4F1CBBE0, 0x10A3227D),
    "impulse0": (1, 5, 1, 4, 448, 0xFFFFFFFF, 0x00000000, 0xBD7CAAD0, 0x266C2942),
}


@pytest.mark.parametrize("name", sorted(KAT))
def test_kat_mono_frame(name):
    """SURVEY.md 8(a) known answers, through the batch encoder on a 1-frame mono input (config 1)."""
    s = signals.families()[name].astype(np.int16)
    descs, words = sela_b200.encode_frames(s, 1)
    d = descs[0]
    wq = words[d["refl_offset"]:d["refl_offset"] + d["refl_words"]]
    wr = words[d["res_offset"]:d["res_offset"] + d["res_words"]]
    got = (d["lpc_order"], d["refl_rice_param"], d["refl_words"], d["res_rice_param"], d["res_words"],
           int(wr[0]), int(wr[-1]), ol.fnv1a32(wq), ol.fnv1a32(wr))
    assert got == KAT[name]
    assert np.array_equal(sela_b200.decode_frames(descs, words, 1), s)


def _stereo_mix(n_frames, seed):
    pcm = synth.sine_noise(44100, 2, n_frames=n_frames, seed=seed)
    f = FRAME
    if n_frames >= 8:
        pcm[f * 3:f * 6, 1] = pcm[f * 3:f * 6, 0] - (pcm[f * 3:f * 6, 1] >> 6)  # near-identical -> diff wins
        pcm[f * 6:f * 7, 1] = pcm[f * 6:f * 7, 0]                                  # identical -> zero diff
        pcm[f * 7:f * 8, :] = 0                                                     # digital silence
    return pcm


# every channel count the ABI admits (1..SELAB200_MAX_CHANNELS): k_encode_units stages a channel of an
# N-channel frame at a stride of N samples
@pytest.mark.parametrize("channels,n_frames", [(1, 9), (2, 24), (3, 5), (8, 4)] +
                         [(c, 3) for c in range(4, 17) if c != 8])
def test_frames_encode_bit_exact_and_roundtrip(O, channels, n_frames):
    pcm = _stereo_mix(n_frames, 3) if channels == 2 else synth.sine_noise(48000, channels, n_frames=n_frames, seed=2)
    d_ref, w_ref = O.encode_frames(pcm, channels)
    d, w = sela_b200.encode_frames(pcm, channels)
    assert d.tobytes() == d_ref.tobytes()
    assert np.array_equal(w, w_ref)
    if channels == 2:
        assert set(d["subframe_type"]) == {0, 1}
    out = sela_b200.decode_frames(d_ref, w_ref, channels)
    assert np.array_equal(out, pcm.reshape(-1))
    assert np.array_equal(out, O.decode_frames(d_ref, w_ref, channels))


def test_frames_edge_signals_stereo(O):
    fam = signals.families()
    names = sorted(fam)
    rng = np.random.default_rng(1)
    frames = []
    for i, n in enumerate(names):
        other = fam[names[(i * 7 + 3) % len(names)]]
        frames.append(np.stack([fam[n], other], axis=1))
    frames.append(np.stack([fam["white_full"], -fam["white_full"] - 1], axis=1))     # inverted channel
    pcm = np.concatenate(frames).astype(np.int16)
    d_ref, w_ref = O.encode_frames(pcm, 2)
    d, w = sela_b200.encode_frames(pcm, 2)
    assert d.tobytes() == d_ref.tobytes()
    assert np.array_equal(w, w_ref)
    assert np.array_equal(sela_b200.decode_frames(d, w, 2), pcm.reshape(-1))


def _malformed_base(O):
    """Two stereo frames whose fields sit at the limits the decoder accepts: an order-100 subframe, a difference
    subframe, an order-0 subframe with a k = 31 residue stream of random bits and an order-1 subframe with a k = 31
    reflection stream."""
    import crafted as CR
    import rice_families as RF
    P = ol.load("port")
    rng = np.random.default_rng(12)
    a = CR.crafted_subframe(P, rng, 100, "small", channel=1)
    b = CR.difference_subframe(P, rng, 2, a, channel=0)
    d = CR.crafted_subframe(P, rng, 1, "small", channel=1)
    refl = lambda s, k: (k, XR.pack_stream(XR.zigzag(s.q), k))
    k31 = next(s for s in RF.family("random") if s[0] == 31)
    subs = [dict(channel=1, order=100, refl=refl(a, 6), res=CR.rice_code(P, a.res)),
            dict(channel=0, type=1, parent=1, order=2, refl=refl(b, 3), res=CR.rice_code(P, b.res)),
            dict(channel=0, order=0, refl=(0, np.zeros(0, np.uint32)), res=k31),
            dict(channel=1, order=1, refl=refl(d, 31), res=CR.rice_code(P, d.res))]
    return RF.layout(subs, 2)


def _to_end(descs, words, i, name, cut=0):
    """Stream `name` of subframe i moved to the end of the arena (offset + words == n_words), minus `cut` words."""
    d, w = descs.copy(), words
    at, n = int(d[name + "_offset"][i]), int(d[name + "_words"][i])
    w = np.concatenate([w, np.full(2, 0xFFFFFFFF, np.uint32), w[at:at + n]])
    d[name + "_offset"][i] = w.size - n
    return d, w[:w.size - cut]


def _edit(**fields):
    def f(d, w):
        d = d.copy()
        for key, (i, v) in fields.items():
            d[key][i] = v
        return d, w
    return f


MALFORMED = [
    ("at the limits", _edit()),
    ("order 101", _edit(lpc_order=(0, 101))),
    ("residue k 32", _edit(res_rice_param=(2, 32))),
    ("residue k 40", _edit(res_rice_param=(1, 40))),
    ("reflection k 32", _edit(refl_rice_param=(3, 32))),
    ("residue at the arena's end", lambda d, w: _to_end(d, w, 2, "res")),
    ("residue one word past it", lambda d, w: _to_end(d, w, 2, "res", 1)),
    ("reflection at the arena's end", lambda d, w: _to_end(d, w, 0, "refl")),
    ("reflection one word past it", lambda d, w: _to_end(d, w, 0, "refl", 1)),
    ("channel = channels", _edit(channel=(2, 2))),
    ("channel 7", _edit(channel=(1, 7))),
    ("parent = channels", _edit(parent_channel=(1, 2))),
    ("duplicate channel", _edit(channel=(3, 0))),
    ("difference of a difference", _edit(subframe_type=(0, 1), parent_channel=(0, 0))),
    ("difference of itself", _edit(parent_channel=(1, 0))),
    ("subframe type 2", _edit(subframe_type=(2, 2))),
    ("samples 2047", _edit(samples=(0, 2047))),
    ("samples 100", _edit(samples=(1, 100))),
    ("residue offset 2^40", _edit(res_offset=(1, 1 << 40))),
    ("residue offset 2^64 - 1", _edit(res_offset=(2, (1 << 64) - 1))),
    ("residue offset 2^64 - words", lambda d, w: _edit(res_offset=(2, (1 << 64) - int(d["res_words"][2])))(d, w)),
    ("reflection offset 2^64 - words",
     lambda d, w: _edit(refl_offset=(0, (1 << 64) - int(d["refl_words"][0])))(d, w)),
    ("truncated arena", lambda d, w: (d, w[:w.size // 2])),
]


def test_decode_rejects_malformed(O):
    """Every descriptor rule at its limit and one past it, and offsets that wrap in 64 bits, through decode_frames,
    verify_frames, decode_frames_device and rice_decode_frames_device: the exact model's acceptance predicate
    (tests/exact_rice.py) decides between the reference's output and SELAB200_ERR_BITSTREAM."""
    base = _malformed_base(O)
    for case, edit in MALFORMED:
        _check_malformed(O, case, *edit(*base))


def _check_malformed(O, case, descs, words):
    import exact_rice as XR
    from gpu_calls import decode_frames_device
    from sela_b200.device import rice_decode_frames
    if XR.accepts(descs, words, 2):
        want = O.decode_frames(descs, words, 2)
        assert np.array_equal(sela_b200.decode_frames(descs, words, 2), want), case
        assert sela_b200.verify_frames(descs, words, 2, want).size == 0, case
        assert np.array_equal(decode_frames_device(descs, words, 2), want), case
    else:
        assert case != "at the limits"
        for call in (lambda: sela_b200.decode_frames(descs, words, 2),
                     lambda: sela_b200.verify_frames(descs, words, 2, np.zeros(descs.size * FRAME, np.int16)),
                     lambda: decode_frames_device(descs, words, 2)):
            with pytest.raises(sela_b200.SelaB200Error) as e:
                call()
            assert e.value.status == -6, case
    if XR.accepts(descs, words, 2, frames=False):
        res, _ = rice_decode_frames(descs, words, 2)
        want, _ = XR.parse_batch([(int(d["res_rice_param"]), words[int(d["res_offset"]):][:int(d["res_words"])])
                                  for d in descs], FRAME)
        assert np.array_equal(res, want), case
    else:
        with pytest.raises(sela_b200.SelaB200Error) as e:
            rice_decode_frames(descs, words, 2)
        assert e.value.status == -6, case


def test_encode_capacity_error():
    pcm = synth.sine_noise(44100, 2, n_frames=4, seed=4)
    with pytest.raises(sela_b200.SelaB200Error) as e:
        sela_b200.encode_frames(pcm, 2, words_capacity=100)
    assert e.value.status == -4
    d, w = sela_b200.encode_frames(pcm, 2)       # and the library still works afterwards
    assert np.array_equal(sela_b200.decode_frames(d, w, 2), pcm.reshape(-1))


def test_empty_batch():
    d, w = sela_b200.encode_frames(np.zeros(0, np.int16), 2)
    assert d.size == 0 and w.size == 0
    assert sela_b200.decode_frames(d, w, 2).size == 0


def test_large_batch_properties(O):
    """BASELINE config-2/3 shape at reduced length (60 s): oracle equality on a sampled subset of
    frames, plus the size-independent properties on everything: exact round trip and
    offsets forming a gap-free prefix sum."""
    pcm = synth.sine_noise(44100, 2, seconds=60, seed=1)
    n_frames = pcm.shape[0] // FRAME
    d, w = sela_b200.encode_frames(pcm, 2)
    sizes = d["refl_words"].astype(np.int64) + d["res_words"]
    assert np.array_equal(d["refl_offset"], np.concatenate([[0], np.cumsum(sizes)[:-1]]))
    assert np.array_equal(d["res_offset"], d["refl_offset"] + d["refl_words"])
    assert w.size == sizes.sum()
    assert np.array_equal(sela_b200.decode_frames(d, w, 2), pcm.reshape(-1))
    pick = np.linspace(0, n_frames - 1, 40).astype(int)
    for f in pick:
        dr, wr = O.encode_frames(pcm[f * FRAME:(f + 1) * FRAME], 2, threads=1)
        for c in range(2):
            a, b = d[2 * f + c], dr[c]
            for name in ("channel", "subframe_type", "parent_channel", "refl_rice_param", "refl_words",
                         "lpc_order", "res_rice_param", "res_words", "samples"):
                assert a[name] == b[name], (f, c, name)
            n = int(sizes[2 * f + c])
            o1, o2 = int(a["refl_offset"]), int(b["refl_offset"])
            assert np.array_equal(w[o1:o1 + n], wr[o2:o2 + n]), (f, c)


def test_pipelined_chunks_match_single_shot(O, monkeypatch):
    """The host-buffer calls stream big batches in chunks (arena fill level chained through the
    scan kernel).  Force many tiny chunks and compare with the oracle."""
    pcm = _stereo_mix(23, 8)
    d_ref, w_ref = O.encode_frames(pcm, 2)
    for cf in ("1", "3", "7"):
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", cf)
        d, w = sela_b200.encode_frames(pcm, 2)
        assert d.tobytes() == d_ref.tobytes() and np.array_equal(w, w_ref), cf
        assert np.array_equal(sela_b200.decode_frames(d, w, 2), pcm.reshape(-1)), cf
    monkeypatch.delenv("SELAB200_CHUNK_FRAMES")


def test_decode_descriptors_in_arbitrary_arena_order(O):
    """Descriptors need not reference the arena in file order: permute the per-subframe word
    blocks and decode through the chunked path."""
    pcm = synth.sine_noise(44100, 2, n_frames=12, seed=6)
    d, w = O.encode_frames(pcm, 2)
    rng = np.random.default_rng(0)
    order = rng.permutation(d.size)
    d2 = d.copy()
    parts, cursor = [], 0
    for idx in order:
        a, n1, b, n2 = int(d["refl_offset"][idx]), int(d["refl_words"][idx]), int(d["res_offset"][idx]), int(d["res_words"][idx])
        parts.append(w[b:b + n2]); d2["res_offset"][idx] = cursor; cursor += n2      # residues first, for a change
        parts.append(w[a:a + n1]); d2["refl_offset"][idx] = cursor; cursor += n1
    w2 = np.concatenate(parts)
    import os
    os.environ["SELAB200_CHUNK_FRAMES"] = "4"
    try:
        assert np.array_equal(sela_b200.decode_frames(d2, w2, 2), pcm.reshape(-1))
    finally:
        del os.environ["SELAB200_CHUNK_FRAMES"]


def test_difference_coding_outside_stereo(O):
    """The reference DEcoder accepts difference-coded subframes at any channel count
    (src/frame/frame_decoder.cpp:40-69) although its encoder only emits them for stereo.  Build a
    3-channel frame whose channel 2 is coded as channel0 - channel2 and check against the oracle."""
    pcm = synth.sine_noise(32000, 3, n_frames=3, seed=12).astype(np.int32)
    pcm[:, 2] = pcm[:, 0] - (pcm[:, 2] >> 4)
    pcm = np.clip(pcm, -32768, 32767).astype(np.int16)
    d, w = O.encode_frames(pcm, 3)
    descs, parts, cursor = d.copy(), [], 0
    for f in range(3):
        frame = pcm[f * FRAME:(f + 1) * FRAME].astype(np.int32)
        for c in range(3):
            i = 3 * f + c
            if c == 2:
                a = O.lpc_analyse(frame[:, 0] - frame[:, 2])
                kq, wq = O.rice_encode(a["q"]); kr, wr = O.rice_encode(a["res"])
                descs[i]["subframe_type"], descs[i]["parent_channel"] = 1, 0
                descs[i]["refl_rice_param"], descs[i]["refl_words"], descs[i]["lpc_order"] = kq, wq.size, a["order"]
                descs[i]["res_rice_param"], descs[i]["res_words"] = kr, wr.size
            else:
                wq = w[int(d[i]["refl_offset"]):int(d[i]["refl_offset"]) + int(d[i]["refl_words"])]
                wr = w[int(d[i]["res_offset"]):int(d[i]["res_offset"]) + int(d[i]["res_words"])]
            descs[i]["refl_offset"] = cursor; parts.append(wq); cursor += wq.size
            descs[i]["res_offset"] = cursor; parts.append(wr); cursor += wr.size
    words = np.concatenate(parts)
    want = O.decode_frames(descs, words, 3)
    assert np.array_equal(want, pcm.reshape(-1))
    assert np.array_equal(sela_b200.decode_frames(descs, words, 3), want)


def test_rice_streams_with_long_unary_runs_and_k_extremes(O):
    rng = np.random.default_rng(77)
    cases = [np.full(64, 1 << 19, np.int32), np.full(2048, -1, np.int32),
             (rng.integers(0, 2, 2048) * (1 << 18)).astype(np.int32),
             rng.integers(-(1 << 23), 1 << 23, 2048).astype(np.int32)]
    vals = np.zeros((len(cases), 2048), np.int32)
    counts = np.array([c.size for c in cases], np.uint32)
    for i, c in enumerate(cases):
        vals[i, :c.size] = c
    k, nw, words = sela_b200.rice_encode(vals, counts, words_stride=40000)
    for i, c in enumerate(cases):
        ko, wo = O.rice_encode(c)
        assert (k[i], nw[i]) == (ko, wo.size), i
        assert np.array_equal(words[i, :nw[i]], wo), i
    out = sela_b200.rice_decode(words, nw, k, counts, out_stride=2048)
    for i, c in enumerate(cases):
        assert np.array_equal(out[i, :c.size], c), i


def test_full_baseline_config2_config3_bit_exact(O):
    """BASELINE configs[1]/[2] at FULL size (44.1 kHz stereo, 10 min, 12 919 frames): the whole
    descriptor table and word arena against the CPU coder, then decode and compare with both the
    CPU decoder's output and the source."""
    pcm = synth.sine_noise(44100, 2, seconds=600, seed=1)
    d, w = sela_b200.encode_frames(pcm, 2)
    d_ref, w_ref = O.encode_frames(pcm, 2)
    assert d.shape == d_ref.shape == (12919 * 2,)
    assert d.tobytes() == d_ref.tobytes()
    assert np.array_equal(w, w_ref)
    out = sela_b200.decode_frames(d, w, 2)
    assert np.array_equal(out, pcm.reshape(-1))
    assert np.array_equal(out, O.decode_frames(d_ref, w_ref, 2))


def test_config4_shape_bit_exact(O):
    """BASELINE configs[3] shape (48 kHz, 8 channels), two minutes of it."""
    pcm = synth.sine_noise(48000, 8, seconds=120, seed=2)
    d, w = sela_b200.encode_frames(pcm, 8)
    d_ref, w_ref = O.encode_frames(pcm, 8)
    assert d.tobytes() == d_ref.tobytes() and np.array_equal(w, w_ref)
    assert not d["subframe_type"].any()          # more than two channels: no difference coding
    assert np.array_equal(sela_b200.decode_frames(d, w, 8), pcm.reshape(-1))


def test_rice_decode_window_boundaries_for_every_k(O):
    """The parser's fast path takes a symbol that fits one 32-bit window (ones + 1 + k <= 32) and hands
    anything longer to the general parser: walk the boundary for every k, at every bit alignment, with
    runs of exactly 31/32/33/63/64/65 ones, against the reference's decoder."""
    rng = np.random.default_rng(5)
    rows = []
    for k in (0, 1, 2, 5, 11, 12, 19, 20, 24, 30, 31):
        edge = [0, 1, max(31 - k - 1, 0), 31 - k, 32 - k, 33 - k if k < 33 else 0, 31, 32, 33, 63, 64, 65, 100]
        qs = []
        for shift in range(0, 37, 3):                      # slide the boundary cases through the bit alignments
            qs += [1] * (shift % 5) + [q for q in edge if q >= 0]
        qs += [int(v) for v in rng.integers(0, 6, 300)]    # ordinary symbols behind them
        us = []
        for q in qs:
            q = min(q, (0xffffffff >> k)) if k else q      # keep (q << k) inside 32 bits: the value itself is tested elsewhere
            us.append((q << k) | int(rng.integers(0, 1 << k)) if k else q)
        rows.append((k, us, XR.pack_stream(us, k)))       # the model's packer at a k the search never picks
    stride = max(r[2].size for r in rows)
    words = np.zeros((len(rows), stride), np.uint32)
    for i, (_, _, w) in enumerate(rows):
        words[i, :w.size] = w
    ks = np.array([r[0] for r in rows], np.uint32)
    counts = np.array([len(r[1]) for r in rows], np.uint32)
    nw = np.array([r[2].size for r in rows], np.uint32)
    out = sela_b200.rice_decode(words, nw, ks, counts, out_stride=int(counts.max()))
    for i, (k, us, w) in enumerate(rows):
        ref = O.rice_decode(w, k, len(us))
        assert np.array_equal(out[i, :len(us)], ref), k
        want = np.array([(u >> 1) ^ -(u & 1) for u in us], np.int64).astype(np.int32)
        assert np.array_equal(ref, want), k            # and the reference agrees with the textbook inverse


def test_adversarial_frames_fit_their_slots(O):
    """The batch encoder packs every analysis unit into a private 1 600-word slot (1 568 for the residues, 24.5
    bits per sample) and refuses a frame that does not fit, where data::SelaSubFrame would carry up to 65 535
    words (src/include/data/sela_sub_frame.hpp:30-44).  16-bit audio cannot get there: with k = 19 a stream costs
    20 bits per sample plus (u >> 19), so 1 568 words need residues beyond 2^21, and a predictor fitted to the
    frame itself does not amplify a 17-bit signal sixteen-fold.  Worst cases -- full-scale alternation, anti-
    correlated stereo noise (17-bit difference), sign-flipping noise, chirps through the band edge, isolated
    full-scale impulses -- must encode, equal the reference, and stay far inside the slot."""
    rng = np.random.default_rng(99)
    n = 2048
    t = np.arange(n)
    mono = {
        "alternate_full": np.where(t % 2 == 0, 32767, -32768),
        "alternate_pairs": np.where((t // 2) % 2 == 0, 32767, -32768),
        "noise_full": rng.integers(-32768, 32768, n),
        "sign_noise": rng.choice([-32768, 32767], n),
        "chirp": np.round(32767 * np.sin(np.pi * t * t / (2.0 * n))).astype(np.int64),
        "chirp_clipped": np.clip(np.round(60000 * np.sin(np.pi * t * t / (1.3 * n))), -32768, 32767).astype(np.int64),
        "impulses": np.where(t % 257 == 0, 32767, 0) - np.where(t % 263 == 1, 32768, 0),
        "step_train": np.where((t // 101) % 2 == 0, 32767, -32768),
        "near_unstable": np.round(32767 * np.cos(np.pi * t * 0.999)).astype(np.int64),
    }
    frames = []
    for name, a in mono.items():
        a = np.asarray(a, np.int64).astype(np.int16)
        frames.append(np.stack([a, a], axis=1))                                  # identical channels
        frames.append(np.stack([a, (-a.astype(np.int32) - 1).clip(-32768, 32767).astype(np.int16)], axis=1))  # inverted: a 17-bit difference
        frames.append(np.stack([a, rng.integers(-32768, 32768, n).astype(np.int16)], axis=1))
    x = rng.integers(-32768, 32768, n).astype(np.int16)
    frames.append(np.stack([x, (~x)], axis=1))                                   # anti-correlated full-scale noise
    pcm = np.concatenate(frames).astype(np.int16)
    d, w = sela_b200.encode_frames(pcm, 2)
    d_ref, w_ref = O.encode_frames(pcm, 2)
    assert d.tobytes() == d_ref.tobytes() and np.array_equal(w, w_ref)
    assert int(d["res_words"].max()) <= 1344, int(d["res_words"].max())         # 21 bits per sample: k = 19 and one more bit
    assert int(d["refl_words"].max()) <= 29
    assert np.array_equal(sela_b200.decode_frames(d, w, 2), O.decode_frames(d_ref, w_ref, 2))
    for ch in (1, 3):                                                            # the non-stereo staging path
        m = np.concatenate([np.asarray(a, np.int64).astype(np.int16) for a in mono.values()])
        m = m[: (m.size // (n * ch)) * n * ch].reshape(-1, ch)
        dm, wm = sela_b200.encode_frames(m, ch)
        dr, wr = O.encode_frames(m, ch)
        assert dm.tobytes() == dr.tobytes() and np.array_equal(wm, wr)
        assert int(dm["res_words"].max()) <= 1344


def test_order_zero_subframe_at_any_word_offset(O):
    """A subframe with no coefficient words (order 0, zero reflection words) decodes as a zero predictor in the
    reference; the decoder must not call that an overrun, whatever 16-byte phase its (empty) stream sits at."""
    rng = np.random.default_rng(3)
    res = np.round(rng.laplace(0, 40, FRAME)).astype(np.int32)
    k, nw, words = sela_b200.rice_encode(res[None, :], np.array([FRAME], np.uint32), words_stride=2048)
    body = words[0, :nw[0]]
    for pad in range(5):
        arena = np.concatenate([np.full(pad, 0xFFFFFFFF, np.uint32), body])
        d = np.zeros(1, _lib_desc())
        d["lpc_order"] = 0
        d["refl_words"] = 0
        d["refl_offset"] = pad
        d["res_rice_param"] = k[0]
        d["res_words"] = nw[0]
        d["samples"] = FRAME
        d["res_offset"] = pad
        out = sela_b200.decode_frames(d, arena, 1)
        assert np.array_equal(out, res.astype(np.int16)), pad                    # zero predictor: samples = residues


def _lib_desc():
    from sela_b200 import _lib
    return _lib.DESC_DTYPE
