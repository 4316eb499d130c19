"""Lossless encodes (selab200_encode_frames_lossless, _encode_container_lossless, the device-resident form and
`sela -L`): every subframe the reference decoder would not bring back to its source is re-coded with a tie-free
predictor, inside the format (DESIGN.md 7.2).

The expected output comes from the CPU model in exact_lossless.py, built on the plain-C port
(oracle/liboracle.so): the tie criterion in NumPy (int64 wrap), and the repair rule -- candidates, rounds, fewest
words, first candidate on a tie -- over the port's lpc_coefficients and rice_size.  Every decode check uses the
port's decoder, and the compiled reference where it has been built.  test_lossless_repair.py drives the repair
through chosen predictors and planted ties."""
import ctypes as C
import pathlib
import subprocess

import numpy as np
import pytest

import analysis_corpus
import oracle_lib as ol
from exact_lossless import (analyse, as_tuples, check_against_model, expected_report, fir, model_batch, repair,
                            repair_edit)
from sela_b200 import _lib, synth, wavio

GOLD = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
CASES = sorted(k[4:] for k in GOLD.files if k.startswith("pcm_"))
FRAME = 2048
ROOT = pathlib.Path(__file__).resolve().parent.parent
BIN = ROOT / "sela_b200" / "host" / "bin"
REF_CLI = ROOT / "oracle" / "_ref" / "sela_ref_cli"
LOSSY = GOLD["pcm_oct_reference_lossy"].reshape(2, FRAME, 8)
L0 = LOSSY[0, :, 1].astype(np.int64)  # order 86, a tie at sample 1
L1 = LOSSY[1, :, 4].astype(np.int64)  # order 29, a tie at sample 1


def _n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


TWO_GPUS = pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")


# ------------------------------------------------------------------- CPU --

def test_criterion_flags_exactly_the_units_that_do_not_decode():
    """Every analysis-corpus unit and every golden unit: the tie test fires iff the port's decode of the port's
    encode differs from the source, and the first tie is the first wrong sample."""
    O = ol.load("port")
    gold = [analysis_corpus.units(GOLD["pcm_" + c], GOLD["pcm_" + c].shape[1]) for c in CASES]
    flagged = []
    for s in np.concatenate([analysis_corpus.all_units()] + gold):
        a = O.lpc_analyse(s.astype(np.int32))
        res, tie = fir(s, a["c"], a["order"])
        assert np.array_equal(res, a["res"])
        dec = O.lpc_synthesise(res, a["order"], a["q"])
        wrong = dec != s
        assert tie.any() == wrong.any()
        if tie.any():
            assert np.argmax(tie) == np.argmax(wrong)
            flagged.append(int(np.argmax(tie)))
    assert len(flagged) > 2 and flagged[-2:] == [1, 1]  # the corpus has lossy units too; then the two golden ones


def test_repair_model_on_the_golden_lossy_units():
    O = ol.load("port")
    for s, order, cand, edit, words in ((L0, 86, 1, (0, +1), 824), (L1, 29, 2, (1, -1), 819)):
        u = analyse(O, s)
        assert u.order == order and u.tie
        w = repair(O, u)
        assert (w.cand, w.order, w.words) == (cand, order, words)
        j, d = edit
        assert np.array_equal(w.q[:order] - u.q[:order], np.eye(order, dtype=np.int32)[j] * d)
        assert w.words < u.words
        checkers = [O] + ([ol.load("ref")] if ol.have_ref() else [])
        for D in checkers:
            assert np.array_equal(D.lpc_synthesise(w.res, w.order, w.q[:w.order]), s)


def test_candidate_numbering():
    assert [repair_edit(2, c) for c in range(5)] == [(2, 0, -1), (2, 0, 1), (2, 1, -1), (2, 1, 1), (1, 0, 0)]
    assert [repair_edit(5, c) for c in range(14)] == [
        (5, 0, -1), (5, 0, 1), (5, 1, -1), (5, 1, 1), (5, 4, -1), (5, 4, 1), (4, 0, 0),
        (5, 2, -1), (5, 2, 1), (5, 3, -1), (5, 3, 1), (3, 0, 0), (2, 0, 0), (1, 0, 0)]
    for o in range(2, 101):
        eds = [repair_edit(o, c) for c in range(3 * o - 1)]
        assert len(set(eds)) == len(eds) and eds[-1] == (1, 0, 0)


def test_lossless_entry_points_have_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = _lib.lib()
    assert L.selab200_init(0) == -1
    pcm = np.zeros(2048, np.int16)
    descs = np.zeros(1, _lib.DESC_DTYPE)
    words = np.zeros(4096, np.uint32)
    rep = np.zeros(1, _lib.LOSSLESS_DTYPE)
    n, used = C.c_size_t(0), C.c_size_t(0)
    blob = np.zeros(1 << 16, np.uint8)
    assert L.selab200_encode_frames_lossless(pcm.ctypes.data, 1, 1, descs.ctypes.data, words.ctypes.data, words.size,
                                             C.addressof(used), rep.ctypes.data, 1, C.addressof(n)) == -7
    assert L.selab200_encode_container_lossless(pcm.ctypes.data, 1, 1, 44100, 16, blob.ctypes.data, blob.size,
                                                C.addressof(used), rep.ctypes.data, 1, C.addressof(n)) == -7
    assert L.selab200_encode_frames_lossless_device(pcm.ctypes.data, 1, 1, descs.ctypes.data, words.ctypes.data,
                                                    words.size, blob.ctypes.data, rep.ctypes.data, blob.ctypes.data,
                                                    blob.ctypes.data, blob.ctypes.data, blob.size, None) == -7
    pred = np.zeros(1, _lib.PREDICTOR_DTYPE)
    assert L.selab200_encode_lossless_forced(pcm.ctypes.data, 1, 1, pred.ctypes.data, descs.ctypes.data,
                                             words.ctypes.data, words.size, C.addressof(used), rep.ctypes.data, 1,
                                             C.addressof(n)) == -7
    assert L.selab200_encode_lossless_workspace_bytes(10, 2) > L.selab200_encode_workspace_bytes(10, 2)
    assert _lib.LOSSLESS_DTYPE.itemsize == 16
    import sela_b200
    from sela_b200 import codec
    with pytest.raises(sela_b200.SelaB200Error):
        sela_b200.encode_frames_lossless(pcm, 1)
    with pytest.raises(sela_b200.SelaB200Error):
        codec.encode_lossless_forced(pcm, 1, [(1, [0])])


# ------------------------------------------------------------------- GPU --

@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if c != "oct_reference_lossy"])
def test_golden_cases_keep_the_reference_bytes(case):
    import sela_b200
    pcm = GOLD["pcm_" + case]
    ch = pcm.shape[1]
    blob, rep = sela_b200.encode_container_lossless(pcm, ch, 44100)
    assert rep.size == 0
    assert blob.tobytes() == sela_b200.encode_container(pcm, ch, 44100).tobytes()
    descs, words, rep2 = sela_b200.encode_frames_lossless(pcm, ch)
    assert rep2.size == 0
    assert descs.tobytes() == GOLD["descs_" + case].tobytes() and np.array_equal(words, GOLD["words_" + case])


@pytest.mark.gpu
def test_golden_lossy_case():
    import sela_b200
    O = ol.load("port")
    pcm = GOLD["pcm_oct_reference_lossy"]
    descs, words, rep = sela_b200.encode_frames_lossless(pcm, 8)
    model = model_batch(O, pcm, 8)
    assert sorted(model) == [0, 1]
    assert as_tuples(rep) == expected_report(model) == [(0, 1, 86, 827, 86, 824), (1, 4, 29, 820, 29, 819)]
    check_against_model(O, descs, words, pcm, 8, model)
    # every other subframe is the reference's, word for word
    gd, gw = GOLD["descs_oct_reference_lossy"].view(_lib.DESC_DTYPE), GOLD["words_oct_reference_lossy"]
    for i in range(16):
        if (i // 8, i % 8) in ((0, 1), (1, 4)):
            continue
        a, b = descs[i], gd[i]
        for fld in ("lpc_order", "refl_rice_param", "res_rice_param", "refl_words", "res_words", "subframe_type"):
            assert a[fld] == b[fld], (i, fld)
        for off, n in (("refl_offset", "refl_words"), ("res_offset", "res_words")):
            assert np.array_equal(words[int(a[off]):int(a[off]) + int(a[n])], gw[int(b[off]):int(b[off]) + int(b[n])])
    blob, rep2 = sela_b200.encode_container_lossless(pcm, 8, 48000)
    assert as_tuples(rep2) == as_tuples(rep)
    assert blob.tobytes() == wavio.pack_container(descs, words, 48000, 8)
    assert sela_b200.verify_container(blob, pcm)[1].size == 0


def _noise(n, amp, seed):
    return np.random.default_rng(seed).integers(-amp, amp + 1, n).astype(np.int64)


def _constructed(kind):
    """One frame (planar channels) built from the lossy units L0, L1."""
    if kind == "mono":
        return [L0]
    if kind == "three":
        return [_noise(FRAME, 3000, 1), L0, L1]
    if kind == "stereo_ch0":
        return [L0, _noise(FRAME, 30000, 2)]
    if kind == "stereo_ch1":  # wide noise on ch0: the difference loses, ch1 is coded on its own
        return [_noise(FRAME, 30000, 3), L0]
    if kind == "stereo_difference":  # ch0 - ch1 = L0, and the wide noise on ch1 makes the difference win
        amp = 32767 - int(np.abs(L0).max())
        x = _noise(FRAME, amp, 4)
        return [L0 + x, x]
    if kind == "stereo_both_sides":  # ch1 = L1 and ch0 - ch1 = L0: both side candidates have a tie
        return [L0 + L1, L1]
    raise ValueError(kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["mono", "three", "stereo_ch0", "stereo_ch1", "stereo_difference",
                                  "stereo_both_sides"])
def test_constructed_frames(kind):
    import sela_b200
    O = ol.load("port")
    planes = _constructed(kind)
    assert all(np.abs(p).max() <= 32767 for p in planes)
    ch = len(planes)
    pcm = np.stack(planes, axis=1).astype(np.int16)
    ref = sela_b200.encode_container(pcm, ch, 44100)
    assert sela_b200.verify_container(ref, pcm)[1].size > 0  # the reference encoding is lossy
    model = model_batch(O, pcm, ch)
    assert list(model) == [0]
    if kind == "stereo_difference":
        assert model[0][1][0][0] == 1 and model[0][0][1][1] == 1  # the re-coded difference is emitted
    if kind == "stereo_both_sides":
        units = [analyse(O, s) for s in analysis_corpus.units(pcm, 2)]
        assert units[1].tie and units[2].tie
    descs, words, rep = sela_b200.encode_frames_lossless(pcm, ch)
    assert as_tuples(rep) == expected_report(model)
    check_against_model(O, descs, words, pcm, ch, model)
    blob, rep2 = sela_b200.encode_container_lossless(pcm, ch, 44100)
    assert as_tuples(rep2) == as_tuples(rep)
    assert sela_b200.verify_container(blob, pcm)[1].size == 0


def _spliced_oct(n_frames, positions, seed=4):
    """8-channel batch with the two golden lossy frames at `positions` (frame A, B, A, ... in turn)."""
    pcm = synth.sine_noise(48000, 8, n_frames=n_frames, seed=seed).reshape(n_frames, FRAME, 8)
    for i, f in enumerate(positions):
        pcm[f] = LOSSY[i % 2]
    return pcm.reshape(-1, 8)


def _expected_spliced(positions):
    a, b = (0, 1, 86, 827, 86, 824), (1, 4, 29, 820, 29, 819)
    return sorted((f,) + (a if i % 2 == 0 else b)[1:] for i, f in enumerate(positions))


@pytest.mark.gpu
def test_spliced_lossy_frames_at_the_edges_and_a_chunk_boundary(monkeypatch):
    import sela_b200
    monkeypatch.setenv("SELAB200_CHUNK_FRAMES", "128")
    n = 1000
    pos = [0, 127, 128, n - 1]
    pcm = _spliced_oct(n, pos)
    blob, rep = sela_b200.encode_container_lossless(pcm, 8, 48000)
    assert as_tuples(rep) == _expected_spliced(pos)
    assert sela_b200.verify_container(blob, pcm)[1].size == 0
    descs, words, rep2 = sela_b200.encode_frames_lossless(pcm, 8)
    assert as_tuples(rep2) == as_tuples(rep)
    assert blob.tobytes() == wavio.pack_container(descs, words, 48000, 8)
    # every frame that was lossless already keeps the reference encoder's bytes
    d0, w0 = sela_b200.encode_frames(pcm, 8)
    keep = np.ones(n, bool)
    keep[pos] = False
    a, b = descs.reshape(n, 8), d0.reshape(n, 8)
    for fld in ("lpc_order", "refl_words", "res_words", "subframe_type"):
        assert np.array_equal(a[keep][fld], b[keep][fld])
    assert np.array_equal(sela_b200.decode_frames(descs, words, 8), pcm.reshape(-1))
    # capacity: the total always, at most `capacity` entries written
    L = _lib.lib()
    few = np.zeros(2, _lib.LOSSLESS_DTYPE)
    cnt, used = C.c_size_t(0), C.c_size_t(0)
    p16 = np.ascontiguousarray(pcm, np.int16)
    cap = L.selab200_encode_words_bound(n, 8)
    dd = np.zeros(n * 8, _lib.DESC_DTYPE)
    ww = np.zeros(cap, np.uint32)
    _lib.check(L.selab200_encode_frames_lossless(p16.ctypes.data, n, 8, dd.ctypes.data, ww.ctypes.data, cap,
                                                 C.addressof(used), few.ctypes.data, 2, C.addressof(cnt)))
    assert cnt.value == 4 and as_tuples(few) == as_tuples(rep)[:2]


@pytest.mark.gpu
def test_all_lossy_batch():
    """Every frame one of the golden lossy frames, a few thousand of them over several chunks."""
    import sela_b200
    n = 3000
    pcm = np.concatenate([LOSSY] * (n // 2)).reshape(-1, 8)
    blob, rep = sela_b200.encode_container_lossless(pcm, 8, 48000)
    assert as_tuples(rep) == _expected_spliced(list(range(n)))
    assert sela_b200.verify_container(blob, pcm)[1].size == 0


@pytest.mark.gpu
def test_device_form_equals_host_forms():
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    n = 300
    pos = [0, 150, n - 1]
    pcm = _spliced_oct(n, pos, seed=7)
    dev = torch.device("cuda", 0)
    codec = DeviceCodec(n, 8, device=0)
    t = torch.from_numpy(np.ascontiguousarray(pcm).reshape(-1)).to(dev)
    codec.encode_lossless(t)
    codec.check_status()
    rep = codec.lossless_report()
    n_words = int(codec.words_used.item())
    descs, words, rep2 = sela_b200.encode_frames_lossless(pcm, 8)
    assert as_tuples(rep) == as_tuples(rep2) == _expected_spliced(pos)
    assert codec.descs.cpu().numpy().tobytes() == descs.tobytes()
    assert np.array_equal(codec.words[:n_words].cpu().numpy().view(np.uint32), words)
    # clean input: the same as the plain encode, and an empty report
    clean = synth.sine_noise(48000, 8, n_frames=n, seed=7).reshape(-1)
    tc = torch.from_numpy(clean).to(dev)
    codec.encode_lossless(tc)
    codec.check_status()
    assert codec.lossless_report().size == 0
    d1, w1 = codec.descs.clone(), codec.words[:int(codec.words_used.item())].clone()
    codec.encode(tc)
    codec.check_status()
    assert torch.equal(d1, codec.descs) and torch.equal(w1, codec.words[:int(codec.words_used.item())])


@pytest.mark.gpu
@pytest.mark.parametrize("slots", [[0, 0], pytest.param([0, 1], marks=TWO_GPUS)], ids=["0-0", "0-1"])
def test_two_devices_give_the_same_bytes(slots):
    import sela_b200
    n = 1200
    pos = [0, 599, 600, n - 1]
    pcm = _spliced_oct(n, pos)
    blob1, rep1 = sela_b200.encode_container_lossless(pcm, 8, 48000, device=0)
    d1, w1, r1 = sela_b200.encode_frames_lossless(pcm, 8, device=0)
    blob2, rep2 = sela_b200.encode_container_lossless(pcm, 8, 48000, device=slots)
    d2, w2, r2 = sela_b200.encode_frames_lossless(pcm, 8, device=slots)
    _lib.init(0)
    assert blob1.tobytes() == blob2.tobytes()
    assert d1.tobytes() == d2.tobytes() and np.array_equal(w1, w2)
    assert as_tuples(rep1) == as_tuples(rep2) == as_tuples(r1) == as_tuples(r2) == _expected_spliced(pos)


@pytest.mark.gpu
def test_full_file():
    """The config-4-shaped 10-minute 8-channel file: exactly frames 8975 / 1 and 13577 / 4 are re-coded."""
    import sela_b200
    pcm = synth.sine_noise(48000, 8, 600, seed=2)
    blob, rep = sela_b200.encode_container_lossless(pcm, 8, 48000)
    assert [(f, c) for f, c, *_ in as_tuples(rep)] == [(8975, 1), (13577, 4)]
    n = pcm.shape[0] // FRAME
    assert sela_b200.verify_container(blob, pcm[:n * FRAME])[1].size == 0


# ------------------------------------------------------------------- CLI --

def _run(*cmd):
    return subprocess.run([str(c) for c in cmd], capture_output=True, text=True, timeout=600)


@pytest.mark.gpu
def test_cli_lossless_mode(tmp_path):
    if not (BIN / "sela").exists():
        subprocess.run(["make", "-C", str(ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    sela = BIN / "sela"
    lossy = _spliced_oct(5, [1, 3])
    clean = synth.sine_noise(44100, 2, n_frames=9, seed=2)
    wavio.write_wav(tmp_path / "lossy.wav", lossy, 48000)
    wavio.write_wav(tmp_path / "clean.wav", clean, 44100)
    for name, n_recoded in (("clean", 0), ("lossy", 2)):
        wav = tmp_path / (name + ".wav")
        p = _run(sela, "-L", wav, tmp_path / (name + ".L.sela"))
        assert p.returncode == 0, (p.stdout, p.stderr)
        assert "Re-coded %d subframes" % n_recoded in p.stdout
        assert _run(sela, "-e", wav, tmp_path / (name + ".e.sela")).returncode == 0
        written = (tmp_path / (name + ".L.sela")).read_bytes()
        assert (written == (tmp_path / (name + ".e.sela")).read_bytes()) == (n_recoded == 0)
        t = _run(sela, "-t", tmp_path / (name + ".L.sela"), wav)
        assert t.returncode == 0 and "Verified" in t.stdout, (t.stdout, t.stderr)
        if REF_CLI.exists():
            assert _run(REF_CLI, "-d", tmp_path / (name + ".L.sela"), tmp_path / (name + ".ref.wav")).returncode == 0
            _, _, pcm = wavio.read_wav_pcm(tmp_path / (name + ".ref.wav"))
            assert np.array_equal(pcm.reshape(-1), (clean if name == "clean" else lossy).reshape(-1))
    assert "-L" in _run(sela).stdout
