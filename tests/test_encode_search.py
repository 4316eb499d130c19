"""Order-search encodes (selab200_encode_frames_search, _encode_container_search, the device-resident form and
`sela -S`): every analysis unit coded at the tie-free predictor order 1..100 with the fewest words, inside the format
(DESIGN.md 7.3).

The expected output comes from the CPU model in exact_search.py (the exact analysis model's quantiser, the port's
predictors, the FIR with the tie test, Rice words, the winner rule and the stereo decision).  Its per-unit form costs
about 30 ms per unit and is used on small batches; the corpus batches are compared whole with its batched form
(about 15 ms per unit, pinned to the per-unit form in test_exact_search.py).  The 4 800-frame batch and the chunked
host forms are compared on chosen frames and checked as a whole through ref_words and decoding.  Every decode check
uses the device decoder, the port's, and the compiled reference's where it has been built."""
import ctypes as C
import pathlib
import subprocess

import numpy as np
import pytest

import analysis_corpus
import exact_lossless as xl
import exact_search as xs
import gpu_calls
import oracle_lib as ol
import signals
from sela_b200 import _lib, codec, synth, wavio

GOLD = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
FRAME = 2048
ROOT = pathlib.Path(__file__).resolve().parent.parent
BIN = ROOT / "sela_b200" / "host" / "bin"
REF_CLI = ROOT / "oracle" / "_ref" / "sela_ref_cli"


def _decoders():
    return [ol.load("port")] + ([ol.load("ref")] if ol.have_ref() else [])


def _check(pcm, ch, frames=None, preds=None, got=None, batched=False):
    """The search of batch `pcm` (host form, or `got` = (descs, words, ref_words)) against the model on `frames` (all
    by default; the batched model, which takes whole batches, with `batched`), ref_words against the default
    encoder's words, and the whole batch decoding back."""
    import sela_b200
    O = ol.load("port")
    pcm = np.asarray(pcm, np.int16).reshape(-1)
    if got is None:
        got = codec.encode_search_forced(pcm, ch, preds) if preds is not None else sela_b200.encode_frames_search(pcm, ch)
    descs, words, ref_words = got
    if batched:
        assert frames is None
        model, model_ref = xs.model_batch_all(pcm, ch, preds)[:2]
    else:
        model, model_ref = xs.model_batch(O, pcm, ch, frames=frames, preds=preds)
    xs.check_frames(O, descs, words, pcm, ch, model)
    assert np.array_equal(gpu_calls.decode_frames_device(descs, words, ch), pcm)
    if preds is None:
        d0, w0 = sela_b200.encode_frames(pcm, ch)
        assert ref_words == w0.size
        for f in model:
            fd = d0[f * ch:(f + 1) * ch]
            assert model_ref[f] == int(fd["refl_words"].sum()) + int(fd["res_words"].sum())
    elif frames is None:
        assert ref_words == sum(model_ref.values())
    return descs, words, ref_words, model


# ------------------------------------------------------------------- CPU --

def test_search_entry_points_have_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = _lib.lib()
    assert L.selab200_init(0) == -1
    pcm = np.zeros(2048, np.int16)
    descs = np.zeros(1, _lib.DESC_DTYPE)
    words = np.zeros(4096, np.uint32)
    used, ref = C.c_size_t(0), C.c_size_t(0)
    blob = np.zeros(1 << 16, np.uint8)
    assert L.selab200_encode_frames_search(pcm.ctypes.data, 1, 1, descs.ctypes.data, words.ctypes.data, words.size,
                                           C.addressof(used), C.addressof(ref)) == -7
    assert L.selab200_encode_container_search(pcm.ctypes.data, 1, 1, 44100, 16, blob.ctypes.data, blob.size,
                                              C.addressof(used), C.addressof(ref)) == -7
    assert L.selab200_encode_frames_search_device(pcm.ctypes.data, 1, 1, descs.ctypes.data, words.ctypes.data,
                                                  words.size, blob.ctypes.data, blob.ctypes.data, blob.ctypes.data,
                                                  blob.ctypes.data, blob.size, None) == -7
    pred = np.zeros(1, _lib.PREDICTOR_DTYPE)
    assert L.selab200_encode_search_forced(pcm.ctypes.data, 1, 1, pred.ctypes.data, descs.ctypes.data,
                                           words.ctypes.data, words.size, C.addressof(used), C.addressof(ref)) == -7
    assert L.selab200_encode_search_workspace_bytes(10, 2) > L.selab200_encode_workspace_bytes(10, 2)
    import sela_b200
    with pytest.raises(sela_b200.SelaB200Error):
        sela_b200.encode_frames_search(pcm, 1)


# ------------------------------------------------------------------- GPU --

@pytest.mark.gpu
@pytest.mark.parametrize("batch", [b[0] for b in analysis_corpus.batches()])
def test_corpus_batches(batch):
    """Every analysis-corpus batch whole (mono, stereo, 3 and 8 channels, every 3rd BASELINE frame), against the
    batched model."""
    _, pcm, ch = next(b for b in analysis_corpus.batches() if b[0] == batch)
    _check(pcm, ch, batched=True)


@pytest.mark.gpu
def test_families_and_random_frames():
    fam = np.stack([v for v in signals.families().values()]).astype(np.int16).reshape(-1)
    _check(fam, 1)
    descs, words, ref_words, model = _check(signals.random_frames(16, 3).astype(np.int16).reshape(-1), 1)
    assert words.size < ref_words  # the threshold order is far from the best on random frames


@pytest.mark.gpu
def test_baseline_slice():
    pcm = synth.sine_noise(44100, 2, n_frames=12, seed=1)
    descs, words, ref_words, model = _check(pcm, 2)
    assert words.size <= ref_words


@pytest.mark.gpu
def test_golden_lossy_frames_lose_their_tied_reference_order():
    """oct_reference_lossy: frame 0 channel 1 (order 86) and frame 1 channel 4 (order 29) tie at the reference order;
    the search must code them at another order, and the file decodes back under every decoder."""
    pcm = GOLD["pcm_oct_reference_lossy"]
    descs, words, ref_words, model = _check(pcm, 8)
    d = descs.reshape(2, 8)
    O = ol.load("port")
    for f, c, o in ((0, 1, 86), (1, 4, 29)):
        assert xl.analyse(O, pcm.reshape(2, FRAME, 8)[f, :, c].astype(np.int64)).tie
        assert int(d[f][c]["lpc_order"]) != o
    for D in _decoders():
        assert np.array_equal(D.decode_frames(descs, words, 8), pcm.reshape(-1))


@pytest.mark.gpu
def test_searched_frames_are_never_larger_without_a_tie():
    """Per frame, the searched words are at most the default encoder's wherever the default's units have no tie."""
    import sela_b200
    O = ol.load("port")
    pcm = np.concatenate([synth.sine_noise(44100, 2, n_frames=30, seed=5).reshape(-1),
                          analysis_corpus.batches()[1][1][:FRAME * 30].reshape(-1)])
    descs, words, ref_words = sela_b200.encode_frames_search(pcm, 2)
    d0, w0 = sela_b200.encode_frames(pcm, 2)
    assert ref_words == w0.size
    units = analysis_corpus.units(pcm, 2)
    for f in range(pcm.size // (2 * FRAME)):
        tie = any(xl.analyse(O, units[3 * f + k]).tie for k in range(3))
        size = lambda d: int(d["refl_words"].sum()) + int(d["res_words"].sum())
        assert tie or size(descs[2 * f:2 * f + 2]) <= size(d0[2 * f:2 * f + 2]), f


# ---- forced cases ----

def _analysed_preds(pcm, ch):
    """(order, q[100]) per unit as the analysis gives them."""
    qs, refs = xs.all_q(analysis_corpus.units(pcm, ch))
    return [(int(o), q) for o, q in zip(refs, qs)]


@pytest.mark.gpu
def test_forced_equal_words_reference_order_then_lowest():
    """two_tone with q = [10, 5, 0, ...]: orders 2..8 cost 984 words, 9 on 985.  The reference order wins inside
    that set, the lowest order outside it."""
    s = signals.families()["two_tone"].astype(np.int16)
    q = np.zeros(100, np.int32)
    q[:2] = [10, 5]
    pcm = np.tile(s, 6)
    refs = [5, 2, 8, 20, 1, 100]
    descs, words, ref_words, model = _check(pcm, 1, preds=[(r, q) for r in refs])
    assert [int(d["lpc_order"]) for d in descs] == [5, 2, 8, 2, 2, 2]
    assert all(int(d["refl_words"]) + int(d["res_words"]) == 984 for d in descs)


@pytest.mark.gpu
def test_forced_tie_at_the_winner_makes_the_runner_up_win():
    """A tie planted at the order that would win: the search codes the unit at the best order without one."""
    O = ol.load("port")
    rng = np.random.default_rng(3)
    base = signals.random_frames(6, 3).astype(np.int64)
    planted = []
    for s in base:
        q, ref = xs.all_q(s[None])
        win, _, _, _ = xs.search_unit(O, s, q[0], ref[0])
        if win.order < 2:
            continue
        c = xs.predictors(O, q[0])[win.order, :win.order + 1]
        t = s.copy()
        if xl.place_tie(t, c, 1000, rng=rng):
            w2, _, _, tie = xs.search_unit(O, t, q[0], ref[0])
            assert tie[win.order - 1] and w2.order != win.order
            planted.append((t, (int(ref[0]), q[0])))
    assert len(planted) >= 3
    pcm = np.concatenate([t for t, _ in planted]).astype(np.int16)
    _check(pcm, 1, preds=[p for _, p in planted])
    _check(pcm, 1)  # and through the analysis


@pytest.mark.gpu
def test_forced_stereo_decision_flips_after_the_search():
    """ch1 = ch0 - a smooth small signal: with the difference unit's reference order forced to 1, the reference
    keeps ch1 independent; after the search the predictable difference wins."""
    O = ol.load("port")
    t = np.arange(FRAME * 3)
    ch0 = (9000 * np.sin(t * 0.013) + 5000 * np.sin(t * 0.0021)).astype(np.int64)
    ch1 = ch0 - (1500 * np.sin(t * 0.031)).astype(np.int64)
    pcm = np.stack([ch0, ch1], axis=1).astype(np.int16).reshape(-1)
    preds = _analysed_preds(pcm, 2)
    for f in range(3):
        preds[3 * f + 2] = (1, preds[3 * f + 2][1])
    descs, words, ref_words, model = _check(pcm, 2, preds=preds)
    _, ref_words_model = xs.model_batch(O, pcm, 2, preds=preds)
    d = descs.reshape(3, 2)
    assert all(int(d[f][1]["subframe_type"]) == 1 for f in range(3))
    units = analysis_corpus.units(pcm, 2)
    for f in range(3):  # the reference's decision: ch1 independent
        a = xs.search_unit(O, units[3 * f + 1], preds[3 * f + 1][1], preds[3 * f + 1][0])[1]
        b = xs.search_unit(O, units[3 * f + 2], preds[3 * f + 2][1], 1)[1]
        assert not b.words < a.words
    assert ref_words == sum(ref_words_model.values())


@pytest.mark.gpu
def test_forced_order_100():
    """Reference order 100 and every q non-zero: every order 1..100 is a candidate, the last slice ends at 100."""
    pcm = signals.random_frames(4, 9).astype(np.int16).reshape(-1)
    preds = _analysed_preds(pcm, 1)
    preds = [(100, np.clip(np.where(q == 0, 1, q), -64, 63)) for _, q in preds]
    _check(pcm, 1, preds=preds)


@pytest.mark.gpu
def test_forced_domain():
    import sela_b200
    pcm = np.zeros(FRAME, np.int16)
    for order, q0 in ((0, 0), (101, 0), (5, 64), (5, -65)):
        q = np.zeros(100, np.int32)
        q[50] = q0
        with pytest.raises(sela_b200.SelaB200Error) as e:
            codec.encode_search_forced(pcm, 1, [(order, q)])
        assert e.value.status == -5


@pytest.mark.gpu
def test_batch_large_enough_for_the_grid_to_loop():
    """4 800 stereo frames (14 400 units: more than the candidate and repack grids of 32 warps per SM), compared with
    the model on frames at both ends and across the middle."""
    pcm = synth.sine_noise(44100, 2, n_frames=4800, seed=11)
    pcm[:FRAME * 4] = analysis_corpus.batches()[1][1][:FRAME * 4]
    _check(pcm, 2, frames=[0, 1, 2, 3, 1500, 2401, 4798, 4799])


# ---- host forms ----

@pytest.mark.gpu
def test_container_is_the_file_writer_of_the_searched_frames():
    import sela_b200
    pcm = np.concatenate([synth.sine_noise(48000, 8, n_frames=20, seed=2).reshape(-1),
                          GOLD["pcm_oct_reference_lossy"].reshape(-1)])
    descs, words, ref_words = sela_b200.encode_frames_search(pcm, 8)
    blob, ref_bytes = sela_b200.encode_container_search(pcm, 8, 48000)
    assert blob.tobytes() == wavio.pack_container(descs, words, 48000, 8)
    assert ref_bytes == sela_b200.encode_container(pcm, 8, 48000).size
    assert ref_bytes - blob.size == 4 * (ref_words - words.size)
    info, out = sela_b200.decode_container(blob)
    assert np.array_equal(out, pcm)


@pytest.mark.gpu
def test_host_forms_equal_the_device_form_under_small_chunks(monkeypatch):
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    n = 700
    pcm = synth.sine_noise(44100, 2, n_frames=n, seed=4).reshape(-1)
    codec_ = DeviceCodec(n, 2, device=0)
    codec_.encode_search(torch.from_numpy(pcm).to(torch.device("cuda", 0)))
    codec_.check_status()
    n_words = int(codec_.words_used.item())
    d_dev = codec_.descs.cpu().numpy().tobytes()
    w_dev = codec_.words[:n_words].cpu().numpy().view(np.uint32)
    ref_dev = int(codec_.ref_words.item())
    blob0, ref_bytes0 = sela_b200.encode_container_search(pcm, 2, 44100)
    for chunk in ("64", "100", "512"):
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", chunk)
        descs, words, ref_words = sela_b200.encode_frames_search(pcm, 2)
        assert descs.tobytes() == d_dev and np.array_equal(words, w_dev) and ref_words == ref_dev
        blob, ref_bytes = sela_b200.encode_container_search(pcm, 2, 44100)
        assert blob.tobytes() == blob0.tobytes() and ref_bytes == ref_bytes0
    monkeypatch.delenv("SELAB200_CHUNK_FRAMES")
    assert ref_dev == sela_b200.encode_frames(pcm, 2)[1].size
    _check(pcm, 2, frames=[0, 350, 699], got=(np.frombuffer(d_dev, _lib.DESC_DTYPE), w_dev, ref_dev))


# ------------------------------------------------------------------- CLI --

def _run(*cmd):
    return subprocess.run([str(c) for c in cmd], capture_output=True, text=True, timeout=600)


@pytest.mark.gpu
def test_cli_search_mode(tmp_path):
    if not (BIN / "sela").exists():
        subprocess.run(["make", "-C", str(ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    sela = BIN / "sela"
    pcm = synth.sine_noise(44100, 2, n_frames=9, seed=2)
    wav = tmp_path / "in.wav"
    # a partial frame at the end, which neither encoder codes
    wavio.write_wav(wav, np.concatenate([pcm, pcm[:700]]), 44100)
    p = _run(sela, "-S", wav, tmp_path / "s.sela")
    assert p.returncode == 0, (p.stdout, p.stderr)
    assert _run(sela, "-e", wav, tmp_path / "e.sela").returncode == 0
    written, ref = (tmp_path / "s.sela").stat().st_size, (tmp_path / "e.sela").stat().st_size
    assert "Wrote %d bytes (-e: %d bytes)" % (written, ref) in p.stdout
    assert written <= ref
    t = _run(sela, "-t", tmp_path / "s.sela", wav)
    assert t.returncode == 0 and "Verified" in t.stdout, (t.stdout, t.stderr)
    if REF_CLI.exists():
        assert _run(REF_CLI, "-d", tmp_path / "s.sela", tmp_path / "ref.wav").returncode == 0
        _, _, out = wavio.read_wav_pcm(tmp_path / "ref.wav")
        assert np.array_equal(out.reshape(-1), pcm.reshape(-1))
    assert "-S" in _run(sela).stdout
