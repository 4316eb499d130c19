"""Window-search encodes (selab200_encode_frames_search_windows, _encode_container_search_windows, the device-resident
form and `sela -W`): the order search, and every unit also searched from the analysis of each selected apodisation
window, coded from the analysis and order with the fewest words (DESIGN.md 7.6).

The expected output comes from the CPU model in exact_window.py, compared word for word and descriptor for
descriptor, with both totals and every (unit, window, order) record through the trace.  The large batch is compared
on sampled frames and checked as a whole through its totals and decoding."""
import pathlib
import subprocess

import numpy as np
import pytest

import analysis_corpus
import exact_lossless as xl
import exact_search as xs
import exact_window as xw
import oracle_lib as ol
import signals
from sela_b200 import _lib, codec, synth, wavio

pytestmark = pytest.mark.gpu

GOLD = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
FRAME = 2048
ROOT = pathlib.Path(__file__).resolve().parent.parent
BIN = ROOT / "sela_b200" / "host" / "bin"
REF_CLI = ROOT / "oracle" / "_ref" / "sela_ref_cli"
MASKS = (1, 2, 4, 8, 16, 31)


def _tables(mask):
    return np.array([codec.analysis_window(i) for i in xw.mask_rows(mask)])


def _frame_words(descs, ch):
    d = descs.reshape(-1, ch)
    return (d["refl_words"].astype(np.int64) + d["res_words"]).sum(axis=1)


def _check_trace(trace, mw, name=""):
    """Every (unit, window, order) record equals the model's and was sized exactly once.  An order whose predictor
    leaves the conversion's domain is flagged as tied; its other fields are not defined by the model."""
    assert (trace["visits"] == 1).all(), (name, np.argwhere(trace["visits"] != 1)[:4])
    got = trace.reshape(-1, xs.MAX_ORDER)
    dom = mw["domain"]
    for field in xs.TRACE_FIELDS:
        want = mw[field]
        bad = np.argwhere((got[field].astype(want.dtype) != want) & (dom | (field == "tie")))
        assert not bad.size, (name, field, bad[:4])


def _check(pcm, ch, mask=1, tables=None, preds=None, name=""):
    """Batch `pcm` through the tracing entry against the model: the stream, both totals and every record; the
    production entry (the forced one with preds) gives the same stream."""
    import sela_b200
    O = ol.load("port")
    pcm = np.asarray(pcm, np.int16).reshape(-1)
    fixed = tables is None
    tables = _tables(mask) if fixed else np.atleast_2d(tables)
    descs, words, base_words, n_window, trace, keys = codec.encode_search_windows_trace(pcm, ch, tables, preds)
    model, base, mw, _, chosen = xw.model_batch(pcm, ch, tables, preds)
    assert np.array_equal(keys, mw["unit_keys"]), (name, np.flatnonzero(keys != mw["unit_keys"])[:4])
    xw.check_frames(O, descs, words, pcm, ch, model)
    assert base_words == sum(base.values()), name
    assert n_window == int((chosen >= 0).sum()), name
    assert words.size == sum(sum(c.words for c, _ in em) for em in model.values())
    got = _frame_words(descs, ch)
    assert (got <= np.array([base[f] for f in sorted(base)])).all(), name
    _check_trace(trace, mw, name)
    if fixed:
        if preds is None:
            d2, w2, b2, n2 = sela_b200.encode_frames_search_windows(pcm, ch, mask)
            ds, ws, _ = sela_b200.encode_frames_search(pcm, ch)
            assert ws.size == base_words
        else:
            d2, w2, b2, n2 = codec.encode_search_windows_forced(pcm, ch, mask, preds)
        assert d2.tobytes() == descs.tobytes() and np.array_equal(w2, words) and (b2, n2) == (base_words, n_window)
    return descs, words, model, mw, chosen


def _analysed_preds(pcm, ch, mask):
    """What the encoder's analyses give for every unit and every (unit, window), as forced predictors."""
    S = analysis_corpus.units(pcm, ch)
    q, o = xs.all_q(S)
    qw = np.stack([xw.window_q(S, t) for t in _tables(mask)], axis=1)
    return [(int(a), b.copy()) for a, b in zip(o, q)] + [(0, r.copy()) for r in qw.reshape(-1, xs.MAX_ORDER)]


# ---- the model, word for word ----

@pytest.mark.parametrize("batch", ["stereo_pairs", "three_channels", "stereo_sine_noise", "eight_channels", "mono"])
def test_corpus_batches(batch):
    _, pcm, ch = next(b for b in analysis_corpus.batches() if b[0] == batch)
    pcm = np.asarray(pcm).reshape(-1, FRAME, ch)
    n = pcm.shape[0]
    keep = np.unique(np.linspace(0, n - 1, min(n, 8 if ch <= 3 else 3)).astype(int))
    _check(pcm[keep].reshape(-1, ch), ch, 1, name=batch)


def test_signal_families_full_mask():
    pcm = np.stack([v for v in signals.families().values()]).reshape(-1, 1)
    _check(pcm, 1, 31, name="families")


@pytest.mark.parametrize("mask", MASKS)
def test_random_frames_every_single_window_and_all(mask):
    pcm = signals.random_frames(12, 5).reshape(-1, 1)
    _check(pcm, 1, mask, name="random %d" % mask)


@pytest.mark.parametrize("mask", MASKS)
def test_music_like_every_single_window_and_all(mask):
    _, _, _, _, chosen = _check(xw.music_like(3, 2, 11), 2, mask, name="music %d" % mask)
    if mask in (1, 31):
        assert (chosen >= 0).sum() >= 2


def test_baseline_shaped_frames():
    _check(synth.sine_noise(44100, 2, n_frames=6, seed=1), 2, 1, name="baseline stereo")
    _check(synth.sine_noise(48000, 8, n_frames=2, seed=9).astype(np.int16), 8, 31, name="config-4 shape")


def test_golden_lossy_frames():
    """oct_reference_lossy: two units tie at the reference order.  No emitted subframe has a tie."""
    import sela_b200
    pcm = GOLD["pcm_oct_reference_lossy"]
    descs, words, _, _, _ = _check(pcm, 8, 31, name="oct_reference_lossy")
    assert np.array_equal(sela_b200.decode_frames(descs, words, 8), np.asarray(pcm).reshape(-1))


# ---- the trace ----

def test_all_ones_window_equals_the_order_search():
    """A window of all ones is the plain analysis: every record equals the order search's record of the same unit, no
    window is strictly better, and the output is the order search's, byte for byte."""
    import sela_b200
    for pcm, ch in ((xw.music_like(2, 2, 3), 2), (synth.sine_noise(48000, 3, n_frames=2, seed=4), 3)):
        pcm = np.asarray(pcm, np.int16).reshape(-1)
        descs, words, base_words, n_window, trace, _ = codec.encode_search_windows_trace(pcm, ch, np.ones((1, FRAME)))
        _, _, _, _, strace = codec.encode_search_trace(pcm, ch)
        for field in xs.TRACE_FIELDS + ("visits",):
            assert np.array_equal(trace[:, 0][field], strace[field]), field
        ds, ws, _ = sela_b200.encode_frames_search(pcm, ch)
        assert n_window == 0 and descs.tobytes() == ds.tobytes() and np.array_equal(words, ws)
        assert base_words == ws.size


# ---- forced analyses ----

def test_forced_tie_at_the_window_winner_moves_it():
    """A tie planted at the order a window wins at: that order is no candidate any more."""
    O = ol.load("port")
    pcm = xw.music_like(1, 1, 21).astype(np.int64)
    preds = _analysed_preds(pcm.astype(np.int16), 1, 1)
    model, _, mw, Qw, chosen = xw.model_batch(pcm.astype(np.int16), 1, _tables(1), preds)
    assert chosen[0] == 0
    won = model[0][0][0].order
    assert won >= 2
    s = pcm[:, 0].copy()
    assert xl.place_tie(s, O.lpc_coefficients(Qw[0, 0], won), 700)
    pcm[:, 0] = s
    _, _, model2, mw2, _ = _check(pcm.astype(np.int16), 1, 1, preds=preds, name="planted tie")
    assert mw2["tie"][0, won - 1] and model2[0][0][0].order != won


def test_forced_window_equal_to_the_search_keeps_the_search():
    """Every window record takes the unit's own q: its best equals the order search's words, which is not strictly
    fewer, so the order search's winner stays (with its bytes)."""
    import sela_b200
    pcm = xw.music_like(2, 2, 23).reshape(-1)
    S = analysis_corpus.units(pcm.reshape(-1, 2), 2)
    q, o = xs.all_q(S)
    preds = [(int(a), b.copy()) for a, b in zip(o, q)] + [(0, b.copy()) for b in q]
    descs, words, _, _, chosen = _check(pcm, 2, 1, preds=preds, name="equal to -S")
    ds, ws, _ = codec.encode_search_forced(pcm, 2, preds[:len(S)])
    assert (chosen < 0).all() and descs.tobytes() == ds.tobytes() and np.array_equal(words, ws)


def test_forced_two_equal_windows_take_the_lower():
    """Windows 0 and 2 of the mask given the same q: equal words at every order, so both code the same bytes; the
    device's window keys (which _check compares with the model's) show that it chose the lower window."""
    pcm = xw.music_like(2, 1, 29)
    preds = _analysed_preds(pcm, 1, 5)
    U = 2
    for u in range(U):
        preds[U + 2 * u + 1] = (0, preds[U + 2 * u][1].copy())
    _, _, _, mw, chosen = _check(pcm, 1, 5, preds=preds, name="equal windows")
    assert np.array_equal(mw["words"][0::2], mw["words"][1::2])
    assert (chosen >= 0).any() and (chosen <= 0).all()
    assert ((mw["unit_keys"] >> np.uint64(8)) & np.uint64(0xff) == 0).all()


def test_forced_winners_at_order_100_and_both_sides_of_every_slice_edge():
    """Frames periodic with period o, the order search given nothing to predict with (every q zero, which at
    order >= 2 is a poor predictor), and the window record the predictor s[i] = s[i - o]: q[o - 1] = -64 (k = -1),
    q[0] = q[1] = 26 (k near 0) and every other q 0.  Orders below o predict next to nothing and orders above it
    cost more reflection words, so the window wins at exactly o.  A window can never win at order 1: the order-1
    predictor is zero whatever q is, so it takes exactly the order search's order-1 words."""
    rng = np.random.default_rng(5)
    edges = (100, 40, 41, 64, 65, 84, 85)
    frames, base, records = [], [], []
    for o in edges:
        frames.append(np.tile(rng.integers(-5000, 5000, o), FRAME // o + 1)[:FRAME])
        base.append((1, np.zeros(100, np.int32)))
        q = np.zeros(100, np.int32)
        q[:2] = 26
        q[o - 1] = -64
        records.append((0, q))
    pcm = np.array(frames, np.int16).reshape(-1, 1)
    _, _, model, mw, chosen = _check(pcm, 1, 1, preds=base + records, name="edges")
    assert (chosen == 0).all()
    assert [model[f][0][0].order for f in range(len(edges))] == list(edges)
    cut = [(1, np.zeros(100, np.int32))] * 2
    _, _, model, _, chosen = _check(pcm[:FRAME], 1, 1, preds=cut, name="order 1")
    assert chosen[0] < 0 and model[0][0][0].order == 1


def test_forced_domain():
    import sela_b200
    pcm = np.zeros(FRAME, np.int16)
    good = [(1, np.zeros(100, np.int32))] * 2
    for rec in ((101, 0), (0, 0)):
        q = np.zeros(100, np.int32)
        with pytest.raises(sela_b200.SelaB200Error) as e:
            codec.encode_search_windows_forced(pcm, 1, 1, [(rec[0], q), good[1]])
        assert e.value.status == -5
    for q0 in (64, -65):
        q = np.zeros(100, np.int32)
        q[2] = q0
        with pytest.raises(sela_b200.SelaB200Error) as e:
            codec.encode_search_windows_forced(pcm, 1, 1, [good[0], (0, q)])
        assert e.value.status == -5


def test_invalid_mask():
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    pcm = synth.sine_noise(44100, 2, n_frames=2, seed=1).reshape(-1)
    dc = DeviceCodec(2, 2, device=0)
    t = torch.from_numpy(pcm).to(torch.device("cuda", 0))
    for mask in (0, 32, 33, 1 << 31):
        for call in (lambda: sela_b200.encode_frames_search_windows(pcm, 2, mask),
                     lambda: sela_b200.encode_container_search_windows(pcm, 2, 44100, mask),
                     lambda: dc.encode_search_windows(t, mask)):
            with pytest.raises(sela_b200.SelaB200Error) as e:
                call()
            assert e.value.status == -3 and "window mask" in str(e.value)


# ---- scale and host forms ----

def test_batch_large_enough_for_the_grids_to_loop():
    """1 450 stereo frames: 4 350 units, past the 4 224 warps of the candidate and repack grids, and with two windows
    8 700 window analyses past the analysis grid."""
    import sela_b200
    O = ol.load("port")
    pcm = np.concatenate([xw.music_like(10, 2, 43), synth.sine_noise(44100, 2, n_frames=1440, seed=6)]).reshape(-1)
    descs, words, base_words, n_window = sela_b200.encode_frames_search_windows(pcm, 2, 5)
    ds, ws, _ = sela_b200.encode_frames_search(pcm, 2)
    assert base_words == ws.size and words.size <= base_words and n_window > 0
    assert (_frame_words(descs, 2) <= _frame_words(ds, 2)).all()
    assert np.array_equal(sela_b200.decode_frames(descs, words, 2), pcm)
    d = descs.reshape(-1, 2)
    frames = pcm.reshape(-1, FRAME, 2)
    for f in (0, 9, 10, 1449):
        em = xw.model_batch(frames[f].reshape(-1), 2, _tables(5))[0][0]
        assert [(int(s["subframe_type"]), int(s["lpc_order"]), int(s["refl_words"]) + int(s["res_words"]))
                for s in d[f]] == [(t, u.order, u.words) for u, t in em], f
        for s, (u, _) in zip(d[f], em):
            _, wr = O.rice_encode(u.res)
            assert np.array_equal(words[int(s["res_offset"]):int(s["res_offset"]) + int(s["res_words"])], wr)


def test_host_forms_and_container_equal_the_device_form(monkeypatch):
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    for ch, n, mask in ((2, 120, 1), (3, 60, 31)):
        pcm = xw.music_like(n, ch, 51 + ch).reshape(-1)
        dc = DeviceCodec(n, ch, device=0)
        dc.encode_search_windows(torch.from_numpy(pcm).to(torch.device("cuda", 0)), mask)
        dc.check_status()
        n_words = int(dc.words_used.item())
        d_dev = dc.descs.cpu().numpy().tobytes()
        w_dev = dc.words[:n_words].cpu().numpy().view(np.uint32)
        totals = (int(dc.base_words.item()), int(dc.n_window.item()))
        blob0, base_bytes0, nw0 = sela_b200.encode_container_search_windows(pcm, ch, 48000, mask)
        assert blob0.tobytes() == wavio.pack_container(np.frombuffer(d_dev, _lib.DESC_DTYPE), w_dev, 48000, ch)
        assert base_bytes0 == sela_b200.encode_container_search(pcm, ch, 48000)[0].size and nw0 == totals[1]
        assert np.array_equal(sela_b200.decode_container(blob0)[1], pcm)
        for chunk in ("16", "50"):
            monkeypatch.setenv("SELAB200_CHUNK_FRAMES", chunk)
            descs, words, base_words, n_window = sela_b200.encode_frames_search_windows(pcm, ch, mask)
            assert descs.tobytes() == d_dev and np.array_equal(words, w_dev) and (base_words, n_window) == totals
            blob, base_bytes, nw = sela_b200.encode_container_search_windows(pcm, ch, 48000, mask)
            assert blob.tobytes() == blob0.tobytes() and (base_bytes, nw) == (base_bytes0, nw0)
        monkeypatch.delenv("SELAB200_CHUNK_FRAMES")
        assert totals[1] > 0 and n_words < totals[0]


def test_window_search_after_the_device_set_changes():
    """Setting the library up for another set of devices sets its contexts up again, each with the window table of
    its own device: the window search then gives the same bytes on every device and in every form."""
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    pcm = xw.music_like(8, 2, 63).reshape(-1)
    want = sela_b200.encode_frames_search_windows(pcm, 2, 1, device=0)
    assert want[3] > 0
    for dev in (1, [1, 0], [0, 1], [1], 0):
        got = sela_b200.encode_frames_search_windows(pcm, 2, 1, device=dev)
        assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1]) and got[2:] == want[2:], dev
    for dev in (1, 0):
        dc = DeviceCodec(8, 2, device=dev)
        dc.encode_search_windows(torch.from_numpy(pcm).to(torch.device("cuda", dev)), 1)
        dc.check_status()
        assert dc.descs.cpu().numpy().tobytes() == want[0].tobytes(), dev
        assert (int(dc.base_words.item()), int(dc.n_window.item())) == want[2:], dev
    _lib.init(0)


# ------------------------------------------------------------------- CLI --

def _run(*cmd):
    return subprocess.run([str(c) for c in cmd], capture_output=True, text=True, timeout=600)


@pytest.mark.parametrize("ch", [1, 2, 6])
def test_cli_window_mode(tmp_path, ch):
    if not (BIN / "sela").exists():
        subprocess.run(["make", "-C", str(ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    sela = BIN / "sela"
    pcm = xw.music_like(4, ch, 70 + ch)
    wav = tmp_path / "in.wav"
    wavio.write_wav(wav, np.concatenate([pcm, pcm[:700]]), 48000)   # a partial frame at the end, which is not coded
    w = _run(sela, "-W", wav, tmp_path / "w.sela")
    assert w.returncode == 0, (w.stdout, w.stderr)
    assert _run(sela, "-S", wav, tmp_path / "s.sela").returncode == 0
    written, base = (tmp_path / "w.sela").stat().st_size, (tmp_path / "s.sela").stat().st_size
    assert "Wrote %d bytes (-S: %d bytes), " % (written, base) in w.stdout and "units coded from the window" in w.stdout
    assert written <= base
    t = _run(sela, "-t", tmp_path / "w.sela", wav)
    assert t.returncode == 0 and "Verified" in t.stdout, (t.stdout, t.stderr)
    if REF_CLI.exists():
        assert _run(REF_CLI, "-d", tmp_path / "w.sela", tmp_path / "ref.wav").returncode == 0
        _, _, out = wavio.read_wav_pcm(tmp_path / "ref.wav")
        assert np.array_equal(out.reshape(-1), pcm.reshape(-1))
    assert "-W" in _run(sela).stdout
