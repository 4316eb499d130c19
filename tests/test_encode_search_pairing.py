"""Search + pairing encodes (selab200_encode_frames_search_pairing, _encode_container_search_pairing, the
device-resident form and `sela -B`): the channel pairing on top of the order search, every channel and every channel
difference coded at its cheapest tie-free order (DESIGN.md 7.5).

The expected output comes from the CPU model in exact_search_pairing.py (the batched search model for the base and
every candidate, exact_pairing.assign for the choice), compared word for word, descriptor for descriptor, par[] and
every candidate's record at every order through the trace.  The large batch is compared on sampled frames and checked
as a whole through its totals, the device verifier and decoding."""
import pathlib
import subprocess

import numpy as np
import pytest

import analysis_corpus
import exact_lossless as xl
import exact_pairing as xp
import exact_search as xs
import exact_search_pairing as xsp
import gpu_calls
import oracle_lib as ol
from sela_b200 import _lib, codec, synth, wavio

pytestmark = pytest.mark.gpu

GOLD = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
FRAME = 2048
ROOT = pathlib.Path(__file__).resolve().parent.parent
BIN = ROOT / "sela_b200" / "host" / "bin"
REF_CLI = ROOT / "oracle" / "_ref" / "sela_ref_cli"


def _frame_words(descs, ch):
    d = descs.reshape(-1, ch)
    return (d["refl_words"].astype(np.int64) + d["res_words"]).sum(axis=1)


def _totals(descs, words, base_words, n_diff, pcm, ch):
    """base_words is the search's words; no frame is larger than the search's, nor than the pairing's on frames in
    which the lossless encode re-codes nothing; the stream verifies and decodes back."""
    import sela_b200
    assert n_diff == int((descs["subframe_type"] == 1).sum())
    ds, ws, _ = sela_b200.encode_frames_search(pcm, ch)
    assert base_words == ws.size and words.size <= base_words
    got = _frame_words(descs, ch)
    assert (got <= _frame_words(ds, ch)).all()
    dp, wp, _, _ = sela_b200.encode_frames_pairing(pcm, ch)
    _, _, recoded = sela_b200.encode_frames_lossless(pcm, ch)
    clean = np.ones(got.size, bool)
    clean[np.asarray(recoded["frame"], int)] = False
    assert (got[clean] <= _frame_words(dp, ch)[clean]).all()
    assert sela_b200.verify_frames(descs, words, ch, pcm).size == 0
    assert np.array_equal(sela_b200.decode_frames(descs, words, ch), pcm)
    assert np.array_equal(gpu_calls.decode_frames_device(descs, words, ch), pcm)


def _check_trace(trace, ch, m, index, name=""):
    """Every candidate's record at every order equals the model's, visited once; the others are never visited."""
    n_frames = trace.shape[0]
    sized = np.zeros(trace.shape[:3], bool)
    for (f, p, c), row in index.items():
        sized[f, p, c] = True
    assert (trace["visits"][~sized] == 0).all(), name
    bad = np.argwhere(trace["visits"][sized] != 1)
    assert not bad.size, (name, bad[:4])
    rows = np.array([index[f, p, c] for f in range(n_frames) for p in range(ch) for c in range(ch)
                     if sized[f, p, c]], int)
    got = trace[sized]
    for field in xs.TRACE_FIELDS:
        want = m[field][rows]
        bad = np.argwhere(got[field].astype(want.dtype) != want)
        assert not bad.size, (name, field, bad[:4])


def _check(pcm, ch, preds=None, name=""):
    """Batch `pcm` through the tracing entry against the model: the stream, par[], the totals and every candidate
    record at every order; the production entry gives the same stream."""
    import sela_b200
    O = ol.load("port")
    pcm = np.asarray(pcm, np.int16).reshape(-1)
    descs, words, base_words, n_diff, par, trace = codec.encode_search_pairing_trace(pcm, ch, preds)
    model, m, index, _, _ = xsp.model_batch(pcm, ch, preds)
    xsp.check_batch(O, descs, words, pcm, ch, model)
    assert base_words == sum(v["base_words"] for v in model.values())
    assert words.size == sum(v["words"] for v in model.values())
    for f, v in model.items():
        assert tuple(par[f]) == v["par"], (name, f)
    if index:
        assert m["domain"].all()
        _check_trace(trace, ch, m, index, name)
    else:
        assert (trace["visits"] == 0).all()
    if preds is None:
        _totals(descs, words, base_words, n_diff, pcm, ch)
        d2, w2, b2, n2 = sela_b200.encode_frames_search_pairing(pcm, ch)
    else:
        assert n_diff == int((descs["subframe_type"] == 1).sum()) and words.size <= base_words
        d2, w2, b2, n2 = codec.encode_search_pairing_forced(pcm, ch, preds)
    assert d2.tobytes() == descs.tobytes() and np.array_equal(w2, words) and (b2, n2) == (base_words, n_diff)
    return descs, words, model, m, index


def _analysed_preds(pcm, ch):
    """What the encoder's analysis gives for every base unit and every candidate, as forced search predictors
    (every q and the reference order)."""
    planes = np.asarray(pcm, np.int64).reshape(-1, FRAME, ch).transpose(0, 2, 1)
    q, o = xs.all_q(analysis_corpus.units(pcm, ch))
    d = np.array([fr[p] - fr[c] for fr in planes for p in range(ch) for c in range(ch) if p != c]).reshape(-1, FRAME)
    qc, oc = xs.all_q(d)
    return [(int(a), b.copy()) for a, b in zip(o, q)] + [(int(a), b.copy()) for a, b in zip(oc, qc)]


@pytest.mark.parametrize("name", [f[0] for f in xp.families()])
def test_correlated_families(name):
    _, pcm, ch = next(f for f in xp.families() if f[0] == name)
    descs, words, model, _, _ = _check(pcm, ch, name=name)
    if name in ("common_source_8", "dual_mono_in_six", "equal_and_negated"):
        assert (descs["subframe_type"] == 1).any()


@pytest.mark.parametrize("batch", ["stereo_pairs", "three_channels", "stereo_sine_noise", "eight_channels", "mono"])
def test_corpus_batches(batch):
    _, pcm, ch = next(b for b in analysis_corpus.batches() if b[0] == batch)
    pcm = np.asarray(pcm).reshape(-1, FRAME, ch)
    n = pcm.shape[0]
    keep = np.unique(np.linspace(0, n - 1, min(n, 24 if ch <= 3 else 8)).astype(int))   # a spread of the batch
    _check(pcm[keep].reshape(-1, ch), ch, name=batch)


def test_mono_is_the_order_search():
    import sela_b200
    pcm = synth.sine_noise(44100, 1, n_frames=5, seed=3).astype(np.int16).reshape(-1)
    descs, words, base_words, n_diff = sela_b200.encode_frames_search_pairing(pcm, 1)
    d0, w0, _ = sela_b200.encode_frames_search(pcm, 1)
    assert descs.tobytes() == d0.tobytes() and np.array_equal(words, w0) and (base_words, n_diff) == (w0.size, 0)


def test_baseline_shaped_frames_and_independent_noise():
    _check(synth.sine_noise(44100, 2, n_frames=6, seed=1), 2, name="baseline stereo")
    _check(synth.sine_noise(48000, 8, n_frames=2, seed=9).astype(np.int16), 8, name="config-4 shape")


def test_golden_lossy_frames():
    """oct_reference_lossy: two units tie at the reference order.  The search never emits a tied order; the file
    decodes back under every decoder."""
    _check(GOLD["pcm_oct_reference_lossy"], 8, name="oct_reference_lossy")


def test_sixteen_channels():
    import sela_b200
    pcm = xp.common_source(1, 16, 21).reshape(-1)
    descs, words, base_words, n_diff = sela_b200.encode_frames_search_pairing(pcm, 16)
    _totals(descs, words, base_words, n_diff, pcm, 16)
    O = ol.load("port")
    xsp.check_batch(O, descs, words, pcm, 16, xsp.model_batch(pcm, 16)[0])
    assert n_diff >= 8


# ---- forced predictors ----

def test_forced_tie_in_the_winner_moves_the_winner():
    """A tie planted at the order a difference wins at: another order or another assignment wins."""
    O = ol.load("port")
    _, pcm, ch = next(f for f in xp.families() if f[0] == "common_source_3")
    pcm = pcm[:FRAME].copy()
    preds = _analysed_preds(pcm, ch)
    model, m, index, _, _ = xsp.model_batch(pcm, ch, preds)
    par = model[0]["par"]
    c, p = next((c, p) for c, p in enumerate(par) if p != c and model[0]["cands"][p, c].order >= 2)
    won = model[0]["cands"][p, c].order
    _, q = preds[len(analysis_corpus.units(pcm, ch)) + xp.candidate_index(ch, 0, p, c)]
    chp, chc = pcm[:, p].astype(np.int64), pcm[:, c].astype(np.int64)
    assert xl.place_tie_difference(chp, chc, O.lpc_coefficients(np.asarray(q, np.int32), won), 700)
    pcm[:, p] = chp
    _, _, model2, m2, index2 = _check(pcm, ch, preds, name="planted tie")
    assert m2["tie"][index2[0, p, c], won - 1] and model2[0]["cands"][p, c].order != won


def test_forced_stereo_first_channel_against_the_second():
    """ch0 alone and the base's difference made expensive (every q zero: every order predicts nothing), so coding ch0
    against ch1 wins."""
    pcm = xp.common_source(2, 2, 31)
    preds = _analysed_preds(pcm, 2)
    for f in range(2):
        preds[3 * f] = (1, np.zeros(100, np.int32))
        preds[3 * f + 2] = (1, np.zeros(100, np.int32))
    descs, words, model, _, _ = _check(pcm, 2, preds, name="stereo ch0 against ch1")
    assert all(v["par"] == (1, 1) for v in model.values())
    d = descs.reshape(-1, 2)
    assert (d[:, 0]["subframe_type"] == 1).all() and (d[:, 0]["parent_channel"] == 1).all()


def test_forced_equal_totals():
    """Every q zero on channels that are equal or negated: every order of every unit and candidate takes the same
    residues, so equal totals everywhere, resolved by the fewest differences and then the smallest parent vector."""
    rng = np.random.default_rng(3)
    a = rng.integers(-200, 200, FRAME)
    for chans in ([a, a, a], [a, -a, a, -a], [a, a]):
        pcm = np.stack(chans, axis=1).astype(np.int16)
        ch = pcm.shape[1]
        n = (3 if ch == 2 else ch) + ch * (ch - 1)
        _check(pcm, ch, [(1, np.zeros(100, np.int32))] * n, name="equal totals %d" % ch)


def test_forced_reference_order_100_and_slice_edges():
    """Candidates whose reference order is 100, or an order at either side of a slice edge (40/41, 64/65, 84/85),
    with q zero past it, so that no higher order takes fewer words and the winner lies at or below it."""
    ch = 3
    pcm = xp.common_source(2, ch, 71)
    preds = _analysed_preds(pcm, ch)
    n_units = 2 * ch
    edges = (100, 40, 41, 64, 65, 84, 85)
    for i in range(n_units, len(preds)):
        o = edges[(i - n_units) % len(edges)]
        q = np.asarray(preds[i][1], np.int32).copy()
        q[o:] = 0
        preds[i] = (o, q)
    _, _, model, m, index = _check(pcm, ch, preds, name="edges")
    slices = {int(np.searchsorted([41, 65, 85], o, side="right")) for o in m["order"]}
    assert len(slices) >= 2, slices


def test_forced_domain():
    import sela_b200
    pcm = np.zeros(FRAME * 3, np.int16)
    good = [(1, np.zeros(100, np.int32))] * 9
    for order, q0 in ((101, 0), (0, 0), (5, 64), (5, -65)):
        q = np.zeros(100, np.int32)
        q[2] = q0
        with pytest.raises(sela_b200.SelaB200Error) as e:
            codec.encode_search_pairing_forced(pcm, 3, good[:8] + [(order, q)])
        assert e.value.status == -5


# ---- scale and host forms ----

def test_batch_large_enough_for_the_candidate_grid_to_loop():
    """540 frames of 8 channels: 4 320 units, past the 4 224 warps of the candidate grid, and 30 240 candidates."""
    import sela_b200
    O = ol.load("port")
    pcm = np.concatenate([xp.common_source(270, 8, 41), synth.sine_noise(48000, 8, n_frames=270, seed=6).astype(np.int16)])
    pcm = pcm.reshape(-1)
    descs, words, base_words, n_diff = sela_b200.encode_frames_search_pairing(pcm, 8)
    _totals(descs, words, base_words, n_diff, pcm, 8)
    d = descs.reshape(-1, 8)
    frames = pcm.reshape(-1, FRAME, 8)
    for f in (0, 269, 270, 539):
        model = xsp.model_batch(frames[f].reshape(-1), 8)[0][0]
        em = model["emitted"]
        assert [(int(s["subframe_type"]), int(s["parent_channel"]), int(s["lpc_order"]),
                 int(s["refl_words"]) + int(s["res_words"])) for s in d[f]] == [(t, p, u.order, u.words) for u, t, p in em]
        for s, (u, _, _) in zip(d[f], em):
            kr, wr = O.rice_encode(u.res)
            assert np.array_equal(words[int(s["res_offset"]):int(s["res_offset"]) + int(s["res_words"])], wr)
    assert n_diff > 270


def test_host_forms_and_container_equal_the_device_form(monkeypatch):
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    for ch, n in ((2, 120), (6, 60)):
        pcm = (xp.common_source(n, 2, 51) if ch == 2 else xp.dual_mono_in_six(n, 52)).reshape(-1)
        dc = DeviceCodec(n, ch, device=0)
        dc.encode_search_pairing(torch.from_numpy(pcm).to(torch.device("cuda", 0)))
        dc.check_status()
        n_words = int(dc.words_used.item())
        d_dev = dc.descs.cpu().numpy().tobytes()
        w_dev = dc.words[:n_words].cpu().numpy().view(np.uint32)
        totals = (int(dc.base_words.item()), int(dc.n_difference.item()))
        blob0, base_bytes0, nd0 = sela_b200.encode_container_search_pairing(pcm, ch, 48000)
        assert blob0.tobytes() == wavio.pack_container(np.frombuffer(d_dev, _lib.DESC_DTYPE), w_dev, 48000, ch)
        assert base_bytes0 == sela_b200.encode_container_search(pcm, ch, 48000)[0].size and nd0 == totals[1]
        assert np.array_equal(sela_b200.decode_container(blob0)[1], pcm)
        for chunk in ("16", "50"):
            monkeypatch.setenv("SELAB200_CHUNK_FRAMES", chunk)
            descs, words, base_words, n_diff = sela_b200.encode_frames_search_pairing(pcm, ch)
            assert descs.tobytes() == d_dev and np.array_equal(words, w_dev) and (base_words, n_diff) == totals
            blob, base_bytes, nd = sela_b200.encode_container_search_pairing(pcm, ch, 48000)
            assert blob.tobytes() == blob0.tobytes() and (base_bytes, nd) == (base_bytes0, nd0)
        monkeypatch.delenv("SELAB200_CHUNK_FRAMES")
        assert totals[1] > 0


# ------------------------------------------------------------------- CLI --

def _run(*cmd):
    return subprocess.run([str(c) for c in cmd], capture_output=True, text=True, timeout=600)


@pytest.mark.parametrize("name", ["common_source_8", "dual_mono_in_six", "common_source_stereo"])
def test_cli_best_mode(tmp_path, name):
    if not (BIN / "sela").exists():
        subprocess.run(["make", "-C", str(ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    sela = BIN / "sela"
    _, pcm, ch = next(f for f in xp.families() if f[0] == name)
    wav = tmp_path / "in.wav"
    wavio.write_wav(wav, np.concatenate([pcm, pcm[:700]]), 48000)   # a partial frame at the end, which is not coded
    b = _run(sela, "-B", wav, tmp_path / "b.sela")
    assert b.returncode == 0, (b.stdout, b.stderr)
    assert _run(sela, "-S", wav, tmp_path / "s.sela").returncode == 0
    written, base = (tmp_path / "b.sela").stat().st_size, (tmp_path / "s.sela").stat().st_size
    assert "Wrote %d bytes (-S: %d bytes), " % (written, base) in b.stdout and "difference subframes" in b.stdout
    assert written <= base
    t = _run(sela, "-t", tmp_path / "b.sela", wav)
    assert t.returncode == 0 and "Verified" in t.stdout, (t.stdout, t.stderr)
    if REF_CLI.exists():
        assert _run(REF_CLI, "-d", tmp_path / "b.sela", tmp_path / "ref.wav").returncode == 0
        _, _, out = wavio.read_wav_pcm(tmp_path / "ref.wav")
        assert np.array_equal(out.reshape(-1), pcm.reshape(-1))
    assert "-B" in _run(sela).stdout
