"""Channel-pairing encodes (selab200_encode_frames_pairing, _encode_container_pairing, the device-resident form and
`sela -P`): every channel of a frame coded alone or as its difference from another, whichever valid assignment takes
the fewest words (DESIGN.md 7.4).

The expected output comes from the CPU model in exact_pairing.py (the lossless model as the base, the port's analysis
of every ordered pair, the tie criterion, Rice words, and the choice by enumeration), compared word for word and
descriptor for descriptor.  The large batch is compared on chosen frames and checked as a whole through base_words,
the device verifier and decoding."""
import pathlib
import subprocess

import numpy as np
import pytest

import analysis_corpus
import exact_lossless as xl
import exact_pairing as xp
import gpu_calls
import oracle_lib as ol
from sela_b200 import _lib, codec, synth, wavio

pytestmark = pytest.mark.gpu

GOLD = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
FRAME = 2048
ROOT = pathlib.Path(__file__).resolve().parent.parent
BIN = ROOT / "sela_b200" / "host" / "bin"
REF_CLI = ROOT / "oracle" / "_ref" / "sela_ref_cli"


def _totals(descs, words, base_words, n_diff, pcm, ch):
    import sela_b200
    assert n_diff == int((descs["subframe_type"] == 1).sum())
    assert words.size <= base_words
    assert base_words == sela_b200.encode_frames_lossless(pcm, ch)[1].size
    assert sela_b200.verify_frames(descs, words, ch, pcm).size == 0
    assert np.array_equal(sela_b200.decode_frames(descs, words, ch), pcm)
    assert np.array_equal(gpu_calls.decode_frames_device(descs, words, ch), pcm)


def _check(pcm, ch, preds=None):
    """Batch `pcm` through the tracing entry against the model: the stream, par[], the totals and every candidate
    record; the production entry gives the same stream."""
    import sela_b200
    O = ol.load("port")
    pcm = np.asarray(pcm, np.int16).reshape(-1)
    descs, words, base_words, n_diff, par, trace = codec.encode_pairing_trace(pcm, ch, preds)
    model = xp.model_batch(O, pcm, ch, preds)
    xp.check_batch(O, descs, words, pcm, ch, model)
    assert base_words == sum(m["base_words"] for m in model.values())
    assert words.size == sum(m["words"] for m in model.values())
    for f, m in model.items():
        assert tuple(par[f]) == m["par"], f
        for p in range(ch):
            for c in range(ch):
                r = trace[f, p, c]
                if p == c or (ch == 2 and p == 0):   # stereo (0, 1): the base's unit, not sized again
                    assert int(r["visits"]) == 0
                    continue
                assert int(r["visits"]) == 1, (f, p, c)
                want = xp.trace_record(O, m["cands"][p, c])
                got = {k: int(r[k]) for k in want if k != "order"}
                got["order"] = int(r["reserved"][0])
                assert got == want, (f, p, c)
    if preds is None:
        _totals(descs, words, base_words, n_diff, pcm, ch)
        d2, w2, b2, n2 = sela_b200.encode_frames_pairing(pcm, ch)
    else:
        assert n_diff == int((descs["subframe_type"] == 1).sum()) and words.size <= base_words
        d2, w2, b2, n2 = codec.encode_pairing_forced(pcm, ch, preds)
    assert d2.tobytes() == descs.tobytes() and np.array_equal(w2, words) and (b2, n2) == (base_words, n_diff)
    return descs, words, model


def _analysed_preds(O, pcm, ch):
    """What the encoder's analysis gives for every base unit and every candidate, as forced predictors."""
    planes = np.asarray(pcm, np.int64).reshape(-1, FRAME, ch).transpose(0, 2, 1)
    base = [xl.analyse(O, s) for s in analysis_corpus.units(pcm, ch)]
    cands = [xl.analyse(O, fr[p] - fr[c]) for fr in planes for p in range(ch) for c in range(ch) if p != c]
    return [(u.order, u.q.copy()) for u in base + cands]


@pytest.mark.parametrize("name", [f[0] for f in xp.families()])
def test_correlated_families(name):
    _, pcm, ch = next(f for f in xp.families() if f[0] == name)
    descs, words, model = _check(pcm, ch)
    if name in ("common_source_8", "dual_mono_in_six", "equal_and_negated"):
        assert (descs["subframe_type"] == 1).any()


@pytest.mark.parametrize("batch", ["stereo_pairs", "three_channels", "stereo_sine_noise", "eight_channels", "mono"])
def test_corpus_batches(batch):
    _, pcm, ch = next(b for b in analysis_corpus.batches() if b[0] == batch)
    pcm = np.asarray(pcm).reshape(-1, ch)
    if batch in ("stereo_pairs", "mono"):   # a spread of the batch: the model costs seconds per frame
        keep = np.arange(0, pcm.shape[0] // FRAME, 9 if batch == "stereo_pairs" else 40)
        pcm = pcm.reshape(-1, FRAME, ch)[keep].reshape(-1, ch)
    _check(pcm, ch)


def test_baseline_shaped_frames_and_independent_noise():
    import sela_b200
    _check(synth.sine_noise(44100, 2, n_frames=6, seed=1), 2)
    pcm = synth.sine_noise(48000, 8, n_frames=3, seed=9).astype(np.int16).reshape(-1)
    descs, words, model = _check(pcm, 8)
    d0, w0, _ = sela_b200.encode_frames_lossless(pcm, 8)   # no difference wins: the lossless encode's bytes
    assert descs.tobytes() == d0.tobytes() and np.array_equal(words, w0)


def test_golden_lossy_frames_never_emit_a_tied_unit():
    """oct_reference_lossy: two units tie at the reference order.  The base repairs them; no tied candidate is
    emitted, and the file decodes back under every decoder."""
    pcm = GOLD["pcm_oct_reference_lossy"]
    descs, words, model = _check(pcm, 8)
    for m in model.values():
        for c, p in enumerate(m["par"]):
            assert p == c or (p, c) not in m["tied"]


def test_sixteen_channels():
    import sela_b200
    pcm = xp.common_source(1, 16, 21).reshape(-1)
    descs, words, base_words, n_diff = sela_b200.encode_frames_pairing(pcm, 16)
    _totals(descs, words, base_words, n_diff, pcm, 16)
    O = ol.load("port")
    xp.check_batch(O, descs, words, pcm, 16, xp.model_batch(O, pcm, 16))
    assert n_diff >= 8


# ---- forced predictors ----

def test_forced_tie_in_the_winner_gives_the_runner_up():
    O = ol.load("port")
    _, pcm, ch = next(f for f in xp.families() if f[0] == "common_source_3")
    pcm = pcm[:FRAME].copy()
    preds = _analysed_preds(O, pcm, ch)
    m = xp.model_batch(O, pcm, ch, preds)[0]
    c, p = next((c, p) for c, p in enumerate(m["par"]) if p != c)
    order, q = preds[ch + xp.candidate_index(ch, 0, p, c)]
    chp, chc = pcm[:, p].astype(np.int64), pcm[:, c].astype(np.int64)
    assert xl.place_tie_difference(chp, chc, O.lpc_coefficients(q, order), 700)
    pcm[:, p] = chp
    descs, words, model = _check(pcm, ch, preds)
    assert (p, c) in model[0]["tied"] and model[0]["par"][c] != p


def test_forced_stereo_first_channel_against_the_second():
    """ch0 is made expensive alone (order 1: its residue is the signal), so coding it against ch1 wins."""
    O = ol.load("port")
    pcm = xp.common_source(2, 2, 31)
    preds = _analysed_preds(O, pcm, 2)
    for f in range(2):
        preds[3 * f] = (1, np.zeros(100, np.int32))
        preds[3 * f + 2] = (1, np.zeros(100, np.int32))   # and the base's own difference too
    descs, words, model = _check(pcm, 2, preds)
    assert all(m["par"] == (1, 1) for m in model.values())
    d = descs.reshape(-1, 2)
    assert (d[:, 0]["subframe_type"] == 1).all() and (d[:, 0]["parent_channel"] == 1).all()


def test_forced_flagged_stereo_loser_stays_tied():
    """ch1 alone has a tie and loses to the difference: the lossless select clears its flag and does not repair it.
    The pairing still may not emit it, so ch0 against ch1 (which needs ch1 alone) is out, whatever it would cost."""
    O = ol.load("port")
    pcm = xp.common_source(1, 2, 33).copy()
    preds = _analysed_preds(O, pcm, 2)
    preds[0] = (1, np.zeros(100, np.int32))   # without the tie, ch0 against ch1 would win
    order, q = preds[1]
    ch1 = pcm[:, 1].astype(np.int64)
    assert xl.place_tie(ch1, O.lpc_coefficients(q, order), 900)
    pcm[:, 1] = ch1
    planes = pcm.astype(np.int64).T
    m = xp.model_frame(O, planes, preds[:3], {(0, 1): preds[3], (1, 0): preds[4]})
    assert m["par"] == (0, 0) and m["base_words"] == m["words"]
    assert xl.Unit(O, planes[1], *preds[1]).tie
    _check(pcm, 2, preds)


def test_forced_equal_totals():
    """Every unit and candidate at order 1 (the residue is the signal) on channels that are equal or negated: many
    equal totals, resolved by the fewest differences and then the smallest parent vector."""
    O = ol.load("port")
    rng = np.random.default_rng(3)
    a = rng.integers(-200, 200, FRAME)
    for chans in ([a, a, a], [a, -a, a, -a], [a, a]):
        pcm = np.stack(chans, axis=1).astype(np.int16)
        ch = pcm.shape[1]
        n = (3 if ch == 2 else ch) + ch * (ch - 1)
        _check(pcm, ch, [(1, np.zeros(100, np.int32))] * n)


def test_forced_domain():
    import sela_b200
    pcm = np.zeros(FRAME * 3, np.int16)
    good = [(1, np.zeros(100, np.int32))] * 9
    for order, q0 in ((101, 0), (5, 64), (5, -65)):
        q = np.zeros(100, np.int32)
        q[2] = q0
        with pytest.raises(sela_b200.SelaB200Error) as e:
            codec.encode_pairing_forced(pcm, 3, good[:8] + [(order, q)])
        assert e.value.status == -5


# ---- scale and host forms ----

def test_batch_large_enough_for_every_grid_to_loop():
    """900 frames of 8 channels: 50 400 candidates and 7 200 subframes, past every fixed grid and scan tile."""
    import sela_b200
    O = ol.load("port")
    pcm = np.concatenate([xp.common_source(450, 8, 41), synth.sine_noise(48000, 8, n_frames=450, seed=6).astype(np.int16)])
    pcm = pcm.reshape(-1)
    descs, words, base_words, n_diff = sela_b200.encode_frames_pairing(pcm, 8)
    _totals(descs, words, base_words, n_diff, pcm, 8)
    frames = [0, 449, 450, 899]
    model = xp.model_batch(O, pcm, 8, frames=frames)
    d = descs.reshape(-1, 8)
    for f in frames:
        em = model[f]["emitted"]
        assert [(int(s["subframe_type"]), int(s["parent_channel"]), int(s["lpc_order"]),
                 int(s["refl_words"]) + int(s["res_words"])) for s in d[f]] == [(t, p, u.order, u.words) for u, t, p in em]
        for s, (u, _, _) in zip(d[f], em):
            kr, wr = O.rice_encode(u.res)
            assert np.array_equal(words[int(s["res_offset"]):int(s["res_offset"]) + int(s["res_words"])], wr)
    assert n_diff > 450 and not (d[450:]["subframe_type"] == 1).any()


def test_host_forms_and_container_equal_the_device_form(monkeypatch):
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    for ch, n in ((2, 300), (6, 120)):
        pcm = (xp.common_source(n, 2, 51) if ch == 2 else xp.dual_mono_in_six(n, 52)).reshape(-1)
        dc = DeviceCodec(n, ch, device=0)
        dc.encode_pairing(torch.from_numpy(pcm).to(torch.device("cuda", 0)))
        dc.check_status()
        n_words = int(dc.words_used.item())
        d_dev = dc.descs.cpu().numpy().tobytes()
        w_dev = dc.words[:n_words].cpu().numpy().view(np.uint32)
        totals = (int(dc.base_words.item()), int(dc.n_difference.item()))
        blob0, base_bytes0, nd0 = sela_b200.encode_container_pairing(pcm, ch, 48000)
        assert blob0.tobytes() == wavio.pack_container(np.frombuffer(d_dev, _lib.DESC_DTYPE), w_dev, 48000, ch)
        assert base_bytes0 == sela_b200.encode_container_lossless(pcm, ch, 48000)[0].size and nd0 == totals[1]
        assert np.array_equal(sela_b200.decode_container(blob0)[1], pcm)
        for chunk in ("32", "100"):
            monkeypatch.setenv("SELAB200_CHUNK_FRAMES", chunk)
            descs, words, base_words, n_diff = sela_b200.encode_frames_pairing(pcm, ch)
            assert descs.tobytes() == d_dev and np.array_equal(words, w_dev) and (base_words, n_diff) == totals
            blob, base_bytes, nd = sela_b200.encode_container_pairing(pcm, ch, 48000)
            assert blob.tobytes() == blob0.tobytes() and (base_bytes, nd) == (base_bytes0, nd0)
        monkeypatch.delenv("SELAB200_CHUNK_FRAMES")
        assert totals[1] > 0


def test_other_encodes_keep_their_bytes():
    """The default and lossless encodes of a pairing family equal the port's and the lossless model's."""
    import sela_b200
    O = ol.load("port")
    _, pcm, ch = next(f for f in xp.families() if f[0] == "dual_mono_in_six")
    pcm = pcm.reshape(-1)
    d, w = sela_b200.encode_frames(pcm, ch)
    do, wo = O.encode_frames(pcm, ch)
    assert np.array_equal(w, wo) and all(np.array_equal(d[k], do[k]) for k in xp.DESC_FIELDS)
    dl, wl, _ = sela_b200.encode_frames_lossless(pcm, ch)
    xl.check_against_model(O, dl, wl, pcm, ch, xl.model_batch(O, pcm, ch, every=True))


# ------------------------------------------------------------------- CLI --

def _run(*cmd):
    return subprocess.run([str(c) for c in cmd], capture_output=True, text=True, timeout=600)


@pytest.mark.parametrize("name", ["common_source_8", "dual_mono_in_six", "equal_and_negated", "common_source_stereo",
                                  "full_scale_opposite_3"])
def test_cli_pairing_mode(tmp_path, name):
    if not (BIN / "sela").exists():
        subprocess.run(["make", "-C", str(ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    sela = BIN / "sela"
    _, pcm, ch = next(f for f in xp.families() if f[0] == name)
    wav = tmp_path / "in.wav"
    wavio.write_wav(wav, np.concatenate([pcm, pcm[:700]]), 48000)   # a partial frame at the end, which is not coded
    p = _run(sela, "-P", wav, tmp_path / "p.sela")
    assert p.returncode == 0, (p.stdout, p.stderr)
    assert _run(sela, "-L", wav, tmp_path / "l.sela").returncode == 0
    written, base = (tmp_path / "p.sela").stat().st_size, (tmp_path / "l.sela").stat().st_size
    assert "Wrote %d bytes (-L: %d bytes), " % (written, base) in p.stdout and "difference subframes" in p.stdout
    assert written <= base
    t = _run(sela, "-t", tmp_path / "p.sela", wav)
    assert t.returncode == 0 and "Verified" in t.stdout, (t.stdout, t.stderr)
    if REF_CLI.exists():
        assert _run(REF_CLI, "-d", tmp_path / "p.sela", tmp_path / "ref.wav").returncode == 0
        _, _, out = wavio.read_wav_pcm(tmp_path / "ref.wav")
        assert np.array_equal(out.reshape(-1), pcm.reshape(-1))
    assert "-P" in _run(sela).stdout
