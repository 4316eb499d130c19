"""Guided order-search encodes (selab200_encode_frames_search_guided, _encode_container_search_guided, the
device-resident form and `sela -F`): every analysis unit coded at the tie-free order with the fewest words among the K
orders a reflection-coefficient estimate ranks best, order 1 and the reference order (DESIGN.md 7.7).

The expected output comes from the CPU model in exact_search_guided.py, whose per-order table is exact_search's batched
model.  One table per batch serves every K.  The trace hook checks every unit's estimates bit for bit, its order mask,
and the record of every order sized, once each; unlisted orders are never visited."""
import ctypes as C
import pathlib
import subprocess

import numpy as np
import pytest

import analysis_corpus
import exact_lossless as xl
import exact_search as xs
import exact_search_guided as xg
import exact_window
import gpu_calls
import oracle_lib as ol
import signals
from sela_b200 import _lib, codec, synth, wavio

GOLD = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
FRAME = 2048
ROOT = pathlib.Path(__file__).resolve().parent.parent
BIN = ROOT / "sela_b200" / "host" / "bin"
REF_CLI = ROOT / "oracle" / "_ref" / "sela_ref_cli"
KS = (1, 2, 4, 8, 100)


def _table(pcm, ch, preds=None):
    S, Q, refs = xg.unit_inputs(pcm, ch, preds)
    return S, Q, refs, xs.search_units(S, Q, refs)


def _check(pcm, ch, K, table, preds=None, got=None):
    """The guided search of batch `pcm` (host form, or the trace hook with `preds`, or `got` = (descs, words,
    ref_words)) against the model; the batch decodes back on the device; ref_words is the default encoder's (the
    model's with preds).  -> (descs, words, ref_words, g)."""
    import sela_b200
    O = ol.load("port")
    pcm = np.asarray(pcm, np.int16).reshape(-1)
    if got is None:
        got = (codec.encode_search_guided_trace(pcm, ch, K, preds)[:3] if preds is not None
               else sela_b200.encode_frames_search_guided(pcm, ch, K))
    descs, words, ref_words = got
    model, model_ref, g = xg.model_batch(pcm, ch, K, table=table)
    xs.check_frames(O, descs, words, pcm, ch, model)
    assert np.array_equal(gpu_calls.decode_frames_device(descs, words, ch), pcm)
    assert ref_words == sum(model_ref.values())
    if preds is None:
        assert ref_words == sela_b200.encode_frames(pcm, ch)[1].size
    return descs, words, ref_words, g


def _check_trace(pcm, ch, K, table, preds=None):
    """The trace hook: E bit for bit, the listed orders, every listed order sized exactly once with the model's
    record, no other order visited; and its output the model's."""
    pcm = np.asarray(pcm, np.int16).reshape(-1)
    descs, words, ref_words, trace, est, listed = codec.encode_search_guided_trace(pcm, ch, K, preds)
    g = _check(pcm, ch, K, table, preds=preds, got=(descs, words, ref_words))[3]
    assert np.array_equal(est.view(np.uint64), g["E"].view(np.uint64))
    assert np.array_equal(listed, g["listed"])
    assert np.array_equal(trace["visits"], listed.astype(np.uint32))
    m = g["m"]
    for f in xs.TRACE_FIELDS:
        got = trace[f].astype(m[f].dtype)
        assert np.array_equal(got[listed], m[f][listed]), f
    return g


# ------------------------------------------------------------------- CPU --

def test_guided_entry_points_have_no_cpu_fallback():
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
    assert L.selab200_encode_frames_search_guided(pcm.ctypes.data, 1, 1, 4, descs.ctypes.data, words.ctypes.data,
                                                  words.size, C.addressof(used), C.addressof(ref)) == -7
    assert L.selab200_encode_container_search_guided(pcm.ctypes.data, 1, 1, 4, 44100, 16, blob.ctypes.data,
                                                     blob.size, C.addressof(used), C.addressof(ref)) == -7
    assert L.selab200_encode_frames_search_guided_device(pcm.ctypes.data, 1, 1, 4, descs.ctypes.data,
                                                         words.ctypes.data, words.size, blob.ctypes.data,
                                                         blob.ctypes.data, blob.ctypes.data, blob.ctypes.data,
                                                         blob.size, None) == -7
    import sela_b200
    with pytest.raises(sela_b200.SelaB200Error):
        sela_b200.encode_frames_search_guided(pcm, 1, 4)


# ------------------------------------------------------------------- GPU --

def _sources():
    """The signal families, random frames, music-like frames, BASELINE-shaped frames and the golden
    oct_reference_lossy frames, then 6 frames of every analysis-corpus batch."""
    out = [("families", np.stack([v for v in signals.families().values()]).astype(np.int16).reshape(-1), 1),
           ("random", signals.random_frames(12, 3).astype(np.int16).reshape(-1), 1),
           ("music_like", exact_window.music_like(8, 2, 11).reshape(-1), 2),
           ("baseline", synth.sine_noise(44100, 2, n_frames=8, seed=1).reshape(-1), 2),
           ("oct_reference_lossy", GOLD["pcm_oct_reference_lossy"].reshape(-1), 8)]
    for name, pcm, ch in analysis_corpus.batches():
        n = pcm.size // (FRAME * ch)
        frames = sorted(set(np.linspace(0, n - 1, min(n, 6)).astype(int).tolist()))
        out.append((name, np.asarray(pcm, np.int16).reshape(n, -1)[frames].reshape(-1), ch))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", [s[0] for s in _sources()])
def test_every_k_against_the_model(name):
    """K = 1, 2, 4, 8, 100 against the model word for word and descriptor for descriptor; every unit at least its
    order-search words, and at most its reference words where the reference order has no tie; K = 100 byte-identical
    to the order search.  One K also through the trace."""
    import sela_b200
    _, pcm, ch = next(s for s in _sources() if s[0] == name)
    table = _table(pcm, ch)
    m, refs = table[3], table[2]
    for K in KS:
        descs, words, ref_words, g = _check(pcm, ch, K, table)
        w = m["words"][np.arange(len(refs)), g["order"] - 1]
        assert (w >= m["words"][np.arange(len(refs)), m["order"] - 1]).all()
        ref_tie = m["tie"][np.arange(len(refs)), refs - 1]
        assert (ref_tie | (w <= m["ref_words"])).all()
        if K == 100:
            d, wd, rw = sela_b200.encode_frames_search(pcm, ch)
            assert descs.tobytes() == d.tobytes() and np.array_equal(words, wd) and ref_words == rw
    _check_trace(pcm, ch, 4, table)


@pytest.mark.gpu
def test_golden_tied_reference_orders_lose():
    """oct_reference_lossy: frame 0 channel 1 (order 86) and frame 1 channel 4 (order 29) tie at the reference order;
    the guided search codes them at another order at every K."""
    pcm = GOLD["pcm_oct_reference_lossy"]
    table = _table(pcm, 8)
    for K in (1, 4):
        d = _check(pcm, 8, K, table)[0].reshape(2, 8)
        for f, c, o in ((0, 1, 86), (1, 4, 29)):
            assert int(d[f][c]["lpc_order"]) != o


# ---- forced cases ----

def _analysed_preds(pcm, ch):
    qs, refs = xs.all_q(analysis_corpus.units(pcm, ch))
    return [(int(o), q) for o, q in zip(refs, qs)]


@pytest.mark.gpu
def test_forced_tie_at_the_best_ranked_order_makes_the_next_listed_order_win():
    """A tie planted at the order the estimate ranks best: the unit is coded at another listed order, as the model
    says."""
    O = ol.load("port")
    rng = np.random.default_rng(5)
    base = np.concatenate([signals.random_frames(8, 3), exact_window.music_like(8, 1, 4).reshape(8, FRAME)])
    planted = []
    for s in base.astype(np.int64):
        q, ref = xs.all_q(s[None])
        top = int(np.argmin(xg.ranks(xg.estimates(q))[0])) + 1
        if top < 2 or top == ref[0]:
            continue
        c = xs.predictors(O, q[0])[top, :top + 1]
        t = s.copy()
        if xl.place_tie(t, c, 1000, rng=rng):
            planted.append((t, (int(ref[0]), q[0]), top))
    assert len(planted) >= 3
    pcm = np.concatenate([t for t, _, _ in planted]).astype(np.int16)
    preds = [p for _, p, _ in planted]
    table = _table(pcm, 1, preds)
    for K in (1, 2, 4):
        descs = _check(pcm, 1, K, table, preds=preds)[0]
        g = _check_trace(pcm, 1, K, table, preds)
        for n, (_, _, top) in enumerate(planted):
            assert g["m"]["tie"][n, top - 1] and int(descs[n]["lpc_order"]) != top


@pytest.mark.gpu
def test_forced_k1_lists_only_the_top_order_order_1_and_the_reference():
    pcm = signals.random_frames(6, 7).astype(np.int16).reshape(-1)
    preds = _analysed_preds(pcm, 1)
    preds = [(50 + 7 * n, q) for n, (_, q) in enumerate(preds)]
    table = _table(pcm, 1, preds)
    g = _check_trace(pcm, 1, 1, table, preds)
    assert (g["listed"].sum(axis=1) <= 3).all() and g["listed"][:, 0].all()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 4])
def test_forced_listed_orders_at_order_100_and_around_the_slice_edges(K):
    """q[X - 1] = -64 (k = -1) makes E zero from order X on, so X ranks first and X + 1 .. next: listed orders at
    order 100 and on both sides of the order search's slice edges 40 | 41, 64 | 65, 84 | 85."""
    xs_ = (40, 41, 64, 65, 84, 85, 99, 100)
    pcm = exact_window.music_like(len(xs_), 1, 9).reshape(-1)
    preds = []
    for (_, q), x in zip(_analysed_preds(pcm, 1), xs_):
        q = np.clip(np.where(q == 0, 1, q), -64, 63)
        q[x - 1] = -64
        preds.append((3, q))
    table = _table(pcm, 1, preds)
    assert table[3]["domain"].all()
    g = _check_trace(pcm, 1, K, table, preds)
    for n, x in enumerate(xs_):
        assert g["listed"][n, x - 1] and g["E"][n, x - 1] == 0.0
        assert all(g["listed"][n, o - 1] for o in range(x, min(x + K, 101)))


@pytest.mark.gpu
def test_forced_tied_reference_order():
    """The reference order forced to an order whose FIR ties: it is listed and sized but never chosen."""
    O = ol.load("port")
    rng = np.random.default_rng(8)
    s = signals.random_frames(3, 11).astype(np.int64)
    out, preds = [], []
    for u in s:
        q, _ = xs.all_q(u[None])
        c = xs.predictors(O, q[0])[30, :31]
        t = u.copy()
        if xl.place_tie(t, c, 1500, rng=rng):
            out.append(t)
            preds.append((30, q[0]))
    assert out
    pcm = np.concatenate(out).astype(np.int16)
    table = _table(pcm, 1, preds)
    for K in (1, 4):
        descs = _check(pcm, 1, K, table, preds=preds)[0]
        assert table[3]["tie"][:, 29].all() and (descs["lpc_order"] != 30).all()


@pytest.mark.gpu
def test_batch_large_enough_for_the_grids_to_loop():
    """4 800 stereo frames (14 400 units, more than the estimate and listed-order grids of 32 warps per SM), compared
    with the model on frames at both ends and across the middle."""
    import sela_b200
    O = ol.load("port")
    pcm = synth.sine_noise(44100, 2, n_frames=4800, seed=11)
    pcm[:FRAME * 4] = analysis_corpus.batches()[1][1][:FRAME * 4]
    descs, words, ref_words = sela_b200.encode_frames_search_guided(pcm, 2, 4)
    assert ref_words == sela_b200.encode_frames(pcm, 2)[1].size
    frames = [0, 1, 2, 3, 1500, 2401, 4798, 4799]
    sub = pcm.reshape(4800, -1)[frames].reshape(-1)
    model, _, _ = xg.model_batch(sub, 2, 4)
    xl.check_against_model(O, descs, words, pcm, 2, {f: (model[n], []) for n, f in enumerate(frames)})


# ---- host forms ----

@pytest.mark.gpu
def test_host_container_and_small_chunks_equal_the_device_form(monkeypatch):
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    n = 700
    pcm = synth.sine_noise(44100, 2, n_frames=n, seed=4).reshape(-1)
    codec_ = DeviceCodec(n, 2, device=0)
    codec_.encode_search_guided(torch.from_numpy(pcm).to(torch.device("cuda", 0)), 4)
    codec_.check_status()
    n_words = int(codec_.words_used.item())
    d_dev = codec_.descs.cpu().numpy().tobytes()
    w_dev = codec_.words[:n_words].cpu().numpy().view(np.uint32)
    ref_dev = int(codec_.ref_words.item())
    blob0, ref_bytes0 = sela_b200.encode_container_search_guided(pcm, 2, 44100, 4)
    assert blob0.tobytes() == wavio.pack_container(np.frombuffer(d_dev, _lib.DESC_DTYPE), w_dev, 44100, 2)
    assert ref_bytes0 == sela_b200.encode_container(pcm, 2, 44100).size
    for chunk in ("64", "100", "512"):
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", chunk)
        descs, words, ref_words = sela_b200.encode_frames_search_guided(pcm, 2, 4)
        assert descs.tobytes() == d_dev and np.array_equal(words, w_dev) and ref_words == ref_dev
        blob, ref_bytes = sela_b200.encode_container_search_guided(pcm, 2, 44100, 4)
        assert blob.tobytes() == blob0.tobytes() and ref_bytes == ref_bytes0
    monkeypatch.delenv("SELAB200_CHUNK_FRAMES")
    assert ref_dev == sela_b200.encode_frames(pcm, 2)[1].size
    info, out = sela_b200.decode_container(blob0)
    assert np.array_equal(out, pcm)
    O = ol.load("port")
    frames = [0, 350, 699]
    model, _, _ = xg.model_batch(pcm.reshape(n, -1)[frames].reshape(-1), 2, 4)
    xl.check_against_model(O, np.frombuffer(d_dev, _lib.DESC_DTYPE), w_dev, pcm, 2,
                           {f: (model[i], []) for i, f in enumerate(frames)})


@pytest.mark.gpu
def test_candidate_counts_outside_1_to_100_are_rejected():
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    pcm = synth.sine_noise(44100, 2, n_frames=2, seed=1).reshape(-1)
    codec_ = DeviceCodec(2, 2, device=0)
    d_pcm = torch.from_numpy(pcm).to(torch.device("cuda", 0))
    for K in (0, 101):
        for call in (lambda: sela_b200.encode_frames_search_guided(pcm, 2, K),
                     lambda: sela_b200.encode_container_search_guided(pcm, 2, 44100, K),
                     lambda: codec.encode_search_guided_trace(pcm, 2, K),
                     lambda: codec_.encode_search_guided(d_pcm, K)):
            with pytest.raises(sela_b200.SelaB200Error) as e:
                call()
            assert e.value.status == -3


# ------------------------------------------------------------------- CLI --

def _run(*cmd):
    return subprocess.run([str(c) for c in cmd], capture_output=True, text=True, timeout=600)


@pytest.mark.gpu
def test_cli_guided_search_mode(tmp_path):
    if not (BIN / "sela").exists():
        subprocess.run(["make", "-C", str(ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    sela = BIN / "sela"
    pcm = synth.sine_noise(44100, 2, n_frames=9, seed=2)
    wav = tmp_path / "in.wav"
    wavio.write_wav(wav, np.concatenate([pcm, pcm[:700]]), 44100)
    p = _run(sela, "-F", wav, tmp_path / "f.sela")
    assert p.returncode == 0, (p.stdout, p.stderr)
    assert _run(sela, "-e", wav, tmp_path / "e.sela").returncode == 0
    assert _run(sela, "-S", wav, tmp_path / "s.sela").returncode == 0
    written, ref = (tmp_path / "f.sela").stat().st_size, (tmp_path / "e.sela").stat().st_size
    assert "Wrote %d bytes (-e: %d bytes)" % (written, ref) in p.stdout
    assert (tmp_path / "s.sela").stat().st_size <= written <= ref
    t = _run(sela, "-t", tmp_path / "f.sela", wav)
    assert t.returncode == 0 and "Verified" in t.stdout, (t.stdout, t.stderr)
    if REF_CLI.exists():
        assert _run(REF_CLI, "-d", tmp_path / "f.sela", tmp_path / "ref.wav").returncode == 0
        _, _, out = wavio.read_wav_pcm(tmp_path / "ref.wav")
        assert np.array_equal(out.reshape(-1), pcm.reshape(-1))
    assert "-F" in _run(sela).stdout
