"""Whole batches at the sizes the project runs, against the tiled per-frame model of tests/batch_model.py: the
encode scan past 32 and 64 CTAs with stereo ties at its CTA edges, the decode plan past its second 64-CTA stride
and at both of its bounds, and every chunk plan of the host calls, with fill levels chained across chunks.

Memory: every one-call case is sized from selab200_*_workspace_bytes and stays under 4 GB of device memory; host
calls stay at or below 5 000 frames (their device buffers are kept for the rest of the process)."""
import gc

import numpy as np
import pytest
import torch

import batch_model as B
import gpu_calls
import sela_b200
from sela_b200 import _lib, wavio
from sela_b200.device import DeviceCodec

pytestmark = pytest.mark.gpu
FRAME = 2048
LIMIT = 4 << 30
SENTINEL = 0x5A5A          # PCM pre-fill: a stale buffer that already holds the right samples must not pass


@pytest.fixture(autouse=True)
def _release():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def codec_bytes(n_frames, ch, words=None, verify=False):
    """Device memory of a DeviceCodec case: descriptors, arena, both workspaces, input and output PCM."""
    L = _lib.lib()
    n_sub = n_frames * ch
    cap = L.selab200_encode_words_bound(n_frames, ch) if words is None else words
    total = (n_sub * 32 + cap * 4 + L.selab200_encode_workspace_bytes(n_frames, ch)
             + L.selab200_decode_workspace_bytes(n_frames, ch) + 2 * n_sub * FRAME * 2)
    if verify:
        total += L.selab200_verify_workspace_bytes(n_frames, ch)
    return total


def first_bad_subframe(got, want):
    g = np.frombuffer(got.tobytes(), np.uint8).reshape(-1, 32)
    w = np.frombuffer(want.tobytes(), np.uint8).reshape(-1, 32)
    bad = np.flatnonzero((g != w).any(axis=1))
    return "%d subframes differ, first %s" % (bad.size, bad[:4].tolist())


def first_bad_frame(got, want, ch):
    bad = np.flatnonzero((got.reshape(-1, FRAME * ch) != want.reshape(-1, FRAME * ch)).any(axis=1))
    return "%d frames differ, first %s" % (bad.size, bad[:4].tolist())


# ------------------------------------------------------------------------------ one-call encode --

def _special(bank):
    return [bank.index(n) for n in (B.TIES if bank.channels == 2 else ("lossy_a", "lossy_b"))]


@pytest.mark.parametrize("ch,n", B.DEVICE_BATCHES, ids=["stereo12919", "stereo33000", "oct8200"])
def test_device_encode_and_decode_one_call(ch, n):
    """DeviceCodec.encode on the whole batch: descriptors byte for byte, words and words_used against the model,
    ties / lossy frames on both sides of the scan's CTA edges; then its decode into sentinel-filled PCM.  At
    33 000 stereo frames: exactly `used` words of capacity succeed, one fewer is CAPACITY."""
    bank = B.encode_bank(ch)
    rng = np.random.default_rng(n)
    idx = rng.integers(0, len(bank), n)
    special = _special(bank)
    at = [f for f in B.EDGE_FRAMES if f < n] + [n - 1]
    idx[at] = [special[j % len(special)] for j in range(len(at))]
    want = B.tile(bank, idx)
    verify = ch == 8
    assert codec_bytes(n, ch, verify=verify) < LIMIT
    if ch == 2:   # the predicted stereo decisions at the edges: ties keep R, one word less takes the difference
        types = want.descs.reshape(n, 2)[at, 1]["subframe_type"]
        assert types.tolist() == [B.TIES[bank.names[idx[f]]][1] for f in at]

    dev = torch.device("cuda", 0)
    codec = DeviceCodec(n, ch, device=0)
    codec.descs.fill_(0xFF)
    pcm = torch.from_numpy(want.pcm).to(dev)
    codec.encode(pcm)
    codec.check_status()
    used = int(codec.words_used.item())
    got_descs = codec.descs.cpu().numpy()
    assert got_descs.tobytes() == want.descs.tobytes(), first_bad_subframe(got_descs, want.descs)
    assert used == want.used
    got_words = codec.words[:used].cpu().numpy().view(np.uint32)
    assert np.array_equal(got_words, want.words), np.flatnonzero(got_words != want.words)[:4]

    out = torch.full((n * ch * FRAME,), SENTINEL, dtype=torch.int16, device=dev)
    codec.decode(out, used)
    codec.check_status()
    got = out.cpu().numpy()
    assert np.array_equal(got, want.decoded), first_bad_frame(got, want.decoded, ch)
    del out
    if verify:
        codec.verify(pcm, used)
        rep = codec.verify_report()
        assert want.report.size > 0 and rep.tolist() == want.report.tolist()

    if n == 33000:
        codec.capacity = used
        codec.encode(pcm)
        codec.check_status()
        assert int(codec.words_used.item()) == used
        codec.capacity = used - 1
        codec.encode(pcm)
        with pytest.raises(sela_b200.SelaB200Error) as e:
            codec.check_status()
        assert e.value.status == -4
    del codec, pcm


# --------------------------------------------------------------------------------- decode plan --

def _plan_batch(case):
    rng = np.random.default_rng(len(case))
    if case == "frames16":
        bank = B.frames16_bank()
        return bank, rng.integers(0, bank.descs.shape[0], B.FRAMES16)
    bank = B.decode_bank()
    if case == "templates26":
        idx = B.by_width(bank, B.PLAN_26, rng)
        w = bank.widths[idx, 0]
        j = int(np.flatnonzero(w != w[1023])[0])                 # subframes 1023 and 1024 of different widths
        if w[1024] == w[1023]:
            idx[[1024, j]] = idx[[j, 1024]]
        return bank, idx
    if case == "odd_order100":
        return bank, rng.choice(np.flatnonzero(bank.descs[:, 0]["lpc_order"] == 100), sum(B.PLAN_ODD13))
    return bank, B.by_width(bank, B.PLAN_WIDTH1, rng)


@pytest.mark.parametrize("case", ["templates26", "odd_order100", "width1", "frames16"])
def test_decode_plan_past_64_ctas(case):
    """One decode call of a tiled crafted batch against the exact samples: MAX_TEMPLATES templates shuffled so
    that every plan CTA is mixed (92 CTAs); an odd count of order-100 subframes (the synthesis_warps bound, 65
    CTAs); all width 1 with a partial last warp; 16-channel frames with difference subframes (66 CTAs)."""
    bank, idx = _plan_batch(case)
    ch = bank.channels
    descs, words, want = bank.tile(idx)
    n_frames = descs.size // ch
    assert codec_bytes(n_frames, ch, words=words.size + 8) < LIMIT
    if case == "templates26":
        assert bank.widths[idx[1023], 0] != bank.widths[idx[1024], 0]
        assert len(B.segment_templates(np.bincount(bank.widths[idx, 0], minlength=14)[1:])) == B.MAX_TEMPLATES
    got = gpu_calls.decode_frames_device(descs, words, ch, fill=SENTINEL)
    assert np.array_equal(got, want), first_bad_frame(got, want, ch)


# ----------------------------------------------------------------------------------- host calls --

def _host_case(ch, n, forced, monkeypatch):
    if forced is None:
        monkeypatch.delenv("SELAB200_CHUNK_FRAMES", raising=False)
    else:
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", str(forced))
    bank = B.encode_bank(ch)
    return B.tile(bank, B.host_idx(bank, n, forced, _special(bank), seed=n * 10 + ch))


@pytest.mark.parametrize("ch", [2, 8])
@pytest.mark.parametrize("n,forced", B.HOST_PLANS, ids=["%d-%s" % c for c in B.HOST_PLANS])
def test_host_calls_at_every_chunk_plan(monkeypatch, ch, n, forced):
    """encode_frames, decode_frames, encode_container / decode_container, verify_frames and
    encode_container_verified at every chunk plan, ties / lossy frames on both sides of every chunk edge."""
    want = _host_case(ch, n, forced, monkeypatch)
    rate = 44100 if ch == 2 else 48000
    descs, words = sela_b200.encode_frames(want.pcm, ch)
    assert descs.tobytes() == want.descs.tobytes(), first_bad_subframe(descs, want.descs)
    assert np.array_equal(words, want.words), np.flatnonzero(words[:want.used] != want.words[:words.size])[:4]
    got = sela_b200.decode_frames(want.descs, want.words, ch)
    assert np.array_equal(got, want.decoded), first_bad_frame(got, want.decoded, ch)
    blob = sela_b200.encode_container(want.pcm, ch, rate)
    packed = wavio.pack_container(want.descs, want.words, rate, ch)
    assert blob.tobytes() == packed
    info, got = sela_b200.decode_container(blob)
    assert info["n_frames"] == n and np.array_equal(got, want.decoded), first_bad_frame(got, want.decoded, ch)
    if ch == 8:
        assert want.report.size > 0
    rep = sela_b200.verify_frames(want.descs, want.words, ch, want.pcm)
    assert rep.tolist() == want.report.tolist()
    blob, rep = sela_b200.encode_container_verified(want.pcm, ch, rate)
    assert blob.tobytes() == packed and rep.tolist() == want.report.tolist()


def test_host_capacity_on_a_tapered_plan(monkeypatch):
    want = _host_case(2, 2048, None, monkeypatch)
    descs, words = sela_b200.encode_frames(want.pcm, 2, words_capacity=want.used)
    assert descs.tobytes() == want.descs.tobytes() and np.array_equal(words, want.words)
    with pytest.raises(sela_b200.SelaB200Error) as e:
        sela_b200.encode_frames(want.pcm, 2, words_capacity=want.used - 1)
    assert e.value.status == -4


@pytest.fixture(scope="module")
def oct_lossless():
    """The 8-channel bank through the library's own lossless encode, one frame at a time in one call."""
    return B.lossless_bank(B.encode_bank(8), lambda pcm, ch: sela_b200.encode_frames_lossless(pcm, ch))


@pytest.mark.parametrize("n,forced", [(2048, None), (500, 7)])
def test_lossless_at_multi_chunk_plans(monkeypatch, oct_lossless, n, forced):
    """encode_frames_lossless of a tiled batch is the lossless encode of its bank frames laid end to end, with the
    re-coded pairs reported at their batch frame numbers; it decodes back to its source."""
    bank = oct_lossless
    assert bank.records.size > 0
    if forced is None:
        monkeypatch.delenv("SELAB200_CHUNK_FRAMES", raising=False)
    else:
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", str(forced))
    recoded = sorted(set(bank.records["frame"].tolist()))
    want = B.tile(bank, B.host_idx(bank, n, forced, recoded, seed=n))
    descs, words, rep = sela_b200.encode_frames_lossless(want.pcm, 8)
    assert descs.tobytes() == want.descs.tobytes(), first_bad_subframe(descs, want.descs)
    assert np.array_equal(words, want.words)
    assert want.report.size > 0 and rep.tolist() == want.report.tolist()
    assert np.array_equal(sela_b200.decode_frames(descs, words, 8), want.pcm)
