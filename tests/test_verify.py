"""Verify: decode coded frames and compare them with their source PCM, reporting every (frame, channel) that
differs (selab200_verify_frames, _encode_container_verified, _container_verify, the device-resident core,
and `sela -V` / `sela -t`).

The expected report always comes from `expected_report` below, a NumPy comparison of decoded output with the
source: on the golden vectors the decoded output is the REFERENCE decoder's (decoded_*), elsewhere
sela_b200.decode_frames (which the golden tests pin to the reference decoder)."""
import ctypes as C
import os
import pathlib
import subprocess

import numpy as np
import pytest

from sela_b200 import _lib, synth, wavio

GOLD = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
CASES = sorted(k[4:] for k in GOLD.files if k.startswith("pcm_"))
FRAME = 2048
ROOT = pathlib.Path(__file__).resolve().parent.parent
BIN = ROOT / "sela_b200" / "host" / "bin"
REF_CLI = ROOT / "oracle" / "_ref" / "sela_ref_cli"
# frame 8975 / 13577 of synth.sine_noise(48000, 8, 600, seed=2), on which the reference is not lossless
LOSSY = GOLD["pcm_oct_reference_lossy"]


def _n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


TWO_GPUS = pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")


def expected_report(decoded, source, channels):
    """One entry per (frame, channel) whose decoded samples differ from the source, in (frame, channel) order."""
    d = np.asarray(decoded, np.int16).reshape(-1, FRAME, channels).astype(np.int32)
    s = np.asarray(source, np.int16).reshape(-1, FRAME, channels).astype(np.int32)
    diff = d != s
    out = []
    for f, c in zip(*np.nonzero(diff.any(axis=1))):
        first = int(np.argmax(diff[f, :, c]))
        out.append((int(f), int(c), first, int(diff[f, :, c].sum()), int(d[f, first, c] - s[f, first, c])))
    return out


def as_tuples(report):
    return [(int(e["frame"]), int(e["channel"]), int(e["first_sample"]), int(e["n_differing"]), int(e["first_delta"]))
            for e in report]


# ------------------------------------------------------------------ CPU --

def test_expected_report_on_the_golden_vectors():
    """The reference decoder departs from the source at sample 1 of frame 0 channel 1 and frame 1 channel 4 of
    oct_reference_lossy, and nowhere on every other golden case."""
    for case in CASES:
        pcm = GOLD["pcm_" + case]
        rep = expected_report(GOLD["decoded_" + case], pcm, pcm.shape[1])
        if case == "oct_reference_lossy":
            assert [(f, c, first) for f, c, first, _, _ in rep] == [(0, 1, 1), (1, 4, 1)]
        else:
            assert rep == [], case


def test_verify_dtype_matches_header():
    assert _lib.VERIFY_DTYPE.itemsize == 16
    assert {n: _lib.VERIFY_DTYPE.fields[n][1] for n in _lib.VERIFY_DTYPE.names} == {
        "frame": 0, "channel": 4, "first_sample": 6, "n_differing": 8, "first_delta": 12}


def test_verify_entry_points_have_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = _lib.lib()
    assert L.selab200_init(0) == -1
    pcm = np.zeros(2048, np.int16)
    descs = np.zeros(1, _lib.DESC_DTYPE)
    words = np.zeros(16, np.uint32)
    rep = np.zeros(1, _lib.VERIFY_DTYPE)
    n = C.c_size_t(0)
    used = C.c_size_t(0)
    blob = np.zeros(1 << 16, np.uint8)
    assert L.selab200_verify_frames(descs.ctypes.data, 1, 1, words.ctypes.data, 16, pcm.ctypes.data, rep.ctypes.data,
                                    1, C.addressof(n)) == -7
    assert L.selab200_encode_container_verified(pcm.ctypes.data, 1, 1, 44100, 16, blob.ctypes.data, blob.size,
                                                C.addressof(used), rep.ctypes.data, 1, C.addressof(n)) == -7
    assert L.selab200_verify_frames_device(descs.ctypes.data, 1, 1, words.ctypes.data, 16, pcm.ctypes.data,
                                           rep.ctypes.data, blob.ctypes.data, blob.ctypes.data, blob.ctypes.data,
                                           blob.size, None) == -7
    h = C.c_void_p(0)
    info = np.zeros(1, _lib.INFO_DTYPE)
    header = np.frombuffer(b"SeLa" + bytes(11), np.uint8).copy()
    assert L.selab200_container_open(header.ctypes.data, header.size, C.addressof(h), info.ctypes.data) == -7
    assert L.selab200_container_verify(None, pcm.ctypes.data, rep.ctypes.data, 1, C.addressof(n)) == -7
    assert L.selab200_verify_workspace_bytes(10, 2) >= L.selab200_decode_workspace_bytes(10, 2) + 10 * 2 * 4096
    import sela_b200
    with pytest.raises(sela_b200.SelaB200Error):
        sela_b200.verify_frames(descs, words, 1, pcm)


# ------------------------------------------------------------------ GPU --

def _stereo_with_difference_frames(n_frames, seed):
    pcm = synth.sine_noise(44100, 2, n_frames=n_frames, seed=seed)
    pcm[FRAME * 2:FRAME * 5, 1] = pcm[FRAME * 2:FRAME * 5, 0] - (pcm[FRAME * 2:FRAME * 5, 1] >> 5)
    return pcm


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_verify_frames_on_golden(case):
    import sela_b200
    pcm = GOLD["pcm_" + case]
    ch = pcm.shape[1]
    descs = GOLD["descs_" + case].view(sela_b200.DESC_DTYPE)
    rep = sela_b200.verify_frames(descs, GOLD["words_" + case], ch, pcm)
    assert as_tuples(rep) == expected_report(GOLD["decoded_" + case], pcm, ch)
    assert (len(rep) == 2) == (case == "oct_reference_lossy")


@pytest.mark.gpu
@pytest.mark.parametrize("case,frame,channel,sample", [
    ("mono_config1", 0, 0, 1234), ("three", 1, 2, 0), ("oct", 0, 5, 2047), ("oct", 1, 0, 77),
    ("stereo", 2, 0, 100), ("stereo", 3, 1, 2000)])
def test_one_flipped_source_sample_is_exactly_one_entry(case, frame, channel, sample):
    """Frames 2 and 3 of the stereo case are difference-coded: a source sample changed on either channel
    reports that channel only (the decoded output is right, the source is not)."""
    import sela_b200
    pcm = GOLD["pcm_" + case].copy()
    ch = pcm.shape[1]
    descs = GOLD["descs_" + case].view(sela_b200.DESC_DTYPE)
    if case == "stereo":
        assert descs.reshape(-1, 2)[frame]["subframe_type"].any()
    old = int(pcm[frame * FRAME + sample, channel])
    pcm[frame * FRAME + sample, channel] = old ^ 0x40
    rep = sela_b200.verify_frames(descs, GOLD["words_" + case], ch, pcm)
    assert as_tuples(rep) == [(frame, channel, sample, 1, old - (old ^ 0x40))]
    assert as_tuples(rep) == expected_report(GOLD["decoded_" + case], pcm, ch)


@pytest.mark.gpu
def test_corrupt_parent_reports_both_channels():
    """A residue word of the parent of a difference-coded subframe changed: the parent decodes wrong, and so does
    the child that is coded against it.  Both appear."""
    import sela_b200
    pcm = _stereo_with_difference_frames(8, seed=3)
    descs, words = sela_b200.encode_frames(pcm, 2)
    d2 = descs.reshape(-1, 2)
    frame = int(np.nonzero(d2["subframe_type"].any(axis=1))[0][0])
    child = int(np.nonzero(d2[frame]["subframe_type"])[0][0])
    parent = int(d2[frame][child]["parent_channel"])
    p = d2[frame][parent]
    found = None
    for w in range(int(p["res_offset"]) + int(p["res_words"]) - 1, int(p["res_offset"]), -1):
        for bit in range(32):
            bad = words.copy()
            bad[w] ^= np.uint32(1 << bit)
            try:
                out = sela_b200.decode_frames(descs, bad, 2)
            except sela_b200.SelaB200Error:
                continue
            exp = expected_report(out, pcm, 2)
            if exp:
                found = (bad, exp)
                break
        if found:
            break
    assert found, "no bit of the parent's residue stream decodes to a wrong but well-formed stream"
    bad, exp = found
    assert sorted({(f, c) for f, c, *_ in exp}) == [(frame, 0), (frame, 1)]
    assert as_tuples(sela_b200.verify_frames(descs, bad, 2, pcm)) == exp


@pytest.mark.gpu
def test_malformed_descriptors_fail_as_decode_does():
    import sela_b200
    pcm = GOLD["pcm_three"]
    for field, value in (("lpc_order", 101), ("samples", 2047), ("res_words", 60000), ("channel", 7)):
        descs = GOLD["descs_three"].view(sela_b200.DESC_DTYPE).copy()
        descs[1][field] = value
        with pytest.raises(sela_b200.SelaB200Error) as e:
            sela_b200.verify_frames(descs, GOLD["words_three"], 3, pcm)
        assert e.value.status == -6, field


def _spliced_oct(n_frames, positions, seed=4):
    """8-channel batch with the two golden lossy frames at `positions` (frame A, B, A, ... in turn)."""
    pcm = synth.sine_noise(48000, 8, n_frames=n_frames, seed=seed).reshape(n_frames, FRAME, 8)
    lossy = LOSSY.reshape(2, FRAME, 8)
    expect = []
    for i, f in enumerate(positions):
        pcm[f] = lossy[i % 2]
        expect.append((f, 1 if i % 2 == 0 else 4))
    return pcm.reshape(-1, 8), sorted(expect)


@pytest.mark.gpu
def test_encode_container_verified_baseline_stereo():
    """BASELINE-sized stereo batch (12 919 frames, several pipeline chunks): same bytes as encode_container, and the
    report equals the NumPy comparison of the decoded output."""
    import sela_b200
    pcm = _stereo_with_difference_frames(12919, seed=1)
    blob, rep = sela_b200.encode_container_verified(pcm, 2, 44100)
    assert blob.tobytes() == sela_b200.encode_container(pcm, 2, 44100).tobytes()
    info, out = sela_b200.decode_container(blob)
    assert as_tuples(rep) == expected_report(out, pcm, 2)
    info2, rep2 = sela_b200.verify_container(blob, pcm)
    assert info2 == info and as_tuples(rep2) == as_tuples(rep)


@pytest.mark.gpu
def test_spliced_lossy_frames_at_the_edges_and_a_chunk_boundary(monkeypatch):
    """The golden lossy frames spliced in at the first frame, both sides of a chunk boundary and the last frame
    (frames are independent: they stay lossy anywhere) -- every host form reports exactly those positions."""
    import sela_b200
    monkeypatch.setenv("SELAB200_CHUNK_FRAMES", "128")
    n = 1000
    pcm, expect = _spliced_oct(n, [0, 127, 128, n - 1])
    blob, rep = sela_b200.encode_container_verified(pcm, 8, 48000)
    assert blob.tobytes() == sela_b200.encode_container(pcm, 8, 48000).tobytes()
    assert [(f, c) for f, c, *_ in as_tuples(rep)] == expect
    descs, words = sela_b200.encode_frames(pcm, 8)
    exp = expected_report(sela_b200.decode_frames(descs, words, 8), pcm, 8)
    assert as_tuples(rep) == exp
    assert as_tuples(sela_b200.verify_frames(descs, words, 8, pcm)) == exp
    assert as_tuples(sela_b200.verify_container(blob, pcm)[1]) == exp
    # capacity: the total always, at most `capacity` entries written
    L = _lib.lib()
    few = np.zeros(2, _lib.VERIFY_DTYPE)
    cnt = C.c_size_t(0)
    p16 = np.ascontiguousarray(pcm, np.int16)
    _lib.check(L.selab200_verify_frames(descs.ctypes.data, n, 8, words.ctypes.data, words.size, p16.ctypes.data,
                                        few.ctypes.data, 2, C.addressof(cnt)))
    assert cnt.value == 4 and as_tuples(few) == exp[:2]


@pytest.mark.gpu
def test_full_file_acceptance():
    """The config-4-shaped 10-minute file: exactly frame 8975 channel 1 and frame 13577 channel 4 do not come back."""
    import sela_b200
    pcm = synth.sine_noise(48000, 8, 600, seed=2)
    blob, rep = sela_b200.encode_container_verified(pcm, 8, 48000)
    assert [(f, c) for f, c, *_ in as_tuples(rep)] == [(8975, 1), (13577, 4)]
    assert all(first == 1 for _, _, first, _, _ in as_tuples(rep))
    info, rep2 = sela_b200.verify_container(blob, pcm)
    assert as_tuples(rep2) == as_tuples(rep)


@pytest.mark.gpu
def test_device_codec_verify_agrees_with_host_forms():
    import torch
    import sela_b200
    from sela_b200.device import DeviceCodec
    n = 300
    pcm, expect = _spliced_oct(n, [0, 150, n - 1], seed=7)
    dev = torch.device("cuda", 0)
    codec = DeviceCodec(n, 8, device=0)
    t = torch.from_numpy(np.ascontiguousarray(pcm).reshape(-1)).to(dev)
    codec.encode(t)
    codec.check_status()
    n_words = int(codec.words_used.item())
    codec.verify(t, n_words)
    rep = codec.verify_report()
    descs, words = sela_b200.encode_frames(pcm, 8)
    assert as_tuples(rep) == as_tuples(sela_b200.verify_frames(descs, words, 8, pcm))
    assert [(f, c) for f, c, *_ in as_tuples(rep)] == expect
    clean = synth.sine_noise(48000, 8, n_frames=n, seed=7).reshape(-1)
    tc = torch.from_numpy(clean).to(dev)
    codec.encode(tc)
    codec.verify(tc, int(codec.words_used.item()))
    assert codec.verify_report().size == 0
    # a decode error surfaces from verify_report
    codec.descs.view(-1, 32)[3, 10] = 7         # samples = 2055
    codec.verify(tc, int(codec.words_used.item()))
    with pytest.raises(sela_b200.SelaB200Error):
        codec.verify_report()


@pytest.mark.gpu
@pytest.mark.parametrize("slots", [[0, 0], pytest.param([0, 1], marks=TWO_GPUS)], ids=["0-0", "0-1"])
def test_two_devices_give_the_same_report_with_global_frames(slots):
    import sela_b200
    n = 1200
    pcm, expect = _spliced_oct(n, [0, 599, 600, n - 1])
    descs, words = sela_b200.encode_frames(pcm, 8, device=0)
    one = as_tuples(sela_b200.verify_frames(descs, words, 8, pcm, device=0))
    blob1, rep1 = sela_b200.encode_container_verified(pcm, 8, 48000, device=0)
    assert [(f, c) for f, c, *_ in one] == expect
    two = as_tuples(sela_b200.verify_frames(descs, words, 8, pcm, device=slots))
    blob2, rep2 = sela_b200.encode_container_verified(pcm, 8, 48000, device=slots)
    _, rep3 = sela_b200.verify_container(blob2, pcm, device=slots)
    assert _lib.lib().selab200_device_count() == 2
    _lib.init(0)
    assert blob1.tobytes() == blob2.tobytes()
    assert two == one == as_tuples(rep1) == as_tuples(rep2) == as_tuples(rep3)


# ------------------------------------------------------------------ CLI --

def _run(*cmd, env=None):
    return subprocess.run([str(c) for c in cmd], capture_output=True, text=True, timeout=600,
                          env=dict(os.environ, **env) if env else None)


@pytest.mark.gpu
def test_cli_verify_and_test_modes(tmp_path):
    if not (BIN / "sela").exists():
        subprocess.run(["make", "-C", str(ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    sela = BIN / "sela"
    lossy_pcm, _ = _spliced_oct(5, [1, 3])
    clean_pcm = _stereo_with_difference_frames(9, seed=2)
    wavio.write_wav(tmp_path / "lossy.wav", np.concatenate([lossy_pcm, lossy_pcm[:300]]), 48000)  # + a partial frame
    wavio.write_wav(tmp_path / "clean.wav", clean_pcm, 44100)
    for name, lossy in (("lossy", True), ("clean", False)):
        wav = tmp_path / (name + ".wav")
        p = _run(sela, "-V", wav, tmp_path / (name + ".V.sela"))
        assert p.returncode == (2 if lossy else 0), (p.stdout, p.stderr)
        assert _run(sela, "-e", wav, tmp_path / (name + ".e.sela")).returncode == 0
        written = (tmp_path / (name + ".V.sela")).read_bytes()
        assert written == (tmp_path / (name + ".e.sela")).read_bytes()
        if REF_CLI.exists():
            assert _run(REF_CLI, "-e", wav, tmp_path / (name + ".ref.sela")).returncode == 0
            assert written == (tmp_path / (name + ".ref.sela")).read_bytes()
        t = _run(sela, "-t", tmp_path / (name + ".V.sela"), wav)
        assert t.returncode == (2 if lossy else 0), (t.stdout, t.stderr)
        for q in (p, t):
            if lossy:
                lines = [ln for ln in q.stderr.splitlines() if ln.startswith("frame ")]
                assert [ln.split(":")[0] for ln in lines] == ["frame 1 channel 1", "frame 3 channel 4"]
                assert "differs from sample 1 on" in lines[0]
                assert "Verify failed: 2 " in q.stderr
            else:
                assert "Verified" in q.stdout and q.stderr == ""
    # -t refuses a WAV that does not match the header; errors exit with 1
    wavio.write_wav(tmp_path / "mono.wav", clean_pcm[:, :1], 44100)
    wavio.write_wav(tmp_path / "rate.wav", clean_pcm, 48000)
    wavio.write_wav(tmp_path / "short.wav", clean_pcm[:FRAME * 8], 44100)
    for wav, msg in (("mono.wav", "channels"), ("rate.wav", "sample rate"), ("short.wav", "whole frames")):
        t = _run(sela, "-t", tmp_path / "clean.V.sela", tmp_path / wav)
        assert t.returncode == 1 and msg in t.stderr, (wav, t.stderr)
    (tmp_path / "junk.sela").write_bytes(b"NotSela" + bytes(40))
    t = _run(sela, "-t", tmp_path / "junk.sela", tmp_path / "clean.wav")
    assert t.returncode == 1 and "Magic number is incorrect" in t.stderr
    assert "-V" in _run(sela).stdout and "-t" in _run(sela).stdout
