"""Random access: sample-accurate clips from open containers (selab200_container_decode_clips, DESIGN.md 7.8).

The expected value is always the whole-file decode, sliced: decode_container on the GPU and the port's decode
(oracle_lib) of the same container, parsed on the CPU.  The expected frames_decoded is the number of distinct
(container, frame) pairs the clips cover, counted here."""
import ctypes as C
import pathlib
import struct
import subprocess

import numpy as np
import pytest

import oracle_lib as ol
from sela_b200 import ClipDecoder, SelaB200Error, _lib, codec, synth, wavio

ROOT = pathlib.Path(__file__).resolve().parent.parent
BIN = ROOT / "sela_b200" / "host" / "bin"
REF_CLI = ROOT / "oracle" / "_ref" / "sela_ref_cli"
GOLD = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
FRAME = 2048
ARGUMENT, BITSTREAM = -3, -6


def parse_container(blob):
    """CPU parse of a .sela byte stream -> (channels, descriptors, words), the layout the encoder returns."""
    blob = bytes(blob)
    channels, n_frames = blob[10], struct.unpack_from("<I", blob, 11)[0]
    at, words, descs = 15, [], []
    for _ in range(n_frames):
        assert blob[at:at + 4] == wavio.SELA_SYNC
        at += 4
        for _ in range(channels):
            ch, typ, parent, rk, rn, order = struct.unpack_from("<BBBBHB", blob, at)
            refl = np.frombuffer(blob, "<u4", rn, at + 7)
            at += 7 + 4 * rn
            k, n, samples = struct.unpack_from("<BHH", blob, at)
            res = np.frombuffer(blob, "<u4", n, at + 5)
            at += 5 + 4 * n
            off = sum(w.size for w in words)
            descs.append((ch, typ, parent, rk, rn, order, k, n, samples, 0, off, off + rn))
            words += [refl, res]
    d = np.array(descs, dtype=_lib.DESC_DTYPE)
    return channels, d, (np.concatenate(words) if words else np.zeros(0, np.uint32)).astype(np.uint32)


def expected(blobs):
    """Per container: [n_frames * 2048, channels] of decode_container, after checking it against the port's decode."""
    O = ol.load("port")
    out = []
    for b in blobs:
        info, pcm = codec.decode_container(b)
        ch, d, w = parse_container(b)
        assert np.array_equal(pcm, O.decode_frames(d, w, ch).reshape(-1))
        out.append(pcm.reshape(-1, info["channels"]))
    return out


def covered(containers, starts, length):
    pairs = set()
    for c, s in zip(np.broadcast_to(containers, np.shape(starts)).tolist(), list(starts)):
        pairs.update((c, f) for f in range(s // FRAME, (s + length - 1) // FRAME + 1))
    return len(pairs)


def check_clips(dec, whole, containers, starts, length, device=False):
    containers = np.broadcast_to(np.asarray(containers), np.shape(starts))
    got = dec.decode_device(containers, starts, length).cpu().numpy() if device else dec.decode(containers, starts,
                                                                                                   length)
    want = np.stack([whole[c][s:s + length] for c, s in zip(containers.tolist(), list(starts))])
    assert got.shape == want.shape and np.array_equal(got, want)
    assert dec.frames_decoded == covered(containers, starts, length)
    return got


def _pcm(channels, n_frames, seed):
    pcm = synth.sine_noise(44100, channels, n_frames=n_frames, seed=seed)
    if channels >= 2:
        pcm[FRAME:FRAME * 4, 1] = pcm[FRAME:FRAME * 4, 0] - (pcm[FRAME:FRAME * 4, 1] >> 5)
    return pcm


def _raw(dec, clips, length, out, device=False):
    """The C call itself, on arrays the test owns: (status, frames_decoded, last error)."""
    L = _lib.lib()
    n = C.c_uint64(12345)
    fn = L.selab200_container_decode_clips_device if device else L.selab200_container_decode_clips
    rc = fn(C.addressof(dec._array), len(dec._handles), clips.ctypes.data if clips is not None else None,
            0 if clips is None else clips.size, length, out, C.addressof(n))
    return rc, n.value, L.selab200_last_error().decode()


def _clips(pairs):
    c = np.zeros(len(pairs), _lib.CLIP_DTYPE)
    for i, (k, s) in enumerate(pairs):
        c[i]["container"], c[i]["start"] = k, s
    return c


# ------------------------------------------------------------------ CPU --

def test_clip_dtype_layout():
    d = _lib.CLIP_DTYPE
    assert d.itemsize == 16
    assert (d.fields["container"][1], d.fields["reserved"][1], d.fields["start"][1]) == (0, 4, 8)
    header = _lib.HEADER_PATH.read_text()
    assert "typedef struct selab200_clip {   /* 16 bytes */" in header


def test_entry_points_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = _lib.lib()
    assert L.selab200_init(0) == -1
    clips = _clips([(0, 0)])
    out = np.zeros(16, np.int16)
    n = C.c_uint64(0)
    handles = (C.c_void_p * 1)()
    for fn in (L.selab200_container_decode_clips, L.selab200_container_decode_clips_device):
        rc = fn(C.addressof(handles), 1, clips.ctypes.data, 1, 8, out.ctypes.data, C.addressof(n))
        assert rc in (-1, -7)        # NO_DEVICE / NOT_INIT: nothing computed on the CPU
    assert not out.any()


# ------------------------------------------------------------------ GPU --

@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 2, 3, 8])
def test_clip_shapes(channels):
    """Forced clip shapes and seeded random ones from three containers, interleaved, against both expected values."""
    blobs = [codec.encode_container(_pcm(channels, n, 10 + channels + n), channels, 44100) for n in (9, 5, 12)]
    whole = expected(blobs)
    total = [w.shape[0] for w in whole]
    rng = np.random.default_rng(channels)
    forced = [(0, 0, 1), (0, 0, 2048), (1, 2048, 2048), (2, 100, 2048), (0, total[0] - 1, 1),
              (1, total[1] - 2048, 2048), (2, total[2] - 777, 777), (0, 2047, 2), (0, 4095, 3)]
    for k in range(3):
        for n in (1, 3, 5, 7, 9, 15, 17, 4097, 3 * FRAME + 5):     # every byte phase of the gather, both sides
            for s in (0, 1, 3, 7, 2041, 4093):
                if s + n <= total[k]:
                    forced.append((k, s, n))
    with ClipDecoder(blobs) as dec:
        assert [i["n_frames"] for i in dec.info] == [9, 5, 12] and dec.channels == channels
        for k, s, n in forced:
            check_clips(dec, whole, [k], [s], n)
        for length in (1, 6, 2048, 5000, 11 * FRAME + 3):
            ks = rng.integers(0, 3, 40)
            ks = ks[[t for t in range(40) if total[ks[t]] >= length]]
            starts = [int(rng.integers(0, total[k] - length + 1)) for k in ks]
            # duplicates, nested and overlapping clips
            ks = np.concatenate([ks, ks[:5], ks[:5]])
            starts = starts + starts[:5] + [min(s + 1, total[k] - length) for k, s in zip(ks[:5], starts[:5])]
            got = check_clips(dec, whole, ks, starts, length)
            assert np.array_equal(got, check_clips(dec, whole, ks, starts, length, device=True))
        # a clip nested in another, one across many frame boundaries, and a whole container
        check_clips(dec, whole, [2, 2, 2], [0, 4000, 4100], 9 * FRAME)
        check_clips(dec, whole, [1], [0], total[1])


def _mode_blobs():
    pcm8 = synth.sine_noise(44100, 8, n_frames=4, seed=21)
    pcm8[:, 5] = pcm8[:, 3] - (pcm8[:, 5] >> 6)          # channel 5 follows channel 3: a difference, parent 3
    pcm2 = _pcm(2, 7, 22)
    return {
        "e": codec.encode_container(pcm2, 2, 44100),
        "L": codec.encode_container_lossless(pcm2, 2, 44100)[0],
        "S": codec.encode_container_search(pcm2, 2, 44100)[0],
        "P": codec.encode_container_pairing(pcm8, 8, 44100)[0],
        "B": codec.encode_container_search_pairing(pcm2, 2, 44100)[0],
        "W": codec.encode_container_search_windows(pcm2, 2, 44100)[0],
        "F": codec.encode_container_search_guided(pcm2, 2, 44100)[0],
    }


@pytest.mark.gpu
def test_every_encode_mode():
    blobs = _mode_blobs()
    _, d, _ = parse_container(blobs["P"])
    assert ((d["subframe_type"] == 1) & (d["parent_channel"] != 0)).any()
    rng = np.random.default_rng(3)
    for mode, blob in blobs.items():
        whole = expected([blob])
        total = whole[0].shape[0]
        with ClipDecoder([blob]) as dec:
            starts = [0, total - 3001] + [int(s) for s in rng.integers(0, total - 3001, 20)]
            check_clips(dec, whole, 0, starts, 3001)
            check_clips(dec, whole, 0, starts, 3001, device=True)


@pytest.mark.gpu
def test_lossy_reference_frames():
    """Clips over frames the reference decoder does not decode back to their source equal the reference output."""
    blob = wavio.pack_container(GOLD["descs_oct_reference_lossy"], GOLD["words_oct_reference_lossy"], 44100, 8)
    ref = GOLD["decoded_oct_reference_lossy"].reshape(-1, 8)
    src = GOLD["pcm_oct_reference_lossy"].reshape(-1, 8)
    with ClipDecoder([blob]) as dec:
        for s, n in ((0, 4096), (1000, 3000), (2040, 9)):
            got = dec.decode(0, [s], n)[0]
            assert np.array_equal(got, ref[s:s + n])
        assert not np.array_equal(dec.decode(0, [0], 4096)[0], src)


@pytest.mark.gpu
def test_malformed_frame_fails_only_clips_that_cover_it():
    pcm = _pcm(2, 8, 5)
    blob = codec.encode_container(pcm, 2, 44100)
    _, d, _ = parse_container(blob)
    at = 15 + 4 * (5 + 1) + 12 * (5 * 2 + 1) + 4 * int(d[5 * 2 + 1]["refl_offset"])   # frame 5, subframe 1
    bad = bytearray(blob)
    bad[at + 6] = 101                                      # its order byte: the walk accepts it, the device does not
    assert codec.container_info(bytes(bad))["n_frames"] == 8
    with pytest.raises(SelaB200Error) as e:
        codec.decode_container(bytes(bad))
    assert e.value.status == BITSTREAM
    whole = expected([blob])
    with ClipDecoder([bytes(bad)]) as dec:
        for s, n in ((0, 5 * FRAME), (6 * FRAME, 2 * FRAME), (100, 3000), (7 * FRAME - 10, 50)):
            check_clips(dec, whole, 0, [s], n)
        for s, n in ((5 * FRAME, 1), (5 * FRAME - 1, 2), (0, 8 * FRAME), (6 * FRAME - 1, 1)):
            with pytest.raises(SelaB200Error) as e:
                dec.decode(0, [s], n)
            assert e.value.status == BITSTREAM, (s, n)
        check_clips(dec, whole, 0, [0, 6 * FRAME], 100)   # the decoder is usable after a failed call


@pytest.mark.gpu
def test_rejections_leave_the_output_alone():
    blobs = [codec.encode_container(_pcm(2, n, 30 + n), 2, 44100) for n in (3, 4)]
    mono = codec.encode_container(_pcm(1, 2, 33), 1, 44100)
    total = [3 * FRAME, 4 * FRAME]
    whole = expected(blobs)
    with ClipDecoder(blobs) as dec:
        out = np.full(4 * 2 * 64 + 16, 0x5A5A, np.int16)

        def call(pairs, length, reserved=None, buf=out):
            c = _clips(pairs)
            if reserved is not None:
                c[reserved]["reserved"] = 1
            return _raw(dec, c, length, buf.ctypes.data if buf is not None else None)

        ok = [(0, 0), (1, total[1] - 64), (0, 5), (1, 7)]
        assert call(ok, 64)[:2] == (0, 3)         # frames (0, 0), (1, 0) and (1, 3)
        got = out[:4 * 64 * 2].reshape(4, 64, 2)
        assert np.array_equal(got, np.stack([whole[k][s:s + 64] for k, s in ok]))
        assert (out[4 * 64 * 2:] == 0x5A5A).all()
        cases = [
            (ok[:3] + [(0, total[0] - 64 + 1)], 64, None, "clip 3"),   # one sample past the end
            (ok[:2] + [(2, 0), (0, 0)], 64, None, "clip 2"),             # container index == n_handles
            (ok, 64, 1, "clip 1"),                                       # reserved field
            (ok, 0, None, "clip 0"),                                     # length 0
            ([(0, total[0])], 1, None, "clip 0"),                        # starts at the end
            ([(0, 2 ** 64 - 1)], 2, None, "clip 0"),                     # start + length wraps 64 bits
        ]
        for pairs, length, reserved, where in cases:
            out[:] = 0x1234
            rc, n, err = call(pairs, length, reserved)
            assert rc == ARGUMENT and where in err and n == 0, (pairs, length, err)
            assert (out == 0x1234).all()
        # at the limits: ends exactly at the end, last container index, length 1
        assert call([(0, total[0] - 64), (1, total[1] - 64)], 64)[0] == 0
        assert call([(1, total[1] - 1)], 1)[0] == 0
        # null pointers, and the empty batch
        assert call(ok, 64, buf=None)[0] == ARGUMENT
        L = _lib.lib()
        n = C.c_uint64(0)
        c = _clips(ok)
        assert L.selab200_container_decode_clips(None, 2, c.ctypes.data, 4, 64, out.ctypes.data, C.addressof(n)) \
            == ARGUMENT
        assert L.selab200_container_decode_clips(C.addressof(dec._array), 2, None, 4, 64, out.ctypes.data,
                                                 C.addressof(n)) == ARGUMENT
        assert L.selab200_container_decode_clips(C.addressof(dec._array), 2, c.ctypes.data, 4, 64, out.ctypes.data,
                                                 None) == ARGUMENT
        out[:] = 0x1234
        assert _raw(dec, None, 64, out.ctypes.data)[:2] == (0, 0)
        assert (out == 0x1234).all()
        assert dec.decode(0, [], 64).shape == (0, 64, 2)
    with ClipDecoder([blobs[0], mono]) as dec:               # channel counts differ
        out[:] = 0x1234
        rc, _, err = _raw(dec, _clips([(0, 0)]), 8, out.ctypes.data)
        assert rc == ARGUMENT and "channels" in err and (out == 0x1234).all()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk_frames", [None, "3"])
def test_large_batch(monkeypatch, chunk_frames):
    """4096 clips over 16 containers; with SELAB200_CHUNK_FRAMES=3 the selection takes many groups and chunks."""
    if chunk_frames:
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", chunk_frames)
    blobs = [codec.encode_container(_pcm(2, 6 + k % 5, 50 + k), 2, 44100) for k in range(16)]
    whole = expected(blobs)
    rng = np.random.default_rng(9)
    length = 1500
    ks = rng.integers(0, 16, 4096)
    starts = [int(rng.integers(0, whole[k].shape[0] - length + 1)) for k in ks]
    with ClipDecoder(blobs) as dec:
        clips = _clips(list(zip(ks.tolist(), starts)))
        out = np.full(4096 * length * 2 + 64, 0x2B2B, np.int16)
        rc, n, err = _raw(dec, clips, length, out.ctypes.data)
        assert rc == 0, err
        want = np.stack([whole[k][s:s + length] for k, s in zip(ks.tolist(), starts)])
        assert np.array_equal(out[:-64].reshape(want.shape), want)
        assert (out[-64:] == 0x2B2B).all()
        assert n == covered(ks, starts, length)
        got = dec.decode_device(ks, starts, length).cpu().numpy()
        assert np.array_equal(got, want) and dec.frames_decoded == n


@pytest.mark.gpu
def test_right_after_open_and_on_two_devices():
    """A call straight after the open of a long file (its upload still running), and with two devices initialised
    the same result as with one."""
    import torch
    pcm = synth.sine_noise(44100, 2, seconds=600, seed=1)
    blob = codec.encode_container(pcm, 2, 44100)
    other = codec.encode_container(_pcm(2, 7, 2), 2, 44100)
    n_frames = pcm.shape[0] // FRAME
    starts = [n_frames * FRAME - 44100, 0, 12345678, n_frames * FRAME // 2]
    want = np.stack([pcm[s:s + 44100] for s in starts])    # BASELINE frames decode back to their source
    with ClipDecoder([blob]) as dec:
        assert np.array_equal(dec.decode(0, starts, 44100), want)
    with ClipDecoder([blob]) as dec:
        assert np.array_equal(dec.decode_device(0, starts, 44100).cpu().numpy(), want)
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the two-device case needs two")
    whole = expected([blob, other])
    try:
        with ClipDecoder([blob, other], device=[0, 1]) as dec:
            got = check_clips(dec, whole, [1, 0, 1], [0, 99999, 5000], 4000)
            assert np.array_equal(got, check_clips(dec, whole, [1, 0, 1], [0, 99999, 5000], 4000, device=True))
    finally:
        _lib.init(0)
    with ClipDecoder([blob, other]) as dec:
        assert np.array_equal(dec.decode([1, 0, 1], [0, 99999, 5000], 4000), got)


@pytest.mark.gpu
def test_cli_range(tmp_path):
    if not (BIN / "sela").exists():
        subprocess.run(["make", "-C", str(ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    pcm = _pcm(2, 9, 41)
    wavio.write_wav(tmp_path / "in.wav", pcm, 44100)

    def run(*args):
        p = subprocess.run([str(a) for a in args], capture_output=True, text=True, timeout=300)
        assert p.returncode == 0, (args, p.stdout[-300:], p.stderr[-300:])

    run(BIN / "sela", "-e", tmp_path / "in.wav", tmp_path / "a.sela")
    run(BIN / "sela", "-d", tmp_path / "a.sela", tmp_path / "full.wav")
    full = (tmp_path / "full.wav").read_bytes()
    wavs = [full]
    if REF_CLI.exists():
        run(REF_CLI, "-d", tmp_path / "a.sela", tmp_path / "ref.wav")
        wavs.append((tmp_path / "ref.wav").read_bytes())
    for first, count in ((0, 9 * FRAME), (0, 1), (5000, 7777), (9 * FRAME - 3, 3)):
        run(BIN / "sela", "-R", tmp_path / "a.sela", tmp_path / "r.wav", first, count)
        got = (tmp_path / "r.wav").read_bytes()
        for w in wavs:
            assert got[:4] == w[:4] and got[8:40] == w[8:40]          # every header field but the two sizes
            assert struct.unpack_from("<I", got, 4)[0] == 36 + 4 * count
            assert struct.unpack_from("<I", got, 40)[0] == 4 * count
            assert got[44:] == w[44 + 4 * first:44 + 4 * (first + count)]
    p = subprocess.run([str(BIN / "sela"), "-R", str(tmp_path / "a.sela"), str(tmp_path / "r.wav"), "18000", "500"],
                       capture_output=True, text=True, timeout=300)
    assert p.returncode == 1 and "clip 0" in p.stderr
