"""Clips of chosen channels, as int16, float32 or a float32 mean (selab200_container_decode_clips_select, DESIGN.md 7.9).

The expected value is the whole-file decode sliced, as in test_decode_clips.py, with the columns picked and converted
in NumPy; every comparison is exact, float32 included.  The expected subframes_decoded is counted here from the parsed
descriptors: per covered frame the selected channels' subframes and the parents of the selected difference-coded ones."""
import ctypes as C
import pathlib
import struct
import subprocess

import numpy as np
import pytest

import test_decode_clips as base
from sela_b200 import ClipDecoder, SelaB200Error, _lib, clips as clips_mod, codec, synth, wavio

FRAME = base.FRAME
ARGUMENT, BITSTREAM = base.ARGUMENT, base.BITSTREAM
F32, MEAN = _lib.CLIP_FLOAT32, _lib.CLIP_MEAN
KINDS = [(np.int16, False), (np.float32, False), (np.float32, True)]


def pick(x, sel, dtype, mean):
    """x: [..., length, C] int16 -> the selected columns, converted as the rule says."""
    cols = x[..., list(range(x.shape[-1])) if sel is None else list(sel)]
    if mean:
        s = cols.astype(np.int64).sum(-1, keepdims=True)
        return s.astype(np.float32) / np.float32(32768 * cols.shape[-1])
    return cols.astype(np.float32) / np.float32(32768) if dtype == np.float32 else cols


def needed(descs, channels, frames, sel):
    """Subframes decoded for the given frames of one container: selected ones plus parents of selected differences."""
    n = 0
    for f in frames:
        fd = descs[f * channels:(f + 1) * channels]
        pos = {int(fd[p]["channel"]): p for p in range(channels)}
        need = set()
        for c in (range(channels) if sel is None else sel):
            p = pos[c]
            need.add(p)
            if fd[p]["subframe_type"] == 1:
                need.add(pos[int(fd[p]["parent_channel"])])
        n += len(need)
    return n


def covered_frames(containers, starts, length):
    pairs = set()
    for c, s in zip(np.broadcast_to(containers, np.shape(starts)).tolist(), list(starts)):
        pairs.update((c, f) for f in range(s // FRAME, (s + length - 1) // FRAME + 1))
    return pairs


def check_select(dec, whole, parsed, containers, starts, length, sel, dtype, mean, device=False):
    containers = np.broadcast_to(np.asarray(containers), np.shape(starts))
    if device:
        import torch
        got = dec.decode_device(containers, starts, length, channels=sel,
                                dtype=torch.float32 if dtype == np.float32 else torch.int16, mean=mean).cpu().numpy()
    else:
        got = dec.decode(containers, starts, length, channels=sel, dtype=dtype, mean=mean)
    want = np.stack([pick(whole[c][s:s + length], sel, dtype, mean) for c, s in zip(containers.tolist(), list(starts))])
    assert got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got, want), (sel, dtype, mean)
    pairs = covered_frames(containers, starts, length)
    assert dec.frames_decoded == len(pairs)
    by_container = {}
    for c, f in pairs:
        by_container.setdefault(c, []).append(f)
    assert dec.subframes_decoded == sum(needed(parsed[c][1], parsed[c][0], fs, sel) for c, fs in by_container.items())
    return got


def _raw(dec, clips, length, sel, flags, out, device=False):
    """The C call itself: (status, frames_decoded, subframes_decoded, last error)."""
    L = _lib.lib()
    n, m = C.c_uint64(12345), C.c_uint64(6789)
    fn = L.selab200_container_decode_clips_select_device if device else L.selab200_container_decode_clips_select
    s = None if sel is None else np.ascontiguousarray(sel, np.uint8)
    rc = fn(C.addressof(dec._array), len(dec._handles), clips.ctypes.data if clips is not None else None,
            0 if clips is None else clips.size, length, s.ctypes.data if s is not None else None,
            0 if s is None else s.size, flags, out, C.addressof(n), C.addressof(m))
    return rc, n.value, m.value, L.selab200_last_error().decode()


# ------------------------------------------------------------------ CPU --

def test_select_entry_points_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = _lib.lib()
    assert L.selab200_init(0) == -1
    clips = base._clips([(0, 0)])
    out = np.zeros(16, np.float32)
    n, m = C.c_uint64(0), C.c_uint64(0)
    handles = (C.c_void_p * 1)()
    sel = np.zeros(1, np.uint8)
    for fn in (L.selab200_container_decode_clips_select, L.selab200_container_decode_clips_select_device):
        rc = fn(C.addressof(handles), 1, clips.ctypes.data, 1, 8, sel.ctypes.data, 1, F32, out.ctypes.data,
                C.addressof(n), C.addressof(m))
        assert rc in (-1, -7)        # NO_DEVICE / NOT_INIT: nothing computed on the CPU
    assert not out.any()


def test_python_arguments_raise_before_any_call(monkeypatch):
    import torch

    def no_call():
        raise AssertionError("the library was called")

    dec = ClipDecoder.__new__(ClipDecoder)
    dec._handles, dec._bufs, dec.info, dec.channels, dec.device = [1], [], [{"channels": 2}], 2, 0
    dec._array = (C.c_void_p * 1)(1)
    monkeypatch.setattr(clips_mod, "lib", no_call)
    bad = [dict(dtype=np.float64), dict(dtype=np.int32), dict(mean=True), dict(mean=True, dtype=np.int16),
           dict(channels=[]), dict(channels=[256]), dict(channels=[-1]), dict(channels=[0] * 256)]
    for kw in bad:
        with pytest.raises(ValueError):
            dec.decode(0, [0], 16, **kw)
    for kw in (dict(dtype=torch.float64), dict(dtype=torch.int32), dict(mean=True), dict(channels=[300])):
        with pytest.raises(ValueError):
            dec.decode_device(0, [0], 16, **kw)
    with pytest.raises(ValueError):                       # the clip arguments are checked before the call too
        dec.decode(0, [0], 1 << 32, channels=[0])
    dec._handles = []


# ------------------------------------------------------------------ GPU --

def _selections(channels):
    sels = [[c] for c in range(channels)] + [list(range(channels)), list(range(channels))[::-1], None]
    sels += [[0, 0], [channels - 1, 0, channels - 1]]
    return sels


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 2, 3, 8])
def test_select_shapes(channels):
    """Every kind of output and selection, clips of many byte phases from three containers, both forms."""
    blobs = [codec.encode_container(base._pcm(channels, n, 10 + channels + n), channels, 44100) for n in (9, 5, 12)]
    whole = base.expected(blobs)
    parsed = [base.parse_container(b) for b in blobs]
    total = [w.shape[0] for w in whole]
    shapes = [([0], [0], 1), ([2], [total[2] - 777], 777), ([0, 1, 2, 0], [1, 3, 2041, 4093], 17),
              ([1, 2, 0], [7, 100, 2047], 2 * FRAME + 5), ([2, 2], [0, 4000], 9 * FRAME), ([1], [0], total[1])]
    with ClipDecoder(blobs) as dec:
        for sel in _selections(channels):
            for dtype, mean in KINDS:
                for ks, starts, n in shapes:
                    got = check_select(dec, whole, parsed, ks, starts, n, sel, dtype, mean)
                    dev = check_select(dec, whole, parsed, ks, starts, n, sel, dtype, mean, device=True)
                    assert np.array_equal(got, dev)
        # every output phase of the device form: the output starts 2 (int16) or 4 (float32) bytes past alignment
        import torch
        clips = base._clips([(1, 5), (0, 2049)])
        for sel, flags, size in (([0], 0, 2), ([channels - 1, 0], 0, 2), ([0], F32, 4), (None, F32 | MEAN, 4)):
            n_out = 1 if flags & MEAN else len(sel)
            for shift in range(0, 16, size):
                buf = torch.zeros(2 * 3001 * n_out * size + 32, dtype=torch.uint8, device="cuda")
                rc, _, _, err = _raw(dec, clips, 3001, sel, flags, buf.data_ptr() + shift, device=True)
                assert rc == 0, err
                raw = buf.cpu().numpy()
                got = raw[shift:shift + 2 * 3001 * n_out * size].view(np.float32 if flags & F32 else np.int16)
                want = np.stack([pick(whole[k][s:s + 3001], sel, np.float32 if flags & F32 else np.int16,
                                      bool(flags & MEAN)) for k, s in ((1, 5), (0, 2049))])
                assert np.array_equal(got.reshape(want.shape), want)
                assert not raw[:shift].any() and not raw[shift + 2 * 3001 * n_out * size:].any()


@pytest.mark.gpu
def test_full_selection_equals_decode_clips():
    blobs = [codec.encode_container(base._pcm(3, n, 60 + n), 3, 44100) for n in (6, 4)]
    rng = np.random.default_rng(4)
    with ClipDecoder(blobs) as dec:
        ks = rng.integers(0, 2, 50)
        starts = [int(rng.integers(0, (6 if k == 0 else 4) * FRAME - 2500)) for k in ks]
        clips = base._clips(list(zip(ks.tolist(), starts)))
        a = np.full(50 * 2500 * 3 + 8, 0x3C3C, np.int16)
        b = a.copy()
        assert base._raw(dec, clips, 2500, a.ctypes.data)[0] == 0
        rc, frames, subs, err = _raw(dec, clips, 2500, None, 0, b.ctypes.data)
        assert rc == 0, err
        assert np.array_equal(a, b)
        assert frames == base.covered(ks, starts, 2500) and subs == 3 * frames


@pytest.mark.gpu
def test_every_encode_mode():
    """Every channel alone, and the mean, in files of every encode mode; in the -P file channel 5 is a difference
    from channel 3, so selecting it alone decodes its parent without returning it."""
    blobs = base._mode_blobs()
    _, d, _ = base.parse_container(blobs["P"])
    fd = d.reshape(-1, 8)
    assert ((fd["subframe_type"] == 1) & (fd["channel"] == 5) & (fd["parent_channel"] == 3)).any()
    rng = np.random.default_rng(3)
    for mode, blob in blobs.items():
        whole = base.expected([blob])
        parsed = [base.parse_container(blob)]
        ch = parsed[0][0]
        total = whole[0].shape[0]
        starts = [0, total - 3001] + [int(s) for s in rng.integers(0, total - 3001, 6)]
        with ClipDecoder([blob]) as dec:
            for c in range(ch):
                check_select(dec, whole, parsed, 0, starts, 3001, [c], np.int16, False)
            check_select(dec, whole, parsed, 0, starts, 3001, None, np.float32, True, device=True)
            check_select(dec, whole, parsed, 0, starts, 3001, [ch - 1, 0], np.float32, False, device=True)
        if mode == "P":
            with ClipDecoder([blob]) as dec:
                dec.decode(0, [0], 4 * FRAME, channels=[5])
                diffs = int((fd["subframe_type"][fd["channel"] == 5] == 1).sum())
                assert dec.subframes_decoded == 4 + diffs          # channel 5 in every frame, its parent where coded


@pytest.mark.gpu
def test_permuted_subframe_order():
    """Subframes stored in the order channel 2, 0, 1, and channel 0 a difference from channel 2 (a parent with a
    higher channel number, stored in front of it)."""
    pcm = synth.sine_noise(44100, 3, n_frames=5, seed=77)
    descs, words = codec.encode_frames(pcm, 3)
    d = descs.copy().reshape(-1, 3)
    d["subframe_type"][:, 0], d["parent_channel"][:, 0] = 1, 2
    crafted = d[:, [2, 0, 1]].reshape(-1)
    blob = wavio.pack_container(crafted, words, 44100, 3)
    whole = base.expected([blob])
    x = pcm.reshape(-1, 3)
    want = x.copy()
    want[:, 0] = (x[:, 2].astype(np.int32) - x[:, 0]).astype(np.uint16).view(np.int16)
    assert np.array_equal(whole[0], want)
    parsed = [base.parse_container(blob)]
    with ClipDecoder([blob]) as dec:
        for sel in ([0], [1], [2], [0, 1], [1, 0, 2], None):
            for dtype, mean in KINDS:
                check_select(dec, whole, parsed, [0, 0], [3, 2 * FRAME - 7], 2 * FRAME + 1, sel, dtype, mean)
        dec.decode(0, [0], 5 * FRAME, channels=[0])
        assert dec.subframes_decoded == 10
        dec.decode(0, [0], 5 * FRAME, channels=[1])
        assert dec.subframes_decoded == 5


@pytest.mark.gpu
def test_lossy_reference_frames():
    blob = wavio.pack_container(base.GOLD["descs_oct_reference_lossy"], base.GOLD["words_oct_reference_lossy"],
                                44100, 8)
    ref = base.GOLD["decoded_oct_reference_lossy"].reshape(-1, 8)
    src = base.GOLD["pcm_oct_reference_lossy"].reshape(-1, 8)
    lossy = [c for c in range(8) if not np.array_equal(ref[:, c], src[:, c])]
    assert lossy
    with ClipDecoder([blob]) as dec:
        for s, n in ((0, 4096), (1000, 3000), (2040, 9)):
            for sel in ([c] for c in range(8)):
                assert np.array_equal(dec.decode(0, [s], n, channels=sel)[0], ref[s:s + n][:, sel])
            assert np.array_equal(dec.decode(0, [s], n, channels=lossy[::-1])[0], ref[s:s + n][:, lossy[::-1]])
            assert np.array_equal(dec.decode(0, [s], n, dtype=np.float32, mean=True)[0],
                                  pick(ref[s:s + n], None, np.float32, True))


@pytest.mark.gpu
def test_subframe_counts_default_encode():
    blob = codec.encode_container(synth.sine_noise(44100, 8, n_frames=10, seed=8), 8, 44100)
    with ClipDecoder([blob]) as dec:
        dec.decode(0, [100, 7000], 9000, dtype=np.float32)
        full = dec.subframes_decoded
        frames = dec.frames_decoded
        dec.decode(0, [100, 7000], 9000, channels=[6])
        assert dec.subframes_decoded * 8 == full and dec.frames_decoded == frames


@pytest.mark.gpu
def test_mixed_channel_counts():
    blobs = [codec.encode_container(base._pcm(c, n, 80 + c), c, 44100) for c, n in ((1, 4), (2, 5), (8, 3))]
    whole = base.expected(blobs)
    parsed = [base.parse_container(b) for b in blobs]
    ks, starts = [0, 1, 2, 1, 0, 2], [0, 3000, 10, 7000, 4000, 2 * FRAME]
    with ClipDecoder(blobs) as dec:
        for dtype in (np.int16, np.float32):
            check_select(dec, whole, parsed, ks, starts, 2000, [0], dtype, False)
            check_select(dec, whole, parsed, ks, starts, 2000, [0], dtype, False, device=True)
        check_select(dec, whole, parsed, ks, starts, 2000, None, np.float32, True)
        check_select(dec, whole, parsed, ks, starts, 2000, None, np.float32, True, device=True)
        check_select(dec, whole, parsed, ks, starts, 2000, [0, 0], np.float32, True)
        with pytest.raises(SelaB200Error) as e:           # every channel as int16 needs one channel count
            dec.decode(ks, starts, 2000)
        assert e.value.status == ARGUMENT
        with pytest.raises(SelaB200Error) as e:
            dec.decode(ks, starts, 2000, dtype=np.float32)
        assert e.value.status == ARGUMENT
        with pytest.raises(SelaB200Error) as e:           # channel 1 is past the mono container's channels
            dec.decode(ks, starts, 2000, channels=[1])
        assert e.value.status == ARGUMENT
        check_select(dec, whole, parsed, [1, 2], [0, 5], 3000, [1], np.int16, False)
        check_select(dec, whole, parsed, [2, 2], [0, 5], 3000, None, np.float32, False)


def _corrupt_residues(blob, descs, channels, frame, pos):
    """Every residue word of the subframe at `pos` of `frame` set to ones: its Rice stream runs past its end."""
    sub = frame * channels + pos
    at = 15 + 4 * (frame + 1) + 12 * (sub + 1) + 4 * int(descs[sub]["res_offset"])
    bad = bytearray(blob)
    bad[at:at + 4 * int(descs[sub]["res_words"])] = b"\xff" * (4 * int(descs[sub]["res_words"]))
    return bytes(bad)


@pytest.mark.gpu
def test_malformed_subframes():
    # a header-rule violation in an unselected subframe fails every call that covers its frame
    pcm = synth.sine_noise(44100, 3, n_frames=6, seed=90)
    blob = codec.encode_container(pcm, 3, 44100)
    whole = base.expected([blob])
    parsed = [base.parse_container(blob)]
    _, d, _ = parsed[0]
    assert (d["subframe_type"] == 0).all()
    sub = 4 * 3 + 2                                       # frame 4, position 2
    at = 15 + 4 * 5 + 12 * sub + 4 * int(d[sub]["refl_offset"])
    bad = bytearray(blob)
    bad[at + 6] = 101                                     # its order byte: the walk accepts it, the rules do not
    other = int(d[sub]["channel"])
    keep = [c for c in range(3) if c != other]
    with ClipDecoder([bytes(bad)]) as dec:
        for s, n in ((4 * FRAME, 1), (3 * FRAME, 2 * FRAME)):
            with pytest.raises(SelaB200Error) as e:
                dec.decode(0, [s], n, channels=keep)
            assert e.value.status == BITSTREAM
        check_select(dec, whole, parsed, 0, [0, 5 * FRAME], FRAME, keep, np.int16, False)   # uncovered: no failure

    # a stream-level fault: only a decoded subframe fails the call
    sub = 2 * 3 + 1
    bad = _corrupt_residues(blob, d, 3, 2, 1)
    with pytest.raises(SelaB200Error) as e:
        codec.decode_container(bad)
    assert e.value.status == BITSTREAM
    faulty = int(d[sub]["channel"])
    keep = [c for c in range(3) if c != faulty]
    with ClipDecoder([bad]) as dec:
        for dtype, mean in KINDS:
            check_select(dec, whole, parsed, 0, [0, 2 * FRAME + 5], 3 * FRAME, keep, dtype, mean)
        for sel in ([faulty], keep + [faulty], None):
            with pytest.raises(SelaB200Error) as e:
                dec.decode(0, [2 * FRAME + 100], 10, channels=sel, dtype=np.float32)
            assert e.value.status == BITSTREAM
        check_select(dec, whole, parsed, 0, [0, 3 * FRAME], 2 * FRAME, [faulty], np.int16, False)
        check_select(dec, whole, parsed, 0, [0, 5 * FRAME], 100, keep, np.int16, False)    # usable after a failure

    # the same fault in the parent of a selected difference
    blob = base._mode_blobs()["P"]
    whole = base.expected([blob])
    parsed = [base.parse_container(blob)]
    _, d, _ = parsed[0]
    fd = d.reshape(-1, 8)
    f = int(np.nonzero((fd["subframe_type"] == 1).any(1))[0][0])
    diff_pos = int(np.nonzero(fd["subframe_type"][f] == 1)[0][0])
    child, parent = int(fd[f, diff_pos]["channel"]), int(fd[f, diff_pos]["parent_channel"])
    parent_pos = int(np.nonzero(fd["channel"][f] == parent)[0][0])
    bad = _corrupt_residues(blob, d, 8, f, parent_pos)
    free = [c for c in range(8) if c not in (child, parent) and
            not ((fd["channel"][f] == c) & (fd["subframe_type"][f] == 1) & (fd["parent_channel"][f] == parent)).any()]
    with ClipDecoder([bad]) as dec:
        with pytest.raises(SelaB200Error) as e:
            dec.decode(0, [f * FRAME], FRAME, channels=[child])
        assert e.value.status == BITSTREAM
        check_select(dec, whole, parsed, 0, [f * FRAME], FRAME, free, np.int16, False)


@pytest.mark.gpu
def test_rejections_leave_the_output_alone():
    blobs = [codec.encode_container(base._pcm(2, n, 30 + n), 2, 44100) for n in (3, 4)]
    mono = codec.encode_container(base._pcm(1, 2, 33), 1, 44100)
    total = [3 * FRAME, 4 * FRAME]
    whole = base.expected(blobs)
    with ClipDecoder(blobs + [mono]) as dec:
        out = np.full(4 * 255 * 64 * 2 + 16, 0x5A5A, np.int16)
        ok = [(0, 0), (1, total[1] - 64), (0, 5), (1, 7)]

        def call(pairs, length, sel, flags, reserved=None, buf=out):
            c = base._clips(pairs)
            if reserved is not None:
                c[reserved]["reserved"] = 1
            return _raw(dec, c, length, sel, flags, buf.ctypes.data if buf is not None else None)

        rc, frames, subs, err = call(ok, 64, [0], 0)      # channel 0 of a default stereo encode is independent
        assert (rc, frames, subs) == (0, 3, 3), err
        assert np.array_equal(out[:4 * 64].reshape(4, 64, 1), np.stack([whole[k][s:s + 64, :1] for k, s in ok]))
        assert (out[4 * 64:] == 0x5A5A).all()
        # at the limits: every flag, channel C - 1, 255 selected channels, the last sample, the mono container's mean
        assert call(ok, 64, [1, 0], F32 | MEAN)[0] == 0
        assert call(ok, 64, [0] * 255, F32)[0] == 0
        assert call(ok, 64, [1] * 255, F32 | MEAN)[0] == 0
        assert call([(2, 2 * FRAME - 1)], 1, [0], 0)[0] == 0
        assert call([(0, 0), (2, 0)], 64, None, F32 | MEAN)[0] == 0
        cases = [
            (ok, 64, [1], 4, ""),                                   # an unknown flag bit
            (ok, 64, [1], 0x80000000, ""),
            (ok, 64, [1], MEAN, ""),                                # MEAN without FLOAT32
            (ok, 64, [0] * 256, F32, ""),                           # 256 selected channels
            (ok, 64, [2], 0, "clip 0"),                             # channel 2 of a stereo container
            (ok[:3] + [(2, 0)], 64, [1], 0, "clip 3"),              # channel 1 of the mono container
            ([(0, 0), (2, 0)], 64, None, F32, "clip 1"),            # every channel of containers of 2 and 1 channels
            ([(2, 0), (0, 0)], 64, None, 0, "clip 1"),
            (ok[:3] + [(0, total[0] - 64 + 1)], 64, [0], 0, "clip 3"),   # one sample past the end
            (ok[:2] + [(3, 0)], 64, [0], 0, "clip 2"),                   # container index == n_handles
            (ok, 0, [0], 0, "clip 0"),                                   # length 0
            ([(0, 2 ** 64 - 1)], 2, [0], F32, "clip 0"),                 # start + length wraps 64 bits
        ]
        for pairs, length, sel, flags, where in cases:
            out[:] = 0x1234
            rc, n, m, err = call(pairs, length, sel, flags)
            assert rc == ARGUMENT and where in err and n == 0 and m == 0, (pairs, length, sel, flags, err)
            assert (out == 0x1234).all()
        out[:] = 0x1234
        rc, n, m, err = call(ok, 64, [0], 0, reserved=2)
        assert rc == ARGUMENT and "clip 2" in err and (out == 0x1234).all()
        # select and n_select disagree
        L = _lib.lib()
        c = base._clips(ok)
        n, m = C.c_uint64(0), C.c_uint64(0)
        sel = np.zeros(1, np.uint8)
        for fn in (L.selab200_container_decode_clips_select, L.selab200_container_decode_clips_select_device):
            assert fn(C.addressof(dec._array), 3, c.ctypes.data, 4, 64, None, 1, 0, out.ctypes.data, C.addressof(n),
                      C.addressof(m)) == ARGUMENT
            assert fn(C.addressof(dec._array), 3, c.ctypes.data, 4, 64, sel.ctypes.data, 0, 0, out.ctypes.data,
                      C.addressof(n), C.addressof(m)) == ARGUMENT
        assert L.selab200_container_decode_clips_select(C.addressof(dec._array), 3, c.ctypes.data, 4, 64,
                                                        sel.ctypes.data, 1, 0, out.ctypes.data, C.addressof(n),
                                                        None) == ARGUMENT
        assert call(ok, 64, [0], 0, buf=None)[0] == ARGUMENT
        assert (out == 0x1234).all()
        assert _raw(dec, None, 64, [0], 0, out.ctypes.data)[:3] == (0, 0, 0)     # the empty batch
        # the device form: float32 output 4-byte aligned, int16 2-byte aligned
        import torch
        buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
        assert _raw(dec, c, 64, [0], F32, buf.data_ptr() + 2, device=True)[0] == ARGUMENT
        assert _raw(dec, c, 64, [0], 0, buf.data_ptr() + 1, device=True)[0] == ARGUMENT
        assert not buf.any()
        assert _raw(dec, c, 64, [0], F32, buf.data_ptr() + 4, device=True)[0] == 0
        assert _raw(dec, c, 64, [0], 0, buf.data_ptr() + 2, device=True)[0] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("chunk_frames", [None, "3"])
def test_large_batch(monkeypatch, chunk_frames):
    """4096 clips over 16 containers of 2, 3 and 8 channels; with SELAB200_CHUNK_FRAMES=3 the selection takes many
    groups (12 subframes each, or one whole frame's) and chunks."""
    if chunk_frames:
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", chunk_frames)
    blobs = [codec.encode_container(base._pcm((2, 3, 8)[k % 3], 6 + k % 5, 50 + k), (2, 3, 8)[k % 3], 44100)
             for k in range(16)]
    whole = base.expected(blobs)
    parsed = [base.parse_container(b) for b in blobs]
    rng = np.random.default_rng(9)
    length = 1500
    ks = rng.integers(0, 16, 4096)
    starts = [int(rng.integers(0, whole[k].shape[0] - length + 1)) for k in ks]
    with ClipDecoder(blobs) as dec:
        check_select(dec, whole, parsed, ks, starts, length, [1, 0], np.int16, False)
        check_select(dec, whole, parsed, ks, starts, length, None, np.float32, True, device=True)
        check_select(dec, whole, parsed, ks, starts, length, [1], np.float32, False, device=True)


@pytest.mark.gpu
def test_cli_range_channels(tmp_path):
    if not (base.BIN / "sela").exists():
        subprocess.run(["make", "-C", str(base.ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    pcm = base._pcm(3, 9, 43)
    wavio.write_wav(tmp_path / "in.wav", pcm, 44100)

    def run(*args):
        p = subprocess.run([str(a) for a in args], capture_output=True, text=True, timeout=300)
        assert p.returncode == 0, (args, p.stdout[-300:], p.stderr[-300:])

    sela = base.BIN / "sela"
    run(sela, "-e", tmp_path / "in.wav", tmp_path / "a.sela")
    for first, count in ((0, 9 * FRAME), (5000, 7777), (9 * FRAME - 3, 3)):
        run(sela, "-R", tmp_path / "a.sela", tmp_path / "full.wav", first, count)
        full = (tmp_path / "full.wav").read_bytes()
        cols = np.frombuffer(full, np.int16, offset=44).reshape(count, 3)
        for sel in ([0, 2], [2], [1, 1, 0]):
            run(sela, "-R", tmp_path / "a.sela", tmp_path / "r.wav", first, count, ",".join(map(str, sel)))
            got = (tmp_path / "r.wav").read_bytes()
            assert struct.unpack_from("<H", got, 22)[0] == len(sel)
            assert struct.unpack_from("<I", got, 40)[0] == 2 * len(sel) * count
            assert struct.unpack_from("<I", got, 4)[0] == 36 + 2 * len(sel) * count
            assert got[24:28] == full[24:28] and got[34:36] == full[34:36]       # sample rate, bits per sample
            assert np.array_equal(np.frombuffer(got, np.int16, offset=44).reshape(count, len(sel)), cols[:, sel])
    for bad in ("3", "0,,1", "x"):
        p = subprocess.run([str(sela), "-R", str(tmp_path / "a.sela"), str(tmp_path / "r.wav"), "0", "10", bad],
                           capture_output=True, text=True, timeout=300)
        assert p.returncode == 1, bad
