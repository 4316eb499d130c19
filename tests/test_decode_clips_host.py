"""Clips from host-resident containers (selab200_container_open_host, DESIGN.md 7.10).

A host-resident handle keeps its image in page-locked host memory and each clip call fetches only the bytes of the
subframes it decodes.  Every result is compared bit for bit with the same call on device-resident handles over the
same bytes, counters included, and the bytes fetched with expected_fetch, a CPU model of the fetch rule over
parse_container's descriptors."""
import ctypes as C
import os

import numpy as np
import pytest

import test_decode_clips as base
import test_decode_clips_select as sel_base
from sela_b200 import ClipDecoder, SelaB200Error, _lib, codec, synth

FRAME = base.FRAME
ARGUMENT, BITSTREAM = base.ARGUMENT, base.BITSTREAM
F32, MEAN = _lib.CLIP_FLOAT32, _lib.CLIP_MEAN
# (channels, dtype, mean): the four forms; channels "all" with int16 is the plain call (selab200_container_decode_clips)
FORMS = [("all", np.int16, False), ("sel", np.int16, False), ("all", np.float32, False), ("all", np.float32, True)]


# ------------------------------------------------------------------ the fetch rule, on the CPU --

def _group_size(full, channels):
    """Frames per group of the plain call (full), subframes per group of the selecting call."""
    env = os.environ.get("SELAB200_CHUNK_FRAMES")
    if env and int(env) > 0:
        return min(4 * int(env), 1 << 20)
    return max(1, 32768 // channels) if full else 32768


def _subframe_ranges(parsed, k, f, positions):
    """Byte ranges [at, end) the unpack reads for the given positions of frame f of container k."""
    ch, d, _ = parsed[k]
    out = []
    for p in positions:
        s = d[f * ch + p]
        at = 15 + 4 * (f + 1) + 12 * (f * ch + p) + 4 * int(s["refl_offset"]) + 7
        out.append((at, at + 4 * int(s["refl_words"]) + 5 + 4 * int(s["res_words"]) + 3))
    return out


def _positions(parsed, k, f, select):
    """Positions a frame needs: the selected channels and the parents of the selected difference-coded ones."""
    ch, d, _ = parsed[k]
    fd = d[f * ch:(f + 1) * ch]
    pos = {int(fd[p]["channel"]): p for p in range(ch)}
    need = set()
    for c in (range(ch) if select is None else select):
        need.add(pos[c])
        if fd[pos[c]]["subframe_type"] == 1:
            need.add(pos[int(fd[pos[c]]["parent_channel"])])
    return sorted(need)


def expected_fetch(blobs, clips, length, select, full=False, host=None):
    """Bytes a clip call fetches from host-resident images.  clips: (container, start) pairs; full: the plain int16
    call over every channel (groups of whole frames), else the selecting call (groups of subframes, cut at frames);
    host: per container whether it is host-resident (default: all)."""
    parsed = [base.parse_container(b) for b in blobs]
    host = [True] * len(blobs) if host is None else host
    keys = sorted({(k, f) for k, s in clips for f in range(s // FRAME, (s + length - 1) // FRAME + 1)})
    groups, rows = [], 0
    for i, (k, f) in enumerate(keys):     # each group: the (container, ranges) of its subframes in selection order
        ch = parsed[k][0]
        pos = list(range(ch)) if full else _positions(parsed, k, f, select)
        if full:
            cut = i % _group_size(True, parsed[keys[0][0]][0]) == 0
        else:
            cut = i == 0 or rows + len(pos) > _group_size(False, 1)
        if cut:
            groups.append([])
            rows = 0
        rows += len(pos)
        groups[-1] += [(k, r) for r in _subframe_ranges(parsed, k, f, pos)]
    total = 0
    for g in groups:
        run = None                         # (container, lo, hi)
        for k, (a, b) in g:
            if not host[k]:
                continue
            lo, hi = a & ~15, (b + 15) & ~15
            if run and run[0] == k and lo <= run[2]:
                run = (k, run[1], max(run[2], hi))
                continue
            if run:
                total += run[2] - run[1]
            run = (k, lo, hi)
        if run:
            total += run[2] - run[1]
    return total


def test_fetch_model_rule(monkeypatch):
    """The model on hand-made descriptors: ranges rounded out to 16 bytes, merged when they touch, cut at groups."""
    d = np.zeros(2, _lib.DESC_DTYPE)
    d["refl_words"], d["res_words"] = 1, [1, 3]
    d["refl_offset"], d["res_offset"] = [0, 2], [1, 3]
    import struct
    blob = b"SeLa" + struct.pack("<IHBI", 44100, 16, 1, 2)
    for fr in range(2):
        blob += b"\x00\xff\x55\xaa" + struct.pack("<BBBBHB", 0, 0, 0, 0, 1, 1) + b"\0" * 4 + \
            struct.pack("<BHH", 0, int(d[fr]["res_words"]), 2048) + b"\0" * 4 * int(d[fr]["res_words"])
    # frame 0 reads [26, 26 + 4 + 5 + 4 + 3) = [26, 42) -> [16, 48); frame 1 [50, 74) -> [48, 80): they touch
    assert expected_fetch([blob], [(0, 0)], 1, None) == 32
    assert expected_fetch([blob], [(0, 0)], 4096, None) == 64
    assert expected_fetch([blob], [(0, 0)], 4096, None, host=[False]) == 0
    monkeypatch.setenv("SELAB200_CHUNK_FRAMES", "1")        # groups of 4 frames or subframes: still one group
    assert expected_fetch([blob], [(0, 0)], 4096, None, full=True) == 64
    assert _group_size(True, 8) == _group_size(False, 1) == 4


# ------------------------------------------------------------------ helpers --

def _raw_select(handles, clips, length, sel, flags, out, device=False):
    """The selecting C call on a handle list: (status, frames, subframes, bytes fetched, last error)."""
    L = _lib.lib()
    arr = (C.c_void_p * len(handles))(*handles)
    n, m, b = C.c_uint64(0), C.c_uint64(0), C.c_uint64(77)
    fn = L.selab200_container_decode_clips_select_device if device else L.selab200_container_decode_clips_select
    s = None if sel is None else np.ascontiguousarray(sel, np.uint8)
    rc = fn(C.addressof(arr), len(handles), clips.ctypes.data, clips.size, length,
            None if s is None else s.ctypes.data, 0 if s is None else s.size, flags, out, C.addressof(n),
            C.addressof(m))
    err = L.selab200_last_error().decode()
    assert L.selab200_clip_bytes_fetched(C.addressof(b)) == 0
    return rc, n.value, m.value, b.value, err


def _decode(dec, ks, starts, length, form, device):
    sel, dtype, mean = form
    if device:
        import torch
        t = torch.float32 if dtype == np.float32 else torch.int16
        return dec.decode_device(ks, starts, length, channels=sel, dtype=t, mean=mean).cpu().numpy()
    return dec.decode(ks, starts, length, channels=sel, dtype=dtype, mean=mean)


def _same(host, dev, blobs, ks, starts, length, form, device=False):
    """host-resident decoder == device-resident decoder, counters included; bytes_fetched == the model."""
    a = _decode(host, ks, starts, length, form, device)
    b = _decode(dev, ks, starts, length, form, device)
    assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), form
    assert (host.frames_decoded, host.subframes_decoded) == (dev.frames_decoded, dev.subframes_decoded)
    assert dev.bytes_fetched == 0
    ks = np.broadcast_to(np.asarray(ks), np.shape(starts)).tolist()
    full = form[0] is None and form[1] == np.int16
    assert host.bytes_fetched == expected_fetch(blobs, list(zip(ks, list(starts))), length, form[0], full=full), form
    return a


def _forms(channels):
    return [(None if c == "all" else [channels - 1, 0][:min(2, channels)], t, m) for c, t, m in FORMS]


def _open(blob, host):
    L = _lib.lib()
    buf = np.frombuffer(bytes(blob), np.uint8).copy()
    info = np.zeros(1, _lib.INFO_DTYPE)
    h = C.c_void_p(0)
    fn = L.selab200_container_open_host if host else L.selab200_container_open
    rc = fn(buf.ctypes.data, buf.size, C.addressof(h), info.ctypes.data)
    return rc, h.value, info, L.selab200_last_error().decode(), buf


# ------------------------------------------------------------------ CPU --

def test_entry_points_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = _lib.lib()
    assert L.selab200_init(0) == -1
    import struct
    blob = np.frombuffer(b"SeLa" + struct.pack("<IHBI", 44100, 16, 2, 0), np.uint8).copy()
    h = C.c_void_p(0)
    info = np.zeros(1, _lib.INFO_DTYPE)
    assert L.selab200_container_open_host(blob.ctypes.data, blob.size, C.addressof(h), info.ctypes.data) in (-1, -7)
    assert h.value is None
    b = C.c_uint64(5)
    assert L.selab200_clip_bytes_fetched(C.addressof(b)) in (-1, -7)     # NO_DEVICE / NOT_INIT: no CPU path
    assert b.value == 5


# ------------------------------------------------------------------ GPU --

@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 2, 3, 8])
def test_host_equals_device(channels):
    """Every form, both outputs, clips of many phases from three containers."""
    blobs = [codec.encode_container(base._pcm(channels, n, 10 + channels + n), channels, 44100) for n in (9, 5, 12)]
    total = [9 * FRAME, 5 * FRAME, 12 * FRAME]
    shapes = [([0], [0], 1), ([2], [total[2] - 777], 777), ([0, 1, 2, 0], [1, 3, 2041, 4093], 17),
              ([1, 2, 0], [7, 100, 2047], 2 * FRAME + 5), ([2, 2], [0, 4000], 9 * FRAME), ([1], [0], total[1])]
    with ClipDecoder(blobs, host_resident=True) as host, ClipDecoder(blobs) as dev:
        for form in _forms(channels):
            for ks, starts, n in shapes:
                for device in (False, True):
                    _same(host, dev, blobs, ks, starts, n, form, device)


@pytest.mark.gpu
def test_mixed_call():
    """Host- and device-resident handles of 2, 3 and 8 channels in one selecting call equal the all-device call."""
    blobs = [codec.encode_container(base._pcm(c, n, 80 + c), c, 44100) for c, n in ((2, 5), (3, 4), (8, 3), (2, 6))]
    mask = [True, False, True, False]
    pairs = [(0, 0), (1, 3000), (2, 10), (3, 7000), (0, 4000), (2, 2 * FRAME), (1, 0), (3, 0), (0, 3 * FRAME - 1)]
    clips = base._clips(pairs)
    with ClipDecoder(blobs, host_resident=True) as host, ClipDecoder(blobs) as dev:
        mixed = [host._handles[k] if mask[k] else dev._handles[k] for k in range(4)]
        for sel, flags, size in (([0], 0, 2), ([1, 0], F32, 4), (None, F32 | MEAN, 4), ([0, 0, 1], 0, 2)):
            n_out = 1 if flags & MEAN else len(sel)
            a = np.full(len(pairs) * 2000 * n_out * size // 2 + 8, 0x3C3C, np.int16)
            b = a.copy()
            ra = _raw_select(mixed, clips, 2000, sel, flags, a.ctypes.data)
            rb = _raw_select(dev._handles, clips, 2000, sel, flags, b.ctypes.data)
            assert ra[0] == 0 and rb[0] == 0, (ra, rb)
            assert np.array_equal(a, b) and ra[1:3] == rb[1:3] and rb[3] == 0
            assert ra[3] == expected_fetch(blobs, pairs, 2000, sel, host=mask) > 0
            import torch
            buf = torch.zeros(a.size * 2, dtype=torch.uint8, device="cuda")
            rc = _raw_select(mixed, clips, 2000, sel, flags, buf.data_ptr(), device=True)
            assert rc[0] == 0 and rc[1:4] == ra[1:4]
            assert np.array_equal(buf.cpu().numpy().view(np.int16)[:-8], a[:-8])


@pytest.mark.gpu
def test_caller_bytes_are_not_kept():
    blobs = [codec.encode_container(base._pcm(2, 6, 5), 2, 44100), codec.encode_container(base._pcm(2, 4, 6), 2, 44100)]
    whole = base.expected(blobs)
    owned = [bytearray(b) for b in blobs]
    with ClipDecoder(owned, host_resident=True) as host:
        assert host._bufs == []
        for o in owned:
            o[:] = bytes(len(o))                            # overwritten straight after the open
        del owned
        got = host.decode([0, 1, 0], [0, 100, 5000], 3000, channels=[1])
        want = np.stack([whole[k][s:s + 3000, [1]] for k, s in ((0, 0), (1, 100), (0, 5000))])
        assert np.array_equal(got, want)
        assert np.array_equal(host.decode(0, [17], 9000), whole[0][17:9017][None])


@pytest.mark.gpu
def test_run_edges():
    blobs = [codec.encode_container(base._pcm(2, 7, 31), 2, 44100), codec.encode_container(base._pcm(2, 5, 32), 2, 44100)]
    total = [7 * FRAME, 5 * FRAME]
    cases = [
        ([0], [0], 100),                                    # at sample 0
        ([0, 1], [total[0] - 500, total[1] - 1], 1),       # ending exactly at the end: rounding reaches the padding
        ([1], [total[1] - 3000], 3000),
        ([0], [FRAME + 5], 100),                            # inside one frame
        ([0, 0, 0], [100, 900, 100], 2500),                 # overlapping and repeated
        ([1, 1, 0, 0], [4 * FRAME, 2 * FRAME, 5 * FRAME, 0], 1000),   # reverse order
    ]
    with ClipDecoder(blobs, host_resident=True) as host, ClipDecoder(blobs) as dev:
        for ks, starts, n in cases:
            for form in _forms(2):
                for device in (False, True):
                    _same(host, dev, blobs, ks, starts, n, form, device)

    # channel pairing: channel 5 is a difference from channel 3, so its parent is fetched with it
    blob = base._mode_blobs()["P"]
    _, d, _ = base.parse_container(blob)
    fd = d.reshape(-1, 8)
    assert ((fd["subframe_type"] == 1) & (fd["channel"] == 5) & (fd["parent_channel"] == 3)).any()
    with ClipDecoder([blob], host_resident=True) as host, ClipDecoder([blob]) as dev:
        for starts, n in (([0], 4 * FRAME), ([FRAME - 3, 100], 2 * FRAME)):
            _same(host, dev, [blob], 0, starts, n, ([5], np.int16, False))
            pairs = [(0, s) for s in starts]
            alone = expected_fetch([blob], pairs, n, [5])
            assert host.bytes_fetched == alone
        # the parents' bytes are in it: more than channel 5's own subframes take, each rounded out on its own
        parsed = [base.parse_container(blob)]
        own = sum(((b + 15) & ~15) - (a & ~15) for f in range(fd.shape[0])
                  for a, b in _subframe_ranges(parsed, 0, f, [int(np.nonzero(fd["channel"][f] == 5)[0][0])]))
        _same(host, dev, [blob], 0, [0], 4 * FRAME, ([5], np.int16, False))
        assert host.bytes_fetched > own
        # every channel of the file: about the covered frames' bytes
        _same(host, dev, [blob], 0, [0], 4 * FRAME, (None, np.int16, False))
        assert host.bytes_fetched <= len(blob) + 16 and host.bytes_fetched >= len(blob) - 15 - 16


@pytest.mark.gpu
@pytest.mark.parametrize("chunk_frames", [None, "3"])
def test_large_batch(monkeypatch, chunk_frames):
    """4096 clips over 16 containers; with SELAB200_CHUNK_FRAMES=3 many groups, chunks and fetch pieces, so every
    staging region is reused across groups."""
    if chunk_frames:
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", chunk_frames)
    blobs = [codec.encode_container(base._pcm(2, 6 + k % 5, 50 + k), 2, 44100) for k in range(16)]
    rng = np.random.default_rng(9)
    length = 1500
    ks = rng.integers(0, 16, 4096)
    starts = [int(rng.integers(0, (6 + k % 5) * FRAME - length + 1)) for k in ks]
    with ClipDecoder(blobs, host_resident=True) as host, ClipDecoder(blobs) as dev:
        _same(host, dev, blobs, ks, starts, length, (None, np.int16, False))
        _same(host, dev, blobs, ks, starts, length, ([1], np.float32, False), device=True)
        _same(host, dev, blobs, ks, starts, length, (None, np.float32, True), device=True)


@pytest.mark.gpu
def test_open_errors_match():
    pcm = base._pcm(2, 6, 3)
    blob = bytes(codec.encode_container(pcm, 2, 44100))
    _, d, _ = base.parse_container(blob)
    at = 15 + 4 * (4 + 2 * 12) + 4 * int(d[8]["refl_offset"])      # frame 4's sync word
    bad_sync = bytearray(blob)
    bad_sync[at + 1] ^= 0x40
    more = bytearray(blob)
    more[11:15] = (500).to_bytes(4, "little")
    cases = [blob[:14], b"RIFF" + blob[4:], blob[:15], blob[:17], bytes(bad_sync), bytes(more),
             blob + b"\x00\xff\x55\xaa junk"] + [blob[:len(blob) - cut] for cut in (1, 5, 7, 640, len(blob) - 19,
                                                                                  len(blob) - 27)]
    _lib.init(0)
    L = _lib.lib()
    for c in cases:
        rc_d, h_d, info_d, err_d, _ = _open(c, False)
        rc_h, h_h, info_h, err_h, _ = _open(c, True)
        assert (rc_h, err_h if rc_h else "") == (rc_d, err_d if rc_d else ""), (len(c), err_d, err_h)
        assert bytes(info_h) == bytes(info_d) or rc_d
        assert (h_h is None) == (h_d is None) == (rc_d != 0)
        L.selab200_container_close(h_d)
        L.selab200_container_close(h_h)
    assert any(_open(c, True)[0] == BITSTREAM for c in cases)


@pytest.mark.gpu
def test_malformed_and_rejected():
    pcm = base._pcm(2, 8, 5)
    blob = codec.encode_container(pcm, 2, 44100)
    whole = base.expected([blob])
    _, d, _ = base.parse_container(blob)
    at = 15 + 4 * (5 + 1) + 12 * (5 * 2 + 1) + 4 * int(d[5 * 2 + 1]["refl_offset"])   # frame 5, subframe 1
    bad = bytearray(blob)
    bad[at + 6] = 101                                       # its order byte: the walk accepts it, the rules do not
    with ClipDecoder([bytes(bad)], host_resident=True) as dec:
        for s, n in ((0, 5 * FRAME), (6 * FRAME, 2 * FRAME)):
            assert np.array_equal(dec.decode(0, [s], n), whole[0][s:s + n][None])
            assert np.array_equal(dec.decode(0, [s], n, channels=[0]), whole[0][s:s + n, :1][None])
        for s, n in ((5 * FRAME, 1), (0, 8 * FRAME)):
            for kw in ({}, dict(channels=[0])):
                with pytest.raises(SelaB200Error) as e:
                    dec.decode(0, [s], n, **kw)
                assert e.value.status == BITSTREAM

    # a residue stream that runs past its words: only a call that decodes its subframe fails
    blob3 = codec.encode_container(synth.sine_noise(44100, 3, n_frames=6, seed=90), 3, 44100)
    whole3 = base.expected([blob3])
    _, d3, _ = base.parse_container(blob3)
    bad3 = sel_base._corrupt_residues(blob3, d3, 3, 2, 1)
    faulty = int(d3[2 * 3 + 1]["channel"])
    keep = [c for c in range(3) if c != faulty]
    with ClipDecoder([bad3], host_resident=True) as dec:
        assert np.array_equal(dec.decode(0, [2 * FRAME + 5], 3 * FRAME, channels=keep),
                              whole3[0][2 * FRAME + 5:5 * FRAME + 5, keep][None])
        for kw in (dict(channels=[faulty]), {}):
            with pytest.raises(SelaB200Error) as e:
                dec.decode(0, [2 * FRAME + 100], 10, **kw)
            assert e.value.status == BITSTREAM
        assert np.array_equal(dec.decode(0, [3 * FRAME], 100), whole3[0][3 * FRAME:3 * FRAME + 100][None])

    # a rejected call writes nothing
    with ClipDecoder([blob], host_resident=True) as dec:
        out = np.full(4 * 64 * 2 + 16, 0x1234, np.int16)
        for pairs, length, sel in (([(0, 0), (0, 8 * FRAME - 63)], 64, [0]), ([(0, 0), (1, 0)], 64, None),
                                   ([(0, 0)], 0, [1]), ([(0, 0)], 64, [2])):
            rc, n, m, b, err = _raw_select(dec._handles, base._clips(pairs), length, sel, 0, out.ctypes.data)
            assert rc == ARGUMENT and (n, m, b) == (0, 0, 0), err
            if sel != [2]:
                rc, n, err = base._raw(dec, base._clips(pairs), length, out.ctypes.data)
                assert rc == ARGUMENT and n == 0, err
        assert (out == 0x1234).all()


@pytest.mark.gpu
def test_decode_and_verify_on_a_host_handle():
    import torch
    pcm = base._pcm(2, 600, 7)
    blob = codec.encode_container(pcm, 2, 44100)
    src = pcm.reshape(-1).copy()
    src[5 * 2 * FRAME + 7] ^= 3                             # two differing (frame, channel) pairs
    src[550 * 2 * FRAME + 2 * 100 + 1] ^= 1

    def run():
        L = _lib.lib()
        out = {}
        for host in (False, True):
            rc, h, info, err, keep = _open(blob, host)
            assert rc == 0, err
            try:
                pcm_out = np.empty(int(info[0]["n_frames"]) * 2 * FRAME, np.int16)
                assert L.selab200_container_decode(C.c_void_p(h), pcm_out.ctypes.data) == 0
                rep = np.zeros(1200, _lib.VERIFY_DTYPE)
                n = C.c_size_t(0)
                assert L.selab200_container_verify(C.c_void_p(h), src.ctypes.data, rep.ctypes.data, rep.size,
                                                   C.addressof(n)) == 0
                out[host] = (pcm_out, rep[:n.value].copy())
            finally:
                L.selab200_container_close(C.c_void_p(h))
        assert np.array_equal(out[True][0], out[False][0])
        assert out[True][1].tobytes() == out[False][1].tobytes() and out[True][1].size >= 2
        return out[True]

    _lib.init(0)
    one = run()
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the two-device part needs two")
    try:
        _lib.init([0, 1])                                    # 600 frames: each device decodes a block
        two = run()
    finally:
        _lib.init(0)
    assert np.array_equal(one[0], two[0]) and one[1].tobytes() == two[1].tobytes()


@pytest.mark.gpu
def test_python_decoder():
    import torch
    blobs = [codec.encode_container(base._pcm(8, 5, 61), 8, 44100)]
    whole = base.expected(blobs)
    dec = ClipDecoder(blobs, host_resident=True)
    assert dec.host_resident and dec.bytes_fetched == 0 and dec.info[0]["channels"] == 8
    got = dec.decode(0, [10, 3000], 4000, channels=[0])
    assert np.array_equal(got, np.stack([whole[0][s:s + 4000, :1] for s in (10, 3000)]))
    one = dec.bytes_fetched
    assert one == expected_fetch(blobs, [(0, 10), (0, 3000)], 4000, [0]) > 0
    got = dec.decode_device(0, [10, 3000], 4000)
    assert got.device.type == "cuda" and np.array_equal(got.cpu().numpy(), np.stack([whole[0][s:s + 4000]
                                                                                      for s in (10, 3000)]))
    assert dec.bytes_fetched == expected_fetch(blobs, [(0, 10), (0, 3000)], 4000, None, full=True) > 4 * one
    m = dec.decode_device(0, [0], 100, dtype=torch.float32, mean=True)
    assert m.shape == (1, 100, 1) and dec.bytes_fetched == expected_fetch(blobs, [(0, 0)], 100, None)
    dec.close()
    assert dec._handles == []
    with pytest.raises(ValueError):
        dec.decode(0, [0], 10)
