"""The multi-device host calls on one GPU: selab200_init_devices with the same device in several slots.

Every slot is a context of its own (streams, events, pools, worker thread), so a slot list such as [0, 0, 0] runs all
of the block code -- the split into blocks, the worker threads, the re-basing of descriptor offsets and container
bodies, the merged counters and records, the per-block uploads of open containers, the first failing block's status --
on one device.  Each call is compared byte for byte, field for field, with the same call on one slot, whose results
the other test files pin to the oracle port and the exact models; plain encode and decode are also compared with the
oracle port here.  What repeats cannot reach is a kernel on one device reading another device's memory: [0, 1] and
[1, 0] run where a second GPU exists."""
import ctypes as C
import os
import pathlib
import subprocess

import numpy as np
import pytest

import oracle_lib as ol
import sela_b200
from sela_b200 import _lib, codec, synth, wavio
from sela_b200.clips import ClipDecoder

pytestmark = pytest.mark.gpu

FRAME = 2048
BLOCK_MIN = 256           # frames per device below which a batch stays on the primary (use_all_devices)
MAX_SLOTS = 16            # kMaxDevices
ROOT = pathlib.Path(__file__).resolve().parent.parent
BIN = ROOT / "sela_b200" / "host" / "bin"
GOLD = np.load(pathlib.Path(__file__).parent / "golden" / "golden_frames.npz")
LOSSY = GOLD["pcm_oct_reference_lossy"].reshape(2, FRAME, 8)   # frame 0 is lossy on channel 1, frame 1 on channel 4


def _n_gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


_two = pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")
SLOT_LISTS = [pytest.param([0, 0], id="0-0"), pytest.param([0, 0, 0], id="0-0-0"),
              pytest.param([0] * MAX_SLOTS, id="0x16"),
              pytest.param([0, 1], id="0-1", marks=_two), pytest.param([1, 0], id="1-0", marks=_two)]

# Per slot count D: the batch sizes around the block edges and the channel count each one runs with.  "chunks" is
# 256 D frames again with SELAB200_CHUNK_FRAMES=3, so that every block is cut into many pipeline chunks.
SIZES = ("one_block", "equal_blocks", "remainder", "chunks")
CHANNELS = {2: (1, 16, 2, 8), 3: (2, 8, 16, 1), MAX_SLOTS: (8, 1, 2, 2)}


def n_frames_for(size, d):
    return {"one_block": BLOCK_MIN * d - 1, "equal_blocks": BLOCK_MIN * d, "remainder": BLOCK_MIN * d + d - 1,
            "chunks": BLOCK_MIN * d}[size]


def blocks(n_frames, d):
    """The D-way split of device_parts: n/D frames each, the last block takes the rest -> [(f0, nf)]."""
    per = n_frames // d
    return [(per * i, n_frames - per * i if i == d - 1 else per) for i in range(d)]


def edge_frames(n_frames, d):
    """The first and the last frame of every block of the D-way split (also where the batch is not split)."""
    return sorted({f for f0, nf in blocks(n_frames, d) for f in (f0, f0 + nf - 1)})


@pytest.fixture
def slots(request):
    """The slot list of the test; whatever the test does, the library is bound to device 0 alone afterwards."""
    try:
        yield list(request.param)
    finally:
        _lib.init(0)


@pytest.fixture(scope="module")
def port():
    return ol.load("port")


def special_pcm(n_frames, channels, d, seed):
    """A music-like batch whose block-edge frames are, in turn, a golden frame the reference decoder does not
    reproduce (both of them), a stereo frame the encoder codes as a difference, and silence."""
    pcm = synth.sine_noise(48000, channels, n_frames=n_frames, seed=seed).reshape(n_frames, FRAME, channels)
    for i, f in enumerate(edge_frames(n_frames, d)):
        kind = i % 4
        if kind < 2:            # the lossy channel (1 or 4) first, then the others of the golden frame in turn
            cols = [(j + (1, 4)[kind]) % 8 for j in range(channels)]
            pcm[f] = LOSSY[kind][:, cols]
        elif kind == 2:
            if channels >= 2:
                pcm[f, :, 1] = pcm[f, :, 0] - (pcm[f, :, 1] >> 5)
            else:               # mono has no difference subframe: full-scale noise instead
                pcm[f, :, 0] = np.random.default_rng(seed + f).choice(np.array([-32768, 32767], np.int16), FRAME)
        else:
            pcm[f] = 0
    return pcm.reshape(-1, channels)


def flipped(pcm, n_frames, channels, d):
    """The source with one sample changed on both sides of every block edge, and in the first and the last frame."""
    src = pcm.copy().reshape(n_frames, FRAME, channels)
    frames = {0, n_frames - 1}
    for f0, _ in blocks(n_frames, d)[1:]:
        frames |= {f0 - 1, f0}
    for f in sorted(frames):
        src[f, (f * 7) % FRAME, f % channels] ^= 0x40
    return src.reshape(-1, channels)


def expected_report(decoded, source, channels):
    """Every (frame, channel) whose decoded samples differ from the source, in (frame, channel) order."""
    dd = np.asarray(decoded, np.int16).reshape(-1, FRAME, channels).astype(np.int32)
    s = np.asarray(source, np.int16).reshape(-1, FRAME, channels).astype(np.int32)
    diff = dd != s
    out = []
    for f, c in zip(*np.nonzero(diff.any(axis=1))):
        first = int(np.argmax(diff[f, :, c]))
        out.append((int(f), int(c), first, int(diff[f, :, c].sum()), int(dd[f, first, c] - s[f, first, c])))
    return out


def verify_tuples(report):
    return [tuple(int(e[k]) for k in ("frame", "channel", "first_sample", "n_differing", "first_delta"))
            for e in report]


def canon(x):
    """A result of any call in a form that compares exactly: arrays by dtype and bytes."""
    if isinstance(x, np.ndarray):
        return (x.dtype.str, x.shape, x.tobytes())
    if isinstance(x, (tuple, list)):
        return tuple(canon(v) for v in x)
    if isinstance(x, dict):
        return tuple(sorted((k, canon(v)) for k, v in x.items()))
    return x


def launches():
    return _lib.lib().selab200_launch_count()


def slot_launches(d):
    return [_lib.lib().selab200_slot_launch_count(i) for i in range(d)]


# ----------------------------------------------------------------------------------------------- host-resident --

def host_resident(blob, pcm=None):
    """selab200_container_open_host, then decode (pcm None) or verify against pcm -> (status, message, result)."""
    L = _lib.lib()
    buf = np.ascontiguousarray(blob, np.uint8)
    info = np.zeros(1, _lib.INFO_DTYPE)
    h = C.c_void_p(0)
    _lib.check(L.selab200_container_open_host(buf.ctypes.data, buf.size, C.addressof(h), info.ctypes.data))
    try:
        n = int(info[0]["n_frames"]) * int(info[0]["channels"])
        if pcm is None:
            out = np.full(n * FRAME, 0x2B2B, np.int16)
            rc = L.selab200_container_decode(h, out.ctypes.data)
        else:
            src = np.ascontiguousarray(pcm, np.int16).reshape(-1)
            out = np.zeros(max(n, 1), _lib.VERIFY_DTYPE)
            cnt = C.c_size_t(0)
            rc = L.selab200_container_verify(h, src.ctypes.data, out.ctypes.data, out.size, C.addressof(cnt))
            out = out[:cnt.value]
        return rc, L.selab200_last_error().decode() if rc else "", out if rc == 0 else None
    finally:
        L.selab200_container_close(h)


def device_resident(blob):
    """selab200_container_open + decode -> (status, message, pcm or None)."""
    L = _lib.lib()
    buf = np.ascontiguousarray(blob, np.uint8)
    info = np.zeros(1, _lib.INFO_DTYPE)
    h = C.c_void_p(0)
    _lib.check(L.selab200_container_open(buf.ctypes.data, buf.size, C.addressof(h), info.ctypes.data))
    try:
        out = np.full(int(info[0]["n_frames"]) * int(info[0]["channels"]) * FRAME, 0x2B2B, np.int16)
        rc = L.selab200_container_decode(h, out.ctypes.data)
        return rc, L.selab200_last_error().decode() if rc else "", out if rc == 0 else None
    finally:
        L.selab200_container_close(h)


# ------------------------------------------------------------------------------------------------ every call --

def encode_calls(pcm, ch, device):
    """Every encode mode in both forms, every counter it returns."""
    r = {}
    r["frames"] = sela_b200.encode_frames(pcm, ch, device=device)
    r["frames_lossless"] = sela_b200.encode_frames_lossless(pcm, ch, device=device)
    r["frames_search"] = sela_b200.encode_frames_search(pcm, ch, device=device)
    for c in (1, 4):
        r["frames_guided%d" % c] = sela_b200.encode_frames_search_guided(pcm, ch, c, device=device)
    r["frames_pairing"] = sela_b200.encode_frames_pairing(pcm, ch, device=device)
    r["frames_search_pairing"] = sela_b200.encode_frames_search_pairing(pcm, ch, device=device)
    for m in (1, 31):
        r["frames_windows%d" % m] = sela_b200.encode_frames_search_windows(pcm, ch, m, device=device)
    r["container"] = sela_b200.encode_container(pcm, ch, 48000, device=device)
    r["container_verified"] = sela_b200.encode_container_verified(pcm, ch, 48000, device=device)
    r["container_lossless"] = sela_b200.encode_container_lossless(pcm, ch, 48000, device=device)
    r["container_search"] = sela_b200.encode_container_search(pcm, ch, 48000, device=device)
    for c in (1, 4):
        r["container_guided%d" % c] = sela_b200.encode_container_search_guided(pcm, ch, 48000, c, device=device)
    r["container_pairing"] = sela_b200.encode_container_pairing(pcm, ch, 48000, device=device)
    r["container_search_pairing"] = sela_b200.encode_container_search_pairing(pcm, ch, 48000, device=device)
    for m in (1, 31):
        r["container_windows%d" % m] = sela_b200.encode_container_search_windows(pcm, ch, 48000, m, device=device)
    return r


def decode_calls(descs, words, blob, source, ch, n_frames, d, device):
    """Every decode-side call: frames, open containers of both kinds, and both clip calls (on the primary)."""
    r = {}
    r["decode_frames"] = sela_b200.decode_frames(descs, words, ch, device=device)
    r["verify_frames"] = sela_b200.verify_frames(descs, words, ch, source, device=device)
    r["container_decode"] = sela_b200.decode_container(blob, device=device)
    r["container_verify"] = sela_b200.verify_container(blob, source, device=device)
    _lib.init(device)
    r["host_decode"] = host_resident(blob)
    r["host_verify"] = host_resident(blob, source)
    # clips across every block edge, the first sample and the last
    total = n_frames * FRAME
    starts = [0, total - 3000] + [max(0, f0 * FRAME - 1000) for f0, _ in blocks(n_frames, d)[1:]]
    pick = [ch - 1, 0] if ch > 1 else [0, 0]
    for host in (False, True):
        with ClipDecoder([blob], device=device, host_resident=host) as dec:
            r["clips", host] = (dec.decode(0, starts, 3000), dec.frames_decoded)
            r["clips_select", host] = (dec.decode(0, starts, 3000, channels=pick, dtype=np.float32),
                                       dec.decode(0, starts, 3000, dtype=np.float32, mean=True),
                                       dec.subframes_decoded)
    return r


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("slots", SLOT_LISTS, indirect=True)
def test_every_call_equals_one_slot(slots, size, port, monkeypatch):
    d = len(slots)
    n = n_frames_for(size, d)
    ch = CHANNELS[d][SIZES.index(size)]
    split = n >= BLOCK_MIN * d
    one = [slots[0]]
    pcm = special_pcm(n, ch, d, seed=d * 10 + SIZES.index(size))
    source = flipped(pcm, n, ch, d)

    # Which slot coded which frames, seen in the kernel launches of each slot: with several blocks, slot i issues
    # those of one slot coding block i on its own; with one block, the primary issues those of the whole batch.  With
    # 4-frame chunks a block of 257 frames has one chunk more than a block of 256, so the counts tell the sizes apart.
    monkeypatch.setenv("SELAB200_CHUNK_FRAMES", "1")
    _lib.init(one)
    l0 = launches()
    sela_b200.encode_frames(pcm, ch, device=one)
    whole = launches() - l0
    per_block = []
    for f0, nf in blocks(n, d):
        l0 = launches()
        sela_b200.encode_frames(pcm[f0 * FRAME:(f0 + nf) * FRAME], ch, device=one)
        per_block.append(launches() - l0)
    _lib.init(slots)
    assert _lib.lib().selab200_device_count() == d
    before = slot_launches(d)
    sela_b200.encode_frames(pcm, ch, device=slots)
    issued = [b - a for a, b in zip(before, slot_launches(d))]
    assert issued == (per_block if split else [whole] + [0] * (d - 1))
    if size == "remainder":   # the last block is the larger one
        assert per_block[-1] > per_block[0]
    if size == "chunks":
        monkeypatch.setenv("SELAB200_CHUNK_FRAMES", "3")
    else:
        monkeypatch.delenv("SELAB200_CHUNK_FRAMES")

    _lib.init(one)
    want = sela_b200.encode_frames(pcm, ch, device=one)
    got = sela_b200.encode_frames(pcm, ch, device=slots)
    assert canon(got) == canon(want)
    d_ref, w_ref = port.encode_frames(pcm, ch)
    assert got[0].tobytes() == d_ref.tobytes() and np.array_equal(got[1], w_ref)

    enc_one = encode_calls(pcm, ch, one)
    enc = encode_calls(pcm, ch, slots)
    for k in enc_one:
        assert canon(enc[k]) == canon(enc_one[k]), k
    # the encoded forms agree with each other: the container is the packed arena, its verify report is empty or
    # agrees with the lossless records, and the records carry global frames in (frame, channel) order
    assert enc["container"].tobytes() == wavio.pack_container(got[0], got[1], 48000, ch)
    assert enc["container_verified"][0].tobytes() == enc["container"].tobytes()
    recoded = [(int(e["frame"]), int(e["channel"])) for e in enc["frames_lossless"][2]]
    lossy = [(int(e["frame"]), int(e["channel"])) for e in enc["container_verified"][1]]
    assert lossy == sorted(set(lossy)) and (ch == 2 or lossy == recoded)   # stereo: a difference repeats an error
    for rec in (enc["frames_lossless"][2], enc["container_lossless"][1]):
        keys = [(int(e["frame"]), int(e["channel"])) for e in rec]
        assert keys == recoded == sorted(set(keys))
    if ch >= 8:   # the golden lossy channels sit at block edges: the repair finds them in every block
        assert {f for i, f in enumerate(edge_frames(n, d)) if i % 4 < 2} <= {f for f, _ in recoded}

    if ch >= 2:   # the difference-coded edge frames: both pairing modes code a channel as a difference there
        assert enc["frames_pairing"][3] > 0 and enc["frames_search_pairing"][3] > 0
    descs, words = got
    blob = enc["container"]
    dec_one = decode_calls(descs, words, blob, source, ch, n, d, one)
    dec = decode_calls(descs, words, blob, source, ch, n, d, slots)
    for k in dec_one:
        assert canon(dec[k]) == canon(dec_one[k]), k
    out = dec["decode_frames"]
    assert np.array_equal(out, port.decode_frames(d_ref, w_ref, ch))
    assert np.array_equal(dec["container_decode"][1], out)
    assert dec["host_decode"][0] == 0 and np.array_equal(dec["host_decode"][2], out)
    report = expected_report(out, source, ch)
    assert len(report) >= 2 * d and [r[:2] for r in report] == sorted(r[:2] for r in report)
    assert verify_tuples(dec["verify_frames"]) == report
    assert verify_tuples(dec["container_verify"][1]) == report
    assert verify_tuples(dec["host_verify"][2]) == report


# ------------------------------------------------------------------------------------ records and capacities --

def _records_call(fn, args, dtype, capacity):
    """fn(*args, entries, capacity, &n_entries) with entries guarded past `capacity` -> (rc, n_entries, entries)."""
    entries = np.zeros(capacity + 4, dtype)
    entries.view(np.uint8)[:] = 0xA5
    n = C.c_size_t(12345)
    rc = fn(*args, entries.ctypes.data, capacity, C.addressof(n))
    return rc, n.value, entries


@pytest.mark.parametrize("slots", SLOT_LISTS, indirect=True)
def test_records_and_capacities(slots):
    """With a small `capacity` only the first records are written and n_entries is the total; an output one word (one
    byte) too small fails as on one slot, with the same size, and nothing past the capacity is written."""
    L = _lib.lib()
    d = len(slots)
    ch, n = 8, BLOCK_MIN * d + d - 1
    pcm = special_pcm(n, ch, d, seed=3)
    source = flipped(pcm, n, ch, d)
    cap_words = L.selab200_encode_words_bound(n, ch)
    results = {}
    for key in ([slots[0]], slots):
        _lib.init(key)
        r = {}
        # lossless records, arena form
        descs = np.zeros(n * ch, _lib.DESC_DTYPE)
        words = np.zeros(cap_words, np.uint32)
        used = C.c_size_t(0)
        args = (pcm.ctypes.data, n, ch, descs.ctypes.data, words.ctypes.data, cap_words, C.addressof(used))
        rc, total, _ = _records_call(L.selab200_encode_frames_lossless, args, _lib.LOSSLESS_DTYPE, 0)
        assert rc == 0 and total >= 2
        rc, n2, ent = _records_call(L.selab200_encode_frames_lossless, args, _lib.LOSSLESS_DTYPE, 1)
        assert rc == 0 and n2 == total
        assert (ent.view(np.uint8)[16:] == 0xA5).all()
        r["lossless"] = (total, ent[:1].tobytes(), descs.tobytes(), words[:used.value].tobytes())
        full = sela_b200.encode_frames_lossless(pcm, ch, device=key)[2]
        assert full.size == total and full[:1].tobytes() == ent[:1].tobytes()
        # verify records: every flipped sample, a capacity of two
        d0, w0 = sela_b200.encode_frames(pcm, ch, device=key)
        args = (d0.ctypes.data, n, ch, w0.ctypes.data, w0.size, np.ascontiguousarray(source).ctypes.data)
        rc, total, _ = _records_call(L.selab200_verify_frames, args, _lib.VERIFY_DTYPE, 0)
        rc2, n2, ent = _records_call(L.selab200_verify_frames, args, _lib.VERIFY_DTYPE, 2)
        assert rc == rc2 == 0 and n2 == total >= 2 * d
        assert (ent.view(np.uint8)[32:] == 0xA5).all()
        r["verify"] = (total, ent[:2].tobytes())
        # the word arena one word too small
        need = w0.size
        words = np.full(need + 64, 0xDEADBEEF, np.uint32)
        used = C.c_size_t(0)
        rc = L.selab200_encode_frames(pcm.ctypes.data, n, ch, descs.ctypes.data, words.ctypes.data, need - 1,
                                      C.addressof(used))
        assert rc == -4 and (words[need - 1:] == 0xDEADBEEF).all()
        r["arena"] = (rc, used.value, L.selab200_last_error())
        # the container one byte too small
        blob = sela_b200.encode_container(pcm, ch, 48000, device=key)
        out = np.full(blob.size + 64, 0x5A, np.uint8)
        used = C.c_size_t(0)
        rc = L.selab200_encode_container(pcm.ctypes.data, n, ch, 48000, 16, out.ctypes.data, blob.size - 1,
                                         C.addressof(used))
        assert rc == -4 and (out[blob.size - 1:] == 0x5A).all()
        r["container"] = (rc, used.value, L.selab200_last_error())
        results[len(key)] = r
    assert results[1] == results[d]
    assert results[d]["arena"][1] == need and results[d]["container"][1] == blob.size


# ------------------------------------------------------------------------------------------------- bad input --

def _corrupt_container(blob, frames):
    """The container with the first subframe of each frame in `frames` claiming 2055 samples."""
    _, offsets = codec.container_frame_offsets(blob)
    bad = blob.copy()
    for f in frames:
        at = int(offsets[f]) + 4
        refl_words = int(bad[at + 4]) | int(bad[at + 5]) << 8
        at2 = at + 7 + 4 * refl_words
        bad[at2 + 3:at2 + 5] = np.frombuffer(np.uint16(2055).tobytes(), np.uint8)
    return bad


@pytest.mark.parametrize("slots", SLOT_LISTS, indirect=True)
def test_a_malformed_subframe_fails_as_on_one_slot(slots):
    """A malformed subframe in the first block only, in the last only, and in both: every decode-side call fails with
    one slot's status and message, which names the first malformed subframe of the batch."""
    L = _lib.lib()
    d = len(slots)
    ch, n = 2, BLOCK_MIN * d
    pcm = special_pcm(n, ch, d, seed=5)
    parts = blocks(n, d)
    first, last = parts[0][0] + parts[0][1] - 1, parts[-1][0]
    for where in ([first], [last], [first, last]):
        seen = []
        for key in ([slots[0]], slots):
            _lib.init(key)
            descs, words = sela_b200.encode_frames(pcm, ch, device=key)
            blob = sela_b200.encode_container(pcm, ch, 48000, device=key)
            bad = descs.copy()
            for f in where:
                bad[f * ch]["samples"] = 2055
            out = np.empty(pcm.size, np.int16)
            r = [L.selab200_decode_frames(bad.ctypes.data, n, ch, words.ctypes.data, words.size, out.ctypes.data),
                 L.selab200_last_error()]
            rep = np.zeros(n * ch, _lib.VERIFY_DTYPE)
            cnt = C.c_size_t(0)
            r += [L.selab200_verify_frames(bad.ctypes.data, n, ch, words.ctypes.data, words.size, pcm.ctypes.data,
                                           rep.ctypes.data, rep.size, C.addressof(cnt)), L.selab200_last_error()]
            broken = _corrupt_container(blob, where)
            r += list(device_resident(broken)[:2]) + list(host_resident(broken)[:2]) + \
                list(host_resident(broken, pcm)[:2])
            seen.append(r)
        assert seen[0] == seen[1], where
        assert seen[1][0::2] == [-6] * 5, where
        # every message names the first malformed subframe, the one in the first failing block
        names = "(the first malformed descriptor: frame %d, channel 0)" % where[0]
        assert all(names in (m.decode() if isinstance(m, bytes) else m) for m in seen[1][1::2]), (where, seen[1])


# ----------------------------------------------------------------------------------------- device-set changes --

def test_window_search_and_device_forms_as_the_slot_list_changes():
    """[0] -> [0, 0] -> [0, 0, 0] -> [0]: after every change the window search gives one slot's bytes on the host
    and through a *_device call, which runs on the first slot of its device."""
    import torch
    from sela_b200.device import DeviceCodec
    ch, n = 2, 3 * BLOCK_MIN
    pcm = special_pcm(n, ch, 3, seed=7).reshape(-1)
    dc = DeviceCodec(n, ch, device=0)
    pcm_dev = torch.from_numpy(pcm).to(torch.device("cuda", 0))
    want = None
    try:
        for key in ([0], [0, 0], [0, 0, 0], [0]):
            _lib.init(key)
            assert _lib.lib().selab200_device_count() == len(key)
            got = sela_b200.encode_frames_search_windows(pcm, ch, 31, device=key)
            dc.encode_search_windows(pcm_dev, 31)
            dc.check_status()
            dev = (dc.descs.cpu().numpy().tobytes(),
                   dc.words[:int(dc.words_used.item())].cpu().numpy().view(np.uint32).tobytes(),
                   int(dc.base_words.item()), int(dc.n_window.item()))
            want = want or canon(got)
            assert canon(got) == want, key
            assert dev == (got[0].tobytes(), got[1].tobytes(), got[2], got[3]), key
        assert got[3] > 0
    finally:
        _lib.init(0)


def test_device_lists_the_library_accepts():
    """Any device may repeat, up to 16 entries; the count and the range are still checked."""
    L = _lib.lib()
    have = _n_gpus()
    try:
        for key in ([0, 0], [0] * MAX_SLOTS, [0, 0, 0]):
            arr = (C.c_int * len(key))(*key)
            assert L.selab200_init_devices(len(key), C.addressof(arr)) == 0
            assert L.selab200_device_count() == len(key)
        arr = (C.c_int * (MAX_SLOTS + 1))(*([0] * (MAX_SLOTS + 1)))
        assert L.selab200_init_devices(MAX_SLOTS + 1, C.addressof(arr)) == -3
        arr = (C.c_int * 2)(0, have)
        assert L.selab200_init_devices(2, C.addressof(arr)) == -3
    finally:
        _lib._initialised = None
        _lib.init(0)


# ------------------------------------------------------------------------------------------------------ CLI --

def test_cli_on_two_slots_of_one_device(tmp_path):
    """SELAB200_DEVICES=0,0 against SELAB200_DEVICE=0: -e and -d byte for byte, on a batch cut into two blocks."""
    if not (BIN / "sela").exists():
        subprocess.run(["make", "-C", str(ROOT / "sela_b200" / "host")], check=True, capture_output=True)
    sela = BIN / "sela"
    pcm = special_pcm(2 * BLOCK_MIN + 1, 2, 2, seed=9)
    wavio.write_wav(tmp_path / "in.wav", pcm, 48000)
    out = {}
    for name, env in (("one", {"SELAB200_DEVICE": "0"}), ("two", {"SELAB200_DEVICES": "0,0"})):
        base = {k: v for k, v in os.environ.items() if k not in ("SELAB200_DEVICE", "SELAB200_DEVICES")}
        e = subprocess.run([str(sela), "-e", str(tmp_path / "in.wav"), str(tmp_path / (name + ".sela"))],
                           capture_output=True, text=True, timeout=600, env=dict(base, **env))
        assert e.returncode == 0, e.stderr
        p = subprocess.run([str(sela), "-d", str(tmp_path / (name + ".sela")), str(tmp_path / (name + ".wav"))],
                           capture_output=True, text=True, timeout=600, env=dict(base, **env))
        assert p.returncode == 0, p.stderr
        out[name] = ((tmp_path / (name + ".sela")).read_bytes(), (tmp_path / (name + ".wav")).read_bytes())
    assert out["one"] == out["two"]
    assert out["one"][0] == sela_b200.encode_container(pcm, 2, 48000).tobytes()
    decoded = sela_b200.decode_container(out["one"][0])[1]       # the golden frames do not decode back to their source
    assert np.array_equal(wavio.read_wav_pcm(tmp_path / "two.wav")[2].reshape(-1), decoded)
