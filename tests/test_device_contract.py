"""The device-resident entry points (the *_device calls of include/sela_b200.h) under their whole contract.

Every call here goes straight to the C ABI on buffers this file owns: each buffer has exactly its documented size and
sits inside a larger allocation poisoned with 0x00, 0xFF, 0xA5 or seeded random bytes, with guard bytes on both sides.
A call must then produce the expected outputs byte for byte whatever the workspace and the outputs held before, reset
every counter it reports, and leave every byte it does not own unchanged: the guards, the word arena from
*d_words_used to its capacity, the PCM around an unaligned d_pcm or d_pcm_out.  Expected values: the oracle port for
the plain encode, the decode and the Rice residues; the host-buffer twin on the same PCM for every other mode (the
exact-model tests pin those twins).

  poison       every call on every pattern, with stream = NULL (the legacy default stream)
  leftovers    mode A, then mode B in the same workspace, then A again: each result is a fresh call's
  stream       each call on a torch stream behind a sleep, inputs copied in and outputs cloned on that stream, one
               synchronisation at the very end; an event recorded right after the call is still pending when it returns
  two streams  two calls interleaved on two streams, each behind its own sleep; the Rice-only call, whose split table
               lives in library scratch shared by every call, waits for the previous one (this cannot force the bad
               interleaving without the ordering; it shows that the second call waits)
  phases       non-stereo d_pcm and every d_pcm_out at byte phases 2, 4, .., 14 of a 16-byte block, inside other samples
  rejections   misaligned stereo PCM or verify reference, a workspace one byte short: SELAB200_ERR_ARGUMENT, no launch,
               nothing written
  devices      one pass with every buffer on device 1 (needs two GPUs)

Audit: every workspace region and device output of each call, and what writes it in the same call before any kernel
reads it (c_abi.cu unless another file is named).  No region is read before it is written, so poison never becomes an
address or an index.

  encode, every mode (encode_device, encode_layout)
    d_status, d_words_used      cudaMemsetAsync 0 before the first kernel; k_encode_scan reads *d_words_used
    d_ref_words                 memset 0 (search, guided); k_search_ref_words adds to it
    d_base_words                memset 0 (pairing, search + pairing, windows); k_pairing_select / k_window_base_words add
    d_n_difference, d_n_window  memset 0; k_pairing_select / k_window_repack add
    d_entries, d_n_entries      memset 0 (lossless), every record; k_lossless_report fills the re-coded pairs
    means                       k_unit_means, every unit
    units (UnitRecord)          k_encode_units / k_search_units, one CTA per unit; the repair, pairing and window
                                repacks rewrite them before k_encode_sizes reads them
    slots                       the unit kernels' pack, every unit; the repacks rewrite theirs; read by k_encode_gather
    residues                    each warp's row is written by its FIR before its Rice pass reads it; the head: tmp[1 + b]
                                by k_encode_sizes (every CTA b), tmp[0] by k_encode_scan's last CTA
    d_descs                     k_encode_scan, every subframe (k_pairing_patch after it)
    d_words                     k_encode_gather: [0, *d_words_used), nothing after a non-zero status
    repair count (lossless)     memset 0 (launch_encoder); frames, orig and units are appended under it and read
                                only below it (lossless.cuh)
    repair best                 set to kNoCandidate where k_lossless_select lists the unit
    SearchUnit (search modes)   k_search_units writes q, ref_order, ref_words and best of every unit (kernels.cuh)
    masks (guided)              k_search_estimate, every unit (search_guided.cuh)
    stale (pairing)             k_pairing_capture, every frame; search + pairing: memset 0 (launch_search_pairing)
    pair means                  k_pairing_means, every candidate (p, c) the later kernels read
    pair table                  k_pairing_candidates / k_search_pairing_table, every candidate; stereo (0, 1) by
                                k_pairing_select (pairing.cuh, search_pairing.cuh)
    par                         k_pairing_select, every frame and channel
    pair_search                 k_search_pairing_units, every candidate
    window su                   k_window_units, every (unit, window): q, ref_order, ref_words, best (window.cuh)
    window key                  memset 0xff (launch_windows)
  decode (decode_device)
    d_status                    memset 0
    ws_q                        k_rice_decode(refl): the lpc_order coefficients the synthesis reads of each subframe
    ws_res                      the residue pass: 2048 samples of every subframe (split decoder, then the general
                                parser on every flagged stream; or the general parser alone)
    seg_index                   memset 0xff, then k_decode_plan
    width counts (aux head)     k_decode_width_counts, every plan CTA, before k_decode_plan reads them
    split table, flags (aux)    k_rice_split_index, every stream (rice_vs.cuh); memset 0 where nothing is split
    d_pcm_out                   k_synthesise_segments, every sample of the independent subframes; k_diff_fixup the rest
  verify (verify_device): the decode's regions, then
    d_status, d_n_differing     memset 0
    d_entries                   memset 0, every record; k_verify_compare fills the differing pairs
    decoded PCM (workspace)     the decode, every sample
  rice_decode_frames_device
    d_status                    memset 0
    split table, flags (g.aux)  as in the decode; ordered after the previous user of g.aux by ev_rice (aux_for)
    d_residues                  every sample of every subframe

Run on the H100:  python -m pytest tests/test_device_contract.py -m gpu -q
"""
import ctypes as C
import functools
import time
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

import batch_model as B
import oracle_lib as ol
from sela_b200 import _lib, codec
from test_decode_clips import _pcm

pytestmark = pytest.mark.gpu

FRAME = 2048
ARGUMENT = -3
GUARD = 256                  # poisoned bytes on each side of every buffer
PATTERNS = ["00", "ff", "a5", "random"]
SLEEP = 200_000_000          # torch.cuda._sleep cycles: about 0.1 s
LONG_SLEEP = 1_000_000_000   # about 0.5 s
PHASES = list(range(2, 16, 2))


def L():
    return _lib.lib()


@functools.lru_cache(maxsize=None)
def O():
    return ol.load("port")


def u64(v):
    return np.array([v], "<u8").view(np.uint8)


def i32(v):
    return np.array([v], "<i4").view(np.uint8)


def as_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(-1)


# ------------------------------------------------------------------------------------------------ signals --

@functools.lru_cache(maxsize=None)
def signal(name):
    """(interleaved int16 PCM, channels)."""
    if name == "stereo":   # the stereo ties (difference wins by one word, loses by one, equal totals) and families
        bank = B.encode_bank(2)
        idx = [bank.index(n) for n in B.TIES] + list(range(8))
        return bank.pcm[idx].reshape(-1), 2
    if name == "oct":      # two frames the reference decoder does not reproduce, correlated channels, noise
        bank = B.encode_bank(8)
        idx = [bank.index(n) for n in ("lossy_a", "identical_0", "inverted_0", "sine_noise_0", "random_0",
                                       "full_noise_0", "lossy_b")]
        return bank.pcm[idx].reshape(-1), 8
    if name == "big":      # 1 040 stereo subframes: the encode scan and the decode plan span two CTAs
        bank = B.encode_bank(2)
        idx = np.random.default_rng(7).integers(0, len(bank), 520)
        idx[[511, 512, 513, 519]] = [bank.index(n) for n in B.TIES]
        return bank.pcm[idx].reshape(-1), 2
    ch = int(name[2:])     # "chN": two frames of sine + noise, channel 1 close to channel 0
    return np.ascontiguousarray(_pcm(ch, 2, seed=ch)).reshape(-1), ch


def frames(name):
    pcm, ch = signal(name)
    return pcm.size // (FRAME * ch), ch


# ------------------------------------------------------------------------------------------------- modes --

# encode mode -> (entry point, the counters it takes after d_words_used (before d_status), takes a mode argument)
ENCODE = {
    "plain": ("selab200_encode_frames_device", [], False),
    "lossless": ("selab200_encode_frames_lossless_device", ["entries", "n_entries"], False),
    "search": ("selab200_encode_frames_search_device", ["ref_words"], False),
    "guided": ("selab200_encode_frames_search_guided_device", ["ref_words"], True),
    "pairing": ("selab200_encode_frames_pairing_device", ["base_words", "n_difference"], False),
    "search_pairing": ("selab200_encode_frames_search_pairing_device", ["base_words", "n_difference"], False),
    "windows": ("selab200_encode_frames_search_windows_device", ["base_words", "n_window"], True),
}
ENCODE_FORMS = ["plain", "lossless", "search", "guided4", "pairing", "search_pairing", "windows1"]


def split_mode(mode):
    for kind in ("guided", "windows"):
        if mode.startswith(kind):
            return kind, int(mode[len(kind):])
    return mode, 0


def encode_ws_bytes(kind, arg, n, ch):
    if kind == "windows":
        return L().selab200_encode_search_windows_workspace_bytes(n, ch, arg)
    name = {"plain": "encode", "lossless": "encode_lossless", "search": "encode_search", "guided": "encode_search_guided",
            "pairing": "encode_pairing", "search_pairing": "encode_search_pairing"}[kind]
    return getattr(L(), "selab200_%s_workspace_bytes" % name)(n, ch)


@functools.lru_cache(maxsize=None)
def expected_encode(mode, name):
    """(descs, words, {counter or record buffer: expected bytes}) of `mode` on signal `name`."""
    pcm, ch = signal(name)
    n, _ = frames(name)
    kind, arg = split_mode(mode)
    if kind == "plain":
        d, w = O().encode_frames(pcm, ch)
        return d, w, {}
    if kind == "lossless":
        d, w, rep = codec.encode_frames_lossless(pcm, ch)
        full = np.zeros(n * ch, _lib.LOSSLESS_DTYPE)
        full[rep["frame"].astype(np.int64) * ch + rep["channel"]] = rep
        return d, w, {"entries": as_bytes(full), "n_entries": u64(rep.size)}
    if kind in ("search", "guided"):
        d, w, ref = (codec.encode_frames_search(pcm, ch) if kind == "search"
                     else codec.encode_frames_search_guided(pcm, ch, candidates=arg))
        return d, w, {"ref_words": u64(ref)}
    if kind in ("pairing", "search_pairing"):
        fn = codec.encode_frames_pairing if kind == "pairing" else codec.encode_frames_search_pairing
        d, w, base, nd = fn(pcm, ch)
        return d, w, {"base_words": u64(base), "n_difference": u64(nd)}
    d, w, base, nw = codec.encode_frames_search_windows(pcm, ch, windows=arg)
    return d, w, {"base_words": u64(base), "n_window": u64(nw)}


@functools.lru_cache(maxsize=None)
def expected_decode(name):
    pcm, ch = signal(name)
    d, w, _ = expected_encode("plain", name)
    return O().decode_frames(d, w, ch)


@functools.lru_cache(maxsize=None)
def expected_verify(name):
    pcm, ch = signal(name)
    n, _ = frames(name)
    d, w, _ = expected_encode("plain", name)
    rep = codec.verify_frames(d, w, ch, pcm)
    full = np.zeros(n * ch, _lib.VERIFY_DTYPE)
    full[rep["frame"].astype(np.int64) * ch + rep["channel"]] = rep
    return full, rep.size


@functools.lru_cache(maxsize=None)
def expected_residues(name):
    d, w, _ = expected_encode("plain", name)
    out = np.zeros((d.size, FRAME), np.int32)
    for i, s in enumerate(d):
        a = int(s["res_offset"])
        out[i] = O().rice_decode(w[a:a + int(s["res_words"])], int(s["res_rice_param"]), int(s["samples"]))
    return out


# ------------------------------------------------------------------------------------------------- cases --

@dataclass
class Case:
    """One call: `args` names buffers (str) or passes values (int); the stream comes last."""
    fn: str
    args: list
    sizes: dict                                  # buffer -> bytes
    inputs: dict                                 # buffer -> its bytes
    want: dict                                   # buffer -> expected bytes of its head; the rest keeps its poison
    scratch: tuple = ("ws",)                     # contents not checked (its guards are)
    phases: dict = field(default_factory=dict)   # buffer -> byte offset from a 256-byte boundary


def encode_case(mode, name, phases=None, short=0):
    pcm, ch = signal(name)
    n, _ = frames(name)
    kind, arg = split_mode(mode)
    fn, counters, with_arg = ENCODE[kind]
    cap = int(L().selab200_encode_words_bound(n, ch))
    ws = encode_ws_bytes(kind, arg, n, ch) - short
    args = ["pcm", n, ch] + ([arg] if with_arg else []) + ["descs", "words", cap, "used"] + counters + \
        ["status", "ws", ws]
    sizes = {"pcm": pcm.size * 2, "descs": n * ch * 32, "words": cap * 4, "used": 8, "status": 4, "ws": ws}
    sizes.update({c: n * ch * 16 if c == "entries" else 8 for c in counters})
    d, w, extra = expected_encode(mode, name)
    want = {"descs": as_bytes(d), "words": as_bytes(w.astype(np.uint32)), "used": u64(w.size), "status": i32(0)}
    want.update(extra)
    return Case(fn, args, sizes, {"pcm": as_bytes(pcm)}, want, phases=phases or {})


def coded(name):
    d, w, _ = expected_encode("plain", name)
    return d, w.astype(np.uint32)


def decode_case(name, phases=None, short=0):
    n, ch = frames(name)
    d, w = coded(name)
    ws = L().selab200_decode_workspace_bytes(n, ch) - short
    sizes = {"descs": d.size * 32, "words": w.size * 4, "pcm_out": d.size * FRAME * 2, "status": 4, "ws": ws}
    return Case("selab200_decode_frames_device", ["descs", n, ch, "words", w.size, "pcm_out", "status", "ws", ws],
                sizes, {"descs": as_bytes(d), "words": as_bytes(w)},
                {"pcm_out": as_bytes(expected_decode(name)), "status": i32(0)}, phases=phases or {})


def verify_case(name, phases=None, short=0):
    pcm, ch = signal(name)
    n, _ = frames(name)
    d, w = coded(name)
    ws = L().selab200_verify_workspace_bytes(n, ch) - short
    full, count = expected_verify(name)
    sizes = {"descs": d.size * 32, "words": w.size * 4, "ref": pcm.size * 2, "entries": d.size * 16, "count": 8,
             "status": 4, "ws": ws}
    return Case("selab200_verify_frames_device",
                ["descs", n, ch, "words", w.size, "ref", "entries", "count", "status", "ws", ws], sizes,
                {"descs": as_bytes(d), "words": as_bytes(w), "ref": as_bytes(pcm)},
                {"entries": as_bytes(full), "count": u64(count), "status": i32(0)}, phases=phases or {})


def rice_case(name):
    n, ch = frames(name)
    d, w = coded(name)
    sizes = {"descs": d.size * 32, "words": w.size * 4, "residues": d.size * FRAME * 4, "status": 4}
    return Case("selab200_rice_decode_frames_device", ["descs", n, ch, "words", w.size, "residues", "status"], sizes,
                {"descs": as_bytes(d), "words": as_bytes(w)},
                {"residues": as_bytes(expected_residues(name)), "status": i32(0)}, scratch=())


def case(cid, **kw):
    """"enc-<mode>-<signal>", "dec-<signal>", "verify-<signal>", "rice-<signal>"."""
    parts = cid.split("-")
    if parts[0] == "enc":
        return encode_case(parts[1], parts[2], **kw)
    return {"dec": decode_case, "verify": verify_case, "rice": rice_case}[parts[0]](parts[1], **kw)


CASES = ["enc-plain-stereo", "enc-plain-oct", "enc-plain-big",
         "enc-lossless-stereo", "enc-lossless-oct",
         "enc-search-stereo", "enc-search-oct",
         "enc-guided1-oct", "enc-guided4-stereo", "enc-guided100-oct",
         "enc-pairing-stereo", "enc-pairing-oct",
         "enc-search_pairing-stereo", "enc-search_pairing-oct",
         "enc-windows1-stereo", "enc-windows31-oct",
         "dec-stereo", "dec-oct", "dec-big",
         "verify-stereo", "verify-oct",
         "rice-stereo", "rice-oct", "rice-big"]


# ---------------------------------------------------------------------------------------------- buffers --

def poison(pattern, n, rng):
    if pattern == "random":
        return rng.integers(0, 256, n, dtype=np.uint8)
    return np.full(n, int(pattern, 16), np.uint8)


class Run:
    """The buffers of one call, each `phase` bytes past a 256-byte boundary inside an allocation poisoned with
    `pattern` that leaves at least GUARD bytes on either side.  shared: buffer -> (allocation, its poison), used as it
    is (leftovers of earlier calls included)."""

    def __init__(self, c, pattern, device=0, seed=0, shared=None):
        self.c, self.device = c, torch.device("cuda", device)
        rng = np.random.default_rng(seed)
        self.mem, self.poison, self.at = {}, {}, {}
        for name, size in c.sizes.items():
            self.at[name] = GUARD + c.phases.get(name, 0)
            if shared and name in shared:
                self.mem[name], self.poison[name] = shared[name]
                continue
            total = (self.at[name] + size + GUARD + 255) & ~255
            self.poison[name] = poison(pattern, total, rng)
            self.mem[name] = torch.from_numpy(self.poison[name]).to(self.device)
            assert self.mem[name].data_ptr() % 256 == 0
        self.stage = {k: torch.from_numpy(v.copy()).to(self.device) for k, v in c.inputs.items()}

    def ptr(self, name):
        return self.mem[name].data_ptr() + self.at[name]

    def view(self, name):
        return self.mem[name][self.at[name]:self.at[name] + self.c.sizes[name]]

    def load(self):
        """The inputs over their poison, on the current stream."""
        for name, t in self.stage.items():
            self.view(name).copy_(t)

    def call(self, stream):
        a = [self.ptr(x) if isinstance(x, str) else x for x in self.c.args]
        return getattr(L(), self.c.fn)(*a, stream)

    def snapshot(self):
        """Every allocation, cloned on the current stream."""
        return {k: m.clone() for k, m in self.mem.items()}

    def check(self, snap, written=True, what=""):
        """Outputs (written) or nothing (not written) over the poison and the inputs; scratch: only its guards."""
        for name, t in snap.items():
            got = t.cpu().numpy()
            want = self.poison[name].copy()
            lo, size = self.at[name], self.c.sizes[name]
            if name in self.c.inputs:
                want[lo:lo + size] = self.c.inputs[name]
            if written and name in self.c.want:
                exp = self.c.want[name]
                want[lo:lo + exp.size] = exp
            if name in self.c.scratch:
                got = np.concatenate([got[:lo], got[lo + size:]])
                want = np.concatenate([want[:lo], want[lo + size:]])
            if not np.array_equal(got, want):
                bad = np.flatnonzero(got != want) - lo
                pytest.fail("%s%s: %d bytes differ, first at %s (relative to the buffer, size %d)"
                            % (what, name, bad.size, bad[:8].tolist(), size))


def run(c, pattern="random", device=0, seed=0, shared=None, stream=None):
    """One call on the NULL stream: poison, inputs, call, outputs checked."""
    r = Run(c, pattern, device, seed, shared)
    r.load()
    rc = r.call(stream)
    assert rc == 0, L().selab200_last_error().decode()
    snap = r.snapshot()
    torch.cuda.synchronize(r.device)
    r.check(snap)
    return r


@pytest.fixture(scope="module", autouse=True)
def _init():
    _lib.init(0)
    yield
    torch.cuda.synchronize()


# --------------------------------------------------------------------------------------------- the tests --

def test_signals_reach_the_special_cases():
    """Stereo frames where the difference wins, a pairing that chooses parents, lossless repairs and a verify report
    on the lossy frames, and a batch above one scan CTA."""
    d, _, _ = expected_encode("plain", "stereo")
    assert (d["subframe_type"] == 1).any()
    for mode in ("pairing", "search_pairing"):
        assert int(expected_encode(mode, "oct")[2]["n_difference"].view("<u8")[0]) > 0
    assert int(expected_encode("lossless", "oct")[2]["n_entries"].view("<u8")[0]) > 0
    assert expected_verify("oct")[1] > 0
    assert np.prod(frames("big")) > B.SCAN_TILE


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("cid", CASES)
def test_poisoned_buffers(cid, pattern):
    run(case(cid), pattern, seed=len(cid))


@pytest.mark.parametrize("a,b", [("enc-windows31-oct", "enc-search_pairing-stereo"),
                                 ("enc-pairing-oct", "enc-lossless-stereo"),
                                 ("enc-guided100-stereo", "enc-plain-big"),
                                 ("verify-oct", "dec-big")])
def test_workspace_leftovers(a, b):
    """A, then B in the same workspace, then A again: every result is a fresh call's."""
    ca, cb = case(a), case(b)
    size = max(ca.sizes["ws"], cb.sizes["ws"])
    ca.sizes["ws"] = cb.sizes["ws"] = size           # one allocation; each call is passed its own workspace size
    p = poison("random", GUARD + size + GUARD, np.random.default_rng(3))
    shared = {"ws": (torch.from_numpy(p).cuda(), p)}
    for c in (ca, cb, ca):
        run(c, shared=shared)


@pytest.mark.parametrize("cid", CASES)
def test_caller_stream(cid):
    """Sleep, inputs, call and output clones on a stream of the caller's; one synchronisation at the end.  Work on
    another stream would read the poison or run before the inputs land; a host wait would find the event done."""
    c = case(cid)
    run(c, "a5")                    # kernels loaded and library scratch grown before the timed part
    r = Run(c, "random", seed=11)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP)
        r.load()
        rc = r.call(s.cuda_stream)
        ev = torch.cuda.Event()
        ev.record(s)
        pending = not ev.query()
        snap = r.snapshot()
    torch.cuda.synchronize()
    assert rc == 0, L().selab200_last_error().decode()
    assert pending, "the call waited for its stream"
    r.check(snap)


@pytest.mark.parametrize("a,b", [("enc-windows31-oct", "dec-big"), ("enc-lossless-oct", "verify-stereo"),
                                 ("rice-big", "rice-oct"), ("enc-search_pairing-oct", "rice-stereo")])
def test_two_streams_interleaved(a, b):
    """Two calls, each on its own stream behind its own sleep, issued alternately twice: serial results."""
    cs = [case(a), case(b)]
    for c in cs:
        run(c, "a5")
    runs = [[Run(c, "random", seed=10 * k + i) for i, c in enumerate(cs)] for k in range(2)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    snaps = []
    for k in range(2):
        for i, s in enumerate(streams):
            with torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP // (1 + i))
                runs[k][i].load()
                assert runs[k][i].call(s.cuda_stream) == 0, L().selab200_last_error().decode()
                snaps.append((runs[k][i], runs[k][i].snapshot()))
    torch.cuda.synchronize()
    for r, snap in snaps:
        r.check(snap)


def test_rice_calls_on_two_streams_wait_for_each_other():
    """The Rice-only call keeps its split table in library scratch: call B on stream 2 must wait for call A, issued
    on stream 1 behind a long sleep, rather than overwrite A's table before A has read it."""
    ca, cb = case("rice-big"), case("rice-oct")
    for c in (ca, cb):
        run(c, "a5")
    ra, rb = Run(ca, "random", seed=1), Run(cb, "random", seed=2)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        torch.cuda._sleep(LONG_SLEEP)
        ra.load()
        assert ra.call(s1.cuda_stream) == 0
        snap_a = ra.snapshot()
    with torch.cuda.stream(s2):
        rb.load()
        assert rb.call(s2.cuda_stream) == 0
        done_b = torch.cuda.Event()
        done_b.record(s2)
        snap_b = rb.snapshot()
    time.sleep(0.05)
    waited = not done_b.query()
    torch.cuda.synchronize()
    assert waited, "call B completed while call A's stream was still asleep"
    ra.check(snap_a, what="A ")
    rb.check(snap_b, what="B ")


@pytest.mark.parametrize("mode", ENCODE_FORMS)
@pytest.mark.parametrize("channels", [1, 3, 5, 8, 16])
def test_encode_pcm_at_every_phase(channels, mode):
    """Non-stereo d_pcm 2, 4, .., 14 bytes past a 16-byte boundary, random samples around it."""
    for phase in PHASES:
        run(encode_case(mode, "ch%d" % channels, phases={"pcm": phase}), seed=phase)


@pytest.mark.parametrize("channels", [1, 2, 3, 5, 8, 16])
def test_decode_output_at_every_phase(channels):
    """d_pcm_out 2, 4, .., 14 bytes past a 16-byte boundary, the samples on both sides unchanged."""
    for phase in PHASES:
        run(decode_case("ch%d" % channels, phases={"pcm_out": phase}), seed=phase)


def rejected(c):
    """The call returns SELAB200_ERR_ARGUMENT, launches nothing and writes nothing."""
    r = Run(c, "a5")
    r.load()
    torch.cuda.synchronize()
    before = L().selab200_launch_count()
    rc = r.call(None)
    assert L().selab200_launch_count() == before
    snap = r.snapshot()
    torch.cuda.synchronize()
    assert rc == ARGUMENT, rc
    r.check(snap, written=False)


def test_rejections():
    for mode in ENCODE_FORMS:
        for phase in PHASES:
            rejected(encode_case(mode, "stereo", phases={"pcm": phase}))
        rejected(encode_case(mode, "stereo", short=1))
        rejected(encode_case(mode, "ch3", short=1))
    for phase in PHASES:
        rejected(verify_case("oct", phases={"ref": phase}))
    rejected(verify_case("oct", short=1))
    rejected(decode_case("stereo", short=1))


def test_buffers_on_device_one():
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the pass with every buffer on device 1 needs a second one")
    _lib.init([0, 1])
    try:
        for cid in ("enc-plain-stereo", "enc-lossless-oct", "enc-search_pairing-oct", "enc-windows31-oct",
                    "enc-guided4-stereo", "dec-big", "verify-oct", "rice-oct"):
            run(case(cid), device=1)
    finally:
        torch.cuda.synchronize(1)
        _lib.init(0)
