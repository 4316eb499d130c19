"""Host-side Python mirror of the reference's operator interface for the hot path.

Function names follow the reference classes they stand for (argument meaning and
error behaviour as in include/sela_b200.h):

    encode_frames / decode_frames   sela::Encoder/Decoder::processFrames
                                    (= frame::FrameEncoder/FrameDecoder::process per frame)
    lpc_residues / lpc_samples      lpc::ResidueGenerator / lpc::SampleGenerator ::process
    rice_encode / rice_decode       rice::RiceEncoder / rice::RiceDecoder ::process
    encode_container / decode_container / container_info
                                    sela::Encoder::process + file::SelaFile::writeToFile, and
                                    file::SelaFile::readFromFile + sela::Decoder::processFrames,
                                    on the byte-packed .sela stream
    verify_frames / encode_container_verified / verify_container
                                    not in the reference: decode coded frames and compare them with
                                    their source PCM, reporting every (frame, channel) that differs
                                    (the format is not lossless for every input, DESIGN.md 7)
    encode_frames_lossless / encode_container_lossless
                                    not in the reference: encodes that decode back to their source, re-coding
                                    the few subframes the reference decoder would not reproduce (DESIGN.md 7.2)
    encode_frames_search / encode_container_search
                                    not in the reference: smaller files at a higher encode cost, every subframe
                                    coded at the predictor order with the fewest words (DESIGN.md 7.3)
    encode_trace / quantise_probe   for tests: the batch encoder's analysis intermediates, its
    / fir_probe / fir_tie_probe     order threshold and quantiser on chosen values, its FIR residual
                                    (and tie test) on chosen signals and predictors, and the lossless
    encode_frames_pairing / encode_container_pairing
                                    the encoder with the channel pairing (DESIGN.md 7.4), and its tests-only
                                    forms encode_pairing_forced / encode_pairing_trace
    encode_frames_search_pairing / encode_container_search_pairing
                                    the order search and the channel pairing together (DESIGN.md 7.5), and its
                                    tests-only forms encode_search_pairing_forced / encode_search_pairing_trace
    encode_frames_search_windows / encode_container_search_windows / analysis_window
                                    the order search over apodised analyses (DESIGN.md 7.6), its window table, and
                                    its tests-only forms encode_search_windows_forced / encode_search_windows_trace
    encode_frames_search_guided / encode_container_search_guided
                                    the order search over the orders an estimate ranks best (DESIGN.md 7.7), and its
                                    tests-only form encode_search_guided_trace
    encode_lossless_forced          encode with chosen predictors, and the order search with chosen
    / encode_search_forced          coefficients

Everything computes on the GPU through the C ABI; NumPy only carries host buffers.
The C++ mirror of the same interface (data::, frame::, file::, sela:: classes and
the `sela` CLI) is in sela_b200/host/.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import (DESC_DTYPE, FRAME, INFO_DTYPE, LOSSLESS_DTYPE, MAX_ORDER, PREDICTOR_DTYPE,  # noqa: F401
                   SEARCH_TRACE_DTYPE, SEARCH_UNIT_DTYPE, TRACE_DTYPE, VERIFY_DTYPE, SelaB200Error, check, init, lib)


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def encode_frames(pcm, channels, words_capacity=None, device=0):
    """pcm: int16, n_frames*2048*channels interleaved samples -> (descs, words)."""
    init(device)
    pcm = _c(pcm, np.int16).reshape(-1)
    n_frames = pcm.size // (FRAME * channels)
    if n_frames * FRAME * channels != pcm.size:
        raise ValueError("pcm must hold whole 2048-sample frames")
    L = lib()
    cap = words_capacity if words_capacity is not None else L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used = C.c_size_t(0)
    check(L.selab200_encode_frames(pcm.ctypes.data, n_frames, channels, descs.ctypes.data, words.ctypes.data,
                                   cap, C.addressof(used)))
    return descs, words[:used.value].copy()


def encode_trace(pcm, channels, device=0):
    """encode_frames on one batch through the tracing analysis kernel -> (descs, words, trace).

    trace: TRACE_DTYPE[n_units], one record per analysis unit, frame after frame; within a frame the channels,
    or for stereo ch0, ch1 and ch0 - ch1."""
    init(device)
    pcm = _c(pcm, np.int16).reshape(-1)
    n_frames = pcm.size // (FRAME * channels)
    if n_frames * FRAME * channels != pcm.size:
        raise ValueError("pcm must hold whole 2048-sample frames")
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    trace = np.zeros(n_frames * (3 if channels == 2 else channels), TRACE_DTYPE)
    used = C.c_size_t(0)
    check(L.selab200_encode_trace(pcm.ctypes.data, n_frames, channels, descs.ctypes.data, words.ctypes.data, cap,
                                  C.addressof(used), trace.ctypes.data))
    return descs, words[:used.value].copy(), trace


def quantise_probe(k, device=0):
    """float64 k[n] -> int32 [n, 4]: the encoder's q of each k as coefficient 0, 1 and any later one, and
    whether |k| > 0.05 (the coefficient counts for the order)."""
    init(device)
    k = _c(k, np.float64).reshape(-1)
    out = np.zeros((k.size, 4), np.int32)
    check(lib().selab200_quantise_probe(k.ctypes.data, k.size, out.ctypes.data))
    return out


def fir_probe(samples, orders, c, wide, device=0):
    """The encoder's FIR residual on chosen signals: samples int32 [n, 2048] (-32768..32767 as a channel row, or
    |s| <= 65535 with wide=True as a 17-bit row), orders [n], c int64 [n, 101] (the Q35 predictor, c[:, 0] unused)
    -> residues int32 [n, 2048]."""
    init(device)
    samples = _c(samples, np.int32).reshape(-1, FRAME)
    n = samples.shape[0]
    orders = _c(orders, np.int32).reshape(n)
    c = _c(c, np.int64).reshape(n, MAX_ORDER + 1)
    res = np.zeros((n, FRAME), np.int32)
    check(lib().selab200_fir_probe(samples.ctypes.data, orders.ctypes.data, c.ctypes.data, n, int(bool(wide)),
                                   res.ctypes.data))
    return res


def fir_tie_probe(samples, orders, c, wide, device=0):
    """fir_probe through the lossless encode's FIR, which also tests every output for a tie -> (residues int32
    [n, 2048], ties bool[n]: whether any output of the signal ties)."""
    init(device)
    samples = _c(samples, np.int32).reshape(-1, FRAME)
    n = samples.shape[0]
    orders = _c(orders, np.int32).reshape(n)
    c = _c(c, np.int64).reshape(n, MAX_ORDER + 1)
    res = np.zeros((n, FRAME), np.int32)
    ties = np.zeros(max(n, 1), np.uint8)
    check(lib().selab200_fir_tie_probe(samples.ctypes.data, orders.ctypes.data, c.ctypes.data, n, int(bool(wide)),
                                       res.ctypes.data, ties.ctypes.data))
    return res, ties[:n].astype(bool)


def encode_lossless_forced(pcm, channels, predictors, device=0):
    """encode_frames_lossless on one batch, every analysis unit coded with its predictor from `predictors`
    (PREDICTOR_DTYPE[n_units], or a sequence of (order, q) pairs, in encode_trace's unit order) instead of its
    analysis' -> (descs, words, report)."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    n_units = n_frames * (3 if channels == 2 else channels)
    if isinstance(predictors, np.ndarray) and predictors.dtype == PREDICTOR_DTYPE:
        pred = _c(predictors, PREDICTOR_DTYPE)
    else:
        pred = np.zeros(len(predictors), PREDICTOR_DTYPE)
        for rec, (order, q) in zip(pred, predictors):
            rec["order"] = order
            rec["q"][:order] = np.asarray(q)[:order]
    if pred.size != n_units:
        raise ValueError("%d predictors for %d analysis units" % (pred.size, n_units))
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used = C.c_size_t(0)
    report = np.zeros(max(n_frames * channels, 1), LOSSLESS_DTYPE)
    n = C.c_size_t(0)
    check(L.selab200_encode_lossless_forced(pcm.ctypes.data, n_frames, channels, pred.ctypes.data, descs.ctypes.data,
                                            words.ctypes.data, cap, C.addressof(used), report.ctypes.data, report.size,
                                            C.addressof(n)))
    return descs, words[:used.value].copy(), report[:n.value].copy()


def decode_frames(descs, words, channels, device=0):
    """(descs, words) -> int16 interleaved PCM, n_frames*2048*channels samples."""
    init(device)
    descs = _c(descs, DESC_DTYPE)
    words = _c(words, np.uint32)
    n_frames = descs.size // channels
    if n_frames * channels != descs.size:
        raise ValueError("descs must hold `channels` subframes per frame")
    pcm = np.empty(n_frames * FRAME * channels, np.int16)
    check(lib().selab200_decode_frames(descs.ctypes.data, n_frames, channels, words.ctypes.data, words.size,
                                       pcm.ctypes.data))
    return pcm


def lpc_residues(samples, device=0):
    """int32 [n_sub, 2048] -> (order u8[n_sub], q int32[n_sub,100], residues int32[n_sub,2048])."""
    init(device)
    samples = _c(samples, np.int32).reshape(-1, FRAME)
    n = samples.shape[0]
    order = np.zeros(n, np.uint8)
    q = np.zeros((n, MAX_ORDER), np.int32)
    res = np.zeros((n, FRAME), np.int32)
    check(lib().selab200_lpc_residues(samples.ctypes.data, n, order.ctypes.data, q.ctypes.data, res.ctypes.data))
    return order, q, res


def lpc_samples(residues, order, q, device=0):
    init(device)
    residues = _c(residues, np.int32).reshape(-1, FRAME)
    n = residues.shape[0]
    order = _c(order, np.uint8).reshape(n)
    qq = np.zeros((n, MAX_ORDER), np.int32)
    q = np.asarray(q)
    qq[:, :q.shape[1]] = q
    out = np.zeros((n, FRAME), np.int32)
    check(lib().selab200_lpc_samples(residues.ctypes.data, n, order.ctypes.data, qq.ctypes.data, out.ctypes.data))
    return out


def rice_encode(values, counts=None, words_stride=None, device=0):
    """values int32 [n_streams, stride] (stride <= 2048) -> (k u32[n], n_words u32[n], words u32[n, words_stride])."""
    init(device)
    values = _c(values, np.int32)
    if values.ndim == 1:
        values = values.reshape(1, -1)
    n, stride = values.shape
    counts = np.full(n, stride, np.uint32) if counts is None else _c(counts, np.uint32)
    if words_stride is None:
        words_stride = stride * 2 + 8
    k = np.zeros(n, np.uint32)
    nw = np.zeros(n, np.uint32)
    words = np.zeros((n, words_stride), np.uint32)
    check(lib().selab200_rice_encode(values.ctypes.data, counts.ctypes.data, n, stride, k.ctypes.data,
                                     nw.ctypes.data, words.ctypes.data, words_stride))
    return k, nw, words


def rice_decode(words, n_words, k, counts, out_stride=None, device=0):
    init(device)
    words = _c(words, np.uint32)
    if words.ndim == 1:
        words = words.reshape(1, -1)
    n, words_stride = words.shape
    n_words = _c(n_words, np.uint32).reshape(n)
    k = _c(k, np.uint32).reshape(n)
    counts = _c(counts, np.uint32).reshape(n)
    if out_stride is None:
        out_stride = int(counts.max()) if n else 0
    out = np.zeros((n, max(out_stride, 1)), np.int32)
    check(lib().selab200_rice_decode(words.ctypes.data, n_words.ctypes.data, words_stride, k.ctypes.data,
                                     counts.ctypes.data, n, out.ctypes.data, out_stride))
    return out


def encode_container(pcm, channels, sample_rate, bits_per_sample=16, capacity=None, device=0):
    """int16 interleaved PCM (whole frames) -> the bytes of the .sela file (uint8 array)."""
    init(device)
    pcm = _c(pcm, np.int16).reshape(-1)
    n_frames = pcm.size // (FRAME * channels)
    if n_frames * FRAME * channels != pcm.size:
        raise ValueError("pcm must hold whole 2048-sample frames")
    L = lib()
    cap = capacity if capacity is not None else L.selab200_container_bound(n_frames, channels)
    out = np.empty(max(cap, 1), np.uint8)
    used = C.c_size_t(0)
    check(L.selab200_encode_container(pcm.ctypes.data, n_frames, channels, sample_rate, bits_per_sample,
                                      out.ctypes.data, cap, C.addressof(used)))
    return out[:used.value]


def container_info(container):
    """Header fields and frame walk of a .sela byte stream (host only, no device needed)."""
    buf = _c(np.frombuffer(container, np.uint8) if isinstance(container, (bytes, bytearray)) else container, np.uint8)
    info = np.zeros(1, INFO_DTYPE)
    check(lib().selab200_container_info_get(buf.ctypes.data, buf.size, info.ctypes.data))
    return {k: int(info[0][k]) for k in INFO_DTYPE.names if k != "reserved"}


def container_frame_offsets(container):
    """(info dict, uint64 array of n_frames+1 byte offsets: frame starts and the end) -- host only."""
    buf = _c(np.frombuffer(container, np.uint8) if isinstance(container, (bytes, bytearray)) else container, np.uint8)
    info = np.zeros(1, INFO_DTYPE)
    L = lib()
    check(L.selab200_container_info_get(buf.ctypes.data, buf.size, info.ctypes.data))
    offsets = np.zeros(int(info[0]["n_frames"]) + 1, np.uint64)
    check(L.selab200_container_frame_offsets(buf.ctypes.data, buf.size, offsets.ctypes.data, offsets.size,
                                             info.ctypes.data))
    return {k: int(info[0][k]) for k in INFO_DTYPE.names if k != "reserved"}, offsets


def decode_container(container, device=0):
    """.sela byte stream -> (info dict, int16 interleaved PCM of info['n_frames'] frames)."""
    init(device)
    buf = _c(np.frombuffer(container, np.uint8) if isinstance(container, (bytes, bytearray)) else container, np.uint8)
    L = lib()
    info = np.zeros(1, INFO_DTYPE)
    handle = C.c_void_p(0)
    check(L.selab200_container_open(buf.ctypes.data, buf.size, C.addressof(handle), info.ctypes.data))
    try:
        n = int(info[0]["n_frames"]) * int(info[0]["channels"]) * FRAME
        pcm = np.empty(n, np.int16)
        check(L.selab200_container_decode(handle, pcm.ctypes.data))
    finally:
        L.selab200_container_close(handle)
    return {k: int(info[0][k]) for k in INFO_DTYPE.names if k != "reserved"}, pcm


def _whole_frames(pcm, channels):
    pcm = _c(pcm, np.int16).reshape(-1)
    n_frames = pcm.size // (FRAME * channels)
    if n_frames * FRAME * channels != pcm.size:
        raise ValueError("pcm must hold whole 2048-sample frames")
    return pcm, n_frames


def verify_frames(descs, words, channels, pcm, device=0):
    """Decode (descs, words) as decode_frames does and compare with pcm (int16, interleaved, the same frames)
    -> VERIFY_DTYPE array: one entry per (frame, channel) whose decoded samples differ, in that order."""
    init(device)
    descs = _c(descs, DESC_DTYPE)
    words = _c(words, np.uint32)
    n_frames = descs.size // channels
    if n_frames * channels != descs.size:
        raise ValueError("descs must hold `channels` subframes per frame")
    pcm, n_pcm = _whole_frames(pcm, channels)
    if n_pcm != n_frames:
        raise ValueError("pcm holds %d frames, descs %d" % (n_pcm, n_frames))
    report = np.zeros(max(descs.size, 1), VERIFY_DTYPE)
    n = C.c_size_t(0)
    check(lib().selab200_verify_frames(descs.ctypes.data, n_frames, channels, words.ctypes.data, words.size,
                                       pcm.ctypes.data, report.ctypes.data, report.size, C.addressof(n)))
    return report[:n.value].copy()


def encode_container_verified(pcm, channels, sample_rate, bits_per_sample=16, capacity=None, device=0):
    """encode_container, plus a check that the returned bytes decode back to pcm -> (bytes, report), the
    report as verify_frames returns it.  The bytes are those encode_container returns."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = capacity if capacity is not None else L.selab200_container_bound(n_frames, channels)
    out = np.empty(max(cap, 1), np.uint8)
    used = C.c_size_t(0)
    report = np.zeros(max(n_frames * channels, 1), VERIFY_DTYPE)
    n = C.c_size_t(0)
    check(L.selab200_encode_container_verified(pcm.ctypes.data, n_frames, channels, sample_rate, bits_per_sample,
                                               out.ctypes.data, cap, C.addressof(used), report.ctypes.data,
                                               report.size, C.addressof(n)))
    return out[:used.value], report[:n.value].copy()


def verify_container(container, pcm, device=0):
    """.sela byte stream and the PCM it should decode to (int16 interleaved, info['n_frames'] frames)
    -> (info dict, report as verify_frames returns it)."""
    init(device)
    buf = _c(np.frombuffer(container, np.uint8) if isinstance(container, (bytes, bytearray)) else container, np.uint8)
    L = lib()
    info = np.zeros(1, INFO_DTYPE)
    handle = C.c_void_p(0)
    check(L.selab200_container_open(buf.ctypes.data, buf.size, C.addressof(handle), info.ctypes.data))
    try:
        n_frames, channels = int(info[0]["n_frames"]), int(info[0]["channels"])
        pcm = _c(pcm, np.int16).reshape(-1)
        if pcm.size != n_frames * channels * FRAME:
            raise ValueError("pcm holds %d samples, the container %d frames of %d channels"
                             % (pcm.size, n_frames, channels))
        report = np.zeros(max(n_frames * channels, 1), VERIFY_DTYPE)
        n = C.c_size_t(0)
        check(L.selab200_container_verify(handle, pcm.ctypes.data, report.ctypes.data, report.size, C.addressof(n)))
    finally:
        L.selab200_container_close(handle)
    return {k: int(info[0][k]) for k in INFO_DTYPE.names if k != "reserved"}, report[:n.value].copy()


def encode_frames_lossless(pcm, channels, words_capacity=None, device=0):
    """encode_frames, lossless -> (descs, words, report).  report: LOSSLESS_DTYPE array, one entry per re-coded
    (frame, channel) in that order: the reference encoder's order and words there, and the emitted ones."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = words_capacity if words_capacity is not None else L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used = C.c_size_t(0)
    report = np.zeros(max(n_frames * channels, 1), LOSSLESS_DTYPE)
    n = C.c_size_t(0)
    check(L.selab200_encode_frames_lossless(pcm.ctypes.data, n_frames, channels, descs.ctypes.data, words.ctypes.data,
                                            cap, C.addressof(used), report.ctypes.data, report.size, C.addressof(n)))
    return descs, words[:used.value].copy(), report[:n.value].copy()


def encode_container_lossless(pcm, channels, sample_rate, bits_per_sample=16, capacity=None, device=0):
    """encode_container, lossless -> (bytes, report), the report as encode_frames_lossless returns it."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = capacity if capacity is not None else L.selab200_container_bound(n_frames, channels)
    out = np.empty(max(cap, 1), np.uint8)
    used = C.c_size_t(0)
    report = np.zeros(max(n_frames * channels, 1), LOSSLESS_DTYPE)
    n = C.c_size_t(0)
    check(L.selab200_encode_container_lossless(pcm.ctypes.data, n_frames, channels, sample_rate, bits_per_sample,
                                               out.ctypes.data, cap, C.addressof(used), report.ctypes.data,
                                               report.size, C.addressof(n)))
    return out[:used.value], report[:n.value].copy()


def encode_frames_search(pcm, channels, words_capacity=None, device=0):
    """encode_frames with the order search (DESIGN.md 7.3) -> (descs, words, ref_words): ref_words is the number of
    words encode_frames writes for the same frames."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = words_capacity if words_capacity is not None else L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used, ref = C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_frames_search(pcm.ctypes.data, n_frames, channels, descs.ctypes.data, words.ctypes.data,
                                          cap, C.addressof(used), C.addressof(ref)))
    return descs, words[:used.value].copy(), ref.value


def encode_container_search(pcm, channels, sample_rate, bits_per_sample=16, capacity=None, device=0):
    """encode_container with the order search -> (bytes, ref_bytes): ref_bytes is the size of encode_container's
    output for the same frames."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = capacity if capacity is not None else L.selab200_container_bound(n_frames, channels)
    out = np.empty(max(cap, 1), np.uint8)
    used, ref = C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_container_search(pcm.ctypes.data, n_frames, channels, sample_rate, bits_per_sample,
                                             out.ctypes.data, cap, C.addressof(used), C.addressof(ref)))
    return out[:used.value], ref.value


def encode_search_forced(pcm, channels, predictors, device=0):
    """encode_frames_search on one batch, every analysis unit taking its 100 quantised reflection coefficients and
    its reference order from `predictors` (PREDICTOR_DTYPE[n_units], or a sequence of (order, q[100]) pairs, in
    encode_trace's unit order) instead of its analysis -> (descs, words, ref_words)."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    pred = _search_predictors(predictors, n_frames * (3 if channels == 2 else channels))
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used, ref = C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_search_forced(pcm.ctypes.data, n_frames, channels, pred.ctypes.data, descs.ctypes.data,
                                          words.ctypes.data, cap, C.addressof(used), C.addressof(ref)))
    return descs, words[:used.value].copy(), ref.value


def _search_predictors(predictors, n_units):
    if isinstance(predictors, np.ndarray) and predictors.dtype == PREDICTOR_DTYPE:
        pred = _c(predictors, PREDICTOR_DTYPE)
    else:
        pred = np.zeros(len(predictors), PREDICTOR_DTYPE)
        for rec, (order, q) in zip(pred, predictors):
            rec["order"] = order
            rec["q"][:] = np.asarray(q)[:MAX_ORDER]
    if pred.size != n_units:
        raise ValueError("%d predictors for %d analysis units" % (pred.size, n_units))
    return pred


def encode_search_trace(pcm, channels, predictors=None, device=0):
    """encode_frames_search (encode_search_forced's with `predictors`) on one batch through the tracing search
    kernels -> (descs, words, ref_words, units, trace).

    units: SEARCH_UNIT_DTYPE[n_units], every analysis unit's q[100], reference order and words and winning key;
    trace: SEARCH_TRACE_DTYPE[n_units, 100], the record of every unit at every order 1..100 (column order - 1).
    Units in encode_trace's order."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    n_units = n_frames * (3 if channels == 2 else channels)
    pred = None if predictors is None else _search_predictors(predictors, n_units)
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    units = np.zeros(n_units, SEARCH_UNIT_DTYPE)
    trace = np.zeros((n_units, MAX_ORDER), SEARCH_TRACE_DTYPE)
    used, ref = C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_search_trace(pcm.ctypes.data, n_frames, channels, None if pred is None else pred.ctypes.data,
                                         descs.ctypes.data, words.ctypes.data, cap, C.addressof(used),
                                         C.addressof(ref), units.ctypes.data, trace.ctypes.data))
    return descs, words[:used.value].copy(), ref.value, units, trace


def encode_frames_search_guided(pcm, channels, candidates=4, words_capacity=None, device=0):
    """encode_frames with the guided order search (DESIGN.md 7.7) -> (descs, words, ref_words): the order search over
    the `candidates` (1..100) orders a reflection-coefficient estimate ranks best, order 1 and the reference order.
    ref_words is the number of words encode_frames writes for the same frames; candidates=100 gives
    encode_frames_search's output."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = words_capacity if words_capacity is not None else L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used, ref = C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_frames_search_guided(pcm.ctypes.data, n_frames, channels, candidates, descs.ctypes.data,
                                                 words.ctypes.data, cap, C.addressof(used), C.addressof(ref)))
    return descs, words[:used.value].copy(), ref.value


def encode_container_search_guided(pcm, channels, sample_rate, candidates=4, bits_per_sample=16, capacity=None,
                                   device=0):
    """encode_container with the guided order search -> (bytes, ref_bytes): ref_bytes is the size of
    encode_container's output for the same frames."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = capacity if capacity is not None else L.selab200_container_bound(n_frames, channels)
    out = np.empty(max(cap, 1), np.uint8)
    used, ref = C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_container_search_guided(pcm.ctypes.data, n_frames, channels, candidates, sample_rate,
                                                    bits_per_sample, out.ctypes.data, cap, C.addressof(used),
                                                    C.addressof(ref)))
    return out[:used.value], ref.value


def encode_search_guided_trace(pcm, channels, candidates, predictors=None, device=0):
    """encode_frames_search_guided (with `predictors`, every unit's q[100] and reference order as encode_search_forced
    takes them) on one batch through the tracing kernels -> (descs, words, ref_words, trace, estimates, masks).

    trace: SEARCH_TRACE_DTYPE[n_units, 100], the record of every order sized (column order - 1; visits 0 where the
    order was not sized); estimates: float64 [n_units, 100], E_order at order - 1; masks: bool [n_units, 100], the
    listed orders.  Units in encode_trace's order."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    n_units = n_frames * (3 if channels == 2 else channels)
    pred = None if predictors is None else _search_predictors(predictors, n_units)
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    trace = np.zeros((n_units, MAX_ORDER), SEARCH_TRACE_DTYPE)
    est = np.zeros((n_units, MAX_ORDER), np.float64)
    masks = np.zeros((n_units, 4), np.uint32)
    used, ref = C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_search_guided_trace(pcm.ctypes.data, n_frames, channels, candidates,
                                                None if pred is None else pred.ctypes.data, descs.ctypes.data,
                                                words.ctypes.data, cap, C.addressof(used), C.addressof(ref),
                                                trace.ctypes.data, est.ctypes.data, masks.ctypes.data))
    listed = ((masks[:, np.arange(MAX_ORDER) // 32] >> (np.arange(MAX_ORDER) % 32).astype(np.uint32)) & 1).astype(bool)
    return descs, words[:used.value].copy(), ref.value, trace, est, listed


def encode_frames_pairing(pcm, channels, words_capacity=None, device=0):
    """encode_frames with the channel pairing (DESIGN.md 7.4) -> (descs, words, base_words, n_difference): base_words
    is the number of words encode_frames_lossless writes for the same frames, n_difference the number of difference
    subframes emitted."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = words_capacity if words_capacity is not None else L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used, base, nd = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_frames_pairing(pcm.ctypes.data, n_frames, channels, descs.ctypes.data, words.ctypes.data,
                                           cap, C.addressof(used), C.addressof(base), C.addressof(nd)))
    return descs, words[:used.value].copy(), base.value, nd.value


def encode_container_pairing(pcm, channels, sample_rate, bits_per_sample=16, capacity=None, device=0):
    """encode_container with the channel pairing -> (bytes, base_bytes, n_difference): base_bytes is the size of
    encode_container_lossless's output for the same frames."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = capacity if capacity is not None else L.selab200_container_bound(n_frames, channels)
    out = np.empty(max(cap, 1), np.uint8)
    used, base, nd = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_container_pairing(pcm.ctypes.data, n_frames, channels, sample_rate, bits_per_sample,
                                              out.ctypes.data, cap, C.addressof(used), C.addressof(base),
                                              C.addressof(nd)))
    return out[:used.value], base.value, nd.value


def _pairing_predictors(predictors, n_frames, channels, every_q=False):
    """every_q: the search's form, q[0..99] whatever the order."""
    n = n_frames * ((3 if channels == 2 else channels) + channels * (channels - 1))
    if isinstance(predictors, np.ndarray) and predictors.dtype == PREDICTOR_DTYPE:
        pred = _c(predictors, PREDICTOR_DTYPE)
    else:
        pred = np.zeros(len(predictors), PREDICTOR_DTYPE)
        for rec, (order, q) in zip(pred, predictors):
            rec["order"] = order
            n_q = MAX_ORDER if every_q else order
            rec["q"][:n_q] = np.asarray(q)[:n_q]
    if pred.size != n:
        raise ValueError("%d predictors for %d units and candidates" % (pred.size, n))
    return pred


def encode_pairing_trace(pcm, channels, predictors=None, device=0):
    """encode_frames_pairing on one batch, and what the pairing kernels saw -> (descs, words, base_words,
    n_difference, par, trace).

    predictors (None: analyse): PREDICTOR_DTYPE records or (order, q) pairs, the base's analysis units in
    encode_trace's order, then one per candidate in (frame, p, c) order without p = c.  par: uint8 [n_frames,
    channels], the parent chosen per channel.  trace: SEARCH_TRACE_DTYPE [n_frames, channels, channels], entry
    [f, p, c] the candidate ch_p - ch_c as it was sized, its order in reserved[0]."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    pred = None if predictors is None else _pairing_predictors(predictors, n_frames, channels)
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    par = np.zeros((n_frames, channels), np.uint8)
    trace = np.zeros((n_frames, channels, channels), SEARCH_TRACE_DTYPE)
    used, base, nd = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_pairing_trace(pcm.ctypes.data, n_frames, channels,
                                          None if pred is None else pred.ctypes.data, descs.ctypes.data,
                                          words.ctypes.data, cap, C.addressof(used), C.addressof(base),
                                          C.addressof(nd), par.ctypes.data, trace.ctypes.data))
    return descs, words[:used.value].copy(), base.value, nd.value, par, trace


def encode_pairing_forced(pcm, channels, predictors, device=0):
    """encode_frames_pairing on one batch with every unit and candidate coded with its predictor from `predictors`
    (as encode_pairing_trace takes them) -> (descs, words, base_words, n_difference)."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    pred = _pairing_predictors(predictors, n_frames, channels)
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used, base, nd = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_pairing_forced(pcm.ctypes.data, n_frames, channels, pred.ctypes.data, descs.ctypes.data,
                                           words.ctypes.data, cap, C.addressof(used), C.addressof(base),
                                           C.addressof(nd)))
    return descs, words[:used.value].copy(), base.value, nd.value


def encode_frames_search_pairing(pcm, channels, words_capacity=None, device=0):
    """encode_frames with the order search and the channel pairing together (DESIGN.md 7.5) -> (descs, words,
    base_words, n_difference): base_words is the number of words encode_frames_search writes for the same frames,
    n_difference the number of difference subframes emitted."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = words_capacity if words_capacity is not None else L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used, base, nd = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_frames_search_pairing(pcm.ctypes.data, n_frames, channels, descs.ctypes.data,
                                                  words.ctypes.data, cap, C.addressof(used), C.addressof(base),
                                                  C.addressof(nd)))
    return descs, words[:used.value].copy(), base.value, nd.value


def encode_container_search_pairing(pcm, channels, sample_rate, bits_per_sample=16, capacity=None, device=0):
    """encode_container with the order search and the channel pairing -> (bytes, base_bytes, n_difference):
    base_bytes is the size of encode_container_search's output for the same frames."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = capacity if capacity is not None else L.selab200_container_bound(n_frames, channels)
    out = np.empty(max(cap, 1), np.uint8)
    used, base, nd = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_container_search_pairing(pcm.ctypes.data, n_frames, channels, sample_rate,
                                                     bits_per_sample, out.ctypes.data, cap, C.addressof(used),
                                                     C.addressof(base), C.addressof(nd)))
    return out[:used.value], base.value, nd.value


def encode_search_pairing_trace(pcm, channels, predictors=None, device=0):
    """encode_frames_search_pairing on one batch through the tracing candidate kernels -> (descs, words, base_words,
    n_difference, par, trace).

    predictors (None: analyse): PREDICTOR_DTYPE records or (order, q[100]) pairs, as encode_search_forced takes
    them: the base's analysis units in encode_trace's order, then one per candidate in (frame, p, c) order without
    p = c.  par: uint8 [n_frames, channels], the parent chosen per channel.  trace: SEARCH_TRACE_DTYPE [n_frames,
    channels, channels, 100], entry [f, p, c, order - 1] the candidate ch_p - ch_c at that order."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    pred = None if predictors is None else _pairing_predictors(predictors, n_frames, channels, every_q=True)
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    par = np.zeros((n_frames, channels), np.uint8)
    trace = np.zeros((n_frames, channels, channels, MAX_ORDER), SEARCH_TRACE_DTYPE)
    used, base, nd = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_search_pairing_trace(pcm.ctypes.data, n_frames, channels,
                                                 None if pred is None else pred.ctypes.data, descs.ctypes.data,
                                                 words.ctypes.data, cap, C.addressof(used), C.addressof(base),
                                                 C.addressof(nd), par.ctypes.data, trace.ctypes.data))
    return descs, words[:used.value].copy(), base.value, nd.value, par, trace


def encode_search_pairing_forced(pcm, channels, predictors, device=0):
    """encode_frames_search_pairing on one batch with every unit and candidate taking its q[0..99] and reference
    order from `predictors` (as encode_search_pairing_trace takes them) -> (descs, words, base_words, n_difference)."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    pred = _pairing_predictors(predictors, n_frames, channels, every_q=True)
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used, base, nd = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_search_pairing_forced(pcm.ctypes.data, n_frames, channels, pred.ctypes.data,
                                                  descs.ctypes.data, words.ctypes.data, cap, C.addressof(used),
                                                  C.addressof(base), C.addressof(nd)))
    return descs, words[:used.value].copy(), base.value, nd.value


def analysis_window(index):
    """Row `index` (0..4) of the window search's table (DESIGN.md 7.6) -> float64 [2048], the exact doubles the
    encoder multiplies by: 0 Tukey(0.5), 1 Tukey(0.25), 2 Hann, 3 and 4 Tukey(0.5) over the first and the second half
    of the frame.  Needs no device."""
    out = np.zeros(FRAME, np.float64)
    check(lib().selab200_analysis_window(int(index), out.ctypes.data))
    return out


def encode_frames_search_windows(pcm, channels, windows=1, words_capacity=None, device=0):
    """encode_frames with the window search (DESIGN.md 7.6) -> (descs, words, base_words, n_window).  windows: a mask
    over analysis_window's rows (1: Tukey(0.5)).  base_words is the number of words encode_frames_search writes for
    the same frames, n_window the number of analysis units coded from a window."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = words_capacity if words_capacity is not None else L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used, base, nw = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_frames_search_windows(pcm.ctypes.data, n_frames, channels, windows, descs.ctypes.data,
                                                  words.ctypes.data, cap, C.addressof(used), C.addressof(base),
                                                  C.addressof(nw)))
    return descs, words[:used.value].copy(), base.value, nw.value


def encode_container_search_windows(pcm, channels, sample_rate, windows=1, bits_per_sample=16, capacity=None,
                                    device=0):
    """encode_container with the window search -> (bytes, base_bytes, n_window): base_bytes is the size of
    encode_container_search's output for the same frames."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    L = lib()
    cap = capacity if capacity is not None else L.selab200_container_bound(n_frames, channels)
    out = np.empty(max(cap, 1), np.uint8)
    used, base, nw = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_container_search_windows(pcm.ctypes.data, n_frames, channels, windows, sample_rate,
                                                     bits_per_sample, out.ctypes.data, cap, C.addressof(used),
                                                     C.addressof(base), C.addressof(nw)))
    return out[:used.value], base.value, nw.value


def _window_predictors(predictors, n_units, n_windows):
    """(order, q[100]) pairs: the units' as encode_search_forced takes them, then the (unit, window) records'."""
    pred = np.zeros(len(predictors), PREDICTOR_DTYPE)
    for rec, (order, q) in zip(pred, predictors):
        rec["order"] = order
        rec["q"][:] = np.asarray(q)[:MAX_ORDER]
    if pred.size != n_units * (1 + n_windows):
        raise ValueError("%d predictors for %d units and %d windows" % (pred.size, n_units, n_windows))
    return pred


def encode_search_windows_forced(pcm, channels, windows, predictors, device=0):
    """encode_frames_search_windows on one batch with every unit's q[0..99] and reference order, then every
    (unit, window) record's q[0..99] (windows in increasing bit order; its order is not read), from `predictors`
    ((order, q[100]) pairs) -> (descs, words, base_words, n_window)."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    n_units = n_frames * (3 if channels == 2 else channels)
    pred = _window_predictors(predictors, n_units, bin(windows & 31).count("1"))
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    used, base, nw = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_search_windows_forced(pcm.ctypes.data, n_frames, channels, windows, pred.ctypes.data,
                                                  descs.ctypes.data, words.ctypes.data, cap, C.addressof(used),
                                                  C.addressof(base), C.addressof(nw)))
    return descs, words[:used.value].copy(), base.value, nw.value


def encode_search_windows_trace(pcm, channels, tables, predictors=None, device=0):
    """The window search on one batch with the windows `tables` (float64 [n, 2048], 1 <= n <= 5) in place of the
    table's (encode_search_windows_forced's q with `predictors`), through the tracing candidate kernel -> (descs,
    words, base_words, n_window, trace, keys): trace SEARCH_TRACE_DTYPE [n_units, n, 100], entry [u, w, order - 1]
    unit u (encode_trace's order) coded from window w at that order; keys uint64 [n_units], unit u's best window
    candidate as words << 16 | w << 8 | order."""
    init(device)
    pcm, n_frames = _whole_frames(pcm, channels)
    tables = np.ascontiguousarray(np.atleast_2d(tables), np.float64)
    n_windows = tables.shape[0]
    if tables.shape[1] != FRAME:
        raise ValueError("a window has 2048 values")
    n_units = n_frames * (3 if channels == 2 else channels)
    pred = None if predictors is None else _window_predictors(predictors, n_units, n_windows)
    L = lib()
    cap = L.selab200_encode_words_bound(n_frames, channels)
    descs = np.zeros(n_frames * channels, DESC_DTYPE)
    words = np.empty(max(cap, 1), np.uint32)
    trace = np.zeros((n_units, n_windows, MAX_ORDER), SEARCH_TRACE_DTYPE)
    keys = np.zeros(n_units, np.uint64)
    used, base, nw = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    check(L.selab200_encode_search_windows_trace(pcm.ctypes.data, n_frames, channels, tables.ctypes.data, n_windows,
                                                 None if pred is None else pred.ctypes.data, descs.ctypes.data,
                                                 words.ctypes.data, cap, C.addressof(used), C.addressof(base),
                                                 C.addressof(nw), trace.ctypes.data, keys.ctypes.data))
    return descs, words[:used.value].copy(), base.value, nw.value, trace, keys
