"""Device-resident entry points for callers that already hold the data in HBM.

PyTorch is used only for what it is good at here: device memory (tensors), streams
and events.  The work itself is the C ABI's *_device calls, enqueued on the
current torch stream without synchronising.
"""
import ctypes as C

import torch

from ._lib import FRAME, check, init, lib


class DeviceCodec:
    """Pre-allocated descriptor table, word arena and workspaces for a fixed batch shape."""

    def __init__(self, n_frames, channels, device=None, words_capacity=None):
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        init(self.device.index)
        L = lib()
        self.n_frames, self.channels = n_frames, channels
        self.n_sub = n_frames * channels
        self.capacity = words_capacity or L.selab200_encode_words_bound(n_frames, channels)
        dev = self.device
        self.descs = torch.zeros(self.n_sub * 32, dtype=torch.uint8, device=dev)
        self.words = torch.zeros(self.capacity, dtype=torch.int32, device=dev)
        self.words_used = torch.zeros(1, dtype=torch.int64, device=dev)
        self.status = torch.zeros(2, dtype=torch.int32, device=dev)
        self.enc_ws_bytes = L.selab200_encode_workspace_bytes(n_frames, channels)
        self.dec_ws_bytes = L.selab200_decode_workspace_bytes(n_frames, channels)
        self.enc_ws = torch.zeros(self.enc_ws_bytes, dtype=torch.uint8, device=dev)
        self.dec_ws = torch.zeros(self.dec_ws_bytes, dtype=torch.uint8, device=dev)

    def encode(self, pcm):
        """pcm: int16 cuda tensor, n_frames*2048*channels interleaved. Asynchronous."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.numel() == self.n_sub * FRAME
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(lib().selab200_encode_frames_device(
            pcm.data_ptr(), self.n_frames, self.channels, self.descs.data_ptr(), self.words.data_ptr(),
            self.capacity, self.words_used.data_ptr(), self.status.data_ptr(), self.enc_ws.data_ptr(),
            self.enc_ws_bytes, C.c_void_p(stream)))

    def encode_lossless(self, pcm):
        """encode, lossless (DESIGN.md 7.2): also fills the per-pair records of re-coded subframes on the device.
        Asynchronous, and the host never waits for what the check finds; lossless_report() collects the report.
        The lossless buffers are allocated on first use."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.numel() == self.n_sub * FRAME
        L = lib()
        if not hasattr(self, "ll_ws"):
            self.ll_ws_bytes = L.selab200_encode_lossless_workspace_bytes(self.n_frames, self.channels)
            self.ll_ws = torch.zeros(self.ll_ws_bytes, dtype=torch.uint8, device=self.device)
            self.ll_entries = torch.zeros(max(self.n_sub, 1) * 16, dtype=torch.uint8, device=self.device)
            self.ll_count = torch.zeros(1, dtype=torch.int64, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(L.selab200_encode_frames_lossless_device(
            pcm.data_ptr(), self.n_frames, self.channels, self.descs.data_ptr(), self.words.data_ptr(),
            self.capacity, self.words_used.data_ptr(), self.ll_entries.data_ptr(), self.ll_count.data_ptr(),
            self.status.data_ptr(), self.ll_ws.data_ptr(), self.ll_ws_bytes, C.c_void_p(stream)))

    def lossless_report(self):
        """Synchronises: the report of the last encode_lossless, a LOSSLESS_DTYPE array of the re-coded
        (frame, channel) pairs in order."""
        import numpy as np
        from ._lib import LOSSLESS_DTYPE
        if int(self.ll_count.item()) == 0:
            return np.zeros(0, LOSSLESS_DTYPE)
        rec = self.ll_entries.cpu().numpy().view(LOSSLESS_DTYPE)[:self.n_sub]
        return rec[rec["words"] != 0].copy()

    def encode_search(self, pcm):
        """encode with the order search (DESIGN.md 7.3).  Asynchronous; self.ref_words (int64 cuda tensor) receives
        the words encode() writes for the same frames.  The search workspace is allocated on first use."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.numel() == self.n_sub * FRAME
        L = lib()
        if not hasattr(self, "search_ws"):
            self.search_ws_bytes = L.selab200_encode_search_workspace_bytes(self.n_frames, self.channels)
            self.search_ws = torch.zeros(self.search_ws_bytes, dtype=torch.uint8, device=self.device)
            self.ref_words = torch.zeros(1, dtype=torch.int64, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(L.selab200_encode_frames_search_device(
            pcm.data_ptr(), self.n_frames, self.channels, self.descs.data_ptr(), self.words.data_ptr(),
            self.capacity, self.words_used.data_ptr(), self.ref_words.data_ptr(), self.status.data_ptr(),
            self.search_ws.data_ptr(), self.search_ws_bytes, C.c_void_p(stream)))

    def encode_search_guided(self, pcm, candidates=4):
        """encode with the guided order search (DESIGN.md 7.7) over `candidates` (1..100) ranked orders.
        Asynchronous; self.ref_words (int64 cuda tensor) receives the words encode() writes for the same frames.  The
        workspace is allocated on first use."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.numel() == self.n_sub * FRAME
        L = lib()
        if not hasattr(self, "guided_ws"):
            self.guided_ws_bytes = L.selab200_encode_search_guided_workspace_bytes(self.n_frames, self.channels)
            self.guided_ws = torch.zeros(self.guided_ws_bytes, dtype=torch.uint8, device=self.device)
        if not hasattr(self, "ref_words"):
            self.ref_words = torch.zeros(1, dtype=torch.int64, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(L.selab200_encode_frames_search_guided_device(
            pcm.data_ptr(), self.n_frames, self.channels, candidates, self.descs.data_ptr(), self.words.data_ptr(),
            self.capacity, self.words_used.data_ptr(), self.ref_words.data_ptr(), self.status.data_ptr(),
            self.guided_ws.data_ptr(), self.guided_ws_bytes, C.c_void_p(stream)))

    def encode_pairing(self, pcm):
        """encode with the channel pairing (DESIGN.md 7.4).  Asynchronous; self.base_words and self.n_difference
        (int64 cuda tensors) receive the words encode_lossless() writes for the same frames and the number of
        difference subframes.  The pairing workspace is allocated on first use."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.numel() == self.n_sub * FRAME
        L = lib()
        if not hasattr(self, "pairing_ws"):
            self.pairing_ws_bytes = L.selab200_encode_pairing_workspace_bytes(self.n_frames, self.channels)
            self.pairing_ws = torch.zeros(self.pairing_ws_bytes, dtype=torch.uint8, device=self.device)
            self.base_words = torch.zeros(1, dtype=torch.int64, device=self.device)
            self.n_difference = torch.zeros(1, dtype=torch.int64, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(L.selab200_encode_frames_pairing_device(
            pcm.data_ptr(), self.n_frames, self.channels, self.descs.data_ptr(), self.words.data_ptr(),
            self.capacity, self.words_used.data_ptr(), self.base_words.data_ptr(), self.n_difference.data_ptr(),
            self.status.data_ptr(), self.pairing_ws.data_ptr(), self.pairing_ws_bytes, C.c_void_p(stream)))

    def encode_search_pairing(self, pcm):
        """encode with the order search and the channel pairing together (DESIGN.md 7.5).  Asynchronous;
        self.base_words and self.n_difference (int64 cuda tensors) receive the words encode_search() writes for the
        same frames and the number of difference subframes.  The workspace is allocated on first use."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.numel() == self.n_sub * FRAME
        L = lib()
        if not hasattr(self, "search_pairing_ws"):
            self.search_pairing_ws_bytes = L.selab200_encode_search_pairing_workspace_bytes(self.n_frames,
                                                                                            self.channels)
            self.search_pairing_ws = torch.zeros(self.search_pairing_ws_bytes, dtype=torch.uint8, device=self.device)
        if not hasattr(self, "base_words"):
            self.base_words = torch.zeros(1, dtype=torch.int64, device=self.device)
            self.n_difference = torch.zeros(1, dtype=torch.int64, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(L.selab200_encode_frames_search_pairing_device(
            pcm.data_ptr(), self.n_frames, self.channels, self.descs.data_ptr(), self.words.data_ptr(),
            self.capacity, self.words_used.data_ptr(), self.base_words.data_ptr(), self.n_difference.data_ptr(),
            self.status.data_ptr(), self.search_pairing_ws.data_ptr(), self.search_pairing_ws_bytes,
            C.c_void_p(stream)))

    def encode_search_windows(self, pcm, windows=1):
        """encode with the window search (DESIGN.md 7.6) over the window mask `windows`.  Asynchronous;
        self.base_words and self.n_window (int64 cuda tensors) receive the words encode_search() writes for the same
        frames and the number of analysis units coded from a window.  The workspace of the largest mask used so far
        is allocated on first use."""
        assert pcm.dtype == torch.int16 and pcm.is_cuda and pcm.numel() == self.n_sub * FRAME
        L = lib()
        need = L.selab200_encode_search_windows_workspace_bytes(self.n_frames, self.channels, windows)
        if getattr(self, "windows_ws_bytes", 0) < need:
            self.windows_ws_bytes = need
            self.windows_ws = torch.zeros(need, dtype=torch.uint8, device=self.device)
        if not hasattr(self, "base_words"):
            self.base_words = torch.zeros(1, dtype=torch.int64, device=self.device)
        if not hasattr(self, "n_window"):
            self.n_window = torch.zeros(1, dtype=torch.int64, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(L.selab200_encode_frames_search_windows_device(
            pcm.data_ptr(), self.n_frames, self.channels, windows, self.descs.data_ptr(), self.words.data_ptr(),
            self.capacity, self.words_used.data_ptr(), self.base_words.data_ptr(), self.n_window.data_ptr(),
            self.status.data_ptr(), self.windows_ws.data_ptr(), self.windows_ws_bytes, C.c_void_p(stream)))

    def decode(self, pcm_out, n_words):
        """Decode self.descs / self.words[:n_words] into pcm_out (int16 cuda tensor). Asynchronous."""
        assert pcm_out.dtype == torch.int16 and pcm_out.is_cuda and pcm_out.numel() == self.n_sub * FRAME
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(lib().selab200_decode_frames_device(
            self.descs.data_ptr(), self.n_frames, self.channels, self.words.data_ptr(), int(n_words),
            pcm_out.data_ptr(), self.status.data_ptr() + 4, self.dec_ws.data_ptr(), self.dec_ws_bytes,
            C.c_void_p(stream)))

    def verify(self, pcm_ref, n_words):
        """Decode self.descs / self.words[:n_words] and compare with pcm_ref (int16 cuda tensor, 16-byte aligned):
        per-pair records and the count of differing pairs stay on the device.  Asynchronous; verify_report()
        collects the result.  The verify buffers are allocated on first use."""
        assert pcm_ref.dtype == torch.int16 and pcm_ref.is_cuda and pcm_ref.numel() == self.n_sub * FRAME
        L = lib()
        if not hasattr(self, "ver_ws"):
            self.ver_ws_bytes = L.selab200_verify_workspace_bytes(self.n_frames, self.channels)
            self.ver_ws = torch.zeros(self.ver_ws_bytes, dtype=torch.uint8, device=self.device)
            self.ver_entries = torch.zeros(max(self.n_sub, 1) * 16, dtype=torch.uint8, device=self.device)
            self.ver_count = torch.zeros(1, dtype=torch.int64, device=self.device)
            self.ver_status = torch.zeros(1, dtype=torch.int32, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        check(L.selab200_verify_frames_device(
            self.descs.data_ptr(), self.n_frames, self.channels, self.words.data_ptr(), int(n_words),
            pcm_ref.data_ptr(), self.ver_entries.data_ptr(), self.ver_count.data_ptr(), self.ver_status.data_ptr(),
            self.ver_ws.data_ptr(), self.ver_ws_bytes, C.c_void_p(stream)))

    def verify_report(self):
        """Synchronises; raises if the last verify's decode reported an error, else returns its report: a
        VERIFY_DTYPE array of the differing (frame, channel) pairs in order (per-pair records copied only
        when there are any)."""
        import numpy as np
        from ._lib import SelaB200Error, STATUS_NAMES, VERIFY_DTYPE
        st = int(self.ver_status.item())
        if st != 0:
            raise SelaB200Error(st, "verify reported %s" % STATUS_NAMES.get(st, st))
        if int(self.ver_count.item()) == 0:
            return np.zeros(0, VERIFY_DTYPE)
        rec = self.ver_entries.cpu().numpy().view(VERIFY_DTYPE)[:self.n_sub]
        return rec[rec["n_differing"] != 0].copy()

    def check_status(self):
        """Synchronises; raises if either the last encode or decode reported an error."""
        from ._lib import SelaB200Error, STATUS_NAMES
        st = self.status.cpu().tolist()
        for what, s in zip(("encode", "decode"), st):
            if s != 0:
                raise SelaB200Error(s, "%s kernel reported %s" % (what, STATUS_NAMES.get(s, s)))


def rice_decode_frames(descs, words, channels, device=0):
    """Residue streams of every subframe -> int32 [n_sub, 2048] (the Rice-decode kernel on its own,
    selab200_rice_decode_frames_device).  descs: numpy array of DESC_DTYPE, words: uint32 arena.
    Returns (residues, n_flagged)."""
    import numpy as np
    from ._lib import DESC_DTYPE
    init(device)
    dev = torch.device("cuda", device)
    L = lib()
    n_sub = descs.size
    assert n_sub % channels == 0
    d_descs = torch.from_numpy(np.ascontiguousarray(descs).view(np.uint8).reshape(-1).copy()).to(dev)
    w = np.ascontiguousarray(words, dtype=np.uint32)
    d_words = torch.zeros(w.size + 8, dtype=torch.int32, device=dev)
    d_words[:w.size] = torch.from_numpy(w.view(np.int32)).to(dev)
    out = torch.empty(n_sub * FRAME, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    check(L.selab200_rice_decode_frames_device(d_descs.data_ptr(), n_sub // channels, channels, d_words.data_ptr(),
                                               w.size, out.data_ptr(), status.data_ptr(), C.c_void_p(stream)))
    torch.cuda.synchronize(dev)
    st = int(status.item())
    if st != 0:
        from ._lib import SelaB200Error, STATUS_NAMES
        raise SelaB200Error(st, "rice decode kernel reported %s" % STATUS_NAMES.get(st, st))
    flagged = C.c_uint32(0)
    check(L.selab200_rice_decode_flagged(C.addressof(flagged)))
    return out.cpu().numpy().reshape(n_sub, FRAME), flagged.value
