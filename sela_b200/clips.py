"""Random access into .sela files: sample-accurate clips from open containers (DESIGN.md 7.8).

    with ClipDecoder([blob_a, blob_b]) as dec:
        x = dec.decode(0, [44100 * 30], 44100)            # np.int16 [1, 44100, channels]
        y = dec.decode_device([0, 1], [0, 4096], 2048)    # torch.int16 cuda [2, 2048, channels]
        z = dec.decode(0, [0], 2048, channels=[0], dtype=np.float32)   # np.float32 [1, 2048, 1], channel 0 / 32768
        m = dec.decode_device([0, 1], [0, 0], 2048, dtype=torch.float32, mean=True)   # the mono mix [2, 2048, 1]

Opening a container uploads its whole byte image to the device and walks its frame headers once; the decoder keeps
the handles (and the byte buffers they read) open until close(), so each call decodes only the frames its clips
cover, each of them once.  With `channels`, `dtype` or `mean` only the subframes the chosen channels need are
decoded (DESIGN.md 7.9), and containers of different channel counts may share a call.

With host_resident=True the images stay in page-locked host memory instead, for a corpus larger than the device
memory it may take, and each call fetches over PCIe only the bytes of the subframes it decodes (DESIGN.md 7.10):

    with ClipDecoder(blobs, host_resident=True) as dec:
        x = dec.decode_device(ks, starts, 44100, channels=[0])
        dec.bytes_fetched                                  # the bytes that call read from host memory
"""
import ctypes as C

import numpy as np

from ._lib import CLIP_DTYPE, CLIP_FLOAT32, CLIP_MAX_SELECT, CLIP_MEAN, INFO_DTYPE, check, init, lib


class ClipDecoder:
    """Open containers (bytes, bytearray or uint8 arrays of whole .sela files) for clip decoding on `device` (an int,
    or a list of devices whose first, the primary, holds the images and runs the decode).  Containers may differ in
    channel count; a call that returns every channel as int16 still needs one count.

    host_resident: open every container with selab200_container_open_host: the handle keeps its own page-locked copy
    of the image, no device memory holds it, and the decoder keeps no reference to the caller's bytes."""

    def __init__(self, containers, device=0, host_resident=False):
        init(device)
        self.device = device[0] if isinstance(device, (list, tuple)) else device
        self._bufs, self._handles, self.info = [], [], []
        L = lib()
        try:
            for c in containers:
                buf = np.ascontiguousarray(np.frombuffer(c, np.uint8) if isinstance(c, (bytes, bytearray)) else c,
                                           np.uint8)
                info = np.zeros(1, INFO_DTYPE)
                handle = C.c_void_p(0)
                opener = L.selab200_container_open_host if host_resident else L.selab200_container_open
                check(opener(buf.ctypes.data, buf.size, C.addressof(handle), info.ctypes.data))
                if not host_resident:
                    self._bufs.append(buf)  # the handle reads these bytes until it is closed
                self._handles.append(handle.value)
                self.info.append({k: int(info[0][k]) for k in INFO_DTYPE.names if k != "reserved"})
        except Exception:
            self.close()
            raise
        self._array = (C.c_void_p * max(len(self._handles), 1))(*self._handles)
        self.channels = self.info[0]["channels"] if self.info else 0
        self.host_resident = bool(host_resident)
        self.frames_decoded = self.subframes_decoded = self.bytes_fetched = 0

    def _clips(self, container_index, starts, length):
        if not self._handles:
            raise ValueError("the decoder is closed or holds no containers")
        starts = np.atleast_1d(np.asarray(starts, dtype=np.uint64)).reshape(-1)
        clips = np.zeros(starts.size, CLIP_DTYPE)
        clips["container"] = np.broadcast_to(np.asarray(container_index, dtype=np.uint32), starts.shape)
        clips["start"] = starts
        if not 0 <= int(length) < 1 << 32:
            raise ValueError("length must fit 32 bits")
        return clips, int(length)

    def _select(self, channels, dtype, mean):
        """(select array or None, flags), or None for the plain int16 call over every channel."""
        if dtype not in (np.int16, np.float32):
            raise ValueError("dtype must be int16 or float32")
        if mean and dtype != np.float32:
            raise ValueError("mean needs dtype float32")
        if channels is None:
            return None if dtype == np.int16 else (None, CLIP_FLOAT32 | (CLIP_MEAN if mean else 0))
        sel = [int(c) for c in np.atleast_1d(np.asarray(channels)).reshape(-1)]
        if not 1 <= len(sel) <= CLIP_MAX_SELECT or not all(0 <= c < 256 for c in sel):
            raise ValueError("channels must be 1..%d channel numbers in 0..255" % CLIP_MAX_SELECT)
        return (np.array(sel, np.uint8),
                (CLIP_FLOAT32 if dtype == np.float32 else 0) | (CLIP_MEAN if mean else 0))

    def _n_out(self, clips, select, flags):
        if flags & CLIP_MEAN:
            return 1
        if select is not None:
            return select.size
        return self.info[int(clips["container"][0])]["channels"] if clips.size else self.channels

    def _call(self, device, clips, length, select, flags, out_ptr):
        n, m = C.c_uint64(0), C.c_uint64(0)
        fn = (lib().selab200_container_decode_clips_select_device if device
              else lib().selab200_container_decode_clips_select)
        check(fn(C.addressof(self._array), len(self._handles), clips.ctypes.data, clips.size, length,
                 select.ctypes.data if select is not None else None, 0 if select is None else select.size, flags,
                 out_ptr, C.addressof(n), C.addressof(m)))
        self.frames_decoded, self.subframes_decoded = n.value, m.value
        self._fetched()

    def _fetched(self):
        b = C.c_uint64(0)
        check(lib().selab200_clip_bytes_fetched(C.addressof(b)))
        self.bytes_fetched = b.value

    def decode(self, container_index, starts, length, channels=None, dtype=np.int16, mean=False):
        """Clip i = samples [starts[i], starts[i] + length) of container container_index (an int, or one per clip)
        -> np.int16 [n, length, channels], equal to the same rows of decode_container's output.

        channels: a list of channel numbers (any order, repeats allowed) to return, in that order; dtype np.float32
        returns sample / 32768; mean (float32) returns one channel, the mean of the chosen ones (of every channel of
        each clip's own container without `channels`).  Only the subframes these channels need are decoded."""
        dtype = np.dtype(dtype).type
        choice = self._select(channels, dtype, mean)
        clips, length = self._clips(container_index, starts, length)
        if choice is None:
            out = np.empty((clips.size, length, self.channels), np.int16)
            n = C.c_uint64(0)
            check(lib().selab200_container_decode_clips(C.addressof(self._array), len(self._handles),
                                                        clips.ctypes.data, clips.size, length, out.ctypes.data,
                                                        C.addressof(n)))
            self.frames_decoded = n.value
            self.subframes_decoded = n.value * self.channels
            self._fetched()
            return out
        select, flags = choice
        out = np.empty((clips.size, length, self._n_out(clips, select, flags)), dtype)
        self._call(False, clips, length, select, flags, out.ctypes.data)
        return out

    def decode_device(self, container_index, starts, length, channels=None, dtype=None, mean=False):
        """decode() into a torch tensor on the primary device, dtype torch.int16 (default) or torch.float32; returns
        once it is written."""
        import torch
        dtype = torch.int16 if dtype is None else dtype
        if dtype not in (torch.int16, torch.float32):
            raise ValueError("dtype must be torch.int16 or torch.float32")
        choice = self._select(channels, np.float32 if dtype == torch.float32 else np.int16, mean)
        clips, length = self._clips(container_index, starts, length)
        dev = torch.device("cuda", self.device)
        n_out = self.channels if choice is None else self._n_out(clips, *choice)
        out = torch.empty((clips.size, length, n_out), dtype=dtype, device=dev)
        torch.cuda.current_stream(dev).synchronize()  # the library writes on its own streams
        if choice is None:
            n = C.c_uint64(0)
            check(lib().selab200_container_decode_clips_device(C.addressof(self._array), len(self._handles),
                                                               clips.ctypes.data, clips.size, length,
                                                               C.c_void_p(out.data_ptr()), C.addressof(n)))
            self.frames_decoded = n.value
            self.subframes_decoded = n.value * self.channels
            self._fetched()
            return out
        self._call(True, clips, length, *choice, C.c_void_p(out.data_ptr()))
        return out

    def close(self):
        L = lib()
        for h in self._handles:
            L.selab200_container_close(C.c_void_p(h))
        self._handles, self._bufs = [], []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
