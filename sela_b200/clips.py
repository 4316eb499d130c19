"""Random access into .sela files: sample-accurate clips from open containers (DESIGN.md 7.8).

    with ClipDecoder([blob_a, blob_b]) as dec:
        x = dec.decode(0, [44100 * 30], 44100)            # np.int16 [1, 44100, channels]
        y = dec.decode_device([0, 1], [0, 4096], 2048)    # torch.int16 cuda [2, 2048, channels]

Opening a container uploads its whole byte image to the device and walks its frame headers once; the decoder keeps
the handles (and the byte buffers they read) open until close(), so each call decodes only the frames its clips
cover, each of them once.
"""
import ctypes as C

import numpy as np

from ._lib import CLIP_DTYPE, INFO_DTYPE, check, init, lib


class ClipDecoder:
    """Open containers (bytes, bytearray or uint8 arrays of whole .sela files) for clip decoding on `device` (an int,
    or a list of devices whose first, the primary, holds the images and runs the decode).  All containers must have
    the same channel count."""

    def __init__(self, containers, device=0):
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
                check(L.selab200_container_open(buf.ctypes.data, buf.size, C.addressof(handle), info.ctypes.data))
                self._bufs.append(buf)  # the handle reads these bytes until it is closed
                self._handles.append(handle.value)
                self.info.append({k: int(info[0][k]) for k in INFO_DTYPE.names if k != "reserved"})
        except Exception:
            self.close()
            raise
        self._array = (C.c_void_p * max(len(self._handles), 1))(*self._handles)
        self.channels = self.info[0]["channels"] if self.info else 0
        self.frames_decoded = 0

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

    def decode(self, container_index, starts, length):
        """Clip i = samples [starts[i], starts[i] + length) of container container_index (an int, or one per clip)
        -> np.int16 [n, length, channels], equal to the same rows of decode_container's output."""
        clips, length = self._clips(container_index, starts, length)
        out = np.empty((clips.size, length, self.channels), np.int16)
        n = C.c_uint64(0)
        check(lib().selab200_container_decode_clips(C.addressof(self._array), len(self._handles), clips.ctypes.data,
                                                    clips.size, length, out.ctypes.data, C.addressof(n)))
        self.frames_decoded = n.value
        return out

    def decode_device(self, container_index, starts, length):
        """decode() into a torch.int16 tensor [n, length, channels] on the primary device; returns once it is
        written."""
        import torch
        clips, length = self._clips(container_index, starts, length)
        dev = torch.device("cuda", self.device)
        out = torch.empty((clips.size, length, self.channels), dtype=torch.int16, device=dev)
        torch.cuda.current_stream(dev).synchronize()  # the library writes on its own streams
        n = C.c_uint64(0)
        check(lib().selab200_container_decode_clips_device(C.addressof(self._array), len(self._handles),
                                                           clips.ctypes.data, clips.size, length,
                                                           C.c_void_p(out.data_ptr()), C.addressof(n)))
        self.frames_decoded = n.value
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
