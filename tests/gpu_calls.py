"""Device calls the GPU tests share (TEST INFRASTRUCTURE)."""
import numpy as np
import torch

from sela_b200.device import DeviceCodec

FRAME = 2048


def decode_frames_device(descs, words, channels, fill=None):
    """selab200_decode_frames_device on (descs, words) -> int16 PCM; raises what the device status says.  fill: an
    int16 the output is set to first (by default it is left as allocated, which may hold an earlier result)."""
    n_frames = descs.size // channels
    codec = DeviceCodec(n_frames, channels, words_capacity=max(words.size, 1) + 8)
    codec.descs.copy_(torch.from_numpy(np.ascontiguousarray(descs).view(np.uint8).reshape(-1).copy()))
    codec.words[:words.size].copy_(torch.from_numpy(np.ascontiguousarray(words, np.uint32).view(np.int32)))
    if fill is None:
        out = torch.empty(descs.size * FRAME, dtype=torch.int16, device=codec.device)
    else:
        out = torch.full((descs.size * FRAME,), fill, dtype=torch.int16, device=codec.device)
    codec.decode(out, words.size)
    codec.check_status()
    return out.cpu().numpy()
