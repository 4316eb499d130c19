"""Batch-path encodes of constant frames against the compiled reference.

On a constant frame x - mean is pure rounding noise, so the order in which the mean's sum is taken decides q[0].
The batch encoder computes every analysis unit's mean in its own kernel (k_unit_means, one lane per unit); these
tests drive that kernel through every way it reads its input: mono, stereo (ch0, ch1 and the difference), an
N-channel layout, and PCM that does not start on a 16-byte boundary.
Run on the H100:  python -m pytest tests -m gpu -q
"""
import numpy as np
import pytest

import oracle_lib as ol
import sela_b200

pytestmark = pytest.mark.gpu

FRAME = 2048
# the levels of test_gpu_parity.py::test_lpc_residues_dc_levels
LEVELS = np.array(list(range(-32768, 32768, 131)) + [-1, 1, 32767], np.int64)


@pytest.fixture(scope="module")
def O():
    return ol.best()


def _constant_frames(levels):
    """levels: [n_frames, channels] -> interleaved int16 PCM, every frame and channel constant."""
    lv = np.asarray(levels, np.int64)
    return np.repeat(lv[:, None, :], FRAME, axis=1).astype(np.int16).reshape(-1, lv.shape[1])


def _check(O, pcm, channels):
    d_ref, w_ref = O.encode_frames(pcm, channels)
    d, w = sela_b200.encode_frames(pcm, channels)
    assert d.tobytes() == d_ref.tobytes()
    assert np.array_equal(w, w_ref)
    return d


def test_dc_mono(O):
    _check(O, _constant_frames(LEVELS[:, None]), 1)


def test_dc_stereo_two_levels(O):
    # ch1 at another level than ch0: the ch1 unit and the difference unit (ch0 - ch1, 17 bits) are constant too
    other = LEVELS[(np.arange(LEVELS.size) * 37 + 11) % LEVELS.size]
    pcm = _constant_frames(np.stack([LEVELS, other], axis=1))
    d = _check(O, pcm, 2)
    assert (d["subframe_type"] == 1).any()  # some frames emit the difference unit


def test_dc_eight_channels(O):
    n = (LEVELS.size + 7) // 8
    lv = np.resize(np.roll(LEVELS, 5), n * 8).reshape(n, 8)
    _check(O, _constant_frames(lv), 8)


@pytest.mark.parametrize("channels", [1, 3])
def test_dc_unaligned_device_pcm(O, channels):
    """PCM that starts 2 bytes past a 16-byte boundary (device-resident call, any channel count but 2)."""
    import torch
    from sela_b200.device import DeviceCodec

    n = LEVELS.size // channels
    pcm = _constant_frames(LEVELS[:n * channels].reshape(n, channels))
    d_ref, w_ref = O.encode_frames(pcm, channels)
    flat = torch.from_numpy(pcm.reshape(-1).copy())
    buf = torch.zeros(flat.numel() + 8, dtype=torch.int16, device="cuda")
    dev_pcm = buf[1:1 + flat.numel()]
    dev_pcm.copy_(flat.cuda())
    assert dev_pcm.data_ptr() % 16 == 2
    codec = DeviceCodec(n, channels)
    codec.encode(dev_pcm)
    codec.check_status()
    used = int(codec.words_used.item())
    descs = codec.descs.cpu().numpy().view(d_ref.dtype)
    assert descs.tobytes() == d_ref.tobytes()
    assert used == w_ref.size
    assert np.array_equal(codec.words[:used].cpu().numpy().view(np.uint32), w_ref)
