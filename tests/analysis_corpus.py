"""The signals the encoder's analysis is checked on, as PCM batches that run every kind of analysis unit.

batches() returns (name, pcm, channels): interleaved int16 PCM of whole 2048-sample frames.  units() turns a
batch into the signals of its analysis units in the batch encoder's order: frame after frame, within a frame
channel 0..C-1, or for stereo ch0, ch1 and the difference ch0 - ch1 (as int32: 17 bits).  The CPU tests
(test_exact_analysis.py) analyse exactly these units, and the GPU tests (test_analysis_trace.py) trace them.

The frames: every test-signal family, three seeded sets of random frames, full-scale pairs whose difference
needs 17 bits, multichannel sine_noise, every 3rd frame of 60 s of the BASELINE synthetic, the 504 DC levels,
digital silence (the NaN path: lag 0 is 0) and +-1-LSB noise.
"""
import functools

import numpy as np

import signals
from sela_b200 import synth

FRAME = 2048
DC_LEVELS = np.array(list(range(-32768, 32768, 131)) + [-1, 1, 32767], np.int64)


def _interleave(planes):
    """planes: [n_frames, channels, 2048] -> interleaved int16 [n_frames * 2048, channels]."""
    planes = np.asarray(planes, np.int64)
    assert planes.min() >= -32768 and planes.max() <= 32767
    return planes.transpose(0, 2, 1).reshape(-1, planes.shape[1]).astype(np.int16)


@functools.lru_cache(maxsize=1)
def batches():
    rng = np.random.default_rng(2024)
    fam = np.stack([v.astype(np.int64) for v in signals.families().values()])
    silence = np.zeros((1, FRAME), np.int64)
    lsb = rng.integers(-1, 2, (2, FRAME))
    dc = np.repeat(DC_LEVELS[:, None], FRAME, axis=1)
    mono = np.concatenate([fam, signals.random_frames(192, 21), dc, silence, lsb])

    # stereo: every random frame paired with another; families paired with a rotation of themselves; ch1 the
    # negated ch0 plus a little noise, or independent full scale (differences up to 65535); equal channels
    # (a silent difference) and +-1-LSB noise in both channels
    r11 = signals.random_frames(300, 11).astype(np.int64)
    a = rng.integers(-32768, 32768, (8, FRAME))
    anti = np.clip(-a + rng.integers(-40, 41, a.shape), -32768, 32767)
    pairs = np.concatenate([
        np.stack([r11[0::2], r11[1::2]], axis=1),
        np.stack([fam, np.roll(fam, 3, axis=0)], axis=1),
        np.stack([a, anti], axis=1),
        np.stack([rng.integers(-32768, 32768, (8, FRAME)), rng.integers(-32768, 32768, (8, FRAME))], axis=1),
        np.stack([fam[:1], fam[:1]], axis=1),
        rng.integers(-1, 2, (2, 2, FRAME)),
    ])

    r5 = signals.random_frames(64, 5).astype(np.int64)[:63]
    three = r5.reshape(21, 3, FRAME)

    baseline = synth.sine_noise(44100, 2, seconds=60, seed=1)
    n = baseline.shape[0] // FRAME
    baseline = baseline[:n * FRAME].reshape(n, FRAME, 2)[::3].reshape(-1, 2)

    return (
        ("mono", _interleave(mono[:, None, :]), 1),
        ("stereo_pairs", _interleave(pairs), 2),
        ("three_channels", _interleave(three), 3),
        ("stereo_sine_noise", synth.sine_noise(44100, 2, n_frames=24, seed=3).astype(np.int16), 2),
        ("eight_channels", synth.sine_noise(48000, 8, n_frames=24, seed=2).astype(np.int16), 8),
        ("stereo_baseline_every_3rd", np.ascontiguousarray(baseline, np.int16), 2),
    )


def units(pcm, channels):
    """The analysis units' signals of a batch, int64 [n_units, 2048], in the batch encoder's order."""
    planes = np.asarray(pcm, np.int64).reshape(-1, FRAME, channels).transpose(0, 2, 1)
    if channels == 2:
        planes = np.concatenate([planes, planes[:, :1] - planes[:, 1:]], axis=1)
    return planes.reshape(-1, FRAME)


@functools.lru_cache(maxsize=1)
def all_units():
    """Every batch's units, concatenated -> int64 [n, 2048]."""
    return np.concatenate([units(pcm, ch) for _, pcm, ch in batches()])
