"""CPU-only: the encode workspace sizes of every mode.  Callers of the *_device encodes size their buffers with these
functions, so their values are part of the interface: they are pinned here over a grid of shapes."""
import pytest

from sela_b200 import _lib

MODES = ("selab200_encode_workspace_bytes", "selab200_encode_lossless_workspace_bytes",
         "selab200_encode_search_workspace_bytes", "selab200_encode_pairing_workspace_bytes")

# (n_frames, channels) -> bytes of [plain, lossless, search, pairing]
SIZES = {
    (0, 1): (256, 512, 256, 512),
    (0, 8): (256, 512, 256, 512),
    (1, 1): (15360, 16384, 15776, 17408),
    (2, 1): (29952, 30976, 30784, 32000),
    (1, 2): (44544, 45568, 45792, 46592),
    (33, 2): (1449216, 1454848, 1490400, 1458944),
    (7, 3): (307712, 309504, 316448, 311552),
    (100, 5): (7316480, 7341568, 7524480, 7403008),
    (3, 16): (702720, 705536, 722688, 724480),
    (512, 2): (22475008, 22551040, 23113984, 22603264),
    (4096, 8): (479461632, 481051136, 493093120, 487391744),
    (12919, 2): (567092992, 569005568, 583215904, 570323456),
    (14062, 8): (1646041856, 1651498240, 1692840192, 1673266432),
}


@pytest.mark.parametrize("shape", sorted(SIZES))
def test_encode_workspace_bytes(shape):
    L = _lib.lib()
    assert tuple(getattr(L, name)(*shape) for name in MODES) == SIZES[shape]


def test_every_mode_holds_the_plain_encode():
    L = _lib.lib()
    for shape in SIZES:
        plain, lossless, search, pairing = (getattr(L, name)(*shape) for name in MODES)
        assert plain % 256 == 0 and lossless % 256 == 0 and pairing % 256 == 0
        assert plain <= search and plain < lossless <= pairing
