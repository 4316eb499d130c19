"""ctypes loader for the in-tree CUDA extension (sela_b200/libsela_b200.so).

There is no CPU fallback: if the shared library is missing this raises, and if
no CUDA device is present every compute call returns SELAB200_ERR_NO_DEVICE
(surfaced as SelaB200Error).
"""
import ctypes as C
import pathlib

import numpy as np

PKG = pathlib.Path(__file__).resolve().parent
LIB_PATH = PKG / "libsela_b200.so"
HEADER_PATH = PKG.parent / "include" / "sela_b200.h"

FRAME = 2048
MAX_ORDER = 100

# mirrors selab200_subframe_desc (include/sela_b200.h), 32 bytes
DESC_DTYPE = np.dtype([
    ("channel", "u1"), ("subframe_type", "u1"), ("parent_channel", "u1"),
    ("refl_rice_param", "u1"), ("refl_words", "<u2"), ("lpc_order", "u1"),
    ("res_rice_param", "u1"), ("res_words", "<u2"), ("samples", "<u2"),
    ("reserved", "<u4"), ("refl_offset", "<u8"), ("res_offset", "<u8"),
], align=True)
assert DESC_DTYPE.itemsize == 32

# mirrors selab200_container_info
INFO_DTYPE = np.dtype([
    ("sample_rate", "<u4"), ("bits_per_sample", "<u2"), ("channels", "u1"), ("reserved", "u1"),
    ("header_frames", "<u4"), ("n_frames", "<u4"), ("n_words", "<u8"), ("n_bytes_used", "<u8"),
], align=True)
assert INFO_DTYPE.itemsize == 32

# mirrors selab200_analysis_trace, 2832 bytes
TRACE_DTYPE = np.dtype([
    ("mean", "<f8"), ("ac", "<f8", (101,)), ("k", "<f8", (100,)), ("c", "<i8", (101,)),
    ("q", "<i4", (100,)), ("order", "<i4"), ("reserved", "<i4"),
], align=True)
assert TRACE_DTYPE.itemsize == 2832

# mirrors selab200_verify_entry, 16 bytes
VERIFY_DTYPE = np.dtype([
    ("frame", "<u4"), ("channel", "<u2"), ("first_sample", "<u2"), ("n_differing", "<u4"), ("first_delta", "<i4"),
], align=True)
assert VERIFY_DTYPE.itemsize == 16

# mirrors selab200_lossless_entry, 16 bytes
LOSSLESS_DTYPE = np.dtype([
    ("frame", "<u4"), ("channel", "<u2"), ("ref_order", "u1"), ("order", "u1"), ("ref_words", "<u4"), ("words", "<u4"),
], align=True)
assert LOSSLESS_DTYPE.itemsize == 16

# mirrors selab200_predictor, 404 bytes
PREDICTOR_DTYPE = np.dtype([("order", "<i4"), ("q", "<i4", (100,))], align=True)
assert PREDICTOR_DTYPE.itemsize == 404

# mirrors selab200_search_trace, 32 bytes
SEARCH_TRACE_DTYPE = np.dtype([
    ("pred_digest", "<u8"), ("res_digest", "<u8"), ("res_words", "<u4"), ("visits", "<u4"), ("refl_words", "<u2"),
    ("refl_k", "u1"), ("res_k", "u1"), ("tie", "u1"), ("reserved", "u1", (3,)),
], align=True)
assert SEARCH_TRACE_DTYPE.itemsize == 32

# mirrors selab200_search_unit, 416 bytes
SEARCH_UNIT_DTYPE = np.dtype([("q", "<i4", (100,)), ("ref_order", "<u4"), ("ref_words", "<u4"), ("best", "<u8")],
                             align=True)
assert SEARCH_UNIT_DTYPE.itemsize == 416

# mirrors selab200_clip, 16 bytes
CLIP_DTYPE = np.dtype([("container", "<u4"), ("reserved", "<u4"), ("start", "<u8")], align=True)
assert CLIP_DTYPE.itemsize == 16
CLIP_FLOAT32, CLIP_MEAN, CLIP_MAX_SELECT = 1, 2, 255   # selab200_container_decode_clips_select

STATUS_NAMES = {0: "OK", -1: "NO_DEVICE", -2: "CUDA", -3: "ARGUMENT", -4: "CAPACITY", -5: "RANGE",
                -6: "BITSTREAM", -7: "NOT_INIT"}


class SelaB200Error(RuntimeError):
    def __init__(self, status, message):
        super().__init__("selab200 status %d (%s): %s" % (status, STATUS_NAMES.get(status, "?"), message))
        self.status = status


_lib = None

_V, _U32, _SZ, _I = C.c_void_p, C.c_uint32, C.c_size_t, C.c_int
_SIGNATURES = {
    "selab200_init": (_I, [_I]),
    "selab200_init_devices": (_I, [_I, _V]),
    "selab200_device_count": (_I, []),
    "selab200_shutdown": (None, []),
    "selab200_last_error": (C.c_char_p, []),
    "selab200_abi_version": (_I, []),
    "selab200_launch_count": (C.c_uint64, []),
    "selab200_slot_launch_count": (C.c_uint64, [_I]),
    "selab200_selftest": (_I, [_V]),
    "selab200_host_alloc": (_V, [_SZ]),
    "selab200_host_free": (None, [_V]),
    "selab200_encode_words_bound": (_SZ, [_U32, _U32]),
    "selab200_encode_frames": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V]),
    "selab200_decode_frames": (_I, [_V, _U32, _U32, _V, _SZ, _V]),
    "selab200_encode_workspace_bytes": (_SZ, [_U32, _U32]),
    "selab200_encode_frames_device": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V, _V, _SZ, _V]),
    "selab200_decode_workspace_bytes": (_SZ, [_U32, _U32]),
    "selab200_decode_frames_device": (_I, [_V, _U32, _U32, _V, _SZ, _V, _V, _V, _SZ, _V]),
    "selab200_rice_decode_frames_device": (_I, [_V, _U32, _U32, _V, _SZ, _V, _V, _V]),
    "selab200_rice_decode_flagged": (_I, [_V]),
    "selab200_container_bound": (_SZ, [_U32, _U32]),
    "selab200_encode_container": (_I, [_V, _U32, _U32, _U32, C.c_uint16, _V, _SZ, _V]),
    "selab200_container_info_get": (_I, [_V, _SZ, _V]),
    "selab200_container_frame_offsets": (_I, [_V, _SZ, _V, _SZ, _V]),
    "selab200_container_open": (_I, [_V, _SZ, _V, _V]),
    "selab200_container_open_host": (_I, [_V, _SZ, _V, _V]),
    "selab200_container_decode": (_I, [_V, _V]),
    "selab200_container_close": (None, [_V]),
    "selab200_container_decode_clips": (_I, [_V, _U32, _V, _U32, _U32, _V, _V]),
    "selab200_container_decode_clips_device": (_I, [_V, _U32, _V, _U32, _U32, _V, _V]),
    "selab200_container_decode_clips_select": (_I, [_V, _U32, _V, _U32, _U32, _V, _U32, _U32, _V, _V, _V]),
    "selab200_container_decode_clips_select_device": (_I, [_V, _U32, _V, _U32, _U32, _V, _U32, _U32, _V, _V, _V]),
    "selab200_clip_bytes_fetched": (_I, [_V]),
    "selab200_verify_workspace_bytes": (_SZ, [_U32, _U32]),
    "selab200_verify_frames_device": (_I, [_V, _U32, _U32, _V, _SZ, _V, _V, _V, _V, _V, _SZ, _V]),
    "selab200_verify_frames": (_I, [_V, _U32, _U32, _V, _SZ, _V, _V, _SZ, _V]),
    "selab200_encode_container_verified": (_I, [_V, _U32, _U32, _U32, C.c_uint16, _V, _SZ, _V, _V, _SZ, _V]),
    "selab200_container_verify": (_I, [_V, _V, _V, _SZ, _V]),
    "selab200_encode_lossless_workspace_bytes": (_SZ, [_U32, _U32]),
    "selab200_encode_frames_lossless_device": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V, _V, _V, _V, _SZ, _V]),
    "selab200_encode_frames_lossless": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V, _SZ, _V]),
    "selab200_encode_container_lossless": (_I, [_V, _U32, _U32, _U32, C.c_uint16, _V, _SZ, _V, _V, _SZ, _V]),
    "selab200_encode_search_workspace_bytes": (_SZ, [_U32, _U32]),
    "selab200_encode_frames_search_device": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V, _V, _V, _SZ, _V]),
    "selab200_encode_frames_search": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V]),
    "selab200_encode_container_search": (_I, [_V, _U32, _U32, _U32, C.c_uint16, _V, _SZ, _V, _V]),
    "selab200_encode_pairing_workspace_bytes": (_SZ, [_U32, _U32]),
    "selab200_encode_frames_pairing_device": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V, _V, _V, _V, _SZ, _V]),
    "selab200_encode_frames_pairing": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V, _V]),
    "selab200_encode_container_pairing": (_I, [_V, _U32, _U32, _U32, C.c_uint16, _V, _SZ, _V, _V, _V]),
    "selab200_encode_search_pairing_workspace_bytes": (_SZ, [_U32, _U32]),
    "selab200_encode_frames_search_pairing_device": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V, _V, _V, _V, _SZ, _V]),
    "selab200_encode_frames_search_pairing": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V, _V]),
    "selab200_encode_container_search_pairing": (_I, [_V, _U32, _U32, _U32, C.c_uint16, _V, _SZ, _V, _V, _V]),
    "selab200_encode_search_windows_workspace_bytes": (_SZ, [_U32, _U32, _U32]),
    "selab200_encode_frames_search_windows_device": (_I, [_V, _U32, _U32, _U32, _V, _V, _SZ, _V, _V, _V, _V, _V, _SZ,
                                                          _V]),
    "selab200_encode_frames_search_windows": (_I, [_V, _U32, _U32, _U32, _V, _V, _SZ, _V, _V, _V]),
    "selab200_encode_container_search_windows": (_I, [_V, _U32, _U32, _U32, _U32, C.c_uint16, _V, _SZ, _V, _V, _V]),
    "selab200_analysis_window": (_I, [_I, _V]),
    "selab200_encode_search_guided_workspace_bytes": (_SZ, [_U32, _U32]),
    "selab200_encode_frames_search_guided_device": (_I, [_V, _U32, _U32, _U32, _V, _V, _SZ, _V, _V, _V, _V, _SZ, _V]),
    "selab200_encode_frames_search_guided": (_I, [_V, _U32, _U32, _U32, _V, _V, _SZ, _V, _V]),
    "selab200_encode_container_search_guided": (_I, [_V, _U32, _U32, _U32, _U32, C.c_uint16, _V, _SZ, _V, _V]),
    "selab200_lpc_residues": (_I, [_V, _U32, _V, _V, _V]),
    "selab200_lpc_samples": (_I, [_V, _U32, _V, _V, _V]),
    "selab200_rice_encode": (_I, [_V, _V, _U32, _U32, _V, _V, _V, _U32]),
    "selab200_rice_decode": (_I, [_V, _V, _U32, _V, _V, _U32, _V, _U32]),
    "selab200_encode_trace": (_I, [_V, _U32, _U32, _V, _V, _SZ, _V, _V]),
    "selab200_quantise_probe": (_I, [_V, _SZ, _V]),
    "selab200_fir_probe": (_I, [_V, _V, _V, _U32, _I, _V]),
    "selab200_fir_tie_probe": (_I, [_V, _V, _V, _U32, _I, _V, _V]),
    "selab200_encode_lossless_forced": (_I, [_V, _U32, _U32, _V, _V, _V, _SZ, _V, _V, _SZ, _V]),
    "selab200_encode_search_forced": (_I, [_V, _U32, _U32, _V, _V, _V, _SZ, _V, _V]),
    "selab200_encode_search_trace": (_I, [_V, _U32, _U32, _V, _V, _V, _SZ, _V, _V, _V, _V]),
    "selab200_encode_pairing_forced": (_I, [_V, _U32, _U32, _V, _V, _V, _SZ, _V, _V, _V]),
    "selab200_encode_pairing_trace": (_I, [_V, _U32, _U32, _V, _V, _V, _SZ, _V, _V, _V, _V, _V]),
    "selab200_encode_search_pairing_forced": (_I, [_V, _U32, _U32, _V, _V, _V, _SZ, _V, _V, _V]),
    "selab200_encode_search_pairing_trace": (_I, [_V, _U32, _U32, _V, _V, _V, _SZ, _V, _V, _V, _V, _V]),
    "selab200_encode_search_windows_forced": (_I, [_V, _U32, _U32, _U32, _V, _V, _V, _SZ, _V, _V, _V]),
    "selab200_encode_search_windows_trace": (_I, [_V, _U32, _U32, _V, _U32, _V, _V, _V, _SZ, _V, _V, _V, _V, _V]),
    "selab200_encode_search_guided_trace": (_I, [_V, _U32, _U32, _U32, _V, _V, _V, _SZ, _V, _V, _V, _V, _V]),
}


def exported_symbols():
    return sorted(_SIGNATURES)


def lib():
    """Load the extension (raises if it has not been built)."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise ImportError("%s not built: run `python -m sela_b200.build` (nvcc, sm_90a). "
                              "There is no CPU fallback." % LIB_PATH)
        L = C.CDLL(str(LIB_PATH))
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)           # AttributeError if the symbol is missing
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(status):
    if status != 0:
        raise SelaB200Error(status, lib().selab200_last_error().decode(errors="replace"))


_initialised = None


def init(device=0):
    """Bind the library to `device` (an int) or to several devices (a list/tuple: device[0] is the primary)."""
    global _initialised
    key = tuple(device) if isinstance(device, (list, tuple)) else (device,)
    if _initialised != key:
        arr = (C.c_int * len(key))(*key)
        check(lib().selab200_init_devices(len(key), C.addressof(arr)))
        _initialised = key
