"""sela_b200 -- H100-native implementation of SELA's per-frame encode/decode hot path.

CUDA kernels (sm_90a) behind the C ABI of include/sela_b200.h; this package holds
the kernels (csrc/), the C++ mirror of the reference interface (host/) and a thin
Python mirror used by the tests and bench.py.  No CPU fallback.
"""
from .clips import ClipDecoder  # noqa: F401
from .codec import (DESC_DTYPE, FRAME, LOSSLESS_DTYPE, VERIFY_DTYPE, SelaB200Error, container_info,  # noqa: F401
                    decode_container, decode_frames, encode_container, encode_container_lossless,
                    encode_container_search, encode_container_verified, encode_frames, encode_frames_lossless,
                    encode_frames_search, encode_container_pairing, encode_frames_pairing,
                    encode_container_search_pairing, encode_frames_search_pairing,
                    encode_container_search_windows, encode_frames_search_windows, analysis_window,
                    encode_container_search_guided, encode_frames_search_guided, init,
                    lpc_residues, lpc_samples, rice_decode, rice_encode, verify_container, verify_frames)
