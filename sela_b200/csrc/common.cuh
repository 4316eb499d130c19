// common.cuh -- shared definitions for the sm_90a kernels of the SELA hot path.
//
// One warp owns one subframe (one channel of one 2048-sample frame).  All
// floating point that feeds the bitstream goes through the *_rn intrinsics below:
// they are never contracted into FMAs, so every operation rounds exactly once, in
// the reference's order (SURVEY.md 7.3-H1).  The translation units are also built
// with -fmad=false as a second line of defence.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/sela_b200.h"

namespace selab200 {

constexpr int kFrame    = SELAB200_FRAME_SAMPLES; // 2048
constexpr int kMaxOrder = SELAB200_MAX_LPC_ORDER; // 100
constexpr int kMaxRice  = SELAB200_MAX_RICE_PARAM; // 20 (k searched in [0, 20))
constexpr int kQ        = 35;                      // CORRECTION_FACTOR, src/include/lpc.hpp:8
constexpr unsigned kFull = 0xffffffffu;

// The decoder's offset, 2^31: s ^ 2^31 == s + 2^31 maps every int32 onto [0, 2^32), so the
// same unsigned products are exact for any sample a stream can decode to (lpc.cuh, K6).
constexpr uint32_t kSynthBias = 0x80000000u;

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double dsqrt(double a) { return __dsqrt_rn(a); }

__device__ __forceinline__ double shfl_d(double v, int src)
{
    return __shfl_sync(kFull, v, src);
}
__device__ __forceinline__ double shfl_down_d(double v, int delta)
{
    return __shfl_down_sync(kFull, v, delta);
}
__device__ __forceinline__ unsigned long long shfl_u64(unsigned long long v, int src)
{
    return __shfl_sync(kFull, v, src);
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// Inclusive prefix sum over the warp.
__device__ __forceinline__ uint32_t warp_scan_inclusive_u32(uint32_t v)
{
    const int lane = lane_id();
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(kFull, v, o);
        if (lane >= o)
            v += t;
    }
    return v;
}

// Every signal buffer in shared memory is preceded by kHistoryPad zero samples: the
// history "before the frame" that the filters read as s = 0.
constexpr int kHistoryPad = 128;

// The signal one warp analyses, held in ONE int16 row of shared memory: a 16-bit channel of
// the frame, or a 17-bit signal d (the difference d = ch0 - ch1 of src/frame/frame_encoder.cpp:20-24,
// or any row of the stage operator selab200_lpc_residues) split as d >> 1 in the row and d & 1 in a
// 2048-bit side array (so a 17-bit unit needs no more shared memory than a plain one and 24 units fit
// an SM).  `a` points at sample 0 (16-byte aligned, kHistoryPad zeros in front); `lo` is nullptr for a
// plain channel, else bit j of lo[] is d[j] & 1 (kHistoryPad zero bits in front as well).
struct Signal {
    const int16_t *a;
    const uint32_t *lo;
    __device__ __forceinline__ int at(int j) const
    {
        int v = a[j];
        if (lo)
            v = (v << 1) | (int)((lo[j >> 5] >> (j & 31)) & 1u);
        return v;
    }
};

// Stages one 17-bit row (|s| <= 65535) of global memory as a Signal: s >> 1 into row[0..2048), s & 1 into
// lo[0..64).  The kHistoryPad zeros in front of both are the caller's.
__device__ __forceinline__ void stage_17bit_row(const int32_t *src, int16_t *row, uint32_t *lo)
{
    const int lane = lane_id();
    for (int it = 0; it < kFrame / 32; it++) {
        const int s = src[it * 32 + lane];
        row[it * 32 + lane] = (int16_t)(s >> 1);
        const uint32_t bits = __ballot_sync(kFull, s & 1);
        if (lane == 0)
            lo[it] = bits;
    }
}

// A stream of `words` words at word `offset` lies inside an arena of n_words words.  Written without a sum:
// offset + words <= n_words wraps in 64 bits for offset = 2^64 - w and would accept a stream that starts in
// front of the arena.
__host__ __device__ __forceinline__ bool words_in_arena(unsigned long long offset, unsigned long long words,
                                                        unsigned long long n_words)
{
    return words <= n_words && offset <= n_words - words;
}

// The decoder's acceptance of one subframe descriptor (frame_check in kernels.cuh adds the rules that span a
// frame).  The host uses the same range test to decide which words a batch references.
__host__ __device__ __forceinline__ bool desc_ok(const selab200_subframe_desc &d, uint32_t channels,
                                                 unsigned long long n_words)
{
    return d.channel < channels && d.parent_channel < channels && d.subframe_type <= 1 &&
           d.lpc_order <= kMaxOrder && d.refl_rice_param < 32 && d.res_rice_param < 32 &&
           d.samples == kFrame && words_in_arena(d.refl_offset, d.refl_words, n_words) &&
           words_in_arena(d.res_offset, d.res_words, n_words) &&
           !(d.subframe_type == 1 && d.parent_channel == d.channel);
}

// Device-side status: first error wins (codes are negative, so take the min).
__device__ __forceinline__ void raise_status(int32_t *status, int code)
{
    if (status)
        atomicMin(status, code);
}

} // namespace selab200
