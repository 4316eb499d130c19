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

// Offset that makes every in-domain ENCODER sample (|s| <= 65535) a non-negative 18-bit
// number, so int64 x int32 products need one IMAD.WIDE.U32 + one IMAD (see lpc.cuh).
// The decoder does not use it: its samples can be any int32 (kSynthBias).
constexpr int      kSampleBias = 1 << 17;
constexpr uint32_t kSampleBiasU = 1u << 17;
// The decoder's offset, 2^31: s ^ 2^31 == s + 2^31 maps every int32 onto [0, 2^32), so the
// same unsigned products are exact for any sample a stream can decode to (lpc.cuh, K6).
constexpr uint32_t kSynthBias = 0x80000000u;
__device__ __forceinline__ uint32_t synth_biased(int s) { return (uint32_t)s ^ kSynthBias; }

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

// d = a*b + c with a 32x32->64 multiply (IMAD.WIDE.U32).  Spelled in PTX because NVVM
// likes to hoist the zero-extension of a loop-invariant operand into a 64-bit register,
// after which ptxas emits a full 64x32 multiply (an extra IMAD + IADD per tap).
__device__ __forceinline__ unsigned long long mad_wide_u32(uint32_t a, uint32_t b, unsigned long long c)
{
    unsigned long long d;
    asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(d) : "r"(a), "r"(b), "l"(c));
    return d;
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

__device__ __forceinline__ void unpack8(const uint4 v, int (&s)[8])
{
    s[0] = (int)(v.x << 16) >> 16; s[1] = (int)v.x >> 16;
    s[2] = (int)(v.y << 16) >> 16; s[3] = (int)v.y >> 16;
    s[4] = (int)(v.z << 16) >> 16; s[5] = (int)v.z >> 16;
    s[6] = (int)(v.w << 16) >> 16; s[7] = (int)v.w >> 16;
}

// The signal one warp analyses, held in ONE int16 row of shared memory: a channel of the
// frame, or the 17-bit difference d = ch0 - ch1 (src/frame/frame_encoder.cpp:20-24) split as
// d >> 1 in the row and d & 1 in a 2048-bit side array (so a difference unit needs no more
// shared memory than a plain one and 24 units fit an SM).  `a` points at sample 0 (16-byte
// aligned, kHistoryPad zeros in front); `lo` is nullptr for a plain channel, else bit j of
// lo[] is d[j] & 1 (kHistoryPad zero bits in front as well).
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
    // samples [8g, 8g+8) biased by 2^17 (g >= -kHistoryPad/8)
    __device__ __forceinline__ void load8(int g, uint32_t (&w)[8]) const
    {
        int s[8];
        unpack8(*reinterpret_cast<const uint4 *>(a + 8 * g), s);
        if (lo) {
            const uint32_t bits = reinterpret_cast<const uint8_t *>(lo)[g];
#pragma unroll
            for (int r = 0; r < 8; r++)
                s[r] = (s[r] << 1) | (int)((bits >> r) & 1u);
        }
#pragma unroll
        for (int r = 0; r < 8; r++)
            w[r] = (uint32_t)(s[r] + kSampleBias);
    }
};

// int32 signal in shared memory (stage-level entry points), same conventions.
struct PlainSignal {
    const int32_t *s;
    __device__ __forceinline__ int at(int j) const { return s[j]; }
    __device__ __forceinline__ void load8(int g, uint32_t (&w)[8]) const
    {
        const int4 v0 = *reinterpret_cast<const int4 *>(s + 8 * g);
        const int4 v1 = *reinterpret_cast<const int4 *>(s + 8 * g + 4);
        w[0] = (uint32_t)(v0.x + kSampleBias); w[1] = (uint32_t)(v0.y + kSampleBias);
        w[2] = (uint32_t)(v0.z + kSampleBias); w[3] = (uint32_t)(v0.w + kSampleBias);
        w[4] = (uint32_t)(v1.x + kSampleBias); w[5] = (uint32_t)(v1.y + kSampleBias);
        w[6] = (uint32_t)(v1.z + kSampleBias); w[7] = (uint32_t)(v1.w + kSampleBias);
    }
};

// Device-side status: first error wins (codes are negative, so take the min).
__device__ __forceinline__ void raise_status(int32_t *status, int code)
{
    if (status)
        atomicMin(status, code);
}

} // namespace selab200
