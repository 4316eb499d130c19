// lpc.cuh -- warp-level LPC analysis / synthesis (kernels K1, K2, K3, K6 of SURVEY.md 2).
//
// One warp processes one 2048-sample signal.  The double-precision front end
// reproduces the reference's operation order and rounding exactly
// (src/lpc/residue_generator.cpp:12-96, src/lpc/linear_predictor.cpp:16-61):
// parallelism is taken ACROSS lags / coefficients, never across the terms of a sum.
#pragma once

#include "common.cuh"
#include "lpc_tables.cuh"

namespace selab200 {

// Per-warp shared memory.  The predictor (shared by encoder and decoder):
struct CoefSmem {
    uint32_t clo[112];           // low / high words of the Q35 coefficients c[1..], tap j at index
    int32_t  chi[112];           //   j-1, zero padded: the FIR reads them in blocks of 8
    int32_t  q[104];             // quantised reflection coefficients
};
// Analysis scratch (3 KB).  The ring is dead once the autocorrelation is done; the
// reflection coefficients (kk) and the step-up row (t) then live in its bytes.
struct AnalysisScratch {
    double ring[256]; // the d = x - mean ring of the autocorrelation (swizzled)
    double ac[128];   // autocorrelation (raw, then normalised)
    __device__ __forceinline__ double *kk() { return ring; }        // k[0..99]
    __device__ __forceinline__ double *t() { return ring + 104; }   // step-up scratch [0..99]
};
using LpcSmem = AnalysisScratch;
// k[0..99] and the step-up row t[0..99] occupy doubles [0, 204) of the ring; from here to the end of ac[] the
// scratch is free after warp_schur() (which reads ac[] into registers first): the encoder puts its CoefSmem there.
constexpr size_t kCoefAlias = 208 * sizeof(double);

__device__ __forceinline__ long long coef_at(const CoefSmem &cf, int j) // c[j], j >= 1
{
    return (long long)(((unsigned long long)(uint32_t)cf.chi[j - 1] << 32) | cf.clo[j - 1]);
}

// ---------------------------------------------------------------------------
// ring addressing: 256 doubles = 128 chunks of 16 B (a 128-sample tile plus the 127
// samples of history the furthest lane still needs).  Odd 128-byte rows have their
// chunk pairs swapped so that the "own window" LDS.128 of the autocorrelation (lanes
// 32 B apart) is bank-conflict free.
__device__ __forceinline__ int ring_chunk(int chunk)
{
    chunk &= 127;
    return chunk ^ ((chunk >> 3) & 1);
}
__device__ __forceinline__ int ring_index(int p) // logical sample index (may be negative)
{
    return (ring_chunk(p >> 1) << 1) | (p & 1);
}

// x[j] = (double)s[j] / 32767  (quantizeSamples, residue_generator.cpp:12-18).
// Correctly rounded quotient without the division subroutine: q0 = s*rcp, one exact
// FMA residual, one FMA correction (Markstein).  Equality with IEEE division is
// verified EXHAUSTIVELY over the whole input domain |s| <= 65535 -- on the CPU in
// tests/test_host_logic.py and on the device by selab200_selftest().
__device__ __forceinline__ double sample_to_x(int s)
{
    const double rcp = 1.0 / 32767.0;
    const double a = (double)s;
    const double q0 = __dmul_rn(a, rcp);
    const double r = __fma_rn(-q0, 32767.0, a);
    return __fma_rn(r, rcp, q0);
}
__device__ __forceinline__ double sample_to_x_div(int s) { return ddiv((double)s, 32767.0); }

// ---------------------------------------------------------------------------
// K1a: the mean of generateAutoCorrelation (residue_generator.cpp:26-30): ONE sequential
// chain  sum = sum + x[j]  over j = 0..2047, then sum / 2048.  Run by one LANE per signal
// (k_unit_means, 32 signals per warp): the only definition of the chain.
struct MeanChain {
    double sum = 0.0;
    __device__ __forceinline__ void add(int s) { sum = dadd(sum, sample_to_x(s)); }
    __device__ __forceinline__ double mean() const { return ddiv(sum, (double)kFrame); } // exact: power of two
};

// ---------------------------------------------------------------------------
// K1: mean-removed autocorrelation, lags 0..100, + normalisation.
// generateAutoCorrelation (residue_generator.cpp:20-45).  Result in sm.ac[0..100].
//
//  - mean: from k_unit_means (MeanChain), computed before the warp starts;
//  - lane l owns lags 4l..4l+3 (lanes 0..25 useful).  For step j the four products
//    are d[j]*d[j-4l-m]; each accumulator is a sequential chain over j, exactly
//    `ac[i] += d[j]*d[j-i]` with the multiply rounded before the add;
//  - j < i terms are fed as d[negative] = +0.0: acc + (+-0) leaves a +0.0
//    accumulator unchanged, so starting the chain at j = 0 instead of j = i is
//    bit-identical;
//  - WINDOW (the window search, DESIGN.md 7.6): d[j] = (x[j] - mean) * win[j], one more
//    rounded multiply per staged value.  The 32 lanes read 32 different j, so win is read
//    through L1 (a __constant__ table would serialise them).
template <typename Sig, bool WINDOW = false>
__device__ void warp_autocorrelation(const Sig &sig, LpcSmem &sm, const double mean, const double *win = nullptr)
{
    const int lane = lane_id();

    // logical d[-128..-1] = 0  -> chunks 64..127 (the upper half of the ring)
    {
        double2 *r2 = reinterpret_cast<double2 *>(sm.ring);
        r2[64 + lane] = make_double2(0.0, 0.0);
        r2[96 + lane] = make_double2(0.0, 0.0);
    }
    double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
    double p1 = 0.0, p2 = 0.0, p3 = 0.0; // d[4G-1], d[4G-2], d[4G-3]
    const char *ringb = reinterpret_cast<const char *>(sm.ring);
    // Groups are processed 8 at a time (g = g0 + i, g0 a multiple of 8), which makes the
    // swizzle bit of every access loop-invariant: for the broadcast group it is (i>>2)&1, a
    // compile-time constant; for the lane's own group G = g - lane it is ((i - lane)>>2)&1.
    // The physical byte offset of chunk 2G is then (32*g0 + own_off[i]) & 2047.
    int own_off[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int rel = i - lane;
        own_off[i] = 16 * (2 * rel + ((rel >> 2) & 1));
    }

    for (int tile = 0; tile < kFrame / 128; tile++) {
        __syncwarp();
#pragma unroll
        for (int r = 0; r < 4; r++) {
            int j = tile * 128 + r * 32 + lane;
            if constexpr (WINDOW)
                sm.ring[ring_index(j)] = dmul(dsub(sample_to_x(sig.at(j)), mean), __ldg(win + j));
            else
                sm.ring[ring_index(j)] = dsub(sample_to_x(sig.at(j)), mean);
        }
        __syncwarp();
        for (int blk = 0; blk < 4; blk++) {
            const int gb = (tile * 32 + blk * 8) * 32; // byte offset of chunk 2*g0 before wrapping
            const char *bbase = ringb + (gb & 2047);    // 256-byte aligned: the 8 broadcast groups never wrap
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int oo = (gb + own_off[i]) & 2047;
                const double2 o0 = *reinterpret_cast<const double2 *>(ringb + oo);
                const double2 o1 = *reinterpret_cast<const double2 *>(ringb + (oo ^ 16));
                constexpr int kSw[8] = {0, 0, 0, 0, 16, 16, 16, 16};
                const double2 b0 = *reinterpret_cast<const double2 *>(bbase + ((32 * i) ^ kSw[i]));
                const double2 b1 = *reinterpret_cast<const double2 *>(bbase + ((32 * i + 16) ^ kSw[i]));
                const double c0 = o0.x, c1 = o0.y, c2 = o1.x, c3 = o1.y; // d[4G..4G+3]
                // u = 0  (j = 4g)
                acc0 = dadd(acc0, dmul(b0.x, c0));
                acc1 = dadd(acc1, dmul(b0.x, p1));
                acc2 = dadd(acc2, dmul(b0.x, p2));
                acc3 = dadd(acc3, dmul(b0.x, p3));
                // u = 1
                acc0 = dadd(acc0, dmul(b0.y, c1));
                acc1 = dadd(acc1, dmul(b0.y, c0));
                acc2 = dadd(acc2, dmul(b0.y, p1));
                acc3 = dadd(acc3, dmul(b0.y, p2));
                // u = 2
                acc0 = dadd(acc0, dmul(b1.x, c2));
                acc1 = dadd(acc1, dmul(b1.x, c1));
                acc2 = dadd(acc2, dmul(b1.x, c0));
                acc3 = dadd(acc3, dmul(b1.x, p1));
                // u = 3
                acc0 = dadd(acc0, dmul(b1.y, c3));
                acc1 = dadd(acc1, dmul(b1.y, c2));
                acc2 = dadd(acc2, dmul(b1.y, c1));
                acc3 = dadd(acc3, dmul(b1.y, c0));
                p1 = c3;
                p2 = c2;
                p3 = c1;
            }
        }
    }
    __syncwarp();
    sm.ac[4 * lane + 0] = acc0;
    sm.ac[4 * lane + 1] = acc1;
    sm.ac[4 * lane + 2] = acc2;
    sm.ac[4 * lane + 3] = acc3;
    __syncwarp();
    // normalise (residue_generator.cpp:41-44): ac[i] /= ac[0] for i >= 1, then ac[0] = 1
    const double ac0 = sm.ac[0];
    __syncwarp();
#pragma unroll
    for (int t = 0; t < 4; t++) {
        int i = lane + 32 * t;
        if (i >= 1 && i <= kMaxOrder)
            sm.ac[i] = ddiv(sm.ac[i], ac0);
    }
    if (lane == 0)
        sm.ac[0] = 1.0;
    __syncwarp();
}

// ---------------------------------------------------------------------------
// K2a: Schur recursion -> 100 reflection coefficients in sm.kk
// generateReflectionCoefficients (residue_generator.cpp:47-68).
// Lane l holds generator elements j = 4l..4l+3 in registers; every per-element
// update is independent, the only serial piece is k[i] = -g1[0]/err.
__device__ void warp_schur(LpcSmem &sm)
{
    const int lane = lane_id();
    double *kk = sm.kk(); // overlays the ring, which the autocorrelation no longer needs
    double g0[4], g1[4];
#pragma unroll
    for (int m = 0; m < 4; m++) {
        int j = 4 * lane + m;
        double v = (j < kMaxOrder) ? sm.ac[j + 1] : 0.0;
        g0[m] = v;
        g1[m] = v;
    }
    double err = sm.ac[0];
    double head = shfl_d(g1[0], 0);
    double k = ddiv(-head, err);
    err = dadd(err, dmul(head, k));
    if (lane == 0)
        kk[0] = k;
    for (int i = 1; i < kMaxOrder; i++) {
        const double kp = k;
        const double nxt = shfl_down_d(g1[0], 1); // g1[4(l+1)] of the previous sweep
        double up[4] = {g1[1], g1[2], g1[3], nxt};
#pragma unroll
        for (int m = 0; m < 4; m++) {
            double n1 = dadd(up[m], dmul(kp, g0[m]));
            double n0 = dadd(dmul(up[m], kp), g0[m]);
            g1[m] = n1;
            g0[m] = n0;
        }
        head = shfl_d(g1[0], 0);
        k = ddiv(-head, err);
        err = dadd(err, dmul(head, k));
        if (lane == 0)
            kk[i] = k;
    }
    __syncwarp();
}

// ---------------------------------------------------------------------------
// K2b: order selection + 7-bit quantisation
// generateoptimalLpcOrder / quantizeReflectionCoefficients (residue_generator.cpp:70-96).
// The threshold and the quantiser of one coefficient are also run on their own, on chosen inputs, by the test
// entry selab200_quantise_probe (k_quantise_probe).

// Whether k counts for the order: the order is one past the last such coefficient (residue_generator.cpp:73).
__device__ __forceinline__ bool reflection_significant(double kv) { return fabs(kv) > 0.05; }

// q of coefficient i with value kv: i = 0 and i = 1 through the square-root companding, the rest linearly.
// k outside [-1, 1] makes the square root NaN, and a NaN quantises to 0 (residue_generator.cpp:85-94).
__device__ __forceinline__ int quantise_reflection(int i, double kv)
{
    const double sqrt2 = 1.4142135623730950488016887242096; // src/include/lpc.hpp:9
    double v;
    if (i == 0)
        v = floor(dmul(64.0, dadd(-1.0, dmul(sqrt2, dsqrt(dadd(kv, 1.0))))));
    else if (i == 1)
        v = floor(dmul(64.0, dadd(-1.0, dmul(sqrt2, dsqrt(dadd(-kv, 1.0))))));
    else
        v = floor(dmul(64.0, kv));
    return isnan(v) ? 0 : __double2int_rz(v);
}

__device__ int warp_order_and_quantise(LpcSmem &sm, CoefSmem &cf)
{
    const int lane = lane_id();
    const double *kk = sm.kk();
    int best = -1;
#pragma unroll
    for (int t = 0; t < 4; t++) {
        int i = lane + 32 * t;
        if (i < kMaxOrder && reflection_significant(kk[i]))
            best = i;
    }
    best = __reduce_max_sync(kFull, best);
    const int order = best < 0 ? 1 : best + 1; // default 1 (src/include/lpc.hpp:76)

#pragma unroll
    for (int t = 0; t < 4; t++) {
        int i = lane + 32 * t;
        if (i < order) {
            cf.q[i] = quantise_reflection(i, kk[i]);
        } else if (i < 104) {
            cf.q[i] = 0;
        }
    }
    __syncwarp();
    return order;
}

// ---------------------------------------------------------------------------
// K2c: de-quantise + step-up -> Q35 integer predictor (cf.clo/chi, tap j at index j-1)
// LinearPredictor::dequantizeReflectionCoefficients / generatelinearPredictionCoefficients
// (src/lpc/linear_predictor.cpp:16-61).  Shared by encoder and decoder.
// Table indices are clamped to [0,127] (the reference reads out of bounds there).
__device__ __forceinline__ double dequantise(int i, int q)
{
    int idx = q + 64;
    idx = idx < 0 ? 0 : (idx > 127 ? 127 : idx);
    if (i == 0)
        return __longlong_as_double((long long)selab200_FIRST_BITS[idx]);
    if (i == 1)
        return idx == 0 ? __longlong_as_double((long long)SELAB200_SECOND0_BITS)
                        : -__longlong_as_double((long long)selab200_FIRST_BITS[idx]);
    return (double)(idx - 64) / 64.0; // exact
}

__device__ void warp_coefficients(CoefSmem &cf, double *t, int order)
{
    const int lane = lane_id();
    for (int i = lane; i < 112; i += 32) {
        cf.clo[i] = 0;
        cf.chi[i] = 0;
    }
    __syncwarp();
    if (order <= 1)
        return; // a single zero reflection coefficient -> c[1] = 0 (linear_predictor.cpp:19-22)
    for (int i = 0; i < order; i++) {
        const double ki = dequantise(i, cf.q[i]);
        const int half = i >> 1;
        for (int j = lane; j < half; j += 32) {
            double a = t[j];
            double b = t[i - 1 - j];
            t[j] = dadd(a, dmul(ki, b));
            t[i - 1 - j] = dadd(b, dmul(ki, a));
        }
        if (lane == 0) {
            if (i & 1) {
                double mid = t[half];
                t[half] = dadd(mid, dmul(mid, ki));
            }
            t[i] = ki;
        }
        __syncwarp();
    }
    const double scale = 34359738368.0; // 2^35
    for (int m = lane; m < order; m += 32) {
        const long long v = __double2ll_rz(dmul(scale, -t[m]));
        cf.clo[m] = (uint32_t)v;
        cf.chi[m] = (int32_t)(v >> 32);
    }
    __syncwarp();
}

// ---------------------------------------------------------------------------
// K3: integer FIR residual.  generateResidues (residue_generator.cpp:98-119):
//   r[i] = s[i] - (int32)((2^34 + sum_{j=1..order} c[j]*s[i-j]) >> 35),  s[<0] = 0
// on the tensor cores.  With the outputs folded as i = 8a + b (a < 256, b < 8) the Toeplitz product is a GEMM,
//   Y[a][b] = sum_m A[a][m] * B[m][b],   A[a][m] = s[8a + 7 - m],   B[m][b] = c[m + b - 7] (0 outside 1..order),
// over K = order + 8 rounded up to 32: 1-4 k-steps of mma.sync m16n8k32 for each of the 16 M-tiles (16 rows a,
// 128 outputs) of a signal.  It is made exact with byte limbs:
//  - a coefficient is split into L signed digits, c = sum_{p<L} e_p * 256^p (mod 2^64) with e_p in [-128, 128):
//    e_p is byte p of (c + H) ^ H, H = 0x8080...80.  L (0..8) is the largest number any tap needs, so it is the
//    same for the whole warp;
//  - a 16-bit sample is u8 + 256 * s8 (its two bytes); a 17-bit one is u8 + 256 * u8 + 65536 * s8 (the top limb
//    is 0 or -1);
//  - all limb products of weight 256^k (k < 8) go into one int32 accumulator T[k]: at most 3 * 128 products of
//    magnitude <= 255 * 128, so |T[k]| < 2^24 and every T[k] is exact;
//  - the sum is sum_k T[k] * 256^k, formed mod 2^64; weights 256^k with k >= 8 are multiples of 2^64.
// So every int64 coefficient, saturated ones included, gives the same sum mod 2^64 as the reference's int64
// arithmetic: bit-identical residues.  Integer adds wrap identically in any order.
// Group g = lane / 4 and t = lane % 4 of the mma fragments: the A-register of rows (a, m..m+3), m = 4t (+16), holds
// samples 8a + 4 - m .. 8a + 7 - m in reverse order -- one 8-byte load at a 4-aligned sample, bytes picked by PRMT.
// The B-register of column g, rows m..m+3, holds e_p(c[m + g - 7 ..]): 4 bytes at offset m + g of digit plane p.
constexpr int kPlaneWords = 34; // a digit plane: bytes x = m + b < 135 of B, byte x = e_p(c[x - 7])
constexpr size_t kPlaneBytes = 8 * kPlaneWords * 4;

// The digit planes of c[1..112] into planes[8][kPlaneWords]; returns L.  planes may overlay anything but cf once
// every lane is past its last read of it (the __syncwarp below).
__device__ int warp_fir_planes(const CoefSmem &cf, uint32_t *planes)
{
    const unsigned long long H = 0x8080808080808080ull;
    const int lane = lane_id();
    __syncwarp();
    int nd = 0;
    for (int w = lane; w < kPlaneWords; w += 32) {
        unsigned long long e[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int j = 4 * w + i - 7;
            const unsigned long long c = (j >= 1 && j <= 112) ? (unsigned long long)coef_at(cf, j) : 0ull;
            e[i] = (c + H) ^ H;
            nd = max(nd, (64 - __clzll((long long)e[i]) + 7) >> 3);
        }
#pragma unroll
        for (int p = 0; p < 8; p++) {
            uint32_t v = 0;
#pragma unroll
            for (int i = 0; i < 4; i++)
                v |= (uint32_t)((e[i] >> (8 * p)) & 0xffu) << (8 * i);
            planes[p * kPlaneWords + w] = v;
        }
    }
    __syncwarp();
    return __reduce_max_sync(kFull, nd);
}

__device__ __forceinline__ uint32_t prmt(uint32_t x, uint32_t y, uint32_t sel) // selector bit 3: replicate the sign
{
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(x), "r"(y), "r"(sel));
    return d;
}

// d += A * B on one m16n8k32 tile: A bytes unsigned or signed, B bytes signed.
template <bool ASIGNED>
__device__ __forceinline__ void mma_s8(int32_t (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    if constexpr (ASIGNED)
        asm("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
            : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    else
        asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
            : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ unsigned long long mad_wide_s32(int32_t a, int32_t b, unsigned long long c)
{
    unsigned long long d;
    asm("mad.wide.s32 %0, %1, %2, %3;" : "=l"(d) : "r"(a), "r"(b), "l"(c));
    return d;
}

// WIDE: sig is a 17-bit signal (sig.lo != nullptr).  planes: 1088 bytes of scratch (see warp_fir_planes).
// CHECK: also return, to every lane, whether some output is a tie -- a prediction the decoder rounds differently,
// (int32)((2^34 + P) >> 35) + (int32)((2^34 - P) >> 35) != 0 with 2^34 - P = 2^35 - sum mod 2^64 (DESIGN.md 7.2).
// The unit then does not decode back to its source under the reference decoder; without one it does.
template <bool WIDE, bool CHECK = false>
__device__ bool warp_fir_residual(const Signal &sig, const CoefSmem &cf, int order, uint32_t *planes, int32_t *res)
{
    bool tie = false;
    constexpr int NL = WIDE ? 3 : 2; // sample limbs: u8, (u8,) s8
    const int lane = lane_id();
    const int g = lane >> 2, t = lane & 3;
    const int nd = warp_fir_planes(cf, planes);
    const int ksteps = (order + 8 + 31) >> 5;
    const uint32_t *pg = planes + t + (g >> 2); // word of byte 4t + g of a plane; shifted by 8 * (g & 3) bits
    const uint32_t sh = 8 * (g & 3);
    for (int mt = 0; mt < kFrame / 128; mt++) {
        int32_t T[8][4];
#pragma unroll
        for (int k = 0; k < 8; k++)
            T[k][0] = T[k][1] = T[k][2] = T[k][3] = 0;
        for (int ks = 0; ks < ksteps; ks++) {
            // A-registers 0..3: rows a = 16mt + g (+8), k = 32ks + 4t (+16): samples from s0 + kOff[r]
            const int s0 = 128 * mt + 8 * g + 4 - 4 * t - 32 * ks;
            constexpr int kOff[4] = {0, 64, -16, 48};
            uint32_t A[NL][4];
#pragma unroll
            for (int r = 0; r < 4; r++) {
                const int j = s0 + kOff[r];
                const uint2 v = *reinterpret_cast<const uint2 *>(sig.a + j);
                if constexpr (WIDE) {
                    // d = 2h + p: the bytes of 2h (bit 15 of the lower h moves into bit 0 of the upper one: masked),
                    // the parity bits p[j + 3 - i] into bit 0 of byte i, and the sign of h as the top limb
                    const uint32_t x = v.x << 1, y = v.y << 1;
                    const uint32_t nib = (sig.lo[j >> 5] >> (j & 31)) & 0xfu;
                    const uint32_t par = ((nib * 0x08040201u) >> 3) & 0x01010101u;
                    A[0][r] = (prmt(x, y, 0x0246) & 0xfefefefeu) | par;
                    A[1][r] = prmt(x, y, 0x1357);
                    A[2][r] = prmt(v.x, v.y, 0x9bdf);
                } else {
                    A[0][r] = prmt(v.x, v.y, 0x0246);
                    A[1][r] = prmt(v.x, v.y, 0x1357);
                }
            }
            const uint32_t *pk = pg + 8 * ks;
#pragma unroll
            for (int p = 0; p < 8; p++) {
                if (p < nd) {
                    const uint32_t *w = pk + p * kPlaneWords;
                    const uint32_t b0 = __funnelshift_r(w[0], w[1], sh);
                    const uint32_t b1 = __funnelshift_r(w[4], w[5], sh);
                    // limb l of the sample has weight 256^l: its products with e_p go to T[p + l]
                    mma_s8<false>(T[p], A[0], b0, b1);
                    if (p + 1 < 8)
                        mma_s8<!WIDE>(T[p + 1], A[1], b0, b1);
                    if constexpr (WIDE)
                        if (p + 2 < 8)
                            mma_s8<true>(T[p + 2], A[2], b0, b1);
                }
            }
        }
        // T[k][r]: output i = 128mt + 8g + 2t + (r & 1) + 64 * (r >> 1)
        const int i0 = 128 * mt + 8 * g + 2 * t;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int i = i0 + 64 * h;
            const uint32_t pair = *reinterpret_cast<const uint32_t *>(sig.a + i);
            int s[2] = {(int)(pair << 16) >> 16, (int)pair >> 16};
            if constexpr (WIDE) {
                const uint32_t bits = sig.lo[i >> 5] >> (i & 31);
                s[0] = 2 * s[0] + (int)(bits & 1u);
                s[1] = 2 * s[1] + (int)((bits >> 1) & 1u);
            }
            int32_t out[2];
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int r = 2 * h + e;
                unsigned long long sum = 1ull << (kQ - 1);
#pragma unroll
                for (int k = 0; k < 4; k++)
                    sum = mad_wide_s32(T[k][r], 1 << (8 * k), sum);
                const uint32_t top = (uint32_t)T[4][r] + ((uint32_t)T[5][r] << 8) + ((uint32_t)T[6][r] << 16) +
                                     ((uint32_t)T[7][r] << 24); // weights 2^32 .. 2^56: only the high word
                sum += (unsigned long long)top << 32;
                out[e] = s[e] - (int32_t)((long long)sum >> kQ);
                if constexpr (CHECK)
                    tie |= (int32_t)((long long)sum >> kQ) + (int32_t)((long long)((1ull << kQ) - sum) >> kQ) != 0;
            }
            *reinterpret_cast<int2 *>(res + i) = make_int2(out[0], out[1]);
        }
    }
    __syncwarp();
    if constexpr (CHECK)
        return __any_sync(kFull, tie);
    return false;
}

// ---------------------------------------------------------------------------
// K6: integer IIR synthesis.  SampleGenerator::generateSamples
// (src/lpc/sample_generator.cpp:11-30):
//   s[i] = r[i] - (int)((2^34 - sum_{j=1..order} c[j]*s[i-j]) >> 35),  s[<0] = 0
// Decoded samples can be any int32: they enter the products biased by 2^31 (kSynthBias), so that
// c*s' needs one IMAD.WIDE.U32 (low word of c) and one IMAD (high word), and the bias is taken
// out once per output (segment_state):
//   sum_j c[j]*s[i-j] = sum_j c[j]*s'[i-j] - 2^31 * sum_j c[j].
// Products and sums wrap mod 2^64, which cancels exactly: the result is the reference's int64
// sum wherever that sum does not overflow.
// A true recurrence, evaluated in TRANSPOSED form: a lane owns kTapsPerLane consecutive taps
// and the partial sums of the outputs those taps will feed next.  When s[i] becomes
// known every lane adds c[j]*s'[i] to the accumulator of output i+j; the accumulator
// of output i+1 (tap 1, first lane) is then complete, that lane finishes the sample and
// broadcasts it, and every accumulator moves one tap down (one 64-bit shuffle per
// lane, register renaming inside a lane).  Critical path per sample: the two multiplies of
// tap 1, a shift-and-add, an add and ONE shuffle -- instead of a five-level reduction.
//
// A warp runs as many subframes as fit, each on a SEGMENT of consecutive lanes.  A subframe of
// order o owns n = max(1, ceil(o / kTapsPerLane)) lanes; lane k of the segment owns taps kTapsPerLane*k + 1 ..
// kTapsPerLane*(k+1) (zero beyond o).  Every segment runs the recurrence at once: the segment's top lane starts a new
// output where the others take the accumulator of the lane above, and the finished sample reaches the segment from its
// first lane.  Taps per lane are fixed, so the multiplies a warp issues follow the orders it holds.
constexpr int kTapsPerLane = 8;
constexpr int kMaxWidth = (kMaxOrder + kTapsPerLane - 1) / kTapsPerLane; // 13 lanes for order 100
constexpr int kSegBlock = 16; // samples per staging block
constexpr int kSegRow = 20;   // words per staging row: the rows of eight segments sit on eight distinct 4-bank groups
static_assert(kSegBlock % kTapsPerLane == 0, "the register of slot 0 must be static inside a block");

__device__ __forceinline__ int segment_width(int order)
{
    return order <= kTapsPerLane ? 1 : (order + kTapsPerLane - 1) / kTapsPerLane;
}

struct SegSmem {
    int32_t q[32 * kTapsPerLane]; // the segment at lanes S.. : q[kTapsPerLane*S + i]
    union {
        double t[32 * kTapsPerLane];  // step-up rows, indexed like q (a segment of n lanes has room for 8n >= order)
        int32_t out[32 * kSegRow];    // finished samples of the current block, row = segment ordinal
    };
    int32_t in[2][32 * kSegRow];      // residues of the next two blocks, row = segment ordinal
    const int32_t *row_res[32];       // per segment ordinal: its residue row
    void *row_out[32];                //   where its samples go (int16 PCM of its channel, or its residue row)
    int row_mode[32];                 //   0: nothing, 1: PCM, 2: residue row (difference subframe)
};

// warp_coefficients for every segment at once: each segment steps its own order up with its own n lanes
// (k = lane - start), the loop runs to the largest order in the warp.  Same operations in the same order per
// element as warp_coefficients.  Returns this lane's taps kTapsPerLane*k + 1 .. as Q35 words.
__device__ __forceinline__ void segment_coefficients(SegSmem &sm, int start, int k, int n, int order, int order_max,
                                                     uint32_t (&cl)[kTapsPerLane], uint32_t (&ch)[kTapsPerLane])
{
    double *t = sm.t + kTapsPerLane * start;
    const int32_t *q = sm.q + kTapsPerLane * start;
    const bool live = order > 1 && k < n; // order <= 1: a single zero reflection coefficient -> c[1] = 0
    for (int i = 0; i < order_max; i++) {
        if (live && i < order) {
            const double ki = dequantise(i, q[i]);
            const int half = i >> 1;
            for (int j = k; j < half; j += n) {
                double a = t[j];
                double b = t[i - 1 - j];
                t[j] = dadd(a, dmul(ki, b));
                t[i - 1 - j] = dadd(b, dmul(ki, a));
            }
            if (k == 0) {
                if (i & 1) {
                    double mid = t[half];
                    t[half] = dadd(mid, dmul(mid, ki));
                }
                t[i] = ki;
            }
        }
        __syncwarp();
    }
    const double scale = 34359738368.0; // 2^35
#pragma unroll
    for (int m = 0; m < kTapsPerLane; m++) {
        const int j = kTapsPerLane * k + m; // tap j + 1
        const long long v = (live && j < order) ? __double2ll_rz(dmul(scale, -t[j])) : 0;
        cl[m] = (uint32_t)v;
        ch[m] = (uint32_t)((unsigned long long)v >> 32);
    }
    __syncwarp(); // t is dead: its bytes become the output rows
}

struct SegState {
    uint32_t cl[kTapsPerLane];
    uint32_t ch[kTapsPerLane];
    unsigned long long acc[kTapsPerLane];
    uint32_t sp;
    unsigned long long fresh; // what the accumulator of a new output starts from: ~(2^34 + 2^31 * sum_j c[j])
};

// Accumulators before the first product: slot m of lane k is output j = kTapsPerLane*k + m + 1, and it starts with
// what the samples before the subframe contribute in biased form, 2^31 * sum_{j < j' <= order} c[j'] (s[<0] = 0 is
// s' = 2^31).  Every output then carries the bias of every tap.  Every output also starts from
// fresh = ~(2^34 + 2^31 * sum_j c[j]), so that its finished accumulator is a = ~y with y = 2^34 - sum_j c[j]*s[i-j],
// the reference's operand of the rounding shift (mod 2^64).  Then -(int32)(y >> 35) == (int32)(a >> 35) + 1 for every
// 64-bit y, because an arithmetic shift commutes with ~: finishing a sample is a shift-and-add and an add.
__device__ __forceinline__ void segment_state(SegState &st, int k, int n, int src)
{
    unsigned long long tot = 0, loc[kTapsPerLane];
#pragma unroll
    for (int m = kTapsPerLane - 1; m >= 0; m--) {
        loc[m] = tot; // taps above m in this lane
        tot += ((unsigned long long)st.ch[m] << 32) | st.cl[m];
    }
    unsigned long long incl = tot; // sum over lanes k.. of the segment
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long x = __shfl_down_sync(kFull, incl, o);
        if (k + o < n)
            incl += x;
    }
    const unsigned long long above = incl - tot;
    st.fresh = ~((1ull << (kQ - 1)) + (__shfl_sync(kFull, incl, src) << 31));
#pragma unroll
    for (int m = 0; m < kTapsPerLane; m++)
        st.acc[m] = ((above + loc[m]) << 31) + st.fresh;
}

// acc += c * s' mod 2^64, c = ch:cl: one IMAD.WIDE.U32 with the accumulator as addend and one IMAD into its high word.
// Spelled as a carry chain: ptxas fuses mad.lo.cc + madc.hi into that IMAD.WIDE.U32, while it splits mad.wide.u32 with
// a register addend into a product into RZ plus an IADD3 / IADD3.X pair (four instructions per tap instead of two).
__device__ __forceinline__ unsigned long long segment_tap(unsigned long long acc, uint32_t cl, uint32_t ch, uint32_t sp)
{
    unsigned long long d;
    asm("{\n\t.reg .u32 lo, hi;\n\t"
        "mov.b64 {lo, hi}, %4;\n\t"
        "mad.lo.u32 hi, %2, %3, hi;\n\t"
        "mad.lo.cc.u32 lo, %1, %3, lo;\n\t"
        "madc.hi.u32 hi, %1, %3, hi;\n\t"
        "mov.b64 %0, {lo, hi};\n\t}"
        : "=l"(d) : "r"(cl), "r"(ch), "r"(sp), "l"(acc));
    return d;
}

// One block of kSegBlock outputs.  in_row / out_row: this segment's staging rows; src: its first lane.  The staging
// rows of finished samples hold them biased (s' = s ^ kSynthBias), four to a store.
// FIRST: block 0, whose output 0 is s[0] = r[0].
template <bool FIRST>
__device__ __forceinline__ void segment_block(SegState &st, const int32_t *in_row, int32_t *out_row, int src, bool top,
                                              bool first)
{
#pragma unroll
    for (int g = 0; g < kSegBlock; g += 4) {
        const int4 r4 = *reinterpret_cast<const int4 *>(in_row + g);
        const uint32_t r[4] = {(uint32_t)r4.x, (uint32_t)r4.y, (uint32_t)r4.z, (uint32_t)r4.w};
        uint32_t s[4];
#pragma unroll
        for (int h = 0; h < 4; h++) {
            const int e = g + h;
            if (FIRST && e == 0) {
                st.sp = r[0] ^ kSynthBias;
            } else {
                const int u = (e + kTapsPerLane - 1) % kTapsPerLane; // == (t - 1) % kTapsPerLane, static
#pragma unroll
                for (int m = 0; m < kTapsPerLane; m++)
                    st.acc[(m + u) % kTapsPerLane] =
                        segment_tap(st.acc[(m + u) % kTapsPerLane], st.cl[m], st.ch[m], st.sp);
                const unsigned long long done = st.acc[u];
                const unsigned long long incoming = __shfl_down_sync(kFull, done, 1);
                // s' = r - (int32)(y >> 35) + 2^31 = r + (int32)(done >> 35) + 1 + 2^31 (segment_state)
                const uint32_t v = r[h] + (uint32_t)((int32_t)(done >> 32) >> (kQ - 32)) + (1u + kSynthBias);
                st.sp = __shfl_sync(kFull, v, src);
                st.acc[u] = top ? st.fresh : incoming;
            }
            s[h] = st.sp;
        }
        if (first)
            *reinterpret_cast<int4 *>(out_row + g) = make_int4((int)s[0], (int)s[1], (int)s[2], (int)s[3]);
    }
}

// The recurrence of every segment of a warp, called by all 32 lanes once sm.row_res / row_out / row_mode are set for
// every segment ordinal.  This lane is lane k of segment `seg` (of n_seg), n lanes from lane `start`; order is 0 on
// lanes past the last segment, q points at the segment's quantised reflection coefficients.  Row modes: 0 nothing,
// 1 int16 PCM (sample t at row_out + t * stride), 2 int32 row.  Residues arrive kSegBlock at a time per segment
// through cp.async (whole 64-byte pieces of every row, two blocks ahead); finished samples are parked in a staging
// row per segment and leave kSegBlock at a time, a 32-byte or 64-byte run per segment and instruction.
__device__ __forceinline__ void segment_synthesis(SegSmem &sm, int start, int k, int n, int seg, int n_seg, int order,
                                                  const int32_t *q, uint32_t stride)
{
    const int lane = lane_id();
    // residues of block B -> in[B & 1]: eight rows per instruction, four 16-byte pieces per row
    auto fetch = [&](int B) {
        for (int i = lane >> 2; i < n_seg; i += 8) {
            const int32_t *src = sm.row_res[i] + kSegBlock * B + 4 * (lane & 3);
            const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&sm.in[B & 1][i * kSegRow + 4 * (lane & 3)]);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    fetch(0);
    fetch(1);

    // ---- predictors: every segment steps its own order up at once ----
    for (int i = k; i < order; i += n)
        sm.q[kTapsPerLane * start + i] = q[i];
    __syncwarp();
    int order_max = order;
#pragma unroll
    for (int o = 16; o; o >>= 1)
        order_max = max(order_max, __shfl_xor_sync(kFull, order_max, o));
    SegState st;
    segment_coefficients(sm, start, k, n, order, order_max, st.cl, st.ch);
    segment_state(st, k, n, start);

    // ---- recurrence + output ----
    const bool top = k == n - 1, first = k == 0;
    int32_t *out_row = sm.out + seg * kSegRow;
    for (int B = 0; B < kFrame / kSegBlock; B++) {
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncwarp();
        const int32_t *in_row = sm.in[B & 1] + seg * kSegRow;
        if (B == 0)
            segment_block<true>(st, in_row, out_row, start, top, first);
        else
            segment_block<false>(st, in_row, out_row, start, top, first);
        __syncwarp();
        for (int i = lane >> 4; i < n_seg; i += 2) {
            const int mode = sm.row_mode[i];
            const int e = lane & 15, t = kSegBlock * B + e;
            const int v = (int)((uint32_t)sm.out[i * kSegRow + e] ^ kSynthBias);
            if (mode == 1)
                static_cast<int16_t *>(sm.row_out[i])[(size_t)t * stride] = (int16_t)(uint16_t)v;
            else if (mode == 2)
                static_cast<int32_t *>(sm.row_out[i])[t] = v;
        }
        if (B + 2 < kFrame / kSegBlock)
            fetch(B + 2);
        else
            asm volatile("cp.async.commit_group;" ::: "memory");
    }
}

} // namespace selab200
