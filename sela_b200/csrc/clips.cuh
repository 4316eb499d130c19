// clips.cuh -- the clip decode (selab200_container_decode_clips, DESIGN.md 7.8): sample ranges of open containers.
//
// The host selects the (container, frame) pairs a batch of clips covers, sorted and deduplicated, and gives every
// selected subframe a compact descriptor re-based into one word arena plus the device address of its reflection
// words in its container's byte image.  Two kernels of their own; the decode in between is decode_device, unchanged:
//   k_clip_unpack  one warp per selected subframe: both word arrays from any open container (any byte alignment)
//                  into the compact arena (16-byte aligned), as k_container_unpack does for one file in file order;
//   k_clip_gather  one CTA row per piece of a clip: its bytes out of the decoded frames into the output, aligned
//                  16-byte stores fed by funnel-shifted aligned loads, int16 stores only at the two ragged ends.
// Host-resident containers (DESIGN.md 7.10) add k_clip_fetch in front of k_clip_unpack: the selected subframes' bytes
// from mapped host memory into a device staging buffer.
#pragma once

#include "kernels.cuh"

namespace selab200 {

// One selected subframe's word arrays from its container's byte image (src: the device address of its reflection
// words; the residue words follow them after 5 bytes of header) into arena + the descriptor's re-based offsets.
__global__ void __launch_bounds__(256) k_clip_unpack(const unsigned long long *src, const selab200_subframe_desc *descs,
                                                     uint32_t n_sub, uint32_t *arena)
{
    const uint32_t sub = blockIdx.x * 8 + warp_id();
    if (sub >= n_sub)
        return;
    const selab200_subframe_desc d = descs[sub];
    const unsigned long long a = src[sub];
    // get_words_at_byte takes the alignment from its byte offset: address the image from the 16-byte block below
    const uint8_t *base = reinterpret_cast<const uint8_t *>(a & ~15ull);
    const unsigned long long D = a & 15;
    get_words_at_byte(base, D, arena + d.refl_offset, d.refl_words);
    get_words_at_byte(base, D + 4ull * d.refl_words + 5, arena + d.res_offset, d.res_words);
}

// A run of output bytes: `bytes` bytes from decoded-frame byte src to output byte dst (both even).
struct ClipPiece {
    unsigned long long src, dst, bytes;
};

// The 16 bytes at byte phase 4q + 2h of the 32 bytes in w (h: 0 or 1; q uniform across the CTA).
template <int Q>
__device__ __forceinline__ uint4 clip_window(const uint32_t (&w)[8], uint32_t sh)
{
    return make_uint4(__funnelshift_r(w[Q], w[Q + 1], sh), __funnelshift_r(w[Q + 1], w[Q + 2], sh),
                      __funnelshift_r(w[Q + 2], w[Q + 3], sh), __funnelshift_r(w[Q + 3], w[Q + 4], sh));
}

// Piece blockIdx.x; the CTAs of grid row y take every gridDim.y-th 256-block stretch of its aligned body.  Reads at
// most 15 bytes past a piece's last source byte (the decoded-frame buffer is padded).
__global__ void __launch_bounds__(256) k_clip_gather(const uint8_t *frames, uint8_t *out, const ClipPiece *pieces)
{
    const ClipPiece p = pieces[blockIdx.x];
    const unsigned long long d0 = reinterpret_cast<unsigned long long>(out) + p.dst, d1 = d0 + p.bytes;
    const unsigned long long s0 = reinterpret_cast<unsigned long long>(frames) + p.src;
    const unsigned long long a0 = (d0 + 15) & ~15ull, a1 = d1 & ~15ull; // the aligned body [a0, a1) (empty if a1 <= a0)
    const unsigned long long off = s0 - d0;                                // source address = destination + off
    if (blockIdx.y == 0 && threadIdx.x < 16) { // ragged ends: up to 7 samples in front of the body, 7 behind it
        const unsigned long long x = threadIdx.x < 8 ? d0 + 2 * threadIdx.x : (a1 > a0 ? a1 : a0) + 2 * (threadIdx.x - 8);
        const bool mine = threadIdx.x < 8 ? x < a0 && x < d1 : x < d1 && x >= a0;
        if (mine)
            *reinterpret_cast<int16_t *>(x) = *reinterpret_cast<const int16_t *>(x + off);
    }
    if (a1 <= a0)
        return;
    const unsigned long long n_blocks = (a1 - a0) >> 4;
    const uint32_t phase = (uint32_t)(off & 15), q = phase >> 2, sh = 8 * (phase & 3);
    for (unsigned long long b = (unsigned long long)blockIdx.y * blockDim.x + threadIdx.x; b < n_blocks;
         b += (unsigned long long)gridDim.y * blockDim.x) {
        const unsigned long long x = a0 + 16 * b;
        const uint4 *s = reinterpret_cast<const uint4 *>((x + off) & ~15ull);
        uint4 v = __ldg(s);
        if (phase) {
            const uint4 u = __ldg(s + 1);
            const uint32_t w[8] = {v.x, v.y, v.z, v.w, u.x, u.y, u.z, u.w};
            switch (q) {
            case 0: v = clip_window<0>(w, sh); break;
            case 1: v = clip_window<1>(w, sh); break;
            case 2: v = clip_window<2>(w, sh); break;
            default: v = clip_window<3>(w, sh); break;
            }
        }
        *reinterpret_cast<uint4 *>(x) = v;
    }
}

// ---- channel-selecting clip decode (selab200_container_decode_clips_select, DESIGN.md 7.9) ----
//
// The needed subframes are decoded as mono frames, one [2048] int16 row each.  A row-table entry names the row of
// one selected channel in a frame and, for a difference-coded channel, the row of its parent (else kNoParentRow).

constexpr uint32_t kNoParentRow = 0xffffffffu;
constexpr uint32_t kSelectTileBytes = 16384; // output bytes staged per pass of k_clip_gather_select

// Samples [t0, t0 + count) of one frame of one clip (count <= 2048), written from output byte dst on.
struct SelectPiece {
    unsigned long long dst;
    uint32_t rows;     // row-table index of the first selected channel of the frame
    uint32_t n;        // selected channels: the mean's divisor, else the output channels
    uint32_t t0, count;
};

// Sample t of a table entry: the row's, or (uint16)(parent - difference) as k_diff_fixup computes it.
__device__ __forceinline__ int16_t select_sample(const int16_t *rows, uint2 e, uint32_t t)
{
    const int16_t v = __ldg(rows + (size_t)e.x * kFrame + t);
    if (e.y == kNoParentRow)
        return v;
    return (int16_t)(uint16_t)((uint32_t)__ldg(rows + (size_t)e.y * kFrame + t) - (uint32_t)v);
}

// Piece blockIdx.x.  Per pass a tile of whole samples [samples][n_out] is staged in shared memory at the 16-byte
// phase of its destination, reading every row along its samples; then it goes out as aligned 16-byte stores, with
// OUT-wide stores only at the tile's ragged ends.  OUT is int16_t or float (x / 32768, exact); MEAN (float) writes
// one value per sample, the exact integer sum over the n channels divided by 32768 n, rounded to nearest.
template <typename OUT, bool MEAN>
__global__ void __launch_bounds__(256) k_clip_gather_select(const int16_t *rows, const uint2 *table, uint8_t *out,
                                                            const SelectPiece *pieces)
{
    __shared__ __align__(16) uint8_t tile[kSelectTileBytes + 16];
    const SelectPiece p = pieces[blockIdx.x];
    const uint32_t n_out = MEAN ? 1 : p.n, sample_bytes = n_out * (uint32_t)sizeof(OUT);
    const uint32_t per = kSelectTileBytes / sample_bytes; // samples per pass
    const uint2 *e = table + p.rows;
    for (uint32_t s0 = 0; s0 < p.count; s0 += per) {
        const uint32_t ns = min(per, p.count - s0);
        const unsigned long long d0 = reinterpret_cast<unsigned long long>(out) + p.dst + (unsigned long long)s0 * sample_bytes;
        const unsigned long long d1 = d0 + (unsigned long long)ns * sample_bytes, base = d0 & ~15ull;
        OUT *t = reinterpret_cast<OUT *>(tile + (d0 & 15));
        for (uint32_t k = threadIdx.x; k < ns; k += blockDim.x) {
            const uint32_t at = p.t0 + s0 + k;
            if (MEAN) {
                int32_t S = 0;
                for (uint32_t j = 0; j < p.n; j++)
                    S += select_sample(rows, e[j], at);
                t[k] = __fdiv_rn((float)S, (float)(32768 * p.n));
            } else {
                for (uint32_t j = 0; j < n_out; j++) {
                    const int16_t v = select_sample(rows, e[j], at);
                    if constexpr (sizeof(OUT) == 2)
                        t[k * n_out + j] = v;
                    else
                        t[k * n_out + j] = (float)v * (1.0f / 32768);
                }
            }
        }
        __syncthreads();
        const unsigned long long a0 = (d0 + 15) & ~15ull, a1 = d1 & ~15ull; // the aligned body [a0, a1)
        for (unsigned long long x = a0 + 16ull * threadIdx.x; x < a1; x += 16ull * blockDim.x)
            *reinterpret_cast<uint4 *>(x) = *reinterpret_cast<const uint4 *>(tile + (x - base));
        if (threadIdx.x < 32) { // ragged ends: fewer than 16 bytes in front of the body and behind it
            const unsigned long long x = threadIdx.x < 16 ? d0 + sizeof(OUT) * threadIdx.x
                                                          : (a1 > a0 ? a1 : a0) + sizeof(OUT) * (threadIdx.x - 16);
            const bool mine = threadIdx.x < 16 ? x < a0 && x < d1 : x < d1 && x >= a0;
            if (mine)
                *reinterpret_cast<OUT *>(x) = *reinterpret_cast<const OUT *>(tile + (x - base));
        }
        __syncthreads();
    }
}

// ---- host-resident images (selab200_container_open_host, DESIGN.md 7.10) ----
//
// A host-resident container keeps its byte image in mapped, page-locked host memory.  Per group the host merges the
// byte ranges of the selected subframes into runs, 16-byte aligned at both ends, and k_clip_fetch copies each run
// over PCIe into a device staging buffer at a 16-byte aligned offset, so every subframe keeps its 16-byte phase and
// k_clip_unpack reads it from the staging buffer unchanged.

// A run: `bytes` bytes (a multiple of 16) from the mapped image address src to the staging address dst (both
// 16-byte aligned).
struct FetchRun {
    unsigned long long src, dst, bytes;
};

constexpr uint32_t kFetchLoads = 8; // independent 16-byte loads each thread has in flight before its first store
// CTAs per k_clip_fetch launch.  Mapped reads reach about 22 GB/s from 16 CTAs on up (H100 SXM, 700 W); more CTAs
// only take SMs from the decode of earlier chunks (DESIGN.md 7.10).
constexpr uint32_t kFetchCtas = 32;

// Runs blockIdx.x, blockIdx.x + gridDim.x, ...; the CTAs of grid row y take every gridDim.y-th stretch of
// kFetchLoads * 256 16-byte blocks of a run.  A read of mapped memory crosses PCIe and takes microseconds, so each
// thread issues all kFetchLoads loads of a stretch (each warp's coalesced into 512 contiguous bytes) before it stores
// any.  The grid is small: a CTA spends its time waiting on PCIe, and the decode kernels of earlier chunks need the SMs.
__global__ void __launch_bounds__(256) k_clip_fetch(const FetchRun *runs, uint32_t n_runs)
{
    for (uint32_t i = blockIdx.x; i < n_runs; i += gridDim.x) {
        const FetchRun r = runs[i];
        const uint4 *s = reinterpret_cast<const uint4 *>(r.src);
        uint4 *d = reinterpret_cast<uint4 *>(r.dst);
        const unsigned long long n = r.bytes >> 4, stretch = (unsigned long long)kFetchLoads * blockDim.x;
        for (unsigned long long b0 = blockIdx.y * stretch + threadIdx.x; b0 < n; b0 += gridDim.y * stretch) {
            uint4 v[kFetchLoads];
#pragma unroll
            for (uint32_t k = 0; k < kFetchLoads; k++)
                if (b0 + k * blockDim.x < n)
                    v[k] = __ldg(s + b0 + k * blockDim.x);
#pragma unroll
            for (uint32_t k = 0; k < kFetchLoads; k++)
                if (b0 + k * blockDim.x < n)
                    d[b0 + k * blockDim.x] = v[k];
        }
    }
}

} // namespace selab200
