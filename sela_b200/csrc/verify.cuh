// verify.cuh -- the kernels of the verify path (sm_90a): decoded PCM against its source.
//
//   k_verify_compare      CTA per frame: per (frame, channel) the first differing sample, the count and the
//                         delta there, plus a device-wide count of differing pairs
//   k_verify_guard_descs  the encoder's descriptors of a chunk, or empty ones once the encoder has failed
//                         (encode_container_verified unpacks and decodes only what the encoder really wrote)
//
// The decode before the compare is the ordinary decoder (k_container_unpack, the Rice kernels, synthesis).
#pragma once

#include "kernels.cuh"

namespace selab200 {

constexpr int kVerifyThreads = 256;
constexpr int kVerifyUnroll = 4; // 16-byte vectors of each input a thread has in flight

// The samples of one differing 16-byte piece (8 interleaved samples starting at sample 8v of the frame).
// Sample s of the frame belongs to channel s % C, position s / C.  The first difference of a channel is
// kept as one key, position << 17 | (delta + 65535), so that a single atomicMin finds it together with
// its delta (|delta| <= 65535 for int16 samples).
__device__ __noinline__ void verify_piece(int4 x, int4 y, uint32_t v, uint32_t channels, uint32_t *count,
                                          uint32_t *key)
{
    const uint32_t xs[4] = {(uint32_t)x.x, (uint32_t)x.y, (uint32_t)x.z, (uint32_t)x.w};
    const uint32_t ys[4] = {(uint32_t)y.x, (uint32_t)y.y, (uint32_t)y.z, (uint32_t)y.w};
#pragma unroll
    for (int w = 0; w < 4; w++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int a = (int16_t)(xs[w] >> (16 * h)), b = (int16_t)(ys[w] >> (16 * h));
            if (a != b) {
                const uint32_t s = 8 * v + 2 * w + h, c = s % channels;
                atomicAdd(&count[c], 1u);
                atomicMin(&key[c], ((s / channels) << 17) | (uint32_t)(a - b + 65535));
            }
        }
}

// decoded, source: interleaved int16, n_frames frames of 2048 * C samples, both 16-byte aligned (a frame is
// 4096 * C bytes, so every frame is).  entries[f * C + c] receives the record of a differing pair (frame =
// frame_base + f) and is left untouched otherwise; *n_differing counts the differing pairs.  Nothing is
// compared once *status reports a decode error: the decoded samples are not defined then.
__global__ void __launch_bounds__(kVerifyThreads) k_verify_compare(const int16_t *decoded, const int16_t *source,
                                                                   uint32_t channels, uint32_t frame_base,
                                                                   const int32_t *status,
                                                                   selab200_verify_entry *entries,
                                                                   unsigned long long *n_differing)
{
    __shared__ uint32_t s_count[SELAB200_MAX_CHANNELS], s_key[SELAB200_MAX_CHANNELS];
    if (*status != 0)
        return;
    if (threadIdx.x < SELAB200_MAX_CHANNELS) {
        s_count[threadIdx.x] = 0;
        s_key[threadIdx.x] = 0xffffffffu;
    }
    __syncthreads();
    const uint32_t f = blockIdx.x;
    const uint32_t vecs = channels * (kFrame / 8);
    const int4 *a = reinterpret_cast<const int4 *>(decoded) + (size_t)f * vecs;
    const int4 *b = reinterpret_cast<const int4 *>(source) + (size_t)f * vecs;
    for (uint32_t v0 = threadIdx.x; v0 < vecs; v0 += kVerifyUnroll * kVerifyThreads) {
        int4 x[kVerifyUnroll], y[kVerifyUnroll];
#pragma unroll
        for (int j = 0; j < kVerifyUnroll; j++) {
            const uint32_t v = v0 + j * kVerifyThreads;
            x[j] = y[j] = make_int4(0, 0, 0, 0);
            if (v < vecs) {
                x[j] = __ldcs(a + v);
                y[j] = __ldcs(b + v);
            }
        }
#pragma unroll
        for (int j = 0; j < kVerifyUnroll; j++)
            if (((x[j].x ^ y[j].x) | (x[j].y ^ y[j].y) | (x[j].z ^ y[j].z) | (x[j].w ^ y[j].w)) != 0)
                verify_piece(x[j], y[j], v0 + j * kVerifyThreads, channels, s_count, s_key);
    }
    __syncthreads();
    const uint32_t c = threadIdx.x;
    if (c < channels && s_count[c] != 0) {
        selab200_verify_entry e;
        e.frame = frame_base + f;
        e.channel = (uint16_t)c;
        e.first_sample = (uint16_t)(s_key[c] >> 17);
        e.n_differing = s_count[c];
        e.first_delta = (int32_t)(s_key[c] & 0x1ffffu) - 65535;
        entries[(size_t)f * channels + c] = e;
        atomicAdd(n_differing, 1ull);
    }
}

// out[i] = descs[i] while *status is 0; otherwise an all-zero descriptor (no words, rejected by the decoder).
__global__ void __launch_bounds__(256) k_verify_guard_descs(const selab200_subframe_desc *descs, uint32_t n,
                                                            const int32_t *status, selab200_subframe_desc *out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    selab200_subframe_desc d = descs[i];
    if (*reinterpret_cast<const volatile int32_t *>(status) != 0)
        memset(&d, 0, sizeof d);
    out[i] = d;
}

} // namespace selab200
