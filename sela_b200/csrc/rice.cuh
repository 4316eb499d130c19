// rice.cuh -- Golomb-Rice coding (kernels K4 / K5 of SURVEY.md 2).
//
// Bit layout (src/rice/rice_encoder.cpp:35-71): stream bit b lives in word b/32 at
// bit b%32 (LSB first); a symbol is u>>k ones, one zero, then the k low bits of u
// MSB FIRST; the last word is zero padded.  u is the zig-zag of the int32 input.
#pragma once

#include "common.cuh"

namespace selab200 {

// convertSignedToUnsigned (rice_encoder.cpp:12-18), 32-bit domain
__device__ __forceinline__ uint32_t zigzag(int32_t v)
{
    return ((uint32_t)v << 1) ^ (uint32_t)(v >> 31);
}
// convertUnsignedToSigned (src/rice/rice_decoder.cpp:46-52)
__device__ __forceinline__ int32_t unzigzag(uint32_t u)
{
    return (int32_t)(u >> 1) ^ -(int32_t)(u & 1);
}

struct RiceChoice {
    uint32_t k;
    uint32_t bits;    // requiredBits (saturated at 0xffffffff)
    uint32_t words;   // ceil(bits / 32)
    uint32_t my_bits; // code length at k of THIS lane's values (rice_lane_range), mod 2^32
};

// The values a lane owns, in the parameter search and in the packer alike: `per` consecutive
// values [lo, hi), per a multiple of 4, so that every lane's range of a 16-byte aligned row starts
// on a 16-byte boundary and is read as int4.  Rows must therefore be 16-byte aligned and readable
// up to the next multiple of 4 values; the values past n are never coded.
__device__ __forceinline__ void rice_lane_range(int n, int &lo, int &hi)
{
    const int per = (((n + 31) >> 5) + 3) & ~3;
    const int first = lane_id() * per;
    lo = first < n ? first : n;
    hi = lo + per < n ? lo + per : n;
}

// calculateOptimumRiceParam (rice_encoder.cpp:20-33): first arg-min over k = 0..19 of
// sum(u >> k) + n*(1 + k).  vals: n <= 2048 int32 inputs (see rice_lane_range).
// Every lane returns the same k, bits and words, and its own my_bits.
//
// The 20 sums are not accumulated one by one.  With S_k = sum_i (u_i >> k) and C_k the
// number of inputs whose bit k is set,  S_k = 2*S_{k+1} + C_k  exactly, so S_19 plus
// the 19 bit counts suffice.  The counts come from a bit-sliced (Harley-Seal) vertical
// counter: each lane folds its own range (at most 64 values) into 7 planes with carry-save
// adders (about two LOP3 per word instead of forty shift+adds), and a ballot per (plane, bit)
// finishes the cross-lane sum; the totals do not depend on how the values are split.  Unrolled
// over k, the recursion gives the lane's own share at the chosen k from its own planes, so the
// packer needs no counting pass:  sum_own (u >> k) = (sum_own u >> 19) << (19 - k) + sum_p 2^p (plane_p >> k).
__device__ __forceinline__ void csa(uint32_t &hi, uint32_t &lo, uint32_t a, uint32_t b, uint32_t c)
{
    const uint32_t u = a ^ b;
    hi = (a & b) | (u & c);
    lo = u ^ c;
}

// vals: generic pointer (shared or global memory).  Deliberately NOT inlined and written as
// compact loops: the encoder kernel is instruction-fetch bound (81 KB of code, 16 warps in
// different phases per SM), so straight-line code that runs once costs more in I-cache misses
// than it saves in issue slots.
__device__ __noinline__ RiceChoice warp_rice_choose(const int32_t *vals, int n)
{
    int lo, hi;
    rice_lane_range(n, lo, hi);
    // bit planes of weight 1, 2, 4, 8 (carry-save side) and 16, 32, 64 (ripple side)
    uint32_t ones = 0, twos = 0, fours = 0, eights = 0, p16 = 0, p32 = 0, p64 = 0;
    unsigned long long top = 0; // sum of u >> 19
#pragma unroll 1
    for (int b0 = lo; b0 < hi; b0 += 16) {
        uint32_t w[16];
#pragma unroll
        for (int v = 0; v < 4; v++) {
            const int i = b0 + 4 * v;
            const int4 x = i < hi ? *reinterpret_cast<const int4 *>(vals + i) : make_int4(0, 0, 0, 0);
            const int32_t e[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const uint32_t u = i + c < hi ? zigzag(e[c]) : 0u;
                top += u >> (kMaxRice - 1);
                w[4 * v + c] = u & ((1u << (kMaxRice - 1)) - 1);
            }
        }
        uint32_t e8[2];
#pragma unroll
        for (int b = 0; b < 2; b++) {
            uint32_t f4[2];
#pragma unroll
            for (int c = 0; c < 2; c++) {
                const int t = b * 8 + c * 4;
                uint32_t ta, tb;
                csa(ta, ones, ones, w[t], w[t + 1]);
                csa(tb, ones, ones, w[t + 2], w[t + 3]);
                csa(f4[c], twos, twos, ta, tb);
            }
            csa(e8[b], fours, fours, f4[0], f4[1]);
        }
        uint32_t c16;
        csa(c16, eights, eights, e8[0], e8[1]);
        const uint32_t c32 = p16 & c16; // ripple the weight-16 carry into the upper planes
        p16 ^= c16;
        const uint32_t c64 = p32 & c32;
        p32 ^= c32;
        p64 ^= c64;
    }
    const uint32_t planes[7] = {ones, twos, fours, eights, p16, p32, p64};
    unsigned long long s_k = warp_sum_u64(top);                            // S_19
    unsigned long long best = s_k + (unsigned long long)n * kMaxRice;      // k = 19
    uint32_t best_k = kMaxRice - 1;
#pragma unroll 1
    for (int k = kMaxRice - 2; k >= 0; k--) {
        uint32_t count = 0;
#pragma unroll
        for (int p = 0; p < 7; p++)
            count += (uint32_t)__popc(__ballot_sync(kFull, (planes[p] >> k) & 1u)) << p;
        s_k = 2 * s_k + count;
        const unsigned long long total = s_k + (unsigned long long)n * (1 + k);
        if (total <= best) { // descending k with <= keeps the FIRST (lowest) arg-min
            best = total;
            best_k = k;
        }
    }
    RiceChoice c;
    c.k = best_k;
    c.bits = best > 0xffffffffull ? 0xffffffffu : (uint32_t)best;
    const unsigned long long wds = (best + 31) >> 5;
    c.words = wds > 0xffffffffull ? 0xffffffffu : (uint32_t)wds;
    unsigned long long mine = (top << (kMaxRice - 1 - best_k)) + (unsigned long long)(hi - lo) * (1 + best_k);
#pragma unroll
    for (int p = 0; p < 7; p++)
        mine += (unsigned long long)(planes[p] >> best_k) << p;
    c.my_bits = (uint32_t)mine;
    return c;
}

// generateEncodedBits + writeInts (rice_encoder.cpp:35-71).  Lane l codes its range of
// rice_lane_range; a warp prefix sum of the lanes' code lengths (c.my_bits, from
// warp_rice_choose) gives each lane its first bit.  Words wholly inside a lane's range are
// plain stores; the (at most two) words it shares with a neighbour are OR-ed into the
// pre-zeroed destination.  dst: `c.words` uint32 in global memory.
// Values arrive as int4, loaded one vector (four symbols) ahead of the symbol that codes
// them, so no load sits on the symbol-to-symbol chain.  A symbol is emitted as pieces of at
// most 32 bits (runs of ones, then "0 + payload") through ONE staging/flush site -- compact
// code, see warp_rice_choose.
__device__ __noinline__ void warp_rice_pack(const int32_t *vals, int n, const RiceChoice c, uint32_t *dst)
{
    const int lane = lane_id();
    for (uint32_t w = lane; w < c.words; w += 32)
        dst[w] = 0;
    __syncwarp();

    int lo, hi;
    rice_lane_range(n, lo, hi);
    const uint32_t k = c.k;
    const uint32_t end = warp_scan_inclusive_u32(c.my_bits);
    const uint32_t start = end - c.my_bits;

    // 64-bit staging: bits [0, fill) of `stage` are pending for word index `widx`; fill < 32
    unsigned long long stage = 0;
    uint32_t fill = start & 31;
    uint32_t widx = start >> 5;
    const int4 *src = reinterpret_cast<const int4 *>(vals + lo);
    int4 next = lo < hi ? src[0] : make_int4(0, 0, 0, 0);
    for (int i = lo; i < hi; i += 4) {
        int4 cur = next;
        if (i + 4 < hi)
            next = src[((i - lo) >> 2) + 1];
        const int m = hi - i < 4 ? hi - i : 4;
#pragma unroll 1
        for (int e = 0; e < m; e++) {
            const uint32_t u = zigzag(cur.x);
            cur.x = cur.y;
            cur.y = cur.z;
            cur.z = cur.w;
            uint32_t ones = u >> k;
            // "0 then the k payload bits MSB first" == bit-reversed low k bits, LSB first, after a zero
            const uint32_t tail = (k ? (__brev(u) >> (32 - k)) : 0u) << 1;
            // Common case: the whole symbol (ones, the zero, the payload) fits one 32-bit piece.
            // Otherwise the run of ones goes out 32 at a time and the rest follows.
            bool last;
            do {
                uint32_t bits, len;
                if (ones + 1 + k <= 32) {
                    bits = (tail << ones) | ((1u << ones) - 1);
                    len = ones + 1 + k;
                    last = true;
                } else if (ones >= 32) {
                    bits = 0xffffffffu;
                    len = 32;
                    ones -= 32;
                    last = false;
                } else {
                    bits = (1u << ones) - 1;
                    len = ones;
                    ones = 0;
                    last = false;
                }
                stage |= (unsigned long long)bits << fill;
                fill += len;
                if (fill >= 32) {
                    const uint32_t value = (uint32_t)stage;
                    const uint32_t b0 = widx << 5;
                    if (b0 >= start && b0 + 32 <= end)
                        dst[widx] = value;
                    else if (value)
                        atomicOr(&dst[widx], value);
                    widx++;
                    stage >>= 32;
                    fill -= 32;
                }
            } while (!last);
        }
    }
    if (fill && hi > lo) {
        const uint32_t value = (uint32_t)stage;
        if (value)
            atomicOr(&dst[widx], value);
    }
    __syncwarp();
}

// rice::RiceDecoder (src/rice/rice_decoder.cpp:11-52), ONE LANE PER STREAM: the parse
// is inherently sequential, so the parallelism is across streams (subframes); the 32
// lanes of a warp run the same branch-free scalar parser on 32 different streams.
//
// Words reach the parser through a per-warp shared-memory ring, ring[w & (RING-1)][lane]
// (bank = lane for every access, so neither the parser's reads nor the refill's writes
// ever conflict).  Each lane keeps its own ring topped up with 16-byte loads from its own
// stream (aligned down; the words in front of the stream are skipped, words past its end
// read as zero -- bounded, unlike the reference), issued one batch ahead of use.
// The parser runs in symbol lockstep (see below): step n decodes symbol n of every lane, the
// common case from a single 32-bit window; ring refills happen at batch boundaries only.
// Margins: a fast step consumes at most one word and looks one ahead, the general parser tops the
// ring up itself; loads issued at one boundary are committed at the next, so 3 + 4*BATCH committed
// words ahead of a lane at every boundary is ample -- the top-up keeps about RING, and a lane
// that still falls short refills on the spot.
struct RiceLaneStream {
    const uint32_t *src;
    uint32_t n_words, k, count;
    int32_t *out;
};

// A lane's view of its stream and ring.  rb = ring + lane; vector v of vp holds words
// [4v, 4v+4) counted from the 16-byte aligned base; words >= total read as zero.
struct RiceRingView {
    uint32_t *rb;
    const uint4 *vp;
    uint32_t nvec, total;
};
template <int RING>
__device__ __forceinline__ uint4 ring_fetch(const RiceRingView &rv, uint32_t w) // words [w, w+4), w % 4 == 0
{
    return (w >> 2) < rv.nvec ? __ldg(rv.vp + (w >> 2)) : make_uint4(0, 0, 0, 0);
}
template <int RING>
__device__ __forceinline__ void ring_commit(const RiceRingView &rv, uint32_t w, const uint4 v)
{
    const uint32_t r = (w & (RING - 1)) * 32;
    const uint32_t x = w + 0 < rv.total ? v.x : 0u; // words past the stream's end read as zero
    rv.rb[r] = x;
    rv.rb[r + 32] = w + 1 < rv.total ? v.y : 0u;
    rv.rb[r + 64] = w + 2 < rv.total ? v.z : 0u;
    rv.rb[r + 96] = w + 3 < rv.total ? v.w : 0u;
    if (r == 0)
        rv.rb[RING * 32] = x; // mirror row: word w+1 is always one row below word w
}
template <int RING>
__device__ __forceinline__ uint32_t ring_window(const uint32_t *rb, uint32_t at)
{
    const uint32_t r = ((at >> 5) & (RING - 1)) * 32;
    return __funnelshift_r(rb[r], rb[r + 32], at);
}

// General parser for ONE symbol of any length starting at bit `pos` (the fast path handles symbols
// that fit a 32-bit window).  Tops the ring up synchronously as it goes and leaves `ahead` committed
// words in front of the new position.  Out of line on purpose: it runs for a handful of symbols per
// stream at most, and eight inlined copies would quadruple the kernel.  Returns {u, pos, committed}.
template <int RING>
__device__ __noinline__ uint4 rice_slow_symbol(uint32_t *rb, const uint4 *vp, uint32_t nvec, uint32_t total,
                                               uint32_t pos, uint32_t committed, uint32_t k, uint32_t ahead)
{
    const RiceRingView rv{rb, vp, nvec, total};
    auto ensure = [&](uint32_t words_ahead) {
        while (committed < (pos >> 5) + words_ahead) {
            ring_commit<RING>(rv, committed, ring_fetch<RING>(rv, committed));
            committed += 4;
        }
    };
    uint32_t q = 0;
    while (true) {
        ensure(3);
        const uint32_t ones = __clz(__brev(~ring_window<RING>(rb, pos))); // 32: no terminator in this window
        q += ones;
        if (ones < 32) {
            pos += ones + 1;
            break;
        }
        pos += 32;
        if (pos > total * 32u + 64) // ran off the stream; words past the end read as zero, so the loop
            break;                  // would end by itself one window later -- belt and braces
    }
    ensure(3);
    const uint32_t payload = (__brev(ring_window<RING>(rb, pos)) >> 1) >> (31 - k);
    pos += k;
    ensure(ahead); // the fast steps that follow in this batch read ahead of pos without checking
    return make_uint4((q << k) | payload, pos, committed, 0u); // uint32 shift as in rice_decoder.cpp:37
}

// Returns (per lane) false if the stream needed more bits than n_words holds.
template <int RING, int BATCH>
__device__ bool warp_rice_decode32(uint32_t *ring, const RiceLaneStream st)
{
    constexpr uint32_t kNeed = 3 + 4 * BATCH; // committed words a lane must have ahead at a boundary
    static_assert(kNeed + 8 <= RING && (RING & (RING - 1)) == 0 && RING % 32 == 0, "ring too small for the batch");
    uint32_t *rb = ring + lane_id();
    // 16-byte view of the stream: vector v holds words [4v, 4v+4) counted from the aligned base
    const uintptr_t addr = reinterpret_cast<uintptr_t>(st.src);
    const uint32_t skip = (uint32_t)(addr >> 2) & 3u;
    const uint4 *vp = reinterpret_cast<const uint4 *>(addr & ~(uintptr_t)15);
    const uint32_t total = st.n_words ? st.n_words + skip : 0; // words from the aligned base
    const uint32_t nvec = (total + 3) >> 2;

    const RiceRingView rv{rb, vp, nvec, total};
    // fetch only ISSUES the load; nothing touches the value until commit, a batch later
    auto fetch = [&](uint32_t w) -> uint4 { return ring_fetch<RING>(rv, w); };
    auto commit = [&](uint32_t w, const uint4 v) { ring_commit<RING>(rv, w, v); };
    uint32_t loaded = 0;    // words [.., loaded) have been requested
    uint32_t committed = 0; // words [.., committed) are in the ring
    for (; loaded < RING; loaded += 32) { // initial fill, eight loads in flight at a time
        uint4 f[8];
#pragma unroll
        for (int t = 0; t < 8; t++)
            f[t] = fetch(loaded + 4 * t);
#pragma unroll
        for (int t = 0; t < 8; t++)
            commit(loaded + 4 * t, f[t]);
    }
    committed = loaded;

    // ---- symbol-lockstep parser --------------------------------------------------------------
    // Step n decodes symbol n of EVERY lane's stream, so the output index, the store schedule and
    // the loop bound are warp-uniform and only `pos` (and the ring fill) are per-lane state.
    // Fast path: the whole symbol (ones, terminator, k payload bits) lies inside ONE 32-bit window
    //     pos -> LDS pair -> funnel shift -> brev -> clz -> pos'
    // with the payload cut from the same window.  A lane whose symbol is longer than the window
    // (a unary run of 32 - k ones or more: rare) flags the step; if any lane did, those lanes redo
    // the symbol with the general, refilling parser under a (divergent) branch.
    uint32_t pos = skip * 32;
    const uint32_t k = st.k, count = st.count;
    const uint32_t kshift = 31 - k; // payload = (t >> 1) >> (31 - k), valid for k = 0 too
    uint32_t max_count = count;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const uint32_t other = __shfl_xor_sync(kFull, max_count, o);
        max_count = other > max_count ? other : max_count;
    }
    const bool vec_out = (reinterpret_cast<uintptr_t>(st.out) & 15) == 0;
    uint4 pend0 = make_uint4(0, 0, 0, 0), pend1 = pend0;
    uint32_t n_pend = 0; // per lane: 0, 1 or 2 vectors in flight, for words [committed, committed + 4*n_pend)
    auto window = [&](uint32_t at) -> uint32_t { return ring_window<RING>(rb, at); };
    auto slow_symbol = [&]() -> uint32_t {
        if (n_pend > 0) // the general parser commits on its own: retire what is in flight first
            commit(committed, pend0);
        if (n_pend > 1)
            commit(committed + 4, pend1);
        committed += 4 * n_pend;
        n_pend = 0;
        const uint4 r = rice_slow_symbol<RING>(rb, vp, nvec, total, pos, committed, k, kNeed);
        pos = r.y;
        committed = r.z;
        loaded = loaded > committed ? loaded : committed;
        return r.x;
    };

    for (uint32_t n = 0; n < max_count; n += BATCH) {
        // ---- batch boundary (per lane, predicated) ----
        const bool live = n < count;
        if (n_pend > 0)
            commit(committed, pend0);
        if (n_pend > 1)
            commit(committed + 4, pend1);
        committed += 4 * n_pend;
        n_pend = 0;
        const uint32_t wi = pos >> 5;
        while (live && committed < wi + kNeed) { // rare: this lane outran its top-up
            commit(committed, fetch(committed));
            committed += 4;
            loaded = committed;
        }
        if (live && loaded + 4 <= wi + RING) { // room for one more vector without touching unread words
            pend0 = fetch(loaded);
            loaded += 4;
            n_pend = 1;
            if (loaded + 4 <= wi + RING) {
                pend1 = fetch(loaded);
                loaded += 4;
                n_pend = 2;
            }
        }
        // ---- BATCH symbols ----
        int32_t v[BATCH];
#pragma unroll
        for (int e = 0; e < BATCH; e++) {
            const bool active = n + e < count;
            const uint32_t b = __brev(window(pos));
            const uint32_t ones = __clz(~b);        // trailing ones of the window (32: all ones)
            const uint32_t len = ones + 1 + k;
            const bool need_slow = active && len > 32;
            const uint32_t t = __funnelshift_lc(0u, b, ones + 1); // b << (ones + 1), 0 for a shift of 32
            uint32_t u = (ones << k) | ((t >> 1) >> kshift);
            if (__any_sync(kFull, need_slow)) {
                if (need_slow)
                    u = slow_symbol();
                else if (active)
                    pos += len;
            } else if (active) {
                pos += len;
            }
            v[e] = unzigzag(u);
        }
        // ---- stores: symbols n .. n+BATCH-1 of this lane's row ----
        if (n + BATCH <= count && vec_out) {
#pragma unroll
            for (int e = 0; e < BATCH; e += 4)
                *reinterpret_cast<int4 *>(st.out + n + e) = make_int4(v[e], v[e + 1], v[e + 2], v[e + 3]);
        } else {
#pragma unroll
            for (int e = 0; e < BATCH; e++)
                if (n + e < count)
                    st.out[n + e] = v[e];
        }
    }
    // nothing to decode is never an overrun (a stream of zero words starts `skip` words into its first vector)
    return count == 0 || pos <= total * 32u;
}

} // namespace selab200
