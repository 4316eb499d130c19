// search.cuh -- the kernels of the order search (sm_90a, DESIGN.md 7.3): every unit is coded at the predictor order
// 1..100 with the fewest words whose FIR has no tie, inside the format.
//
//   k_search_units<S, T, FORCE>  the ordinary analysis kernel (encode_unit<kUnitSearch>): codes the unit at the
//                              reference order into its slot, and leaves all 100 q, the reference order and its words
//                              in the unit's SearchUnit
//   k_search_candidates<S, T>  warp per (unit, slice of orders): carries one step-up forward through the slice's
//                              orders; per order the FIR with the tie check and both Rice sizes; a tie-free order
//                              enters the unit's atomicMin key
//   k_search_repack<S>         warp per unit whose winner is not the reference order: the winner packed into the
//                              unit's slot, record rewritten
//   k_search_ref_words         thread per frame: the words the reference encoder's choice takes (its orders, its
//                              stereo decision), summed into one counter
// Then k_encode_sizes / k_encode_scan / k_encode_gather(_container) run as for every encode, and the stereo decision
// there sees the searched sizes.  The candidate and repack kernels have grids of a fixed size and loop over the work.
// T (tests only, selab200_encode_search_trace): the tracing instantiations, which also write the record of every
// (unit, order) to a trace buffer.
#pragma once

#include "kernels.cuh"

namespace selab200 {

// The orders 1..100 in slices of about equal work, one warp per (unit, slice).  An order costs its FIR k-steps
// ((order + 8) / 32 rounded up: 1 up to order 24, then 2, 3, 4) and two Rice sizings, which cost about a k-step
// together; a slice also repeats the step-up of the orders below it, which is small beside these.
constexpr int kSearchSlices = 4;
__host__ __device__ constexpr int search_slice_first(int s) // first order of slice s; s = kSearchSlices: 101
{
    return s == 0 ? 1 : s == 1 ? 41 : s == 2 ? 65 : s == 3 ? 85 : kMaxOrder + 1;
}

// Shared memory of a search warp: the signal as stage_unit stages it, the step-up row, the predictor and the FIR's
// digit planes.
constexpr size_t kSearchStepBytes = 104 * sizeof(double);
template <bool STEREO>
constexpr size_t search_smem_bytes()
{
    return unit_signal_bytes<STEREO>() + kSearchStepBytes + sizeof(CoefSmem) + kPlaneBytes;
}

// One iteration i of the step-up of warp_coefficients (the same operations in the same order): afterwards t[0..i]
// is the predictor of order i + 1, for i >= 1.
__device__ __forceinline__ void step_up(double *t, int i, int q)
{
    const int lane = lane_id();
    const double ki = dequantise(i, q);
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

// What search_orders sizes or packs (see there).
enum { kOrdersUnit = 0, kOrdersPair = 1, kOrdersWindow = 2, kOrdersListed = 3 };

// Unit `unit` at the orders o_lo..o_hi, one after the other, on one carried step-up.  The order-1 predictor is zero
// (linear_predictor.cpp:19-22), not row 0 of the step-up.  res: the warp's residue row.
//   PACK = false  every order but the reference order (the analysis kernel has sized that one): FIR with the tie
//                 check, Rice sizes, a tie-free order into su[unit].best
//   PACK = true   (o_lo = o_hi) FIR, Rice, pack into the unit's slot and rewrite its record
// TRACE (PACK = false, tests only, selab200_encode_search_trace): each order's record into trace as well.
// KIND says what `unit` is:
//   kOrdersUnit    (order search, this file) an analysis unit, at `unit` of su and trace
//   kOrdersPair    (search + pairing, search_pairing.cuh; STEREO = true for its shared memory layout): the candidate
//                  (frame, par, c) at ((frame * C + par) * C + c) of su and trace, its signal ch_par - ch_c from
//                  stage_pair, its FIR always the wide one; PACK packs into unit `out`.  Other kinds leave `out` unused
//   kOrdersWindow  (window search, window.cuh): the record (analysis unit u, window w) at u * n_win + w of su and
//                  trace, its signal unit u's; a tie-free order enters wkey[u] as words << 16 | w << 8 | order, and
//                  PACK packs into u.  An order whose predictor leaves the domain of the int64 conversion
//                  (|2^35 t| >= 2^62, undefined in the reference; a window's clamped q can get there) counts as tied:
//                  it is never eligible
//   kOrdersListed  (PACK = false; guided order search, search_guided.cuh): an analysis unit, of which only the orders
//                  whose bit o - 1 is set in listed[unit] are sized; the step-up still runs through every order below
//                  the highest one sized
template <int KIND, bool STEREO, bool PACK, bool TRACE = false>
__device__ __forceinline__ void search_orders(const EncodeParams &p, SearchUnit *su, const uint32_t unit, int o_lo,
                                              int o_hi, int32_t *res, selab200_search_trace *trace = nullptr,
                                              uint32_t out = 0, uint32_t n_win = 1,
                                              unsigned long long *wkey = nullptr, const uint4 *listed = nullptr)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr size_t kSigBytes = unit_signal_bytes<STEREO>();
    double *t = reinterpret_cast<double *>(smem_raw + kSigBytes);
    CoefSmem &cf = *reinterpret_cast<CoefSmem *>(smem_raw + kSigBytes + kSearchStepBytes);
    uint32_t *planes = reinterpret_cast<uint32_t *>(smem_raw + kSigBytes + kSearchStepBytes + sizeof(CoefSmem));
    static_assert(kSearchStepBytes % 16 == 0 && sizeof(CoefSmem) % 16 == 0, "search shared memory layout");
    constexpr bool PAIR = KIND == kOrdersPair, WINDOW = KIND == kOrdersWindow, LISTED = KIND == kOrdersListed;
    static_assert(!PAIR || STEREO, "a pair is staged as the stereo difference is");
    static_assert(!LISTED || !PACK, "a list of a unit's orders to size");

    const int lane = lane_id();
    const uint32_t src = WINDOW ? unit / n_win : unit; // the analysis unit whose signal is coded
    const bool wide = PAIR || (STEREO && src % 3 == 2);
    const uint32_t dst = PAIR ? out : src;
    Signal sig;
    if constexpr (PAIR)
        sig = stage_pair(p, unit / (p.channels * p.channels), unit / p.channels % p.channels, unit % p.channels,
                         smem_raw);
    else
        sig = stage_unit<STEREO>(p, src, smem_raw);
    SearchUnit &s = su[unit];
    const int ref = (int)s.ref_order;
    for (int i = lane; i < 104; i += 32)
        cf.q[i] = i < kMaxOrder ? s.q[i] : 0;
    for (int i = lane; i < 112; i += 32) {
        cf.clo[i] = 0;
        cf.chi[i] = 0;
    }
    __syncwarp();
    const double scale = 34359738368.0; // 2^35
    int done = 0;                       // step-up iterations applied to t
    uint4 mask{};
    if constexpr (LISTED)
        mask = listed[unit];
    for (int o = o_lo; o <= o_hi; o++) {
        if (!PACK && o == ref)
            continue;
        if constexpr (LISTED) {
            const int b = o - 1;
            const uint32_t m = b < 32 ? mask.x : b < 64 ? mask.y : b < 96 ? mask.z : mask.w;
            if (!((m >> (b & 31)) & 1u))
                continue;
        }
        bool outside = false; // WINDOW: the predictor leaves the conversion's domain
        if (o >= 2) {
            for (; done < o; done++)
                step_up(t, done, cf.q[done]);
            for (int m = lane; m < o; m += 32) {
                if constexpr (WINDOW)
                    outside |= !(fabs(dmul(scale, -t[m])) < 4611686018427387904.0); // 2^62
                const long long v = __double2ll_rz(dmul(scale, -t[m]));
                cf.clo[m] = (uint32_t)v;
                cf.chi[m] = (int32_t)(v >> 32);
            }
            __syncwarp();
            if constexpr (WINDOW)
                outside = __any_sync(kFull, outside);
        }
        const bool tie = (wide ? warp_fir_residual<true, !PACK>(sig, cf, o, planes, res)
                               : warp_fir_residual<false, !PACK>(sig, cf, o, planes, res)) ||
                         outside;
        const RiceChoice cq = warp_rice_choose(cf.q, o);
        const RiceChoice cr = warp_rice_choose(res, kFrame);
        if constexpr (!PACK) {
            if constexpr (TRACE)
                search_trace_record(trace, unit, o, cf, res, tie, cq, cr);
            const unsigned long long words = cq.words + cr.words;
            if constexpr (WINDOW) {
                if (lane == 0 && !tie)
                    atomicMin(&wkey[src], words << 16 | (unsigned long long)(unit % n_win) << 8 | (unsigned long long)o);
            } else {
                if (lane == 0 && !tie)
                    atomicMin(&s.best, words << 8 | (unsigned long long)o);
            }
        } else {
            const bool too_large = pack_slot(p, dst, cf.q, o, res, cq, cr);
            write_record(p, dst, o, cq, cr, too_large ? 1u : 0u);
        }
        __syncwarp();
    }
}

// The search's analysis kernel: encode_unit for unit blockIdx.x.  FORCE and `pred` (tests only,
// selab200_encode_search_forced): the unit's q[0..99] and reference order are pred[unit]'s.  TRACE (tests only,
// selab200_encode_search_trace): the reference order's record into trace as well.
template <bool STEREO, bool TRACE, bool FORCE = false>
__global__ void __launch_bounds__(32) k_search_units(EncodeParams p, const selab200_predictor *pred, SearchUnit *su,
                                                     selab200_search_trace *trace)
{
    encode_unit<STEREO, TRACE, kUnitSearch, FORCE>(p, nullptr, blockIdx.x, nullptr, 0, pred, su, trace);
}

// Work item w = (unit w / kSearchSlices, slice w % kSearchSlices): the slices of a unit go to neighbouring warps,
// which read the same PCM.  Residue row = the warp's (the grid is at most the batch's units).  TRACE (tests only,
// selab200_encode_search_trace): every order's record into trace as well.
template <bool STEREO, bool TRACE>
__global__ void __launch_bounds__(32) k_search_candidates(EncodeParams p, SearchUnit *su, selab200_search_trace *trace)
{
    const size_t work = (size_t)encode_units(p.n_frames, p.channels) * kSearchSlices;
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const int sl = (int)(w % kSearchSlices);
        __syncwarp();
        search_orders<kOrdersUnit, STEREO, false, TRACE>(p, su, (uint32_t)(w / kSearchSlices), search_slice_first(sl),
                                                         search_slice_first(sl + 1) - 1, res, trace);
    }
    discard_row(res);
}

template <bool STEREO>
__global__ void __launch_bounds__(32) k_search_repack(EncodeParams p, SearchUnit *su)
{
    const uint32_t n = encode_units(p.n_frames, p.channels);
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    for (uint32_t u = blockIdx.x; u < n; u += gridDim.x) {
        const int o = (int)(su[u].best & 0xffu);
        if (o == 0 || o > kMaxOrder) // the reference order won (its slot and record stand); > 100: no tie-free
            continue;                // order, which cannot happen (order 1 has none)
        __syncwarp();
        search_orders<kOrdersUnit, STEREO, true>(p, su, u, o, o, res);
    }
}

// The words of the reference encoder's subframes of each frame (its orders, its stereo decision: difference iff
// strictly fewer words) into *ref_words.
__global__ void __launch_bounds__(256) k_search_ref_words(EncodeParams p, const SearchUnit *su,
                                                          unsigned long long *ref_words)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long w = 0;
    if (f < p.n_frames) {
        if (p.channels == 2) {
            const SearchUnit *fs = su + (size_t)f * 3;
            const uint32_t a = fs[1].ref_words, d = fs[2].ref_words;
            w = (unsigned long long)fs[0].ref_words + (d < a ? d : a);
        } else {
            const SearchUnit *fs = su + (size_t)f * p.channels;
            for (uint32_t c = 0; c < p.channels; c++)
                w += fs[c].ref_words;
        }
    }
    w = warp_sum_u64(w);
    if (lane_id() == 0 && w)
        atomicAdd(ref_words, w);
}

} // namespace selab200
