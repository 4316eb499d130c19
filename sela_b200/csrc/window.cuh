// window.cuh -- the kernels of the window search (sm_90a, DESIGN.md 7.6): the order search of 7.3, and every unit
// also analysed once per selected apodisation window and searched over orders 1..100 from that analysis; a unit is
// coded from the window analysis and order with the fewest words when that is strictly fewer than the order search's.
//
//   the order search (search.cuh) runs first, unchanged: the base
//   k_window_base_words          thread per frame: the words the order search writes (its records, its stereo
//                                decision), summed into one counter
//   k_window_units<S>            warp per (unit, window): stage_unit, the autocorrelation of the windowed signal, Schur,
//                                and all 100 q into the (unit, window) SearchUnit with ref_order = 0.  Nothing is packed
//   k_window_candidates<S, T>    warp per (unit, window, slice of orders): search_orders on the unit's signal with the
//                                record's q; a tie-free order enters the unit's window key
//   k_window_repack<S>           warp per unit whose window key has strictly fewer words than the order search's
//                                winner: that window's q at that order packed into the unit's slot, record rewritten
// Then k_encode_sizes / k_encode_scan / k_encode_gather(_container) run as for every encode.  The warp kernels have
// grids of a fixed size and loop over the work.  T (tests only, selab200_encode_search_windows_trace): the tracing
// instantiation, which writes the record of every (unit, window, order) to trace at (unit * n + w) * 100 + order - 1.
#pragma once

#include "search.cuh"

namespace selab200 {

// The fixed window table (selab200_analysis_window): bit i of a window mask selects row i.  The host computes the
// rows once and copies them here when it sets the device up (init_slot in c_abi.cu).
constexpr int kAnalysisWindows = 5;
__device__ double d_analysis_windows[kAnalysisWindows * kFrame];

struct WindowParams {
    const double *table;               // [.][2048]; record w of a unit uses the row of the w-th set bit of mask
    uint32_t mask, n;                  // n = popcount(mask), at most kAnalysisWindows
    SearchUnit *su;                    // [n_units][n]: every q of each window analysis, ref_order 0
    unsigned long long *key;           // [n_units]: words << 16 | w << 8 | order of the best window candidate
    unsigned long long *n_window;      // += the units coded from a window
    const selab200_predictor *pred;    // tests only: [n_units][n], the records' q in place of the analyses'
    selab200_search_trace *trace;      // tests only: [n_units][n][100]
};

// The words of the order search's subframes of each frame, as k_encode_scan would emit them now, into *base_words.
__global__ void __launch_bounds__(256) k_window_base_words(EncodeParams p, unsigned long long *base_words)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long w = 0;
    if (f < p.n_frames)
        for (uint32_t c = 0; c < p.channels; c++) {
            UnitRecord u;
            choose_record(p.units, p.channels, f * p.channels + c, u);
            w += (unsigned long long)u.refl_words + u.res_words;
        }
    w = warp_sum_u64(w);
    if (lane_id() == 0 && w)
        atomicAdd(base_words, w);
}

// Work item w = (unit w / n, window w % n): the windows of a unit go to neighbouring warps, which read the same PCM.
// The analysis is encode_unit's up to the quantiser, with d[j] * win[j] in the autocorrelation; every q is kept,
// clamped to [-64, 63]: a windowed analysis of a near-singular signal can round to |k| > 1, whose q the quantiser puts
// outside the range the decoders read (the reference's dequantiser would index past its table).
template <bool STEREO>
__global__ void __launch_bounds__(32) k_window_units(EncodeParams p, WindowParams wp)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    AnalysisScratch &scratch = *reinterpret_cast<AnalysisScratch *>(smem_raw + unit_signal_bytes<STEREO>());
    const int lane = lane_id();
    const size_t work = (size_t)encode_units(p.n_frames, p.channels) * wp.n;
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const uint32_t unit = (uint32_t)(w / wp.n), win = (uint32_t)(w % wp.n);
        SearchUnit &s = wp.su[w];
        __syncwarp();
        if (wp.pred) {
            for (int i = lane; i < kMaxOrder; i += 32)
                s.q[i] = wp.pred[w].q[i];
        } else {
            const Signal sig = stage_unit<STEREO>(p, unit, smem_raw);
            const double *row = wp.table + (size_t)(__fns(wp.mask, 0, (int)win + 1)) * kFrame;
            warp_autocorrelation<Signal, true>(sig, scratch, shfl_d(lane == 0 ? p.means[unit] : 0.0, 0), row);
            warp_schur(scratch);
            for (int i = lane; i < kMaxOrder; i += 32) // into the range the decoder reads (see the comment above)
                s.q[i] = min(max(quantise_reflection(i, scratch.kk()[i]), -64), 63);
        }
        if (lane == 0) {
            s.ref_order = 0;
            s.ref_words = 0;
            s.best = kNoCandidate;
        }
    }
}

// Work item w = ((unit, window) w / kSearchSlices, slice w % kSearchSlices), numbered densely: the slices and windows
// of a unit go to neighbouring warps, which read the same PCM.  Residue row = the warp's.
template <bool STEREO, bool TRACE>
__global__ void __launch_bounds__(32) k_window_candidates(EncodeParams p, WindowParams wp)
{
    const size_t work = (size_t)encode_units(p.n_frames, p.channels) * wp.n * kSearchSlices;
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const int sl = (int)(w % kSearchSlices);
        __syncwarp();
        search_orders<kOrdersWindow, STEREO, false, TRACE>(p, wp.su, (uint32_t)(w / kSearchSlices),
                                                           search_slice_first(sl), search_slice_first(sl + 1) - 1, res,
                                                           wp.trace, 0, wp.n, wp.key);
    }
    discard_row(res);
}

// A warp per unit at a time.  su: the order search's records, whose best holds its winner's words.
template <bool STEREO>
__global__ void __launch_bounds__(32) k_window_repack(EncodeParams p, WindowParams wp, const SearchUnit *su)
{
    const uint32_t n = encode_units(p.n_frames, p.channels);
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    unsigned long long count = 0;
    for (uint32_t u = blockIdx.x; u < n; u += gridDim.x) {
        const unsigned long long key = wp.key[u];
        if (key == kNoCandidate || (key >> 16) >= (su[u].best >> 8)) // no window strictly better: -S's bytes stand
            continue;
        __syncwarp();
        search_orders<kOrdersWindow, STEREO, true>(p, wp.su, u * wp.n + (uint32_t)((key >> 8) & 0xffu),
                                                   (int)(key & 0xffu), (int)(key & 0xffu), res, nullptr, 0, wp.n);
        count++;
    }
    discard_row(res);
    if (lane_id() == 0 && count)
        atomicAdd(wp.n_window, count);
}

} // namespace selab200
