// search_pairing.cuh -- the kernels of the search + pairing (sm_90a, DESIGN.md 7.5): the channel pairing of 7.4 on top
// of the order search of 7.3, every channel and every channel difference coded at its cheapest tie-free order.
//
//   the order search (search.cuh) runs first: the base.  Every searched unit is tie-free, so no unit is stale
//   k_pairing_means                 lane per (frame, p, c): the mean of ch_p - ch_c, as for the pairing
//   k_search_pairing_units<T>       warp per (frame, p, c), p != c: pair_unit's analysis in its search mode: all 100
//                                   q, the reference order coded with the tie check, the candidate's SearchUnit and,
//                                   if that order is tie-free, its key.  Nothing is packed.  Stereo (0, 1) is the
//                                   base's searched unit 2 and is not run again
//   k_search_pairing_candidates<T>  warp per (candidate, slice of orders): search_orders<kOrdersPair>, as
//                                   k_search_candidates runs it on a unit
//   k_search_pairing_table          thread per (frame, p, c): the candidate's searched words into the PairRecord table
//   k_pairing_select                unchanged: the valid assignment with the fewest words -> par[frame][C]
//   k_search_pairing_repack         warp per winning difference: search_orders packs it at its searched order into the
//                                   slot and record of channel c; stereo (1, 0) makes unit 2 lose, as k_pairing_repack
//   k_pairing_patch                 after k_encode_scan, unchanged
// The candidates' SearchUnits are indexed [n_frames][C][C] like the table.  The warp kernels have grids of a fixed
// size and loop over the work.  T (tests only, selab200_encode_search_pairing_trace): the tracing instantiations,
// which write the record of every (candidate, order) to q.trace at ((frame * C + p) * C + c) * 100 + order - 1.
#pragma once

#include "pairing.cuh"
#include "search.cuh"

namespace selab200 {

// The warp kernels number the candidates densely, (frame, p, c) in order without p = c and stereo (0, 1): a work
// index over all [C][C] entries would leave warps idle, because the grid's stride is a multiple of C * C for small C
// and every warp would meet the same (p, c) each time round.
__device__ __forceinline__ uint32_t search_pairing_per_frame(uint32_t C)
{
    return C == 2 ? 1u : C * (C - 1);
}

// Candidate k of the batch -> its index (frame * C + par) * C + c.
__device__ __forceinline__ uint32_t search_pairing_candidate(uint32_t C, size_t k)
{
    const uint32_t per = search_pairing_per_frame(C), f = (uint32_t)(k / per), j = (uint32_t)(k % per);
    const uint32_t par = C == 2 ? 1u : j / (C - 1), r = C == 2 ? 0u : j % (C - 1);
    const uint32_t c = r < par ? r : r + 1;
    return (f * C + par) * C + c;
}

// TRACE: the reference order's record into q.trace as well.
template <bool TRACE>
__global__ void __launch_bounds__(32) k_search_pairing_units(EncodeParams p, PairingParams q, SearchUnit *su)
{
    const uint32_t C = p.channels;
    const size_t work = (size_t)p.n_frames * search_pairing_per_frame(C);
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const uint32_t idx = search_pairing_candidate(C, w);
        pair_unit<false, true, TRACE>(p, q, idx / (C * C), idx / C % C, idx % C, res, 0, su);
    }
    discard_row(res);
}

// Work item w = (candidate w / kSearchSlices, slice w % kSearchSlices), candidates numbered densely in (frame, p, c)
// order: the slices of a candidate and the candidates of a frame go to neighbouring warps, which read the same PCM.
// TRACE: every order's record into trace as well.
template <bool TRACE>
__global__ void __launch_bounds__(32) k_search_pairing_candidates(EncodeParams p, SearchUnit *su,
                                                                  selab200_search_trace *trace)
{
    const uint32_t C = p.channels;
    const size_t work = (size_t)p.n_frames * search_pairing_per_frame(C) * kSearchSlices;
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const uint32_t idx = search_pairing_candidate(C, w / kSearchSlices);
        const int sl = (int)(w % kSearchSlices);
        __syncwarp();
        search_orders<kOrdersPair, true, false, TRACE>(p, su, idx, search_slice_first(sl),
                                                       search_slice_first(sl + 1) - 1, res, trace);
    }
    discard_row(res);
}

// The candidates' searched keys into the table (the PairRecord comment says what the fields hold).  Every candidate
// has a key: order 1 never ties.
__global__ void __launch_bounds__(256) k_search_pairing_table(EncodeParams p, PairingParams q, const SearchUnit *su)
{
    const uint32_t C = p.channels;
    const size_t n = (size_t)p.n_frames * C * C, i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !pairing_is_candidate(C, (uint32_t)(i / C % C), (uint32_t)(i % C)))
        return;
    const unsigned long long best = su[i].best;
    const uint32_t o = (uint32_t)(best & 0xffu);
    PairRecord r;
    r.refl_words = 0;
    r.res_words = (uint32_t)(best >> 8);
    r.order = (uint8_t)(o ? o : su[i].ref_order);
    r.refl_k = r.res_k = 0;
    r.tie = 0;
    r.pad = 0;
    q.table[i] = r;
}

// A warp per subframe at a time; every winning candidate is packed at its searched order into channel c's slot and
// record.  Stereo: (0, 1) is the base's unit 2, which choose_unit picks by itself; (1, 0) goes to unit 0, and unit 2
// is given a size that loses.
__global__ void __launch_bounds__(32) k_search_pairing_repack(EncodeParams p, PairingParams q, SearchUnit *su)
{
    const uint32_t C = p.channels, n_sub = p.n_frames * C;
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    for (uint32_t sub = blockIdx.x; sub < n_sub; sub += gridDim.x) {
        const uint32_t f = sub / C, c = sub % C, par = q.par[sub];
        if (!pairing_is_candidate(C, par, c))
            continue;
        const uint32_t idx = (f * C + par) * C + c;
        const int key_order = (int)(su[idx].best & 0xffu); // 0: the reference order won
        const int o = key_order ? key_order : (int)su[idx].ref_order;
        __syncwarp();
        search_orders<kOrdersPair, true, true>(p, su, idx, o, o, res, nullptr, pairing_unit(C, f, c));
        if (C == 2 && lane_id() == 0)
            p.units[(size_t)f * 3 + 2].res_words = kPairNone;
    }
    discard_row(res);
}

} // namespace selab200
