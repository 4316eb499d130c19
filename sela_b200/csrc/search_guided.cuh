// search_guided.cuh -- the kernels of the guided order search (sm_90a, DESIGN.md 7.7): the order search of 7.3 with
// its candidates cut down to the K orders a reflection-coefficient estimate of the prediction error ranks best,
// order 1 and the reference order.
//
//   k_search_units<S>            the order search's analysis kernel, unchanged (search.cuh)
//   k_search_estimate<T>         warp per unit: E_o = P_o * R_o for o = 1..100 (one lane, sequentially), the rank of
//                                every order by (E_o, o), and the unit's order mask: rank < K, order 1, the reference
//                                order
//   k_search_listed<S, T>        warp per unit: search_orders over the listed orders, on one carried step-up; a
//                                tie-free order enters the unit's atomicMin key, as in k_search_candidates
//   k_search_ref_words, k_search_repack<S>   as for the order search (search.cuh), unchanged
// Then k_encode_sizes / k_encode_scan / k_encode_gather(_container) run as for every encode.  The estimate and listed
// kernels have grids of a fixed size and loop over the units.  T (tests only, selab200_encode_search_guided_trace):
// the tracing instantiations, which write every unit's E[100] and the record of every order sized.
#pragma once

#include "search.cuh"

namespace selab200 {

// r = 2^(1/256), rounded to the nearest double: a cost of 4 bits per coefficient over a 2048-sample frame, as a
// factor on the prediction error per order.
constexpr double kGuidedOrderCost = 0x1.00b1afa5abcbfp+0;

struct GuidedParams {
    uint32_t candidates; // K, 1..100
    uint4 *masks;        // [n_units]: bit o - 1 set for every listed order o
    double *estimates;   // tests only: [n_units][100], E_o at o - 1
};

// The estimate of every order and the unit's mask.  a_i = 1 - k_i^2 with k_i the coefficient the step-up
// dequantises; P_1 = 1, P_o = P_{o-1} a_{o-1} (P_2 = a_0 a_1); R_o = r^o; E_o = P_o R_o, every operation rounded as
// written and in this order.  An order's rank is the number of orders before it by (E, order).
template <bool TRACE>
__global__ void __launch_bounds__(32) k_search_estimate(EncodeParams p, const SearchUnit *su, GuidedParams gp)
{
    __shared__ double a[kMaxOrder];
    __shared__ double e[kMaxOrder];
    const int lane = lane_id();
    const uint32_t n = encode_units(p.n_frames, p.channels);
    for (uint32_t u = blockIdx.x; u < n; u += gridDim.x) {
        const SearchUnit &s = su[u];
        __syncwarp();
        for (int i = lane; i < kMaxOrder; i += 32) {
            const double k = dequantise(i, s.q[i]);
            a[i] = dsub(1.0, dmul(k, k));
        }
        __syncwarp();
        if (lane == 0) {
            double P = 1.0, R = kGuidedOrderCost;
            e[0] = dmul(P, R);
            P = a[0];
            for (int o = 2; o <= kMaxOrder; o++) {
                P = dmul(P, a[o - 1]);
                R = dmul(R, kGuidedOrderCost);
                e[o - 1] = dmul(P, R);
            }
        }
        __syncwarp();
        const int ref = (int)s.ref_order;
        uint32_t words[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int o = 32 * j + lane + 1;
            bool listed = false;
            if (o <= kMaxOrder) {
                const double eo = e[o - 1];
                int rank = 0;
#pragma unroll 4
                for (int m = 0; m < kMaxOrder; m++) {
                    const double em = e[m];
                    rank += (em < eo || (em == eo && m + 1 < o)) ? 1 : 0;
                }
                listed = rank < (int)gp.candidates || o == 1 || o == ref;
                if constexpr (TRACE)
                    gp.estimates[(size_t)u * kMaxOrder + o - 1] = eo;
            }
            words[j] = __ballot_sync(kFull, listed);
        }
        if (lane == 0)
            gp.masks[u] = make_uint4(words[0], words[1], words[2], words[3]);
    }
}

// Work item: unit u, every listed order but the reference one.  Residue row = the warp's.
template <bool STEREO, bool TRACE>
__global__ void __launch_bounds__(32) k_search_listed(EncodeParams p, SearchUnit *su, GuidedParams gp,
                                                      selab200_search_trace *trace)
{
    const uint32_t n = encode_units(p.n_frames, p.channels);
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    for (uint32_t u = blockIdx.x; u < n; u += gridDim.x) {
        __syncwarp();
        search_orders<kOrdersListed, STEREO, false, TRACE>(p, su, u, 1, kMaxOrder, res, trace, 0, 1, nullptr,
                                                           gp.masks);
    }
    discard_row(res);
}

} // namespace selab200
