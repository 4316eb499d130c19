// pairing.cuh -- the kernels of the channel pairing (sm_90a, DESIGN.md 7.4): every channel of a frame is coded alone
// or as its difference from another, independently coded channel of the frame, whichever assignment of the whole
// frame takes the fewest words, for any channel count, inside the format.
//
//   the lossless encode (lossless.cuh) runs first: the base.  k_pairing_capture, in front of k_lossless_select, keeps
//   the tie flags that kernel clears (a flagged stereo candidate that loses stays tied, it is only never emitted)
//   k_pairing_means        lane per (frame, p, c): the mean of ch_p - ch_c (MeanChain)
//   k_pairing_candidates   warp per (frame, p, c), p != c: ch_p - ch_c staged as the stereo difference is, analysed,
//                          FIR with the tie check, both Rice sizes -> a 16-byte record of the frame's [C][C] table.
//                          Nothing is packed.  Stereo (0, 1) is the base's unit 2 and is not run again
//   k_pairing_select       CTA per frame: the valid assignment with the fewest words over all 2^C sets of independent
//                          channels -> par[frame][C]; the base's words and the differences chosen into two counters
//   k_pairing_repack       warp per winning difference: run again and packed into the slot and record of channel c
//   k_pairing_patch        thread per subframe, after k_encode_scan: type and parent of the winners' descriptors
// k_encode_sizes / k_encode_scan / k_encode_gather(_container) run unchanged on the records as the repack left them;
// the container gather takes type and parent from the descriptors.  Stereo has three units per frame and the decision
// inside choose_unit: with ch0 coded against ch1 the difference goes to unit 0 and unit 2 is made to lose.
// The candidate and repack kernels have grids of a fixed size and loop over the work.
#pragma once

#include "lossless.cuh"

namespace selab200 {

// One candidate (p, c) of a frame.  In the search + pairing (search_pairing.cuh) k_search_pairing_table fills it from
// the candidate's searched key: res_words the searched words (reflection + residue), order the searched order,
// refl_words, refl_k and res_k 0, tie 0 (every searched order is tie-free).  k_pairing_select reads only the sum of
// the two word counts and tie.
struct __align__(16) PairRecord {
    uint32_t refl_words, res_words;
    uint8_t order, refl_k, res_k, tie;
    uint32_t pad;
};

struct PairingParams {
    PairRecord *table;                  // [n_frames][C][C], entry p * C + c; the diagonal is unused
    double *means;                      // [n_frames][C][C]
    uint8_t *par;                       // [n_frames][C]
    uint32_t *stale;                    // [n_frames] bit k: unit k of the frame has a tie that the base left alone
    unsigned long long *base_words;     // += the words of the base's subframes
    unsigned long long *n_difference;   // += the difference subframes chosen
    const selab200_predictor *pred;     // tests only: the candidates' predictors, (frame, p, c) order without p = c
    selab200_search_trace *trace;       // tests only: [n_frames][C][C] records of the candidates as they were sized
};

__device__ __forceinline__ bool pairing_is_candidate(uint32_t channels, uint32_t p, uint32_t c)
{
    return p != c && !(channels == 2 && p == 0); // stereo (0, 1): the base's unit 2
}

// The unit of the workspace that holds channel c's independent coding.
__device__ __forceinline__ uint32_t pairing_unit(uint32_t channels, uint32_t frame, uint32_t c)
{
    return frame * units_per_frame(channels) + c;
}

// In front of k_lossless_select: the flagged units of the frames that kernel will not list.  It clears their flags
// because they are not emitted; they still have their ties, and the pairing must neither emit them nor use them as
// parents.
__global__ void __launch_bounds__(256) k_pairing_capture(EncodeParams p, PairingParams q)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.n_frames)
        return;
    const uint32_t per = units_per_frame(p.channels);
    const UnitRecord *fu = p.units + (size_t)f * per;
    uint32_t flagged = 0;
    for (uint32_t k = 0; k < per; k++)
        flagged |= ((fu[k].flags >> 1) & 1u) << k;
    bool emitted = false;
    for (uint32_t c = 0; flagged && c < p.channels; c++) {
        UnitRecord u;
        emitted |= (flagged >> choose_record(fu, p.channels, c, u).unit) & 1u;
    }
    q.stale[f] = emitted ? 0u : flagged;
}

__global__ void __launch_bounds__(128) k_pairing_means(EncodeParams p, PairingParams q)
{
    const uint32_t C = p.channels;
    const size_t n = (size_t)p.n_frames * C * C, i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const uint32_t c = (uint32_t)(i % C), par = (uint32_t)(i / C % C);
    if (!pairing_is_candidate(C, par, c))
        return;
    const int16_t *src = p.pcm + i / ((size_t)C * C) * kFrame * C;
    MeanChain chain;
    for (int j = 0; j < kFrame; j++)
        chain.add((int)src[(size_t)j * C + par] - (int)src[(size_t)j * C + c]);
    q.means[i] = chain.mean();
}

// Candidate (par, c) of `frame` by one warp, with the steps of encode_unit on a stereo difference (stage_pair in
// kernels.cuh stages it).  res: the warp's residue row.
//   PACK = false  FIR with the tie check, Rice sizes, the candidate's record into the table
//   PACK = true   FIR, Rice, pack into the slot of unit `out` and rewrite its record
//   SEARCH        (PACK = false; search + pairing, search_pairing.cuh) as kUnitSearch does for a unit: every q and
//                 the reference order's words and key into su[(frame, par, c)], nothing into the table.  TRACE: the
//                 reference order's search record into q.trace
template <bool PACK, bool SEARCH = false, bool TRACE = false>
__device__ __forceinline__ void pair_unit(const EncodeParams &p, const PairingParams &q, uint32_t frame, uint32_t par,
                                          uint32_t c, int32_t *res, uint32_t out, SearchUnit *su = nullptr)
{
    static_assert(!SEARCH || !PACK, "the search packs through search_orders");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr size_t kSigBytes = unit_signal_bytes<true>();
    AnalysisScratch &scratch = *reinterpret_cast<AnalysisScratch *>(smem_raw + kSigBytes);
    CoefSmem &cf = *reinterpret_cast<CoefSmem *>(smem_raw + kSigBytes + kCoefAlias);
    const int lane = lane_id();
    const uint32_t C = p.channels;
    const size_t idx = ((size_t)frame * C + par) * C + c;
    const Signal sig = stage_pair(p, frame, par, c, smem_raw);
    warp_autocorrelation(sig, scratch, shfl_d(lane == 0 ? q.means[idx] : 0.0, 0));
    warp_schur(scratch);
    int order = warp_order_and_quantise(scratch, cf);
    if (q.pred) { // tests only: q past the forced order is zero (the entry point checks it)
        const selab200_predictor &f = q.pred[((size_t)frame * C + par) * (C - 1) + (c < par ? c : c - 1)];
        for (int i = lane; i < kMaxOrder; i += 32)
            cf.q[i] = f.q[i];
        order = f.order;
        __syncwarp();
    }
    warp_coefficients(cf, scratch.t(), order);
    if constexpr (SEARCH)
        copy_every_q(su[idx].q, cf, scratch, q.pred != nullptr);
    uint32_t *planes = reinterpret_cast<uint32_t *>(scratch.ring); // over k[] and the step-up row, dead now
    const bool tie = warp_fir_residual<true, !PACK>(sig, cf, order, planes, res);
    const RiceChoice cq = warp_rice_choose(cf.q, order);
    const RiceChoice cr = warp_rice_choose(res, kFrame);
    if constexpr (SEARCH) {
        if constexpr (TRACE)
            search_trace_record(q.trace, (uint32_t)idx, order, cf, res, tie, cq, cr);
        write_search_ref(su[idx], order, cq, cr, tie);
    } else if constexpr (!PACK) {
        if (q.trace) {
            search_trace_record(q.trace + idx, 0, 1, cf, res, tie, cq, cr);
            if (lane == 0)
                q.trace[idx].reserved[0] = (uint8_t)order;
        }
        if (lane == 0) {
            PairRecord r;
            r.refl_words = cq.words;
            r.res_words = cr.words;
            r.order = (uint8_t)order;
            r.refl_k = (uint8_t)cq.k;
            r.res_k = (uint8_t)cr.k;
            r.tie = tie ? 1 : 0;
            r.pad = 0;
            q.table[idx] = r;
        }
    } else {
        const bool too_large = pack_slot(p, out, cf.q, order, res, cq, cr);
        write_record(p, out, order, cq, cr, too_large ? 1u : 0u);
    }
    __syncwarp();
}

// Work item w = (frame, p, c) in that order: the candidates of a frame go to neighbouring warps, which read the same
// PCM.  Residue row = the warp's (the grid is at most the batch's units).
__global__ void __launch_bounds__(32) k_pairing_candidates(EncodeParams p, PairingParams q)
{
    const uint32_t C = p.channels;
    const size_t work = (size_t)p.n_frames * C * C;
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    for (size_t w = blockIdx.x; w < work; w += gridDim.x) {
        const uint32_t c = (uint32_t)(w % C), par = (uint32_t)(w / C % C);
        if (!pairing_is_candidate(C, par, c))
            continue;
        pair_unit<false>(p, q, (uint32_t)(w / ((size_t)C * C)), par, c, res, 0);
    }
    discard_row(res);
}

// Rule 3 and 4 of DESIGN.md 7.4 for one frame per CTA at a time.  An assignment is fixed by its set S of independent
// channels: every other channel takes its cheapest valid parent in S, the lowest between equal words.  The key
// (words << 8 | differences, par[0..C) as nibbles, par[0] highest) orders the assignments as rule 4 does.
constexpr uint32_t kPairNone = 0xffffffffu;
__global__ void __launch_bounds__(128) k_pairing_select(EncodeParams p, PairingParams q)
{
    __shared__ uint32_t I[SELAB200_MAX_CHANNELS];                         // words of channel c alone; kPairNone: tied
    __shared__ uint32_t D[SELAB200_MAX_CHANNELS][SELAB200_MAX_CHANNELS]; // words of (p, c); kPairNone: tied
    __shared__ unsigned long long best[4][2];
    static_assert(SELAB200_MAX_CHANNELS <= 16, "the key holds a parent per nibble");
    const uint32_t C = p.channels, per = units_per_frame(C);
    const int lane = lane_id(), warp = warp_id();
    for (uint32_t f = blockIdx.x; f < p.n_frames; f += gridDim.x) {
        const UnitRecord *fu = p.units + (size_t)f * per;
        PairRecord *ft = q.table + (size_t)f * C * C;
        const uint32_t stale = q.stale[f];
        __syncthreads();
        if (threadIdx.x == 0 && C == 2) { // the base's difference unit, as the base left it
            PairRecord r;
            r.refl_words = fu[2].refl_words;
            r.res_words = fu[2].res_words;
            r.order = (uint8_t)fu[2].order;
            r.refl_k = (uint8_t)fu[2].refl_k;
            r.res_k = (uint8_t)fu[2].res_k;
            r.tie = (stale >> 2) & 1u;
            r.pad = 0;
            ft[1] = r;
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < C * C; i += blockDim.x) {
            const uint32_t par = i / C, c = i % C;
            if (par == c) {
                I[c] = (stale >> c) & 1u ? kPairNone : fu[c].refl_words + fu[c].res_words;
            } else {
                const PairRecord r = ft[i];
                D[par][c] = r.tie ? kPairNone : r.refl_words + r.res_words;
            }
        }
        if (threadIdx.x == 0) { // what the lossless encode emits for this frame
            unsigned long long w = 0;
            for (uint32_t c = 0; c < C; c++) {
                UnitRecord u;
                choose_record(fu, C, c, u);
                w += (unsigned long long)u.refl_words + u.res_words;
            }
            atomicAdd(q.base_words, w);
        }
        __syncthreads();
        unsigned long long k1 = ~0ull, k2 = ~0ull;
        for (uint32_t S = 1 + threadIdx.x; S < (1u << C); S += blockDim.x) {
            unsigned long long words = 0, pars = 0;
            bool ok = true;
            for (uint32_t c = 0; c < C && ok; c++) {
                uint32_t w = kPairNone, parent = c;
                if ((S >> c) & 1u) {
                    w = I[c];
                } else {
                    for (uint32_t m = S; m; m &= m - 1) {
                        const uint32_t par = __ffs(m) - 1;
                        if (D[par][c] < w) {
                            w = D[par][c];
                            parent = par;
                        }
                    }
                }
                ok = w != kPairNone;
                words += w;
                pars = pars << 4 | parent;
            }
            const unsigned long long a = words << 8 | (C - __popc(S));
            if (ok && (a < k1 || (a == k1 && pars < k2))) {
                k1 = a;
                k2 = pars;
            }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long a = __shfl_xor_sync(kFull, k1, o), b = __shfl_xor_sync(kFull, k2, o);
            if (a < k1 || (a == k1 && b < k2)) {
                k1 = a;
                k2 = b;
            }
        }
        if (lane == 0) {
            best[warp][0] = k1;
            best[warp][1] = k2;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < 4; w++)
                if (best[w][0] < k1 || (best[w][0] == k1 && best[w][1] < k2)) {
                    k1 = best[w][0];
                    k2 = best[w][1];
                }
            // the base's own assignment is valid, so there is a minimum
            for (uint32_t c = 0; c < C; c++)
                q.par[(size_t)f * C + c] = (uint8_t)((k2 >> (4 * (C - 1 - c))) & 15u);
            if (k1 & 0xffu)
                atomicAdd(q.n_difference, k1 & 0xffu);
        }
    }
}

// A warp per subframe at a time; the winners that are not packed yet are run again and packed.  Stereo: (0, 1) is
// the base's unit 2, which the decision in choose_unit picks by itself (it won on strictly fewer words, or channel
// 1 alone is tied); (1, 0) goes to unit 0, and unit 2 is given a size that loses.
__global__ void __launch_bounds__(32) k_pairing_repack(EncodeParams p, PairingParams q)
{
    const uint32_t C = p.channels, n_sub = p.n_frames * C;
    int32_t *res = p.residues + (size_t)blockIdx.x * kFrame;
    for (uint32_t sub = blockIdx.x; sub < n_sub; sub += gridDim.x) {
        const uint32_t f = sub / C, c = sub % C, par = q.par[sub];
        if (!pairing_is_candidate(C, par, c))
            continue;
        pair_unit<true>(p, q, f, par, c, res, pairing_unit(C, f, c));
        if (C == 2 && lane_id() == 0)
            p.units[(size_t)f * 3 + 2].res_words = kPairNone;
    }
    discard_row(res);
}

// After k_encode_scan: the winners' descriptors say what they are.
__global__ void __launch_bounds__(256) k_pairing_patch(EncodeParams p, PairingParams q)
{
    const uint32_t sub = blockIdx.x * blockDim.x + threadIdx.x;
    if (sub >= p.n_frames * p.channels)
        return;
    const uint32_t par = q.par[sub];
    if (par != sub % p.channels) {
        p.descs[sub].subframe_type = 1;
        p.descs[sub].parent_channel = (uint8_t)par;
    }
}

} // namespace selab200
