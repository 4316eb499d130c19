// kernels.cuh -- the __global__ kernels of the SELA hot path (sm_90a).
//
//   encode   k_unit_means<KIND> (lane per analysis unit: the mean of its samples)
//            k_encode_units<STEREO> (warp per analysis unit: PCM -> ... -> Rice pack into a private slot; its
//            CHECK instantiation also flags ties, and lossless.cuh re-codes flagged units through encode_unit;
//            search.cuh runs its kUnitSearch mode and codes other orders on the staged signal of stage_unit)
//            k_encode_sizes + k_encode_scan (stereo decision, prefix sum, descriptors)
//            k_encode_gather / k_encode_gather_container (slot -> word arena / .sela byte stream)
//   decode   k_container_unpack (.sela bytes -> word arena)
//            k_decode_width_counts + k_decode_plan (subframes packed into synthesis warps by segment width)
//            k_rice_decode<RING,BATCH> (lane per stream: reflection streams, flagged residue streams)
//            k_rice_split_index / k_rice_decode_vc (rice_vs.cuh: residue streams, lane per part of a stream)
//            k_synthesise_segments (+ k_diff_fixup for difference-coded subframes)
//   stage-level entry points   k_unit_means + k_lpc_residues, k_lpc_samples, k_rice_encode, k_rice_decode_streams
#pragma once

#include "lpc.cuh"
#include "rice.cuh"
#include "rice_vs.cuh"

namespace selab200 {

// ------------------------------------------------------------------- means --
//
// k_unit_means<KIND>: the mean of every analysis unit (K1a, MeanChain), one LANE per unit, 32 units per
// warp, a warp per CTA.  All 32 lanes of a warp used to run the same 2048-step chain of dependent adds
// inside k_encode_units; here each lane runs its own unit's.  The units of a warp cover a few consecutive
// rows of the input (frames of interleaved PCM, or planar signals); tile by tile (64 samples of every row)
// the warp copies those rows into shared memory with aligned 16-byte loads, issued one tile ahead of the
// chains, and each lane reads its own samples from there.
//   kMeanPcm     unit u = channel u % C of frame u / C, interleaved int16 PCM, any channel count C
//   kMeanStereo  unit u = ch0, ch1 or ch0 - ch1 of frame u / 3 (interleaved int16, 16-byte aligned)
//   kMeanPlanar  unit u = int32 row u of 2048 samples (16-byte aligned)
// A row is read in whole aligned 16-byte pieces, so up to 15 bytes around it: never past the 16-byte
// block that holds the input's first or last byte.
enum { kMeanPcm = 0, kMeanStereo = 1, kMeanPlanar = 2 };
constexpr int kMeanTile = 64;  // samples per row per tile
constexpr int kMeanSlots = 16; // 16-byte pieces per lane per tile (at most 512 per warp, see mean_tiling)

struct MeanTiling {
    uint32_t units_per_row; // units that read one row
    uint32_t step;          // bytes from one sample of a row to the next
    uint32_t row_stride;    // bytes from one row to the next (a multiple of 16)
    uint32_t rows_max;      // rows a warp's 32 units can cover
    uint32_t row_words;     // shared-memory words per staged row
};

// Row pitch in shared memory: the lanes of one row read at most `span` neighbouring words at a time, and a
// pitch of d words (mod 32), d >= span and odd, puts the rows of a warp on different banks.
__host__ __device__ inline MeanTiling mean_tiling(int kind, uint32_t channels)
{
    MeanTiling t;
    uint32_t span = 1;
    if (kind == kMeanPcm) {
        t.units_per_row = channels;
        t.step = 2 * channels;
        t.row_stride = (uint32_t)kFrame * 2 * channels;
        t.rows_max = 31 / channels + 2 < 32 ? 31 / channels + 2 : 32;
        span = (2 * channels + 5) / 4;
    } else {
        t.units_per_row = kind == kMeanStereo ? 3 : 1;
        t.step = 4;
        t.row_stride = (uint32_t)kFrame * 4;
        t.rows_max = kind == kMeanStereo ? 12 : 32;
    }
    const uint32_t d = span | 1u;
    const uint32_t need = kMeanTile * t.step / 4 + 4; // the tile plus the piece it may start inside
    t.row_words = need + ((d - need) & 31u);
    return t;
}

template <int KIND>
__global__ void __launch_bounds__(32) k_unit_means(const void *src, uint32_t n_units, uint32_t channels, double *means)
{
    extern __shared__ __align__(16) uint32_t staged[]; // [rows_max][row_words]
    const MeanTiling mt = mean_tiling(KIND, channels);
    const int lane = lane_id();
    const uint32_t u0 = blockIdx.x * 32, u = u0 + lane;
    const uint32_t u_last = u0 + 31 < n_units ? u0 + 31 : n_units - 1;
    const uint32_t first = u0 / mt.units_per_row, n_rows = u_last / mt.units_per_row - first + 1;
    const uint32_t mine = u < n_units ? u : u_last; // lanes past the end shadow the last unit
    const uint32_t row = mine / mt.units_per_row - first, role = mine % mt.units_per_row;

    // the warp's rows start `mis` bytes into an aligned piece; staged row r holds the tile's bytes from there
    const char *base = static_cast<const char *>(src) + (size_t)first * mt.row_stride;
    const uint32_t mis = (uint32_t)reinterpret_cast<uintptr_t>(base) & 15u;
    const uint4 *pieces = reinterpret_cast<const uint4 *>(base - mis);
    const uint32_t tile_pieces = kMeanTile * mt.step / 16;
    const uint32_t per_row = (mis + kMeanTile * mt.step + 15) / 16, total = n_rows * per_row;
    // slot s of this lane: piece v = lane + 32 s of the tile, i.e. piece v % per_row of row v / per_row
    uint32_t goff[kMeanSlots], soff[kMeanSlots];
#pragma unroll
    for (int s = 0; s < kMeanSlots; s++) {
        const uint32_t v = lane + 32 * s, r = v / per_row, k = v - r * per_row;
        goff[s] = r * (mt.row_stride / 16) + k;
        soff[s] = r * mt.row_words + 4 * k;
    }
    uint4 buf[kMeanSlots];
    auto fetch = [&](int t) {
#pragma unroll
        for (int s = 0; s < kMeanSlots; s++)
            if (lane + 32 * s < total)
                buf[s] = pieces[goff[s] + t * tile_pieces];
    };
    const char *at = reinterpret_cast<const char *>(staged) + row * mt.row_words * 4 + mis + (KIND == kMeanPcm ? 2 * role : 0);

    MeanChain chain;
    fetch(0);
    for (int t = 0; t < kFrame / kMeanTile; t++) {
        __syncwarp();
#pragma unroll
        for (int s = 0; s < kMeanSlots; s++)
            if (lane + 32 * s < total) {
                staged[soff[s]] = buf[s].x;
                staged[soff[s] + 1] = buf[s].y;
                staged[soff[s] + 2] = buf[s].z;
                staged[soff[s] + 3] = buf[s].w;
            }
        __syncwarp();
        if (t + 1 < kFrame / kMeanTile)
            fetch(t + 1);
#pragma unroll 8
        for (int j = 0; j < kMeanTile; j++) {
            int x;
            if (KIND == kMeanPcm) {
                x = *reinterpret_cast<const int16_t *>(at + j * mt.step);
            } else if (KIND == kMeanStereo) {
                const uint32_t pair = *reinterpret_cast<const uint32_t *>(at + 4 * j);
                const int a = (int)(pair << 16) >> 16, b = (int)pair >> 16;
                x = role == 0 ? a : role == 1 ? b : a - b;
            } else {
                x = *reinterpret_cast<const int32_t *>(at + 4 * j);
            }
            chain.add(x);
        }
    }
    if (u < n_units)
        means[u] = chain.mean();
}

inline size_t unit_means_smem_bytes(const MeanTiling &mt) { return (size_t)mt.rows_max * mt.row_words * 4; }

// ------------------------------------------------------------------ encode --
//
// Five launches, no inter-CTA dependency inside any of them:
//   k_unit_means     one LANE per analysis unit: the mean of its samples (see above).
//   k_encode_units   one WARP per analysis unit (a channel, or for stereo the three
//                    candidates ch0 / ch1 / ch0-ch1 of a frame): PCM -> autocorrelation ->
//                    Schur -> quantise -> step-up -> FIR -> Rice parameter search -> Rice
//                    pack into the unit's private slot of a scratch arena + a 32-byte
//                    unit record.  No barriers, no atomics between units.
//   k_encode_sizes,  1024 subframes per CTA: stereo decision (difference wins iff strictly fewer
//   k_encode_scan    words, src/frame/frame_encoder.cpp:63-72), exclusive prefix sum of the chosen
//                    sizes in file order, descriptors, total (see there).
//   k_encode_gather  one warp per emitted subframe: slot -> final arena offset.

constexpr uint32_t kSlotWords = 1600;     // per-unit scratch slot (refl words first, then residue words)
constexpr uint32_t kSlotReflWords = 32;   // 100 coefficients * (8 + 1) bits <= 29 words

struct __align__(16) UnitRecord {         // 32 bytes
    uint32_t order;
    uint32_t refl_k, refl_words;
    uint32_t res_k, res_words;
    uint32_t flags;                       // 1 = too large for the slot / the uint16 fields
    uint32_t pad[2];
};

struct EncodeParams {
    const int16_t *pcm;            // [n_frames][2048][channels] interleaved
    uint32_t n_frames, channels;
    selab200_subframe_desc *descs; // [n_frames*channels]
    uint32_t *words;
    unsigned long long capacity;   // words
    unsigned long long *words_used;
    int32_t *status;
    UnitRecord *units;             // workspace [n_units]
    uint32_t *slots;               // workspace [n_units][kSlotWords]
    double *means;                 // workspace [n_units]: k_unit_means
    int32_t *residues;             // workspace [n_units][2048]: FIR output, re-read by the Rice stages (L2-resident)
};

__host__ __device__ inline uint32_t encode_units(uint32_t n_frames, uint32_t channels)
{
    return channels == 2 ? n_frames * 3u : n_frames * channels;
}

// ---- lossless repair (DESIGN.md 7.2) ----
// A unit whose FIR has a tie does not decode back to its source.  The repair codes it with a slightly different
// predictor, chosen from the candidates of a unit of order o >= 2 with quantised coefficients q[0..o):
//   round 1: q[j] - 1, q[j] + 1 for j = 0, 1, o-1 (increasing j, each once), then order o-1;
//   round 2: q[j] - 1, q[j] + 1 for every other j (2 .. o-2), then orders o-2, o-3, .. 1.
// An edit that leaves [-64, 63] is no candidate.  Order 1 has no tie (c[1] = 0), so round 2 always has one.  The
// winner is the tie-free candidate of the first round that has any with the fewest words, ties to the earlier
// candidate.  Candidates are numbered 0 .. 3o-2 in this order, round 1 first.
struct PredictorEdit {
    int order, j, delta; // code at `order`; q[j] += delta where delta != 0
};
__host__ __device__ inline int repair_round1(int o) { return o == 2 ? 5 : 7; }
__host__ __device__ inline int repair_candidates(int o) { return o < 2 ? 0 : 3 * o - 1; }
constexpr int kRepairRound2Max = 3 * kMaxOrder - 1 - 7;
__host__ __device__ inline PredictorEdit repair_edit(int o, int c)
{
    PredictorEdit e{o, 0, 0};
    const int n1 = repair_round1(o);
    if (c < n1) {
        if (c == n1 - 1) {
            e.order = o - 1;
        } else {
            e.j = (c >> 1) < 2 ? (c >> 1) : o - 1;
            e.delta = (c & 1) ? 1 : -1;
        }
        return e;
    }
    c -= n1;
    const int n_edits = o > 3 ? 2 * (o - 3) : 0;
    if (c < n_edits) {
        e.j = 2 + (c >> 1);
        e.delta = (c & 1) ? 1 : -1;
    } else {
        e.order = o - 2 - (c - n_edits);
    }
    return e;
}

// A unit being repaired: its index in the batch, its order as analysed, and the best candidate so far as the key
// round << 63 | words << 32 | candidate (all ones: none yet), so that one atomicMin keeps the winner.
struct RepairUnit {
    uint32_t unit, order;
    unsigned long long best;
};
constexpr unsigned long long kNoCandidate = ~0ull;

// ---- order search (DESIGN.md 7.3) ----
// What the search's analysis leaves per unit for the candidate kernels (search.cuh): all 100 quantised reflection
// coefficients, the reference encoder's order and its words (reflection + residue), and the best order so far as the
// key words << 8 | (order == ref_order ? 0 : order), so that one atomicMin keeps the fewest words and, between equal
// words, the reference order, else the lowest.  q is kept as int32, as the quantiser produces it.
struct __align__(16) SearchUnit {
    int32_t q[kMaxOrder];
    uint32_t ref_order, ref_words;
    unsigned long long best;
};
static_assert(sizeof(SearchUnit) == 416, "SearchUnit layout");

// The search trace (tests only, selab200_encode_search_trace): the record of unit `unit` at order o, written by the
// warp that sized that order, once its FIR (predictor cf, residues res, tie) and both Rice choices are done.  The
// digests are those of include/sela_b200.h, over c[1..100] as the FIR read them and the whole residue row.
constexpr unsigned long long kDigestK = 0x9E3779B97F4A7C15ull, kDigestK2 = 0xD6E8FEB86659FD93ull;
__device__ __noinline__ void search_trace_record(selab200_search_trace *trace, uint32_t unit, int o,
                                                 const CoefSmem &cf, const int32_t *res, bool tie, RiceChoice cq,
                                                 RiceChoice cr)
{
    const int lane = lane_id();
    __syncwarp();
    unsigned long long dp = 0, dr = 0;
    for (int j = lane + 1; j <= kMaxOrder; j += 32)
        dp += ((unsigned long long)coef_at(cf, j) + (unsigned long long)j * kDigestK2) * kDigestK;
    for (int i = lane; i < kFrame; i += 32)
        dr += ((unsigned long long)i << 32 | (uint32_t)res[i]) * kDigestK;
    dp = warp_sum_u64(dp);
    dr = warp_sum_u64(dr);
    if (lane == 0) {
        selab200_search_trace &r = trace[(size_t)unit * kMaxOrder + (o - 1)];
        r.pred_digest = dp;
        r.res_digest = dr;
        r.res_words = cr.words;
        r.refl_words = (uint16_t)cq.words;
        r.refl_k = (uint8_t)cq.k;
        r.res_k = (uint8_t)cr.k;
        r.tie = tie ? 1 : 0;
        atomicAdd(&r.visits, 1u);
    }
    __syncwarp();
}

// ---- the coding tail of every warp that codes a unit (encode_unit, pair_unit in pairing.cuh, search_orders in
// search.cuh) ----

// The residue row res is dead.  It only ever lived in L2 (written and re-read by this warp within microseconds); tell
// L2 to drop the dirty lines instead of writing 8 KB back to HBM.
__device__ __forceinline__ void discard_row(int32_t *res)
{
    __syncwarp();
    for (int l = lane_id(); l < kFrame * 4 / 128; l += 32)
        asm volatile("discard.global.L2 [%0], 128;" ::"l"(res + l * 32) : "memory");
}

// Every q of an analysis into dst[0..100) for the order search: from k[] (still intact), or as forced (cf.q).
__device__ __forceinline__ void copy_every_q(int32_t *dst, const CoefSmem &cf, AnalysisScratch &scratch, bool forced)
{
    for (int i = lane_id(); i < kMaxOrder; i += 32)
        dst[i] = forced ? cf.q[i] : quantise_reflection(i, scratch.kk()[i]);
    __syncwarp();
}

// The predictor q[0..order) and the residue row Rice-packed into the slot of unit `unit`, if both fit; returns
// whether they do not (flag 1 of the record).
__device__ __forceinline__ bool pack_slot(const EncodeParams &p, uint32_t unit, const int32_t *q, int order,
                                          const int32_t *res, RiceChoice cq, RiceChoice cr)
{
    const bool too_large = cq.words > kSlotReflWords || cr.words > kSlotWords - kSlotReflWords;
    uint32_t *slot = p.slots + (size_t)unit * kSlotWords;
    if (!too_large) {
        warp_rice_pack(q, order, cq, slot);
        warp_rice_pack(res, kFrame, cr, slot + kSlotReflWords);
    }
    return too_large;
}

// Lane 0 writes the record of unit `unit`.
__device__ __forceinline__ void write_record(const EncodeParams &p, uint32_t unit, int order, RiceChoice cq,
                                             RiceChoice cr, uint32_t flags)
{
    if (lane_id() == 0) {
        UnitRecord u;
        u.order = order;
        u.refl_k = cq.k;
        u.refl_words = cq.words;
        u.res_k = cr.k;
        u.res_words = cr.words;
        u.flags = flags;
        u.pad[0] = u.pad[1] = 0;
        p.units[unit] = u;
    }
}

// Lane 0 writes the reference order's entry of a search record: the order, its words, and as the best so far that
// order (key words << 8 | 0), if it has no tie.
__device__ __forceinline__ void write_search_ref(SearchUnit &s, int order, RiceChoice cq, RiceChoice cr, bool tie)
{
    if (lane_id() == 0) {
        s.ref_order = order;
        s.ref_words = cq.words + cr.words;
        s.best = tie ? kNoCandidate : (unsigned long long)(cq.words + cr.words) << 8;
    }
}

// What encode_unit does with the unit:
//   kUnitEncode     analyse, FIR, Rice, pack into the unit's slot and write its record (production)
//   kUnitCheck      kUnitEncode, and bit 1 of the record's flags when the FIR has a tie
//   kUnitCandidate  analyse, apply candidate `cand`, FIR with the tie check, Rice sizes: a tie-free candidate enters
//                   ru->best; nothing is packed
//   kUnitRepack     analyse, apply candidate `cand`, FIR, Rice, pack into the unit's slot and rewrite its record
//   kUnitSearch     kUnitEncode with the tie check, and su[unit] filled in: every q, the reference order and words,
//                   and as the best so far the reference order, if it has no tie
enum { kUnitEncode = 0, kUnitCheck = 1, kUnitCandidate = 2, kUnitRepack = 3, kUnitSearch = 4 };

// Stages the signal of analysis unit `unit` at smem, as one planar int16 row with kHistoryPad zeros in front (for a
// stereo difference d = ch0 - ch1: d >> 1 in the row, d & 1 in the bit array behind it).
template <bool STEREO>
__device__ __forceinline__ Signal stage_unit(const EncodeParams &p, const uint32_t unit, unsigned char *smem)
{
    constexpr int kRow = kHistoryPad + kFrame;
    int16_t *s16 = reinterpret_cast<int16_t *>(smem);                    // [pad + 2048]
    uint32_t *lo_bits = reinterpret_cast<uint32_t *>(smem + kRow * 2);    // [pad/32 + 64] (stereo only)
    const int lane = lane_id();
    const uint32_t frame = STEREO ? unit / 3 : unit / p.channels;
    const uint32_t role = STEREO ? unit % 3 : unit % p.channels; // stereo: 0 ch0, 1 ch1, 2 ch0-ch1

    // ---- stage the signal (de-interleave to one planar int16 row, zero history in front) ----
    const int16_t *src = p.pcm + (size_t)frame * kFrame * p.channels;
    for (int j = lane; j < kHistoryPad / 2; j += 32)
        reinterpret_cast<uint32_t *>(s16)[j] = 0;
    int16_t *row = s16 + kHistoryPad;
    Signal sig;
    sig.a = row;
    sig.lo = nullptr;
    if (STEREO) {
        const uint4 *src128 = reinterpret_cast<const uint4 *>(src); // 4 stereo sample pairs per load
        if (role < 2) {
            const uint32_t sel = role ? 0x7632 : 0x5410;
            for (int j = lane; j < kFrame / 4; j += 32) {
                const uint4 v = src128[j];
                reinterpret_cast<uint2 *>(row)[j] = make_uint2(__byte_perm(v.x, v.y, sel), __byte_perm(v.z, v.w, sel));
            }
        } else {
            // difference d = ch0 - ch1 (17 bits): d >> 1 into the row, d & 1 into the bit array
            if (lane < kHistoryPad / 32)
                lo_bits[lane] = 0;
            uint32_t *lo = lo_bits + kHistoryPad / 32;
            for (int it = 0; it < kFrame / 128; it++) {
                const uint4 v = src128[it * 32 + lane];
                const uint32_t pr[4] = {v.x, v.y, v.z, v.w};
                int d[4];
#pragma unroll
                for (int e = 0; e < 4; e++)
                    d[e] = ((int)(pr[e] << 16) >> 16) - ((int)pr[e] >> 16);
                const uint32_t h01 = ((uint32_t)(d[0] >> 1) & 0xffffu) | ((uint32_t)(d[1] >> 1) << 16);
                const uint32_t h23 = ((uint32_t)(d[2] >> 1) & 0xffffu) | ((uint32_t)(d[3] >> 1) << 16);
                reinterpret_cast<uint2 *>(row)[it * 32 + lane] = make_uint2(h01, h23);
                uint32_t nib = (d[0] & 1) | ((d[1] & 1) << 1) | ((d[2] & 1) << 2) | ((d[3] & 1) << 3);
                nib <<= 4 * (lane & 7);
                nib |= __shfl_xor_sync(kFull, nib, 1);
                nib |= __shfl_xor_sync(kFull, nib, 2);
                nib |= __shfl_xor_sync(kFull, nib, 4);
                if ((lane & 7) == 0)
                    lo[it * 4 + (lane >> 3)] = nib;
            }
            sig.lo = lo;
        }
    } else {
        for (int j = lane; j < kFrame; j += 32)
            row[j] = src[(size_t)j * p.channels + role];
    }
    __syncwarp();
    return sig;
}

// Stages d = ch_par - ch_c of `frame` (17 bits) at smem as stage_unit stages the stereo difference: d >> 1 in the
// int16 row, d & 1 in the bit array behind it, kHistoryPad zeros in front of both.  The channel pairing's candidates
// (pairing.cuh, search_pairing.cuh).
__device__ __forceinline__ Signal stage_pair(const EncodeParams &p, uint32_t frame, uint32_t par, uint32_t c,
                                             unsigned char *smem)
{
    constexpr int kRow = kHistoryPad + kFrame;
    int16_t *s16 = reinterpret_cast<int16_t *>(smem);
    uint32_t *lo_bits = reinterpret_cast<uint32_t *>(smem + kRow * 2);
    const int lane = lane_id();
    const int16_t *src = p.pcm + (size_t)frame * kFrame * p.channels;
    for (int j = lane; j < kHistoryPad / 2; j += 32)
        reinterpret_cast<uint32_t *>(s16)[j] = 0;
    if (lane < kHistoryPad / 32)
        lo_bits[lane] = 0;
    int16_t *row = s16 + kHistoryPad;
    uint32_t *lo = lo_bits + kHistoryPad / 32;
    for (int it = 0; it < kFrame / 32; it++) {
        const size_t j = (size_t)(it * 32 + lane) * p.channels;
        const int d = (int)src[j + par] - (int)src[j + c];
        row[it * 32 + lane] = (int16_t)(d >> 1);
        const uint32_t bits = __ballot_sync(kFull, d & 1);
        if (lane == 0)
            lo[it] = bits;
    }
    __syncwarp();
    Signal sig;
    sig.a = row;
    sig.lo = lo;
    return sig;
}

// Shared memory of the signal staged by stage_unit.
template <bool STEREO>
__host__ __device__ constexpr size_t unit_signal_bytes()
{
    return (size_t)(kHistoryPad + kFrame) * 2 + (STEREO ? (kHistoryPad + kFrame) / 8 : 0);
}

// The work of one analysis unit by one warp.
// TRACE (tests only, selab200_encode_trace): also copies the unit's analysis intermediates to trace[unit] as they
// are produced.  Production runs TRACE = false, where none of it exists and `trace` is null.  In kUnitSearch
// (selab200_encode_search_trace) TRACE writes the reference order's search record to strace instead.
// FORCE (tests only, selab200_encode_lossless_forced): the unit is coded with the predictor pred[unit] in place of the
// one its analysis chose; every step after the quantiser, the repair's edits included, runs as in production.
// SEARCH (kUnitSearch only): the units' search records.
template <bool STEREO, bool TRACE, int MODE, bool FORCE = false>
__device__ __forceinline__ void encode_unit(const EncodeParams &p, selab200_analysis_trace *trace, const uint32_t unit,
                                            RepairUnit *ru, uint32_t cand, const selab200_predictor *pred = nullptr,
                                            SearchUnit *su = nullptr, selab200_search_trace *strace = nullptr)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr size_t kSigBytes = unit_signal_bytes<STEREO>();
    AnalysisScratch &scratch = *reinterpret_cast<AnalysisScratch *>(smem_raw + kSigBytes);
    // The predictor lives in the part of the analysis scratch that is dead once the Schur recursion has taken
    // the autocorrelation into registers (the tail of the ring and ac[]): 7.7 instead of 9 KB per unit, 29
    // instead of 23 units per SM.
    static_assert(kCoefAlias + sizeof(CoefSmem) <= sizeof(AnalysisScratch) && kCoefAlias % 16 == 0, "predictor alias");
    CoefSmem &cf = *reinterpret_cast<CoefSmem *>(smem_raw + kSigBytes + kCoefAlias);

    const int lane = lane_id();
    const uint32_t role = STEREO ? unit % 3 : unit % p.channels; // stereo: 0 ch0, 1 ch1, 2 ch0-ch1
    const Signal sig = stage_unit<STEREO>(p, unit, smem_raw);

    // ---- analysis ----
    // the residue row: the unit's own, or in the repair (which runs several candidates of a unit at once) the warp's
    int32_t *res = p.residues + (size_t)(MODE == kUnitEncode || MODE == kUnitCheck ? unit : blockIdx.x) * kFrame;
    // one lane loads the mean and the warp gets it by shuffle: a warp-wide load of p.means[unit] moves the unit
    // index out of the uniform registers, and the stereo kernel then needs 78 registers instead of 72
    warp_autocorrelation(sig, scratch, shfl_d(lane == 0 ? p.means[unit] : 0.0, 0));
    constexpr bool kTraceAnalysis = TRACE && MODE != kUnitSearch;
    if constexpr (kTraceAnalysis) { // before warp_schur: the predictor overlays ac[] from warp_order_and_quantise on
        selab200_analysis_trace &tr = trace[unit];
        if (lane == 0)
            tr.mean = p.means[unit];
        for (int i = lane; i <= kMaxOrder; i += 32)
            tr.ac[i] = scratch.ac[i];
    }
    warp_schur(scratch);
    int order = warp_order_and_quantise(scratch, cf);
    if constexpr (FORCE) { // q past the forced order is zero (the entry point checks it), as the quantiser leaves it
        const selab200_predictor &f = pred[unit];
        for (int i = lane; i < kMaxOrder; i += 32)
            cf.q[i] = f.q[i];
        order = f.order;
        __syncwarp();
    }
    if constexpr (MODE == kUnitCandidate || MODE == kUnitRepack) {
        const PredictorEdit e = repair_edit(order, (int)cand);
        if (e.delta) {
            const int v = cf.q[e.j] + e.delta;
            if (v < -64 || v > 63)
                return; // no candidate (the whole warp)
            __syncwarp();
            if (lane == 0)
                cf.q[e.j] = v;
        } else {
            for (int i = e.order + lane; i < order; i += 32)
                cf.q[i] = 0;
        }
        __syncwarp();
        order = e.order;
    }
    warp_coefficients(cf, scratch.t(), order);
    if constexpr (kTraceAnalysis) { // k[] (ring[0, 100)) is still intact: t[] and the predictor lie behind it
        selab200_analysis_trace &tr = trace[unit];
        for (int i = lane; i < kMaxOrder; i += 32) {
            tr.k[i] = scratch.kk()[i];
            tr.q[i] = cf.q[i];
        }
        for (int i = lane; i <= kMaxOrder; i += 32)
            tr.c[i] = i == 0 ? 0 : coef_at(cf, i);
        if (lane == 0)
            tr.order = order;
    }
    if constexpr (MODE == kUnitSearch)
        copy_every_q(su[unit].q, cf, scratch, FORCE);
    // the digit planes of the FIR overlay k[] and the step-up row, dead now (the trace has copied k)
    static_assert(kPlaneBytes <= kCoefAlias, "FIR digit planes");
    uint32_t *planes = reinterpret_cast<uint32_t *>(scratch.ring);
    constexpr bool kCheck = MODE == kUnitCheck || MODE == kUnitCandidate || MODE == kUnitSearch;
    bool tie;
    if (STEREO && role == 2)
        tie = warp_fir_residual<true, kCheck>(sig, cf, order, planes, res);
    else
        tie = warp_fir_residual<false, kCheck>(sig, cf, order, planes, res);

    // ---- Rice: parameter search, then pack into this unit's slot ----
    const RiceChoice cq = warp_rice_choose(cf.q, order);
    const RiceChoice cr = warp_rice_choose(res, kFrame);
    if constexpr (TRACE && MODE == kUnitSearch)
        search_trace_record(strace, unit, order, cf, res, tie, cq, cr);
    if constexpr (MODE == kUnitCandidate) {
        discard_row(res);
        const unsigned long long round = cand >= (uint32_t)repair_round1(ru->order) ? 1ull : 0ull;
        if (lane == 0 && !tie)
            atomicMin(&ru->best, round << 63 | (unsigned long long)(cq.words + cr.words) << 32 | cand);
        return;
    }
    const bool too_large = pack_slot(p, unit, cf.q, order, res, cq, cr);
    discard_row(res);
    // flag 2: not lossless (kUnitCheck only)
    write_record(p, unit, order, cq, cr, (too_large ? 1u : 0u) | (MODE != kUnitSearch && tie ? 2u : 0u));
    if constexpr (MODE == kUnitSearch)
        write_search_ref(su[unit], order, cq, cr, tie);
}

// k_encode_units: encode_unit for unit blockIdx.x.  CHECK: the kUnitCheck instantiation (lossless encodes).
// `trace` and `pred` (FORCE, tests only) are kernel arguments of their own rather than fields of EncodeParams: a
// longer EncodeParams would move the parameter offsets of the kernels that take arguments after it.
template <bool STEREO, bool TRACE = false, bool CHECK = false, bool FORCE = false>
__global__ void __launch_bounds__(32) k_encode_units(EncodeParams p, selab200_analysis_trace *trace,
                                                     const selab200_predictor *pred)
{
    encode_unit<STEREO, TRACE, CHECK ? kUnitCheck : kUnitEncode, FORCE>(p, trace, blockIdx.x, nullptr, 0, pred);
}

template <bool STEREO>
constexpr size_t encode_smem_bytes()
{
    return (size_t)(kHistoryPad + kFrame) * 2 + (STEREO ? (kHistoryPad + kFrame) / 8 : 0) + sizeof(AnalysisScratch);
}

// Warp copy of n words, eight loads in flight per lane before the first store (a load-store-load-store loop leaves
// ONE: the in-order issue stops at every store until its load has landed).  The source is read once and dead after.
__device__ __forceinline__ void warp_copy_words(uint32_t *__restrict__ dst, const uint32_t *__restrict__ src, uint32_t n, int lane)
{
    for (uint32_t w = lane; w < n; w += 256) {
        uint32_t v[8];
#pragma unroll
        for (int j = 0; j < 8; j++)
            v[j] = w + 32 * j < n ? __ldcs(src + w + 32 * j) : 0u;
#pragma unroll
        for (int j = 0; j < 8; j++)
            if (w + 32 * j < n)
                dst[w + 32 * j] = v[j];
    }
}

// Which unit is emitted for output subframe (frame, channel), and as what.
struct Emit {
    uint32_t unit, type, parent;
};
__device__ __forceinline__ Emit choose_unit(const UnitRecord *units, uint32_t channels, uint32_t sub)
{
    Emit e;
    if (channels != 2) {
        e.unit = sub;
        e.type = 0;
        e.parent = sub % channels;
        return e;
    }
    const uint32_t frame = sub >> 1;
    if ((sub & 1) == 0) {
        e.unit = 3 * frame;
        e.type = 0;
        e.parent = 0;
        return e;
    }
    const UnitRecord a = units[3 * frame + 1], d = units[3 * frame + 2];
    const bool diff_wins = (unsigned long long)d.refl_words + d.res_words <
                           (unsigned long long)a.refl_words + a.res_words; // strictly smaller
    e.unit = 3 * frame + (diff_wins ? 2 : 1);
    e.type = diff_wins ? 1 : 0;
    e.parent = diff_wins ? 0 : 1;
    return e;
}

// The unit emitted for subframe `sub` together with its record (for a stereo side channel the winner is one of the
// two records the decision reads anyway).
__device__ __forceinline__ Emit choose_record(const UnitRecord *units, uint32_t channels, uint32_t sub, UnitRecord &u)
{
    Emit e;
    if (channels != 2 || (sub & 1) == 0) {
        e.unit = channels != 2 ? sub : 3 * (sub >> 1);
        e.type = 0;
        e.parent = channels != 2 ? sub % channels : 0;
        u = units[e.unit];
        return e;
    }
    const uint32_t frame = sub >> 1;
    const UnitRecord a = units[3 * frame + 1], d = units[3 * frame + 2];
    const bool diff_wins = (unsigned long long)d.refl_words + d.res_words <
                           (unsigned long long)a.refl_words + a.res_words; // strictly smaller
    e.unit = 3 * frame + (diff_wins ? 2 : 1);
    e.type = diff_wins ? 1 : 0;
    e.parent = diff_wins ? 0 : 1;
    u = diff_wins ? d : a;
    return e;
}

// Block-wide inclusive scan of one 64-bit value per thread (1024 threads); warp_tot[31] is the block total afterwards.
__device__ __forceinline__ unsigned long long block_scan_inclusive_u64(unsigned long long v, unsigned long long *warp_tot)
{
    const int lane = lane_id(), warp = warp_id();
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(kFull, v, o);
        if (lane >= o)
            v += t;
    }
    if (lane == 31)
        warp_tot[warp] = v;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = warp_tot[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(kFull, w, o);
            if (lane >= o)
                w += t;
        }
        warp_tot[lane] = w; // inclusive over warps
    }
    __syncthreads();
    return v + (warp ? warp_tot[warp - 1] : 0ull);
}

// The scan of the emitted sizes (stereo decision, exclusive prefix sum in file order, descriptors, fill level) in two
// launches of 1024 subframes per CTA, coalesced record loads in both:
//   k_encode_sizes   CTA b: total words of its 1024 subframes -> tmp[1 + b]           (independent of earlier chunks)
//   k_encode_scan    CTA b: fill level so far (*words_used, left by the previous chunk of a pipelined call) + the
//                    totals of the CTAs before it + a block scan -> descriptors; the last CTA leaves the new fill level
//                    in tmp[0] (the host side copies it to *words_used: other CTAs may still be reading the old one).
// tmp is the head of the residue workspace, dead once k_encode_units has finished.
constexpr uint32_t kScanTile = 1024;

__global__ void __launch_bounds__(kScanTile) k_encode_sizes(EncodeParams p)
{
    __shared__ unsigned long long warp_tot[32];
    const uint32_t n_sub = p.n_frames * p.channels;
    const uint32_t sub = blockIdx.x * kScanTile + threadIdx.x;
    unsigned long long size = 0;
    if (sub < n_sub) {
        UnitRecord u;
        choose_record(p.units, p.channels, sub, u);
        size = (unsigned long long)u.refl_words + u.res_words;
    }
    block_scan_inclusive_u64(size, warp_tot);
    if (threadIdx.x == 0)
        reinterpret_cast<unsigned long long *>(p.residues)[1 + blockIdx.x] = warp_tot[31];
}

__global__ void __launch_bounds__(kScanTile) k_encode_scan(EncodeParams p)
{
    __shared__ unsigned long long warp_tot[32];
    __shared__ unsigned long long before;
    unsigned long long *tmp = reinterpret_cast<unsigned long long *>(p.residues);
    const uint32_t n_sub = p.n_frames * p.channels;
    const uint32_t sub = blockIdx.x * kScanTile + threadIdx.x;
    const int lane = lane_id(), warp = warp_id();
    if (warp == 0) { // words in front of this CTA
        unsigned long long s = lane == 0 ? *p.words_used : 0ull;
        for (uint32_t b = lane; b < blockIdx.x; b += 32)
            s += tmp[1 + b];
        s = warp_sum_u64(s);
        if (lane == 0)
            before = s;
    }
    Emit e;
    UnitRecord u;
    unsigned long long size = 0;
    bool bad = false;
    if (sub < n_sub) {
        e = choose_record(p.units, p.channels, sub, u);
        size = (unsigned long long)u.refl_words + u.res_words;
        bad = u.flags != 0 || u.refl_words > 0xffffu || u.res_words > 0xffffu;
    }
    const unsigned long long incl = block_scan_inclusive_u64(size, warp_tot); // its barriers also publish `before`
    if (sub < n_sub) {
        const unsigned long long off = before + incl - size;
        selab200_subframe_desc v;
        v.channel = (uint8_t)(sub % p.channels);
        v.subframe_type = (uint8_t)e.type;
        v.parent_channel = (uint8_t)e.parent;
        v.refl_rice_param = (uint8_t)u.refl_k;
        v.refl_words = (uint16_t)u.refl_words;
        v.lpc_order = (uint8_t)u.order;
        v.res_rice_param = (uint8_t)u.res_k;
        v.res_words = (uint16_t)u.res_words;
        v.samples = (uint16_t)kFrame;
        v.reserved = 0;
        v.refl_offset = off;
        v.res_offset = off + u.refl_words;
        p.descs[sub] = v;
    }
    if (bad)
        raise_status(p.status, SELAB200_ERR_RANGE); // a stream the uint16 word counts cannot describe
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
        const unsigned long long fill = before + warp_tot[31];
        tmp[0] = fill;
        if (fill > p.capacity)
            raise_status(p.status, SELAB200_ERR_CAPACITY);
    }
}

// One warp per emitted subframe; 8 warps per CTA.
__global__ void __launch_bounds__(256) k_encode_gather(EncodeParams p)
{
    const uint32_t sub = blockIdx.x * 8 + warp_id();
    const uint32_t n_sub = p.n_frames * p.channels;
    if (sub >= n_sub || *reinterpret_cast<volatile int32_t *>(p.status) != 0)
        return;
    const int lane = lane_id();
    const Emit e = choose_unit(p.units, p.channels, sub);
    const selab200_subframe_desc d = p.descs[sub];
    const uint32_t *slot = p.slots + (size_t)e.unit * kSlotWords;
    warp_copy_words(p.words + d.refl_offset, slot, d.refl_words, lane);
    warp_copy_words(p.words + d.res_offset, slot + kSlotReflWords, d.res_words, lane);
}

// --------------------------------------------------------------- container --
//
// The .sela container (src/file/sela_file.cpp:105-137) is byte-packed: a 15-byte file header,
// then per frame the sync word 0xAA55FF00 (little endian: 00 FF 55 AA) and per subframe
//   channel, type, parent, reflK (u8 each), reflInts (u16), order (u8), refl words,
//   resK (u8), resInts (u16), samples (u16), residue words.
// With the word arena laid out in file order (refl words then residue words, subframe after
// subframe), the byte position of everything follows from the subframe's global index g, its
// frame f = g / channels and the arena offset W of its first word:
//   header of g at  15 + 4*(f+1) + 12*g + 4*W.
// Word arrays therefore sit at arbitrary byte alignments; the kernels below move them with
// aligned 32-bit accesses and a funnel shift, byte stores only at the two ragged ends.
constexpr unsigned long long kContainerHeaderBytes = 15;
constexpr uint32_t kSubframeHeaderBytes = 12;

__device__ __forceinline__ unsigned long long container_subframe_byte(unsigned long long g, uint32_t channels,
                                                                       unsigned long long first_word)
{
    return kContainerHeaderBytes + 4ull * (g / channels + 1) + (unsigned long long)kSubframeHeaderBytes * g +
           4ull * first_word;
}

// n words from src (aligned) to byte address out + D (any alignment).
__device__ __forceinline__ void put_words_at_byte(uint8_t *out, unsigned long long D, const uint32_t *src, uint32_t n)
{
    const int lane = lane_id();
    if (n == 0)
        return;
    const uint32_t s = (uint32_t)(D & 3);
    uint32_t *dst = reinterpret_cast<uint32_t *>(out + (D - s));
    if (s == 0) {
        warp_copy_words(dst, src, n, lane);
        return;
    }
    // aligned word t = high bytes of src[t-1], low bytes of src[t]; four words per lane loaded before the first store
    for (uint32_t t0 = 1 + lane; t0 < n; t0 += 128) {
        uint32_t v[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t t = t0 + 32 * j;
            v[j] = t < n ? __funnelshift_l(src[t - 1], src[t], 8 * s) : 0u;
        }
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (t0 + 32 * j < n)
                dst[t0 + 32 * j] = v[j];
    }
    if (lane < (int)(4 - s))
        out[D + lane] = (uint8_t)(src[0] >> (8 * lane));
    else if (lane >= 4 && lane < (int)(4 + s))
        out[D - s + 4ull * n + (lane - 4)] = (uint8_t)(src[n - 1] >> (8 * (4 - s + (lane - 4))));
}

// n words from byte address in + D (any alignment) to dst (aligned).  Reads the aligned word
// that holds the last byte, i.e. at most 3 bytes past the array (the buffer is padded).
__device__ __forceinline__ void get_words_at_byte(const uint8_t *in, unsigned long long D, uint32_t *dst, uint32_t n)
{
    const int lane = lane_id();
    const uint32_t s = (uint32_t)(D & 3);
    const uint32_t *src = reinterpret_cast<const uint32_t *>(in + (D - s));
    for (uint32_t t0 = lane; t0 < n; t0 += 128) { // four words per lane loaded before the first store
        uint32_t v[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t t = t0 + 32 * j;
            v[j] = t < n ? (s ? __funnelshift_r(src[t], src[t + 1], 8 * s) : src[t]) : 0u;
        }
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (t0 + 32 * j < n)
                dst[t0 + 32 * j] = v[j];
    }
}

// Encoder output straight into the container: k_encode_gather with byte-packed destinations
// and the headers written in place.  One warp per emitted subframe; `sub_base` is the global
// index of this chunk's first subframe.
__global__ void __launch_bounds__(256) k_encode_gather_container(EncodeParams p, uint8_t *container,
                                                                 unsigned long long sub_base)
{
    const uint32_t sub = blockIdx.x * 8 + warp_id();
    const uint32_t n_sub = p.n_frames * p.channels;
    if (sub >= n_sub || *reinterpret_cast<volatile int32_t *>(p.status) != 0)
        return;
    const int lane = lane_id();
    const Emit e = choose_unit(p.units, p.channels, sub);
    const selab200_subframe_desc d = p.descs[sub];
    const uint32_t *slot = p.slots + (size_t)e.unit * kSlotWords;
    const unsigned long long g = sub_base + sub;
    const unsigned long long at = container_subframe_byte(g, p.channels, d.refl_offset);
    if (g % p.channels == 0 && lane >= 12 && lane < 16) {
        const uint32_t sync = 0xAA55FF00u;
        container[at - 4 + (lane - 12)] = (uint8_t)(sync >> (8 * (lane - 12)));
    }
    const unsigned long long at2 = at + 7 + 4ull * d.refl_words;
    if (lane < 12) {
        uint8_t v;
        switch (lane) {
        case 0: v = d.channel; break;
        case 1: v = d.subframe_type; break;
        case 2: v = d.parent_channel; break;
        case 3: v = d.refl_rice_param; break;
        case 4: v = (uint8_t)d.refl_words; break;
        case 5: v = (uint8_t)(d.refl_words >> 8); break;
        case 6: v = d.lpc_order; break;
        case 7: v = d.res_rice_param; break;
        case 8: v = (uint8_t)d.res_words; break;
        case 9: v = (uint8_t)(d.res_words >> 8); break;
        case 10: v = (uint8_t)d.samples; break;
        default: v = (uint8_t)(d.samples >> 8); break;
        }
        container[lane < 7 ? at + lane : at2 + (lane - 7)] = v;
    }
    put_words_at_byte(container, at + 7, slot, d.refl_words);
    put_words_at_byte(container, at2 + 5, slot + kSlotReflWords, d.res_words);
}

// Decoder input straight from the container: realign the word arrays of each subframe into the
// (16-byte aligned) arena the Rice decoder reads.  descs[] come from the host's header walk and
// carry arena offsets in file order.  One warp per subframe.
__global__ void __launch_bounds__(256) k_container_unpack(const uint8_t *container, const selab200_subframe_desc *descs,
                                                          uint32_t n_sub, uint32_t channels, unsigned long long sub_base,
                                                          uint32_t *arena)
{
    const uint32_t sub = blockIdx.x * 8 + warp_id();
    if (sub >= n_sub)
        return;
    const selab200_subframe_desc d = descs[sub];
    const unsigned long long at = container_subframe_byte(sub_base + sub, channels, d.refl_offset);
    get_words_at_byte(container, at + 7, arena + d.refl_offset, d.refl_words);
    get_words_at_byte(container, at + 7 + 4ull * d.refl_words + 5, arena + d.res_offset, d.res_words);
}

// ------------------------------------------------------------------ decode --

// Acceptance of a whole frame (its ch descriptors fd[0..ch)): every subframe passes desc_ok (common.cuh), the channel fields form
// a permutation and every parent is an independent subframe.  The host applies it too (the channel-selecting clip
// decode checks every covered frame, decoded subframes or not).
__host__ __device__ __forceinline__ bool frame_check(const selab200_subframe_desc *fd, uint32_t ch, unsigned long long n_words)
{
    bool ok = true;
    unsigned seen = 0, type_mask = 0; // by channel: seen, difference-coded
    for (uint32_t i = 0; i < ch; i++) {
        const selab200_subframe_desc d = fd[i];
        const bool good = desc_ok(d, ch, n_words) && !((seen >> d.channel) & 1);
        ok &= good;
        if (good) {
            seen |= 1u << d.channel;
            type_mask |= (unsigned)(d.subframe_type & 1) << d.channel;
        }
    }
    for (uint32_t i = 0; i < ch && ok; i++) {
        const selab200_subframe_desc d = fd[i];
        if (d.subframe_type == 1 && ((type_mask >> d.parent_channel) & 1))
            ok = false;
    }
    return ok;
}

struct DecodeParams {
    const selab200_subframe_desc *descs;
    uint32_t n_frames, channels;
    const uint32_t *words;
    unsigned long long n_words;
    int16_t *pcm_out;
    int32_t *status;
    int32_t *ws_q;   // [n_sub][128]
    int32_t *ws_res; // [n_sub][2048]
    uint32_t *seg_index; // [synthesis_warps(n_sub)][32]: subframe whose segment starts at that lane (k_decode_plan)
    const uint32_t *rice_flags; // residue pass of k_rice_decode: when set, only streams with a non-zero flag (rice_vs.cuh)
};

// K5: one lane per stream, 2 warps per CTA.  which = 0: reflection streams (-> ws_q), 1: residue
// streams (-> ws_res).
constexpr int kRiceWarps = 2;
constexpr int kRiceRing = 64, kRiceBatch = 8;
template <int RING, int BATCH>
__global__ void __launch_bounds__(32 * kRiceWarps) k_rice_decode(DecodeParams p, int which)
{
    __shared__ uint32_t ring[kRiceWarps][(RING + 1) * 32];
    const uint32_t sub = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n_sub = p.n_frames * p.channels;
    RiceLaneStream st;
    st.src = p.words;
    st.n_words = 0;
    st.k = 0;
    st.count = 0;
    st.out = nullptr;
    if (sub < n_sub) {
        const selab200_subframe_desc d = p.descs[sub];
        if (!desc_ok(d, p.channels, p.n_words)) {
            raise_status(p.status, SELAB200_ERR_BITSTREAM);
        } else if (which == 0) {
            st.src = p.words + d.refl_offset;
            st.n_words = d.refl_words;
            st.k = d.refl_rice_param;
            st.count = d.lpc_order;
            st.out = p.ws_q + (size_t)sub * 128;
        } else if (!p.rice_flags || p.rice_flags[sub]) {
            st.src = p.words + d.res_offset;
            st.n_words = d.res_words;
            st.k = d.res_rice_param;
            st.count = d.samples;
            st.out = p.ws_res + (size_t)sub * kFrame;
        }
    }
    if (which == 1 && p.rice_flags && __ballot_sync(kFull, st.count != 0) == 0)
        return; // nothing flagged in this warp (the usual case)
    if (!warp_rice_decode32<RING, BATCH>(ring[warp_id()], st))
        raise_status(p.status, SELAB200_ERR_BITSTREAM);
}

// Packing plan of the batch synthesis kernel: which subframes share a warp, and on which lanes.  A warp holds
// segments of widths 1..kMaxWidth lanes (segment_width) summing to at most 32.  Subframes of the same width are
// interchangeable, so the plan is made from the width counts alone, as a short list of warp TEMPLATES: the widest
// width left opens a warp, which is then filled greedily, widest first, with whatever still fits; the template is
// repeated as often as the counts allow.  Templates are laid out widest first, so the warps with the most lanes in
// use start first.  Every template either takes the last subframes of some width or is followed by one that does
// (after a template limited by room, the first width it exhausted to below its copies is taken whole by the next),
// so there are at most 2 * kMaxWidth templates.  Every warp but the last holds at least two segments, so there are
// at most n_sub / 2 + 1 warps.  On the BASELINE synthetic 93 % of the issued multiply slots are predictor taps.
//   k_decode_width_counts  CTA b: how many of its subframes have each width -> tmp[b]
//   k_decode_plan          CTA b: width totals of all CTAs -> templates (every CTA computes them, one thread);
//                          counts of the CTAs before it + the rank inside the CTA -> the subframe's rank among its
//                          width -> template, repeat and lane: seg_index[warp][first lane] = subframe.
// tmp is the head of the Rice decoder's scratch, which is not in use yet.  seg_index is pre-set to kNoSegment.
constexpr uint32_t kNoSegment = 0xffffffffu;
constexpr int kMaxTemplates = 2 * kMaxWidth;

struct WidthCounts {
    uint32_t n[16]; // by segment width; [0]: no subframe
};
struct SegTemplate {
    uint32_t repeats, first_warp;
    uint8_t copies[16], lane0[16]; // by width: segments per warp, first lane of the first of them
};

__device__ __forceinline__ int subframe_width(const DecodeParams &p, uint32_t u)
{
    const int order = p.descs[u].lpc_order;
    return segment_width(order > kMaxOrder ? 0 : order);
}

// Per-warp width counts of a 1024-thread CTA into cnt[warp][width]; returns the thread's rank among the threads of
// its warp with the same width.
__device__ __forceinline__ uint32_t warp_width_counts(int w, uint32_t (*cnt)[16])
{
    const int lane = lane_id();
    uint32_t rank = 0;
#pragma unroll
    for (int v = 0; v < 16; v++) {
        const unsigned b = __ballot_sync(kFull, w == v);
        if (w == v)
            rank = __popc(b & ((1u << lane) - 1u));
        if (lane == 0)
            cnt[warp_id()][v] = __popc(b);
    }
    return rank;
}

__global__ void __launch_bounds__(kScanTile) k_decode_width_counts(DecodeParams p, WidthCounts *tmp)
{
    __shared__ uint32_t cnt[32][16];
    const uint32_t u = blockIdx.x * kScanTile + threadIdx.x;
    warp_width_counts(u < p.n_frames * p.channels ? subframe_width(p, u) : 0, cnt);
    __syncthreads();
    if (threadIdx.x < 16) {
        uint32_t s = 0;
        for (int w = 0; w < 32; w++)
            s += cnt[w][threadIdx.x];
        tmp[blockIdx.x].n[threadIdx.x] = s;
    }
}

// The templates for the width counts c[1..kMaxWidth]; returns how many.
__device__ int segment_templates(uint32_t (&c)[16], SegTemplate *tpl)
{
    int nt = 0;
    uint32_t warp = 0;
    for (;;) {
        SegTemplate t;
        int room = 32;
        uint32_t rep = 0xffffffffu;
#pragma unroll
        for (int v = 15; v >= 1; v--) {
            const uint32_t k = v > kMaxWidth ? 0u : min(c[v], (uint32_t)(room / v));
            t.copies[v] = (uint8_t)k;
            t.lane0[v] = (uint8_t)(32 - room);
            room -= (int)k * v;
            if (k)
                rep = min(rep, c[v] / k);
        }
        if (room == 32)
            return nt;
#pragma unroll
        for (int v = 1; v < 16; v++)
            c[v] -= rep * t.copies[v];
        t.copies[0] = t.lane0[0] = 0;
        t.repeats = rep;
        t.first_warp = warp;
        warp += rep;
        tpl[nt++] = t;
    }
}

__global__ void __launch_bounds__(kScanTile) k_decode_plan(DecodeParams p, const WidthCounts *tmp)
{
    __shared__ uint32_t cnt[32][16];
    __shared__ uint32_t part_all[kScanTile / 16][16], part_before[kScanTile / 16][16];
    __shared__ uint32_t total[16], before[16];
    __shared__ SegTemplate tpl[kMaxTemplates];
    const uint32_t n_units = p.n_frames * p.channels;
    const uint32_t u = blockIdx.x * kScanTile + threadIdx.x;
    const int w = u < n_units ? subframe_width(p, u) : 0;
    const uint32_t rank = warp_width_counts(w, cnt);
    {
        const int v = threadIdx.x & 15, g = threadIdx.x >> 4;
        uint32_t all = 0, pre = 0;
        for (uint32_t b = g; b < gridDim.x; b += kScanTile / 16) {
            const uint32_t x = tmp[b].n[v];
            all += x;
            if (b < blockIdx.x)
                pre += x;
        }
        part_all[g][v] = all;
        part_before[g][v] = pre;
    }
    __syncthreads();
    if (threadIdx.x < 16) {
        const int v = threadIdx.x;
        uint32_t all = 0, pre = 0, run = 0;
        for (int g = 0; g < kScanTile / 16; g++)
            all += part_all[g][v], pre += part_before[g][v];
        total[v] = all;
        before[v] = pre;
        for (int x = 0; x < 32; x++) { // exclusive prefix over the warps of this CTA
            const uint32_t c = cnt[x][v];
            cnt[x][v] = run;
            run += c;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t c[16];
#pragma unroll
        for (int v = 0; v < 16; v++)
            c[v] = v ? total[v] : 0u;
        segment_templates(c, tpl);
    }
    __syncthreads();
    if (u >= n_units)
        return;
    const uint32_t r = before[w] + cnt[warp_id()][w] + rank; // rank among all subframes of width w
    uint32_t acc = 0;
    int t = 0;
    for (;; t++) {
        const uint32_t m = tpl[t].repeats * tpl[t].copies[w];
        if (r < acc + m)
            break;
        acc += m;
    }
    const uint32_t k = tpl[t].copies[w], j = r - acc, rep = j / k;
    const uint32_t lane = tpl[t].lane0[w] + (j - rep * k) * (uint32_t)w;
    p.seg_index[((size_t)tpl[t].first_warp + rep) * 32 + lane] = u;
}

// Upper bound of the number of synthesis warps (see above).
__host__ __device__ inline size_t synthesis_warps(size_t n_sub) { return n_sub / 2 + 1; }

// K6, batch form: one warp = the segments k_decode_plan put there (segment_synthesis), every valid frame at any
// channel count.  A difference-coded subframe leaves its decoded difference in its residue row for k_diff_fixup.
__global__ void __launch_bounds__(32) k_synthesise_segments(DecodeParams p)
{
    __shared__ __align__(16) SegSmem sm;
    const uint32_t ch = p.channels;
    const int lane = lane_id();
    const uint32_t entry = p.seg_index[(size_t)blockIdx.x * 32 + lane];
    const unsigned starts = __ballot_sync(kFull, entry != kNoSegment);
    if (!(starts & 1u))
        return; // beyond the last warp of the plan
    const int start = 31 - __clz(starts & (0xffffffffu >> (31 - lane))); // the last segment start at or below
    const uint32_t sub = __shfl_sync(kFull, entry, start);
    const int seg = __popc(starts & ((1u << start) - 1u)); // segment ordinal
    const int n_seg = __popc(starts);
    const int k = lane - start;
    const uint32_t frame = sub / ch, pos = sub % ch;
    const selab200_subframe_desc *fd = p.descs + (size_t)frame * ch;
    const int n = subframe_width(p, sub);
    const bool exists = k < n; // lanes past the last segment hold zero taps and store nothing

    const bool frame_ok = frame_check(fd, ch, p.n_words); // every lane of the segment redundantly
    if (!frame_ok && k == 0)
        raise_status(p.status, SELAB200_ERR_BITSTREAM);
    const selab200_subframe_desc mine = fd[pos];
    const bool proc = exists && frame_ok;
    const bool diff = proc && mine.subframe_type == 1;
    int16_t *out = p.pcm_out + (size_t)frame * kFrame * ch;
    int32_t *row = p.ws_res + (size_t)sub * kFrame;
    if (k == 0) {
        sm.row_res[seg] = row;
        // a difference signal goes back into its (already consumed) residue row; k_diff_fixup turns it into
        // parent - difference once the parent is complete
        sm.row_out[seg] = diff ? static_cast<void *>(row) : static_cast<void *>(out + mine.channel);
        sm.row_mode[seg] = !proc ? 0 : diff ? 2 : 1;
    }
    __syncwarp();
    segment_synthesis(sm, start, k, n, seg, n_seg, proc ? mine.lpc_order : 0, p.ws_q + (size_t)sub * 128, ch);

    if (exists && !frame_ok) { // malformed frame: silence
        for (int t = k; t < kFrame; t += n)
            out[(size_t)t * ch + pos] = 0;
    }
}

// Difference reconstruction (frame_decoder.cpp:40-69): after k_synthesise_segments the residue row of a
// difference-coded subframe holds the decoded difference, and its parent, always an independent subframe, is complete
// in the PCM; the channel is parent - difference.  Both are taken mod 2^16, which is all the int16 output keeps, in
// unsigned arithmetic, so that no int32 difference can overflow.  One CTA per frame, any channel count; frames without
// a difference subframe return at once.
__global__ void __launch_bounds__(128) k_diff_fixup(DecodeParams p)
{
    const uint32_t frame = blockIdx.x, ch = p.channels;
    const selab200_subframe_desc *fd = p.descs + (size_t)frame * ch;
    bool any = false; // nearly every frame has no difference subframe: it returns before the whole check
    for (uint32_t pos = 0; pos < ch; pos++)
        any |= fd[pos].subframe_type == 1;
    if (!any || !frame_check(fd, ch, p.n_words)) // the synthesis kernel has already reported a violation
        return;
    int16_t *out = p.pcm_out + (size_t)frame * kFrame * ch;
    for (uint32_t pos = 0; pos < ch; pos++) {
        const selab200_subframe_desc d = fd[pos];
        if (d.subframe_type != 1)
            continue;
        const int32_t *diff = p.ws_res + ((size_t)frame * ch + pos) * kFrame;
        for (int t = threadIdx.x; t < kFrame; t += blockDim.x)
            out[(size_t)t * ch + d.channel] =
                (int16_t)(uint16_t)((uint32_t)out[(size_t)t * ch + d.parent_channel] - (uint32_t)diff[t]);
    }
}

// ------------------------------------------------------------ stage level --

// A 17-bit signal staged as a Signal in static shared memory (the stage-level kernels): the row, the parity bits, and
// kHistoryPad zeros in front of both.
struct Row17 {
    __align__(16) int16_t a[kHistoryPad + kFrame];
    uint32_t lo[(kHistoryPad + kFrame) / 32];
    __device__ __forceinline__ Signal stage(const int32_t *src)
    {
        const int lane = lane_id();
        for (int i = lane; i < kHistoryPad / 2; i += 32)
            reinterpret_cast<uint32_t *>(a)[i] = 0;
        if (lane < kHistoryPad / 32)
            lo[lane] = 0;
        stage_17bit_row(src, a + kHistoryPad, lo + kHistoryPad / 32);
        __syncwarp();
        return Signal{a + kHistoryPad, lo + kHistoryPad / 32};
    }
};

// lpc::ResidueGenerator::process for one signal per (1-warp) CTA; the means come from
// k_unit_means<kMeanPlanar> over the same samples.
__global__ void __launch_bounds__(32) k_lpc_residues(const int32_t *samples, const double *means, uint32_t n_sub,
                                                     uint8_t *order_out, int32_t *q_out, int32_t *residues)
{
    __shared__ __align__(16) AnalysisScratch scratch;
    __shared__ __align__(16) CoefSmem cf;
    __shared__ __align__(16) Row17 row;
    const uint32_t sub = blockIdx.x;
    const int lane = lane_id();
    const Signal sig = row.stage(samples + (size_t)sub * kFrame);
    warp_autocorrelation(sig, scratch, means[sub]);
    warp_schur(scratch);
    const int order = warp_order_and_quantise(scratch, cf);
    warp_coefficients(cf, scratch.t(), order);
    warp_fir_residual<true>(sig, cf, order, reinterpret_cast<uint32_t *>(scratch.ring), residues + (size_t)sub * kFrame);
    for (int i = lane; i < kMaxOrder; i += 32)
        q_out[(size_t)sub * kMaxOrder + i] = i < order ? cf.q[i] : 0;
    if (lane == 0)
        order_out[sub] = (uint8_t)order;
}

// selab200_fir_probe: the encoder's FIR on chosen samples and predictors, a warp per signal.  wide = 0: the int16 row
// of a channel unit (|s| <= 32767), else the row + parity bits of a 17-bit unit (|s| <= 65535).
// CHECK (selab200_fir_tie_probe): the instantiation with the tie test, whose flag goes to ties[signal].
template <bool CHECK = false>
__global__ void __launch_bounds__(32) k_fir_probe(const int32_t *samples, const int32_t *orders, const long long *c,
                                                  int wide, int32_t *residues, uint8_t *ties)
{
    __shared__ __align__(16) AnalysisScratch scratch;
    __shared__ __align__(16) CoefSmem cf;
    __shared__ __align__(16) Row17 row;
    const uint32_t sub = blockIdx.x;
    const int lane = lane_id();
    const int32_t *src = samples + (size_t)sub * kFrame;
    Signal sig = row.stage(src);
    if (!wide) {
        for (int j = lane; j < kFrame; j += 32)
            row.a[kHistoryPad + j] = (int16_t)src[j];
        sig.lo = nullptr;
    }
    const int order = orders[sub];
    for (int i = lane; i < 112; i += 32) { // c[1..order] as the step-up leaves it: zero past the order
        const long long v = i < order ? c[(size_t)sub * (kMaxOrder + 1) + i + 1] : 0;
        cf.clo[i] = (uint32_t)v;
        cf.chi[i] = (int32_t)(v >> 32);
    }
    __syncwarp();
    uint32_t *planes = reinterpret_cast<uint32_t *>(scratch.ring);
    int32_t *res = residues + (size_t)sub * kFrame;
    const bool tie = wide ? warp_fir_residual<true, CHECK>(sig, cf, order, planes, res)
                          : warp_fir_residual<false, CHECK>(sig, cf, order, planes, res);
    if (CHECK && lane == 0)
        ties[sub] = tie;
}

// lpc::SampleGenerator::process for one signal per (1-warp) CTA: the decoder's recurrence on one segment at lane 0.
__global__ void __launch_bounds__(32) k_lpc_samples(const int32_t *residues, uint32_t n_sub, const uint8_t *order_in,
                                                    const int32_t *q_in, int32_t *samples)
{
    __shared__ __align__(16) SegSmem sm;
    const uint32_t sub = blockIdx.x;
    const int lane = lane_id();
    const int order = min((int)order_in[sub], kMaxOrder);
    const int n = segment_width(order);
    if (lane == 0) {
        sm.row_res[0] = residues + (size_t)sub * kFrame;
        sm.row_out[0] = samples + (size_t)sub * kFrame;
        sm.row_mode[0] = 2;
    }
    __syncwarp();
    segment_synthesis(sm, 0, lane, n, 0, 1, lane < n ? order : 0, q_in + (size_t)sub * kMaxOrder, 1);
}

// selab200_quantise_probe: the encoder's order threshold and quantiser on chosen k, a thread per value.
__global__ void k_quantise_probe(const double *k, uint32_t n, int32_t *out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const double kv = k[i];
    out[4 * (size_t)i + 0] = quantise_reflection(0, kv);
    out[4 * (size_t)i + 1] = quantise_reflection(1, kv);
    out[4 * (size_t)i + 2] = quantise_reflection(2, kv);
    out[4 * (size_t)i + 3] = reflection_significant(kv) ? 1 : 0;
}

// Exhaustive device check of sample_to_x against IEEE division over |s| <= 65535.
__global__ void k_selftest_scaling(uint32_t *mismatches)
{
    const int s = (int)(blockIdx.x * blockDim.x + threadIdx.x) - 65535;
    if (s > 65535)
        return;
    if (__double_as_longlong(sample_to_x(s)) != __double_as_longlong(sample_to_x_div(s)))
        atomicAdd(mismatches, 1u);
}

// rice::RiceEncoder::process, one stream per (1-warp) CTA.  Stream rows lie `pitch` values apart,
// pitch a multiple of 4 and values 16-byte aligned (rice_lane_range).
__global__ void __launch_bounds__(32) k_rice_encode(const int32_t *values, const uint32_t *counts, uint32_t pitch,
                                                    uint32_t *k_out, uint32_t *n_words_out, uint32_t *words,
                                                    uint32_t words_stride, int32_t *status)
{
    const uint32_t st = blockIdx.x;
    const int32_t *v = values + (size_t)st * pitch;
    const int n = (int)counts[st];
    RiceChoice c = warp_rice_choose(v, n);
    if (lane_id() == 0) {
        k_out[st] = c.k;
        n_words_out[st] = c.words;
    }
    if (c.words > words_stride) {
        if (lane_id() == 0)
            raise_status(status, SELAB200_ERR_CAPACITY);
        return;
    }
    warp_rice_pack(v, n, c, words + (size_t)st * words_stride);
}

// rice::RiceDecoder::process, one stream per lane.
__global__ void __launch_bounds__(32 * kRiceWarps) k_rice_decode_streams(
    const uint32_t *words, const uint32_t *n_words, uint32_t words_stride, const uint32_t *k,
    const uint32_t *counts, uint32_t n_streams, int32_t *out, uint32_t out_stride, int32_t *status)
{
    __shared__ uint32_t ring[kRiceWarps][(kRiceRing + 1) * 32];
    const uint32_t st_i = blockIdx.x * blockDim.x + threadIdx.x;
    RiceLaneStream st;
    st.src = words;
    st.n_words = 0;
    st.k = 0;
    st.count = 0;
    st.out = nullptr;
    if (st_i < n_streams) {
        if (k[st_i] >= 32 || counts[st_i] > out_stride || n_words[st_i] > words_stride) {
            raise_status(status, SELAB200_ERR_BITSTREAM);
        } else {
            st.src = words + (size_t)st_i * words_stride;
            st.n_words = n_words[st_i];
            st.k = k[st_i];
            st.count = counts[st_i];
            st.out = out + (size_t)st_i * out_stride;
        }
    }
    warp_rice_decode32<kRiceRing, kRiceBatch>(ring[warp_id()], st);
}

} // namespace selab200
