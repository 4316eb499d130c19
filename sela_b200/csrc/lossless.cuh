// lossless.cuh -- the kernels of the lossless encode (sm_90a, DESIGN.md 7.2): every subframe that the reference
// decoder would not bring back to its source is coded with a slightly different predictor, inside the format.
//
//   k_encode_units<S, false, true>   the ordinary analysis kernel, which also flags units whose FIR has a tie
//   k_lossless_select                frame per thread: frames whose emitted subframes include a flagged unit
//                                    -> the repair lists; the flag of every other unit is cleared
//   k_lossless_candidates<S>         warp per (listed unit, candidate of one round): the candidate's words, if it has
//                                    no tie (encode_unit<kUnitCandidate>); round 2 only for units round 1 left empty
//   k_lossless_repack<S>             warp per listed unit: the winner packed into the unit's slot, record rewritten
//   k_lossless_report                thread per listed frame: the emitted subframes that differ from the reference's
// Then k_encode_sizes / k_encode_scan / k_encode_gather(_container) run as for every encode, and the stereo
// decision there sees the repaired sizes.  The lists are counted on the device: the repair kernels have grids of a
// fixed size and loop over whatever the select kernel listed, so a batch without a flagged unit costs their
// launches and nothing else, and the host never waits for a count.
#pragma once

#include "kernels.cuh"

namespace selab200 {

struct RepairParams {
    uint32_t *count;                  // [0] frames listed, [1] units listed
    uint32_t *frames;                 // [n_frames] listed frames (batch-local)
    UnitRecord *orig;                 // [n_frames][units per frame] the records of a listed frame before the repair
    RepairUnit *units;                // [n_units] listed units
    selab200_lossless_entry *entries; // [n_frames * channels] per (frame, channel); untouched where nothing changed
    unsigned long long *n_entries;    // entries written
    uint32_t frame_base;              // frame number of the batch's first frame in the report
};

__host__ __device__ inline uint32_t units_per_frame(uint32_t channels) { return channels == 2 ? 3u : channels; }

__global__ void __launch_bounds__(256) k_lossless_select(EncodeParams p, RepairParams r)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.n_frames)
        return;
    const uint32_t per = units_per_frame(p.channels);
    UnitRecord *fu = p.units + (size_t)f * per;
    uint32_t flagged = 0;
    for (uint32_t k = 0; k < per; k++)
        flagged |= ((fu[k].flags >> 1) & 1u) << k;
    if (!flagged)
        return;
    bool emitted = false; // the reference's decision, on the records as the reference encoder has them
    for (uint32_t c = 0; c < p.channels; c++) {
        UnitRecord u;
        emitted |= (flagged >> choose_record(fu, p.channels, c, u).unit) & 1u;
    }
    if (!emitted) { // a flagged stereo candidate that loses: the frame keeps the reference's bytes
        for (uint32_t k = 0; k < per; k++)
            if ((flagged >> k) & 1u)
                fu[k].flags &= ~2u;
        return;
    }
    const uint32_t i = atomicAdd(&r.count[0], 1u);
    r.frames[i] = f;
    for (uint32_t k = 0; k < per; k++)
        r.orig[(size_t)i * per + k] = fu[k];
    for (uint32_t k = 0; k < per; k++)
        if ((flagged >> k) & 1u) {
            RepairUnit ru;
            ru.unit = f * per + k;
            ru.order = fu[k].order;
            ru.best = kNoCandidate;
            r.units[atomicAdd(&r.count[1], 1u)] = ru;
        }
}

// Round 0: the candidates of round 1 of every listed unit; round 1: those of round 2, for units without a round-1
// winner.  A warp per (unit, candidate) at a time, residue row = the warp's (the grid is at most the batch's units).
// FORCE and `pred` as for k_encode_units (tests only).
template <bool STEREO, bool FORCE = false>
__global__ void __launch_bounds__(32) k_lossless_candidates(EncodeParams p, RepairParams r, int round,
                                                            const selab200_predictor *pred)
{
    const uint32_t n = *reinterpret_cast<volatile uint32_t *>(&r.count[1]);
    const uint32_t stride = round == 0 ? 7u : (uint32_t)kRepairRound2Max;
    for (size_t w = blockIdx.x; w < (size_t)n * stride; w += gridDim.x) {
        RepairUnit *ru = r.units + w / stride;
        const int o = (int)ru->order, n1 = repair_round1(o);
        const uint32_t cand = (uint32_t)(w % stride) + (round == 0 ? 0u : (uint32_t)n1);
        if (round == 0 ? cand >= (uint32_t)n1
                       : cand >= (uint32_t)repair_candidates(o) || ru->best < (1ull << 63)) // round 1 has a winner
            continue;
        __syncwarp();
        encode_unit<STEREO, false, kUnitCandidate, FORCE>(p, nullptr, ru->unit, ru, cand, pred);
    }
}

template <bool STEREO, bool FORCE = false>
__global__ void __launch_bounds__(32) k_lossless_repack(EncodeParams p, RepairParams r, const selab200_predictor *pred)
{
    const uint32_t n = *reinterpret_cast<volatile uint32_t *>(&r.count[1]);
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        const RepairUnit ru = r.units[i];
        if (ru.best == kNoCandidate) // cannot happen (order 1 is a candidate); the flag left set fails the scan
            continue;
        __syncwarp();
        encode_unit<STEREO, false, kUnitRepack, FORCE>(p, nullptr, ru.unit, nullptr, (uint32_t)ru.best, pred);
    }
}

// Per listed frame and channel: the subframe the reference encoder emits (its decision on the records before the
// repair) against the one emitted now.  An entry where the emitted unit differs or was re-coded.
__global__ void __launch_bounds__(256) k_lossless_report(EncodeParams p, RepairParams r)
{
    const uint32_t n = *reinterpret_cast<volatile uint32_t *>(&r.count[0]);
    const uint32_t per = units_per_frame(p.channels);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t f = r.frames[i];
        const UnitRecord *ref = r.orig + (size_t)i * per, *now = p.units + (size_t)f * per;
        for (uint32_t c = 0; c < p.channels; c++) {
            UnitRecord a, b;
            const Emit ea = choose_record(ref, p.channels, c, a), eb = choose_record(now, p.channels, c, b);
            if (ea.unit == eb.unit && !(ref[eb.unit].flags & 2u))
                continue;
            selab200_lossless_entry e;
            e.frame = r.frame_base + f;
            e.channel = (uint16_t)c;
            e.ref_order = (uint8_t)a.order;
            e.order = (uint8_t)b.order;
            e.ref_words = a.refl_words + a.res_words;
            e.words = b.refl_words + b.res_words;
            r.entries[(size_t)f * p.channels + c] = e;
            atomicAdd(r.n_entries, 1ull);
        }
    }
}

} // namespace selab200
