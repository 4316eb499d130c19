// ref_shim.cpp -- C interface over the UNMODIFIED reference classes.
//
// TEST INFRASTRUCTURE ONLY.  Compiled by oracle/Makefile together with the
// reference sources where they lie under $(SELA_REF) (default /root/reference)
// into oracle/_ref/libsela_ref.so.  No reference source is copied into this
// repository; this file only calls the reference's public classes
// (frame::FrameEncoder/FrameDecoder, lpc::ResidueGenerator/SampleGenerator,
// rice::RiceEncoder/RiceDecoder) and reads some of their private members: the
// multithreaded CPU baseline's sela::Encoder/Decoder::processFrames, and the
// normalised autocorrelation ResidueGenerator leaves behind (opened with the
// usual `#define private public` around the includes, nothing else is touched).
//
// It exports the same symbols as oracle/sela_oracle.c, except the port-only
// sela_oracle_lpc_mean and sela_oracle_quantise_probe, so tests and bench.py can load
// either library: sela_oracle_kind() tells them apart ("reference"), and
// sela_oracle_internals() says which internals each fills.

#include <chrono>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <string>
#include <thread>
#include <vector>

// Every standard header the reference headers pull in (<cstdint>, <string>, <vector>) is included above, so
// the define below only reaches the reference's own classes.
#define private public
#include "frame.hpp"
#include "lpc.hpp"
#include "rice.hpp"
#include "sela/decoder.hpp"
#include "sela/encoder.hpp"
#undef private

#include "sela_oracle.h"

namespace {
const uint32_t kFrame = SELA_ORACLE_FRAME;

std::vector<data::WavFrame> demux(const int16_t *pcm, uint32_t n_frames, uint32_t channels)
{
    std::vector<data::WavFrame> frames;
    frames.reserve(n_frames);
    for (uint32_t f = 0; f < n_frames; f++) {
        std::vector<std::vector<int32_t>> planes(channels, std::vector<int32_t>(kFrame));
        const int16_t *src = pcm + (size_t)f * kFrame * channels;
        for (uint32_t j = 0; j < kFrame; j++)
            for (uint32_t c = 0; c < channels; c++)
                planes[c][j] = src[(size_t)j * channels + c];
        frames.push_back(data::WavFrame(16, std::move(planes)));
    }
    return frames;
}

int flatten(const std::vector<data::SelaFrame> &frames, size_t first_desc, sela_oracle_desc *descs,
            uint32_t *words, size_t cap, size_t *used)
{
    size_t d = first_desc;
    for (const data::SelaFrame &fr : frames) {
        for (const data::SelaSubFrame &sf : fr.subFrames) {
            size_t need = sf.encodedReflectionCoefficients.size() + sf.encodedResidues.size();
            if (*used + need > cap)
                return -1;
            sela_oracle_desc &o = descs[d++];
            std::memset(&o, 0, sizeof o);
            o.channel = sf.channel;
            o.subframe_type = sf.subFrameType;
            o.parent_channel = sf.parentChannelNumber;
            o.refl_rice_param = sf.reflectionCoefficientRiceParam;
            o.refl_words = sf.reflectionCoefficientRequiredInts;
            o.lpc_order = sf.optimumLpcOrder;
            o.res_rice_param = sf.residueRiceParam;
            o.res_words = sf.residueRequiredInts;
            o.samples = sf.samplesPerChannel;
            o.refl_offset = *used;
            std::memcpy(words + *used, sf.encodedReflectionCoefficients.data(),
                        sf.encodedReflectionCoefficients.size() * 4);
            *used += sf.encodedReflectionCoefficients.size();
            o.res_offset = *used;
            std::memcpy(words + *used, sf.encodedResidues.data(), sf.encodedResidues.size() * 4);
            *used += sf.encodedResidues.size();
        }
    }
    return 0;
}

data::SelaFrame unflatten(const sela_oracle_desc *descs, uint32_t n_sub, const uint32_t *words)
{
    data::SelaFrame fr(16);
    fr.subFrames.reserve(n_sub);
    for (uint32_t i = 0; i < n_sub; i++) {
        const sela_oracle_desc &d = descs[i];
        std::vector<uint32_t> refl(words + d.refl_offset, words + d.refl_offset + d.refl_words);
        std::vector<uint32_t> res(words + d.res_offset, words + d.res_offset + d.res_words);
        data::RiceEncodedData reflData(d.refl_rice_param, d.lpc_order, std::move(refl));
        data::RiceEncodedData resData(d.res_rice_param, d.samples, std::move(res));
        fr.subFrames.push_back(data::SelaSubFrame(d.channel, d.subframe_type, d.parent_channel, reflData, resData));
    }
    return fr;
}
} // namespace

extern "C" {

const char *sela_oracle_kind(void) { return "reference"; }

const char *sela_oracle_internals(void) { return "ac"; }

int sela_oracle_online_cores(void)
{
    unsigned n = std::thread::hardware_concurrency();
    return n ? (int)n : 1;
}

void sela_oracle_lpc_analyse(const int32_t *s, size_t n, uint8_t *order, int32_t *q, int64_t *c,
                             int32_t *res, double *refl, double *ac)
{
    // Not observable here, so left untouched: dequantizeReflectionCoefficients replaces the raw
    // reflection coefficients with de-quantised ones.
    (void)refl;
    data::LpcDecodedData in(16, std::vector<int32_t>(s, s + n));
    lpc::ResidueGenerator gen(in);
    data::LpcEncodedData enc = gen.process();
    if (ac) // lags 0..100 after normalisation (residue_generator.cpp:40-44); process() leaves them alone
        std::memcpy(ac, gen.autocorrelationFactors.data(), (SELA_ORACLE_MAX_ORDER + 1) * sizeof(double));
    *order = enc.optimalLpcOrder;
    if (q)
        std::memcpy(q, enc.quantizedReflectionCoefficients.data(), enc.quantizedReflectionCoefficients.size() * 4);
    if (res)
        std::memcpy(res, enc.residues.data(), enc.residues.size() * 4);
    if (c)
        sela_oracle_lpc_coefficients(enc.quantizedReflectionCoefficients.data(), enc.optimalLpcOrder, c);
}

void sela_oracle_lpc_coefficients(const int32_t *q, uint8_t order, int64_t *c)
{
    lpc::LinearPredictor lp(std::vector<int32_t>(q, q + order), order);
    lp.dequantizeReflectionCoefficients();
    lp.generatelinearPredictionCoefficients();
    std::memcpy(c, lp.linearPredictionCoefficients.data(), lp.linearPredictionCoefficients.size() * 8);
}

void sela_oracle_lpc_synthesise(const int32_t *res, size_t n, uint8_t order, const int32_t *q, int32_t *s)
{
    data::LpcEncodedData enc(order, 16, std::vector<int32_t>(q, q + order), std::vector<int32_t>(res, res + n));
    data::LpcDecodedData dec = lpc::SampleGenerator(enc).process();
    std::memcpy(s, dec.samples.data(), dec.samples.size() * 4);
}

size_t sela_oracle_rice_encode(const int32_t *x, size_t n, uint32_t *k_out, uint32_t *words, size_t cap)
{
    data::RiceDecodedData in(std::vector<int32_t>(x, x + n));
    data::RiceEncodedData enc = rice::RiceEncoder(in).process();
    if (k_out)
        *k_out = enc.optimumRiceParam;
    if (enc.encodedData.size() <= cap)
        std::memcpy(words, enc.encodedData.data(), enc.encodedData.size() * 4);
    return enc.encodedData.size();
}

size_t sela_oracle_rice_size(const int32_t *x, size_t n, uint32_t *k_out, uint64_t *bits_out)
{
    data::RiceDecodedData in(std::vector<int32_t>(x, x + n));
    data::RiceEncodedData enc = rice::RiceEncoder(in).process();
    if (k_out)
        *k_out = enc.optimumRiceParam;
    if (bits_out)
        *bits_out = 0; // requiredBits is private in the reference
    return enc.encodedData.size();
}

void sela_oracle_rice_decode(const uint32_t *words, size_t n_words, uint32_t k, uint32_t count, int32_t *out)
{
    data::RiceEncodedData enc(k, count, std::vector<uint32_t>(words, words + n_words));
    data::RiceDecodedData dec = rice::RiceDecoder(enc).process();
    std::memcpy(out, dec.decodedData.data(), dec.decodedData.size() * 4);
}

int sela_oracle_frame_encode_i32(const int32_t *const *chs, uint32_t channels, uint32_t n,
                                 sela_oracle_desc *descs, uint32_t *words, size_t cap, size_t *used)
{
    std::vector<std::vector<int32_t>> planes;
    for (uint32_t c = 0; c < channels; c++)
        planes.push_back(std::vector<int32_t>(chs[c], chs[c] + n));
    data::WavFrame wf(16, std::move(planes));
    std::vector<data::SelaFrame> one;
    one.push_back(frame::FrameEncoder(wf).process());
    return flatten(one, 0, descs, words, cap, used);
}

int sela_oracle_frame_decode_i32(const sela_oracle_desc *descs, uint32_t n_sub, const uint32_t *words,
                                 int32_t *const *out)
{
    data::SelaFrame fr = unflatten(descs, n_sub, words);
    data::WavFrame wf = frame::FrameDecoder(fr).process();
    for (size_t c = 0; c < wf.samples.size(); c++)
        std::memcpy(out[c], wf.samples[c].data(), wf.samples[c].size() * 4);
    return 0;
}

// The reference's own multithreaded path: sela::Encoder::processFrames
// (src/sela/encoder.cpp:40-92), hardware_concurrency() std::threads.  `threads`
// is ignored on purpose (the reference has no such knob) unless it is 1, which
// runs the reference's per-frame class in a plain loop for single-core timing.
int sela_oracle_encode_frames(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                              sela_oracle_desc *descs, uint32_t *words, size_t cap, size_t *used, int threads)
{
    *used = 0;
    std::vector<data::SelaFrame> out;
    if (threads == 1) {
        std::vector<data::WavFrame> frames = demux(pcm, n_frames, channels);
        out.reserve(n_frames);
        for (const data::WavFrame &wf : frames)
            out.push_back(frame::FrameEncoder(wf).process());
    } else {
        std::ifstream none;
        sela::Encoder enc(none);
        enc.wavFile.wavChunk.dataSubChunk.wavFrames = demux(pcm, n_frames, channels);
        enc.processFrames(out);
    }
    return flatten(out, 0, descs, words, cap, used);
}

int sela_oracle_decode_frames(const sela_oracle_desc *descs, uint32_t n_frames, uint32_t channels,
                              const uint32_t *words, int16_t *pcm_out, int threads)
{
    std::vector<data::SelaFrame> in;
    in.reserve(n_frames);
    for (uint32_t f = 0; f < n_frames; f++)
        in.push_back(unflatten(descs + (size_t)f * channels, channels, words));
    std::vector<data::WavFrame> out;
    if (threads == 1) {
        out.reserve(n_frames);
        for (const data::SelaFrame &sf : in)
            out.push_back(frame::FrameDecoder(sf).process());
    } else {
        std::ifstream none;
        sela::Decoder dec(none);
        dec.selaFile.selaFrames = std::move(in);
        dec.processFrames(out);
    }
    for (uint32_t f = 0; f < n_frames; f++) {
        int16_t *dst = pcm_out + (size_t)f * kFrame * channels;
        for (uint32_t j = 0; j < kFrame; j++)
            for (uint32_t c = 0; c < channels; c++)
                dst[(size_t)j * channels + c] = (int16_t)(uint16_t)out[f].samples[c][j];
    }
    return 0;
}

// Timing helpers for bench.py: processFrames ONLY (SURVEY.md 8d), demux/flatten excluded.
// Returns seconds (steady_clock) for `reps` repetitions' median is left to the caller.
double sela_oracle_time_encode(const int16_t *pcm, uint32_t n_frames, uint32_t channels, int threads)
{
    (void)threads; // the reference always uses hardware_concurrency()
    std::ifstream none;
    sela::Encoder enc(none);
    enc.wavFile.wavChunk.dataSubChunk.wavFrames = demux(pcm, n_frames, channels);
    std::vector<data::SelaFrame> out;
    auto t0 = std::chrono::steady_clock::now();
    enc.processFrames(out);
    auto t1 = std::chrono::steady_clock::now();
    return std::chrono::duration<double>(t1 - t0).count();
}

double sela_oracle_time_decode(const sela_oracle_desc *descs, uint32_t n_frames, uint32_t channels,
                               const uint32_t *words, int threads)
{
    (void)threads;
    std::ifstream none;
    sela::Decoder dec(none);
    dec.selaFile.selaFrames.reserve(n_frames);
    for (uint32_t f = 0; f < n_frames; f++)
        dec.selaFile.selaFrames.push_back(unflatten(descs + (size_t)f * channels, channels, words));
    std::vector<data::WavFrame> out;
    auto t0 = std::chrono::steady_clock::now();
    dec.processFrames(out);
    auto t1 = std::chrono::steady_clock::now();
    return std::chrono::duration<double>(t1 - t0).count();
}

} // extern "C"
