// sela_host.cpp -- C++ mirror of the reference's operator interface over the CUDA C ABI.
//
// Host glue only (container parsing, value-struct <-> flat-buffer conversion); every
// sample is analysed, filtered and coded on the GPU through include/sela_b200.h.
// Device errors become `throw data::Exception(...)` (src/include/data/exception.hpp:7-14).
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include <thread>

#include "sela_api.hpp"
#include "../../../include/sela_b200.h"

namespace {

constexpr uint32_t kFrame = SELAB200_FRAME_SAMPLES;

[[noreturn]] void raise(const std::string &what)
{
    throw data::Exception(std::string(what));
}

void check(int status)
{
    if (status != SELAB200_OK)
        raise(std::string("sela_b200: ") + selab200_last_error());
}

void ensure_device()
{
    static std::mutex m;
    static bool ready = false;
    std::lock_guard<std::mutex> lock(m);
    if (ready)
        return;
    // SELAB200_DEVICES = "0,1,2,3" (or "all"): the batch calls then cut the frames into one block per device;
    // SELAB200_DEVICE = n: one device (default: device 0 -- a CUDA context per GPU is not free, and one
    // ten-minute file is a few milliseconds of work).
    if (const char *list = std::getenv("SELAB200_DEVICES")) {
        std::vector<int> ids;
        if (std::string(list) == "all") {
            int dev = 0;
            while (dev < 16 && selab200_init(dev) == SELAB200_OK) // probe how many there are
                ids.push_back(dev++);
        } else {
            for (const char *c = list; *c;) {
                ids.push_back(std::atoi(c));
                while (*c && *c != ',')
                    c++;
                if (*c == ',')
                    c++;
            }
        }
        if (ids.empty())
            ids.push_back(0);
        check(selab200_init_devices((int)ids.size(), ids.data()));
    } else {
        const char *env = std::getenv("SELAB200_DEVICE");
        check(selab200_init(env ? std::atoi(env) : 0));
    }
    ready = true;
}

// Pinned staging buffer (RAII) for the batch calls.
template <typename T>
struct Pinned {
    T *p = nullptr;
    size_t n = 0;
    explicit Pinned(size_t count) : n(count)
    {
        p = static_cast<T *>(selab200_host_alloc(std::max<size_t>(count, 1) * sizeof(T)));
        if (!p)
            raise("sela_b200: pinned host allocation failed");
    }
    ~Pinned() { selab200_host_free(p); }
    Pinned(const Pinned &) = delete;
    Pinned &operator=(const Pinned &) = delete;
};

int16_t narrow_sample(int32_t v)
{
    if (v < INT16_MIN || v > INT16_MAX)
        raise("sela_b200: sample outside the 16-bit range (only 16-bit audio is supported)");
    return (int16_t)v;
}

data::SelaFrame frame_from_descs(const selab200_subframe_desc *d, uint32_t channels, const uint32_t *words, uint8_t bits)
{
    data::SelaFrame out(bits);
    out.subFrames.reserve(channels);
    for (uint32_t c = 0; c < channels; c++) {
        const selab200_subframe_desc &s = d[c];
        data::RiceEncodedData refl(s.refl_rice_param, s.lpc_order,
                                   std::vector<uint32_t>(words + s.refl_offset, words + s.refl_offset + s.refl_words));
        data::RiceEncodedData res(s.res_rice_param, s.samples,
                                  std::vector<uint32_t>(words + s.res_offset, words + s.res_offset + s.res_words));
        out.subFrames.push_back(data::SelaSubFrame(s.channel, s.subframe_type, s.parent_channel, refl, res));
    }
    return out;
}

size_t frame_words(const data::SelaFrame &f)
{
    size_t n = 0;
    for (const data::SelaSubFrame &s : f.subFrames)
        n += s.encodedReflectionCoefficients.size() + s.encodedResidues.size();
    return n;
}

void flatten_frame(const data::SelaFrame &f, selab200_subframe_desc *d, uint32_t *words, size_t &cursor)
{
    for (const data::SelaSubFrame &s : f.subFrames) {
        std::memset(d, 0, sizeof *d);
        d->channel = s.channel;
        d->subframe_type = s.subFrameType;
        d->parent_channel = s.parentChannelNumber;
        d->refl_rice_param = s.reflectionCoefficientRiceParam;
        d->refl_words = (uint16_t)s.encodedReflectionCoefficients.size();
        d->lpc_order = s.optimumLpcOrder;
        d->res_rice_param = s.residueRiceParam;
        d->res_words = (uint16_t)s.encodedResidues.size();
        d->samples = s.samplesPerChannel;
        d->refl_offset = cursor;
        std::copy(s.encodedReflectionCoefficients.begin(), s.encodedReflectionCoefficients.end(), words + cursor);
        cursor += s.encodedReflectionCoefficients.size();
        d->res_offset = cursor;
        std::copy(s.encodedResidues.begin(), s.encodedResidues.end(), words + cursor);
        cursor += s.encodedResidues.size();
        d++;
    }
}

// little-endian field readers over a byte buffer
struct Bytes {
    const std::vector<char> &b;
    uint32_t u8(size_t o) const { return (uint8_t)b[o]; }
    uint32_t u16(size_t o) const { return u8(o) | (u8(o + 1) << 8); }
    uint32_t u32(size_t o) const { return u16(o) | (u16(o + 2) << 16); }
    std::string tag(size_t o) const { return std::string(b.begin() + o, b.begin() + o + 4); }
};

std::vector<char> slurp(std::ifstream &in)
{
    std::vector<char> contents;
    in.seekg(0, std::ios::end);
    const std::streamoff size = in.tellg();
    contents.resize(size > 0 ? (size_t)size : 0);
    in.seekg(0, std::ios::beg);
    if (!contents.empty())
        in.read(contents.data(), (std::streamsize)contents.size());
    return contents;
}

template <typename T>
void put(std::ofstream &out, const T &v)
{
    out.write(reinterpret_cast<const char *>(&v), sizeof v);
}

// Staging memory of the file-to-file drivers, one pair (input, output) per host thread.
// One-shot use (the CLI coding one file): plain heap memory, released when the call returns --
// page-locking 200 MB costs more than the pageable copies it would save.  Batch mode
// (sela::setBatchMode, many files per process): page-locked, kept and reused from file to file, so
// that uploads and downloads run at full PCIe speed and overlap the kernels.
std::atomic<bool> g_batch_mode{false};

struct HostBuffer {
    char *p = nullptr;
    size_t cap = 0;
    bool pinned = false;
    void release()
    {
        if (p && pinned)
            selab200_host_free(p);
        else
            delete[] p;
        p = nullptr;
        cap = 0;
    }
    // uninitialised memory: no value-initialisation pass over 100 MB
    char *ensure(size_t n)
    {
        const bool want_pinned = g_batch_mode.load();
        if (p && n <= cap && pinned == want_pinned)
            return p;
        release();
        const size_t want = want_pinned ? n + n / 4 + 4096 : n + 1;
        pinned = want_pinned;
        p = pinned ? static_cast<char *>(selab200_host_alloc(want)) : new char[want];
        if (!p)
            raise("sela_b200: host staging allocation failed");
        cap = want;
        return p;
    }
    ~HostBuffer() { release(); }
};
thread_local HostBuffer t_input, t_output;
struct StagingScope { // one-shot use gives the memory back; batch mode keeps it for the next file
    ~StagingScope()
    {
        if (!g_batch_mode.load()) {
            t_input.release();
            t_output.release();
        }
    }
};

struct RawFile {
    char *data = nullptr;
    size_t size = 0;
    const uint8_t *bytes() const { return reinterpret_cast<const uint8_t *>(data); }
};
// Whole file into this thread's input staging buffer.
RawFile slurp_raw(std::ifstream &in)
{
    RawFile f;
    in.seekg(0, std::ios::end);
    const std::streamoff size = in.tellg();
    f.size = size > 0 ? (size_t)size : 0;
    f.data = t_input.ensure(f.size + 1);
    in.seekg(0, std::ios::beg);
    if (f.size)
        in.read(f.data, (std::streamsize)f.size);
    return f;
}

// RIFF walk of file::WavFile::readFromFile (src/file/wav_file.cpp:39-179) without the copies:
// same acceptance rules, same messages, same order of checks.
struct WavSpan {
    std::string id;
    uint32_t size;
    size_t body;
};
struct WavLayout {
    uint32_t chunkSize = 0;
    data::WavFormatSubChunk fmt; // scalar fields only; subChunkData left empty
    size_t fmtIndex = 0, dataIndex = 0;
    std::vector<WavSpan> spans;  // every sub-chunk in file order
};
struct ByteView {
    const char *b;
    uint32_t u8(size_t o) const { return (uint8_t)b[o]; }
    uint32_t u16(size_t o) const { return u8(o) | (u8(o + 1) << 8); }
    uint32_t u32(size_t o) const { return u16(o) | (u16(o + 2) << 16); }
    std::string tag(size_t o) const { return std::string(b + o, b + o + 4); }
};
WavLayout scan_wav(const char *contents, size_t n)
{
    const ByteView rd{contents};
    WavLayout w;
    if (n < 44)
        raise("File is too small, probably not a wav file.");
    if (rd.tag(0) != "RIFF")
        raise("chunkId is not RIFF, probably not a wav file.");
    w.chunkSize = rd.u32(4);
    if ((size_t)w.chunkSize > n)
        raise("chunkSize exceeds file size, probably a corrupted file");
    if (rd.tag(8) != "WAVE")
        raise("format is not WAVE, probably not a wav file.");
    bool haveFmt = false, haveData = false;
    size_t at = 12;
    while (at < n) {
        if (at + 8 > n)
            raise("truncated sub-chunk header, probably a corrupted file");
        WavSpan span{rd.tag(at), rd.u32(at + 4), at + 8};
        if (span.body + span.size > n)
            raise("sub-chunk exceeds file size, probably a corrupted file");
        if (span.id == "fmt ") {
            if (span.size < 16)
                raise("fmt subChunk is too small");
            data::WavFormatSubChunk &fmt = w.fmt;
            fmt.subChunkId = span.id;
            fmt.subChunkSize = span.size;
            fmt.audioFormat = (int16_t)rd.u16(span.body);
            fmt.numChannels = (uint16_t)rd.u16(span.body + 2);
            fmt.sampleRate = rd.u32(span.body + 4);
            fmt.byteRate = rd.u32(span.body + 8);
            fmt.blockAlign = (uint16_t)rd.u16(span.body + 12);
            fmt.bitsPerSample = (uint16_t)rd.u16(span.body + 14);
            if (fmt.bitsPerSample != 16)
                raise("Only 16bits per sample wav is supported.");
            w.fmtIndex = w.spans.size();
            haveFmt = true;
        } else if (span.id == "data") {
            if (!haveFmt)
                raise("Probably corrupt wav, data subChunk present without fmt subChunk.");
            w.dataIndex = w.spans.size();
            haveData = true;
        }
        w.spans.push_back(span);
        at = span.body + span.size;
    }
    if (!haveFmt)
        raise("fmt subChunk is missing from file");
    if (!haveData)
        raise("data subChunk is missing from file");
    return w;
}

// SELA_B200_TIMING=1: phase wall times of the file-level drivers on stderr.
struct Phase {
    const char *name;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    explicit Phase(const char *n) : name(n) {}
    ~Phase()
    {
        static const bool on = std::getenv("SELA_B200_TIMING") != nullptr;
        if (on)
            std::fprintf(stderr, "[sela_b200] %-22s %8.2f ms\n", name,
                         std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    }
};

// Device bring-up (CUDA context creation, a few hundred ms) on a helper thread while the caller
// reads its input file; join() rethrows what ensure_device() threw.
struct DeviceWarmup {
    std::exception_ptr error;
    std::thread worker;
    DeviceWarmup()
        : worker([this] {
              try {
                  Phase p("device init");
                  ensure_device();
              } catch (...) {
                  error = std::current_exception();
              }
          })
    {
    }
    void join()
    {
        if (worker.joinable())
            worker.join();
        if (error)
            std::rethrow_exception(error);
    }
    ~DeviceWarmup()
    {
        if (worker.joinable())
            worker.join();
    }
};

void write_wav_header(std::ofstream &outputFile, const data::WavChunk &wavChunk)
{
    const data::WavFormatSubChunk &fmt = wavChunk.formatSubChunk;
    outputFile << wavChunk.chunkId;
    put(outputFile, wavChunk.chunkSize);
    outputFile << wavChunk.format;
    outputFile << fmt.subChunkId;
    put(outputFile, fmt.subChunkSize);
    put(outputFile, fmt.audioFormat);
    put(outputFile, fmt.numChannels);
    put(outputFile, fmt.sampleRate);
    put(outputFile, fmt.byteRate);
    put(outputFile, fmt.blockAlign);
    put(outputFile, fmt.bitsPerSample);
    outputFile << wavChunk.dataSubChunk.subChunkId;
    put(outputFile, wavChunk.dataSubChunk.subChunkSize);
}

} // namespace

// ------------------------------------------------------------------- rice --

namespace rice {

RiceEncoder::RiceEncoder(const data::RiceDecodedData &decodedData) : input(decodedData.decodedData) {}

// rice::RiceEncoder::process (src/rice/rice_encoder.cpp:73-81)
data::RiceEncodedData RiceEncoder::process()
{
    ensure_device();
    const uint32_t n = (uint32_t)input.size();
    if (n > kFrame)
        raise("sela_b200: rice::RiceEncoder handles at most 2048 values per stream");
    uint32_t count = n, k = 0, n_words = 0;
    const uint32_t stride = std::max<uint32_t>(n, 1);
    std::vector<int32_t> values(stride, 0);
    std::copy(input.begin(), input.end(), values.begin());
    uint32_t cap = 2 * stride + 8;
    std::vector<uint32_t> words(cap);
    int rc = selab200_rice_encode(values.data(), &count, 1, stride, &k, &n_words, words.data(), cap);
    if (rc == SELAB200_ERR_CAPACITY) { // rare: more than ~64 bits per value
        cap = n_words;
        words.assign(cap, 0);
        rc = selab200_rice_encode(values.data(), &count, 1, stride, &k, &n_words, words.data(), cap);
    }
    check(rc);
    words.resize(n_words);
    return data::RiceEncodedData((int32_t)k, (int32_t)n, std::move(words));
}

RiceDecoder::RiceDecoder(const data::RiceEncodedData &encodedData)
    : input(encodedData.encodedData), dataCount(encodedData.dataCount), optimumRiceParam(encodedData.optimumRiceParam)
{
}

// rice::RiceDecoder::process (src/rice/rice_decoder.cpp:54-61)
data::RiceDecodedData RiceDecoder::process()
{
    ensure_device();
    uint32_t n_words = (uint32_t)input.size(), k = optimumRiceParam, count = dataCount;
    std::vector<uint32_t> words(std::max<size_t>(input.size(), 1), 0);
    std::copy(input.begin(), input.end(), words.begin());
    std::vector<int32_t> out(std::max<uint32_t>(count, 1), 0);
    check(selab200_rice_decode(words.data(), &n_words, (uint32_t)words.size(), &k, &count, 1, out.data(),
                               (uint32_t)out.size()));
    out.resize(count);
    return data::RiceDecodedData(std::move(out));
}

} // namespace rice

// -------------------------------------------------------------------- lpc --

namespace lpc {

ResidueGenerator::ResidueGenerator(const data::LpcDecodedData &data) : samples(data.samples), bitsPerSample(data.bitsPerSample) {}

// lpc::ResidueGenerator::process (src/lpc/residue_generator.cpp:121-134)
data::LpcEncodedData ResidueGenerator::process()
{
    ensure_device();
    if (samples.size() != kFrame)
        raise("sela_b200: lpc::ResidueGenerator needs exactly 2048 samples (the codec's frame size)");
    uint8_t order = 0;
    std::vector<int32_t> q(SELAB200_MAX_LPC_ORDER), res(kFrame);
    check(selab200_lpc_residues(samples.data(), 1, &order, q.data(), res.data()));
    q.resize(order);
    return data::LpcEncodedData(order, bitsPerSample, std::move(q), std::move(res));
}

SampleGenerator::SampleGenerator(const data::LpcEncodedData &encodedData) : encoded(encodedData) {}

// lpc::SampleGenerator::process (src/lpc/sample_generator.cpp:32-39)
data::LpcDecodedData SampleGenerator::process()
{
    ensure_device();
    if (encoded.residues.size() != kFrame)
        raise("sela_b200: lpc::SampleGenerator needs exactly 2048 residues (the codec's frame size)");
    uint8_t order = encoded.optimalLpcOrder;
    std::vector<int32_t> q(SELAB200_MAX_LPC_ORDER, 0), out(kFrame);
    std::copy_n(encoded.quantizedReflectionCoefficients.begin(),
                std::min<size_t>(encoded.quantizedReflectionCoefficients.size(), q.size()), q.begin());
    check(selab200_lpc_samples(encoded.residues.data(), 1, &order, q.data(), out.data()));
    return data::LpcDecodedData(encoded.bitsPerSample, std::move(out));
}

} // namespace lpc

// ------------------------------------------------------------------ frame --

namespace frame {

FrameEncoder::FrameEncoder(const data::WavFrame &wavFrame) : wavFrame(wavFrame) {}

// frame::FrameEncoder::process (src/frame/frame_encoder.cpp:11-102)
data::SelaFrame FrameEncoder::process()
{
    ensure_device();
    const uint32_t channels = (uint32_t)wavFrame.samples.size();
    if (channels == 0 || channels > SELAB200_MAX_CHANNELS)
        raise("sela_b200: unsupported channel count");
    for (const std::vector<int32_t> &plane : wavFrame.samples)
        if (plane.size() != kFrame)
            raise("sela_b200: frame::FrameEncoder needs 2048 samples per channel (the codec's frame size)");
    std::vector<int16_t> pcm((size_t)kFrame * channels);
    for (uint32_t j = 0; j < kFrame; j++)
        for (uint32_t c = 0; c < channels; c++)
            pcm[(size_t)j * channels + c] = narrow_sample(wavFrame.samples[c][j]);
    std::vector<selab200_subframe_desc> descs(channels);
    const size_t cap = selab200_encode_words_bound(1, channels);
    std::vector<uint32_t> words(cap);
    size_t used = 0;
    check(selab200_encode_frames(pcm.data(), 1, channels, descs.data(), words.data(), cap, &used));
    return frame_from_descs(descs.data(), channels, words.data(), wavFrame.bitsPerSample);
}

FrameDecoder::FrameDecoder(const data::SelaFrame &selaFrame) : selaFrame(selaFrame) {}

// frame::FrameDecoder::process (src/frame/frame_decoder.cpp:11-72)
data::WavFrame FrameDecoder::process()
{
    ensure_device();
    const uint32_t channels = (uint32_t)selaFrame.subFrames.size();
    if (channels == 0 || channels > SELAB200_MAX_CHANNELS)
        raise("sela_b200: unsupported channel count");
    std::vector<selab200_subframe_desc> descs(channels);
    std::vector<uint32_t> words(frame_words(selaFrame) + 4);
    size_t cursor = 0;
    flatten_frame(selaFrame, descs.data(), words.data(), cursor);
    std::vector<int16_t> pcm((size_t)kFrame * channels);
    check(selab200_decode_frames(descs.data(), 1, channels, words.data(), cursor, pcm.data()));
    std::vector<std::vector<int32_t>> planes(channels, std::vector<int32_t>(kFrame));
    for (uint32_t j = 0; j < kFrame; j++)
        for (uint32_t c = 0; c < channels; c++)
            planes[c][j] = pcm[(size_t)j * channels + c];
    return data::WavFrame(selaFrame.bitsPerSample, std::move(planes));
}

} // namespace frame

// ------------------------------------------------------------------- file --

namespace file {

// file::WavFile::WavFile (src/file/wav_file.cpp:7-37): canonical 44-byte header fields
WavFile::WavFile(uint32_t sampleRate, uint16_t bitsPerSample, uint16_t numChannels, std::vector<data::WavFrame> &&wavFrames)
{
    size_t payload = 0;
    for (const data::WavFrame &f : wavFrames)
        payload += f.samples.size() * (f.samples.empty() ? 0 : f.samples[0].size()) * (bitsPerSample / 8);
    wavChunk.chunkId = "RIFF";
    wavChunk.chunkSize = (uint32_t)(payload + 36);
    wavChunk.format = "WAVE";
    data::WavFormatSubChunk &fmt = wavChunk.formatSubChunk;
    fmt.subChunkId = "fmt ";
    fmt.subChunkSize = 16;
    fmt.audioFormat = 1;
    fmt.numChannels = numChannels;
    fmt.sampleRate = sampleRate;
    fmt.byteRate = (sampleRate * numChannels * bitsPerSample) / 8;
    fmt.blockAlign = (uint16_t)((numChannels * bitsPerSample) / 8);
    fmt.bitsPerSample = bitsPerSample;
    data::WavDataSubChunk &dat = wavChunk.dataSubChunk;
    dat.subChunkId = "data";
    dat.subChunkSize = (uint32_t)payload;
    dat.bitsPerSample = (uint8_t)bitsPerSample;
    dat.channels = (uint8_t)numChannels;
    dat.wavFrames = std::move(wavFrames);
}

// file::WavFile::readFromFile (src/file/wav_file.cpp:39-179): same acceptance rules and messages
// (scan_wav), then the reference's value structs filled from the spans it found.
void WavFile::readFromFile(std::ifstream &inputFile)
{
    const std::vector<char> contents = slurp(inputFile);
    const WavLayout w = scan_wav(contents.data(), contents.size());
    wavChunk.chunkId = "RIFF";
    wavChunk.chunkSize = w.chunkSize;
    wavChunk.format = "WAVE";
    wavChunk.wavSubChunks.clear();
    for (size_t i = 0; i < w.spans.size(); i++) {
        const WavSpan &span = w.spans[i];
        const auto first = contents.begin() + span.body, last = first + span.size;
        if (span.id == "fmt ") { // a later fmt chunk replaces an earlier one, as in the reference's loop
            data::WavFormatSubChunk fmt;
            const ByteView rd{contents.data()};
            fmt.subChunkId = span.id;
            fmt.subChunkSize = span.size;
            fmt.subChunkData.assign(first, last);
            fmt.audioFormat = (int16_t)rd.u16(span.body);
            fmt.numChannels = (uint16_t)rd.u16(span.body + 2);
            fmt.sampleRate = rd.u32(span.body + 4);
            fmt.byteRate = rd.u32(span.body + 8);
            fmt.blockAlign = (uint16_t)rd.u16(span.body + 12);
            fmt.bitsPerSample = (uint16_t)rd.u16(span.body + 14);
            wavChunk.formatSubChunk = fmt;
        } else if (span.id == "data") {
            data::WavDataSubChunk dat;
            dat.subChunkId = span.id;
            dat.subChunkSize = span.size;
            dat.bitsPerSample = 0; // the reference leaves these two zero as well (wav_file.cpp:84-85,134-135)
            dat.channels = 0;
            dat.subChunkData.assign(first, last);
            wavChunk.dataSubChunk = dat;
        } else {
            data::WavSubChunk other;
            other.subChunkId = span.id;
            other.subChunkSize = span.size;
            other.subChunkData.assign(first, last);
            wavChunk.wavSubChunks.push_back(other);
        }
    }
    demuxSamples();
}

// file::WavFile::demuxSamples (src/file/wav_file.cpp:181-220): whole frames only, the tail is dropped
void WavFile::demuxSamples()
{
    const uint32_t channels = wavChunk.formatSubChunk.numChannels;
    if (channels == 0)
        raise("fmt subChunk declares zero channels");
    const std::vector<int8_t> &raw = wavChunk.dataSubChunk.subChunkData;
    const size_t sampleCount = (raw.size() * 8) / wavChunk.formatSubChunk.bitsPerSample;
    const size_t n_frames = sampleCount / (samplesPerChannelPerFrame * channels);
    std::vector<data::WavFrame> &frames = wavChunk.dataSubChunk.wavFrames;
    frames.clear();
    frames.reserve(n_frames);
    const int16_t *pcm = reinterpret_cast<const int16_t *>(raw.data()); // little-endian host
    for (size_t f = 0; f < n_frames; f++) {
        std::vector<std::vector<int32_t>> planes(channels, std::vector<int32_t>(samplesPerChannelPerFrame));
        const int16_t *src = pcm + f * samplesPerChannelPerFrame * channels;
        for (size_t j = 0; j < samplesPerChannelPerFrame; j++)
            for (uint32_t c = 0; c < channels; c++)
                planes[c][j] = src[j * channels + c];
        frames.push_back(data::WavFrame((uint8_t)wavChunk.formatSubChunk.bitsPerSample, std::move(planes)));
    }
}

// file::WavFile::writeToFile (src/file/wav_file.cpp:222-267): same bytes for every channel count
// (the reference has a fast path for stereo only; the layout is identical)
void WavFile::writeToFile(std::ofstream &outputFile)
{
    write_wav_header(outputFile, wavChunk);
    std::vector<int16_t> block;
    for (const data::WavFrame &f : wavChunk.dataSubChunk.wavFrames) {
        const size_t channels = f.samples.size();
        const size_t n = channels ? f.samples[0].size() : 0;
        block.resize(n * channels);
        for (size_t j = 0; j < n; j++)
            for (size_t c = 0; c < channels; c++)
                block[j * channels + c] = (int16_t)(uint16_t)f.samples[c][j];
        outputFile.write(reinterpret_cast<const char *>(block.data()), (std::streamsize)(block.size() * 2));
    }
}

// file::SelaFile::SelaFile (src/file/sela_file.cpp:10-17)
SelaFile::SelaFile(uint32_t sampleRate, uint16_t bitsPerSample, uint8_t channels, std::vector<data::SelaFrame> &&frames)
    : selaFrames(frames)
{
    selaHeader.sampleRate = sampleRate;
    selaHeader.bitsPerSample = bitsPerSample;
    selaHeader.channels = channels;
    selaHeader.numFrames = (uint32_t)selaFrames.size();
}

// file::SelaFile::readFromFile (src/file/sela_file.cpp:19-103).  Container: 15-byte header
// ("SeLa", rate u32, bits u16, channels u8, frames u32) then per frame the sync word
// 0xAA55FF00 and per subframe 3+4 header bytes, refl words, 5 header bytes, residue words.
// Stops quietly at the first bad sync word, as the reference does; unlike it, never reads
// past the end of the buffer.
void SelaFile::readFromFile(std::ifstream &inputFile)
{
    const std::vector<char> contents = slurp(inputFile);
    const Bytes rd{contents};
    if (contents.size() < 15)
        raise("File is too small, probably not a sela file.");
    if (rd.tag(0) != "SeLa")
        raise("Magic number is incorrect, probably not a sela file.");
    selaHeader.sampleRate = rd.u32(4);
    selaHeader.bitsPerSample = (uint16_t)rd.u16(8);
    selaHeader.channels = (uint8_t)rd.u8(10);
    selaHeader.numFrames = rd.u32(11);
    size_t at = 15;
    auto need = [&](size_t n) {
        if (at + n > contents.size())
            raise("sela file is truncated");
    };
    auto words_at = [&](size_t count) {
        need(count * 4);
        std::vector<uint32_t> w(count);
        if (count)
            std::memcpy(w.data(), contents.data() + at, count * 4); // little-endian host
        at += count * 4;
        return w;
    };
    selaFrames.clear();
    // numFrames is only a promise: never reserve more frames than the bytes could hold
    selaFrames.reserve(std::min<size_t>(selaHeader.numFrames,
                                        contents.size() / (4 + 12 * std::max<size_t>(1, selaHeader.channels))));
    for (uint32_t f = 0; f < selaHeader.numFrames; f++) {
        if (at + 4 > contents.size() || rd.u32(at) != 0xAA55FF00u)
            break;
        at += 4;
        data::SelaFrame frame((uint8_t)selaHeader.bitsPerSample);
        frame.subFrames.reserve(selaHeader.channels);
        for (uint32_t c = 0; c < selaHeader.channels; c++) {
            need(7);
            const uint8_t channel = (uint8_t)rd.u8(at), type = (uint8_t)rd.u8(at + 1), parent = (uint8_t)rd.u8(at + 2);
            const uint8_t reflK = (uint8_t)rd.u8(at + 3);
            const uint16_t reflInts = (uint16_t)rd.u16(at + 4);
            const uint8_t order = (uint8_t)rd.u8(at + 6);
            at += 7;
            data::RiceEncodedData refl(reflK, order, words_at(reflInts));
            need(5);
            const uint8_t resK = (uint8_t)rd.u8(at);
            const uint16_t resInts = (uint16_t)rd.u16(at + 1), samples = (uint16_t)rd.u16(at + 3);
            at += 5;
            data::RiceEncodedData res(resK, samples, words_at(resInts));
            frame.subFrames.push_back(data::SelaSubFrame(channel, type, parent, refl, res));
        }
        selaFrames.push_back(frame);
    }
}

// file::SelaFile::writeToFile (src/file/sela_file.cpp:105-137)
void SelaFile::writeToFile(std::ofstream &outputFile)
{
    outputFile.write(reinterpret_cast<const char *>(selaHeader.magicNumber), 4);
    put(outputFile, selaHeader.sampleRate);
    put(outputFile, selaHeader.bitsPerSample);
    put(outputFile, selaHeader.channels);
    put(outputFile, selaHeader.numFrames);
    for (const data::SelaFrame &frame : selaFrames) {
        put(outputFile, frame.syncWord);
        for (const data::SelaSubFrame &s : frame.subFrames) {
            put(outputFile, s.channel);
            put(outputFile, s.subFrameType);
            put(outputFile, s.parentChannelNumber);
            put(outputFile, s.reflectionCoefficientRiceParam);
            put(outputFile, s.reflectionCoefficientRequiredInts);
            put(outputFile, s.optimumLpcOrder);
            outputFile.write(reinterpret_cast<const char *>(s.encodedReflectionCoefficients.data()),
                             (std::streamsize)(s.encodedReflectionCoefficients.size() * 4));
            put(outputFile, s.residueRiceParam);
            put(outputFile, s.residueRequiredInts);
            put(outputFile, s.samplesPerChannel);
            outputFile.write(reinterpret_cast<const char *>(s.encodedResidues.data()),
                             (std::streamsize)(s.encodedResidues.size() * 4));
        }
    }
}

} // namespace file

// ------------------------------------------------------------------- sela --

namespace sela {

void Encoder::readFrames() { wavFile.readFromFile(ifStream); }

// sela::Encoder::processFrames (src/sela/encoder.cpp:40-92): the reference fans the frames
// out over hardware_concurrency() threads; here the whole file is ONE batch on the GPU
// and the frames come back in order.
void Encoder::processFrames(std::vector<data::SelaFrame> &encodedSelaFrames)
{
    ensure_device();
    const std::vector<data::WavFrame> &frames = wavFile.wavChunk.dataSubChunk.wavFrames;
    const uint32_t n_frames = (uint32_t)frames.size();
    encodedSelaFrames.reserve(n_frames);
    if (n_frames == 0)
        return;
    const uint32_t channels = (uint32_t)frames[0].samples.size();
    if (channels == 0 || channels > SELAB200_MAX_CHANNELS)
        raise("sela_b200: unsupported channel count");
    const size_t n_samples = (size_t)n_frames * channels * kFrame;
    Pinned<int16_t> pcm(n_samples);
    const std::vector<int8_t> &raw = wavFile.wavChunk.dataSubChunk.subChunkData;
    if (raw.size() >= n_samples * 2) {
        std::memcpy(pcm.p, raw.data(), n_samples * 2); // the data chunk IS the interleaved layout
    } else {
        for (uint32_t f = 0; f < n_frames; f++)
            for (uint32_t j = 0; j < kFrame; j++)
                for (uint32_t c = 0; c < channels; c++)
                    pcm.p[((size_t)f * kFrame + j) * channels + c] = narrow_sample(frames[f].samples[c][j]);
    }
    const size_t cap = selab200_encode_words_bound(n_frames, channels);
    Pinned<selab200_subframe_desc> descs((size_t)n_frames * channels);
    Pinned<uint32_t> words(cap);
    size_t used = 0;
    check(selab200_encode_frames(pcm.p, n_frames, channels, descs.p, words.p, cap, &used));
    const uint8_t bits = frames[0].bitsPerSample;
    for (uint32_t f = 0; f < n_frames; f++)
        encodedSelaFrames.push_back(frame_from_descs(descs.p + (size_t)f * channels, channels, words.p, bits));
}

// sela::Encoder::process (src/sela/encoder.cpp:94-99)
file::SelaFile Encoder::process()
{
    std::vector<data::SelaFrame> frames;
    readFrames();
    processFrames(frames);
    const data::WavFormatSubChunk &fmt = wavFile.wavChunk.formatSubChunk;
    return file::SelaFile(fmt.sampleRate, fmt.bitsPerSample, (uint8_t)fmt.numChannels, std::move(frames));
}

// The library's report in the mirror's terms.
static std::vector<VerifyEntry> mirror_report(const std::vector<selab200_verify_entry> &raw, size_t n)
{
    std::vector<VerifyEntry> out;
    out.reserve(n);
    for (size_t i = 0; i < n && i < raw.size(); i++)
        out.push_back(VerifyEntry{raw[i].frame, raw[i].channel, raw[i].first_sample, raw[i].n_differing, raw[i].first_delta});
    return out;
}

// process() + file::SelaFile::writeToFile() without the detour through per-frame value structs:
// the data chunk is handed to the device where it lies in the file buffer, and what comes back is
// the .sela byte stream.  Output is byte-identical to the two-step path (tests/test_host_cli.py).
void Encoder::processTo(std::ofstream &outputFile) { encodeTo(outputFile, nullptr, nullptr); }

void Encoder::processTo(std::ofstream &outputFile, std::vector<VerifyEntry> &report) { encodeTo(outputFile, &report, nullptr); }

void Encoder::processLosslessTo(std::ofstream &outputFile, std::vector<RecodedEntry> &recoded)
{
    encodeTo(outputFile, nullptr, &recoded);
}

size_t Encoder::processSearchTo(std::ofstream &outputFile, size_t &refBytes)
{
    const std::streampos at = outputFile.tellp();
    encodeTo(outputFile, nullptr, nullptr, &refBytes);
    return (size_t)(outputFile.tellp() - at);
}

size_t Encoder::processPairingTo(std::ofstream &outputFile, size_t &losslessBytes, size_t &differences)
{
    const std::streampos at = outputFile.tellp();
    encodeTo(outputFile, nullptr, nullptr, &losslessBytes, &differences);
    return (size_t)(outputFile.tellp() - at);
}

size_t Encoder::processSearchPairingTo(std::ofstream &outputFile, size_t &searchBytes, size_t &differences)
{
    const std::streampos at = outputFile.tellp();
    encodeTo(outputFile, nullptr, nullptr, &searchBytes, &differences, true);
    return (size_t)(outputFile.tellp() - at);
}

size_t Encoder::processSearchWindowsTo(std::ofstream &outputFile, uint32_t windows, size_t &searchBytes,
                                       size_t &windowUnits)
{
    const std::streampos at = outputFile.tellp();
    encodeTo(outputFile, nullptr, nullptr, &searchBytes, &windowUnits, false, windows);
    return (size_t)(outputFile.tellp() - at);
}

size_t Encoder::processSearchGuidedTo(std::ofstream &outputFile, uint32_t candidates, size_t &refBytes)
{
    const std::streampos at = outputFile.tellp();
    encodeTo(outputFile, nullptr, nullptr, &refBytes, nullptr, false, 0, candidates);
    return (size_t)(outputFile.tellp() - at);
}

// processTo(); with `report` through selab200_encode_container_verified (same bytes), with `recoded` through
// selab200_encode_container_lossless, with `refBytes` through selab200_encode_container_search, with `differences`
// as well through selab200_encode_container_pairing, and with `searchBase` too through
// selab200_encode_container_search_pairing.  With `windows` (and refBytes, differences) through
// selab200_encode_container_search_windows, `differences` receiving the units coded from a window.  With
// `candidates` (and refBytes) through selab200_encode_container_search_guided.
void Encoder::encodeTo(std::ofstream &outputFile, std::vector<VerifyEntry> *report, std::vector<RecodedEntry> *recoded,
                       size_t *refBytes, size_t *differences, bool searchBase, uint32_t windows, uint32_t candidates)
{
    if (differences)
        *differences = 0;
    if (report)
        report->clear();
    if (recoded)
        recoded->clear();
    StagingScope staging;
    DeviceWarmup warmup; // CUDA context creation overlaps the file read
    if (g_batch_mode.load())
        warmup.join();   // page-locked staging needs the device; it is up after the first file anyway
    RawFile file;
    {
        Phase p("read input");
        file = slurp_raw(ifStream);
    }
    const WavLayout w = scan_wav(file.data, file.size);
    const WavSpan &dat = w.spans[w.dataIndex];
    const uint32_t channels = w.fmt.numChannels;
    if (channels == 0)
        raise("fmt subChunk declares zero channels");
    // file::WavFile::demuxSamples (src/file/wav_file.cpp:181-220): whole frames only
    const size_t sampleCount = ((size_t)dat.size * 8) / w.fmt.bitsPerSample;
    const size_t n_frames = sampleCount / ((size_t)kFrame * channels);
    warmup.join();
    if (n_frames > 0 && channels > SELAB200_MAX_CHANNELS)
        raise("sela_b200: unsupported channel count");
    if (n_frames > UINT32_MAX)
        raise("sela_b200: too many frames");
    if (n_frames == 0) { // header only, as SelaFile::writeToFile does for an empty frame list
        file::SelaFile(w.fmt.sampleRate, w.fmt.bitsPerSample, (uint8_t)channels, {}).writeToFile(outputFile);
        if (refBytes)
            *refBytes = 15;
        return;
    }
    const size_t cap = selab200_container_bound((uint32_t)n_frames, channels);
    uint8_t *out = reinterpret_cast<uint8_t *>(t_output.ensure(cap));
    size_t used = 0;
    if (report) {
        Phase p("encode + verify (device)");
        std::vector<selab200_verify_entry> raw(n_frames * channels);
        size_t n = 0;
        check(selab200_encode_container_verified(reinterpret_cast<const int16_t *>(file.data + dat.body),
                                                 (uint32_t)n_frames, channels, w.fmt.sampleRate, w.fmt.bitsPerSample,
                                                 out, cap, &used, raw.data(), raw.size(), &n));
        *report = mirror_report(raw, n);
    } else if (recoded) {
        Phase p("lossless encode (device)");
        std::vector<selab200_lossless_entry> raw(n_frames * channels);
        size_t n = 0;
        check(selab200_encode_container_lossless(reinterpret_cast<const int16_t *>(file.data + dat.body),
                                                 (uint32_t)n_frames, channels, w.fmt.sampleRate, w.fmt.bitsPerSample,
                                                 out, cap, &used, raw.data(), raw.size(), &n));
        for (size_t i = 0; i < n && i < raw.size(); i++)
            recoded->push_back(RecodedEntry{raw[i].frame, raw[i].channel, raw[i].ref_order, raw[i].order,
                                            raw[i].ref_words, raw[i].words});
    } else if (windows) {
        Phase p("window-search encode (device)");
        check(selab200_encode_container_search_windows(reinterpret_cast<const int16_t *>(file.data + dat.body),
                                                       (uint32_t)n_frames, channels, windows, w.fmt.sampleRate,
                                                       w.fmt.bitsPerSample, out, cap, &used, refBytes, differences));
    } else if (candidates) {
        Phase p("guided order-search encode (device)");
        check(selab200_encode_container_search_guided(reinterpret_cast<const int16_t *>(file.data + dat.body),
                                                      (uint32_t)n_frames, channels, candidates, w.fmt.sampleRate,
                                                      w.fmt.bitsPerSample, out, cap, &used, refBytes));
    } else if (differences && searchBase) {
        Phase p("order-search + pairing encode (device)");
        check(selab200_encode_container_search_pairing(reinterpret_cast<const int16_t *>(file.data + dat.body),
                                                       (uint32_t)n_frames, channels, w.fmt.sampleRate,
                                                       w.fmt.bitsPerSample, out, cap, &used, refBytes, differences));
    } else if (differences) {
        Phase p("pairing encode (device)");
        check(selab200_encode_container_pairing(reinterpret_cast<const int16_t *>(file.data + dat.body),
                                                (uint32_t)n_frames, channels, w.fmt.sampleRate, w.fmt.bitsPerSample,
                                                out, cap, &used, refBytes, differences));
    } else if (refBytes) {
        Phase p("order-search encode (device)");
        check(selab200_encode_container_search(reinterpret_cast<const int16_t *>(file.data + dat.body),
                                               (uint32_t)n_frames, channels, w.fmt.sampleRate, w.fmt.bitsPerSample,
                                               out, cap, &used, refBytes));
    } else {
        Phase p("encode (device)");
        check(selab200_encode_container(reinterpret_cast<const int16_t *>(file.data + dat.body), (uint32_t)n_frames,
                                        channels, w.fmt.sampleRate, w.fmt.bitsPerSample, out, cap, &used));
    }
    Phase p("write output");
    outputFile.write(reinterpret_cast<const char *>(out), (std::streamsize)used);
}

void Decoder::readFrames() { selaFile.readFromFile(ifStream); }

// process() + file::WavFile::writeToFile() in one step: the .sela bytes go to the device as they
// lie in the file (the library walks the frame headers while the upload runs), interleaved int16
// PCM -- the WAV data chunk -- comes back.
void Decoder::processTo(std::ofstream &outputFile)
{
    StagingScope staging;
    DeviceWarmup warmup;
    if (g_batch_mode.load())
        warmup.join();
    RawFile file;
    {
        Phase p("read input");
        file = slurp_raw(ifStream);
    }
    warmup.join();
    selab200_container *handle = nullptr;
    selab200_container_info info;
    {
        Phase p("open (upload + walk)");
        if (selab200_container_open(file.bytes(), file.size, &handle, &info) != SELAB200_OK)
            raise(selab200_last_error()); // the reader's own messages (too small / magic / truncated)
    }
    struct Closer {
        selab200_container *h;
        ~Closer() { selab200_container_close(h); }
    } closer{handle};
    if (info.n_frames > 0 && (info.channels == 0 || info.channels > SELAB200_MAX_CHANNELS))
        raise("sela_b200: unsupported channel count");
    const size_t n_samples = (size_t)info.n_frames * info.channels * kFrame;
    int16_t *pcm = reinterpret_cast<int16_t *>(t_output.ensure((n_samples + 1) * 2));
    {
        Phase p("decode (device)");
        check(selab200_container_decode(handle, pcm));
    }
    Phase p("write output");
    // header exactly as file::WavFile::WavFile computes it from the decoded frames (wav_file.cpp:7-37)
    file::WavFile shell(info.sample_rate, info.bits_per_sample, info.channels, {});
    const size_t payload = n_samples * (info.bits_per_sample / 8);
    shell.wavChunk.chunkSize = (uint32_t)(payload + 36);
    shell.wavChunk.dataSubChunk.subChunkSize = (uint32_t)payload;
    write_wav_header(outputFile, shell.wavChunk);
    outputFile.write(reinterpret_cast<const char *>(pcm), (std::streamsize)(n_samples * 2));
}

// processTo() for one sample range: the container opens as for processTo(), and one clip comes back.
void Decoder::processRangeTo(std::ofstream &outputFile, uint64_t firstSample, uint64_t nSamples)
{
    processRangeTo(outputFile, firstSample, nSamples, {});
}

// The same for the channels listed (all of them if the list is empty): only the subframes they need are decoded.
void Decoder::processRangeTo(std::ofstream &outputFile, uint64_t firstSample, uint64_t nSamples,
                             const std::vector<uint8_t> &channels)
{
    StagingScope staging;
    DeviceWarmup warmup;
    RawFile file;
    {
        Phase p("read input");
        file = slurp_raw(ifStream);
    }
    warmup.join();
    selab200_container *handle = nullptr;
    selab200_container_info info;
    {
        Phase p("open (upload + walk)");
        if (selab200_container_open(file.bytes(), file.size, &handle, &info) != SELAB200_OK)
            raise(selab200_last_error());
    }
    struct Closer {
        selab200_container *h;
        ~Closer() { selab200_container_close(h); }
    } closer{handle};
    if (nSamples == 0 || nSamples > 0xffffffffull)
        raise("sela_b200: the sample count must be in [1, 2^32 - 1]");
    if (info.channels == 0 || info.channels > SELAB200_MAX_CHANNELS)
        raise("sela_b200: unsupported channel count");
    const uint32_t n_out = channels.empty() ? info.channels : (uint32_t)channels.size();
    const size_t n_values = (size_t)nSamples * n_out;
    int16_t *pcm = reinterpret_cast<int16_t *>(t_output.ensure((n_values + 1) * 2));
    {
        Phase p("decode range (device)");
        const selab200_clip clip{0, 0, firstSample};
        uint64_t frames = 0, subframes = 0;
        if (channels.empty())
            check(selab200_container_decode_clips(&handle, 1, &clip, 1, (uint32_t)nSamples, pcm, &frames));
        else
            check(selab200_container_decode_clips_select(&handle, 1, &clip, 1, (uint32_t)nSamples, channels.data(),
                                                         (uint32_t)channels.size(), 0, pcm, &frames, &subframes));
    }
    Phase p("write output");
    file::WavFile shell(info.sample_rate, info.bits_per_sample, (uint16_t)n_out, {});
    const size_t payload = n_values * (info.bits_per_sample / 8);
    shell.wavChunk.chunkSize = (uint32_t)(payload + 36);
    shell.wavChunk.dataSubChunk.subChunkSize = (uint32_t)payload;
    write_wav_header(outputFile, shell.wavChunk);
    outputFile.write(reinterpret_cast<const char *>(pcm), (std::streamsize)(n_values * 2));
}

// The .sela stream against a WAV file: the .sela bytes go to the device as processTo() sends them, the WAV's
// data chunk goes up chunk by chunk from where it lies in the file buffer, and only the report comes back.
std::vector<VerifyEntry> Decoder::verifyAgainst(std::ifstream &wavInput)
{
    StagingScope staging;
    DeviceWarmup warmup;
    if (g_batch_mode.load())
        warmup.join();
    RawFile file;
    char *wav = nullptr;
    size_t wav_size = 0;
    {
        Phase p("read inputs");
        file = slurp_raw(ifStream);
        wavInput.seekg(0, std::ios::end);
        const std::streamoff size = wavInput.tellg();
        wav_size = size > 0 ? (size_t)size : 0;
        wav = t_output.ensure(wav_size + 1);
        wavInput.seekg(0, std::ios::beg);
        if (wav_size)
            wavInput.read(wav, (std::streamsize)wav_size);
    }
    const WavLayout w = scan_wav(wav, wav_size);
    const WavSpan &dat = w.spans[w.dataIndex];
    warmup.join();
    selab200_container *handle = nullptr;
    selab200_container_info info;
    {
        Phase p("open (upload + walk)");
        if (selab200_container_open(file.bytes(), file.size, &handle, &info) != SELAB200_OK)
            raise(selab200_last_error());
    }
    struct Closer {
        selab200_container *h;
        ~Closer() { selab200_container_close(h); }
    } closer{handle};
    const uint32_t channels = w.fmt.numChannels;
    if (channels != info.channels)
        raise("the WAV file has " + std::to_string(channels) + " channels, the sela file " + std::to_string(info.channels));
    if (w.fmt.sampleRate != info.sample_rate)
        raise("the WAV file's sample rate is " + std::to_string(w.fmt.sampleRate) + " Hz, the sela file's " +
              std::to_string(info.sample_rate) + " Hz");
    // file::WavFile::demuxSamples (src/file/wav_file.cpp:181-220): whole frames only
    const size_t wav_frames = channels ? ((size_t)dat.size * 8 / w.fmt.bitsPerSample) / ((size_t)kFrame * channels) : 0;
    if (wav_frames != info.header_frames)
        raise("the WAV file holds " + std::to_string(wav_frames) + " whole frames, the sela header declares " +
              std::to_string(info.header_frames));
    if (info.n_frames != info.header_frames)
        raise("the sela file holds " + std::to_string(info.n_frames) + " of the " + std::to_string(info.header_frames) +
              " frames its header declares");
    if (info.n_frames > 0 && (channels == 0 || channels > SELAB200_MAX_CHANNELS))
        raise("sela_b200: unsupported channel count");
    std::vector<selab200_verify_entry> raw((size_t)info.n_frames * channels);
    size_t n = 0;
    {
        Phase p("verify (device)");
        check(selab200_container_verify(handle, reinterpret_cast<const int16_t *>(wav + dat.body), raw.data(), raw.size(), &n));
    }
    return mirror_report(raw, n);
}

// sela::Decoder::processFrames (src/sela/decoder.cpp:41-92)
void Decoder::processFrames(std::vector<data::WavFrame> &decodedWavFrames)
{
    ensure_device();
    const std::vector<data::SelaFrame> &frames = selaFile.selaFrames;
    const uint32_t n_frames = (uint32_t)frames.size();
    decodedWavFrames.reserve(n_frames);
    if (n_frames == 0)
        return;
    const uint32_t channels = (uint32_t)frames[0].subFrames.size();
    if (channels == 0 || channels > SELAB200_MAX_CHANNELS)
        raise("sela_b200: unsupported channel count");
    size_t total_words = 0;
    for (const data::SelaFrame &f : frames) {
        if (f.subFrames.size() != channels)
            raise("sela_b200: frames with differing channel counts");
        total_words += frame_words(f);
    }
    Pinned<selab200_subframe_desc> descs((size_t)n_frames * channels);
    Pinned<uint32_t> words(total_words + 4);
    size_t cursor = 0;
    for (uint32_t f = 0; f < n_frames; f++)
        flatten_frame(frames[f], descs.p + (size_t)f * channels, words.p, cursor);
    Pinned<int16_t> pcm((size_t)n_frames * channels * kFrame);
    check(selab200_decode_frames(descs.p, n_frames, channels, words.p, cursor, pcm.p));
    const uint8_t bits = (uint8_t)selaFile.selaHeader.bitsPerSample;
    for (uint32_t f = 0; f < n_frames; f++) {
        std::vector<std::vector<int32_t>> planes(channels, std::vector<int32_t>(kFrame));
        const int16_t *src = pcm.p + (size_t)f * channels * kFrame;
        for (uint32_t j = 0; j < kFrame; j++)
            for (uint32_t c = 0; c < channels; c++)
                planes[c][j] = src[(size_t)j * channels + c];
        decodedWavFrames.push_back(data::WavFrame(bits, std::move(planes)));
    }
}

// sela::Decoder::process (src/sela/decoder.cpp:94-99)
file::WavFile Decoder::process()
{
    std::vector<data::WavFrame> frames;
    readFrames();
    processFrames(frames);
    return file::WavFile(selaFile.selaHeader.sampleRate, selaFile.selaHeader.bitsPerSample,
                         selaFile.selaHeader.channels, std::move(frames));
}

void setBatchMode(bool on) { g_batch_mode.store(on); }

void Player::play(const file::WavFile &)
{
    raise("playback is not part of this build (libao output is out of scope); decode with -d instead");
}

} // namespace sela
