// sela_api.hpp -- the reference's operator interface for the hot path and its callers,
// re-implemented on top of the CUDA C ABI (include/sela_b200.h).  Class names, method
// names, argument meaning and error behaviour follow the reference; none of the
// computation happens on the CPU.
//
//   rice::RiceEncoder / RiceDecoder           src/include/rice.hpp:10-42
//   lpc::ResidueGenerator / SampleGenerator   src/include/lpc.hpp:86-116
//   frame::FrameEncoder / FrameDecoder        src/include/frame.hpp:8-24
//   file::WavFile / SelaFile                  src/include/file/wav_file.hpp:10-19, sela_file.hpp:10-18
//   sela::Encoder / Decoder                   src/include/sela/encoder.hpp:9-22, decoder.hpp:9-22
//   sela::Player                              src/include/sela/player.hpp:27 (stub: no audio device here)
//
// Errors from the device layer surface as `throw data::Exception(message)`, the
// reference's convention.
#pragma once

#include <fstream>

#include "sela_types.hpp"

constexpr uint8_t MAX_LPC_ORDER = 100;   // src/include/lpc.hpp:7
constexpr uint8_t CORRECTION_FACTOR = 35; // src/include/lpc.hpp:8
constexpr uint8_t MAX_RICE_PARAM = 20;   // src/include/rice.hpp:7

namespace rice {
class RiceEncoder {
    const std::vector<int32_t> &input;

public:
    explicit RiceEncoder(const data::RiceDecodedData &decodedData);
    data::RiceEncodedData process();
};
class RiceDecoder {
    const std::vector<uint32_t> &input;
    uint32_t dataCount;
    uint32_t optimumRiceParam;

public:
    explicit RiceDecoder(const data::RiceEncodedData &encodedData);
    data::RiceDecodedData process();
};
} // namespace rice

namespace lpc {
class ResidueGenerator {
    const std::vector<int32_t> &samples;
    uint8_t bitsPerSample;

public:
    explicit ResidueGenerator(const data::LpcDecodedData &data);
    data::LpcEncodedData process();
};
class SampleGenerator {
    const data::LpcEncodedData &encoded;

public:
    explicit SampleGenerator(const data::LpcEncodedData &encodedData);
    data::LpcDecodedData process();
};
} // namespace lpc

namespace frame {
class FrameEncoder {
    const data::WavFrame &wavFrame;

public:
    explicit FrameEncoder(const data::WavFrame &wavFrame);
    data::SelaFrame process();
};
class FrameDecoder {
    const data::SelaFrame &selaFrame;

public:
    explicit FrameDecoder(const data::SelaFrame &selaFrame);
    data::WavFrame process();
};
} // namespace frame

namespace file {
class WavFile {
public:
    size_t samplesPerChannelPerFrame = 2048;
    void demuxSamples();
    data::WavChunk wavChunk;
    WavFile() {}
    WavFile(uint32_t sampleRate, uint16_t bitsPerSample, uint16_t numChannels, std::vector<data::WavFrame> &&wavFrames);
    void readFromFile(std::ifstream &inputFile);
    void writeToFile(std::ofstream &outputFile);
};
class SelaFile {
public:
    data::SelaHeader selaHeader;
    std::vector<data::SelaFrame> selaFrames;
    void readFromFile(std::ifstream &inputFile);
    void writeToFile(std::ofstream &outputFile);
    SelaFile() {}
    SelaFile(uint32_t sampleRate, uint16_t bitsPerSample, uint8_t channels, std::vector<data::SelaFrame> &&selaFrames);
};
} // namespace file

namespace sela {
// Not in the reference: one decoded (frame, channel) that differs from its source (selab200_verify_entry).
// The format is not lossless for every input: encoder and decoder round the prediction differently when it
// lands exactly on a half, and the decoded channel drifts away from the source from that sample on.
struct VerifyEntry {
    uint32_t frame;
    uint16_t channel;
    uint16_t firstSample;      // first differing sample, within the frame
    uint32_t differingSamples; // how many of the frame's 2048 samples differ
    int32_t firstDelta;        // decoded - source at firstSample
};

// Not in the reference: one subframe a lossless encode emits in place of the reference encoder's
// (selab200_lossless_entry): that subframe's order and words (reflection + residue), and the emitted one's.
struct RecodedEntry {
    uint32_t frame;
    uint16_t channel;
    uint8_t refOrder, order;
    uint32_t refWords, words;
};

class Encoder {
    void readFrames();
    void processFrames(std::vector<data::SelaFrame> &encodedSelaFrames);
    void encodeTo(std::ofstream &outputFile, std::vector<VerifyEntry> *report, std::vector<RecodedEntry> *recoded,
                  size_t *refBytes = nullptr, size_t *differences = nullptr, bool searchBase = false,
                  uint32_t windows = 0, uint32_t candidates = 0);
    std::ifstream &ifStream;
    file::WavFile wavFile;

public:
    explicit Encoder(std::ifstream &ifStream) : ifStream(ifStream) {}
    file::SelaFile process();
    // Not in the reference: process() + SelaFile::writeToFile() in one step, byte-identical output.
    // The WAV data chunk goes to the device as it lies in the file and the .sela byte stream comes
    // back ready to write (selab200_encode_container): no per-frame value structs on the host.
    void processTo(std::ofstream &outputFile);
    // Not in the reference: processTo() that also proves what it wrote (`flac --verify`): the bytes are decoded
    // on the device and compared with the WAV's whole frames.  Same bytes as processTo(); `report` receives
    // every (frame, channel) that does not decode back to its source, in order (empty: lossless).
    void processTo(std::ofstream &outputFile, std::vector<VerifyEntry> &report);
    // Not in the reference: processTo() writing a file that decodes back to its source under the unmodified
    // reference decoder (selab200_encode_container_lossless).  Frames without a tie keep processTo()'s bytes;
    // `recoded` receives every (frame, channel) coded differently, in order.
    void processLosslessTo(std::ofstream &outputFile, std::vector<RecodedEntry> &recoded);
    // Not in the reference: processTo() writing a smaller file at a higher encode cost: every subframe at the
    // predictor order with the fewest words whose FIR has no tie (selab200_encode_container_search), so it also
    // decodes back to its source under the unmodified reference decoder.  Returns the bytes written; `refBytes`
    // receives the bytes processTo() writes for the same input.
    size_t processSearchTo(std::ofstream &outputFile, size_t &refBytes);
    // Not in the reference: processLosslessTo() writing a smaller file of correlated channels: every channel of a
    // frame coded alone or as its difference from another channel of the frame, whichever assignment takes the
    // fewest words (selab200_encode_container_pairing).  Returns the bytes written; `losslessBytes` receives the
    // bytes processLosslessTo() writes for the same input, `differences` the number of difference subframes.
    size_t processPairingTo(std::ofstream &outputFile, size_t &losslessBytes, size_t &differences);
    // Not in the reference: the smallest of these files, at the highest encode cost: processPairingTo() on top of
    // processSearchTo(), every channel and every channel difference at the order with the fewest words
    // (selab200_encode_container_search_pairing).  Returns the bytes written; `searchBytes` receives the bytes
    // processSearchTo() writes for the same input, `differences` the number of difference subframes.
    size_t processSearchPairingTo(std::ofstream &outputFile, size_t &searchBytes, size_t &differences);
    // Not in the reference: processSearchTo(), and every subframe also searched from the analysis of each window in
    // the mask `windows` (bit 0 Tukey(0.5), 1 Tukey(0.25), 2 Hann, 3 and 4 Tukey(0.5) over each half frame), coded
    // from whichever analysis and order takes the fewest words (selab200_encode_container_search_windows).  Returns
    // the bytes written; `searchBytes` receives the bytes processSearchTo() writes for the same input, `windowUnits`
    // the number of analysis units coded from a window.
    size_t processSearchWindowsTo(std::ofstream &outputFile, uint32_t windows, size_t &searchBytes,
                                  size_t &windowUnits);
    // Not in the reference: processSearchTo() over only the `candidates` (1..100) orders a reflection-coefficient
    // estimate ranks best, order 1 and the reference order (selab200_encode_container_search_guided).  Returns the
    // bytes written; `refBytes` receives the bytes processTo() writes for the same input.
    size_t processSearchGuidedTo(std::ofstream &outputFile, uint32_t candidates, size_t &refBytes);
};
class Decoder {
    void readFrames();
    void processFrames(std::vector<data::WavFrame> &decodedWavFrames);
    std::ifstream &ifStream;
    file::SelaFile selaFile;

public:
    explicit Decoder(std::ifstream &ifStream) : ifStream(ifStream) {}
    file::WavFile process();
    // Not in the reference: process() + WavFile::writeToFile() in one step, byte-identical output
    // (selab200_container_open / _decode: the .sela bytes go to the device as they lie in the file).
    void processTo(std::ofstream &outputFile);
    // Not in the reference: processTo() for samples [firstSample, firstSample + nSamples) of every channel only
    // (selab200_container_decode_clips: only the frames the range covers are decoded).  The header is the one
    // processTo() writes for that many samples; the data chunk equals the same bytes of processTo()'s.
    void processRangeTo(std::ofstream &outputFile, uint64_t firstSample, uint64_t nSamples);
    // The same for only the channels listed, in that order (repeats allowed): a WAV of that many channels, from only
    // the subframes they need (selab200_container_decode_clips_select).  An empty list means every channel.
    void processRangeTo(std::ofstream &outputFile, uint64_t firstSample, uint64_t nSamples,
                        const std::vector<uint8_t> &channels);
    // Not in the reference: decode this .sela stream on the device and compare it with the whole frames of the
    // WAV file `wavInput` (its partial final frame is ignored, as the encoder ignores it).  Returns every
    // (frame, channel) that differs, in order.  Throws data::Exception if the WAV's channels, sample rate or
    // whole-frame count disagree with the .sela header.
    std::vector<VerifyEntry> verifyAgainst(std::ifstream &wavInput);
};
// Not in the reference.  On: the processTo() drivers keep page-locked staging buffers per host thread
// and reuse them from file to file (a process that codes many files, e.g. `sela -E`); off (default):
// plain memory, released when the call returns.
void setBatchMode(bool on);

class Player {
public:
    void play(const file::WavFile &wavFile); // always throws: playback (libao) is out of scope
};
} // namespace sela
