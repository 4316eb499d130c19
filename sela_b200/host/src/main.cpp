// sela -- command-line front end over the GPU codec.  Same contract as the reference CLI
// (src/main.cpp:16-27, 53-107): `-e in.wav out.sela`, `-d in.sela out.wav`, `-p in.sela`;
// banner on stdout, data::Exception caught by value -> message on stderr, exit status 1.
// (-p needs an audio device and is not built here: it reports that and fails.)
// Not in the reference: `-V in.wav out.sela` (encode, then prove the written bytes decode back to the WAV)
// and `-t in.sela in.wav` (test a coded file against a WAV).  Exit status 0 when every frame decodes to its
// source, 2 when some do not (one stderr line per (frame, channel), then a summary), 1 on errors.
// `-L in.wav out.sela`: a lossless encode (a file that decodes back to the WAV under the reference decoder, the same
// bytes as -e where -e's already do), one line with the number of re-coded subframes.
// `-S in.wav out.sela`: a smaller file at a higher encode cost (every subframe at the predictor order with the fewest
// words, and decoding back to the WAV under the reference decoder), one line with the bytes written and the bytes -e
// writes.
// `-P in.wav out.sela`: a smaller file of correlated channels at a higher encode cost (every channel of a frame coded
// alone or as its difference from another, whichever takes the fewest words, for any channel count, and decoding back
// to the WAV under the reference decoder), one line with the bytes written, the bytes -L writes and the number of
// difference subframes.
// `-B in.wav out.sela` ("best"): -S and -P together, every channel and every channel difference at the order with the
// fewest words; the smallest file of these modes at the highest encode cost, decoding back to the WAV under the
// reference decoder.  One line with the bytes written, the bytes -S writes and the number of difference subframes.
// `-W in.wav out.sela`: -S, and every subframe also searched from a Tukey(0.5)-windowed analysis, coded from whichever
// analysis and order takes the fewest words; a file at most -S's size, decoding back to the WAV under the reference
// decoder.  One line with the bytes written, the bytes -S writes and the number of units coded from the window.
// `-F in.wav out.sela` ("fast search"): -S over only the 4 orders a reflection-coefficient estimate ranks best, order 1
// and the reference order; most of -S's saving at a fraction of its cost, decoding back to the WAV under the
// reference decoder.  One line with the bytes written and the bytes -e writes.
// `-R in.sela out.wav first_sample n_samples` (random access): the WAV -d writes, cut to samples
// [first_sample, first_sample + n_samples) of every channel; only the frames that range covers are decoded.  With a
// fifth argument `c0,c1,...` the WAV holds just those channels, in that order, decoded from only the subframes they
// need.
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "sela_api.hpp"

namespace {
// `sela -E out_dir a.wav b.wav ...` / `sela -D out_dir a.sela b.sela ...` (not in the reference):
// many files in ONE process, so that the CUDA context is created once, staging buffers stay
// page-locked, and a few host threads read and write files while another file is on the GPU.
// Output names: <out_dir>/<input base name>.sela|.wav.  A file that fails is reported on stderr
// (reference messages) and the others still run; exit status 1 if any failed.
int run_batch(bool encode, const std::string &out_dir, const std::vector<std::string> &inputs)
{
    sela::setBatchMode(true);
    std::atomic<size_t> next{0}, failed{0};
    std::mutex log;
    unsigned workers = 8;
    if (const char *env = std::getenv("SELA_B200_WORKERS"))
        workers = (unsigned)std::max(1, std::atoi(env));
    workers = (unsigned)std::min<size_t>(workers, inputs.size());
    auto work = [&] {
        for (;;) {
            const size_t i = next.fetch_add(1);
            if (i >= inputs.size())
                return;
            const std::string &in_path = inputs[i];
            std::string base = in_path.substr(in_path.find_last_of('/') + 1);
            const size_t dot = base.find_last_of('.');
            if (dot != std::string::npos && dot > 0)
                base.resize(dot);
            const std::string out_path = out_dir + "/" + base + (encode ? ".sela" : ".wav");
            try {
                std::ifstream in(in_path, std::ios::binary);
                if (!in)
                    throw data::Exception("cannot open input file");
                std::ofstream out(out_path, std::ios::binary);
                if (!out)
                    throw data::Exception("cannot open output file " + out_path);
                if (encode)
                    sela::Encoder(in).processTo(out);
                else
                    sela::Decoder(in).processTo(out);
            } catch (data::Exception e) {
                std::lock_guard<std::mutex> lock(log);
                std::cerr << in_path << ": " << e.exceptionMessage << std::endl;
                failed++;
            }
        }
    };
    std::vector<std::thread> pool;
    for (unsigned t = 0; t < workers; t++)
        pool.emplace_back(work);
    for (std::thread &t : pool)
        t.join();
    std::cout << (encode ? "Encoded " : "Decoded ") << inputs.size() - failed.load() << " of " << inputs.size()
              << " files" << std::endl;
    return failed.load() ? 1 : 0;
}

// The verify modes' output; returns their exit status.
int print_report(const std::vector<sela::VerifyEntry> &report)
{
    if (report.empty()) {
        std::cout << "Verified: every frame decodes to its source" << std::endl;
        return 0;
    }
    for (const sela::VerifyEntry &e : report)
        std::cerr << "frame " << e.frame << " channel " << e.channel << ": differs from sample " << e.firstSample
                  << " on, " << e.differingSamples << " samples differ, first delta " << e.firstDelta << "\n";
    std::cerr << "Verify failed: " << report.size() << " (frame, channel) pairs do not decode to their source"
              << std::endl;
    return 2;
}

int usage(const std::string &prog)
{
    std::cout << "Usage: \n\n"
              << "Encoding a file:\n" << prog << " -e path/to/input.wav path/to/output.sela\n\n"
              << "Decoding a file:\n" << prog << " -d path/to/input.sela path/to/output.wav\n\n"
              << "Playing a file:\n" << prog << " -p path/to/input.sela\n\n"
              << "Encoding a file and verifying that it decodes back to the input (H100 build):\n" << prog
              << " -V path/to/input.wav path/to/output.sela\n\n"
              << "Encoding a file so that it decodes back to the input (H100 build):\n" << prog
              << " -L path/to/input.wav path/to/output.sela\n\n"
              << "Encoding a file smaller, searching every subframe's predictor order (H100 build):\n" << prog
              << " -S path/to/input.wav path/to/output.sela\n\n"
              << "Encoding a file smaller, pairing the channels of every frame (H100 build):\n" << prog
              << " -P path/to/input.wav path/to/output.sela\n\n"
              << "Encoding a file smallest, searching the predictor orders and pairing the channels (H100 build):\n"
              << prog << " -B path/to/input.wav path/to/output.sela\n\n"
              << "Encoding a file smaller, searching the predictor orders over windowed analyses (H100 build):\n"
              << prog << " -W path/to/input.wav path/to/output.sela\n\n"
              << "Encoding a file smaller, searching the predictor orders an estimate ranks best (H100 build):\n"
              << prog << " -F path/to/input.wav path/to/output.sela\n\n"
              << "Decoding samples [first, first + count) of every channel of a file (H100 build):\n" << prog
              << " -R path/to/input.sela path/to/output.wav first count [c0,c1,...]\n\n"
              << "Testing a file against a wav file (H100 build):\n" << prog << " -t path/to/input.sela path/to/input.wav\n\n"
              << "Many files in one process (H100 build):\n" << prog << " -E out_dir a.wav b.wav ...\n"
              << prog << " -D out_dir a.sela b.sela ..." << std::endl;
    return 0;
}
} // namespace

int main(int argc, char **argv)
{
    std::cout << "SimplE Lossless Audio v2 (H100 build). Released under MIT license" << std::endl;
    const std::string prog = argv[0];
    if (argc < 2)
        return usage(prog);
    // One GPU is all this process uses: hide the others from the driver before it starts, so that
    // cuInit does not bring up every device of an 8-GPU box (the bulk of a short run's wall time).
    if (!std::getenv("CUDA_VISIBLE_DEVICES")) {
        const char *dev = std::getenv("SELAB200_DEVICE");
        setenv("CUDA_VISIBLE_DEVICES", dev ? dev : "0", 1);
        setenv("SELAB200_DEVICE", "0", 1);
    }
    // SELA_B200_CLASSIC=1: the reference's two-step call sequence (process(), then writeToFile())
    // instead of the fused file-to-file drivers; same bytes, more host work.
    const bool classic = std::getenv("SELA_B200_CLASSIC") != nullptr;
    int status = 0;
    try {
        const std::string mode = argv[1];
        if ((mode == "-E" || mode == "-D") && argc >= 4) {
            std::cout << (mode == "-E" ? "Encoding " : "Decoding ") << argc - 3 << " files into " << argv[2] << std::endl;
            const int rc = run_batch(mode == "-E", argv[2], std::vector<std::string>(argv + 3, argv + argc));
            std::cout.flush();
            std::cerr.flush();
            std::_Exit(rc);
        } else if (mode == "-e" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Encoding: " << argv[2] << std::endl;
            if (classic) {
                file::SelaFile coded = sela::Encoder(in).process();
                coded.writeToFile(out);
            } else {
                sela::Encoder(in).processTo(out);
            }
        } else if (mode == "-d" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Decoding: " << argv[2] << std::endl;
            if (classic) {
                file::WavFile pcm = sela::Decoder(in).process();
                pcm.writeToFile(out);
            } else {
                sela::Decoder(in).processTo(out);
            }
        } else if (mode == "-R" && (argc == 6 || argc == 7)) {
            uint64_t first = 0, count = 0;
            std::vector<uint8_t> channels;
            try {
                first = std::stoull(argv[4]);
                count = std::stoull(argv[5]);
            } catch (const std::exception &) {
                throw data::Exception("first sample and sample count must be non-negative integers");
            }
            if (argc == 7) {
                const std::string list = argv[6];
                size_t at = 0;
                while (at <= list.size()) {
                    const size_t end = std::min(list.find(',', at), list.size());
                    const std::string item = list.substr(at, end - at);
                    if (item.empty() || item.find_first_not_of("0123456789") != std::string::npos || item.size() > 3 ||
                        std::stoul(item) > 255)
                        throw data::Exception("channels must be a comma-separated list of numbers in [0, 255]");
                    channels.push_back((uint8_t)std::stoul(item));
                    at = end + 1;
                }
            }
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Decoding samples " << first << " to " << first + count << ": " << argv[2] << std::endl;
            sela::Decoder(in).processRangeTo(out, first, count, channels);
        } else if (mode == "-V" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Encoding and verifying: " << argv[2] << std::endl;
            std::vector<sela::VerifyEntry> report;
            sela::Encoder(in).processTo(out, report);
            status = print_report(report);
        } else if (mode == "-L" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Encoding losslessly: " << argv[2] << std::endl;
            std::vector<sela::RecodedEntry> recoded;
            sela::Encoder(in).processLosslessTo(out, recoded);
            std::cout << "Re-coded " << recoded.size() << " subframes" << std::endl;
        } else if (mode == "-S" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Encoding with the order search: " << argv[2] << std::endl;
            size_t refBytes = 0;
            const size_t written = sela::Encoder(in).processSearchTo(out, refBytes);
            std::cout << "Wrote " << written << " bytes (-e: " << refBytes << " bytes)" << std::endl;
        } else if (mode == "-P" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Encoding with the channel pairing: " << argv[2] << std::endl;
            size_t losslessBytes = 0, differences = 0;
            const size_t written = sela::Encoder(in).processPairingTo(out, losslessBytes, differences);
            std::cout << "Wrote " << written << " bytes (-L: " << losslessBytes << " bytes), " << differences
                      << " difference subframes" << std::endl;
        } else if (mode == "-B" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Encoding with the order search and the channel pairing: " << argv[2] << std::endl;
            size_t searchBytes = 0, differences = 0;
            const size_t written = sela::Encoder(in).processSearchPairingTo(out, searchBytes, differences);
            std::cout << "Wrote " << written << " bytes (-S: " << searchBytes << " bytes), " << differences
                      << " difference subframes" << std::endl;
        } else if (mode == "-W" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Encoding with the order search over Tukey(0.5)-windowed analyses: " << argv[2] << std::endl;
            size_t searchBytes = 0, windowUnits = 0;
            const size_t written = sela::Encoder(in).processSearchWindowsTo(out, 1u, searchBytes, windowUnits);
            std::cout << "Wrote " << written << " bytes (-S: " << searchBytes << " bytes), " << windowUnits
                      << " units coded from the window" << std::endl;
        } else if (mode == "-F" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ofstream out(argv[3], std::ios::binary);
            std::cout << "Encoding with the order search over the 4 best-ranked orders: " << argv[2] << std::endl;
            size_t refBytes = 0;
            const size_t written = sela::Encoder(in).processSearchGuidedTo(out, 4u, refBytes);
            std::cout << "Wrote " << written << " bytes (-e: " << refBytes << " bytes)" << std::endl;
        } else if (mode == "-t" && argc == 4) {
            std::ifstream in(argv[2], std::ios::binary);
            std::ifstream wav(argv[3], std::ios::binary);
            std::cout << "Testing: " << argv[2] << " against " << argv[3] << std::endl;
            status = print_report(sela::Decoder(in).verifyAgainst(wav));
        } else if (mode == "-p" && argc == 3) {
            std::ifstream in(argv[2], std::ios::binary);
            std::cout << "Playing: " << argv[2] << std::endl;
            file::WavFile pcm = sela::Decoder(in).process();
            sela::Player().play(pcm);
        } else {
            return usage(prog);
        }
    } catch (data::Exception e) {
        std::cerr << e.exceptionMessage << std::endl;
        return 1;
    }
    // Output files are closed (their streams went out of scope above).  Leave without tearing the
    // CUDA context down piece by piece: the driver reclaims everything with the process, and the
    // orderly teardown of a context holding ~1 GB costs a few hundred ms.
    std::cout.flush();
    std::cerr.flush();
    std::_Exit(status);
}
