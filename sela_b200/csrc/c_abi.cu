// c_abi.cu -- the extern "C" boundary declared in include/sela_b200.h.
//
// Host-side plumbing only: device selection, a grow-only device workspace, the
// launches.  No algorithm lives here and there is no CPU fallback: without a
// CUDA device every compute entry point returns SELAB200_ERR_NO_DEVICE.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "clips.cuh"
#include "lossless.cuh"
#include "pairing.cuh"
#include "search.cuh"
#include "search_guided.cuh"
#include "search_pairing.cuh"
#include "verify.cuh"
#include "window.cuh"

using namespace selab200;

namespace {

thread_local char g_error[512] = "";
std::mutex g_mutex;
std::atomic<uint64_t> g_launches{0};

int fail(int code, const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof g_error, fmt, ap);
    va_end(ap);
    return code;
}

#define CUDA_TRY(expr)                                                                      \
    do {                                                                                    \
        cudaError_t e_ = (expr);                                                            \
        if (e_ != cudaSuccess)                                                              \
            return fail(SELAB200_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e_)); \
    } while (0)

struct DeviceBuffer {
    void *ptr = nullptr;
    size_t bytes = 0;
    int ensure(size_t need)
    {
        if (need <= bytes)
            return 0;
        if (ptr)
            cudaFree(ptr);
        ptr = nullptr;
        bytes = 0;
        size_t want = need + need / 8 + 4096;
        cudaError_t e = cudaMalloc(&ptr, want);
        if (e != cudaSuccess)
            return fail(SELAB200_ERR_CUDA, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
        bytes = want;
        return 0;
    }
    void release()
    {
        if (ptr)
            cudaFree(ptr);
        ptr = nullptr;
        bytes = 0;
    }
};

// The counters of the host-buffer, test and stage calls: at the front of g.small on the device, and in the pinned
// g.h_small they come down to.  The encode counters (status .. n_window) are reset and read back as one block.
struct Counters {
    int32_t status;                  // the device status of the call
    uint64_t used;                   // encode: the word arena's fill level
    unsigned long long ref_words;    // search: the words the reference encoder's choice takes
    unsigned long long base_words;   // pairing: the words of its base, the lossless encode (search_pairing: the search)
    unsigned long long n_difference; // pairing, search_pairing: the difference subframes chosen
    unsigned long long n_window;     // search_windows: the units coded from a window
    uint32_t selftest;               // selab200_selftest: the mismatches
    // host side only (collect_records): a count of set records, and the decode status that follows a verify count
    unsigned long long n_records;
    int32_t records_status;
};
constexpr size_t kEncodeCounterBytes = offsetof(Counters, selftest);
static_assert(offsetof(Counters, records_status) == offsetof(Counters, n_records) + 8, "VerifyArea order");
static_assert(sizeof(Counters) <= 256, "g.small holds the counters");

constexpr int kMaxChunks = 72;
constexpr int kLanes = 8; // concurrent compute streams of the pipelined host calls

struct Context {
    bool ready = false;
    int device = -1;
    int sms = 0;                                   // streaming multiprocessors of `device`
    cudaStream_t stream = nullptr;                 // stage-level calls
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr; // pipelined batch calls: copy engines ...
    cudaStream_t s_compute[kLanes] = {};           // ... and compute lanes
    cudaEvent_t ev_h2d[kMaxChunks], ev_done[kMaxChunks], ev_scan[kMaxChunks], ev_reset;
    cudaEvent_t ev_rice;                           // after the last kernel of the last Rice-only device call (aux)
    bool events = false;
    DeviceBuffer in, descs, words, work, lane_work[kLanes], aux;
    DeviceBuffer small;                            // Counters
    DeviceBuffer verify;                           // verify paths: count, status, per-pair records (VerifyArea)
    DeviceBuffer lossless;                         // lossless host paths: count, per-pair records of re-coded subframes
    DeviceBuffer clip_src, clip_pieces, clip_out;  // clip decode: source addresses, gather pieces, host-form staging
    DeviceBuffer clip_rows;                        // channel-selecting clip decode: the gather's row table
    DeviceBuffer clip_runs, clip_stage;            // host-resident images: a group's fetch runs and their staging
    Counters *h_small = nullptr;                   // pinned: where g.small's counters come down
    unsigned long long *h_totals = nullptr;        // pinned: arena fill level after each chunk
    size_t last_rice_n_sub = 0;                    // selab200_rice_decode_frames_device bookkeeping (flag count query)
    cudaStream_t last_rice_stream = nullptr;
    std::vector<struct ContainerBuffers> *spare = nullptr; // recycled container buffers of this device
    const double *windows = nullptr;               // d_analysis_windows on `device`, filled by init_slot
    std::atomic<uint64_t> launches{0};             // kernel launches of this slot since init_slot (selab200_slot_launch_count)
};

// One context per device the library was initialised for (selab200_init / selab200_init_devices), slot 0 the
// primary.  Everything below reaches "the" context through `g`, a thread-local pointer: an API call runs on
// the primary (or, for the *_device forms, on the device that owns the caller's pointers); the multi-device
// host-buffer calls give every device a worker thread of its own that points `g` at that device's context.
// Contexts share nothing, so the workers never contend.
constexpr int kMaxDevices = 16;
Context g_slots[kMaxDevices];
int g_n_ctx = 0;
Context *g_last_rice_ctx = nullptr; // the context selab200_rice_decode_frames_device last ran on (flag count query)
thread_local Context *tl_ctx = &g_slots[0];
#define g (*tl_ctx)

Counters *device_counters() { return static_cast<Counters *>(g.small.ptr); }

// What a container handle owns besides the walk result: the device image of the bytes, a pinned
// descriptor table and the upload events.  Recycled through a small free list, because a process
// that decodes many files would otherwise pay cudaMalloc/cudaFree (a device-wide sync) and
// cudaMallocHost/cudaFreeHost for every one of them.
struct ContainerBuffers {
    static constexpr int kPieces = 8;
    void *d_bytes = nullptr;
    size_t d_cap = 0;
    selab200_subframe_desc *h_descs = nullptr;
    size_t h_cap = 0; // descriptors
    cudaEvent_t ev_piece[kPieces] = {};
    void destroy()
    {
        for (cudaEvent_t &e : ev_piece)
            if (e) {
                cudaEventDestroy(e);
                e = nullptr;
            }
        if (d_bytes)
            cudaFree(d_bytes);
        if (h_descs)
            cudaFreeHost(h_descs);
        d_bytes = nullptr;
        h_descs = nullptr;
        d_cap = h_cap = 0;
    }
};

std::vector<ContainerBuffers> g_spare_store[kMaxDevices]; // guarded by g_mutex; Context::spare points here
#define g_spare_buffers (*g.spare)
constexpr size_t kMaxSpareBuffers = 16;

// On every exit from a pipelined call -- error paths included -- nothing may still be
// reading or writing the caller's host buffers.
struct PipelineDrain {
    ~PipelineDrain()
    {
        if (g.s_h2d)
            cudaStreamSynchronize(g.s_h2d);
        for (int i = 0; i < kLanes; i++)
            if (g.s_compute[i])
                cudaStreamSynchronize(g.s_compute[i]);
        if (g.s_d2h)
            cudaStreamSynchronize(g.s_d2h);
    }
};

// g.aux, the library's scratch, holding at least `bytes`, for work that `stream` is about to enqueue.  The Rice-only
// device call leaves its split table and flags there and returns before its kernels have run, on a stream of the
// caller's; whatever uses aux next waits for those kernels first (ev_rice), without a host synchronisation.  Growing
// aux frees the old buffer, which synchronises the device.
int aux_for(size_t bytes, cudaStream_t stream)
{
    if (int rc = g.aux.ensure(bytes))
        return rc;
    CUDA_TRY(cudaStreamWaitEvent(stream, g.ev_rice, 0));
    return 0;
}

// Chunking of the pipelined host-buffer calls (encode_host, decode_pipeline): about
// eight chunks, enough to overlap PCIe with compute, each still several waves of warps, workspace bounded
// for huge batches.  SELAB200_CHUNK_FRAMES forces the chunk size (tools/e2e_chunk_sweep.py sweeps it on the
// BASELINE batch; tests use it to get many chunks).
uint32_t chunk_frames_for(uint32_t n_frames)
{
    if (const char *env = std::getenv("SELAB200_CHUNK_FRAMES")) { // tuning / tests only
        long v = std::atol(env);
        if (v > 0) {
            uint32_t c = (uint32_t)v;
            while ((n_frames + c - 1) / c > (uint32_t)kMaxChunks)
                c *= 2;
            return c;
        }
    }
    constexpr uint32_t kParts = 8;
    uint32_t c = (n_frames + kParts - 1) / kParts;
    if (c < 512) c = 512;
    if (c > 16384) c = 16384;
    while ((n_frames + c - 1) / c > (uint32_t)kMaxChunks)
        c *= 2;
    return c;
}

// Chunk boundaries of a pipelined host-buffer call.  Equal chunks, except that the first and the last
// are cut into shrinking pieces: what a pipeline cannot hide is the upload of the first chunk before any
// kernel runs and the download of the last chunk after the last kernel, so those two are made small.  The
// decoder gains from it as well: small batches cut every Rice stream into parts (rice_vs.cuh), so a small
// chunk does not starve its Rice kernel.  With SELAB200_CHUNK_FRAMES every chunk has the size it asks for.
struct ChunkPlan {
    std::vector<uint32_t> start; // n_chunks + 1 boundaries
    uint32_t max_frames = 0;     // largest chunk (sizes the per-lane workspace)
    uint32_t chunks() const { return (uint32_t)start.size() - 1; }
};

ChunkPlan plan_chunks(uint32_t n_frames)
{
    ChunkPlan p;
    const uint32_t cf = chunk_frames_for(n_frames);
    const uint32_t n_base = (n_frames + cf - 1) / cf;
    const bool taper = !std::getenv("SELAB200_CHUNK_FRAMES") && n_base >= 4 && n_base + 6 <= (uint32_t)kMaxChunks;
    p.start.push_back(0);
    for (uint32_t c = 0; c < n_base; c++) {
        const uint32_t f0 = c * cf, f1 = (f0 + cf <= n_frames) ? f0 + cf : n_frames, len = f1 - f0;
        if (taper && c == 0 && len >= 512) {
            p.start.push_back(f0 + len / 8);
            p.start.push_back(f0 + len / 2);
        } else if (taper && c == n_base - 1 && len >= 512) {
            p.start.push_back(f0 + len / 2);
            p.start.push_back(f0 + len / 2 + len / 4);
            p.start.push_back(f0 + len / 2 + len / 4 + len / 8);
        }
        p.start.push_back(f1);
    }
    for (uint32_t c = 0; c + 1 < p.start.size(); c++)
        p.max_frames = std::max(p.max_frames, p.start[c + 1] - p.start[c]);
    return p;
}

const char *status_text(int s)
{
    switch (s) {
    case SELAB200_ERR_CAPACITY: return "output word arena too small";
    case SELAB200_ERR_RANGE: return "value outside the representable domain (16-bit audio / uint16 word counts)";
    case SELAB200_ERR_BITSTREAM: return "malformed subframe descriptor or Rice stream";
    default: return "device reported an error";
    }
}

// Points `g` at the primary context for the calling thread (g_mutex held) and selects its device.
int require_ready()
{
    tl_ctx = &g_slots[0];
    if (g_n_ctx == 0 || !g.ready)
        return fail(SELAB200_ERR_NOT_INIT, "selab200_init() has not been called (or found no CUDA device)");
    // the current device is per host thread; callers may arrive on a thread other than init()'s
    cudaError_t e = cudaSetDevice(g.device);
    if (e != cudaSuccess)
        return fail(SELAB200_ERR_CUDA, "cudaSetDevice(%d) failed: %s", g.device, cudaGetErrorString(e));
    return 0;
}

// The *_device forms run on the device that owns the caller's buffers: points `g` at that device's context.
int require_ready_for(const void *device_ptr)
{
    if (g_n_ctx == 0)
        return require_ready();
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, device_ptr) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        return fail(SELAB200_ERR_ARGUMENT, "not a device pointer");
    }
    for (int i = 0; i < g_n_ctx; i++)
        if (g_slots[i].ready && g_slots[i].device == attr.device) {
            tl_ctx = &g_slots[i];
            cudaError_t e = cudaSetDevice(g.device);
            if (e != cudaSuccess)
                return fail(SELAB200_ERR_CUDA, "cudaSetDevice(%d) failed: %s", g.device, cudaGetErrorString(e));
            return 0;
        }
    return fail(SELAB200_ERR_ARGUMENT, "the buffers live on device %d, which the library was not initialised for "
                                       "(selab200_init / selab200_init_devices)", attr.device);
}

int check_channels(uint32_t channels)
{
    if (channels == 0 || channels > SELAB200_MAX_CHANNELS)
        return fail(SELAB200_ERR_ARGUMENT, "channels must be in [1, %d]", SELAB200_MAX_CHANNELS);
    return 0;
}

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// Raises a kernel's dynamic shared-memory limit; remembered per (kernel, device): the attribute call is a
// host round trip that would otherwise precede every launch.
template <typename K>
int set_smem(K kernel, size_t bytes)
{
    static std::mutex m;
    static std::vector<std::pair<std::pair<const void *, int>, size_t>> done;
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    const std::pair<const void *, int> key(reinterpret_cast<const void *>(kernel), dev);
    std::lock_guard<std::mutex> lock(m);
    for (auto &e : done)
        if (e.first == key) {
            if (e.second >= bytes)
                return 0;
            CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
            e.second = bytes;
            return 0;
        }
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    done.emplace_back(key, bytes);
    return 0;
}

int launch_check(const char *what)
{
    g_launches.fetch_add(1, std::memory_order_relaxed);
    g.launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        return fail(SELAB200_ERR_CUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
    return 0;
}

// kernel<<<grid, block, smem, stream>>>(args...) with the kernel's dynamic shared-memory limit raised to smem first,
// and the launch checked (`name` in the error).
template <typename... Params, typename... Args>
int launch(void (*kernel)(Params...), size_t grid, unsigned block, size_t smem, cudaStream_t stream, const char *name,
           const Args &...args)
{
    if (smem)
        if (int rc = set_smem(kernel, smem))
            return rc;
    kernel<<<(unsigned)grid, block, smem, stream>>>(args...);
    return launch_check(name);
}

// The mean of every analysis unit (k_unit_means<KIND>, a warp per 32 units) into means[n_units].
template <int KIND>
int launch_unit_means(const void *src, size_t n_units, uint32_t channels, double *means, cudaStream_t stream)
{
    return launch(k_unit_means<KIND>, (n_units + 31) / 32, 32, unit_means_smem_bytes(mean_tiling(KIND, channels)),
                  stream, "k_unit_means", src, (uint32_t)n_units, channels, means);
}

// The lossless encode (lossless.cuh) in place of k_encode_units: the analysis with the tie check,
// k_encode_units<S, false, true>, then the repair.  Every repair launch has a grid of a fixed size: nothing here
// depends on what the check found.  The warp kernels use at most one residue row per unit of the batch.  FORCE: the
// units' predictors are d_pred's (selab200_encode_lossless_forced).  pairing: the base of a pairing encode, which
// keeps the tie flags that the select kernel clears and takes no report.
template <bool STEREO, bool FORCE>
int launch_lossless(const EncodeParams &p, const RepairParams &r, size_t n_frames, size_t n_units, cudaStream_t stream,
                    const selab200_predictor *d_pred, const PairingParams *pairing)
{
    constexpr size_t smem = encode_smem_bytes<STEREO>();
    const size_t frame_ctas = (n_frames + 255) / 256, warps = std::min(n_units, (size_t)g.sms * 32);
    if (int rc = launch(k_encode_units<STEREO, false, true, FORCE>, n_units, 32, smem, stream, "k_encode_units", p,
                        nullptr, d_pred))
        return rc;
    if (pairing)
        if (int rc = launch(k_pairing_capture, frame_ctas, 256, 0, stream, "k_pairing_capture", p, *pairing))
            return rc;
    if (int rc = launch(k_lossless_select, frame_ctas, 256, 0, stream, "k_lossless_select", p, r))
        return rc;
    for (int round = 0; round < 2; round++)
        if (int rc = launch(k_lossless_candidates<STEREO, FORCE>, warps, 32, smem, stream, "k_lossless_candidates", p, r,
                            round, d_pred))
            return rc;
    if (int rc = launch(k_lossless_repack<STEREO, FORCE>, warps, 32, smem, stream, "k_lossless_repack", p, r, d_pred))
        return rc;
    if (pairing)
        return 0;
    return launch(k_lossless_report, std::min(frame_ctas, (size_t)g.sms), 256, 0, stream, "k_lossless_report", p, r);
}

// The order search (search.cuh) in place of k_encode_units: analysis, candidates, repack, and the reference encoder's
// words added to *d_ref_words.  The warp kernels have grids of a fixed size, at most one residue row per unit of the
// batch.  d_ref_words null (the base of a search + pairing): k_search_ref_words is not run.  FORCE: the units' q and
// reference orders are d_pred's (selab200_encode_search_forced).  TRACE: the analysis and candidate kernels are their
// tracing instantiations, which write every (unit, order) record to d_trace (selab200_encode_search_trace).  gp
// (guided order search, search_guided.cuh): the estimate, and every unit's listed orders sized by k_search_listed in
// place of k_search_candidates; with TRACE, every unit's estimates to gp->estimates as well.
template <bool STEREO, bool FORCE, bool TRACE>
int launch_search(const EncodeParams &p, SearchUnit *su, size_t n_frames, size_t n_units,
                  unsigned long long *d_ref_words, cudaStream_t stream, const selab200_predictor *d_pred,
                  selab200_search_trace *d_trace, const GuidedParams *gp)
{
    constexpr size_t smem = encode_smem_bytes<STEREO>(), smem_orders = search_smem_bytes<STEREO>();
    const size_t warps = std::min(n_units, (size_t)g.sms * 32);
    if (int rc = launch(k_search_units<STEREO, TRACE, FORCE>, n_units, 32, smem, stream, "k_search_units", p, d_pred,
                        su, d_trace))
        return rc;
    if (gp) {
        if (int rc = launch(k_search_estimate<TRACE>, warps, 32, 0, stream, "k_search_estimate", p, su, *gp))
            return rc;
        if (int rc = launch(k_search_listed<STEREO, TRACE>, warps, 32, smem_orders, stream, "k_search_listed", p, su, *gp,
                            d_trace))
            return rc;
    } else if (int rc = launch(k_search_candidates<STEREO, TRACE>, warps, 32, smem_orders, stream, "k_search_candidates",
                               p, su, d_trace)) {
        return rc;
    }
    if (d_ref_words)
        if (int rc = launch(k_search_ref_words, (n_frames + 255) / 256, 256, 0, stream, "k_search_ref_words", p, su,
                            d_ref_words))
            return rc;
    return launch(k_search_repack<STEREO>, warps, 32, smem_orders, stream, "k_search_repack", p, su);
}

// The channel pairing (pairing.cuh) between the lossless repair and the scan: means, candidates, choice, and the
// winning differences packed in place of their channels.  The warp kernels have grids of a fixed size, at most one
// residue row per unit of the batch.
int launch_pairing(const EncodeParams &p, const PairingParams &q, size_t n_frames, size_t n_units, cudaStream_t stream)
{
    constexpr size_t smem = encode_smem_bytes<true>();
    const size_t n_pairs = n_frames * p.channels * p.channels, warps = std::min(n_units, (size_t)g.sms * 32);
    if (int rc = launch(k_pairing_means, (n_pairs + 127) / 128, 128, 0, stream, "k_pairing_means", p, q))
        return rc;
    if (int rc = launch(k_pairing_candidates, warps, 32, smem, stream, "k_pairing_candidates", p, q))
        return rc;
    if (int rc = launch(k_pairing_select, std::min(n_frames, (size_t)g.sms * 16), 128, 0, stream, "k_pairing_select", p,
                        q))
        return rc;
    return launch(k_pairing_repack, warps, 32, smem, stream, "k_pairing_repack", p, q);
}

// The search + pairing (search_pairing.cuh) between the order search and the scan: means, the candidates' analysis
// and search, the table, the choice, and the winning differences packed at their searched orders in place of their
// channels.  The warp kernels have grids of a fixed size, at most one residue row per unit of the batch.  TRACE: the
// candidates' analysis and search kernels are their tracing instantiations, which write to q.trace.
template <bool TRACE>
int launch_search_pairing(const EncodeParams &p, const PairingParams &q, SearchUnit *cand, size_t n_frames,
                          size_t n_units, cudaStream_t stream)
{
    constexpr size_t smem = encode_smem_bytes<true>(), smem_orders = search_smem_bytes<true>();
    const size_t n_pairs = n_frames * p.channels * p.channels, warps = std::min(n_units, (size_t)g.sms * 32);
    CUDA_TRY(cudaMemsetAsync(q.stale, 0, n_frames * sizeof(uint32_t), stream)); // every searched unit is tie-free
    if (int rc = launch(k_pairing_means, (n_pairs + 127) / 128, 128, 0, stream, "k_pairing_means", p, q))
        return rc;
    if (int rc = launch(k_search_pairing_units<TRACE>, warps, 32, smem, stream, "k_search_pairing_units", p, q, cand))
        return rc;
    if (int rc = launch(k_search_pairing_candidates<TRACE>, warps, 32, smem_orders, stream,
                        "k_search_pairing_candidates", p, cand, q.trace))
        return rc;
    if (int rc = launch(k_search_pairing_table, (n_pairs + 255) / 256, 256, 0, stream, "k_search_pairing_table", p, q,
                        cand))
        return rc;
    if (int rc = launch(k_pairing_select, std::min(n_frames, (size_t)g.sms * 16), 128, 0, stream, "k_pairing_select", p,
                        q))
        return rc;
    return launch(k_search_pairing_repack, warps, 32, smem_orders, stream, "k_search_pairing_repack", p, q, cand);
}

// The window table of the window search (DESIGN.md 7.6), computed once on the host: row i is the window of mask bit
// i.  Tukey(p) over n samples: L = floor(p (n - 1) / 2) samples 0.5 (1 - cos(pi i / L)) at each end, 1 between.
const double *analysis_window_table()
{
    static const std::vector<double> table = [] {
        std::vector<double> t((size_t)kAnalysisWindows * kFrame, 1.0);
        const auto tukey = [](double *w, int n, double frac) {
            const int L = (int)std::floor(frac * (n - 1) / 2);
            for (int i = 0; i < L; i++) {
                const double v = 0.5 * (1.0 - std::cos(M_PI * i / L));
                w[i] = v;
                w[n - 1 - i] = v;
            }
        };
        double *row = t.data();
        tukey(row, kFrame, 0.5);                                    // 0: Tukey(0.5)
        tukey(row + kFrame, kFrame, 0.25);                          // 1: Tukey(0.25)
        for (int i = 0; i < kFrame; i++)                            // 2: Hann
            row[2 * kFrame + i] = 0.5 - 0.5 * std::cos(2 * M_PI * i / (kFrame - 1));
        std::fill(row + 3 * kFrame + kFrame / 2, row + 4 * kFrame, 0.0); // 3: Tukey(0.5) over the first half
        tukey(row + 3 * kFrame, kFrame / 2, 0.5);
        std::fill(row + 4 * kFrame, row + 4 * kFrame + kFrame / 2, 0.0); // 4: Tukey(0.5) over the second half
        tukey(row + 4 * kFrame + kFrame / 2, kFrame / 2, 0.5);
        return t;
    }();
    return table.data();
}

// A window mask names at least one window and none past the table.
int check_windows(uint32_t windows)
{
    if (windows == 0 || (windows >> kAnalysisWindows) != 0)
        return fail(SELAB200_ERR_ARGUMENT, "window mask 0x%x must select windows among bits 0..%d", windows,
                    kAnalysisWindows - 1);
    return 0;
}

// The window search (window.cuh) after the order search and before the scan: the order search's words added to
// *d_base_words, the window analyses, their candidates, and the units whose best window candidate has strictly fewer
// words repacked.  su: the order search's SearchUnits.  The warp kernels have grids of a fixed size, the candidate
// and repack kernels at most one residue row per unit of the batch.  TRACE: the candidate kernel is its tracing
// instantiation (wp.trace).
template <bool STEREO, bool TRACE>
int launch_windows(const EncodeParams &p, const WindowParams &wp, const SearchUnit *su, size_t n_frames,
                   size_t n_units, unsigned long long *d_base_words, cudaStream_t stream)
{
    constexpr size_t smem = encode_smem_bytes<STEREO>(), smem_orders = search_smem_bytes<STEREO>();
    const size_t cap = (size_t)g.sms * 32, warps = std::min(n_units, cap);
    if (int rc = launch(k_window_base_words, (n_frames + 255) / 256, 256, 0, stream, "k_window_base_words", p,
                        d_base_words))
        return rc;
    CUDA_TRY(cudaMemsetAsync(wp.key, 0xff, n_units * sizeof(unsigned long long), stream));
    if (int rc = launch(k_window_units<STEREO>, std::min(n_units * wp.n, cap), 32, smem, stream, "k_window_units", p, wp))
        return rc;
    if (int rc = launch(k_window_candidates<STEREO, TRACE>, warps, 32, smem_orders, stream, "k_window_candidates", p, wp))
        return rc;
    return launch(k_window_repack<STEREO>, warps, 32, smem_orders, stream, "k_window_repack", p, wp, su);
}

// Which encoder an encode call runs.  lossless: re-code every subframe the reference decoder would not reproduce
// (DESIGN.md 7.2).  search: code every subframe at the predictor order with the fewest words (7.3).  pairing: code
// channels as differences wherever that takes fewer words, on top of the lossless encode (7.4).  search_pairing: the
// pairing on top of the search, every channel and every difference at its cheapest order (7.5).  search_windows: the
// search, and every unit also searched from the analysis of each selected window (7.6).  search_guided: the search
// over the orders an estimate ranks best, order 1 and the reference order (7.7).
enum class EncodeMode { plain, lossless, search, pairing, search_pairing, search_windows, search_guided };

// The guided order search's candidate count names 1..100 orders.
int check_candidates(uint32_t candidates)
{
    if (candidates == 0 || candidates > (uint32_t)kMaxOrder)
        return fail(SELAB200_ERR_ARGUMENT, "%u candidates: must be 1..%d", candidates, kMaxOrder);
    return 0;
}

// Where every region of an encode workspace lies, as byte offsets from its base, and its size.  Every mode has the
// plain encode's regions; lossless and pairing add the repair lists, search the SearchUnits, and pairing the pairing
// tables behind the repair lists.  search_pairing has the SearchUnits (every region padded), the pairing tables and
// the candidates' SearchUnits.  search_windows has the SearchUnits, one per (unit, window) and the units' window keys.
// search_guided has the SearchUnits (padded) and a 16-byte order mask per unit.  The offsets of the regions a mode
// lacks are 0.
struct EncodeLayout {
    size_t units, slots, means, residues;                       // EncodeParams
    size_t repair_count, repair_frames, repair_orig, repair_units; // RepairParams
    size_t search;                                              // SearchUnit[n_units]
    size_t pair_search;                                         // search_pairing: SearchUnit[n_frames][C][C]
    size_t pair_table, pair_means, par, stale;                  // PairingParams
    size_t window_search, window_keys;                          // search_windows: WindowParams::su and ::key
    size_t masks;                                               // search_guided: GuidedParams::masks
    size_t bytes;                                               // selab200_encode_*_workspace_bytes
};

EncodeLayout encode_layout(EncodeMode mode, uint32_t n_frames, uint32_t channels, uint32_t n_windows = 0)
{
    const size_t n_units = encode_units(n_frames, channels), n_sub = (size_t)n_frames * channels;
    const size_t n_pairs = n_sub * channels;
    EncodeLayout l{};
    size_t at = 0;
    auto region = [&at](size_t bytes) {
        const size_t o = at;
        at += align256(bytes);
        return o;
    };
    l.units = region(n_units * sizeof(UnitRecord));
    l.slots = region(n_units * (size_t)kSlotWords * 4);
    l.means = region(n_units * sizeof(double));
    l.residues = region(n_units * (size_t)kFrame * 4 + 256);
    if (mode == EncodeMode::search) { // the last region, not padded
        l.search = at;
        l.bytes = at + n_units * sizeof(SearchUnit);
        return l;
    }
    if (mode == EncodeMode::search_windows) {
        l.search = region(n_units * sizeof(SearchUnit));
        l.window_search = region(n_units * n_windows * sizeof(SearchUnit));
        l.window_keys = region(n_units * sizeof(unsigned long long));
    }
    if (mode == EncodeMode::search_guided) {
        l.search = region(n_units * sizeof(SearchUnit));
        l.masks = region(n_units * sizeof(uint4));
    }
    if (mode == EncodeMode::lossless || mode == EncodeMode::pairing) {
        l.repair_count = region(256);
        l.repair_frames = region((size_t)n_frames * 4);
        l.repair_orig = region(n_units * sizeof(UnitRecord));
        l.repair_units = region(n_units * sizeof(RepairUnit));
    }
    if (mode == EncodeMode::search_pairing)
        l.search = region(n_units * sizeof(SearchUnit));
    if (mode == EncodeMode::pairing || mode == EncodeMode::search_pairing) {
        l.pair_table = region(n_pairs * sizeof(PairRecord));
        l.pair_means = region(n_pairs * sizeof(double));
        l.par = region(n_sub);
        l.stale = region((size_t)n_frames * 4);
    }
    if (mode == EncodeMode::search_pairing)
        l.pair_search = region(n_pairs * sizeof(SearchUnit));
    l.bytes = at;
    return l;
}

// Where a lossless encode reports its re-coded subframes: the batch's per-pair records, their count, and the frame
// number of the batch's first frame.
struct LosslessArgs {
    selab200_lossless_entry *entries;
    unsigned long long *n_entries;
    uint32_t frame_base;
};

// ---- device-resident cores (no synchronisation) --------------------------

// Which encoder encode_device runs, how it chains into a pipelined call, and what it produces besides the word arena.
// The defaults are a stand-alone plain batch.  The fields from `lossless` on are read only by the modes they name.
struct EncodeOptions {
    EncodeMode mode = EncodeMode::plain;
    bool fresh = true;                          // reset status, the arena fill level and the mode's counters and
                                                // records first; the pipelined host path resets once and then
                                                // chains chunks through *d_used
    cudaEvent_t before_scan = nullptr;          // the scan waits for it (the previous chunk's scan on another lane)
    cudaEvent_t after_scan = nullptr;           // recorded once this batch's fill level has been taken
    unsigned long long *h_fill_after = nullptr; // pinned: receives the fill level this batch leaves behind
    uint8_t *d_container = nullptr;             // gather into this byte-packed .sela image instead of the arena ...
    unsigned long long sub_base = 0;            // ... where the batch's first subframe is subframe sub_base
    LosslessArgs lossless{};                    // lossless: where the re-coded pairs are reported
    unsigned long long *d_ref_words = nullptr;  // search: += the reference encoder's words
    unsigned long long *d_base_words = nullptr; // pairing, search_pairing: += the words of its base, the lossless
                                                // encode or the search ...
    unsigned long long *d_n_difference = nullptr; // ... and the difference subframes chosen
    uint32_t windows = 0;                         // search_windows: the window mask ...
    unsigned long long *d_n_window = nullptr;     // ... += the units coded from a window
    uint32_t candidates = 0;                      // search_guided: K, the orders listed by rank
    // tests only
    selab200_analysis_trace *d_trace = nullptr;      // plain: the tracing unit kernel writes every unit's analysis here
    const selab200_predictor *d_pred = nullptr;      // lossless, search, pairing, search_pairing: every unit's
                                                     // predictor (pairing, search_pairing: its base's units)
    const selab200_predictor *d_pair_pred = nullptr; // pairing, search_pairing: the candidates' predictors
                                                     // (PairingParams::pred)
    selab200_search_trace *d_search_trace = nullptr; // search, pairing, search_pairing, search_windows: the tracing
                                                     // kernels write every (unit, order) / candidate / (candidate,
                                                     // order) / (unit, window, order) record here
    const selab200_predictor *d_window_pred = nullptr; // search_windows: the (unit, window) records' q
    const double *d_windows = nullptr;               // search_windows: the table the mask indexes (null: the fixed one)
    double *d_estimates = nullptr;                   // search_guided, with d_search_trace: every unit's E[100]
};

// The launches of encode mode o.mode up to the scan: the units' means, then the mode's kernels in place of
// k_encode_units.  STEREO: two channels, three units per frame.  FORCE: o.d_pred is set.  TRACE: o.d_trace or
// o.d_search_trace is set.  q: the pairing's tables (pairing, search_pairing).
template <bool STEREO, bool FORCE, bool TRACE>
int launch_encoder(const EncodeOptions &o, const EncodeLayout &l, char *ws, const EncodeParams &p,
                   const PairingParams &q, uint32_t n_windows, cudaStream_t stream)
{
    const size_t n_frames = p.n_frames, n_units = encode_units(p.n_frames, p.channels);
    if (int rc = launch_unit_means<STEREO ? kMeanStereo : kMeanPcm>(p.pcm, n_units, p.channels, p.means, stream))
        return rc;
    SearchUnit *su = reinterpret_cast<SearchUnit *>(ws + l.search);
    switch (o.mode) {
    case EncodeMode::plain:
        return launch(k_encode_units<STEREO, TRACE>, n_units, 32, encode_smem_bytes<STEREO>(), stream, "k_encode_units",
                      p, o.d_trace, nullptr);
    case EncodeMode::lossless:
    case EncodeMode::pairing: {
        const bool pairing = o.mode == EncodeMode::pairing;
        const LosslessArgs la = pairing ? LosslessArgs{} : o.lossless; // the pairing's base takes no report
        RepairParams r;
        r.count = reinterpret_cast<uint32_t *>(ws + l.repair_count);
        r.frames = reinterpret_cast<uint32_t *>(ws + l.repair_frames);
        r.orig = reinterpret_cast<UnitRecord *>(ws + l.repair_orig);
        r.units = reinterpret_cast<RepairUnit *>(ws + l.repair_units);
        r.entries = la.entries;
        r.n_entries = la.n_entries;
        r.frame_base = la.frame_base;
        CUDA_TRY(cudaMemsetAsync(r.count, 0, 2 * sizeof(uint32_t), stream));
        if (int rc = launch_lossless<STEREO, FORCE>(p, r, n_frames, n_units, stream, o.d_pred, pairing ? &q : nullptr))
            return rc;
        return pairing ? launch_pairing(p, q, n_frames, n_units, stream) : 0;
    }
    case EncodeMode::search:
    case EncodeMode::search_guided: {
        GuidedParams gp{o.candidates, reinterpret_cast<uint4 *>(ws + l.masks), o.d_estimates};
        return launch_search<STEREO, FORCE, TRACE>(p, su, n_frames, n_units, o.d_ref_words, stream, o.d_pred,
                                                   o.d_search_trace, o.mode == EncodeMode::search_guided ? &gp : nullptr);
    }
    // the base of a search + pairing or a window search takes no reference words and no trace (its candidates are
    // traced)
    case EncodeMode::search_pairing:
        if (int rc = launch_search<STEREO, FORCE, false>(p, su, n_frames, n_units, nullptr, stream, o.d_pred, nullptr,
                                                         nullptr))
            return rc;
        return launch_search_pairing<TRACE>(p, q, reinterpret_cast<SearchUnit *>(ws + l.pair_search), n_frames, n_units,
                                            stream);
    case EncodeMode::search_windows: {
        if (int rc = launch_search<STEREO, FORCE, false>(p, su, n_frames, n_units, nullptr, stream, o.d_pred, nullptr,
                                                         nullptr))
            return rc;
        WindowParams wp;
        wp.table = o.d_windows ? o.d_windows : g.windows;
        wp.mask = o.windows;
        wp.n = n_windows;
        wp.su = reinterpret_cast<SearchUnit *>(ws + l.window_search);
        wp.key = reinterpret_cast<unsigned long long *>(ws + l.window_keys);
        wp.n_window = o.d_n_window;
        wp.pred = o.d_window_pred;
        wp.trace = o.d_search_trace;
        return launch_windows<STEREO, TRACE>(p, wp, su, n_frames, n_units, o.d_base_words, stream);
    }
    }
    return 0;
}
using EncodeLaunch = int (*)(const EncodeOptions &, const EncodeLayout &, char *, const EncodeParams &,
                             const PairingParams &, uint32_t, cudaStream_t);

int encode_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels, selab200_subframe_desc *d_descs,
                  uint32_t *d_words, size_t capacity, uint64_t *d_used, int32_t *d_status, void *d_ws,
                  size_t ws_bytes, cudaStream_t stream, const EncodeOptions &o = EncodeOptions())
{
    if (int rc = check_channels(channels))
        return rc;
    const bool search_windows = o.mode == EncodeMode::search_windows;
    if (search_windows && !o.d_windows)
        if (int rc = check_windows(o.windows))
            return rc;
    const bool search_guided = o.mode == EncodeMode::search_guided;
    if (search_guided)
        if (int rc = check_candidates(o.candidates))
            return rc;
    const uint32_t n_windows = search_windows ? (uint32_t)__builtin_popcount(o.windows) : 0;
    const EncodeLayout l = encode_layout(o.mode, n_frames, channels, n_windows);
    if (ws_bytes < l.bytes)
        return fail(SELAB200_ERR_ARGUMENT, "encode workspace too small");
    if (channels == 2 && (reinterpret_cast<uintptr_t>(d_pcm) & 15) != 0) // the stereo kernel reads 16 bytes (4 sample pairs) at a time
        return fail(SELAB200_ERR_ARGUMENT, "stereo PCM must be 16-byte aligned on the device");
    const bool search_pairing = o.mode == EncodeMode::search_pairing;
    const bool pairing = o.mode == EncodeMode::pairing || search_pairing; // the pairing tables, counters and patch
    const size_t n_sub = (size_t)n_frames * channels;
    if (o.fresh) {
        CUDA_TRY(cudaMemsetAsync(d_status, 0, sizeof(int32_t), stream));
        CUDA_TRY(cudaMemsetAsync(d_used, 0, sizeof(uint64_t), stream));
        if (o.mode == EncodeMode::lossless) {
            CUDA_TRY(cudaMemsetAsync(o.lossless.n_entries, 0, sizeof(unsigned long long), stream));
            if (n_sub)
                CUDA_TRY(cudaMemsetAsync(o.lossless.entries, 0, n_sub * sizeof(selab200_lossless_entry), stream));
        }
        if (o.mode == EncodeMode::search || search_guided)
            CUDA_TRY(cudaMemsetAsync(o.d_ref_words, 0, sizeof(unsigned long long), stream));
        if (pairing) {
            CUDA_TRY(cudaMemsetAsync(o.d_base_words, 0, sizeof(unsigned long long), stream));
            CUDA_TRY(cudaMemsetAsync(o.d_n_difference, 0, sizeof(unsigned long long), stream));
        }
        if (search_windows) {
            CUDA_TRY(cudaMemsetAsync(o.d_base_words, 0, sizeof(unsigned long long), stream));
            CUDA_TRY(cudaMemsetAsync(o.d_n_window, 0, sizeof(unsigned long long), stream));
        }
    }
    if (n_frames == 0)
        return 0;
    char *ws = static_cast<char *>(d_ws);
    EncodeParams p;
    p.pcm = d_pcm;
    p.n_frames = n_frames;
    p.channels = channels;
    p.descs = d_descs;
    p.words = d_words;
    p.capacity = capacity;
    p.words_used = reinterpret_cast<unsigned long long *>(d_used);
    p.status = d_status;
    p.units = reinterpret_cast<UnitRecord *>(ws + l.units);
    p.slots = reinterpret_cast<uint32_t *>(ws + l.slots);
    p.means = reinterpret_cast<double *>(ws + l.means);
    p.residues = reinterpret_cast<int32_t *>(ws + l.residues);
    PairingParams q{};
    if (pairing) {
        q.table = reinterpret_cast<PairRecord *>(ws + l.pair_table);
        q.means = reinterpret_cast<double *>(ws + l.pair_means);
        q.par = reinterpret_cast<uint8_t *>(ws + l.par);
        q.stale = reinterpret_cast<uint32_t *>(ws + l.stale);
        q.base_words = o.d_base_words;
        q.n_difference = o.d_n_difference;
        q.pred = o.d_pair_pred;
        q.trace = o.d_search_trace;
    }
    // the one place where the call's stereo layout, forced predictors and trace buffer become template arguments
    constexpr EncodeLaunch kLaunch[8] = {
        launch_encoder<false, false, false>, launch_encoder<false, false, true>, launch_encoder<false, true, false>,
        launch_encoder<false, true, true>,   launch_encoder<true, false, false>, launch_encoder<true, false, true>,
        launch_encoder<true, true, false>,   launch_encoder<true, true, true>};
    const bool force = o.d_pred != nullptr, trace = o.d_trace || o.d_search_trace;
    if (int rc = kLaunch[(channels == 2) * 4 + force * 2 + trace](o, l, ws, p, q, n_windows, stream))
        return rc;
    const size_t scan_ctas = (n_sub + kScanTile - 1) / kScanTile;
    if (int rc = launch(k_encode_sizes, scan_ctas, kScanTile, 0, stream, "k_encode_sizes", p))
        return rc;
    if (o.before_scan)
        CUDA_TRY(cudaStreamWaitEvent(stream, o.before_scan, 0));
    if (int rc = launch(k_encode_scan, scan_ctas, kScanTile, 0, stream, "k_encode_scan", p))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(d_used, p.residues, 8, cudaMemcpyDeviceToDevice, stream)); // the new fill level (see k_encode_scan)
    if (pairing)
        if (int rc = launch(k_pairing_patch, (n_sub + 255) / 256, 256, 0, stream, "k_pairing_patch", p, q))
            return rc;
    // The fill level this chunk leaves behind must be captured BEFORE the next chunk's scan (on the
    // other compute lane) may overwrite *d_used: copy it out now and only then release the event.
    if (o.h_fill_after)
        CUDA_TRY(cudaMemcpyAsync(o.h_fill_after, d_used, 8, cudaMemcpyDeviceToHost, stream));
    if (o.after_scan)
        CUDA_TRY(cudaEventRecord(o.after_scan, stream));
    if (o.d_container) // byte-packed .sela stream instead of the word arena
        return launch(k_encode_gather_container, (n_sub + 7) / 8, 256, 0, stream, "k_encode_gather_container", p,
                      o.d_container, o.sub_base);
    return launch(k_encode_gather, (n_sub + 7) / 8, 256, 0, stream, "k_encode_gather", p);
}

// K5 launch: 64-word rings (8.3 KB per warp), eight parser steps per batch.
int launch_rice_decode(const DecodeParams &p, int which, cudaStream_t stream)
{
    const size_t n_sub = (size_t)p.n_frames * p.channels;
    const unsigned blocks = (unsigned)((n_sub + 32 * kRiceWarps - 1) / (32 * kRiceWarps));
    k_rice_decode<kRiceRing, kRiceBatch><<<blocks, 32 * kRiceWarps, 0, stream>>>(p, which);
    return launch_check(which ? "k_rice_decode(res)" : "k_rice_decode(refl)");
}

// Residue streams (K5 proper).  Large batches: one lane per stream through k_rice_decode_vc.  Smaller
// ones: every stream is cut into S parts first (k_rice_split_index), so that a batch of BASELINE's
// size still fills the machine.  SELAB200_RICE_SPLIT = 0 (first-generation kernel only), 1, 2, 4, 8, 16
// overrides the choice.  aux: n_sub * 64 bytes (split table + per-stream flags).
int rice_split_log2(size_t n_sub)
{
    if (const char *env = std::getenv("SELAB200_RICE_SPLIT")) {
        const long v = std::atol(env);
        if (v <= 0)
            return -1;
        int l = 0;
        while ((1 << (l + 1)) <= v && l < 4)
            l++;
        return l;
    }
    // One lane per stream (S = 1) through k_rice_decode_vc wins once every SM has a few warps of its own (about
    // 80 streams per SM): the two split passes then cost more than the extra warps bring.  Below that the
    // machine is starved and the streams are cut until there are about 270 parts per SM.  Both thresholds
    // scale with the SM count of the device.
    const size_t sms = (size_t)g.sms;
    if (n_sub >= 81 * sms)
        return 0;
    int l = 0;
    while (l < 4 && (n_sub << l) < 270 * sms)
        l++;
    return l;
}

template <int LOG2S>
int launch_split_index(const RiceVsParams &q, size_t n_sub, cudaStream_t stream)
{
    const unsigned blocks = (unsigned)(((n_sub << LOG2S) + 32 * kVsWarps - 1) / (32 * kVsWarps));
    if (int rc = set_smem(k_rice_split_index<LOG2S>, kSplitSmemBytes))
        return rc;
    k_rice_split_index<LOG2S><<<blocks, 32 * kVsWarps, kSplitSmemBytes, stream>>>(q);
    return launch_check("k_rice_split_index");
}

int launch_rice_residues(const DecodeParams &p, void *aux, cudaStream_t stream)
{
    const size_t n_sub = (size_t)p.n_frames * p.channels;
    const int log2s = rice_split_log2(n_sub);
    if (log2s < 0 || (reinterpret_cast<uintptr_t>(p.ws_res) & 15) != 0) {
        // the general parser alone: nothing is flagged.  Zero the flags that selab200_rice_decode_flagged counts,
        // which would otherwise count whatever the last call that used this scratch left there.
        CUDA_TRY(cudaMemsetAsync(static_cast<uint32_t *>(aux) + n_sub * 15, 0, n_sub * 4, stream));
        return launch_rice_decode(p, 1, stream);
    }
    RiceVsParams q;
    q.descs = p.descs;
    q.n_sub = (uint32_t)n_sub;
    q.channels = p.channels;
    q.words = p.words;
    q.n_words = p.n_words;
    q.out = p.ws_res;
    q.table = static_cast<uint32_t *>(aux);
    q.flags = q.table + n_sub * 15;
    q.status = p.status;
    int rc = 0;
    switch (log2s) {
    case 0: CUDA_TRY(cudaMemsetAsync(q.flags, 0, n_sub * 4, stream)); break;
    case 1: rc = launch_split_index<1>(q, n_sub, stream); break;
    case 2: rc = launch_split_index<2>(q, n_sub, stream); break;
    case 3: rc = launch_split_index<3>(q, n_sub, stream); break;
    default: rc = launch_split_index<4>(q, n_sub, stream); break;
    }
    if (rc)
        return rc;
    const size_t n_vs = n_sub << log2s;
    const unsigned vs_blocks = (unsigned)((n_vs + 32 * kVsWarps - 1) / (32 * kVsWarps));
    if (int rc2 = set_smem(k_rice_decode_vc, kVcSmemBytes))
        return rc2;
    k_rice_decode_vc<<<vs_blocks, 32 * kVsWarps, kVcSmemBytes, stream>>>(q, log2s);
    if (int rc2 = launch_check("k_rice_decode_vc"))
        return rc2;
    DecodeParams pf = p; // whatever was flagged: the general lane-per-stream parser decodes it again
    pf.rice_flags = q.flags;
    return launch_rice_decode(pf, 1, stream);
}

int decode_device(const selab200_subframe_desc *d_descs, uint32_t n_frames, uint32_t channels,
                  const uint32_t *d_words, size_t n_words, int16_t *d_pcm, int32_t *d_status, void *d_ws,
                  size_t ws_bytes, cudaStream_t stream, bool fresh = true)
{
    if (int rc = check_channels(channels))
        return rc;
    if (ws_bytes < selab200_decode_workspace_bytes(n_frames, channels))
        return fail(SELAB200_ERR_ARGUMENT, "decode workspace too small");
    if (fresh)
        CUDA_TRY(cudaMemsetAsync(d_status, 0, sizeof(int32_t), stream));
    if (n_frames == 0)
        return 0;
    const size_t n_sub = (size_t)n_frames * channels;
    DecodeParams p;
    p.descs = d_descs;
    p.n_frames = n_frames;
    p.channels = channels;
    p.words = d_words;
    p.n_words = n_words;
    p.pcm_out = d_pcm;
    p.status = d_status;
    p.ws_q = static_cast<int32_t *>(d_ws);
    p.ws_res = reinterpret_cast<int32_t *>(static_cast<char *>(d_ws) + align256(n_sub * 128 * 4));
    p.seg_index = reinterpret_cast<uint32_t *>(reinterpret_cast<char *>(p.ws_res) + align256(n_sub * kFrame * 4));
    p.rice_flags = nullptr;
    const size_t n_warps = synthesis_warps(n_sub);
    void *rice_aux = reinterpret_cast<char *>(p.seg_index) + align256(n_warps * 32 * 4);
    CUDA_TRY(cudaMemsetAsync(p.seg_index, 0xff, n_warps * 32 * 4, stream));
    const unsigned plan_ctas = (unsigned)((n_sub + kScanTile - 1) / kScanTile);
    k_decode_width_counts<<<plan_ctas, kScanTile, 0, stream>>>(p, static_cast<WidthCounts *>(rice_aux));
    if (int rc = launch_check("k_decode_width_counts"))
        return rc;
    k_decode_plan<<<plan_ctas, kScanTile, 0, stream>>>(p, static_cast<const WidthCounts *>(rice_aux));
    if (int rc = launch_check("k_decode_plan"))
        return rc;
    if (int rc = launch_rice_decode(p, 0, stream))
        return rc;
    if (int rc = launch_rice_residues(p, rice_aux, stream))
        return rc;
    k_synthesise_segments<<<(unsigned)n_warps, 32, 0, stream>>>(p);
    if (int rc = launch_check("k_synthesise_segments"))
        return rc;
    if (channels == 1) // desc_ok admits no difference subframe: its parent would have to be another channel
        return 0;
    k_diff_fixup<<<n_frames, 128, 0, stream>>>(p);
    return launch_check("k_diff_fixup");
}

int read_status(cudaStream_t stream, const int32_t *d_status)
{
    CUDA_TRY(cudaMemcpyAsync(&g.h_small->status, d_status, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    if (g.h_small->status != 0)
        return fail(g.h_small->status, "%s", status_text(g.h_small->status));
    return 0;
}

// Decode as decode_device does into the PCM scratch behind the decode workspace, then compare with d_ref.
// `fresh`: reset status, count and the per-pair records first (a stand-alone batch); the pipelined host
// paths reset once and point every chunk at its slice of the records.  Frames in the records are numbered
// from frame_base.
int verify_device(const selab200_subframe_desc *d_descs, uint32_t n_frames, uint32_t channels, const uint32_t *d_words,
                  size_t n_words, const int16_t *d_ref, selab200_verify_entry *d_entries, unsigned long long *d_count,
                  int32_t *d_status, void *d_ws, size_t ws_bytes, cudaStream_t stream, bool fresh = true,
                  uint32_t frame_base = 0)
{
    if (int rc = check_channels(channels))
        return rc;
    if (ws_bytes < selab200_verify_workspace_bytes(n_frames, channels))
        return fail(SELAB200_ERR_ARGUMENT, "verify workspace too small");
    if ((reinterpret_cast<uintptr_t>(d_ref) & 15) != 0)
        return fail(SELAB200_ERR_ARGUMENT, "source PCM must be 16-byte aligned on the device");
    const size_t n_sub = (size_t)n_frames * channels;
    if (fresh) {
        CUDA_TRY(cudaMemsetAsync(d_status, 0, sizeof(int32_t), stream));
        CUDA_TRY(cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), stream));
        if (n_sub)
            CUDA_TRY(cudaMemsetAsync(d_entries, 0, n_sub * sizeof(selab200_verify_entry), stream));
    }
    if (n_frames == 0)
        return 0;
    const size_t dec_bytes = align256(selab200_decode_workspace_bytes(n_frames, channels));
    int16_t *d_decoded = reinterpret_cast<int16_t *>(static_cast<char *>(d_ws) + dec_bytes);
    if (int rc = decode_device(d_descs, n_frames, channels, d_words, n_words, d_decoded, d_status, d_ws, dec_bytes,
                               stream, false))
        return rc;
    k_verify_compare<<<n_frames, kVerifyThreads, 0, stream>>>(d_decoded, d_ref, channels, frame_base, d_status,
                                                              d_entries, d_count);
    return launch_check("k_verify_compare");
}

// What the host-buffer verify paths keep on the device (g.verify): the count of differing pairs and a
// status word, the per-pair records of the whole batch, and -- for encode_container_verified only -- the
// guarded descriptors and the word arena the container image is unpacked into (file-order offsets, as
// the encoder assigned them, so every chunk lands in its own range).
struct VerifyArea {
    unsigned long long *count = nullptr;
    int32_t *status = nullptr;
    selab200_verify_entry *entries = nullptr;
    selab200_subframe_desc *descs = nullptr;
    uint32_t *arena = nullptr;
};

// Sizes g.verify for n_sub pairs (and arena_words unpacked words, if any) and resets count, status and records
// on `stream`.
int verify_area(size_t n_sub, size_t arena_words, cudaStream_t stream, VerifyArea &v)
{
    const size_t e_bytes = align256(n_sub * sizeof(selab200_verify_entry));
    const size_t d_bytes = arena_words ? align256(n_sub * sizeof(selab200_subframe_desc)) : 0;
    if (int rc = g.verify.ensure(256 + e_bytes + d_bytes + (arena_words ? arena_words * 4 + 64 : 0)))
        return rc;
    char *b = static_cast<char *>(g.verify.ptr);
    v.count = reinterpret_cast<unsigned long long *>(b);
    v.status = reinterpret_cast<int32_t *>(b + 8);
    v.entries = reinterpret_cast<selab200_verify_entry *>(b + 256);
    v.descs = arena_words ? reinterpret_cast<selab200_subframe_desc *>(b + 256 + e_bytes) : nullptr;
    v.arena = arena_words ? reinterpret_cast<uint32_t *>(b + 256 + e_bytes + d_bytes) : nullptr;
    CUDA_TRY(cudaMemsetAsync(b, 0, 256 + n_sub * sizeof(selab200_verify_entry), stream));
    return 0;
}

// A per-pair record that says something: a verify record with differing samples, a lossless record of a re-coded
// subframe.  Every other record is all zeros.
bool record_set(const selab200_verify_entry &e) { return e.n_differing != 0; }
bool record_set(const selab200_lossless_entry &e) { return e.words != 0; }

// Once the records are complete (the caller has synchronised the lanes that write them): the set ones of the
// n records at d_records, in order.  The records come down only when the count at d_count is not zero.  A
// non-null d_status is a decode status that lies right behind the count (VerifyArea): it comes down in the same
// copy, and a non-zero status fails the call.
template <typename T>
int collect_records(const unsigned long long *d_count, const int32_t *d_status, const T *d_records, size_t n,
                    cudaStream_t stream, std::vector<T> &out)
{
    out.clear();
    CUDA_TRY(cudaMemcpyAsync(&g.h_small->n_records, d_count, d_status ? 16 : 8, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    const unsigned long long count = g.h_small->n_records;
    const int32_t st = d_status ? g.h_small->records_status : 0;
    if (st != 0)
        return fail(st, "%s", status_text(st));
    if (count == 0)
        return 0;
    std::vector<T> all(n);
    CUDA_TRY(cudaMemcpyAsync(all.data(), d_records, n * sizeof(T), cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    out.reserve((size_t)count);
    for (const T &e : all)
        if (record_set(e))
            out.push_back(e);
    return 0;
}

// The records of a host-buffer call: *n_entries = all of them, at most `capacity` entries written.
template <typename T>
int deliver_records(const std::vector<T> &records, T *entries, size_t capacity, size_t *n_entries)
{
    *n_entries = records.size();
    if (capacity && !records.empty())
        memcpy(entries, records.data(), std::min(capacity, records.size()) * sizeof(T));
    return 0;
}

} // namespace

extern "C" {

int selab200_abi_version(void) { return SELAB200_ABI_VERSION; }
const char *selab200_last_error(void) { return g_error; }
uint64_t selab200_launch_count(void) { return g_launches.load(); }

uint64_t selab200_slot_launch_count(int slot)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    return slot >= 0 && slot < g_n_ctx ? g_slots[slot].launches.load() : 0;
}

// (g_mutex held; `g` points at the slot to set up)
static int init_slot(int device, int slot)
{
    CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) // sm_90a code loads on compute capability 9.0 only
        return fail(SELAB200_ERR_NO_DEVICE, "device %d is sm_%d%d; this build targets sm_90a only", device,
                    prop.major, prop.minor);
    CUDA_TRY(cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&g.s_h2d, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&g.s_d2h, cudaStreamNonBlocking));
    for (int i = 0; i < kLanes; i++)
        CUDA_TRY(cudaStreamCreateWithFlags(&g.s_compute[i], cudaStreamNonBlocking));
    for (int i = 0; i < kMaxChunks; i++) {
        CUDA_TRY(cudaEventCreateWithFlags(&g.ev_h2d[i], cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&g.ev_done[i], cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&g.ev_scan[i], cudaEventDisableTiming));
    }
    CUDA_TRY(cudaEventCreateWithFlags(&g.ev_reset, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&g.ev_rice, cudaEventDisableTiming));
    g.events = true;
    CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&g.h_small), sizeof(Counters)));
    CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&g.h_totals), (kMaxChunks + 1) * 8));
    if (int rc = g.small.ensure(256))
        return rc;
    // The window search's table, copied before any stream of the context can launch a kernel that reads it: a
    // pageable copy may still be in flight when cudaMemcpyToSymbol returns, and the streams above do not wait for it.
    CUDA_TRY(cudaMemcpyToSymbol(d_analysis_windows, analysis_window_table(), sizeof(d_analysis_windows)));
    CUDA_TRY(cudaDeviceSynchronize());
    void *table = nullptr;
    CUDA_TRY(cudaGetSymbolAddress(&table, d_analysis_windows));
    g.windows = static_cast<const double *>(table);
    g.spare = &g_spare_store[slot];
    g.launches = 0;
    g.device = device;
    g.sms = prop.multiProcessorCount;
    g.ready = true;
    return 0;
}

static void shutdown_slot()
{
    if (g.device >= 0)
        cudaSetDevice(g.device);
    if (g.stream)
        cudaStreamSynchronize(g.stream);
    if (g.spare) {
        for (ContainerBuffers &b : *g.spare)
            b.destroy();
        g.spare->clear();
    }
    g.in.release();
    g.descs.release();
    g.words.release();
    g.work.release();
    for (int i = 0; i < kLanes; i++)
        g.lane_work[i].release();
    g.aux.release();
    g.verify.release();
    g.lossless.release();
    g.clip_src.release();
    g.clip_pieces.release();
    g.clip_out.release();
    g.clip_rows.release();
    g.clip_runs.release();
    g.clip_stage.release();
    g.small.release();
    if (g.h_small)
        cudaFreeHost(g.h_small);
    g.h_small = nullptr;
    if (g.h_totals)
        cudaFreeHost(g.h_totals);
    g.h_totals = nullptr;
    for (cudaStream_t st : {g.stream, g.s_h2d, g.s_d2h})
        if (st)
            cudaStreamDestroy(st);
    for (int i = 0; i < kLanes; i++) {
        if (g.s_compute[i])
            cudaStreamDestroy(g.s_compute[i]);
        g.s_compute[i] = nullptr;
    }
    g.stream = g.s_h2d = g.s_d2h = nullptr;
    if (g.events) {
        for (int i = 0; i < kMaxChunks; i++) {
            cudaEventDestroy(g.ev_h2d[i]);
            cudaEventDestroy(g.ev_done[i]);
            cudaEventDestroy(g.ev_scan[i]);
        }
        cudaEventDestroy(g.ev_reset);
        cudaEventDestroy(g.ev_rice);
    }
    g.events = false;
    g.ready = false;
    g.device = -1;
    g.windows = nullptr; // the address belongs to this device; a slot set up again may get another
    g.last_rice_n_sub = 0;
    if (g_last_rice_ctx == tl_ctx)
        g_last_rice_ctx = nullptr;
}

static void shutdown_all()
{
    for (int i = 0; i < g_n_ctx; i++) {
        tl_ctx = &g_slots[i];
        shutdown_slot();
    }
    g_n_ctx = 0;
    tl_ctx = &g_slots[0];
}

int selab200_init_devices(int count, const int *devices)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (count < 1 || count > kMaxDevices || !devices)
        return fail(SELAB200_ERR_ARGUMENT, "device count must be in [1, %d]", kMaxDevices);
    bool same = count == g_n_ctx;
    for (int i = 0; same && i < count; i++)
        same = g_slots[i].ready && g_slots[i].device == devices[i];
    if (same) {
        tl_ctx = &g_slots[0];
        return 0;
    }
    int have = 0;
    cudaError_t e = cudaGetDeviceCount(&have);
    if (e != cudaSuccess || have == 0)
        return fail(SELAB200_ERR_NO_DEVICE, "no CUDA device available (%s); this library has no CPU path",
                    e == cudaSuccess ? "count == 0" : cudaGetErrorString(e));
    // A device may be listed more than once: every entry is a context of its own, and contexts share nothing (the
    // device globals are constant tables, which every slot of a device writes with the same contents).
    for (int i = 0; i < count; i++)
        if (devices[i] < 0 || devices[i] >= have)
            return fail(SELAB200_ERR_ARGUMENT, "device %d out of range (have %d)", devices[i], have);
    // a different set of devices than before: everything the old contexts own (streams, events, pools) lives on
    // the old devices, so they are torn down completely before the new ones are set up
    shutdown_all();
    for (int i = 0; i < count; i++) {
        tl_ctx = &g_slots[i];
        if (int rc = init_slot(devices[i], i)) {
            char keep[sizeof g_error];
            memcpy(keep, g_error, sizeof keep);
            g_n_ctx = i + 1;
            shutdown_all();
            memcpy(g_error, keep, sizeof keep);
            return rc;
        }
    }
    g_n_ctx = count;
    tl_ctx = &g_slots[0];
    CUDA_TRY(cudaSetDevice(g_slots[0].device));
    return 0;
}

int selab200_init(int device) { return selab200_init_devices(1, &device); }

int selab200_device_count(void)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    return g_n_ctx;
}

void selab200_shutdown(void)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    shutdown_all();
}

void *selab200_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) {
        fail(SELAB200_ERR_CUDA, "cudaMallocHost(%zu) failed", bytes);
        return nullptr;
    }
    return p;
}

void selab200_host_free(void *p)
{
    if (p)
        cudaFreeHost(p);
}

size_t selab200_encode_words_bound(uint32_t n_frames, uint32_t channels)
{
    // A subframe never exceeds its scratch slot (larger streams are refused with
    // SELAB200_ERR_RANGE): residues <= 1568 words (24.5 bits/sample), coefficients <= 32.
    return (size_t)n_frames * channels * kSlotWords + 64;
}

size_t selab200_encode_workspace_bytes(uint32_t n_frames, uint32_t channels)
{
    return encode_layout(EncodeMode::plain, n_frames, channels).bytes;
}

size_t selab200_encode_lossless_workspace_bytes(uint32_t n_frames, uint32_t channels)
{
    return encode_layout(EncodeMode::lossless, n_frames, channels).bytes;
}

size_t selab200_encode_pairing_workspace_bytes(uint32_t n_frames, uint32_t channels)
{
    return encode_layout(EncodeMode::pairing, n_frames, channels).bytes;
}

size_t selab200_encode_search_workspace_bytes(uint32_t n_frames, uint32_t channels)
{
    return encode_layout(EncodeMode::search, n_frames, channels).bytes;
}

size_t selab200_encode_search_pairing_workspace_bytes(uint32_t n_frames, uint32_t channels)
{
    return encode_layout(EncodeMode::search_pairing, n_frames, channels).bytes;
}

size_t selab200_encode_search_windows_workspace_bytes(uint32_t n_frames, uint32_t channels, uint32_t windows)
{
    return encode_layout(EncodeMode::search_windows, n_frames, channels, (uint32_t)__builtin_popcount(windows)).bytes;
}

size_t selab200_encode_search_guided_workspace_bytes(uint32_t n_frames, uint32_t channels)
{
    return encode_layout(EncodeMode::search_guided, n_frames, channels).bytes;
}

int selab200_analysis_window(int index, double *out)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (index < 0 || index >= kAnalysisWindows || !out)
        return fail(SELAB200_ERR_ARGUMENT, "window %d is not in the table (0..%d), or out is null", index,
                    kAnalysisWindows - 1);
    memcpy(out, analysis_window_table() + (size_t)index * kFrame, kFrame * sizeof(double));
    return 0;
}

size_t selab200_decode_workspace_bytes(uint32_t n_frames, uint32_t channels)
{
    const size_t n_sub = (size_t)n_frames * channels;
    return align256(n_sub * 128 * 4) + align256(n_sub * kFrame * 4) + align256(synthesis_warps(n_sub) * 32 * 4) +
           align256(n_sub * 64) + 256;
}

size_t selab200_verify_workspace_bytes(uint32_t n_frames, uint32_t channels)
{
    // the decode workspace, then the decoded PCM
    return align256(selab200_decode_workspace_bytes(n_frames, channels)) + align256((size_t)n_frames * channels * kFrame * 2);
}

int selab200_encode_frames_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                  selab200_subframe_desc *d_descs, uint32_t *d_words, size_t words_capacity,
                                  uint64_t *d_words_used, int32_t *d_status, void *d_workspace,
                                  size_t workspace_bytes, void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_pcm ? require_ready_for(d_pcm) : require_ready())
        return rc;
    if (!d_pcm || !d_descs || !d_words || !d_words_used || !d_status || !d_workspace)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    return encode_device(d_pcm, n_frames, channels, d_descs, d_words, words_capacity, d_words_used, d_status,
                         d_workspace, workspace_bytes, (cudaStream_t)stream);
}

int selab200_encode_frames_lossless_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                           selab200_subframe_desc *d_descs, uint32_t *d_words, size_t words_capacity,
                                           uint64_t *d_words_used, selab200_lossless_entry *d_entries,
                                           uint64_t *d_n_entries, int32_t *d_status, void *d_workspace,
                                           size_t workspace_bytes, void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_pcm ? require_ready_for(d_pcm) : require_ready())
        return rc;
    if (!d_pcm || !d_descs || !d_words || !d_words_used || !d_entries || !d_n_entries || !d_status || !d_workspace)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    EncodeOptions o;
    o.mode = EncodeMode::lossless;
    o.lossless = LosslessArgs{d_entries, reinterpret_cast<unsigned long long *>(d_n_entries), 0};
    return encode_device(d_pcm, n_frames, channels, d_descs, d_words, words_capacity, d_words_used, d_status,
                         d_workspace, workspace_bytes, (cudaStream_t)stream, o);
}

int selab200_encode_frames_search_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                         selab200_subframe_desc *d_descs, uint32_t *d_words, size_t words_capacity,
                                         uint64_t *d_words_used, uint64_t *d_ref_words, int32_t *d_status,
                                         void *d_workspace, size_t workspace_bytes, void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_pcm ? require_ready_for(d_pcm) : require_ready())
        return rc;
    if (!d_pcm || !d_descs || !d_words || !d_words_used || !d_ref_words || !d_status || !d_workspace)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    EncodeOptions o;
    o.mode = EncodeMode::search;
    o.d_ref_words = reinterpret_cast<unsigned long long *>(d_ref_words);
    return encode_device(d_pcm, n_frames, channels, d_descs, d_words, words_capacity, d_words_used, d_status,
                         d_workspace, workspace_bytes, (cudaStream_t)stream, o);
}

int selab200_encode_frames_pairing_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                          selab200_subframe_desc *d_descs, uint32_t *d_words, size_t words_capacity,
                                          uint64_t *d_words_used, uint64_t *d_base_words, uint64_t *d_n_difference,
                                          int32_t *d_status, void *d_workspace, size_t workspace_bytes, void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_pcm ? require_ready_for(d_pcm) : require_ready())
        return rc;
    if (!d_pcm || !d_descs || !d_words || !d_words_used || !d_base_words || !d_n_difference || !d_status || !d_workspace)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    EncodeOptions o;
    o.mode = EncodeMode::pairing;
    o.d_base_words = reinterpret_cast<unsigned long long *>(d_base_words);
    o.d_n_difference = reinterpret_cast<unsigned long long *>(d_n_difference);
    return encode_device(d_pcm, n_frames, channels, d_descs, d_words, words_capacity, d_words_used, d_status,
                         d_workspace, workspace_bytes, (cudaStream_t)stream, o);
}

int selab200_encode_frames_search_pairing_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                                 selab200_subframe_desc *d_descs, uint32_t *d_words,
                                                 size_t words_capacity, uint64_t *d_words_used, uint64_t *d_base_words,
                                                 uint64_t *d_n_difference, int32_t *d_status, void *d_workspace,
                                                 size_t workspace_bytes, void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_pcm ? require_ready_for(d_pcm) : require_ready())
        return rc;
    if (!d_pcm || !d_descs || !d_words || !d_words_used || !d_base_words || !d_n_difference || !d_status || !d_workspace)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    EncodeOptions o;
    o.mode = EncodeMode::search_pairing;
    o.d_base_words = reinterpret_cast<unsigned long long *>(d_base_words);
    o.d_n_difference = reinterpret_cast<unsigned long long *>(d_n_difference);
    return encode_device(d_pcm, n_frames, channels, d_descs, d_words, words_capacity, d_words_used, d_status,
                         d_workspace, workspace_bytes, (cudaStream_t)stream, o);
}

int selab200_encode_frames_search_windows_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                                uint32_t windows, selab200_subframe_desc *d_descs, uint32_t *d_words,
                                                size_t words_capacity, uint64_t *d_words_used, uint64_t *d_base_words,
                                                uint64_t *d_n_window, int32_t *d_status, void *d_workspace,
                                                size_t workspace_bytes, void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_pcm ? require_ready_for(d_pcm) : require_ready())
        return rc;
    if (!d_pcm || !d_descs || !d_words || !d_words_used || !d_base_words || !d_n_window || !d_status || !d_workspace)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    if (int rc = check_windows(windows))
        return rc;
    EncodeOptions o;
    o.mode = EncodeMode::search_windows;
    o.windows = windows;
    o.d_base_words = reinterpret_cast<unsigned long long *>(d_base_words);
    o.d_n_window = reinterpret_cast<unsigned long long *>(d_n_window);
    return encode_device(d_pcm, n_frames, channels, d_descs, d_words, words_capacity, d_words_used, d_status,
                         d_workspace, workspace_bytes, (cudaStream_t)stream, o);
}

int selab200_encode_frames_search_guided_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                                uint32_t candidates, selab200_subframe_desc *d_descs, uint32_t *d_words,
                                                size_t words_capacity, uint64_t *d_words_used, uint64_t *d_ref_words,
                                                int32_t *d_status, void *d_workspace, size_t workspace_bytes,
                                                void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_pcm ? require_ready_for(d_pcm) : require_ready())
        return rc;
    if (!d_pcm || !d_descs || !d_words || !d_words_used || !d_ref_words || !d_status || !d_workspace)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    if (int rc = check_candidates(candidates))
        return rc;
    EncodeOptions o;
    o.mode = EncodeMode::search_guided;
    o.candidates = candidates;
    o.d_ref_words = reinterpret_cast<unsigned long long *>(d_ref_words);
    return encode_device(d_pcm, n_frames, channels, d_descs, d_words, words_capacity, d_words_used, d_status,
                         d_workspace, workspace_bytes, (cudaStream_t)stream, o);
}

int selab200_decode_frames_device(const selab200_subframe_desc *d_descs, uint32_t n_frames, uint32_t channels,
                                  const uint32_t *d_words, size_t n_words, int16_t *d_pcm_out, int32_t *d_status,
                                  void *d_workspace, size_t workspace_bytes, void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_descs ? require_ready_for(d_descs) : require_ready())
        return rc;
    if (!d_descs || !d_words || !d_pcm_out || !d_status || !d_workspace)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    return decode_device(d_descs, n_frames, channels, d_words, n_words, d_pcm_out, d_status, d_workspace,
                         workspace_bytes, (cudaStream_t)stream);
}

int selab200_verify_frames_device(const selab200_subframe_desc *d_descs, uint32_t n_frames, uint32_t channels,
                                  const uint32_t *d_words, size_t n_words, const int16_t *d_pcm_ref,
                                  selab200_verify_entry *d_entries, uint64_t *d_n_differing, int32_t *d_status,
                                  void *d_workspace, size_t workspace_bytes, void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_descs ? require_ready_for(d_descs) : require_ready())
        return rc;
    if (!d_descs || !d_words || !d_pcm_ref || !d_entries || !d_n_differing || !d_status || !d_workspace)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    return verify_device(d_descs, n_frames, channels, d_words, n_words, d_pcm_ref, d_entries,
                         reinterpret_cast<unsigned long long *>(d_n_differing), d_status, d_workspace, workspace_bytes,
                         (cudaStream_t)stream);
}

int selab200_rice_decode_frames_device(const selab200_subframe_desc *d_descs, uint32_t n_frames, uint32_t channels,
                                       const uint32_t *d_words, size_t n_words, int32_t *d_residues,
                                       int32_t *d_status, void *stream)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = d_descs ? require_ready_for(d_descs) : require_ready())
        return rc;
    if (!d_descs || !d_words || !d_residues || !d_status)
        return fail(SELAB200_ERR_ARGUMENT, "null device pointer");
    if (int rc = check_channels(channels))
        return rc;
    CUDA_TRY(cudaMemsetAsync(d_status, 0, sizeof(int32_t), (cudaStream_t)stream));
    if (n_frames == 0)
        return 0;
    DecodeParams p;
    p.descs = d_descs;
    p.n_frames = n_frames;
    p.channels = channels;
    p.words = d_words;
    p.n_words = n_words;
    p.pcm_out = nullptr;
    p.status = d_status;
    p.ws_q = nullptr;
    p.ws_res = d_residues;
    p.seg_index = nullptr;
    p.rice_flags = nullptr;
    if (int rc = aux_for((size_t)n_frames * channels * 64 + 256, (cudaStream_t)stream))
        return rc;
    g.last_rice_n_sub = (size_t)n_frames * channels;
    g.last_rice_stream = (cudaStream_t)stream;
    g_last_rice_ctx = tl_ctx;
    const int rc = launch_rice_residues(p, g.aux.ptr, (cudaStream_t)stream);
    CUDA_TRY(cudaEventRecord(g.ev_rice, (cudaStream_t)stream)); // the next user of aux waits for this call
    return rc;
}

int selab200_rice_decode_flagged(uint32_t *n_flagged)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!n_flagged)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    *n_flagged = 0;
    if (g_last_rice_ctx && g_last_rice_ctx->ready) { // the device the last call ran on, which need not be the primary
        tl_ctx = g_last_rice_ctx;
        CUDA_TRY(cudaSetDevice(g.device));
    }
    const size_t n = g.last_rice_n_sub;
    if (n == 0 || g.aux.bytes < n * 64)
        return 0;
    std::vector<uint32_t> flags(n);
    CUDA_TRY(cudaStreamSynchronize(g.last_rice_stream));
    CUDA_TRY(cudaMemcpy(flags.data(), static_cast<uint32_t *>(g.aux.ptr) + n * 15, n * 4, cudaMemcpyDeviceToHost));
    uint32_t c = 0;
    for (uint32_t f : flags)
        c += f != 0;
    *n_flagged = c;
    return 0;
}

} // extern "C"

static_assert(sizeof(selab200_analysis_trace) == 2832, "selab200_analysis_trace layout (include/sela_b200.h)");
static_assert(sizeof(selab200_lossless_entry) == 16, "selab200_lossless_entry layout (include/sela_b200.h)");
static_assert(sizeof(selab200_predictor) == 404, "selab200_predictor layout (include/sela_b200.h)");

// Bytes of container in front of frame f when `words` Rice words precede it.
static unsigned long long container_frame_byte(unsigned long long f, uint32_t channels, unsigned long long words)
{
    return kContainerHeaderBytes + 4 * f + (unsigned long long)kSubframeHeaderBytes * f * channels + 4 * words;
}

// Host-buffer batch calls.  Pipelined in chunks of frames (plan_chunks) over three engines:
//   s_h2d      PCM (encode) / descriptors + words (decode) of chunk c+1 .. go up
//   s_compute  compute lanes run the kernels of chunk c, so that the tails of one chunk overlap the head of the
//              next.  Encode alternates two lanes (its scans are chained by events because each needs the arena
//              fill level its predecessor left in *d_used) and verifies, if asked, on the others; decode gives
//              every chunk a lane of its own, up to kLanes.
//   s_d2h      results of chunk c-1 come down
// With pinned host buffers (selab200_host_alloc) the three overlap; pageable memory works
// but serialises inside the driver.

// Where the pipelined encoder puts its output.
enum class EncodeForm { arena, container };
struct EncodeTarget {
    EncodeForm form;
    // Leave the word arena / container body on the device (g.words) instead of copying it out chunk by chunk:
    // with several devices, every device's block is placed once the sizes of the blocks before it are known.
    bool defer;
    selab200_subframe_desc *descs; // arena: one descriptor per subframe (written even with `defer`)
    uint32_t *words;               // arena: the Rice words (unused with `defer`)
    uint8_t *container;            // container: the whole .sela stream, header written by the caller (unused with `defer`)
    size_t words_capacity;         // Rice words the output holds
    bool verify = false;           // container: also verify the image, chunk by chunk on the device (Result::report)
};

// What a host-buffer call returns besides its output arrays: for one block of frames (DevicePart), or, summed with
// add(), for the whole call.  The lists' frames are file-global.
struct Result {
    size_t words = 0;                  // encode: the words used (for CAPACITY: the size the caller needs)
    unsigned long long ref_words = 0;  // search: the words the reference encoder's choice takes
    unsigned long long base_words = 0; // pairing: the words of its base, the lossless encode (search_pairing: the search)
    unsigned long long n_difference = 0; // pairing, search_pairing: the difference subframes chosen
    unsigned long long n_window = 0;   // search_windows: the units coded from a window
    size_t ref_bytes = 0;              // container search / pairing / search_pairing: the size of the output it is
                                       // measured against
    std::vector<selab200_lossless_entry> recoded; // lossless: the re-coded (frame, channel) pairs
    std::vector<selab200_verify_entry> report;    // verify: the (frame, channel) pairs that do not decode back
    void add(const Result &b)
    {
        words += b.words;
        ref_words += b.ref_words;
        base_words += b.base_words;
        n_difference += b.n_difference;
        n_window += b.n_window;
        recoded.insert(recoded.end(), b.recoded.begin(), b.recoded.end());
        report.insert(report.end(), b.report.begin(), b.report.end());
    }
};

// Once the encode on `stream` is done: its counters (g.small) into r, and its status.
static int read_counters(cudaStream_t stream, Result &r)
{
    CUDA_TRY(cudaMemcpyAsync(g.h_small, device_counters(), kEncodeCounterBytes, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    const Counters &c = *g.h_small;
    r.words = (size_t)c.used;
    r.ref_words = c.ref_words;
    r.base_words = c.base_words;
    r.n_difference = c.n_difference;
    r.n_window = c.n_window;
    return c.status ? fail(c.status, "%s", status_text(c.status)) : 0;
}

// g.lossless sized for n_sub pairs: the count of re-coded pairs, then their per-pair records.
static int lossless_area(size_t n_sub, LosslessArgs &la)
{
    if (int rc = g.lossless.ensure(256 + n_sub * sizeof(selab200_lossless_entry)))
        return rc;
    la.n_entries = static_cast<unsigned long long *>(g.lossless.ptr);
    la.entries = reinterpret_cast<selab200_lossless_entry *>(static_cast<char *>(g.lossless.ptr) + 256);
    return 0;
}

// The pipelined encoder over host buffers, running `mode`, into r; frames numbered from frame_base in what it
// reports.  arg: the mode's parameter, the window search's mask or the guided order search's candidate count.
static int encode_host(const int16_t *pcm, uint32_t n_frames, uint32_t channels, const EncodeTarget &t,
                       EncodeMode mode, uint32_t arg, uint32_t frame_base, Result &r)
{
    const size_t words_capacity = t.words_capacity;
    const bool to_container = t.form == EncodeForm::container;
    if (n_frames == 0)
        return 0;
    PipelineDrain drain;
    const ChunkPlan plan = plan_chunks(n_frames);
    const uint32_t n_chunks = plan.chunks();
    const size_t n_sub = (size_t)n_frames * channels;
    const size_t frame_bytes = (size_t)channels * kFrame * 2;
    const bool verify = t.verify && to_container;
    const bool lossless = mode == EncodeMode::lossless;
    const uint32_t windows = mode == EncodeMode::search_windows ? arg : 0;
    const size_t ws_bytes = encode_layout(mode, plan.max_frames, channels, (uint32_t)__builtin_popcount(windows)).bytes;
    if (int rc = g.in.ensure(n_sub * kFrame * 2)) return rc;
    if (int rc = g.descs.ensure(n_sub * sizeof(selab200_subframe_desc))) return rc;
    if (int rc = g.words.ensure(container_frame_byte(n_frames, channels, words_capacity) + 64)) return rc;
    LosslessArgs records{}; // lossless: the re-coded pairs of the whole batch
    if (lossless)
        if (int rc = lossless_area(n_sub, records)) return rc;
    constexpr int kEncLanes = 2;
    for (int i = 0; i < kEncLanes && (uint32_t)i < n_chunks; i++)
        if (int rc = g.lane_work[i].ensure(ws_bytes)) return rc;
    // verify: chunk c is checked on lane kEncLanes + c % kVerifyLanes once its gather is done, so that the check
    // (a decode: latency-bound Rice kernels) overlaps the encode of the chunks after it instead of queueing in front
    constexpr int kVerifyLanes = kLanes - kEncLanes;
    for (int i = 0; verify && i < kVerifyLanes && (uint32_t)i < n_chunks; i++)
        if (int rc = g.lane_work[kEncLanes + i].ensure(selab200_verify_workspace_bytes(plan.max_frames, channels))) return rc;
    Counters *d_ctr = device_counters(); // the mode's counters are summed over the chunks
    int16_t *d_pcm = static_cast<int16_t *>(g.in.ptr);
    selab200_subframe_desc *d_descs = static_cast<selab200_subframe_desc *>(g.descs.ptr);
    uint32_t *d_words = static_cast<uint32_t *>(g.words.ptr);
    // every offset the encoder hands out while its status is clean lies below both of these
    const size_t arena_words = std::min(words_capacity, selab200_encode_words_bound(n_frames, channels));
    VerifyArea va;
    if (verify)
        if (int rc = verify_area(n_sub, arena_words, g.s_compute[0], va)) return rc;

    CUDA_TRY(cudaMemsetAsync(d_ctr, 0, kEncodeCounterBytes, g.s_compute[0]));
    if (lossless)
        CUDA_TRY(cudaMemsetAsync(g.lossless.ptr, 0, 256 + n_sub * sizeof(selab200_lossless_entry), g.s_compute[0]));
    CUDA_TRY(cudaEventRecord(g.ev_reset, g.s_compute[0]));
    for (int i = 1; i < kLanes; i++)
        CUDA_TRY(cudaStreamWaitEvent(g.s_compute[i], g.ev_reset, 0));
    for (uint32_t c = 0; c < n_chunks; c++) {
        const uint32_t f0 = plan.start[c], nf = plan.start[c + 1] - f0;
        CUDA_TRY(cudaMemcpyAsync(d_pcm + (size_t)f0 * channels * kFrame, pcm + (size_t)f0 * channels * kFrame,
                                 nf * frame_bytes, cudaMemcpyHostToDevice, g.s_h2d));
        CUDA_TRY(cudaEventRecord(g.ev_h2d[c], g.s_h2d));
        cudaStream_t cs = g.s_compute[c % kEncLanes];
        DeviceBuffer &ws = g.lane_work[c % kEncLanes];
        CUDA_TRY(cudaStreamWaitEvent(cs, g.ev_h2d[c], 0));
        EncodeOptions o;
        o.mode = mode;
        o.fresh = false;
        o.before_scan = c ? g.ev_scan[c - 1] : nullptr;
        o.after_scan = g.ev_scan[c];
        o.h_fill_after = &g.h_totals[c + 1];
        o.d_container = to_container ? static_cast<uint8_t *>(g.words.ptr) : nullptr;
        o.sub_base = (unsigned long long)f0 * channels;
        if (lossless)
            o.lossless = LosslessArgs{records.entries + (size_t)f0 * channels, records.n_entries, frame_base + f0};
        o.d_ref_words = &d_ctr->ref_words;
        o.d_base_words = &d_ctr->base_words;
        o.d_n_difference = &d_ctr->n_difference;
        o.windows = windows;
        o.d_n_window = &d_ctr->n_window;
        o.candidates = mode == EncodeMode::search_guided ? arg : 0;
        if (int rc = encode_device(d_pcm + (size_t)f0 * channels * kFrame, nf, channels, d_descs + (size_t)f0 * channels,
                                   d_words, words_capacity, &d_ctr->used, &d_ctr->status, ws.ptr, ws.bytes, cs, o))
            return rc;
        CUDA_TRY(cudaEventRecord(g.ev_done[c], cs));
        if (verify) {
            // The bytes just gathered, read back the way a reader does: the word arrays unpacked from the image,
            // decoded, and compared with the PCM this chunk already holds.  The guard hands the unpack empty
            // descriptors once the encoder has failed (offsets past the arena), and the call fails anyway.
            const size_t chunk_sub = (size_t)nf * channels;
            selab200_subframe_desc *vd = va.descs + (size_t)f0 * channels;
            cudaStream_t vs = g.s_compute[kEncLanes + c % kVerifyLanes];
            DeviceBuffer &vws = g.lane_work[kEncLanes + c % kVerifyLanes];
            CUDA_TRY(cudaStreamWaitEvent(vs, g.ev_done[c], 0));
            k_verify_guard_descs<<<(unsigned)((chunk_sub + 255) / 256), 256, 0, vs>>>(d_descs + (size_t)f0 * channels,
                                                                                   (uint32_t)chunk_sub, &d_ctr->status, vd);
            if (int rc = launch_check("k_verify_guard_descs"))
                return rc;
            k_container_unpack<<<(unsigned)((chunk_sub + 7) / 8), 256, 0, vs>>>(static_cast<const uint8_t *>(g.words.ptr), vd,
                                                                               (uint32_t)chunk_sub, channels,
                                                                               (unsigned long long)f0 * channels, va.arena);
            if (int rc = launch_check("k_container_unpack"))
                return rc;
            if (int rc = verify_device(vd, nf, channels, va.arena, arena_words, d_pcm + (size_t)f0 * channels * kFrame,
                                       va.entries + (size_t)f0 * channels, va.count, va.status, vws.ptr, vws.bytes, vs,
                                       false, frame_base + f0))
                return rc;
        }
    }
    g.h_totals[0] = 0;
    for (uint32_t c = 0; c < n_chunks; c++) {
        const uint32_t f0 = plan.start[c], nf = plan.start[c + 1] - f0;
        CUDA_TRY(cudaEventSynchronize(g.ev_done[c]));
        const unsigned long long lo = g.h_totals[c], hi = g.h_totals[c + 1];
        if (hi > words_capacity || hi < lo)
            break; // capacity exceeded: reported through the status word below
        if (t.defer) {
            if (!to_container)
                CUDA_TRY(cudaMemcpyAsync(t.descs + (size_t)f0 * channels, d_descs + (size_t)f0 * channels,
                                         (size_t)nf * channels * sizeof(selab200_subframe_desc), cudaMemcpyDeviceToHost,
                                         g.s_d2h));
            continue;
        }
        if (to_container) {
            const unsigned long long b0 = container_frame_byte(f0, channels, lo);
            const unsigned long long b1 = container_frame_byte(f0 + nf, channels, hi);
            CUDA_TRY(cudaMemcpyAsync(t.container + b0, static_cast<uint8_t *>(g.words.ptr) + b0, b1 - b0,
                                     cudaMemcpyDeviceToHost, g.s_d2h));
            continue;
        }
        CUDA_TRY(cudaMemcpyAsync(t.descs + (size_t)f0 * channels, d_descs + (size_t)f0 * channels,
                                 (size_t)nf * channels * sizeof(selab200_subframe_desc), cudaMemcpyDeviceToHost,
                                 g.s_d2h));
        CUDA_TRY(cudaMemcpyAsync(t.words + lo, d_words + lo, (hi - lo) * 4, cudaMemcpyDeviceToHost, g.s_d2h));
    }
    for (int i = 0; i < (verify ? kLanes : kEncLanes); i++)
        CUDA_TRY(cudaStreamSynchronize(g.s_compute[i]));
    if (int rc = read_counters(g.s_d2h, r))
        return rc;
    if (lossless)
        if (int rc = collect_records(records.n_entries, nullptr, records.entries, n_sub, g.s_d2h, r.recoded))
            return rc;
    return verify ? collect_records(va.count, va.status, va.entries, n_sub, g.s_d2h, r.report) : 0;
}

// The words n descriptors reference, [lo, hi) (descriptors need not be in arena order); hi <= lo if none.
static void words_referenced(const selab200_subframe_desc *dc, size_t n, size_t n_words, unsigned long long &lo,
                             unsigned long long &hi)
{
    lo = ~0ull;
    hi = 0;
    for (size_t i = 0; i < n; i++) {
        const unsigned long long a0 = dc[i].refl_offset, a1 = a0 + dc[i].refl_words;
        const unsigned long long b0 = dc[i].res_offset, b1 = b0 + dc[i].res_words;
        // out-of-range descriptors are rejected on the device (desc_ok), by the same wrap-free test
        if (words_in_arena(a0, dc[i].refl_words, n_words) && words_in_arena(b0, dc[i].res_words, n_words)) {
            lo = a0 < lo ? a0 : lo;
            lo = b0 < lo ? b0 : lo;
            hi = a1 > hi ? a1 : hi;
            hi = b1 > hi ? b1 : hi;
        }
    }
}

struct selab200_container {
    const uint8_t *bytes = nullptr; // the caller's bytes, or (host-resident) the handle's page-locked copy
    size_t n_bytes = 0;
    selab200_container_info info{};
    ContainerBuffers buf;
    size_t piece_bytes = 0;
    int n_pieces = 0;
    // selab200_container_open_host: no device image (buf.d_bytes stays null); the page-locked copy is mapped, and
    // clip calls fetch what they read from it through `mapped`, its device address
    bool host = false;
    const uint8_t *mapped = nullptr;
};

// One host-to-device copy.
struct Upload {
    void *dst = nullptr;
    const void *src = nullptr;
    size_t bytes = 0;
};

// One group of the clip decode's selection: frames of any open containers, numbered from 0 in (container, frame)
// order.  Per subframe a descriptor re-based into one compact arena of n_words words, the file byte of its reflection
// words and their device address: in its container's image, or for a host-resident container in the staging buffer
// its fetch run goes to (plan_fetch).  Per frame its container and the end of the bytes it reads (+3 bytes of slack),
// which say which upload pieces a chunk waits for.
struct ClipSelection {
    std::vector<selab200_subframe_desc> descs;
    std::vector<unsigned long long> src, at;
    std::vector<const selab200_container *> frame_h;
    std::vector<unsigned long long> frame_end;
    // host-resident subframes (plan_fetch): the group's fetch runs in selection order, each with its first subframe,
    // and per subframe its run (-1: a device-resident image)
    std::vector<FetchRun> runs;
    std::vector<size_t> run_first;
    std::vector<int64_t> run;
};

// Where the decode-side pipeline's coded input comes from, frames numbered file-globally in the first two cases: the
// caller's descriptor and word arrays (h == nullptr), an open container whose byte image is unpacked into the word
// arena on the device, or a clip selection (sel: descs are its descriptors, n_words its arena) unpacked from the
// images of several open containers.  start() sizes the arena for the block of frames [F0, F0 + NF) and uploads what
// the block needs as a whole; chunk() puts one chunk's descriptors and words on the device, then `also` on the stream
// that carried the descriptors, and makes the chunk's lane wait for all of it.
struct CodedInput {
    const selab200_subframe_desc *descs; // the whole file's descriptors, in host memory
    const uint32_t *words;               // caller arrays: the words the descriptors reference
    size_t n_words;
    const selab200_container *h;         // or an open container
    const ClipSelection *sel = nullptr;  // or a clip selection
    // set by start()
    uint32_t channels = 0;
    uint32_t *arena = nullptr;           // the decoder's word array, addressed by the descriptors' offsets
    const uint8_t *d_bytes = nullptr;    // container: the byte image on this device, addressed by file offset
    bool primary = true;
    std::vector<int> fetched;            // clip selection: per chunk, the fetch piece (g.ev_h2d) it waits for, or -1

    int start(uint32_t F0, uint32_t NF, uint32_t ch, const ChunkPlan &plan)
    {
        channels = ch;
        if (sel) { // re-based descriptors: the arena is addressed from 0
            if (int rc = g.words.ensure(n_words * 4 + 96)) return rc;
            arena = reinterpret_cast<uint32_t *>(static_cast<char *>(g.words.ptr) + 16); // 16 bytes of slack in front
            if (int rc = g.clip_src.ensure(sel->src.size() * sizeof(unsigned long long))) return rc;
            return fetch(plan);
        }
        if (!h) {
            if (int rc = g.words.ensure(n_words * 4 + 16)) return rc;
            arena = static_cast<uint32_t *>(g.words.ptr);
            return 0;
        }
        // The arena keeps the descriptors' file-order offsets: it is addressed through a pointer shifted back by the
        // block's first word, so nothing is re-based.
        const unsigned long long w_lo = descs[(size_t)F0 * ch].refl_offset;
        const selab200_subframe_desc &tail = descs[(size_t)(F0 + NF) * ch - 1];
        const unsigned long long w_hi = tail.res_offset + tail.res_words;
        if (int rc = g.words.ensure((size_t)(w_hi - w_lo) * 4 + 96)) return rc;
        // 16 bytes of slack in front (the Rice decoder reads whole 16-byte vectors), the 16-byte phase of file order kept
        arena = reinterpret_cast<uint32_t *>(static_cast<char *>(g.words.ptr) + 16 + ((w_lo * 4) & 15)) - w_lo;
        // The primary device holds the whole byte image (uploaded by selab200_container_open, in pieces with events);
        // any other device, and every device for a host-resident image, uploads just the bytes of its block.
        primary = tl_ctx == &g_slots[0] && !h->host;
        d_bytes = static_cast<const uint8_t *>(h->buf.d_bytes);
        if (!primary) {
            const unsigned long long b0 = container_frame_byte(F0, ch, w_lo) & ~3ull; // the unpack kernel reads aligned 32-bit words
            const size_t end = std::min<size_t>(h->n_bytes, (size_t)container_frame_byte(F0 + NF, ch, w_hi) + 4);
            if (int rc = aux_for(end - (size_t)b0 + 64, g.s_h2d)) return rc;
            CUDA_TRY(cudaMemcpyAsync(g.aux.ptr, h->bytes + b0, end - (size_t)b0, cudaMemcpyHostToDevice, g.s_h2d));
            CUDA_TRY(cudaEventRecord(g.ev_h2d[0], g.s_h2d));
            d_bytes = static_cast<const uint8_t *>(g.aux.ptr) - b0;
        }
        return 0;
    }

    // The selection's fetch runs (plan_fetch) go up on s_h2d in one piece per chunk, the runs that start in the chunk,
    // each followed by event g.ev_h2d[c]; a chunk waits for the piece that holds its last run.  Staging is written once
    // per group: decode_pipeline drains before the next group's fetch starts.
    int fetch(const ChunkPlan &plan)
    {
        const uint32_t n_chunks = plan.chunks();
        fetched.assign(n_chunks, -1);
        if (sel->runs.empty())
            return 0;
        if (int rc = g.clip_runs.ensure(sel->runs.size() * sizeof(FetchRun))) return rc;
        const FetchRun *d_runs = static_cast<const FetchRun *>(g.clip_runs.ptr);
        CUDA_TRY(cudaMemcpyAsync(g.clip_runs.ptr, sel->runs.data(), sel->runs.size() * sizeof(FetchRun),
                                 cudaMemcpyHostToDevice, g.s_h2d));
        std::vector<int> piece(sel->runs.size());
        size_t r = 0;
        for (uint32_t c = 0; c < n_chunks; c++) {
            const size_t r0 = r, end = (size_t)plan.start[c + 1] * channels;
            unsigned long long widest = 0;
            for (; r < sel->runs.size() && sel->run_first[r] < end; r++) {
                piece[r] = (int)c;
                widest = std::max(widest, sel->runs[r].bytes);
            }
            if (r == r0)
                continue;
            const unsigned long long per_cta = 16ull * kFetchLoads * 256;
            const unsigned rows = (unsigned)std::min<unsigned long long>(kFetchCtas, (widest + per_cta - 1) / per_cta);
            const unsigned cols = (unsigned)std::min<size_t>(r - r0, std::max(1u, kFetchCtas / rows));
            k_clip_fetch<<<dim3(cols, rows), 256, 0, g.s_h2d>>>(d_runs + r0, (uint32_t)(r - r0));
            if (int rc = launch_check("k_clip_fetch"))
                return rc;
            CUDA_TRY(cudaEventRecord(g.ev_h2d[c], g.s_h2d));
        }
        for (uint32_t c = 0; c < n_chunks; c++) // runs follow selection order: a chunk's last host subframe reads last
            for (size_t i = (size_t)plan.start[c + 1] * channels; i > (size_t)plan.start[c] * channels; i--)
                if (sel->run[i - 1] >= 0) {
                    fetched[c] = piece[(size_t)sel->run[i - 1]];
                    break;
                }
        return 0;
    }

    // Chunk c, frames [f0, f0 + nf): its descriptors to d_descs and its words to the arena, for `lane` to decode.
    int chunk(uint32_t c, uint32_t f0, uint32_t nf, selab200_subframe_desc *d_descs, cudaStream_t lane, const Upload &also)
    {
        const selab200_subframe_desc *dc = descs + (size_t)f0 * channels;
        const size_t n = (size_t)nf * channels;
        // a container's descriptors go up on the chunk's own lane: s_h2d is still busy with the container bytes
        const cudaStream_t carrier = h || sel ? lane : g.s_h2d;
        CUDA_TRY(cudaMemcpyAsync(d_descs, dc, n * sizeof(*dc), cudaMemcpyHostToDevice, carrier));
        if (sel) {
            unsigned long long *d_src = static_cast<unsigned long long *>(g.clip_src.ptr) + (size_t)f0 * channels;
            CUDA_TRY(cudaMemcpyAsync(d_src, sel->src.data() + (size_t)f0 * channels, n * sizeof(unsigned long long),
                                     cudaMemcpyHostToDevice, lane));
            // every device-resident container the chunk reads: the upload piece that holds the last byte it reads
            // there; every host-resident one: the fetch piece that holds its last run
            if (fetched[c] >= 0)
                CUDA_TRY(cudaStreamWaitEvent(lane, g.ev_h2d[fetched[c]], 0));
            for (uint32_t f = f0; f < f0 + nf; f++) {
                const selab200_container *c = sel->frame_h[f];
                if (c->host || (f + 1 < f0 + nf && sel->frame_h[f + 1] == c))
                    continue; // frames of one container are in file order: its last frame here reads furthest
                const int piece = std::min(c->n_pieces - 1, (int)(sel->frame_end[f] / c->piece_bytes));
                CUDA_TRY(cudaStreamWaitEvent(lane, c->buf.ev_piece[piece], 0));
            }
            k_clip_unpack<<<(unsigned)((n + 7) / 8), 256, 0, lane>>>(d_src, d_descs, (uint32_t)n, arena);
            if (int rc = launch_check("k_clip_unpack"))
                return rc;
        } else if (!h) {
            unsigned long long lo, hi;
            words_referenced(dc, n, n_words, lo, hi);
            if (hi > lo)
                CUDA_TRY(cudaMemcpyAsync(arena + lo, words + lo, (hi - lo) * 4, cudaMemcpyHostToDevice, g.s_h2d));
        } else {
            cudaEvent_t uploaded = g.ev_h2d[0];
            if (primary) { // the container bytes this chunk reads end with its last subframe (+3 bytes of slack)
                const selab200_subframe_desc &last = dc[n - 1];
                const unsigned long long end_byte =
                    container_frame_byte(f0 + nf, channels, last.res_offset + last.res_words) + 3;
                uploaded = h->buf.ev_piece[std::min(h->n_pieces - 1, (int)(end_byte / h->piece_bytes))];
            }
            CUDA_TRY(cudaStreamWaitEvent(lane, uploaded, 0));
            k_container_unpack<<<(unsigned)((n + 7) / 8), 256, 0, lane>>>(d_bytes, d_descs, (uint32_t)n, channels,
                                                                           (unsigned long long)f0 * channels, arena);
            if (int rc = launch_check("k_container_unpack"))
                return rc;
        }
        if (also.bytes)
            CUDA_TRY(cudaMemcpyAsync(also.dst, also.src, also.bytes, cudaMemcpyHostToDevice, carrier));
        if (!h && !sel) {
            CUDA_TRY(cudaEventRecord(g.ev_h2d[c], g.s_h2d));
            CUDA_TRY(cudaStreamWaitEvent(lane, g.ev_h2d[c], 0));
        }
        return 0;
    }
};

// A decode of frames [F0, F0 + NF) of `in` that ended in BITSTREAM: if a descriptor there fails the device's own
// descriptor test (desc_ok), the message names the first one, by file frame and channel, so that the error is the same
// however the frames were split into blocks.  A fault inside a Rice stream keeps the plain text, and so does a clip
// selection, whose frames are numbered by the selection rather than by a file.
static int name_malformed(const CodedInput &in, uint32_t F0, uint32_t NF, uint32_t channels, int rc)
{
    if (rc != SELAB200_ERR_BITSTREAM || in.sel)
        return rc;
    for (size_t i = (size_t)F0 * channels; i < (size_t)(F0 + NF) * channels; i++)
        if (!desc_ok(in.descs[i], channels, in.n_words))
            return fail(rc, "%s (the first malformed descriptor: frame %zu, channel %zu)", status_text(rc),
                        i / channels, i % channels);
    return rc;
}

// Frames [F0, F0 + NF) of `in` through the chunk pipeline on the device of the current context.  Without `report`
// the decoded samples come down into pcm_out, or, if pcm_out is null, stay in g.in for the caller (the clip decode);
// with it, each lane compares them on the device with `source` (verify_device) and only the differing pairs come
// back.  pcm_out, source and the report's frames are file-global.
static int decode_pipeline(CodedInput in, uint32_t F0, uint32_t NF, uint32_t channels, int16_t *pcm_out,
                           const int16_t *source, std::vector<selab200_verify_entry> *report)
{
    if (report)
        report->clear();
    if (NF == 0)
        return 0;
    PipelineDrain drain;
    // Every chunk gets its own compute lane (up to kLanes): the Rice kernel is one lane per stream
    // and latency-bound (a fixed time however small the chunk), so the chunks' Rice kernels must
    // overlap each other and the synthesis kernels of earlier chunks rather than queue up.
    const ChunkPlan plan = plan_chunks(NF);
    const uint32_t n_chunks = plan.chunks();
    const size_t n_sub = (size_t)NF * channels;
    const size_t frame_bytes = (size_t)channels * kFrame * 2;
    const size_t ws_bytes = report ? selab200_verify_workspace_bytes(plan.max_frames, channels)
                                   : selab200_decode_workspace_bytes(plan.max_frames, channels);
    if (int rc = g.in.ensure(n_sub * kFrame * 2)) return rc;
    if (int rc = g.descs.ensure(n_sub * sizeof(selab200_subframe_desc))) return rc;
    for (int i = 0; i < kLanes && (uint32_t)i < n_chunks; i++)
        if (int rc = g.lane_work[i].ensure(ws_bytes)) return rc;
    if (int rc = in.start(F0, NF, channels, plan)) return rc;
    int32_t *d_status = &device_counters()->status;
    int16_t *d_pcm = static_cast<int16_t *>(g.in.ptr);
    selab200_subframe_desc *d_descs = static_cast<selab200_subframe_desc *>(g.descs.ptr);
    VerifyArea va;
    if (report) {
        if (int rc = verify_area(n_sub, 0, g.s_compute[0], va)) return rc;
    } else {
        CUDA_TRY(cudaMemsetAsync(d_status, 0, sizeof(int32_t), g.s_compute[0]));
    }
    CUDA_TRY(cudaEventRecord(g.ev_reset, g.s_compute[0]));
    for (int i = 1; i < kLanes; i++)
        CUDA_TRY(cudaStreamWaitEvent(g.s_compute[i], g.ev_reset, 0));
    for (uint32_t c = 0; c < n_chunks; c++) {
        const uint32_t f0 = plan.start[c], nf = plan.start[c + 1] - f0; // within the block
        const size_t at = (size_t)f0 * channels, file_at = (size_t)(F0 + f0) * channels; // the chunk's first subframe
        cudaStream_t cs = g.s_compute[c % kLanes];
        DeviceBuffer &ws = g.lane_work[c % kLanes];
        // verify: the chunk's source PCM goes up with its coded input
        const Upload src = report ? Upload{d_pcm + at * kFrame, source + file_at * kFrame, nf * frame_bytes} : Upload{};
        if (int rc = in.chunk(c, F0 + f0, nf, d_descs + at, cs, src))
            return rc;
        if (report) {
            if (int rc = verify_device(d_descs + at, nf, channels, in.arena, in.n_words, d_pcm + at * kFrame,
                                       va.entries + at, va.count, va.status, ws.ptr, ws.bytes, cs, false, F0 + f0))
                return rc;
            continue;
        }
        if (int rc = decode_device(d_descs + at, nf, channels, in.arena, in.n_words, d_pcm + at * kFrame, d_status,
                                   ws.ptr, ws.bytes, cs, false))
            return rc;
        CUDA_TRY(cudaEventRecord(g.ev_done[c], cs));
        CUDA_TRY(cudaStreamWaitEvent(g.s_d2h, g.ev_done[c], 0));
        if (pcm_out)
            CUDA_TRY(cudaMemcpyAsync(pcm_out + file_at * kFrame, d_pcm + at * kFrame, nf * frame_bytes,
                                     cudaMemcpyDeviceToHost, g.s_d2h));
    }
    if (!report)
        return name_malformed(in, F0, NF, channels, read_status(g.s_d2h, d_status));
    for (int i = 0; i < kLanes && (uint32_t)i < n_chunks; i++)
        CUDA_TRY(cudaStreamSynchronize(g.s_compute[i]));
    return name_malformed(in, F0, NF, channels, collect_records(va.count, va.status, va.entries, n_sub, g.s_d2h, *report));
}

// ---- every initialised device at once ----------------------------------------------------------
//
// Frames are independent (src/sela/encoder.cpp:40-92 hands contiguous ranges of them to its threads); with more
// than one device the host-buffer calls do the same with the devices: device d codes the contiguous block
// frame_block(d) on a worker thread of its own, with its own context (streams, pools), straight from / into
// disjoint ranges of the caller's buffers.  Only the encoder needs a second step: where a block's words land
// depends on the sizes of the blocks before it, so the workers leave the words on their devices and the
// calling thread copies them out (all devices at once) when every size is known, re-basing the descriptors'
// offsets on the way.  The byte-packed container works the same way: a block's body is position independent
// (DESIGN.md 6).
struct DevicePart {
    uint32_t f0 = 0, nf = 0;
    int rc = 0;
    char err[sizeof g_error] = "";
    Result res; // this block's
};

static std::vector<DevicePart> device_parts(uint32_t n_frames)
{
    // n/D frames each, the last device takes the rest: the reference's thread split (src/sela/encoder.cpp:58-73)
    std::vector<DevicePart> parts((size_t)g_n_ctx);
    const uint32_t per = n_frames / (uint32_t)g_n_ctx;
    for (int d = 0; d < g_n_ctx; d++) {
        parts[d].f0 = per * d;
        parts[d].nf = d == g_n_ctx - 1 ? n_frames - per * d : per;
    }
    return parts;
}

static bool use_all_devices(uint32_t n_frames)
{
    return g_n_ctx > 1 && n_frames >= 256u * (uint32_t)g_n_ctx;
}

template <typename F>
static int run_on_devices(std::vector<DevicePart> &parts, F work)
{
    std::vector<std::thread> threads;
    for (int d = 0; d < g_n_ctx; d++)
        threads.emplace_back([&, d] {
            tl_ctx = &g_slots[d];
            DevicePart &p = parts[d];
            cudaError_t e = cudaSetDevice(g.device);
            p.rc = e == cudaSuccess ? work(p) : fail(SELAB200_ERR_CUDA, "cudaSetDevice(%d) failed: %s", g.device, cudaGetErrorString(e));
            if (p.rc)
                memcpy(p.err, g_error, sizeof p.err);
        });
    for (std::thread &t : threads)
        t.join();
    tl_ctx = &g_slots[0];
    cudaSetDevice(g.device);
    for (const DevicePart &p : parts)
        if (p.rc) {
            memcpy(g_error, p.err, sizeof g_error);
            return p.rc;
        }
    return 0;
}

// What run_blocks did: its blocks, and their results summed, the lists one after the other.  Blocks are contiguous
// and in frame order, so the joined lists are in order too.
struct Blocks {
    int rc = 0;
    std::vector<DevicePart> parts;
    Result total;
};

// Runs work(block) over frames [0, n_frames) of a host-buffer call: as one block on the primary context, or, with
// enough frames for several devices (use_all_devices), as one block per device, each on its own worker thread.
template <typename F>
static Blocks run_blocks(uint32_t n_frames, F work)
{
    Blocks b;
    if (use_all_devices(n_frames)) {
        b.parts = device_parts(n_frames);
        b.rc = run_on_devices(b.parts, work);
    } else {
        b.parts.resize(1);
        b.parts[0].nf = n_frames;
        b.rc = work(b.parts[0]);
    }
    for (const DevicePart &p : b.parts)
        b.total.add(p.res);
    return b;
}

// The encoder's second step with several devices: every device's block (left on the device, EncodeTarget::defer)
// goes out once the sizes of all blocks are known, and the descriptors' offsets are re-based to file order.
static int place_blocks(const std::vector<DevicePart> &parts, uint32_t channels, const EncodeTarget &t, size_t total)
{
    if (total > t.words_capacity)
        return fail(SELAB200_ERR_CAPACITY, "%s", status_text(SELAB200_ERR_CAPACITY));
    const bool to_container = t.form == EncodeForm::container;
    size_t base = 0;
    for (int d = 0; d < g_n_ctx; d++) { // every device's block goes out at once, each over its own link
        tl_ctx = &g_slots[d];
        const DevicePart &p = parts[d];
        CUDA_TRY(cudaSetDevice(g.device));
        if (to_container) {
            const size_t body = (size_t)container_frame_byte(p.nf, channels, p.res.words) - kContainerHeaderBytes;
            const size_t at = (size_t)container_frame_byte(p.f0, channels, base);
            if (body)
                CUDA_TRY(cudaMemcpyAsync(t.container + at, static_cast<uint8_t *>(g.words.ptr) + kContainerHeaderBytes, body,
                                         cudaMemcpyDeviceToHost, g.s_d2h));
        } else if (p.res.words) {
            CUDA_TRY(cudaMemcpyAsync(t.words + base, g.words.ptr, p.res.words * 4, cudaMemcpyDeviceToHost, g.s_d2h));
        }
        base += p.res.words;
    }
    if (!to_container) { // meanwhile: descriptor offsets from block-local to file order
        size_t b = 0;
        for (const DevicePart &p : parts) {
            if (b)
                for (size_t i = (size_t)p.f0 * channels; i < (size_t)(p.f0 + p.nf) * channels; i++) {
                    t.descs[i].refl_offset += b;
                    t.descs[i].res_offset += b;
                }
            b += p.res.words;
        }
    }
    int rc2 = 0;
    for (int d = 0; d < g_n_ctx; d++) {
        tl_ctx = &g_slots[d];
        cudaSetDevice(g.device);
        cudaError_t e = cudaStreamSynchronize(g.s_d2h);
        if (e != cudaSuccess && !rc2)
            rc2 = fail(SELAB200_ERR_CUDA, "download from device %d failed: %s", g.device, cudaGetErrorString(e));
    }
    tl_ctx = &g_slots[0];
    cudaSetDevice(g.device);
    return rc2;
}

// Every host-buffer encode: encode_host on each block of run_blocks, then, with several blocks, place_blocks.  r: the
// results of all blocks.  arg: the mode's parameter (encode_host).
static int encode_blocks(const int16_t *pcm, uint32_t n_frames, uint32_t channels, const EncodeTarget &t,
                         EncodeMode mode, Result &r, uint32_t arg = 0)
{
    const bool split = use_all_devices(n_frames);
    const size_t per_frame = (size_t)channels * kFrame;
    Blocks b = run_blocks(n_frames, [&](DevicePart &p) {
        EncodeTarget block = t;
        if (split) { // the block stays on its device; its words are counted from its own start
            block.defer = true;
            block.descs = t.descs ? t.descs + (size_t)p.f0 * channels : nullptr;
            block.words = nullptr;
            block.container = nullptr;
            block.words_capacity = selab200_encode_words_bound(p.nf, channels);
        }
        return encode_host(pcm + p.f0 * per_frame, p.nf, channels, block, mode, arg, p.f0, p.res);
    });
    r = std::move(b.total);
    if (b.rc || !split)
        return b.rc;
    return place_blocks(b.parts, channels, t, r.words);
}

extern "C" {

int selab200_encode_frames(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                           selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                           size_t *words_used)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!pcm || !descs || !words || !words_used)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    Result r;
    const int rc = encode_blocks(pcm, n_frames, channels, EncodeTarget{EncodeForm::arena, false, descs, words, nullptr,
                                                                       words_capacity}, EncodeMode::plain, r);
    *words_used = r.words;
    return rc;
}

int selab200_encode_frames_lossless(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                    selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                    size_t *words_used, selab200_lossless_entry *entries, size_t capacity,
                                    size_t *n_entries)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!pcm || !descs || !words || !words_used || (!entries && capacity) || !n_entries)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    *n_entries = 0;
    Result r;
    const int rc = encode_blocks(pcm, n_frames, channels, EncodeTarget{EncodeForm::arena, false, descs, words, nullptr,
                                                                       words_capacity}, EncodeMode::lossless, r);
    *words_used = r.words;
    return rc ? rc : deliver_records(r.recoded, entries, capacity, n_entries);
}

int selab200_encode_frames_search(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                  selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                  size_t *words_used, size_t *ref_words)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!pcm || !descs || !words || !words_used || !ref_words)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    Result r;
    const int rc = encode_blocks(pcm, n_frames, channels, EncodeTarget{EncodeForm::arena, false, descs, words, nullptr,
                                                                       words_capacity}, EncodeMode::search, r);
    *words_used = r.words;
    *ref_words = (size_t)r.ref_words;
    return rc;
}

int selab200_encode_frames_pairing(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                   selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                   size_t *words_used, size_t *base_words, size_t *n_difference)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!pcm || !descs || !words || !words_used || !base_words || !n_difference)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    Result r;
    const int rc = encode_blocks(pcm, n_frames, channels, EncodeTarget{EncodeForm::arena, false, descs, words, nullptr,
                                                                       words_capacity}, EncodeMode::pairing, r);
    *words_used = r.words;
    *base_words = (size_t)r.base_words;
    *n_difference = (size_t)r.n_difference;
    return rc;
}

int selab200_encode_frames_search_pairing(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                          selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                          size_t *words_used, size_t *base_words, size_t *n_difference)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!pcm || !descs || !words || !words_used || !base_words || !n_difference)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    Result r;
    const int rc = encode_blocks(pcm, n_frames, channels, EncodeTarget{EncodeForm::arena, false, descs, words, nullptr,
                                                                       words_capacity}, EncodeMode::search_pairing, r);
    *words_used = r.words;
    *base_words = (size_t)r.base_words;
    *n_difference = (size_t)r.n_difference;
    return rc;
}

int selab200_encode_frames_search_windows(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t windows,
                                         selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                         size_t *words_used, size_t *base_words, size_t *n_window)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!pcm || !descs || !words || !words_used || !base_words || !n_window)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    if (int rc = check_windows(windows))
        return rc;
    Result r;
    const int rc = encode_blocks(pcm, n_frames, channels, EncodeTarget{EncodeForm::arena, false, descs, words, nullptr,
                                                                       words_capacity}, EncodeMode::search_windows, r,
                                 windows);
    *words_used = r.words;
    *base_words = (size_t)r.base_words;
    *n_window = (size_t)r.n_window;
    return rc;
}

int selab200_encode_frames_search_guided(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t candidates,
                                        selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                        size_t *words_used, size_t *ref_words)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!pcm || !descs || !words || !words_used || !ref_words)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    if (int rc = check_candidates(candidates))
        return rc;
    Result r;
    const int rc = encode_blocks(pcm, n_frames, channels, EncodeTarget{EncodeForm::arena, false, descs, words, nullptr,
                                                                       words_capacity}, EncodeMode::search_guided, r,
                                 candidates);
    *words_used = r.words;
    *ref_words = (size_t)r.ref_words;
    return rc;
}

size_t selab200_container_bound(uint32_t n_frames, uint32_t channels)
{
    return (size_t)container_frame_byte(n_frames, channels, selab200_encode_words_bound(n_frames, channels));
}

} // extern "C"

// selab200_encode_container in every mode, and with `verify` its verified form (g_mutex held by the caller).
static int encode_container_impl(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t sample_rate,
                                 uint16_t bits_per_sample, uint8_t *container, size_t capacity, size_t *bytes_used,
                                 EncodeMode mode, bool verify, Result &r, uint32_t arg = 0)
{
    if (int rc = require_ready())
        return rc;
    if ((!pcm && n_frames) || !container || !bytes_used)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    const unsigned long long fixed = container_frame_byte(n_frames, channels, 0);
    *bytes_used = (size_t)fixed;
    if (capacity < fixed)
        return fail(SELAB200_ERR_CAPACITY, "container buffer too small: %zu bytes, need more than %llu", capacity, fixed);
    // file::SelaFile::writeToFile, header part (src/file/sela_file.cpp:107-112)
    const uint8_t header[15] = {'S', 'e', 'L', 'a',
                                (uint8_t)sample_rate, (uint8_t)(sample_rate >> 8), (uint8_t)(sample_rate >> 16), (uint8_t)(sample_rate >> 24),
                                (uint8_t)bits_per_sample, (uint8_t)(bits_per_sample >> 8), (uint8_t)channels,
                                (uint8_t)n_frames, (uint8_t)(n_frames >> 8), (uint8_t)(n_frames >> 16), (uint8_t)(n_frames >> 24)};
    memcpy(container, header, sizeof header);
    const EncodeTarget t{EncodeForm::container, false, nullptr, nullptr, container, (size_t)((capacity - fixed) / 4),
                         verify};
    const int rc = encode_blocks(pcm, n_frames, channels, t, mode, r, arg);
    *bytes_used = (size_t)container_frame_byte(n_frames, channels, r.words);
    r.ref_bytes = (size_t)container_frame_byte(n_frames, channels,
                                               mode == EncodeMode::pairing || mode == EncodeMode::search_pairing ||
                                                       mode == EncodeMode::search_windows
                                                   ? r.base_words
                                                   : r.ref_words);
    return rc;
}

extern "C" {

int selab200_encode_container(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t sample_rate,
                              uint16_t bits_per_sample, uint8_t *container, size_t capacity, size_t *bytes_used)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    Result r;
    return encode_container_impl(pcm, n_frames, channels, sample_rate, bits_per_sample, container, capacity, bytes_used,
                                 EncodeMode::plain, false, r);
}

int selab200_encode_container_verified(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t sample_rate,
                                       uint16_t bits_per_sample, uint8_t *container, size_t capacity, size_t *bytes_used,
                                       selab200_verify_entry *entries, size_t entries_capacity, size_t *n_entries)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!n_entries || (!entries && entries_capacity)) {
        if (int rc = require_ready())
            return rc;
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    }
    *n_entries = 0;
    Result r;
    if (int rc = encode_container_impl(pcm, n_frames, channels, sample_rate, bits_per_sample, container, capacity,
                                       bytes_used, EncodeMode::plain, true, r))
        return rc;
    return deliver_records(r.report, entries, entries_capacity, n_entries);
}

int selab200_encode_container_lossless(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t sample_rate,
                                       uint16_t bits_per_sample, uint8_t *container, size_t capacity, size_t *bytes_used,
                                       selab200_lossless_entry *entries, size_t entries_capacity, size_t *n_entries)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!n_entries || (!entries && entries_capacity)) {
        if (int rc = require_ready())
            return rc;
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    }
    *n_entries = 0;
    Result r;
    if (int rc = encode_container_impl(pcm, n_frames, channels, sample_rate, bits_per_sample, container, capacity,
                                       bytes_used, EncodeMode::lossless, false, r))
        return rc;
    return deliver_records(r.recoded, entries, entries_capacity, n_entries);
}

int selab200_encode_container_search(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t sample_rate,
                                     uint16_t bits_per_sample, uint8_t *container, size_t capacity, size_t *bytes_used,
                                     size_t *ref_bytes)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!ref_bytes) {
        if (int rc = require_ready())
            return rc;
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    }
    Result r;
    const int rc = encode_container_impl(pcm, n_frames, channels, sample_rate, bits_per_sample, container, capacity,
                                         bytes_used, EncodeMode::search, false, r);
    *ref_bytes = r.ref_bytes;
    return rc;
}

int selab200_encode_container_pairing(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t sample_rate,
                                      uint16_t bits_per_sample, uint8_t *container, size_t capacity, size_t *bytes_used,
                                      size_t *base_bytes, size_t *n_difference)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!base_bytes || !n_difference) {
        if (int rc = require_ready())
            return rc;
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    }
    Result r;
    const int rc = encode_container_impl(pcm, n_frames, channels, sample_rate, bits_per_sample, container, capacity,
                                         bytes_used, EncodeMode::pairing, false, r);
    *base_bytes = r.ref_bytes;
    *n_difference = (size_t)r.n_difference;
    return rc;
}

int selab200_encode_container_search_pairing(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                             uint32_t sample_rate, uint16_t bits_per_sample, uint8_t *container,
                                             size_t capacity, size_t *bytes_used, size_t *base_bytes,
                                             size_t *n_difference)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!base_bytes || !n_difference) {
        if (int rc = require_ready())
            return rc;
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    }
    Result r;
    const int rc = encode_container_impl(pcm, n_frames, channels, sample_rate, bits_per_sample, container, capacity,
                                         bytes_used, EncodeMode::search_pairing, false, r);
    *base_bytes = r.ref_bytes;
    *n_difference = (size_t)r.n_difference;
    return rc;
}

int selab200_encode_container_search_windows(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                            uint32_t windows, uint32_t sample_rate, uint16_t bits_per_sample,
                                            uint8_t *container, size_t capacity, size_t *bytes_used,
                                            size_t *base_bytes, size_t *n_window)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!base_bytes || !n_window) {
        if (int rc = require_ready())
            return rc;
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    }
    if (int rc = check_windows(windows))
        return rc;
    Result r;
    const int rc = encode_container_impl(pcm, n_frames, channels, sample_rate, bits_per_sample, container, capacity,
                                         bytes_used, EncodeMode::search_windows, false, r, windows);
    *base_bytes = r.ref_bytes;
    *n_window = (size_t)r.n_window;
    return rc;
}

int selab200_encode_container_search_guided(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                           uint32_t candidates, uint32_t sample_rate, uint16_t bits_per_sample,
                                           uint8_t *container, size_t capacity, size_t *bytes_used, size_t *ref_bytes)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!ref_bytes) {
        if (int rc = require_ready())
            return rc;
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    }
    if (int rc = check_candidates(candidates))
        return rc;
    Result r;
    const int rc = encode_container_impl(pcm, n_frames, channels, sample_rate, bits_per_sample, container, capacity,
                                         bytes_used, EncodeMode::search_guided, false, r, candidates);
    *ref_bytes = r.ref_bytes;
    return rc;
}

int selab200_decode_frames(const selab200_subframe_desc *descs, uint32_t n_frames, uint32_t channels,
                           const uint32_t *words, size_t n_words, int16_t *pcm_out)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!descs || !pcm_out || (!words && n_words))
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    const CodedInput in{descs, words, n_words, nullptr};
    return run_blocks(n_frames, [&](DevicePart &p) {
        return decode_pipeline(in, p.f0, p.nf, channels, pcm_out, nullptr, nullptr);
    }).rc;
}

int selab200_verify_frames(const selab200_subframe_desc *descs, uint32_t n_frames, uint32_t channels,
                           const uint32_t *words, size_t n_words, const int16_t *pcm, selab200_verify_entry *entries,
                           size_t capacity, size_t *n_entries)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (((!descs || !pcm) && n_frames) || (!words && n_words) || (!entries && capacity) || !n_entries)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    *n_entries = 0;
    const CodedInput in{descs, words, n_words, nullptr};
    const Blocks b = run_blocks(n_frames, [&](DevicePart &p) {
        return decode_pipeline(in, p.f0, p.nf, channels, nullptr, pcm, &p.res.report);
    });
    if (b.rc)
        return b.rc;
    return deliver_records(b.total.report, entries, capacity, n_entries);
}

// ---- .sela container, decode side ----------------------------------------------------------

} // extern "C"

namespace {

// file::SelaFile::readFromFile (src/file/sela_file.cpp:19-103) without the copies: validates the
// header, then hops from frame to frame.  With `descs` it also emits one descriptor per subframe,
// arena offsets assigned in file order.  Messages match the host mirror's reader.
int walk_container(const uint8_t *b, size_t n, selab200_container_info *info,
                   std::vector<selab200_subframe_desc> *descs, uint64_t *frame_bytes = nullptr,
                   size_t frame_capacity = 0)
{
    memset(info, 0, sizeof *info);
    if (n < 15)
        return fail(SELAB200_ERR_BITSTREAM, "File is too small, probably not a sela file.");
    if (memcmp(b, "SeLa", 4) != 0)
        return fail(SELAB200_ERR_BITSTREAM, "Magic number is incorrect, probably not a sela file.");
    auto u16 = [&](size_t o) { return (uint32_t)b[o] | ((uint32_t)b[o + 1] << 8); };
    auto u32 = [&](size_t o) { return u16(o) | (u16(o + 2) << 16); };
    info->sample_rate = u32(4);
    info->bits_per_sample = (uint16_t)u16(8);
    info->channels = b[10];
    info->header_frames = u32(11);
    const uint32_t channels = info->channels;
    size_t at = 15;
    unsigned long long words = 0;
    uint32_t f = 0;
    for (; f < info->header_frames; f++) {
        if (at + 4 > n || u32(at) != 0xAA55FF00u)
            break;
        if (frame_bytes && f < frame_capacity)
            frame_bytes[f] = at;
        at += 4;
        for (uint32_t c = 0; c < channels; c++) {
            if (at + 7 > n)
                return fail(SELAB200_ERR_BITSTREAM, "sela file is truncated");
            const uint32_t refl_words = u16(at + 4);
            const size_t at2 = at + 7 + 4 * (size_t)refl_words;
            if (at2 + 5 > n)
                return fail(SELAB200_ERR_BITSTREAM, "sela file is truncated");
            const uint32_t res_words = u16(at2 + 1);
            if (at2 + 5 + 4 * (size_t)res_words > n)
                return fail(SELAB200_ERR_BITSTREAM, "sela file is truncated");
            if (descs) {
                selab200_subframe_desc d;
                d.channel = b[at];
                d.subframe_type = b[at + 1];
                d.parent_channel = b[at + 2];
                d.refl_rice_param = b[at + 3];
                d.refl_words = (uint16_t)refl_words;
                d.lpc_order = b[at + 6];
                d.res_rice_param = b[at2];
                d.res_words = (uint16_t)res_words;
                d.samples = (uint16_t)u16(at2 + 3);
                d.reserved = 0;
                d.refl_offset = words;
                d.res_offset = words + refl_words;
                descs->push_back(d);
            }
            words += refl_words + res_words;
            at = at2 + 5 + 4 * (size_t)res_words;
        }
    }
    info->n_frames = f;
    info->n_words = words;
    info->n_bytes_used = at;
    if (frame_bytes && f < frame_capacity)
        frame_bytes[f] = at;
    return 0;
}

} // namespace

// ---- clip decode (DESIGN.md 7.8) --------------------------------------------------------------------------------
//
// The selection -- every (container, frame) some clip covers, sorted and deduplicated -- is cut into groups of at most
// clip_group_frames() frames.  Each group goes through decode_pipeline as a ClipSelection and stays decoded in g.in
// until the pieces of the clips that fall in it are cut out (k_clip_gather), so the call's device memory is bounded by
// a group and a gather batch whatever the number of clips.  A clip's frames are consecutive in the selection, so a
// clip is one run of decoded rows, split only where a group ends.
constexpr uint32_t kClipGroupSubframes = 32768;
constexpr size_t kClipPieceBatch = 65536;              // pieces per gather launch (the device piece table)
constexpr size_t kClipStagingBytes = (size_t)64 << 20; // host form: output bytes per gather launch

// Frames per group; with SELAB200_CHUNK_FRAMES (tests, tuning) four chunks of that size.
static uint32_t clip_group_frames(uint32_t channels)
{
    if (const char *env = std::getenv("SELAB200_CHUNK_FRAMES")) {
        const long v = std::atol(env);
        if (v > 0)
            return (uint32_t)std::min<long>(4 * v, 1l << 20);
    }
    return std::max<uint32_t>(1, kClipGroupSubframes / channels);
}

// Bytes of host-resident images the last clip call fetched (selab200_clip_bytes_fetched); g_mutex guards it.
static uint64_t g_clip_bytes_fetched = 0;

// The fetch runs of one group (DESIGN.md 7.10).  Each host-resident subframe reads the bytes [at, end) of its image,
// from its reflection words to 3 bytes past its residue words (what get_words_at_byte touches); rounded out to
// [at & ~15, (end + 15) & ~15), the ranges of one container that touch or overlap, taken in selection order, merge
// into one run.  Runs are staged back to back in g.clip_stage, so a run keeps its 16-byte phase, and each such
// subframe's src is re-pointed into its run's staging.  Host images are page-aligned, so file offsets and mapped
// addresses have the same 16-byte phase.
static int plan_fetch(ClipSelection &sel, uint32_t channels)
{
    sel.runs.clear();
    sel.run_first.clear();
    sel.run.assign(sel.src.size(), -1);
    std::vector<const selab200_container *> run_h;
    unsigned long long staged = 0;
    for (size_t i = 0; i < sel.src.size(); i++) {
        const selab200_container *h = sel.frame_h[i / channels];
        if (!h->host)
            continue;
        const selab200_subframe_desc &d = sel.descs[i];
        const unsigned long long lo = sel.at[i] & ~15ull;
        const unsigned long long hi = (sel.at[i] + 4ull * d.refl_words + 5 + 4ull * d.res_words + 3 + 15) & ~15ull;
        // runs hold file offsets (src) and staging offsets (dst) until the staging buffer is placed
        FetchRun *last = sel.runs.empty() ? nullptr : &sel.runs.back();
        if (last && run_h.back() == h && lo <= last->src + last->bytes) {
            if (hi > last->src + last->bytes) {
                staged += hi - (last->src + last->bytes);
                last->bytes = hi - last->src;
            }
        } else {
            sel.runs.push_back(FetchRun{lo, staged, hi - lo});
            sel.run_first.push_back(i);
            run_h.push_back(h);
            staged += hi - lo;
        }
        sel.run[i] = (int64_t)sel.runs.size() - 1;
    }
    if (sel.runs.empty())
        return 0;
    g_clip_bytes_fetched += staged;
    if (int rc = g.clip_stage.ensure(staged)) return rc;
    const unsigned long long stage = reinterpret_cast<unsigned long long>(g.clip_stage.ptr);
    for (size_t i = 0; i < sel.src.size(); i++)
        if (sel.run[i] >= 0) {
            const FetchRun &r = sel.runs[(size_t)sel.run[i]];
            sel.src[i] = stage + r.dst + (sel.at[i] - r.src);
        }
    for (size_t r = 0; r < sel.runs.size(); r++) {
        sel.runs[r].src += reinterpret_cast<unsigned long long>(run_h[r]->mapped);
        sel.runs[r].dst += stage;
    }
    return 0;
}

// The pieces of one group, in output order, out of g.in into `out` (device form) or, through the staging buffer
// g.clip_out, into host memory.  On g.s_d2h; returns when every piece is written.
static int clip_gather(const std::vector<ClipPiece> &pieces, uint8_t *out, bool device_out)
{
    const cudaStream_t s = g.s_d2h;
    if (int rc = g.clip_pieces.ensure(kClipPieceBatch * sizeof(ClipPiece))) return rc;
    if (!device_out)
        if (int rc = g.clip_out.ensure(kClipStagingBytes)) return rc;
    uint8_t *staging = static_cast<uint8_t *>(g.clip_out.ptr);
    std::vector<ClipPiece> batch, copies; // copies (host form): staging offset, host offset, bytes
    size_t i = 0;
    unsigned long long done = 0; // bytes of pieces[i] already gathered (host form: a piece may span batches)
    while (i < pieces.size()) {
        batch.clear();
        copies.clear();
        unsigned long long staged = 0, widest = 0;
        while (i < pieces.size() && batch.size() < kClipPieceBatch) {
            const ClipPiece &p = pieces[i];
            unsigned long long take = p.bytes - done;
            if (!device_out) {
                if (staged == kClipStagingBytes)
                    break;
                take = std::min<unsigned long long>(take, kClipStagingBytes - staged);
                if (!copies.empty() && copies.back().dst + copies.back().bytes == p.dst + done)
                    copies.back().bytes += take;
                else
                    copies.push_back(ClipPiece{staged, p.dst + done, take});
            }
            batch.push_back(ClipPiece{p.src + done, device_out ? p.dst + done : staged, take});
            staged += take;
            widest = std::max(widest, take);
            done += take;
            if (done == p.bytes) {
                i++;
                done = 0;
            }
        }
        const unsigned rows = (unsigned)std::min<unsigned long long>(64, std::max(1ull, (widest / 16 + 255) / 256));
        CUDA_TRY(cudaMemcpyAsync(g.clip_pieces.ptr, batch.data(), batch.size() * sizeof(ClipPiece),
                                 cudaMemcpyHostToDevice, s));
        k_clip_gather<<<dim3((unsigned)batch.size(), rows), 256, 0, s>>>(
            static_cast<const uint8_t *>(g.in.ptr), device_out ? out : staging,
            static_cast<const ClipPiece *>(g.clip_pieces.ptr));
        if (int rc = launch_check("k_clip_gather"))
            return rc;
        for (const ClipPiece &c : copies)
            CUDA_TRY(cudaMemcpyAsync(out + c.dst, staging + c.src, c.bytes, cudaMemcpyDeviceToHost, s));
    }
    CUDA_TRY(cudaStreamSynchronize(s));
    return 0;
}

// Both forms of selab200_container_decode_clips, on the primary context (require_ready done, g_mutex held).
static int decode_clips(selab200_container *const *handles, uint32_t n_handles, const selab200_clip *clips,
                        uint32_t n_clips, uint32_t length, uint8_t *out, bool device_out, uint64_t *frames_decoded)
{
    g_clip_bytes_fetched = 0;
    if (!frames_decoded)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    *frames_decoded = 0;
    if (n_clips == 0)
        return 0;
    if (!handles || !clips || !out)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (length == 0)
        return fail(SELAB200_ERR_ARGUMENT, "clip 0: length must be at least 1");
    for (uint32_t i = 0; i < n_handles; i++) {
        if (!handles[i])
            return fail(SELAB200_ERR_ARGUMENT, "handles[%u] is null", i);
        if (handles[i]->info.channels != handles[0]->info.channels)
            return fail(SELAB200_ERR_ARGUMENT, "handles[%u] has %u channels, handles[0] %u", i,
                        (unsigned)handles[i]->info.channels, (unsigned)handles[0]->info.channels);
    }
    for (uint32_t i = 0; i < n_clips; i++) {
        const selab200_clip &c = clips[i];
        if (c.container >= n_handles)
            return fail(SELAB200_ERR_ARGUMENT, "clip %u: container %u, but %u handles", i, c.container, n_handles);
        if (c.reserved != 0)
            return fail(SELAB200_ERR_ARGUMENT, "clip %u: reserved field is not 0", i);
        const unsigned long long total = (unsigned long long)handles[c.container]->info.n_frames * kFrame;
        if (c.start > total || length > total - c.start)
            return fail(SELAB200_ERR_ARGUMENT, "clip %u: samples [%llu, %llu + %u) outside the %llu samples of its container",
                        i, (unsigned long long)c.start, (unsigned long long)c.start, length, total);
    }
    const uint32_t C = handles[0]->info.channels;
    if (int rc = check_channels(C))
        return rc;
    const unsigned long long clip_bytes = (unsigned long long)length * C * 2;
    if (clip_bytes > ~0ull / n_clips)
        return fail(SELAB200_ERR_ARGUMENT, "output of %u clips of %u samples does not fit 64 bits", n_clips, length);

    // the selection: (container << 32 | frame), sorted and deduplicated
    std::vector<unsigned long long> keys;
    for (uint32_t i = 0; i < n_clips; i++) {
        const unsigned long long f0 = clips[i].start / kFrame, f1 = (clips[i].start + length - 1) / kFrame;
        for (unsigned long long f = f0; f <= f1; f++)
            keys.push_back((unsigned long long)clips[i].container << 32 | f);
    }
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    *frames_decoded = keys.size();

    // every clip as rows [r0, r0 + length) of the selection decoded back to back, cut at group ends
    const unsigned long long group_rows = (unsigned long long)clip_group_frames(C) * kFrame;
    const size_t n_groups = (keys.size() * kFrame + group_rows - 1) / group_rows;
    std::vector<std::vector<ClipPiece>> pieces(n_groups);
    for (uint32_t i = 0; i < n_clips; i++) {
        const unsigned long long key = (unsigned long long)clips[i].container << 32 | clips[i].start / kFrame;
        const unsigned long long k = (unsigned long long)(std::lower_bound(keys.begin(), keys.end(), key) - keys.begin());
        const unsigned long long r0 = k * kFrame + clips[i].start % kFrame, r1 = r0 + length;
        for (unsigned long long grp = r0 / group_rows; grp <= (r1 - 1) / group_rows; grp++) {
            const unsigned long long lo = std::max(r0, grp * group_rows), hi = std::min(r1, (grp + 1) * group_rows);
            pieces[grp].push_back(ClipPiece{(lo - grp * group_rows) * C * 2, i * clip_bytes + (lo - r0) * C * 2,
                                            (hi - lo) * C * 2});
        }
    }

    ClipSelection sel;
    for (size_t grp = 0; grp < n_groups; grp++) {
        const size_t s0 = grp * (size_t)(group_rows / kFrame), s1 = std::min(keys.size(), s0 + (size_t)(group_rows / kFrame));
        const uint32_t nf = (uint32_t)(s1 - s0);
        sel.descs.resize((size_t)nf * C);
        sel.src.resize((size_t)nf * C);
        sel.at.resize((size_t)nf * C);
        sel.frame_h.resize(nf);
        sel.frame_end.resize(nf);
        unsigned long long words = 0;
        for (uint32_t s = 0; s < nf; s++) {
            const selab200_container *h = handles[keys[s0 + s] >> 32];
            const unsigned long long f = keys[s0 + s] & 0xffffffffull;
            const unsigned long long image = reinterpret_cast<unsigned long long>(h->buf.d_bytes);
            for (uint32_t c = 0; c < C; c++) {
                selab200_subframe_desc d = h->buf.h_descs[f * C + c];
                const unsigned long long at = container_frame_byte(f, C, d.refl_offset) + 4 + (unsigned long long)kSubframeHeaderBytes * c + 7;
                sel.src[(size_t)s * C + c] = image + at;
                sel.at[(size_t)s * C + c] = at;
                sel.frame_end[s] = at + 4ull * d.refl_words + 5 + 4ull * d.res_words + 3;
                d.refl_offset = words;
                d.res_offset = words + d.refl_words;
                words += (unsigned long long)d.refl_words + d.res_words;
                sel.descs[(size_t)s * C + c] = d;
            }
            sel.frame_h[s] = h;
        }
        if (int rc = plan_fetch(sel, C))
            return rc;
        CodedInput in{sel.descs.data(), nullptr, (size_t)words, nullptr, &sel};
        if (int rc = decode_pipeline(in, 0, nf, C, nullptr, nullptr, nullptr))
            return rc;
        if (int rc = clip_gather(pieces[grp], out, device_out))
            return rc;
    }
    return 0;
}

// ---- channel-selecting clip decode (DESIGN.md 7.9) ---------------------------------------------------------------
//
// The selection of decode_clips, flattened: every subframe a covered frame needs -- its selected channels and the
// parents of the selected difference-coded ones -- becomes one mono frame of a ClipSelection, in file order, with
// channel, type and parent 0.  decode_pipeline decodes a group of them with channels = 1 into [n][2048] int16 rows (an
// independent subframe's samples, a difference subframe's difference, both mod 2^16 as in the full decode), and
// k_clip_gather_select cuts the clips out of the rows through a row table: per covered frame and selected channel the
// row of its subframe and, for a difference-coded one, the row of its parent.  A frame's subframes stay in one group.

// The pieces of one group out of g.in into `out` (device form) or, through the staging buffer g.clip_out, into host
// memory; pieces are never split (one is at most 2048 * 255 * 4 bytes).  On g.s_d2h; returns when all are written.
template <typename OUT, bool MEAN>
static int clip_gather_select(const std::vector<SelectPiece> &pieces, const std::vector<uint2> &table, uint8_t *out,
                              bool device_out)
{
    const cudaStream_t s = g.s_d2h;
    if (int rc = g.clip_pieces.ensure(kClipPieceBatch * sizeof(SelectPiece))) return rc;
    if (int rc = g.clip_rows.ensure(table.size() * sizeof(uint2))) return rc;
    if (!device_out)
        if (int rc = g.clip_out.ensure(kClipStagingBytes)) return rc;
    CUDA_TRY(cudaMemcpyAsync(g.clip_rows.ptr, table.data(), table.size() * sizeof(uint2), cudaMemcpyHostToDevice, s));
    uint8_t *staging = static_cast<uint8_t *>(g.clip_out.ptr);
    std::vector<SelectPiece> batch;
    std::vector<ClipPiece> copies; // host form: staging offset, host offset, bytes
    for (size_t i = 0; i < pieces.size();) {
        batch.clear();
        copies.clear();
        unsigned long long staged = 0;
        for (; i < pieces.size() && batch.size() < kClipPieceBatch; i++) {
            SelectPiece p = pieces[i];
            if (!device_out) {
                const unsigned long long bytes = (unsigned long long)p.count * (MEAN ? 1 : p.n) * sizeof(OUT);
                if (staged + bytes > kClipStagingBytes)
                    break;
                if (!copies.empty() && copies.back().dst + copies.back().bytes == p.dst)
                    copies.back().bytes += bytes;
                else
                    copies.push_back(ClipPiece{staged, p.dst, bytes});
                p.dst = staged;
                staged += bytes;
            }
            batch.push_back(p);
        }
        CUDA_TRY(cudaMemcpyAsync(g.clip_pieces.ptr, batch.data(), batch.size() * sizeof(SelectPiece),
                                 cudaMemcpyHostToDevice, s));
        k_clip_gather_select<OUT, MEAN><<<(unsigned)batch.size(), 256, 0, s>>>(
            static_cast<const int16_t *>(g.in.ptr), static_cast<const uint2 *>(g.clip_rows.ptr),
            device_out ? out : staging, static_cast<const SelectPiece *>(g.clip_pieces.ptr));
        if (int rc = launch_check("k_clip_gather_select"))
            return rc;
        for (const ClipPiece &c : copies)
            CUDA_TRY(cudaMemcpyAsync(out + c.dst, staging + c.src, c.bytes, cudaMemcpyDeviceToHost, s));
    }
    CUDA_TRY(cudaStreamSynchronize(s));
    return 0;
}

// Both forms of selab200_container_decode_clips_select, on the primary context (require_ready done, g_mutex held).
static int decode_clips_select(selab200_container *const *handles, uint32_t n_handles, const selab200_clip *clips,
                               uint32_t n_clips, uint32_t length, const uint8_t *select, uint32_t n_select,
                               uint32_t flags, uint8_t *out, bool device_out, uint64_t *frames_decoded,
                               uint64_t *subframes_decoded)
{
    g_clip_bytes_fetched = 0;
    if (!frames_decoded || !subframes_decoded)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    *frames_decoded = 0;
    *subframes_decoded = 0;
    if (flags & ~(SELAB200_CLIP_FLOAT32 | SELAB200_CLIP_MEAN))
        return fail(SELAB200_ERR_ARGUMENT, "unknown flag bits 0x%x", flags & ~(SELAB200_CLIP_FLOAT32 | SELAB200_CLIP_MEAN));
    const bool f32 = flags & SELAB200_CLIP_FLOAT32, mean = flags & SELAB200_CLIP_MEAN;
    if (mean && !f32)
        return fail(SELAB200_ERR_ARGUMENT, "SELAB200_CLIP_MEAN needs SELAB200_CLIP_FLOAT32");
    if (!select && n_select)
        return fail(SELAB200_ERR_ARGUMENT, "select is null but n_select is %u", n_select);
    if (select && !n_select)
        return fail(SELAB200_ERR_ARGUMENT, "n_select is 0 but select is not null");
    if (n_select > SELAB200_CLIP_MAX_SELECT)
        return fail(SELAB200_ERR_ARGUMENT, "n_select is %u, more than %u", n_select, SELAB200_CLIP_MAX_SELECT);
    if (n_clips == 0)
        return 0;
    if (!handles || !clips || !out)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (length == 0)
        return fail(SELAB200_ERR_ARGUMENT, "clip 0: length must be at least 1");
    for (uint32_t i = 0; i < n_handles; i++)
        if (!handles[i])
            return fail(SELAB200_ERR_ARGUMENT, "handles[%u] is null", i);
    uint32_t top = 0; // the highest channel selected
    for (uint32_t j = 0; j < n_select; j++)
        top = std::max<uint32_t>(top, select[j]);
    for (uint32_t i = 0; i < n_clips; i++) {
        const selab200_clip &c = clips[i];
        if (c.container >= n_handles)
            return fail(SELAB200_ERR_ARGUMENT, "clip %u: container %u, but %u handles", i, c.container, n_handles);
        if (c.reserved != 0)
            return fail(SELAB200_ERR_ARGUMENT, "clip %u: reserved field is not 0", i);
        const unsigned long long total = (unsigned long long)handles[c.container]->info.n_frames * kFrame;
        if (c.start > total || length > total - c.start)
            return fail(SELAB200_ERR_ARGUMENT, "clip %u: samples [%llu, %llu + %u) outside the %llu samples of its container",
                        i, (unsigned long long)c.start, (unsigned long long)c.start, length, total);
        const uint32_t C = handles[c.container]->info.channels, C0 = handles[clips[0].container]->info.channels;
        if (select && top >= C)
            return fail(SELAB200_ERR_ARGUMENT, "clip %u: channel %u selected, but its container has %u channels", i, top, C);
        if (!select && !mean && C != C0)
            return fail(SELAB200_ERR_ARGUMENT, "clip %u: its container has %u channels, clip 0's %u: a full selection "
                                               "without SELAB200_CLIP_MEAN needs one channel count", i, C, C0);
    }
    const uint32_t n_out = mean ? 1 : select ? n_select : handles[clips[0].container]->info.channels;
    const unsigned long long sample_bytes = (unsigned long long)n_out * (f32 ? 4 : 2);
    const unsigned long long clip_bytes = length * sample_bytes;
    if (clip_bytes > ~0ull / n_clips)
        return fail(SELAB200_ERR_ARGUMENT, "output of %u clips of %u samples does not fit 64 bits", n_clips, length);

    // the selection: (container << 32 | frame), sorted and deduplicated
    std::vector<unsigned long long> keys;
    for (uint32_t i = 0; i < n_clips; i++) {
        const unsigned long long f0 = clips[i].start / kFrame, f1 = (clips[i].start + length - 1) / kFrame;
        for (unsigned long long f = f0; f <= f1; f++)
            keys.push_back((unsigned long long)clips[i].container << 32 | f);
    }
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());

    // Per covered frame: the header rules over all its subframes, the positions it needs (a bit each), and where its
    // rows and row-table entries start in its group.  Groups are cut at frame ends.
    const uint32_t group_subs = clip_group_frames(1);
    std::vector<uint32_t> need(keys.size()), key_group(keys.size()), key_tab(keys.size());
    std::vector<size_t> group_key0;
    std::vector<std::vector<uint2>> tables;
    uint64_t n_need = 0;
    uint32_t rows = 0;
    for (size_t k = 0; k < keys.size(); k++) {
        const uint32_t ci = (uint32_t)(keys[k] >> 32);
        const unsigned long long f = keys[k] & 0xffffffffull;
        const selab200_container *h = handles[ci];
        const uint32_t C = h->info.channels;
        const selab200_subframe_desc *fd = h->buf.h_descs + f * C;
        if (!frame_check(fd, C, h->info.n_words))
            return fail(SELAB200_ERR_BITSTREAM, "container %u, frame %llu: a subframe header breaks the format", ci, f);
        uint32_t pos[SELAB200_MAX_CHANNELS]; // channel -> position in the frame (a permutation, by frame_check)
        for (uint32_t p = 0; p < C; p++)
            pos[fd[p].channel] = p;
        const uint32_t n_sel = select ? n_select : C;
        uint32_t m = 0;
        for (uint32_t j = 0; j < n_sel; j++) {
            const uint32_t p = pos[select ? select[j] : j];
            m |= 1u << p;
            if (fd[p].subframe_type == 1)
                m |= 1u << pos[fd[p].parent_channel];
        }
        const uint32_t n = (uint32_t)__builtin_popcount(m);
        if (k == 0 || rows + n > group_subs) {
            group_key0.push_back(k);
            tables.emplace_back();
            rows = 0;
        }
        std::vector<uint2> &tab = tables.back();
        need[k] = m;
        key_group[k] = (uint32_t)(group_key0.size() - 1);
        key_tab[k] = (uint32_t)tab.size();
        const auto row = [&](uint32_t p) { return rows + (uint32_t)__builtin_popcount(m & ((1u << p) - 1)); };
        for (uint32_t j = 0; j < n_sel; j++) {
            const uint32_t p = pos[select ? select[j] : j];
            tab.push_back(make_uint2(row(p), fd[p].subframe_type == 1 ? row(pos[fd[p].parent_channel]) : kNoParentRow));
        }
        rows += n;
        n_need += n;
    }
    *frames_decoded = keys.size();
    *subframes_decoded = n_need;

    // every clip as pieces of at most one frame each
    std::vector<std::vector<SelectPiece>> pieces(group_key0.size());
    for (uint32_t i = 0; i < n_clips; i++) {
        const selab200_clip &c = clips[i];
        const uint32_t n = select ? n_select : handles[c.container]->info.channels;
        const unsigned long long f0 = c.start / kFrame, end = c.start + length;
        const size_t k0 = std::lower_bound(keys.begin(), keys.end(), (unsigned long long)c.container << 32 | f0) - keys.begin();
        for (unsigned long long s = c.start; s < end;) {
            const uint32_t t0 = (uint32_t)(s % kFrame), count = (uint32_t)std::min<unsigned long long>(kFrame - t0, end - s);
            const size_t k = k0 + (size_t)(s / kFrame - f0);
            pieces[key_group[k]].push_back(SelectPiece{i * clip_bytes + (s - c.start) * sample_bytes, key_tab[k], n, t0, count});
            s += count;
        }
    }

    ClipSelection sel;
    for (size_t grp = 0; grp < group_key0.size(); grp++) {
        const size_t k1 = grp + 1 < group_key0.size() ? group_key0[grp + 1] : keys.size();
        sel.descs.clear();
        sel.src.clear();
        sel.at.clear();
        sel.frame_h.clear();
        sel.frame_end.clear();
        unsigned long long words = 0;
        for (size_t k = group_key0[grp]; k < k1; k++) {
            const selab200_container *h = handles[keys[k] >> 32];
            const unsigned long long f = keys[k] & 0xffffffffull;
            const uint32_t C = h->info.channels;
            const unsigned long long image = reinterpret_cast<unsigned long long>(h->buf.d_bytes);
            for (uint32_t p = 0; p < C; p++) {
                if (!((need[k] >> p) & 1))
                    continue;
                selab200_subframe_desc d = h->buf.h_descs[f * C + p];
                const unsigned long long at = container_frame_byte(f, C, d.refl_offset) + 4 + (unsigned long long)kSubframeHeaderBytes * p + 7;
                sel.src.push_back(image + at);
                sel.at.push_back(at);
                sel.frame_end.push_back(at + 4ull * d.refl_words + 5 + 4ull * d.res_words + 3);
                sel.frame_h.push_back(h);
                d.channel = 0;
                d.subframe_type = 0;
                d.parent_channel = 0;
                d.refl_offset = words;
                d.res_offset = words + d.refl_words;
                words += (unsigned long long)d.refl_words + d.res_words;
                sel.descs.push_back(d);
            }
        }
        if (int rc = plan_fetch(sel, 1))
            return rc;
        CodedInput in{sel.descs.data(), nullptr, (size_t)words, nullptr, &sel};
        if (int rc = decode_pipeline(in, 0, (uint32_t)sel.descs.size(), 1, nullptr, nullptr, nullptr))
            return rc;
        const int rc = !f32  ? clip_gather_select<int16_t, false>(pieces[grp], tables[grp], out, device_out)
                       : mean ? clip_gather_select<float, true>(pieces[grp], tables[grp], out, device_out)
                              : clip_gather_select<float, false>(pieces[grp], tables[grp], out, device_out);
        if (rc)
            return rc;
    }
    return 0;
}

extern "C" {

int selab200_container_decode_clips(selab200_container *const *handles, uint32_t n_handles, const selab200_clip *clips,
                                    uint32_t n_clips, uint32_t length, int16_t *pcm_out, uint64_t *frames_decoded)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    return decode_clips(handles, n_handles, clips, n_clips, length, reinterpret_cast<uint8_t *>(pcm_out), false,
                        frames_decoded);
}

int selab200_container_decode_clips_device(selab200_container *const *handles, uint32_t n_handles,
                                           const selab200_clip *clips, uint32_t n_clips, uint32_t length,
                                           int16_t *d_pcm_out, uint64_t *frames_decoded)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (d_pcm_out && n_clips) { // the primary holds every open image, so the output must live there too
        cudaPointerAttributes attr;
        if (cudaPointerGetAttributes(&attr, d_pcm_out) != cudaSuccess || attr.type != cudaMemoryTypeDevice ||
            attr.device != g.device) {
            cudaGetLastError();
            return fail(SELAB200_ERR_ARGUMENT, "d_pcm_out is not device memory of the primary device (%d)", g.device);
        }
        if (reinterpret_cast<uintptr_t>(d_pcm_out) & 1)
            return fail(SELAB200_ERR_ARGUMENT, "d_pcm_out is not 2-byte aligned");
    }
    return decode_clips(handles, n_handles, clips, n_clips, length, reinterpret_cast<uint8_t *>(d_pcm_out), true,
                        frames_decoded);
}

int selab200_container_decode_clips_select(selab200_container *const *handles, uint32_t n_handles,
                                           const selab200_clip *clips, uint32_t n_clips, uint32_t length,
                                           const uint8_t *select, uint32_t n_select, uint32_t flags, void *out,
                                           uint64_t *frames_decoded, uint64_t *subframes_decoded)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    return decode_clips_select(handles, n_handles, clips, n_clips, length, select, n_select, flags,
                               static_cast<uint8_t *>(out), false, frames_decoded, subframes_decoded);
}

int selab200_container_decode_clips_select_device(selab200_container *const *handles, uint32_t n_handles,
                                                  const selab200_clip *clips, uint32_t n_clips, uint32_t length,
                                                  const uint8_t *select, uint32_t n_select, uint32_t flags,
                                                  void *d_out, uint64_t *frames_decoded, uint64_t *subframes_decoded)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (d_out && n_clips) { // the primary holds every open image, so the output must live there too
        cudaPointerAttributes attr;
        if (cudaPointerGetAttributes(&attr, d_out) != cudaSuccess || attr.type != cudaMemoryTypeDevice ||
            attr.device != g.device) {
            cudaGetLastError();
            return fail(SELAB200_ERR_ARGUMENT, "d_out is not device memory of the primary device (%d)", g.device);
        }
        const unsigned align = flags & SELAB200_CLIP_FLOAT32 ? 4 : 2;
        if (reinterpret_cast<uintptr_t>(d_out) & (align - 1))
            return fail(SELAB200_ERR_ARGUMENT, "d_out is not %u-byte aligned", align);
    }
    return decode_clips_select(handles, n_handles, clips, n_clips, length, select, n_select, flags,
                               static_cast<uint8_t *>(d_out), true, frames_decoded, subframes_decoded);
}

int selab200_container_info_get(const uint8_t *container, size_t n_bytes, selab200_container_info *info)
{
    if (!container || !info)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    return walk_container(container, n_bytes, info, nullptr);
}

int selab200_container_frame_offsets(const uint8_t *container, size_t n_bytes, uint64_t *offsets, size_t capacity,
                                     selab200_container_info *info)
{
    if (!container || !offsets || !info)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = walk_container(container, n_bytes, info, nullptr, offsets, capacity))
        return rc;
    if ((size_t)info->n_frames + 1 > capacity)
        return fail(SELAB200_ERR_CAPACITY, "offset table too small: %zu entries, need %u", capacity, info->n_frames + 1);
    return 0;
}

void selab200_container_close(selab200_container *h)
{
    if (!h)
        return;
    std::lock_guard<std::mutex> lock(g_mutex);
    tl_ctx = &g_slots[0]; // container handles belong to the primary device
    if (g.ready)
        cudaSetDevice(g.device); // the caller may be on a thread that never selected the device
    if (g.s_h2d)
        cudaStreamSynchronize(g.s_h2d); // the upload reads the caller's bytes
    if (g.ready && g_spare_buffers.size() < kMaxSpareBuffers)
        g_spare_buffers.push_back(h->buf);
    else
        h->buf.destroy();
    if (h->host && h->bytes)
        cudaFreeHost(const_cast<uint8_t *>(h->bytes));
    delete h;
}

// The frame walk of both opens: h->info, and the descriptors in h->buf's pinned table the chunked uploads stream from.
static int walk_into(selab200_container *h, const uint8_t *container, size_t n_bytes)
{
    // One walk, into a growing host vector (numFrames is not trusted for sizing), then a pinned copy.
    std::vector<selab200_subframe_desc> descs;
    descs.reserve(n_bytes / 2048 + 16);
    if (int rc = walk_container(container, n_bytes, &h->info, &descs))
        return rc;
    if (descs.empty())
        return 0;
    if (h->buf.h_cap < descs.size()) {
        if (h->buf.h_descs)
            cudaFreeHost(h->buf.h_descs);
        h->buf.h_descs = nullptr;
        h->buf.h_cap = 0;
        const size_t want = descs.size() + descs.size() / 4 + 64;
        if (cudaMallocHost(reinterpret_cast<void **>(&h->buf.h_descs), want * sizeof(selab200_subframe_desc)) != cudaSuccess)
            return fail(SELAB200_ERR_CUDA, "cudaMallocHost(%zu) failed", want * sizeof(selab200_subframe_desc));
        h->buf.h_cap = want;
    }
    memcpy(h->buf.h_descs, descs.data(), descs.size() * sizeof(selab200_subframe_desc));
    return 0;
}

// Both opens end here: the handle out, or on failure the handle closed and the failure's message kept.
static int open_done(int rc, selab200_container *h, selab200_container **handle, selab200_container_info *info)
{
    if (rc != 0) {
        char keep[sizeof g_error];
        memcpy(keep, g_error, sizeof keep);
        selab200_container_close(h);
        memcpy(g_error, keep, sizeof keep);
        return rc;
    }
    *info = h->info;
    *handle = h;
    return 0;
}

int selab200_container_open(const uint8_t *container, size_t n_bytes, selab200_container **handle,
                            selab200_container_info *info)
{
    if (!container || !handle || !info)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    *handle = nullptr;
    selab200_container_info probe;
    if (int rc = walk_container(container, n_bytes < 15 ? n_bytes : 15, &probe, nullptr)) // header checks only
        return rc;
    selab200_container *h = nullptr;
    int rc = 0;
    {
        std::lock_guard<std::mutex> lock(g_mutex);
        if ((rc = require_ready()) != 0)
            return rc;
        h = new selab200_container;
        h->bytes = container;
        h->n_bytes = n_bytes;
        // recycled buffers: the smallest spare that is large enough, else any spare (it is regrown below)
        if (!g_spare_buffers.empty()) {
            size_t pick = 0;
            for (size_t i = 0; i < g_spare_buffers.size(); i++)
                if (g_spare_buffers[i].d_cap >= n_bytes + 64 &&
                    (g_spare_buffers[pick].d_cap < n_bytes + 64 || g_spare_buffers[i].d_cap < g_spare_buffers[pick].d_cap))
                    pick = i;
            h->buf = g_spare_buffers[pick];
            g_spare_buffers.erase(g_spare_buffers.begin() + pick);
        }
        cudaError_t e = cudaSuccess;
        if (h->buf.d_cap < n_bytes + 64) {
            if (h->buf.d_bytes)
                cudaFree(h->buf.d_bytes);
            h->buf.d_bytes = nullptr;
            h->buf.d_cap = 0;
            const size_t want = n_bytes + n_bytes / 8 + 4096;
            e = cudaMalloc(&h->buf.d_bytes, want);
            if (e != cudaSuccess)
                rc = fail(SELAB200_ERR_CUDA, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
            else
                h->buf.d_cap = want;
        }
        // start the upload first: the DMA engine streams the bytes while this thread walks them
        h->piece_bytes = ((n_bytes + ContainerBuffers::kPieces - 1) / ContainerBuffers::kPieces + 255) & ~(size_t)255;
        for (int i = 0; rc == 0 && (size_t)i * h->piece_bytes < n_bytes; i++) {
            const size_t lo = (size_t)i * h->piece_bytes;
            const size_t len = lo + h->piece_bytes <= n_bytes ? h->piece_bytes : n_bytes - lo;
            if (!h->buf.ev_piece[i])
                e = cudaEventCreateWithFlags(&h->buf.ev_piece[i], cudaEventDisableTiming);
            if (e == cudaSuccess)
                e = cudaMemcpyAsync(static_cast<uint8_t *>(h->buf.d_bytes) + lo, container + lo, len, cudaMemcpyHostToDevice, g.s_h2d);
            if (e == cudaSuccess)
                e = cudaEventRecord(h->buf.ev_piece[i], g.s_h2d);
            if (e != cudaSuccess)
                rc = fail(SELAB200_ERR_CUDA, "container upload failed: %s", cudaGetErrorString(e));
            h->n_pieces = i + 1;
        }
    }
    if (rc == 0)
        rc = walk_into(h, container, n_bytes);
    return open_done(rc, h, handle, info);
}

int selab200_container_open_host(const uint8_t *container, size_t n_bytes, selab200_container **handle,
                                 selab200_container_info *info)
{
    if (!container || !handle || !info)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    *handle = nullptr;
    selab200_container_info probe;
    if (int rc = walk_container(container, n_bytes < 15 ? n_bytes : 15, &probe, nullptr)) // header checks only
        return rc;
    {
        std::lock_guard<std::mutex> lock(g_mutex);
        if (int rc = require_ready())
            return rc;
    }
    selab200_container *h = new selab200_container;
    h->host = true;
    h->n_bytes = n_bytes;
    int rc = walk_into(h, container, n_bytes);
    if (rc == 0) {
        // the image in page-locked memory the handle owns, mapped into every device's address space; the padding
        // covers the reads of the last subframe's fetch run (3 bytes of slack, rounded out to 16)
        void *p = nullptr;
        cudaError_t e = cudaHostAlloc(&p, n_bytes + 64, cudaHostAllocMapped | cudaHostAllocPortable);
        void *d = nullptr;
        if (e == cudaSuccess) {
            h->bytes = static_cast<const uint8_t *>(p);
            memcpy(p, container, n_bytes);
            memset(static_cast<uint8_t *>(p) + n_bytes, 0, 64);
            e = cudaHostGetDevicePointer(&d, p, 0);
        }
        if (e != cudaSuccess)
            rc = fail(SELAB200_ERR_CUDA, "page-locked image of %zu bytes: %s", n_bytes + 64, cudaGetErrorString(e));
        h->mapped = static_cast<const uint8_t *>(d);
    }
    return open_done(rc, h, handle, info);
}

int selab200_clip_bytes_fetched(uint64_t *bytes)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!bytes)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    *bytes = g_clip_bytes_fetched;
    return 0;
}

int selab200_container_decode(selab200_container *h, int16_t *pcm_out)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!h)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    const uint32_t n_frames = h->info.n_frames, channels = h->info.channels;
    if (n_frames == 0)
        return 0;
    if (!pcm_out)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    // with several devices the primary (which holds the whole image) takes the first block
    const CodedInput in{h->buf.h_descs, nullptr, (size_t)h->info.n_words, h};
    return run_blocks(n_frames, [&](DevicePart &p) {
        return decode_pipeline(in, p.f0, p.nf, channels, pcm_out, nullptr, nullptr);
    }).rc;
}

int selab200_container_verify(selab200_container *h, const int16_t *pcm, selab200_verify_entry *entries, size_t capacity,
                              size_t *n_entries)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!h || !n_entries || (!entries && capacity))
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    *n_entries = 0;
    const uint32_t n_frames = h->info.n_frames, channels = h->info.channels;
    if (n_frames == 0)
        return 0;
    if (!pcm)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    const CodedInput in{h->buf.h_descs, nullptr, (size_t)h->info.n_words, h};
    const Blocks b = run_blocks(n_frames, [&](DevicePart &p) {
        return decode_pipeline(in, p.f0, p.nf, channels, nullptr, pcm, &p.res.report);
    });
    if (b.rc)
        return b.rc;
    return deliver_records(b.total.report, entries, capacity, n_entries);
}

int selab200_selftest(uint32_t *mismatches)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!mismatches)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    uint32_t *d = &device_counters()->selftest;
    CUDA_TRY(cudaMemsetAsync(d, 0, sizeof *d, g.stream));
    k_selftest_scaling<<<(131071 + 255) / 256, 256, 0, g.stream>>>(d);
    if (int rc = launch_check("k_selftest_scaling"))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(&g.h_small->selftest, d, sizeof *d, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaStreamSynchronize(g.stream));
    *mismatches = g.h_small->selftest;
    return 0;
}

int selab200_quantise_probe(const double *k, size_t n, int32_t *out)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!k || !out)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (n == 0)
        return 0;
    if (n > 0xffffffffu)
        return fail(SELAB200_ERR_ARGUMENT, "at most 2^32 - 1 values per call");
    if (int rc = g.in.ensure(n * sizeof(double))) return rc;
    if (int rc = g.work.ensure(n * 4 * sizeof(int32_t))) return rc;
    CUDA_TRY(cudaMemcpyAsync(g.in.ptr, k, n * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    k_quantise_probe<<<(unsigned)((n + 255) / 256), 256, 0, g.stream>>>(static_cast<const double *>(g.in.ptr), (uint32_t)n,
                                                                       static_cast<int32_t *>(g.work.ptr));
    if (int rc = launch_check("k_quantise_probe"))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(out, g.work.ptr, n * 4 * sizeof(int32_t), cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaStreamSynchronize(g.stream));
    return 0;
}

static_assert(sizeof(selab200_search_trace) == 32, "selab200_search_trace layout (include/sela_b200.h)");
static_assert(sizeof(selab200_search_unit) == sizeof(SearchUnit) &&
                  offsetof(selab200_search_unit, ref_order) == offsetof(SearchUnit, ref_order) &&
                  offsetof(selab200_search_unit, best) == offsetof(SearchUnit, best),
              "selab200_search_unit mirrors SearchUnit");

// What a test hook returns besides descriptors and words (encode_batch): host pointers, null where the hook has none.
struct BatchOutputs {
    size_t *words_used = nullptr;
    size_t *ref_words = nullptr;                           // search
    size_t *base_words = nullptr, *n_difference = nullptr; // pairing, search_pairing (base_words: search_windows)
    size_t *n_window = nullptr;                            // search_windows ...
    uint64_t *window_keys = nullptr;                       // ... and its units' window keys
    selab200_lossless_entry *entries = nullptr;            // lossless: the re-coded pairs
    size_t entries_capacity = 0, *n_entries = nullptr;
    selab200_analysis_trace *analysis = nullptr;           // plain: the tracing unit kernel's records
    selab200_search_trace *trace = nullptr;                // search, pairing, search_pairing: the tracing kernels'
                                                           // records ...
    selab200_search_unit *units = nullptr;                 // ... and the search records (search)
    uint8_t *par = nullptr;                                // ... and the pairing's choice (pairing, search_pairing)
    double *estimates = nullptr;                           // search_guided, with trace: every unit's E[100] ...
    uint32_t *masks = nullptr;                             // ... and its order mask, 4 words
};

// A test hook's predictors: every order in min_order..kMaxOrder, every q in [-64, 63], and with zero_past, every q
// past the order zero.  noun: what a predictor is called in the messages.
static int check_predictors(const selab200_predictor *pred, size_t n, int min_order, bool zero_past, const char *noun)
{
    for (size_t u = 0; u < n; u++) {
        const int o = pred[u].order;
        if (o < min_order || o > kMaxOrder)
            return fail(SELAB200_ERR_RANGE, "order %d of %s %zu outside %d..%d", o, noun, u, min_order, kMaxOrder);
        for (int i = 0; i < kMaxOrder; i++) {
            const int q = pred[u].q[i];
            if (zero_past && (i < o ? q < -64 || q > 63 : q != 0))
                return fail(SELAB200_ERR_RANGE, "q[%d] = %d of %s %zu (order %d) outside [-64, 63], or not zero "
                            "past the order", i, q, noun, u, o);
            if (!zero_past && (q < -64 || q > 63))
                return fail(SELAB200_ERR_RANGE, "q[%d] = %d of %s %zu outside [-64, 63]", i, q, noun, u);
        }
    }
    return 0;
}

// For tests: one unpipelined batch of `mode` through encode_device on g.stream.  pred (lossless: required): every
// unit's predictor, for the pairing and the search + pairing followed by the candidates', for the window search by
// the (unit, window) records' (include/sela_b200.h).  arg: the window search's mask, or the guided order search's
// candidate count; with window_table (host, popcount(mask) rows of 2048) the mask selects that table's rows in place
// of the fixed table's.
static int encode_batch(EncodeMode mode, const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                        const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                        size_t words_capacity, const BatchOutputs &out, uint32_t arg = 0,
                        const double *window_table = nullptr)
{
    if (int rc = require_ready())
        return rc;
    const bool search_guided = mode == EncodeMode::search_guided;
    const uint32_t windows = mode == EncodeMode::search_windows ? arg : 0;
    const bool lossless = mode == EncodeMode::lossless, search = mode == EncodeMode::search || search_guided,
               search_pairing = mode == EncodeMode::search_pairing,
               search_windows = mode == EncodeMode::search_windows,
               pairing = mode == EncodeMode::pairing || search_pairing;
    const bool every_q = search || search_pairing || search_windows; // q[0..99] and a reference order 1..100
    if (!pcm || !descs || !words || !out.words_used || (mode == EncodeMode::plain && !out.analysis) ||
        (lossless && (!pred || (!out.entries && out.entries_capacity) || !out.n_entries)) ||
        (search && !out.ref_words) || (pairing && (!out.base_words || !out.n_difference)) ||
        (search_windows && (!out.base_words || !out.n_window)))
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (int rc = check_channels(channels))
        return rc;
    if (search_windows && !window_table)
        if (int rc = check_windows(windows))
            return rc;
    if (search_guided)
        if (int rc = check_candidates(arg))
            return rc;
    *out.words_used = 0;
    if (lossless)
        *out.n_entries = 0;
    if (search)
        *out.ref_words = 0;
    if (pairing)
        *out.base_words = *out.n_difference = 0;
    if (search_windows)
        *out.base_words = *out.n_window = 0;
    if (n_frames == 0)
        return 0;
    const size_t n_sub = (size_t)n_frames * channels, n_units = encode_units(n_frames, channels);
    const uint32_t n_windows = search_windows ? (uint32_t)__builtin_popcount(windows) : 0;
    const size_t n_pred = pairing ? n_units + n_sub * (channels - 1) : n_units + n_units * n_windows;
    if (pred) {
        const size_t n_first = search_windows ? n_units : n_pred;
        if (int rc = check_predictors(pred, n_first, every_q ? 1 : 0, !every_q, pairing ? "predictor" : "unit"))
            return rc;
        if (search_windows) // the window records' order is not read
            if (int rc = check_predictors(pred + n_units, n_pred - n_units, 0, false, "window record"))
                return rc;
    }
    const EncodeLayout l = encode_layout(mode, n_frames, channels, n_windows);
    const size_t pred_bytes = pred ? align256(n_pred * sizeof(selab200_predictor)) : 0;
    const size_t n_records = search_pairing   ? n_sub * channels * kMaxOrder
                             : pairing        ? n_sub * channels
                             : search_windows ? n_units * n_windows * kMaxOrder
                                              : n_units * kMaxOrder;
    const size_t trace_bytes = out.analysis ? n_units * sizeof(selab200_analysis_trace)
                               : out.trace  ? n_records * sizeof(selab200_search_trace)
                                            : 0;
    const size_t table_bytes = window_table ? (size_t)n_windows * kFrame * sizeof(double) : 0;
    const size_t est_bytes = out.estimates ? n_units * kMaxOrder * sizeof(double) : 0;
    if (int rc = g.in.ensure(n_sub * kFrame * 2)) return rc;
    if (int rc = g.descs.ensure(n_sub * sizeof(selab200_subframe_desc))) return rc;
    if (int rc = g.words.ensure(words_capacity * 4 + 64)) return rc;
    if (int rc = g.work.ensure(l.bytes)) return rc;
    if (int rc = aux_for(pred_bytes + align256(trace_bytes) + align256(table_bytes) + est_bytes, g.stream)) return rc;
    Counters *d_ctr = device_counters();
    const selab200_predictor *d_pred = static_cast<const selab200_predictor *>(g.aux.ptr);
    void *d_trace = static_cast<char *>(g.aux.ptr) + pred_bytes;
    double *d_table = reinterpret_cast<double *>(static_cast<char *>(g.aux.ptr) + pred_bytes + align256(trace_bytes));
    double *d_est = reinterpret_cast<double *>(reinterpret_cast<char *>(d_table) + align256(table_bytes));
    EncodeOptions o; // fresh: encode_device resets the counters and records
    o.mode = mode;
    if (lossless)
        if (int rc = lossless_area(n_sub, o.lossless)) return rc;
    o.d_ref_words = &d_ctr->ref_words;
    o.d_base_words = &d_ctr->base_words;
    o.d_n_difference = &d_ctr->n_difference;
    o.windows = windows;
    o.d_n_window = &d_ctr->n_window;
    o.candidates = search_guided ? arg : 0;
    o.d_estimates = est_bytes ? d_est : nullptr;
    o.d_pred = pred ? d_pred : nullptr;
    o.d_pair_pred = pred && pairing ? d_pred + n_units : nullptr;
    o.d_window_pred = pred && search_windows ? d_pred + n_units : nullptr;
    o.d_windows = window_table ? d_table : nullptr;
    o.d_trace = out.analysis ? static_cast<selab200_analysis_trace *>(d_trace) : nullptr;
    o.d_search_trace = out.trace ? static_cast<selab200_search_trace *>(d_trace) : nullptr;
    if (trace_bytes)
        CUDA_TRY(cudaMemsetAsync(d_trace, 0, trace_bytes, g.stream));
    CUDA_TRY(cudaMemcpyAsync(g.in.ptr, pcm, n_sub * kFrame * 2, cudaMemcpyHostToDevice, g.stream));
    if (pred)
        CUDA_TRY(cudaMemcpyAsync(g.aux.ptr, pred, n_pred * sizeof(selab200_predictor), cudaMemcpyHostToDevice, g.stream));
    if (table_bytes)
        CUDA_TRY(cudaMemcpyAsync(d_table, window_table, table_bytes, cudaMemcpyHostToDevice, g.stream));
    if (int rc = encode_device(static_cast<const int16_t *>(g.in.ptr), n_frames, channels,
                               static_cast<selab200_subframe_desc *>(g.descs.ptr), static_cast<uint32_t *>(g.words.ptr),
                               words_capacity, &d_ctr->used, &d_ctr->status, g.work.ptr, g.work.bytes, g.stream, o))
        return rc;
    const char *ws = static_cast<const char *>(g.work.ptr);
    if (out.units)
        CUDA_TRY(cudaMemcpyAsync(out.units, ws + l.search, n_units * sizeof(SearchUnit), cudaMemcpyDeviceToHost, g.stream));
    if (out.par)
        CUDA_TRY(cudaMemcpyAsync(out.par, ws + l.par, n_sub, cudaMemcpyDeviceToHost, g.stream));
    if (out.window_keys)
        CUDA_TRY(cudaMemcpyAsync(out.window_keys, ws + l.window_keys, n_units * sizeof(uint64_t), cudaMemcpyDeviceToHost,
                                 g.stream));
    if (out.masks)
        CUDA_TRY(cudaMemcpyAsync(out.masks, ws + l.masks, n_units * sizeof(uint4), cudaMemcpyDeviceToHost, g.stream));
    if (est_bytes)
        CUDA_TRY(cudaMemcpyAsync(out.estimates, d_est, est_bytes, cudaMemcpyDeviceToHost, g.stream));
    if (trace_bytes)
        CUDA_TRY(cudaMemcpyAsync(out.analysis ? static_cast<void *>(out.analysis) : static_cast<void *>(out.trace),
                                 d_trace, trace_bytes, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaMemcpyAsync(descs, g.descs.ptr, n_sub * sizeof(selab200_subframe_desc), cudaMemcpyDeviceToHost, g.stream));
    Result r;
    const int status = read_counters(g.stream, r);
    *out.words_used = r.words;
    if (search)
        *out.ref_words = (size_t)r.ref_words;
    if (pairing) {
        *out.base_words = (size_t)r.base_words;
        *out.n_difference = (size_t)r.n_difference;
    }
    if (search_windows) {
        *out.base_words = (size_t)r.base_words;
        *out.n_window = (size_t)r.n_window;
    }
    if (status)
        return status;
    if (r.words > words_capacity)
        return fail(SELAB200_ERR_CAPACITY, "%s", status_text(SELAB200_ERR_CAPACITY));
    CUDA_TRY(cudaMemcpyAsync(words, g.words.ptr, r.words * 4, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaStreamSynchronize(g.stream));
    if (!lossless)
        return 0;
    if (int rc = collect_records(o.lossless.n_entries, nullptr, o.lossless.entries, n_sub, g.stream, r.recoded))
        return rc;
    return deliver_records(r.recoded, out.entries, out.entries_capacity, out.n_entries);
}

// For tests: one unpipelined batch through encode_device with the tracing unit kernel (include/sela_b200.h).
int selab200_encode_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels, selab200_subframe_desc *descs,
                          uint32_t *words, size_t words_capacity, size_t *words_used, selab200_analysis_trace *trace)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    BatchOutputs out;
    out.words_used = words_used;
    out.analysis = trace;
    return encode_batch(EncodeMode::plain, pcm, n_frames, channels, nullptr, descs, words, words_capacity, out);
}

// For tests: one unpipelined lossless batch through encode_device, every unit coded with its predictor from pred.
int selab200_encode_lossless_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                    const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                    size_t words_capacity, size_t *words_used, selab200_lossless_entry *entries,
                                    size_t entries_capacity, size_t *n_entries)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    BatchOutputs out;
    out.words_used = words_used;
    out.entries = entries;
    out.entries_capacity = entries_capacity;
    out.n_entries = n_entries;
    return encode_batch(EncodeMode::lossless, pcm, n_frames, channels, pred, descs, words, words_capacity, out);
}

// For tests: one unpipelined order-search batch through encode_device, every unit's q[0..99] and reference order
// from pred.
int selab200_encode_search_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                  const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                  size_t words_capacity, size_t *words_used, size_t *ref_words)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!pred)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    BatchOutputs out;
    out.words_used = words_used;
    out.ref_words = ref_words;
    return encode_batch(EncodeMode::search, pcm, n_frames, channels, pred, descs, words, words_capacity, out);
}

// For tests: selab200_encode_search_forced (or, without pred, the unforced search) through the tracing search
// kernels, with the search records and the tracing kernels' records.
int selab200_encode_search_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                 const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                 size_t words_capacity, size_t *words_used, size_t *ref_words,
                                 selab200_search_unit *units, selab200_search_trace *trace)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!units || !trace)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    BatchOutputs out;
    out.words_used = words_used;
    out.ref_words = ref_words;
    out.units = units;
    out.trace = trace;
    return encode_batch(EncodeMode::search, pcm, n_frames, channels, pred, descs, words, words_capacity, out);
}

// For tests: one unpipelined pairing batch through encode_device.  pred: the base's units' predictors, then the
// candidates'.
int selab200_encode_pairing_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                   const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                   size_t words_capacity, size_t *words_used, size_t *base_words, size_t *n_difference)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!pred)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    BatchOutputs out;
    out.words_used = words_used;
    out.base_words = base_words;
    out.n_difference = n_difference;
    return encode_batch(EncodeMode::pairing, pcm, n_frames, channels, pred, descs, words, words_capacity, out);
}

// For tests: selab200_encode_pairing_forced (or, without pred, the unforced pairing) with the choice, par, and the
// candidates' trace records.
int selab200_encode_pairing_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                  const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                  size_t words_capacity, size_t *words_used, size_t *base_words, size_t *n_difference,
                                  uint8_t *par, selab200_search_trace *trace)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!par || !trace)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    BatchOutputs out;
    out.words_used = words_used;
    out.base_words = base_words;
    out.n_difference = n_difference;
    out.par = par;
    out.trace = trace;
    return encode_batch(EncodeMode::pairing, pcm, n_frames, channels, pred, descs, words, words_capacity, out);
}

// For tests: one unpipelined search + pairing batch through encode_device.  pred: the base's units' q[0..99] and
// reference orders, then the candidates'.
int selab200_encode_search_pairing_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                          const selab200_predictor *pred, selab200_subframe_desc *descs,
                                          uint32_t *words, size_t words_capacity, size_t *words_used,
                                          size_t *base_words, size_t *n_difference)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!pred)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    BatchOutputs out;
    out.words_used = words_used;
    out.base_words = base_words;
    out.n_difference = n_difference;
    return encode_batch(EncodeMode::search_pairing, pcm, n_frames, channels, pred, descs, words, words_capacity, out);
}

// For tests: selab200_encode_search_pairing_forced (or, without pred, the unforced search + pairing) through the
// tracing candidate kernels, with the choice, par, and every (candidate, order) record.
int selab200_encode_search_pairing_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                         const selab200_predictor *pred, selab200_subframe_desc *descs,
                                         uint32_t *words, size_t words_capacity, size_t *words_used,
                                         size_t *base_words, size_t *n_difference, uint8_t *par,
                                         selab200_search_trace *trace)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!par || !trace)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    BatchOutputs out;
    out.words_used = words_used;
    out.base_words = base_words;
    out.n_difference = n_difference;
    out.par = par;
    out.trace = trace;
    return encode_batch(EncodeMode::search_pairing, pcm, n_frames, channels, pred, descs, words, words_capacity, out);
}

// For tests: one unpipelined window-search batch through encode_device.  pred: the units' q[0..99] and reference
// orders, then the q of every (unit, window) record.
int selab200_encode_search_windows_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t windows,
                                          const selab200_predictor *pred, selab200_subframe_desc *descs,
                                          uint32_t *words, size_t words_capacity, size_t *words_used,
                                          size_t *base_words, size_t *n_window)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!pred)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    BatchOutputs out;
    out.words_used = words_used;
    out.base_words = base_words;
    out.n_window = n_window;
    return encode_batch(EncodeMode::search_windows, pcm, n_frames, channels, pred, descs, words, words_capacity, out,
                        windows);
}

// For tests: the window search with the given window rows (or, with pred, selab200_encode_search_windows_forced's)
// through the tracing candidate kernel, with every (unit, window, order) record and every unit's window key.
int selab200_encode_search_windows_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                         const double *windows, uint32_t n_windows, const selab200_predictor *pred,
                                         selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                         size_t *words_used, size_t *base_words, size_t *n_window,
                                         selab200_search_trace *trace, uint64_t *keys)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!windows || !trace || !keys)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (n_windows < 1 || n_windows > (uint32_t)kAnalysisWindows)
        return fail(SELAB200_ERR_ARGUMENT, "%u windows: must be 1..%d", n_windows, kAnalysisWindows);
    BatchOutputs out;
    out.words_used = words_used;
    out.base_words = base_words;
    out.n_window = n_window;
    out.trace = trace;
    out.window_keys = keys;
    return encode_batch(EncodeMode::search_windows, pcm, n_frames, channels, pred, descs, words, words_capacity, out,
                        (1u << n_windows) - 1, windows);
}

// For tests: the guided order search on one unpipelined batch (with pred, every unit's q[0..99] and reference order
// from it, as selab200_encode_search_forced takes them) through the tracing kernels, with every sized order's record,
// every unit's E[100] and its order mask.
int selab200_encode_search_guided_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t candidates,
                                        const selab200_predictor *pred, selab200_subframe_desc *descs,
                                        uint32_t *words, size_t words_capacity, size_t *words_used, size_t *ref_words,
                                        selab200_search_trace *trace, double *estimates, uint32_t *masks)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (!trace || !estimates || !masks)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    BatchOutputs out;
    out.words_used = words_used;
    out.ref_words = ref_words;
    out.trace = trace;
    out.estimates = estimates;
    out.masks = masks;
    return encode_batch(EncodeMode::search_guided, pcm, n_frames, channels, pred, descs, words, words_capacity, out,
                        candidates);
}

// selab200_fir_probe, and with `ties` selab200_fir_tie_probe (g_mutex held by the caller).
static int fir_probe(const int32_t *samples, const int32_t *orders, const int64_t *c, uint32_t n, int wide,
                     int32_t *residues, uint8_t *ties)
{
    if (int rc = require_ready())
        return rc;
    if (!samples || !orders || !c || !residues)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (n == 0)
        return 0;
    const int hi = wide ? 65535 : 32767, lo = wide ? -65535 : -32768;
    for (size_t i = 0; i < (size_t)n * kFrame; i++)
        if (samples[i] > hi || samples[i] < lo)
            return fail(SELAB200_ERR_RANGE, "sample %zu = %d outside the domain of the row form", i, samples[i]);
    for (uint32_t i = 0; i < n; i++)
        if (orders[i] < 0 || orders[i] > kMaxOrder)
            return fail(SELAB200_ERR_RANGE, "order %d of signal %u outside 0..%d", orders[i], i, kMaxOrder);
    const size_t sig = (size_t)n * kFrame * 4, cb = (size_t)n * (kMaxOrder + 1) * 8;
    if (int rc = g.in.ensure(sig)) return rc;
    if (int rc = g.work.ensure(sig)) return rc;
    if (int rc = aux_for(cb + (size_t)n * 5, g.stream)) return rc;
    long long *d_c = static_cast<long long *>(g.aux.ptr);
    int32_t *d_orders = reinterpret_cast<int32_t *>(d_c + (size_t)n * (kMaxOrder + 1));
    uint8_t *d_ties = reinterpret_cast<uint8_t *>(d_orders + n);
    CUDA_TRY(cudaMemcpyAsync(g.in.ptr, samples, sig, cudaMemcpyHostToDevice, g.stream));
    CUDA_TRY(cudaMemcpyAsync(d_c, c, cb, cudaMemcpyHostToDevice, g.stream));
    CUDA_TRY(cudaMemcpyAsync(d_orders, orders, (size_t)n * 4, cudaMemcpyHostToDevice, g.stream));
    if (ties)
        k_fir_probe<true><<<n, 32, 0, g.stream>>>(static_cast<const int32_t *>(g.in.ptr), d_orders, d_c, wide,
                                                  static_cast<int32_t *>(g.work.ptr), d_ties);
    else
        k_fir_probe<<<n, 32, 0, g.stream>>>(static_cast<const int32_t *>(g.in.ptr), d_orders, d_c, wide,
                                            static_cast<int32_t *>(g.work.ptr), nullptr);
    if (int rc = launch_check("k_fir_probe"))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(residues, g.work.ptr, sig, cudaMemcpyDeviceToHost, g.stream));
    if (ties)
        CUDA_TRY(cudaMemcpyAsync(ties, d_ties, n, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaStreamSynchronize(g.stream));
    return 0;
}

int selab200_fir_probe(const int32_t *samples, const int32_t *orders, const int64_t *c, uint32_t n, int wide,
                       int32_t *residues)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    return fir_probe(samples, orders, c, n, wide, residues, nullptr);
}

int selab200_fir_tie_probe(const int32_t *samples, const int32_t *orders, const int64_t *c, uint32_t n, int wide,
                           int32_t *residues, uint8_t *ties)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!ties)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    return fir_probe(samples, orders, c, n, wide, residues, ties);
}

// ---------------------------------------------------------------- stages --

int selab200_lpc_residues(const int32_t *samples, uint32_t n_sub, uint8_t *order, int32_t *q, int32_t *residues)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!samples || !order || !q || !residues)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (n_sub == 0)
        return 0;
    for (size_t i = 0; i < (size_t)n_sub * kFrame; i++)
        if (samples[i] > 65535 || samples[i] < -65535)
            return fail(SELAB200_ERR_RANGE, "sample %zu = %d outside the 17-bit domain of 16-bit audio", i, samples[i]);
    const size_t sig = (size_t)n_sub * kFrame * 4;
    if (int rc = g.in.ensure(sig)) return rc;
    if (int rc = g.work.ensure(sig)) return rc;
    if (int rc = aux_for(align256((size_t)n_sub * sizeof(double)) + (size_t)n_sub * kMaxOrder * 4 + n_sub + 256, g.stream)) return rc;
    double *d_means = static_cast<double *>(g.aux.ptr);
    int32_t *d_q = reinterpret_cast<int32_t *>(static_cast<char *>(g.aux.ptr) + align256((size_t)n_sub * sizeof(double)));
    uint8_t *d_order = reinterpret_cast<uint8_t *>(d_q + (size_t)n_sub * kMaxOrder);
    CUDA_TRY(cudaMemcpyAsync(g.in.ptr, samples, sig, cudaMemcpyHostToDevice, g.stream));
    if (int rc = launch_unit_means<kMeanPlanar>(g.in.ptr, n_sub, 1, d_means, g.stream))
        return rc;
    k_lpc_residues<<<n_sub, 32, 0, g.stream>>>(static_cast<const int32_t *>(g.in.ptr), d_means, n_sub, d_order, d_q,
                                               static_cast<int32_t *>(g.work.ptr));
    if (int rc = launch_check("k_lpc_residues"))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(residues, g.work.ptr, sig, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaMemcpyAsync(q, d_q, (size_t)n_sub * kMaxOrder * 4, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaMemcpyAsync(order, d_order, n_sub, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaStreamSynchronize(g.stream));
    return 0;
}

int selab200_lpc_samples(const int32_t *residues, uint32_t n_sub, const uint8_t *order, const int32_t *q,
                         int32_t *samples)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!residues || !order || !q || !samples)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (n_sub == 0)
        return 0;
    for (uint32_t i = 0; i < n_sub; i++)
        if (order[i] > kMaxOrder)
            return fail(SELAB200_ERR_BITSTREAM, "order[%u] = %u exceeds %d", i, order[i], kMaxOrder);
    const size_t sig = (size_t)n_sub * kFrame * 4;
    if (int rc = g.in.ensure(sig)) return rc;
    if (int rc = g.work.ensure(sig)) return rc;
    if (int rc = aux_for((size_t)n_sub * kMaxOrder * 4 + n_sub + 256, g.stream)) return rc;
    int32_t *d_q = static_cast<int32_t *>(g.aux.ptr);
    uint8_t *d_order = reinterpret_cast<uint8_t *>(d_q + (size_t)n_sub * kMaxOrder);
    CUDA_TRY(cudaMemcpyAsync(g.in.ptr, residues, sig, cudaMemcpyHostToDevice, g.stream));
    CUDA_TRY(cudaMemcpyAsync(d_q, q, (size_t)n_sub * kMaxOrder * 4, cudaMemcpyHostToDevice, g.stream));
    CUDA_TRY(cudaMemcpyAsync(d_order, order, n_sub, cudaMemcpyHostToDevice, g.stream));
    k_lpc_samples<<<n_sub, 32, 0, g.stream>>>(static_cast<const int32_t *>(g.in.ptr), n_sub, d_order, d_q,
                                              static_cast<int32_t *>(g.work.ptr));
    if (int rc = launch_check("k_lpc_samples"))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(samples, g.work.ptr, sig, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaStreamSynchronize(g.stream));
    return 0;
}

int selab200_rice_encode(const int32_t *values, const uint32_t *counts, uint32_t n_streams, uint32_t stride,
                         uint32_t *rice_param, uint32_t *n_words, uint32_t *words, uint32_t words_stride)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!values || !counts || !rice_param || !n_words || !words)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (stride > (uint32_t)kFrame)
        return fail(SELAB200_ERR_ARGUMENT, "stride %u exceeds %d values per stream", stride, kFrame);
    for (uint32_t i = 0; i < n_streams; i++)
        if (counts[i] > stride)
            return fail(SELAB200_ERR_ARGUMENT, "counts[%u] exceeds stride", i);
    if (n_streams == 0)
        return 0;
    // on the device every stream row starts 16-byte aligned (the encoder reads int4, rice_lane_range)
    const uint32_t pitch = (stride + 3) & ~3u;
    const size_t vbytes = (size_t)n_streams * pitch * 4, wbytes = (size_t)n_streams * words_stride * 4;
    if (int rc = g.in.ensure(vbytes + 16)) return rc;
    if (int rc = g.words.ensure(wbytes + 16)) return rc;
    if (int rc = aux_for((size_t)n_streams * 12 + 256, g.stream)) return rc;
    uint32_t *d_counts = static_cast<uint32_t *>(g.aux.ptr);
    uint32_t *d_k = d_counts + n_streams, *d_nw = d_k + n_streams;
    int32_t *d_status = &device_counters()->status;
    CUDA_TRY(cudaMemsetAsync(d_status, 0, 4, g.stream));
    if (stride)
        CUDA_TRY(cudaMemcpy2DAsync(g.in.ptr, (size_t)pitch * 4, values, (size_t)stride * 4, (size_t)stride * 4, n_streams,
                                   cudaMemcpyHostToDevice, g.stream));
    CUDA_TRY(cudaMemcpyAsync(d_counts, counts, (size_t)n_streams * 4, cudaMemcpyHostToDevice, g.stream));
    k_rice_encode<<<n_streams, 32, 0, g.stream>>>(static_cast<const int32_t *>(g.in.ptr), d_counts, pitch, d_k,
                                                  d_nw, static_cast<uint32_t *>(g.words.ptr), words_stride, d_status);
    if (int rc = launch_check("k_rice_encode"))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(rice_param, d_k, (size_t)n_streams * 4, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaMemcpyAsync(n_words, d_nw, (size_t)n_streams * 4, cudaMemcpyDeviceToHost, g.stream));
    CUDA_TRY(cudaMemcpyAsync(words, g.words.ptr, wbytes, cudaMemcpyDeviceToHost, g.stream));
    return read_status(g.stream, d_status);
}

int selab200_rice_decode(const uint32_t *words, const uint32_t *n_words, uint32_t words_stride,
                         const uint32_t *rice_param, const uint32_t *counts, uint32_t n_streams, int32_t *out,
                         uint32_t out_stride)
{
    std::lock_guard<std::mutex> lock(g_mutex);
    if (int rc = require_ready())
        return rc;
    if (!words || !n_words || !rice_param || !counts || !out)
        return fail(SELAB200_ERR_ARGUMENT, "null pointer");
    if (n_streams == 0)
        return 0;
    const size_t wbytes = (size_t)n_streams * words_stride * 4, obytes = (size_t)n_streams * out_stride * 4;
    if (int rc = g.words.ensure(wbytes + 16)) return rc;
    if (int rc = g.work.ensure(obytes + 16)) return rc;
    if (int rc = aux_for((size_t)n_streams * 12 + 256, g.stream)) return rc;
    uint32_t *d_nw = static_cast<uint32_t *>(g.aux.ptr);
    uint32_t *d_k = d_nw + n_streams, *d_counts = d_k + n_streams;
    int32_t *d_status = &device_counters()->status;
    CUDA_TRY(cudaMemsetAsync(d_status, 0, 4, g.stream));
    CUDA_TRY(cudaMemsetAsync(g.work.ptr, 0, obytes, g.stream));
    CUDA_TRY(cudaMemcpyAsync(g.words.ptr, words, wbytes, cudaMemcpyHostToDevice, g.stream));
    CUDA_TRY(cudaMemcpyAsync(d_nw, n_words, (size_t)n_streams * 4, cudaMemcpyHostToDevice, g.stream));
    CUDA_TRY(cudaMemcpyAsync(d_k, rice_param, (size_t)n_streams * 4, cudaMemcpyHostToDevice, g.stream));
    CUDA_TRY(cudaMemcpyAsync(d_counts, counts, (size_t)n_streams * 4, cudaMemcpyHostToDevice, g.stream));
    k_rice_decode_streams<<<(n_streams + 32 * kRiceWarps - 1) / (32 * kRiceWarps), 32 * kRiceWarps, 0, g.stream>>>(
        static_cast<const uint32_t *>(g.words.ptr), d_nw, words_stride, d_k, d_counts, n_streams,
        static_cast<int32_t *>(g.work.ptr), out_stride, d_status);
    if (int rc = launch_check("k_rice_decode_streams"))
        return rc;
    CUDA_TRY(cudaMemcpyAsync(out, g.work.ptr, obytes, cudaMemcpyDeviceToHost, g.stream));
    return read_status(g.stream, d_status);
}

} // extern "C"
