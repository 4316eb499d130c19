/*
 * sela_b200.h -- C ABI of the H100-native SELA per-frame encode/decode hot path.
 *
 * This is the drop-in boundary (SURVEY.md 8b).  The reference has no FFI; its
 * boundary is a set of C++ classes over std::vector-owning value structs.  Each
 * entry point below names the reference interface it replaces (paths relative
 * to the reference tree) and is what a reference-side binding would call; the
 * C++ mirror of the reference classes that sits on top of it lives in
 * sela_b200/host/ (see INTEGRATION.md).
 *
 * Conventions
 *   - plain pointers and sizes only; the caller owns every buffer it passes;
 *     the library owns device memory, streams and its workspace.
 *   - every function returns SELAB200_OK (0) or a negative selab200_status;
 *     selab200_last_error() returns a thread-local description.  The C++ shim
 *     turns a non-zero status into `throw data::Exception(...)`, the reference's
 *     error convention (src/include/data/exception.hpp:7-14, src/main.cpp:101-105).
 *   - there is NO CPU fallback: without a CUDA device every compute entry point
 *     fails with SELAB200_ERR_NO_DEVICE.
 *   - one process drives one GPU (selab200_init(device)) or several
 *     (selab200_init_devices); calls are synchronous unless they take a stream
 *     (the *_device forms), and are serialised by an internal mutex -- inside a
 *     call every device works on its own thread with its own context.
 *   - a "subframe" is one channel of one 2048-sample frame
 *     (src/include/file/wav_file.hpp:12); frames are independent.
 */
#ifndef SELA_B200_H_
#define SELA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SELAB200_ABI_VERSION     2 /* 2: selab200_init_devices, selab200_device_count, selab200_rice_decode_flagged */
#define SELAB200_FRAME_SAMPLES   2048 /* src/include/file/wav_file.hpp:12 */
#define SELAB200_MAX_LPC_ORDER   100  /* src/include/lpc.hpp:7            */
#define SELAB200_MAX_RICE_PARAM  20   /* src/include/rice.hpp:7           */
#define SELAB200_MAX_CHANNELS    16

typedef enum selab200_status {
    SELAB200_OK              = 0,
    SELAB200_ERR_NO_DEVICE   = -1, /* no CUDA device / extension not usable        */
    SELAB200_ERR_CUDA        = -2, /* a CUDA runtime call failed                    */
    SELAB200_ERR_ARGUMENT    = -3, /* null pointer, bad channel count, ...          */
    SELAB200_ERR_CAPACITY    = -4, /* output word arena too small                   */
    SELAB200_ERR_RANGE       = -5, /* sample outside the 16-bit domain              */
    SELAB200_ERR_BITSTREAM   = -6, /* malformed subframe descriptor / Rice stream   */
    SELAB200_ERR_NOT_INIT    = -7
} selab200_status;

/* One coded subframe.  Field-for-field data::SelaSubFrame
 * (src/include/data/sela_sub_frame.hpp:7-29) with the two word vectors replaced
 * by offsets (in uint32 words) into a flat arena.  32 bytes, naturally aligned. */
typedef struct selab200_subframe_desc {
    uint8_t  channel;
    uint8_t  subframe_type;     /* 0 independent, 1 difference-coded            */
    uint8_t  parent_channel;
    uint8_t  refl_rice_param;   /* reflectionCoefficientRiceParam               */
    uint16_t refl_words;        /* reflectionCoefficientRequiredInts            */
    uint8_t  lpc_order;         /* optimumLpcOrder                              */
    uint8_t  res_rice_param;    /* residueRiceParam                             */
    uint16_t res_words;         /* residueRequiredInts                          */
    uint16_t samples;           /* samplesPerChannel                            */
    uint32_t reserved;          /* zero                                         */
    uint64_t refl_offset;       /* encodedReflectionCoefficients -> words[...]  */
    uint64_t res_offset;        /* encodedResidues               -> words[...]  */
} selab200_subframe_desc;

/* ------------------------------------------------------------ life cycle -- */

/* Bind this process to CUDA device `device` (>= 0) and create the streams and
 * workspace.  Idempotent for the same device; a different device than before
 * tears the old context down first (its streams and pools belong to the old device). */
int  selab200_init(int device);
/* Several devices of one box (SURVEY.md 8b: selagpu_init(device_count, device_ids)): every device gets a
 * context of its own (streams, events, pools).  The host-buffer batch calls (selab200_encode_frames,
 * selab200_decode_frames, selab200_encode_container, selab200_container_decode and their verify, lossless and
 * search forms) then cut the frames into one contiguous block per device
 * -- n/D frames each, the last device takes the rest, the way sela::Encoder::processFrames cuts them for its
 * threads (src/sela/encoder.cpp:58-73) -- and run the blocks concurrently, reading and writing disjoint ranges
 * of the caller's buffers; results are byte-identical to a single device's.  A batch is split only when every
 * device gets at least 256 frames; a smaller one runs on the primary alone.  devices[0] is the primary: it
 * serves the stage-level calls and holds the byte image of an open container.  The *_device forms run on the first
 * entry that holds the device owning the buffers they are given.
 * A device may be listed more than once ({0, 0, 0}): every entry is an independent context on that device, with
 * its own worker thread, streams and pools, and takes a block of its own, exactly as a distinct device would. */
int  selab200_init_devices(int count, const int *devices);
int  selab200_device_count(void);
void selab200_shutdown(void);
const char *selab200_last_error(void);
int  selab200_abi_version(void);
/* Number of kernel launches issued by this process so far (bench bookkeeping). */
uint64_t selab200_launch_count(void);
/* For tests: kernel launches issued on slot `slot` (an entry of selab200_init_devices) since the slots were last set
 * up; 0 for a slot that is not set up.  Shows which slot coded which block of a split call. */
uint64_t selab200_slot_launch_count(int slot);

/* Device self-test: counts inputs s in [-65535, 65535] for which the kernels'
 * division-free s/32767 differs from IEEE division (must be 0). */
int selab200_selftest(uint32_t *mismatches);

/* Pinned host memory for the host-buffer calls (pageable memory also works, slower). */
void *selab200_host_alloc(size_t bytes);
void  selab200_host_free(void *p);

/* Safe arena size (in words) for encoding n_frames x channels subframes of 16-bit
 * audio: every stream the Rice coder can produce for in-domain input fits. */
size_t selab200_encode_words_bound(uint32_t n_frames, uint32_t channels);

/* ------------------------------------------------- batch coder (frames) -- */

/* Replaces sela::Encoder::processFrames (src/sela/encoder.cpp:40-92), i.e.
 * frame::FrameEncoder::process (src/frame/frame_encoder.cpp:11-102) over every
 * frame.  pcm: interleaved little-endian int16 exactly as the WAV data chunk
 * (src/file/wav_file.cpp:194-200), n_frames*2048*channels samples.  channels==2
 * triggers the difference-coding decision for channel 1.  descs:
 * n_frames*channels entries in frame order, channel order.  words: arena of
 * words_capacity uint32; subframes are laid out in file order (refl words then
 * residue words, src/file/sela_file.cpp:120-135); *words_used receives the total. */
int selab200_encode_frames(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                           selab200_subframe_desc *descs, uint32_t *words,
                           size_t words_capacity, size_t *words_used);

/* Replaces sela::Decoder::processFrames (src/sela/decoder.cpp:41-92), i.e.
 * frame::FrameDecoder::process (src/frame/frame_decoder.cpp:11-72) over every
 * frame.  pcm_out: interleaved int16, n_frames*2048*channels samples (the
 * layout file::WavFile::writeToFile emits, src/file/wav_file.cpp:244-266).
 * Descriptors are validated (order <= 100, rice params < 32, samples == 2048,
 * channel/parent < channels, offsets inside n_words); invalid input returns
 * SELAB200_ERR_BITSTREAM instead of the reference's undefined behaviour.  The message then names the first invalid
 * descriptor by frame and channel (a stream that runs past its words is not named), with one device or several; so do
 * selab200_verify_frames, selab200_container_decode and selab200_container_verify. */
int selab200_decode_frames(const selab200_subframe_desc *descs, uint32_t n_frames,
                           uint32_t channels, const uint32_t *words, size_t n_words,
                           int16_t *pcm_out);

/* Device-resident forms: every pointer is a device pointer, work is enqueued on
 * `stream` (a cudaStream_t; NULL is the legacy default stream, as everywhere in CUDA) and the call
 * returns without synchronising.  d_status (int32, device) receives 0 or a
 * selab200_status once the stream has drained; d_words_used is a device uint64.
 * workspace: selab200_*_workspace_bytes() bytes of device memory, 256-aligned; its contents need not be
 * initialised, and the call overwrites them.  Every counter and status a call reports is reset on
 * `stream` by the call itself.  d_words must be
 * 16-byte aligned and readable up to the next 16-byte boundary past its last word (the Rice
 * decoder fetches 16 bytes at a time); cudaMalloc / torch allocations satisfy both.  d_pcm (stereo) must
 * be 16-byte aligned as well; any other d_pcm and every d_pcm_out need 2-byte alignment only.  Any d_pcm
 * is read in whole aligned 16-byte pieces, so the 16-byte blocks that hold its first and last byte must
 * be readable (every allocation's are).  An encode writes d_words[0 .. *d_words_used) and no word past
 * it (none at all once the status is not 0).  A call rejected with SELAB200_ERR_ARGUMENT (a misaligned
 * stereo d_pcm or verify d_pcm_ref, a workspace too small, ...) enqueues nothing and writes nothing. */
size_t selab200_encode_workspace_bytes(uint32_t n_frames, uint32_t channels);
int selab200_encode_frames_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                  selab200_subframe_desc *d_descs, uint32_t *d_words,
                                  size_t words_capacity, uint64_t *d_words_used,
                                  int32_t *d_status, void *d_workspace, size_t workspace_bytes,
                                  void *stream);
size_t selab200_decode_workspace_bytes(uint32_t n_frames, uint32_t channels);
int selab200_decode_frames_device(const selab200_subframe_desc *d_descs, uint32_t n_frames,
                                  uint32_t channels, const uint32_t *d_words, size_t n_words,
                                  int16_t *d_pcm_out, int32_t *d_status, void *d_workspace,
                                  size_t workspace_bytes, void *stream);

/* The Rice-decode kernel (K5 of SURVEY.md 2) on its own, device resident: the residue streams of
 * every subframe -> d_residues[subframe][2048] int32, i.e. rice::RiceDecoder::process
 * (src/rice/rice_decoder.cpp:54-61) over a batch.  Algorithmic bytes: the words read + 4 B per
 * sample written (SURVEY.md 8d).  Asynchronous on `stream`.  Its split table and flags live in scratch
 * the library owns, which every such call shares: before it touches that scratch, each call's stream waits on
 * the device for the last kernel of the call before it, on whichever stream that one ran, so calls on
 * different streams run one after the other (no host synchronisation).  A batch larger than every earlier one grows the
 * scratch, which synchronises the device once. */
int selab200_rice_decode_frames_device(const selab200_subframe_desc *d_descs, uint32_t n_frames,
                                       uint32_t channels, const uint32_t *d_words, size_t n_words,
                                       int32_t *d_residues, int32_t *d_status, void *stream);
/* How many streams of the last selab200_rice_decode_frames_device call the fast decoder handed to the
 * general lane-per-stream parser (streams it could not split, or that hold a symbol its windows do not
 * cover; results are identical either way).  Synchronises.  Diagnostics / bench bookkeeping. */
int selab200_rice_decode_flagged(uint32_t *n_flagged);

/* ------------------------------------------------ .sela container level -- */

/* The byte-packed file format of file::SelaFile (src/file/sela_file.cpp:19-137): 15-byte header
 * ("SeLa", sampleRate u32, bitsPerSample u16, channels u8, numFrames u32, little endian), then
 * per frame the sync word 0xAA55FF00 and per subframe
 *   channel, type, parent, reflK (u8), reflInts (u16), order (u8), refl words,
 *   resK (u8), resInts (u16), samples (u16), residue words.
 * These entry points move whole containers: the encoder's gather kernel writes the byte stream
 * in place (headers included), the decoder realigns the word arrays on the device, so the host
 * never builds per-subframe vectors (SURVEY.md 8f, row f2).  Bytes are identical to what
 * file::SelaFile::writeToFile emits for the frames selab200_encode_frames returns. */
typedef struct selab200_container_info {
    uint32_t sample_rate;
    uint16_t bits_per_sample;
    uint8_t  channels;
    uint8_t  reserved;
    uint32_t header_frames;  /* the numFrames field                                            */
    uint32_t n_frames;       /* frames present: the walk stops quietly at the first bad sync
                                word, as the reference reader does (sela_file.cpp:48-56)       */
    uint64_t n_words;        /* Rice words of those frames                                     */
    uint64_t n_bytes_used;   /* bytes of the container those frames (and the header) occupy    */
} selab200_container_info;

/* Worst-case container size for n_frames x channels subframes of 16-bit audio. */
size_t selab200_container_bound(uint32_t n_frames, uint32_t channels);

/* WAV data chunk -> complete .sela byte stream: sela::Encoder::process + file::SelaFile::writeToFile
 * (src/sela/encoder.cpp:94-99, src/file/sela_file.cpp:105-137).  pcm as in selab200_encode_frames.
 * SELAB200_ERR_CAPACITY if `capacity` bytes do not suffice (*bytes_used = the size needed). */
int selab200_encode_container(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                              uint32_t sample_rate, uint16_t bits_per_sample,
                              uint8_t *container, size_t capacity, size_t *bytes_used);

/* Host-only parse of a container (no device needed): header fields and the frame walk of
 * file::SelaFile::readFromFile (src/file/sela_file.cpp:19-103).  Errors (SELAB200_ERR_BITSTREAM)
 * carry the message the host mirror throws for the same file: too small, bad magic, truncated. */
int selab200_container_info_get(const uint8_t *container, size_t n_bytes, selab200_container_info *info);

/* Same walk, also returning where each frame starts: offsets[i] = byte position of frame i's sync
 * word, offsets[n_frames] = one past the last frame.  Frames are independent, so a byte range
 * [offsets[a], offsets[b]) behind a 15-byte header that says b-a frames is itself a container --
 * which is how a file is cut into per-GPU blocks (sela_b200/distributed.py).  Host only.
 * SELAB200_ERR_CAPACITY if capacity < n_frames + 1 (info is filled in either way). */
int selab200_container_frame_offsets(const uint8_t *container, size_t n_bytes, uint64_t *offsets,
                                     size_t capacity, selab200_container_info *info);

/* Complete .sela byte stream -> interleaved int16 PCM (the WAV data chunk):
 * file::SelaFile::readFromFile + sela::Decoder::processFrames.  open: parses the header, starts
 * the upload and walks the frame headers on the host meanwhile (the walk is a pointer chase
 * through the byte stream -- inherently serial, microseconds per thousand frames; everything
 * that touches the payload runs on the device).  `container` must stay valid until close.
 * decode: pcm_out receives info.n_frames * channels * 2048 samples. */
typedef struct selab200_container selab200_container;
int  selab200_container_open(const uint8_t *container, size_t n_bytes, selab200_container **handle,
                             selab200_container_info *info);
int  selab200_container_decode(selab200_container *handle, int16_t *pcm_out);
void selab200_container_close(selab200_container *handle);

/* A host-resident open (DESIGN.md 7.10): for a corpus larger than the device memory it may take.  The same header
 * checks, errors, messages, frame walk and info as selab200_container_open for the same bytes, but the handle copies
 * the image into page-locked host memory it owns (mapped into the devices' address space, 64 bytes of padding) and
 * allocates no device memory for it.  Unlike selab200_container_open, the caller's buffer may be freed or overwritten
 * as soon as this returns.  The handle works in every call that takes one, mixed freely with device-resident handles,
 * with results bit for bit those of a device-resident handle over the same bytes; selab200_container_close closes it.
 *   - the clip calls fetch over PCIe only the bytes of the subframes they decode: per subframe [a & ~15, (b + 15) & ~15)
 *     with a its first reflection byte and b 3 bytes past its last residue byte, merged, in selection order, with the
 *     previous range of the same container when they touch or overlap, within one decode group (the groups the clip
 *     calls document); each merged run is fetched once per group.  Device memory for the fetched bytes is bounded by
 *     one group's;
 *   - selab200_container_decode and selab200_container_verify upload each device's block of the image per call. */
int  selab200_container_open_host(const uint8_t *container, size_t n_bytes, selab200_container **handle,
                                  selab200_container_info *info);

/* Random access (DESIGN.md 7.8): a batch of clips of `length` samples each from any of n_handles open containers with
 * the same channel count.  Clip i is samples [start, start + length) of every channel of handles[clips[i].container],
 * i.e. rows start .. start + length - 1 of that container's selab200_container_decode output viewed as
 * [n_frames * 2048][channels], bit for bit.  The output is interleaved int16, [n_clips][length][channels], clips back
 * to back; nothing past n_clips * length * channels samples is written.  Every (container, frame) that some clip
 * covers is decoded exactly once per call however many clips overlap it; *frames_decoded receives their number.
 * Frames no clip covers are neither decoded nor checked: a malformed frame fails the call (SELAB200_ERR_BITSTREAM)
 * only if a clip covers it.  SELAB200_ERR_ARGUMENT, with the clip index in selab200_last_error(), for length 0, a
 * clip past its container's end (ending exactly at the end is accepted), a container index >= n_handles, a non-zero
 * reserved field, handles of different channel counts and null pointers; n_clips == 0 is SELAB200_OK and writes
 * nothing.  Device memory apart from a device-form output does not grow with n_clips: the covered frames are decoded
 * in groups (fewer frames each under SELAB200_CHUNK_FRAMES).  With several devices initialised the clips decode on the
 * primary, which holds every open image; one call's clips are not spread over devices. */
typedef struct selab200_clip {   /* 16 bytes */
    uint32_t container;          /* index into handles[]          */
    uint32_t reserved;           /* must be 0                     */
    uint64_t start;              /* first sample (per channel)    */
} selab200_clip;

/* host output: pcm_out holds n_clips * length * channels int16 */
int selab200_container_decode_clips(selab200_container *const *handles, uint32_t n_handles, const selab200_clip *clips,
                                    uint32_t n_clips, uint32_t length, int16_t *pcm_out, uint64_t *frames_decoded);
/* the same, into device memory of the primary device (2-byte aligned); synchronises: returns once the output is
 * written */
int selab200_container_decode_clips_device(selab200_container *const *handles, uint32_t n_handles,
                                           const selab200_clip *clips, uint32_t n_clips, uint32_t length,
                                           int16_t *d_pcm_out, uint64_t *frames_decoded);

/* Clips of chosen channels (DESIGN.md 7.9): the clips above, but only the channels select[0 .. n_select) (any order,
 * repeats allowed; select == NULL with n_select == 0: every channel 0 .. C-1 of each clip's own container), and only
 * the subframes those channels need are decoded.  With x the [length][C] rows of a clip as above, the output is
 * [n_clips][length][n_out], clips back to back, n_out = 1 with SELAB200_CLIP_MEAN, else the number of channels
 * selected:
 *   int16 (flags 0):  out[t][j] = x[t][select[j]], bit for bit;
 *   FLOAT32:          (float)x[t][select[j]] / 32768.0f (exact);
 *   FLOAT32 | MEAN:   (float)S / (float)(32768 * n), IEEE round-to-nearest, S the exact integer sum of the n selected
 *                     samples of the row (both operands exact: the value is defined to the last bit).
 * Containers of different channel counts may share a call, except in a full selection without MEAN (n_out must be
 * one count).  *frames_decoded is as above; *subframes_decoded receives the subframes decoded: per covered frame
 * those of the selected channels and the parents of the selected difference-coded ones, each once.  A covered frame
 * fails the call (SELAB200_ERR_BITSTREAM, before anything is decoded) when any of its subframe headers breaks the
 * decoder's descriptor and frame rules, decoded or not; a stream that ends inside its words is found only in the
 * subframes that are decoded, since only those streams are parsed.  SELAB200_ERR_ARGUMENT, with the clip index where
 * one applies, for everything the clip call rejects (except handles of different channel counts), flag bits other
 * than the two below, MEAN without FLOAT32, select == NULL with n_select != 0 or the reverse, n_select > 255, a
 * selected channel >= the channel count of a container some clip reads, and a full selection without MEAN over
 * clips of containers with different channel counts.  A rejected call writes no output. */
#define SELAB200_CLIP_FLOAT32 1u   /* float32 output instead of int16                                    */
#define SELAB200_CLIP_MEAN    2u   /* one output channel: the mean of the selected ones (needs FLOAT32) */
#define SELAB200_CLIP_MAX_SELECT 255u

/* host output: out holds n_clips * length * n_out int16 or float */
int selab200_container_decode_clips_select(selab200_container *const *handles, uint32_t n_handles,
                                           const selab200_clip *clips, uint32_t n_clips, uint32_t length,
                                           const uint8_t *select, uint32_t n_select, uint32_t flags, void *out,
                                           uint64_t *frames_decoded, uint64_t *subframes_decoded);
/* the same, into device memory of the primary device (2-byte aligned for int16, 4-byte for float32); synchronises */
int selab200_container_decode_clips_select_device(selab200_container *const *handles, uint32_t n_handles,
                                                  const selab200_clip *clips, uint32_t n_clips, uint32_t length,
                                                  const uint8_t *select, uint32_t n_select, uint32_t flags,
                                                  void *d_out, uint64_t *frames_decoded, uint64_t *subframes_decoded);

/* *bytes receives the bytes of host-resident images (selab200_container_open_host) the process's last clip call
 * fetched, by the rule above: the sum of its runs' lengths over all its groups; 0 if it read only device-resident
 * images.  SELAB200_ERR_NOT_INIT before selab200_init; diagnostics and bench bookkeeping. */
int selab200_clip_bytes_fetched(uint64_t *bytes);

/* ------------------------------------------------------------- verify -- */

/* The format is not lossless for every input: encoder and decoder round the Q35 prediction differently
 * when it lands exactly on a half (DESIGN.md 7), and from that sample on the decoded channel drifts away
 * from its source.  Verifying coded frames against PCM means decoding them exactly as
 * selab200_decode_frames does (which equals the reference decoder) and comparing with the PCM sample for
 * sample.  The report holds one entry per decoded output (frame, channel) that differs, in (frame,
 * channel) order; a wrong parent makes its difference-coded sibling wrong as well, and both appear. */
typedef struct selab200_verify_entry {   /* 16 bytes */
    uint32_t frame;          /* frame index in the batch / file                               */
    uint16_t channel;
    uint16_t first_sample;   /* 0..2047, within the frame                                      */
    uint32_t n_differing;    /* 1..2048 (0 only in the device-resident per-pair array)         */
    int32_t  first_delta;    /* decoded - source at first_sample                               */
} selab200_verify_entry;

/* Device-resident core: decode (d_descs, d_words) as selab200_decode_frames_device does and compare with
 * d_pcm_ref.  d_entries: n_frames*channels records, one per (frame, channel) in frame order, channel order;
 * a differing pair's record is filled in, every other one is zeroed (n_differing == 0).  *d_n_differing
 * (uint64, device) receives the number of differing pairs.  Stream-ordered, no synchronisation; d_status
 * as for decode (the records are all zero after a decode error).  Alignment rules as for the other *_device
 * forms; d_pcm_ref must also be 16-byte aligned (it is read as 16-byte vectors). */
size_t selab200_verify_workspace_bytes(uint32_t n_frames, uint32_t channels);
int selab200_verify_frames_device(const selab200_subframe_desc *d_descs, uint32_t n_frames, uint32_t channels,
                                  const uint32_t *d_words, size_t n_words, const int16_t *d_pcm_ref,
                                  selab200_verify_entry *d_entries, uint64_t *d_n_differing, int32_t *d_status,
                                  void *d_workspace, size_t workspace_bytes, void *stream);

/* Host-buffer forms.  A report with differences is SELAB200_OK; malformed streams fail as decode does
 * (SELAB200_ERR_BITSTREAM).  *n_entries always receives the number of differing pairs, of which the first
 * `capacity` are written to entries.  With several devices the frames are split as for the other batch
 * calls; frame indices in the report are those of the whole batch. */

/* selab200_decode_frames + compare with pcm (n_frames*2048*channels interleaved samples), pipelined. */
int selab200_verify_frames(const selab200_subframe_desc *descs, uint32_t n_frames, uint32_t channels,
                           const uint32_t *words, size_t n_words, const int16_t *pcm,
                           selab200_verify_entry *entries, size_t capacity, size_t *n_entries);

/* selab200_encode_container, and a check that the bytes it returns decode back to pcm (`flac --verify`).
 * The container bytes are identical to selab200_encode_container's.  Each chunk's byte image is unpacked
 * on the device, decoded and compared with the PCM the chunk already holds in device memory, on the
 * chunk's compute lane while the next chunk encodes: neither PCM nor bytes cross PCIe a second time. */
int selab200_encode_container_verified(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                       uint32_t sample_rate, uint16_t bits_per_sample, uint8_t *container,
                                       size_t capacity, size_t *bytes_used, selab200_verify_entry *entries,
                                       size_t entries_capacity, size_t *n_entries);

/* Instead of selab200_container_decode on an open container: compare its info.n_frames frames with pcm. */
int selab200_container_verify(selab200_container *handle, const int16_t *pcm, selab200_verify_entry *entries,
                              size_t capacity, size_t *n_entries);

/* ----------------------------------------------------------- lossless -- */

/* Encodes that decode back to their source (DESIGN.md 7.2).  A subframe has a tie when, at some sample, the
 * encoder's and the decoder's rounding of the prediction differ; it then does not decode back to its source.  The
 * lossless forms find such subframes while encoding, and in every frame where the reference encoder would emit one,
 * code each subframe candidate that has a tie with a slightly different predictor: one quantised reflection
 * coefficient moved by 1, or a lower order, whichever tie-free choice costs the fewest words.  The output is an
 * ordinary stream that the unmodified reference decoder reads; every other frame keeps the reference encoder's
 * bytes.  The report holds one entry per emitted (frame, channel) that differs from the reference encoder's, in
 * (frame, channel) order: the order and words (reflection + residue) of the reference's subframe and of the one
 * emitted.  Frame indices are those of the whole batch / file. */
typedef struct selab200_lossless_entry { /* 16 bytes */
    uint32_t frame;
    uint16_t channel;
    uint8_t  ref_order;      /* the reference encoder's subframe                                */
    uint8_t  order;          /* the emitted subframe                                            */
    uint32_t ref_words;
    uint32_t words;          /* 0 only in the device-resident per-pair array, where nothing changed */
} selab200_lossless_entry;

/* selab200_encode_frames, lossless.  *n_entries receives the number of re-coded subframes, of which the first
 * `capacity` are written to entries.  Frames are split over devices as for the other batch calls. */
int selab200_encode_frames_lossless(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                    selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                    size_t *words_used, selab200_lossless_entry *entries, size_t capacity,
                                    size_t *n_entries);

/* selab200_encode_container, lossless; report as selab200_encode_frames_lossless. */
int selab200_encode_container_lossless(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                       uint32_t sample_rate, uint16_t bits_per_sample, uint8_t *container,
                                       size_t capacity, size_t *bytes_used, selab200_lossless_entry *entries,
                                       size_t entries_capacity, size_t *n_entries);

/* Device-resident form of selab200_encode_frames_lossless: arguments as selab200_encode_frames_device, with
 * selab200_encode_lossless_workspace_bytes() of workspace.  d_entries: n_frames*channels records, one per
 * (frame, channel) in frame order, channel order; a re-coded pair's record is filled in, every other one is zeroed
 * (words == 0).  *d_n_entries (uint64, device) receives the number of re-coded pairs.  Stream-ordered, no
 * synchronisation: the repair runs on the device whatever it finds. */
size_t selab200_encode_lossless_workspace_bytes(uint32_t n_frames, uint32_t channels);
int selab200_encode_frames_lossless_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                           selab200_subframe_desc *d_descs, uint32_t *d_words,
                                           size_t words_capacity, uint64_t *d_words_used,
                                           selab200_lossless_entry *d_entries, uint64_t *d_n_entries,
                                           int32_t *d_status, void *d_workspace, size_t workspace_bytes,
                                           void *stream);

/* ------------------------------------------------------- order search -- */

/* Smaller files at a higher encode cost (DESIGN.md 7.3), like `flac -8`.  The reference encoder takes the predictor
 * order from a threshold on the reflection coefficients; the search forms code every analysis unit (a channel, or
 * for stereo ch0, ch1 and ch0 - ch1) at the order 1..100 with the fewest words (reflection + residue) among those
 * whose FIR has no tie, so that every subframe decodes back to its source under the reference decoder.  Between equal
 * words the reference encoder's order wins if it is among them, else the lowest order.  The stereo decision then runs
 * as always on the searched units.  The output is an ordinary stream that the unmodified reference decoder reads.
 * *ref_words receives the words the reference encoder's choice takes for the same frames (the words_used of
 * selab200_encode_frames), so that the caller sees the saving.  Frames are split over devices as for the other batch
 * calls. */
int selab200_encode_frames_search(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                  selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                  size_t *words_used, size_t *ref_words);

/* selab200_encode_container, with the order search; *ref_bytes receives the size of selab200_encode_container's
 * output for the same frames. */
int selab200_encode_container_search(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                     uint32_t sample_rate, uint16_t bits_per_sample, uint8_t *container,
                                     size_t capacity, size_t *bytes_used, size_t *ref_bytes);

/* Device-resident form of selab200_encode_frames_search: arguments as selab200_encode_frames_device, with
 * selab200_encode_search_workspace_bytes() of workspace; *d_ref_words (uint64, device) receives the reference
 * encoder's words.  Stream-ordered, no synchronisation. */
size_t selab200_encode_search_workspace_bytes(uint32_t n_frames, uint32_t channels);
int selab200_encode_frames_search_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                         selab200_subframe_desc *d_descs, uint32_t *d_words, size_t words_capacity,
                                         uint64_t *d_words_used, uint64_t *d_ref_words, int32_t *d_status,
                                         void *d_workspace, size_t workspace_bytes, void *stream);

/* ----------------------------------------------- guided order search -- */

/* Most of the order search's saving at a fraction of its cost (DESIGN.md 7.7), like the middle presets of other
 * lossless codecs.  Each analysis unit is searched as selab200_encode_frames_search searches it, but only over the
 * `candidates` (K, 1..100) orders an estimate ranks best, order 1 and the reference encoder's order.  The estimate of
 * order o is E_o = P_o * r^o, with P_1 = 1 and P_o = prod_{i<o} (1 - k_i^2) over the dequantised reflection
 * coefficients k_i, and r = 2^(1/256) (4 bits per coefficient over a 2048-sample frame); orders rank by (E_o, o),
 * lower first.  The winner and tie rules are the order search's, so every unit takes at least the order search's
 * words, and at most the reference encoder's where its order has no tie; every output decodes back to its source
 * under this decoder and the unmodified reference decoder; K = 100 is byte-identical to the order search.  A
 * candidate count of 0 or above 100 -> SELAB200_ERR_ARGUMENT.  *ref_words as selab200_encode_frames_search's.  Frames
 * are split over devices as for the other batch calls. */
int selab200_encode_frames_search_guided(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t candidates,
                                         selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                         size_t *words_used, size_t *ref_words);

/* selab200_encode_container, with the guided order search; *ref_bytes receives the size of
 * selab200_encode_container's output for the same frames. */
int selab200_encode_container_search_guided(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                            uint32_t candidates, uint32_t sample_rate, uint16_t bits_per_sample,
                                            uint8_t *container, size_t capacity, size_t *bytes_used,
                                            size_t *ref_bytes);

/* Device-resident form of selab200_encode_frames_search_guided: arguments as selab200_encode_frames_device, with
 * selab200_encode_search_guided_workspace_bytes() of workspace; *d_ref_words (uint64, device) receives the reference
 * encoder's words.  Stream-ordered, no synchronisation. */
size_t selab200_encode_search_guided_workspace_bytes(uint32_t n_frames, uint32_t channels);
int selab200_encode_frames_search_guided_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                                uint32_t candidates, selab200_subframe_desc *d_descs, uint32_t *d_words,
                                                size_t words_capacity, uint64_t *d_words_used, uint64_t *d_ref_words,
                                                int32_t *d_status, void *d_workspace, size_t workspace_bytes,
                                                void *stream);

/* ---------------------------------------------------- channel pairing -- */

/* Smaller files of correlated channels at a higher encode cost (DESIGN.md 7.4).  The format can code any channel of
 * a frame as `parent - difference` against any independently coded channel of the frame; the reference encoder only
 * ever tries channel 1 against channel 0 of a stereo file.  The pairing forms start from the lossless encode, size
 * the difference ch_p - ch_c of every ordered pair of channels of every frame, coded as the stereo difference is, and
 * emit per frame the assignment (each channel alone, or against one independently coded parent) with the fewest words
 * in total; between equal totals the fewest difference subframes, then the lexicographically smallest parent vector.
 * A subframe whose FIR has a tie is never emitted, so every output decodes back to its source, under this decoder and
 * under the unmodified reference decoder.  A frame in which no difference wins keeps the bytes of the lossless encode.
 * channels == 1 is the lossless encode.  *base_words receives the words_used of selab200_encode_frames_lossless for
 * the same frames (words_used <= base_words always), *n_difference the number of difference subframes emitted.
 * Frames are split over devices as for the other batch calls. */
int selab200_encode_frames_pairing(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                   selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                   size_t *words_used, size_t *base_words, size_t *n_difference);

/* selab200_encode_container, with the pairing; *base_bytes receives the size of selab200_encode_container_lossless's
 * output for the same frames. */
int selab200_encode_container_pairing(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                      uint32_t sample_rate, uint16_t bits_per_sample, uint8_t *container,
                                      size_t capacity, size_t *bytes_used, size_t *base_bytes, size_t *n_difference);

/* Device-resident form of selab200_encode_frames_pairing: arguments as selab200_encode_frames_device, with
 * selab200_encode_pairing_workspace_bytes() of workspace; *d_base_words and *d_n_difference (uint64, device) receive
 * the two totals.  Stream-ordered, no synchronisation. */
size_t selab200_encode_pairing_workspace_bytes(uint32_t n_frames, uint32_t channels);
int selab200_encode_frames_pairing_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                          selab200_subframe_desc *d_descs, uint32_t *d_words, size_t words_capacity,
                                          uint64_t *d_words_used, uint64_t *d_base_words, uint64_t *d_n_difference,
                                          int32_t *d_status, void *d_workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------ order search + pairing -- */

/* The smallest files of these encodes, at the highest encode cost (DESIGN.md 7.5): the order search and the channel
 * pairing together, like the "maximum" setting of other lossless codecs.  The base is selab200_encode_frames_search's
 * encode of the frame; then every ordered pair (p, c), p != c, of a frame is the difference ch_p - ch_c coded at its
 * searched order (the order 1..100 with the fewest words whose FIR has no tie; between equal words the reference
 * encoder's order, else the lowest), and the pairing's choice runs on these words: the assignment with the fewest
 * words in total, then the fewest difference subframes, then the lexicographically smallest parent vector.  Every
 * frame takes at most the words of selab200_encode_frames_search on it, and every output decodes back to its source
 * under this decoder and the unmodified reference decoder.  channels == 1 is the order search.  *base_words receives
 * the words_used of selab200_encode_frames_search for the same frames (words_used <= base_words always),
 * *n_difference the number of difference subframes emitted.  Frames are split over devices as for the other batch
 * calls. */
int selab200_encode_frames_search_pairing(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                          selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                          size_t *words_used, size_t *base_words, size_t *n_difference);

/* selab200_encode_container, with the search + pairing; *base_bytes receives the size of
 * selab200_encode_container_search's output for the same frames. */
int selab200_encode_container_search_pairing(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                             uint32_t sample_rate, uint16_t bits_per_sample, uint8_t *container,
                                             size_t capacity, size_t *bytes_used, size_t *base_bytes,
                                             size_t *n_difference);

/* Device-resident form of selab200_encode_frames_search_pairing: arguments as selab200_encode_frames_device, with
 * selab200_encode_search_pairing_workspace_bytes() of workspace; *d_base_words and *d_n_difference (uint64, device)
 * receive the two totals.  Stream-ordered, no synchronisation. */
size_t selab200_encode_search_pairing_workspace_bytes(uint32_t n_frames, uint32_t channels);
int selab200_encode_frames_search_pairing_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                                 selab200_subframe_desc *d_descs, uint32_t *d_words,
                                                 size_t words_capacity, uint64_t *d_words_used, uint64_t *d_base_words,
                                                 uint64_t *d_n_difference, int32_t *d_status, void *d_workspace,
                                                 size_t workspace_bytes, void *stream);

/* ------------------------------------------------------ window search -- */

/* The order search with apodised analyses (DESIGN.md 7.6), like the apodisation option of other lossless codecs.
 * Each analysis unit is coded as selab200_encode_frames_search codes it, unless one of the selected windows does
 * strictly better: the unit's signal minus its mean, multiplied by the window, is analysed as the reference analyses
 * the plain signal (autocorrelation, Schur recursion, all 100 quantised coefficients, each clamped to [-64, 63]),
 * and searched over orders 1..100 as the order search does (the FIR of every order with its tie check, both Rice
 * sizes; an order whose predictor leaves the domain of the Q35 conversion counts as tied).  The unit takes the
 * tie-free window candidate with the fewest words if that is strictly fewer than the order search's winner (between
 * equal words the lower window bit, then the lower order).  The stereo decision then runs as always.  So every frame
 * takes at most the words of selab200_encode_frames_search, a file no window improves is byte-identical to it, and
 * every output decodes back to its source under this decoder and the unmodified reference decoder.
 *
 * windows: a mask over the rows of the fixed window table (selab200_analysis_window): bit 0 Tukey(0.5), 1 Tukey(0.25),
 * 2 Hann, 3 Tukey(0.5) over samples 0..1023 and zero after, 4 Tukey(0.5) over samples 1024..2047 and zero before.  A
 * mask of 0 or with a bit above 4 -> SELAB200_ERR_ARGUMENT.  Each window costs about one more order search.
 * *base_words receives the words_used of selab200_encode_frames_search for the same frames, *n_window the number of
 * analysis units (channels; for stereo ch0, ch1 and ch0 - ch1) coded from a window.  Frames are split over devices
 * as for the other batch calls. */
int selab200_encode_frames_search_windows(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t windows,
                                          selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                          size_t *words_used, size_t *base_words, size_t *n_window);

/* selab200_encode_container, with the window search; *base_bytes receives the size of
 * selab200_encode_container_search's output for the same frames. */
int selab200_encode_container_search_windows(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                             uint32_t windows, uint32_t sample_rate, uint16_t bits_per_sample,
                                             uint8_t *container, size_t capacity, size_t *bytes_used,
                                             size_t *base_bytes, size_t *n_window);

/* Device-resident form of selab200_encode_frames_search_windows: arguments as selab200_encode_frames_device, with
 * selab200_encode_search_windows_workspace_bytes() of workspace (it grows with the number of windows in the mask);
 * *d_base_words and *d_n_window (uint64, device) receive the two totals.  Stream-ordered, no synchronisation. */
size_t selab200_encode_search_windows_workspace_bytes(uint32_t n_frames, uint32_t channels, uint32_t windows);
int selab200_encode_frames_search_windows_device(const int16_t *d_pcm, uint32_t n_frames, uint32_t channels,
                                                 uint32_t windows, selab200_subframe_desc *d_descs, uint32_t *d_words,
                                                 size_t words_capacity, uint64_t *d_words_used, uint64_t *d_base_words,
                                                 uint64_t *d_n_window, int32_t *d_status, void *d_workspace,
                                                 size_t workspace_bytes, void *stream);

/* Row `index` (0..4) of the window table into out[2048]: the exact doubles the window search multiplies by.  Needs
 * no device and no selab200_init.  Another index or a null out -> SELAB200_ERR_ARGUMENT. */
int selab200_analysis_window(int index, double *out);

/* ------------------------------------------ stage level (host buffers) -- */

/* lpc::ResidueGenerator::process (src/lpc/residue_generator.cpp:121-134) for
 * n_sub independent 2048-sample signals.  samples: [n_sub][2048] int32 in the
 * 17-bit domain |s| <= 65535 (16-bit channels and their L-R difference).
 * Outputs: order[n_sub]; q[n_sub][100] (first order[i] valid, rest 0);
 * residues[n_sub][2048]. */
int selab200_lpc_residues(const int32_t *samples, uint32_t n_sub, uint8_t *order,
                          int32_t *q, int32_t *residues);

/* lpc::SampleGenerator::process (src/lpc/sample_generator.cpp:32-39) for n_sub independent
 * 2048-sample residue signals.  order[i] <= 100 (larger is clamped to 100); q: [n_sub][100], the
 * first order[i] used, each in [-64, 63] (values outside are clamped to the table ends, where the
 * reference reads out of bounds).  residues: any int32.  samples[n_sub][2048] equal the reference's
 * wherever its int64 arithmetic does not overflow (every partial prediction sum below 2^62 in
 * magnitude) and every sample fits in int32; outside that the reference is undefined. */
int selab200_lpc_samples(const int32_t *residues, uint32_t n_sub, const uint8_t *order,
                         const int32_t *q, int32_t *samples);

/* rice::RiceEncoder::process (src/rice/rice_encoder.cpp:73-81) for n_streams
 * independent inputs.  values: [n_streams][stride] int32, counts[i] <= stride
 * <= 2048 used from row i.  Outputs per stream: rice_param, n_words, and the
 * words at words[i*words_stride ...]; SELAB200_ERR_CAPACITY if a stream needs
 * more than words_stride words (n_words[] still holds the required sizes). After
 * SELAB200_ERR_CAPACITY, rice_param[] holds every stream's parameter and every
 * stream that fits has its words; the rows of the others are undefined. */
int selab200_rice_encode(const int32_t *values, const uint32_t *counts, uint32_t n_streams,
                         uint32_t stride, uint32_t *rice_param, uint32_t *n_words,
                         uint32_t *words, uint32_t words_stride);

/* rice::RiceDecoder::process (src/rice/rice_decoder.cpp:54-61) for n_streams
 * inputs: words[i*words_stride ... +n_words[i]) -> out[i*out_stride ... +counts[i]).
 * Reads past n_words[i] see zero bits (the reference would read out of bounds). */
int selab200_rice_decode(const uint32_t *words, const uint32_t *n_words, uint32_t words_stride,
                         const uint32_t *rice_param, const uint32_t *counts, uint32_t n_streams,
                         int32_t *out, uint32_t out_stride);

/* --------------------------------------------------- tests: internals -- */

/* The floating-point analysis of one analysis unit of the batch encoder, as the encoder computed it:
 * the intermediates of lpc::ResidueGenerator (src/lpc/residue_generator.cpp:20-96) and the predictor
 * of LinearPredictor::generatelinearPredictionCoefficients (src/lpc/linear_predictor.cpp:30-61).
 * 2 832 bytes, naturally aligned. */
typedef struct selab200_analysis_trace {
    double  mean;     /* mean of s/32767                                       */
    double  ac[101];  /* autocorrelation lags 0..100 after normalisation       */
    double  k[100];   /* reflection coefficients from the Schur recursion      */
    int64_t c[101];   /* Q35 predictor, c[0] = 0, zero past the order          */
    int32_t q[100];   /* quantised k, zero past the order                      */
    int32_t order;
    int32_t reserved; /* zero                                                  */
} selab200_analysis_trace;

/* For tests: selab200_encode_frames on one device and one batch, through the same kernels except that the
 * analysis kernel is its tracing instantiation, which also writes every analysis unit's intermediates to
 * trace.  The units are frame after frame; within a frame channel 0..channels-1, or for stereo channel 0,
 * channel 1 and the difference channel 0 - channel 1.  trace: n_frames*3 records for stereo, else
 * n_frames*channels.  descs, words and *words_used as selab200_encode_frames. */
int selab200_encode_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                          selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                          size_t *words_used, selab200_analysis_trace *trace);

/* For tests: the encoder's order threshold and reflection-coefficient quantiser on chosen values
 * (src/lpc/residue_generator.cpp:70-96), the device functions the encoder runs.  For every k[i]:
 * out[4i+0], out[4i+1], out[4i+2] = q of k[i] as coefficient 0, as coefficient 1 and as any later
 * coefficient; out[4i+3] = 1 if |k[i]| > 0.05, else 0. */
int selab200_quantise_probe(const double *k, size_t n, int32_t *out);

/* For tests: the encoder's FIR residual (src/lpc/residue_generator.cpp:98-119), the device function the encoder
 * runs, on chosen signals and predictors.  samples: [n][2048]; wide = 0 stages them as the int16 row of a channel
 * unit (-32768..32767), wide != 0 as the row and parity bits of a 17-bit unit (|s| <= 65535); anything outside
 * -> SELAB200_ERR_RANGE.  orders[n] in 0..100; c: [n][101], the Q35 predictor, c[i][1..orders[i]] used (any int64).
 * residues: [n][2048], s[t] - (int32)((2^34 + sum_j c[j] * s[t-j]) >> 35) with the sum taken mod 2^64. */
int selab200_fir_probe(const int32_t *samples, const int32_t *orders, const int64_t *c, uint32_t n, int wide,
                       int32_t *residues);

/* For tests: selab200_fir_probe through the instantiation of the FIR that the lossless encode runs, which also tests
 * every output for a tie: (int32)((2^34 + sum) >> 35) + (int32)((2^34 - sum) >> 35) != 0, both sums taken mod
 * 2^64 (DESIGN.md 7.2).  Arguments and domain as selab200_fir_probe; ties[n] receives 1 for a signal with a tie
 * at any output, else 0. */
int selab200_fir_tie_probe(const int32_t *samples, const int32_t *orders, const int64_t *c, uint32_t n, int wide,
                           int32_t *residues, uint8_t *ties);

/* A quantised predictor: the order and the quantised reflection coefficients, zero past the order. */
typedef struct selab200_predictor { /* 404 bytes */
    int32_t order;   /* 0..100 */
    int32_t q[100];  /* [-64, 63] */
} selab200_predictor;

/* For tests: selab200_encode_frames_lossless on one device and one batch, except that every analysis unit is coded
 * with the predictor pred[unit] instead of the one its analysis chooses.  pred holds one record per analysis unit,
 * in the order of selab200_encode_trace's.  Everything after the quantiser runs as in the lossless encode: the tie
 * test, the repair (whose candidates edit the given predictor), the stereo decision and the report.  A predictor
 * outside the domain (order, q or a non-zero q past the order) -> SELAB200_ERR_RANGE.  The other arguments as
 * selab200_encode_frames_lossless. */
int selab200_encode_lossless_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                    const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                    size_t words_capacity, size_t *words_used, selab200_lossless_entry *entries,
                                    size_t entries_capacity, size_t *n_entries);

/* For tests: selab200_encode_frames_search on one device and one batch, except that every analysis unit takes
 * pred[unit].q[0..99] as its 100 quantised reflection coefficients (values past the order included) and
 * pred[unit].order as the reference encoder's order, instead of what its analysis gives.  pred holds one record per
 * analysis unit, in the order of selab200_encode_trace's.  An order outside 1..100 or any q outside [-64, 63] ->
 * SELAB200_ERR_RANGE.  The other arguments as selab200_encode_frames_search. */
int selab200_encode_search_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                  const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                  size_t words_capacity, size_t *words_used, size_t *ref_words);

/* One candidate order of one analysis unit in the order search, as the search sized it.  32 bytes, naturally
 * aligned.  With K = 0x9E3779B97F4A7C15 and K2 = 0xD6E8FEB86659FD93, all sums mod 2^64:
 *   pred_digest = sum_{j=1..100} (c[j] + j * K2) * K, c the Q35 predictor the FIR ran (zero past the order);
 *   res_digest  = sum_{i<2048} ((i << 32) | (uint32)r[i]) * K, r the residues.
 * Every term is a bijection of its element, so any one changed coefficient or residue changes the digest. */
typedef struct selab200_search_trace {
    uint64_t pred_digest;
    uint64_t res_digest;
    uint32_t res_words;  /* residue Rice words                                               */
    uint32_t visits;     /* how many times the order was sized (atomic): 1                   */
    uint16_t refl_words; /* reflection-coefficient Rice words                                */
    uint8_t  refl_k;     /* reflection-coefficient Rice parameter                            */
    uint8_t  res_k;      /* residue Rice parameter                                           */
    uint8_t  tie;        /* 1 if the FIR has a tie at any output                             */
    uint8_t  reserved[3];
} selab200_search_trace;

/* What the order search's analysis left for one analysis unit: every quantised reflection coefficient, the
 * reference encoder's order and its words, and the winner's key words << 8 | (order == ref_order ? 0 : order).
 * 416 bytes. */
typedef struct selab200_search_unit {
    int32_t  q[100];
    uint32_t ref_order;
    uint32_t ref_words;
    uint64_t best;
} selab200_search_unit;

/* For tests: selab200_encode_frames_search on one device and one batch (selab200_encode_search_forced's when pred
 * is not NULL), through the tracing instantiations of the search kernels.  trace[unit * 100 + order - 1] receives
 * the record of every analysis unit at every order 1..100: the reference order's from the analysis kernel, every
 * other order's from the candidate kernel.  units[unit] receives the unit's search record once the candidates have
 * run.  descs, words, *words_used and *ref_words as selab200_encode_frames_search. */
int selab200_encode_search_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                 const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                 size_t words_capacity, size_t *words_used, size_t *ref_words,
                                 selab200_search_unit *units, selab200_search_trace *trace);

/* For tests: selab200_encode_frames_pairing on one device and one batch, except that every unit is coded with a given
 * predictor, as selab200_encode_lossless_forced codes the base's.  pred holds the base's analysis units first, in
 * selab200_encode_trace's order, then one record per candidate in (frame, p, c) order with the p = c entries skipped
 * (n_frames * channels * (channels - 1) records; stereo (0, 1) is the base's difference unit and its record is not
 * read).  A predictor outside the domain -> SELAB200_ERR_RANGE. */
int selab200_encode_pairing_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                   const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                   size_t words_capacity, size_t *words_used, size_t *base_words,
                                   size_t *n_difference);

/* For tests: selab200_encode_frames_pairing on one device and one batch (selab200_encode_pairing_forced's when pred is
 * not NULL), and what the pairing kernels saw.  trace[(frame * channels + p) * channels + c] receives the record of
 * the candidate ch_p - ch_c as it was sized, in the layout of the order search's trace with the candidate's order in
 * reserved[0]; every p != c is visited once, except stereo (0, 1), which is the base's unit and is not sized again
 * (visits 0), and the p = c records stay zero.  par[frame * channels + c] receives the parent chosen for channel c
 * (c itself: coded alone). */
int selab200_encode_pairing_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                  const selab200_predictor *pred, selab200_subframe_desc *descs, uint32_t *words,
                                  size_t words_capacity, size_t *words_used, size_t *base_words, size_t *n_difference,
                                  uint8_t *par, selab200_search_trace *trace);

/* For tests: selab200_encode_frames_search_pairing on one device and one batch, except that every unit and every
 * candidate takes its q[0..99] and reference order from pred, as selab200_encode_search_forced takes them.  pred holds
 * the base's analysis units first, in selab200_encode_trace's order, then one record per candidate in (frame, p, c)
 * order with the p = c entries skipped, as selab200_encode_pairing_forced orders them (stereo (0, 1) is the base's
 * searched difference unit and its record is not read).  An order outside 1..100 or a q outside [-64, 63] ->
 * SELAB200_ERR_RANGE. */
int selab200_encode_search_pairing_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                          const selab200_predictor *pred, selab200_subframe_desc *descs,
                                          uint32_t *words, size_t words_capacity, size_t *words_used,
                                          size_t *base_words, size_t *n_difference);

/* For tests: selab200_encode_frames_search_pairing on one device and one batch
 * (selab200_encode_search_pairing_forced's when pred is not NULL), through the tracing instantiations of the
 * candidate kernels.  trace[((frame * channels + p) * channels + c) * 100 + order - 1] receives the record of the
 * candidate ch_p - ch_c at every order 1..100: the reference order's from the analysis kernel, every other order's
 * from the search kernel.  Stereo (0, 1), which is the base's unit, and the p = c records keep visits 0.
 * par[frame * channels + c] receives the parent chosen for channel c (c itself: coded alone). */
int selab200_encode_search_pairing_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                         const selab200_predictor *pred, selab200_subframe_desc *descs,
                                         uint32_t *words, size_t words_capacity, size_t *words_used,
                                         size_t *base_words, size_t *n_difference, uint8_t *par,
                                         selab200_search_trace *trace);

/* For tests: selab200_encode_frames_search_windows on one device and one batch, except that every analysis unit and
 * every (unit, window) record takes its q[0..99] from pred.  pred holds the units first, as
 * selab200_encode_search_forced takes them (q[0..99] and a reference order 1..100), then n_units * popcount(windows)
 * records in (unit, window) order, windows in increasing bit order, whose q[0..99] are the window analyses' (their
 * order, 0..100, is not read).  A value out of range -> SELAB200_ERR_RANGE. */
int selab200_encode_search_windows_forced(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t windows,
                                          const selab200_predictor *pred, selab200_subframe_desc *descs,
                                          uint32_t *words, size_t words_capacity, size_t *words_used,
                                          size_t *base_words, size_t *n_window);

/* For tests: selab200_encode_frames_search_windows on one device and one batch with the n_windows (1..5) windows
 * windows[n_windows][2048] in place of the table's (selab200_encode_search_windows_forced's q when pred is not NULL),
 * through the tracing candidate kernel.  trace[((unit * n_windows) + w) * 100 + order - 1] receives the record of
 * unit `unit` (selab200_encode_trace's order) coded from window w at every order 1..100; keys[unit] receives the
 * unit's best window candidate as words << 16 | w << 8 | order (all ones: none). */
int selab200_encode_search_windows_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                                         const double *windows, uint32_t n_windows, const selab200_predictor *pred,
                                         selab200_subframe_desc *descs, uint32_t *words, size_t words_capacity,
                                         size_t *words_used, size_t *base_words, size_t *n_window,
                                         selab200_search_trace *trace, uint64_t *keys);

/* For tests: selab200_encode_frames_search_guided on one device and one batch (with pred, every unit's q[0..99] and
 * reference order from it, as selab200_encode_search_forced takes them), through the tracing instantiations of the
 * search kernels.  trace[unit * 100 + order - 1] receives the record of every order sized (the reference order's
 * from the analysis kernel, every other listed order's from the listed-order kernel); the records of unlisted orders
 * keep visits 0.  estimates[unit * 100 + order - 1] receives E_order, masks[unit * 4 + (order - 1) / 32] bit
 * (order - 1) % 32 whether the order is listed. */
int selab200_encode_search_guided_trace(const int16_t *pcm, uint32_t n_frames, uint32_t channels, uint32_t candidates,
                                        const selab200_predictor *pred, selab200_subframe_desc *descs,
                                        uint32_t *words, size_t words_capacity, size_t *words_used, size_t *ref_words,
                                        selab200_search_trace *trace, double *estimates, uint32_t *masks);

#ifdef __cplusplus
}
#endif
#endif /* SELA_B200_H_ */
