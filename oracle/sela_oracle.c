/*
 * sela_oracle.c -- plain-C CPU restatement of SELA's per-frame hot path.
 *
 * TEST INFRASTRUCTURE ONLY (see sela_oracle.h).  Build: oracle/Makefile, which
 * passes -O2 -ffp-contract=off: the reference is compiled by GCC for baseline
 * x86-64 (no FMA), every double operation rounds once, and the arithmetic below
 * keeps the reference's operation ORDER (sums are sequential in j, products
 * round before they are added) because the doubles are floored/thresholded into
 * integers that reach the bitstream (SURVEY.md 7.3-H1).
 *
 * Citations are /root/reference-relative file:line.
 */
#define _POSIX_C_SOURCE 200809L
#include "sela_oracle.h"

#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include "lpc_tables.inc"

#define MAXO SELA_ORACLE_MAX_ORDER

static double bits2d(unsigned long long b)
{
    double d;
    memcpy(&d, &b, sizeof d);
    return d;
}

/* Table look-ups of LinearPredictor::dequantizeReflectionCoefficients
 * (src/lpc/linear_predictor.cpp:23-27; tables src/include/lpc.hpp:10-71).
 * The reference indexes q+64 without a bound check (UB outside [-64,63]); the
 * oracle clamps, which is the behaviour the CUDA path documents too. */
static int clamp_idx(int32_t q)
{
    int i = q + 64;
    return i < 0 ? 0 : (i > 127 ? 127 : i);
}
static double deq_first(int32_t q) { return bits2d(sela_oracle_FIRST_BITS[clamp_idx(q)]); }
static double deq_second(int32_t q)
{
    int i = clamp_idx(q);
    return i == 0 ? bits2d(SELA_ORACLE_SECOND0_BITS) : -bits2d(sela_oracle_FIRST_BITS[i]);
}
static double deq_higher(int32_t q) { return (double)(clamp_idx(q) - 64) / 64.0; }

const char *sela_oracle_kind(void) { return "port"; }

int sela_oracle_online_cores(void)
{
    long n = sysconf(_SC_NPROCESSORS_ONLN);
    return n > 0 ? (int)n : 1;
}

/* ------------------------------------------------------------------ LPC -- */

/* src/lpc/linear_predictor.cpp:16-61 */
void sela_oracle_lpc_coefficients(const int32_t *q, uint8_t order, int64_t *c)
{
    double khat[MAXO];
    double t[MAXO];
    int n_k;

    /* dequantize: order <= 1 collapses to a single zero coefficient (:19-22) */
    if (order <= 1) {
        khat[0] = 0.0;
        n_k = 1;
    } else {
        khat[0] = deq_first(q[0]);
        khat[1] = deq_second(q[1]);
        for (int i = 2; i < order; i++)
            khat[i] = deq_higher(q[i]);
        n_k = order;
    }
    (void)n_k;

    /* step-up recursion, in place, pairs (j, i-1-j) updated from OLD values (:39-50) */
    for (int i = 0; i < order; i++) {
        t[i] = khat[i];
        int half = i >> 1;
        int j;
        for (j = 0; j < half; j++) {
            double old_j = t[j];
            t[j] = t[j] + khat[i] * t[i - 1 - j];
            t[i - 1 - j] = t[i - 1 - j] + khat[i] * old_j;
        }
        if (i & 1)
            t[j] = t[j] + t[j] * khat[i];
    }

    /* Q35 conversion, truncation toward zero (:57-60); 2^35 is exact in double */
    const double scale = 34359738368.0;
    c[0] = 0;
    for (int m = 0; m < order; m++)
        c[1 + m] = (int64_t)(scale * (-t[m]));
}

/* quantizeReflectionCoefficients (src/lpc/residue_generator.cpp:80-96) for coefficient i of value k */
static int32_t quantise_one(int i, double k)
{
    const double sqrt2 = 1.4142135623730950488016887242096; /* lpc.hpp:9 */
    double v;
    if (i == 0)
        v = floor(64.0 * (-1.0 + (sqrt2 * sqrt(k + 1.0))));
    else if (i == 1)
        v = floor(64.0 * (-1.0 + (sqrt2 * sqrt(-k + 1.0))));
    else
        v = floor(64.0 * k);
    return isnan(v) ? 0 : (int32_t)v;
}

void sela_oracle_quantise_probe(const double *k, size_t n, int32_t *out)
{
    for (size_t i = 0; i < n; i++) {
        out[4 * i + 0] = quantise_one(0, k[i]);
        out[4 * i + 1] = quantise_one(1, k[i]);
        out[4 * i + 2] = quantise_one(2, k[i]);
        out[4 * i + 3] = fabs(k[i]) > 0.05; /* generateoptimalLpcOrder, :73 */
    }
}

const char *sela_oracle_internals(void) { return "ac refl mean quantise"; }

/* quantizeSamples (src/lpc/residue_generator.cpp:12-18) into x[n] and the mean of
 * generateAutoCorrelation (:26-30): true division by INT16_MAX (lpc.hpp:93), one sequential sum */
static double samples_and_mean(const int32_t *s, size_t n, double *x)
{
    for (size_t j = 0; j < n; j++)
        x[j] = (double)s[j] / 32767.0;
    double sum = 0.0;
    for (size_t j = 0; j < n; j++)
        sum = sum + x[j];
    return sum / (double)n;
}

double sela_oracle_lpc_mean(const int32_t *s, size_t n)
{
    double *x = (double *)malloc(n * sizeof(double));
    const double mean = samples_and_mean(s, n, x);
    free(x);
    return mean;
}

/* src/lpc/residue_generator.cpp:12-134 */
void sela_oracle_lpc_analyse(const int32_t *s, size_t n, uint8_t *order_out, int32_t *q,
                             int64_t *c, int32_t *res, double *refl_out, double *ac_out)
{
    double *x = (double *)malloc(n * sizeof(double));
    double *d = (double *)malloc(n * sizeof(double));
    double ac[MAXO + 1];
    double k[MAXO];
    double g0[MAXO], g1[MAXO];
    int32_t q_local[MAXO];
    int64_t c_local[MAXO + 1];

    /* generateAutoCorrelation (:20-45): sequential sum, sequential lags */
    const double mean = samples_and_mean(s, n, x);
    for (size_t j = 0; j < n; j++)
        d[j] = x[j] - mean;            /* same value every time the reference recomputes it */
    for (size_t i = 0; i <= MAXO; i++) {
        double a = 0.0;
        for (size_t j = i; j < n; j++) {
            double p = d[j] * d[j - i];
            a = a + p;
        }
        ac[i] = a;
    }
    for (size_t i = 1; i <= MAXO; i++)
        ac[i] = ac[i] / ac[0];
    ac[0] = 1.0;
    if (ac_out)
        memcpy(ac_out, ac, sizeof ac);

    /* generateReflectionCoefficients (:47-68): Schur, always all 100 */
    for (int i = 0; i < MAXO; i++)
        g0[i] = g1[i] = ac[i + 1];
    double err = ac[0];
    k[0] = -g1[0] / err;
    err = err + g1[0] * k[0];
    for (int i = 1; i < MAXO; i++) {
        double kp = k[i - 1];
        for (int j = 0; j < MAXO - i; j++) {
            double up = g1[j + 1];     /* both updates read the not-yet-overwritten g1[j+1] */
            g1[j] = up + kp * g0[j];
            g0[j] = up * kp + g0[j];
        }
        k[i] = -g1[0] / err;
        err = err + g1[0] * k[i];
    }
    if (refl_out)
        memcpy(refl_out, k, sizeof k);

    /* generateoptimalLpcOrder (:70-78); default 1 (lpc.hpp:76) */
    uint8_t order = 1;
    for (int i = MAXO - 1; i >= 0; i--) {
        if (fabs(k[i]) > 0.05) {
            order = (uint8_t)(i + 1);
            break;
        }
    }

    /* quantizeReflectionCoefficients (:80-96) */
    for (int i = 0; i < order; i++)
        q_local[i] = quantise_one(i, k[i]);

    sela_oracle_lpc_coefficients(q_local, order, c_local);

    /* generateResidues (:98-119) */
    if (res) {
        const int64_t half = (int64_t)1 << (SELA_ORACLE_Q - 1);
        res[0] = s[0];
        for (size_t i = 1; i <= (size_t)order && i < n; i++) {
            int64_t acc = half;
            for (size_t j = 1; j <= i; j++)
                acc += c_local[j] * (int64_t)s[i - j];
            res[i] = s[i] - (int32_t)(acc >> SELA_ORACLE_Q);
        }
        for (size_t i = (size_t)order + 1; i < n; i++) {
            int64_t acc = half;
            for (size_t j = 0; j <= (size_t)order; j++)
                acc += c_local[j] * (int64_t)s[i - j];
            res[i] = s[i] - (int32_t)(acc >> SELA_ORACLE_Q);
        }
    }

    *order_out = order;
    if (q)
        memcpy(q, q_local, order * sizeof(int32_t));
    if (c)
        memcpy(c, c_local, ((size_t)order + 1) * sizeof(int64_t));
    free(x);
    free(d);
}

/* src/lpc/sample_generator.cpp:11-39 */
void sela_oracle_lpc_synthesise(const int32_t *res, size_t n, uint8_t order, const int32_t *q,
                                int32_t *s)
{
    int64_t c[MAXO + 1];
    sela_oracle_lpc_coefficients(q, order, c);
    const int64_t half = (int64_t)1 << (SELA_ORACLE_Q - 1);

    memset(s, 0, n * sizeof(int32_t));
    s[0] = res[0];
    for (size_t i = 1; i <= (size_t)order && i < n; i++) {
        int64_t acc = half;
        for (size_t j = 1; j <= i; j++)
            acc -= c[j] * (int64_t)s[i - j];
        s[i] = res[i] - (int32_t)(acc >> SELA_ORACLE_Q);
    }
    for (size_t i = (size_t)order + 1; i < n; i++) {
        int64_t acc = half;
        for (size_t j = 0; j <= (size_t)order; j++)
            acc -= c[j] * (int64_t)s[i - j];   /* s[i] is still 0 here, c[0] is 0 */
        s[i] = res[i] - (int32_t)(acc >> SELA_ORACLE_Q);
    }
}

/* ----------------------------------------------------------------- Rice -- */

/* convertSignedToUnsigned (src/rice/rice_encoder.cpp:12-18): the shift and the
 * negation are done in int32, then widened. */
static uint64_t zigzag(int32_t v)
{
    int32_t t = v < 0 ? (int32_t)(-(int32_t)((uint32_t)v << 1)) - 1 : (int32_t)((uint32_t)v << 1);
    return (uint64_t)(int64_t)t;
}

/* calculateOptimumRiceParam (src/rice/rice_encoder.cpp:20-33): first arg-min over k=0..19 */
size_t sela_oracle_rice_size(const int32_t *x, size_t n, uint32_t *k_out, uint64_t *bits_out)
{
    uint64_t best = 0;
    uint32_t best_k = 0;
    for (uint32_t k = 0; k < SELA_ORACLE_MAX_K; k++) {
        uint64_t total = 0;
        for (size_t i = 0; i < n; i++)
            total += (zigzag(x[i]) >> k) + 1 + k;
        if (k == 0 || total < best) {
            best = total;
            best_k = k;
        }
    }
    if (k_out)
        *k_out = best_k;
    if (bits_out)
        *bits_out = best;
    /* requiredInts = ceil((float)requiredBits / 32) (:63); float keeps 24 bits, exact
     * for every size the uint16 word-count field can hold. */
    return (size_t)ceil((float)best / 32);
}

/* generateEncodedBits + writeInts (src/rice/rice_encoder.cpp:35-71): stream bit b
 * lands in word b/32 at bit b%32; unary ones, a zero, then k bits MSB first. */
size_t sela_oracle_rice_encode(const int32_t *x, size_t n, uint32_t *k_out, uint32_t *words,
                               size_t words_cap)
{
    uint32_t k;
    uint64_t bits;
    size_t n_words = sela_oracle_rice_size(x, n, &k, &bits);
    if (k_out)
        *k_out = k;
    if (n_words > words_cap)
        return n_words;
    memset(words, 0, n_words * sizeof(uint32_t));
    uint64_t pos = 0;
    for (size_t i = 0; i < n; i++) {
        uint64_t u = zigzag(x[i]);
        uint64_t ones = u >> k;
        for (uint64_t t = 0; t < ones; t++, pos++)
            words[pos >> 5] |= 1u << (pos & 31);
        pos++; /* the terminating zero */
        for (int b = (int)k - 1; b >= 0; b--, pos++)
            if ((u >> b) & 1)
                words[pos >> 5] |= 1u << (pos & 31);
    }
    return n_words;
}

/* src/rice/rice_decoder.cpp:11-52 */
void sela_oracle_rice_decode(const uint32_t *words, size_t n_words, uint32_t k, uint32_t count,
                             int32_t *out)
{
    (void)n_words; /* the reference does not bounds-check either (:31-41) */
    uint32_t pos = 0;
    for (uint32_t i = 0; i < count; i++) {
        uint32_t ones = 0;
        while ((words[pos >> 5] >> (pos & 31)) & 1) {
            ones++;
            pos++;
        }
        pos++;
        uint64_t u = (uint32_t)(ones << k);      /* uint32 shift, then widened (:37) */
        for (uint32_t b = 1; b < k + 1; b++, pos++)
            u |= (uint64_t)((words[pos >> 5] >> (pos & 31)) & 1) << (k - b);
        out[i] = (int32_t)((u & 1) ? -(int64_t)((u + 1) >> 1) : (int64_t)(u >> 1));
    }
}

/* ---------------------------------------------------------------- frame -- */

typedef struct {
    uint8_t order;
    uint32_t refl_k, res_k;
    size_t refl_words, res_words;
    uint32_t *refl, *res; /* malloc'd */
} coded_channel;

static void code_channel(const int32_t *s, size_t n, coded_channel *o)
{
    int32_t q[MAXO];
    int32_t *res = (int32_t *)malloc(n * sizeof(int32_t));
    sela_oracle_lpc_analyse(s, n, &o->order, q, NULL, res, NULL, NULL);
    o->refl_words = sela_oracle_rice_size(q, o->order, NULL, NULL);
    o->refl = (uint32_t *)malloc((o->refl_words + 1) * sizeof(uint32_t));
    sela_oracle_rice_encode(q, o->order, &o->refl_k, o->refl, o->refl_words);
    o->res_words = sela_oracle_rice_size(res, n, NULL, NULL);
    o->res = (uint32_t *)malloc((o->res_words + 1) * sizeof(uint32_t));
    sela_oracle_rice_encode(res, n, &o->res_k, o->res, o->res_words);
    free(res);
}

static int emit_subframe(const coded_channel *cc, uint8_t ch, uint8_t type, uint8_t parent,
                         uint32_t n, sela_oracle_desc *d, uint32_t *words, size_t cap, size_t *used)
{
    if (*used + cc->refl_words + cc->res_words > cap)
        return -1;
    memset(d, 0, sizeof *d);
    d->channel = ch;
    d->subframe_type = type;
    d->parent_channel = parent;
    d->refl_rice_param = (uint8_t)cc->refl_k;
    d->refl_words = (uint16_t)cc->refl_words;
    d->lpc_order = cc->order;
    d->res_rice_param = (uint8_t)cc->res_k;
    d->res_words = (uint16_t)cc->res_words;
    d->samples = (uint16_t)n;
    d->refl_offset = *used;
    memcpy(words + *used, cc->refl, cc->refl_words * 4);
    *used += cc->refl_words;
    d->res_offset = *used;
    memcpy(words + *used, cc->res, cc->res_words * 4);
    *used += cc->res_words;
    return 0;
}

/* frame::FrameEncoder::process (src/frame/frame_encoder.cpp:11-102) */
int sela_oracle_frame_encode_i32(const int32_t *const *chs, uint32_t channels, uint32_t n,
                                 sela_oracle_desc *descs, uint32_t *words, size_t cap, size_t *used)
{
    int rc = 0;
    for (uint32_t i = 0; i < channels && rc == 0; i++) {
        coded_channel actual;
        code_channel(chs[i], n, &actual);
        if (i == 1 && channels == 2) { /* exactly stereo, second channel (:18) */
            int32_t *diff = (int32_t *)malloc(n * sizeof(int32_t));
            for (uint32_t j = 0; j < n; j++)
                diff[j] = chs[0][j] - chs[1][j];
            coded_channel dc;
            code_channel(diff, n, &dc);
            free(diff);
            /* strictly smaller word count wins for the difference (:63-72) */
            if (dc.refl_words + dc.res_words < actual.refl_words + actual.res_words)
                rc = emit_subframe(&dc, 1, 1, 0, n, &descs[i], words, cap, used);
            else
                rc = emit_subframe(&actual, 1, 0, 1, n, &descs[i], words, cap, used);
            free(dc.refl);
            free(dc.res);
        } else {
            rc = emit_subframe(&actual, (uint8_t)i, 0, (uint8_t)i, n, &descs[i], words, cap, used);
        }
        free(actual.refl);
        free(actual.res);
    }
    return rc;
}

static void decode_subframe(const sela_oracle_desc *d, const uint32_t *words, int32_t *out)
{
    int32_t q[256];
    int32_t *res = (int32_t *)malloc((size_t)d->samples * sizeof(int32_t) + 4);
    sela_oracle_rice_decode(words + d->refl_offset, d->refl_words, d->refl_rice_param, d->lpc_order, q);
    sela_oracle_rice_decode(words + d->res_offset, d->res_words, d->res_rice_param, d->samples, res);
    sela_oracle_lpc_synthesise(res, d->samples, d->lpc_order, q, out);
    free(res);
}

/* frame::FrameDecoder::process (src/frame/frame_decoder.cpp:11-72): independent
 * subframes first, then dependent ones as parent - difference; output slot is the
 * subframe's channel field. */
int sela_oracle_frame_decode_i32(const sela_oracle_desc *descs, uint32_t n_sub,
                                 const uint32_t *words, int32_t *const *out)
{
    for (uint32_t i = 0; i < n_sub; i++)
        if (descs[i].subframe_type == 0)
            decode_subframe(&descs[i], words, out[descs[i].channel]);
    for (uint32_t i = 0; i < n_sub; i++)
        if (descs[i].subframe_type == 1) {
            const sela_oracle_desc *d = &descs[i];
            int32_t *diff = (int32_t *)malloc((size_t)d->samples * sizeof(int32_t) + 4);
            decode_subframe(d, words, diff);
            for (uint32_t j = 0; j < d->samples; j++)
                out[d->channel][j] = out[d->parent_channel][j] - diff[j];
            free(diff);
        }
    return 0;
}

/* --------------------------------------------------------------- batches -- */

typedef struct {
    const int16_t *pcm;
    int16_t *pcm_out;
    uint32_t channels, begin, end;
    sela_oracle_desc *descs;        /* encode: out (offsets local to this segment) */
    const sela_oracle_desc *cdescs; /* decode: in */
    const uint32_t *cwords;
    uint32_t *seg_words;            /* encode: malloc'd by the worker */
    size_t seg_used;
} seg_job;

static void *encode_worker(void *arg)
{
    seg_job *job = (seg_job *)arg;
    const uint32_t ch = job->channels, n = SELA_ORACLE_FRAME;
    size_t cap = 0;
    int32_t **planes = (int32_t **)malloc(ch * sizeof(int32_t *));
    for (uint32_t c = 0; c < ch; c++)
        planes[c] = (int32_t *)malloc(n * sizeof(int32_t));
    job->seg_words = NULL;
    job->seg_used = 0;
    for (uint32_t f = job->begin; f < job->end; f++) {
        /* demux exactly as src/file/wav_file.cpp:194-200: sign-extended int16 */
        const int16_t *src = job->pcm + (size_t)f * n * ch;
        for (uint32_t j = 0; j < n; j++)
            for (uint32_t c = 0; c < ch; c++)
                planes[c][j] = src[(size_t)j * ch + c];
        size_t need = job->seg_used + (size_t)ch * 2 * 70000;
        if (need > cap) {
            cap = need * 2;
            job->seg_words = (uint32_t *)realloc(job->seg_words, cap * sizeof(uint32_t));
        }
        sela_oracle_frame_encode_i32((const int32_t *const *)planes, ch, n,
                                     job->descs + (size_t)f * ch, job->seg_words, cap, &job->seg_used);
    }
    for (uint32_t c = 0; c < ch; c++)
        free(planes[c]);
    free(planes);
    return NULL;
}

static void *decode_worker(void *arg)
{
    seg_job *job = (seg_job *)arg;
    const uint32_t ch = job->channels, n = SELA_ORACLE_FRAME;
    int32_t **planes = (int32_t **)malloc(ch * sizeof(int32_t *));
    for (uint32_t c = 0; c < ch; c++)
        planes[c] = (int32_t *)calloc(65536, sizeof(int32_t));
    for (uint32_t f = job->begin; f < job->end; f++) {
        sela_oracle_frame_decode_i32(job->cdescs + (size_t)f * ch, ch, job->cwords, planes);
        int16_t *dst = job->pcm_out + (size_t)f * n * ch;
        for (uint32_t j = 0; j < n; j++)
            for (uint32_t c = 0; c < ch; c++)
                dst[(size_t)j * ch + c] = (int16_t)(uint16_t)planes[c][j]; /* wav_file.cpp:249-251 */
    }
    for (uint32_t c = 0; c < ch; c++)
        free(planes[c]);
    free(planes);
    return NULL;
}

/* Thread split of sela::Encoder::processFrames (src/sela/encoder.cpp:58-73):
 * framesPerThread = N / T contiguous frames each, the last thread takes the rest. */
static void split(uint32_t n_frames, int threads, int t, uint32_t *b, uint32_t *e)
{
    uint32_t per = n_frames / (uint32_t)threads;
    *b = per * (uint32_t)t;
    *e = (t == threads - 1) ? n_frames : per * (uint32_t)(t + 1);
}

int sela_oracle_encode_frames(const int16_t *pcm, uint32_t n_frames, uint32_t channels,
                              sela_oracle_desc *descs, uint32_t *words, size_t cap, size_t *used,
                              int threads)
{
    if (threads <= 0)
        threads = sela_oracle_online_cores();
    seg_job *jobs = (seg_job *)calloc((size_t)threads, sizeof(seg_job));
    pthread_t *tid = (pthread_t *)calloc((size_t)threads, sizeof(pthread_t));
    for (int t = 0; t < threads; t++) {
        jobs[t].pcm = pcm;
        jobs[t].channels = channels;
        jobs[t].descs = descs;
        split(n_frames, threads, t, &jobs[t].begin, &jobs[t].end);
        pthread_create(&tid[t], NULL, encode_worker, &jobs[t]);
    }
    int rc = 0;
    size_t total = 0;
    for (int t = 0; t < threads; t++) {
        pthread_join(tid[t], NULL);
        /* concatenate segments in thread order (src/sela/encoder.cpp:80-84) */
        if (rc == 0 && total + jobs[t].seg_used <= cap) {
            if (jobs[t].seg_used)
                memcpy(words + total, jobs[t].seg_words, jobs[t].seg_used * sizeof(uint32_t));
            for (size_t i = (size_t)jobs[t].begin * channels; i < (size_t)jobs[t].end * channels; i++) {
                descs[i].refl_offset += total;
                descs[i].res_offset += total;
            }
            total += jobs[t].seg_used;
        } else {
            rc = -1;
        }
        free(jobs[t].seg_words);
    }
    *used = total;
    free(jobs);
    free(tid);
    return rc;
}

int sela_oracle_decode_frames(const sela_oracle_desc *descs, uint32_t n_frames, uint32_t channels,
                              const uint32_t *words, int16_t *pcm_out, int threads)
{
    if (threads <= 0)
        threads = sela_oracle_online_cores();
    seg_job *jobs = (seg_job *)calloc((size_t)threads, sizeof(seg_job));
    pthread_t *tid = (pthread_t *)calloc((size_t)threads, sizeof(pthread_t));
    for (int t = 0; t < threads; t++) {
        jobs[t].pcm_out = pcm_out;
        jobs[t].channels = channels;
        jobs[t].cdescs = descs;
        jobs[t].cwords = words;
        split(n_frames, threads, t, &jobs[t].begin, &jobs[t].end);
        pthread_create(&tid[t], NULL, decode_worker, &jobs[t]);
    }
    for (int t = 0; t < threads; t++)
        pthread_join(tid[t], NULL);
    free(jobs);
    free(tid);
    return 0;
}

static double now_s(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

double sela_oracle_time_encode(const int16_t *pcm, uint32_t n_frames, uint32_t channels, int threads)
{
    size_t cap = (size_t)n_frames * channels * 4096 + 1024, used = 0;
    sela_oracle_desc *descs = (sela_oracle_desc *)malloc((size_t)n_frames * channels * sizeof *descs);
    uint32_t *words = (uint32_t *)malloc(cap * sizeof(uint32_t));
    double t0 = now_s();
    sela_oracle_encode_frames(pcm, n_frames, channels, descs, words, cap, &used, threads);
    double t1 = now_s();
    free(descs);
    free(words);
    return t1 - t0;
}

double sela_oracle_time_decode(const sela_oracle_desc *descs, uint32_t n_frames, uint32_t channels,
                               const uint32_t *words, int threads)
{
    int16_t *pcm = (int16_t *)malloc((size_t)n_frames * channels * SELA_ORACLE_FRAME * sizeof(int16_t));
    double t0 = now_s();
    sela_oracle_decode_frames(descs, n_frames, channels, words, pcm, threads);
    double t1 = now_s();
    free(pcm);
    return t1 - t0;
}
