/*
 * oracle/gcadpcm.c — CPU ORACLE (test infrastructure, not product) for Nintendo GC-ADPCM.
 *
 * Restates, in plain C with IEEE-754 double / wrapping int32 semantics, what the reference does in
 *   Codecs/GcAdpcm/GcAdpcmCoefficients.cs, GcAdpcmEncoder.cs, GcAdpcmDecoder.cs, GcAdpcmMath.cs and
 *   Utilities/Helpers.cs:32-58 (paths relative to VGAudio's src/VGAudio/).
 * Must be compiled with -ffp-contract=off and without -ffast-math: RyuJIT emits separate SSE2
 * mul/add, and the silent-channel case relies on NaN comparison semantics (SURVEY.md Appendix A.4, A.19).
 *
 * Pinning: see vgoracle.h.  The reference cannot be executed in this environment (no .NET), so the
 * encoded bytes are checked through the reference's own round-trip properties, not a golden stream.
 */
#include "vgoracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <stdatomic.h>
#include <unistd.h>

enum { FRAME_BYTES = 8, FRAME_SAMPLES = 14, FRAME_NIBBLES = 16 };

/* ------------------------------------------------------------------------------------------------
 * small helpers
 * ---------------------------------------------------------------------------------------------- */

/* C# int arithmetic is unchecked: do add/mul in uint32 and reinterpret (SURVEY.md A.7). */
static inline int32_t wrap_add(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
static inline int32_t wrap_sub(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }
static inline int32_t wrap_mul(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); }
/* >> on a negative int is an arithmetic shift in C#; gcc does the same for signed operands. */
static inline int32_t sar(int32_t a, int n) { return a >> n; }

/* Helpers.Clamp16 (Utilities/Helpers.cs:32-39), Clamp4 (:41-48) */
static inline int32_t sat16(int32_t v) { return v > 32767 ? 32767 : (v < -32768 ? -32768 : v); }
static inline int32_t sat4(int32_t v) { return v > 7 ? 7 : (v < -8 ? -8 : v); }
/* Helpers.CombineNibbles (:58) */
static inline uint8_t nibbles(int hi, int lo) { return (uint8_t)((hi << 4) | (lo & 0xF)); }
/* Helpers.GetHighNibbleSigned / GetLowNibbleSigned (:50-56): two's complement 4-bit */
static inline int32_t snib(int v) { v &= 0xF; return v >= 8 ? v - 16 : v; }

/* Extensions.DivideByRoundUp (Utilities/Extensions.cs:145): (int)Math.Ceiling((double)v / d) */
int vgo_divide_by_round_up(int value, int divisor) { return (int)ceil((double)value / (double)divisor); }

/* ------------------------------------------------------------------------------------------------
 * GcAdpcmMath.cs:7-47
 * ---------------------------------------------------------------------------------------------- */
int vgo_gc_nibble_count_to_sample_count(int nibble_count)
{
    int whole = nibble_count / FRAME_NIBBLES, rest = nibble_count % FRAME_NIBBLES;
    return FRAME_SAMPLES * whole + (rest < 2 ? 0 : rest - 2);
}
int vgo_gc_sample_count_to_nibble_count(int sample_count)
{
    int whole = sample_count / FRAME_SAMPLES, rest = sample_count % FRAME_SAMPLES;
    return FRAME_NIBBLES * whole + (rest == 0 ? 0 : rest + 2);
}
int vgo_gc_nibble_to_sample(int nibble)
{
    return FRAME_SAMPLES * (nibble / FRAME_NIBBLES) + nibble % FRAME_NIBBLES - 2;
}
int vgo_gc_sample_to_nibble(int sample)
{
    return FRAME_NIBBLES * (sample / FRAME_SAMPLES) + sample % FRAME_SAMPLES + 2;
}
int vgo_gc_sample_count_to_byte_count(int sample_count)
{
    int nib = vgo_gc_sample_count_to_nibble_count(sample_count);
    return nib / 2 + (nib & 1); /* Extensions.DivideBy2RoundUp :146 */
}
int vgo_gc_byte_count_to_sample_count(int byte_count) { return vgo_gc_nibble_count_to_sample_count(byte_count * 2); }

/* ------------------------------------------------------------------------------------------------
 * Coefficient analysis, phase 1: one candidate record per frame (GcAdpcmCoefficients.cs:40-61)
 * Arrays are 1-based 3x3 / length-3 like the reference so the index arithmetic reads the same.
 * ---------------------------------------------------------------------------------------------- */

/* InnerProductMerge :112-120 — win[0..13] previous frame, win[14..27] current frame */
static void autocorr_neg(double out[3], const int16_t win[28])
{
    for (int lag = 0; lag <= 2; lag++) {
        double acc = 0.0;
        for (int t = 0; t < 14; t++)
            acc -= (double)((int32_t)win[14 + t - lag] * (int32_t)win[14 + t]);
        out[lag] = acc;
    }
}

/* OuterProductMerge :122-131 */
static void covariance(double m[3][3], const int16_t win[28])
{
    for (int a = 1; a <= 2; a++)
        for (int b = 1; b <= 2; b++) {
            double acc = 0.0;
            for (int t = 0; t < 14; t++)
                acc += (double)((int32_t)win[14 + t - a] * (int32_t)win[14 + t - b]);
            m[a][b] = acc;
        }
}

/* AnalyzeRanges :133-208 — scaled partial-pivot LU of the 2x2 block; returns a VGO_GC_REJ_* reason to REJECT the frame,
 * 0 to keep it */
static int lu_reject(double m[3][3], int perm[3], double inv_row_max[3])
{
    for (int r = 1; r <= 2; r++) {
        double big = fmax(fabs(m[r][1]), fabs(m[r][2]));
        if (big < 4.9406564584124654e-324) /* double.Epsilon: smallest denormal (A.2) */
            return VGO_GC_REJ_BIG;
        inv_row_max[r] = 1.0 / big;
    }

    int pivot_row = 0;
    for (int col = 1; col <= 2; col++) {
        for (int r = 1; r < col; r++) {
            double t = m[r][col];
            for (int k = 1; k < r; k++) t -= m[r][k] * m[k][col];
            m[r][col] = t;
        }
        double best = 0.0;
        for (int r = col; r <= 2; r++) {
            double t = m[r][col];
            for (int k = 1; k < col; k++) t -= m[r][k] * m[k][col];
            m[r][col] = t;
            t = fabs(t) * inv_row_max[r];
            if (t >= best) { best = t; pivot_row = r; }
        }
        if (pivot_row != col) {
            for (int k = 1; k <= 2; k++) {
                double t = m[pivot_row][k];
                m[pivot_row][k] = m[col][k];
                m[col][k] = t;
            }
            inv_row_max[pivot_row] = inv_row_max[col];
        }
        perm[col] = pivot_row;
        if (col != 2) {
            double t = 1.0 / m[col][col];
            for (int r = col + 1; r <= 2; r++) m[r][col] *= t;
        }
    }

    double lo = 1.0e10, hi = 0.0;
    for (int d = 1; d <= 2; d++) {
        double t = fabs(m[d][d]);
        if (t < lo) lo = t;
        if (t > hi) hi = t;
    }
    return lo / hi < 1.0e-10 ? VGO_GC_REJ_RANGE : 0;
}

/* BidirectionalFilter :210-237 — permuted forward substitution, then back substitution */
static void lu_solve(double m[3][3], const int perm[3], double v[3])
{
    for (int i = 1, first_nz = 0; i <= 2; i++) {
        int src = perm[i];
        double t = v[src];
        v[src] = v[i];
        if (first_nz != 0) {
            for (int k = first_nz; k <= i - 1; k++) t -= v[k] * m[i][k];
        } else if (t != 0.0) {
            first_nz = i;
        }
        v[i] = t;
    }
    for (int i = 2; i > 0; i--) {
        double t = v[i];
        for (int k = i + 1; k <= 2; k++) t -= v[k] * m[i][k];
        v[i] = t / m[i][i];
    }
    v[0] = 1.0;
}

/* QuadraticMerge :239-255 — returns a VGO_GC_REJ_* reason to REJECT, 0 to keep */
static int to_reflection(double v[3])
{
    double k2 = v[2];
    double den = 1.0 - (k2 * k2);
    if (den == 0.0) return VGO_GC_REJ_DEN;
    double a = (v[0] - (k2 * k2)) / den;
    double b = (v[1] - (v[1] * k2)) / den;
    v[0] = a;
    v[1] = b;
    return fabs(b) > 1.0 ? VGO_GC_REJ_K1 : 0;
}

/* FinishRecord :257-283 (both overloads share the arithmetic) */
static void finish_record(double in[3], double out[3])
{
    for (int z = 1; z <= 2; z++) {
        if (in[z] >= 1.0) in[z] = 0.9999999999;
        else if (in[z] <= -1.0) in[z] = -0.9999999999;
    }
    out[0] = 1.0;
    out[1] = (in[2] * in[1]) + in[1];
    out[2] = in[2];
}

/* MatrixFilter :285-305 — step-down from the stored record to a direct-form vector */
static void record_to_direct(const double rec[3], double dst[3], double m[3][3])
{
    m[2][0] = 1.0;
    for (int i = 1; i <= 2; i++) m[2][i] = -rec[i];
    for (int i = 2; i > 0; i--) {
        double den = 1.0 - (m[i][i] * m[i][i]);
        for (int y = 1; y <= i; y++)
            m[i - 1][y] = ((m[i][i] * m[i][y]) + m[i][y]) / den;
    }
    dst[0] = 1.0;
    for (int i = 1; i <= 2; i++) {
        dst[i] = 0.0;
        for (int y = 1; y <= i; y++) dst[i] += m[i][y] * dst[i - y];
    }
}

/* MergeFinishRecord :307-333 */
static void centroid_from_mean(const double src[3], double dst[3])
{
    double k[3] = {0.0, 0.0, 0.0};
    double err = src[0];
    dst[0] = 1.0;
    for (int i = 1; i <= 2; i++) {
        double acc = 0.0;
        for (int y = 1; y < i; y++) acc += dst[y] * src[i - y];
        if (err > 0.0) dst[i] = -(acc + src[i]) / err;
        else dst[i] = 0.0;
        k[i] = dst[i];
        for (int y = 1; y < i; y++) dst[y] += dst[i] * dst[i - y];
        err *= 1.0 - (dst[i] * dst[i]);
    }
    finish_record(k, dst);
}

/* ContrastVectors :335-342 */
static double contrast(const double c[3], const double rec[3])
{
    double q = (rec[2] * rec[1] + -rec[1]) / (1.0 - rec[2] * rec[2]);
    double e0 = (c[0] * c[0]) + (c[1] * c[1]) + (c[2] * c[2]);
    double e1 = (c[0] * c[1]) + (c[1] * c[2]);
    double e2 = c[0] * c[2];
    return e0 + (2.0 * q * e1) + (2.0 * (-rec[1] * q + -rec[2]) * e2);
}

/* Trace of one refinement pass: the record's minimum distance `least` is shared by more than one centroid (vgo_gc_coef_trace) */
static void note_tie(vgo_gc_coef_pass *st, const double best[8][3], const double dist[8], int count, double least, int z)
{
    int lo = -1, hi = -1, n = 0, same = 1;
    for (int c = 0; c < count; c++) {
        if (!(dist[c] == least)) continue;
        if (lo < 0) lo = c;
        else if (memcmp(best[c], best[lo], sizeof best[c]) != 0) same = 0;
        hi = c;
        n++;
    }
    if (n < 2) return;
    if (same) st->ties_same++;
    else st->ties_distinct++;
    if (st->tie_record < 0) {
        st->tie_record = z;
        st->tie_lo = lo;
        st->tie_hi = hi;
    }
}

/* After a pass: the centroids and bucket counts it leaves (vgo_gc_coef_trace) */
static void note_pass(vgo_gc_coef_pass *st, const double best[8][3], const int *hits, int count)
{
    st->count = count;
    for (int z = 0; z < 8; z++) {
        st->cent[z][0] = best[z][1];
        st->cent[z][1] = best[z][2];
        st->hits[z] = z < count ? hits[z] : 0;
        if (z < count && hits[z] == 0) st->empty++;
    }
}

/* FilterRecords :344-396 — two rounds of nearest-centroid assignment + ordered mean.  st == NULL on the normal path,
 * else the trace of the two rounds; recording only reads values the loop computes anyway. */
static void refine_centroids(double best[8][3], int count, const double (*records)[3], int n_records, vgo_gc_coef_pass *st)
{
    double sums[8][3];
    double m[3][3];
    int hits[8];
    double direct[3];
    double dist[8];
    memset(m, 0, sizeof m);

    for (int round = 0; round < 2; round++) {
        for (int c = 0; c < count; c++) {
            hits[c] = 0;
            for (int i = 0; i <= 2; i++) sums[c][i] = 0.0;
        }
        for (int z = 0; z < n_records; z++) {
            int pick = 0;
            double least = 1.0e30;
            for (int c = 0; c < count; c++) {
                double d = contrast(best[c], records[z]);
                dist[c] = d;
                if (d < least) { least = d; pick = c; }
            }
            if (st && least < 1.0e30) note_tie(&st[round], (const double (*)[3])best, dist, count, least, z);
            hits[pick]++;
            record_to_direct(records[z], direct, m);
            for (int i = 0; i <= 2; i++) sums[pick][i] += direct[i];
        }
        for (int c = 0; c < count; c++)
            if (hits[c] > 0)
                for (int y = 0; y <= 2; y++) sums[c][y] /= hits[c];
        for (int c = 0; c < count; c++) centroid_from_mean(sums[c], best[c]);
        if (st) note_pass(&st[round], (const double (*)[3])best, hits, count);
    }
}

/* One frame of phase 1.  win holds previous+current frame.  Returns 0 (VGO_GC_ACCEPTED) and fills rec[0..2] if the
 * frame gives a record, else the VGO_GC_REJ_* reason it was rejected for. */
static int frame_record(const int16_t win[28], double rec[3])
{
    double v[3], m[3][3], scratch[3];
    int perm[3] = {0, 0, 0};
    int why;
    memset(m, 0, sizeof m);
    autocorr_neg(v, win);
    if (!(fabs(v[0]) > 10.0)) return VGO_GC_REJ_QUIET;
    covariance(m, win);
    if ((why = lu_reject(m, perm, scratch)) != 0) return why;
    lu_solve(m, perm, v);
    if ((why = to_reflection(v)) != 0) return why;
    finish_record(v, rec);
    return VGO_GC_ACCEPTED;
}

/* short rounding of the final coefficients, GcAdpcmCoefficients.cs:94-108.  Math.Round = half-to-even. */
static int16_t quantise_coef(double v)
{
    double d = -v * 2048.0;
    if (d > 0.0) return d > 32767.0 ? 32767 : (int16_t)nearbyint(d);
    if (d < -32768.0) return -32768;
    if (d != d) return 0; /* (short)(int)NaN on x64 = (short)0x80000000 = 0; unreachable in practice (A.19) */
    return (int16_t)nearbyint(d);
}

static int collect_records(const int16_t *source, int length, double (*records)[3], double *rec_out,
                           double *dir_out, uint8_t *accepted_out, uint8_t *outcome_out)
{
    int16_t win[28];
    double m[3][3];
    int n_records = 0, frame = 0;
    memset(win, 0, sizeof win);
    memset(m, 0, sizeof m);
    for (int pos = 0, left = length; pos < length; pos += 14, left -= 14, frame++) {
        int take = left < 14 ? left : 14;
        memset(win + 14, 0, 14 * sizeof(int16_t));
        memcpy(win + 14, source + pos, (size_t)take * sizeof(int16_t));
        double rec[3];
        int why = frame_record(win, rec);
        int ok = why == VGO_GC_ACCEPTED;
        if (ok && records) memcpy(records[n_records], rec, sizeof rec);
        if (accepted_out) accepted_out[frame] = (uint8_t)ok;
        if (outcome_out) outcome_out[frame] = (uint8_t)why;
        if (rec_out) { rec_out[2 * frame] = ok ? rec[1] : 0.0; rec_out[2 * frame + 1] = ok ? rec[2] : 0.0; }
        if (dir_out) {
            double d[3] = {0.0, 0.0, 0.0};
            if (ok) record_to_direct(rec, d, m);
            dir_out[2 * frame] = d[1];
            dir_out[2 * frame + 1] = d[2];
        }
        n_records += ok;
        memmove(win, win + 14, 14 * sizeof(int16_t));
    }
    return n_records;
}

int vgo_gc_coef_records(const int16_t *source, int length, double *rec_out, double *dir_out, uint8_t *accepted_out)
{
    return collect_records(source, length, NULL, rec_out, dir_out, accepted_out, NULL);
}

/* CalculateCoefficients :9-110.  trace_out == NULL on the normal path, else the facts of every pass and frame
 * (vgo_gc_coef_trace); recording only reads values the loops compute anyway, so the arithmetic is the same either way. */
static void calculate_coefficients(const int16_t *source, int length, int16_t coefs_out[16], vgo_gc_refine_trace *trace_out,
                                   uint8_t *outcome_out)
{
    int n_frames = vgo_divide_by_round_up(length, FRAME_SAMPLES);
    double (*records)[3] = malloc(sizeof(double[3]) * (size_t)(n_frames > 0 ? n_frames : 1));
    double best[8][3];
    double m[3][3];
    double mean[3], nudge[3];
    memset(best, 0, sizeof best);
    memset(m, 0, sizeof m);

    int n_records = collect_records(source, length, records, NULL, NULL, NULL, outcome_out);

    /* ordered mean of the direct-form vectors :63-76 */
    mean[0] = 1.0; mean[1] = 0.0; mean[2] = 0.0;
    for (int z = 0; z < n_records; z++) {
        record_to_direct(records[z], best[0], m);
        for (int y = 1; y <= 2; y++) mean[y] += best[0][y];
    }
    for (int y = 1; y <= 2; y++) mean[y] /= n_records; /* 0/0 = NaN when no frame qualified (A.19) */
    centroid_from_mean(mean, best[0]);
    if (trace_out) {
        memset(trace_out, 0, sizeof *trace_out);
        for (int p = 0; p < VGO_GC_COEF_PASSES; p++) trace_out->pass[p].tie_record = trace_out->pass[p].tie_lo = trace_out->pass[p].tie_hi = -1;
        trace_out->n_frames = n_frames;
        trace_out->n_records = n_records;
        note_pass(&trace_out->pass[0], (const double (*)[3])best, &n_records, 1);
    }

    /* three split-and-refine generations: 1 -> 2 -> 4 -> 8 centroids :79-91 */
    int count = 1;
    for (int gen = 0; gen < 3;) {
        nudge[0] = 0.0; nudge[1] = -1.0; nudge[2] = 0.0;
        for (int i = 0; i < count; i++)
            for (int y = 0; y <= 2; y++)
                best[count + i][y] = (0.01 * nudge[y]) + best[i][y];
        ++gen;
        count = 1 << gen;
        refine_centroids(best, count, (const double (*)[3])records, n_records,
                         trace_out ? &trace_out->pass[2 * gen - 1] : NULL);
    }

    for (int z = 0; z < 8; z++) {
        coefs_out[z * 2] = quantise_coef(best[z][1]);
        coefs_out[z * 2 + 1] = quantise_coef(best[z][2]);
    }
    free(records);
}

void vgo_gc_calculate_coefficients(const int16_t *source, int length, int16_t coefs_out[16])
{
    calculate_coefficients(source, length, coefs_out, NULL, NULL);
}

void vgo_gc_coef_trace(const int16_t *source, int length, vgo_gc_refine_trace *trace_out, uint8_t *outcome_out,
                       int16_t coefs_out[16])
{
    calculate_coefficients(source, length, coefs_out, trace_out, outcome_out);
}

int vgo_gc_refine_trace_size(void) { return (int)sizeof(vgo_gc_refine_trace); }

/* ------------------------------------------------------------------------------------------------
 * Encoder (GcAdpcmEncoder.cs)
 * ---------------------------------------------------------------------------------------------- */

typedef struct {
    int32_t recon[16]; /* PcmOut */
    int32_t nib[14];   /* AdpcmOut */
    int32_t scale_power;
    double error;      /* TotalDistance */
} gc_trial;

/* |v| without the overflow of abs(INT32_MIN) */
static inline uint32_t uabs32(int32_t v) { return v < 0 ? 0u - (uint32_t)v : (uint32_t)v; }

/* DspEncodeCoef :96-171 for one predictor pair (c0 = coefs[2p], c1 = coefs[2p+1]).  st == NULL on the encoding path;
 * otherwise the facts of the scale chain are recorded there (vgo_gc_encode_trace).  Recording only reads values the
 * loop computes anyway, so the arithmetic is the same either way. */
static void try_predictor(const int16_t pcm[16], int n, int16_t c0, int16_t c1, gc_trial *t, vgo_gc_pred_trace *st)
{
    int32_t peak = 0;
    int32_t over;

    t->recon[0] = pcm[0];
    t->recon[1] = pcm[1];

    /* residual range against the RAW neighbours (:107-115); "/ 2048" truncates toward zero (A.6) */
    for (int s = 0; s < n; s++) {
        int64_t wide = (int64_t)pcm[s] * c1 + (int64_t)pcm[s + 1] * c0;
        int32_t guess = wrap_add(wrap_mul(pcm[s], c1), wrap_mul(pcm[s + 1], c0)) / 2048;
        if (st && wide != (int32_t)wide) st->wrapped = 1;
        int32_t diff = sat16(wrap_sub(pcm[s + 2], guess));
        if (abs(diff) > abs(peak)) peak = diff;
    }

    /* first scale guess (:118-124) */
    int32_t sp = 0;
    while (sp <= 12 && (peak > 7 || peak < -8)) {
        peak /= 2;
        sp++;
    }
    sp = sp <= 1 ? -1 : sp - 2;
    if (st) st->first_sp = (int8_t)(sp + 1);

    /* quantise / reconstruct, growing the scale until the nibbles fit (:127-170) */
    do {
        sp++;
        int32_t scale = (1 << sp) * 2048;
        t->error = 0.0;
        over = 0;

        for (int s = 0; s < n; s++) {
            int32_t want = wrap_mul(pcm[s + 2], 2048);
            int32_t guess = wrap_add(wrap_mul(t->recon[s], c1), wrap_mul(t->recon[s + 1], c0));
            int32_t diff = wrap_sub(want, guess);
            if (st) {
                int64_t wide = (int64_t)t->recon[s] * c1 + (int64_t)t->recon[s + 1] * c0;
                if (wide != (int32_t)wide || (int64_t)want - guess != diff) st->wrapped = 1;
                if (uabs32(diff) > st->max_abs_diff) st->max_abs_diff = uabs32(diff);
            }
            /* int -> float32 -> divide in float32 -> widen -> add float32 literal widened -> truncate (A.5) */
            float ratio = (float)diff / (float)scale;
            int32_t raw = (diff > 0) ? (int32_t)((double)ratio + (double)0.4999999f)
                                     : (int32_t)((double)ratio - (double)0.4999999f);
            int32_t q = sat4(raw);
            if (q != raw) {
                int32_t excess = abs(raw - q);
                if (excess > over) over = excess;
            }
            t->nib[s] = q;

            int32_t fixed = wrap_add(guess, wrap_mul(q, scale));
            int32_t out = sat16(sar(wrap_add(fixed, 1024), 11));
            t->recon[s + 2] = out;
            double miss = (double)(pcm[s + 2] - out);
            t->error += miss * miss;
        }

        /* DEVIATION (termination guard): with hostile coefficient sets the pass at scalePower 12 can still
         * overflow by more than 248; the reference then bumps 13 -> 11 (:166-168), re-enters the loop, repeats the
         * identical pass at 12 and NEVER terminates (found by fuzzing this restatement).  Coefficients produced by
         * CalculateCoefficients cannot reach it (|diff| < 2^29 there).  Oracle and CUDA kernel both treat a pass
         * at scalePower 12 as final, which changes nothing for any input on which the reference halts. */
        const int pass_power = sp;
        if (st) {
            st->over[st->n_passes++] = over;  /* every pass raises sp by at least one: at most 13 passes */
            if (over + 8 > 256 && pass_power < 12) st->bumped = 1;
            if (pass_power >= 12 && over > 1) st->final12 = 1;
        }
        for (int32_t x = over + 8; x > 256; x >>= 1)
            if (++sp >= 12) sp = 11;
        if (pass_power >= 12) { sp = 12; break; }
    } while (sp < 12 && over > 1);

    t->scale_power = sp;
    if (st) {
        st->final_sp = (int8_t)sp;
        st->error = 0;
        for (int s = 0; s < n; s++) {
            int64_t miss = (int64_t)pcm[s + 2] - t->recon[s + 2];
            st->error += (uint64_t)(miss * miss);
        }
    }
}

/* DspEncodeFrame :48-94; st == NULL on the encoding path, else the frame's trace record */
static void dsp_encode_frame(int16_t pcm_in_out[16], int sample_count, uint8_t adpcm_out[8], const int16_t coefs[16],
                             vgo_gc_frame_trace *st)
{
    gc_trial trial[8];
    if (st) memset(st, 0, sizeof *st);
    for (int p = 0; p < 8; p++)
        try_predictor(pcm_in_out, sample_count, coefs[2 * p], coefs[2 * p + 1], &trial[p], st ? &st->pred[p] : NULL);

    int pick = 0;
    double least = 1.7976931348623157e308; /* double.MaxValue; strict < keeps the first minimum (A.9) */
    for (int p = 0; p < 8; p++)
        if (trial[p].error < least) { least = trial[p].error; pick = p; }
    if (st) {
        st->winner = (int8_t)pick;
        for (int p = 0; p < 8; p++)
            if (p != pick && st->pred[p].error == st->pred[pick].error) st->tie = 1;
    }

    for (int s = 0; s < sample_count; s++) pcm_in_out[s + 2] = (int16_t)trial[pick].recon[s + 2];
    adpcm_out[0] = nibbles(pick, trial[pick].scale_power);
    for (int s = sample_count; s < 14; s++) trial[pick].nib[s] = 0;
    for (int i = 0; i < 7; i++) adpcm_out[i + 1] = nibbles(trial[pick].nib[2 * i], trial[pick].nib[2 * i + 1]);
}

void vgo_gc_dsp_encode_frame(int16_t pcm_in_out[16], int sample_count, uint8_t adpcm_out[8], const int16_t coefs[16])
{
    dsp_encode_frame(pcm_in_out, sample_count, adpcm_out, coefs, NULL);
}

/* Encode :14-46; trace_out == NULL on the encoding path, else one record per frame */
static void encode(const int16_t *pcm, int pcm_length, const int16_t coefs[16], int sample_count, int16_t history1,
                   int16_t history2, uint8_t *adpcm_out, vgo_gc_frame_trace *trace_out)
{
    if (sample_count == -1) sample_count = pcm_length;
    int16_t window[2 + FRAME_SAMPLES];
    uint8_t packed[FRAME_BYTES];
    window[0] = history2;
    window[1] = history1;

    int n_frames = vgo_divide_by_round_up(sample_count, FRAME_SAMPLES);
    for (int f = 0; f < n_frames; f++) {
        int take = sample_count - f * FRAME_SAMPLES;
        if (take > FRAME_SAMPLES) take = FRAME_SAMPLES;
        memcpy(window + 2, pcm + (size_t)f * FRAME_SAMPLES, (size_t)take * sizeof(int16_t));
        memset(window + 2 + take, 0, (size_t)(FRAME_SAMPLES - take) * sizeof(int16_t));

        dsp_encode_frame(window, FRAME_SAMPLES, packed, coefs, trace_out ? &trace_out[f] : NULL);

        memcpy(adpcm_out + (size_t)f * FRAME_BYTES, packed, (size_t)vgo_gc_sample_count_to_byte_count(take));
        window[0] = window[14];
        window[1] = window[15];
    }
}

void vgo_gc_encode(const int16_t *pcm, int pcm_length, const int16_t coefs[16],
                   int sample_count, int16_t history1, int16_t history2, uint8_t *adpcm_out)
{
    encode(pcm, pcm_length, coefs, sample_count, history1, history2, adpcm_out, NULL);
}

void vgo_gc_encode_trace(const int16_t *pcm, int pcm_length, const int16_t coefs[16], int sample_count,
                         int16_t history1, int16_t history2, uint8_t *adpcm_out, vgo_gc_frame_trace *trace_out)
{
    encode(pcm, pcm_length, coefs, sample_count, history1, history2, adpcm_out, trace_out);
}

int vgo_gc_frame_trace_size(void) { return (int)sizeof(vgo_gc_frame_trace); }

/* ------------------------------------------------------------------------------------------------
 * Decoder (GcAdpcmDecoder.cs:10-54)
 * ---------------------------------------------------------------------------------------------- */
void vgo_gc_decode(const uint8_t *adpcm, const int16_t coefs[16], int sample_count,
                   int16_t history1, int16_t history2, int16_t *pcm_out)
{
    if (sample_count == 0) return;
    int n_frames = vgo_divide_by_round_up(sample_count, FRAME_SAMPLES);
    int done = 0;
    size_t in = 0;
    int32_t h1 = history1, h2 = history2;

    for (int f = 0; f < n_frames; f++) {
        uint8_t head = adpcm[in++];
        int32_t scale = (1 << (head & 0xF)) * 2048;
        int p = (head >> 4) & 0xF;
        int32_t c1 = coefs[p * 2], c2 = coefs[p * 2 + 1];
        int take = sample_count - done;
        if (take > FRAME_SAMPLES) take = FRAME_SAMPLES;

        for (int s = 0; s < take; s++) {
            int32_t q = (s % 2 == 0) ? snib(adpcm[in] >> 4) : snib(adpcm[in++]);
            int32_t guess = wrap_add(wrap_mul(c1, h1), wrap_mul(c2, h2));
            int32_t fixed = wrap_add(guess, wrap_mul(scale, q));
            int32_t out = sat16(sar(wrap_add(fixed, 1024), 11));
            h2 = h1;
            h1 = out;
            pcm_out[done++] = (int16_t)out;
        }
    }
}

/* GcAdpcmSeekTable.CreateSeekTable (Formats/GcAdpcm/GcAdpcmSeekTable.cs:25-38) on decoded PCM. out: entries*2 shorts. */
int vgo_gc_seek_table(const int16_t *pcm, int length, int samples_per_entry, int16_t *out)
{
    if (samples_per_entry <= 0) return 0;
    int entries = vgo_divide_by_round_up(length, samples_per_entry);
    memset(out, 0, sizeof(int16_t) * 2 * (size_t)entries);
    for (int i = 1; i < entries; i++) { /* the first entry should always be 0 */
        out[i * 2] = pcm[i * samples_per_entry - 1];
        out[i * 2 + 1] = pcm[i * samples_per_entry - 2];
    }
    return entries;
}

/* GcAdpcmLoopContext(adpcm, pcm, loopStart) (Formats/GcAdpcm/GcAdpcmLoopContext.cs:17-26): pred/scale, hist1, hist2. */
void vgo_gc_loop_context(const uint8_t *adpcm, const int16_t *pcm, int loop_start, int16_t out[3])
{
    out[0] = adpcm[loop_start / FRAME_SAMPLES * FRAME_BYTES]; /* GcAdpcmDecoder.GetPredictorScale :56-59 */
    out[1] = loop_start < 1 ? 0 : pcm[loop_start - 1];
    out[2] = loop_start < 2 ? 0 : pcm[loop_start - 2];
}

/* ------------------------------------------------------------------------------------------------
 * Batch drivers = the reference's Parallel.For over channels (Formats/GcAdpcm/GcAdpcmFormat.cs:65-68,
 * :45-48; EncodeChannel :129-135).  This is what bench.py times as the CPU baseline.
 * ---------------------------------------------------------------------------------------------- */
typedef void (*channel_fn)(void *ctx, int channel);

typedef struct {
    channel_fn fn;
    void *ctx;
    int n_channels;
    atomic_int next; /* dynamic schedule: each worker pulls the next unclaimed channel */
} pool_job;

static void *pool_worker(void *arg)
{
    pool_job *job = arg;
    for (;;) {
        int c = atomic_fetch_add(&job->next, 1);
        if (c >= job->n_channels) break;
        job->fn(job->ctx, c);
    }
    return NULL;
}

/* Runs fn(ctx, c) for c in [0, n_channels) on n_threads workers (<= 0: all online cores). Returns threads used. */
static int for_each_channel(channel_fn fn, void *ctx, int n_channels, int n_threads)
{
    if (n_threads <= 0) n_threads = (int)sysconf(_SC_NPROCESSORS_ONLN);
    if (n_threads < 1) n_threads = 1;
    if (n_threads > n_channels) n_threads = n_channels > 0 ? n_channels : 1;
    pool_job job = {fn, ctx, n_channels, 0};
    pthread_t *tid = malloc(sizeof(pthread_t) * (size_t)n_threads);
    int started = 0;
    for (int t = 1; t < n_threads; t++)
        if (pthread_create(&tid[started], NULL, pool_worker, &job) == 0) started++;
    pool_worker(&job);
    for (int t = 0; t < started; t++) pthread_join(tid[t], NULL);
    free(tid);
    return started + 1;
}

typedef struct {
    const int16_t *pcm; int64_t pcm_stride; int sample_count;
    int16_t *coefs; uint8_t *adpcm; int64_t adpcm_stride;
} enc_ctx;

static void encode_one(void *p, int c)
{
    enc_ctx *k = p;
    const int16_t *src = k->pcm + (int64_t)c * k->pcm_stride;
    int16_t *co = k->coefs + 16 * (int64_t)c;
    vgo_gc_calculate_coefficients(src, k->sample_count, co);
    vgo_gc_encode(src, k->sample_count, co, -1, 0, 0, k->adpcm + (int64_t)c * k->adpcm_stride);
}

int vgo_gc_encode_batch(const int16_t *pcm, int64_t pcm_stride, int n_channels, int sample_count,
                        int16_t *coefs_out, uint8_t *adpcm_out, int64_t adpcm_stride, int n_threads)
{
    enc_ctx k = {pcm, pcm_stride, sample_count, coefs_out, adpcm_out, adpcm_stride};
    return for_each_channel(encode_one, &k, n_channels, n_threads);
}

typedef struct {
    const uint8_t *adpcm; int64_t adpcm_stride; const int16_t *coefs; int sample_count;
    int16_t *pcm; int64_t pcm_stride;
} dec_ctx;

static void decode_one(void *p, int c)
{
    dec_ctx *k = p;
    vgo_gc_decode(k->adpcm + (int64_t)c * k->adpcm_stride, k->coefs + 16 * (int64_t)c, k->sample_count, 0, 0,
                  k->pcm + (int64_t)c * k->pcm_stride);
}

int vgo_gc_decode_batch(const uint8_t *adpcm, int64_t adpcm_stride, const int16_t *coefs, int n_channels,
                        int sample_count, int16_t *pcm_out, int64_t pcm_stride, int n_threads)
{
    dec_ctx k = {adpcm, adpcm_stride, coefs, sample_count, pcm_out, pcm_stride};
    return for_each_channel(decode_one, &k, n_channels, n_threads);
}
