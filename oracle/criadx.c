/*
 * oracle/criadx.c — CPU ORACLE (test infrastructure, not product) for the CRI ADX 4-bit ADPCM codec.
 *
 * Restates Codecs/CriAdx/CriAdxCodec.cs (paths relative to VGAudio's src/VGAudio/) in plain C.
 * PARITY UNPINNED: the reference has no test of any kind for this codec (SURVEY.md §4/§8c: no file under
 * src/VGAudio.Tests mentions Adx) and cannot be executed here (no .NET), so this restatement is argued line by line
 * and checked only through self-consistency properties (encode->decode tracking, encoder reconstruction == decoder).
 */
#include "vgoracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

static inline int32_t sat16(int32_t v) { return v > 32767 ? 32767 : (v < -32768 ? -32768 : v); }
static inline int32_t sat4(int32_t v) { return v > 7 ? 7 : (v < -8 ? -8 : v); }
static inline int32_t snib(int v) { v &= 0xF; return v >= 8 ? v - 16 : v; }
static inline int32_t wmul(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); }
static inline int32_t wadd(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }

/* (int)double on x64 = cvttsd2si: out-of-range and NaN give 0x80000000 (SURVEY.md A.8) */
static inline int32_t cast_double_to_int(double v)
{
    if (!(v > -2147483649.0 && v < 2147483648.0)) return INT32_MIN;
    return (int32_t)v;
}

/* Helpers.Log2 (Utilities/Helpers.cs:146-161): floor(log2(v)) for v > 0 */
static int floor_log2(int value)
{
    int r = 0;
    while (value > 1) { value >>= 1; r++; }
    return r;
}

/* CriAdxCodec.Coefs (:186-191) */
static const int16_t kFixed[4][2] = {{0, 0}, {0x0F00, 0}, {0x1CC0, (int16_t)0xF300}, {0x1880, (int16_t)0xF240}};

/* CalculateCoefficients (:173-184) */
void vgo_adx_calculate_coefficients(int highpass_freq, int sample_rate, int16_t coefs_out[2])
{
    double sqrt2 = sqrt(2.0);
    double a = sqrt2 - cos(2.0 * 3.14159265358979323846 * highpass_freq / sample_rate);
    double b = sqrt2 - 1;
    double c = (a - sqrt((a + b) * (a - b))) / b;
    coefs_out[0] = (int16_t)cast_double_to_int(c * 8192);
    coefs_out[1] = (int16_t)cast_double_to_int(c * c * -4096);
}

int vgo_adx_encoded_byte_count(int pcm_length, int padding, int frame_size)
{
    int spf = (frame_size - 2) * 2;
    return vgo_divide_by_round_up(pcm_length + padding, spf) * frame_size; /* :59-61,67 */
}

/* CalculateScale (:149-165) */
static int calc_scale(int max_distance, double *gain, int *scale_to_write, int exponential)
{
    int scale = (max_distance - 1) / 7 + 1;
    if (scale > 0x1000) scale = 0x1000;
    *scale_to_write = scale - 1;
    if (exponential) {
        int power = *scale_to_write == 0 ? 0 : floor_log2(*scale_to_write) + 1;
        scale = 1 << power;
        *scale_to_write = 12 - power;
        max_distance = 8 * scale - 1;
    }
    *gain = max_distance == 0 ? 0 : (double)32767 / max_distance;
    return scale;
}

/* ScaleShortToNibble (:167-171) */
static int32_t short_to_nibble(int32_t sample)
{
    int sgn = (sample > 0) - (sample < 0);
    sample = (sample + (32767 / 14) * sgn) / (32767 / 7);
    return sat4(sample);
}

/* EncodeFrame (:107-147).  pcm[0..1] = history, pcm[2..] = samples; rewritten with the reconstruction.  rec == NULL on
 * the normal path; otherwise the frame's facts are added to it (recording reads values the frame computes anyway). */
static void encode_frame(int16_t *pcm, uint8_t *adpcm_out, const int16_t coefs[2], int samples_per_frame, int type,
                         int version, vgo_adx_frame_trace *rec)
{
    int max_distance = 0;
    int32_t nib[512];
    if (rec) { rec->hist_in[0] = pcm[1]; rec->hist_in[1] = pcm[0]; }
    for (int i = 0; i < samples_per_frame; i++) {
        int32_t predicted = (wmul(pcm[i + 1], coefs[0]) >> 12) + (wmul(pcm[i], coefs[1]) >> 12);
        int32_t d = pcm[i + 2] - predicted;
        int32_t distance = abs(sat16(d));
        if (rec) { rec->clip1_hi += d > 32767; rec->clip1_lo += d < -32768; }
        if (distance > max_distance) max_distance = distance;
    }
    double gain;
    int scale_out;
    if (rec) {
        rec->max_distance = max_distance;
        rec->scale_raw = (max_distance - 1) / 7 + 1;
        rec->scale_lin = (rec->scale_raw > 0x1000 ? 0x1000 : rec->scale_raw) - 1;
        rec->power = type == 4 ? (rec->scale_lin == 0 ? 0 : floor_log2(rec->scale_lin) + 1) : -1;
    }
    int scale = calc_scale(max_distance, &gain, &scale_out, type == 4);
    /* the maxDistance the gain is computed from (8 * scale - 1 for the Exponential type) */
    const int md_gain = type == 4 ? 8 * scale - 1 : max_distance;
    if (rec) { rec->scale_out = scale_out; rec->md_gain = md_gain; }

    for (int i = 0; i < samples_per_frame; i++) {
        int32_t predicted = (wmul(pcm[i + 1], coefs[0]) >> 12) + (wmul(pcm[i], coefs[1]) >> 12);
        int32_t v4_predicted = wadd(wmul(pcm[i + 1], coefs[0]), wmul(pcm[i], coefs[1])) >> 12;
        int32_t raw = pcm[i + 2] - predicted;
        int32_t cast = cast_double_to_int(raw * gain);
        int32_t scaled = sat16(cast);
        int32_t q = short_to_nibble(scaled);
        nib[i] = q;
        int32_t decoded_distance = sat16(wmul(scale, q));
        if (version == 4) predicted = v4_predicted;
        int32_t recon = decoded_distance + predicted;
        if (rec) {
            double prod = raw * gain;
            rec->cast_ovf += !(prod > -2147483649.0 && prod < 2147483648.0);
            rec->clip2_hi += cast > 32767;
            rec->clip2_lo += cast < -32768;
            rec->nibbles[q & 15]++;
            if (md_gain > 0)
                for (int k = 1; k <= 7; k++)
                    rec->ties[k] += (int64_t)abs(raw) * 32767 == (int64_t)(4681 * k - 2340) * md_gain;
            rec->recon_hi += recon > 32767;
            rec->recon_lo += recon < -32768;
            rec->v4_differs += v4_predicted != (wmul(pcm[i + 1], coefs[0]) >> 12) + (wmul(pcm[i], coefs[1]) >> 12);
        }
        pcm[i + 2] = (int16_t)sat16(recon);
    }
    adpcm_out[0] = (uint8_t)((scale_out >> 8) & 0x1f);
    adpcm_out[1] = (uint8_t)scale_out;
    for (int i = 0; i < samples_per_frame / 2; i++)
        adpcm_out[i + 2] = (uint8_t)((nib[2 * i] << 4) | (nib[2 * i + 1] & 0xF));
    if (rec) { rec->hist_out[0] = pcm[samples_per_frame + 1]; rec->hist_out[1] = pcm[samples_per_frame]; }
}

void vgo_adx_encode_frame(int16_t *pcm, uint8_t *adpcm_out, const int16_t coefs[2], int samples_per_frame, int type,
                          int version)
{
    encode_frame(pcm, adpcm_out, coefs, samples_per_frame, type, version, NULL);
}

/* Encode (:56-105).  Returns the value the reference leaves in config.History (:73), 0 if untouched.  trace == NULL on
 * the normal path, else one record per frame. */
static int encode(const int16_t *pcm, int pcm_length, int sample_rate, int frame_size, int version, int padding, int type,
                  int filter, uint8_t *adpcm_out, vgo_adx_frame_trace *trace)
{
    int sample_count = pcm_length + padding;
    int spf = (frame_size - 2) * 2;
    int frame_count = vgo_divide_by_round_up(sample_count, spf);
    int padding_remaining = padding;
    int16_t coefs[2];
    if (type == 2) { coefs[0] = kFixed[filter & 3][0]; coefs[1] = kFixed[filter & 3][1]; }
    else vgo_adx_calculate_coefficients(500, sample_rate, coefs);

    int16_t *buf = calloc((size_t)spf + 2, sizeof(int16_t));
    uint8_t *frame = calloc((size_t)frame_size, 1);
    memset(adpcm_out, 0, (size_t)frame_count * frame_size);
    if (trace) memset(trace, 0, (size_t)frame_count * sizeof *trace);
    int history = 0;
    if (version == 4 && padding == 0 && pcm_length > 0) {
        buf[0] = pcm[0];
        buf[1] = pcm[0];
        history = pcm[0];
    }
    for (int i = 0; i < frame_count; i++) {
        int to_copy = sample_count - i * spf;
        if (to_copy > spf) to_copy = spf;
        int start = 2;
        vgo_adx_frame_trace *rec = trace ? trace + i : NULL;
        if (rec) { rec->frame = i; rec->power = -1; }
        if (padding_remaining != 0) {
            while (padding_remaining > 0 && to_copy > 0) { padding_remaining--; to_copy--; start++; }
            if (rec && start > 2) rec->layout |= VGO_ADX_FRAME_PADDED;
            if (to_copy == 0) {
                if (rec) rec->layout |= VGO_ADX_FRAME_SKIPPED;
                continue;
            }
        }
        if (rec && start - 2 + to_copy < spf) rec->layout |= VGO_ADX_FRAME_PARTIAL;
        int src = i * spf - padding;
        if (src < 0) src = 0;
        memcpy(buf + start, pcm + src, (size_t)to_copy * sizeof(int16_t));
        memset(buf + start + to_copy, 0, (size_t)(spf - to_copy - start + 2) * sizeof(int16_t));
        encode_frame(buf, frame, coefs, spf, type, version, rec);
        if (type == 2) frame[0] |= (uint8_t)(filter << 5);
        memcpy(adpcm_out + (size_t)i * frame_size, frame, (size_t)frame_size);
        buf[0] = buf[spf];
        buf[1] = buf[spf + 1];
    }
    free(buf);
    free(frame);
    return history;
}

int vgo_adx_encode(const int16_t *pcm, int pcm_length, int sample_rate, int frame_size, int version, int padding,
                   int type, int filter, uint8_t *adpcm_out)
{
    return encode(pcm, pcm_length, sample_rate, frame_size, version, padding, type, filter, adpcm_out, NULL);
}

int vgo_adx_encode_trace(const int16_t *pcm, int pcm_length, int sample_rate, int frame_size, int version, int padding,
                         int type, int filter, uint8_t *adpcm_out, vgo_adx_frame_trace *trace_out)
{
    return encode(pcm, pcm_length, sample_rate, frame_size, version, padding, type, filter, adpcm_out, trace_out);
}

int vgo_adx_frame_trace_size(void) { return (int)sizeof(vgo_adx_frame_trace); }

/* Decode (:9-54) */
void vgo_adx_decode(const uint8_t *adpcm, int sample_count, int sample_rate, int highpass_freq, int frame_size,
                    int version, int history, int padding, int type, int16_t *pcm_out)
{
    int spf = (frame_size - 2) * 2;
    int16_t calc[2];
    vgo_adx_calculate_coefficients(highpass_freq, sample_rate, calc);
    int hist1 = history, hist2 = history;
    int frame_count = vgo_divide_by_round_up(sample_count, spf);
    int current = 0;
    int start_sample = padding > 0 ? padding % spf : 0;
    int in = padding / spf * frame_size;

    for (int i = 0; i < frame_count; i++) {
        int filter_num = ((adpcm[in] >> 4) & 0xF) >> 1;
        /* the reference indexes a 1-entry table for non-Fixed types (any other filter bits throw); Fixed has 4 */
        const int16_t *co = type == 2 ? kFixed[filter_num & 3] : calc;
        int16_t scale = (int16_t)((adpcm[in] << 8 | adpcm[in + 1]) & 0x1FFF);
        scale = (int16_t)(type == 4 ? 1 << ((12 - scale) & 31) : scale + 1);
        in += 2 + start_sample / 2;
        int to_read = sample_count - current;
        if (to_read > spf) to_read = spf;
        for (int s = start_sample; s < to_read; s++) {
            int32_t sample = s % 2 == 0 ? snib(adpcm[in] >> 4) : snib(adpcm[in++]);
            if (version == 4)
                sample = wadd(wmul(scale, sample), wadd(wmul(hist1, co[0]), wmul(hist2, co[1])) >> 12);
            else
                sample = wadd(wadd(wmul(scale, sample), wmul(hist1, co[0]) >> 12), wmul(hist2, co[1]) >> 12);
            int32_t out = sat16(sample);
            hist2 = hist1;
            hist1 = out;
            pcm_out[current++] = (int16_t)out;
        }
        start_sample = 0;
    }
}
