/* hcakeys.c - the key search of HcaReader.FindKey for type-56 .hca files (Containers/Hca/HcaReader.cs:32, 238-252) with
 * CriHcaEncryption.FindKey / TestKey / FindFirstNonEmptyFrame / FrameEmpty (Codecs/CriHca/CriHcaEncryption.cs:34-87)
 * and CriHcaPacking.UnpackingWasSuccessful / FrameEmpty (Codecs/CriHca/CriHcaPacking.cs:207-229) - TEST INFRASTRUCTURE.
 *
 * The key list is the caller's (the reference's CriHcaEncryptionKeys list is not carried).  One frame state is kept for
 * every key and frame, as the reference's FindKey keeps one CriHcaFrame.
 *
 * Outcome of one (file, key): 0 TestKey accepts it, else 1 + 3 * j + r with j the window frame it stops at and r 0 a bad
 * sync word (InvalidDataException out of FindKey), 1 a scale-factor delta out of range, 2 UnpackingWasSuccessful false.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "vgoracle.h"

#pragma GCC diagnostic push
#pragma GCC diagnostic ignored "-Wunused-const-variable"
#include "hca_tables.inc"
#pragma GCC diagnostic pop

/* ------------------------------------------------------------------------------------------------
 * One CriHcaFrame (CriHcaFrame.cs, CriHcaChannel.cs) with what UnpackFrame reads and writes.  FindKey keeps one for every
 * key and frame, and so does this file: nothing is cleared between calls but what UnpackFrame itself clears.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    int type, coded_count, delta_bits;
    int scale_factors[128], resolution[128], intensity[8], hfr_scales[8], quantized[8][128];
} key_channel;

typedef struct {
    vgo_hca_info hca;
    key_channel ch[8];
    uint8_t ath[128];
    int noise_level, eval_boundary;
} key_frame;

/* GetChannelTypes (CriHcaFrame.cs:34-52): 0 discrete, 1 stereo primary, 2 stereo secondary */
static void key_channel_types(const vgo_hca_info *h, int types[8])
{
    static const int t2[] = {1, 2}, t3[] = {1, 2, 0}, t4a[] = {1, 2, 0, 0}, t4b[] = {1, 2, 1, 2}, t5a[] = {1, 2, 0, 0, 0},
                     t5b[] = {1, 2, 0, 1, 2}, t6[] = {1, 2, 0, 0, 1, 2}, t7[] = {1, 2, 0, 0, 1, 2, 0},
                     t8[] = {1, 2, 0, 0, 1, 2, 1, 2};
    memset(types, 0, sizeof(int) * 8);
    const int per_track = h->channel_count / (h->track_count > 0 ? h->track_count : 1);
    if (h->stereo_band_count == 0 || per_track == 1) return;
    const int *src = NULL;
    switch (per_track) {
    case 2: src = t2; break;
    case 3: src = t3; break;
    case 4: src = h->channel_config != 0 ? t4a : t4b; break;
    case 5: src = h->channel_config > 2 ? t5a : t5b; break;
    case 6: src = t6; break;
    case 7: src = t7; break;
    case 8: src = t8; break;
    default: return;
    }
    memcpy(types, src, sizeof(int) * (size_t)per_track);
}

/* new CriHcaFrame(hca) (CriHcaFrame.cs:20-32) with AthCurve = UseAthCurve ? ScaleAthCurve(SampleRate) : new byte[128] */
static key_frame *key_frame_new(const vgo_hca_info *h)
{
    key_frame *f = calloc(1, sizeof *f);
    int types[8];
    f->hca = *h;
    key_channel_types(h, types);
    for (int c = 0; c < h->channel_count && c < 8; c++) {
        f->ch[c].type = types[c];
        f->ch[c].coded_count = types[c] == 2 ? h->base_band_count : h->base_band_count + h->stereo_band_count;
    }
    if (h->use_ath_curve) { /* ScaleAthCurve :60-84 */
        int acc = 0, i;
        for (i = 0; i < 128; i++) {
            acc += h->sample_rate;
            const int index = acc >> 13;
            if (index >= (int)sizeof kHcaAthCurve) break;
            f->ath[i] = kHcaAthCurve[index];
        }
        for (; i < 128; i++) f->ath[i] = 0xff;
    }
    return f;
}

/* BitReader (Utilities/BitReader.cs): PeekInt reads bits past the end as zero */
typedef struct { const uint8_t *buf; int length_bits, pos; } key_reader;
static int kr_peek(const key_reader *r, int count)
{
    int v = 0;
    for (int i = 0; i < count; i++) {
        const int p = r->pos + i;
        v = (v << 1) | (p < r->length_bits ? (r->buf[p >> 3] >> (7 - (p & 7))) & 1 : 0);
    }
    return v;
}
static int kr_read(key_reader *r, int count) { const int v = kr_peek(r, count); r->pos += count; return v; }

/* CalculateResolution (CriHcaPacking.cs:60-69) */
static int key_resolution(int scale_factor, int noise_level)
{
    if (scale_factor == 0) return 0;
    int p = noise_level - 5 * scale_factor / 2 + 2;
    p = p < 0 ? 0 : (p > 58 ? 58 : p);
    return kHcaScaleToResolutionCurve[p];
}

/* DeltaDecode (:180-205) */
static int key_delta_decode(key_reader *r, int delta_bits, int data_bits, int count, int *out)
{
    out[0] = kr_read(r, data_bits);
    const int max_delta = 1 << (delta_bits - 1), max_value = (1 << data_bits) - 1;
    for (int i = 1; i < count; i++) {
        const int delta = kr_read(r, delta_bits) - (max_delta - 1); /* ReadOffsetBinary, OffsetBias.Positive */
        if (delta < max_delta) {
            const int value = out[i - 1] + delta;
            if (value < 0 || value > max_value) return 0;
            out[i] = value;
        } else {
            out[i] = kr_read(r, data_bits);
        }
    }
    return 1;
}

/* UnpackFrame (:10-15) without its last test: -2 the sync word is not 0xFFFF (InvalidDataException), 1 a scale-factor
 * delta out of range (UnpackFrameHeader returns false), 0 the frame was read to its end; *pos_out the bit position then */
static int key_unpack(key_frame *f, const uint8_t *data, int *pos_out)
{
    key_reader r = {data, f->hca.frame_size * 8, 0};
    if (kr_read(&r, 16) != 0xffff) return -2; /* UnpackFrameHeader :71-107 */
    f->noise_level = kr_read(&r, 9);
    f->eval_boundary = kr_read(&r, 7);
    for (int c = 0; c < f->hca.channel_count; c++) {
        key_channel *ch = &f->ch[c];
        ch->delta_bits = kr_read(&r, 3); /* ReadScaleFactors :109-128 */
        if (ch->delta_bits == 0) {
            memset(ch->scale_factors, 0, sizeof ch->scale_factors);
        } else if (ch->delta_bits >= 6) {
            for (int i = 0; i < ch->coded_count; i++) ch->scale_factors[i] = kr_read(&r, 6);
        } else if (!key_delta_decode(&r, ch->delta_bits, 6, ch->coded_count, ch->scale_factors)) {
            return 1;
        }
        for (int i = 0; i < f->eval_boundary; i++)
            ch->resolution[i] = key_resolution(ch->scale_factors[i], f->ath[i] + f->noise_level - 1);
        for (int i = f->eval_boundary; i < ch->coded_count; i++)
            ch->resolution[i] = key_resolution(ch->scale_factors[i], f->ath[i] + f->noise_level);
        if (ch->type == 2) {
            for (int i = 0; i < 8; i++) ch->intensity[i] = kr_read(&r, 4); /* ReadIntensity :130-136 */
        } else if (f->hca.hfr_group_count > 0) {
            for (int i = 0; i < f->hca.hfr_group_count; i++) ch->hfr_scales[i] = kr_read(&r, 6); /* :138-144 */
        }
    }
    for (int sf = 0; sf < 8; sf++) /* ReadSpectralCoefficients :146-178 */
        for (int c = 0; c < f->hca.channel_count; c++) {
            key_channel *ch = &f->ch[c];
            for (int s = 0; s < ch->coded_count; s++) {
                const int resolution = ch->resolution[s];
                int bits = kHcaQuantizedSpectrumMaxBits[resolution];
                const int code = kr_peek(&r, bits);
                if (resolution < 8) {
                    bits = kHcaQuantizedSpectrumBits[resolution][code];
                    ch->quantized[sf][s] = kHcaQuantizedSpectrumValue[resolution][code];
                } else {
                    const int q = code / 2 * (1 - (code % 2 * 2)); /* sign-magnitude, the low bit is the sign */
                    if (q == 0) bits--;
                    ch->quantized[sf][s] = q;
                }
                r.pos += bits;
            }
        }
    *pos_out = r.pos;
    return 0;
}

#define FRAMES_TO_TEST 10

/* CriHcaEncryption.FrameEmpty (:77-87): bytes [2, size - 2) all zero */
int vgo_hca_key_frame_empty(const uint8_t *frame, int size)
{
    for (int i = 2; i < size - 2; i++)
        if (frame[i] != 0) return 0;
    return 1;
}

/* FindFirstNonEmptyFrame (:65-75) over the encrypted frames, and TestKey's window end (:50-51) */
void vgo_hca_key_window(const uint8_t *frames, int frame_count, int frame_size, int *start_out, int *end_out)
{
    int start = 0;
    for (int i = 0; i < frame_count; i++)
        if (!vgo_hca_key_frame_empty(frames + (size_t)i * frame_size, frame_size)) { start = i; break; }
    *start_out = start;
    *end_out = frame_count < start + FRAMES_TO_TEST ? frame_count : start + FRAMES_TO_TEST;
}

/* TestKey (:48-63) with one key's decryption table on the state's frame; no_crc 1 leaves the last two bytes as they are
 * instead of writing CryptFrame's CRC there (it exists only to show which outcomes the CRC decides).  remaining_out
 * (may be null, FRAMES_TO_TEST entries): Remaining after each window frame that reached UnpackingWasSuccessful. */
static int test_key(key_frame *state, const vgo_hca_info *h, const uint8_t *frames, const uint8_t *table, int start, int end,
                    int no_crc, int *remaining_out, uint8_t *buffer)
{
    const int fs = h->frame_size;
    for (int i = start; i < end; i++) {
        const int j = i - start;
        memcpy(buffer, frames + (size_t)i * fs, (size_t)fs);
        if (no_crc) { /* CryptFrame's substitution alone */
            for (int b = 0; b < fs - 2; b++) buffer[b] = table[buffer[b]];
        } else {
            vgo_hca_crypt_frame(buffer, fs, table); /* CryptFrame (:20-32) */
        }
        int pos = 0;
        const int rc = key_unpack(state, buffer, &pos);
        if (rc == -2) return 1 + 3 * j;
        if (rc == 1) return 1 + 3 * j + 1;
        const int remaining = fs * 8 - pos; /* BitReader.Remaining */
        if (remaining_out) remaining_out[j] = remaining;
        /* UnpackingWasSuccessful (:207-214) with FrameEmpty (:216-229) */
        const int noise = state->noise_level;
        int delta_any = 0;
        for (int c = 0; c < h->channel_count; c++) delta_any |= state->ch[c].delta_bits > 0;
        const int frame_empty = noise == 0 && !delta_any;
        const int ok = (remaining >= 16 && remaining <= 128) || frame_empty || (noise == 0 && remaining >= 16);
        if (!ok) return 1 + 3 * j + 2;
    }
    return 0;
}

/* Every (key) outcome of one file: outcome_out[n_keys], remaining_out[n_keys][FRAMES_TO_TEST] (may be null, entries of
 * frames that did not reach UnpackingWasSuccessful are left as they are) */
void vgo_hca_key_outcomes(const vgo_hca_info *h, const uint8_t *frames, const uint64_t *key_codes, int n_keys, int no_crc,
                          int32_t *outcome_out, int32_t *remaining_out)
{
    int start, end;
    vgo_hca_key_window(frames, h->frame_count, h->frame_size, &start, &end);
    key_frame *state = key_frame_new(h);
    uint8_t *buffer = malloc((size_t)h->frame_size + 1);
    for (int k = 0; k < n_keys; k++) {
        uint8_t dec[256], enc[256];
        vgo_hca_key_tables(56, key_codes[k], dec, enc);
        int rem[FRAMES_TO_TEST];
        for (int j = 0; j < FRAMES_TO_TEST; j++) rem[j] = INT32_MIN;
        outcome_out[k] = test_key(state, h, frames, dec, start, end, no_crc, rem, buffer);
        if (remaining_out)
            for (int j = 0; j < FRAMES_TO_TEST; j++)
                if (rem[j] != INT32_MIN) remaining_out[(size_t)k * FRAMES_TO_TEST + j] = rem[j];
    }
    free(buffer);
    free(state);
}

/* CriHcaEncryption.FindKey (:34-46) as HcaReader.FindKey calls it for "ciph" 56: the index of the first key TestKey
 * accepts, or -1.  *status_out: 0 found, 1 a bad sync word thrown out of FindKey (InvalidDataException), 2 no key
 * ("Cannot find key to decrypt HCA file.") */
int vgo_hca_find_key(const vgo_hca_info *h, const uint8_t *frames, const uint64_t *key_codes, int n_keys, int *status_out)
{
    int start, end, found = -1;
    vgo_hca_key_window(frames, h->frame_count, h->frame_size, &start, &end);
    key_frame *state = key_frame_new(h);
    uint8_t *buffer = malloc((size_t)h->frame_size + 1);
    *status_out = 2;
    for (int k = 0; k < n_keys; k++) {
        uint8_t dec[256], enc[256];
        vgo_hca_key_tables(56, key_codes[k], dec, enc);
        const int outcome = test_key(state, h, frames, dec, start, end, 0, NULL, buffer);
        if (outcome == 0) { *status_out = 0; found = k; break; }
        if ((outcome - 1) % 3 == 0) { *status_out = 1; break; }
    }
    free(buffer);
    free(state);
    return found;
}
