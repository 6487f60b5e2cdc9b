/* containers.c — CPU restatement of the container layer either side of the codec path (SURVEY.md §8f rank 2-4):
 * WAVE front end, DSP / ADX / HCA writers, the DSP reader, CRI ADX / HCA encryption.  TEST INFRASTRUCTURE (see
 * vgoracle.h): only tests/, smoke() and bench.py's CPU legs may load it.
 *
 * Pins the reference holds for this layer: build -> parse round trips only (src/VGAudio.Tests/Containers/DspTests.cs:9-19,
 * WaveTests.cs:9-55 through BuildParseTests.cs:9-16); no golden file bytes, no encryption test => header bytes and
 * key schedules are "parity unpinned" like the codecs' payloads.  Citations are relative to VGAudio's src/VGAudio/.
 */
#include <stdlib.h>
#include <string.h>

#include "vgoracle.h"

static void be16(uint8_t *p, int v) { p[0] = (uint8_t)(v >> 8); p[1] = (uint8_t)v; }
static void be32(uint8_t *p, int32_t v) { p[0] = (uint8_t)((uint32_t)v >> 24); p[1] = (uint8_t)((uint32_t)v >> 16); p[2] = (uint8_t)((uint32_t)v >> 8); p[3] = (uint8_t)v; }
static void le16(uint8_t *p, int v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); }
static void le32(uint8_t *p, int32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)((uint32_t)v >> 8); p[2] = (uint8_t)((uint32_t)v >> 16); p[3] = (uint8_t)((uint32_t)v >> 24); }
static int rd_le16(const uint8_t *p) { return p[0] | (p[1] << 8); }
static int rd_le16s(const uint8_t *p) { return (int16_t)(p[0] | (p[1] << 8)); }
static int32_t rd_le32(const uint8_t *p) { return (int32_t)((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24)); }
static int rd_be16s(const uint8_t *p) { return (int16_t)((p[0] << 8) | p[1]); }
static int32_t rd_be32(const uint8_t *p) { return (int32_t)(((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3]); }
static int next_multiple(int value, int multiple) /* Utilities/Helpers.cs:71-80 */
{
    if (multiple <= 0) return value;
    if (value % multiple == 0) return value;
    return value + multiple - value % multiple;
}

/* ============================================================================================================
 * WAVE front end: RiffParser.ParseRiff (Utilities/Riff/RiffParser.cs:38-86), the chunk classes next to it,
 * WaveReader.ReadFile / ValidateWaveFile (Containers/Wave/WaveReader.cs:13-51, :71-95)
 * ============================================================================================================ */
static const uint8_t kPcmGuid[16] = {0x01, 0x00, 0x00, 0x00, 0x00, 0x00, 0x10, 0x00, 0x80, 0x00, 0x00, 0xAA, 0x00, 0x38, 0x9B, 0x71};

int vgo_wave_parse(const uint8_t *f, int64_t len, vgo_wave_info *out)
{
    memset(out, 0, sizeof *out);
    if (len < 12) return VGO_E_TRUNCATED;                       /* EndOfStreamException in RiffChunk.Parse */
    if (memcmp(f, "RIFF", 4) != 0) return VGO_E_NOT_RIFF;       /* RiffChunk.cs:20-23 */
    const int32_t riff_size = rd_le32(f + 4);
    const int is_wave = memcmp(f + 8, "WAVE", 4) == 0;
    int64_t pos = 12;
    const int64_t end = 8 + (int64_t)riff_size;                 /* RiffParser.cs:46-47 */
    int have_fmt = 0, have_data = 0, have_smpl = 0, have_ext = 0;
    int format_tag = 0, channels = 0, block_align = 0, bits = 0;
    int32_t sample_rate = 0, data_chunk_size = 0, loop_start = 0, loop_end = 0;
    int64_t data_off = 0, data_avail = 0;
    int smpl_loops = 0;
    uint8_t sub_format[16] = {0};
    while (pos + 8 < end) {                                     /* :50 */
        if (pos + 8 > len) return VGO_E_TRUNCATED;
        const uint8_t *id = f + pos;
        const int32_t size = rd_le32(f + pos + 4);
        const int64_t body = pos + 8;
        if (size < 0) return VGO_E_TRUNCATED;
        if (memcmp(id, "fmt ", 4) == 0) {                       /* WaveFmtChunk.cs:16-34 */
            if (body + 16 > len) return VGO_E_TRUNCATED;
            format_tag = rd_le16(f + body);
            channels = rd_le16s(f + body + 2);
            sample_rate = rd_le32(f + body + 4);
            block_align = rd_le16s(f + body + 12);
            bits = rd_le16s(f + body + 14);
            have_ext = 0;
            if (format_tag == 0xFFFE) {                         /* WaveFormatExtensible.cs:20-27 */
                if (body + 16 + 24 > len) return VGO_E_TRUNCATED;
                memcpy(sub_format, f + body + 16 + 8, 16);
                have_ext = 1;
            }
            have_fmt = 1;
        } else if (memcmp(id, "smpl", 4) == 0) {                /* WaveSmplChunk.cs:18-44 */
            if (body + 36 > len) return VGO_E_TRUNCATED;
            smpl_loops = rd_le32(f + body + 28);
            if (smpl_loops < 0) return VGO_E_TRUNCATED;         /* new SampleLoop[negative] throws */
            if (body + 36 + 24ll * smpl_loops > len) return VGO_E_TRUNCATED;
            if (smpl_loops > 0) { loop_start = rd_le32(f + body + 36 + 8); loop_end = rd_le32(f + body + 36 + 12); }
            have_smpl = 1;
        } else if (memcmp(id, "data", 4) == 0) {                /* WaveDataChunk.cs:11-17: ReadBytes returns what is left */
            data_chunk_size = size;
            data_off = body;
            data_avail = len - body < size ? (len - body < 0 ? 0 : len - body) : size;
            have_data = 1;
        }
        const int64_t chunk_end = body + size;
        pos = chunk_end + (chunk_end & 1);                      /* :83 sub-chunks are 2-byte aligned */
    }
    /* ValidateWaveFile, in its order */
    if (!is_wave) return VGO_E_NOT_WAVE;
    if (!have_fmt) return VGO_E_NO_FMT;
    if (!have_data) return VGO_E_NO_DATA;
    const int bytes_per_sample = (bits + 7) / 8;                /* DivideByRoundUp for the positive values that pass below */
    if (format_tag != 0x0001 && format_tag != 0xFFFE) return VGO_E_NOT_PCM;
    if (bits != 16 && bits != 8) return VGO_E_BITS;
    if (channels == 0) return VGO_E_CHANNELS;
    if (block_align != bytes_per_sample * channels) return VGO_E_BLOCK_ALIGN;
    if (have_ext && memcmp(sub_format, kPcmGuid, 16) != 0) return VGO_E_NOT_PCM;
    if (channels < 0) return VGO_E_CHANNELS;                    /* new short[negative][] throws in InterleavedByteToShort */
    out->channel_count = channels;
    out->sample_rate = sample_rate;
    out->bits_per_sample = bits;
    out->data_offset = data_off;
    out->data_size = data_avail;
    (void)data_chunk_size;
    /* the format's SampleCount is the decoded arrays' length (Interleave.cs:190, Pcm16FormatBuilder.cs:17) */
    out->sample_count = (int32_t)(data_avail / bytes_per_sample / channels);
    if (have_smpl && smpl_loops > 0) {                          /* WaveReader.cs:33-38 */
        out->loop_start = loop_start;
        out->loop_end = loop_end;
        out->looping = loop_end > loop_start;
    }
    if (out->looping) {                                         /* AudioFormatBaseBuilder.WithLoop :23-50 */
        if (loop_start < 0 || loop_start > out->sample_count || loop_end < 0 || loop_end > out->sample_count)
            return VGO_E_LOOP;
    } else {
        out->loop_start = 0;                                    /* WithLoop(false) :52-58 */
        out->loop_end = 0;
    }
    return 0;
}

/* InterleavedByteToShort (Utilities/Interleave.cs:188-207) */
void vgo_wave_read16(const uint8_t *f, const vgo_wave_info *w, int16_t *const *channels)
{
    const uint8_t *d = f + w->data_offset;
    for (int i = 0; i < w->sample_count; i++)
        for (int o = 0; o < w->channel_count; o++) {
            const int64_t off = ((int64_t)i * w->channel_count + o) * 2;
            channels[o][i] = (int16_t)(d[off] | (d[off + 1] << 8));
        }
}

/* 8-bit data: DeInterleave(bytesPerSample = 1) then Pcm8Codec.Decode (Codecs/Pcm8/Pcm8Codec.cs:23) when PCM16 is asked for */
void vgo_wave_read8_as16(const uint8_t *f, const vgo_wave_info *w, int16_t *const *channels)
{
    const uint8_t *d = f + w->data_offset;
    for (int i = 0; i < w->sample_count; i++)
        for (int o = 0; o < w->channel_count; o++)
            channels[o][i] = (int16_t)((d[(int64_t)i * w->channel_count + o] - 0x80) << 8);
}

/* WaveWriter, 16-bit codec (Containers/Wave/WaveWriter.cs:24-153): only here so that the reference's own pin for the
 * reader - WaveWriter -> WaveReader returns the same audio (WaveTests.cs) - can be replayed */
static int wave_channel_mask(int n)
{
    switch (n) { case 4: return 0x0033; case 5: return 0x0133; case 6: return 0x0633; case 7: return 0x01f3; case 8: return 0x06f3; default: return (1 << n) - 1; }
}
int64_t vgo_wave_file_size(int channels, int samples, int looping)
{
    const int fmt = channels > 2 ? 40 : 16;
    return 8 + 4 + 8 + fmt + 8 + (int64_t)channels * samples * 2 + (looping ? 8 + 0x3c : 0);
}
void vgo_wave_write16(const int16_t *const *pcm, int channels, int samples, int sample_rate, int looping, int loop_start, int loop_end, uint8_t *out)
{
    const int fmt = channels > 2 ? 40 : 16;
    const int64_t total = vgo_wave_file_size(channels, samples, looping);
    memset(out, 0, (size_t)total);
    uint8_t *p = out;
    memcpy(p, "RIFF", 4); le32(p + 4, (int32_t)(total - 8)); memcpy(p + 8, "WAVE", 4); p += 12;
    memcpy(p, "fmt ", 4); le32(p + 4, fmt);
    le16(p + 8, channels > 2 ? 0xFFFE : 1); le16(p + 10, channels); le32(p + 12, sample_rate);
    le32(p + 16, sample_rate * 2 * channels); le16(p + 20, 2 * channels); le16(p + 22, 16);
    if (channels > 2) { le16(p + 24, 22); le16(p + 26, 16); le32(p + 28, wave_channel_mask(channels)); memcpy(p + 32, kPcmGuid, 16); }
    p += 8 + fmt;
    if (looping) {
        memcpy(p, "smpl", 4); le32(p + 4, 0x3c);
        le32(p + 8 + 28, 1);                                   /* seven zero ints, then the loop count */
        le32(p + 8 + 36 + 8, loop_start); le32(p + 8 + 36 + 12, loop_end);
        p += 8 + 0x3c;
    }
    memcpy(p, "data", 4); le32(p + 4, channels * samples * 2); p += 8;
    for (int i = 0; i < samples; i++)                           /* ShortToInterleavedByte (Interleave.cs:169-186) */
        for (int j = 0; j < channels; j++) le16(p + ((int64_t)i * channels + j) * 2, pcm[j][i]);
}

/* ============================================================================================================
 * DSP: DspWriter (Containers/Dsp/DspWriter.cs:17-108), DspReader (Containers/Dsp/DspReader.cs:15-127)
 * ============================================================================================================ */
static int dsp_alignment(const vgo_dsp_desc *d) { return next_multiple(d->loop_start, d->loop_point_alignment) - d->loop_start; }
static int dsp_loop_end(const vgo_dsp_desc *d) { return d->loop_end + dsp_alignment(d); }
static int dsp_sample_count(const vgo_dsp_desc *d) /* :22 */
{
    const int le = dsp_loop_end(d);
    return d->trim_file && d->looping ? le : (d->sample_count > le ? d->sample_count : le);
}
static int dsp_audio_data_size(const vgo_dsp_desc *d) /* :105-106 */
{
    return next_multiple(vgo_gc_sample_count_to_byte_count(dsp_sample_count(d)), d->channel_count == 1 ? 1 : 8);
}
int64_t vgo_dsp_file_size(const vgo_dsp_desc *d) { return (int64_t)(0x60 + dsp_audio_data_size(d)) * d->channel_count; }

/* adpcm[c]: the channel's GetAdpcmAudio() = SampleCountToByteCount(d->sample_count) bytes; coefs [ch][16];
 * gain [ch] (may be NULL = 0); start_hist [ch][2] (may be NULL = 0,0; PredScale is adpcm[c][0], GcAdpcmChannel.cs:44);
 * loop_ctx [ch][3] = PredScale, Hist1, Hist2 (ignored unless looping) */
int vgo_dsp_write(const vgo_dsp_desc *d, const uint8_t *const *adpcm, const int16_t *coefs, const int16_t *gain,
                  const int16_t *start_hist, const int16_t *loop_ctx, uint8_t *out)
{
    const int ch = d->channel_count;
    const int sc = dsp_sample_count(d);
    const int in_size = vgo_gc_sample_count_to_byte_count(d->sample_count);
    const int data_size = dsp_audio_data_size(d);
    const int bpi = vgo_gc_sample_count_to_byte_count(d->samples_per_interleave);
    if (ch < 1 || d->samples_per_interleave < 1 || d->samples_per_interleave % 14 != 0) return VGO_E_ARG;
    if (ch == 1 && vgo_gc_sample_count_to_byte_count(sc) > in_size) return VGO_E_ARG; /* Stream.Write past the array: ArgumentException */
    memset(out, 0, (size_t)vgo_dsp_file_size(d));
    const int align = dsp_alignment(d);
    const int start_addr = vgo_gc_sample_to_nibble(d->looping ? d->loop_start + align : 0);   /* :33 */
    const int end_addr = vgo_gc_sample_to_nibble(d->looping ? dsp_loop_end(d) : sc - 1);     /* :34 */
    for (int i = 0; i < ch; i++) {                                                            /* WriteHeader :54-84 */
        uint8_t *h = out + 0x60 * i;
        be32(h + 0x00, sc);
        be32(h + 0x04, vgo_gc_sample_count_to_nibble_count(sc));
        be32(h + 0x08, d->sample_rate);
        be16(h + 0x0c, d->looping ? 1 : 0);
        be16(h + 0x0e, 0);
        be32(h + 0x10, start_addr);
        be32(h + 0x14, end_addr);
        be32(h + 0x18, vgo_gc_sample_to_nibble(0));
        for (int k = 0; k < 16; k++) be16(h + 0x1c + 2 * k, coefs[i * 16 + k]);
        be16(h + 0x3c, gain ? gain[i] : 0);
        be16(h + 0x3e, in_size > 0 ? adpcm[i][0] : 0);
        be16(h + 0x40, start_hist ? start_hist[2 * i] : 0);
        be16(h + 0x42, start_hist ? start_hist[2 * i + 1] : 0);
        if (d->looping) for (int k = 0; k < 3; k++) be16(h + 0x44 + 2 * k, loop_ctx[3 * i + k]);
        be16(h + 0x4a, ch == 1 ? 0 : ch);
        be16(h + 0x4c, ch == 1 ? 0 : bpi / 8);
    }
    uint8_t *data = out + 0x60 * ch;                                                          /* WriteData :86-99 */
    if (ch == 1) memcpy(data, adpcm[0], (size_t)vgo_gc_sample_count_to_byte_count(sc));
    else vgo_interleave(adpcm, ch, in_size, bpi, data_size, data);
    return 0;
}

/* DspReader.ReadHeader (:57-104): validation in the reference's order */
int vgo_dsp_parse(const uint8_t *f, int64_t len, vgo_dsp_info *o)
{
    memset(o, 0, sizeof *o);
    if (len < 0x60) return VGO_E_TRUNCATED;
    o->sample_count = rd_be32(f);
    o->nibble_count = rd_be32(f + 4);
    o->sample_rate = rd_be32(f + 8);
    o->looping = rd_be16s(f + 0x0c) == 1;
    o->format = rd_be16s(f + 0x0e);
    o->start_address = rd_be32(f + 0x10);
    o->end_address = rd_be32(f + 0x14);
    o->current_address = rd_be32(f + 0x18);
    o->channel_count = rd_be16s(f + 0x4a);
    o->frames_per_interleave = rd_be16s(f + 0x4c);
    if (o->channel_count == 0) o->channel_count = 1;
    if (o->channel_count < 0 || o->channel_count > VGO_DSP_MAX_CHANNELS) return VGO_E_CHANNELS;
    if (len < 0x60ll * o->channel_count) return VGO_E_TRUNCATED;
    for (int i = 0; i < o->channel_count; i++) {
        const uint8_t *h = f + 0x60 * i;
        for (int k = 0; k < 16; k++) o->coefs[i][k] = (int16_t)rd_be16s(h + 0x1c + 2 * k);
        o->gain[i] = (int16_t)rd_be16s(h + 0x3c);
        for (int k = 0; k < 3; k++) { o->start_ctx[i][k] = (int16_t)rd_be16s(h + 0x3e + 2 * k); o->loop_ctx[i][k] = (int16_t)rd_be16s(h + 0x44 + 2 * k); }
    }
    if (len < 0x60 + (int64_t)vgo_gc_sample_count_to_byte_count(o->sample_count)) return VGO_E_TRUNCATED;  /* :90-93 */
    if (vgo_gc_sample_count_to_nibble_count(o->sample_count) != o->nibble_count) return VGO_E_NIBBLES;    /* :95-98 */
    if (o->format != 0) return VGO_E_NOT_PCM;                                                              /* :100-103 */
    o->loop_start = vgo_gc_nibble_to_sample(o->start_address);                                             /* DspStructure.cs:69-73 */
    o->loop_end = vgo_gc_nibble_to_sample(o->end_address);
    return 0;
}

/* DspReader.ReadData (:106-119): outputs[c] holds SampleCountToByteCount(sample_count) bytes */
int vgo_dsp_read_data(const uint8_t *f, int64_t len, const vgo_dsp_info *o, uint8_t *const *outputs)
{
    const int bytes = vgo_gc_sample_count_to_byte_count(o->sample_count);
    const uint8_t *data = f + 0x60 * o->channel_count;
    if (o->channel_count == 1) {
        const int64_t avail = len - 0x60;
        memset(outputs[0], 0, (size_t)bytes);
        memcpy(outputs[0], data, (size_t)(avail < bytes ? avail : bytes));
        return 0;
    }
    const int data_len = next_multiple(bytes, 8) * o->channel_count;
    if (len - 0x60ll * o->channel_count < data_len) return VGO_E_TRUNCATED;  /* Interleave.cs:122-129 */
    if (o->frames_per_interleave <= 0) return VGO_E_ARG;
    return vgo_deinterleave(data, data_len, o->frames_per_interleave * 8, o->channel_count, bytes, outputs);
}

/* ============================================================================================================
 * CRI ADX: key schedule (Codecs/CriAdx/CriAdxKey.cs), EncryptDecrypt (CriAdxEncryption.cs:8-44), AdxWriter
 * (Containers/Adx/AdxWriter.cs:12-146)
 * ============================================================================================================ */
static int g_primes[0x400];
static int g_primes_ready;
static void adx_primes(void) /* CriAdxKey.BuildPrimesTable :68-75 over Helpers.GetPrimes(0x8000) (Helpers.cs:115-139) */
{
    if (g_primes_ready) return;
    static uint8_t sieve[0x4000];
    memset(sieve, 0, sizeof sieve);
    for (int i = 3; i * i < 0x8000; i += 2) {
        if (sieve[i >> 1]) continue;
        for (int j = i * i; j < 0x8000; j += i * 2) sieve[j >> 1] = 1;
    }
    int n = 0;
    for (int i = 1; i < 0x4000 && n < 0x400; i++) {           /* primes >= 0x4000 (BinarySearch insertion point) */
        const int p = i * 2 + 1;
        if (!sieve[i] && p >= 0x4000) g_primes[n++] = p;
    }
    g_primes_ready = 1;
}
void vgo_adx_key_from_code(uint64_t key_code, int32_t key[3]) /* :18-24 */
{
    key_code--;
    key[0] = (int)((key_code >> 27) & 0x7fff);
    key[1] = (int)(((key_code >> 12) & 0x7ffc) | 1);
    key[2] = (int)(((key_code << 1) & 0x7fff) | 1);
}
void vgo_adx_key_from_string(const char *s, int32_t key[3]) /* :26-41 (chars as UTF-16 code units; ASCII here) */
{
    adx_primes();
    int seed = g_primes[0x100], mult = g_primes[0x200], inc = g_primes[0x300];
    for (; *s; s++) {
        const int c = (unsigned char)*s;
        seed = g_primes[seed * g_primes[c + 0x80] % 0x400];
        mult = g_primes[mult * g_primes[c + 0x80] % 0x400];
        inc = g_primes[inc * g_primes[c + 0x80] % 0x400];
    }
    key[0] = seed; key[1] = mult; key[2] = inc;
}
/* EncryptDecryptChannel :16-44 */
void vgo_adx_crypt_channel(uint8_t *adpcm, int length, const int32_t key[3], int encryption_type, int frame_size, int channel_num, int channel_count)
{
    int x = key[0];
    const int frames = (length + frame_size - 1) / frame_size;
    for (int i = 0; i < channel_num; i++) x = (x * key[1] + key[2]) & 0x7fff;
    for (int i = 0; i < frames; i++) {
        const int pos = i * frame_size;
        int not_empty = 0;
        for (int k = pos; k < pos + frame_size; k++) if (adpcm[k]) { not_empty = 1; break; }
        if (not_empty) {
            adpcm[pos] ^= (uint8_t)(x >> 8);
            if (encryption_type == 9) adpcm[pos] &= 0x1f;
            adpcm[pos + 1] ^= (uint8_t)x;
        }
        for (int c = 0; c < channel_count; c++) x = (x * key[1] + key[2]) & 0x7fff;
    }
}

static int adx_bytes(int samples, int frame_size) /* CriAdxHelpers.SampleCountToByteCount */
{
    const int npf = frame_size * 2, spf = npf - 4;
    const int extra = samples % spf;
    const int nib = npf * (samples / spf) + (extra == 0 ? 0 : extra + 4);
    return (nib + 1) / 2;
}
typedef struct { int sample_count, frame_count, base_header, alignment_bytes, header_size, audio_offset, audio_size, footer_offset, footer_size; } adx_geom;
static void adx_geometry(const vgo_adx_desc *d, adx_geom *g)
{
    const int spf = (d->frame_size - 2) * 2;
    const int sample_count = d->sample_count + d->alignment_samples;      /* CriAdxFormat.SampleCount :16 */
    const int loop_start = d->loop_start + d->alignment_samples, loop_end = d->loop_end + d->alignment_samples;
    g->sample_count = d->trim_file && d->looping ? loop_end + spf * 3 : sample_count;   /* :21 */
    g->frame_count = (g->sample_count + spf - 1) / spf;
    g->base_header = d->looping ? (d->version == 4 ? 60 : 52) : (d->version == 4 ? 36 : 32);
    g->alignment_bytes = 0;
    if (d->looping) {                                                       /* CalculateAlignmentBytes :57-68 */
        const int off = adx_bytes(loop_start, d->frame_size) * d->channel_count + g->base_header + 4;
        g->alignment_bytes = next_multiple(off, 0x800) - off;
        if (d->version == 3) g->alignment_bytes += d->alignment_samples / spf * 0x800;
    }
    g->header_size = g->base_header + g->alignment_bytes;
    g->audio_offset = g->header_size + 4;
    g->audio_size = d->frame_size * g->frame_count * d->channel_count;
    g->footer_offset = g->audio_offset + g->audio_size;
    g->footer_size = d->looping ? next_multiple(g->footer_offset + d->frame_size, 0x800) - g->footer_offset : d->frame_size;
}
int64_t vgo_adx_file_size(const vgo_adx_desc *d) { adx_geom g; adx_geometry(d, &g); return (int64_t)g.audio_offset + g.audio_size + g.footer_size; }

/* audio[c]: channel c's encoded frames, audio_len bytes each (CriAdxChannel.Audio); history[c]: CriAdxChannel.History;
 * key: NULL = no encryption.  d->sample_count / loop points are the UNALIGNED values of the PCM the format was made from. */
int vgo_adx_write(const vgo_adx_desc *d, const uint8_t *const *audio, int audio_len, const int16_t *history, const int32_t *key, uint8_t *out)
{
    adx_geom g;
    adx_geometry(d, &g);
    const int ch = d->channel_count;
    if (ch < 1 || ch > 255 || d->frame_size < 3) return VGO_E_ARG;
    memset(out, 0, (size_t)vgo_adx_file_size(d));
    const int loop_start = d->loop_start + d->alignment_samples, loop_end = d->loop_end + d->alignment_samples;
    uint8_t *p = out;                                                       /* WriteHeader :80-119 */
    be16(p, 0x8000); be16(p + 2, g.header_size); p[4] = (uint8_t)d->type; p[5] = (uint8_t)d->frame_size; p[6] = 4; p[7] = (uint8_t)ch;
    be32(p + 8, d->sample_rate); be32(p + 12, g.sample_count);
    be16(p + 16, d->type != 2 ? d->highpass_frequency : 0);
    p[18] = (uint8_t)d->version; p[19] = (uint8_t)d->encryption_type;
    p += 20;
    if (d->version == 4) {
        be32(p, 0); p += 4;
        for (int i = 0; i < ch; i++) { be16(p, history[i]); be16(p + 2, history[i]); p += 4; }
        if (ch == 1) { be32(p, 0); p += 4; }
    }
    be16(p, d->alignment_samples); be16(p + 2, d->looping ? 1 : 0); be32(p + 4, d->looping ? 1 : 0);
    be32(p + 8, loop_start);
    be32(p + 12, g.audio_offset + adx_bytes(loop_start, d->frame_size) * ch);                             /* LoopStartOffset :35 */
    be32(p + 16, loop_end);
    be32(p + 20, g.audio_offset + next_multiple(adx_bytes(loop_end, d->frame_size), d->frame_size) * ch); /* LoopEndOffset :36 */
    memcpy(out + g.header_size - 2, "(c)CRI", 6);
    /* WriteData :121-133: an encrypted COPY of the audio, frame-interleaved */
    const int out_size = g.frame_count * d->frame_size;
    uint8_t **tmp = (uint8_t **)malloc(sizeof(uint8_t *) * (size_t)ch);
    for (int c = 0; c < ch; c++) {
        tmp[c] = (uint8_t *)malloc((size_t)audio_len + 1);
        memcpy(tmp[c], audio[c], (size_t)audio_len);
        if (key) vgo_adx_crypt_channel(tmp[c], audio_len, key, d->encryption_type, d->frame_size, c, ch);
    }
    vgo_interleave((const uint8_t *const *)tmp, ch, audio_len, d->frame_size, out_size, out + g.audio_offset);
    for (int c = 0; c < ch; c++) free(tmp[c]);
    free(tmp);
    be16(out + g.footer_offset, 0x8001);                                    /* WriteFooter :135-140 */
    be16(out + g.footer_offset + 2, g.footer_size - 4);
    return 0;
}

/* ============================================================================================================
 * CRI HCA: key tables (Codecs/CriHca/CriHcaKey.cs), CryptFrame (CriHcaEncryption.cs:21-33), HcaWriter
 * (Containers/Hca/HcaWriter.cs:56-185)
 * ============================================================================================================ */
static void hca_random_row(uint8_t seed, uint8_t row[16]) /* CreateRandomRow :117-131 */
{
    int x = seed >> 4;
    const int mult = ((seed & 1) << 3) | 5, inc = (seed & 0xe) | 1;
    for (int i = 0; i < 16; i++) { x = (x * mult + inc) % 16; row[i] = (uint8_t)x; }
}
/* key_type 0, 1 (CriHcaKey(Type) :17-34) or 56 (CriHcaKey(ulong) :9-15); tables are 256 bytes each */
int vgo_hca_key_tables(int key_type, uint64_t key_code, uint8_t *decrypt, uint8_t *encrypt)
{
    memset(decrypt, 0, 256);
    if (key_type == 0) {
        for (int i = 0; i < 256; i++) decrypt[i] = (uint8_t)i;
    } else if (key_type == 1) {                                 /* CreateDecryptionTableType1 :80-98 */
        int x = 0, pos = 1;
        for (int i = 0; i < 256; i++) {
            x = (x * 13 + 11) % 256;
            if (x != 0 && x != 0xff) decrypt[pos++] = (uint8_t)x;
        }
        decrypt[0xff] = 0xff;
    } else if (key_type == 56) {                                /* CreateDecryptionTable :43-66 + CreateTable :100-115 + ShuffleTable :145-161 */
        const uint64_t k = key_code - 1;
        uint8_t kc[8], seed[16], t[256], row[16], col[16];
        for (int i = 0; i < 8; i++) kc[i] = (uint8_t)(k >> (8 * i));
        seed[0] = kc[1]; seed[1] = kc[6] ^ kc[1]; seed[2] = kc[2] ^ kc[3]; seed[3] = kc[2]; seed[4] = kc[1] ^ kc[2]; seed[5] = kc[3] ^ kc[4];
        seed[6] = kc[3]; seed[7] = kc[2] ^ kc[3]; seed[8] = kc[4] ^ kc[5]; seed[9] = kc[4]; seed[10] = kc[3] ^ kc[4]; seed[11] = kc[5] ^ kc[6];
        seed[12] = kc[5]; seed[13] = kc[4] ^ kc[5]; seed[14] = kc[6] ^ kc[1]; seed[15] = kc[6];
        hca_random_row(kc[0], row);
        for (int r = 0; r < 16; r++) {
            hca_random_row(seed[r], col);
            for (int c = 0; c < 16; c++) t[16 * r + c] = (uint8_t)((row[r] << 4) | col[c]);   /* CombineNibbles(high, low) */
        }
        uint8_t x = 0;
        int pos = 1;
        for (int i = 0; i < 256; i++) {
            x = (uint8_t)(x + 17);
            if (t[x] != 0 && t[x] != 0xff) decrypt[pos++] = t[x];
        }
        decrypt[0xff] = 0xff;
    } else {
        return VGO_E_ARG;
    }
    for (int i = 0; i < 256; i++) encrypt[decrypt[i]] = (uint8_t)i;   /* InvertTable :163-174 */
    return 0;
}
void vgo_hca_crypt_frame(uint8_t *frame, int frame_size, const uint8_t *table) /* CryptFrame :21-33 */
{
    for (int b = 0; b < frame_size - 2; b++) frame[b] = table[frame[b]];
    const uint16_t crc = vgo_crc16(frame, frame_size - 2);
    frame[frame_size - 2] = (uint8_t)(crc >> 8);
    frame[frame_size - 1] = (uint8_t)crc;
}

/* frames: frame_count x frame_size bytes (CriHcaFormat.AudioData); encrypt_table: NULL = none (then key_type is ignored);
 * comment: NULL or "" = none; volume as float32 bits (1.0f = no rva chunk).  out: header_size + frame_count*frame_size */
int vgo_hca_write(const vgo_hca_info *h, const uint8_t *frames, const uint8_t *encrypt_table, int key_type,
                  const char *comment, uint32_t volume_bits, uint8_t *out)
{
    const int masked = encrypt_table != NULL;
    const int64_t total = (int64_t)h->header_size + (int64_t)h->frame_size * h->frame_count;
    memset(out, 0, (size_t)total);
    uint8_t *p = out;
#define HCA_ID(s, n) do { for (int _i = 0; _i < (n); _i++) { uint8_t _b = (uint8_t)(s)[_i]; if (masked && _b) _b |= 0x80; p[_i] = _b; } p += (n); } while (0)
    HCA_ID("HCA\0", 4); be16(p, 0x0200); be16(p + 2, h->header_size); p += 4;                       /* :80-85 */
    HCA_ID("fmt\0", 4); p[0] = (uint8_t)h->channel_count; p[1] = (uint8_t)(h->sample_rate >> 16); be16(p + 2, h->sample_rate);
    be32(p + 4, h->frame_count); be16(p + 8, h->inserted_samples); be16(p + 10, h->appended_samples); p += 12;   /* :87-99 */
    HCA_ID("comp", 4); be16(p, h->frame_size); p[2] = (uint8_t)h->min_resolution; p[3] = (uint8_t)h->max_resolution;
    p[4] = (uint8_t)h->track_count; p[5] = (uint8_t)h->channel_config; p[6] = (uint8_t)h->total_band_count; p[7] = (uint8_t)h->base_band_count;
    p[8] = (uint8_t)h->stereo_band_count; p[9] = (uint8_t)h->bands_per_hfr_group; be16(p + 10, 0); p += 12;      /* :101-114 */
    if (h->looping) {                                                                                /* :116-125 */
        HCA_ID("loop", 4); be32(p, h->loop_start_frame); be32(p + 4, h->loop_end_frame); be16(p + 8, h->pre_loop_samples); be16(p + 10, h->post_loop_samples); p += 12;
    }
    HCA_ID("ciph", 4); be16(p, masked ? key_type : 0); p += 2;                                       /* :127-131, :41 */
    if (volume_bits != 0x3F800000u) { HCA_ID("rva\0", 4); be32(p, (int32_t)volume_bits); p += 4; }   /* :133-142 */
    int blank = 1;                                                                                   /* string.IsNullOrWhiteSpace */
    if (comment) for (const char *c = comment; *c; c++) if (*c != ' ' && *c != '\t' && *c != '\n' && *c != '\r' && *c != '\v' && *c != '\f') blank = 0;
    if (blank) { HCA_ID("pad", 3); }                                                                 /* :150-153 ("pad" is 3 bytes) */
    else { HCA_ID("comm\0", 5); const size_t n = strlen(comment); memcpy(p, comment, n); p += n + 1; } /* :144-148 WriteUTF8Z */
#undef HCA_ID
    if (p - out > h->header_size - 2) return VGO_E_ARG;
    const uint16_t crc = vgo_crc16(out, h->header_size - 2);                                         /* :72-76 */
    be16(out + h->header_size - 2, crc);
    uint8_t *d = out + h->header_size;                                                               /* WriteData :172-178 (+ Crypt :38-44) */
    memcpy(d, frames, (size_t)h->frame_size * (size_t)h->frame_count);
    if (encrypt_table) for (int f = 0; f < h->frame_count; f++) vgo_hca_crypt_frame(d + (size_t)f * h->frame_size, h->frame_size, encrypt_table);
    return 0;
}
