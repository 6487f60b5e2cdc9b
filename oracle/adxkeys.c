/* adxkeys.c — the key search of VGAudio.Tools/CrackAdx/GuessAdx.cs, restated in plain C.  TEST INFRASTRUCTURE: the
 * GPU search (vgaudio_b200/csrc/adx_keys.cu) is compared against it on boxes small enough for one CPU thread.
 * Everything runs in the reference's order: Run's index loop outside, the files inside, TryScale's mult and inc loops. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "vgoracle.h"

/* The entry points (bound by tests/adx_key_oracle.py; vgoracle.h is not extended for them):
 *   vgo_adx_key_load      LoadFiles (:79-97) + AdxFile (:276-300) on one image.  *type is the search's revision so far
 *                         (0 before the first file); returns 0 when the file is loaded (at most cap scales written),
 *                         1 when it is of another revision, negative where ReadMetadata or the audio read throws.
 *   vgo_adx_key_list      the revision's lists (:48-71): which 0 seeds, 1 multipliers, 2 increments; returns the count.
 *   vgo_adx_key_is_valid  KeyIsValid (:217-229).
 *   vgo_adx_guess_box     Run (:113-124) over scale indices [i0, i1), multipliers [m0, m1) and increments [c0, c1) of the
 *                         lists: TryScale for every index and file, FindStartingKey, AddKey's dedup and KeyIsValid on
 *                         every file; files without a frame add no candidates and validate every key.  Returns the
 *                         number of keys (ascending, at most cap written); stats = candidates tried, frame steps, full
 *                         matches.
 *   vgo_adx_key_confidence  GetReencodeConfidence (:231-263) for one image the reader chain accepts: out = differing
 *                         bytes short, compared bytes short, differing bytes full, compared bytes full (C# int sums);
 *                         returns 0, or -1 where the chain throws. */
int vgo_adx_key_load(const uint8_t *f, int64_t len, int *type, int *frame_size, int *start_frame, uint16_t *scales, int cap, int *n_frames);
int vgo_adx_key_list(int revision, int which, int32_t *out);
int vgo_adx_key_is_valid(int revision, const int32_t key[3], const uint16_t *scales, int n_frames);
int vgo_adx_guess_box(int revision, int n_files, const uint16_t *const *scales, const int *n_frames, const int *start_frame, int i0, int i1,
                      int m0, int m1, int c0, int c1, int32_t *keys_out, int cap, uint64_t stats[3]);
int vgo_adx_key_confidence(const uint8_t *f, int64_t len, const int32_t key[3], int32_t out[4]);

/* Common.GetPrimes(0x8000) (VGAudio.Tools/Common.cs) from its first prime above 0x4000, 0x400 of them (GuessAdx.cs:51-57) */
static const int *key_primes(void)
{
    static int primes[0x400];
    static int ready;
    if (!ready) {
        static uint8_t composite[0x8000];
        for (int i = 2; i * i < 0x8000; i++)
            if (!composite[i])
                for (int j = i * i; j < 0x8000; j += i) composite[j] = 1;
        int n = 0;
        for (int p = 0x4000; p < 0x8000 && n < 0x400; p++)
            if (!composite[p]) primes[n++] = p;
        ready = 1;
    }
    return primes;
}

typedef struct {
    int ok;
    int header_size, type, frame_size, channel_count, sample_rate, sample_count, highpass, version, revision;
    int inserted, looping, loop_start, loop_end;
} key_hdr;

/* AdxReader.ReadHeader (Containers/Adx/AdxReader.cs:70-109), big-endian; ok = 0 on a read past the image or a bad signature */
static key_hdr read_header(const uint8_t *f, int64_t len)
{
    key_hdr h;
    memset(&h, 0, sizeof h);
    int64_t pos = 0;
    int past = 0;
#define U8() (pos < len ? f[pos++] : (past = 1, pos++, 0))
    int sig = U8() << 8; sig |= U8();
    if (past || sig != 0x8000) return h;
    int v = U8() << 8; v |= U8(); h.header_size = (int16_t)v;
    h.type = U8(); h.frame_size = U8(); (void)U8(); h.channel_count = U8();
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) r = r << 8 | (uint32_t)U8();
    h.sample_rate = (int32_t)r;
    r = 0;
    for (int i = 0; i < 4; i++) r = r << 8 | (uint32_t)U8();
    h.sample_count = (int32_t)r;
    v = U8() << 8; v |= U8(); h.highpass = (int16_t)v;
    h.version = U8(); h.revision = U8();
    if (h.version >= 4) {
        pos += 4;
        for (int c = 0; c < h.channel_count * 4; c++) (void)U8();
        if (h.channel_count == 1) pos += 4;
    }
    if (past) return h;
    if (pos + 24 <= h.header_size) {
        v = U8() << 8; v |= U8(); h.inserted = (int16_t)v;
        v = U8() << 8; v |= U8();
        if ((int16_t)v > 0) {
            int32_t w[5];
            for (int k = 0; k < 5; k++) { r = 0; for (int i = 0; i < 4; i++) r = r << 8 | (uint32_t)U8(); w[k] = (int32_t)r; }
            h.looping = 1; h.loop_start = w[1]; h.loop_end = w[3];
        }
        if (past) return h;
    }
#undef U8
    h.ok = 1;
    return h;
}

/* AdxStructure.AudioDataLength (AdxStructure.cs:30): DivideByRoundUp through a double, C# int products */
static int64_t audio_data_length(const key_hdr *h)
{
    const int spf = (h->frame_size - 2) * 2;
    const double q = (double)h->sample_count / spf;
    const int32_t frames = (isnan(q) || q >= 2147483648.0 || q < -2147483648.0) ? INT32_MIN : (int32_t)ceil(q);
    return (int32_t)((uint32_t)h->frame_size * (uint32_t)frames * (uint32_t)h->channel_count);
}

int vgo_adx_key_load(const uint8_t *f, int64_t len, int *type, int *frame_size, int *start_frame, uint16_t *scales, int cap, int *n_frames)
{
    const key_hdr h = read_header(f, len);
    if (!h.ok) return -1;
    if (*type == 0) *type = h.revision;
    if (h.revision != *type) return 1;
    if (h.frame_size == 0) return -2;
    const int64_t n = audio_data_length(&h);
    const int64_t off = (int64_t)h.header_size + 4;
    if (n < 0) return -3;
    if (off < 0) return -4;
    const int fs = h.frame_size;
    *frame_size = fs;
    *n_frames = (int)(n / fs);
    for (int64_t i = 0; i < n / fs && i < cap; i++) {
        const int64_t p = off + i * fs;
        scales[i] = (uint16_t)((p < len ? f[p] : 0) << 8 | (p + 1 < len ? f[p + 1] : 0));
    }
    *start_frame = 0;
    for (int64_t i = 0; i < n && off + i < len; i++)
        if (f[off + i]) { *start_frame = (int)(i / fs); break; }
    return 0;
}

int vgo_adx_key_list(int revision, int which, int32_t *out)
{
    int n = 0;
    if (revision == 8) {
        const int *primes = key_primes();
        for (int i = 0; i < 0x400; i++) if (out) out[n++] = primes[i]; else n++;
        return n;
    }
    for (int x = 0; x < 0x2000; x++) {
        const int take = which == 0 ? 1 : which == 1 ? (x & 3) == 1 : (x & 1) == 1;
        if (take) { if (out) out[n] = x; n++; }
    }
    return n;
}

static int mask_of(int revision) { return revision == 8 ? 0xE000 : 0x1000; }
static int max_seed_of(int revision) { return revision == 8 ? 0x8000 : 0x2000; }

int vgo_adx_key_is_valid(int revision, const int32_t key[3], const uint16_t *scales, int n_frames)
{
    const int mask = mask_of(revision);
    int x = key[0];
    for (int i = 0; i < n_frames; i++) {
        const int s = scales[i];
        if (((s ^ x) & mask) != 0 && s != 0) return 0;
        x = (x * key[1] + key[2]) & 0x7fff;
    }
    return 1;
}

static int cmp_key(const void *a, const void *b)
{
    const int32_t *x = a, *y = b;
    for (int i = 0; i < 3; i++) if (x[i] != y[i]) return x[i] < y[i] ? -1 : 1;
    return 0;
}

int vgo_adx_guess_box(int revision, int n_files, const uint16_t *const *scales, const int *n_frames, const int *start_frame, int i0, int i1,
                      int m0, int m1, int c0, int c1, int32_t *keys_out, int cap, uint64_t stats[3])
{
    int32_t *seeds = malloc(0x2000 * sizeof *seeds), *mults = malloc(0x2000 * sizeof *mults), *incs = malloc(0x2000 * sizeof *incs);
    const int n_seeds = vgo_adx_key_list(revision, 0, seeds);
    vgo_adx_key_list(revision, 1, mults);
    vgo_adx_key_list(revision, 2, incs);
    uint8_t *listed = calloc(0x8000, 1);
    for (int i = 0; i < n_seeds; i++) listed[seeds[i]] = 1;
    const int mask = mask_of(revision), smask = max_seed_of(revision) - 1;
    int n_found = 0, found_cap = 64;
    int32_t *found = malloc((size_t)found_cap * 3 * sizeof *found);
    stats[0] = stats[1] = stats[2] = 0;
    for (int index = i0; index < i1; index++) {
        for (int f = 0; f < n_files; f++) {
            if (n_frames[f] == 0) continue; /* on purpose: the reference throws at Scales[StartFrame] */
            const uint16_t *sc = scales[f];
            const int start = start_frame[f];
            const int seed = (sc[start] ^ index) & smask;
            if (start == 0 && !listed[seed]) continue;
            for (int m = m0; m < m1; m++) {
                for (int c = c0; c < c1; c++) {
                    const int mult = mults[m], inc = incs[c];
                    int x = seed, match = 1;
                    stats[0]++;
                    for (int i = start; i < n_frames[f]; i++) {
                        const int s = sc[i];
                        stats[1]++;
                        if (((s ^ x) & mask) != 0 && s != 0) { match = 0; break; }
                        x = (x * mult + inc) & 0x7fff;
                    }
                    if (!match) continue;
                    stats[2]++;
                    /* FindStartingKey: the first listed seed, in ascending order, that reaches `seed` after `start` steps */
                    int real = -1;
                    if (start == 0) real = seed;
                    else
                        for (int k = 0; k < n_seeds && real < 0; k++) {
                            int y = seeds[k];
                            for (int i = 0; i < start; i++) y = (y * mult + inc) & 0x7fff;
                            if ((y & smask) == seed) real = seeds[k];
                        }
                    if (real < 0) continue;
                    const int32_t key[3] = {real, mult, inc};
                    int valid = 1;
                    for (int g = 0; g < n_files && valid; g++) valid = vgo_adx_key_is_valid(revision, key, scales[g], n_frames[g]);
                    if (!valid) continue;
                    if (n_found == found_cap) { found_cap *= 2; found = realloc(found, (size_t)found_cap * 3 * sizeof *found); }
                    memcpy(found + 3 * n_found++, key, sizeof key);
                }
            }
        }
    }
    /* AddKey's TriedKeys: each distinct key once */
    qsort(found, (size_t)n_found, 3 * sizeof *found, cmp_key);
    int n = 0;
    for (int i = 0; i < n_found; i++)
        if (n == 0 || cmp_key(found + 3 * i, found + 3 * (n - 1)) != 0) memmove(found + 3 * n++, found + 3 * i, 3 * sizeof *found);
    for (int i = 0; i < n && i < cap; i++) memcpy(keys_out + 3 * i, found + 3 * i, 3 * sizeof *found);
    free(found); free(listed); free(seeds); free(mults); free(incs);
    return n;
}

int vgo_adx_key_confidence(const uint8_t *f, int64_t len, const int32_t key[3], int32_t out[4])
{
    const key_hdr h = read_header(f, len);
    if (!h.ok || h.frame_size < 3 || h.channel_count == 0) return -1;
    const int fs = h.frame_size, ch = h.channel_count, spf = (fs - 2) * 2;
    const int64_t n = audio_data_length(&h), off = (int64_t)h.header_size + 4;
    if (n < 0 || off < 0 || off + n > len) return -1;
    const int row_len = (int)(n / ch), frames = row_len / fs;
    const int samples = h.sample_count - h.inserted;
    const int ls = h.looping ? h.loop_start - h.inserted : 0, le = h.looping ? h.loop_end - h.inserted : 0;
    if (h.looping && (ls < 0 || ls > samples || le < 0 || le > samples || le < ls)) return -1;
    if (samples < 0) return -1;
    const int pad = h.inserted > 0 ? h.inserted : 0;
    if (samples > 0 && ((int64_t)(pad / spf) + (samples + spf - 1) / spf) * fs > row_len) return -1;
    /* the re-encode: default CriAdxParameters, alignment to the loop start (CriAdxFormat.cs:57-64) */
    const int mult = ch == 1 ? 64 : 32, align = (ls + mult - 1) / mult * mult - ls;
    if (samples == 0 && align == 0) return -1; /* CriAdxCodec.Encode reads pcm[0] */
    const int enc_len = vgo_adx_encoded_byte_count(samples, align, 18);
    uint8_t *row = malloc((size_t)row_len + 1), *enc = malloc((size_t)enc_len + 1);
    int16_t *pcm = malloc(((size_t)samples + 1) * sizeof *pcm);
    for (int t = 0; t < 4; t++) out[t] = 0;
    const int n_short = fs * 100 < row_len ? fs * 100 : row_len;
    for (int c = 0; c < ch; c++) {
        for (int j = 0; j < frames; j++) memcpy(row + (size_t)j * fs, f + off + ((int64_t)j * ch + c) * fs, (size_t)fs);
        vgo_adx_crypt_channel(row, row_len, key, h.revision, fs, c, ch);
        vgo_adx_decode(row, samples, h.sample_rate, h.highpass, fs, h.version, 0, h.inserted, h.type, pcm);
        vgo_adx_encode(pcm, samples, h.sample_rate, 18, 4, align, 3, 0, enc);
        int d_short = -2, d_full = -2;
        if (enc_len == row_len) {
            d_short = d_full = 0;
            for (int i = 0; i < row_len; i++) {
                const int d = row[i] != enc[i];
                d_full += d;
                if (i < n_short) d_short += d;
            }
        }
        out[0] = (int32_t)((uint32_t)out[0] + (uint32_t)d_short);
        out[1] = (int32_t)((uint32_t)out[1] + (uint32_t)n_short);
        out[2] = (int32_t)((uint32_t)out[2] + (uint32_t)d_full);
        out[3] = (int32_t)((uint32_t)out[3] + (uint32_t)row_len);
    }
    free(row); free(enc); free(pcm);
    return 0;
}
