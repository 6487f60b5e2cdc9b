/*
 * vgoracle.h — CPU ORACLE for the VGAudio hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This is a plain-C restatement of the reference's (Thealexbarney/VGAudio, C#)
 * per-channel codec arithmetic.  It exists so the CUDA kernels can be checked
 * bit-for-bit; it is NOT part of the product.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.
 *
 * Parity status (see DESIGN.md §Oracle):
 *   - GcAdpcmMath helpers ........ pinned by the reference's own KAT tables
 *                                  (src/VGAudio.Tests/Formats/GcAdpcm/GcAdpcmHelpersTests.cs:8-100)
 *   - GC-ADPCM encode/decode ..... pinned by the reference's round-trip properties
 *                                  (GcAdpcmFormatTests.cs:87-157 ramps exact; GcAdpcmAlignmentTests.cs:64-108
 *                                  sine <= 2 LSB and encoder-reconstruction == decoder).
 *                                  The reference holds NO golden bitstream and cannot be run here
 *                                  (no .NET toolchain) => encoded BYTES are "parity unpinned".
 *   - CRI ADX ...................... reference has zero tests => "parity unpinned".
 *   - CRI HCA tables ............... pinned bit-exact by CriHcaTableTests.cs literals; encoder output unpinned.
 *
 *   - Interleave / DeInterleave ... pinned by the reference's golden vectors (Tests/Utilities/InterleaveTests.cs,
 *                                  DeinterleaveTests.cs), replayed literally in tests/test_interleave_reference_vectors.py
 *   - seek table / loop context .... pinned by the KATs of GcAdpcmLoopContextTests.cs / GcAdpcmSeekTableTests.cs
 *   - containers (containers.c) .... build -> parse round trips only (WaveTests.cs, DspTests.cs): file bytes unpinned
 *
 * All file:line citations are relative to VGAudio's src/VGAudio/.
 * Build: see oracle/Makefile (gcc -O2 -ffp-contract=off -fno-fast-math).
 */
#ifndef VGORACLE_H
#define VGORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- GcAdpcmMath (Codecs/GcAdpcm/GcAdpcmMath.cs:7-47) ---- */
int vgo_gc_nibble_count_to_sample_count(int nibble_count);
int vgo_gc_sample_count_to_nibble_count(int sample_count);
int vgo_gc_nibble_to_sample(int nibble);
int vgo_gc_sample_to_nibble(int sample);
int vgo_gc_sample_count_to_byte_count(int sample_count);
int vgo_gc_byte_count_to_sample_count(int byte_count);
/* Utilities/Extensions.cs:145 */
int vgo_divide_by_round_up(int value, int divisor);

/* ---- GcAdpcmCoefficients.CalculateCoefficients (Codecs/GcAdpcm/GcAdpcmCoefficients.cs:9-110) ---- */
void vgo_gc_calculate_coefficients(const int16_t *source, int length, int16_t coefs_out[16]);

/* Phase-1 only (GcAdpcmCoefficients.cs:40-61): one (accepted, r1, r2) triple per 14-sample frame,
 * NOT compacted, plus the direct-form vector MatrixFilter (:285-305) derives from it.
 * rec_out: [frames][2] = record[z,1], record[z,2];  dir_out: [frames][2] = MatrixFilter dst[1], dst[2].
 * Returns the number of accepted records.  Used to test the GPU phase-1 kernel in isolation. */
int vgo_gc_coef_records(const int16_t *source, int length, double *rec_out, double *dir_out, uint8_t *accepted_out);

/* CalculateCoefficients with a record of every refinement pass and of every frame's phase-1 outcome, so that tests can
 * compare a kernel pass by pass and show which rare paths an input reaches.  Same coefficients as
 * vgo_gc_calculate_coefficients.  Passes are numbered as gc_coef_refine_kernel numbers them: 0 is the ordered mean
 * (:63-76), 1..6 are split + two FilterRecords rounds with 2, 4 and 8 centroids (:79-91, :344-396). */
enum { VGO_GC_COEF_PASSES = 7 };
/* phase-1 outcome of a frame (:40-61, :133-255) */
enum { VGO_GC_ACCEPTED = 0, VGO_GC_REJ_QUIET = 1 /* |v0| <= 10 */, VGO_GC_REJ_BIG = 2 /* a row max < double.Epsilon */,
       VGO_GC_REJ_RANGE = 3 /* lo / hi < 1e-10 */, VGO_GC_REJ_DEN = 4 /* 1 - k2^2 == 0 */, VGO_GC_REJ_K1 = 5 /* |k1| > 1 */ };
typedef struct vgo_gc_coef_pass {
    double cent[8][2];       /* best[z][1], best[z][2] after the pass, raw doubles (centroids the pass does not use: 0) */
    int32_t hits[8];         /* records per bucket (pass 0: all records in bucket 0; unused buckets 0) */
    int32_t count;           /* centroids of the pass: 1, 2, 2, 4, 4, 8, 8 */
    int32_t empty;           /* buckets below count without a record */
    int32_t ties_same;       /* records whose minimum distance (< 1e30) is shared by centroids that are all bit-identical */
    int32_t ties_distinct;   /* ... shared by centroids of which two differ in some bit */
    int32_t tie_record;      /* the first tied record (record order), -1: none */
    int32_t tie_lo, tie_hi;  /* its lowest and highest centroid index at the minimum: the record went to tie_lo */
    int32_t pad;
} vgo_gc_coef_pass;
typedef struct vgo_gc_refine_trace {
    vgo_gc_coef_pass pass[VGO_GC_COEF_PASSES];
    int32_t n_frames, n_records;
} vgo_gc_refine_trace;
/* outcome_out [frames]: VGO_GC_ACCEPTED or the VGO_GC_REJ_* reason; either pointer may be NULL */
void vgo_gc_coef_trace(const int16_t *source, int length, vgo_gc_refine_trace *trace_out, uint8_t *outcome_out,
                       int16_t coefs_out[16]);
int vgo_gc_refine_trace_size(void); /* sizeof(vgo_gc_refine_trace), checked by the Python wrapper */

/* ---- GcAdpcmEncoder (Codecs/GcAdpcm/GcAdpcmEncoder.cs) ---- */
/* Encode :14-46.  sample_count == -1 means pcm_length.  adpcm_out holds SampleCountToByteCount(sample_count) bytes. */
void vgo_gc_encode(const int16_t *pcm, int pcm_length, const int16_t coefs[16],
                   int sample_count, int16_t history1, int16_t history2, uint8_t *adpcm_out);
/* DspEncodeFrame :48-94.  pcm_in_out[0..1] = history (older first), [2..15] = samples; rewritten with the
 * reconstructed samples. */
void vgo_gc_dsp_encode_frame(int16_t pcm_in_out[16], int sample_count, uint8_t adpcm_out[8], const int16_t coefs[16]);

/* Encode with a per-frame record of the reference-level facts of DspEncodeCoef's scale chain (:118-170) and of the
 * argmin (:66-76), so that tests can show which rare paths an input reaches.  Same bytes as vgo_gc_encode. */
typedef struct vgo_gc_pred_trace {
    uint64_t error;          /* final TotalDistance as an exact integer */
    uint32_t max_abs_diff;   /* max |want - guess| over all passes (wrapping int32 diff) */
    int32_t over[13];        /* maxOverflow of every pass, in order (a chain has at most 13 passes) */
    int8_t first_sp;         /* scalePower of the first pass */
    int8_t n_passes;         /* number of do/while passes */
    int8_t final_sp;         /* scalePower written to the header */
    uint8_t bumped;          /* some pass at a power < 12 had over + 8 > 256 (:166-168) */
    uint8_t final12;         /* the chain ended on a pass at scalePower 12 with over > 1 */
    uint8_t wrapped;         /* some prediction sum (residual pass or any pass), or a pass's want - guess, wrapped int32 */
    uint8_t pad[2];
} vgo_gc_pred_trace;
typedef struct vgo_gc_frame_trace {
    vgo_gc_pred_trace pred[8];
    int8_t winner;           /* the predictor written to the header */
    uint8_t tie;             /* another predictor has exactly the winner's error */
    uint8_t pad[6];
} vgo_gc_frame_trace;
void vgo_gc_encode_trace(const int16_t *pcm, int pcm_length, const int16_t coefs[16], int sample_count,
                         int16_t history1, int16_t history2, uint8_t *adpcm_out, vgo_gc_frame_trace *trace_out);
int vgo_gc_frame_trace_size(void); /* sizeof(vgo_gc_frame_trace), checked by the Python wrapper */

/* ---- GcAdpcmDecoder.Decode (Codecs/GcAdpcm/GcAdpcmDecoder.cs:10-54) ---- */
void vgo_gc_decode(const uint8_t *adpcm, const int16_t coefs[16], int sample_count,
                   int16_t history1, int16_t history2, int16_t *pcm_out);

/* ---- batch drivers: the reference's Parallel.For over channels (Formats/GcAdpcm/GcAdpcmFormat.cs:58-74,
 * :42-54, :129-135) restated with a pthread pool (dynamic schedule); n_threads <= 0 means all host cores.  Channel c lives at
 * pcm + c*pcm_stride (samples) / adpcm + c*adpcm_stride (bytes).  Returns threads used. ---- */
int vgo_gc_seek_table(const int16_t *pcm, int length, int samples_per_entry, int16_t *out); /* GcAdpcmSeekTable.cs:25-38 */
void vgo_gc_loop_context(const uint8_t *adpcm, const int16_t *pcm, int loop_start, int16_t out[3]); /* GcAdpcmLoopContext.cs:17-26 */
int vgo_gc_encode_batch(const int16_t *pcm, int64_t pcm_stride, int n_channels, int sample_count,
                        int16_t *coefs_out /* [n_channels][16] */, uint8_t *adpcm_out, int64_t adpcm_stride,
                        int n_threads);
int vgo_gc_decode_batch(const uint8_t *adpcm, int64_t adpcm_stride, const int16_t *coefs, int n_channels,
                        int sample_count, int16_t *pcm_out, int64_t pcm_stride, int n_threads);

/* ---- CRI ADX (Codecs/CriAdx/CriAdxCodec.cs) — PARITY UNPINNED: the reference has no ADX test at all ---- */
/* type: 2 Fixed, 3 Linear, 4 Exponential (CriAdxType.cs:3-8) */
void vgo_adx_calculate_coefficients(int highpass_freq, int sample_rate, int16_t coefs_out[2]); /* :173-184 */
int vgo_adx_encoded_byte_count(int pcm_length, int padding, int frame_size);
void vgo_adx_encode_frame(int16_t *pcm, uint8_t *adpcm_out, const int16_t coefs[2], int samples_per_frame, int type,
                          int version); /* :107-147 */
/* Encode :56-105; returns the History value the reference writes back into the config (:73) */
int vgo_adx_encode(const int16_t *pcm, int pcm_length, int sample_rate, int frame_size, int version, int padding,
                   int type, int filter, uint8_t *adpcm_out);
/* Encode with one record per frame of the facts of EncodeFrame's rare paths (:107-171), so that tests can show which of
 * them an input reaches.  Same bytes and return value as vgo_adx_encode; recording only reads values the frame computes
 * anyway.  A frame the padding skips (`continue`, :87) keeps a zero record apart from frame, layout and power = -1. */
enum { VGO_ADX_FRAME_SKIPPED = 1 /* all padding: `continue`, the frame stays zero */,
       VGO_ADX_FRAME_PADDED = 2 /* leading padding samples */, VGO_ADX_FRAME_PARTIAL = 4 /* zero-filled tail */ };
typedef struct vgo_adx_frame_trace {
    int32_t frame, layout;       /* frame index, VGO_ADX_FRAME_* */
    int32_t hist_in[2];          /* (hist1, hist2) the frame starts from: pcmBuffer[1], pcmBuffer[0] */
    int32_t hist_out[2];         /* the reconstructed pair it hands on */
    int32_t max_distance;        /* pass 1 (:112-118) */
    int32_t clip1_hi, clip1_lo;  /* pass-1 distances Clamp16 clipped at +32767 / -32768 */
    int32_t scale_raw;           /* CalculateScale (:149-165): (maxDistance - 1) / 7 + 1 before the 0x1000 clamp */
    int32_t scale_lin;           /* scale - 1 after the clamp: the Linear scaleOut, the Exponential power's argument */
    int32_t scale_out;           /* the value written to the header */
    int32_t power;               /* Exponential: the power of two (0..12); -1 for the other types */
    int32_t md_gain;             /* the maxDistance of gain = 32767 / maxDistance (8 * scale - 1 for Exponential) */
    int32_t nibbles[16];         /* histogram of the written nibbles, by nibble & 15 */
    int32_t ties[8];             /* [k], k = 1..7: samples with |raw| * 32767 == (4681 k - 2340) * md_gain */
    int32_t cast_ovf;            /* raw * gain outside int32: (int) gives INT_MIN */
    int32_t clip2_hi, clip2_lo;  /* Clamp16 of the scaled distance (:126) */
    int32_t recon_hi, recon_lo;  /* Clamp16 of the reconstruction (:133) */
    int32_t v4_differs;          /* samples where version 4's prediction differs from version 3's */
} vgo_adx_frame_trace;
int vgo_adx_encode_trace(const int16_t *pcm, int pcm_length, int sample_rate, int frame_size, int version, int padding,
                         int type, int filter, uint8_t *adpcm_out, vgo_adx_frame_trace *trace_out);
int vgo_adx_frame_trace_size(void); /* sizeof(vgo_adx_frame_trace), checked by the Python wrapper */
/* Decode :9-54 */
void vgo_adx_decode(const uint8_t *adpcm, int sample_count, int sample_rate, int highpass_freq, int frame_size,
                    int version, int history, int padding, int type, int16_t *pcm_out);

/* ---- CRI HCA (Codecs/CriHca, Utilities/Mdct.cs) — tables pinned by the reference's test literals, frame bytes
 * PARITY UNPINNED (the reference never runs its encoder/decoder in a test) ---- */
typedef struct vgo_hca_params { /* CriHcaParameters.cs:3-15 (+ CodecParameters.SampleCount) */
    int32_t quality;       /* CriHcaQuality: 0 NotSet, 1 Highest, 2 High, 3 Middle, 4 Low, 5 Lowest */
    int32_t bitrate;       /* 0 = derive from quality */
    int32_t limit_bitrate;
    int32_t channel_count, sample_rate, sample_count;
    int32_t looping, loop_start, loop_end;
} vgo_hca_params;
typedef struct vgo_hca_info { /* HcaInfo.cs:5-48, the fields the codec uses */
    int32_t channel_count, sample_rate, sample_count, frame_count, inserted_samples, appended_samples;
    int32_t header_size, frame_size, min_resolution, max_resolution, track_count, channel_config;
    int32_t total_band_count, base_band_count, stereo_band_count, hfr_band_count, bands_per_hfr_group, hfr_group_count;
    int32_t bitrate;
    int32_t looping, loop_start_frame, loop_end_frame, pre_loop_samples, post_loop_samples; /* HcaInfo.cs:29-33 */
    int32_t use_ath_curve; /* HcaInfo.cs:38: decode side only (old files); the encoder always writes 0 */
} vgo_hca_info;
int vgo_hca_init(const vgo_hca_params *p, vgo_hca_info *info_out);              /* CriHcaEncoder.Initialize :61-114 */
int vgo_hca_encode(const int16_t *const *pcm, const vgo_hca_params *p, vgo_hca_info *info_out, uint8_t *frames_out);
/* test helper (NOT in the reference): a well-formed stream whose resolutions use the ATH curve, for the decoder's ATH path */
int vgo_hca_encode_ath(const int16_t *const *pcm, const vgo_hca_params *p, vgo_hca_info *info_out, uint8_t *frames_out);
int vgo_hca_spectra(const int16_t *const *pcm, const vgo_hca_params *p, double *spectra_out);
int vgo_hca_decode(const vgo_hca_info *h, const uint8_t *frames, int16_t *const *pcm_out); /* CriHcaDecoder.Decode :11-25 */
int vgo_hca_unpack_ok(const vgo_hca_info *h, const uint8_t *frames);             /* test helper: all frames well-formed */

/* Encode with one record per frame of the facts of EncodeFrame's rare paths, so that tests can show which of them an
 * input reaches.  Same return value and frame bytes as vgo_hca_encode; recording only reads values the stages compute
 * anyway.  Frames after a failing one are not encoded (their records stay zero). */
enum { VGO_HCA_IS_SILENT = 1 /* el == er == 0 */, VGO_HCA_IS_ET_ZERO = 2 /* et == 0 (anti-phase pair) */,
       VGO_HCA_IS_CLAMP_LOW = 4 /* ratio < 0.5 */, VGO_HCA_IS_CLAMP_HIGH = 8 /* ratio > sqrt(2)/2 (or +inf) */ };
enum { VGO_HCA_HFR_AVG_ZERO = 1 /* source average == 0 */, VGO_HCA_HFR_AVG_NAN = 2 /* no source band: 0/0 */ };
typedef struct vgo_hca_frame_trace {
    int32_t noise_level, eval_boundary;
    int32_t drop_rounds;        /* `highest -= 2` rounds of CalculateNoiseLevel (:457-485) */
    int32_t status;             /* EncodeFrame's outcome: 0, -2 "Bitrate is set too low.", -3 other failure */
    int32_t delta_bits[8];      /* per channel, as written */
    int32_t escapes[8];         /* per channel: deltas written as escape + raw value */
    int32_t coded[8];           /* per channel: CodedScaleFactorCount */
    int32_t res_hist[16];       /* coded bands of every channel per resolution */
    int32_t clamped;            /* scaled coefficients clamped to +-0.999999999999 (ScaleSpectra :651-671) */
    int32_t sf_zero, sf_max;    /* coded bands with scale factor 0 / 63, after band dropping */
    int8_t intensity[8][8];     /* [channel][subframe]: index written for a stereo secondary, else -1 */
    uint8_t is_flags[8][8];     /* [secondary channel][subframe]: VGO_HCA_IS_* */
    uint8_t hfr_flags[8][8];    /* [channel][group]: VGO_HCA_HFR_* of CalculateHfrScale's source average */
    int8_t hfr_scale[8][8];     /* [channel][group]: scale written, -1 where none */
} vgo_hca_frame_trace;
int vgo_hca_encode_trace(const int16_t *const *pcm, const vgo_hca_params *p, vgo_hca_info *info_out, uint8_t *frames_out,
                         vgo_hca_frame_trace *trace_out);
int vgo_hca_frame_trace_size(void); /* sizeof(vgo_hca_frame_trace), checked by the Python wrapper */

/* Decode with one record per frame.  A frame that does not unpack the way the reference's happy path does is recorded
 * and not decoded further (its PCM counts stay zero); vgo_hca_decode's PCM is unchanged for every other frame. */
enum { VGO_HCA_UNPACK_OK = 0, VGO_HCA_UNPACK_BAD_SYNC = 1, VGO_HCA_UNPACK_BAD_DELTA = 2, VGO_HCA_UNPACK_INTENSITY_15 = 3 };
typedef struct vgo_hca_dframe_trace {
    int32_t unpack;                 /* VGO_HCA_UNPACK_* */
    int32_t delta_bits[8];          /* per channel, as read (-1 past the channel count or an early stop) */
    int32_t hfr_index_min, hfr_index_max; /* ScaleConversion index of ReconstructHighFrequency; -1 if none */
    int32_t pcm_in_range, pcm_clip_high, pcm_clip_low, pcm_out_of_int32; /* PcmFloatToShort outcomes */
} vgo_hca_dframe_trace;
int vgo_hca_decode_trace(const vgo_hca_info *h, const uint8_t *frames, int16_t *const *pcm_out, vgo_hca_dframe_trace *trace_out);
int vgo_hca_decode_trace_size(void); /* sizeof(vgo_hca_dframe_trace) */
void vgo_hca_mdct_run(const double *blocks, int n, double *spectra_out);         /* Mdct.RunMdct :63-92, state from zero */
void vgo_hca_imdct_run(const double *spectra, int n, double *blocks_out);        /* Mdct.RunImdct :94-119 */
void vgo_hca_mdct_tables(double *sin_out, double *cos_out, int *shuffle_out, int bits); /* :183-208 */
uint16_t vgo_crc16(const uint8_t *data, int size);                               /* Crc16.Compute, poly 0x8005 */

/* ---- Utilities/Interleave.cs:9-41, :81-117 (bytes) ---- */
int vgo_interleave(const uint8_t *const *inputs, int count, int in_size, int interleave_size, int out_size, uint8_t *output);
int vgo_deinterleave(const uint8_t *input, int length, int interleave_size, int count, int out_size, uint8_t *const *outputs);


/* ---- container layer either side of the codec path (containers.c; SURVEY.md 8f rank 2-4).  The reference pins this layer
 * by build -> parse round trips only (Tests/Containers/DspTests.cs, WaveTests.cs): file BYTES are "parity unpinned" ---- */
enum { VGO_E_ARG = -1, VGO_E_TRUNCATED = -2, VGO_E_NOT_RIFF = -3, VGO_E_NOT_WAVE = -4, VGO_E_NO_FMT = -5, VGO_E_NO_DATA = -6,
       VGO_E_NOT_PCM = -7, VGO_E_BITS = -8, VGO_E_CHANNELS = -9, VGO_E_BLOCK_ALIGN = -10, VGO_E_LOOP = -11, VGO_E_NIBBLES = -12 };
typedef struct vgo_wave_info { /* WaveStructure.cs + where the data chunk's payload sits in the file */
    int32_t channel_count, sample_rate, bits_per_sample, sample_count, looping, loop_start, loop_end, reserved;
    int64_t data_offset, data_size;
} vgo_wave_info;
int vgo_wave_parse(const uint8_t *file, int64_t len, vgo_wave_info *out);        /* RiffParser.cs:38-86, WaveReader.cs:13-95 */
void vgo_wave_read16(const uint8_t *file, const vgo_wave_info *w, int16_t *const *channels);      /* Interleave.cs:188-207 */
void vgo_wave_read8_as16(const uint8_t *file, const vgo_wave_info *w, int16_t *const *channels);  /* + Pcm8Codec.cs:23 */
int64_t vgo_wave_file_size(int channels, int samples, int looping);              /* WaveWriter.cs:24-29 */
void vgo_wave_write16(const int16_t *const *pcm, int channels, int samples, int sample_rate, int looping, int loop_start,
                      int loop_end, uint8_t *out);                               /* WaveWriter.cs:52-132 */

typedef struct vgo_dsp_desc { /* what DspWriter reads from GcAdpcmFormat + DspConfiguration */
    int32_t channel_count, sample_rate, sample_count, looping, loop_start, loop_end;
    int32_t samples_per_interleave /* 0x3800 */, loop_point_alignment /* 1 */, trim_file /* 1 */;
} vgo_dsp_desc;
int64_t vgo_dsp_file_size(const vgo_dsp_desc *d);                                /* DspWriter.cs:17 */
int vgo_dsp_write(const vgo_dsp_desc *d, const uint8_t *const *adpcm, const int16_t *coefs, const int16_t *gain,
                  const int16_t *start_hist, const int16_t *loop_ctx, uint8_t *out);   /* DspWriter.cs:42-99 */
#define VGO_DSP_MAX_CHANNELS 64
typedef struct vgo_dsp_info { /* DspStructure.cs */
    int32_t sample_count, nibble_count, sample_rate, looping, format, start_address, end_address, current_address;
    int32_t channel_count, frames_per_interleave, loop_start, loop_end;
    int16_t coefs[VGO_DSP_MAX_CHANNELS][16], gain[VGO_DSP_MAX_CHANNELS], start_ctx[VGO_DSP_MAX_CHANNELS][3], loop_ctx[VGO_DSP_MAX_CHANNELS][3];
} vgo_dsp_info;
int vgo_dsp_parse(const uint8_t *file, int64_t len, vgo_dsp_info *out);          /* DspReader.cs:57-104 */
int vgo_dsp_read_data(const uint8_t *file, int64_t len, const vgo_dsp_info *o, uint8_t *const *outputs); /* :106-119 */

typedef struct vgo_adx_desc { /* what AdxWriter reads from CriAdxFormat + AdxConfiguration; sample_count and the loop points
                                 are the UNALIGNED values (the format adds alignment_samples, CriAdxFormat.cs:16-18) */
    int32_t channel_count, sample_rate, sample_count, looping, loop_start, loop_end, alignment_samples;
    int32_t frame_size, version, type, highpass_frequency, encryption_type, trim_file;
} vgo_adx_desc;
void vgo_adx_key_from_code(uint64_t key_code, int32_t key[3]);                   /* CriAdxKey.cs:18-24: seed, mult, inc */
void vgo_adx_key_from_string(const char *s, int32_t key[3]);                     /* CriAdxKey.cs:26-41 */
void vgo_adx_crypt_channel(uint8_t *adpcm, int length, const int32_t key[3], int encryption_type, int frame_size,
                           int channel_num, int channel_count);                  /* CriAdxEncryption.cs:16-44 */
int64_t vgo_adx_file_size(const vgo_adx_desc *d);                                /* AdxWriter.cs:18 */
int vgo_adx_write(const vgo_adx_desc *d, const uint8_t *const *audio, int audio_len, const int16_t *history,
                  const int32_t *key, uint8_t *out);                             /* AdxWriter.cs:70-140 */

int vgo_hca_key_tables(int key_type, uint64_t key_code, uint8_t *decrypt, uint8_t *encrypt); /* CriHcaKey.cs */
void vgo_hca_crypt_frame(uint8_t *frame, int frame_size, const uint8_t *table);  /* CriHcaEncryption.cs:21-33 */
int vgo_hca_write(const vgo_hca_info *h, const uint8_t *frames, const uint8_t *encrypt_table, int key_type,
                  const char *comment, uint32_t volume_bits, uint8_t *out);      /* HcaWriter.cs:37-178 */

#ifdef __cplusplus
}
#endif
#endif
