// common.cuh — shared device helpers for the sm_90a codec kernels.
//
// Numeric contract (SURVEY.md Appendix A): the reference is C# compiled by RyuJIT for x64, i.e. IEEE-754
// binary64/binary32 with NO fused multiply-add, wrapping (unchecked) int32 arithmetic, truncating integer
// division and arithmetic right shifts.  The whole library is compiled with --fmad=false -prec-div=true
// -prec-sqrt=true; where a fused operation is wanted for speed it is written explicitly (__fmaf_rn) together
// with the argument for why its single rounding cannot differ.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace vgb {

constexpr int kGcFrameSamples = 14;
constexpr int kGcFrameBytes = 8;
constexpr int kGcFrameNibbles = 16;

// C# unchecked int32 arithmetic: do it in uint32 so C++ has no UB and wraps identically (A.7).
__host__ __device__ __forceinline__ int32_t wadd(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
__host__ __device__ __forceinline__ int32_t wsub(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }
__host__ __device__ __forceinline__ int32_t wmul(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); }

// Helpers.Clamp16 / Clamp4 (Utilities/Helpers.cs:32-48)
__host__ __device__ __forceinline__ int32_t clamp16(int32_t v) { return v > 32767 ? 32767 : (v < -32768 ? -32768 : v); }
__host__ __device__ __forceinline__ int32_t clamp4(int32_t v) { return v > 7 ? 7 : (v < -8 ? -8 : v); }

// GcAdpcmMath.cs:20-27,46 / Extensions.cs:145-146
__host__ __device__ __forceinline__ int32_t gc_sample_count_to_nibble_count(int32_t n)
{
    int32_t whole = n / kGcFrameSamples, rest = n % kGcFrameSamples;
    return kGcFrameNibbles * whole + (rest == 0 ? 0 : rest + 2);
}
__host__ __device__ __forceinline__ int32_t gc_sample_count_to_byte_count(int32_t n)
{
    int32_t nib = gc_sample_count_to_nibble_count(n);
    return nib / 2 + (nib & 1);
}
__host__ __device__ __forceinline__ int32_t gc_nibble_count_to_sample_count(int32_t nib)
{
    int32_t whole = nib / kGcFrameNibbles, rest = nib % kGcFrameNibbles;
    return kGcFrameSamples * whole + (rest < 2 ? 0 : rest - 2);
}
// DivideByRoundUp for non-negative operands (the reference goes through a double; identical for n < 2^31).
__host__ __device__ __forceinline__ int32_t div_round_up(int32_t a, int32_t b) { return (int32_t)(((int64_t)a + b - 1) / b); }

// Per-batch channel tables, all resident in HBM (uploaded once per call).
struct GcChannelTable {
    const int64_t *pcm_off;    // [ch] sample offset of the channel in the PCM slab (multiple of 8)
    const int64_t *adpcm_off;  // [ch] byte offset of the channel in the ADPCM slab (multiple of 16)
    const int64_t *rec_off;    // [ch] frame offset of the channel in the record slab (multiple of 32)
    const int32_t *n_samples;  // [ch] PCM length (coefficient analysis length / decode sample count)
    const int32_t *enc_count;  // [ch] samples to encode (<= n_samples)
    int16_t *hist;             // [ch][2] running history: [0] = hist1 (newest), [1] = hist2
    int32_t *status;           // decode: lowest channel index whose stream selects a predictor 8..15 (INT_MAX: none); may be null
    int32_t n_channels;
};

// Time-parallel encoding (gc_encode.cu): segment bookkeeping of one encode launch, all in the caller's workspace.
constexpr int kGcMinSegFrames = 4096; // default shortest segment (gc_encode_min_segment_frames): longer than the run-on tail
constexpr int kGcMaxSegments = 256;
constexpr int kGcStatWords = 18;      // GcSegArgs::stats
struct GcSegArgs {
    uint32_t *trace;             // [rec_off[ch] + frame] the pair (hist1 + 32768) | (hist2 + 32768) << 16 a frame hands on
    uint32_t *used_start;        // [ch][seg_count] the pair a boundary's run-on started from
    unsigned long long *stats;   // [0] frames re-encoded by run-ons, [1] by the cascade, [2] boundaries left to the cascade,
                                 // [3] longest run-on, [4 + b] run-ons of 2^b .. 2^(b+1)-1 frames (b = 13: longer)
    int32_t seg_count;
    int32_t min_seg_frames;      // no segment shorter than this
};

// One channel of a seek-table / loop-context request (gc_decode_kernel<true>).
struct GcTapChannel {
    int64_t out_off;            // first short of the channel in the tap slab: [entries * 2 seek shorts][hist1][hist2]
    int32_t samples_per_entry;  // 0: no seek table
    int32_t loop_start;         // < 0: no loop context
};

// One channel of a loop-alignment batch (gc_align_tail_kernel, GcAdpcmAlignment.cs:44-55).
struct GcAlignChannel {
    int64_t src_off;     // first sample of the channel's decoded prefix [0, loop_end) in the PCM slab
    int64_t dst_off;     // first sample of the channel's tail row (multiple of 8)
    int32_t loop_start, loop_end;
    int32_t keep;        // samplesToKeep: whole frames below loop_end
    int32_t count;       // samplesToEncode: the tail's length
};

// One channel of a CRI ADX batch (mirror of CriAdxParameters, Codecs/CriAdx/CriAdxParameters.cs:3-13, plus layout).
struct AdxChannel {
    int64_t pcm_off;     // sample offset in the PCM slab
    int64_t adpcm_off;   // byte offset in the ADPCM slab
    int32_t n_samples;   // encode: pcm.Length; decode: sampleCount
    int32_t frame_size, version, padding, type, filter;
    int32_t history;     // decode only (CriAdxParameters.History)
    int16_t coef0, coef1;  // fixed-table pair or CalculateCoefficients (host, once per distinct sample rate)
    int64_t trace_off;     // encode: first word of the channel in the trace slab of the time-parallel encoder (whole frames)
};

// Time-parallel ADX encoding (adx.cu): bookkeeping of one launch.  trace == nullptr: plain serial encode.
constexpr int kAdxMinSegFrames = 4096;  // a boundary's run-on is some hundred frames here (the fixed predictor's error decays slowly); VGB_ADX_MIN_SEG_FRAMES overrides
constexpr int kAdxMaxSegments = 64;
struct AdxSegArgs {
    uint32_t *trace;             // [trace_off[ch] + frame] the reconstructed pair a whole frame hands on
    uint32_t *used_start;        // [ch][seg_count] the pair a boundary's run-on started from
    unsigned long long *stats;   // [0] frames re-encoded by run-ons, [1] by the cascade, [2] boundaries repaired by the cascade
    int32_t seg_count;
    int32_t min_seg_frames;
};

// Time-parallel ADX decoding (adx.cu, the adx_decode_seg_kernel family).  CriAdxCodec.Decode (:9-54) walks frames
// 0..frames-1 from byte (padding / spf) * frame_size: the HEAD frame 0 yields samples start..min(spf, n)-1 of its frame
// (k0 of them), every BODY frame after it all spf samples, and at most one TAIL frame the rest; samples no frame reaches
// stay 0.  Only body frames are cut into segments.
struct AdxDecGeom {
    int32_t spf, start, frames, k0, body;
    int64_t in0;  // byte of the head frame in the channel's row
};
__host__ __device__ __forceinline__ AdxDecGeom adx_dec_geom(int32_t n, int32_t frame_size, int32_t padding)
{
    AdxDecGeom g;
    g.spf = (frame_size - 2) * 2;
    g.start = padding > 0 ? padding % g.spf : 0;                                      // :21
    g.in0 = (int64_t)(padding / g.spf) * frame_size;                                  // :22
    g.frames = n > 0 ? div_round_up(n, g.spf) : 0;                                    // :19
    const int32_t k0 = (n < g.spf ? n : g.spf) - g.start;
    g.k0 = g.frames > 0 && k0 > 0 ? k0 : 0;
    const int32_t full = 1 + (n - g.k0) / g.spf;                                      // head + whole frames after it
    g.body = g.frames > 0 ? (full < g.frames ? full : g.frames) - 1 : 0;
    return g;
}
struct AdxDecChannel {
    int64_t pcm_off;     // sample offset of the channel's output
    int64_t adpcm_off;   // byte offset of the channel's row (the fast path wants a multiple of 16)
    int64_t trace_off;   // first word of the channel in the trace slab (one word per body frame)
    int32_t n_samples, frame_size, version, padding, type;
    int32_t history;     // initial hist1 = hist2 (:16-17)
    int16_t coef0, coef1;  // CalculateCoefficients (Linear / Exponential; Fixed frames pick their own)
};
constexpr int kAdxDecMinSegFrames = 512;  // run-ons measured at p99 62 / max 101 frames; VGB_ADX_DEC_MIN_SEG_FRAMES overrides
constexpr int kAdxDecMaxSegments = 256;
constexpr int kAdxDecStatWords = 4;
struct AdxDecSegArgs {
    uint32_t *trace;             // [trace_off[ch] + body frame] the pair (hist1 & 0xffff) | hist2 << 16 after the frame
    uint32_t *used_start;        // [ch][kAdxDecMaxSegments] the pair a boundary's run-on started from
    unsigned long long *stats;   // [0] frames decoded by run-ons, [1] by the cascade, [2] boundaries the cascade repaired,
                                 // [3] longest run-on
    int32_t *status;             // [ch] bit 0: a Fixed-type frame selects a filter 4..7, bit 1: another type's frame a filter 1..7
    int32_t seg_count;
    int32_t min_seg_frames;
};

// ---- CRI HCA ------------------------------------------------------------------------------------------------
// per-stream status codes the encoder kernel can raise (mapped to the reference's exceptions by the C ABI)
constexpr int32_t VGB_HCA_BITRATE_TOO_LOW = 1;   // InvalidDataException("Bitrate is set too low.") CriHcaEncoder.cs:469-472
constexpr int32_t VGB_HCA_NOT_IMPLEMENTED = 2;   // NotImplementedException, CriHcaEncoder.cs:499
constexpr int32_t VGB_HCA_BIT_OVERFLOW = 3;      // InvalidOperationException, BitWriter.cs:30-33
constexpr int32_t VGB_HCA_BAD_SYNC = 4;          // InvalidDataException("Invalid frame header"), CriHcaPacking.cs:73-77
constexpr int32_t VGB_HCA_BAD_INDEX = 6;         // intensity index 15: IndexOutOfRangeException in ApplyIntensityStereo
constexpr int32_t VGB_HCA_BAD_DELTA = 5;         // UnpackFrame returns false (scale-factor delta out of range)

// Stream-independent encoder configuration = the HcaInfo fields EncodeFrame reads (HcaInfo.cs:5-48) + channel types
// (CriHcaFrame.GetChannelTypes :34-52).
struct HcaConfig {
    int32_t channel_count, frame_size;
    int32_t base_band_count, stereo_band_count, total_band_count, hfr_band_count, bands_per_hfr_group, hfr_group_count;
    int32_t channel_type[8];  // 0 Discrete, 1 StereoPrimary, 2 StereoSecondary
    uint8_t ath[128];         // decoder: CriHcaFrame.AthCurve (CriHcaFrame.cs:31), all zero unless HcaInfo.UseAthCurve
};

struct HcaStream {
    int64_t pcm_off;         // sample offset of channel 0 of the stream in the PCM slab
    int64_t channel_stride;  // samples between consecutive channels of the stream
    int64_t frames_off;      // byte offset of the stream's first frame in the output slab
    int64_t dct_off;         // decoder: index of the stream's first frame in the seam scratch (frames)
    int32_t sample_count, frame_count;
    int32_t inserted_samples, reserved;  // decoder: HcaInfo.InsertedSamples (CopyPcmToOutput, CriHcaDecoder.cs:26-37)
    // encoder: the input as one virtual stream (CriHcaEncoder.Encode :126-272): pre_zero zeros, pre_fill copies of the
    // first sample, sample_count source samples, post_count samples from loop_start on, zeros
    int32_t pre_zero, pre_fill, post_count, loop_start, src_count, last_chunk;
};

// Read-only codec tables, resident in HBM (uploaded once per device).  Values: the reference's test literals
// (hca_tables.inc) + host-computed trig/CRC/dead-zone tables (same formulas and libm as the oracle).
struct HcaTables {
    const double *window;                 // [128] MdctWindow (float32 data widened, CriHcaTables.cs:18)
    const double *sin_tab[8], *cos_tab[8];  // Mdct trig tables by size bits 0..7 (Mdct.cs:183-195)
    const int32_t *shuffle;               // [128] (Mdct.cs:197-208)
    double mdct_scale, sqrt2;
    const double *dequantizer_scaling, *quantizer_scaling;  // [64]
    const double *inv_step, *dead_zone;   // [16] QuantizerInverseStepSize, QuantizerDeadZone
    const double *intensity_bounds;       // [14]
    const uint8_t *scale_to_resolution;   // [59]
    const uint8_t *quantized_max_bits;    // [16]
    const uint8_t (*quantize_bits)[16];   // [8][16] QuantizeSpectrumBits
    const uint8_t (*quantize_value)[16];  // [8][16] QuantizeSpectrumValue
    const uint16_t *crc_table;            // [256] Crc16 (poly 0x8005)
    // decoder side
    const double *step_size;              // [16] QuantizerStepSize
    const double *intensity_ratio;        // [15]
    const double *scale_conversion;       // [128]
    const uint8_t (*dequantize_bits)[16]; // [8][16] QuantizedSpectrumBits
    const int8_t (*dequantize_value)[16]; // [8][16] QuantizedSpectrumValue
};

}  // namespace vgb
