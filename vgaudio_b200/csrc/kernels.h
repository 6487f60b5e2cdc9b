// kernels.h — host-callable launchers of the sm_90a kernels (internal to libvgaudio_b200.so).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace vgb {

// c_abi.cu — raises cudaFuncAttributeMaxDynamicSharedMemorySize of `kernel` on the current device to `bytes` when it is
// lower; never lowers it.  The attribute belongs to the kernel on a device, not to the calling thread: every bound device
// needs it, and two threads launching one kernel on one device with different sizes (a device bound twice) must not
// lower it under each other's launch.
cudaError_t raise_dynamic_smem(const void *kernel, size_t bytes);
template <class Kernel>
cudaError_t raise_dynamic_smem(Kernel *kernel, size_t bytes) { return raise_dynamic_smem(reinterpret_cast<const void *>(kernel), bytes); }

// gc_coefs.cu — GcAdpcmCoefficients.CalculateCoefficients (Codecs/GcAdpcm/GcAdpcmCoefficients.cs:9-110)
void launch_gc_coef_frames(const int16_t *pcm, const GcChannelTable &tab, double2 *records, uint32_t *mask,
                           int max_frames, int frame_begin, int frame_end, cudaStream_t stream);
void launch_gc_coef_refine(const GcChannelTable &tab, const double2 *records, const uint32_t *mask,
                           int16_t *coefs_out, cudaStream_t stream);
// the refinement with a record of every pass (vgb_gcadpcm_debug_refine_trace): warps 4 or 8 picks the CTA width directly
void launch_gc_coef_refine_tap(const GcChannelTable &tab, const double2 *records, const uint32_t *mask, int16_t *coefs_out,
                               int warps, double *tap_cent, int32_t *tap_hits, cudaStream_t stream);

// gc_encode.cu — GcAdpcmEncoder.Encode / DspEncodeFrame / DspEncodeCoef (Codecs/GcAdpcm/GcAdpcmEncoder.cs:14-171)
int gc_encode_pick_segments(int n_channels, int max_frames, int *min_seg_out = nullptr);  // segments per channel (and the shortest segment) for the time-parallel encode
void launch_gc_encode(const int16_t *pcm, const GcChannelTable &tab, const int16_t *coefs, uint8_t *adpcm,
                      int max_frames, int frame_begin, int frame_end, GcSegArgs seg, cudaStream_t stream);
void launch_gc_encode_frames(int16_t *pcm_in_out, const int32_t *sample_count, const int16_t *coefs, int n_frames,
                             uint8_t *adpcm_out, cudaStream_t stream);

// gc_decode.cu — GcAdpcmDecoder.Decode (Codecs/GcAdpcm/GcAdpcmDecoder.cs:10-54)
void launch_gc_decode(const uint8_t *adpcm, const GcChannelTable &tab, const int16_t *coefs, int16_t *pcm,
                      int max_frames, int frame_begin, int frame_end, cudaStream_t stream);

// the time-parallel decode (chain / run-on / cascade); seg.trace, seg.status and seg.stats live in the caller's workspace
int gc_decode_pick_segments(int n_channels, int max_full_frames, int *min_seg_out);
void launch_gc_decode_seg(const uint8_t *adpcm, const GcDecChannel *tab, int n_channels, int16_t *pcm, GcDecSegArgs seg,
                          cudaStream_t stream);

// seek table (GcAdpcmSeekTable.cs:25-38) and loop context (GcAdpcmLoopContext.cs:17-26) of already encoded channels
void launch_gc_taps(const uint8_t *adpcm, const GcChannelTable &tab, const int16_t *coefs, const GcTapChannel *taps,
                    int16_t *tap_slab, int max_frames, cudaStream_t stream);

// gc_align.cu — GcAdpcmAlignment's tail (Formats/GcAdpcm/GcAdpcmAlignment.cs:44-55): per channel, the samples to re-encode
// into the 16-byte aligned row tail + dst_off, and the history pair into hist_enc[2c..] and hist_dec[2c..]
void launch_gc_align_tail(const int16_t *pcm, const GcAlignChannel *chans, int n_channels, int16_t *tail, int16_t *hist_enc,
                          int16_t *hist_dec, cudaStream_t stream);

// adx.cu — CriAdxCodec.Encode / Decode (Codecs/CriAdx/CriAdxCodec.cs:9-171)
int adx_encode_pick_segments(int n_channels, int max_whole_frames, int *min_seg_out = nullptr);
void launch_adx_encode(const int16_t *pcm, const AdxChannel *tab, int n_channels, uint8_t *adpcm, int16_t *history_out,
                       AdxSegArgs seg, cudaStream_t stream);  // seg.trace == nullptr: one segment (plain serial encode)
void launch_adx_decode(const uint8_t *adpcm, const AdxChannel *tab, int n_channels, int16_t *pcm, int32_t *status,
                       cudaStream_t stream);  // status[0] / [1]: lowest channel whose Fixed-type / other-type frame selects a filter
                                             // the reference cannot index (atomicMin), may be null
// the time-parallel decode (chain / run-on / cascade); seg.status, seg.stats and the trace live in the caller's workspace
int adx_decode_pick_segments(int n_channels, int max_body_frames, int *min_seg_out);
void launch_adx_decode_seg(const uint8_t *adpcm, const AdxDecChannel *tab, int n_channels, int16_t *pcm, AdxDecSegArgs seg,
                           cudaStream_t stream);

// hca.cu — CriHcaEncoder.EncodeFrame + CriHcaPacking.PackFrame (Codecs/CriHca/CriHcaEncoder.cs:271-286)
size_t hca_encode_smem_bytes(const HcaConfig &cfg);
cudaError_t launch_hca_encode(const int16_t *pcm, const HcaStream *streams, int n_streams, int max_frames,
                              const HcaConfig &cfg, const HcaTables &tables, uint8_t *frames_out, int32_t *status_out,
                              cudaStream_t stream);

// CriHcaPacking.UnpackFrame + CriHcaDecoder.DecodeFrame (Codecs/CriHca/CriHcaDecoder.cs:62-192)
size_t hca_decode_smem_bytes(const HcaConfig &cfg);
size_t hca_decode_parsed_bytes(const HcaConfig &cfg, int64_t total_frames);  // scratch between the parse and frame kernels
cudaError_t launch_hca_decode(const uint8_t *frames, const HcaStream *streams, int n_streams, int max_frames,
                              int64_t total_frames, const HcaConfig &cfg, const HcaTables &tables, uint8_t *parsed_scratch,
                              double *edge_scratch, int16_t *pcm, int32_t *status_out,
                              cudaStream_t stream);  // edge_scratch: 2*128 doubles per channel-frame

// Mdct.RunMdct / RunImdct (Utilities/Mdct.cs:63-119), the codec's 128-point instance, n_sequences x n_blocks blocks of 128 doubles
cudaError_t launch_hca_mdct128(const double *in, double *out, int n_sequences, int n_blocks, bool inverse, const HcaTables &tables,
                               cudaStream_t stream);

// interleave.cu — InterleaveExtensions.Interleave / DeInterleave (Utilities/Interleave.cs:9-166) for n_items payloads
cudaError_t launch_interleave(const void *in, int64_t in_channel_stride, int64_t in_item_stride, void *out, int64_t out_item_stride,
                              int n_items, int count, int64_t in_size, int64_t interleave, int64_t out_size, cudaStream_t stream);
cudaError_t launch_deinterleave(const void *in, int64_t in_item_stride, void *out, int64_t out_channel_stride, int64_t out_item_stride,
                                int n_items, int count, int64_t in_size, int64_t interleave, int64_t out_size, cudaStream_t stream);

// containers.cu — HpsReader.ToAudioStream's concatenation (Containers/Hps/HpsReader.cs:37-50): piece i copies len bytes
// from in + src_off to rows + dst_off; tile_first numbers its first CTA of kHpsGatherTile bytes (the launch has as many
// CTAs as the pieces' tiles together, 256 threads each)
struct HpsPiece {
    int64_t src_off, dst_off;
    int32_t len, tile_first;
};
constexpr int kHpsGatherTile = 8192;
__global__ void __launch_bounds__(256) hps_gather_kernel(const uint8_t *__restrict__ in, const HpsPiece *__restrict__ pieces, int n_pieces,
                                                          uint8_t *__restrict__ rows);

// adx_keys.cu — the key search of VGAudio.Tools/CrackAdx/GuessAdx.cs (TryScale :160-189, FindStartingKey :191-215,
// KeyIsValid :217-229) and the byte comparison of its re-encode confidence (Common.DiffArrays).
// A file's frames as the search reads them: frame i's scale s becomes one word (s & mask) | (s ? mask : 0) << 16, so
// that a key stream value x fails the frame exactly when ((x ^ w) & (w >> 16)) != 0.
struct AdxKeyFileDev {
    int64_t word_off;     // its words in the search's word array, frame 0 first
    int32_t frames;       // Scales.Length
    int32_t start;        // StartFrame
    int32_t first_scale;  // Scales[StartFrame]
    int32_t pad;
};
struct AdxKeyHit { int32_t seed, mult, inc; };
struct AdxKeySearch {
    const uint32_t *words;
    const AdxKeyFileDev *files;   // every file of the search: a key is kept only when it is valid on all of them
    int32_t n_files, file;        // file: the one whose TryScale this launch runs
    const int32_t *mults, *incs;  // the multiplier and increment lists of the box
    int32_t n_mult, n_inc;
    int32_t index0, n_index;      // scale indices index0 .. index0 + n_index - 1
    uint32_t seed_mask;           // MaxSeed - 1
    int32_t check_seed;           // revision 8: a seed must be in seed_bits (the prime list), for StartFrame 0 and FindStartingKey
    const uint32_t *seed_bits;    // 0x8000 bits
    unsigned long long *tried;    // kAdxKeyTried slots, zeroed: the keys already validated
    AdxKeyHit *hits;              // keys valid on every file, in no order, duplicates possible
    unsigned long long *n_hits;   // all of them are counted; only the first cap are stored
    uint32_t cap;
    unsigned long long *stats;    // [0] candidates tried, [1] frame steps, [2] full matches
};
constexpr int kAdxKeyTried = 1 << 16;
constexpr int kAdxKeyStage = 12288;  // words of the scanned file staged in shared memory (48 KiB)
cudaError_t launch_adx_key_search(const AdxKeySearch &a, int frames_after_start, cudaStream_t stream);
// out[2r] / out[2r+1]: the bytes of rows a + a_off[r] and b + b_off[r] that differ among their first n[2r] / n[2r+1]
cudaError_t launch_adx_byte_diff(const uint8_t *a, const int64_t *a_off, const uint8_t *b, const int64_t *b_off, const int32_t *n,
                                 int n_rows, int32_t *out, cudaStream_t stream);

// hca_keys.cu — HcaReader.FindKey's frame test (CriHcaEncryption.FindKey / TestKey, Codecs/CriHca/CriHcaEncryption.cs:34-87)
// over a list of type-56 key tables, one CTA per file.  Outcome of a (file, key): 0 pass, else 1 + 3 * j + r with j the
// window frame it stops at and r 0 a bad sync word, 1 a scale-factor delta out of range, 2 UnpackingWasSuccessful false.
constexpr int kHcaKeyWindow = 10;  // CriHcaEncryption.FramesToTest
struct HcaKeyFileDev {
    HcaConfig cfg;
    int64_t frames_off;  // the window's first byte in the search's frame bytes
    int32_t window;      // frames in the window, 0..kHcaKeyWindow
    int32_t pad;
};
struct HcaKeySearch {
    const uint8_t *frames;
    const HcaKeyFileDev *files;
    int32_t n_files, n_keys;
    const uint8_t *tables;   // [n_keys][256] decryption tables, 16-byte aligned
    int32_t every;           // 1: every outcome to outcomes[f * n_keys + k]; 0: first[2f] the decisive key of lowest index
                             // (or -1), first[2f + 1] its outcome
    int32_t max_channels;    // the largest channel count of the files (sizes the shared resolutions)
    int32_t *outcomes, *first;
    unsigned long long *stats;  // [0] (file, key) walks started, [1] frames unpacked: added to
};
cudaError_t launch_hca_key_search(const HcaKeySearch &a, cudaStream_t stream);

}  // namespace vgb
