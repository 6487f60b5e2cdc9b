/*
 * vgaudio_b200.h — C ABI of libvgaudio_b200.so: the H100 (sm_90a) batch codec engine that replaces the
 * per-channel CPU hot path of Thealexbarney/VGAudio.
 *
 * This header is the drop-in boundary.  Every entry point names the reference interface it replaces
 * (paths relative to VGAudio's src/VGAudio/).  The reference-side binding (C# P/Invoke) a maintainer
 * would add is shown in INTEGRATION.md and bindings/csharp/.
 *
 * Conventions
 *   - cdecl, plain pointers and sizes only; all buffers are caller-owned, nothing allocated here crosses the
 *     boundary except through vgb_host_alloc/vgb_host_free.
 *   - Every function returns an int32 status: VGB_OK (0) or a negative VGB_E_* code; vgb_last_error() gives the
 *     thread-local message.  The C# shim maps the codes back to the exception types the reference throws.
 *   - "host" entry points take HOST pointers and perform the H2D/D2H copies themselves (pinned memory is used
 *     directly, pageable memory is staged).  "_dev" entry points take DEVICE pointers that are already resident
 *     in HBM and a cudaStream_t (passed as void*); they never touch host memory and never synchronise.
 *   - There is NO CPU fallback: without a usable CUDA device every codec call fails with VGB_E_CUDA.
 *   - Thread-safe: concurrent calls from different host threads are serialised per device workspace.
 */
#ifndef VGAUDIO_B200_H
#define VGAUDIO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VGB_OK        0
#define VGB_E_ARG    -1  /* ArgumentException / ArgumentOutOfRangeException on the C# side */
#define VGB_E_DATA   -2  /* InvalidDataException */
#define VGB_E_STATE  -3  /* InvalidOperationException */
#define VGB_E_CUDA   -4  /* no device / CUDA runtime failure */
#define VGB_E_NCCL   -5  /* NCCL missing or a collective failed (vgb_nccl_*, vgb_scatterv_dev, vgb_gatherv_dev) */
#define VGB_E_NOMEM  -6  /* OutOfMemoryException */

#define VGB_ABI_VERSION 1

/* ---------------------------------------------------------------------------------------------------------
 * Library / device control
 * ------------------------------------------------------------------------------------------------------- */
int32_t vgb_abi_version(void);
/* Bind the calling process to CUDA device `device` (>= 0) and create the workspace.  Idempotent. */
int32_t vgb_init(int32_t device, uint32_t flags);
int32_t vgb_shutdown(void);
/* Bind several devices (SURVEY §8b's vgb_init(n_devices, flags); the reference's counterpart is Parallel.ForEach over
 * files, src/VGAudio.Cli/Batch.cs:24-25).  devices[0] becomes the primary device (the one the *_dev entry points, timers
 * and debug taps use); every host-pointer codec *_batch call and both batch converters (vgb_convert_wave_batch,
 * vgb_convert_dsp_to_wave_batch) are then sharded over all bound devices by greedy longest-first bin packing of the
 * units' sample counts - one worker thread and one H2D / kernel / D2H pipeline per device, each over its own PCIe link,
 * results written straight into the caller's arrays (no collective: host data reaches a GPU fastest over that GPU's own
 * link).  The single-shot container calls (vgb_*_read_batch, vgb_*_write_batch, vgb_*_crypt_batch) stay on the primary.
 * A device may be listed more than once. */
int32_t vgb_init_devices(const int32_t *devices, int32_t n_devices, uint32_t flags);
int32_t vgb_device_count(void);

/* ---------------------------------------------------------------------------------------------------------
 * The one exchange step of a multi-GPU job whose data is already resident in HBM (SURVEY §8e): scatterv of PCM from a
 * root rank, gatherv of bitstreams back.  One rank per GPU (one process per GPU under torchrun, or one thread per device);
 * grouped ncclSend / ncclRecv with per-rank byte counts - no padding to the longest shard, no host round trip.  NCCL is
 * bound at run time (dlopen of libnccl.so.2, preferring the copy the process already loaded); every failure is
 * VGB_E_NCCL.  The reference has no counterpart: its Parallel.ForEach over files (src/VGAudio.Cli/Batch.cs:24-25) shares
 * one address space.
 *   vgb_nccl_unique_id   rank 0 creates the 128-byte id and hands it to the others (any out-of-band channel)
 *   vgb_nccl_init        every rank, with its CUDA device current (after vgb_init): joins the communicator
 *   vgb_scatterv_dev     root: bytes [send_offset[r], +counts[r]) of d_send go to rank r's d_recv; asynchronous on stream
 *   vgb_gatherv_dev      rank r's counts[r] bytes at d_send land at d_recv + recv_offset[r] on the root
 *   vgb_sendrecv_dev     one NCCL group of arbitrary sends and receives (both directions at once: the pipelined batch path
 *                        scatters chunk k+1 while it gathers chunk k-1 over the full-duplex links)
 *   vgb_partition_lpt    greedy longest-first bin packing of units (files / channels) onto parts by weight (samples):
 *                        part_out[u] = part of unit u, load_out[p] = summed weight (may be NULL)
 * ------------------------------------------------------------------------------------------------------- */
#define VGB_NCCL_ID_BYTES 128
int32_t vgb_nccl_unique_id(uint8_t *id_out /* [VGB_NCCL_ID_BYTES] */);
int32_t vgb_nccl_init(const uint8_t *id, int32_t n_ranks, int32_t rank);
int32_t vgb_nccl_shutdown(void);
int32_t vgb_nccl_version(void); /* e.g. 22809; 0 when NCCL cannot be loaded */
int32_t vgb_scatterv_dev(const void *d_send, const int64_t *send_offset, const int64_t *counts /* [n_ranks] bytes */,
                         void *d_recv, int32_t root, void *cuda_stream);
int32_t vgb_gatherv_dev(const void *d_send, void *d_recv, const int64_t *recv_offset, const int64_t *counts /* [n_ranks] bytes */,
                        int32_t root, void *cuda_stream);
int32_t vgb_sendrecv_dev(const void *const *send_ptr, const int64_t *send_bytes, const int32_t *send_peer, int32_t n_send,
                         void *const *recv_ptr, const int64_t *recv_bytes, const int32_t *recv_peer, int32_t n_recv, void *cuda_stream);
int32_t vgb_partition_lpt(const int64_t *weight, int32_t n_units, int32_t n_parts, int32_t *part_out, int64_t *load_out);
const char *vgb_last_error(void);
/* Pinned host memory, so the host entry points can DMA straight from/to the caller's buffers. */
int32_t vgb_host_alloc(void **ptr_out, uint64_t bytes);
int32_t vgb_host_free(void *ptr);
/* Number of kernel launches issued by this library since vgb_init (bench.py reports it as gpu_launches). */
int64_t vgb_kernel_launch_count(void);

/* ---------------------------------------------------------------------------------------------------------
 * GcAdpcmMath (Codecs/GcAdpcm/GcAdpcmMath.cs:7-47) — so the caller can size its output arrays first
 * ------------------------------------------------------------------------------------------------------- */
int32_t vgb_gcadpcm_sample_count_to_byte_count(int32_t sample_count);   /* :46 */
int32_t vgb_gcadpcm_byte_count_to_sample_count(int32_t byte_count);     /* :47 */
int32_t vgb_gcadpcm_sample_count_to_nibble_count(int32_t sample_count); /* :20-27 */
int32_t vgb_gcadpcm_nibble_count_to_sample_count(int32_t nibble_count); /* :11-18 */
int32_t vgb_gcadpcm_sample_to_nibble(int32_t sample);                   /* :38-44 */
int32_t vgb_gcadpcm_nibble_to_sample(int32_t nibble);                   /* :29-36 */

/* Mirror of GcAdpcmParameters : CodecParameters (Codecs/GcAdpcm/GcAdpcmParameters.cs:3-7,
 * Codecs/CodecParameters.cs:3-17).  sample_count == -1 means "the whole input" exactly as in
 * GcAdpcmEncoder.Encode (GcAdpcmEncoder.cs:17) / GcAdpcmDecoder.Decode (GcAdpcmDecoder.cs:12). */
typedef struct vgb_gc_params {
    int32_t sample_count;
    int16_t history1;
    int16_t history2;
} vgb_gc_params;

/* IProgressReport.ReportAdd (IProgressReport.cs:3-28) — invoked from the calling host thread between device
 * chunks with the number of frames finished since the last call; the deltas sum to the reference's
 * SetTotal value (GcAdpcmFormat.cs:62-63). */
typedef void (*vgb_progress_cb)(void *user, int64_t frames_done_delta);

/* ---------------------------------------------------------------------------------------------------------
 * GC-ADPCM, host buffers.  One call replaces one Parallel.For over channels.
 * ------------------------------------------------------------------------------------------------------- */

/* GcAdpcmCoefficients.CalculateCoefficients (GcAdpcmCoefficients.cs:9-110) for n_channels independent
 * channels.  pcm[c] points at n_samples[c] int16 samples; coefs_out is [n_channels][16]. */
int32_t vgb_gcadpcm_coefs_batch(const int16_t *const *pcm, const int32_t *n_samples, int32_t n_channels,
                                int16_t *coefs_out);

/* GcAdpcmFormat.EncodeFromPcm16's loop body (Formats/GcAdpcm/GcAdpcmFormat.cs:65-68 -> EncodeChannel :129-135
 * = CalculateCoefficients + GcAdpcmEncoder.Encode, GcAdpcmEncoder.cs:14-46) for every channel at once.
 *   params      NULL (all defaults) or [n_channels]
 *   coefs_in    NULL = run the coefficient analysis; else [n_channels][16] (GcAdpcmEncoder.Encode only)
 *   coefs_out   [n_channels][16], receives the coefficients used (may alias coefs_in)
 *   adpcm_out   adpcm_out[c] receives SampleCountToByteCount(sample_count) bytes
 *   cb/user     optional progress callback */
int32_t vgb_gcadpcm_encode_batch(const int16_t *const *pcm, const int32_t *n_samples, const vgb_gc_params *params,
                                 const int16_t *coefs_in, int32_t n_channels, int16_t *coefs_out,
                                 uint8_t *const *adpcm_out, vgb_progress_cb cb, void *user);

/* GcAdpcmFormat.ToPcm16's loop body (GcAdpcmFormat.cs:45-48 -> GcAdpcmChannel.GetPcmAudio, GcAdpcmChannel.cs:57-60
 * -> GcAdpcmDecoder.Decode, GcAdpcmDecoder.cs:10-54).  n_bytes[c] is the length of adpcm[c]; params[c].sample_count
 * == -1 decodes ByteCountToSampleCount(n_bytes[c]) samples.  pcm_out[c] receives sample_count samples.
 * VGB_E_DATA: a frame header selects a predictor outside 0..7 (IndexOutOfRangeException at GcAdpcmDecoder.cs:31-32);
 * the message names the lowest such channel.  The device-resident variant below decodes such a frame with the lookup
 * wrapped (predictor & 7) and leaves the lowest such channel in its workspace, where vgb_gcadpcm_decode_dev_status
 * reports it. */
int32_t vgb_gcadpcm_decode_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int16_t *coefs,
                                 const vgb_gc_params *params, int32_t n_channels, int16_t *const *pcm_out);

/* GcAdpcmEncoder.DspEncodeFrame (GcAdpcmEncoder.cs:48-94) for n_frames INDEPENDENT frames (the IDspTool /
 * GcAdpcmAlignment use, Formats/GcAdpcm/GcAdpcmAlignment.cs:57).  pcm_in_out is [n_frames][16]: two history samples
 * (older first) then 14 samples, rewritten with the reconstruction; sample_count[f] in 0..14 (NULL = 14);
 * coefs is [n_frames][16]; adpcm_out is [n_frames][8]. */
int32_t vgb_gcadpcm_encode_frames(int16_t *pcm_in_out, const int32_t *sample_count, const int16_t *coefs,
                                  int32_t n_frames, uint8_t *adpcm_out);

/* ---------------------------------------------------------------------------------------------------------
 * GC-ADPCM, device-resident ("_dev").  Channel c occupies
 *      d_pcm   + pcm_offset[c]    .. n_samples[c] samples      (pcm_offset in samples, multiple of 8)
 *      d_adpcm + adpcm_offset[c]  .. byte count of the channel (adpcm_offset in bytes, multiple of 16)
 * The offset/length tables are HOST arrays (they are tiny and are uploaded on `stream`); both slabs must be
 * padded so that each channel's region is readable/writable up to the next multiple of 16 bytes.
 * vgb_gcadpcm_workspace_bytes() tells how much scratch HBM the call needs for the given total frame count.
 * Base pointers: d_pcm, d_adpcm and d_workspace must be 16-byte aligned, d_coefs_in / d_coefs_out / d_coefs 2-byte
 * aligned (the kernels read and write them with 16-byte vector and cp.async accesses); VGB_E_ARG otherwise, before any
 * device work.
 * ------------------------------------------------------------------------------------------------------- */
uint64_t vgb_gcadpcm_workspace_bytes(int64_t total_frames, int32_t n_channels);

int32_t vgb_gcadpcm_encode_dev(const int16_t *d_pcm, const int64_t *pcm_offset, const int32_t *n_samples,
                               const vgb_gc_params *params, int32_t n_channels,
                               const int16_t *d_coefs_in, int16_t *d_coefs_out,
                               uint8_t *d_adpcm, const int64_t *adpcm_offset,
                               void *d_workspace, uint64_t workspace_bytes, void *cuda_stream);

int32_t vgb_gcadpcm_coefs_dev(const int16_t *d_pcm, const int64_t *pcm_offset, const int32_t *n_samples,
                              int32_t n_channels, int16_t *d_coefs_out,
                              void *d_workspace, uint64_t workspace_bytes, void *cuda_stream);

int32_t vgb_gcadpcm_decode_dev(const uint8_t *d_adpcm, const int64_t *adpcm_offset, const int16_t *d_coefs,
                               const vgb_gc_params *params /* sample_count must be >= 0 */, int32_t n_channels,
                               int16_t *d_pcm, const int64_t *pcm_offset,
                               void *d_workspace, uint64_t workspace_bytes, void *cuda_stream);
/* vgb_gcadpcm_decode_dev is asynchronous; a frame header that selects a predictor outside 0..7 (the reference's
 * IndexOutOfRangeException, GcAdpcmDecoder.cs:31-32) leaves the lowest such channel in the workspace.  This call
 * synchronises the stream and maps it: VGB_OK or VGB_E_DATA. */
int32_t vgb_gcadpcm_decode_dev_status(const void *d_workspace, int32_t n_channels, void *cuda_stream);

/* ---------------------------------------------------------------------------------------------------------
 * Post-encode channel rebuild (SURVEY.md 8f rank 1): what GcAdpcmChannelBuilder.GetSeekTable / GetLoopContext
 * (Formats/GcAdpcm/GcAdpcmChannelBuilder.cs:176-202) compute by decoding the whole channel again on the CPU.
 *   seek table    GcAdpcmSeekTable.CreateSeekTable (GcAdpcmSeekTable.cs:25-38): entry i = (pcm[i*spe - 1], pcm[i*spe - 2]),
 *                 entry 0 = (0, 0), entries = ceil(sample_count / spe)
 *   loop context  GcAdpcmLoopContext (GcAdpcmLoopContext.cs:17-26): predictor/scale byte of the frame holding the loop
 *                 start (GcAdpcmDecoder.GetPredictorScale :56-59), hist1 = pcm[loop_start - 1], hist2 = pcm[loop_start - 2]
 *   alignment     GcAdpcmAlignment (GcAdpcmAlignment.cs:20-63): the re-encode that moves an unaligned loop start onto a
 *                 multiple, below (vgb_gcadpcm_alignment, vgb_gcadpcm_align_batch)
 * ------------------------------------------------------------------------------------------------------- */
typedef struct vgb_gc_tap_params {
    int32_t sample_count;
    int32_t samples_per_seek_table_entry; /* 0: no seek table (GetSeekTable returns null) */
    int32_t loop_start;                   /* < 0: no loop context */
} vgb_gc_tap_params;

int32_t vgb_gcadpcm_seek_entry_count(int32_t sample_count, int32_t samples_per_entry);

/* adpcm / n_bytes / coefs as in vgb_gcadpcm_decode_batch.  seek_table_out[c] receives entry_count * 2 shorts (may be
 * NULL when the channel asks for no table); loop_context_out is [n_channels][3] = pred_scale, hist1, hist2 (zeros for
 * a channel without a loop; may be NULL when no channel has one). */
int32_t vgb_gcadpcm_seek_context_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int16_t *coefs,
                                       const vgb_gc_tap_params *params, int32_t n_channels,
                                       int16_t *const *seek_table_out, int16_t *loop_context_out);

/* Loop points of one channel before alignment (GcAdpcmAlignment's constructor arguments) and the geometry after it. */
typedef struct vgb_gc_align_params { int32_t multiple, loop_start, loop_end; } vgb_gc_align_params;
typedef struct vgb_gc_alignment { int32_t alignment_needed, loop_start_aligned, sample_count_aligned; } vgb_gc_alignment;

/* GcAdpcmAlignment's geometry (GcAdpcmAlignment.cs:22-31 with Helpers.GetNextMultiple / LoopPointsAreAligned,
 * Helpers.cs:71-83; C# `%` truncates toward zero).  Host only, needs no device.  Every field is 0 when no alignment is
 * needed, as in the reference.  A multiple <= 0 leaves the loop start where it is, yet a negative multiple that does not
 * divide the loop start still counts as "alignment needed": the tail is then re-encoded with no shift.
 * VGB_E_ARG (out zeroed) when alignment is needed and the loop points are unusable, as for vgb_gcadpcm_align_batch. */
int32_t vgb_gcadpcm_alignment(const vgb_gc_align_params *p, vgb_gc_alignment *out);

/* new GcAdpcmAlignment(multiple, loopStart, loopEnd, adpcm, coefs) for n_channels channels, each with its own params;
 * adpcm / n_bytes / coefs as in vgb_gcadpcm_decode_batch.  For a channel that needs alignment:
 *   adpcm_aligned_out[c]  SampleCountToByteCount(sample_count_aligned) bytes (AdpcmAligned): the first loop_end / 14
 *                         whole frames of adpcm[c], then the re-encoded tail
 *   pcm_aligned_out       NULL, or pcm_aligned_out[c] receives sample_count_aligned samples (PcmAligned)
 * Channels that need no alignment are skipped: their output rows may be NULL and are not written.
 * Only the first SampleCountToByteCount(loop_end) bytes of a channel are read; the first decode starts from history
 * (0, 0), not from the channel's start context (:41-42).  Errors, checked only on channels that need alignment:
 *   VGB_E_ARG   before any device work: a negative loop point, loop_end < loop_start, n_bytes[c] shorter than loop_end
 *               samples, sample_count_aligned past INT32_MAX, or loop_start == loop_end while the start moves.  The last
 *               is a deliberate difference: the reference's tail loop (:48) then steps by zero and never ends.
 *   VGB_E_DATA  a frame header below loop_end selects a predictor outside 0..7 (IndexOutOfRangeException in the first
 *               Decode); the message names the lowest such channel.  The output rows are then unspecified.
 * Sharded over the bound devices like the other host-pointer batch calls (weights: loop_end). */
int32_t vgb_gcadpcm_align_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int16_t *coefs,
                                const vgb_gc_align_params *params, int32_t n_channels,
                                uint8_t *const *adpcm_aligned_out, int16_t *const *pcm_aligned_out);

/* ---------------------------------------------------------------------------------------------------------
 * Block (de)interleave of channel payloads (SURVEY.md 8f rank 2): InterleaveExtensions.Interleave / DeInterleave
 * (Utilities/Interleave.cs:9-166), the byte shuffle the container writers / readers run next to the codec path
 * (AdxWriter.cs:131, BrstmWriter.cs:294, WaveReader.cs:47 ...).  Blocks of interleave_size bytes per channel, a shorter
 * last block on either side, only min(in, out) blocks / bytes copied, the rest of the output zero; out_size == -1
 * means in_size.  The _dev entry points work on n_items payloads resident in HBM (strides in bytes), which is how the
 * shuffle fuses behind an encode; the host entry points handle one payload like the reference calls.
 * ------------------------------------------------------------------------------------------------------- */
int32_t vgb_interleave_dev(const void *d_in, int64_t in_channel_stride, int64_t in_item_stride, void *d_out, int64_t out_item_stride,
                           int32_t n_items, int32_t count, int64_t in_size, int32_t interleave_size, int64_t out_size, void *cuda_stream);
int32_t vgb_deinterleave_dev(const void *d_in, int64_t in_item_stride, void *d_out, int64_t out_channel_stride, int64_t out_item_stride,
                             int32_t n_items, int32_t count, int64_t in_size, int32_t interleave_size, int64_t out_size, void *cuda_stream);
/* inputs[count] of in_size bytes -> output of out_size * count bytes (T[] Interleave<T>(this T[][] inputs, ...), :9-41) */
int32_t vgb_interleave(const uint8_t *const *inputs, int32_t count, int32_t in_size, int32_t interleave_size, int32_t out_size,
                       uint8_t *output);
/* input of `length` bytes -> outputs[count] of out_size bytes (T[][] DeInterleave<T>(this T[] input, ...), :81-117);
 * VGB_E_ARG when length is not divisible by count (ArgumentOutOfRangeException) */
int32_t vgb_deinterleave(const uint8_t *input, int32_t length, int32_t interleave_size, int32_t count, int32_t out_size,
                         uint8_t *const *outputs);

/* Per-kernel device time (ms, CUDA events on the launching stream) of the most recent *_dev or host call on this
 * thread's workspace: [0] GC coefficient phase 1, [1] GC coefficient refinement, [2] GC encode, [3] GC decode,
 * [4] ADX encode, [5] ADX decode, [6] HCA encode, [7] HCA decode (all kernels), [8] interleave, [9] deinterleave.  Only filled when
 * vgb_set_kernel_timing(1) was called; bench.py / tools/secondary_bench.py use it for the roofline objects. */
int32_t vgb_set_kernel_timing(int32_t enabled);
int32_t vgb_last_kernel_ms(float *ms_out, int32_t n);

/* Device timeline of the last host GC-ADPCM encode call, ms since its first copy was enqueued: per channel group
 * [H2D landed, kernels finished, D2H finished] (evidence of the copy/compute overlap; bench.py reports it). */
int32_t vgb_debug_last_timeline(float *ms_out, int32_t n);
/* same call, per channel group: when its coefficient kernels finished (ms since the first copy was enqueued) */
int32_t vgb_debug_last_coefs_done(float *ms_out, int32_t n);

/* Bookkeeping of the most recent GC-ADPCM encode launch, which runs time-parallel (every channel's frame range is
 * cut into segments encoded concurrently, then spliced at the boundaries; gc_encode.cu): out[0] segments per channel,
 * out[1] frames re-encoded by the boundary run-ons, out[2] frames re-encoded by the serial cascade (the fallback when a
 * boundary does not re-lock inside its segment), out[3] boundaries the cascade had to repair, out[4] the longest
 * run-on in frames, out[5 + b] the number of run-ons of 2^b .. 2^(b+1)-1 frames (b = 0..13, the last one open).  n = how
 * many words to fill (up to 19).  bench.py reports (out[1] + out[2]) / frames as `fallback_frames_frac`.  Synchronises
 * the device.  The words live in the workspace of that launch: after a vgb_gcadpcm_encode_dev the caller's workspace
 * must still be allocated (and not yet reused) when this is called.  VGB_GC_SEGMENTS=<n> in the environment forces the
 * segment count (1 = the plain serial loop of GcAdpcmEncoder.cs:30-43). */
int32_t vgb_gcadpcm_debug_splice_stats(uint64_t *out, int32_t n);

/* Debug/test taps (tests/ only): run coefficient phase 1 and return, per frame, the direct-form pair and the
 * accept flag the refinement consumes.  Host buffers; dir_out [frames][2] doubles, accepted_out [frames] bytes. */
int32_t vgb_gcadpcm_debug_records(const int16_t *pcm, int32_t n_samples, double *dir_out, uint8_t *accepted_out);
/* Debug/test tap (tests/ only): coefficient phase 1 and the refinement for a ragged batch, with what every refinement
 * pass leaves: pass 0 is the ordered mean, passes 1..6 split and reassign with 2, 2, 4, 4, 8, 8 centroids.  warps (4 or 8)
 * picks the refinement's CTA width directly.  Host buffers: cent_out [ch][7][8][2] doubles (c1, c2 of every centroid),
 * hits_out [ch][7][8] (records per bucket), coefs_out [ch][16]. */
int32_t vgb_gcadpcm_debug_refine_trace(const int16_t *const *pcm, const int32_t *n_samples, int32_t n_channels, int32_t warps,
                                       double *cent_out, int32_t *hits_out, int16_t *coefs_out);

/* ---------------------------------------------------------------------------------------------------------
 * CRI ADX (Codecs/CriAdx/CriAdxCodec.cs), host buffers.  One call replaces one Parallel.For over channels
 * (Formats/CriAdx/CriAdxFormat.cs:67-81 encode, :37-49 decode).
 * ------------------------------------------------------------------------------------------------------- */

/* Mirror of CriAdxParameters : CodecParameters (Codecs/CriAdx/CriAdxParameters.cs:3-13).
 * type: 2 = Fixed, 3 = Linear, 4 = Exponential (CriAdxType.cs:3-8). */
typedef struct vgb_adx_params {
    int32_t sample_rate;         /* default 48000 */
    int32_t highpass_frequency;  /* default 500 (decode only; Encode hard-codes 500, CriAdxCodec.cs:63) */
    int32_t frame_size;          /* default 18 */
    int32_t version;             /* default 4 */
    int32_t history;             /* decode: initial hist1 = hist2 (CriAdxCodec.cs:16-17) */
    int32_t padding;
    int32_t type;                /* default 3 (Linear) */
    int32_t filter;              /* Fixed only: 0..3 */
} vgb_adx_params;

/* CriAdxCodec.CalculateCoefficients(highpassFreq, sampleRate) (CriAdxCodec.cs:173-184): the two Q12 prediction
 * coefficients of the Linear / Exponential types.  Pure host arithmetic (doubles, truncating casts). */
int32_t vgb_adx_calculate_coefficients(int32_t highpass_frequency, int32_t sample_rate, int16_t *coefs_out);

/* frameCount * FrameSize of CriAdxCodec.Encode (CriAdxCodec.cs:59-61,67) */
int32_t vgb_adx_encoded_byte_count(int32_t pcm_length, int32_t padding, int32_t frame_size);

/* CriAdxCodec.Encode(short[] pcm, CriAdxParameters config) (CriAdxCodec.cs:56-105) for every channel.
 * params is [n_channels]; history_out[c] receives the value the reference writes back into config.History (:73,
 * read by CriAdxFormat.cs:80); adpcm_out[c] receives vgb_adx_encoded_byte_count(...) bytes. */
int32_t vgb_adx_encode_batch(const int16_t *const *pcm, const int32_t *n_samples, const vgb_adx_params *params,
                             int32_t n_channels, int16_t *history_out, uint8_t *const *adpcm_out,
                             vgb_progress_cb cb, void *user);

/* Device-resident variant of vgb_adx_encode_batch (same semantics, asynchronous on `cuda_stream`): d_pcm / d_adpcm are HBM
 * slabs, channel c at pcm_offset[c] samples (a multiple of 8) / adpcm_offset[c] bytes (even); d_history_out ([n] shorts)
 * may be NULL; d_workspace holds the channel table and the bookkeeping of the time-parallel encoder (one word per
 * 32-sample frame; vgb_adx_workspace_bytes(total samples, channels)).  d_pcm must be 16-byte aligned (the encoder
 * copies it with cp.async), d_adpcm and d_history_out 2-byte aligned, d_workspace 8-byte aligned; VGB_E_ARG otherwise.
 * The multi-GPU batch path and bench.py's device-resident figures use it. */
uint64_t vgb_adx_workspace_bytes(int64_t total_samples, int32_t n_channels);
int32_t vgb_adx_encode_dev(const int16_t *d_pcm, const int64_t *pcm_offset, const int32_t *n_samples, const vgb_adx_params *params,
                           int32_t n_channels, int16_t *d_history_out, uint8_t *d_adpcm, const int64_t *adpcm_offset,
                           void *d_workspace, uint64_t workspace_bytes, void *cuda_stream);

/* CriAdxCodec.Decode(byte[] adpcm, int sampleCount, CriAdxParameters config) (CriAdxCodec.cs:9-54).
 * n_bytes[c] = length of adpcm[c]; pcm_out[c] receives sample_count[c] samples.
 * VGB_E_DATA: a Fixed-type frame selects a filter outside 0..3 (IndexOutOfRangeException at CriAdxCodec.Coefs, :186-191). */
int32_t vgb_adx_decode_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int32_t *sample_count,
                             const vgb_adx_params *params, int32_t n_channels, int16_t *const *pcm_out);

/* Device-resident, time-parallel variant of vgb_adx_decode_batch (same rules for params, sample_count and n_bytes, except
 * that any sample rate is taken, as CriAdxCodec.Decode takes it; asynchronous on `cuda_stream`): channel c reads n_bytes[c] bytes at d_adpcm + adpcm_offset[c] and writes
 * sample_count[c] samples to d_pcm + pcm_offset[c], zeros included where the padding logic produces none.  Each
 * channel's frames are cut into segments decoded concurrently and spliced where a frame-end history pair matches
 * (adx.cu; the segment count follows the SM and channel counts, VGB_ADX_DEC_SEGMENTS / VGB_ADX_DEC_MIN_SEG_FRAMES in the
 * environment force it / the shortest segment).  18-byte frames whose row starts at a 16-byte aligned address take the
 * fast path, and the output store width follows the address of each row; any base pointer and offset and any frame size
 * 3..255 decode bit-exactly.  d_pcm must be 2-byte aligned and d_workspace 8-byte aligned (VGB_E_ARG otherwise).  A frame
 * that yields no sample (the head frame when sample_count <= padding % samples per frame) never indexes the coefficient
 * table, so its filter number is not checked, as in the reference.  The workspace (vgb_adx_decode_workspace_bytes from
 * the same sample counts and params) holds the channel table, per-channel status words and the splice bookkeeping:
 * vgb_adx_decode_dev_status synchronises the stream and returns VGB_E_DATA for the lowest channel whose Fixed-type
 * frame selects a filter 4..7, with vgb_adx_decode_batch's message. */
uint64_t vgb_adx_decode_workspace_bytes(const int32_t *sample_count, const vgb_adx_params *params, int32_t n_channels);
int32_t vgb_adx_decode_dev(const uint8_t *d_adpcm, const int64_t *adpcm_offset, const int32_t *n_bytes, const int32_t *sample_count,
                           const vgb_adx_params *params, int32_t n_channels, int16_t *d_pcm, const int64_t *pcm_offset,
                           void *d_workspace, uint64_t workspace_bytes, void *cuda_stream);
int32_t vgb_adx_decode_dev_status(const void *d_workspace, int32_t n_channels, void *cuda_stream);
/* Bookkeeping of the most recent vgb_adx_decode_dev on this thread's context (its workspace must still be allocated;
 * criadx.decode_dev returns it for that reason):
 * out[0] segments per channel, out[1] frames decoded by the boundary run-ons, out[2] frames decoded by the serial
 * cascade (boundaries whose run-on did not lock inside its segment), out[3] boundaries the cascade repaired, out[4] the
 * longest run-on in frames.  n = how many words to fill (up to 5).  Synchronises the device. */
int32_t vgb_adx_debug_decode_stats(uint64_t *out, int32_t n);

/* ---------------------------------------------------------------------------------------------------------
 * CRI HCA encode (Codecs/CriHca/CriHcaEncoder.cs), host buffers.  One call replaces CriHcaFormat.EncodeFromPcm16
 * (Formats/CriHca/CriHcaFormat.cs:34-84, single-threaded in the reference) for a batch of streams.
 * ------------------------------------------------------------------------------------------------------- */

/* Mirror of CriHcaParameters : CodecParameters (Codecs/CriHca/CriHcaParameters.cs:3-15).
 * quality = CriHcaQuality (CriHcaQuality.cs:3-10): 0 NotSet, 1 Highest, 2 High, 3 Middle, 4 Low, 5 Lowest. */
typedef struct vgb_hca_params {
    int32_t quality, bitrate, limit_bitrate;
    int32_t channel_count, sample_rate, sample_count;
    int32_t looping, loop_start, loop_end;
} vgb_hca_params;

/* The HcaInfo fields the codec and the container writer need (Codecs/CriHca/HcaInfo.cs:5-48). */
typedef struct vgb_hca_info {
    int32_t channel_count, sample_rate, sample_count, frame_count, inserted_samples, appended_samples;
    int32_t header_size, frame_size, min_resolution, max_resolution, track_count, channel_config;
    int32_t total_band_count, base_band_count, stereo_band_count, hfr_band_count, bands_per_hfr_group, hfr_group_count;
    int32_t bitrate;
    int32_t looping, loop_start_frame, loop_end_frame, pre_loop_samples, post_loop_samples; /* HcaInfo.cs:29-33 */
    /* HcaInfo.UseAthCurve (HcaInfo.cs:38; set by HcaReader for version < 2.0 files without an ath chunk and for ath
     * type 1, HcaReader.cs:116,201): the decoder adds ScaleAthCurve(sample_rate) (CriHcaFrame.cs:60-84) to the noise level
     * when it derives resolutions (CriHcaPacking.cs:79-95).  vgb_hca_query / the encoder always write 0. */
    int32_t use_ath_curve;
} vgb_hca_info;

/* CriHcaEncoder.Initialize (CriHcaEncoder.cs:61-114): stream parameters for one configuration, so the caller can
 * allocate frame_count * frame_size bytes per stream.  Pure host integer logic. */
int32_t vgb_hca_query(const vgb_hca_params *params, vgb_hca_info *info_out);

/* Encode n_streams streams.  All streams of a call share channel_count / sample_rate / quality / bitrate /
 * limit_bitrate (one band layout); sample_count and the loop points may differ.  For a looping stream
 * params.sample_count is the PCM length the caller holds, info.sample_count becomes min(loop_end, sample_count)
 * (CriHcaEncoder.cs:89-99).  pcm is a flat table [n_streams * channel_count]
 * (stream-major) of channel pointers, frames_out[s] receives frame_count(s) * frame_size bytes, info_out is
 * [n_streams].  Errors: VGB_E_ARG (> 8 channels, mismatched streams, loop points outside 0 <= start < end, start < sample_count), VGB_E_DATA ("Bitrate is set too
 * low.", CriHcaEncoder.cs:469-472), VGB_E_STATE (bit writer overflow). */
int32_t vgb_hca_encode_batch(const int16_t *const *pcm, const vgb_hca_params *params, int32_t n_streams,
                             vgb_hca_info *info_out, uint8_t *const *frames_out, vgb_progress_cb cb, void *user);

/* Device-resident variant of vgb_hca_encode_batch (asynchronous on `cuda_stream`): channel c of stream s starts at
 * pcm_offset[s] + c * channel_stride[s] samples of d_pcm; its frames go to d_frames + frames_offset[s]
 * (info.frame_count * info.frame_size bytes, from vgb_hca_query).  The per-stream status of the encoder (the reference's
 * "Bitrate is set too low." ...) stays in the workspace: vgb_hca_encode_dev_status synchronises the stream and maps it.
 * d_pcm must be 2-byte and d_workspace 8-byte aligned (VGB_E_ARG otherwise); d_frames and the offsets may be odd. */
uint64_t vgb_hca_workspace_bytes(int32_t n_streams);
int32_t vgb_hca_encode_dev(const int16_t *d_pcm, const int64_t *pcm_offset, const int64_t *channel_stride, const vgb_hca_params *params,
                           int32_t n_streams, vgb_hca_info *info_out, uint8_t *d_frames, const int64_t *frames_offset,
                           void *d_workspace, uint64_t workspace_bytes, void *cuda_stream);
int32_t vgb_hca_encode_dev_status(const void *d_workspace, int32_t n_streams, void *cuda_stream);

/* Mdct.RunMdct(double[] input, double[] output) / RunImdct (Utilities/Mdct.cs:63-92 / :94-119) of the codec's instance
 * (128 points, CriHcaTables.MdctWindow, scale sqrt(2/128); CriHcaChannel.cs:19) for n_sequences independent sequences of
 * n_blocks blocks; every sequence starts from a fresh Mdct object's zero state.  in / out: [sequence][block][128] doubles
 * on the host.  Unit-parity taps: results are bit-identical to the reference's fp64 operation order (no FMA). */
int32_t vgb_mdct128_batch(const double *in, int32_t n_sequences, int32_t n_blocks, double *out);
int32_t vgb_imdct128_batch(const double *in, int32_t n_sequences, int32_t n_blocks, double *out);

/* CRI HCA decode: replaces CriHcaDecoder.Decode (Codecs/CriHca/CriHcaDecoder.cs:11-25) for a batch of streams.
 * info[s] is what the caller's container reader parsed (HcaReader -> HcaInfo); the codec reads channel_count,
 * frame_size, the band layout, track_count / channel_config (channel types), sample_count, frame_count and
 * inserted_samples.  All streams of a call share everything but the last three.  frames[s] = frame_count(s) *
 * frame_size bytes (the reference's byte[][] AudioData, concatenated); pcm_out is a flat table
 * [n_streams * channel_count] (stream-major) of buffers of sample_count(s) samples.  Frames are not CRC-checked
 * (CriHcaPacking.UnpackFrame does not check either).  Errors: VGB_E_DATA ("Invalid frame header" - sync word is not
 * 0xffff, CriHcaPacking.cs:73-77; or a scale-factor delta out of range, where the reference silently keeps decoding
 * with the previous frame's state). */
int32_t vgb_hca_decode_batch(const uint8_t *const *frames, const vgb_hca_info *info, int32_t n_streams,
                             int16_t *const *pcm_out);

/* Device-resident variant of vgb_hca_decode_batch (asynchronous on `cuda_stream`), with the same rules for info (at most
 * 65535 streams): the frames of stream s are frame_count * frame_size bytes at d_frames + frames_offset[s]; channel c of
 * its PCM is written to sample_count samples at d_pcm + pcm_offset[s] + c * channel_stride[s] (channel_stride >=
 * sample_count).  Samples no frame covers (sample_count > frame_count * 1024 - inserted_samples) are not written: clear
 * the buffer first for the reference's fresh short[].  The workspace holds the stream table, the status words, the parse
 * records and the seam addends; vgb_hca_decode_workspace_bytes sizes it from the same info.  The per-stream status of
 * the decoder stays in the workspace: vgb_hca_decode_dev_status synchronises the stream and maps it to VGB_E_DATA with
 * vgb_hca_decode_batch's messages.  d_pcm must be 2-byte aligned and d_workspace 8-byte aligned (the stream table's
 * int64 fields, the fp64 seam addends); VGB_E_ARG otherwise. */
uint64_t vgb_hca_decode_workspace_bytes(const vgb_hca_info *info, int32_t n_streams);
int32_t vgb_hca_decode_dev(const uint8_t *d_frames, const int64_t *frames_offset, const vgb_hca_info *info, int32_t n_streams,
                           int16_t *d_pcm, const int64_t *pcm_offset, const int64_t *channel_stride,
                           void *d_workspace, uint64_t workspace_bytes, void *cuda_stream);
int32_t vgb_hca_decode_dev_status(const void *d_workspace, int32_t n_streams, void *cuda_stream);


/* =====================================================================================================================
 * Containers either side of the codec path (SURVEY.md 8f rank 2-4): the WAVE front end, the DSP / ADX / HCA writers, the
 * DSP reader, CRI encryption, and the batch converter that replaces the CLI's file-level Parallel.ForEach.  All payload
 * movement (de-interleave, block / frame interleave, key streams, substitution + CRC) runs on the GPU; header fields are
 * host integer logic.  Sizes come first (vgb_*_file_size), the caller allocates, the call fills.
 * ===================================================================================================================== */

/* WaveStructure (Containers/Wave/WaveStructure.cs) + where the data chunk's payload sits in the file. */
typedef struct vgb_wave_info {
    int32_t channel_count, sample_rate, bits_per_sample, sample_count;
    int32_t looping, loop_start, loop_end, reserved;
    int64_t data_offset, data_size;
} vgb_wave_info;

/* RiffParser.ParseRiff (Utilities/Riff/RiffParser.cs:38-86) + WaveReader.ReadFile / ValidateWaveFile
 * (Containers/Wave/WaveReader.cs:13-51, :71-95) on a file image in host memory: chunk walk ("fmt ", "smpl", "data";
 * 2-byte alignment; a later chunk of the same id replaces an earlier one), validation in the reference's order with its
 * messages in vgb_last_error() (VGB_E_DATA = InvalidDataException), loop points from the first smpl loop, WithLoop's range
 * check (Formats/AudioFormatBaseBuilder.cs:23-50).  Host only. */
int32_t vgb_wave_parse(const uint8_t *file, int64_t length, vgb_wave_info *info_out);

/* data.Data.InterleavedByteToShort(channelCount) (WaveReader.cs:47, Interleave.cs:188-207) for a batch of parsed files:
 * pcm_out is a flat file-major table of channel rows (sample_count samples each).  8-bit files come out as PCM16 through
 * Pcm8Codec.Decode ((b - 0x80) << 8, Codecs/Pcm8/Pcm8Codec.cs:23), which is what every encoder asks AudioData for.  A
 * description that does not fit its image (data_offset + payload > lengths[i]) is VGB_E_ARG. */
int32_t vgb_wave_read_batch(const uint8_t *const *files, const int64_t *lengths, const vgb_wave_info *info, int32_t n_files,
                            int16_t *const *pcm_out);

/* What DspWriter reads from GcAdpcmFormat and DspConfiguration (Containers/Dsp/DspWriter.cs:17-36, DspConfiguration.cs):
 * sample_count / loop points are the format's; 0 in the three option fields selects the reference's defaults
 * (SamplesPerInterleave 0x3800, LoopPointAlignment 1, TrimFile true). */
typedef struct vgb_dsp_desc {
    int32_t channel_count, sample_rate, sample_count, looping, loop_start, loop_end;
    int32_t samples_per_interleave, loop_point_alignment, no_trim;
} vgb_dsp_desc;
int64_t vgb_dsp_file_size(const vgb_dsp_desc *desc); /* FileSize (:17); negative = VGB_E_* */

/* DspWriter.WriteStream (:42-99) for n_files files: 0x60-byte big-endian header per channel, then the payload (mono: the
 * channel; else Interleave(BytesPerInterleave, AudioDataSize)).  adpcm / coefs ([ch][16]) / gain / start_hist ([ch][2]) /
 * loop_context ([ch][3] = PredScale, Hist1, Hist2, e.g. from vgb_gcadpcm_seek_context_batch) are flat file-major tables
 * over all channels; gain, start_hist may be NULL (zeros), loop_context may be NULL when nothing loops.  adpcm[c] holds
 * SampleCountToByteCount(sample_count) bytes.  files_out[i] receives vgb_dsp_file_size bytes. */
int32_t vgb_dsp_write_batch(const vgb_dsp_desc *files, int32_t n_files, const uint8_t *const *adpcm, const int16_t *coefs,
                            const int16_t *gain, const int16_t *start_hist, const int16_t *loop_context, uint8_t *const *files_out);

#define VGB_DSP_MAX_CHANNELS 64
typedef struct vgb_dsp_info { /* DspStructure (Containers/Dsp/DspStructure.cs) */
    int32_t sample_count, nibble_count, sample_rate, looping, format, start_address, end_address, current_address;
    int32_t channel_count, frames_per_interleave, loop_start, loop_end;
    int16_t coefs[VGB_DSP_MAX_CHANNELS][16], gain[VGB_DSP_MAX_CHANNELS];
    int16_t start_context[VGB_DSP_MAX_CHANNELS][3], loop_context[VGB_DSP_MAX_CHANNELS][3];
} vgb_dsp_info;
/* DspReader.ReadHeader (Containers/Dsp/DspReader.cs:57-104), host only; VGB_E_DATA with the reference's messages. */
int32_t vgb_dsp_parse(const uint8_t *file, int64_t length, vgb_dsp_info *info_out);
/* DspReader.ReadData (:106-119): adpcm_out is a flat file-major table of channel rows, SampleCountToByteCount(sample_count)
 * bytes each; multi-channel payloads are de-interleaved on the device. */
int32_t vgb_dsp_read_batch(const uint8_t *const *files, const int64_t *lengths, const vgb_dsp_info *info, int32_t n_files,
                           uint8_t *const *adpcm_out);

/* What AdxWriter reads from CriAdxFormat and AdxConfiguration (Containers/Adx/AdxWriter.cs:18-55).  sample_count and the
 * loop points are the UNALIGNED values of the PCM (the format adds alignment_samples, CriAdxFormat.cs:16-18);
 * highpass_frequency is 500 for anything the encoder made (CriAdxFormat.cs:84). */
typedef struct vgb_adx_desc {
    int32_t channel_count, sample_rate, sample_count, looping, loop_start, loop_end, alignment_samples;
    int32_t frame_size, version, type, highpass_frequency, encryption_type, no_trim;
} vgb_adx_desc;
typedef struct vgb_adx_key { int32_t seed, mult, inc; } vgb_adx_key; /* CriAdxKey */
int32_t vgb_adx_key_from_code(uint64_t key_code, vgb_adx_key *key_out);       /* CriAdxKey(ulong), CriAdxKey.cs:18-24 */
int32_t vgb_adx_key_from_string(const char *key_string, vgb_adx_key *key_out); /* CriAdxKey(string), :26-41 (ASCII) */
int64_t vgb_adx_file_size(const vgb_adx_desc *desc);                           /* FileSize (:18) */
/* AdxWriter.WriteStream (:70-140): header, frame-interleaved audio (encrypted copy when key != NULL,
 * CriAdxEncryption.EncryptDecrypt), footer.  audio / audio_len / history are flat file-major tables over all channels
 * (channels of a file must have equal lengths); history may be NULL. */
int32_t vgb_adx_write_batch(const vgb_adx_desc *files, int32_t n_files, const uint8_t *const *audio, const int32_t *audio_len,
                            const int16_t *history, const vgb_adx_key *key, uint8_t *const *files_out);
/* CriAdxEncryption.EncryptDecrypt(byte[][] adpcm, key, encryptionType, frameSize) (CriAdxEncryption.cs:8-44) on the
 * channels of one file, in place; length must be a whole number of frames. */
int32_t vgb_adx_crypt_batch(uint8_t *const *audio, int32_t n_channels, int32_t length, const vgb_adx_key *key,
                            int32_t encryption_type, int32_t frame_size);

/* AdxStructure (Containers/Adx/AdxStructure.cs) as AdxReader.ReadHeader / ReadData (Containers/Adx/AdxReader.cs:14-124)
 * leave it, plus where the audio sits: audio_size bytes at audio_offset = header_size + 4, frame-interleaved over the
 * channels.  history[c] is the header's pair of channel c (version >= 4 only), for reporting: ToPcm16 never uses it. */
#define VGB_ADX_MAX_CHANNELS 255
typedef struct vgb_adx_file_info {
    int32_t header_size, type, frame_size, bit_depth, channel_count, sample_rate, sample_count, highpass_frequency;
    int32_t version, revision, inserted_samples, loop_count, looping, loop_type;
    int32_t loop_start_sample, loop_start_byte, loop_end_sample, loop_end_byte;
    int32_t samples_per_frame, reserved;
    int64_t audio_offset, audio_size;
    int16_t history[VGB_ADX_MAX_CHANNELS][2];
} vgb_adx_file_info;
/* AdxReader.ReadFile's header and data reads on a file image, host only: big-endian, HeaderSize and InsertedSamples
 * signed 16-bit; version >= 4 skips 4 bytes and reads two shorts per channel (4 more bytes skipped for mono); nothing
 * past the history when Position + 24 > HeaderSize; the loop fields only when LoopCount > 0.  VGB_E_DATA, naming the
 * file, wherever the reference throws: the signature ("File doesn't have ADX signature (0x80 0x00)"), a read past the
 * image, a frame size or channel count of 0 (division by zero), a negative header offset or audio length, and an audio
 * region shorter than AudioDataLength (Interleave.cs:118-128, "Specified length is greater than the number of bytes
 * remaining in the Stream").  On purpose, where the reference would not throw but no decode can run: frame sizes 1 and 2
 * (no whole sample per frame) and InsertedSamples <= -samples_per_frame (ToPcm16 would index before the audio). */
int32_t vgb_adx_parse(const uint8_t *file, int64_t length, vgb_adx_file_info *info_out);

/* HcaReader.ReadHcaHeader (Containers/Hca/HcaReader.cs:59-121) on a file image, host only: the chunk walk over
 * header_size bytes ("fmt", "comp", "dec", "loop", "ath", "ciph", "rva", "vbr", "comm", "pad"; every id byte masked with
 * 0x7f, so the ids of encrypted files read the same; a later chunk overwrites what an earlier one set), UseAthCurve for
 * an "ath" chunk of type 1 and for version < 0x0200 files without one, track_count at least 1, HcaInfo.CalculateHfrValues
 * when bands_per_hfr_group > 0, sample_count = min(sample_count, LoopEndSample) for looping files.  The "ciph" value goes
 * to *encryption_type_out (0 without the chunk; may be NULL).  VGB_E_DATA for a bad signature, an unknown chunk
 * ("Chunk X is not supported."), a read past `length`, and an image shorter than header_size + frame_count * frame_size
 * (where ReadHcaData, :123-138, would hand short frames to the decoder).  CRCs are not checked, as in the reference. */
int32_t vgb_hca_parse(const uint8_t *file, int64_t length, vgb_hca_info *info_out, int32_t *encryption_type_out);
/* CriHcaKey (Codecs/CriHca/CriHcaKey.cs): key_type 0, 1 or 56 (key_code used by 56 only); 256-byte substitution tables. */
int32_t vgb_hca_key_tables(int32_t key_type, uint64_t key_code, uint8_t *decrypt_out, uint8_t *encrypt_out);
/* CriHcaEncryption.Crypt (CriHcaEncryption.cs:12-33) for a batch of streams, in place: substitution over the first
 * frame_size-2 bytes of every frame, CRC-16 recomputed.  frames[s] = frame_count[s] * frame_size bytes. */
int32_t vgb_hca_crypt_batch(uint8_t *const *frames, const int32_t *frame_count, int32_t n_streams, int32_t frame_size,
                            int32_t key_type, uint64_t key_code, int32_t decrypt);
/* HcaWriter.WriteStream (Containers/Hca/HcaWriter.cs:37-178): chunked header ("HCA", "fmt", "comp", "loop", "ciph", "rva",
 * "comm" / "pad"; ids masked with 0x80 when a key is given), header CRC, frames (encrypted when key_type >= 0; -1 = no key).
 * comment / volume may be NULL (none / 1.0).  files_out[i] receives header_size + frame_count * frame_size bytes. */
int32_t vgb_hca_write_batch(const vgb_hca_info *info, int32_t n_files, const uint8_t *const *frames, int32_t key_type,
                            uint64_t key_code, const char *const *comment, const float *volume, uint8_t *const *files_out);

/* Batch converter: replaces BatchConvert's Parallel.ForEach over files (src/VGAudio.Cli/Batch.cs:24-46, each body =
 * Convert.ConvertFile: WaveReader -> GetFormat<T> (encode) -> writer) for WAVE inputs held in host memory.  Files are
 * coalesced into GPU batches; per batch: one H2D of the raw data chunks, de-interleave -> encode -> (loop context) ->
 * file assembly on the device, one D2H of the finished files; neighbouring batches overlap copies and kernels.
 * Zero-initialised options = the reference's defaults. */
#define VGB_CONTAINER_DSP 1
#define VGB_CONTAINER_ADX 2
#define VGB_CONTAINER_HCA 3
typedef struct vgb_convert_options {
    int32_t out_type;                   /* VGB_CONTAINER_* */
    int32_t no_trim;                    /* Configuration.TrimFile = !no_trim */
    int32_t dsp_samples_per_interleave, dsp_loop_point_alignment;
    int32_t adx_version, adx_frame_size, adx_type, adx_filter_plus1; /* 0 = 4, 18, Linear, filter 2 (AdxConfiguration.cs) */
    int32_t adx_encryption_type, adx_has_key, adx_key_seed, adx_key_mult, adx_key_inc;
    int32_t hca_quality, hca_bitrate, hca_limit_bitrate;             /* CriHcaParameters */
    int32_t hca_key_type;               /* -1 = no key; NOTE: 0 is a key type, set -1 explicitly */
    int32_t reserved;
    uint64_t hca_key_code;
    int64_t group_bytes;                /* input bytes per GPU batch; 0 = an eighth of the job, 64..512 MiB */
} vgb_convert_options;
/* Pass files_out == NULL for the sizing pass: out_sizes[i] = size of output i (0 for a file that failed), status_out[i]
 * (may be NULL) = VGB_OK or the error of file i - a bad file does not stop the batch (Batch.cs:39-43).  The sizing pass
 * runs on the host only and needs no device.  The second pass fills files_out[i] for every file whose status is VGB_OK.
 * cb receives the number of files finished (positive deltas summing to the good files).  With several devices bound
 * (vgb_init_devices) and at least two good files, the second pass is sharded: files weigh sample_count * channel_count
 * + 1024, every device converts its share in groups of its own (group_bytes = 0: an eighth of its share's input, 64..512
 * MiB), and an error of a device's share fails the call with " (device N)" appended to its message. */
int32_t vgb_convert_wave_batch(const uint8_t *const *files, const int64_t *lengths, int32_t n_files, const vgb_convert_options *options,
                               int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out, vgb_progress_cb cb, void *user);
/* The decode direction of the batch job: .dsp file images in, 16-bit WAVE file images out - DspReader (Containers/Dsp/DspReader.cs:15-127)
 * -> GcAdpcmFormat.ToPcm16 (GcAdpcmFormat.cs:42-54, from the header's coefficients and start history) -> WaveWriter
 * (Containers/Wave/WaveWriter.cs:52-132: RIFF / fmt (extensible above two channels) / smpl when looping / data).  Same two-pass
 * protocol, per-file status and sharding over several devices as vgb_convert_wave_batch (files weigh their decoded
 * samples).  A frame header that selects a predictor outside 0..7 fails the whole call (VGB_E_DATA). */
int32_t vgb_convert_dsp_to_wave_batch(const uint8_t *const *files, const int64_t *lengths, int32_t n_files, int64_t *out_sizes,
                                      uint8_t *const *files_out, int32_t *status_out);
/* The decode direction of the batch job for .hca file images: HcaReader.ReadFile -> ToAudioStream (Containers/Hca/HcaReader.cs:20-49)
 * -> CriHcaFormat.ToPcm16 (Formats/CriHca/CriHcaFormat.cs:25-32) -> WaveWriter, with vgb_convert_dsp_to_wave_batch's
 * two-pass protocol and sharding (files weigh frame_count * channel_count).  Decryption follows HcaReader.FindKey
 * (:238-252): "ciph" 1 uses the built-in type-1 table, 56 the table of *key_code, any other value none.  The reference's
 * list of known keys is not carried: a type-56 file without key_code fails with "Cannot find key to decrypt HCA file.",
 * and the given code is not tested against the frames.  Per file, on the device: the frames are copied in, decrypted in
 * place, decoded (vgb_hca_decode_dev, one launch per group of files that share a codec configuration) and joined behind
 * the WAVE header (smpl when looping, extensible fmt above two channels).
 * Per-file errors, each failing that file only (Batch.cs:39-43): a parse error, more than 8 channels or a layout the
 * decoder cannot take, sample_count < 0, 2 GiB of PCM or more, loop points WithLoop rejects (AudioFormatBaseBuilder.cs:23-50),
 * a missing key - all known in the sizing pass - and a decoder status word on the device ("Invalid frame header" ...),
 * known only in the fill pass: such a file gets its status_out entry, out_sizes[i] = 0 and its buffer is not written.
 * Unlike the .dsp direction, where one bad predictor fails the call, a bad frame fails its file alone: a wrong key shows
 * up exactly this way, and one such file must not cost the batch.  With status_out NULL, such a file fails the call
 * (VGB_E_DATA) after every other file has been written. */
int32_t vgb_convert_hca_to_wave_batch(const uint8_t *const *files, const int64_t *lengths, int32_t n_files,
                                      const uint64_t *key_code, int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out);
/* The decode direction of the batch job for .adx file images: AdxReader -> ToAudioStream (Containers/Adx/AdxReader.cs:14-58)
 * -> CriAdxFormat.ToPcm16 (Formats/CriAdx/CriAdxFormat.cs:35-55) -> WaveWriter, with vgb_convert_hca_to_wave_batch's
 * two-pass protocol, per-file status and sharding (files weigh frames * channels).  Per group of files, on the device:
 * the audio regions are copied in, de-interleaved into channel rows, decrypted in place where needed, decoded by the
 * time-parallel decoder (vgb_adx_decode_dev) and joined behind the WAVE header.  The reference's rules kept:
 * ToPcm16 decodes sample_count - inserted_samples samples with padding = inserted_samples, the header's frame size,
 * high-pass, type and version and history 0 (the header's history is never handed to the decoder); the WAVE loop points
 * are the loop samples minus inserted_samples, checked by WithLoop's rules (AudioFormatBaseBuilder.cs:23-50).
 * Keys (*key from vgb_adx_key_from_code / _from_string, or NULL): revision 8 or 9 is decrypted with *key, and fails with
 * "encrypted ADX file (type N) and no key" without one; any other revision is not decrypted.  Two differences on
 * purpose: AdxReader.EncryptionKey would also "decrypt" files of other revisions, but a directory mixes files, so the key
 * goes to types 8 and 9 only; and the reference's built-in key list (CriAdxEncryption.FindKey) is not carried - there is
 * no key search.  A sample rate <= 0 decodes as in the reference (CalculateCoefficients' double math; a rate of 0 gives
 * NaN, which C#'s (int) makes int.MinValue and (short) 0).  Per-file errors, each failing that file only: a parse error, a missing key, bad loop points, a negative
 * unaligned sample count, decoded frames past a channel's audio (IndexOutOfRangeException), 2 GiB of PCM or more, too many
 * channels for the WAVE join - all known in the sizing pass - and a Fixed-type frame with a filter 4..7, found on the
 * device in the fill pass: that file gets its status_out entry, out_sizes[i] = 0 and its buffer is not written.  With
 * status_out NULL such a file fails the call (VGB_E_DATA) after every other file has been written. */
int32_t vgb_convert_adx_to_wave_batch(const uint8_t *const *files, const int64_t *lengths, int32_t n_files, const vgb_adx_key *key,
                                      int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out);
/* Transcoding in the batch job: .dsp, .adx and .hca file images in, another of the three out (Convert.ConvertFile with a
 * coded source: the source's reader, a fresh configuration from the options, source.ToPcm16() -> EncodeFromPcm16).
 * in_type[i] (VGB_CONTAINER_*) names file i's codec: a .dsp file has no signature.  options->out_type, its options and
 * its key describe the output exactly as for vgb_convert_wave_batch; options->group_bytes counts DECODED PCM bytes per
 * GPU batch (0: an eighth of the job's PCM, 64..512 MiB; a batch holds at most 4096 files).  The sources are read as by vgb_convert_{dsp,adx,hca}_to_wave_batch:
 * the PCM, loop points and rate their ToPcm16 yields (.adx: sample_count - inserted_samples samples, loop points shifted;
 * .hca: trimmed at the loop end; .dsp: from the header's start history), and their keys: *in_adx_key decrypts revision 8
 * and 9 .adx files, *in_hca_key_code "ciph" 56 .hca files, "ciph" 1 uses the built-in table; a keyed source without its
 * key fails alone, keys are never applied to other revisions and there is no key search.  No PCM leaves the device:
 * per batch one H2D of the coded regions, the source's decode straight into the encoder's channel rows, encode and file
 * assembly, one D2H of the finished files.  Same two-pass protocol, per-file status, progress and sharding (files weigh
 * sample_count * channel_count + 1024) as vgb_convert_wave_batch.
 * Per-file errors of the sizing pass, each failing that file only: in_type not DSP / ADX / HCA, or equal to out_type
 * (a rewrite in the source's own codec is not performed), the source's parse and planning errors (as its -> WAVE
 * converter, without the WAVE writer's limits), and the target's planning errors (as vgb_convert_wave_batch).
 * In the fill pass, an ADX frame with a filter the reference cannot index or an HCA frame the decoder refuses fails that
 * file alone (status_out entry, out_sizes[i] = 0, buffer not written; without status_out the call fails with VGB_E_DATA
 * after the other files are written), a GC-ADPCM predictor outside 0..7 fails the call (VGB_E_DATA). */
int32_t vgb_transcode_batch(const uint8_t *const *files, const int64_t *lengths, const int32_t *in_type, int32_t n_files,
                            const vgb_convert_options *options, const vgb_adx_key *in_adx_key, const uint64_t *in_hca_key_code,
                            int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out, vgb_progress_cb cb, void *user);
/* Measurement tap: device time of the most recent vgb_convert_wave_batch summed over its (first 32) batches per device,
 * over every device that converted part of it, out[0..3] = WAVE split, encode, loop-context decode, file assembly (ms,
 * CUDA events on the kernel streams); returns the number of batches timed on all devices together. */
int32_t vgb_convert_debug_stage_ms(float *out, int32_t n);

#ifdef __cplusplus
}
#endif
#endif /* VGAUDIO_B200_H */
