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
 * and debug taps use); every host-pointer codec *_batch call and every batch converter (vgb_convert_wave_batch,
 * vgb_convert_{dsp,hca,adx,nw,idsp_hps}_to_wave_batch, vgb_transcode_batch, vgb_transcode_nw_batch, vgb_transcode_from_nw_batch) are then sharded over all bound devices by greedy
 * longest-first bin packing of the units' sample or frame counts - one worker thread and one H2D / kernel / D2H pipeline
 * per device, each over its own PCIe link, results written straight into the caller's arrays (no collective: host data
 * reaches a GPU fastest over that GPU's own link).  The single-shot container calls (vgb_*_read_batch, vgb_*_write_batch, vgb_*_crypt_batch) stay on the primary.
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
/* Bookkeeping of the most recent ADX encode launch on this thread's context (vgb_adx_encode_batch: its last channel group;
 * vgb_adx_encode_dev: the call), whose 18-byte channels without padding are cut into segments encoded concurrently and
 * spliced at the boundaries (adx.cu): out[0] segments per channel, out[1] the shortest segment in frames, out[2] frames
 * re-encoded by the boundary run-ons, out[3] frames re-encoded by the serial cascade (boundaries whose run-on did not
 * lock inside its segment), out[4] boundaries the cascade repaired.  A single-segment launch leaves out[2..4] zero.
 * n = how many words to fill (up to 5).  Synchronises the device.  The words live in the workspace of that launch: after
 * a vgb_adx_encode_dev the caller's workspace must still be allocated (and not yet reused) when this is called.
 * VGB_ADX_SEGMENTS / VGB_ADX_MIN_SEG_FRAMES in the environment force the segment count and the shortest segment. */
int32_t vgb_adx_debug_encode_stats(uint64_t *out, int32_t n);

/* CriAdxCodec.Decode(byte[] adpcm, int sampleCount, CriAdxParameters config) (CriAdxCodec.cs:9-54).
 * n_bytes[c] = length of adpcm[c]; pcm_out[c] receives sample_count[c] samples.
 * VGB_E_DATA for the lowest channel with a frame that yields a sample and whose filter number coefs[filterNum] cannot
 * index (IndexOutOfRangeException, :12,26): a Fixed-type filter outside 0..3 (CriAdxCodec.Coefs, :186-191) or a Linear /
 * Exponential filter other than 0 (a one-row table).  A frame that yields no sample (the head frame when sample_count
 * <= padding % samples per frame) is not checked, as in the reference. */
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
 * vgb_adx_decode_dev_status synchronises the stream and returns VGB_E_DATA for the lowest channel whose frame selects a
 * filter the reference cannot index (Fixed 4..7, other types 1..7), with vgb_adx_decode_batch's message for its kind. */
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

/* BxstmStructure (Containers/NintendoWare/BxstmStructure.cs) as BrstmReader.ReadFile (BrstmReader.cs:12-185) or
 * BCFstmReader.ReadFile (BCFstmReader.cs:14-288) leaves it, reduced to what decoding needs: StreamInfo's codec
 * (NwCodec.cs: 0 PCM8, 1 PCM16, 2 GC-ADPCM), looping, channel count, rate, loop start and sample count, the interleave
 * size and the byte order of the file (BRSTM: always big-endian), the region Stream.DeInterleave reads (audio_length
 * bytes at audio_offset, each reader's ReadDataBlock) and its per-channel output size (Common.SamplesToBytes), and per
 * channel with GC-ADPCM info (Structures/ChannelInfo.cs) the coefficients, gain (BRSTM only) and start / loop contexts
 * (PredScale, Hist1, Hist2).  version is NwVersion.Version; seek_table: 0 none read, 1 read (BRSTM: the standard size),
 * 2 the shortened BRSTM size; region_count / track_count: entries read from REGN / the track info.  The unaligned loop
 * fields (version-dependent, Common.cs:118-157) are read and reported but, as in the reference, not used. */
#define VGB_NW_MAX_CHANNELS 255
typedef struct vgb_nw_info {
    int32_t codec, looping, channel_count, sample_rate, loop_start, sample_count;
    int32_t interleave_size, big_endian;
    uint32_t version;
    int32_t seek_table, region_count, track_count, adpcm_channel_count, samples_per_seek_entry;
    int32_t loop_start_unaligned, loop_end_unaligned, output_size, reserved;
    int64_t audio_offset, audio_length;
    int16_t coefs[VGB_NW_MAX_CHANNELS][16];
    int16_t gain[VGB_NW_MAX_CHANNELS];
    int16_t start_context[VGB_NW_MAX_CHANNELS][3], loop_context[VGB_NW_MAX_CHANNELS][3];
} vgb_nw_info;
/* The two readers on a file image, host only.  Every read and check runs in the reference's order and fails with
 * VGB_E_DATA and the reference's message: the signature ("File has no RSTM header", "File has no CSTM or FSTM header")
 * and byte-order mark, "Actual file length is less than stated length", each block's id and size against the main
 * header (HEAD / ADPC / DATA, INFO / SEEK / REGN / DATA), "Could not read stream/track/channel info.", a read past the
 * image, a negative position, the ADPC / SEEK seek table (BRSTM: the standard and shortened sizes are read, another size
 * is skipped; a zero samples-per-entry divides by zero), the REGN regions (a REGN block in a version without region
 * info dereferences null), the track info, and Stream.DeInterleave's checks (Utilities/Interleave.cs:118-133: the
 * region stays in the image and splits evenly over the channels).  Refused on purpose, where the reference would fail
 * later or read something these readers do not carry: codec 3 (IMA; ToAudioStream returns null) and any codec above
 * it, a GC-ADPCM stream with fewer channel infos than channels, and CWAV / FWAV / CSTP / FSTP images, wave info blocks
 * and prefetch / wave data blocks (BCFstmReader accepts them; "... are not read" - vgb_nw_file_parse with a wave or
 * prefetch type reads them).  vgb_bcfstm_parse accepts CSTM and FSTM alike. */
int32_t vgb_brstm_parse(const uint8_t *file, int64_t length, vgb_nw_info *info_out);
int32_t vgb_bcfstm_parse(const uint8_t *file, int64_t length, vgb_nw_info *info_out);
/* Every NintendoWare reader behind one call, host only; in_type (VGB_CONTAINER_*) names the reader as the file extension
 * does in the reference.  BRSTM, BCSTM and BFSTM behave exactly as vgb_brstm_parse / vgb_bcfstm_parse, through the same
 * code.  BCWAV, BFWAV, BCSTP and BFSTP run the whole BCFstmReader (BCFstmReader.cs:14-288) on any of its six magics:
 * the wave info block (StreamInfo.ReadBfwav: the unaligned loop start from BFWAV 0.1.2 / BCWAV 2.1.1, the channel count
 * peeked from the channel reference table; ChannelInfo.ReadBfstm with the wave channels' audio offsets, GC-ADPCM info
 * without gain), the wave data block and the prefetch data block.  BRWAV runs BrwavReader (BrwavReader.cs,
 * RwavWaveInfo.cs, RwavChannelInfo.cs), big-endian; as in the reference its loop start and sample count go through
 * NibbleToSample whatever the codec, and every channel's coefficients, gain and contexts are read at its ADPCM info
 * offset whatever the codec.  info_out describes what Common.ToAudioStream builds:
 *   - a wave file (a wave data block, or BRWAV): each channel is ReadBytes(SamplesToBytes(sample_count)) at its own
 *     offset behind the DATA header, so a channel's bytes may be shorter than output_size (or empty) at the image's end;
 *     interleave_size = 0; channel_offsets_out[c] (c < channel_count) is the absolute file offset of channel c's bytes;
 *     audio_offset / audio_length span the channels' bytes that lie in the image (0 / 0 when none do);
 *   - a prefetch file (a PDAT block): the region and geometry of the first entry, read as a stream by Stream.DeInterleave
 *     (PDAT size bytes, rows of that size); sample_count = BytesToSamples(size / channel_count) and looping = 0, as
 *     ToAudioStream sets them;
 *   - a stream: as vgb_bcfstm_parse.
 * channel_offsets_out (VGB_NW_MAX_CHANNELS entries, or NULL) is -1 wherever no wave channel is described.  The reference's
 * failures, with its messages: a channel position before the image, a channel reference that is not a wave channel
 * (WaveAudioOffsets[i] is out of range), no channel info at all (a null reference), a wave info block with a stream
 * data block (no audio reference), a PDAT count of 0 (PrefetchData[0] is out of range), a prefetch file of 0 channels
 * (a divide by zero), a negative wave channel length (new byte[n]).  Refused on purpose: codec 3 (IMA) and above, as
 * for the streams, and a wave info block of more than 255 (or fewer than 0) channels.  An in_type that names no
 * NintendoWare reader is VGB_E_ARG. */
int32_t vgb_nw_file_parse(const uint8_t *file, int64_t length, int32_t in_type, vgb_nw_info *info_out, int64_t *channel_offsets_out);

/* IdspStructure (Containers/Idsp/IdspStructure.cs) as IdspReader.ReadFile (Containers/Idsp/IdspReader.cs:13-112) leaves
 * it, big-endian: the main header's fields, looping (set when any channel's flag is 1), and per channel its header
 * (IdspChannelInfo: sample count, nibble count, rate, looping flag, start / end / current address, coefficients, gain,
 * start and loop contexts as PredScale, Hist1, Hist2).  ReadIdspData's Stream.DeInterleave reads audio_length =
 * channel_count * audio_data_length bytes (C# int) at audio_offset = audio_data_offset, in blocks of `interleave`
 * (interleave_size, or audio_data_length when that is 0), into rows of output_size = SampleCountToByteCount(sample_count)
 * bytes: a shorter last block, rows zero-filled or truncated, nothing copied when interleave or the per-channel length
 * is <= 0. */
typedef struct vgb_idsp_info {
    int32_t channel_count, sample_rate, sample_count, loop_start, loop_end, interleave_size;
    int32_t header_size, channel_info_size, audio_data_offset, audio_data_length;
    int32_t looping, interleave, output_size, reserved;
    int64_t audio_offset, audio_length;
    int32_t ch_sample_count[VGB_NW_MAX_CHANNELS], ch_nibble_count[VGB_NW_MAX_CHANNELS], ch_sample_rate[VGB_NW_MAX_CHANNELS];
    int32_t ch_looping[VGB_NW_MAX_CHANNELS], start_address[VGB_NW_MAX_CHANNELS], end_address[VGB_NW_MAX_CHANNELS];
    int32_t current_address[VGB_NW_MAX_CHANNELS];
    int16_t coefs[VGB_NW_MAX_CHANNELS][16];
    int16_t gain[VGB_NW_MAX_CHANNELS];
    int16_t start_context[VGB_NW_MAX_CHANNELS][3], loop_context[VGB_NW_MAX_CHANNELS][3];
} vgb_idsp_info;
/* IdspReader on a file image, host only.  Every read and check runs in the reference's order and fails with VGB_E_DATA
 * and the reference's message: "File has no IDSP header", a read past the image, a negative channel-info position
 * (HeaderSize + i * ChannelInfoSize), and Stream.DeInterleave's checks (Utilities/Interleave.cs:118-133: the region stays
 * in the image, and its length divides evenly by the channel count - zero channels divide by zero, "Attempted to divide
 * by zero."; a negative output size overflows).  Refused on purpose: a channel count above VGB_NW_MAX_CHANNELS (255, the
 * writers' limit) or below 0, right after the main header ("... channels (this reader takes 0..255)"). */
int32_t vgb_idsp_parse(const uint8_t *file, int64_t length, vgb_idsp_info *info_out);

/* HpsStructure (Containers/Hps/HpsStructure.cs) as HpsReader.ReadFile (Containers/Hps/HpsReader.cs:14-163) leaves it,
 * big-endian: rate, channel count, per channel (HpsChannelInfo) the max block size, end address, coefficients, gain and
 * start context; sample_count = NibbleToSample(EndAddress) + 1 of channel 0; looping, loop_start and the loop contexts
 * from VerifyData; the block chain's length and where it starts (first_block = GetNextMultiple(Max(0x80, position after
 * the header), 0x20)); loop_block = the index of the loop block, or -1.  channel_audio_bytes[c] is the length of the
 * channel's concatenated block pieces (ToAudioStream's Sum; INT64 so an overflowing sum can be seen). */
typedef struct vgb_hps_info {
    int32_t sample_rate, channel_count, sample_count, looping, loop_start, block_count;
    int32_t first_block, loop_block;
    int32_t max_block_size[VGB_NW_MAX_CHANNELS], end_address[VGB_NW_MAX_CHANNELS];
    int64_t channel_audio_bytes[VGB_NW_MAX_CHANNELS];
    int16_t coefs[VGB_NW_MAX_CHANNELS][16];
    int16_t gain[VGB_NW_MAX_CHANNELS];
    int16_t start_context[VGB_NW_MAX_CHANNELS][3], loop_context[VGB_NW_MAX_CHANNELS][3];
} vgb_hps_info;
/* One block of the chain (HpsBlock.cs): where it sits, its Size, FinalNibble and NextOffset.  Channel c's piece of the
 * block is ReadBytes(AudioSizeBytes = (FinalNibble + 1) / 2 rounded up) at the block's audio start (its header, 12 + 8 *
 * channel_count bytes, rounded up to a multiple of 0x20) + Size / ChannelCount * c. */
typedef struct vgb_hps_block {
    int32_t offset, size, final_nibble, next_offset;
} vgb_hps_block;
/* HpsReader on a file image, host only: the header, the chain walk `while (nextBlock > currentBlock)` and VerifyData.
 * Every read and check runs in the reference's order and fails with VGB_E_DATA and the reference's message: "File has no
 * HALPST header", a read past the image, a negative position (audio start + Size / ChannelCount * c), a negative
 * AudioSizeBytes ("Non-negative number required."), "Channels have differing sample counts".  ReadBytes at or past the
 * end of the image returns a short or empty piece, as in the reference.  Zero or fewer channels end in VerifyData's
 * First() on an empty list ("Sequence contains no elements.").  Refused on purpose: a channel count above
 * VGB_NW_MAX_CHANNELS (255, the writers' limit), right after the header.  info_out->block_count is always set on
 * success; blocks_out (may be NULL) receives the first min(block_count, block_capacity) blocks. */
int32_t vgb_hps_parse(const uint8_t *file, int64_t length, vgb_hps_info *info_out, vgb_hps_block *blocks_out, int32_t block_capacity);

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
/* NintendoWare streams (BrstmWriter, BCFstmWriter with BxstmConfiguration's defaults: interleave 0x2000 bytes, a seek
 * entry every 0x2000 bytes' worth of samples, BRSTM standard track and seek-table types, BCSTM version 2.1, BFSTM
 * version 0.3, seek table and loop context recalculated).  vgb_convert_wave_batch writes them; vgb_transcode_batch does
 * not take them as a target; vgb_transcode_nw_batch writes them from .adx, .hca and (PCM16 / PCM8 only) .dsp sources;
 * vgb_convert_nw_to_wave_batch reads them.  A looping GC-ADPCM file whose loop start is not
 * a multiple of the loop point alignment goes through GcAdpcmFormat.WithAlignment as in the reference: the loop moves
 * to the next multiple and the tail behind the kept frames is re-encoded on the device. */
#define VGB_CONTAINER_BRSTM 4
#define VGB_CONTAINER_BCSTM 5
#define VGB_CONTAINER_BFSTM 6
/* IDSP (IdspWriter with IdspConfiguration's default block size of 16 bytes: the loop start moves to a multiple of 28
 * samples, and no_trim maps to TrimFile as for .dsp) and HPS (HpsWriter: blocks of at most 0x10000 bytes, the loop start
 * moves to a multiple of one block's samples per channel), both GC-ADPCM only.  vgb_convert_wave_batch writes them;
 * vgb_transcode_batch does not take them as a target; vgb_transcode_nw_batch writes them from .adx and .hca sources;
 * the nw_* options are ignored.  Per-file refusals besides the
 * usual ones (no samples, loop points GcAdpcmAlignment refuses, 2 GiB of output, more than 255 channels - this
 * converter's limit): an HPS file with 3, 7, 11 ... channels, whose block headers HpsWriter writes 0x20 bytes past the
 * block map's offsets; and an HPS file whose loop moved and that has a block starting more than one sample behind the
 * input's last sample, where HpsWriter reads the block's history past the unaligned decode (IndexOutOfRangeException). */
#define VGB_CONTAINER_IDSP 7
#define VGB_CONTAINER_HPS 8
/* NintendoWare wave files and prefetch streams, named by the reader the reference picks for the file extension
 * (src/VGAudio.Cli/ContainerTypes.cs).  They are read only: vgb_nw_file_parse and vgb_convert_nw_to_wave_batch take them;
 * vgb_convert_wave_batch does not take them as a target and vgb_transcode_batch not as a source (the reference has no
 * writer for them).  BCFstmReader accepts any of its six magics under any of the four BCFstmReader types. */
#define VGB_CONTAINER_BRWAV 9    /* BrwavReader: .brwav .rwav */
#define VGB_CONTAINER_BCWAV 10   /* BCFstmReader: .bcwav .cwav .bms */
#define VGB_CONTAINER_BFWAV 11   /* BCFstmReader: .bfwav */
#define VGB_CONTAINER_BCSTP 12   /* BCFstmReader: .bcstp */
#define VGB_CONTAINER_BFSTP 13   /* BCFstmReader: .bfstp */
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
    /* NintendoWare targets (BxstmConfiguration); zero selects the reference's default */
    int32_t nw_codec_plus1;             /* 0 = GC-ADPCM; else NwCodec + 1: 1 = PCM8, 2 = PCM16, 3 = GC-ADPCM */
    int32_t nw_endianness;              /* 0 = the target's (BCSTM little, BFSTM big), 1 = little, 2 = big; BRSTM is always big */
    int32_t nw_loop_point_alignment;    /* 0 = BytesToSamples(0x2000, codec) (14336 for GC-ADPCM) */
    int32_t nw_pad;
    /* AudioData.SetLoop on every source before any encode or write (the CLI's -l / --no-loop, Convert.cs:82-90):
     * loop_mode 0 keeps each source's loop; VGB_LOOP_SET loops every file over [loop_start, loop_end); VGB_LOOP_CLEAR
     * makes every file non-looping.  The source format's WithLoop rules decide per file (see vgb_convert_to_wave_batch).
 * Any other loop_mode fails the whole call with VGB_E_ARG before a file is read, in every call that takes options. */
    int32_t loop_mode, loop_start, loop_end, loop_pad;
} vgb_convert_options;
#define VGB_LOOP_SET   1
#define VGB_LOOP_CLEAR 2
/* Pass files_out == NULL for the sizing pass: out_sizes[i] = size of output i (0 for a file that failed), status_out[i]
 * (may be NULL) = VGB_OK or the error of file i - a bad file does not stop the batch (Batch.cs:39-43).  The sizing pass
 * runs on the host only and needs no device.  The second pass fills files_out[i] for every file whose status is VGB_OK.
 * cb receives the number of files finished (positive deltas summing to the good files).  With several devices bound
 * (vgb_init_devices) and at least two good files, the second pass is sharded: files weigh sample_count * channel_count
 * + 1024, every device converts its share in groups of its own (group_bytes = 0: an eighth of its share's input, 64..512
 * MiB), and an error of a device's share fails the call with " (device N)" appended to its message.  loop_mode sets or
 * clears every WAVE file's loop (its smpl loop otherwise) before the encode, with the rules of vgb_convert_to_wave_batch;
 * a file whose points WithLoop refuses fails alone, and the targets' own refusals then apply to the new loop (an empty
 * loop is refused where the loop start must move, and by the .hca encoder). */
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
 * and the given code is not tested against the frames (HcaReader's EncryptionKey ?? FindKey: a given key wins untested).
 * vgb_hca_find_keys runs FindKey over a caller's list of codes; convert each found key's files with it.  Per file, on the device: the frames are copied in, decrypted in
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
/* HcaReader.FindKey for type-56 files (Containers/Hca/HcaReader.cs:32, 238-252) over the caller's key codes in list
 * order: CriHcaEncryption.FindKey / TestKey (Codecs/CriHca/CriHcaEncryption.cs:34-87).  For each file whose "ciph" is
 * 56: the window is the first frame whose encrypted bytes [2, FrameSize - 2) are not all zero (frame 0 if none) and up to
 * nine frames after it; a key passes when every window frame, decrypted by CryptFrame (table substitution of bytes
 * [0, FrameSize - 2), then their CRC-16 in the last two bytes), unpacks with UnpackingWasSuccessful true
 * (CriHcaPacking.cs:10-229: 16 <= Remaining <= 128, or FrameEmpty, or noise level 0 and Remaining >= 16).  Codes go
 * through CriHcaKey(ulong) (vgb_hca_key_tables), which reads bytes 0..6 of code - 1, so codes equal there are one key;
 * duplicates are legal and the first one wins.  Runs on the device, one file per CTA and one key per lane.
 * key_index_out[i] / file_status_out[i]:
 *   - VGB_OK and the index of the first code FindKey accepts;
 *   - VGB_E_DATA, -1: the first key that passes the window frames before frame j reaches a bad sync word there (an
 *     InvalidDataException("Invalid frame header") out of FindKey: every type-56 table keeps 0x00 and 0xFF, so the sync
 *     word decrypts to 0xFFFF exactly when the raw one is 0xFFFF);
 *   - VGB_HCA_KEY_SKIPPED, -1: "ciph" is not 56 (not searched);
 *   - VGB_HCA_KEY_NOT_FOUND, -1: no listed key passes ("Cannot find key to decrypt HCA file."), every type-56 file when
 *     n_keys is 0;
 *   - the error, -1: vgb_hca_parse refuses the file, or its channel layout is one the decoder cannot take (more than 8
 *     channels, bands out of range).
 * A file with zero frames has an empty window, so the first code passes.  Differences on purpose: the reference throws and
 * ends the run for an unreadable file or a missing key; here each file gets its status and the others are searched.
 * With several devices bound (vgb_init_devices) the files are split over them. */
#define VGB_HCA_KEY_SKIPPED   1
#define VGB_HCA_KEY_NOT_FOUND 2
int32_t vgb_hca_find_keys(const uint8_t *const *files, const int64_t *lengths, int32_t n_files, const uint64_t *key_codes,
                          int32_t n_keys, int32_t *key_index_out, int32_t *file_status_out);
/* Every (file, key) outcome of vgb_hca_find_keys' test, with no skipping across keys: outcome_out[f * n_keys + k] = 0 the
 * key passes, else 1 + 3 * j + r with j the window frame (0..9) it stops at and r 0 a bad sync word, 1 a scale-factor
 * delta out of range, 2 UnpackingWasSuccessful false; -1 for every key of a file that is not searched (not type 56, or
 * refused).  Returns VGB_OK unless the arguments are bad or the device fails. */
int32_t vgb_hca_debug_key_outcomes(const uint8_t *const *files, const int64_t *lengths, int32_t n_files,
                                   const uint64_t *key_codes, int32_t n_keys, int32_t *outcome_out);
/* The counts of the most recent vgb_hca_find_keys / vgb_hca_debug_key_outcomes (every device): out[0] (file, key) pairs
 * walked, [1] frames unpacked, [2] files searched, [3] device time of the search kernels in microseconds (CUDA events
 * around each device's launch, summed over the devices). */
int32_t vgb_hca_debug_key_search_stats(uint64_t *out, int32_t n);
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
 * goes to types 8 and 9 only; and the reference's built-in key list (CriAdxEncryption.FindKey) is not carried: a keyed
 * file needs the caller's key, which vgb_adx_find_keys can recover from the files.  A sample rate <= 0 decodes as in the reference (CalculateCoefficients' double math; a rate of 0 gives
 * NaN, which C#'s (int) makes int.MinValue and (short) 0).  Per-file errors, each failing that file only: a parse error, a missing key, bad loop points, a negative
 * unaligned sample count, decoded frames past a channel's audio (IndexOutOfRangeException), 2 GiB of PCM or more, too many
 * channels for the WAVE join - all known in the sizing pass - and a Fixed-type frame with a filter 4..7, found on the
 * device in the fill pass: that file gets its status_out entry, out_sizes[i] = 0 and its buffer is not written.  With
 * status_out NULL such a file fails the call (VGB_E_DATA) after every other file has been written. */
int32_t vgb_convert_adx_to_wave_batch(const uint8_t *const *files, const int64_t *lengths, int32_t n_files, const vgb_adx_key *key,
                                      int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out);
/* The key search of VGAudio.Tools/CrackAdx/GuessAdx.cs: recovers the CriAdxKey (seed, mult, inc) of keyed .adx files
 * (revisions 8 and 9) from the files alone, with no list of known keys.
 *   - Loading (LoadFiles, GuessAdx.cs:79-97): each image's header as AdxReader.ReadMetadata reads it; the search's
 *     revision is the first read file's (a file of revision 0 read before it sets nothing and is kept, as in the
 *     reference), files of another revision are skipped.  A kept file's AudioDataLength bytes from HeaderSize + 4 are
 *     read, bytes past the image as zero; Scales[i] is the big-endian u16 at i * FrameSize over the raw, interleaved
 *     region (file order = key stream order), StartFrame the frame of the first non-zero byte (0 if none).
 *   - Candidates (:48-71, TryScale :160-189): revision 8 takes the 0x400 primes above 0x4000 as seeds, multipliers and
 *     increments, validation mask 0xE000, MaxSeed 0x8000; revision 9 seeds 0..0x1FFF, multipliers x & 3 == 1 and odd
 *     increments below 0x2000, mask 0x1000, MaxSeed 0x2000.  For every scale index 0..0xFFF and every file:
 *     seed = (Scales[StartFrame] ^ index) & (MaxSeed - 1) (skipped when StartFrame is 0 and the seed is not listed), and
 *     every (mult, inc) walks the frames from StartFrame; a frame fails when ((scale ^ x) & mask) != 0 && scale != 0.
 *   - A full match is wound back to frame 0 (FindStartingKey :191-215; revision 8 drops a seed that is not a listed
 *     prime) and kept when KeyIsValid (:217-229) holds on every loaded file.  The keys are the union over every file's
 *     scan, each distinct key once, sorted ascending by (seed, mult, inc) - the reference logs them in thread order.
 *     Revision 9 only reads the low 13 bits of a key, so a file keyed with a 15-bit key (vgb_adx_key_from_code) is found
 *     as its 13-bit equivalent, which decrypts it byte for byte the same.
 *   - Confidence (AddKey :126-158, GetReencodeConfidence :231-263), per key and file: AdxReader with the key -> ToPcm16
 *     -> CriAdxFormat.EncodeFromPcm16 with default CriAdxParameters (frame size 18, version 4, Linear, the loop-start
 *     alignment of CriAdxFormat.cs:57-89), on the device through the .adx source stage of vgb_convert_adx_to_wave_batch
 *     and the ADX target encode of vgb_convert_wave_batch.  Each channel's decrypted audio is compared with its
 *     re-encode (Common.DiffArrays: bytes that DIFFER, -2 when the lengths differ) over n = channel 0's audio length
 *     ("full") and min(FrameSize * 100, full) ("short"); totals add n per channel.  confidence = 1 - (double)sum of
 *     differences / sum of totals over the files, short and full.
 * keys_out receives *n_keys_out entries; key_code is CriAdxKey.KeyCode.  When more than max_keys keys are valid on every
 * file the call fails (VGB_E_ARG) with nothing written to keys_out: no partial set, whatever the internal buffers hold.
 * *n_keys_out is then the number of keys when the search ran to its end, or 0 when it stopped early (more than max_keys
 * hits per scanned file already prove the set too large).  file_status_out[i] (may be NULL): VGB_OK for a file in the search,
 * VGB_ADX_KEY_SKIPPED for a file of another revision, else the file's read error.  *revision_out (may be NULL): the
 * search's revision.  With several devices bound (vgb_init_devices) the scale indices are split over them, and the
 * keys' confidences are spread over them key by key.
 * Revision 9 scans one file with a non-zero Scales[StartFrame] in place of every file: any key another file's scan finds
 * is valid on that file, and that file's scan finds every such key (the bits the scale pins are the bits validation
 * reads), so the set is the same.
 * Differences on purpose, where the reference throws and ends the whole run:
 *   - a file whose header cannot be read, or whose audio length or offset is invalid, gets that status and is left
 *     out; the revision comes from the first file that is read;
 *   - a first revision other than 8 or 9 (or no file read) fails the call with VGB_E_ARG (a NullReferenceException);
 *   - a file with no whole frame adds no candidates and validates every key (IndexOutOfRangeException at
 *     Scales[StartFrame]);
 *   - a key for which a file's re-read or re-encode throws gets that error as its status and NaN confidences; so does a
 *     sum past int.MaxValue (LINQ's checked Sum, VGB_E_DATA). */
#define VGB_ADX_KEY_SKIPPED 1
typedef struct vgb_adx_found_key {
    vgb_adx_key key;
    int32_t status;                        /* VGB_OK, or the error of the confidence pass (confidences NaN) */
    uint64_t key_code;                     /* CriAdxKey.KeyCode */
    int64_t diff_short, total_short;       /* sums over the files: differing bytes (IdenticalBytesShort) and compared bytes */
    int64_t diff_full, total_full;
    double confidence_short, confidence_full;
} vgb_adx_found_key;
int32_t vgb_adx_find_keys(const uint8_t *const *files, const int64_t *lengths, int32_t n_files, vgb_adx_found_key *keys_out,
                          int32_t max_keys, int32_t *n_keys_out, int32_t *file_status_out, int32_t *revision_out);
/* vgb_adx_find_keys over a box of the search: scale indices [index_first, index_end) of 0..0x1000, multipliers
 * [mult_first, mult_end) and increments [inc_first, inc_end) of the revision's lists (indices into them).  Every file is
 * scanned, as in the reference, unless flags holds VGB_ADX_KEYS_ONE_FILE: then revision 9 over every scale index scans
 * one file as vgb_adx_find_keys does.  Out-of-range boxes are VGB_E_ARG (after the files are read). */
#define VGB_ADX_KEYS_ONE_FILE 1
int32_t vgb_adx_debug_find_keys_box(const uint8_t *const *files, const int64_t *lengths, int32_t n_files, int32_t index_first,
                                    int32_t index_end, int32_t mult_first, int32_t mult_end, int32_t inc_first, int32_t inc_end,
                                    int32_t flags, vgb_adx_found_key *keys_out, int32_t max_keys, int32_t *n_keys_out,
                                    int32_t *file_status_out, int32_t *revision_out);
/* LoadFiles' body for one image, host only: *revision_inout is the search's revision so far (0 before the first file;
 * set from this file's header while it is 0).  Returns VGB_OK with the file's Scales (the first scales_cap of them),
 * their number and StartFrame; VGB_ADX_KEY_SKIPPED for another revision; or the read error. */
int32_t vgb_adx_key_load(const uint8_t *file, int64_t length, int32_t *revision_inout, uint16_t *scales_out, int32_t scales_cap,
                         int32_t *n_frames_out, int32_t *start_frame_out);
/* The counts of the most recent search (any thread, every device): out[0] candidates tried ((seed, mult, inc) triples
 * walked), [1] frame steps (frames tested, the failing one included), [2] full matches (candidates that walked every
 * frame, before FindStartingKey), [3] device time of the search kernels in microseconds (CUDA events around each
 * device's launches, summed over the devices). */
int32_t vgb_adx_debug_key_search_stats(uint64_t *out, int32_t n);
/* The decode direction of the batch job for NintendoWare files: .brstm, .bcstm and .bfstm streams, .brwav, .bcwav and
 * .bfwav wave files and .bcstp / .bfstp prefetch streams in, 16-bit WAVE images out - BrstmReader / BrwavReader /
 * BCFstmReader (vgb_nw_file_parse) -> Common.ToAudioStream (Containers/NintendoWare/Common.cs:45-116) -> ToPcm16 ->
 * WaveWriter.  in_type[i] (VGB_CONTAINER_BRSTM, _BCSTM, _BFSTM, _BRWAV, _BCWAV, _BFWAV, _BCSTP or _BFSTP; any other
 * value, IDSP and HPS included, fails that file) names the reader, as the reference picks one by file extension: BRSTM
 * uses BrstmReader, BRWAV BrwavReader, the others BCFstmReader, which accepts any of its magics (the stream types
 * refuse wave and prefetch files on purpose); the magic is not sniffed, so a .bcstm image passed as BRSTM fails as in
 * the reference.  A wave file's channels are separate runs: their bytes (ReadBytes, short or empty at the image's end)
 * are gathered into the channel rows by hps_gather_kernel, one launch per group, in place of the de-interleave; a
 * prefetch file's first region goes through the de-interleave as a stream.  The sizing pass adds ToAudioStream's checks
 * on such rows: GcAdpcmChannel's "Audio array length is too short for the specified number of samples." (VGB_E_ARG);
 * for PCM, the builders' sample count from channel 0's row ("All channels must have the same sample count", a
 * big-endian PCM16 row of odd length indexes past it, VGB_E_DATA), WithLoop(Looping, LoopStart, SampleCount) against
 * that count, and "Channels parameter cannot be empty or null" for no channels.  The WAVE holds that many samples.  Same two-pass protocol, per-file status and sharding as vgb_convert_adx_to_wave_batch (files weigh
 * sample_count * channel_count).  Per group of files, on the device: one H2D of the DATA regions, the existing
 * de-interleave (Stream.DeInterleave: a shorter last block, rows of SamplesToBytes(sample_count) bytes zero-filled or
 * truncated; an interleave size <= 0 copies nothing, so the rows are zeros), then the GC-ADPCM rows through the
 * time-parallel decoder (from each channel's start context; VGB_GC_DEC_SEGMENTS / VGB_GC_DEC_MIN_SEG_FRAMES force the
 * segment count and the shortest segment, read at each call) and the PCM rows through nw_pcm_kernel (PCM16 byte-swapped
 * when the file is big-endian, PCM8 by Pcm8Codec.DecodeSigned), then the WAVE join behind the host-built header (smpl
 * when looping, extensible fmt above two channels), one D2H of the finished files.  Gain, tracks, regions and seek
 * tables do not change the output and are not read by the decode.  Loop points follow WithLoop(Looping, LoopStart,
 * SampleCount) (AudioFormatBaseBuilder.cs:23-50; VGB_E_ARG with its messages).  Per-file errors, each failing that
 * file only: in_type not one of the eight, a parse error, bad loop points, a negative sample count (refused on purpose:
 * the reference allocates from it), 2 GiB of PCM or more, too many channels for the WAVE join - all known in the sizing
 * pass - and, found on the device in the fill pass, a GC-ADPCM frame header that selects a predictor 8..15 (the
 * reference indexes coefficients[predictor * 2] and throws): that file gets its status_out entry, out_sizes[i] = 0 and
 * its buffer is not written.  With status_out NULL such a file fails the call (VGB_E_DATA) after every other file has
 * been written. */
int32_t vgb_convert_nw_to_wave_batch(const uint8_t *const *files, const int64_t *lengths, const int32_t *in_type, int32_t n_files,
                                     int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out);
/* The decode direction of the batch job for IDSP and HPS streams: .idsp and .hps file images in, 16-bit WAVE images out -
 * IdspReader / HpsReader (vgb_idsp_parse / vgb_hps_parse) -> ToAudioStream -> GcAdpcmFormat.ToPcm16 -> WaveWriter.
 * in_type[i] is VGB_CONTAINER_IDSP or VGB_CONTAINER_HPS and names the reader (no sniffing); anything else fails that
 * file.  Same two-pass protocol, per-file status and sharding as vgb_convert_nw_to_wave_batch (files weigh sample_count *
 * channel_count).  Per group of files, on the device: one H2D of each IDSP audio region and of each HPS file's span of
 * block pieces; IDSP rows by the existing de-interleave, HPS rows by hps_gather_kernel (each channel row is the
 * concatenation of its pieces of every block, as HpsReader.ToAudioStream builds it; rows are cleared first); every row
 * through the time-parallel GC-ADPCM decoder from the header's coefficients and start history (GcAdpcmChannel.GetPcmAudio;
 * the HPS per-block and loop contexts are not used, as in the reference); the WAVE join.  The sizing pass, in the
 * reference's order: a negative sample count (VGB_E_DATA, on purpose), for HPS an overflowing sum of a channel's piece
 * lengths (VGB_E_DATA) and "Audio array length is too short for the specified number of samples." (GcAdpcmChannel,
 * VGB_E_ARG), WithLoop's messages when looping (AudioFormatBaseBuilder.cs:23-50, VGB_E_ARG; IDSP with (LoopStart,
 * LoopEnd), HPS with (LoopStart, SampleCount) - also the WAVE loop), 2 GiB of PCM or more, too many channels for the WAVE
 * join.  In the fill pass a frame header that selects a predictor 8..15 fails its file alone, as in
 * vgb_convert_nw_to_wave_batch; with status_out NULL such a file fails the call (VGB_E_DATA) after every other file has
 * been written. */
int32_t vgb_convert_idsp_hps_to_wave_batch(const uint8_t *const *files, const int64_t *lengths, const int32_t *in_type, int32_t n_files,
                                           int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out);
/* The decode direction of the batch job for every readable source in one call, with the batch's loop setting: in_type[i]
 * names file i's reader (VGB_CONTAINER_DSP, _ADX, _HCA, _BRSTM ... _BFSTP, _IDSP, _HPS; any other value fails that file
 * with VGB_E_ARG).  Each file is read, decoded and written exactly as by the one of vgb_convert_{dsp,adx,hca,nw,
 * idsp_hps}_to_wave_batch that takes its in_type (same two-pass protocol, per-file status, sharding over the bound
 * devices and fill-pass refusals; *adx_key and *hca_key_code as there, NULL for none), and with options NULL or
 * loop_mode 0 its bytes are theirs.  Only the loop_* fields of *options are read: AudioData.SetLoop runs on the
 * source's format before the WAVE is written (Convert.cs:82-90):
 *   - VGB_LOOP_CLEAR (--no-loop): WithLoop(false), no smpl chunk.  An .hca file stays cut at its old loop end.
 *   - VGB_LOOP_SET (-l loop_start-loop_end): WithLoop(true, s, e) (AudioFormatBaseBuilder.cs:23-58) against the sample
 *     count ToPcm16 yields (the unaligned count for .adx, channel 0's row for PCM NintendoWare files), failing the file
 *     with "Loop points must be less than the number of samples and non-negative." or "The loop end must be greater than
 *     the loop start" (VGB_E_ARG); s == e is a loop.  An .hca file then refuses any points but its own ("Changing the
 *     loop points on HCA audio without re-encoding is not supported.") and a loop it does not have ("Adding a loop to
 *     HCA audio without re-encoding is not supported."), VGB_E_ARG.
 * The same rules, at the same point of every source plan, drive vgb_convert_wave_batch (WAVE sources),
 * vgb_transcode_batch and vgb_rewrite_batch through their options.  The files of each reader go through their own
 * groups, .dsp last (a predictor outside 0..7 still fails the call).  Without
 * status_out a fill-pass refusal fails the call (VGB_E_DATA) after the other files are written. */
int32_t vgb_convert_to_wave_batch(const uint8_t *const *files, const int64_t *lengths, const int32_t *in_type, int32_t n_files,
                                  const vgb_convert_options *options, const vgb_adx_key *adx_key, const uint64_t *hca_key_code,
                                  int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out);
/* Bookkeeping of the most recent time-parallel GC-ADPCM decode of vgb_convert_nw_to_wave_batch or
 * vgb_convert_idsp_hps_to_wave_batch on this thread's
 * context (its last group of files): out[0] segments per channel, [1] frames decoded by run-ons, [2] frames decoded by
 * the cascade, [3] boundaries the cascade repaired, [4] longest run-on in frames.  Synchronises the device. */
int32_t vgb_gcadpcm_debug_decode_stats(uint64_t *out, int32_t n);
/* Transcoding in the batch job: .dsp, .adx and .hca file images in, another of the three out (Convert.ConvertFile with a
 * coded source: the source's reader, a fresh configuration from the options, source.ToPcm16() -> EncodeFromPcm16).
 * in_type[i] (VGB_CONTAINER_*) names file i's codec: a .dsp file has no signature.  options->out_type, its options and
 * its key describe the output exactly as for vgb_convert_wave_batch; options->group_bytes counts DECODED PCM bytes per
 * GPU batch (0: an eighth of the job's PCM, 64..512 MiB; a batch holds at most 4096 files).  The sources are read as by vgb_convert_{dsp,adx,hca}_to_wave_batch:
 * the PCM, loop points and rate their ToPcm16 yields (.adx: sample_count - inserted_samples samples, loop points shifted;
 * .hca: trimmed at the loop end; .dsp: from the header's start history), and their keys: *in_adx_key decrypts revision 8
 * and 9 .adx files, *in_hca_key_code "ciph" 56 .hca files, "ciph" 1 uses the built-in table; a keyed source without its
 * key fails alone, keys are never applied to other revisions (vgb_adx_find_keys recovers a key from the files).  No PCM leaves the device:
 * per batch one H2D of the coded regions, the source's decode straight into the encoder's channel rows, encode and file
 * assembly, one D2H of the finished files.  Same two-pass protocol, per-file status, progress and sharding (files weigh
 * sample_count * channel_count + 1024) as vgb_convert_wave_batch.
 * Per-file errors of the sizing pass, each failing that file only: in_type not DSP / ADX / HCA, or equal to out_type
 * (a rewrite in the source's own codec is not performed), the source's parse and planning errors (as its -> WAVE
 * converter, without the WAVE writer's limits), and the target's planning errors (as vgb_convert_wave_batch).
 * In the fill pass, an ADX frame with a filter the reference cannot index or an HCA frame the decoder refuses fails that
 * file alone (status_out entry, out_sizes[i] = 0, buffer not written; without status_out the call fails with VGB_E_DATA
 * after the other files are written), a GC-ADPCM predictor outside 0..7 fails the call (VGB_E_DATA).
 * loop_mode sets or clears every source's loop on the source's format before the re-encode (vgb_convert_to_wave_batch's
 * rules: an .hca source refuses new points and an added loop even here, as CriHcaFormatBuilder does). */
int32_t vgb_transcode_batch(const uint8_t *const *files, const int64_t *lengths, const int32_t *in_type, int32_t n_files,
                            const vgb_convert_options *options, const vgb_adx_key *in_adx_key, const uint64_t *in_hca_key_code,
                            int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out, vgb_progress_cb cb, void *user);
/* Transcoding in the batch job into the NintendoWare streams, IDSP and HPS: .dsp, .adx and .hca file images in,
 * options->out_type (VGB_CONTAINER_BRSTM, _BCSTM, _BFSTM, _IDSP or _HPS; anything else fails the call with VGB_E_ARG)
 * out.  The sources are read exactly as by vgb_transcode_batch (in_type, keys, loop_mode, what ToPcm16 yields); the
 * target is planned and written exactly as by vgb_convert_wave_batch for the same PCM (nw_codec_plus1, nw_endianness,
 * nw_loop_point_alignment, no_trim for IDSP): GC-ADPCM coefficients, encode, GcAdpcmFormat.WithAlignment of a loop start
 * off the alignment, seek table, loop and block contexts, all on the device.  Same two-pass protocol, per-file status,
 * progress, sharding and fill-pass failures as vgb_transcode_batch; options->group_bytes counts a file's decoded PCM plus,
 * for GC-ADPCM, the full decode and ADPCM rows the target keeps resident, as vgb_convert_wave_batch counts it.
 * Per-file errors of the sizing pass besides those of vgb_transcode_batch's sources and vgb_convert_wave_batch's
 * targets: in_type not DSP / ADX / HCA, and a .dsp source into a GC-ADPCM target (IDSP, HPS, or NintendoWare without
 * -f pcm16 / pcm8), where GetFormat<GcAdpcmFormat> hands back the source's own format: a rewrite, which is not performed. */
int32_t vgb_transcode_nw_batch(const uint8_t *const *files, const int64_t *lengths, const int32_t *in_type, int32_t n_files,
                               const vgb_convert_options *options, const vgb_adx_key *in_adx_key, const uint64_t *in_hca_key_code,
                               int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out, vgb_progress_cb cb, void *user);
/* Transcoding in the batch job from the NintendoWare streams, wave and prefetch files, IDSP and HPS: file images of
 * in_type VGB_CONTAINER_BRSTM .. _BFSTP (4..13) in, options->out_type any of the eight coded targets (VGB_CONTAINER_DSP
 * .. _HPS; anything else fails the call with VGB_E_ARG) out.  The sources are read exactly as by
 * vgb_convert_to_wave_batch (the reader in_type names, loop_mode, what ToPcm16 yields: GC-ADPCM, or the header's PCM16 /
 * PCM8); the target is planned and written exactly as by vgb_convert_wave_batch for the same PCM (the output key, ADX
 * type / frame size / version, HCA quality / bitrate, nw_codec_plus1, nw_endianness, nw_loop_point_alignment, no_trim).
 * None of these containers is encrypted: there are no input keys.  Same two-pass protocol, per-file status, progress,
 * group_bytes and sharding over the bound devices as vgb_transcode_batch.
 * A source whose codec is the target's (AudioData.GetFormat<T> hands back its own format) is a rewrite, which is not
 * performed: GC-ADPCM into .dsp / IDSP / HPS / a NintendoWare stream without -f pcm16|pcm8, PCM16 into -f pcm16, PCM8
 * into -f pcm8.  Per-file errors of the sizing pass, in this order: in_type outside 4..13; IDSP / HPS into a GC-ADPCM
 * target (the rewrite message, before the file is read); the reader's and the loop setting's errors, as in
 * vgb_convert_to_wave_batch; a NintendoWare file whose header's codec is the target's (the rewrite message); the
 * target's errors, as in vgb_convert_wave_batch.  Fill pass: a GC-ADPCM frame header selecting a predictor outside 0..7
 * fails its own file with VGB_E_DATA (an HCA target's encoder status of that file is not reported); without status_out
 * the call then fails. */
int32_t vgb_transcode_from_nw_batch(const uint8_t *const *files, const int64_t *lengths, const int32_t *in_type, int32_t n_files,
                                    const vgb_convert_options *options, int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out,
                                    vgb_progress_cb cb, void *user);
/* Rewriting .dsp files into BRSTM, BCSTM, BFSTM, IDSP or HPS without re-encoding (DspReader -> GetFormat<GcAdpcmFormat>
 * hands the writer the source's own ADPCM, Formats/AudioData.cs:20-33).  in_type[i] must be VGB_CONTAINER_DSP (any other
 * value fails that file with VGB_E_ARG); options->out_type is VGB_CONTAINER_BRSTM .. _HPS and nw_codec_plus1 is 0 or 3
 * (GC-ADPCM), else the call fails with VGB_E_ARG.  The loop setting, nw_endianness, nw_loop_point_alignment and no_trim
 * mean what they mean in vgb_convert_wave_batch; the sizes and per-file refusals of the sizing pass are those of
 * vgb_convert_to_wave_batch's .dsp reader and loop setting, then vgb_convert_wave_batch's target for the same PCM
 * description (an HPS file keeps its refusals, except the history read past the unaligned decode when the writer's
 * channels hold no decode: there HpsWriter writes history 0).  Same two-pass protocol, per-file status and sharding over
 * the bound devices as vgb_transcode_batch (no progress callback; group_bytes as there).
 * Every ADPCM byte is copied except the loop tail GcAdpcmAlignment re-encodes when the loop start is not a multiple of
 * the target's alignment.  The output keeps each channel's coefficients, gain and start history (the start
 * predictor/scale is the first ADPCM byte, GcAdpcmChannel.cs:44).  The NintendoWare and HPS writers recalculate the loop
 * context from a decode (history 0) at the unaligned loop start, as does the NintendoWare seek table; IDSP keeps the
 * header's loop context verbatim when the file is read and written with the header's loop start
 * (GcAdpcmChannelBuilder.PreviousLoopContextIsValid), and decodes it otherwise (-l, --no-loop on a looping file).  Fill
 * pass: a frame header selecting a predictor outside 0..7 fails its own file with VGB_E_DATA; without status_out the
 * call then fails. */
int32_t vgb_rewrite_gc_batch(const uint8_t *const *files, const int64_t *lengths, const int32_t *in_type, int32_t n_files,
                             const vgb_convert_options *options, int64_t *out_sizes, uint8_t *const *files_out, int32_t *status_out);
/* Rewriting .adx or .hca files in their own codec without re-encoding: decrypted, re-keyed or left as they are
 * (Convert.ConvertFile with the same container on both sides: the reader decrypts the frames, AudioData.GetFormat<T>
 * hands the writer the source's own CriAdxFormat / CriHcaFormat, Formats/AudioData.cs:20-33, and the writer encrypts
 * them with the output key or writes them in the clear).  options->out_type (VGB_CONTAINER_ADX or _HCA) names both the
 * reader and the writer: every file is read by it.  Same two-pass protocol, per-file status, progress, group_bytes
 * (INPUT bytes per GPU batch; 0: an eighth of the job, 64..512 MiB) and sharding over the bound devices (files weigh
 * their payload bytes) as vgb_transcode_batch; the sizing pass runs on the host only.  No payload byte is touched on
 * the host: per batch one H2D of the frame regions, one kernel pass, one D2H of the finished files.
 * Input keys as in vgb_transcode_batch: *in_adx_key decrypts revision 8 and 9 .adx files, *in_hca_key_code "ciph" 56
 * .hca files, "ciph" 1 uses the built-in table.  The output key: adx_has_key with the adx_key_* fields and
 * adx_encryption_type (the header's encryption byte, written with or without a key), or hca_key_type (-1 none, 0, 1,
 * 56) with hca_key_code.  adx_version, adx_frame_size, adx_type, adx_filter_plus1, hca_quality, hca_bitrate and
 * hca_limit_bitrate are ignored: the writer receives the source's format and they only reach the encoder.
 *   .adx (AdxReader.cs:14-58 -> AdxWriter.cs:18-140): the header is rebuilt from the source's frame size, version,
 *   type byte and high-pass (0 for type 2, Fixed), SampleCount - InsertedSamples samples with AlignmentSamples =
 *   InsertedSamples, the loop points minus InsertedSamples, and a version-4 history block holding each channel's first
 *   history sample twice.  TrimFile (!no_trim) cuts a looping file at LoopEnd + 3 frames, which may be more frames than
 *   the source holds: those stay zero.  Output frame j * channels + c is source frame j * channels + c; its two scale
 *   bytes go through the source's key stream, then the output's, at that step, each side behind its own FrameNotEmpty
 *   test and type-9 mask (adx_rewrite_kernel).
 *   .hca (HcaReader.cs:20-49 -> HcaWriter.cs:21-178): the frames are decrypted where HcaReader decrypts them ("ciph" 1,
 *   or 56 with a key) and encrypted with the output key: bytes [0, FrameSize - 2) through one composed substitution
 *   table and the CRC-16 recomputed (also for an output key of type 0); with neither they are copied verbatim, a wrong
 *   CRC included.  The header is regenerated at the source's header_size: version 0x0200, chunks HCA fmt comp [loop]
 *   ciph [rva] comm|pad, ids masked with 0x80 iff an output key is given, "ciph" the output key's type, else 0 for a
 *   decrypted source and the source's value otherwise; a dec chunk comes out as comp, track_count below 1 as 1, ath and
 *   vbr are dropped (so a version < 2.0 file without ath decodes differently afterwards, as in the reference).  The
 *   comment is ReadUTF8Z's (Utilities/Extensions.cs:60-73: from one byte past the comm id to the first byte 0x00 or
 *   0x01; at the end of the image its last byte is dropped), written as pad when every character is white space to
 *   string.IsNullOrWhiteSpace; rva is kept as its float bits and written whenever the volume is not 1 (NaN included).
 *   Chunks that do not fit in header_size - 2 bytes are written on as the reference's writer does: the header CRC covers
 *   the first header_size - 2 bytes as written, and the CRC and the frames overwrite the rest.
 * Per-file errors of the sizing pass, each failing that file only: the parse errors of vgb_adx_parse / vgb_hca_parse, a
 * keyed source without its key, loop points WithLoop refuses (AudioFormatBaseBuilder.cs:23-50), an InsertedSamples
 * above the sample count or below 0 (VGB_E_ARG), 2 GiB of output or more.  Differences on purpose: an encrypted source
 * without its key fails (the reference would pass the encrypted frames through, an .adx file even labelled with the
 * output's encryption byte); a comment that is not valid UTF-8 fails with VGB_E_DATA (the reference would write U+FFFD
 * in place of the bad bytes); HCA chunks that run past the end of the output file fail with VGB_E_DATA (the reference
 * would grow the file: only a tiny header_size with few frames can do that).  There is no device-side refusal.
 * loop_mode sets or clears every source's loop with vgb_convert_to_wave_batch's rules: an .adx file gets the new
 * (unaligned) points plus AlignmentSamples in its header and TrimFile cuts a looping file at the new loop end, shorter
 * or longer than the source; an .hca file loses its loop chunk with VGB_LOOP_CLEAR (same header size and frames) and
 * takes VGB_LOOP_SET only with its own points. */
int32_t vgb_rewrite_batch(const uint8_t *const *files, const int64_t *lengths, int32_t n_files, const vgb_convert_options *options,
                          const vgb_adx_key *in_adx_key, const uint64_t *in_hca_key_code, int64_t *out_sizes, uint8_t *const *files_out,
                          int32_t *status_out, vgb_progress_cb cb, void *user);
/* Measurement tap: device time of the most recent vgb_convert_wave_batch summed over its (first 32) batches per device,
 * over every device that converted part of it, out[0..3] = WAVE split, encode, loop-context decode, file assembly (ms,
 * CUDA events on the kernel streams); returns the number of batches timed on all devices together. */
int32_t vgb_convert_debug_stage_ms(float *out, int32_t n);

#ifdef __cplusplus
}
#endif
#endif /* VGAUDIO_B200_H */
