// containers.cu — the byte movers either side of the codec path (SURVEY.md §8f rank 2-4), so that a batch goes from
// file bytes to file bytes without leaving HBM:
//   front end  WAVE data chunk -> short[ch][n]        WaveReader.cs:13-51, InterleavedByteToShort (Interleave.cs:188-207)
//   writers    DSP  header + block-interleaved ADPCM   DspWriter.cs:42-99
//              ADX  header + frame-interleaved frames + footer, optional encryption
//                                                      AdxWriter.cs:70-140, CriAdxEncryption.cs:8-44
//              HCA  chunked header + CRC + frames, optional encryption
//                                                      HcaWriter.cs:56-178, CriHcaEncryption.cs:12-33
//   reader     DSP  header parse + payload de-interleave   DspReader.cs:57-119
//   batch      WAVE files in -> encoded files out, files coalesced into GPU batches
//                                                      src/VGAudio.Cli/Batch.cs:11-51 + Convert.cs:18-36
// All of it is HBM-bound byte work (every payload byte read once, written once); headers are a few dozen bytes per file
// and are built on the host, except the fields that only exist on the device (DSP: coefficients, first predictor/scale
// byte, loop context), which the assemble kernel patches in.  Citations are relative to VGAudio's src/VGAudio/.
#include <array>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <deque>

#include "abi.cuh"

using namespace vgb;  // the shared host runtime; common.cuh: GcAdpcmMath helpers, frame constants

namespace {

inline int next_multiple(int value, int multiple)  // Utilities/Helpers.cs:71-80
{
    if (multiple <= 0) return value;
    if (value % multiple == 0) return value;
    return value + multiple - value % multiple;
}

// ---------------------------------------------------------------------------------------------------------------
// device-side descriptors
// ---------------------------------------------------------------------------------------------------------------
constexpr int kTileBytes = 16384;      // output bytes one CTA of an assemble / split kernel produces
constexpr int kSplitSmemSamples = 8192;

struct WaveItem {            // one WAVE data chunk -> channel rows
    int64_t in_off;          // bytes into the input slab (multiple of 16)
    int64_t out_off;         // samples into the PCM slab: row of channel 0 (multiple of 8)
    int64_t out_stride;      // samples between channel rows (multiple of 8)
    int32_t channels, samples, bits, tile_samples;
    int32_t tile_first;      // first tile of this item (exclusive prefix sum)
    int32_t lead;            // zero samples written in front of every row (an encoder's alignment padding made physical)
};

struct DspChan {
    int64_t adpcm_off;       // bytes into the ADPCM slab (multiple of 16)
    int64_t pcm_off;         // samples into the decoded-PCM scratch (looping files), else -1
    int32_t coef_index;      // row of the coefficient table
    int16_t gain, hist1, hist2;
    int16_t loop_ctx[3];     // used when pcm_off < 0 and the file loops (caller-provided context)
    int16_t pad;
};
struct DspFile {
    int64_t out_off;         // bytes into the output slab (multiple of 16)
    int32_t channels, first_ch;
    int32_t in_size;         // bytes of ADPCM a channel holds (SampleCountToByteCount of the encoded length)
    int32_t data_size;       // AudioDataSize (DspWriter.cs:105-106)
    int32_t bpi;             // BytesPerInterleave
    int32_t sample_count, nibble_count, sample_rate, looping, start_addr, end_addr;
    int32_t loop_start;      // the format's LoopStart (where the loop context is taken)
    int32_t tile_first;
    int32_t pad;
};

struct AdxChanRef { int64_t adpcm_off; };
struct AdxFile {
    int64_t out_off;         // bytes into the output slab
    int64_t hdr_off;         // bytes into the header blob (header_size + 4 bytes: header and the "(c)CRI" tail)
    int32_t channels, first_ch;
    int32_t frame_size, frame_count, in_frames;   // frames written / frames a channel holds
    int32_t audio_offset, footer_offset, footer_size;
    int32_t has_key, enc_type, seed, mult, inc;
    int32_t tile_first;
};

// An .adx file rewritten in its own codec (vgb_rewrite_batch): both sides are frame-interleaved with the same channel
// count and frame size, so output frame p (= j * channels + c) is source frame p, which is also its key stream step
struct AdxRewriteFile {
    int64_t out_off;         // bytes into the output slab
    int64_t hdr_off;         // bytes into the header blob (audio_offset bytes)
    int64_t src_off;         // bytes into the input slab: the source's interleaved audio region (multiple of 16)
    int32_t frame_size, frames, src_frames;       // frames written / frames the source holds, over all channels
    int32_t audio_offset, footer_offset, footer_size;
    int32_t dec_type, dec_seed, dec_mult, dec_inc; // the source's key: revision 8 or 9, or dec_type 0 for none
    int32_t has_key, enc_type, seed, mult, inc;    // the output's key and the encryption type its header states
    int32_t tile_first;
};

struct HcaFile {
    int64_t out_off, hdr_off, frames_off;
    int32_t header_size, frame_size, frame_count;
    int32_t tile_first;
};

template <class T>
__device__ __forceinline__ int find_item(const T *items, int n, int tile)
{
    int lo = 0, hi = n - 1;  // last item whose tile_first <= tile
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (items[mid].tile_first <= tile) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---------------------------------------------------------------------------------------------------------------
// WAVE front end: one CTA turns tile_samples sample times of ALL channels of one file from interleaved little-endian
// bytes into channel rows, through shared memory so both sides are coalesced 16-byte accesses.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) wave_split_kernel(const uint8_t *__restrict__ in, const WaveItem *__restrict__ items, int n_items,
                                                          int16_t *__restrict__ pcm)
{
    __shared__ __align__(16) int16_t tile[kSplitSmemSamples];
    const int it = find_item(items, n_items, (int)blockIdx.x);
    const WaveItem w = items[it];
    const int s0 = ((int)blockIdx.x - w.tile_first) * w.tile_samples;
    const int ns = min(w.tile_samples, w.samples - s0);
    if (ns <= 0) return;
    const int ch = w.channels;
    if (s0 == 0 && w.lead > 0)                                  // the first tile also lays down the leading zeros of every row
        for (int t = threadIdx.x; t < w.lead * ch; t += blockDim.x) pcm[w.out_off + (int64_t)(t / w.lead) * w.out_stride + t % w.lead] = 0;
    if (ch == 1 && w.bits == 16 && (w.lead & 7) == 0) {         // mono: the data chunk IS the row
        const uint4 *src = reinterpret_cast<const uint4 *>(in + w.in_off + (int64_t)s0 * 2);
        int16_t *row = pcm + w.out_off + w.lead + s0;
        const int n_vec = ns >> 3;
        for (int v = threadIdx.x; v < n_vec; v += blockDim.x) reinterpret_cast<uint4 *>(row)[v] = src[v];
        for (int e = (n_vec << 3) + threadIdx.x; e < ns; e += blockDim.x) row[e] = reinterpret_cast<const int16_t *>(src)[e];
        return;
    }
    const int n_el = ns * ch;                                   // interleaved elements of this tile
    if (w.bits == 16) {
        const uint8_t *src = in + w.in_off + (int64_t)s0 * ch * 2;   // 16-byte aligned: tile_samples is a multiple of 8
        const int n_vec = n_el >> 3;
        for (int v = threadIdx.x; v < n_vec; v += blockDim.x)
            reinterpret_cast<uint4 *>(tile)[v] = reinterpret_cast<const uint4 *>(src)[v];
        for (int e = (n_vec << 3) + threadIdx.x; e < n_el; e += blockDim.x)
            tile[e] = (int16_t)(src[2 * e] | (src[2 * e + 1] << 8));
    } else {                                                    // 8-bit: Pcm8Codec.Decode (Codecs/Pcm8/Pcm8Codec.cs:23)
        const uint8_t *src = in + w.in_off + (int64_t)s0 * ch;
        for (int e = threadIdx.x; e < n_el; e += blockDim.x) tile[e] = (int16_t)((src[e] - 0x80) << 8);
    }
    __syncthreads();
    // rows out: pairs of samples per thread (rows start on 16-byte boundaries, s0 is even; an odd lead breaks the pairing)
    const int pairs = (ns + 1) >> 1;
    const bool paired = (w.lead & 1) == 0;
    for (int t = threadIdx.x; t < pairs * ch; t += blockDim.x) {
        const int o = t / pairs, i = (t - o * pairs) * 2;
        int16_t *row = pcm + w.out_off + (int64_t)o * w.out_stride + w.lead + s0;
        const uint32_t a = (uint16_t)tile[i * ch + o];
        if (i + 1 < ns) {
            const uint32_t b = (uint16_t)tile[(i + 1) * ch + o];
            if (paired) *reinterpret_cast<uint32_t *>(row + i) = a | (b << 16);
            else { row[i] = (int16_t)a; row[i + 1] = (int16_t)b; }
        } else {
            row[i] = (int16_t)a;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// WAVE writer, 16-bit codec (WaveWriter.WriteDataChunk -> ShortToInterleavedByte, Interleave.cs:169-186): the inverse of
// wave_split_kernel.  Tile 0 of a file also copies the host-built RIFF header.  The data chunk starts at a multiple of four
// bytes (every chunk size the writer emits is one), so the interleaved samples leave as 32-bit words.
// ---------------------------------------------------------------------------------------------------------------
struct WaveJoinItem {
    int64_t pcm_off;         // samples into the PCM slab: row of channel 0
    int64_t pcm_stride;      // samples between channel rows
    int64_t out_off;         // bytes into the output slab (multiple of 16)
    int64_t hdr_off;         // bytes into the header blob
    int32_t header_size, channels, samples, tile_samples;
    int32_t tile_first;
    int32_t pad;
};

__global__ void __launch_bounds__(256) wave_join_kernel(const int16_t *__restrict__ pcm, const WaveJoinItem *__restrict__ items, int n_items,
                                                         const uint8_t *__restrict__ hdr_blob, uint8_t *__restrict__ out)
{
    __shared__ __align__(16) int16_t tile[kSplitSmemSamples];
    const int it = find_item(items, n_items, (int)blockIdx.x);
    const WaveJoinItem w = items[it];
    const int t = (int)blockIdx.x - w.tile_first;
    uint8_t *dst = out + w.out_off;
    if (t == 0)
        for (int k = threadIdx.x; k < w.header_size; k += blockDim.x) dst[k] = hdr_blob[w.hdr_off + k];
    const int s0 = t * w.tile_samples;
    const int ns = min(w.tile_samples, w.samples - s0);
    if (ns <= 0) return;
    const int ch = w.channels;
    for (int k = threadIdx.x; k < ns * ch; k += blockDim.x) {  // rows in (coalesced per row), interleaved order in shared memory
        const int o = k / ns, i = k - o * ns;
        tile[i * ch + o] = pcm[w.pcm_off + (int64_t)o * w.pcm_stride + s0 + i];
    }
    __syncthreads();
    uint8_t *data = dst + w.header_size + (int64_t)s0 * ch * 2;   // 4-byte aligned: s0 * ch is even (tile_samples is a multiple of 8)
    const int n_el = ns * ch, n_words = n_el >> 1;
    for (int k = threadIdx.x; k < n_words; k += blockDim.x) reinterpret_cast<uint32_t *>(data)[k] = reinterpret_cast<const uint32_t *>(tile)[k];
    if ((n_el & 1) && threadIdx.x == 0) reinterpret_cast<int16_t *>(data)[n_el - 1] = tile[n_el - 1];
}

// ---------------------------------------------------------------------------------------------------------------
// NintendoWare PCM rows -> the int16 rows the WAVE join reads (Common.ToPcm16Stream / ToPcm8Stream, Common.cs:99-116):
// PCM16 is ToShortArray in the file's byte order, PCM8 is Pcm8Codec.DecodeSigned (Codecs/Pcm8/Pcm8Codec.cs:41-50).
// wave_split_kernel's 8-bit path reads unsigned interleaved WAVE bytes; these rows are planar, signed and possibly
// big-endian, so they get a kernel of their own instead of a caller switch inside the WAVE front end.  One CTA per
// kNwPcmTile samples of one row; rows start 16-byte aligned on both sides.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kNwPcmTile = 8192;
struct NwPcmRow {
    int64_t in_off;    // bytes into the row slab
    int64_t out_off;   // samples into the PCM slab (multiple of 8)
    int32_t samples, mode;  // mode 0: PCM8 signed, 1: PCM16 little-endian, 2: PCM16 big-endian
    int32_t tile_first, pad;
};

__global__ void __launch_bounds__(256) nw_pcm_kernel(const uint8_t *__restrict__ rows, const NwPcmRow *__restrict__ items, int n_items,
                                                      int16_t *__restrict__ pcm)
{
    const int it = find_item(items, n_items, (int)blockIdx.x);
    const NwPcmRow r = items[it];
    const int s0 = ((int)blockIdx.x - r.tile_first) * kNwPcmTile;
    const int ns = min(kNwPcmTile, r.samples - s0);
    const uint8_t *src = rows + r.in_off;
    int16_t *dst = pcm + r.out_off + s0;
    if (r.mode == 0) {
        for (int k = threadIdx.x; k < ns; k += blockDim.x) dst[k] = (int16_t)((uint32_t)src[s0 + k] << 8);
        return;
    }
    const uint32_t *w = reinterpret_cast<const uint32_t *>(src + (int64_t)s0 * 2);  // two samples per word
    uint32_t *o = reinterpret_cast<uint32_t *>(dst);
    const bool swap = r.mode == 2;
    for (int k = threadIdx.x; k < ns / 2; k += blockDim.x) {
        const uint32_t v = w[k];
        o[k] = swap ? __byte_perm(v, 0, 0x2301) : v;
    }
    if ((ns & 1) && threadIdx.x == 0) {
        const uint8_t *b = src + (int64_t)(s0 + ns - 1) * 2;
        dst[ns - 1] = (int16_t)(swap ? (b[0] << 8 | b[1]) : (b[1] << 8 | b[0]));
    }
}

// ---------------------------------------------------------------------------------------------------------------
// DSP writer.  Tile 0 of a file writes the channel headers (big-endian halfwords), the others 16 KB of the data
// region each: byte q of the region belongs to block b, channel i, offset k (Interleave.cs:43-79 semantics: shorter
// last block on either side, zero fill) and comes from channel i's byte bpi*b + k.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void put_be16(uint8_t *p, int v) { p[0] = (uint8_t)(v >> 8); p[1] = (uint8_t)v; }

__global__ void __launch_bounds__(256) dsp_assemble_kernel(const DspFile *__restrict__ files, int n_files, const DspChan *__restrict__ chans,
                                                            const uint8_t *__restrict__ adpcm, const int16_t *__restrict__ coefs,
                                                            const int16_t *__restrict__ decoded, uint8_t *__restrict__ out)
{
    const int fi = find_item(files, n_files, (int)blockIdx.x);
    const DspFile f = files[fi];
    const int tile = (int)blockIdx.x - f.tile_first;
    uint8_t *dst = out + f.out_off;
    if (tile == 0) {  // WriteHeader (DspWriter.cs:54-84), one halfword per thread-step
        for (int t = threadIdx.x; t < f.channels * 0x30; t += blockDim.x) {
            const int c = t / 0x30, h = (t - c * 0x30) * 2;
            const DspChan cc = chans[f.first_ch + c];
            int v = 0;
            auto hi = [](int32_t x) { return (int)((uint32_t)x >> 16); };
            switch (h) {
            case 0x00: v = hi(f.sample_count); break;    case 0x02: v = f.sample_count; break;
            case 0x04: v = hi(f.nibble_count); break;    case 0x06: v = f.nibble_count; break;
            case 0x08: v = hi(f.sample_rate); break;     case 0x0a: v = f.sample_rate; break;
            case 0x0c: v = f.looping ? 1 : 0; break;     case 0x0e: v = 0; break;
            case 0x10: v = hi(f.start_addr); break;      case 0x12: v = f.start_addr; break;
            case 0x14: v = hi(f.end_addr); break;        case 0x16: v = f.end_addr; break;
            case 0x18: v = 0; break;                     case 0x1a: v = 2; break;   // CurAddr = SampleToNibble(0)
            case 0x3c: v = cc.gain; break;
            case 0x3e: v = f.in_size > 0 ? adpcm[cc.adpcm_off] : 0; break;          // StartContext.PredScale (GcAdpcmChannel.cs:44)
            case 0x40: v = cc.hist1; break;              case 0x42: v = cc.hist2; break;
            case 0x44:  // LoopContext (GcAdpcmLoopContext.cs:17-26): predictor/scale of the loop frame, pcm[ls-1], pcm[ls-2]
                if (f.looping) v = cc.pcm_off >= 0 ? adpcm[cc.adpcm_off + (int64_t)(f.loop_start / kGcFrameSamples) * kGcFrameBytes] : cc.loop_ctx[0];
                break;
            case 0x46: if (f.looping) v = cc.pcm_off >= 0 ? (f.loop_start >= 1 ? decoded[cc.pcm_off + f.loop_start - 1] : 0) : cc.loop_ctx[1]; break;
            case 0x48: if (f.looping) v = cc.pcm_off >= 0 ? (f.loop_start >= 2 ? decoded[cc.pcm_off + f.loop_start - 2] : 0) : cc.loop_ctx[2]; break;
            case 0x4a: v = f.channels == 1 ? 0 : f.channels; break;
            case 0x4c: v = f.channels == 1 ? 0 : f.bpi / kGcFrameBytes; break;
            default:
                if (h >= 0x1c && h < 0x3c) v = coefs[(int64_t)cc.coef_index * 16 + ((h - 0x1c) >> 1)];
                break;  // 0x4e..0x5f: padding
            }
            put_be16(dst + c * 0x60 + h, v);
        }
        return;
    }
    const int ch = f.channels;
    uint8_t *data = dst + 0x60 * ch;
    // a file is below 2 GiB (FileSize is an int in the reference): 32-bit positions, unsigned so the divisions are cheap
    const uint32_t region = (uint32_t)f.data_size * (uint32_t)ch;
    const uint32_t q0 = (uint32_t)(tile - 1) * kTileBytes;
    const int in_blocks = div_round_up(f.in_size, f.bpi), out_blocks = div_round_up(f.data_size, f.bpi);
    const int last_in = f.in_size - (in_blocks - 1) * f.bpi, last_out = f.data_size - (out_blocks - 1) * f.bpi;
    const int copy_blocks = min(in_blocks, out_blocks);
    const uint32_t block_span = (uint32_t)f.bpi * (uint32_t)ch;
#pragma unroll 4  // independent words: the loads of several iterations are in flight together
    for (int w = threadIdx.x; w < kTileBytes / 8; w += blockDim.x) {
        const uint32_t q = q0 + (uint32_t)w * 8;
        if (q >= region) break;
        int b = (int)(q / block_span);
        if (b > out_blocks - 1) b = out_blocks - 1;
        const int cur_out = b == out_blocks - 1 ? last_out : f.bpi;
        const int r = (int)(q - (uint32_t)b * block_span);
        const int i = r / cur_out, k = r - i * cur_out;
        const int cur_in = b == in_blocks - 1 ? last_in : f.bpi;
        const int n = b < copy_blocks ? min(cur_in, cur_out) : 0;
        // fast path: the eight bytes sit in one channel's run and inside the region
        if (k + 8 <= cur_out && q + 8 <= region && i < ch) {
            uint2 v = make_uint2(0u, 0u);
            if (k < n) {
                v = *reinterpret_cast<const uint2 *>(adpcm + chans[f.first_ch + i].adpcm_off + (int64_t)f.bpi * b + k);
                const int valid = n - k;  // bytes of this word that exist in the source block
                if (valid < 8) {
                    const uint64_t m = valid <= 0 ? 0ull : (~0ull >> (8 * (8 - valid)));
                    uint64_t x = ((uint64_t)v.y << 32) | v.x;
                    x &= m;
                    v = make_uint2((uint32_t)x, (uint32_t)(x >> 32));
                }
            }
            *reinterpret_cast<uint2 *>(data + q) = v;
        } else {
            for (int j = 0; j < 8 && q + j < region; j++) {
                const int rr = r + j;
                const int ii = rr / cur_out, kk = rr - ii * cur_out;
                uint8_t byte = 0;
                if (ii < ch && kk < n) byte = adpcm[chans[f.first_ch + ii].adpcm_off + (int64_t)f.bpi * b + kk];
                data[q + j] = byte;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// ADX writer.  Tile 0 copies the host-built header (with the copyright tail) and writes the footer; the others
// interleave frames: thread = (frame, channel), frame_size bytes each, with CriAdxEncryption.EncryptDecryptChannel
// applied on the way (the key stream position of frame j of channel c is c + j * channels steps of the LCG).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kAdxFramesPerTile = 1024;

__global__ void __launch_bounds__(256) adx_assemble_kernel(const AdxFile *__restrict__ files, int n_files, const AdxChanRef *__restrict__ chans,
                                                            const uint8_t *__restrict__ adpcm, const uint8_t *__restrict__ hdr_blob,
                                                            uint8_t *__restrict__ out)
{
    const int fi = find_item(files, n_files, (int)blockIdx.x);
    const AdxFile f = files[fi];
    const int tile = (int)blockIdx.x - f.tile_first;
    uint8_t *dst = out + f.out_off;
    if (tile == 0) {
        // the header; bytes the sequential writer spills past AudioOffset are overwritten by the first frames, which
        // the data tiles own - so only [0, audio_offset) is written here
        for (int t = threadIdx.x; t < f.audio_offset; t += blockDim.x) dst[t] = hdr_blob[f.hdr_off + t];
        for (int t = threadIdx.x; t < f.footer_size; t += blockDim.x) {  // WriteFooter (AdxWriter.cs:135-140)
            const int pad = f.footer_size - 4;
            dst[f.footer_offset + t] = t == 0 ? 0x80 : t == 1 ? 0x01 : t == 2 ? (uint8_t)(pad >> 8) : t == 3 ? (uint8_t)pad : 0;
        }
        return;
    }
    const int ch = f.channels, fs = f.frame_size;
    const int64_t first = (int64_t)(tile - 1) * kAdxFramesPerTile;          // (frame, channel) pairs, frame-major
    const int64_t total = (int64_t)f.frame_count * ch;
    for (int t = threadIdx.x; t < kAdxFramesPerTile; t += blockDim.x) {
        const int64_t p = first + t;
        if (p >= total) break;
        const int j = (int)(p / ch), c = (int)(p - (int64_t)j * ch);
        uint8_t *o = dst + f.audio_offset + p * fs;
        if (j >= f.in_frames) {  // the interleave copies nothing here: the file keeps its zeros
            for (int k = 0; k < fs; k++) o[k] = 0;
            continue;
        }
        const uint8_t *s = adpcm + chans[f.first_ch + c].adpcm_off + (int64_t)j * fs;
        uint32_t any = 0;
        uint8_t b0 = s[0], b1 = s[1];
        if (((fs | f.audio_offset | (int)(f.out_off & 1)) & 1) == 0) {
            // even frame size and offsets (every standard file): halfword moves, half the memory instructions
            const uint16_t *s2 = reinterpret_cast<const uint16_t *>(s);
            uint16_t *o2 = reinterpret_cast<uint16_t *>(o);
            for (int k = 1; k < fs / 2; k++) { const uint16_t v = s2[k]; any |= v; o2[k] = v; }
        } else {
            for (int k = 2; k < fs; k++) { const uint8_t v = s[k]; any |= v; o[k] = v; }
        }
        if (f.has_key && (any | b0 | b1)) {  // FrameNotEmpty (CriAdxEncryption.cs:104-115)
            const int x = adx_key_at(f.seed, f.mult, f.inc, (uint32_t)p);
            b0 ^= (uint8_t)(x >> 8);
            if (f.enc_type == 9) b0 &= 0x1f;
            b1 ^= (uint8_t)x;
        }
        o[0] = b0;
        o[1] = b1;
    }
}

// The same-codec rewrite of .adx files (AdxReader -> AdxWriter without an encode): tile 0 as in adx_assemble_kernel,
// the others move kAdxFramesPerTile frames each from the source's interleaved region, thread = frame.  The scale bytes
// go through the source's key stream, then the output's, both at step p (CriAdxEncryption.cs:8-44), each behind its own
// FrameNotEmpty test: the decryption tests the bytes as read, the encryption the bytes as decrypted.  Frames past the
// source stay zero (Interleave.cs:43-78 copies nothing there) and are never encrypted.
__global__ void __launch_bounds__(256) adx_rewrite_kernel(const AdxRewriteFile *__restrict__ files, int n_files, const uint8_t *__restrict__ src,
                                                           const uint8_t *__restrict__ hdr_blob, uint8_t *__restrict__ out)
{
    const int fi = find_item(files, n_files, (int)blockIdx.x);
    const AdxRewriteFile f = files[fi];
    const int tile = (int)blockIdx.x - f.tile_first;
    uint8_t *dst = out + f.out_off;
    if (tile == 0) {
        for (int t = threadIdx.x; t < f.audio_offset; t += blockDim.x) dst[t] = hdr_blob[f.hdr_off + t];
        for (int t = threadIdx.x; t < f.footer_size; t += blockDim.x) {  // WriteFooter (AdxWriter.cs:135-140)
            const int pad = f.footer_size - 4;
            dst[f.footer_offset + t] = t == 0 ? 0x80 : t == 1 ? 0x01 : t == 2 ? (uint8_t)(pad >> 8) : t == 3 ? (uint8_t)pad : 0;
        }
        return;
    }
    const int fs = f.frame_size;
    const bool halves = ((fs | f.audio_offset | (int)(f.out_off & 1)) & 1) == 0;  // src_off is even
    const int first = (tile - 1) * kAdxFramesPerTile;
    for (int t = threadIdx.x; t < kAdxFramesPerTile; t += blockDim.x) {
        const int p = first + t;
        if (p >= f.frames) break;
        uint8_t *o = dst + f.audio_offset + (int64_t)p * fs;
        if (p >= f.src_frames) {
            for (int k = 0; k < fs; k++) o[k] = 0;
            continue;
        }
        const uint8_t *s = src + f.src_off + (int64_t)p * fs;
        uint32_t any = 0;
        uint8_t b0 = s[0], b1 = s[1];
        if (halves) {
            const uint16_t *s2 = reinterpret_cast<const uint16_t *>(s);
            uint16_t *o2 = reinterpret_cast<uint16_t *>(o);
            for (int k = 1; k < fs / 2; k++) { const uint16_t v = s2[k]; any |= v; o2[k] = v; }
        } else {
            for (int k = 2; k < fs; k++) { const uint8_t v = s[k]; any |= v; o[k] = v; }
        }
        if (f.dec_type && (any | b0 | b1)) {
            const int x = adx_key_at(f.dec_seed, f.dec_mult, f.dec_inc, (uint32_t)p);
            b0 ^= (uint8_t)(x >> 8);
            if (f.dec_type == 9) b0 &= 0x1f;
            b1 ^= (uint8_t)x;
        }
        if (f.has_key && (any | b0 | b1)) {
            const int x = adx_key_at(f.seed, f.mult, f.inc, (uint32_t)p);
            b0 ^= (uint8_t)(x >> 8);
            if (f.enc_type == 9) b0 &= 0x1f;
            b1 ^= (uint8_t)x;
        }
        o[0] = b0;
        o[1] = b1;
    }
}

// AdxWriter's version-4 history block (AdxWriter.cs:99-100): each channel's History, big-endian and twice, taken from the
// encoder's write-back (CriAdxCodec.cs:69-74) on the device; runs behind adx_assemble_kernel and patches the finished
// headers.  Thread = channel row.
struct AdxHistPatch {
    int64_t at;     // byte offset of the row's pair in the output slab
    int32_t bytes;  // how many of its 4 bytes the header keeps: the "(c)CRI" at header_size - 2 overwrites the rest, and
                    // a non-looping file's 36-byte header has no room for more than two channels' pairs (0: version 3)
    int32_t pad;
};
__global__ void adx_history_kernel(const AdxHistPatch *__restrict__ patch, const int16_t *__restrict__ history, int n_rows, uint8_t *__restrict__ out)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const AdxHistPatch p = patch[r];
    const uint32_t h = (uint16_t)history[r];
    for (int j = 0; j < p.bytes; j++) out[p.at + j] = (uint8_t)((j & 1) ? h : h >> 8);
}

// in-place EncryptDecrypt over channel rows (CriAdxEncryption.cs:8-44): thread = (frame, channel)
__global__ void adx_crypt_kernel(uint8_t *__restrict__ adpcm, const int64_t *__restrict__ row_off, int channels, int frames, int frame_size,
                                 int row_len, int seed, int mult, int inc, int enc_type)
{
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (int64_t)frames * channels) return;
    const int j = (int)(p / channels), c = (int)(p - (int64_t)j * channels);
    uint8_t *s = adpcm + row_off[c] + (int64_t)j * frame_size;
    const int n = min(frame_size, row_len - j * frame_size);  // a partial last frame would index past the array in the reference
    uint32_t any = 0;
    for (int k = 0; k < n; k++) any |= s[k];
    if (!any || n < 2) return;
    const int x = adx_key_at(seed, mult, inc, (uint32_t)p);
    uint8_t b0 = s[0] ^ (uint8_t)(x >> 8);
    if (enc_type == 9) b0 &= 0x1f;
    s[0] = b0;
    s[1] ^= (uint8_t)x;
}

// ---------------------------------------------------------------------------------------------------------------
// HCA writer: tile 0 copies the host-built header (CRC included); the others move frames, one WARP per frame.  With a
// key the bytes go through the substitution table and the frame's CRC-16 is recomputed (CriHcaEncryption.cs:21-33):
// each lane runs the table-driven CRC over its slice, slices are joined by crc(A||B) = shift(crc(A), |B|) ^ crc(B).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kHcaFramesPerTile = 8;  // = warps per CTA

__device__ __forceinline__ uint16_t crc16_byte(const uint16_t *tab, uint16_t crc, uint8_t v) { return (uint16_t)((crc << 8) ^ tab[(crc >> 8) ^ v]); }

__global__ void __launch_bounds__(kHcaFramesPerTile * 32) hca_assemble_kernel(const HcaFile *__restrict__ files, int n_files,
                                                                               const uint8_t *__restrict__ frames, const uint8_t *__restrict__ hdr_blob,
                                                                               const uint8_t *__restrict__ sub_table /* null: no key */,
                                                                               uint8_t *__restrict__ out)
{
    __shared__ uint16_t crc_tab[256];
    __shared__ uint8_t sub[256];
    for (int i = threadIdx.x; i < 256 && sub_table; i += blockDim.x) {
        uint16_t v = (uint16_t)(i << 8);                        // Crc16 table, polynomial 0x8005 (Utilities/Crc16.cs)
        for (int k = 0; k < 8; k++) v = (uint16_t)((v & 0x8000) ? (v << 1) ^ 0x8005 : v << 1);
        crc_tab[i] = v;
        sub[i] = sub_table[i];
    }
    __syncthreads();
    const int fi = find_item(files, n_files, (int)blockIdx.x);
    const HcaFile f = files[fi];
    const int tile = (int)blockIdx.x - f.tile_first;
    uint8_t *dst = out + f.out_off;
    if (tile == 0) {
        for (int t = threadIdx.x; t < f.header_size; t += blockDim.x) dst[t] = hdr_blob[f.hdr_off + t];
        return;
    }
    if (!sub_table) {  // no key: the frames are one contiguous run behind the header - 16 KB of it per tile
        const int64_t total = (int64_t)f.frame_size * f.frame_count;
        const int64_t q0 = (int64_t)(tile - 1) * kTileBytes;
        const int nb = (int)min((int64_t)kTileBytes, total - q0);
        const uint8_t *s = frames + f.frames_off + q0;            // 16-byte aligned (frames_off is, q0 is)
        uint8_t *o = dst + f.header_size + q0;
        if (((f.out_off + f.header_size) & 15) == 0) {
            const int n_vec = nb >> 4;
            for (int v = threadIdx.x; v < n_vec; v += blockDim.x) reinterpret_cast<uint4 *>(o)[v] = reinterpret_cast<const uint4 *>(s)[v];
            for (int k = (n_vec << 4) + threadIdx.x; k < nb; k += blockDim.x) o[k] = s[k];
        } else {  // header sizes of looping files are not multiples of 16: aligned loads, byte stores
            for (int v = threadIdx.x; v < (nb + 15) >> 4; v += blockDim.x) {
                const uint4 x = reinterpret_cast<const uint4 *>(s)[v];
                const uint32_t wds[4] = {x.x, x.y, x.z, x.w};
                for (int k = 0; k < 16 && v * 16 + k < nb; k++) o[v * 16 + k] = (uint8_t)(wds[k >> 2] >> (8 * (k & 3)));
            }
        }
        return;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int fr = (tile - 1) * kHcaFramesPerTile + warp;
    if (fr >= f.frame_count) return;
    const uint8_t *s = frames + f.frames_off + (int64_t)fr * f.frame_size;
    uint8_t *o = dst + f.header_size + (int64_t)fr * f.frame_size;
    const int body = f.frame_size - 2;
    const int chunk = (body + 31) / 32;
    const int lo = min(lane * chunk, body), hi = min(lo + chunk, body);
    uint16_t crc = 0;
    for (int k = lo; k < hi; k++) {
        const uint8_t v = sub[s[k]];
        o[k] = v;
        crc = crc16_byte(crc_tab, crc, v);
    }
    // join: lane l absorbs lane l+d's slice (|slice| = bytes between the two lanes' ends)
    int len = hi - lo;  // bytes covered by this lane's crc
    for (int d = 1; d < 32; d <<= 1) {
        const uint16_t other = (uint16_t)__shfl_down_sync(0xFFFFFFFFu, (int)crc, d);
        const int other_len = __shfl_down_sync(0xFFFFFFFFu, len, d);
        if ((lane & (2 * d - 1)) == 0 && lane + d < 32) {
            for (int k = 0; k < other_len; k++) crc = crc16_byte(crc_tab, crc, 0);  // shift by |B| zero bytes
            crc ^= other;
            len += other_len;
        }
    }
    if (lane == 0) { o[body] = (uint8_t)(crc >> 8); o[body + 1] = (uint8_t)crc; }
}

// ---------------------------------------------------------------------------------------------------------------
// NintendoWare stream writers (BrstmWriter.cs, BCFstmWriter.cs).  Tile 0 of a file copies the host-built header
// (everything in front of the audio data: RSTM/HEAD/ADPC/DATA or header/INFO/SEEK/DATA, device fields zero) and, for
// GC-ADPCM, patches what only the device has: each channel's coefficients, its start context (predictor/scale of frame
// 0, zero history) and loop context (GcAdpcmLoopContext.cs:17-26 at the loop start, or the start context when the
// stream does not loop), and the seek table (GcAdpcmSeekTable.cs:25-38, interleaved per entry and resized to the
// writer's entry count, GcAdpcmFormat.BuildSeekTable).  The other tiles write 16 KB of the data region each, with
// InterleaveExtensions.Interleave's block layout (Interleave.cs:43-78) from the channel arrays the writer hands it:
// GC-ADPCM rows (GcAdpcmAlignment.AdpcmAligned when the loop was aligned: the kept frames of the encoded row, then the
// re-encoded tail), PCM16 in the file's byte order, PCM8 as (byte)(s >> 8) (Pcm8Codec.EncodeSigned).  InterleaveSize is
// always 0x2000 and every block ends on a multiple of 32 bytes, so an 8-byte word never straddles two channel runs.
// ---------------------------------------------------------------------------------------------------------------
struct NwChan {
    int64_t row_off;         // GC-ADPCM: bytes into the ADPCM slab (multiple of 16); PCM: samples into the PCM slab (multiple of 8)
    int64_t pcm_off;         // GC-ADPCM: samples into the decoded-PCM slab (the channel decoded in full)
    int64_t tail_off;        // GC-ADPCM, aligned loop: bytes of the re-encoded tail into the tail slab (multiple of 16)
    int32_t coef_index;
    int32_t start_hist;      // GC-ADPCM: the start context's Hist1 | Hist2 << 16 (0 for an encoded channel; a rewrite keeps the source's)
};
struct NwFile {
    int64_t out_off;         // bytes into the output slab (multiple of 16)
    int64_t hdr_off;         // bytes into the header blob
    int32_t hdr_size;        // AudioDataOffset (a multiple of 32)
    int32_t channels, first_ch;
    int32_t codec;           // NwCodec: 0 PCM8, 1 PCM16, 2 GC-ADPCM
    int32_t big_endian;      // byte order of the coefficients, contexts and PCM16 samples
    int32_t in_size;         // bytes of each channel's array (the whole encoded or converted channel, or AdpcmAligned)
    int32_t keep_bytes;      // bytes of that array taken from the encoded row; the rest is the aligned tail (a multiple of 8)
    int32_t data_size;       // AudioDataSize
    int32_t bpi;             // InterleaveSize
    int32_t info_off;        // GC-ADPCM: file offset of channel 0's coefficients
    int32_t info_stride;     // bytes between two channels' coefficients
    int32_t ctx_off;         // start context relative to the coefficients (behind BRSTM's gain)
    int32_t looping, loop_start;  // loop_start: where the loop context is taken (the unaligned loop start, see nw_plan_target)
    int32_t seek_off;        // file offset of the first seek entry
    int32_t seek_entries;    // SeekTableEntryCount (the resized table)
    int32_t chan_entries;    // entries GcAdpcmSeekTable computes from the channel's own length
    int32_t seek_spe, seek_be;
    int32_t tile_first, pad;
};

__device__ __forceinline__ void put16(uint8_t *p, int v, bool be)
{
    if (be) { p[0] = (uint8_t)(v >> 8); p[1] = (uint8_t)v; }
    else { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); }
}

__global__ void __launch_bounds__(256) nw_assemble_kernel(const NwFile *__restrict__ files, int n_files, const NwChan *__restrict__ chans,
                                                           const uint8_t *__restrict__ hdr_blob, const uint8_t *__restrict__ adpcm,
                                                           const uint8_t *__restrict__ tail,
                                                           const int16_t *__restrict__ coefs, const int16_t *__restrict__ decoded,
                                                           const int16_t *__restrict__ pcm, uint8_t *__restrict__ out)
{
    const int fi = find_item(files, n_files, (int)blockIdx.x);
    const NwFile f = files[fi];
    const int tile = (int)blockIdx.x - f.tile_first;
    uint8_t *dst = out + f.out_off;
    const int ch = f.channels;
    if (tile == 0) {
        for (int t = threadIdx.x; t < f.hdr_size; t += blockDim.x) dst[t] = hdr_blob[f.hdr_off + t];
        if (f.codec != 2) return;
        __syncthreads();
        const bool be = f.big_endian != 0;
        for (int t = threadIdx.x; t < ch * 22; t += blockDim.x) {  // 16 coefficients and 2 x 3 context halfwords per channel
            const int c = t / 22, h = t - c * 22;
            const NwChan cc = chans[f.first_ch + c];
            uint8_t *info = dst + f.info_off + c * f.info_stride;
            if (h < 16) { put16(info + 2 * h, coefs[(int64_t)cc.coef_index * 16 + h], be); continue; }
            const int k = h - 16;                  // 0..2 start context, 3..5 loop context
            const bool loop_ctx = k >= 3 && f.looping;
            const int ls = f.loop_start;
            int v = 0;
            switch (loop_ctx ? k - 3 : k % 3) {
            case 0: v = loop_ctx ? adpcm[cc.row_off + (int64_t)(ls / kGcFrameSamples) * kGcFrameBytes] : adpcm[cc.row_off]; break;
            case 1: v = loop_ctx ? (ls >= 1 ? decoded[cc.pcm_off + ls - 1] : 0) : (int16_t)(cc.start_hist & 0xffff); break;
            default: v = loop_ctx ? (ls >= 2 ? decoded[cc.pcm_off + ls - 2] : 0) : (int16_t)((uint32_t)cc.start_hist >> 16); break;
            }
            put16(info + f.ctx_off + 2 * k, v, be);
        }
        const int n_words = f.seek_entries * ch;   // one (hist1, hist2) pair per entry and channel, entry-major
        for (int t = threadIdx.x; t < n_words; t += blockDim.x) {
            const int j = t / ch, c = t - j * ch;
            int h1 = 0, h2 = 0;
            if (j >= 1 && j < f.chan_entries) {   // entry 0 is always zero; entries past the channel's own table are Array.Resize's zeros
                const int64_t at = chans[f.first_ch + c].pcm_off + (int64_t)j * f.seek_spe;
                h1 = decoded[at - 1];
                h2 = decoded[at - 2];
            }
            put16(dst + f.seek_off + 4 * t, h1, f.seek_be != 0);
            put16(dst + f.seek_off + 4 * t + 2, h2, f.seek_be != 0);
        }
        return;
    }
    uint8_t *data = dst + f.hdr_size;
    const uint32_t region = (uint32_t)f.data_size * (uint32_t)ch;  // a file is below 2 GiB (FileSize is an int)
    const uint32_t q0 = (uint32_t)(tile - 1) * kTileBytes;
    const int in_blocks = div_round_up(f.in_size, f.bpi), out_blocks = div_round_up(f.data_size, f.bpi);
    const int last_in = f.in_size - (in_blocks - 1) * f.bpi, last_out = f.data_size - (out_blocks - 1) * f.bpi;
    const int copy_blocks = min(in_blocks, out_blocks);
    const uint32_t block_span = (uint32_t)f.bpi * (uint32_t)ch;
#pragma unroll 4
    for (int w = threadIdx.x; w < kTileBytes / 8; w += blockDim.x) {
        const uint32_t q = q0 + (uint32_t)w * 8;
        if (q >= region) break;
        int b = (int)(q / block_span);
        if (b > out_blocks - 1) b = out_blocks - 1;
        const int cur_out = b == out_blocks - 1 ? last_out : f.bpi;
        const int r = (int)(q - (uint32_t)b * block_span);
        const int i = r / cur_out, k = r - i * cur_out;
        const int cur_in = b == in_blocks - 1 ? last_in : f.bpi;
        const int n = b < copy_blocks ? min(cur_in, cur_out) : 0;
        uint2 v = make_uint2(0u, 0u);
        if (k < n) {
            const int64_t pos = (int64_t)f.bpi * b + k;  // byte of channel i's array (a multiple of 8)
            const NwChan cc = chans[f.first_ch + i];
            if (f.codec == 2) {
                v = pos < f.keep_bytes ? *reinterpret_cast<const uint2 *>(adpcm + cc.row_off + pos)
                                       : *reinterpret_cast<const uint2 *>(tail + cc.tail_off + (pos - f.keep_bytes));
            } else if (f.codec == 1) {
                v = *reinterpret_cast<const uint2 *>(pcm + cc.row_off + pos / 2);
                if (f.big_endian) v = make_uint2(__byte_perm(v.x, 0, 0x2301), __byte_perm(v.y, 0, 0x2301));
            } else {
                const uint4 s = *reinterpret_cast<const uint4 *>(pcm + cc.row_off + pos);
                v = make_uint2(__byte_perm(s.x, s.y, 0x7531), __byte_perm(s.z, s.w, 0x7531));
            }
            const int valid = n - k;
            if (valid < 8) {
                uint64_t x = ((uint64_t)v.y << 32) | v.x;
                x &= ~0ull >> (8 * (8 - valid));
                v = make_uint2((uint32_t)x, (uint32_t)(x >> 32));
            }
        }
        *reinterpret_cast<uint2 *>(data + q) = v;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// IDSP and HPS writers (IdspWriter.cs, HpsWriter.cs), big-endian GC-ADPCM containers.  Their channels are rows of
// NwChan, as for the NintendoWare writer: the array each writer hands on is GetAdpcmAudio(), the encoded row, or when the
// loop moved, its kept frames followed by the re-encoded tail (keep_bytes, a multiple of 8, so an 8-byte word never
// straddles the two).  Tile 0 of a file copies the host-built header and patches what only the device has; the other
// tiles write 16 KB of the rest each.
// ---------------------------------------------------------------------------------------------------------------
struct IdspFile {
    int64_t out_off;         // bytes into the output slab (multiple of 16)
    int64_t hdr_off;         // bytes into the header blob
    int32_t hdr_size;        // HeaderSize = 0x40 + 0x60 * channels
    int32_t channels, first_ch;
    int32_t in_size;         // bytes of each channel's array
    int32_t keep_bytes;      // bytes of that array taken from the encoded row
    int32_t data_size;       // AudioDataSize (a multiple of the 16-byte interleave)
    int32_t ctx_loop_start;  // where the loop context is taken (the unaligned loop start); -1: the header blob's context stays
    int32_t tile_first;
};
struct HpsBlock {
    int32_t at;              // file offset of the block (BlockInfo.Offset)
    int32_t start_sample, byte_in, chan_size;  // StartSample, ByteInIndex (a multiple of 32), ChannelSize
    int32_t written, end_nibble, next;         // WrittenSize, EndNibble, NextOffset
    int32_t pad;
};
struct HpsFile {
    int64_t out_off, hdr_off;
    int32_t hdr_size;        // HeaderSize
    int32_t channels, first_ch;
    int32_t keep_bytes;
    int32_t block_hdr;       // bytes in front of a block's audio: GetNextMultiple(12 + 8 * channels, 0x20)
    int32_t first_block, n_blocks;
    int32_t file_size;
    int32_t tile_first;
    int32_t no_hist;         // the channels' Pcm is null (a rewrite that never decoded before the loop moved): block histories 0
};

__device__ __forceinline__ void put16be(uint8_t *p, int v) { p[0] = (uint8_t)(v >> 8); p[1] = (uint8_t)v; }

// byte `pos` of a channel's array
__device__ __forceinline__ int gc_array_byte(const NwChan &cc, int64_t pos, int keep_bytes, const uint8_t *adpcm, const uint8_t *tail)
{
    return pos < keep_bytes ? adpcm[cc.row_off + pos] : tail[cc.tail_off + (pos - keep_bytes)];
}

// the 8 bytes of a channel's array from `pos` (a multiple of 8), those from `valid` on zero
__device__ __forceinline__ uint2 gc_array_word(const NwChan &cc, int64_t pos, int keep_bytes, const uint8_t *adpcm, const uint8_t *tail, int valid)
{
    uint2 v = pos < keep_bytes ? *reinterpret_cast<const uint2 *>(adpcm + cc.row_off + pos)
                               : *reinterpret_cast<const uint2 *>(tail + cc.tail_off + (pos - keep_bytes));
    if (valid < 8) {
        uint64_t x = ((uint64_t)v.y << 32) | v.x;
        x &= ~0ull >> (8 * (8 - valid));
        v = make_uint2((uint32_t)x, (uint32_t)(x >> 32));
    }
    return v;
}

// IdspWriter: per channel the coefficients, the start context's predictor/scale (Adpcm[0]; its history is in the header
// blob) and the loop context (the first encode's, at the unaligned loop start, or the blob's), then Interleave(16,
// AudioDataSize) (Interleave.cs:43-73):
// AudioDataSize is a multiple of 16, so every block is whole and byte `pos` of a channel is in the file iff pos < in_size.
__global__ void __launch_bounds__(256) idsp_assemble_kernel(const IdspFile *__restrict__ files, int n_files, const NwChan *__restrict__ chans,
                                                             const uint8_t *__restrict__ hdr_blob, const uint8_t *__restrict__ adpcm,
                                                             const uint8_t *__restrict__ tail, const int16_t *__restrict__ coefs,
                                                             const int16_t *__restrict__ decoded, uint8_t *__restrict__ out)
{
    const int fi = find_item(files, n_files, (int)blockIdx.x);
    const IdspFile f = files[fi];
    const int tile = (int)blockIdx.x - f.tile_first;
    uint8_t *dst = out + f.out_off;
    const int ch = f.channels;
    if (tile == 0) {
        for (int t = threadIdx.x; t < f.hdr_size; t += blockDim.x) dst[t] = hdr_blob[f.hdr_off + t];
        __syncthreads();
        const int ls = f.ctx_loop_start;
        for (int t = threadIdx.x; t < ch * 20; t += blockDim.x) {  // 16 coefficients, the start predictor/scale, 3 loop context halfwords
            const int c = t / 20, h = t - c * 20;
            const NwChan cc = chans[f.first_ch + c];
            uint8_t *info = dst + 0x40 + 0x60 * c;
            if (h < 16) put16be(info + 0x1c + 2 * h, coefs[(int64_t)cc.coef_index * 16 + h]);
            else if (h == 16) put16be(info + 0x3e, adpcm[cc.row_off]);
            else if (ls >= 0) {
                const int k = h - 17;
                const int v = k == 0 ? adpcm[cc.row_off + (int64_t)(ls / kGcFrameSamples) * kGcFrameBytes]
                                     : ls >= k ? decoded[cc.pcm_off + ls - k] : 0;
                put16be(info + 0x44 + 2 * k, v);
            }
        }
        return;
    }
    uint8_t *data = dst + f.hdr_size;
    const uint32_t region = (uint32_t)f.data_size * (uint32_t)ch;
    const uint32_t q0 = (uint32_t)(tile - 1) * kTileBytes;
    const uint32_t block_span = 16u * (uint32_t)ch;
#pragma unroll 4
    for (int w = threadIdx.x; w < kTileBytes / 8; w += blockDim.x) {
        const uint32_t q = q0 + (uint32_t)w * 8;
        if (q >= region) break;
        const uint32_t b = q / block_span, r = q - b * block_span;
        const int64_t pos = (int64_t)b * 16 + (r & 15);
        const int valid = f.in_size - (int)pos;
        uint2 v = make_uint2(0u, 0u);
        if (valid > 0) v = gc_array_word(chans[f.first_ch + (int)(r >> 4)], pos, f.keep_bytes, adpcm, tail, valid);
        *reinterpret_cast<uint2 *>(data + q) = v;
    }
}

// HpsWriter: per channel the coefficients and the start context's predictor/scale; per block (WriteBlock) WrittenSize,
// EndNibble, NextOffset and per channel (predictor/scale of GetAdpcmAudio() at StartSample, Hist1 and Hist2 from the
// first encode's full decode, 0), then each channel's ChannelSize bytes, every part padded to 0x20.  Tile 0 writes the
// headers, the other tiles the audio of the blocks.
__global__ void __launch_bounds__(256) hps_assemble_kernel(const HpsFile *__restrict__ files, int n_files, const HpsBlock *__restrict__ blocks,
                                                            const NwChan *__restrict__ chans, const uint8_t *__restrict__ hdr_blob,
                                                            const uint8_t *__restrict__ adpcm, const uint8_t *__restrict__ tail,
                                                            const int16_t *__restrict__ coefs, const int16_t *__restrict__ decoded,
                                                            uint8_t *__restrict__ out)
{
    const int fi = find_item(files, n_files, (int)blockIdx.x);
    const HpsFile f = files[fi];
    const int tile = (int)blockIdx.x - f.tile_first;
    uint8_t *dst = out + f.out_off;
    const int ch = f.channels;
    const HpsBlock *B = blocks + f.first_block;
    if (tile == 0) {
        for (int t = threadIdx.x; t < f.hdr_size; t += blockDim.x) dst[t] = hdr_blob[f.hdr_off + t];
        __syncthreads();
        for (int t = threadIdx.x; t < ch * 17; t += blockDim.x) {  // 16 coefficients and the start predictor/scale
            const int c = t / 17, h = t - c * 17;
            const NwChan cc = chans[f.first_ch + c];
            uint8_t *info = dst + 0x10 + 0x38 * c;
            put16be(info + (h < 16 ? 0x10 + 2 * h : 0x32), h < 16 ? coefs[(int64_t)cc.coef_index * 16 + h] : adpcm[cc.row_off]);
        }
        const int halves = f.block_hdr / 2;
        for (int t = threadIdx.x; t < f.n_blocks * halves; t += blockDim.x) {
            const int bi = t / halves, j = 2 * (t - bi * halves);
            const HpsBlock blk = B[bi];
            int v = 0;
            if (j < 12) {
                const int word = j < 4 ? blk.written : j < 8 ? blk.end_nibble : blk.next;
                v = (j & 2) ? word & 0xffff : (int)((uint32_t)word >> 16);
            } else if (j < 12 + 8 * ch) {
                const int c = (j - 12) >> 3, m = ((j - 12) & 7) >> 1;
                const NwChan cc = chans[f.first_ch + c];
                const int s = blk.start_sample;
                if (m == 0) v = gc_array_byte(cc, blk.byte_in, f.keep_bytes, adpcm, tail);
                else if (m < 3 && s >= m && !f.no_hist) v = decoded[cc.pcm_off + s - m];
            }
            put16be(dst + blk.at + j, v);
        }
        return;
    }
    const int q0 = f.hdr_size + (tile - 1) * kTileBytes;
#pragma unroll 4
    for (int w = threadIdx.x; w < kTileBytes / 8; w += blockDim.x) {
        const int q = q0 + w * 8;
        if (q >= f.file_size) break;
        int lo = 0, hi = f.n_blocks - 1;  // the last block at or before q
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (B[mid].at <= q) lo = mid; else hi = mid - 1;
        }
        const HpsBlock blk = B[lo];
        int r = q - blk.at - f.block_hdr;
        if (r < 0) continue;  // the block's header: tile 0
        const int cpad = (blk.chan_size + 31) & ~31;
        const int i = r / cpad, k = r - i * cpad;
        const int valid = blk.chan_size - k;
        uint2 v = make_uint2(0u, 0u);
        if (valid > 0) v = gc_array_word(chans[f.first_ch + i], (int64_t)blk.byte_in + k, f.keep_bytes, adpcm, tail, valid);
        *reinterpret_cast<uint2 *>(dst + q) = v;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// host state of this translation unit: its own slabs and streams per context (Context::containers), so a converter call
// sharded over several devices gives every worker its own on that worker's device
// ---------------------------------------------------------------------------------------------------------------
constexpr int kWays = 4;  // groups of the batch converter in flight: each has its own working set and kernel stream

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// HPS block pieces -> channel rows (HpsReader.ToAudioStream, Containers/Hps/HpsReader.cs:37-50: each channel's audio is
// the concatenation of its pieces of every block).  One CTA per kHpsGatherTile bytes of one piece.  Hostile chains give
// pieces of any length at any byte of the image and of the row; writer-made files give whole frames at 0x20 multiples on
// both sides.  So each tile copies with the widest word the common alignment of its source and destination allows
// (16, 8 or 4 bytes), byte-wise up to the first aligned address and behind the last whole word, and byte-wise
// throughout when source and destination disagree below 4 bytes.
// ---------------------------------------------------------------------------------------------------------------
namespace vgb {

template <class W>
__device__ __forceinline__ void gather_words(const uint8_t *src, uint8_t *dst, int n)
{
    constexpr int kW = (int)sizeof(W);
    const int head = min(n, (int)((kW - ((uintptr_t)dst & (kW - 1))) & (kW - 1)));
    for (int k = threadIdx.x; k < head; k += blockDim.x) dst[k] = src[k];
    const int words = (n - head) / kW;
    const W *s = reinterpret_cast<const W *>(src + head);
    W *d = reinterpret_cast<W *>(dst + head);
#pragma unroll 4
    for (int k = threadIdx.x; k < words; k += blockDim.x) d[k] = s[k];
    for (int k = head + words * kW + threadIdx.x; k < n; k += blockDim.x) dst[k] = src[k];
}

__global__ void __launch_bounds__(256) hps_gather_kernel(const uint8_t *__restrict__ in, const HpsPiece *__restrict__ pieces, int n_pieces,
                                                          uint8_t *__restrict__ rows)
{
    const int it = find_item(pieces, n_pieces, (int)blockIdx.x);
    const HpsPiece p = pieces[it];
    const int b0 = ((int)blockIdx.x - p.tile_first) * kHpsGatherTile;
    const int n = min(kHpsGatherTile, p.len - b0);
    if (n <= 0) return;
    const uint8_t *src = in + p.src_off + b0;
    uint8_t *dst = rows + p.dst_off + b0;
    const unsigned mis = (unsigned)((uintptr_t)src ^ (uintptr_t)dst);
    if ((mis & 15) == 0) gather_words<uint4>(src, dst, n);
    else if ((mis & 7) == 0) gather_words<uint2>(src, dst, n);
    else if ((mis & 3) == 0) gather_words<uint32_t>(src, dst, n);
    else gather_words<uint8_t>(src, dst, n);
}

}  // namespace vgb

namespace vgb {
// Created on the context's device, used and freed with that device current.  Lock order: ContainerState::mu before
// Context::mu (the *_dev codec calls a converter group makes take the latter).
struct ContainerState {
    std::mutex mu;
    bool ready = false;
    cudaStream_t s_in = nullptr, s_out = nullptr, s_kern[kWays] = {};
    cudaStream_t s_k = nullptr;  // = s_kern[0]: the stream of the single-shot entry points
    cudaEvent_t ev_in[kWays] = {}, ev_split[kWays] = {}, ev_k[kWays] = {}, ev_out[kWays] = {};
    // working set 0 doubles as the single-shot entry points' and the .dsp -> WAVE converter's
    DevBuf in[kWays], out[kWays], tab[kWays], pcms[kWays], encs[kWays], decs[kWays], coefss[kWays], wss[kWays];
    // vgb_transcode_batch's source side: de-interleaved coded rows and the decoder's workspace, whose status words are
    // read after the next group is enqueued, so no encoder may reuse it before then
    DevBuf srcs[kWays], dws[kWays];
    // stage timers of the batch converter: per group 5 events (start, split done, encode done, context done, assembled)
    static constexpr int kTimedGroups = 32, kStageEvents = 5;
    cudaEvent_t stage[kTimedGroups][kStageEvents] = {};
    int timed_groups = 0;
};
}  // namespace vgb

namespace {

using State = vgb::ContainerState;

State &state_of(Context &c)
{
    State *s = c.containers.load(std::memory_order_acquire);
    if (s) return *s;
    std::lock_guard<std::mutex> lock(c.mu);  // the only place that takes Context::mu before a State exists
    s = c.containers.load(std::memory_order_relaxed);
    if (!s) {
        s = new State();
        c.containers.store(s, std::memory_order_release);
    }
    return *s;
}

// the container state of the context this thread works on: the primary's on a caller thread, a worker's own in a
// sharded converter call (as g_ctx is for the codec calls)
#define g_st (state_of(g_ctx))

// readies g_ctx, makes its device current and creates the state's streams and events there; g_st.mu is held
int32_t ensure_state()
{
    VGB_TRY(vgb::abi_ensure_ready());
    if (g_st.ready) return VGB_OK;
    CUDA_TRY(cudaStreamCreateWithFlags(&g_st.s_in, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&g_st.s_out, cudaStreamNonBlocking));
    for (int i = 0; i < kWays; i++) {
        CUDA_TRY(cudaStreamCreateWithFlags(&g_st.s_kern[i], cudaStreamNonBlocking));
        CUDA_TRY(cudaEventCreateWithFlags(&g_st.ev_in[i], cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&g_st.ev_split[i], cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&g_st.ev_k[i], cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&g_st.ev_out[i], cudaEventDisableTiming));
    }
    g_st.s_k = g_st.s_kern[0];
    for (auto &grp : g_st.stage) for (auto &e : grp) CUDA_TRY(cudaEventCreate(&e));
    g_st.ready = true;
    return VGB_OK;
}

void drain_state(State &s)  // with s's device current
{
    if (!s.ready) return;
    cudaStreamSynchronize(s.s_in);
    for (auto st : s.s_kern) cudaStreamSynchronize(st);
    cudaStreamSynchronize(s.s_out);
    (void)cudaGetLastError();
}

struct Drain {  // no copy may be in flight on caller memory once an entry point (or a converter worker) returns
    ~Drain() { drain_state(g_st); }
};

void be16(uint8_t *p, int v) { p[0] = (uint8_t)(v >> 8); p[1] = (uint8_t)v; }
void be32(uint8_t *p, int32_t v) { be16(p, (int)((uint32_t)v >> 16)); be16(p + 2, (int)((uint32_t)v & 0xffff)); }
int32_t rd_le32(const uint8_t *p) { return (int32_t)((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24)); }
int rd_le16(const uint8_t *p) { return p[0] | (p[1] << 8); }
int rd_be16s(const uint8_t *p) { return (int16_t)((p[0] << 8) | p[1]); }
int32_t rd_be32(const uint8_t *p) { return (int32_t)(((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3]); }

// ---- DSP geometry (DspWriter.cs:17-36, :105-106) ----
struct DspGeom { int align, loop_start, loop_end, sample_count, data_size, bpi, in_size; };
int32_t dsp_geometry(const vgb_dsp_desc &d, DspGeom &g, int index)
{
    if (d.channel_count < 1 || d.channel_count > 255) return fail(VGB_E_ARG, "file %d: channel_count %d outside 1..255", index, d.channel_count);
    if (d.sample_count < 0) return fail(VGB_E_ARG, "file %d: negative sample count", index);
    const int spi = d.samples_per_interleave == 0 ? 0x3800 : d.samples_per_interleave;
    if (spi < 1 || spi % 14 != 0)  // DspConfiguration.cs:29-44
        return fail(VGB_E_ARG, "file %d: samples per interleave (%d) must be positive and divisible by 14", index, spi);
    const int lpa = d.loop_point_alignment == 0 ? 1 : d.loop_point_alignment;
    if (d.looping && (d.loop_start < 0 || d.loop_end < d.loop_start || d.loop_end > d.sample_count))
        return fail(VGB_E_ARG, "file %d: loop points %d..%d outside 0..%d", index, d.loop_start, d.loop_end, d.sample_count);
    g.align = next_multiple(d.loop_start, lpa) - d.loop_start;
    g.loop_start = d.loop_start + g.align;
    g.loop_end = d.loop_end + g.align;
    g.sample_count = (!d.no_trim && d.looping) ? g.loop_end : std::max(d.sample_count, g.loop_end);
    g.in_size = gc_sample_count_to_byte_count(d.sample_count);
    g.data_size = next_multiple(gc_sample_count_to_byte_count(g.sample_count), d.channel_count == 1 ? 1 : 8);
    g.bpi = gc_sample_count_to_byte_count(spi);
    // mono: Stream.Write(array, 0, count) with count past the array throws ArgumentException (DspWriter.cs:91)
    if (d.channel_count == 1 && gc_sample_count_to_byte_count(g.sample_count) > g.in_size)
        return fail(VGB_E_ARG, "file %d: the aligned loop end (%d) lies past the encoded audio (%d samples)", index, g.loop_end, d.sample_count);
    return VGB_OK;
}

// ---- ADX geometry (AdxWriter.cs:18-36, :57-68) ----
int adx_bytes(int samples, int frame_size)  // CriAdxHelpers.SampleCountToByteCount
{
    const int npf = frame_size * 2, spf = npf - 4, extra = samples % spf;
    return (npf * (samples / spf) + (extra == 0 ? 0 : extra + 4) + 1) / 2;
}
struct AdxGeom { int sample_count, frame_count, base_header, alignment_bytes, header_size, audio_offset, audio_size, footer_offset, footer_size, loop_start, loop_end; };
int32_t adx_geometry(const vgb_adx_desc &d, AdxGeom &g, int index)
{
    if (d.channel_count < 1 || d.channel_count > 255) return fail(VGB_E_ARG, "file %d: channel_count %d outside 1..255", index, d.channel_count);
    if (d.frame_size < 3 || d.frame_size > 255) return fail(VGB_E_ARG, "file %d: frame_size %d outside 3..255", index, d.frame_size);
    if (d.sample_count < 0 || d.alignment_samples < 0) return fail(VGB_E_ARG, "file %d: negative count", index);
    const int spf = (d.frame_size - 2) * 2;
    g.loop_start = d.loop_start + d.alignment_samples;
    g.loop_end = d.loop_end + d.alignment_samples;
    g.sample_count = (!d.no_trim && d.looping) ? g.loop_end + spf * 3 : d.sample_count + d.alignment_samples;
    g.frame_count = (int)(((int64_t)g.sample_count + spf - 1) / spf);
    g.base_header = d.looping ? (d.version == 4 ? 60 : 52) : (d.version == 4 ? 36 : 32);
    g.alignment_bytes = 0;
    if (d.looping) {
        const int off = adx_bytes(g.loop_start, d.frame_size) * d.channel_count + g.base_header + 4;
        g.alignment_bytes = next_multiple(off, 0x800) - off;
        if (d.version == 3) g.alignment_bytes += d.alignment_samples / spf * 0x800;
    }
    g.header_size = g.base_header + g.alignment_bytes;
    g.audio_offset = g.header_size + 4;
    g.audio_size = d.frame_size * g.frame_count * d.channel_count;
    g.footer_offset = g.audio_offset + g.audio_size;
    g.footer_size = d.looping ? next_multiple(g.footer_offset + d.frame_size, 0x800) - g.footer_offset : d.frame_size;
    return VGB_OK;
}
// WriteHeader (AdxWriter.cs:80-119) into `h` (header_size + 4 bytes... the sequential writer may run past that for
// non-looping files; those bytes belong to the first audio frames and are dropped here)
void adx_build_header(const vgb_adx_desc &d, const AdxGeom &g, const int16_t *history, std::vector<uint8_t> &h)
{
    h.assign((size_t)g.audio_offset + 64 + 4 * (size_t)d.channel_count, 0);
    uint8_t *p = h.data();
    be16(p, 0x8000); be16(p + 2, g.header_size); p[4] = (uint8_t)d.type; p[5] = (uint8_t)d.frame_size; p[6] = 4; p[7] = (uint8_t)d.channel_count;
    be32(p + 8, d.sample_rate); be32(p + 12, g.sample_count);
    be16(p + 16, d.type != 2 ? d.highpass_frequency : 0);
    p[18] = (uint8_t)d.version; p[19] = (uint8_t)d.encryption_type;
    p += 20;
    if (d.version == 4) {
        p += 4;
        for (int i = 0; i < d.channel_count; i++) { const int hv = history ? history[i] : 0; be16(p, hv); be16(p + 2, hv); p += 4; }
        if (d.channel_count == 1) p += 4;
    }
    be16(p, d.alignment_samples); be16(p + 2, d.looping ? 1 : 0); be32(p + 4, d.looping ? 1 : 0);
    be32(p + 8, g.loop_start);
    be32(p + 12, g.audio_offset + adx_bytes(g.loop_start, d.frame_size) * d.channel_count);
    be32(p + 16, g.loop_end);
    be32(p + 20, g.audio_offset + next_multiple(adx_bytes(g.loop_end, d.frame_size), d.frame_size) * d.channel_count);
    std::memcpy(h.data() + g.header_size - 2, "(c)CRI", 6);
    h.resize((size_t)g.audio_offset);
}

// ---- NintendoWare stream geometry (BrstmWriter.cs:24-74, BCFstmWriter.cs:23-83, BxstmConfiguration defaults) ----
struct NwGeom {
    int type = 0, codec = 0, be = 0, channels = 0, rate = 0, looping = 0, loop_start = 0;
    int sample_count = 0;      // the writer's SampleCount: LoopEnd when looping
    int in_samples = 0;        // samples of each channel's array (the whole WAVE channel)
    int spi = 0, bpi = 0;      // SamplesPerInterleave, InterleaveSize
    int audio_data_size = 0, interleave_count = 0, last_samples = 0, last_size_np = 0, last_size = 0;
    int spe = 0;               // SamplesPerSeekTableEntry as the header states it
    int seek_entries = 0, chan_entries = 0;
    int head_size = 0, info1 = 0, info2 = 0, info3 = 0, seek_off = 0, seek_size = 0, data_off = 0, data_size = 0;
    int tracks = 0;
    int aligned = 0, ctx_loop_start = 0, keep = 0, keep_bytes = 0, tail_count = 0, in_size = 0;
    int64_t file_size = 0;
    int audio_offset() const { return data_off + 0x20; }
};

int nw_bytes(int samples, int codec)  // Common.SamplesToBytes
{
    return codec == 2 ? gc_sample_count_to_byte_count(samples) : codec == 1 ? samples * 2 : samples;
}

// type: VGB_CONTAINER_BRSTM / _BCSTM / _BFSTM; codec: NwCodec; be: the file's byte order.  No throw is possible here
// except the ones the caller checks (channel count, FileSize as an int).
void nw_geometry(int type, int codec, int be, int channels, int rate, int samples, bool looping, int loop_start, int loop_end, NwGeom &g)
{
    g = NwGeom{};
    g.type = type; g.codec = codec; g.be = be; g.channels = channels; g.rate = rate; g.looping = looping;
    g.loop_start = looping ? loop_start : 0;
    g.sample_count = looping ? loop_end : samples;
    g.in_samples = samples;
    g.in_size = nw_bytes(samples, codec);
    g.ctx_loop_start = g.loop_start;
    g.keep_bytes = INT_MAX;
    g.spi = codec == 2 ? gc_nibble_count_to_sample_count(0x2000 * 2) : codec == 1 ? 0x1000 : 0x2000;  // BytesToSamples(0x2000)
    g.bpi = nw_bytes(g.spi, codec);
    g.audio_data_size = next_multiple(nw_bytes(g.sample_count, codec), 0x20);
    g.interleave_count = div_round_up(g.sample_count, g.spi);
    g.last_samples = g.sample_count - (g.interleave_count - 1) * g.spi;
    g.last_size_np = nw_bytes(g.last_samples, codec);
    g.last_size = next_multiple(g.last_size_np, 0x20);
    g.tracks = div_round_up(channels, 2);                          // AudioTrack.GetDefaultTrackList
    const bool adpcm = codec == 2;
    const int seek_spe = g.spi;                                    // SamplesPerSeekTableEntry's default equals the interleave's
    g.spe = type == VGB_CONTAINER_BRSTM && !adpcm ? 0 : seek_spe;
    if (adpcm) {
        g.seek_entries = div_round_up(g.sample_count, seek_spe);
        g.chan_entries = div_round_up(samples, seek_spe);
    }
    const int C = channels, T = g.tracks;
    if (type == VGB_CONTAINER_BRSTM) {
        const int h2 = 4 + 8 * T + 0x0c * T, h3 = 4 + 8 * C + (adpcm ? 0x38 : 8) * C;
        g.info2 = h2;
        g.head_size = next_multiple(8 + 24 + 0x34 + h2 + h3, 0x20);
        g.seek_off = adpcm ? 0x40 + g.head_size : 0;
        g.seek_size = adpcm ? next_multiple(8 + g.seek_entries * C * 4, 0x20) : 0;
        g.data_off = 0x40 + g.head_size + g.seek_size;
    } else {
        const bool track_info = type == VGB_CONTAINER_BCSTM;       // version 2.1 has track info, 0.3 does not; both have region info
        g.info1 = 0x38 + 0xc;
        g.info2 = track_info ? 4 + 8 * T : 0;
        g.info3 = 4 + 8 * C + (track_info ? 0x14 * T : 0) + 8 * C + (adpcm ? 0x2e : 0) * C;
        g.head_size = next_multiple(8 + 24 + g.info1 + g.info2 + g.info3, 0x20);
        g.seek_off = adpcm ? 0x40 + g.head_size : 0;
        g.seek_size = adpcm ? next_multiple(8 + g.seek_entries * C * 4, 0x20) : 0;
        g.data_off = 0x40 + g.head_size + g.seek_size;
    }
    g.data_size = 0x20 + g.audio_data_size * C;
    g.file_size = (int64_t)g.data_off + (int64_t)0x20 + (int64_t)g.audio_data_size * C;
}

// A BinaryWriter over a zeroed header image in the file's byte order
struct NwOut {
    std::vector<uint8_t> &h;
    bool be;
    size_t at = 0;
    void u8(int v) { h[at++] = (uint8_t)v; }
    void u16(int v) { if (be) { u8(v >> 8); u8(v); } else { u8(v); u8(v >> 8); } }
    void u32(int32_t v) { const uint32_t u = (uint32_t)v; if (be) { u16((int)(u >> 16)); u16((int)(u & 0xffff)); } else { u16((int)(u & 0xffff)); u16((int)(u >> 16)); } }
    void tag(const char *s) { for (int i = 0; i < 4; i++) u8(s[i]); }
    void ref(int type, int32_t off) { u16(type); u16(0); u32(off); }
};

// Everything in front of the audio data, with the device's fields (coefficients, contexts, seek entries) left zero.
// info_off / info_stride / ctx_off say where the kernel patches them.
void nw_build_header(const NwGeom &g, std::vector<uint8_t> &h, int &info_off, int &info_stride, int &ctx_off)
{
    h.assign((size_t)g.audio_offset(), 0);
    const bool adpcm = g.codec == 2;
    const int C = g.channels, T = g.tracks;
    NwOut w{h, g.type == VGB_CONTAINER_BRSTM || g.be != 0};
    auto track = [&](int t, int &cc, int &left, int &right) { cc = std::min(C - 2 * t, 2); left = 2 * t; right = cc >= 2 ? 2 * t + 1 : 0; };
    if (g.type == VGB_CONTAINER_BRSTM) {  // WriteRstmHeader, WriteHeadBlock (BrstmWriter.cs:139-259)
        const int marker = 0x01000000, h2 = g.info2;
        w.tag("RSTM"); w.u16(0xfeff); w.u16(0x0100); w.u32((int32_t)g.file_size); w.u16(0x40); w.u16(2);
        w.u32(0x40); w.u32(g.head_size); w.u32(g.seek_off); w.u32(g.seek_size); w.u32(g.data_off); w.u32(g.data_size);
        w.at = 0x40;
        w.tag("HEAD"); w.u32(g.head_size);
        w.u32(marker); w.u32(24); w.u32(marker); w.u32(24 + 0x34); w.u32(marker); w.u32(24 + 0x34 + h2);
        w.u8(g.codec); w.u8(g.looping); w.u8(C); w.u8(0); w.u16(g.rate & 0xffff); w.u16(0);  // (ushort)SampleRate
        w.u32(g.loop_start); w.u32(g.sample_count); w.u32(g.audio_offset()); w.u32(g.interleave_count); w.u32(g.bpi); w.u32(g.spi);
        w.u32(g.last_size_np); w.u32(g.last_samples); w.u32(g.last_size); w.u32(g.spe); w.u32(adpcm ? 4 : 0);
        w.u8(T); w.u8(1); w.u16(0);
        const int base2 = 24 + 0x34 + 4;
        for (int t = 0; t < T; t++) { w.u32(0x01010000); w.u32(base2 + 8 * T + 0x0c * t); }
        for (int t = 0; t < T; t++) {
            int cc, l, r;
            track(t, cc, l, r);
            w.u8(0x7f); w.u8(0x40); w.u16(0); w.u32(0); w.u8(cc); w.u8(l); w.u8(r); w.u8(0);
        }
        w.u8(C); w.u8(0); w.u16(0);
        const int base3 = 24 + 0x34 + h2 + 4, cis = adpcm ? 0x38 : 8;
        for (int c = 0; c < C; c++) { w.u32(marker); w.u32(base3 + 8 * C + cis * c); }
        info_off = 0;
        for (int c = 0; c < C; c++) {
            w.u32(marker);
            if (!adpcm) { w.u32(0); continue; }
            w.u32(base3 + 8 * C + cis * c + 8);
            if (c == 0) info_off = (int)w.at;
            w.at += 0x30;  // coefficients, gain, start and loop context, padding
        }
        info_stride = 0x38;
        ctx_off = 0x22;
        if (adpcm) { w.at = (size_t)g.seek_off; w.tag("ADPC"); w.u32(g.seek_size); }
        w.at = (size_t)g.data_off;
        w.tag("DATA"); w.u32(g.data_size); w.u32(0x18);
        return;
    }
    // WriteHeader, WriteInfoBlock (BCFstmWriter.cs:164-332)
    const bool track_info = g.type == VGB_CONTAINER_BCSTM;
    w.tag(g.type == VGB_CONTAINER_BCSTM ? "CSTM" : "FSTM"); w.u16(0xfeff); w.u16(0x40);
    w.u32((track_info ? 0x201 : 3) << 16); w.u32((int32_t)g.file_size);
    w.u16(adpcm ? 3 : 2); w.u16(0);
    w.ref(0x4000, 0x40); w.u32(g.head_size);
    if (adpcm) { w.ref(0x4001, g.seek_off); w.u32(g.seek_size); }
    w.ref(0x4002, g.data_off); w.u32(g.data_size);
    w.at = 0x40;
    w.tag("INFO"); w.u32(g.head_size);
    w.ref(0x4100, 24);
    if (track_info) w.ref(0x0101, 24 + g.info1);
    else { w.u32(0); w.u32(-1); }
    w.ref(0x0101, 24 + g.info1 + g.info2);
    w.u8(g.codec); w.u8(g.looping); w.u8(C); w.u8(0); w.u32(g.rate); w.u32(g.loop_start); w.u32(g.sample_count);
    w.u32(g.interleave_count); w.u32(g.bpi); w.u32(g.spi); w.u32(g.last_size_np); w.u32(g.last_samples); w.u32(g.last_size);
    w.u32(4); w.u32(g.spe); w.ref(0x1F00, 0x18);
    w.ref(0x0100, 0); w.u32(-1);  // region info
    if (track_info) {
        w.u32(T);
        for (int t = 0; t < T; t++) w.ref(0x4101, (4 + 8 * T) + (4 + 8 * C) + 0x14 * t);
    }
    w.u32(C);
    for (int c = 0; c < C; c++) w.ref(0x4102, (4 + 8 * C) + (track_info ? 0x14 * T : 0) + 8 * c);
    if (track_info)
        for (int t = 0; t < T; t++) {
            int cc, l, r;
            track(t, cc, l, r);
            w.u8(0x7f); w.u8(0x40); w.u16(0); w.ref(0x0100, 0xc); w.u32(cc); w.u8(l); w.u8(r); w.u16(0);
        }
    for (int c = 0; c < C; c++) {
        if (adpcm) w.ref(0x0300, 8 * C - 8 * c + 0x2e * c);
        else { w.u32(0); w.u32(-1); }
    }
    info_off = (int)w.at;
    info_stride = 0x2e;
    ctx_off = 0x20;
    if (adpcm) { w.at = (size_t)g.seek_off; w.tag("SEEK"); w.u32(g.seek_size); }
    w.at = (size_t)g.data_off;
    w.tag("DATA"); w.u32(g.data_size);
}

// ---- IDSP (IdspWriter.cs) and HPS (HpsWriter.cs) geometry, after the writers' GcAdpcmFormat.WithAlignment ----
struct GcGeom {
    int type = 0, channels = 0, rate = 0, looping = 0;
    int sample_count = 0;      // IDSP: the writer's SampleCount; HPS: the format's (SampleCountAligned when the loop moved)
    int loop_start = 0, loop_end = 0;  // the format's loop points (aligned), 0 without a loop
    int chan_samples = 0;      // each channel's own SampleCount
    int aligned = 0, ctx_loop_start = 0, keep = 0, keep_bytes = INT_MAX, tail_count = 0, in_size = 0;
    int header_size = 0;
    int audio_data_size = 0;   // IDSP
    int block_hdr = 0;         // HPS
    std::vector<HpsBlock> blocks;  // HPS: CreateBlockMap
    int64_t file_size = 0;
};

int gc_sample_to_nibble(int s) { return s / kGcFrameSamples * 16 + s % kGcFrameSamples + 2; }  // GcAdpcmMath.SampleToNibble
int gc_nibble_to_sample(int n) { return n / 16 * kGcFrameSamples + n % 16 - 2; }                // GcAdpcmMath.NibbleToSample

constexpr int kIdspBlockSize = 16;  // IdspConfiguration.BlockSize's default (BytesPerFrame * 2); the CLI never sets it

void idsp_geometry(bool trim, GcGeom &g)
{
    g.sample_count = trim && g.looping ? g.loop_end : std::max(g.chan_samples, g.loop_end);
    g.audio_data_size = next_multiple(gc_sample_count_to_byte_count(g.sample_count), kIdspBlockSize);
    g.header_size = 0x40 + 0x60 * g.channels;
    g.file_size = (int64_t)g.header_size + (int64_t)g.audio_data_size * g.channels;
}

int hps_channel_size(int channels) { return next_multiple(0x10000 / channels, 0x20); }

// CreateBlockMap (HpsWriter.cs:113-157) for the format's sample count and loop.  False where the reference would leave a
// null entry in its block array (the even split running out of nibbles before the last block).
bool hps_geometry(GcGeom &g)
{
    const int C = g.channels;
    g.sample_count = g.chan_samples;
    g.header_size = next_multiple(std::max(0x80, 0x10 + 0x38 * C), 0x20);
    g.block_hdr = next_multiple(12 + 8 * C, 0x20);
    const int nibbles = gc_sample_count_to_nibble_count(g.sample_count);
    const int max_nibbles = hps_channel_size(C) * C / C * 2;
    const int count = div_round_up(nibbles, max_nibbles);
    const int loop_block = g.looping ? gc_sample_to_nibble(g.loop_start) / max_nibbles : count - 1;
    g.blocks.clear();
    int cur = 0;
    auto add = [&](int size) {
        HpsBlock b{};
        b.start_sample = gc_nibble_to_sample(cur + 2);
        b.byte_in = cur / 2;
        b.end_nibble = size - 1;
        b.chan_size = (size + 1) / 2;
        b.written = next_multiple(b.chan_size, 0x20) * C;
        g.blocks.push_back(b);
        cur += size;
    };
    while ((int)g.blocks.size() < loop_block) add(max_nibbles);
    while (cur < nibbles) {
        const int left = count - (int)g.blocks.size(), rem = nibbles - cur;
        add(std::min(rem, next_multiple(div_round_up(rem, left), 0x40)));
    }
    if ((int)g.blocks.size() != count) return false;
    int64_t at = g.header_size;
    for (HpsBlock &b : g.blocks) {
        b.at = (int32_t)std::min<int64_t>(at, INT_MAX);
        at += next_multiple(4 + 8 * C, 0x20) + b.written;  // BlockInfo.TotalSize
    }
    for (int i = 0; i < count; i++) g.blocks[i].next = i + 1 < count ? g.blocks[i + 1].at : g.looping ? g.blocks[loop_block].at : -1;
    g.file_size = at;
    return true;
}

// Everything the writers put in front of the audio (IDSP) or the first block (HPS), big-endian, with the device's
// fields (coefficients, contexts) left zero
void gc_build_header(const GcGeom &g, std::vector<uint8_t> &h)
{
    h.assign((size_t)g.header_size, 0);
    NwOut w{h, true};
    if (g.type == VGB_CONTAINER_IDSP) {  // WriteHeader (IdspWriter.cs:66-104)
        w.tag("IDSP"); w.u32(0); w.u32(g.channels); w.u32(g.rate); w.u32(g.sample_count); w.u32(g.loop_start); w.u32(g.loop_end);
        w.u32(kIdspBlockSize); w.u32(0x40); w.u32(0x60); w.u32(g.header_size); w.u32(g.audio_data_size);
        for (int c = 0; c < g.channels; c++) {
            w.at = (size_t)(0x40 + 0x60 * c);
            w.u32(g.chan_samples); w.u32(gc_sample_count_to_nibble_count(g.chan_samples)); w.u32(g.rate); w.u16(g.looping); w.u16(0);
            w.u32(gc_sample_to_nibble(g.looping ? g.loop_start : 0));
            w.u32(gc_sample_to_nibble(g.looping ? g.loop_end : g.sample_count - 1));
            w.u32(gc_sample_to_nibble(0));
        }
        return;
    }
    w.tag(" HAL"); w.tag("PST\0");  // WriteHpsHeader, WriteChannelInfo (HpsWriter.cs:63-84)
    w.u32(g.rate); w.u32(g.channels);
    for (int c = 0; c < g.channels; c++) {
        w.at = (size_t)(0x10 + 0x38 * c);
        w.u32(0x10000); w.u32(gc_sample_to_nibble(0)); w.u32(gc_sample_to_nibble(g.sample_count - 1)); w.u32(gc_sample_to_nibble(0));
    }
}

const uint8_t kPcmGuid[16] = {0x01, 0x00, 0x00, 0x00, 0x00, 0x00, 0x10, 0x00, 0x80, 0x00, 0x00, 0xAA, 0x00, 0x38, 0x9B, 0x71};

// ---- WAVE header, 16-bit codec (WaveWriter.cs:24-153): everything in front of the samples ----
int wave_channel_mask(int n)
{
    switch (n) { case 4: return 0x0033; case 5: return 0x0133; case 6: return 0x0633; case 7: return 0x01f3; case 8: return 0x06f3; default: return (int)((1u << n) - 1u); }
}
void le16(uint8_t *p, int v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); }
void le32(uint8_t *p, int32_t v) { le16(p, (int)((uint32_t)v & 0xffff)); le16(p + 2, (int)((uint32_t)v >> 16)); }
void wave_build_header(int channels, int samples, int sample_rate, bool looping, int loop_start, int loop_end, std::vector<uint8_t> &h)
{
    const int fmt = channels > 2 ? 40 : 16;
    const int header = 12 + 8 + fmt + (looping ? 8 + 0x3c : 0) + 8;
    const int64_t data_bytes = (int64_t)channels * samples * 2;
    h.assign((size_t)header, 0);
    uint8_t *p = h.data();
    std::memcpy(p, "RIFF", 4); le32(p + 4, (int32_t)(header - 8 + data_bytes)); std::memcpy(p + 8, "WAVE", 4); p += 12;
    std::memcpy(p, "fmt ", 4); le32(p + 4, fmt);
    le16(p + 8, channels > 2 ? 0xFFFE : 1); le16(p + 10, channels); le32(p + 12, sample_rate);
    le32(p + 16, (int32_t)((uint32_t)sample_rate * 2u * (uint32_t)channels)); le16(p + 20, 2 * channels); le16(p + 22, 16);
    if (channels > 2) { le16(p + 24, 22); le16(p + 26, 16); le32(p + 28, wave_channel_mask(channels)); std::memcpy(p + 32, kPcmGuid, 16); }
    p += 8 + fmt;
    if (looping) {
        std::memcpy(p, "smpl", 4); le32(p + 4, 0x3c);
        le32(p + 8 + 28, 1);
        le32(p + 8 + 36 + 8, loop_start); le32(p + 8 + 36 + 12, loop_end);
        p += 8 + 0x3c;
    }
    std::memcpy(p, "data", 4); le32(p + 4, (int32_t)data_bytes);
}

// ---- HCA header (HcaWriter.cs:56-170) ----
uint16_t crc16_host(const uint8_t *data, size_t n)  // Crc16.Compute (Utilities/Crc16.cs:13-19), polynomial 0x8005
{
    static uint16_t table[256];
    static std::once_flag once;
    std::call_once(once, [] {
        for (int i = 0; i < 256; i++) {
            uint16_t v = (uint16_t)(i << 8);
            for (int k = 0; k < 8; k++) v = (uint16_t)((v & 0x8000) ? (v << 1) ^ 0x8005 : v << 1);
            table[i] = v;
        }
    });
    uint16_t crc = 0;
    for (size_t i = 0; i < n; i++) crc = (uint16_t)((crc << 8) ^ table[(crc >> 8) ^ data[i]]);
    return crc;
}
// The header_size bytes in front of the frames.  ciph: the "ciph" chunk's value; comment: comment_len bytes of UTF-8
// (no zero byte), written as "comm" unless blank (string.IsNullOrWhiteSpace, judged by the caller), else "pad".
// file_size < 0: chunks that do not fit in header_size - 2 bytes are refused (VGB_E_ARG).  Otherwise the reference's
// stream writer is followed: the chunks run on past header_size - 2, the CRC covers the first header_size - 2 bytes as
// written and the CRC and the frames overwrite the rest; chunks running past file_size (where the reference would grow
// the file) are refused (VGB_E_DATA).
int32_t hca_write_header(const vgb_hca_info &h, bool masked, int ciph, const uint8_t *comment, size_t comment_len, bool blank,
                         uint32_t volume_bits, int64_t file_size, std::vector<uint8_t> &out, int index)
{
    if (h.header_size < 8 || h.header_size > 0xffff) return fail(VGB_E_ARG, "file %d: header_size %d", index, h.header_size);
    out.assign((size_t)h.header_size + 64 + comment_len, 0);
    uint8_t *p = out.data();
    auto id = [&](const char *s, int n) { for (int i = 0; i < n; i++) { uint8_t b = (uint8_t)s[i]; if (masked && b) b |= 0x80; p[i] = b; } p += n; };
    id("HCA\0", 4); be16(p, 0x0200); be16(p + 2, h.header_size); p += 4;
    id("fmt\0", 4); p[0] = (uint8_t)h.channel_count; p[1] = (uint8_t)(h.sample_rate >> 16); be16(p + 2, h.sample_rate);
    be32(p + 4, h.frame_count); be16(p + 8, h.inserted_samples); be16(p + 10, h.appended_samples); p += 12;
    id("comp", 4); be16(p, h.frame_size); p[2] = (uint8_t)h.min_resolution; p[3] = (uint8_t)h.max_resolution; p[4] = (uint8_t)h.track_count;
    p[5] = (uint8_t)h.channel_config; p[6] = (uint8_t)h.total_band_count; p[7] = (uint8_t)h.base_band_count; p[8] = (uint8_t)h.stereo_band_count;
    p[9] = (uint8_t)h.bands_per_hfr_group; p += 12;
    if (h.looping) { id("loop", 4); be32(p, h.loop_start_frame); be32(p + 4, h.loop_end_frame); be16(p + 8, h.pre_loop_samples); be16(p + 10, h.post_loop_samples); p += 12; }
    id("ciph", 4); be16(p, ciph); p += 2;
    if (volume_bits != 0x3F800000u) { id("rva\0", 4); be32(p, (int32_t)volume_bits); p += 4; }
    if (blank) id("pad", 3);
    else { id("comm\0", 5); std::memcpy(p, comment, comment_len); p += comment_len + 1; }
    const int64_t end = p - out.data();
    if (end > h.header_size - 2) {
        if (file_size < 0) return fail(VGB_E_ARG, "file %d: header_size %d cannot hold the chunks (%d bytes)", index, h.header_size, (int)end + 2);
        if (end > file_size)
            return fail(VGB_E_DATA, "file %d: the header chunks (%lld bytes) run past the end of the %lld-byte file", index, (long long)end, (long long)file_size);
    }
    out.resize((size_t)h.header_size);
    be16(out.data() + h.header_size - 2, crc16_host(out.data(), (size_t)h.header_size - 2));
    return VGB_OK;
}
// HcaWriter's header for the encoders' files: "ciph" is the key's type, the comment a C string judged blank by its ASCII
// white space, and every chunk fits in header_size - 2 bytes
int32_t hca_build_header(const vgb_hca_info &h, bool masked, int key_type, const char *comment, uint32_t volume_bits,
                         std::vector<uint8_t> &out, int index)
{
    bool blank = true;  // string.IsNullOrWhiteSpace
    if (comment) for (const char *c = comment; *c; c++) if (!std::strchr(" \t\n\r\v\f", *c)) blank = false;
    return hca_write_header(h, masked, masked ? key_type : 0, reinterpret_cast<const uint8_t *>(comment), comment ? std::strlen(comment) : 0, blank,
                            volume_bits, -1, out, index);
}

// CriHcaKey tables (Codecs/CriHca/CriHcaKey.cs:9-174)
void hca_random_row(uint8_t seed, uint8_t row[16])
{
    int x = seed >> 4;
    const int mult = ((seed & 1) << 3) | 5, inc = (seed & 0xe) | 1;
    for (int i = 0; i < 16; i++) { x = (x * mult + inc) % 16; row[i] = (uint8_t)x; }
}
int32_t hca_key_tables(int key_type, uint64_t key_code, uint8_t *dec, uint8_t *enc)
{
    std::memset(dec, 0, 256);
    if (key_type == 0) {
        for (int i = 0; i < 256; i++) dec[i] = (uint8_t)i;
    } else if (key_type == 1) {
        int x = 0, pos = 1;
        for (int i = 0; i < 256; i++) { x = (x * 13 + 11) % 256; if (x != 0 && x != 0xff) dec[pos++] = (uint8_t)x; }
        dec[0xff] = 0xff;
    } else if (key_type == 56) {
        const uint64_t k = key_code - 1;
        uint8_t kc[8], seed[16], t[256], row[16], col[16];
        for (int i = 0; i < 8; i++) kc[i] = (uint8_t)(k >> (8 * i));
        const uint8_t s[16] = {kc[1], (uint8_t)(kc[6] ^ kc[1]), (uint8_t)(kc[2] ^ kc[3]), kc[2], (uint8_t)(kc[1] ^ kc[2]), (uint8_t)(kc[3] ^ kc[4]), kc[3],
                               (uint8_t)(kc[2] ^ kc[3]), (uint8_t)(kc[4] ^ kc[5]), kc[4], (uint8_t)(kc[3] ^ kc[4]), (uint8_t)(kc[5] ^ kc[6]), kc[5],
                               (uint8_t)(kc[4] ^ kc[5]), (uint8_t)(kc[6] ^ kc[1]), kc[6]};
        std::memcpy(seed, s, 16);
        hca_random_row(kc[0], row);
        for (int r = 0; r < 16; r++) {
            hca_random_row(seed[r], col);
            for (int c = 0; c < 16; c++) t[16 * r + c] = (uint8_t)((row[r] << 4) | col[c]);
        }
        uint8_t x = 0;
        int pos = 1;
        for (int i = 0; i < 256; i++) { x = (uint8_t)(x + 17); if (t[x] != 0 && t[x] != 0xff) dec[pos++] = t[x]; }
        dec[0xff] = 0xff;
    } else {
        return fail(VGB_E_ARG, "HCA key type %d (0, 1 or 56)", key_type);
    }
    for (int i = 0; i < 256; i++) enc[dec[i]] = (uint8_t)i;
    return VGB_OK;
}

int wave_tile_samples(int channels)
{
    int t = kSplitSmemSamples / channels / 8 * 8;
    return t < 8 ? 0 : t;
}

}  // namespace

namespace vgb {
void containers_release(Context &c)  // vgb_shutdown, once per bound context
{
    State *s = c.containers.load(std::memory_order_acquire);
    if (!s) return;
    {
        std::lock_guard<std::mutex> lock(s->mu);
        if (s->ready) {
            cudaSetDevice(c.device);  // every stream, event and slab of the state lives on c's device
            drain_state(*s);
            for (int i = 0; i < kWays; i++) {
                s->in[i].release(); s->out[i].release(); s->tab[i].release();
                s->pcms[i].release(); s->encs[i].release(); s->decs[i].release(); s->coefss[i].release(); s->wss[i].release();
                s->srcs[i].release(); s->dws[i].release();
                cudaEventDestroy(s->ev_in[i]); cudaEventDestroy(s->ev_split[i]); cudaEventDestroy(s->ev_k[i]); cudaEventDestroy(s->ev_out[i]);
                cudaStreamDestroy(s->s_kern[i]);
            }
            cudaStreamDestroy(s->s_in); cudaStreamDestroy(s->s_out);
            for (auto &grp : s->stage) for (auto &e : grp) { if (e) cudaEventDestroy(e); e = nullptr; }
            (void)cudaGetLastError();
        }
    }
    c.containers.store(nullptr, std::memory_order_release);
    delete s;
}
}  // namespace vgb

#include "containers_abi.inc"
