// hca.cu — CRI HCA encoder on sm_90a (H100).
//
// Replaces CriHcaEncoder.EncodeFrame and its 12 stages (Codecs/CriHca/CriHcaEncoder.cs:271-286, :420-858),
// CriHcaPacking.PackFrame (CriHcaPacking.cs:17-58, BitWriter.cs:26-98, Crc16.cs) and Mdct.RunMdct/Dct4
// (Utilities/Mdct.cs:63-181).  The reference's streaming front end (CriHcaEncoder.Encode :126-272 driven by
// CriHcaFormat.cs:53-81) is folded into one VIRTUAL input stream per channel - pre-roll, source samples, for a looping
// stream the loop-start audio repeated behind the loop end, zeros - and frame k encodes its k-th 1024-sample window.
//
// Frames are independent given that stream (the MDCT overlap is its previous 128 samples), so ONE CTA OF 128
// THREADS OWNS ONE (stream, frame): massive parallelism across frames, stages inside the CTA separated by barriers.
//   mdct        2 x 64 threads run two 128-point DCT-IV at a time (6 radix-2 stages in shared memory), fp64, same
//               operation order as the reference (a*cos + b*sin as mul, mul, add - no FMA)
//   scale       one thread per band: max |coef| over 8 subframes -> FindScaleFactor (binary search) -> scaled spectra
//   allocation  CalculateUsedBits is an integer sum -> block reduction; the two binary searches (noise level,
//               evaluation boundary) run ~16 probes of it
//   order-sensitive fp64 sums (intensity stereo energies, HFR group averages) stay sequential inside one thread each
//   pack        thread = band sizes and places its own codes (two warp-scan passes over the stream's sections, bits
//               ORed into big-endian words), the CRC is folded by one warp using its linearity
// fp64 throughout like the reference (A.14); with identical tables and operation order the frames are byte-identical
// to the oracle.  ALU/latency bound: ~135 ops per sample (SURVEY.md §8d), algorithmic traffic 2 B/sample in +
// frame_size/1024 B/sample out.
#include "common.cuh"
#include "kernels.h"

namespace vgb {

namespace {

constexpr int kSub = 8, kBins = 128, kFrame = 1024;
constexpr int kMaxSections = 8 + kSub * 8;  // packer: one header per channel + one code row per (subframe, channel)

__device__ __forceinline__ double dclamp(double v, double lo, double hi) { return v < lo ? lo : (v > hi ? hi : v); }

// CalculateResolution (CriHcaPacking.cs:60-69)
__device__ __forceinline__ int hca_resolution(const HcaTables &T, int scale_factor, int noise_level)
{
    if (scale_factor == 0) return 0;
    int pos = noise_level - 5 * scale_factor / 2 + 2;
    pos = min(max(pos, 0), 58);
    return T.scale_to_resolution[pos];
}

// FindScaleFactor (CriHcaEncoder.cs:691-709)
__device__ __forceinline__ int hca_find_scale_factor(const HcaTables &T, double value)
{
    unsigned low = 0, high = 63;
    while (low < high) {
        const unsigned mid = (low + high) / 2;
        if (T.dequantizer_scaling[mid] <= value) low = mid + 1;
        else high = mid;
    }
    return (int)low;
}

// bits one scaled coefficient costs at a resolution (CalculateUsedBits inner loops, :566-592)
__device__ __forceinline__ int hca_coef_bits(const HcaTables &T, int resolution, double scaled)
{
    if (resolution >= 8) {
        const int bits = T.quantized_max_bits[resolution] - 1;
        return bits + (fabs(scaled) >= T.dead_zone[resolution] ? 1 : 0);
    }
    const double inv = T.inv_step[resolution];
    const double up = inv + 1;
    const int down = (int)(inv + 0.5 - 8);
    const int q = (int)(scaled * inv + up) - down;
    return T.quantize_bits[resolution][q];
}

struct BlockSum {  // integer sum over the 128 threads of the CTA, result in every thread
    int *scratch;  // 2 x 4 ints of shared memory, used alternately: ONE barrier per sum (a warp can be at most one call
    int parity;    // ahead of the slowest reader, and that call writes the other half)
    __device__ int operator()(int v)
    {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
        int *mine = scratch + 4 * parity;
        parity ^= 1;
        if ((threadIdx.x & 31) == 0) mine[threadIdx.x >> 5] = v;
        __syncthreads();
        return mine[0] + mine[1] + mine[2] + mine[3];
    }
};

}  // namespace

// Sample `v` of the encoder's virtual input stream (see HcaStream): what CriHcaEncoder.Encode's buffer management
// (EncodePreAudio :175-194, EncodeMainAudio :196-211, SaveLoopAudio :247-257, EncodePostAudio :213-245) feeds to
// EncodeFrame at position v, given the 1024-sample chunks CriHcaFormat.EncodeFromPcm16 (:53-81) hands it.
__device__ __forceinline__ int16_t hca_virtual_sample(const int16_t *src, const HcaStream &st, int64_t v)
{
    if (v < st.pre_zero) return 0;  // before the stream, and the whole silent frames in front of a padded loop
    v -= st.pre_zero;
    if (v < st.pre_fill) return st.src_count > 0 ? src[0] : (int16_t)0;  // pcm[i][0] of the first chunk
    v -= st.pre_fill;
    if (v < st.sample_count) return src[v];
    v -= st.sample_count;
    if (v < st.post_count) {
        // PostAudio[v] = what the format layer's reused 1024-sample chunk buffer held at source position a when the
        // chunk went by: the sample itself; past the end of the PCM the previous chunk's sample at the same offset
        // (the buffer is not cleared, CriHcaFormat.cs:57-61); zero if that chunk was never handed over.
        const int64_t a = (int64_t)st.loop_start + v;
        const int64_t chunk = a >> 10;
        if (chunk > st.last_chunk) return 0;
        if (a < st.src_count) return src[a];
        return chunk >= 1 ? src[a - 1024] : (int16_t)0;
    }
    return 0;
}

// Dynamic shared memory layout per CTA (nch = channel count):
//   double spectra[nch][8][128]; double scaled[nch][128][8]; then the small per-channel state below.
struct HcaChannelState {
    int scale_factors[kBins];
    int resolution[kBins];
    int intensity[kSub];
    int hfr_scales[8];
    double hfr_group_avg[8];
    int header_bits, delta_bits, type, coded_count;
};

__global__ void __launch_bounds__(128)
hca_encode_kernel(const int16_t *__restrict__ pcm, const HcaStream *__restrict__ streams, HcaConfig cfg, HcaTables T,
                  uint8_t *__restrict__ frames_out, int32_t *__restrict__ status_out)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int nch = cfg.channel_count;
    double *spectra = reinterpret_cast<double *>(smem_raw);                   // [nch][8][128]
    double *scaled = spectra + (size_t)nch * kSub * kBins;                    // [nch][128][8]
    double *work = scaled + (size_t)nch * kSub * kBins;                       // [2][128] DCT scratch (+ fold input)
    double *fold = work + 2 * kBins;                                          // [2][128]
    HcaChannelState *chs = reinterpret_cast<HcaChannelState *>(fold + 2 * kBins);  // [nch]
    uint8_t *frame_buf = reinterpret_cast<uint8_t *>(chs + nch);              // [frame_size] (+pad)
    int *red = reinterpret_cast<int *>(frame_buf + ((cfg.frame_size + 15) & ~15));  // [8] reduction / broadcast scratch

    const int tid = threadIdx.x;
    const int s = blockIdx.y;
    const HcaStream st = streams[s];
    const int k = blockIdx.x;  // frame index
    if (k >= st.frame_count) return;
    BlockSum block_sum{red, 0};

    // ---- channel set-up (CriHcaFrame ctor :18-33)
    if (tid < nch) {
        chs[tid].type = cfg.channel_type[tid];
        chs[tid].coded_count = cfg.channel_type[tid] == 2 ? cfg.base_band_count : cfg.base_band_count + cfg.stereo_band_count;
    }

    // ---- PcmToFloat (:845-858) + RunMdct (:834-843, Mdct.cs:63-92): FOUR subframes at a time, one WARP per subframe.  A
    // 128-point DCT-IV stage has exactly 32 butterflies, so a warp owns a whole transform and every step inside it is
    // separated by __syncwarp instead of a CTA barrier (the first version ran two subframes on 64 threads each, half of
    // them idle in the butterfly stages, with nine CTA barriers per pair).  Scratch: the `scaled` array, not yet in use.
    {
        const int wsub = tid >> 5, ln = tid & 31;
        double *t = scaled + wsub * kBins;
        double *in = scaled + (4 + wsub) * kBins;
        for (int c = 0; c < nch; c++) {
            const int16_t *src = pcm + st.pcm_off + (int64_t)c * st.channel_stride;
            for (int sf4 = 0; sf4 < kSub; sf4 += 4) {
                const int sf = sf4 + wsub;
                const int64_t base = (int64_t)k * kFrame + sf * kBins;  // first sample of this subframe
                auto sample = [&](int64_t idx) -> double { return (double)hca_virtual_sample(src, st, idx) * (1.0 / 32768.0); };
#pragma unroll
                for (int h = 0; h < 2; h++) {  // window + fold into the DCT input (Mdct.cs:77-85); `previous` = the 128 samples before this subframe
                    const int i = ln + 32 * h;
                    const double a = T.window[64 - i - 1] * -sample(base + 64 + i);
                    const double b = T.window[64 + i] * sample(base + 64 - i - 1);
                    const double cc = T.window[i] * sample(base - kBins + i);
                    const double d = T.window[kBins - i - 1] * sample(base - kBins + kBins - i - 1);
                    in[i] = a - b;
                    in[64 + i] = cc - d;
                }
                __syncwarp();
#pragma unroll
                for (int h = 0; h < 2; h++) {  // Dct4 pre-twiddle (Mdct.cs:137-147)
                    const int i = ln + 32 * h, i2 = i * 2;
                    const double a = in[i2], b = in[kBins - 1 - i2];
                    const double sn = T.sin_tab[7][i], cs = T.cos_tab[7][i];
                    t[i2] = a * cs + b * sn;
                    t[i2 + 1] = a * sn - b * cs;
                }
                __syncwarp();
#pragma unroll 1
                for (int stage = 0; stage < 6; stage++) {  // (Mdct.cs:148-175): 32 butterflies of two complex pairs each
                    const int block_bits = 6 - stage, half_bits = block_bits - 1;
                    const int block_size = 1 << block_bits, block_half = 1 << half_bits;
                    const int block = ln >> half_bits, j = ln & (block_half - 1);
                    const int front = (block * block_size + j) * 2, back = front + block_size;
                    const double a = t[front] - t[back];
                    const double b = t[front + 1] - t[back + 1];
                    const double sn = T.sin_tab[half_bits][j], cs = T.cos_tab[half_bits][j];
                    const double f0 = t[front] + t[back], f1 = t[front + 1] + t[back + 1];
                    t[front] = f0;
                    t[front + 1] = f1;
                    t[back] = a * cs + b * sn;
                    t[back + 1] = a * sn - b * cs;
                    __syncwarp();
                }
                double *out = spectra + ((size_t)c * kSub + sf) * kBins;
#pragma unroll
                for (int h = 0; h < 4; h++) out[ln + 32 * h] = t[T.shuffle[ln + 32 * h]] * T.mdct_scale;  // (Mdct.cs:177-180)
                __syncwarp();
            }
        }
        __syncthreads();  // the spectra of every subframe and channel are in place; `scaled` is free again
    }

    // ---- EncodeIntensityStereo (:711-764): the energy sums are order-sensitive fp64 -> one thread per (pair, sf)
    if (cfg.stereo_band_count > 0) {
        for (int c = 0; c < nch; c++) {
            if (chs[c].type != 1) continue;
            double *l = spectra + ((size_t)c * kSub) * kBins, *r = spectra + ((size_t)(c + 1) * kSub) * kBins;
            if (tid < kSub) {
                const int sf = tid;
                double el = 0, er = 0, et = 0;
                for (int b = cfg.base_band_count; b < cfg.total_band_count; b++) {
                    el += fabs(l[sf * kBins + b]);
                    er += fabs(r[sf * kBins + b]);
                    et += fabs(l[sf * kBins + b] + r[sf * kBins + b]);
                }
                et *= 2;
                const double elr = er + el;
                const double stored = 2 * el / elr;
                double ratio = elr / et;
                ratio = dclamp(ratio, 0.5, T.sqrt2 / 2);
                int q = 1;
                if (er > 0 || el > 0) {
                    while (q < 13 && T.intensity_bounds[q] >= stored) q++;
                } else {
                    q = 0;
                    ratio = 1;
                }
                chs[c + 1].intensity[sf] = q;
                for (int b = cfg.base_band_count; b < cfg.total_band_count; b++) {
                    l[sf * kBins + b] = (l[sf * kBins + b] + r[sf * kBins + b]) * ratio;
                    r[sf * kBins + b] = 0;
                }
            }
        }
        __syncthreads();
    }

    // ---- CalculateScaleFactors (:673-689) + ScaleSpectra (:651-671): thread = band
    for (int c = 0; c < nch; c++) {
        const int b = tid;
        int sfac = 0;
        if (b < chs[c].coded_count) {
            double mx = 0;
#pragma unroll
            for (int sf = 0; sf < kSub; sf++) {
                const double coeff = fabs(spectra[((size_t)c * kSub + sf) * kBins + b]);
                mx = coeff > mx ? coeff : mx;
            }
            sfac = hca_find_scale_factor(T, mx);
            const double qs = T.quantizer_scaling[sfac];
#pragma unroll
            for (int sf = 0; sf < kSub; sf++) {
                const double coeff = spectra[((size_t)c * kSub + sf) * kBins + b];
                scaled[((size_t)c * kBins + b) * kSub + sf] = sfac == 0 ? 0.0 : dclamp(coeff * qs, -0.999999999999, 0.999999999999);
            }
        }
        chs[c].scale_factors[b] = sfac;
        chs[c].resolution[b] = 0;
    }
    __syncthreads();

    // ---- CalculateHfrGroupAverages (:766-793) + CalculateHfrScale (:795-832): sequential sums, thread = (channel, group)
    if (cfg.hfr_group_count > 0) {
        const int c = tid >> 3, group = tid & 7;
        if (c < nch && group < cfg.hfr_group_count && chs[c].type != 2) {
            const int start = cfg.stereo_band_count + cfg.base_band_count;
            {
                double sum = 0.0;
                int count = 0;
                int band = start + group * cfg.bands_per_hfr_group;
                for (int ii = 0; ii < cfg.bands_per_hfr_group && band < kBins; band++, ii++) {
                    for (int sf = 0; sf < kSub; sf++) sum += fabs(spectra[((size_t)c * kSub + sf) * kBins + band]);
                    count += kSub;
                }
                chs[c].hfr_group_avg[group] = sum / count;
            }
            {
                const int hfr_bands = min(cfg.hfr_band_count, cfg.total_band_count - cfg.hfr_band_count);
                double sum = 0.0;
                int count = 0;
                int band = group * cfg.bands_per_hfr_group;
                for (int ii = 0; ii < cfg.bands_per_hfr_group && band < hfr_bands; band++, ii++) {
                    for (int sf = 0; sf < kSub; sf++) sum += fabs(scaled[((size_t)c * kBins + (start - band - 1)) * kSub + sf]);
                    count += kSub;
                }
                const double avg = sum / count;
                double g = chs[c].hfr_group_avg[group];
                if (avg > 0.0) {
                    const double inv = 1.0 / avg;
                    g *= inv < T.sqrt2 ? inv : T.sqrt2;
                }
                chs[c].hfr_group_avg[group] = g;
                chs[c].hfr_scales[group] = hca_find_scale_factor(T, g);
            }
        }
        __syncthreads();
    }

    // ---- CalculateFrameHeaderLength (:599-649): integers; one thread per channel
    auto header_lengths = [&]() {
        if (tid < nch) {
            HcaChannelState &ch = chs[tid];
            bool empty = true;
            for (int b = 0; b < ch.coded_count; b++)
                if (ch.scale_factors[b] != 0) { empty = false; break; }
            if (empty) {
                ch.header_bits = 3;
                ch.delta_bits = 0;
            } else {
                int min_delta_bits = 6;
                int min_length = 3 + 6 * ch.coded_count;
                for (int delta_bits = 1; delta_bits < 6; delta_bits++) {
                    const int max_delta = (1 << (delta_bits - 1)) - 1;
                    int length = 3 + 6;
                    for (int band = 1; band < ch.coded_count; band++) {
                        const int delta = ch.scale_factors[band] - ch.scale_factors[band - 1];
                        length += abs(delta) > max_delta ? delta_bits + 6 : delta_bits;
                    }
                    if (length < min_length) { min_length = length; min_delta_bits = delta_bits; }
                }
                ch.header_bits = min_length;
                ch.delta_bits = min_delta_bits;
            }
            if (ch.type == 2) ch.header_bits += 32;
            else if (cfg.hfr_group_count > 0) ch.header_bits += 6 * cfg.hfr_group_count;
        }
        __syncthreads();
    };
    header_lengths();

    // ---- CalculateUsedBits (:554-597): integer sum over channels x bands x subframes -> block reduction.  The two
    // searches below probe it ~17 times with different (noise level, boundary); what changes between probes is only
    // the RESOLUTION of a band, so the cost of a band's eight coefficients is tabulated once for all 16 resolutions
    // (the same hca_coef_bits arithmetic) and a probe is one table read per band.
    uint8_t *band_bits = reinterpret_cast<uint8_t *>(red + 8);  // [nch][128][16], sums <= 8 * 12
    for (int c = 0; c < nch; c++) {
        const int b = tid;
        double x[kSub];
#pragma unroll
        for (int sf = 0; sf < kSub; sf++) x[sf] = scaled[((size_t)c * kBins + b) * kSub + sf];
        uint32_t packed[4] = {0, 0, 0, 0};
#pragma unroll
        for (int res = 0; res < 16; res++) {
            int w = 0;
            if (b < chs[c].coded_count) {
#pragma unroll
                for (int sf = 0; sf < kSub; sf++) w += hca_coef_bits(T, res, x[sf]);
            }
            packed[res >> 2] |= (uint32_t)w << ((res & 3) * 8);
        }
        *reinterpret_cast<uint4 *>(band_bits + ((size_t)c * kBins + b) * 16) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
    }
    __syncthreads();
    auto used_bits = [&](int noise_level, int eval_boundary) -> int {
        int mine = 0;
        for (int c = 0; c < nch; c++) {
            const int b = tid;
            if (b < chs[c].coded_count) {
                const int noise = b < eval_boundary ? noise_level - 1 : noise_level;
                const int resolution = hca_resolution(T, chs[c].scale_factors[b], noise);
                mine += band_bits[((size_t)c * kBins + b) * 16 + resolution];
            }
            if (tid == 0) mine += chs[c].header_bits;
        }
        return 16 + 16 + 16 + block_sum(mine);
    };

    // ---- CalculateNoiseLevel (:457-485) with BinarySearchLevel (:502-523); every thread runs the same control flow
    const int available = cfg.frame_size * 8;
    auto search_level = [&]() -> int {
        int low = 0, high = 255, mid_value = 0;
        while (low != high) {
            const int mid = (low + high) / 2;
            mid_value = used_bits(mid, 0);
            if (mid_value > available) low = mid + 1;
            else high = mid;
        }
        return (low == 255 && mid_value > available) ? -1 : low;
    };
    int level = search_level();
    int highest = cfg.base_band_count + cfg.stereo_band_count - 1;
    int status = 0;
    while (level < 0) {
        highest -= 2;
        if (highest < 0) { status = VGB_HCA_BITRATE_TOO_LOW; break; }  // InvalidDataException("Bitrate is set too low.")
        if (tid < nch) {
            chs[tid].scale_factors[highest + 1] = 0;
            chs[tid].scale_factors[highest + 2] = 0;
        }
        __syncthreads();
        header_lengths();
        level = search_level();
    }
    const int noise_level = status ? 0 : level;

    // ---- CalculateEvaluationBoundary (:487-500) with BinarySearchBoundary (:525-552)
    int eval_boundary = 0;
    if (!status && noise_level != 0) {
        int low = 0, high = 127;
        while (abs(high - low) > 1) {
            const int mid = (low + high) / 2;
            const int mid_value = used_bits(noise_level, mid);
            if (available < mid_value) high = mid - 1;
            else low = mid;
        }
        int found;
        if (low == high) found = low < 127 ? low : -1;
        else found = used_bits(noise_level, high) > available ? low : high;
        if (found < 0) status = VGB_HCA_NOT_IMPLEMENTED;  // NotImplementedException (:499)
        else eval_boundary = found;
    }

    // ---- CalculateFrameResolutions (:441-455) + QuantizeSpectra (:420-439): thread = band; quantised values reuse
    // the `spectra` storage as ints (the spectra themselves are no longer needed)
    int *quantized = reinterpret_cast<int *>(spectra);  // [nch][8][128] ints inside the first half of the doubles
    __syncthreads();
    for (int c = 0; c < nch; c++) {
        const int b = tid;
        int resolution = 0;
        if (b < chs[c].coded_count)
            resolution = hca_resolution(T, chs[c].scale_factors[b], b < eval_boundary ? noise_level - 1 : noise_level);
        chs[c].resolution[b] = resolution;
    }
    __syncthreads();
    for (int c = 0; c < nch; c++) {
        const int b = tid;
        int q[kSub];
        const int resolution = chs[c].resolution[b];
        const double inv = T.inv_step[resolution];
        const double up = inv + 1;
        const int down = (int)(inv + 0.5);
#pragma unroll
        for (int sf = 0; sf < kSub; sf++)
            q[sf] = b < chs[c].coded_count ? (int)(scaled[((size_t)c * kBins + b) * kSub + sf] * inv + up) - down : 0;
        __syncthreads();  // every thread has read what it needs from `spectra` long ago; ints alias its first half
#pragma unroll
        for (int sf = 0; sf < kSub; sf++) quantized[((size_t)c * kSub + sf) * kBins + b] = q[sf];
    }
    // ---- PackFrame (CriHcaPacking.cs:17-58), in parallel.  The bitstream is a sequence of SECTIONS - one header per
    // channel (WriteScaleFactors :262-295 + intensity / HFR scales), then one row of spectral codes per (subframe,
    // channel) (WriteSpectra :238-260) - and inside a section thread = band owns one element (0..3 short codes).
    // Pass A sizes every element (warp scans -> per-warp totals), thread 0 turns the totals into section offsets,
    // pass B recomputes the codes and ORs them into the frame at their bit positions.  The frame is held as big-endian
    // 32-bit words in shared memory (bit p of the stream = bit 31 - p%32 of word p/32), converted on the way out.
    uint32_t *words = reinterpret_cast<uint32_t *>(frame_buf);
    const int n_words = (cfg.frame_size + 3) >> 2;
    int *warp_tot = reinterpret_cast<int *>(scaled);      // [sections][4]   (`scaled` is dead after quantisation)
    int *sec_base = warp_tot + kMaxSections * 4;          // [sections]
    int *pack_flag = sec_base + kMaxSections;             // [1] overflow
    __syncthreads();                                      // all reads of `scaled` are done
    for (int w = tid; w < ((cfg.frame_size + 15) & ~15) / 4; w += blockDim.x) words[w] = 0;
    if (tid == 0) *pack_flag = 0;
    const int n_sections = nch + kSub * nch;
    const int lane = tid & 31, warp = tid >> 5;
    const int capacity = cfg.frame_size * 8;              // BitWriter over the whole frame buffer (BitWriter.cs:26-33)

    // the codes thread `tid` contributes to section `sec`, in stream order, through emit(value, bit count)
    auto element = [&](int sec, auto &&emit) {
        if (sec < nch) {
            const HcaChannelState &ch = chs[sec];
            const int db = ch.delta_bits, b = tid;
            if (b == 0) emit((uint32_t)db, 3);
            if (b < ch.coded_count) {
                if (db == 6) {
                    emit((uint32_t)ch.scale_factors[b], 6);
                } else if (db != 0) {
                    if (b == 0) {
                        emit((uint32_t)ch.scale_factors[0], 6);
                    } else {
                        const int max_delta = (1 << (db - 1)) - 1, escape = (1 << db) - 1;
                        const int delta = ch.scale_factors[b] - ch.scale_factors[b - 1];
                        if (abs(delta) > max_delta) {
                            emit((uint32_t)escape, db);
                            emit((uint32_t)ch.scale_factors[b], 6);
                        } else {
                            emit((uint32_t)(max_delta + delta), db);
                        }
                    }
                }
            }
            if (b == max(ch.coded_count - 1, 0)) {  // the channel's trailer rides behind its last scale factor
                if (ch.type == 2) {
                    for (int sf = 0; sf < kSub; sf++) emit((uint32_t)ch.intensity[sf], 4);
                } else if (cfg.hfr_group_count > 0) {
                    for (int g = 0; g < cfg.hfr_group_count; g++) emit((uint32_t)ch.hfr_scales[g], 6);
                }
            }
        } else {
            const int row = sec - nch, sf = row / nch, c = row - sf * nch, b = tid;
            const HcaChannelState &ch = chs[c];
            if (b < ch.coded_count) {
                const int resolution = ch.resolution[b];
                const int q = quantized[((size_t)c * kSub + sf) * kBins + b];
                if (resolution != 0) {
                    if (resolution < 8) {
                        emit((uint32_t)T.quantize_value[resolution][q + 8], (int)T.quantize_bits[resolution][q + 8]);
                    } else {
                        emit((uint32_t)abs(q), (int)T.quantized_max_bits[resolution] - 1);
                        if (q != 0) emit(q > 0 ? 0u : 1u, 1);
                    }
                }
            }
        }
    };
    auto warp_inclusive = [&](int v) {
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int up = __shfl_up_sync(0xFFFFFFFFu, v, o);
            if (lane >= o) v += up;
        }
        return v;
    };

    for (int sec = 0; sec < n_sections; sec++) {  // pass A
        int len = 0;
        element(sec, [&](uint32_t, int n) { len += n; });
        const int incl = warp_inclusive(len);
        if (lane == 31) warp_tot[sec * 4 + warp] = incl;
    }
    __syncthreads();
    if (tid == 0) {
        int running = 32;  // sync word, noise level, evaluation boundary
        for (int sec = 0; sec < n_sections; sec++) {
            sec_base[sec] = running;
            running += warp_tot[sec * 4] + warp_tot[sec * 4 + 1] + warp_tot[sec * 4 + 2] + warp_tot[sec * 4 + 3];
        }
        if (running > capacity) *pack_flag = 1;  // InvalidOperationException (BitWriter.cs:30-33)
        words[0] = 0xffff0000u | ((uint32_t)noise_level << 7) | (uint32_t)eval_boundary;  // 16 + 9 + 7 bits
    }
    __syncthreads();
    for (int sec = 0; sec < n_sections; sec++) {  // pass B
        int len = 0;
        element(sec, [&](uint32_t, int n) { len += n; });
        int pos = sec_base[sec] + warp_inclusive(len) - len;
        for (int w = 0; w < warp; w++) pos += warp_tot[sec * 4 + w];
        element(sec, [&](uint32_t value, int n) {
            if (n > 0 && pos + n <= capacity) {
                const int w = pos >> 5, sh = 32 - (pos & 31) - n;
                if (sh >= 0) {
                    atomicOr(&words[w], value << sh);
                } else {
                    atomicOr(&words[w], value >> -sh);
                    atomicOr(&words[w + 1], value << (32 + sh));
                }
            }
            pos += n;
        });
    }
    __syncthreads();
    if (*pack_flag && !status) status = VGB_HCA_BIT_OVERFLOW;

    // ---- WriteChecksum (:231-236, Crc16.cs): CRC-16 (poly 0x8005, init 0) is linear and ignores leading zero bytes,
    // so the message is right-aligned into 32 equal segments, one per lane of warp 0, and the partial CRCs are folded
    // pairwise: crc(A || B) = crc(A) * x^(8 |B|) + crc(B) in GF(2)[x] / P.
    if (warp == 0) {
        const int n_msg = cfg.frame_size - 2;
        const int seg = (n_msg + 31) / 32, pad = seg * 32 - n_msg;
        auto byte_at = [&](int i) -> uint32_t { return (words[i >> 2] >> (24 - 8 * (i & 3))) & 0xFFu; };
        auto mulmod = [](uint32_t a, uint32_t bb) {  // a * bb mod x^16 + x^15 + x^2 + 1
            uint32_t r = 0;
#pragma unroll
            for (int i = 15; i >= 0; i--) {
                r <<= 1;
                if (r & 0x10000u) r ^= 0x18005u;
                if ((bb >> i) & 1u) r ^= a;
            }
            return r;
        };
        uint32_t crc = 0;
        for (int j = 0; j < seg; j++) {
            const int i = lane * seg + j - pad;
            const uint32_t byte = i >= 0 ? byte_at(i) : 0u;
            crc = ((crc << 8) & 0xFFFFu) ^ T.crc_table[(crc >> 8) ^ byte];
        }
        uint32_t shift = 1;  // x^(8 * seg): multiplier for a right neighbour of one segment
        for (int j = 0; j < 8 * seg; j++) {
            shift <<= 1;
            if (shift & 0x10000u) shift ^= 0x18005u;
        }
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t right = __shfl_down_sync(0xFFFFFFFFu, crc, o);
            if ((lane & (2 * o - 1)) == 0) crc = mulmod(crc, shift) ^ right;
            shift = mulmod(shift, shift);
        }
        if (lane == 0) {  // big-endian CRC in the last two bytes
            const int i0 = cfg.frame_size - 2, i1 = cfg.frame_size - 1;
            atomicOr(&words[i0 >> 2], ((crc >> 8) & 0xFFu) << (24 - 8 * (i0 & 3)));
            atomicOr(&words[i1 >> 2], (crc & 0xFFu) << (24 - 8 * (i1 & 3)));
            if (status) atomicCAS(status_out + s, 0, status);
        }
    }
    __syncthreads();
    uint8_t *dst = frames_out + st.frames_off + (int64_t)k * cfg.frame_size;
    for (int b = tid; b < cfg.frame_size; b += blockDim.x) dst[b] = (uint8_t)(words[b >> 2] >> (24 - 8 * (b & 3)));
    (void)n_words;
}

// ==========================================================================================================
// Decoder: CriHcaPacking.UnpackFrame (CriHcaPacking.cs:10-229) + CriHcaDecoder.DecodeFrame (CriHcaDecoder.cs:62-192)
// ==========================================================================================================
// The only state the reference carries between frames is the IMDCT overlap buffer (Mdct.cs:114-117), and that is a
// pure function of the previous subframe's DCT-IV output.  So decoding splits into two embarrassingly parallel
// kernels: (P) one THREAD per frame parses the bitstream (prefix codes are serial inside a frame, frames are independent)
// into a record of scale factors, resolutions and quantised coefficients; (A) one CTA per (stream, frame): dequantise,
// rebuild the high band and intensity-stereo band, run the eight DCT-IV, window + overlap-add subframes 1..7, convert
// to int16 and write the samples the container asks for (CopyPcmToOutput, CriHcaDecoder.cs:26-37); the two addends of
// subframe 0 (2 KB per channel-frame) are parked in HBM; (B) one CTA per (stream, frame, channel) adds frame k's head
// to frame k-1's tail.
// Malformed input: a wrong sync word raises VGB_HCA_BAD_SYNC (InvalidDataException in the reference); a failed
// scale-factor delta decode raises VGB_HCA_BAD_DELTA (the reference ignores UnpackFrame's `false` and keeps decoding
// with whatever the previous frame left in its buffers - state we deliberately do not carry).

namespace {

// PcmFloatToShort (CriHcaDecoder.cs:168-181)
__device__ __forceinline__ int16_t hca_pcm_float_to_short(double x)
{
    const double v = x * 32768.0;
    const int sample = (v > -2147483649.0 && v < 2147483648.0) ? __double2int_rz(v) : INT32_MIN;  // x64 cvttsd2si (A.8)
    return (int16_t)clamp16(sample);
}

}  // namespace

// ---- parsed-frame record (HBM scratch between the two decoder kernels), per channel:
//   [0,128) scale factors, [128,256) resolutions, [256,264) intensity, [264,272) HFR scales, [272, 272 + 2048) the
//   8 x 128 quantised coefficients as int16
constexpr int kRecScale = 0, kRecRes = 128, kRecIntensity = 256, kRecHfr = 264, kRecQuant = 272;
constexpr int kRecChannelBytes = kRecQuant + kSub * kBins * 2;  // 2320
constexpr int kParseThreads = 64;

// CriHcaPacking.UnpackFrame (CriHcaPacking.cs:10-229), ONE THREAD PER FRAME.  Parsing a frame is inherently serial
// (prefix codes), and a CTA-per-frame kernel that parks 127 threads behind one parser spent 90 % of its warp
// instructions at 1/32 lane efficiency (ncu).  Frames are independent, so here the 32 lanes of a warp parse 32
// different frames; the per-band code descriptors come from shared memory, everything on the bit chain is shifts.
__global__ void __launch_bounds__(kParseThreads)
hca_decode_parse_kernel(const uint8_t *__restrict__ frames, const HcaStream *__restrict__ streams, int n_streams,
                        int64_t total_frames, HcaConfig cfg, HcaTables T, uint8_t *__restrict__ parsed,
                        int32_t *__restrict__ status_out)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ unsigned long long s_lens64[16], s_vals64[16];
    __shared__ uint8_t s_maxbits[16], s_curve[64], s_ath[128];
    uint8_t *sres = smem_raw;  // [nch][128][kParseThreads] resolutions of this thread's frame (thread fastest)
    const int nch = cfg.channel_count, tid = threadIdx.x;
    if (tid < 16) {
        unsigned long long lens = 0, vals = 0;
        if (tid < 8)
            for (int code = 0; code < 16; code++) {
                lens |= (unsigned long long)(T.dequantize_bits[tid][code] & 15u) << (4 * code);
                vals |= (unsigned long long)((unsigned)T.dequantize_value[tid][code] & 15u) << (4 * code);
            }
        s_lens64[tid] = lens;
        s_vals64[tid] = vals;
        s_maxbits[tid] = T.quantized_max_bits[tid];
    }
    if (tid < 59) s_curve[tid] = T.scale_to_resolution[tid];
    for (int b = tid; b < 128; b += kParseThreads) s_ath[b] = cfg.ath[b];
    __syncthreads();

    const int64_t fi = (int64_t)blockIdx.x * kParseThreads + tid;
    if (fi >= total_frames) return;
    int lo = 0, hi = n_streams - 1;  // the stream this frame belongs to: last one whose first frame index <= fi
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (streams[mid].dct_off <= fi) lo = mid; else hi = mid - 1;
    }
    const int s = lo;
    const HcaStream st = streams[s];
    const int64_t k = fi - st.dct_off;
    const uint8_t *src = frames + st.frames_off + k * cfg.frame_size;
    uint8_t *rec = parsed + fi * ((int64_t)nch * kRecChannelBytes);
    const int frame_size = cfg.frame_size;

    // BitReader.ReadInt / PeekInt (Utilities/BitReader.cs:51-99) over the frame's bytes in HBM: a 64-bit window keeps the
    // next bits left-aligned, so a read is a shift; a refill happens once per 32 consumed bits from a word fetched at the
    // previous refill; bits past the end of the frame read as zero, like the reference
    auto word = [&](int i) -> uint32_t {
        uint32_t v = 0;
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (4 * i + j < frame_size) v |= (uint32_t)__ldg(src + 4 * i + j) << (24 - 8 * j);
        return v;
    };
    uint64_t win = ((uint64_t)word(0) << 32) | word(1);
    int avail = 64, next = 2;
    uint32_t ahead = word(2);
    auto peek = [&](int count) -> uint32_t { return (uint32_t)((win >> 1) >> (63 - count)); };
    auto skip = [&](int count) {
        win <<= count;
        avail -= count;
        if (avail <= 32) {
            win |= (uint64_t)ahead << (32 - avail);
            avail += 32;
            ahead = word(++next);
        }
    };
    auto read = [&](int count) -> int { const uint32_t v = peek(count); skip(count); return (int)v; };

    int status = 0;
    if (read(16) != 0xffff) status = VGB_HCA_BAD_SYNC;
    const int noise_level = read(9);
    const int eval_boundary = read(7);
    for (int c = 0; c < nch && !status; c++) {
        uint8_t *rc = rec + (size_t)c * kRecChannelBytes;
        const int type = cfg.channel_type[c];
        const int coded = type == 2 ? cfg.base_band_count : cfg.base_band_count + cfg.stereo_band_count;
        const int delta_bits = read(3);  // ReadScaleFactors (:108-126)
        int prev = 0;
        for (int b = 0; b < kBins; b++) {
            int sf = 0;
            if (b < coded && delta_bits != 0) {
                if (delta_bits >= 6 || b == 0) {
                    sf = read(6);
                } else {  // DeltaDecode (:183-208)
                    const int max_delta = 1 << (delta_bits - 1);
                    const int delta = read(delta_bits) - (max_delta - 1);  // ReadOffsetBinary, OffsetBias.Positive
                    if (delta < max_delta) {
                        sf = prev + delta;
                        if (sf < 0 || sf > 63) { status = VGB_HCA_BAD_DELTA; sf = 0; }
                    } else {
                        sf = read(6);
                    }
                }
            }
            prev = sf;
            int res = 0;
            if (b < coded && sf != 0) {  // CalculateResolution (CriHcaPacking.cs:60-69) of athCurve[b] + noise (:86-94)
                int pos = s_ath[b] + (b < eval_boundary ? noise_level - 1 : noise_level) - 5 * sf / 2 + 2;
                pos = min(max(pos, 0), 58);
                res = s_curve[pos];
            }
            rc[kRecScale + b] = (uint8_t)sf;
            rc[kRecRes + b] = (uint8_t)res;
            sres[((size_t)c * kBins + b) * kParseThreads + tid] = (uint8_t)res;
        }
        if (status) break;
        for (int i = 0; i < 8; i++) { rc[kRecIntensity + i] = 0; rc[kRecHfr + i] = 0; }
        if (type == 2) {
            for (int i = 0; i < kSub; i++) {
                int v = read(4);
                if (v > 14) { status = VGB_HCA_BAD_INDEX; v = 14; }
                rc[kRecIntensity + i] = (uint8_t)v;
            }
        } else if (cfg.hfr_group_count > 0) {
            for (int i = 0; i < cfg.hfr_group_count; i++) rc[kRecHfr + i] = (uint8_t)read(6);
        }
    }
    if (!status) {
        for (int sf = 0; sf < kSub; sf++)  // ReadSpectralCoefficients (:144-181)
            for (int c = 0; c < nch; c++) {
                const int type = cfg.channel_type[c];
                const int coded = type == 2 ? cfg.base_band_count : cfg.base_band_count + cfg.stereo_band_count;
                int16_t *q = reinterpret_cast<int16_t *>(rec + (size_t)c * kRecChannelBytes + kRecQuant) + sf * kBins;
                const uint8_t *rb = sres + (size_t)c * kBins * kParseThreads + tid;
                int res = coded > 0 ? rb[0] : 0;
                for (int b = 0; b < coded; b++) {
                    const int res_next = b + 1 < coded ? rb[(size_t)(b + 1) * kParseThreads] : 0;
                    const int mbits = s_maxbits[res];
                    const unsigned long long lens = s_lens64[res], vals = s_vals64[res];
                    const int code = (int)peek(mbits);
                    // both code families, selected without a branch (lanes parse different frames)
                    const int bits_p = (int)((lens >> (4 * code)) & 15u);
                    const int v_p = (int)((unsigned)(vals >> (4 * code)) << 28) >> 28;
                    const int mag = code >> 1;
                    const int v_s = (code & 1) ? -mag : mag;
                    const int bits_s = mbits - (mag == 0 ? 1 : 0);
                    const bool prefix = mbits <= 4;
                    q[b] = (int16_t)(prefix ? v_p : v_s);
                    skip(prefix ? bits_p : bits_s);
                    res = res_next;
                }
                for (int b = coded; b < kBins; b++) q[b] = 0;
            }
    } else {
        atomicCAS(status_out + s, 0, status);
        for (int e = 0; e < nch * kRecChannelBytes; e++) rec[e] = 0;
    }
}

__global__ void __launch_bounds__(128)
hca_decode_unpack_kernel(const uint8_t *__restrict__ parsed, const HcaStream *__restrict__ streams, HcaConfig cfg,
                         HcaTables T, double *__restrict__ edge, int16_t *__restrict__ pcm)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int nch = cfg.channel_count;
    double *spectra = reinterpret_cast<double *>(smem_raw);                   // [nch][8][128]
    double *work = spectra + (size_t)nch * kSub * kBins;                      // [2][128]
    int *quantized = reinterpret_cast<int *>(work + 2 * kBins);               // [nch][8][128]
    HcaChannelState *chs = reinterpret_cast<HcaChannelState *>(quantized + (size_t)nch * kSub * kBins);

    const int tid = threadIdx.x;
    const int s = blockIdx.y, k = blockIdx.x;
    const HcaStream st = streams[s];
    if (k >= st.frame_count) return;

    // ---- the frame as hca_decode_parse_kernel left it: scale factors, resolutions, side information, quantised
    // coefficients (coalesced reads of the record)
    const uint8_t *rec = parsed + ((int64_t)st.dct_off + k) * ((int64_t)nch * kRecChannelBytes);
    for (int c = 0; c < nch; c++) {
        const uint8_t *rc = rec + (size_t)c * kRecChannelBytes;
        HcaChannelState &ch = chs[c];
        if (tid == 0) {
            ch.type = cfg.channel_type[c];
            ch.coded_count = cfg.channel_type[c] == 2 ? cfg.base_band_count : cfg.base_band_count + cfg.stereo_band_count;
        }
        ch.scale_factors[tid] = rc[kRecScale + tid];
        ch.resolution[tid] = rc[kRecRes + tid];
        if (tid < kSub) { ch.intensity[tid] = rc[kRecIntensity + tid]; ch.hfr_scales[tid] = rc[kRecHfr + tid]; }
        const int16_t *rq = reinterpret_cast<const int16_t *>(rc + kRecQuant);
        int *q = quantized + (size_t)c * kSub * kBins;
#pragma unroll
        for (int j = 0; j < kSub; j++) q[j * kBins + tid] = rq[j * kBins + tid];
    }
    __syncthreads();

    // ---- DequantizeFrame (CriHcaDecoder.cs:72-105): thread = band
    for (int c = 0; c < nch; c++) {
        const int b = tid;
        const double gain = b < chs[c].coded_count ? T.dequantizer_scaling[chs[c].scale_factors[b]] * T.step_size[chs[c].resolution[b]] : 0.0;
#pragma unroll
        for (int sf = 0; sf < kSub; sf++)
            spectra[((size_t)c * kSub + sf) * kBins + b] = b < chs[c].coded_count ? quantized[((size_t)c * kSub + sf) * kBins + b] * gain : 0.0;
    }
    __syncthreads();
    // ---- ReconstructHighFrequency (:106-134): every high band is a scaled copy of a low band
    if (cfg.hfr_group_count != 0) {
        const int total = min(cfg.total_band_count, 127);
        const int start = cfg.base_band_count + cfg.stereo_band_count;
        const int hfr_bands = min(cfg.hfr_band_count, total - cfg.hfr_band_count);
        for (int c = 0; c < nch; c++) {
            if (chs[c].type == 2) continue;
            const int band = tid;
            if (band < hfr_bands && band / cfg.bands_per_hfr_group < cfg.hfr_group_count) {
                const int group = band / cfg.bands_per_hfr_group;
                const int high = start + band, low = start - band - 1;
                const int index = chs[c].hfr_scales[group] - chs[c].scale_factors[low] + 64;
                const double conv = T.scale_conversion[index];
#pragma unroll
                for (int sf = 0; sf < kSub; sf++)
                    spectra[((size_t)c * kSub + sf) * kBins + high] = conv * spectra[((size_t)c * kSub + sf) * kBins + low];
            }
        }
        __syncthreads();
    }
    // ---- ApplyIntensityStereo (:135-157)
    if (cfg.stereo_band_count > 0) {
        for (int c = 0; c < nch; c++) {
            if (chs[c].type != 1) continue;
            const int b = tid;
            if (b >= cfg.base_band_count && b < cfg.total_band_count) {
#pragma unroll
                for (int sf = 0; sf < kSub; sf++) {
                    const double rl = T.intensity_ratio[chs[c + 1].intensity[sf]];
                    const double rr = rl - 2.0;
                    double &l = spectra[((size_t)c * kSub + sf) * kBins + b];
                    spectra[((size_t)(c + 1) * kSub + sf) * kBins + b] = l * rr;
                    l *= rl;
                }
            }
        }
        __syncthreads();
    }

    // ---- the DCT-IV of RunImdct (Mdct.cs:107): two subframes at a time, each output replaces its input in `spectra`
    const int grp = tid >> 6, i = tid & 63;
    double *t = work + grp * kBins;
    for (int c = 0; c < nch; c++) {
        for (int sf2 = 0; sf2 < kSub; sf2 += 2) {
            const int sf = sf2 + grp;
            double *io = spectra + ((size_t)c * kSub + sf) * kBins;
            {
                const int i2 = i * 2;
                const double a = io[i2], b = io[kBins - 1 - i2];
                const double sn = T.sin_tab[7][i], cs = T.cos_tab[7][i];
                t[i2] = a * cs + b * sn;
                t[i2 + 1] = a * sn - b * cs;
            }
            __syncthreads();
#pragma unroll 1
            for (int stage = 0; stage < 6; stage++) {
                const int block_bits = 6 - stage, half_bits = block_bits - 1;
                const int block_size = 1 << block_bits, block_half = 1 << half_bits;
                if (i < 32) {  // a 128-point stage has 32 butterflies of two complex pairs each
                    const int block = i >> half_bits, j = i & (block_half - 1);
                    const int front = (block * block_size + j) * 2, back = front + block_size;
                    const double a = t[front] - t[back];
                    const double b = t[front + 1] - t[back + 1];
                    const double sn = T.sin_tab[half_bits][j], cs = T.cos_tab[half_bits][j];
                    const double f0 = t[front] + t[back], f1 = t[front + 1] + t[back + 1];
                    t[front] = f0;
                    t[front + 1] = f1;
                    t[back] = a * cs + b * sn;
                    t[back + 1] = a * sn - b * cs;
                }
                __syncthreads();
            }
            io[i] = t[T.shuffle[i]] * T.mdct_scale;
            io[64 + i] = t[T.shuffle[64 + i]] * T.mdct_scale;
            __syncthreads();
        }
    }

    // ---- window + overlap-add (Mdct.cs:108-117).  The overlap buffer a subframe sees is a pure function of the
    // previous subframe's DCT output, so subframes 1..7 finish here; subframe 0 needs the previous FRAME's tail, so its
    // two addends go to HBM (head = this frame's products, tail = the overlap terms subframe 7 leaves behind) and
    // hca_decode_seam_kernel adds them.  thread = (h, i): h = 0 -> output[i], h = 1 -> output[i + 64].
    const int h = grp;
    for (int c = 0; c < nch; c++) {
        int16_t *dst = pcm + st.pcm_off + (int64_t)c * st.channel_stride;
        const double *d = spectra + (size_t)c * kSub * kBins;
        double *e = edge + (((size_t)st.dct_off + k) * nch + c) * 2 * kBins;
        auto product = [&](const double *cur) {  // this subframe's own term
            return h == 0 ? T.window[i] * cur[i + 64] : T.window[i + 64] * -cur[kBins - 1 - i];
        };
        auto overlap = [&](const double *prev) {  // what the previous subframe left in the overlap buffer
            return h == 0 ? T.window[kBins - 1 - i] * -prev[64 - i - 1] : T.window[64 - i - 1] * prev[i];
        };
        e[tid] = product(d);
        e[kBins + tid] = overlap(d + 7 * kBins);
#pragma unroll 1
        for (int sf = 1; sf < kSub; sf++) {
            const double a = product(d + sf * kBins), p = overlap(d + (sf - 1) * kBins);
            const int64_t pos = (int64_t)k * kFrame + sf * kBins + tid - st.inserted_samples;
            if (pos >= 0 && pos < st.sample_count) dst[pos] = hca_pcm_float_to_short(h == 0 ? a + p : a - p);
        }
    }
}

// First subframe of every frame: head(k) +/- tail(k-1).  grid: x = frame, y = channel, z = stream; 128 threads.
__global__ void __launch_bounds__(128)
hca_decode_seam_kernel(const double *__restrict__ edge, const HcaStream *__restrict__ streams, HcaConfig cfg,
                       int16_t *__restrict__ pcm)
{
    const int k = blockIdx.x, c = blockIdx.y, s = blockIdx.z;
    const HcaStream st = streams[s];
    if (k >= st.frame_count) return;
    const int nch = cfg.channel_count, tid = threadIdx.x;
    const double a = edge[((((size_t)st.dct_off + k) * nch + c) * 2) * kBins + tid];
    const double p = k > 0 ? edge[((((size_t)st.dct_off + k - 1) * nch + c) * 2 + 1) * kBins + tid] : 0.0;
    const int64_t pos = (int64_t)k * kFrame + tid - st.inserted_samples;
    if (pos >= 0 && pos < st.sample_count)
        pcm[st.pcm_off + (int64_t)c * st.channel_stride + pos] = hca_pcm_float_to_short(tid < 64 ? a + p : a - p);
}

// ---- Mdct.RunMdct / RunImdct (Utilities/Mdct.cs:63-119) for the codec's 128-point instance, as a batch --------------------
// The unit-parity taps SURVEY §8(b) asks for (vgb_mdct128_batch / vgb_imdct128_batch): sequences of 128-sample blocks,
// each sequence starting from the all-zero state of a fresh Mdct object.  Block k of RunMdct reads input blocks k-1 and
// k; block k of RunImdct needs the DCT-IV of spectra k-1 and k: both are independent per block, one CTA of 64 threads
// each.  Same window (CriHcaTables.MdctWindow), scale sqrt(2/128) and operation order as the codec kernels above.
__device__ __forceinline__ void hca_dct4_128(double *t, const double *in, const HcaTables &T, int i)
{
    {   // Dct4 pre-twiddle (Mdct.cs:137-147)
        const int i2 = i * 2;
        const double a = in[i2], b = in[kBins - 1 - i2];
        const double sn = T.sin_tab[7][i], cs = T.cos_tab[7][i];
        __syncthreads();  // `in` may alias `t`
        t[i2] = a * cs + b * sn;
        t[i2 + 1] = a * sn - b * cs;
    }
    __syncthreads();
#pragma unroll 1
    for (int stage = 0; stage < 6; stage++) {  // (Mdct.cs:148-175)
        const int block_bits = 6 - stage, half_bits = block_bits - 1;
        const int block_size = 1 << block_bits, block_half = 1 << half_bits;
        if (i < 32) {
            const int block = i >> half_bits, j = i & (block_half - 1);
            const int front = (block * block_size + j) * 2, back = front + block_size;
            const double a = t[front] - t[back];
            const double b = t[front + 1] - t[back + 1];
            const double sn = T.sin_tab[half_bits][j], cs = T.cos_tab[half_bits][j];
            const double f0 = t[front] + t[back], f1 = t[front + 1] + t[back + 1];
            t[front] = f0;
            t[front + 1] = f1;
            t[back] = a * cs + b * sn;
            t[back + 1] = a * sn - b * cs;
        }
        __syncthreads();
    }
}

// grid: x = block, y = sequence; in/out [seq][blocks][128]
__global__ void __launch_bounds__(64)
hca_mdct128_kernel(const double *__restrict__ in, double *__restrict__ out, int n_blocks, HcaTables T)
{
    __shared__ double fold[kBins], t[kBins];
    const int k = blockIdx.x, i = threadIdx.x;
    const double *cur = in + ((size_t)blockIdx.y * n_blocks + k) * kBins;
    const double *prev = cur - kBins;  // Mdct._mdctPrevious: zeros for the first block (:71)
    auto pv = [&](int j) -> double { return k > 0 ? prev[j] : 0.0; };
    {   // window + fold (Mdct.cs:77-85)
        const double a = T.window[64 - i - 1] * -cur[64 + i];
        const double b = T.window[64 + i] * cur[64 - i - 1];
        const double cc = T.window[i] * pv(i);
        const double d = T.window[kBins - i - 1] * pv(kBins - i - 1);
        fold[i] = a - b;
        fold[64 + i] = cc - d;
    }
    __syncthreads();
    hca_dct4_128(t, fold, T, i);
    double *o = out + ((size_t)blockIdx.y * n_blocks + k) * kBins;
    o[i] = t[T.shuffle[i]] * T.mdct_scale;            // (Mdct.cs:177-180)
    o[64 + i] = t[T.shuffle[64 + i]] * T.mdct_scale;
}

__global__ void __launch_bounds__(64)
hca_imdct128_kernel(const double *__restrict__ in, double *__restrict__ out, int n_blocks, HcaTables T)
{
    __shared__ double cur_d[kBins], prev_d[kBins], t[kBins];
    const int k = blockIdx.x, i = threadIdx.x;
    const double *cur = in + ((size_t)blockIdx.y * n_blocks + k) * kBins;
    hca_dct4_128(t, cur, T, i);                       // Dct4 of this block (Mdct.cs:107)
    cur_d[i] = t[T.shuffle[i]] * T.mdct_scale;
    cur_d[64 + i] = t[T.shuffle[64 + i]] * T.mdct_scale;
    __syncthreads();
    if (k > 0) {                                      // ... and of the previous one: it left the overlap buffer (:114-117)
        hca_dct4_128(t, cur - kBins, T, i);
        prev_d[i] = t[T.shuffle[i]] * T.mdct_scale;
        prev_d[64 + i] = t[T.shuffle[64 + i]] * T.mdct_scale;
    } else {
        prev_d[i] = 0.0;
        prev_d[64 + i] = 0.0;
    }
    __syncthreads();
    double *o = out + ((size_t)blockIdx.y * n_blocks + k) * kBins;
    // output[i] = window[i] * dct[i + 64] + previous[i];  output[i + 64] = window[i + 64] * -dct[127 - i] - previous[i + 64]
    // previous[i] = window[127 - i] * -prevDct[63 - i];   previous[i + 64] = window[63 - i] * prevDct[i]      (:108-117)
    const double p0 = k > 0 ? T.window[kBins - 1 - i] * -prev_d[64 - i - 1] : 0.0;
    const double p1 = k > 0 ? T.window[64 - i - 1] * prev_d[i] : 0.0;
    o[i] = T.window[i] * cur_d[i + 64] + p0;
    o[i + 64] = T.window[i + 64] * -cur_d[kBins - 1 - i] - p1;
}

cudaError_t launch_hca_mdct128(const double *in, double *out, int n_sequences, int n_blocks, bool inverse, const HcaTables &tables,
                               cudaStream_t stream)
{
    if (n_sequences <= 0 || n_blocks <= 0) return cudaSuccess;
    const dim3 grid((unsigned)n_blocks, (unsigned)n_sequences);
    if (inverse) hca_imdct128_kernel<<<grid, 64, 0, stream>>>(in, out, n_blocks, tables);
    else hca_mdct128_kernel<<<grid, 64, 0, stream>>>(in, out, n_blocks, tables);
    return cudaGetLastError();
}

size_t hca_decode_smem_bytes(const HcaConfig &cfg)
{
    const size_t nch = (size_t)cfg.channel_count;
    return nch * kSub * kBins * sizeof(double) + 2 * kBins * sizeof(double) + nch * kSub * kBins * sizeof(int) +
           nch * sizeof(HcaChannelState) + 16;
}

size_t hca_decode_parsed_bytes(const HcaConfig &cfg, int64_t total_frames)
{
    return (size_t)total_frames * (size_t)cfg.channel_count * kRecChannelBytes;
}

cudaError_t launch_hca_decode(const uint8_t *frames, const HcaStream *streams, int n_streams, int max_frames,
                              int64_t total_frames, const HcaConfig &cfg, const HcaTables &tables, uint8_t *parsed_scratch,
                              double *edge_scratch, int16_t *pcm, int32_t *status_out, cudaStream_t stream)
{
    if (n_streams <= 0 || max_frames <= 0 || total_frames <= 0) return cudaSuccess;
    const size_t smem_p = (size_t)cfg.channel_count * kBins * kParseThreads;
    cudaError_t e = raise_dynamic_smem(hca_decode_parse_kernel, smem_p);
    if (e != cudaSuccess) return e;
    const unsigned blocks_p = (unsigned)((total_frames + kParseThreads - 1) / kParseThreads);
    hca_decode_parse_kernel<<<blocks_p, kParseThreads, smem_p, stream>>>(frames, streams, n_streams, total_frames, cfg, tables,
                                                                         parsed_scratch, status_out);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const size_t smem = hca_decode_smem_bytes(cfg);
    e = raise_dynamic_smem(hca_decode_unpack_kernel, smem);
    if (e != cudaSuccess) return e;
    dim3 grid_a((unsigned)max_frames, (unsigned)n_streams);
    hca_decode_unpack_kernel<<<grid_a, 128, smem, stream>>>(parsed_scratch, streams, cfg, tables, edge_scratch, pcm);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    dim3 grid_b((unsigned)max_frames, (unsigned)cfg.channel_count, (unsigned)n_streams);
    hca_decode_seam_kernel<<<grid_b, 128, 0, stream>>>(edge_scratch, streams, cfg, pcm);
    return cudaGetLastError();
}

size_t hca_encode_smem_bytes(const HcaConfig &cfg)
{
    const size_t nch = (size_t)cfg.channel_count;
    return 2 * nch * kSub * kBins * sizeof(double) + 4 * kBins * sizeof(double) + nch * sizeof(HcaChannelState) +
           (size_t)((cfg.frame_size + 15) & ~15) + 8 * sizeof(int) + nch * kBins * 16 + 16;
}

cudaError_t launch_hca_encode(const int16_t *pcm, const HcaStream *streams, int n_streams, int max_frames,
                              const HcaConfig &cfg, const HcaTables &tables, uint8_t *frames_out, int32_t *status_out,
                              cudaStream_t stream)
{
    if (n_streams <= 0 || max_frames <= 0) return cudaSuccess;
    const size_t smem = hca_encode_smem_bytes(cfg);
    cudaError_t e = raise_dynamic_smem(hca_encode_kernel, smem);
    if (e != cudaSuccess) return e;
    dim3 grid((unsigned)max_frames, (unsigned)n_streams);
    hca_encode_kernel<<<grid, 128, smem, stream>>>(pcm, streams, cfg, tables, frames_out, status_out);
    return cudaGetLastError();
}

}  // namespace vgb
