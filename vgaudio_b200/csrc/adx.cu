// adx.cu — CRI ADX 4-bit ADPCM encode / decode on sm_90a (H100).
//
// Replaces CriAdxCodec.Encode / EncodeFrame / Decode (Codecs/CriAdx/CriAdxCodec.cs:9-171).  Like GC-ADPCM the codec
// is a serial recurrence per channel (the next frame starts from the reconstructed last two samples, :98-99,:137),
// but there is no predictor search, so one THREAD owns one channel and the batch supplies the parallelism.  Each
// frame: residual range against raw neighbours (:112-118), CalculateScale (:149-165), then the quantise /
// reconstruct recurrence with its one fp64 multiply + truncation per sample (:126).
// Latency bound (one fp64 multiply, two conversions and ~10 integer ops per sample on the dependent chain);
// algorithmic traffic 2 B/sample in + frame_size/samples_per_frame B/sample out (2.5625 B/sample at 18-byte frames).
// The standard layout (18-byte frames, no padding) streams privately per thread: cp.async copies a frame's 32 samples
// (encoder, four 16-byte chunks) or 8 frames' 144 bytes (decoder, nine chunks) into the thread's own shared-memory ring
// two steps ahead, results leave as halfword / 16-byte stores straight from registers (partial sectors merge in L2), so
// DRAM latency never reaches the recurrence.  Other frame sizes / padded streams / a partial last frame take the general loop.
#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace vgb {

// (int)double on x64 is cvttsd2si: out-of-range and NaN give 0x80000000 (SURVEY.md A.8); CUDA's cvt saturates.
__device__ __forceinline__ int32_t cast_double_to_int_x64(double v)
{
    return (v > -2147483649.0 && v < 2147483648.0) ? __double2int_rz(v) : INT32_MIN;
}

// ScaleShortToNibble (:167-171): (s + 2340*sign(s)) / 4681 truncating, Clamp4
__device__ __forceinline__ int32_t adx_short_to_nibble(int32_t s)
{
    const int32_t sgn = (s > 0) - (s < 0);
    return clamp4((s + 2340 * sgn) / 4681);
}

constexpr int kAdxThreads = 32;   // one warp per CTA: spreads a few thousand channels over all SMs
constexpr int kAdxStages = 3;     // cp.async ring depth (kAdxStages - 1 frames / frame groups in flight)
constexpr int kAdxDecGroup = 8;   // decoder: 8 frames = 144 B = nine 16-byte chunks per thread and step

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src)
{
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}

// a*b + c as ONE multiply-add the compiler may not re-associate
__device__ __forceinline__ int32_t adx_imad(int32_t a, int32_t b, int32_t c)
{
    int32_t d;
    asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// ---------------------------------------------------------------------------------------------------------
// The quantiser of pass 2 (:126,:167-171) in integers.  Reference:
//     scaled = Clamp16((int)(raw * gain)),  gain = 32767.0 / maxDistance (double);   q = Clamp4((scaled +- 2340) / 4681)
// q only counts how many of the thresholds T_k = 4681 k - 2340 (k = 1..7) |scaled| reaches, and truncation / Clamp16 do
// not move a value across an integer threshold, so with a = |raw|:
//     q = sign(raw) * #{ k : a * 32767 >= T_k * maxDistance }
// (the two fp64 roundings move the product by < 1e-11 while a * 32767 / maxDistance is at least 1 / maxDistance away
// from T_k unless equal, which the factorisation 32767 = 7 * 31 * 151 restricts to maxDistance = 4681 j).  Two corner
// cases: maxDistance == 0 gives gain 0 and q = 0; a * 32767 >= 2^31 * maxDistance overflows the (int) cast, which is
// INT_MIN on x64, hence q = -7 whatever the sign.  tools/adx_quantiser_check.c enumerates the identity for every
// maxDistance (0..32768) around every threshold and over the full raw range for small maxDistance: 0 mismatches.
// Per frame: the seven products M_k = T_k * maxDistance (< 2^30) and the overflow bound; per sample a three-step
// binary search over them instead of int->double, fp64 multiply, double->int, a division by 4681 and two clamps.
// ---------------------------------------------------------------------------------------------------------
struct AdxQuant {
    uint32_t m[8];     // m[k] = T_k * maxDistance for k = 1..7 (m[0] unused)
    uint32_t ovf;      // smallest |raw| whose product leaves int32 (0xFFFFFFFF: none below 2^18)
    bool zero;         // maxDistance == 0
};
__device__ __forceinline__ AdxQuant adx_quant_setup(int32_t max_distance)
{
    AdxQuant qz;
#pragma unroll
    for (int k = 1; k < 8; k++) qz.m[k] = (uint32_t)(4681 * k - 2340) * (uint32_t)max_distance;
    qz.m[0] = 0;
    qz.zero = max_distance == 0;
    // a * 32767 >= 2^31 * md  <=>  a >= ceil(2^31 * md / 32767); only md <= 3 can be reached by |raw| < 2^18
    qz.ovf = (max_distance >= 1 && max_distance <= 3) ? (uint32_t)((((uint64_t)max_distance << 31) + 32766u) / 32767u) : 0xFFFFFFFFu;
    return qz;
}
__device__ __forceinline__ int32_t adx_quantise(int32_t raw, const AdxQuant &qz)
{
    const uint32_t a = (uint32_t)abs(raw);
    const uint32_t v = min(a, 65535u) * 32767u;  // |raw| >= 30428 already reaches T_7 for every maxDistance <= 32768
    const bool c4 = v >= qz.m[4];
    const bool c2 = v >= (c4 ? qz.m[6] : qz.m[2]);
    const bool c1 = v >= (c4 ? (c2 ? qz.m[7] : qz.m[5]) : (c2 ? qz.m[3] : qz.m[1]));
    const int32_t k = (c4 ? 4 : 0) + (c2 ? 2 : 0) + (c1 ? 1 : 0);
    int32_t q = raw < 0 ? -k : k;
    q = a >= qz.ovf ? -7 : q;
    return qz.zero ? 0 : q;
}

// EncodeFrame (:107-147) for one whole frame of the standard layout (32 samples in x[], history h2 = pcm[0],
// h1 = pcm[1]); writes the 18 bytes at out16 and leaves the reconstructed pair in (h1, h2).
template <bool kV4>
__device__ __forceinline__ void adx_encode_frame_std(const int32_t (&x)[32], int32_t c0, int32_t c1, bool exponential, int type, int filter,
                                                     int32_t &h1, int32_t &h2, uint16_t *out16)
{
    int32_t max_distance = 0;  // pass 1 (:112-118): neighbours are RAW samples except for the two history slots
    {
        int32_t p0 = h2, p1 = h1;
#pragma unroll
        for (int i = 0; i < 32; i++) {
            const int32_t predicted = (wmul(p1, c0) >> 12) + (wmul(p0, c1) >> 12);
            max_distance = max(max_distance, abs(clamp16(x[i] - predicted)));
            p0 = p1;
            p1 = x[i];
        }
    }
    int32_t scale = (max_distance - 1) / 7 + 1;  // CalculateScale (:149-165)
    if (scale > 0x1000) scale = 0x1000;
    int32_t scale_out = scale - 1;
    if (exponential) {
        const int power = scale_out == 0 ? 0 : (31 - __clz(scale_out)) + 1;
        scale = 1 << power;
        scale_out = 12 - power;
        max_distance = 8 * scale - 1;
    }
    const AdxQuant qz = adx_quant_setup(max_distance);  // gain = 32767.0 / maxDistance, in integers
    const uint32_t hdr0 = ((uint32_t)(scale_out >> 8) & 0x1fu) | (type == 2 ? (uint32_t)(filter << 5) : 0u);
    out16[0] = (uint16_t)((hdr0 & 0xFFu) | (((uint32_t)scale_out & 0xFFu) << 8));  // :140-141
    // pass 2 (:122-138).  Clamp16(scale * q) (:131) is the identity here: scale <= 0x1000 (:151-163) and q in [-8, 7]
    // give a product in [-32768, 28672], so it is left out of the dependent chain.
    uint32_t hw = 0;
#pragma unroll
    for (int i = 0; i < 32; i++) {
        int32_t predicted = (wmul(h1, c0) >> 12) + (wmul(h2, c1) >> 12);
        const int32_t q = adx_quantise(x[i] - predicted, qz);
        if (kV4) predicted = wadd(wmul(h1, c0), wmul(h2, c1)) >> 12;
        const int32_t recon = clamp16(wmul(scale, q) + predicted);
        h2 = h1;
        h1 = recon;
        // byte = (q_even << 4) | q_odd; halfword = byte0 | byte1 << 8
        const int sh = ((i & 1) ? 0 : 4) + ((i & 2) ? 8 : 0);
        hw |= ((uint32_t)q & 0xFu) << sh;
        if ((i & 3) == 3) { out16[1 + (i >> 2)] = (uint16_t)hw; hw = 0; }
    }
}

// ---------------------------------------------------------------------------------------------------------
// TIME-PARALLEL ENCODING, as for GC-ADPCM (gc_encode.cu): a frame depends on its predecessors only through the two
// reconstructed samples it starts from (:98-99,:137), and the fixed high-pass predictor (pole radius ~0.9) forgets a
// wrong pair within a handful of frames.  The whole frames of a standard-layout channel are cut into seg_count segments:
//   kAdxChain    thread = (channel, segment): segment 0 from the true history, the others from the raw samples in
//                front of them; bytes and, per frame, the pair handed on (`trace`) are written
//   kAdxRunOn    thread = (channel, boundary): the chain of segment s-1 runs on into segment s until its pair equals the
//                recorded one (from there the recorded chain is the true one), inside its segment, noting its start pair
//   kAdxCascade  thread = channel: repairs a boundary whose predecessor's end pair changed afterwards (serially, across
//                segment ends if need be), then encodes the partial last frame from the true pair
// Exact by construction: the only test is equality of two int16 pairs.  Channels with another frame size or padding
// keep the plain serial loop (segment 0's thread).
// ---------------------------------------------------------------------------------------------------------
constexpr int kAdxChain = 0, kAdxRunOn = 1, kAdxCascade = 2;
__host__ __device__ __forceinline__ int adx_seg_len(int whole_frames, int seg_count, int min_seg)
{
    const int per = (whole_frames + (seg_count > 0 ? seg_count : 1) - 1) / (seg_count > 0 ? seg_count : 1);
    return per < min_seg ? min_seg : per;
}

// General loop of Encode (:76-101): any frame size, padding, partial frames; frames [f_first, frame_count).
__device__ void adx_encode_general(const AdxChannel &c, const int16_t *__restrict__ src, uint8_t *__restrict__ dst, int f_first,
                                   int32_t &h1, int32_t &h2)
{
    const int spf = (c.frame_size - 2) * 2;
    const int sample_count = c.n_samples + c.padding;            // :59
    const int frame_count = div_round_up(sample_count, spf);     // :61
    const int32_t c0 = c.coef0, c1 = c.coef1;
    const bool v4 = c.version == 4;
    const bool exponential = c.type == 4;
    int padding_remaining = c.padding;
    for (int f = 0; f < f_first && padding_remaining != 0; f++) padding_remaining -= min(padding_remaining, min(sample_count - f * spf, spf));
    for (int f = f_first; f < frame_count; f++) {
        int to_copy = min(sample_count - f * spf, spf);  // :78
        int lead = 0;                                    // zero samples in front (pcmBufferStart - 2)
        if (padding_remaining != 0) {                    // :80-89
            const int eat = min(padding_remaining, to_copy);
            padding_remaining -= eat;
            to_copy -= eat;
            lead = eat;
        }
        uint8_t *out = dst + (int64_t)f * c.frame_size;
        if (to_copy == 0 && lead > 0) {  // `continue`: the frame stays all-zero and the history is untouched
            for (int b = 0; b < c.frame_size; b++) out[b] = 0;
            continue;
        }
        const int64_t first = max((int64_t)f * spf - c.padding, (int64_t)0);  // :90
        auto sample_at = [&](int i) -> int32_t {  // pcmBuffer[i + 2]
            const int k = i - lead;
            return (k >= 0 && k < to_copy) ? (int32_t)__ldg(src + first + k) : 0;
        };
        // pass 1 (:112-118): neighbours are the RAW samples except for the two history slots
        int32_t max_distance = 0;
        {
            int32_t p0 = h2, p1 = h1;
            for (int i = 0; i < spf; i++) {
                const int32_t cur = sample_at(i);
                const int32_t predicted = (wmul(p1, c0) >> 12) + (wmul(p0, c1) >> 12);
                max_distance = max(max_distance, abs(clamp16(cur - predicted)));
                p0 = p1;
                p1 = cur;
            }
        }
        int32_t scale = (max_distance - 1) / 7 + 1;  // CalculateScale (:149-165)
        if (scale > 0x1000) scale = 0x1000;
        int32_t scale_out = scale - 1;
        if (exponential) {
            const int power = scale_out == 0 ? 0 : (31 - __clz(scale_out)) + 1;  // Helpers.Log2 = floor(log2)
            scale = 1 << power;
            scale_out = 12 - power;
            max_distance = 8 * scale - 1;
        }
        const AdxQuant qz = adx_quant_setup(max_distance);
        // pass 2 (:122-138): quantise + reconstruct, feeding the reconstruction back
        uint32_t pair = 0;
        out[0] = (uint8_t)(((scale_out >> 8) & 0x1f) | (c.type == 2 ? (c.filter << 5) : 0));  // :140, :95
        out[1] = (uint8_t)scale_out;                                                           // :141
        for (int i = 0; i < spf; i++) {
            const int32_t cur = sample_at(i);
            int32_t predicted = (wmul(h1, c0) >> 12) + (wmul(h2, c1) >> 12);
            const int32_t q = adx_quantise(cur - predicted, qz);
            const int32_t decoded_distance = clamp16(wmul(scale, q));
            if (v4) predicted = wadd(wmul(h1, c0), wmul(h2, c1)) >> 12;
            const int32_t recon = clamp16(decoded_distance + predicted);
            h2 = h1;
            h1 = recon;
            if (i & 1) out[2 + (i >> 1)] = (uint8_t)(pair | (uint32_t)(q & 0xF));  // CombineNibbles (:145)
            else pair = (uint32_t)(q << 4) & 0xF0u;
        }
    }
}

template <int kMode>
__global__ void __launch_bounds__(kAdxThreads)
adx_encode_kernel(const int16_t *__restrict__ pcm, const AdxChannel *__restrict__ tab, int n_channels,
                  uint8_t *__restrict__ adpcm, int16_t *__restrict__ history_out, AdxSegArgs sa)
{
    __shared__ __align__(16) uint4 enc_ring[kAdxStages][4][kAdxThreads];  // [stage][16-byte chunk of the frame][thread]
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= n_channels) return;
    const AdxChannel c = tab[ch];
    const int16_t *src = pcm + c.pcm_off;
    uint8_t *dst = adpcm + c.adpcm_off;
    const int32_t c0 = c.coef0, c1 = c.coef1;
    const bool v4 = c.version == 4;
    const bool exponential = c.type == 4;
    const bool standard = c.frame_size == 18 && c.padding == 0;
    const int whole = standard ? c.n_samples / 32 : 0;            // frames of the standard layout with all 32 samples
    const int seg_len = adx_seg_len(whole, sa.seg_count, sa.min_seg_frames);
    uint32_t *trace = sa.trace + c.trace_off;                     // [frame] recon pair handed on: (h1 & 0xFFFF) | h2 << 16
    uint32_t *used_start = sa.used_start + (int64_t)ch * sa.seg_count;

    // frames [f_lo, f_hi) of the standard layout from the pair (h1, h2); kSplice: stop once the pair after a frame equals
    // the recorded one.  Returns the number of frames encoded.
    auto run = [&](int f_lo, int f_hi, int32_t &h1, int32_t &h2, bool splice) -> int {
        const uint4 *vin = reinterpret_cast<const uint4 *>(src);  // pcm_off is a multiple of 8 samples
        auto issue = [&](int f) {  // frame f -> ring stage (cp.async: no register scoreboard to wait on)
            if (f < f_hi) {
#pragma unroll
                for (int j = 0; j < 4; j++) cp_async16(&enc_ring[(f - f_lo) % kAdxStages][j][threadIdx.x], vin + (int64_t)f * 4 + j);
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
#pragma unroll
        for (int a = 0; a < kAdxStages - 1; a++) issue(f_lo + a);
        int done = 0;
        for (int f = f_lo; f < f_hi; f++) {
            issue(f + kAdxStages - 1);
            asm volatile("cp.async.wait_group %0;" ::"n"(kAdxStages - 1) : "memory");
            int32_t x[32];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint4 v = enc_ring[(f - f_lo) % kAdxStages][j][threadIdx.x];
                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    x[8 * j + 2 * k] = (int32_t)(int16_t)(w[k] & 0xFFFFu);
                    x[8 * j + 2 * k + 1] = (int32_t)w[k] >> 16;
                }
            }
            uint16_t *out16 = reinterpret_cast<uint16_t *>(dst + (int64_t)f * 18);  // adpcm_off is even
            if (v4) adx_encode_frame_std<true>(x, c0, c1, exponential, c.type, c.filter, h1, h2, out16);
            else adx_encode_frame_std<false>(x, c0, c1, exponential, c.type, c.filter, h1, h2, out16);
            const uint32_t pair = ((uint32_t)h1 & 0xFFFFu) | ((uint32_t)h2 << 16);
            done++;
            if (splice && trace[f] == pair) break;  // the recorded chain continues from exactly this pair
            trace[f] = pair;
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        return done;
    };

    if (kMode == kAdxChain) {
        const int s = blockIdx.y;
        int32_t h2 = 0, h1 = 0;  // pcmBuffer[0], pcmBuffer[1]
        if (s == 0) {
            int16_t hist_cfg = 0;
            if (v4 && c.padding == 0 && c.n_samples > 0) {  // :69-74
                h2 = h1 = src[0];
                hist_cfg = src[0];
            }
            if (history_out) history_out[ch] = hist_cfg;
        }
        if (!standard) {
            if (s == 0) adx_encode_general(c, src, dst, 0, h1, h2);
            return;
        }
        const int f_lo = s * seg_len, f_hi = min(f_lo + seg_len, whole);
        if (f_lo < f_hi) {
            if (s > 0) {  // speculative start: the raw samples in front of the segment
                h1 = src[(int64_t)f_lo * 32 - 1];
                h2 = src[(int64_t)f_lo * 32 - 2];
            }
            run(f_lo, f_hi, h1, h2, false);
        }
        // a single-segment launch has no cascade: the partial last frame follows right here
        if (sa.seg_count == 1 && s == 0) adx_encode_general(c, src, dst, whole, h1, h2);
        return;
    }
    if (!standard) return;
    if (kMode == kAdxRunOn) {
        const int s = blockIdx.y + 1;
        const int f_lo = s * seg_len, f_hi = min(f_lo + seg_len, whole);
        if (f_lo >= f_hi) return;
        const uint32_t start = trace[f_lo - 1];
        used_start[s] = start;
        int32_t h1 = (int32_t)(int16_t)(start & 0xFFFFu), h2 = (int32_t)(int16_t)(start >> 16);
        const int done = run(f_lo, f_hi, h1, h2, true);
        atomicAdd(&sa.stats[0], (unsigned long long)done);
        return;
    }
    // cascade: one thread per channel walks the boundaries in order
    int truth_upto = 0;
    for (int s = 1; s < sa.seg_count; s++) {
        const int f_lo = s * seg_len;
        if (f_lo >= whole) break;
        if (f_lo < truth_upto) continue;
        const uint32_t start = trace[f_lo - 1];
        if (start == used_start[s]) continue;
        int32_t h1 = (int32_t)(int16_t)(start & 0xFFFFu), h2 = (int32_t)(int16_t)(start >> 16);
        const int done = run(f_lo, whole, h1, h2, true);
        truth_upto = f_lo + done;
        atomicAdd(&sa.stats[1], (unsigned long long)done);
        atomicAdd(&sa.stats[2], 1ull);
    }
    {   // the partial last frame (and nothing else) from the true pair
        int32_t h1 = 0, h2 = 0;
        if (whole > 0) {
            const uint32_t last = trace[whole - 1];
            h1 = (int32_t)(int16_t)(last & 0xFFFFu);
            h2 = (int32_t)(int16_t)(last >> 16);
        } else if (v4 && c.n_samples > 0) {
            h2 = h1 = src[0];
        }
        adx_encode_general(c, src, dst, whole, h1, h2);
    }
}

__global__ void __launch_bounds__(kAdxThreads)
adx_decode_kernel(const uint8_t *__restrict__ adpcm, const AdxChannel *__restrict__ tab, int n_channels, int32_t *__restrict__ status,
                  int16_t *__restrict__ pcm)
{
    __shared__ __align__(16) uint4 dec_ring[kAdxStages][9][kAdxThreads];  // [stage][16-byte chunk of the group][thread]
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= n_channels) return;
    const AdxChannel c = tab[ch];
    const uint8_t *src = adpcm + c.adpcm_off;
    int16_t *dst = pcm + c.pcm_off;
    const int spf = (c.frame_size - 2) * 2;
    const int sample_count = c.n_samples;
    const int frame_count = div_round_up(sample_count, spf);
    const bool v4 = c.version == 4;
    int32_t hist1 = c.history, hist2 = c.history;  // :16-17
    uint32_t bad_filter = 0;                       // OR of the header bytes of Fixed-type frames
    int current = 0;
    int start_sample = c.padding > 0 ? c.padding % spf : 0;       // :21
    int64_t in = (int64_t)(c.padding / spf) * c.frame_size;      // :22

    int f_first = 0;
    if (c.frame_size == 18 && c.padding == 0) {
        // ---- standard layout: groups of 8 whole frames (144 B = nine 16-byte chunks) through a cp.async ring
        const int groups = sample_count / (32 * kAdxDecGroup);
        const uint4 *vin = reinterpret_cast<const uint4 *>(src);  // adpcm_off is a multiple of 16
        auto issue = [&](int g) {
            if (g < groups) {
#pragma unroll
                for (int j = 0; j < 9; j++) cp_async16(&dec_ring[g % kAdxStages][j][threadIdx.x], vin + (int64_t)g * 9 + j);
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
#pragma unroll
        for (int a = 0; a < kAdxStages - 1; a++) issue(a);
        for (int g = 0; g < groups; g++) {
            issue(g + kAdxStages - 1);
            asm volatile("cp.async.wait_group %0;" ::"n"(kAdxStages - 1) : "memory");
            uint32_t w[36];  // the group's 144 bytes
#pragma unroll
            for (int j = 0; j < 9; j++) {
                const uint4 v = dec_ring[g % kAdxStages][j][threadIdx.x];
                w[4 * j] = v.x; w[4 * j + 1] = v.y; w[4 * j + 2] = v.z; w[4 * j + 3] = v.w;
            }
#pragma unroll
            for (int fr = 0; fr < kAdxDecGroup; fr++) {
                const int base = 18 * fr;  // byte offset of the frame inside the group (even)
                auto byte_at = [&](int k) -> uint32_t { return (w[(base + k) >> 2] >> (((base + k) & 3) * 8)) & 0xFFu; };
                const uint32_t b0 = byte_at(0), b1 = byte_at(1);
                int32_t c0 = c.coef0, c1 = c.coef1;
                if (c.type == 2) {
                    const int k = ((int)((b0 >> 4) & 0xF) >> 1) & 3;
                    bad_filter |= b0;  // bit 7: filter number 4..7
                    c0 = k == 0 ? 0 : (k == 1 ? 0x0F00 : (k == 2 ? 0x1CC0 : 0x1880));
                    c1 = k == 0 ? 0 : (k == 1 ? 0 : (k == 2 ? (int16_t)0xF300 : (int16_t)0xF240));
                }
                int32_t scale = (int16_t)(((b0 << 8) | b1) & 0x1FFF);
                scale = (int16_t)(c.type == 4 ? (1 << ((12 - scale) & 31)) : scale + 1);
                // history kept with a +32768 bias (hb = h + 32768) so that Clamp16 is one VIMNMX.RELU; the bias is folded
                // into per-frame constants (sums wrap like the reference's int32), the multiply-adds are pinned so that
                // only IMAD -> shift(+add) -> clamp sits on the chain
                const int32_t bias0 = wmul(-32768, c0), bias1 = wmul(-32768, c1);
                int32_t hb1 = hist1 + 32768, hb2 = hist2 + 32768;
                uint32_t o[16];
                // the version test is hoisted: two copies of the 32-sample loop instead of predicating both variants
                auto samples = [&](auto is_v4) {
#pragma unroll
                    for (int s2 = 0; s2 < 32; s2++) {
                        const int byte = base + 2 + (s2 >> 1);
                        const int lo_bit = (byte & 3) * 8 + ((s2 & 1) ? 0 : 4);
                        const int32_t q = (int32_t)(w[byte >> 2] << (28 - lo_bit)) >> 28;
                        const int32_t sq = adx_imad(scale, q, 32768);                         // off the chain
                        int32_t biased;                                                        // sample + 32768
                        if (decltype(is_v4)::value) {
                            const int32_t t = adx_imad(c1, hb2, wadd(bias0, bias1));          // off the chain
                            biased = wadd(adx_imad(c0, hb1, t) >> 12, sq);
                        } else {
                            const int32_t t = wadd(adx_imad(c1, hb2, bias1) >> 12, sq);       // off the chain
                            biased = wadd(adx_imad(c0, hb1, bias0) >> 12, t);
                        }
                        const int32_t ob = __viaddmin_s32_relu(biased, 0, 65535);              // clamp16(sample) + 32768
                        hb2 = hb1;
                        hb1 = ob;
                        if (s2 & 1) o[s2 >> 1] |= (uint32_t)ob << 16; else o[s2 >> 1] = (uint32_t)ob;
                    }
                };
                if (v4) samples(std::true_type{}); else samples(std::false_type{});
#pragma unroll
                for (int j = 0; j < 16; j++) o[j] ^= 0x80008000u;
                hist1 = hb1 - 32768;
                hist2 = hb2 - 32768;

                uint4 *vout = reinterpret_cast<uint4 *>(dst + ((int64_t)g * kAdxDecGroup + fr) * 32);  // pcm_off % 8 == 0
#pragma unroll
                for (int j = 0; j < 4; j++) vout[j] = make_uint4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
            }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        f_first = groups * kAdxDecGroup;
        current = f_first * 32;
        in = (int64_t)f_first * 18;
    }

    for (int f = f_first; f < frame_count; f++) {
        const uint32_t b0 = src[in], b1 = src[in + 1];
        const int filter_num = (int)((b0 >> 4) & 0xF) >> 1;  // :26
        int32_t c0 = c.coef0, c1 = c.coef1;
        if (c.type == 2) {  // CriAdxCodec.Coefs (:186-191); the reference throws for filter numbers 4..7
            const int k = filter_num & 3;
            bad_filter |= b0;
            c0 = k == 0 ? 0 : (k == 1 ? 0x0F00 : (k == 2 ? 0x1CC0 : 0x1880));
            c1 = k == 0 ? 0 : (k == 1 ? 0 : (k == 2 ? (int16_t)0xF300 : (int16_t)0xF240));
        }
        int32_t scale = (int16_t)(((b0 << 8) | b1) & 0x1FFF);                         // :27
        scale = (int16_t)(c.type == 4 ? (1 << ((12 - scale) & 31)) : scale + 1);      // :28 (C# masks the shift count)
        in += 2 + start_sample / 2;
        const int to_read = min(spf, sample_count - current);
        for (int s = start_sample; s < to_read; s++) {
            const uint32_t byte = src[in];
            int32_t sample = (s & 1) == 0 ? ((int32_t)(byte << 24) >> 28) : ((int32_t)(byte << 28) >> 28);
            if (s & 1) in++;
            if (v4) sample = wadd(wmul(scale, sample), wadd(wmul(hist1, c0), wmul(hist2, c1)) >> 12);
            else sample = wadd(wadd(wmul(scale, sample), wmul(hist1, c0) >> 12), wmul(hist2, c1) >> 12);
            const int32_t out = clamp16(sample);
            hist2 = hist1;
            hist1 = out;
            dst[current++] = (int16_t)out;
        }
        start_sample = 0;
    }
    // CriAdxCodec.Coefs[filterNum] (:186-191) has four rows: the reference throws IndexOutOfRangeException for 4..7
    if ((bad_filter & 0x80u) && status) atomicMin(status, ch);
    // `new short[sampleCount]` is zero-initialised: samples the padding logic never produces stay 0 (:14,:31-33)
    for (; current < sample_count; current++) dst[current] = 0;
}

// ---------------------------------------------------------------------------------------------------------
// TIME-PARALLEL DECODING.  adx_decode_kernel runs one thread through a whole channel: right for many-channel batches,
// ~100x too serial for one long stereo track.  The decoder is a state machine on (hist1, hist2), so the encoder's three
// phases carry over with the frame-end pair as the only thing compared (AdxDecGeom names the frames):
//   kAdxChain    thread = (channel, segment) over body frames: segment 0 decodes the head frame from the channel's history
//                and runs on, the others start from (0, 0); output and every body frame's end pair (`trace`) are written
//   kAdxRunOn    thread = (channel, boundary): from the previous segment's recorded end pair, decode on inside the segment
//                until a frame-end pair equals the recorded one (from there the recorded output IS the true one)
//   kAdxCascade  thread = channel: repairs, in order, every boundary whose start pair changed after its run-on read it
//                (a run-on that never locked: digital silence keeps a wrong nonzero pair fixed under the >> 12), across
//                segment ends if need be, then decodes the tail frame and zero-fills what no frame reaches
// Exact by construction: a matching pair at the same frame means identical output from there on.  18-byte frames of a
// row at a 16-byte aligned address read groups of 8 frames (144 B, 8-frame aligned in the row) through the cp.async ring;
// the head, unaligned leftovers, other frame sizes and the tail take the per-byte loop, which reads only the bytes
// CriAdxCodec.Decode reads.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void adx_fixed_coefs(uint32_t b0, int32_t &c0, int32_t &c1)  // CriAdxCodec.Coefs (:186-191)
{
    const int k = ((int)((b0 >> 4) & 0xF) >> 1) & 3;
    c0 = k == 0 ? 0 : (k == 1 ? 0x0F00 : (k == 2 ? 0x1CC0 : 0x1880));
    c1 = k == 0 ? 0 : (k == 1 ? 0 : (k == 2 ? (int16_t)0xF300 : (int16_t)0xF240));
}

// The filter number of a frame header (:26) indexes CriAdxCodec.Coefs, four rows, for the Fixed type and a one-row table
// of the computed pair for every other type: status bit 0 for a Fixed filter 4..7, bit 1 for another type's filter 1..7
// (both IndexOutOfRangeException in the reference)
__device__ __forceinline__ uint32_t adx_filter_fault(uint32_t b0, int type)
{
    return type == 2 ? (b0 >> 7) & 1u : ((b0 & 0xE0u) ? 2u : 0u);
}

// One frame by the reference's loop (:24-51): header at byte fb of src, samples s in [start, to_read) to dst[0..).  A frame
// that yields no sample never indexes the coefficient table, so its filter number is not checked.
__device__ __forceinline__ void adx_dec_frame_general(const AdxDecChannel &c, const uint8_t *__restrict__ src, int64_t fb, int start,
                                                      int to_read, int16_t *__restrict__ dst, int32_t &hist1, int32_t &hist2,
                                                      uint32_t &bad_filter)
{
    const uint32_t b0 = src[fb], b1 = src[fb + 1];
    int32_t c0 = c.coef0, c1 = c.coef1;
    if (c.type == 2) adx_fixed_coefs(b0, c0, c1);
    if (to_read > start) bad_filter |= adx_filter_fault(b0, c.type);  // coefs[filterNum] is indexed in the sample loop only
    int32_t scale = (int16_t)(((b0 << 8) | b1) & 0x1FFF);
    scale = (int16_t)(c.type == 4 ? (1 << ((12 - scale) & 31)) : scale + 1);
    const bool v4 = c.version == 4;
    for (int s = start; s < to_read; s++) {
        const uint32_t byte = src[fb + 2 + s / 2];
        int32_t sample = (s & 1) == 0 ? ((int32_t)(byte << 24) >> 28) : ((int32_t)(byte << 28) >> 28);
        if (v4) sample = wadd(wmul(scale, sample), wadd(wmul(hist1, c0), wmul(hist2, c1)) >> 12);
        else sample = wadd(wadd(wmul(scale, sample), wmul(hist1, c0) >> 12), wmul(hist2, c1) >> 12);
        const int32_t out = clamp16(sample);
        hist2 = hist1;
        hist1 = out;
        dst[s - start] = (int16_t)out;
    }
}

// One 18-byte frame at byte `base` of an 8-frame group w[] (the arithmetic of adx_decode_kernel's fast path); o[]
// receives the 32 samples as halfword pairs.
template <bool kV4>
__device__ __forceinline__ void adx_dec_frame_std(const uint32_t (&w)[36], int base, int32_t coef0, int32_t coef1, int type,
                                                  int32_t &hist1, int32_t &hist2, uint32_t &bad_filter, uint32_t (&o)[16])
{
    auto byte_at = [&](int k) -> uint32_t { return (w[(base + k) >> 2] >> (((base + k) & 3) * 8)) & 0xFFu; };
    const uint32_t b0 = byte_at(0), b1 = byte_at(1);
    int32_t c0 = coef0, c1 = coef1;
    if (type == 2) adx_fixed_coefs(b0, c0, c1);
    bad_filter |= adx_filter_fault(b0, type);
    int32_t scale = (int16_t)(((b0 << 8) | b1) & 0x1FFF);
    scale = (int16_t)(type == 4 ? (1 << ((12 - scale) & 31)) : scale + 1);
    const int32_t bias0 = wmul(-32768, c0), bias1 = wmul(-32768, c1);  // history biased by +32768: Clamp16 is one VIMNMX
    int32_t hb1 = hist1 + 32768, hb2 = hist2 + 32768;
#pragma unroll
    for (int s2 = 0; s2 < 32; s2++) {
        const int byte = base + 2 + (s2 >> 1);
        const int lo_bit = (byte & 3) * 8 + ((s2 & 1) ? 0 : 4);
        const int32_t q = (int32_t)(w[byte >> 2] << (28 - lo_bit)) >> 28;
        const int32_t sq = adx_imad(scale, q, 32768);
        int32_t biased;
        if (kV4) {
            const int32_t t = adx_imad(c1, hb2, wadd(bias0, bias1));
            biased = wadd(adx_imad(c0, hb1, t) >> 12, sq);
        } else {
            const int32_t t = wadd(adx_imad(c1, hb2, bias1) >> 12, sq);
            biased = wadd(adx_imad(c0, hb1, bias0) >> 12, t);
        }
        const int32_t ob = __viaddmin_s32_relu(biased, 0, 65535);
        hb2 = hb1;
        hb1 = ob;
        if (s2 & 1) o[s2 >> 1] |= (uint32_t)ob << 16; else o[s2 >> 1] = (uint32_t)ob;
    }
#pragma unroll
    for (int j = 0; j < 16; j++) o[j] ^= 0x80008000u;
    hist1 = hb1 - 32768;
    hist2 = hb2 - 32768;
}

__host__ __device__ __forceinline__ int adx_dec_seg_len(int body, int seg_count, int min_seg)
{
    const int per = (body + seg_count - 1) / seg_count;
    return ((per > min_seg ? per : min_seg) + 7) & ~7;  // a multiple of 8: interior boundaries fall on 8-frame groups
}

template <int kMode>
__global__ void __launch_bounds__(kAdxThreads)
adx_decode_seg_kernel(const uint8_t *__restrict__ adpcm, const AdxDecChannel *__restrict__ tab, int n_channels, int16_t *__restrict__ pcm,
                      AdxDecSegArgs sa)
{
    __shared__ __align__(16) uint4 ring[kAdxStages][9][kAdxThreads];  // [stage][16-byte chunk of the group][thread]
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= n_channels) return;
    const AdxDecChannel c = tab[ch];
    const uint8_t *src = adpcm + c.adpcm_off;
    int16_t *dst = pcm + c.pcm_off;
    const AdxDecGeom g = adx_dec_geom(c.n_samples, c.frame_size, c.padding);
    const int seg_len = adx_dec_seg_len(g.body, sa.seg_count, sa.min_seg_frames);
    const int a1 = (int)(g.in0 / c.frame_size) + 1;  // row frame of body frame 0
    // boundary s >= 1 sits at body frame s * seg_len - (a1 & 7): a multiple of 8 in the row; the last segment runs to the end
    auto seg_lo = [&](int s) { return s == 0 ? 0 : (s >= sa.seg_count ? g.body : min(g.body, s * seg_len - (a1 & 7))); };
    // both paths are chosen from absolute addresses: the caller's base pointers need not be aligned beyond their type
    const bool fast = c.frame_size == 18 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
    const int64_t out_pos = (int64_t)c.pcm_off + g.k0;  // body frame j writes samples out_pos + 32 j..
    const uintptr_t out_addr = reinterpret_cast<uintptr_t>(pcm + out_pos);  // + 64 j keeps its alignment
    const int store = (out_addr & 15) == 0 ? 16 : ((out_addr & 3) == 0 ? 4 : 2);  // widest store the output's alignment allows
    uint32_t *trace = sa.trace + c.trace_off;
    uint32_t bad_filter = 0;

    // body frames [lo, hi) from (h1, h2); splice: stop after the first frame whose end pair equals the recorded one.
    // Returns the number of frames decoded.
    auto run = [&](int lo, int hi, int32_t &h1, int32_t &h2, bool splice) -> int {
        int j = lo, done = 0;
        auto finish = [&](int jj) -> bool {  // frame jj decoded: record its pair or stop at the recorded one
            const uint32_t pair = ((uint32_t)h1 & 0xFFFFu) | ((uint32_t)h2 << 16);
            done++;
            if (splice && trace[jj] == pair) return true;
            trace[jj] = pair;
            return false;
        };
        auto general = [&](int jj) -> bool {
            adx_dec_frame_general(c, src, g.in0 + (int64_t)(1 + jj) * c.frame_size, 0, g.spf, dst + g.k0 + (int64_t)jj * g.spf, h1, h2, bad_filter);
            return finish(jj);
        };
        if (fast) {
            const int jg = min(hi, lo + ((8 - ((a1 + lo) & 7)) & 7));  // first body frame at a multiple of 8 in the row
            for (; j < jg; j++) if (general(j)) return done;
            const int groups = (hi - j) / kAdxDecGroup;
            const uint4 *vin = reinterpret_cast<const uint4 *>(src + (int64_t)(a1 + j) * 18);
            auto issue = [&](int q) {
                if (q < groups) {
#pragma unroll
                    for (int k = 0; k < 9; k++) cp_async16(&ring[q % kAdxStages][k][threadIdx.x], vin + (int64_t)q * 9 + k);
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
            };
#pragma unroll
            for (int q = 0; q < kAdxStages - 1; q++) issue(q);
            bool stop = false;
            for (int q = 0; q < groups && !stop; q++) {
                issue(q + kAdxStages - 1);
                asm volatile("cp.async.wait_group %0;" ::"n"(kAdxStages - 1) : "memory");
                uint32_t w[36];
#pragma unroll
                for (int k = 0; k < 9; k++) {
                    const uint4 v = ring[q % kAdxStages][k][threadIdx.x];
                    w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
                }
#pragma unroll
                for (int fr = 0; fr < kAdxDecGroup; fr++) {
                    uint32_t o[16];
                    if (c.version == 4) adx_dec_frame_std<true>(w, 18 * fr, c.coef0, c.coef1, c.type, h1, h2, bad_filter, o);
                    else adx_dec_frame_std<false>(w, 18 * fr, c.coef0, c.coef1, c.type, h1, h2, bad_filter, o);
                    const int64_t at = out_pos + (int64_t)(j + fr) * 32;
                    if (store == 16) {
                        uint4 *v = reinterpret_cast<uint4 *>(pcm + at);
#pragma unroll
                        for (int k = 0; k < 4; k++) v[k] = make_uint4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
                    } else if (store == 4) {
                        uint32_t *v = reinterpret_cast<uint32_t *>(pcm + at);
#pragma unroll
                        for (int k = 0; k < 16; k++) v[k] = o[k];
                    } else {
#pragma unroll
                        for (int k = 0; k < 16; k++) { pcm[at + 2 * k] = (int16_t)(o[k] & 0xFFFFu); pcm[at + 2 * k + 1] = (int16_t)(o[k] >> 16); }
                    }
                    if (finish(j + fr)) { stop = true; break; }
                }
                j += kAdxDecGroup;
            }
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            if (stop) return done;
        }
        for (; j < hi; j++) if (general(j)) return done;
        return done;
    };
    // the tail frame from the true pair after the last body frame, then zeros where no frame reaches (:14,:31-33)
    auto tail = [&](int32_t h1, int32_t h2) {
        int64_t produced = g.k0 + (int64_t)g.body * g.spf;
        if (g.frames > 1 + g.body) {
            const int to_read = min(g.spf, c.n_samples - (int)produced);
            adx_dec_frame_general(c, src, g.in0 + (int64_t)(1 + g.body) * c.frame_size, 0, to_read, dst + produced, h1, h2, bad_filter);
            produced += max(to_read, 0);
        }
        for (int64_t s = produced; s < c.n_samples; s++) dst[s] = 0;
    };
    auto report = [&]() { if (bad_filter) atomicOr(&sa.status[ch], (int)bad_filter); };

    if (kMode == kAdxChain) {
        const int s = blockIdx.y;
        const int lo = seg_lo(s), hi = seg_lo(s + 1);
        if (s > 0 && lo >= hi) return;
        int32_t h1 = 0, h2 = 0;  // a guess, for every segment but the first
        if (s == 0) {
            h1 = h2 = c.history;
            if (g.frames > 0) adx_dec_frame_general(c, src, g.in0, g.start, min(g.spf, c.n_samples), dst, h1, h2, bad_filter);
        }
        run(lo, hi, h1, h2, false);
        if (s == 0 && (sa.seg_count == 1 || g.body == 0)) tail(h1, h2);  // else the cascade decodes the tail from the true pair
        report();
        return;
    }
    if (kMode == kAdxRunOn) {
        const int s = blockIdx.y + 1;
        const int lo = seg_lo(s), hi = seg_lo(s + 1);
        if (lo >= hi) return;
        const uint32_t start = trace[lo - 1];
        sa.used_start[(int64_t)ch * kAdxDecMaxSegments + s] = start;
        int32_t h1 = (int32_t)(int16_t)(start & 0xFFFFu), h2 = (int32_t)(int16_t)(start >> 16);
        const int done = run(lo, hi, h1, h2, true);
        atomicAdd(&sa.stats[0], (unsigned long long)done);
        atomicMax(&sa.stats[3], (unsigned long long)done);
        return;
    }
    // cascade: one thread per channel walks the boundaries in order
    int truth_upto = 0;
    for (int s = 1; s < sa.seg_count; s++) {
        const int lo = seg_lo(s);
        if (lo >= g.body) break;
        if (lo < truth_upto) continue;
        const uint32_t start = trace[lo - 1];
        if (start == sa.used_start[(int64_t)ch * kAdxDecMaxSegments + s]) continue;
        int32_t h1 = (int32_t)(int16_t)(start & 0xFFFFu), h2 = (int32_t)(int16_t)(start >> 16);
        const int done = run(lo, g.body, h1, h2, true);
        truth_upto = lo + done;
        atomicAdd(&sa.stats[1], (unsigned long long)done);
        atomicAdd(&sa.stats[2], 1ull);
    }
    if (g.body == 0) return;  // segment 0's chain decoded the whole channel
    const uint32_t last = trace[g.body - 1];
    tail((int32_t)(int16_t)(last & 0xFFFFu), (int32_t)(int16_t)(last >> 16));
    report();
}

// Segments per channel of the time-parallel ADX decode: about four waves of threads over the SMs, no segment shorter
// than the minimum (VGB_ADX_DEC_SEGMENTS / VGB_ADX_DEC_MIN_SEG_FRAMES override both).
int adx_decode_pick_segments(int n_channels, int max_body_frames, int *min_seg_out)
{
    int min_seg = kAdxDecMinSegFrames;
    if (const char *env = std::getenv("VGB_ADX_DEC_MIN_SEG_FRAMES")) {
        const int v = std::atoi(env);
        if (v >= 1) min_seg = v;
    }
    if (min_seg_out) *min_seg_out = min_seg;
    if (const char *env = std::getenv("VGB_ADX_DEC_SEGMENTS")) {
        const int v = std::atoi(env);
        if (v >= 1) return std::min(v, kAdxDecMaxSegments);
    }
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) {
        (void)cudaGetLastError();
        sms = 132;  // H100 SXM
    }
    const long long want = (4ll * sms * 512 + n_channels - 1) / std::max(n_channels, 1);
    const int max_s = std::max(1, std::min(kAdxDecMaxSegments, max_body_frames / min_seg));
    return (int)std::max<long long>(1, std::min<long long>(want, max_s));
}

void launch_adx_decode_seg(const uint8_t *adpcm, const AdxDecChannel *tab, int n_channels, int16_t *pcm, AdxDecSegArgs sa, cudaStream_t stream)
{
    if (n_channels <= 0) return;
    const int blocks = (n_channels + kAdxThreads - 1) / kAdxThreads;
    adx_decode_seg_kernel<kAdxChain><<<dim3(blocks, sa.seg_count), kAdxThreads, 0, stream>>>(adpcm, tab, n_channels, pcm, sa);
    if (sa.seg_count > 1) {
        adx_decode_seg_kernel<kAdxRunOn><<<dim3(blocks, sa.seg_count - 1), kAdxThreads, 0, stream>>>(adpcm, tab, n_channels, pcm, sa);
        adx_decode_seg_kernel<kAdxCascade><<<dim3(blocks, 1), kAdxThreads, 0, stream>>>(adpcm, tab, n_channels, pcm, sa);
    }
}

// Segments per channel of the time-parallel ADX encode: thread-per-item kernels want every SM full of threads
// (~512 resident per SM at this register count), the run-on at a boundary is a handful of frames.
// Shortest segment in frames.  Measured with the oracle on the synthetic set: a chain started from raw history meets the
// true one after 100-600 frames as a rule (quantisation step = maxDistance / 7 is hundreds of LSB on loud material, so the
// two reconstructions rarely coincide twice in a row), hence segments of at least 4096 frames; tests lower it.
int adx_min_segment_frames()
{
    if (const char *env = std::getenv("VGB_ADX_MIN_SEG_FRAMES")) {
        const int v = std::atoi(env);
        if (v >= 1) return v;
    }
    return kAdxMinSegFrames;
}

int adx_encode_pick_segments(int n_channels, int max_whole_frames, int *min_seg_out)
{
    int min_seg = adx_min_segment_frames();
    if (min_seg_out) *min_seg_out = min_seg;
    if (const char *env = std::getenv("VGB_ADX_SEGMENTS")) {
        const int v = std::atoi(env);
        if (v >= 1) return v > kAdxMaxSegments ? kAdxMaxSegments : v;
    }
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) {
            (void)cudaGetLastError();
            sms = 132;  // H100 SXM
        }
    }
    const long long want = (4ll * sms * 512 + n_channels - 1) / std::max(n_channels, 1);  // about four waves of threads
    // a batch that cannot fill the machine with kAdxMinSegFrames-long segments is latency bound: quarter the minimum (the
    // fixed predictor's run-on is some hundred frames, so short segments stay cheap; the batch converter's files of 1-6 s
    // are this case)
    if (!std::getenv("VGB_ADX_MIN_SEG_FRAMES") && max_whole_frames / min_seg < want) min_seg = std::max(64, min_seg / 4);
    if (min_seg_out) *min_seg_out = min_seg;
    const int max_s = std::max(1, std::min(kAdxMaxSegments, max_whole_frames / min_seg));
    return (int)std::max<long long>(1, std::min<long long>(want, max_s));
}

void launch_adx_encode(const int16_t *pcm, const AdxChannel *tab, int n_channels, uint8_t *adpcm, int16_t *history_out,
                       AdxSegArgs sa, cudaStream_t stream)
{
    if (n_channels <= 0) return;
    if (sa.seg_count < 1 || !sa.trace) sa.seg_count = 1;
    if (sa.seg_count > kAdxMaxSegments) sa.seg_count = kAdxMaxSegments;
    if (sa.min_seg_frames <= 0) sa.min_seg_frames = adx_min_segment_frames();  // else: chosen by adx_encode_pick_segments
    const int blocks = (n_channels + kAdxThreads - 1) / kAdxThreads;
    if (sa.stats) cudaMemsetAsync(sa.stats, 0, 4 * sizeof(unsigned long long), stream);
    adx_encode_kernel<kAdxChain><<<dim3(blocks, sa.seg_count), kAdxThreads, 0, stream>>>(pcm, tab, n_channels, adpcm, history_out, sa);
    if (sa.seg_count > 1) {
        adx_encode_kernel<kAdxRunOn><<<dim3(blocks, sa.seg_count - 1), kAdxThreads, 0, stream>>>(pcm, tab, n_channels, adpcm, history_out, sa);
        adx_encode_kernel<kAdxCascade><<<dim3(blocks, 1), kAdxThreads, 0, stream>>>(pcm, tab, n_channels, adpcm, history_out, sa);
    }
}

void launch_adx_decode(const uint8_t *adpcm, const AdxChannel *tab, int n_channels, int16_t *pcm, int32_t *status, cudaStream_t stream)
{
    if (n_channels <= 0) return;
    adx_decode_kernel<<<(n_channels + kAdxThreads - 1) / kAdxThreads, kAdxThreads, 0, stream>>>(adpcm, tab, n_channels, status, pcm);
}

}  // namespace vgb
