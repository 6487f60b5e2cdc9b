// gc_decode.cu — GC-ADPCM decoder on sm_90a (H100).
//
// Replaces GcAdpcmDecoder.Decode (Codecs/GcAdpcm/GcAdpcmDecoder.cs:10-54).  The recurrence
//     s[t] = Clamp16((c1*s[t-1] + c2*s[t-2] + scale*nibble + 1024) >> 11)
// is non-linear (the clamp), so a channel is strictly serial; parallelism is across channels: one THREAD owns one
// channel and streams it privately — no shared-memory transpose:
//   in    groups of 4 frames = 32 B = two 16-byte cp.async copies per thread into the thread's own shared-memory ring,
//         issued three groups (~3500 cycles of decode work) ahead so DRAM latency never reaches the recurrence; the
//         32-byte sector a thread touches is its own, so HBM moves every ADPCM byte exactly once;
//   out   4 frames = 56 samples = 112 B = seven 16-byte stores per thread straight from registers (fire and forget;
//         the two halves of a 32-byte sector are merged in L2 before they reach DRAM).
// Per sample the dependent chain is IMAD -> SHF -> VIADDMNMX.RELU (~13.5 cycles): history is kept with a +32768 bias so
// that Clamp16 is one instruction, the bias and the rounding constant are folded into a per-frame constant, and the
// older-sample product, nibble extraction and scale multiply sit off the chain.  All sums are wrapping int32 like the
// reference (A.7); folding constants is exact in the ring.
// Bound: chain latency at <= 1 warp per SM sub-partition (8192 channels = 256 warps), HBM (2.57 B/sample) above that.
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace vgb {

constexpr int kDecThreads = 32;      // one warp per CTA: 8192 channels -> 256 CTAs spread over all SMs
constexpr int kDecGroupFrames = 4;   // 32 B in, 112 B out per thread
constexpr int kDecAhead = 4;         // ring stages (kDecAhead - 1 groups in flight)

namespace {

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src)
{
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}

// a*b + c as ONE multiply-add the compiler may not re-associate (it otherwise moves the nibble term onto the chain)
__device__ __forceinline__ int32_t dec_imad(int32_t a, int32_t b, int32_t c)
{
    int32_t d;
    asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

struct DecState {
    int32_t hb1, hb2;  // biased history (+32768): newest, older
    uint32_t heads;    // OR of the frame headers seen: bit 7 set = some frame selected a predictor 8..15
};

// 14 samples of one frame (8 bytes in w0,w1; byte 0 = header).  out[0..6] = the 14 samples, two per word.
__device__ __forceinline__ void gc_decode_frame(uint32_t w0, uint32_t w1, const uint32_t *coef_pairs, DecState &st, uint32_t *out)
{
    const uint32_t head = w0 & 0xFFu;
    st.heads |= w0;
    const int sp = (int)(head & 0xFu);  // scale = (1 << sp) * 2048 (GcAdpcmDecoder.cs:28)
    // a hostile header may select pairs 8..15: the reference throws IndexOutOfRangeException; the lookup wraps to stay
    // in bounds and the channel is reported through tab.status (the batch call then returns VGB_E_DATA)
    const uint32_t pair = coef_pairs[(head >> 4) & 7u];
    const int32_t c1 = (int32_t)(int16_t)(pair & 0xFFFFu), c2 = (int32_t)pair >> 16;
    int32_t k = wsub(1024, wmul(32768, wadd(c1, c2)));  // rounding constant minus the bias of both histories
    asm("" : "+r"(k));                                    // one register, not a multiply re-derived for every sample
    const int32_t scale = (int32_t)((1u << sp) * 2048u);
    int32_t hb1 = st.hb1, hb2 = st.hb2;
#pragma unroll
    for (int s = 0; s < 14; s++) {
        const int byte = 1 + s / 2;
        const uint32_t word = byte < 4 ? w0 : w1;
        const int lo_bit = (byte & 3) * 8 + ((s & 1) ? 0 : 4);                 // position of the nibble's lowest bit
        const int32_t q = (int32_t)(word << (28 - lo_bit)) >> 28;              // Helpers.GetHighNibbleSigned/Low (:50-56)
        const int32_t t = dec_imad(c2, hb2, dec_imad(q, scale, k));            // off the chain
        const int32_t v = dec_imad(c1, hb1, t);                                // chain: IMAD
        const int32_t ob = __viaddmin_s32_relu(v >> 11, 32768, 65535);         // chain: shift+bias, clamp
        hb2 = hb1;
        hb1 = ob;
        if (s & 1) out[s / 2] |= (uint32_t)ob << 16; else out[s / 2] = (uint32_t)ob;
    }
#pragma unroll
    for (int j = 0; j < 7; j++) out[j] ^= 0x80008000u;  // remove the bias from both halves
    st.hb1 = hb1;
    st.hb2 = hb2;
}

}  // namespace

// kTaps == false: the decoder proper, every sample goes to `pcm`.
// kTaps == true : the post-encode channel rebuild of the format layer (GcAdpcmChannelBuilder.GetSeekTable /
//                 GetLoopContext, Formats/GcAdpcm/GcAdpcmChannelBuilder.cs:176-202): the reference decodes the whole
//                 channel again only to read pcm[i*spe - 1], pcm[i*spe - 2] (GcAdpcmSeekTable.cs:25-38) and
//                 pcm[loopStart - 1], pcm[loopStart - 2] (GcAdpcmLoopContext.cs:24-26); here the same decode keeps
//                 just those samples.  `pcm` is then the tap slab: per channel [entries*2 seek shorts][hist1][hist2].
template <bool kTaps>
__global__ void __launch_bounds__(kDecThreads)
gc_decode_kernel(const uint8_t *__restrict__ adpcm, GcChannelTable tab, const int16_t *__restrict__ coefs,
                 int16_t *__restrict__ pcm, int frame_begin, int frame_end, const GcTapChannel *__restrict__ taps)
{
    __shared__ uint32_t coef_smem[kDecThreads][9];  // 8 (c1 | c2 << 16) pairs per channel, odd pitch: conflict free
    __shared__ __align__(16) uint4 ring_smem[kDecAhead][2][kDecThreads];  // [stage][half of the 32 bytes][thread]
    const int ch = blockIdx.x * kDecThreads + threadIdx.x;
    if (ch >= tab.n_channels) return;

    const int n = tab.n_samples[ch];
    const int n_frames = div_round_up(n, kGcFrameSamples);
    const int f_hi = min(frame_end, n_frames);
    if (frame_begin >= f_hi) return;
    const uint8_t *src = adpcm + tab.adpcm_off[ch];
    int16_t *dst = pcm + (kTaps ? taps[ch].out_off : tab.pcm_off[ch]);
    const int spe = kTaps ? taps[ch].samples_per_entry : 1;  // (1: keeps the dead divisions of the decoder proper defined)
    const int loop_start = kTaps ? taps[ch].loop_start : -1;
    const int entries = (kTaps && spe > 0) ? div_round_up(n, spe) : 0;
    // taps mode: keep the samples of the run [p0, p0 + cnt) (two per word in o[]) that the seek table / loop context want
    auto keep_taps = [&](int64_t p0, int cnt, const uint32_t (&o)[28]) {
        auto sample_at = [&](int idx) -> int16_t {  // o[] lives in registers: select instead of indexing
            uint32_t w = 0;
#pragma unroll
            for (int j = 0; j < 28; j++) w = (j == (idx >> 1) && j * 2 < cnt + 1) ? o[j] : w;
            return (int16_t)((w >> ((idx & 1) * 16)) & 0xFFFFu);
        };
        if (kTaps && spe > 0) {
            // multiples m of spe with a tap in the run: m - 1 or m - 2 in [p0, p0 + cnt)  <=>  p0 + 1 <= m <= p0 + cnt + 1
            int64_t m = (p0 + 1 + spe - 1) / spe * spe;
            if (m == 0) m = spe;  // the first entry is always zero (GcAdpcmSeekTable.cs:31)
            for (; m <= p0 + cnt + 1; m += spe) {
                const int64_t i = m / spe;
                if (i >= entries) break;
                if (m - 1 >= p0 && m - 1 < p0 + cnt) dst[2 * i] = sample_at((int)(m - 1 - p0));
                if (m - 2 >= p0 && m - 2 < p0 + cnt) dst[2 * i + 1] = sample_at((int)(m - 2 - p0));
            }
        }
        if (loop_start >= 1 && loop_start - 1 >= p0 && loop_start - 1 < p0 + cnt) dst[2 * entries] = sample_at((int)(loop_start - 1 - p0));
        if (loop_start >= 2 && loop_start - 2 >= p0 && loop_start - 2 < p0 + cnt) dst[2 * entries + 1] = sample_at((int)(loop_start - 2 - p0));
    };
    uint32_t *pairs = coef_smem[threadIdx.x];
#pragma unroll
    for (int p = 0; p < 8; p++) {
        const uint32_t c1 = (uint16_t)coefs[(int64_t)ch * 16 + 2 * p], c2 = (uint16_t)coefs[(int64_t)ch * 16 + 2 * p + 1];
        pairs[p] = c1 | (c2 << 16);
    }
    DecState st{tab.hist[2 * ch] + 32768, tab.hist[2 * ch + 1] + 32768, 0u};

    // groups of 4 whole frames whose 56 samples all exist go through the vector path
    const int full_frames = min(f_hi, n / kGcFrameSamples);  // frames with all 14 samples
    const int g_lo = frame_begin / kDecGroupFrames;          // frame_begin is a multiple of 16
    const int g_hi = max(full_frames / kDecGroupFrames, g_lo);
    const uint4 *vin = reinterpret_cast<const uint4 *>(src);

    // Ring of kDecAhead groups per thread in shared memory, filled by cp.async (LDGSTS): asynchronous copies have no
    // register scoreboard, so neither a register rotation nor the compiler's habit of sinking loads next to their
    // first use can shorten the prefetch distance.  A thread only ever reads what it copied itself: no barrier.
    auto issue = [&](int g) {
        if (g < g_hi) {
            const uint4 *p = vin + (int64_t)g * 2;
            uint4 *slot = &ring_smem[g % kDecAhead][0][threadIdx.x];
            cp_async16(slot, p);
            cp_async16(slot + kDecThreads, p + 1);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");  // one (possibly empty) group per step keeps the count exact
    };
#pragma unroll
    for (int a = 0; a < kDecAhead - 1; a++) issue(g_lo + a);
    for (int g = g_lo; g < g_hi; g++) {
        issue(g + kDecAhead - 1);
        asm volatile("cp.async.wait_group %0;" ::"n"(kDecAhead - 1) : "memory");  // group g has landed
        const uint4 a = ring_smem[g % kDecAhead][0][threadIdx.x], b = ring_smem[g % kDecAhead][1][threadIdx.x];
        uint32_t o[28];
        gc_decode_frame(a.x, a.y, pairs, st, o);
        gc_decode_frame(a.z, a.w, pairs, st, o + 7);
        gc_decode_frame(b.x, b.y, pairs, st, o + 14);
        gc_decode_frame(b.z, b.w, pairs, st, o + 21);
        if constexpr (kTaps) {
            const int64_t p0 = (int64_t)g * kDecGroupFrames * kGcFrameSamples;
            bool hit = false;  // rare: one run in samples_per_entry / 56 holds a tap
            if (spe > 0) {
                const int64_t m = (p0 + 57) / spe * spe;  // largest multiple of spe <= p0 + 57
                hit = m >= p0 + 1 && m > 0;
            }
            hit = hit || (loop_start >= 1 && loop_start - 2 < p0 + 56 && loop_start - 1 >= p0);
            if (hit) keep_taps(p0, 56, o);
        } else {
            uint4 *vout = reinterpret_cast<uint4 *>(dst + (int64_t)g * kDecGroupFrames * kGcFrameSamples);
#pragma unroll
            for (int j = 0; j < 7; j++) vout[j] = make_uint4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");

    // the rest (< 4 whole frames, and the channel's partial last frame): byte loads, only the samples that exist
    for (int f = max(g_hi * kDecGroupFrames, frame_begin); f < f_hi; f++) {
        const int take = min(kGcFrameSamples, n - f * kGcFrameSamples);
        const int bytes = 1 + (take + 1) / 2;  // header + nibble bytes present (SampleCountToByteCount)
        uint32_t w[2] = {0, 0};  // bytes the stream does not hold decode as zero nibbles; those samples are not written
        for (int j = 0; j < bytes; j++) w[j >> 2] |= (uint32_t)src[(int64_t)f * kGcFrameBytes + j] << ((j & 3) * 8);
        if constexpr (kTaps) {
            uint32_t o[28];
#pragma unroll
            for (int j = 7; j < 28; j++) o[j] = 0;
            gc_decode_frame(w[0], w[1], pairs, st, o);
            keep_taps((int64_t)f * kGcFrameSamples, take, o);
        } else {
            uint32_t o[7];
            gc_decode_frame(w[0], w[1], pairs, st, o);
            int16_t *d = dst + (int64_t)f * kGcFrameSamples;
            for (int s = 0; s < take; s++) d[s] = (int16_t)((o[s >> 1] >> ((s & 1) * 16)) & 0xFFFFu);
        }
    }

    if ((st.heads & 0x80u) && tab.status) atomicMin(tab.status, ch);
    tab.hist[2 * ch] = (int16_t)(st.hb1 - 32768);  // carried into the next time slice of the same call
    tab.hist[2 * ch + 1] = (int16_t)(st.hb2 - 32768);
}

void launch_gc_decode(const uint8_t *adpcm, const GcChannelTable &tab, const int16_t *coefs, int16_t *pcm,
                      int max_frames, int frame_begin, int frame_end, cudaStream_t stream)
{
    if (tab.n_channels <= 0 || max_frames <= 0) return;
    if (frame_begin >= frame_end || frame_begin >= max_frames) return;
    const int blocks = (tab.n_channels + kDecThreads - 1) / kDecThreads;
    gc_decode_kernel<false><<<blocks, kDecThreads, 0, stream>>>(adpcm, tab, coefs, pcm, frame_begin, frame_end, nullptr);
}

void launch_gc_taps(const uint8_t *adpcm, const GcChannelTable &tab, const int16_t *coefs, const GcTapChannel *taps,
                    int16_t *tap_slab, int max_frames, cudaStream_t stream)
{
    if (tab.n_channels <= 0 || max_frames <= 0) return;
    const int blocks = (tab.n_channels + kDecThreads - 1) / kDecThreads;
    gc_decode_kernel<true><<<blocks, kDecThreads, 0, stream>>>(adpcm, tab, coefs, tap_slab, 0, INT32_MAX, taps);
}

// ---------------------------------------------------------------------------------------------------------
// TIME-PARALLEL DECODING.  gc_decode_kernel runs one thread through a whole channel: right for many-channel batches,
// far too serial for a few long stereo streams (a .brstm track lasts minutes).  The decoder is a state machine on
// (hist1, hist2), so the three phases of the ADX decoder (adx.cu) carry over, with the frame-end pair as the only thing
// compared:
//   kGcChain    thread = (channel, segment) over full frames: segment 0 decodes from the channel's start context, the
//               others from (0, 0); output and every full frame's end pair (`trace`) are written
//   kGcRunOn    thread = (channel, boundary): from the previous segment's recorded end pair, decode on inside the segment
//               until a frame-end pair equals the recorded one (from there the recorded output IS the true one)
//   kGcCascade  thread = channel: repairs, in order, every boundary whose start pair changed after its run-on read it
//               (a run-on that never locked: digital silence can hold a wrong pair under the >> 11), across segment
//               ends if need be, then decodes the partial last frame from the true pair
// Exact by construction: a matching pair after the same frame means identical output from there on.  The per-sample
// chain is gc_decode_frame's (biased history, rounding constant and bias folded per frame).  Interior boundaries fall
// on multiples of 4 frames, so every segment reads 32-byte groups through the same cp.async ring as the serial kernel;
// the chain stores whole groups as 16-byte vectors, run-ons and the cascade store frame by frame (they may stop inside
// a group).
// ---------------------------------------------------------------------------------------------------------
constexpr int kSegThreads = 64;
constexpr int kGcChain = 0, kGcRunOn = 1, kGcCascade = 2;

__host__ __device__ __forceinline__ int gc_dec_seg_len(int full, int seg_count, int min_seg)
{
    const int per = (full + seg_count - 1) / seg_count;
    return (int)((((int64_t)(per > min_seg ? per : min_seg)) + 3) & ~(int64_t)3);  // interior boundaries on 4-frame groups
}

template <int kMode>
__global__ void __launch_bounds__(kSegThreads)
gc_decode_seg_kernel(const uint8_t *__restrict__ adpcm, const GcDecChannel *__restrict__ tab, int n_channels,
                     int16_t *__restrict__ pcm, GcDecSegArgs sa)
{
    __shared__ uint32_t coef_smem[kSegThreads][9];
    __shared__ __align__(16) uint4 ring_smem[kDecAhead][2][kSegThreads];
    const int per_ch = kMode == kGcChain ? sa.seg_count : (kMode == kGcRunOn ? sa.seg_count - 1 : 1);
    const int64_t idx = (int64_t)blockIdx.x * kSegThreads + threadIdx.x;
    if (idx >= (int64_t)n_channels * per_ch) return;
    const int ch = (int)(idx % n_channels);
    const int s = (int)(idx / n_channels) + (kMode == kGcRunOn ? 1 : 0);
    const GcDecChannel &c = tab[ch];
    const int n = c.n_samples;
    const int full = n / kGcFrameSamples, frames = div_round_up(n, kGcFrameSamples);
    const int seg_len = gc_dec_seg_len(full, sa.seg_count, sa.min_seg_frames);
    auto seg_lo = [&](int k) -> int {
        return k == 0 ? 0 : (k >= sa.seg_count ? full : (int)min((int64_t)full, (int64_t)k * seg_len));
    };
    const uint8_t *src = adpcm + c.adpcm_off;
    int16_t *dst = pcm + c.pcm_off;
    uint32_t *trace = sa.trace + c.trace_off;
    uint32_t *pairs = coef_smem[threadIdx.x];
#pragma unroll
    for (int p = 0; p < 8; p++) pairs[p] = (uint32_t)(uint16_t)c.coefs[2 * p] | ((uint32_t)(uint16_t)c.coefs[2 * p + 1] << 16);

    // full frames [lo, hi) from st; splice: stop after the first frame whose end pair equals the recorded one.
    // Returns the number of frames decoded.
    auto run = [&](int lo, int hi, DecState &st, bool splice) -> int {
        int done = 0;
        auto finish = [&](int j) -> bool {  // frame j decoded: record its pair or stop at the recorded one
            const uint32_t pair = (uint32_t)st.hb1 | ((uint32_t)st.hb2 << 16);
            done++;
            if (splice && trace[j] == pair) return true;
            trace[j] = pair;
            return false;
        };
        auto store7 = [&](int j, const uint32_t *o) {  // frame j's 14 samples: 4-byte aligned (pcm_off is a multiple of 8)
            uint32_t *d = reinterpret_cast<uint32_t *>(dst + (int64_t)j * kGcFrameSamples);
#pragma unroll
            for (int k = 0; k < 7; k++) d[k] = o[k];
        };
        const int groups = (hi - lo) / kDecGroupFrames;  // lo is a multiple of 4
        const uint4 *vin = reinterpret_cast<const uint4 *>(src + (int64_t)lo * kGcFrameBytes);
        auto issue = [&](int q) {
            if (q < groups) {
                uint4 *slot = &ring_smem[q % kDecAhead][0][threadIdx.x];
                cp_async16(slot, vin + (int64_t)q * 2);
                cp_async16(slot + kSegThreads, vin + (int64_t)q * 2 + 1);
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
#pragma unroll
        for (int a = 0; a < kDecAhead - 1; a++) issue(a);
        bool stop = false;
        for (int q = 0; q < groups && !stop; q++) {
            issue(q + kDecAhead - 1);
            asm volatile("cp.async.wait_group %0;" ::"n"(kDecAhead - 1) : "memory");
            const uint4 a = ring_smem[q % kDecAhead][0][threadIdx.x], b = ring_smem[q % kDecAhead][1][threadIdx.x];
            const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
            const int j0 = lo + q * kDecGroupFrames;
            if (!splice) {
                uint32_t o[28];
#pragma unroll
                for (int fr = 0; fr < kDecGroupFrames; fr++) {
                    gc_decode_frame(w[2 * fr], w[2 * fr + 1], pairs, st, o + 7 * fr);
                    finish(j0 + fr);
                }
                uint4 *vout = reinterpret_cast<uint4 *>(dst + (int64_t)j0 * kGcFrameSamples);
#pragma unroll
                for (int k = 0; k < 7; k++) vout[k] = make_uint4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
            } else {
#pragma unroll
                for (int fr = 0; fr < kDecGroupFrames; fr++) {
                    uint32_t o[7];
                    gc_decode_frame(w[2 * fr], w[2 * fr + 1], pairs, st, o);
                    store7(j0 + fr, o);
                    if (finish(j0 + fr)) { stop = true; break; }
                }
            }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        if (stop) return done;
        for (int j = lo + groups * kDecGroupFrames; j < hi; j++) {  // whole frames short of a group: 8-byte loads
            const uint2 v = *reinterpret_cast<const uint2 *>(src + (int64_t)j * kGcFrameBytes);
            uint32_t o[7];
            gc_decode_frame(v.x, v.y, pairs, st, o);
            store7(j, o);
            if (finish(j) && splice) break;
        }
        return done;
    };
    // the partial last frame from the true pair after the full frames: byte loads, only the samples that exist
    auto tail = [&](DecState &st) {
        if (frames <= full) return;
        const int take = n - full * kGcFrameSamples;
        const int bytes = 1 + (take + 1) / 2;
        uint32_t w[2] = {0, 0};
        for (int j = 0; j < bytes; j++) w[j >> 2] |= (uint32_t)src[(int64_t)full * kGcFrameBytes + j] << ((j & 3) * 8);
        uint32_t o[7];
        gc_decode_frame(w[0], w[1], pairs, st, o);
        int16_t *d = dst + (int64_t)full * kGcFrameSamples;
        for (int k = 0; k < take; k++) d[k] = (int16_t)((o[k >> 1] >> ((k & 1) * 16)) & 0xFFFFu);
    };
    // GcAdpcmDecoder indexes coefficients[predictor * 2] on every frame that yields samples: 8..15 throws there
    auto report = [&](const DecState &st) { if (st.heads & 0x80u) atomicOr(&sa.status[ch], 1); };
    auto from_pair = [](uint32_t pair) { return DecState{(int32_t)(pair & 0xFFFFu), (int32_t)(pair >> 16), 0u}; };

    if (kMode == kGcChain) {
        const int lo = seg_lo(s), hi = seg_lo(s + 1);
        if (s > 0 && lo >= hi) return;
        DecState st = s == 0 ? DecState{c.hist1 + 32768, c.hist2 + 32768, 0u} : DecState{32768, 32768, 0u};  // a guess but for s = 0
        run(lo, hi, st, false);
        if (s == 0 && (sa.seg_count == 1 || full == 0)) tail(st);  // else the cascade decodes it from the true pair
        report(st);
        return;
    }
    if (kMode == kGcRunOn) {
        const int lo = seg_lo(s), hi = seg_lo(s + 1);
        if (lo >= hi) return;
        const uint32_t start = trace[lo - 1];
        sa.used_start[(int64_t)ch * kGcDecMaxSegments + s] = start;
        DecState st = from_pair(start);
        const int done = run(lo, hi, st, true);
        atomicAdd(&sa.stats[0], (unsigned long long)done);
        atomicMax(&sa.stats[3], (unsigned long long)done);
        return;
    }
    // cascade: one thread per channel walks the boundaries in order
    int truth_upto = 0;
    for (int k = 1; k < sa.seg_count; k++) {
        const int lo = seg_lo(k);
        if (lo >= full) break;
        if (lo < truth_upto) continue;
        const uint32_t start = trace[lo - 1];
        if (start == sa.used_start[(int64_t)ch * kGcDecMaxSegments + k]) continue;
        DecState st = from_pair(start);
        const int done = run(lo, full, st, true);
        truth_upto = lo + done;
        atomicAdd(&sa.stats[1], (unsigned long long)done);
        atomicAdd(&sa.stats[2], 1ull);
    }
    if (full == 0) return;  // segment 0's chain decoded the whole channel
    DecState st = from_pair(trace[full - 1]);
    tail(st);
    report(st);
}

// Segments per channel of the time-parallel decode: about four waves of threads over the SMs, no segment shorter than
// the minimum, at most kGcDecMaxSegments (VGB_GC_DEC_SEGMENTS / VGB_GC_DEC_MIN_SEG_FRAMES override both, read per call).
int gc_decode_pick_segments(int n_channels, int max_full_frames, int *min_seg_out)
{
    int min_seg = kGcDecMinSegFrames;
    if (const char *env = std::getenv("VGB_GC_DEC_MIN_SEG_FRAMES")) {
        const int v = std::atoi(env);
        if (v >= 1) min_seg = v;
    }
    if (min_seg_out) *min_seg_out = min_seg;
    if (const char *env = std::getenv("VGB_GC_DEC_SEGMENTS")) {
        const int v = std::atoi(env);
        if (v >= 1) return std::min(v, kGcDecMaxSegments);
    }
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) {
        (void)cudaGetLastError();
        sms = 132;  // H100 SXM
    }
    const long long want = (4ll * sms * 512 + n_channels - 1) / std::max(n_channels, 1);
    const int max_s = std::max(1, std::min(kGcDecMaxSegments, max_full_frames / min_seg));
    return (int)std::max<long long>(1, std::min<long long>(want, max_s));
}

void launch_gc_decode_seg(const uint8_t *adpcm, const GcDecChannel *tab, int n_channels, int16_t *pcm, GcDecSegArgs sa,
                          cudaStream_t stream)
{
    if (n_channels <= 0) return;
    auto blocks = [&](int per_ch) { return (unsigned)(((int64_t)n_channels * per_ch + kSegThreads - 1) / kSegThreads); };
    gc_decode_seg_kernel<kGcChain><<<blocks(sa.seg_count), kSegThreads, 0, stream>>>(adpcm, tab, n_channels, pcm, sa);
    if (sa.seg_count > 1) {
        gc_decode_seg_kernel<kGcRunOn><<<blocks(sa.seg_count - 1), kSegThreads, 0, stream>>>(adpcm, tab, n_channels, pcm, sa);
        gc_decode_seg_kernel<kGcCascade><<<blocks(1), kSegThreads, 0, stream>>>(adpcm, tab, n_channels, pcm, sa);
    }
}

}  // namespace vgb
