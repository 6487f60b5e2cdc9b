// gc_encode.cu — GC-ADPCM encoder on sm_90a (H100).
//
// Replaces GcAdpcmEncoder.Encode / DspEncodeFrame / DspEncodeCoef (Codecs/GcAdpcm/GcAdpcmEncoder.cs:14-171).
//
// Dependence structure of the reference: frames of one channel are strictly serial (frame k+1 starts from the
// RECONSTRUCTED last two samples of frame k, :40-41,:80), channels are independent, and inside a frame the eight
// predictors are independent while the scale attempts of one predictor form a short chain (:127-170).
//
// Mapping: ONE QUARTER-WARP OWNS ONE CHANNEL (four channels per warp).  Lane & 7 = predictor: the 8 predictors are
// searched in parallel and each lane evaluates 2 consecutive scale powers of its predictor speculatively, as two
// interleaved recurrences (every attempt is a pure function of (samples, history, coefs, scalePower), so the do/while
// chain can be replayed over finished attempts inside the lane; a second round covers one more power; the rare
// overflow "bump" (:166-168) falls back to the literal loop).  The argmin over predictors (strict <, first wins,
// :66-76) is an 8-lane butterfly MIN on an exact integer key; the winner's two newest reconstructed samples are
// broadcast with one SHFL.  PCM is staged through shared memory 16 frames at a time with coalesced 16-byte loads
// (prefetched one chunk ahead), ADPCM bytes are staged and written back 128 bytes at a time.  The per-frame work that
// is paid once per warp (head keys, votes, argmin, broadcast, bookkeeping) is shared by four channels.
//
// Cut into segments (below) the kernel runs several warps per SM sub-partition and is instruction-issue bound; a
// lone warp would be latency bound by the dependent instruction chain of a frame, so that chain is kept short
// (DESIGN.md §gc_encode):
//   * the quantiser's int->float32->float64->int cast chain (:142-144) is replaced by an exactly equivalent
//     integer expression (proved by enumeration, tools/quantiser_check.c): 6 dependent ALU ops per sample instead
//     of 5 conversion-unit/fp64 ops (~55 cycles);
//   * both clamps run as one VIADDMNMX.RELU each by carrying the samples with a +32768 bias and the nibbles with
//     a +8 bias (the biases fold into the multiply-add constants);
//   * the ">> 11" of the reconstruction is taken off the chain: (guess + q*2^K + 1024) >> 11 ==
//     q*2^(K-11) + ((guess + 1024) >> 11) because K >= 11;
//   * the residual pass against raw neighbours (:107-115) is software-pipelined one frame ahead for the 12 samples
//     that do not depend on the reconstructed history.
// The fast expression is exact while |diff| < 2^24 (float32 holds the difference exactly) and, beyond that, whenever
// the float32 rounding provably cannot move the result (gc_pass_end's test); the few frames with a pass that fails the
// test are recomputed with the general exact path (wrapping int32 arithmetic + the float32-rounding-aware integer
// quantiser).
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace vgb {

constexpr uint32_t kFull = 0xFFFFFFFFu;
constexpr int kEncChunkFrames = 16;                                   // frames staged per chunk
constexpr int kEncChunkSamples = kEncChunkFrames * kGcFrameSamples;   // 224 samples = 448 B = 28 x 16 B
constexpr int kEncWarps = 2;                                          // warps per CTA
constexpr int kEncWarpChannels = 4;                                   // channels per warp (8 lanes each)
constexpr int kEncRowPad = 4;                                         // int32 words after each channel's x_buf row: 4 banks apart
#ifndef VGB_ENC_BLOCKS_PER_SM
#define VGB_ENC_BLOCKS_PER_SM 8
#endif
constexpr int kEncChainBlocksPerSm = VGB_ENC_BLOCKS_PER_SM;               // register budget of the chain launch: 8 CTAs x 2 warps = 4 warps per sub-partition
constexpr uint32_t kErrSat = (1u << 27) - 1;                          // one 32-bit argmin while err < 2^27 - 1
// The bits 0x4B000000 + v are the float32 2^23 + v for 0 <= v < 2^23, so a biased sample in [0, 65535] carries its own
// float image.  The staged samples hold x + kStageBias; every integer use of them is a wrapping multiply-add whose
// constant absorbs the image (0x4B000000 * 2048 == 0 modulo 2^32).
constexpr uint32_t kFloatImage = 0x4B000000u;
constexpr uint32_t kStageBias = 32768u + kFloatImage;

template <bool kGeneral>
struct GcTrial {
    uint32_t w0, w1;   // the 8 frame bytes as two little-endian words (byte 0 = header, filled by the winner)
    int32_t r1, r2;    // newest / second newest reconstructed sample
    int32_t over;      // maxOverflow (:132,:147-151)
    uint64_t err;      // TotalDistance (:163) - a sum of squared integers, exact in 64 bits (< 2^36)
    int32_t recon[kGeneral ? 14 : 1];  // full reconstruction, only for the independent-frames entry point
};

// ---------------------------------------------------------------------------------------------------------
// The reference's quantiser cast chain (:142-144)
//     (int)((double)((float)diff / scale) +/- 0.4999999f)
// as integer arithmetic.  scale = 2^shift (11 <= shift <= 23).  (float)diff rounds |diff| to 24 significant bits
// (nearest-even); the division is exact; adding 0.4999999f (= 0.5 - 3*2^-25) in double is exact and the truncation
// then rounds half toward zero.  With a = |diff| this is  m = (a + 2^(shift-1) - 1 - hs) >> shift  where
// hs = 0 if a < 2^24, else half a float32 ulp of a = 2^(floor(log2 a) - 24).  Enumerated against the literal
// chain for every shift in tools/quantiser_check.c.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int32_t gc_quantise_exact(int32_t diff, int shift)
{
    const uint32_t a = diff < 0 ? (0u - (uint32_t)diff) : (uint32_t)diff;
    const uint32_t top = a >> 24;
    const uint32_t hs = top ? (0x80000000u >> __clz(top)) : 0u;  // largest power of two <= top
    const uint32_t m = (a + (1u << (shift - 1)) - 1u - hs) >> shift;
    return diff < 0 ? -(int32_t)m : (int32_t)m;
}

// One pass of the do/while body (:129-164) at a fixed scalePower — general exact form (any coefficients, any
// history; int32 wrap-around like the reference, A.7).  Fed from memory (the frame's 14 samples at `frame`) and only
// reached through the out-of-line wrappers below, so the hot loop neither spills nor grows.
template <bool kGeneral>
__device__ __forceinline__ void gc_attempt_exact(const int16_t *frame, int n, int32_t h1, int32_t h2, int32_t c0,
                                              int32_t c1, int sp, GcTrial<kGeneral> &t)
{
    const int shift = sp + 11;
    const int32_t scale = (int32_t)(1u << shift);  // (1 << scalePower) * 2048
    int32_t r1 = h1, r2 = h2, over = 0;
    uint64_t err = 0;
    uint32_t w0 = 0, w1 = 0;
#pragma unroll
    for (int s = 0; s < 14; s++) {
        if (kGeneral && s >= n) break;
        const int32_t xs = frame[s];
        const int32_t want = xs * 2048;
        const int32_t guess = wadd(wmul(r2, c1), wmul(r1, c0));
        const int32_t diff = wsub(want, guess);
        const int32_t raw = gc_quantise_exact(diff, shift);
        const int32_t q = clamp4(raw);
        over = max(over, abs(raw - q));
        const int32_t out = clamp16(wadd(wadd(guess, wmul(q, scale)), 1024) >> 11);
        const int32_t miss = xs - out;
        err += (uint64_t)((int64_t)miss * miss);
        const int byte = 1 + s / 2, bit = (byte & 3) * 8 + ((s & 1) ? 0 : 4);
        if (byte < 4) w0 |= (uint32_t)(q & 15) << bit; else w1 |= (uint32_t)(q & 15) << bit;
        if (kGeneral) t.recon[s] = out;
        r2 = r1;
        r1 = out;
    }
    t.w0 = w0; t.w1 = w1; t.r1 = r1; t.r2 = r2; t.over = over; t.err = err;
}

// a*b + c as ONE multiply-add the compiler may not re-associate (it would otherwise canonicalise the integer sums
// and put two IMADs plus an add back on the dependent chain).  Wrapping arithmetic, like the reference.
__device__ __forceinline__ int32_t imad(int32_t a, int32_t b, int32_t c)
{
    int32_t d;
    asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// a >> k (arithmetic) the compiler may not commute with a later select.
__device__ __forceinline__ int32_t sar(int32_t a, int k)
{
    int32_t d;
    asm("shr.s32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(k));
    return d;
}

// The literal do/while of DspEncodeCoef (:127-170), used when the speculative window does not cover the chain.
// A pass at scalePower 12 is final: see the termination note in oracle/gcadpcm.c (the reference does not halt there).
template <bool kGeneral>
__device__ __forceinline__ void gc_try_predictor_literal(const int16_t *frame, int n, int32_t h1, int32_t h2, int32_t c0,
                                                         int32_t c1, int sp_first, GcTrial<kGeneral> &t, int &sp_out)
{
    int sp = sp_first - 1;
    do {
        sp++;
        gc_attempt_exact<kGeneral>(frame, n, h1, h2, c0, c1, sp, t);
        const int pass_power = sp;
        for (int v = t.over + 8; v > 256; v >>= 1)
            if (++sp >= 12) sp = 11;
        if (pass_power >= 12) { sp = 12; break; }
    } while (sp < 12 && t.over > 1);
    sp_out = sp;
}

// Residual of one sample against the RAW neighbours (:107-115) folded into an order-preserving key:
// larger |distance| wins, then the EARLIER sample (the reference keeps the first maximum: strict '>'), and the
// sign rides in bit 0 so the signed maxDistance can be rebuilt.  `neg_bias` is added to the prediction sum
// before the division (0 for raw samples, -32768*(c0+c1) when older/newer carry the +32768 bias).
__device__ __forceinline__ uint32_t gc_peak_key(int32_t older, int32_t newer, int32_t cur, int32_t c0, int32_t c1, int s,
                                                int32_t neg_bias = 0)
{
    const int32_t guess = imad(newer, c0, imad(older, c1, neg_bias)) / 2048;  // truncates toward zero (A.6)
    const int32_t diff = clamp16(wsub(cur, guess));
    return ((uint32_t)abs(diff) << 5) | ((uint32_t)(15 - s) << 1) | ((uint32_t)diff >> 31);
}

// The same residual for the channel encoder's hot loop, cheaper on the integer ALU pipe (the busiest unit of that
// kernel): the distance is NOT clamped per sample and the two signs are tracked as two running maxima of
// (+-distance * 16 + order), order = 15 - s, so that a larger |distance| wins and then the earlier sample, exactly the
// reference's strict '>'.  Per sample that is three multiply-adds and the truncating division; the maxima are taken
// two samples at a time.  gc_peak_pack folds the pair back into the key format above (|distance| << 5 | order << 1 |
// sign); Clamp16 (:113) is applied to the winner there - clamping commutes with the maximum, and among clamped
// samples sign and order no longer matter: every |distance| >= 18432 gives scalePower 12 whatever its sign.
// All three samples carry kStageBias, the bias of the staged data; neg_bias = -kStageBias * (c0 + c1) removes it from
// the sum (modulo 2^32: the true sums fit in int32, so the wrapping ones are exact).
__device__ __forceinline__ void gc_peak_terms(int32_t older, int32_t newer, int32_t cur, int32_t c0, int32_t c1, int s,
                                              int32_t neg_bias, int32_t &tp, int32_t &tn)
{
    const int32_t g = imad(newer, c0, imad(older, c1, neg_bias));
    const int32_t q = (int32_t)(g + (int32_t)((uint32_t)(g >> 31) >> 21)) >> 11;  // g / 2048, truncating toward zero (A.6)
    const int32_t d = imad(q, -1, cur);                                           // distance + kStageBias; |distance| < 2^21
    tp = imad(d, 16, (int32_t)(15u - s - kStageBias * 16u));
    tn = imad(d, -16, (int32_t)(15u - s + kStageBias * 16u));
}
__device__ __forceinline__ uint32_t gc_peak_pack(int32_t kp, int32_t kn)
{
    const int32_t k = max(kp, kn);                    // (|distance| << 4) | order of the first largest sample (0: none)
    return ((uint32_t)k << 1) | (uint32_t)(kn > kp);  // sign in bit 0
}
constexpr uint32_t kPeakKeyMax = (32768u << 5) | 1u;  // Clamp16: -32768 (a positive 32767 gives the same scalePower)

// First value scalePower takes inside the do/while (:118-129), from the max-residual key.  Closed form of
//   n = 0; while (n <= 12 && (peak > 7 || peak < -8)) { peak /= 2; n++; }   ("/" truncates toward zero)
// positive peak a: smallest n with a < 8*2^n; negative peak -a: smallest n with a < 9*2^n (a <= 32768 so n <= 12).
// The key holds a in bits 5.., so bitlength(a) = bitlength(key) - 5.
__device__ __forceinline__ int gc_first_scale_power(uint32_t key)
{
    int top;  // index of the highest set bit, -1 for key == 0
    asm("bfind.u32 %0, %1;" : "=r"(top) : "r"(key));
    const int n = max(top - 7, 0);                               // max(bitlength(a) - 3, 0)
    // negative peak with a in [8,9) * 2^(n-1) needs one halving less.  For n > 0 the four bits key >> (n+4) are
    // 8..15, so "== 8" is "< 9"; everything stays in integer registers (a predicate costs ~13 cycles of latency).
    const uint32_t t = key >> ((n + 4) & 31);
    const uint32_t one_less = ((t - 9u) >> 31) & key & ((uint32_t)(-n) >> 31);
    return max(n - 1 - (int)one_less, 0);                        // n <= 1 ? 0 : n - 1
}

// Minimum over the 8 lanes of a quarter-warp (one channel), known to all 8: a butterfly of three SHFL + IMNMX.  Four
// channels per warp would need four REDUX instructions with neutral elements (plus the selects); this is fewer issues.
__device__ __forceinline__ uint32_t quarter_min_u32(uint32_t v)
{
    v = min(v, __shfl_xor_sync(kFull, v, 1));
    v = min(v, __shfl_xor_sync(kFull, v, 2));
    return min(v, __shfl_xor_sync(kFull, v, 4));
}

// DspEncodeFrame (:48-94) for one frame of each of the warp's four channels with the general exact arithmetic and the
// literal scale loop: the rare path of the channel encoder (a pass failed the exactness test, a scale chain left the
// speculative window, an overflow bump).  Warp-uniform call; lane & 7 = predictor, every lane runs its predictor's
// literal loop.  A quarter with `commit` set writes its 8 frame bytes to out8 and gets its winner's biased newest two
// samples back (packed like the hot path); the other quarters' return values are unspecified.
__device__ __noinline__ uint32_t gc_slow_frame(const int16_t *frame, int32_t h1, int32_t h2, int32_t c0, int32_t c1,
                                               int sp_first, int lane, bool commit, uint8_t *out8)
{
    const int pred = lane & 7;
    GcTrial<false> t;
    t.err = 0; t.r1 = 0; t.r2 = 0; t.w0 = 0; t.w1 = 0;
    int sp_final = 0;
    gc_try_predictor_literal<false>(frame, 14, h1, h2, c0, c1, sp_first, t, sp_final);
    const uint64_t full_key = (t.err << 3) | (uint64_t)pred;  // first minimum wins (:66-76)
    const uint32_t hi = (uint32_t)(full_key >> 16);
    const uint32_t min_hi = quarter_min_u32(hi);
    const uint32_t lo = hi == min_hi ? (uint32_t)(full_key & 0xFFFFu) : 0xFFFFFFFFu;
    const uint32_t min_lo = quarter_min_u32(lo);
    if (hi == min_hi && lo == min_lo && commit) {
        const uint32_t head = (uint32_t)((pred << 4) | (sp_final & 0xF));  // CombineNibbles (:83)
        *reinterpret_cast<uint2 *>(out8) = make_uint2(t.w0 | head, t.w1);
    }
    const uint32_t mine = (uint32_t)(t.r1 + 32768) | ((uint32_t)(t.r2 + 32768) << 16);
    return __shfl_sync(kFull, mine, (lane & ~7) | (int)(min_lo & 7u));
}

// One speculative pass of the channel encoder's hot loop: the do/while body (:129-164) at one scalePower, as the
// constants of that power and the running state of the 14-step recurrence.  A lane carries two of them (scale powers
// sp and sp + 1) as independent register sets, so the two recurrences interleave in one straight-line block.
struct GcPass {
    int sp;              // scalePower of the pass (the candidate clamped to 12)
    bool valid;          // the candidate is <= 12: the chain can reach it
    int shift;           // sp + 11
    int32_t mul;         // 2^(shift-11)
    int32_t base_g;      // wf = guess + 1024 - 8*2^shift = c0*p1 + c1*p2 + base_g
    int32_t base_t;      // tm1 = diff + half - 1 = x*2048 + base_t - wf   (x carries +32768: folded in)
    uint32_t near_c;     // 128 << (32 - shift)
    uint32_t near_k;     // (1 << (32 - shift)) + near_c: (tm1 << lsh) + near_k = (tn << lsh) + near_c with tn = tm1 + 1
    int32_t lmul;        // 1 << (32 - shift)
    int32_t r1, r2;      // newest two reconstructed samples (biased +32768)
    int32_t rmin, rmax, raw_even;
    uint32_t nearmin;    // smallest distance of (diff + half) to a multiple of 2^shift, scaled
    uint32_t near_even;  // that distance of the last even sample (folded in with the odd one)
    uint32_t nw0, nw1;   // nibbles, biased +8
    uint32_t elo;        // squared error modulo 2^32 (the wrap is intended; the error is < 14 * 2^32)
    float ef;            // the same sum in float32, within 2^16 of it: the multiple of 2^32 (gc_err_exact)
};

__device__ __forceinline__ void gc_pass_begin(GcPass &P, int sp_raw, int32_t bias_c, int32_t p1, int32_t p2)
{
    P.sp = min(sp_raw, 12);
    P.valid = sp_raw <= 12;
    P.shift = P.sp + 11;
    P.mul = (int32_t)(1u << P.sp);
    P.base_g = wsub(wsub(1024, (int32_t)(8u << P.shift)), bias_c);
    // diff + half - 1 = (x - 32768)*2048 - (guess + 1024 - 8*2^shift) + 1024 - 8*2^shift + 2^(shift-1) - 1
    P.base_t = wadd(P.base_g, wadd(bias_c, (int32_t)(1u << (P.shift - 1))) - 1 - 32768 * 2048);
    const int lsh = 32 - P.shift;
    P.near_c = 128u << lsh;
    P.near_k = (1u << lsh) + P.near_c;
    P.lmul = (int32_t)(1u << lsh);
    P.r1 = p1; P.r2 = p2;
    P.rmin = 0; P.rmax = 0; P.raw_even = 0;
    P.nearmin = 0xFFFFFFFFu;
    P.near_even = 0xFFFFFFFFu;
    P.nw0 = 0; P.nw1 = 0;
    P.elo = 0; P.ef = 0.0f;
}

// Sample s (a compile-time constant once unrolled) of the recurrence; xs = the staged sample (x + kStageBias), and
// xw = xs * 2048 = (x + 32768) * 2048 (shared by the lane's passes).  Per sample the dependent chain is IMAD -> IADD3 ->
// LEA.HI -> SHF -> VIADDMNMX.RELU -> IMAD -> VIADDMNMX.RELU; range of raw (maxOverflow), distance to a rounding
// threshold, squared error and nibble packing ride along as independent work and nothing per sample is kept in
// registers.  The IMAD and the integer ALU pipes each take one warp instruction every two cycles (DESIGN.md §5.3), so
// the side work is split between them: tm1 is rebuilt from wf with one IADD3 instead of its own multiply-adds (modulo
// 2^32, x*2048 + base_m - c0*r1 - c1*r2 == x*2048 + base_t - wf).  The squared error stays off IMAD.WIDE (a 64-bit
// accumulate takes three IMAD slots): a 32-bit IMAD sums it modulo 2^32 and the FP32 pipe, idle otherwise, sums it
// again in float32 (an FP32 instruction costs about half an IMAD slot).  The float images of the sample and of the
// reconstruction are in [2^23, 2^24), so their difference is the exact miss; each FFMA rounds once, by at most 2^11
// below 2^36, so the float sum is within 14 * 2^11 < 2^16 of the exact one (tools/gc_err_check.c checks that bound on
// worst-case frames).
__device__ __forceinline__ void gc_pass_step(GcPass &P, int s, int32_t xs, int32_t xw, int32_t c0, int32_t c1)
{
    const int32_t gn = imad(P.r2, c1, P.base_g);     // r2 term: one step off the chain
    const int32_t wf = imad(P.r1, c0, gn);           // guess + 1024 - 8*2^shift  <- chain
    const int32_t tm1 = wsub(wadd(xw, P.base_t), wf);  // diff + half - 1 (one IADD3: wf comes out of asm, nothing to re-associate)
    // round half toward zero: (diff + half - (diff > 0)) >> shift = (tm1 + (diff <= 0)) >> shift.  diff <= 0 is
    // tm1 < half, and for 0 <= tm1 < half both tm1 and tm1 + 1 shift to 0: only the SIGN of tm1 matters
    const int32_t t2 = tm1 + (int32_t)((uint32_t)tm1 >> 31);
    const int32_t raw = sar(t2, P.shift);
    const int32_t qb = __viaddmin_s32_relu(raw, 8, 15);        // clamp4(raw) + 8
    const int32_t o = imad(qb, P.mul, wf >> 11);
    const int32_t ob = __viaddmin_s32_relu(o, 32768, 65535);   // clamp16(o) + 32768
    P.r2 = P.r1;
    P.r1 = ob;
    if (s & 1) {
        P.rmin = __vimin3_s32(P.rmin, P.raw_even, raw);
        P.rmax = __vimax3_s32(P.rmax, P.raw_even, raw);
    } else {
        P.raw_even = raw;
    }
    const uint32_t near = (uint32_t)imad(tm1, P.lmul, (int32_t)P.near_k);   // (tm1 << lsh) + near_k
    if (s & 1) P.nearmin = __vimin3_u32(P.nearmin, P.near_even, near);
    else P.near_even = near;
    const int32_t obf = (int32_t)((uint32_t)ob | kFloatImage);   // float image of ob: 2^23 + ob
    const int32_t miss = imad(obf, -1, xs);                        // x - out: the images cancel
    P.elo = (uint32_t)imad(miss, miss, (int32_t)P.elo);
    const float mf = __fsub_rn(__int_as_float(xs), __int_as_float(obf));  // x - out, exact
    P.ef = __fmaf_rn(mf, mf, P.ef);  // explicit: the build runs with --fmad=false
    const int byte = 1 + s / 2, bit = (byte & 3) * 8 + ((s & 1) ? 0 : 4);
    if (byte < 4) P.nw0 = (uint32_t)imad(qb, 1 << bit, (int32_t)P.nw0);
    else P.nw1 = (uint32_t)imad(qb, (int32_t)(1u << bit), (int32_t)P.nw1);  // disjoint bit fields: add == or
}

// The pass's verdict, from branch-free flags.  maxOverflow (:147-151) is max(rmax - 7, -8 - rmin, 0); only its
// comparisons are needed, and all of them are thresholds of one number, m = max(rmax + 1, -rmin):
//   over <= 1  <=>  rmax <= 8 and rmin >= -9    <=>  m <= 9
//   over >= 240 <=> rmax >= 247 or rmin <= -248 <=>  m >= 248
//   over > 248 <=>  rmax > 255 or rmin < -256   <=>  m >= 257
// big / huge (|raw| >= threshold) use m >= threshold, which can only err on the careful side.
//   term     the while (:170) fails after this pass: it ends the chain
//   trouble  the pass may differ from the reference's (inexact) or the chain leaves the one-step window (bump :166-168)
__device__ __forceinline__ void gc_pass_end(const GcPass &P, bool &term, bool &trouble)
{
    const int32_t m = __viaddmax_s32(P.rmax, 1, -P.rmin);
    const int32_t m_scaled = imad(m, P.mul, 0);                   // m * 2^(shift-11) <= 2^21
    // predicates combined with non-short-circuit operators: compare-and-combine is one instruction each
    const bool big = m_scaled >= (1 << 13);     // some |diff| >= 2^24 (or one short of it)
    const bool huge = m_scaled >= (1 << 18);    // some |diff| >= 2^29
    const bool over_ge_240 = m >= 248;
    const bool over_gt_248 = m >= 257;
    const bool over_le_1 = m <= 9;
    const bool near = (P.nearmin <= 2u * P.near_c) | over_ge_240;
    trouble = P.valid & ((huge | (big & near)) | ((P.sp < 12) & over_gt_248));
    term = P.valid & (over_le_1 | (P.sp >= 12));
}

// The exact squared error of a pass from its two sums: err = ef + d with |d| < 2^16, and err == elo modulo 2^32.  Only
// the loud-frame argmin needs it; below 2^31, ef already proves err == elo (the tail's saturated key).
__device__ __forceinline__ uint64_t gc_err_exact(float ef, uint32_t elo)
{
    const uint64_t approx = __float2ull_rz(ef);  // a whole number (every float32 >= 2^24 is one, and below it the sum is exact)
    return approx + (uint64_t)(int64_t)(int32_t)(elo - (uint32_t)approx);
}

// ---------------------------------------------------------------------------------------------------------
// TIME-PARALLEL ENCODING (speculate -> verify -> splice).  Frames of a channel are serial only through the two
// reconstructed samples a frame hands to the next (:40-41).  Quantise/reconstruct is error feedback, so a chain that
// starts from a WRONG history re-locks onto the true chain after a few frames (measured with the oracle on the
// synthetic set: median ~10 frames, tail < 1000), and once two chains agree on (hist1, hist2) after the same frame
// they agree forever (a frame's output is a pure function of its samples, the coefficients and the entering pair).
// So the frame range [frame_begin, frame_end) of every channel is cut into seg_count segments of seg_len frames
// (a multiple of 16) and encoded by three launches of the same kernel body:
//   kGcChain    (grid.y = segment)   segment 0 starts from the true history, segment s > 0 from the RAW samples
//               before its first frame; each writes its frame bytes and, per frame, the pair it hands on
//               (`trace`, 4 B per frame).
//   kGcRunOn    (grid.y = boundary)  the chain of segment s-1 runs on into segment s from its own end state
//               (trace[lo-1]), overwriting bytes and trace, until the pair after a frame equals the one recorded
//               there: from that frame on the recorded chain IS the true chain.  Each boundary notes the start pair
//               it used; boundaries run in parallel and stay inside their segment.
//   kGcCascade  (one pass per channel) repairs the rare boundary whose predecessor did not splice inside its segment
//               (its end pair changed after the successor had used it): it runs on serially, across segment ends if
//               need be, until a splice or the end of the channel - the reference's plain serial loop as the last
//               resort - and stores the final history.
// Exact by construction: every byte that stays was produced by a frame step from the true entering pair; the only
// test is equality of two int16 pairs.  Invariant the splice relies on: inside a segment, (bytes[k], trace[k]) is
// always the step from trace[k-1]; only a segment's first frame may sit on a seam.
// ---------------------------------------------------------------------------------------------------------
constexpr int kGcChain = 0, kGcRunOn = 1, kGcCascade = 2;

// frames per segment of a channel with `range_frames` frames to encode (device and host agree on this)
__host__ __device__ __forceinline__ int gc_seg_len(int range_frames, int seg_count, int min_seg_frames)
{
    const int per = (div_round_up(range_frames, seg_count > 0 ? seg_count : 1) + kEncChunkFrames - 1) / kEncChunkFrames * kEncChunkFrames;
    return per < min_seg_frames ? min_seg_frames : per;
}

// grid.x: one QUARTER-WARP per channel (four channels per warp); encodes frames [frame_begin, frame_end) of every
// channel, carrying the history in tab.hist between launches (frame_begin must be a multiple of 16).
//
// Lane & 7 = predictor: the 8 predictors of a channel are searched in parallel and each lane evaluates two consecutive
// scale powers of its predictor speculatively, as two independent recurrences (every pass is a pure function of
// (samples, history, coefs, scalePower), so the reference's do/while chain :127-170 is replayed over finished passes
// inside the lane: the first pass that ends the chain wins).  The reference's first guess is deliberately one power
// low, so on real signals the chain ends at the first pass in ~11 % and at the second in ~88.6 % of predictor-frames;
// when a predictor needs a third pass the warp runs a second round of one pass; a fourth goes to gc_slow_frame.
//
// The per-frame code is DspEncodeFrame (:48-94), written as one software-pipelined block:
//   head     residual keys of samples 0,1 (they need the reconstructed history) + the 12 keys computed one frame
//            ahead -> first scalePower -> the constants of the lane's two passes
//   passes   the two 14-step recurrences (gc_pass_step), interleaved; the next frame's loads / residual keys ride
//            along as independent work
//   verdict  range of raw (maxOverflow), exactness test (gc_pass_end), in-lane replay of the chain
//   tail     one vote (does any predictor need round 1), an 8-lane butterfly MIN for each channel's argmin, one SHFL
//            to broadcast each winner's two newest samples, one ballot for trouble; anything unusual re-runs the frame
//            in gc_slow_frame.
// Exactness of a pass (tools/quantiser_check.c enumerates the quantiser identity):
//   * every |diff| < 2^24: float32 holds diff exactly, the pass is bit-identical to the reference cast chain;
//   * some |diff| >= 2^24 ("big"): the float32 rounding moves a quantiser threshold by hs <= 128, which changes
//     `raw` only if (diff + half) lies within 128 of a multiple of 2^shift ("near"), and then by one - invisible
//     to the clamped nibble when |raw| >= 15, but it could flip the overflow-bump test at 248 (`over >= 240`);
//   * some |diff| >= 2^29 ("huge", hostile coefficients only): the biased sums could wrap.
template <int kMode>
__global__ void __launch_bounds__(kEncWarps * 32, kMode == kGcChain ? kEncChainBlocksPerSm : 1)
gc_encode_kernel(const int16_t *__restrict__ pcm, GcChannelTable tab, const int16_t *__restrict__ coefs,
                 uint8_t *__restrict__ adpcm, int frame_begin, int frame_end, GcSegArgs sa)
{
    __shared__ __align__(16) int16_t in_buf[kEncWarps][kEncWarpChannels][2][kEncChunkSamples];   // [warp][channel][buffer], cp.async target
    // the same samples widened once per chunk, +32768; a channel's row holds both buffers and is padded so that the
    // four channels' broadcast loads of the same sample fall in different banks
    __shared__ __align__(16) int32_t x_buf[kEncWarps][kEncWarpChannels][2 * kEncChunkSamples + kEncRowPad];
    __shared__ __align__(16) uint8_t out_buf[kEncWarps][kEncWarpChannels][kEncChunkFrames * kGcFrameBytes];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qc = lane >> 3, pred = lane & 7;                          // channel of the warp, predictor
    const int ch0 = (blockIdx.x * kEncWarps + warp) * kEncWarpChannels;
    if (ch0 >= tab.n_channels) return;                                  // whole warp beyond the batch
    const bool live = ch0 + qc < tab.n_channels;                        // ragged channel count: upper quarters idle
    const int ch = live ? ch0 + qc : tab.n_channels - 1;

    const int n_enc = live ? tab.enc_count[ch] : 0;
    const int n_frames = div_round_up(n_enc, kGcFrameSamples);
    const int f_end = min(frame_end, n_frames);                         // this channel's end of the frame range
    const int range_frames = max(f_end - frame_begin, 0);
    const int seg_len = gc_seg_len(range_frames, sa.seg_count, sa.min_seg_frames);         // this channel's frames per segment
    const int total_bytes = gc_sample_count_to_byte_count(n_enc);

    const int16_t *src = pcm + tab.pcm_off[ch];
    uint8_t *dst = adpcm + tab.adpcm_off[ch];
    uint32_t *trace = sa.trace + tab.rec_off[ch];                       // [frame] pair handed on: hist1+32768 | (hist2+32768) << 16
    uint32_t *used_start = sa.used_start + (int64_t)ch * sa.seg_count;  // [segment] pair the boundary's run-on started from
    const int32_t c0 = coefs[(int64_t)ch * 16 + 2 * pred];
    const int32_t c1 = coefs[(int64_t)ch * 16 + 2 * pred + 1];
    const int32_t bias_c = wmul(32768, wadd(c0, c1));  // undoes the +32768 bias of both history samples
    const int32_t neg_bias_s = (int32_t)(0u - kStageBias * (uint32_t)wadd(c0, c1));  // undoes kStageBias (gc_peak_terms)
    int16_t (*const in_row)[kEncChunkSamples] = in_buf[warp][qc];
    int32_t *const x_row = x_buf[warp][qc];

    // Stage the 28 16-byte vectors of the chunk starting at `chunk_frame` into buffer b with cp.async (LDGSTS): the
    // copy needs no registers, so it is issued a whole chunk ahead and DRAM latency never shows - a register-staged
    // load was moved next to its first use by the compiler and cost ~1300 cycles per chunk (ncu).
    // Bytes past the encoded sample count are zero-filled by the copy itself (src-size operand; GcAdpcmEncoder.cs:32-34).
    auto stage_chunk = [&](int chunk_frame, int b) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int v = pred + 8 * k;
            if (v < kEncChunkSamples / 8) {
                const int64_t s = (int64_t)chunk_frame * kGcFrameSamples + v * 8;
                int64_t valid = (int64_t)n_enc - s;
                valid = valid < 0 ? 0 : (valid > 8 ? 8 : valid);
                const int16_t *from = valid > 0 ? src + s : src;
                const unsigned to = (unsigned)__cvta_generic_to_shared(&in_row[b][v * 8]);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(to), "l"(from), "r"((int)valid * 2) : "memory");
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    auto staged_wait = [&]() {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncwarp();
    };
    // int16 -> int32 once per chunk (frames pred and pred + 8 of the chunk) instead of a 16-bit load and a sign
    // extension per sample use: the frame loop then reads whole 64-bit pairs, broadcast to the 8 lanes of a channel.
    // Stored as x + kStageBias: the +32768 bias and the float image of the biased sample
    auto widen_chunk = [&](int b) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int f = pred + 8 * h;
            const uint32_t *from = reinterpret_cast<const uint32_t *>(&in_row[b][f * kGcFrameSamples]);
            int2 *to = reinterpret_cast<int2 *>(&x_row[b * kEncChunkSamples + f * kGcFrameSamples]);
#pragma unroll
            for (int k = 0; k < kGcFrameSamples / 2; k++) {
                const uint32_t w = from[k];
                to[k] = make_int2((int32_t)((uint32_t)(int16_t)(w & 0xFFFFu) + kStageBias),
                                  (int32_t)((uint32_t)((int32_t)w >> 16) + kStageBias));
            }
        }
        __syncwarp();
    };
    // residual keys of samples 2..13 (raw samples only) of this lane's predictor
    auto key_rest_of = [&](const int32_t *frame) -> uint32_t {
        int32_t v[14];
#pragma unroll
        for (int j = 0; j < 14; j++) v[j] = frame[j];
        int32_t kp = 0, kn = 0;
#pragma unroll
        for (int j = 2; j < 14; j += 2) {
            int32_t tpa, tna, tpb, tnb;
            gc_peak_terms(v[j - 2], v[j - 1], v[j], c0, c1, j, neg_bias_s, tpa, tna);
            gc_peak_terms(v[j - 1], v[j], v[j + 1], c0, c1, j + 1, neg_bias_s, tpb, tnb);
            kp = __vimax3_s32(kp, tpa, tpb);
            kn = __vimax3_s32(kn, tna, tnb);
        }
        return gc_peak_pack(kp, kn);
    };

    // ---- jobs: a chain job is one segment; a run-on job is one segment boundary; the cascade walks the boundaries ----
    const int job_first = kMode == kGcChain ? (int)blockIdx.y : (kMode == kGcRunOn ? (int)blockIdx.y + 1 : 1);
    const int n_jobs = kMode == kGcCascade ? sa.seg_count - 1 : 1;  // a compile-time 1 for chain and run-on: no job loop
    int truth_upto = 0;           // cascade: frames below this index were finished by an earlier job of this pass
    int reencoded = 0;            // run-on / cascade statistics (frames encoded again)
    int32_t p1 = 0, p2 = 0;       // biased history (newest, older)

    for (int j = 0; j < n_jobs; j++) {
        const int job = job_first + j;
        const int seg_lo = frame_begin + job * seg_len;   // this channel's first frame (a multiple of 16 past frame_begin)
        bool need = live && seg_lo < f_end;
        uint32_t start_pair = 0;
        if (kMode == kGcChain) {
            if (need) {
                if (job == 0) {
                    p1 = tab.hist[2 * ch] + 32768; p2 = tab.hist[2 * ch + 1] + 32768;
                } else {  // speculative start: the raw samples in front of the segment
                    p1 = src[(int64_t)seg_lo * kGcFrameSamples - 1] + 32768; p2 = src[(int64_t)seg_lo * kGcFrameSamples - 2] + 32768;
                }
            }
        } else {
            if (kMode == kGcCascade) __syncwarp();  // trace words written by other lanes in an earlier job
            if (need) start_pair = trace[seg_lo - 1];
            if (kMode == kGcRunOn) {
                if (need && pred == 0) used_start[job] = start_pair;
            } else {
                need = need && seg_lo >= truth_upto && start_pair != used_start[job];
            }
            p1 = (int32_t)(start_pair & 0xFFFFu); p2 = (int32_t)(start_pair >> 16);
        }
        // chain / run-on stay inside their segment; the cascade may run to the end of the channel
        const int seg_hi = kMode == kGcCascade ? f_end : min(seg_lo + seg_len, f_end);
        const int len = need ? seg_hi - seg_lo : 0;
        int len_warp = max(len, __shfl_xor_sync(kFull, len, 8));  // the warp runs until all four channels are done
        len_warp = max(len_warp, __shfl_xor_sync(kFull, len_warp, 16));
        if (len_warp == 0) continue;
        bool spliced = false;      // run-on: the recorded chain was met, the rest of it is final
        int done = 0;              // frames this channel has encoded in this job

    int buf = 0;
    stage_chunk(seg_lo, 0);
    staged_wait();
    widen_chunk(0);
    // pipeline prologue: residual keys of the first frame
    uint32_t key_rest = key_rest_of(x_row);

    for (int rc = 0; rc < len_warp; rc += kEncChunkFrames) {
        const int cf = seg_lo + rc;                                            // this channel's chunk
        // next chunk -> the other buffer (dead since the previous chunk's last frame), awaited before the last frame
        stage_chunk(cf + kEncChunkFrames, buf ^ 1);
        const int frames_warp = min(kEncChunkFrames, len_warp - rc);
        const int frames_here = max(min(kEncChunkFrames, len - rc), 0);    // this channel's share
        const int32_t *chunk = x_row + buf * kEncChunkSamples;
        const int32_t *other = x_row + (buf ^ 1) * kEncChunkSamples;
        uint32_t tr0 = 0, tr1 = 0;           // the pairs frames cf + pred and cf + pred + 8 hand on
        uint32_t tr_old0 = 0, tr_old1 = 0;   // run-on: the pairs recorded there by the chain being met
        if (kMode != kGcChain && !spliced) {
            if (pred < frames_here) tr_old0 = trace[cf + pred];
            if (pred + 8 < frames_here) tr_old1 = trace[cf + pred + 8];
        }
        int frames_done = 0;
        bool all_done = false;

        for (int i = 0; i < frames_warp; i++) {
            if (i == kEncChunkFrames - 1) {  // this frame reads the next chunk's first samples
                staged_wait();
                widen_chunk(buf ^ 1);
            }
            const bool active = i < frames_here && !spliced;  // a finished channel idles while its warp mates go on
            const int32_t *frame = chunk + i * kGcFrameSamples;
            const int32_t *frame_next = (i + 1 < kEncChunkFrames) ? frame + kGcFrameSamples : other;
            // the frame's samples, x + kStageBias (same address for the 8 lanes of a channel: broadcast).  Not carried
            // in registers from the previous frame: 14 registers fewer per thread buy resident warps
            int32_t x[14];
#pragma unroll
            for (int j = 0; j < 14; j++) x[j] = frame[j];

            // ---------------- head ----------------
            int32_t tp0, tn0, tp1, tn1;
            const int32_t p1s = (int32_t)((uint32_t)p1 + kFloatImage), p2s = (int32_t)((uint32_t)p2 + kFloatImage);
            gc_peak_terms(p2s, p1s, x[0], c0, c1, 0, neg_bias_s, tp0, tn0);
            gc_peak_terms(p1s, x[0], x[1], c0, c1, 1, neg_bias_s, tp1, tn1);
            const uint32_t key = min(max(key_rest, gc_peak_pack(max(tp0, tp1), max(tn0, tn1))), kPeakKeyMax);
            const int sp_first = gc_first_scale_power(key);

            // result of this lane's chain-ending pass (or its latest, while unresolved)
            uint32_t w0 = 0, w1 = 0;
            uint32_t elo = 0;   // its squared error modulo 2^32 ...
            float ef = 0.0f;    // ... and in float32 (GcPass)
            int sp = 0;
            int32_t q1 = p1, q2 = p2;  // newest two reconstructed samples of that pass (biased)
            uint32_t key_rest_next = 0;
            bool resolved = !active;   // an idle channel reports "done" so that it never forces a second round
            bool trouble = false;

            // fully unrolled on purpose: in round 0 the next frame's loads/keys must sit in the same straight-line block
            // as the recurrences to be interleaved with them; the round-1 copy is cold code.  Round 0 runs powers
            // sp_first and sp_first + 1, round 1 only sp_first + 2: a chain that needs a fourth power is rare enough
            // (none on the benchmark's signals) to go to gc_slow_frame as unresolved.
#pragma unroll
            for (int round = 0; round < 2; round++) {
                GcPass A, B;
                gc_pass_begin(A, sp_first + 2 * round, bias_c, p1, p2);
                if (round == 0) gc_pass_begin(B, sp_first + 1, bias_c, p1, p2);
#pragma unroll
                for (int s = 0; s < 14; s++) {
                    const int32_t xw = imad(x[s], 2048, 0);
                    gc_pass_step(A, s, x[s], xw, c0, c1);
                    if (round == 0) gc_pass_step(B, s, x[s], xw, c0, c1);
                    // independent work for the NEXT frame rides along (software pipelining), first round only
                    if (round == 0 && s == 4) key_rest_next = key_rest_of(frame_next);
                }
                bool term_a, trouble_a, term_b = false, trouble_b = false;
                gc_pass_end(A, term_a, trouble_a);
                if (round == 0) gc_pass_end(B, term_b, trouble_b);
                // the first pass that ends the chain wins; B only counts when A did not end it.  Round 1 only
                // touches predictors round 0 left unresolved.
                const bool take = round == 0 || !resolved;
                const bool use_b = round == 0 && !term_a;
                if (take) {
                    trouble = trouble | (active & (trouble_a | (use_b & trouble_b)));
                    elo = use_b ? B.elo : A.elo;
                    ef = use_b ? B.ef : A.ef;
                    w0 = (use_b ? B.nw0 : A.nw0) ^ 0x88888800u;  // remove the +8 nibble bias (q & 15 == (q + 8) ^ 8)
                    w1 = (use_b ? B.nw1 : A.nw1) ^ 0x88888888u;
                    sp = use_b ? B.sp : A.sp;
                    q1 = use_b ? B.r1 : A.r1;
                    q2 = use_b ? B.r2 : A.r2;
                    resolved = resolved | term_a | term_b;
                }
                if (round == 0 && !__any_sync(kFull, !resolved)) break;  // warp-uniform: every predictor of the four channels resolved
            }
            // a predictor still unresolved after three powers leaves the window: handled as trouble
            trouble = trouble | !resolved;

            // ---------------- tail: argmin over predictors ----------------
            // first minimum wins (:66-76): the key is monotone in the predictor.  ef < 2^31 proves err < 2^32, so
            // err == elo; otherwise err > 2^31 - 2^16 > kErrSat.
            const uint32_t e_sat = ef < 2147483648.0f ? min(elo, kErrSat) : kErrSat;
            uint32_t best = quarter_min_u32(active ? ((e_sat << 3) | (uint32_t)pred) : 0xFFFFFFFFu);
            const bool sat = (best >> 3) >= kErrSat && best != 0xFFFFFFFFu;
            if (__any_sync(kFull, sat)) {
                // loud frame (warp-uniform): candidate errors of >= 2^27 - 1, reduce on the full 64-bit value
                const uint64_t full_key = active ? ((gc_err_exact(ef, elo) << 3) | (uint64_t)pred) : ~0ull;
                const uint32_t hi = (uint32_t)(full_key >> 16);
                const uint32_t min_hi = quarter_min_u32(hi);
                best = quarter_min_u32(hi == min_hi ? (uint32_t)(full_key & 0xFFFFu) : 0xFFFFFFFFu);  // low 3 bits = winner
            }
            const int best_lane = (lane & ~7) | (int)(best & 7u);
            const uint32_t head = (uint32_t)((pred << 4) | sp);  // CombineNibbles (:83)
            uint8_t *out8 = &out_buf[warp][qc][i * kGcFrameBytes];
            if (lane == best_lane && active) *reinterpret_cast<uint2 *>(out8) = make_uint2(w0 | head, w1);
            // pcmBuffer[0] = pcmBuffer[14]; pcmBuffer[1] = pcmBuffer[15] (:40-41): the winner's two newest samples
            uint32_t packed = __shfl_sync(kFull, (uint32_t)q1 | ((uint32_t)q2 << 16), best_lane);
            // anything unusual (rare): redo the frame with the exact arithmetic and the literal loop (an idle channel
            // raises no trouble)
            const uint32_t trouble_bits = __ballot_sync(kFull, trouble);
            if (trouble_bits != 0u) {
                __syncwarp();  // the fast path's frame bytes are overwritten below by another lane of the warp
                const bool mine = ((trouble_bits >> (lane & ~7)) & 0xFFu) != 0u && active;
                const uint32_t redo = gc_slow_frame(&in_row[buf][i * kGcFrameSamples], p1 - 32768, p2 - 32768, c0, c1, sp_first, lane, mine, out8);
                if (mine) packed = redo;
            }
            if (active) {
                p1 = (int32_t)(packed & 0xFFFFu);
                p2 = (int32_t)(packed >> 16);
                frames_done = i + 1;
                if (pred == i) tr0 = packed;
                if (pred + 8 == i) tr1 = packed;
            }
            if (kMode != kGcChain) {
                // splice test: the pair this frame hands on against the pair recorded after the same frame
                const uint32_t old = __shfl_sync(kFull, i < 8 ? tr_old0 : tr_old1, (lane & ~7) | (i & 7));
                if (active && packed == old) spliced = true;
                all_done = __all_sync(kFull, spliced || rc + i + 1 >= len);
                if (all_done) break;
            }

            key_rest = key_rest_next;
        }
        staged_wait();

        // write the bytes and trace words of the frames encoded in this chunk; only the channel's last frame can be
        // partial (:38)
        if (frames_done > 0) {
            const int64_t byte0 = (int64_t)cf * kGcFrameBytes;
            const int bytes_here = (int)min((int64_t)frames_done * kGcFrameBytes, (int64_t)total_bytes - byte0);
            const int b = pred * 16;
            if (b + 16 <= bytes_here) {
                *reinterpret_cast<uint4 *>(dst + byte0 + b) = *reinterpret_cast<const uint4 *>(&out_buf[warp][qc][b]);
            } else {
                for (int j = b; j < bytes_here; j++) dst[byte0 + j] = out_buf[warp][qc][j];
            }
            if (pred < frames_done) trace[cf + pred] = tr0;
            if (pred + 8 < frames_done) trace[cf + pred + 8] = tr1;
            done += frames_done;
        }
        __syncwarp();
        buf ^= 1;
        if (kMode != kGcChain && all_done) break;
    }
        // ---- end of the job ----
        if (kMode != kGcChain) {
            reencoded += done;
            if (kMode == kGcCascade && need) truth_upto = seg_lo + done;
            if (kMode == kGcRunOn && need && !spliced && pred == 0 && seg_hi < f_end)
                atomicAdd(&sa.stats[2], 1ull);  // this boundary's segment end changed under its successor
            if (kMode == kGcRunOn && need && pred == 0) {  // run-on length statistics: maximum and a log2 histogram
                atomicMax(&sa.stats[3], (unsigned long long)done);
                atomicAdd(&sa.stats[4 + min(31 - __clz(max(done, 1)), 13)], 1ull);
            }
        }
    }

    if (kMode != kGcChain && pred == 0 && reencoded > 0) atomicAdd(&sa.stats[kMode == kGcRunOn ? 0 : 1], (unsigned long long)reencoded);
    // the history the next call continues from (:40-41 carried across launches): the pair the range's last frame hands on
    if ((kMode == kGcCascade || (kMode == kGcChain && sa.seg_count == 1)) && live && range_frames > 0) {
        __syncwarp();
        if (pred == 0) {
            const uint32_t last = trace[f_end - 1];
            tab.hist[2 * ch] = (int16_t)((int32_t)(last & 0xFFFFu) - 32768);
            tab.hist[2 * ch + 1] = (int16_t)((int32_t)(last >> 16) - 32768);
        }
    }
}

// DspEncodeFrame for independent frames with any sample count 0..14: one warp per frame, general exact path
// (IDspTool.DspEncodeFrame / GcAdpcmAlignment use; not a throughput path).
__global__ void __launch_bounds__(128)
gc_encode_frames_kernel(int16_t *__restrict__ pcm_in_out, const int32_t *__restrict__ sample_count,
                        const int16_t *__restrict__ coefs, int n_frames, uint8_t *__restrict__ adpcm_out)
{
    __shared__ int16_t stage[4][16];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = blockIdx.x * (blockDim.x >> 5) + warp;
    if (f >= n_frames) return;
    int16_t *io = pcm_in_out + (int64_t)f * 16;
    const int n = sample_count ? min(max(sample_count[f], 0), 14) : 14;
    if (lane < 16) stage[warp][lane] = io[lane];
    __syncwarp();
    const int16_t *frame = &stage[warp][2];
    const int32_t h2 = stage[warp][0], h1 = stage[warp][1];
    const int pred = lane >> 2, cand = lane & 3;
    const int32_t c0 = coefs[(int64_t)f * 16 + 2 * pred], c1 = coefs[(int64_t)f * 16 + 2 * pred + 1];

    // residual pass (:107-115) over the first n samples
    uint32_t key = 0;
#pragma unroll
    for (int s = 0; s < 14; s++) {
        if (s >= n) break;
        const int32_t older = s == 0 ? h2 : (s == 1 ? h1 : (int32_t)frame[s >= 2 ? s - 2 : 0]);
        const int32_t newer = s == 0 ? h1 : (int32_t)frame[s >= 1 ? s - 1 : 0];
        key = max(key, gc_peak_key(older, newer, frame[s], c0, c1, s));
    }
    const int sp_first = gc_first_scale_power(key);

    // one lane per predictor runs the literal loop; the other three lanes idle
    GcTrial<true> t;
    t.err = 0;
    int sp_final = 0;
    const bool pred_winner = cand == 0;
    if (pred_winner) gc_try_predictor_literal<true>(frame, n, h1, h2, c0, c1, sp_first, t, sp_final);
    const uint64_t full_key = pred_winner ? ((t.err << 5) | (uint64_t)lane) : ~0ull;
    const uint32_t hi = (uint32_t)(full_key >> 16);
    const uint32_t min_hi = __reduce_min_sync(kFull, hi);
    const uint32_t lo = (pred_winner && hi == min_hi) ? (uint32_t)(full_key & 0xFFFFu) : 0xFFFFFFFFu;
    const uint32_t min_lo = __reduce_min_sync(kFull, lo);
    const bool is_winner = pred_winner && hi == min_hi && lo == min_lo;
    if (is_winner) {
        const uint32_t head = (uint32_t)((pred << 4) | (sp_final & 0xF));
        uint32_t w[2] = {t.w0 | head, t.w1};
        for (int j = 0; j < 8; j++) adpcm_out[(int64_t)f * 8 + j] = (uint8_t)(w[j >> 2] >> ((j & 3) * 8));
#pragma unroll
        for (int j = 0; j < 14; j++)
            if (j < n) io[2 + j] = (int16_t)t.recon[j];
    }
}

// Shortest segment, in frames (a multiple of 16).  A boundary costs a run-on of a few dozen frames as a rule, but the
// distribution has a long tail: loud, tonal material (predictor poles next to the unit circle) forgets a wrong history
// only over thousands of frames (measured on C2: 23 552 boundaries, median 8-16 frames, 20 above 1024, longest 3809).
// A run-on that does not splice inside its segment leaves the rest of the channel to the serial cascade, so segments
// stay longer than that tail; VGB_GC_MIN_SEG_FRAMES overrides (the tests use 256 to exercise many segments on short
// inputs).
int gc_encode_min_segment_frames()
{
    if (const char *env = std::getenv("VGB_GC_MIN_SEG_FRAMES")) {
        const int v = std::atoi(env);
        if (v >= kEncChunkFrames) return (v + kEncChunkFrames - 1) / kEncChunkFrames * kEncChunkFrames;
    }
    return kGcMinSegFrames;
}

// How many segments to cut the frame range into.  The chain launch is throughput bound once every SM sub-partition
// holds its resident warps (a lone warp per sub-partition waits on its own dependent chain), so the aim is (a) waves of
// (channel quad, segment) items on this device's SM count and the kernel's occupancy with as little idle issue as
// possible: the count s minimises waves(s) x frames per segment(s), and (b) segments longer than the run-on tail
// (above).  Of equally good counts the largest wins: items differ in time (frames that take the slow path), and a slot
// that runs several items evens that out, while a single wave ends with its slowest item (C2 on H100: 8 segments =
// one wave 37.6 ms, 16 or 24 segments 36.6 ms; tools/seg_sweep.py sweeps the count).
int gc_encode_pick_segments(int n_channels, int max_frames, int *min_seg_out)
{
    int min_seg = gc_encode_min_segment_frames();
    if (min_seg_out) *min_seg_out = min_seg;
    if (const char *env = std::getenv("VGB_GC_SEGMENTS")) {
        const int v = std::atoi(env);
        if (v >= 1) return v > kGcMaxSegments ? kGcMaxSegments : v;
    }
    static int slots = 0;
    if (slots == 0) {
        int dev = 0, sms = 132, per_sm = kEncChainBlocksPerSm;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gc_encode_kernel<kGcChain>, kEncWarps * 32, 0) != cudaSuccess || per_sm < 1) {
            (void)cudaGetLastError();
            per_sm = kEncChainBlocksPerSm;
        }
        slots = sms * per_sm * kEncWarps;  // resident warps of the chain launch
    }
    const int rows = (n_channels + kEncWarpChannels - 1) / kEncWarpChannels;  // warps per segment
    const int five_waves = (int)((5ll * slots + rows - 1) / rows);
    // A batch of SHORT channels too small to fill the machine with kGcMinSegFrames-long segments is latency bound (a
    // segment's serial chain): halve the minimum when a channel yields fewer than eight segments and fewer items than five
    // waves.  More boundaries then end in the cascade, but a few serial repairs cost less than chains twice as long (the
    // batch converter's files of 1-6 s).  Long channels keep the full minimum: with 2048-frame segments the 128-channel
    // groups of the pipelined host call lose more to the cascade's serial repairs than they gain.
    if (!std::getenv("VGB_GC_MIN_SEG_FRAMES") && max_frames / min_seg < std::min(five_waves, 8)) min_seg = std::max(kEncChunkFrames, min_seg / 2);
    if (min_seg_out) *min_seg_out = min_seg;
    const int max_s = std::min(kGcMaxSegments, std::max(1, max_frames / min_seg));
    int best = 1;
    long long best_cost = -1;
    for (int s = 1; s <= max_s; s++) {
        const long long waves = ((long long)rows * s + slots - 1) / slots;
        const long long cost = waves * gc_seg_len(max_frames, s, min_seg);
        if (best_cost < 0 || cost <= best_cost) { best = s; best_cost = cost; }
    }
    return best;
}

void launch_gc_encode(const int16_t *pcm, const GcChannelTable &tab, const int16_t *coefs, uint8_t *adpcm,
                      int max_frames, int frame_begin, int frame_end, GcSegArgs sa, cudaStream_t stream)
{
    if (tab.n_channels <= 0 || max_frames <= 0) return;
    if (frame_begin >= frame_end || frame_begin >= max_frames) return;
    const int per_block = kEncWarps * kEncWarpChannels;
    const int blocks = (tab.n_channels + per_block - 1) / per_block;
    if (sa.seg_count < 1) sa.seg_count = 1;
    if (sa.seg_count > kGcMaxSegments) sa.seg_count = kGcMaxSegments;
    if (sa.min_seg_frames <= 0) sa.min_seg_frames = gc_encode_min_segment_frames();  // else: chosen by gc_encode_pick_segments
    cudaMemsetAsync(sa.stats, 0, kGcStatWords * sizeof(unsigned long long), stream);
    gc_encode_kernel<kGcChain><<<dim3(blocks, sa.seg_count), kEncWarps * 32, 0, stream>>>(pcm, tab, coefs, adpcm, frame_begin, frame_end, sa);
    if (sa.seg_count > 1) {
        gc_encode_kernel<kGcRunOn><<<dim3(blocks, sa.seg_count - 1), kEncWarps * 32, 0, stream>>>(pcm, tab, coefs, adpcm, frame_begin, frame_end, sa);
        gc_encode_kernel<kGcCascade><<<dim3(blocks, 1), kEncWarps * 32, 0, stream>>>(pcm, tab, coefs, adpcm, frame_begin, frame_end, sa);
    }
}

void launch_gc_encode_frames(int16_t *pcm_in_out, const int32_t *sample_count, const int16_t *coefs, int n_frames,
                             uint8_t *adpcm_out, cudaStream_t stream)
{
    if (n_frames <= 0) return;
    int blocks = (n_frames + 3) / 4;
    gc_encode_frames_kernel<<<blocks, 128, 0, stream>>>(pcm_in_out, sample_count, coefs, n_frames, adpcm_out);
}

}  // namespace vgb
