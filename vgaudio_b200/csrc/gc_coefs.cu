// gc_coefs.cu — GC-ADPCM coefficient analysis on sm_90a (H100).
//
// Replaces GcAdpcmCoefficients.CalculateCoefficients (Codecs/GcAdpcm/GcAdpcmCoefficients.cs:9-110) for a whole
// batch of channels.  The reference is one serial fp64 loop per channel; here it is split where the data
// dependences allow it:
//
//   gc_coef_frames_kernel   phase 1 (:40-61): one THREAD per 14-sample frame, all channels x frames in flight.
//                           Each frame is a pure function of 16 samples (two of history).  The five integer
//                           correlations are exact in int64, the 2x2 LU / solve / reflection step is the
//                           reference's fp64 sequence.  The record is stored already pushed through MatrixFilter
//                           (:285-305), because that direct-form pair is the only thing phase 2 ever reads
//                           (it equals ContrastVectors' `val` terms bit for bit - see DESIGN.md §gc_coef_refine).
//                           HBM-bound by design: 2 B/sample in, 16 B + 1 bit per frame out.
//
//   gc_coef_refine_kernel   phase 2 (:63-108): one CTA per channel, producer warps + one consumer warp.  The
//                           nearest-centroid search is parallel over 32 records; the fp64 accumulations are applied
//                           strictly in record order (SURVEY.md A.1) by 16 accumulator lanes (8 buckets x 2
//                           components), because any tree reduction would change the roundings and can flip a 16-bit
//                           coefficient.  Records are compacted per bucket (ballot + popc) so each lane's DADD chain
//                           only contains its own bucket's records.
#include "common.cuh"
#include <cstdlib>

#include "kernels.h"

namespace vgb {

constexpr int kP1Threads = 256;             // frames per CTA tile
constexpr int kP1TileSamples = kP1Threads * kGcFrameSamples;  // 3584 samples = 7168 B = 448 x 16 B

// ---------------------------------------------------------------------------------------------------------
// phase 1: per-frame record
// ---------------------------------------------------------------------------------------------------------

// x[0..1] = the two samples before the frame (older first), x[2..15] = the frame (zero padded).
// Returns true when the reference would append a record (GcAdpcmCoefficients.cs:46-57) and sets d1,d2 to
// MatrixFilter(record)[1..2].
__device__ __forceinline__ bool gc_frame_direct(const int32_t (&x)[16], double &d1, double &d2)
{
    // InnerProductMerge (:112-120): -sum x[t-lag]*x[t].  Every product and partial sum is an integer below
    // 2^34, so the reference's sequential double accumulation is exact and equals the int64 sum.
    long long s0 = 0, s1 = 0, s2 = 0;
#pragma unroll
    for (int t = 0; t < 14; t++) {
        long long a = x[t + 2];
        s0 += a * x[t + 2];
        s1 += a * x[t + 1];
        s2 += a * x[t];
    }
    double v0 = 0.0 - (double)s0;  // "0.0 - s" keeps +0.0 for an all-zero frame like the reference's loop
    double v1 = 0.0 - (double)s1;
    double v2 = 0.0 - (double)s2;
    if (!(fabs(v0) > 10.0)) return false;  // :46

    // OuterProductMerge (:122-131) by sliding the lag-0/lag-1 sums one and two samples back (exact integers).
    long long c11 = s0 - (long long)x[15] * x[15] + (long long)x[1] * x[1];
    long long c22 = c11 - (long long)x[14] * x[14] + (long long)x[0] * x[0];
    long long c12 = s1 - (long long)x[15] * x[14] + (long long)x[1] * x[0];
    double m11 = (double)c11, m12 = (double)c12, m21 = (double)c12, m22 = (double)c22;

    // AnalyzeRanges (:133-208), 2x2 case written out.
    double big1 = fmax(fabs(m11), fabs(m12));
    if (big1 < 4.9406564584124654e-324) return false;  // double.Epsilon (A.2)
    double big2 = fmax(fabs(m21), fabs(m22));
    if (big2 < 4.9406564584124654e-324) return false;
    double inv1 = 1.0 / big1, inv2 = 1.0 / big2;

    int perm1 = 0;
    {
        double best = 0.0;
        double t = fabs(m11) * inv1;
        if (t >= best) { best = t; perm1 = 1; }
        t = fabs(m21) * inv2;
        if (t >= best) { best = t; perm1 = 2; }
    }
    if (perm1 == 2) {  // row swap (:174-183)
        double t = m21; m21 = m11; m11 = t;
        t = m22; m22 = m12; m12 = t;
    }
    {
        double t = 1.0 / m11;  // :187-192
        m21 *= t;
    }
    m22 = m22 - m21 * m12;  // :161-165 for column 2 (the pivot search there can only pick row 2)

    {
        double lo = 1.0e10, hi = 0.0;  // :195-207
        double t = fabs(m11);
        if (t < lo) lo = t;
        if (t > hi) hi = t;
        t = fabs(m22);
        if (t < lo) lo = t;
        if (t > hi) hi = t;
        if (lo / hi < 1.0e-10) return false;
    }

    // BidirectionalFilter (:210-237)
    double a = (perm1 == 2) ? v2 : v1;  // forward substitution with the row permutation
    double b = (perm1 == 2) ? v1 : v2;
    if (a != 0.0) b = b - a * m21;
    b = b / m22;
    a = (a - b * m12) / m11;

    // QuadraticMerge (:239-255)
    double den = 1.0 - (b * b);
    if (den == 0.0) return false;
    double k1 = (a - (a * b)) / den;
    if (fabs(k1) > 1.0) return false;
    double k2 = b;

    // FinishRecord (:257-269)
    if (k1 >= 1.0) k1 = 0.9999999999; else if (k1 <= -1.0) k1 = -0.9999999999;
    if (k2 >= 1.0) k2 = 0.9999999999; else if (k2 <= -1.0) k2 = -0.9999999999;
    double rec1 = (k2 * k1) + k1;
    double rec2 = k2;

    // MatrixFilter (:285-305)
    double n2 = -rec2, n1 = -rec1;
    double den2 = 1.0 - (n2 * n2);
    double p11 = ((n2 * n1) + n1) / den2;
    d1 = 0.0 + p11 * 1.0;
    d2 = (0.0 + n1 * d1) + n2 * 1.0;
    return true;
}

// grid: x = channel, y = tile of 256 frames (strided if the channel has more tiles than gridDim.y)
__global__ void __launch_bounds__(kP1Threads)
gc_coef_frames_kernel(const int16_t *__restrict__ pcm, GcChannelTable tab, double2 *__restrict__ records,
                      uint32_t *__restrict__ accept_mask, int frame_begin, int frame_end)
{
    __shared__ __align__(16) int16_t tile[8 + kP1TileSamples];  // tile[6..7] = two history samples, tile[8..] = frames

    const int ch = blockIdx.x;
    const int n = tab.n_samples[ch];
    const int n_frames = div_round_up(n, kGcFrameSamples);
    const int f_hi = min(frame_end, n_frames);
    const int16_t *src = pcm + tab.pcm_off[ch];
    double2 *rec = records + tab.rec_off[ch];
    uint32_t *mask = accept_mask + (tab.rec_off[ch] >> 5);

    for (int f0 = frame_begin + (int)blockIdx.y * kP1Threads; f0 < f_hi; f0 += (int)gridDim.y * kP1Threads) {
        const int64_t s0 = (int64_t)f0 * kGcFrameSamples;  // first sample of the tile; multiple of 8 -> 16 B aligned
        // coalesced 16-byte loads; samples at or beyond n read as zero (the reference zero-pads, :42-43)
        for (int v = threadIdx.x; v < kP1TileSamples / 8; v += kP1Threads) {
            int64_t s = s0 + (int64_t)v * 8;
            uint4 q = make_uint4(0, 0, 0, 0);
            if (s < n) {
                q = __ldg(reinterpret_cast<const uint4 *>(src + s));
                int valid = (int)min((int64_t)8, (int64_t)n - s);
                if (valid < 8) {
                    uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        if (2 * i >= valid) w[i] = 0;
                        else if (2 * i + 1 >= valid) w[i] &= 0xFFFFu;
                    }
                    q = make_uint4(w[0], w[1], w[2], w[3]);
                }
            }
            *reinterpret_cast<uint4 *>(&tile[8 + v * 8]) = q;
        }
        if (threadIdx.x < 2) {
            int64_t s = s0 - 2 + threadIdx.x;
            tile[6 + threadIdx.x] = (s >= 0 && s < n) ? src[s] : (int16_t)0;
        }
        __syncthreads();

        const int f = f0 + threadIdx.x;
        bool ok = false;
        double d1 = 0.0, d2 = 0.0;
        if (f < f_hi) {
            // 16 samples = 8 aligned 32-bit words at byte offset 28*t + 12: stride of 7 words -> conflict free
            const uint32_t *w = reinterpret_cast<const uint32_t *>(&tile[6 + threadIdx.x * kGcFrameSamples]);
            int32_t x[16];
#pragma unroll
            for (int i = 0; i < 8; i++) {
                uint32_t u = w[i];
                x[2 * i] = (int32_t)(int16_t)(u & 0xFFFFu);
                x[2 * i + 1] = (int32_t)(int16_t)(u >> 16);
            }
            ok = gc_frame_direct(x, d1, d2);
            rec[f] = make_double2(d1, d2);
        }
        uint32_t bits = __ballot_sync(0xFFFFFFFFu, ok);
        if ((threadIdx.x & 31) == 0 && f < f_hi) mask[f >> 5] = bits;
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------------
// phase 2: ordered mean + three split/refine generations, one warp per channel
// ---------------------------------------------------------------------------------------------------------

struct Centroid {
    double e0, e1, e2;  // ContrastVectors' val1, val2, val3 for this centroid (:338-340)
};

// FinishRecord(double[], double[]) (:271-283)
__device__ __forceinline__ void gc_finish(double k1, double k2, double &o1, double &o2)
{
    if (k1 >= 1.0) k1 = 0.9999999999; else if (k1 <= -1.0) k1 = -0.9999999999;
    if (k2 >= 1.0) k2 = 0.9999999999; else if (k2 <= -1.0) k2 = -0.9999999999;
    o1 = (k2 * k1) + k1;
    o2 = k2;
}

// MergeFinishRecord (:307-333) for a 3-vector src -> centroid (1, o1, o2)
__device__ __forceinline__ void gc_centroid_from_mean(double s0, double s1, double s2, double &o1, double &o2)
{
    double err = s0;
    // i = 1
    double acc = 0.0;
    double t1 = (err > 0.0) ? (-(acc + s1) / err) : 0.0;
    double k1 = t1;
    err *= 1.0 - (t1 * t1);
    // i = 2
    acc = 0.0;
    acc += t1 * s1;
    double t2 = (err > 0.0) ? (-(acc + s2) / err) : 0.0;
    double k2 = t2;
    // (dst[1] += dst[2]*dst[1] and the last err update do not reach the output)
    gc_finish(k1, k2, o1, o2);
}

// (short) rounding of :94-108; Math.Round is half-to-even = rint.
__device__ __forceinline__ int16_t gc_quantise_coef(double v)
{
    double d = -v * 2048.0;
    if (d > 0.0) return d > 32767.0 ? (int16_t)32767 : (int16_t)__double2int_rn(d);
    if (d < -32768.0) return (int16_t)-32768;
    if (d != d) return 0;
    return (int16_t)__double2int_rn(d);
}

// ---- phase 2 as a producer/consumer CTA: one CTA of kRefineWarps warps per channel -----------------------------
// The ordered fp64 sums are a serial chain (8.3 cycles per add), everything else - loading the records, the nearest
// centroid search, sorting a block of 32 records into per-bucket queues - is parallel work.  At 1024 channels one
// warp per channel leaves most of the machine idle and each channel pays for both in sequence, so the work is split
// and software-pipelined over CHUNKS of kRefineProducers blocks with one CTA barrier per chunk (no polling):
//   warps 1..P (producers) classify one block of 32 records each and append every record to ITS bucket's queue in
//              the chunk's shared-memory buffer (rank = number of earlier records of the block in the same bucket,
//              from a ballot: record order is preserved inside a bucket);
//   warp 0     (consumer) meanwhile walks the PREVIOUS chunk's blocks in order and lane (bucket, component) adds ONLY
//              its bucket's records, in record order - exactly the reference's sequence of additions.
// W warps per CTA = 1 consumer + (W - 1) producers.  W = 4 keeps eight CTAs per SM (64 registers, 8 x 26 KB of shared
// memory), which holds all 1024 channels of the headline batch at once on H100's 132 SMs (seven would leave 100 channels
// for a second wave); W = 8 (7 producers, 61 KB of queues) is kept for experiments with small batches
// (VGB_REFINE_WIDE_LIMIT).

struct __align__(16) RefineSlot {
    double2 q[8 * 33];    // per-bucket queues of one block of 32 records, bucket b at q + b * refine_row(NB): 33 entries per
                          // row with 8 buckets (the 16 accumulator lanes (bucket, comp) read entry j of all buckets at once,
                          // 528-byte rows put them in 16 distinct bank pairs), 66 / 132 / 264 with 4 / 2 / 1 buckets - room
                          // for the longer padding the consumer's wider steps need when few buckets share the block
    int32_t count[8];     // records per bucket (buckets the pass does not use stay 0)
};
// queue row length and consumer step (entries added per loop iteration; queues are padded to a multiple of it with -0.0)
__host__ __device__ constexpr int refine_row(int nb) { return nb >= 8 ? 33 : (nb == 4 ? 66 : (nb == 2 ? 132 : 264)); }
__host__ __device__ constexpr int refine_step(int nb) { return nb >= 4 ? 4 : (nb == 2 ? 8 : 16); }

template <int W>
struct RefineShared {
    RefineSlot slot[2][W - 1];             // double-buffered chunks
    double cent[8][3];                      // centroids (1, c1, c2)
    double econst[8][3];                    // per-centroid constants of ContrastVectors (:338-340), refreshed every pass
};

// all kRefineWarps warps, once per chunk; PTX named barrier so that the two code paths may use different instructions
template <int W>
__device__ __forceinline__ void refine_chunk_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(W * 32) : "memory"); }

// consumer side of one pass: ordered accumulation (:382-386 / :67-72).  Lane (bucket*2 + comp) walks its bucket's queue
// of every block in block order - a pure DADD chain over exactly the bucket's records, in record order.
struct RefineSum { double acc; int hits; };
template <int NB, int W>
__device__ __forceinline__ RefineSum gc_refine_consume(int lane, int n_blocks, int n_chunks, RefineShared<W> &sh)
{
    constexpr int P = W - 1;
    constexpr int STEP = refine_step(NB), ROW = refine_row(NB);
    const int my_bucket = (lane >> 1) & 7, my_comp = lane & 1;
    double a = 0.0;
    int h = 0;
    refine_chunk_barrier<W>();  // chunk 0 classified
    for (int c = 1; c <= n_chunks; c++) {
        const int first = (c - 1) * P;
        for (int j = 0; j < P && first + j < n_blocks; j++) {
            const RefineSlot &slot = sh.slot[(c - 1) & 1][j];
            const int n_mine = (lane < 16 && my_bucket < NB) ? slot.count[my_bucket] : 0;
            const double *col = reinterpret_cast<const double *>(slot.q + (my_bucket < NB ? my_bucket : 0) * ROW) + my_comp;
            // STEP queue entries per iteration (the producers pad every queue to a multiple of STEP with -0.0, the additive
            // identity): loads issued together, then the bare DADD chain - the shared-memory latency and the loop overhead are
            // paid once per STEP records, so the passes with one or two long queues (STEP 16 / 8) run close to the 8.3 cycles
            // a dependent add costs.  The trip count differs per lane; lanes whose bucket is done simply drop out.
            const int n_pad = (n_mine + STEP - 1) / STEP * STEP;
            for (int j0 = 0; j0 < n_pad; j0 += STEP) {
                double v[STEP];
#pragma unroll
                for (int i = 0; i < STEP; i++) v[i] = col[2 * (j0 + i)];
#pragma unroll
                for (int i = 0; i < STEP; i++) a += v[i];
            }
            h += n_mine;
        }
        refine_chunk_barrier<W>();
    }
    return RefineSum{a, h};
}

// One pass over all records of a channel with COUNT centroids (COUNT == 0: the plain ordered mean of :63-76, every
// record goes to bucket 0), executed by the whole CTA.  On return, in warp 0, lane (bucket*2 + comp) with
// bucket < max(COUNT,1) holds the ordered sum of that component over the bucket's records in `acc` and the record
// count in `hits`.
template <int COUNT, int W>
__device__ __forceinline__ void gc_refine_pass(int warp, int lane, int n_frames, int n_blocks, const double2 *__restrict__ rec,
                                               const uint32_t *__restrict__ mask, RefineShared<W> &sh, double &acc, int &hits)
{
    constexpr int NB = COUNT > 0 ? COUNT : 1;
    constexpr int P = W - 1;
    constexpr int STEP = refine_step(NB), ROW = refine_row(NB);
    const uint32_t lanes_below = (1u << lane) - 1u;
    const int p = warp - 1;                              // producer index (warp 0: unused)
    const int n_chunks = (n_blocks + P - 1) / P;

    auto fetch = [&](int b, double2 &r, uint32_t &okbits) {
        r = make_double2(0.0, 0.0);
        okbits = 0;
        if (warp > 0 && b < n_blocks) {
            okbits = mask[b];
            const int f = b * 32 + lane;
            if (f < n_frames) r = rec[f];
        }
    };
    // producer: classify block b (nearest centroid, parallel over its 32 records) into `slot`
    auto stage = [&](int b, double2 r, uint32_t okbits, RefineSlot &slot) {
        const bool ok = ((okbits >> lane) & 1u) && (b * 32 + lane < n_frames);
        int pick = 0;
        if (COUNT > 1) {
            // ContrastVectors (:335-342); its `val` is r.x and (-rec1*val - rec2) is r.y (DESIGN.md §5.1)
            const double ta = 2.0 * r.x, tb = 2.0 * r.y;
            // all distances first (independent), then a tournament instead of the reference's sequential scan
            // (:373-381: `if (tempVal < value)`, value starting at 1.0e30): a later candidate replaces an earlier one
            // only when strictly smaller, so ties keep the lower index - the same first-minimum rule, depth log2(NB)
            double d[NB];
            int idx[NB];
#pragma unroll
            for (int i = 0; i < NB; i++) {
                const double di = sh.econst[i][0] + (ta * sh.econst[i][1]) + (tb * sh.econst[i][2]);  // smem broadcast
                d[i] = di < 1.0e30 ? di : __longlong_as_double(0x7FF0000000000000ll);  // never wins (also NaN), as in the scan
                idx[i] = i;
            }
#pragma unroll
            for (int step = 1; step < NB; step *= 2) {
#pragma unroll
                for (int i = 0; i + step < NB; i += 2 * step) {
                    const bool right = d[i + step] < d[i];
                    d[i] = right ? d[i + step] : d[i];
                    idx[i] = right ? idx[i + step] : idx[i];
                }
            }
            pick = d[0] < 1.0e30 ? idx[0] : 0;  // nothing below the initial 1.0e30: the index stays 0
        }
        // lanes that picked the same bucket find each other with ONE match instead of a ballot per bucket; records that
        // were not accepted form their own group (key NB) and are not queued
        if (lane < NB) slot.count[lane] = 0;
        const uint32_t mine = __match_any_sync(0xFFFFFFFFu, ok ? pick : NB);
        __syncwarp();
        if (ok) {
            const int rank = __popc(mine & lanes_below);
            if (rank == 0) slot.count[pick] = __popc(mine);  // the group's first lane publishes its size
            slot.q[pick * ROW + rank] = r;
        }
        __syncwarp();
        {   // pad every queue to a multiple of STEP entries with -0.0 (lane = bucket * STEP + i; NB * STEP <= 32)
            const int bucket = lane / STEP, i = lane % STEP;
            if (bucket < NB) {
                const int c = slot.count[bucket];
                if (i < ((STEP - (c % STEP)) % STEP)) slot.q[bucket * ROW + c + i] = make_double2(-0.0, -0.0);
            }
        }
    };
    acc = 0.0;
    hits = 0;
    // Records stream from HBM once per pass (1.6 MB per channel, no reuse): a producer's loads are issued kDepth of
    // its blocks ahead of their use to cover DRAM latency; ring indices are compile-time.
    constexpr int kDepth = 4;
    double2 ring_r[kDepth];
    uint32_t ring_ok[kDepth];
#pragma unroll
    for (int k = 0; k < kDepth; k++) fetch(p + k * P, ring_r[k], ring_ok[k]);

    if (warp == 0) {
        // consumer: deliberately small, rolled code (it is the critical path and must stay in the instruction cache
        // next to the producers' large unrolled loop); inlined so that `sh` stays a shared-window address
        const RefineSum sum = gc_refine_consume<NB, W>(lane, n_blocks, n_chunks, sh);
        acc = sum.acc;
        hits = sum.hits;
        return;
    }
    for (int c0 = 0; c0 <= n_chunks; c0 += kDepth) {  // one extra step drains the pipeline
#pragma unroll
        for (int k = 0; k < kDepth; k++) {
            const int c = c0 + k;
            if (c > n_chunks) break;
            const int b = c * P + p;
            if (b < n_blocks) stage(b, ring_r[k], ring_ok[k], sh.slot[c & 1][p]);
            fetch(b + kDepth * P, ring_r[k], ring_ok[k]);
            refine_chunk_barrier<W>();  // chunk c is classified, chunk c-1 is summed: the two buffers swap roles
        }
    }
}

// The refinement of one channel per CTA.  kTap: warp 0 also writes the centroids (c1, c2) and bucket counts every pass
// leaves to tap_cent [ch][7][8][2] / tap_hits [ch][7][8] (vgb_gcadpcm_debug_refine_trace); the encode path instantiates
// it with kTap = false, which compiles to the same code as without the tap.
template <int W, bool kTap>
__device__ __forceinline__ void gc_coef_refine(GcChannelTable tab, const double2 *__restrict__ records,
                                               const uint32_t *__restrict__ accept_mask, int16_t *__restrict__ coefs_out,
                                               double *__restrict__ tap_cent, int32_t *__restrict__ tap_hits)
{
    extern __shared__ __align__(16) unsigned char refine_smem[];
    RefineShared<W> &sh = *reinterpret_cast<RefineShared<W> *>(refine_smem);
    constexpr int kRefineProducers = W - 1;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ch = blockIdx.x;
    if (ch >= tab.n_channels) return;

    double (*best)[3] = sh.cent;
    const int n_frames = div_round_up(tab.n_samples[ch], kGcFrameSamples);
    const int n_blocks = (n_frames + 31) >> 5;
    const double2 *rec = records + tab.rec_off[ch];
    const uint32_t *mask = accept_mask + (tab.rec_off[ch] >> 5);

    if (threadIdx.x < 8) { best[threadIdx.x][0] = 1.0; best[threadIdx.x][1] = 0.0; best[threadIdx.x][2] = 0.0; }
    if (threadIdx.x < 2 * kRefineProducers * 8) sh.slot[threadIdx.x / (kRefineProducers * 8)][(threadIdx.x / 8) % kRefineProducers].count[threadIdx.x & 7] = 0;
    __syncthreads();

    // pass 0 is the plain ordered mean (:63-76); passes 1..6 are the FilterRecords rounds (:79-91): split, then two
    // rounds of reassign + average with 2, 4, 8 centroids.
    int count = 1;
    for (int pass = 0; pass < 7; pass++) {
        if (pass == 1 || pass == 3 || pass == 5) {
            // split (:82-89): new centroid = (0.01 * (0,-1,0)) + old
            if (warp == 0 && lane < count) {
                best[count + lane][0] = (0.01 * 0.0) + best[lane][0];
                best[count + lane][1] = (0.01 * -1.0) + best[lane][1];
                best[count + lane][2] = (0.01 * 0.0) + best[lane][2];
            }
            count *= 2;
            __syncthreads();
        }
        if (warp == 0 && lane < count) {
            const double a0 = best[lane][0], a1 = best[lane][1], a2 = best[lane][2];
            sh.econst[lane][0] = (a0 * a0) + (a1 * a1) + (a2 * a2);
            sh.econst[lane][1] = (a0 * a1) + (a1 * a2);
            sh.econst[lane][2] = a0 * a2;
        }
        __syncthreads();
        double acc;
        int hits;
        if (pass == 0) gc_refine_pass<0, W>(warp, lane, n_frames, n_blocks, rec, mask, sh, acc, hits);
        else if (count == 2) gc_refine_pass<2, W>(warp, lane, n_frames, n_blocks, rec, mask, sh, acc, hits);
        else if (count == 4) gc_refine_pass<4, W>(warp, lane, n_frames, n_blocks, rec, mask, sh, acc, hits);
        else gc_refine_pass<8, W>(warp, lane, n_frames, n_blocks, rec, mask, sh, acc, hits);

        if (warp == 0) {
            // divide (:73-74 / :388-391) and rebuild the centroids (:76 / :393-394)
            double mean;
            if (pass == 0) mean = acc / (double)hits;  // 0/0 = NaN for a silent channel, as in the reference (A.19)
            else mean = hits > 0 ? acc / (double)hits : acc;
            const double m1 = __shfl_sync(0xFFFFFFFFu, mean, (lane & 7) * 2);
            const double m2 = __shfl_sync(0xFFFFFFFFu, mean, (lane & 7) * 2 + 1);
            const int h = __shfl_sync(0xFFFFFFFFu, hits, (lane & 7) * 2);
            if (lane < count) {
                const double m0 = (pass == 0) ? 1.0 : (h > 0 ? 1.0 : 0.0);  // sum of h ones divided by h
                double o1, o2;
                gc_centroid_from_mean(m0, m1, m2, o1, o2);
                best[lane][0] = 1.0;
                best[lane][1] = o1;
                best[lane][2] = o2;
            }
            if (kTap && lane < 8) {  // each lane its own centroid: just written above, or untouched by this pass
                const int64_t at = ((int64_t)ch * 7 + pass) * 8 + lane;
                tap_cent[2 * at] = best[lane][1];
                tap_cent[2 * at + 1] = best[lane][2];
                tap_hits[at] = h;
            }
        }
        __syncthreads();  // the next pass classifies against the new centroids
    }

    if (threadIdx.x < 16) coefs_out[(int64_t)ch * 16 + threadIdx.x] = gc_quantise_coef(best[threadIdx.x >> 1][1 + (threadIdx.x & 1)]);
}

template <int W>
__global__ void __launch_bounds__(W * 32, W == 4 ? 8 : 3)  // W = 4: 8 CTAs per SM, 1024 channels are resident at once on 132 SMs
gc_coef_refine_kernel(GcChannelTable tab, const double2 *__restrict__ records, const uint32_t *__restrict__ accept_mask,
                      int16_t *__restrict__ coefs_out)
{
    gc_coef_refine<W, false>(tab, records, accept_mask, coefs_out, nullptr, nullptr);
}

template <int W>
__global__ void __launch_bounds__(W * 32, W == 4 ? 8 : 3)
gc_coef_refine_tap_kernel(GcChannelTable tab, const double2 *__restrict__ records, const uint32_t *__restrict__ accept_mask,
                          int16_t *__restrict__ coefs_out, double *__restrict__ tap_cent, int32_t *__restrict__ tap_hits)
{
    gc_coef_refine<W, true>(tab, records, accept_mask, coefs_out, tap_cent, tap_hits);
}

// ---------------------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------------------
void launch_gc_coef_frames(const int16_t *pcm, const GcChannelTable &tab, double2 *records, uint32_t *mask,
                           int max_frames, int frame_begin, int frame_end, cudaStream_t stream)
{
    if (tab.n_channels <= 0 || max_frames <= 0) return;
    int hi = frame_end < max_frames ? frame_end : max_frames;
    if (hi <= frame_begin) return;
    int tiles = (hi - frame_begin + kP1Threads - 1) / kP1Threads;
    if (tiles > 65535) tiles = 65535;
    dim3 grid((unsigned)tab.n_channels, (unsigned)tiles);
    gc_coef_frames_kernel<<<grid, kP1Threads, 0, stream>>>(pcm, tab, records, mask, frame_begin, frame_end);
}

void launch_gc_coef_refine(const GcChannelTable &tab, const double2 *records, const uint32_t *mask,
                           int16_t *coefs_out, cudaStream_t stream)
{
    if (tab.n_channels <= 0) return;
    static int wide_limit = -1;  // batches up to this many channels take the 8-warp CTA (0: never - it measured no faster)
    if (wide_limit < 0) {
        wide_limit = 0;
        if (const char *env = std::getenv("VGB_REFINE_WIDE_LIMIT")) wide_limit = std::atoi(env);  // tuning knob
    }
    if (tab.n_channels <= wide_limit) {
        raise_dynamic_smem(gc_coef_refine_kernel<8>, sizeof(RefineShared<8>));
        gc_coef_refine_kernel<8><<<tab.n_channels, 8 * 32, sizeof(RefineShared<8>), stream>>>(tab, records, mask, coefs_out);
    } else {
        raise_dynamic_smem(gc_coef_refine_kernel<4>, sizeof(RefineShared<4>));
        gc_coef_refine_kernel<4><<<tab.n_channels, 4 * 32, sizeof(RefineShared<4>), stream>>>(tab, records, mask, coefs_out);
    }
}

void launch_gc_coef_refine_tap(const GcChannelTable &tab, const double2 *records, const uint32_t *mask, int16_t *coefs_out,
                               int warps, double *tap_cent, int32_t *tap_hits, cudaStream_t stream)
{
    if (tab.n_channels <= 0) return;
    if (warps == 8) {
        raise_dynamic_smem(gc_coef_refine_tap_kernel<8>, sizeof(RefineShared<8>));
        gc_coef_refine_tap_kernel<8><<<tab.n_channels, 8 * 32, sizeof(RefineShared<8>), stream>>>(tab, records, mask, coefs_out,
                                                                                                  tap_cent, tap_hits);
    } else {
        raise_dynamic_smem(gc_coef_refine_tap_kernel<4>, sizeof(RefineShared<4>));
        gc_coef_refine_tap_kernel<4><<<tab.n_channels, 4 * 32, sizeof(RefineShared<4>), stream>>>(tab, records, mask, coefs_out,
                                                                                                  tap_cent, tap_hits);
    }
}

}  // namespace vgb
