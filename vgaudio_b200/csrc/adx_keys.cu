// adx_keys.cu — the CRI ADX key search of VGAudio.Tools/CrackAdx/GuessAdx.cs on sm_90a (H100).
//
// GuessAdx recovers the LCG key (seed, mult, inc) of revision 8 / 9 .adx files from the files alone: for every scale
// index (0..0xFFF) and every file, TryScale (:160-189) takes seed = (Scales[StartFrame] ^ index) & (MaxSeed - 1) and
// walks every (mult, inc) of the revision's lists over the file's frame scales from StartFrame, stopping at the first
// frame whose scale disagrees with the key stream under the validation mask.  A candidate that walks every frame goes
// to FindStartingKey (:191-215), which winds the key back to frame 0, and to AddKey (:126-158), which keeps it when
// KeyIsValid (:217-229) holds on every file.
//
// The search is integer-only and reads nothing but the scanned file's frame words, which sit in shared memory (up to
// kAdxKeyStage frames from StartFrame; a candidate that outlives them continues from global memory, which only keys
// that are nearly right ever do).  A warp takes one warp-uniform (index, mult) and 32 increments, one per lane, and
// walks frames while any lane is alive: a frame passes with probability 1/4 (revision 8) or 1/2 (revision 9), so a
// warp walks a handful of frames per 32 candidates.  The counts the debug call reports (candidates tried, frame steps,
// full matches) come from the same ballots that drive the loop.  A key that walks every frame is checked on every file
// once (a device table of tried keys, like AddKey's TriedKeys), by the whole warp.
//
// FindStartingKey by jump-ahead: after StartFrame steps the key stream is x = (A * seed0 + B) mod 2^15, with A odd,
// so the seed0 whose state equals `seed` under MaxSeed - 1 is A^-1 * (seed - B) under the same mask - the only one, so
// it is also the first in the reference's ascending seed order.  Revision 8 keeps it only if it is in the prime list.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace vgb {

namespace {

constexpr int kKeyWarps = 8;  // warps per CTA of the search

// ((x ^ w) & (w >> 16)) != 0: the frame's scale disagrees with key stream value x (see AdxKeyFileDev)
__device__ __forceinline__ bool frame_fails(uint32_t x, uint32_t w) { return ((x ^ w) & (w >> 16)) != 0u; }

__device__ __forceinline__ bool seed_listed(const AdxKeySearch &a, uint32_t s) { return (__ldg(a.seed_bits + (s >> 5)) >> (s & 31u)) & 1u; }

// KeyIsValid (:217-229) on every file of the search, from frame 0 with the key's seed, by the whole warp: lane L walks
// the L-th 32nd of each file's frames from the key stream value there (jump-ahead), its loads eight at a time
__device__ bool key_valid_everywhere(const AdxKeySearch &a, uint32_t seed, uint32_t mult, uint32_t inc, int lane)
{
    for (int f = 0; f < a.n_files; f++) {
        const AdxKeyFileDev g = a.files[f];
        const uint32_t *w = a.words + g.word_off;
        const int per = (g.frames + 31) / 32, i0 = min(lane * per, g.frames), i1 = min(i0 + per, g.frames);
        uint32_t x = (uint32_t)adx_key_at((int)seed, (int)mult, (int)inc, (uint32_t)i0);
        bool bad = false;
        for (int i = i0; i < i1 && !bad; i += 8) {
            uint32_t v[8];
#pragma unroll
            for (int k = 0; k < 8; k++) v[k] = i + k < i1 ? __ldg(w + i + k) : 0u;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                bad = bad || frame_fails(x, v[k]);
                x = (x * mult + inc) & 0x7fffu;
            }
        }
        if (__any_sync(0xffffffffu, bad)) return false;
    }
    return true;
}

// AddKey's TriedKeys on the device: true for the first caller with this key.  A full table only stops deduplicating
// (the host dedups again), so the result never depends on its size.
__device__ bool first_try(const AdxKeySearch &a, uint32_t seed, uint32_t mult, uint32_t inc)
{
    const unsigned long long k = ((unsigned long long)seed << 32 | (unsigned long long)mult << 16 | inc) + 1ull;
    uint32_t h = (uint32_t)((k * 0x9E3779B97F4A7C15ull) >> 40) & (kAdxKeyTried - 1);
    for (int probe = 0; probe < 64; probe++, h = (h + 1) & (kAdxKeyTried - 1)) {
        const unsigned long long old = atomicCAS(a.tried + h, 0ull, k);
        if (old == 0ull) return true;
        if (old == k) return false;
    }
    return true;
}

__global__ void __launch_bounds__(kKeyWarps * 32) adx_key_search_kernel(const AdxKeySearch a)
{
    extern __shared__ uint32_t s_words[];
    const AdxKeyFileDev f = a.files[a.file];
    const int n_walk = f.frames - f.start;
    const int staged = min(n_walk, kAdxKeyStage);
    const uint32_t *g_words = a.words + f.word_off + f.start;
    for (int j = threadIdx.x; j < staged; j += blockDim.x) s_words[j] = g_words[j];
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long tried = 0, steps = 0, matches = 0;
    const int64_t n_items = (int64_t)a.n_index * a.n_mult;
    for (int64_t it = (int64_t)blockIdx.x * kKeyWarps + warp; it < n_items; it += (int64_t)gridDim.x * kKeyWarps) {
        const int index = a.index0 + (int)(it / a.n_mult);
        const uint32_t mult = (uint32_t)__ldg(a.mults + (it % a.n_mult));
        const uint32_t seed = ((uint32_t)f.first_scale ^ (uint32_t)index) & a.seed_mask;
        if (f.start == 0 && a.check_seed && !seed_listed(a, seed)) continue;  // :163
        for (int c0 = 0; c0 < a.n_inc; c0 += 32) {
            const bool valid = c0 + lane < a.n_inc;
            const uint32_t inc = valid ? (uint32_t)__ldg(a.incs + c0 + lane) : 0u;
            uint32_t x = seed;
            bool alive = valid;
            tried += (unsigned)__popc(__ballot_sync(0xffffffffu, valid));
            int j = 0;
            unsigned live;
            while (j < staged && (live = __ballot_sync(0xffffffffu, alive)) != 0u) {
                steps += (unsigned)__popc(live);
                alive = alive && !frame_fails(x, s_words[j]);
                x = (x * mult + inc) & 0x7fffu;
                j++;
            }
            while (j < n_walk && (live = __ballot_sync(0xffffffffu, alive)) != 0u) {  // past the staged frames: rare
                steps += (unsigned)__popc(live);
                alive = alive && !frame_fails(x, __ldg(g_words + j));
                x = (x * mult + inc) & 0x7fffu;
                j++;
            }
            unsigned found = __ballot_sync(0xffffffffu, alive);
            matches += (unsigned)__popc(found);
            if (!found) continue;
            // FindStartingKey (:191-215)
            uint32_t seed0 = seed;
            if (alive && f.start > 0) {
                uint32_t A, B;
                adx_key_jump((int)mult, (int)inc, (uint32_t)f.start, A, B);
                uint32_t inv = A;  // A odd: Newton's iteration doubles the correct low bits, 3 -> 24
                for (int k = 0; k < 3; k++) inv *= 2u - A * inv;
                seed0 = (inv * (seed - B)) & a.seed_mask;
                if (a.check_seed && !seed_listed(a, seed0)) alive = false;
            }
            // AddKey (:126-136): each new key is validated on every file by the whole warp, one key after another
            found = __ballot_sync(0xffffffffu, alive);
            while (found) {
                const int src = __ffs(found) - 1;
                found &= found - 1;
                const uint32_t ks = __shfl_sync(0xffffffffu, seed0, src), ki = __shfl_sync(0xffffffffu, inc, src);
                const bool fresh = __shfl_sync(0xffffffffu, lane == 0 ? first_try(a, ks, mult, ki) : false, 0);
                if (!fresh || !key_valid_everywhere(a, ks, mult, ki, lane)) continue;
                if (lane == 0) {
                    const unsigned long long at = atomicAdd(a.n_hits, 1ull);
                    if (at < a.cap) a.hits[at] = AdxKeyHit{(int32_t)ks, (int32_t)mult, (int32_t)ki};
                }
            }
        }
    }
    if (lane == 0) {  // tried, steps and matches are warp-uniform
        atomicAdd(a.stats + 0, tried);
        atomicAdd(a.stats + 1, steps);
        atomicAdd(a.stats + 2, matches);
    }
}

__global__ void __launch_bounds__(256) adx_byte_diff_kernel(const uint8_t *__restrict__ a, const int64_t *__restrict__ a_off,
                                                            const uint8_t *__restrict__ b, const int64_t *__restrict__ b_off,
                                                            const int32_t *__restrict__ n, int32_t *__restrict__ out)
{
    const int r = blockIdx.x;
    const uint8_t *x = a + a_off[r], *y = b + b_off[r];
    const int n_short = n[2 * r], n_full = n[2 * r + 1];
    int d_short = 0, d_full = 0;
    for (int i = threadIdx.x; i < n_full; i += blockDim.x) {
        const int d = x[i] != y[i];
        d_full += d;
        d_short += i < n_short ? d : 0;
    }
    __shared__ int s[2][8];
    for (int o = 16; o; o >>= 1) {
        d_short += __shfl_xor_sync(0xffffffffu, d_short, o);
        d_full += __shfl_xor_sync(0xffffffffu, d_full, o);
    }
    if ((threadIdx.x & 31) == 0) { s[0][threadIdx.x >> 5] = d_short; s[1][threadIdx.x >> 5] = d_full; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int ts = 0, tf = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) { ts += s[0][w]; tf += s[1][w]; }
        out[2 * r] = ts;
        out[2 * r + 1] = tf;
    }
}

}  // namespace

cudaError_t launch_adx_key_search(const AdxKeySearch &a, int frames_after_start, cudaStream_t stream)
{
    const int64_t items = (int64_t)a.n_index * a.n_mult;
    if (items <= 0 || a.n_inc <= 0 || frames_after_start <= 0) return cudaSuccess;
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    const size_t smem = (size_t)std::min(frames_after_start, kAdxKeyStage) * sizeof(uint32_t);
    const int64_t ctas = std::min<int64_t>((items + kKeyWarps - 1) / kKeyWarps, (int64_t)sms * 8);
    adx_key_search_kernel<<<(unsigned)ctas, kKeyWarps * 32, smem, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_adx_byte_diff(const uint8_t *a, const int64_t *a_off, const uint8_t *b, const int64_t *b_off, const int32_t *n,
                                 int n_rows, int32_t *out, cudaStream_t stream)
{
    if (n_rows <= 0) return cudaSuccess;
    adx_byte_diff_kernel<<<(unsigned)n_rows, 256, 0, stream>>>(a, a_off, b, b_off, n, out);
    return cudaGetLastError();
}

}  // namespace vgb
