// interleave.cu — block (de)interleave of channel payloads on sm_90a (H100).
//
// Replaces InterleaveExtensions.Interleave / DeInterleave (Utilities/Interleave.cs:9-166), the byte shuffles the
// container writers / readers run right after / before the codec path (SURVEY.md 8f rank 2): DspWriter / BrstmWriter
// interleave the channels' ADPCM in 0x2000-byte blocks, AdxWriter in frame_size-byte blocks (AdxWriter.cs:131), the WAV
// reader de-interleaves 2-byte samples (WaveReader.cs:47).  Pure data movement: every byte is read once and written
// once, so the kernel is HBM-bound by construction; it moves the widest vector (16/8/4/2/1 bytes) that divides the
// block size, the channel sizes and the strides, four independent elements per thread (loads first, stores after),
// fully coalesced on the interleaved side and in block-sized runs on the planar side; 32-bit index arithmetic per item.
//
// Semantics (identical for both directions, :17-23): blocks of `interleave` bytes per channel; the LAST block of the
// input / output may be shorter (size - (blocks-1)*interleave); only min(inBlocks, outBlocks) blocks are copied and
// in a block only min(currentInputBlock, currentOutputBlock) bytes per channel; the rest of the output stays zero.
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace vgb {

namespace {

struct Shape {
    int64_t in_size, out_size, interleave;  // bytes per channel / per block
    int64_t in_blocks, out_blocks, last_in, last_out, blocks_to_copy;
    int count;
};

__host__ __device__ inline Shape make_shape(int count, int64_t in_size, int64_t interleave, int64_t out_size)
{
    Shape s;
    s.count = count; s.in_size = in_size; s.out_size = out_size; s.interleave = interleave;
    s.in_blocks = (in_size + interleave - 1) / interleave;
    s.out_blocks = (out_size + interleave - 1) / interleave;
    s.last_in = in_size - (s.in_blocks - 1) * interleave;
    s.last_out = out_size - (s.out_blocks - 1) * interleave;
    s.blocks_to_copy = s.in_blocks < s.out_blocks ? s.in_blocks : s.out_blocks;
    return s;
}

constexpr int kIlvThreads = 256, kIlvIter = 4;  // elements per thread: independent loads in flight

// planar [count][in_size] -> interleaved [out_size * count].  A CTA works on kIlvThreads * kIlvIter consecutive output
// elements of ONE item, so all index arithmetic is 32-bit (an item's payload is < 2 GiB) and the item offset is added
// once; one output element of width sizeof(V) per thread and iteration, consecutive threads on consecutive elements.
template <typename V>
__global__ void __launch_bounds__(kIlvThreads)
interleave_kernel(const uint8_t *__restrict__ in, int64_t in_channel_stride, int64_t in_item_stride, uint8_t *__restrict__ out,
                  int64_t out_item_stride, uint32_t blocks_per_item, Shape sh)
{
    const uint32_t item = blockIdx.x / blocks_per_item, bx = blockIdx.x - item * blocks_per_item;
    const uint32_t per_item = (uint32_t)(sh.out_size * sh.count / (int64_t)sizeof(V));
    const uint32_t full_block = (uint32_t)(sh.interleave * sh.count), ilv = (uint32_t)sh.interleave;
    const uint32_t out_blocks = (uint32_t)sh.out_blocks, in_blocks = (uint32_t)sh.in_blocks, to_copy = (uint32_t)sh.blocks_to_copy;
    const uint32_t last_out = (uint32_t)sh.last_out, last_in = (uint32_t)sh.last_in;
    const uint8_t *src = in + (int64_t)item * in_item_stride;
    uint8_t *dst = out + (int64_t)item * out_item_stride;
    V v[kIlvIter];
    uint32_t o[kIlvIter];
#pragma unroll
    for (int k = 0; k < kIlvIter; k++) {
        const uint32_t e = (bx * kIlvIter + k) * kIlvThreads + threadIdx.x;
        o[k] = e * (uint32_t)sizeof(V);                         // byte offset inside the item's output
        v[k] = V{};
        if (e < per_item) {
            const uint32_t b = o[k] / full_block;               // block index (all earlier blocks are full)
            const uint32_t r = o[k] - b * full_block;
            const uint32_t cur_out = b == out_blocks - 1 ? last_out : ilv;
            const uint32_t cur_in = b == in_blocks - 1 ? last_in : ilv;
            const uint32_t ch = r / cur_out, off = r - ch * cur_out;
            if (b < to_copy && off < (cur_in < cur_out ? cur_in : cur_out))
                v[k] = *reinterpret_cast<const V *>(src + (int64_t)ch * in_channel_stride + (ilv * b + off));
        }
    }
#pragma unroll
    for (int k = 0; k < kIlvIter; k++)
        if (o[k] / (uint32_t)sizeof(V) < per_item) *reinterpret_cast<V *>(dst + o[k]) = v[k];
}

// interleaved [in_size * count] -> planar [count][out_size]; elements are walked in the order of the interleaved stream
// (one block of one channel, then the same block of the next channel): reads stay sequential, writes are block runs
template <typename V>
__global__ void __launch_bounds__(kIlvThreads)
deinterleave_kernel(const uint8_t *__restrict__ in, int64_t in_item_stride, uint8_t *__restrict__ out, int64_t out_channel_stride,
                    int64_t out_item_stride, uint32_t blocks_per_item, Shape sh)
{
    const uint32_t item = blockIdx.x / blocks_per_item, bx = blockIdx.x - item * blocks_per_item;
    const uint32_t per_item = (uint32_t)(sh.out_size / (int64_t)sizeof(V)) * (uint32_t)sh.count;
    const uint32_t ilv = (uint32_t)sh.interleave, count = (uint32_t)sh.count;
    const uint32_t block_elems = ilv / (uint32_t)sizeof(V), group = block_elems * count;
    const uint32_t out_blocks = (uint32_t)sh.out_blocks, in_blocks = (uint32_t)sh.in_blocks, to_copy = (uint32_t)sh.blocks_to_copy;
    const uint32_t last_out = (uint32_t)sh.last_out, last_in = (uint32_t)sh.last_in;
    const uint32_t last_elems = last_out / (uint32_t)sizeof(V);
    const uint8_t *src = in + (int64_t)item * in_item_stride;
    uint8_t *dst = out + (int64_t)item * out_item_stride;
    V v[kIlvIter];
    int64_t where[kIlvIter];
#pragma unroll
    for (int k = 0; k < kIlvIter; k++) {
        const uint32_t q = (bx * kIlvIter + k) * kIlvThreads + threadIdx.x;
        v[k] = V{};
        where[k] = -1;
        if (q < per_item) {
            uint32_t b = q / group, ch, off;
            if (b < out_blocks - 1) {
                const uint32_t r = q - b * group;
                ch = r / block_elems;
                off = (r - ch * block_elems) * (uint32_t)sizeof(V);
            } else {  // last output block: last_out bytes per channel
                b = out_blocks - 1;
                const uint32_t r = q - b * group;
                ch = r / last_elems;
                off = (r - ch * last_elems) * (uint32_t)sizeof(V);
            }
            const uint32_t cur_out = b == out_blocks - 1 ? last_out : ilv;
            const uint32_t cur_in = b == in_blocks - 1 ? last_in : ilv;
            if (b < to_copy && off < (cur_in < cur_out ? cur_in : cur_out))
                v[k] = *reinterpret_cast<const V *>(src + ((int64_t)ilv * b * count + cur_in * ch + off));
            where[k] = (int64_t)ch * out_channel_stride + (ilv * b + off);
        }
    }
#pragma unroll
    for (int k = 0; k < kIlvIter; k++)
        if (where[k] >= 0) *reinterpret_cast<V *>(dst + where[k]) = v[k];
}

// ---- TMA variant: the block shuffle as bulk copies -----------------------------------------------------------------------
// A block of one channel is a contiguous run on both sides, so the shuffle is a list of (source, destination, bytes)
// copies.  Here one elected thread per CTA moves them with the bulk-copy engine: cp.async.bulk global -> shared (completion
// on an mbarrier), cp.async.bulk shared -> global, a ring of kBulkStages buffers of kBulkChunk bytes, persistent CTAs
// striding over the chunk list.  No thread touches the data.  Eligible when every size, stride and address is a multiple
// of 16 bytes and the output is fully covered (in_size == out_size); selected with VGB_INTERLEAVE_TMA=1
// (tools/interleave_bench.py compares it with the vector kernels, which stay the default: they keep more bytes in flight).
constexpr int kBulkChunk = 8192, kBulkStages = 4;

__device__ __forceinline__ void bulk_load(void *smem, const void *gsrc, uint32_t bytes, uint64_t *mbar)
{
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem), m = (uint32_t)__cvta_generic_to_shared(mbar);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(m), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(d), "l"(gsrc), "r"(bytes), "r"(m)
                 : "memory");
}
__device__ __forceinline__ void bulk_store(void *gdst, const void *smem, uint32_t bytes)
{
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(s), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *mbar, uint32_t parity)
{
    const uint32_t m = (uint32_t)__cvta_generic_to_shared(mbar);
    uint32_t done = 0;
    while (!done)
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(m), "r"(parity) : "memory");
}

// kDe == false: planar -> interleaved; kDe == true: interleaved -> planar.  chunk list: item x block x channel x chunk.
template <bool kDe>
__global__ void __launch_bounds__(32)
interleave_tma_kernel(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, int64_t planar_channel_stride, int64_t planar_item_stride,
                      int64_t ilv_item_stride, int n_items, Shape sh)
{
    extern __shared__ __align__(128) uint8_t ring[];  // kBulkStages x kBulkChunk
    __shared__ __align__(8) uint64_t mbar[kBulkStages];
    if (threadIdx.x != 0) return;
    for (int s = 0; s < kBulkStages; s++) {
        const uint32_t m = (uint32_t)__cvta_generic_to_shared(&mbar[s]);
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(m) : "memory");
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const int64_t ilv = sh.interleave, blocks = sh.blocks_to_copy;
    const int64_t cpb = (ilv + kBulkChunk - 1) / kBulkChunk;            // chunks per (block, channel), over-counted for a short last block
    const int64_t per_item = blocks * sh.count * cpb, total = per_item * n_items;
    auto locate = [&](int64_t w, const uint8_t *&src, uint8_t *&dst, uint32_t &bytes) {
        const int64_t item = w / per_item, r = w - item * per_item;
        const int64_t b = r / (sh.count * cpb), r2 = r - b * (sh.count * cpb);
        const int64_t c = r2 / cpb, k = r2 - c * cpb;
        const int64_t cur = b == sh.in_blocks - 1 ? sh.last_in : ilv;    // in_size == out_size: both sides agree
        const int64_t off = k * kBulkChunk;
        bytes = off < cur ? (uint32_t)(cur - off < kBulkChunk ? cur - off : kBulkChunk) : 0u;
        const int64_t planar = item * planar_item_stride + c * planar_channel_stride + b * ilv + off;
        const int64_t packed = item * ilv_item_stride + b * ilv * sh.count + c * cur + off;
        src = in + (kDe ? packed : planar);
        dst = out + (kDe ? planar : packed);
    };
    const int64_t first = blockIdx.x, stride = gridDim.x;
    const int64_t n_mine = first < total ? (total - first + stride - 1) / stride : 0;
    uint32_t phase_bits = 0;
    for (int64_t j = 0; j < kBulkStages - 1 && j < n_mine; j++) {
        const uint8_t *src; uint8_t *dst; uint32_t bytes;
        locate(first + j * stride, src, dst, bytes);
        if (bytes) bulk_load(ring + (j % kBulkStages) * kBulkChunk, src, bytes, &mbar[j % kBulkStages]);
    }
    for (int64_t j = 0; j < n_mine; j++) {
        const int s = (int)(j % kBulkStages);
        const int64_t ahead = j + kBulkStages - 1;
        if (ahead < n_mine) {  // the stage the look-ahead load lands in was read by the store of chunk j-1
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            const uint8_t *src; uint8_t *dst; uint32_t bytes;
            locate(first + ahead * stride, src, dst, bytes);
            if (bytes) bulk_load(ring + (ahead % kBulkStages) * kBulkChunk, src, bytes, &mbar[ahead % kBulkStages]);
        }
        const uint8_t *src; uint8_t *dst; uint32_t bytes;
        locate(first + j * stride, src, dst, bytes);
        if (bytes) {
            mbar_wait(&mbar[s], (phase_bits >> s) & 1u);
            phase_bits ^= 1u << s;
            bulk_store(dst, ring + s * kBulkChunk, bytes);
        }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

inline bool tma_wanted() { const char *e = std::getenv("VGB_INTERLEAVE_TMA"); return e && e[0] == '1'; }

template <bool kDe>
cudaError_t launch_tma(const void *in, void *out, int64_t planar_channel_stride, int64_t planar_item_stride, int64_t ilv_item_stride,
                       int n_items, const Shape &sh, cudaStream_t stream)
{
    static int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
    const size_t smem = (size_t)kBulkStages * kBulkChunk;
    auto kern = interleave_tma_kernel<kDe>;
    raise_dynamic_smem(kern, smem);
    const int64_t cpb = (sh.interleave + kBulkChunk - 1) / kBulkChunk;
    const int64_t total = sh.blocks_to_copy * sh.count * cpb * n_items;
    const int grid = (int)std::min<int64_t>(total, (int64_t)sms * 6);
    if (grid <= 0) return cudaSuccess;
    kern<<<grid, 32, smem, stream>>>(static_cast<const uint8_t *>(in), static_cast<uint8_t *>(out), planar_channel_stride, planar_item_stride,
                                     ilv_item_stride, n_items, sh);
    return cudaGetLastError();
}

struct alignas(16) Vec16 { uint32_t x, y, z, w; };

inline int vector_width(std::initializer_list<int64_t> values)
{
    int w = 16;
    for (int64_t v : values)
        while (w > 1 && (v % w) != 0) w >>= 1;
    return w;
}

inline uint32_t blocks_per_item_for(int64_t elements_per_item)
{
    const int64_t per_block = (int64_t)kIlvThreads * kIlvIter;
    return (uint32_t)((elements_per_item + per_block - 1) / per_block);
}

}  // namespace

cudaError_t launch_interleave(const void *in, int64_t in_channel_stride, int64_t in_item_stride, void *out, int64_t out_item_stride,
                              int n_items, int count, int64_t in_size, int64_t interleave, int64_t out_size, cudaStream_t stream)
{
    if (n_items <= 0 || count <= 0 || out_size <= 0) return cudaSuccess;
    const Shape sh = make_shape(count, in_size, interleave, out_size);
    const int w = vector_width({interleave, in_size, out_size, sh.last_in, sh.last_out, in_channel_stride, in_item_stride, out_item_stride,
                                (int64_t)reinterpret_cast<uintptr_t>(in), (int64_t)reinterpret_cast<uintptr_t>(out)});
    if (w == 16 && in_size == out_size && tma_wanted())
        return launch_tma<false>(in, out, in_channel_stride, in_item_stride, out_item_stride, n_items, sh, stream);
    if (out_size * count >= (int64_t)1 << 31 || in_size >= (int64_t)1 << 31) return cudaErrorInvalidValue;  // 32-bit index arithmetic per item
    const uint32_t bpi = blocks_per_item_for(out_size * count / w);
    const int64_t grid64 = (int64_t)bpi * n_items;
    if (grid64 >= (int64_t)1 << 31) return cudaErrorInvalidValue;
    const unsigned grid = (unsigned)grid64;
    const uint8_t *i8 = static_cast<const uint8_t *>(in);
    uint8_t *o8 = static_cast<uint8_t *>(out);
    switch (w) {
    case 16: interleave_kernel<Vec16><<<grid, kIlvThreads, 0, stream>>>(i8, in_channel_stride, in_item_stride, o8, out_item_stride, bpi, sh); break;
    case 8: interleave_kernel<uint64_t><<<grid, kIlvThreads, 0, stream>>>(i8, in_channel_stride, in_item_stride, o8, out_item_stride, bpi, sh); break;
    case 4: interleave_kernel<uint32_t><<<grid, kIlvThreads, 0, stream>>>(i8, in_channel_stride, in_item_stride, o8, out_item_stride, bpi, sh); break;
    case 2: interleave_kernel<uint16_t><<<grid, kIlvThreads, 0, stream>>>(i8, in_channel_stride, in_item_stride, o8, out_item_stride, bpi, sh); break;
    default: interleave_kernel<uint8_t><<<grid, kIlvThreads, 0, stream>>>(i8, in_channel_stride, in_item_stride, o8, out_item_stride, bpi, sh); break;
    }
    return cudaGetLastError();
}

cudaError_t launch_deinterleave(const void *in, int64_t in_item_stride, void *out, int64_t out_channel_stride, int64_t out_item_stride,
                                int n_items, int count, int64_t in_size, int64_t interleave, int64_t out_size, cudaStream_t stream)
{
    if (n_items <= 0 || count <= 0 || out_size <= 0) return cudaSuccess;
    const Shape sh = make_shape(count, in_size, interleave, out_size);
    const int w = vector_width({interleave, in_size, out_size, sh.last_in, sh.last_out, out_channel_stride, in_item_stride, out_item_stride,
                                (int64_t)reinterpret_cast<uintptr_t>(in), (int64_t)reinterpret_cast<uintptr_t>(out)});
    if (w == 16 && in_size == out_size && tma_wanted())
        return launch_tma<true>(in, out, out_channel_stride, out_item_stride, in_item_stride, n_items, sh, stream);
    if (out_size * count >= (int64_t)1 << 31 || in_size * count >= (int64_t)1 << 31) return cudaErrorInvalidValue;
    const uint32_t bpi = blocks_per_item_for(out_size / w * count);
    const int64_t grid64 = (int64_t)bpi * n_items;
    if (grid64 >= (int64_t)1 << 31) return cudaErrorInvalidValue;
    const unsigned grid = (unsigned)grid64;
    const uint8_t *i8 = static_cast<const uint8_t *>(in);
    uint8_t *o8 = static_cast<uint8_t *>(out);
    switch (w) {
    case 16: deinterleave_kernel<Vec16><<<grid, kIlvThreads, 0, stream>>>(i8, in_item_stride, o8, out_channel_stride, out_item_stride, bpi, sh); break;
    case 8: deinterleave_kernel<uint64_t><<<grid, kIlvThreads, 0, stream>>>(i8, in_item_stride, o8, out_channel_stride, out_item_stride, bpi, sh); break;
    case 4: deinterleave_kernel<uint32_t><<<grid, kIlvThreads, 0, stream>>>(i8, in_item_stride, o8, out_channel_stride, out_item_stride, bpi, sh); break;
    case 2: deinterleave_kernel<uint16_t><<<grid, kIlvThreads, 0, stream>>>(i8, in_item_stride, o8, out_channel_stride, out_item_stride, bpi, sh); break;
    default: deinterleave_kernel<uint8_t><<<grid, kIlvThreads, 0, stream>>>(i8, in_item_stride, o8, out_channel_stride, out_item_stride, bpi, sh); break;
    }
    return cudaGetLastError();
}

}  // namespace vgb
