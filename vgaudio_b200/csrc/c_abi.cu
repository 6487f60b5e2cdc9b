// c_abi.cu — the extern "C" boundary of libvgaudio_b200.so (declared in include/vgaudio_b200.h).
//
// Host-side responsibilities only: argument validation with the reference's error behaviour, HBM layout of a
// batch (channel slabs + tables), H2D/D2H movement, kernel sequencing on one stream, timing taps.
// No codec arithmetic happens on the CPU here; without a CUDA device every codec entry point fails (VGB_E_CUDA).
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "../../include/vgaudio_b200.h"
#include "common.cuh"
#include "kernels.h"

using namespace vgb;

namespace {

thread_local std::string g_err;

int32_t fail(int32_t code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

}  // namespace
namespace vgb {
void containers_release();  // containers.cu
int32_t abi_fail(int32_t code, const char *fmt, ...)  // for the other translation units of the boundary (collective.cu)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
}  // namespace vgb
namespace {

#define CUDA_TRY(expr)                                                                                      \
    do {                                                                                                    \
        cudaError_t e_ = (expr);                                                                            \
        if (e_ != cudaSuccess)                                                                              \
            return fail(e_ == cudaErrorMemoryAllocation ? VGB_E_NOMEM : VGB_E_CUDA, "%s failed: %s", #expr, \
                        cudaGetErrorString(e_));                                                            \
    } while (0)

#define VGB_TRY(expr)              \
    do {                           \
        int32_t s_ = (expr);       \
        if (s_ != VGB_OK) return s_; \
    } while (0)

// Grow-only device buffer.
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    int32_t reserve(size_t bytes)
    {
        if (bytes <= cap && p) return VGB_OK;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        if (bytes == 0) bytes = 256;
        size_t want = bytes + bytes / 8 + 4096;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            want = bytes;
            e = cudaMalloc(&p, want);
        }
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            p = nullptr;
            return fail(VGB_E_NOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
        }
        cap = want;
        return VGB_OK;
    }
    void release()
    {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
};

constexpr int kTimers = 10;  // 0 coef phase 1, 1 coef refine, 2 gc encode, 3 gc decode, 4 adx encode, 5 adx decode, 6 hca encode, 7 hca decode, 8 interleave, 9 deinterleave
constexpr int kMaxGroups = 16;   // channel groups of one host call, pipelined: H2D(g+1) || kernels(g) || D2H(g-1)
constexpr int kCompStreams = 4;  // kernel streams the groups rotate over

// One upload of the HCA codec tables per device
struct HcaTableStore {
    bool ready = false;
    void *blob = nullptr;
    HcaTables view{};
};

// Everything the library keeps per bound device.  The entry points reach "their" context through g_ctx: the primary
// device's for a caller thread, a worker's own when a host-pointer batch call is sharded over several devices.
struct Context {
    std::mutex mu;
    bool ready = false;
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t s_in = nullptr, s_out = nullptr, s_comp[kCompStreams] = {};
    cudaEvent_t ev_in[kMaxGroups] = {}, ev_done[kMaxGroups] = {}, ev_out[kMaxGroups] = {}, ev_mid[kMaxGroups] = {}, ev_t0 = nullptr;
    int last_groups = 0;
    DevBuf pcm, adpcm, coefs, ws, misc;
    bool timing = false;
    cudaEvent_t ev[2 * kTimers] = {};
    bool ev_used[kTimers] = {};
    std::atomic<int64_t> launches{0};
    GcSegArgs last_seg{};            // bookkeeping of the most recent encode launch (vgb_gcadpcm_debug_splice_stats)
    HcaTableStore hca_tables;
};

Context g_primary;                               // the device vgb_init / vgb_init_devices binds first
std::vector<std::unique_ptr<Context>> g_extra;   // further devices of vgb_init_devices
thread_local Context *t_ctx = &g_primary;        // the context this thread works on
#define g_ctx (*t_ctx)
#define g_hca_tables (g_ctx.hca_tables)

void hca_tables_release_locked();  // defined next to the HCA table store

int32_t ensure_ready_locked()
{
    if (g_ctx.ready) {
        CUDA_TRY(cudaSetDevice(g_ctx.device));
        return VGB_OK;
    }
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) {
        (void)cudaGetLastError();
        return fail(VGB_E_CUDA, "no CUDA device available (%s): libvgaudio_b200 has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    if (g_ctx.device >= count) return fail(VGB_E_ARG, "device %d out of range (%d devices)", g_ctx.device, count);
    CUDA_TRY(cudaSetDevice(g_ctx.device));
    CUDA_TRY(cudaStreamCreateWithFlags(&g_ctx.stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&g_ctx.s_in, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&g_ctx.s_out, cudaStreamNonBlocking));
    for (int g = 0; g < kCompStreams; g++) CUDA_TRY(cudaStreamCreateWithFlags(&g_ctx.s_comp[g], cudaStreamNonBlocking));
    for (int g = 0; g < kMaxGroups; g++) {
        CUDA_TRY(cudaEventCreate(&g_ctx.ev_in[g]));
        CUDA_TRY(cudaEventCreate(&g_ctx.ev_done[g]));
        CUDA_TRY(cudaEventCreate(&g_ctx.ev_out[g]));
        CUDA_TRY(cudaEventCreate(&g_ctx.ev_mid[g]));
    }
    CUDA_TRY(cudaEventCreate(&g_ctx.ev_t0));
    for (auto &ev : g_ctx.ev) CUDA_TRY(cudaEventCreate(&ev));
    g_ctx.ready = true;
    return VGB_OK;
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

void tick(int slot, bool begin, cudaStream_t stream)
{
    if (!g_ctx.timing) return;
    cudaEventRecord(g_ctx.ev[2 * slot + (begin ? 0 : 1)], stream);
    if (!begin) g_ctx.ev_used[slot] = true;
}

// ---- batch layout ----------------------------------------------------------------------------------------
struct GcLayout {
    int32_t n_channels = 0;
    std::vector<int64_t> pcm_off, adpcm_off, rec_off;
    std::vector<int32_t> n_samples, enc_count;
    std::vector<int16_t> hist;  // [ch][2] = hist1, hist2
    int64_t pcm_total = 0;      // samples, padded
    int64_t adpcm_total = 0;    // bytes, padded
    int64_t rec_total = 0;      // frames, padded to a multiple of 32 per channel
    int32_t max_frames = 0;     // over analysis and encode lengths
    int64_t total_frames = 0;   // sum over channels of encode frames (progress total, GcAdpcmFormat.cs:62)
};

// Workspace carve-up (every region 256-byte aligned).  [0, table_bytes) is the host-built table blob.
struct GcWorkspace {
    size_t off_pcm_off, off_adpcm_off, off_rec_off, off_n_samples, off_enc_count, off_hist, off_records, off_mask;
    size_t off_trace, off_used_start, off_stats;  // time-parallel encode bookkeeping (GcSegArgs)
    size_t off_status;                            // decode: first channel with an out-of-range predictor index
    size_t table_bytes;
    size_t total;
};

GcWorkspace carve(int64_t rec_total_frames, int32_t n_channels)
{
    GcWorkspace w{};
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o = align_up(o + bytes, 256); return at; };
    const size_t n = (size_t)(n_channels > 0 ? n_channels : 1);
    w.off_pcm_off = take(n * 8);
    w.off_adpcm_off = take(n * 8);
    w.off_rec_off = take(n * 8);
    w.off_n_samples = take(n * 4);
    w.off_enc_count = take(n * 4);
    w.off_hist = take(n * 4);
    w.table_bytes = o;
    w.off_records = take((size_t)rec_total_frames * sizeof(double2));
    w.off_mask = take((size_t)(rec_total_frames / 32 + 1) * 4);
    w.off_trace = take((size_t)rec_total_frames * 4);
    w.off_used_start = take(n * kGcMaxSegments * 4);
    w.off_stats = take(kGcStatWords * 8);
    w.off_status = take(16);
    w.total = o;
    return w;
}

// upper bound of the padded record slab for a given total frame count (what workspace_bytes promises)
int64_t padded_rec_bound(int64_t total_frames, int32_t n_channels) { return total_frames + 32ll * n_channels + 32; }

GcChannelTable table_view(void *ws, const GcWorkspace &w, int32_t n_channels)
{
    char *b = static_cast<char *>(ws);
    GcChannelTable t;
    t.pcm_off = reinterpret_cast<const int64_t *>(b + w.off_pcm_off);
    t.adpcm_off = reinterpret_cast<const int64_t *>(b + w.off_adpcm_off);
    t.rec_off = reinterpret_cast<const int64_t *>(b + w.off_rec_off);
    t.n_samples = reinterpret_cast<const int32_t *>(b + w.off_n_samples);
    t.enc_count = reinterpret_cast<const int32_t *>(b + w.off_enc_count);
    t.hist = reinterpret_cast<int16_t *>(b + w.off_hist);
    t.status = reinterpret_cast<int32_t *>(b + w.off_status);
    t.n_channels = n_channels;
    return t;
}

GcSegArgs seg_view(void *ws, const GcWorkspace &w, int32_t seg_count)
{
    char *b = static_cast<char *>(ws);
    GcSegArgs a;
    a.trace = reinterpret_cast<uint32_t *>(b + w.off_trace);
    a.used_start = reinterpret_cast<uint32_t *>(b + w.off_used_start);
    a.stats = reinterpret_cast<unsigned long long *>(b + w.off_stats);
    a.seg_count = seg_count;
    a.min_seg_frames = 0;  // the caller stores gc_encode_pick_segments' choice; 0 lets launch_gc_encode take the default
    return a;
}

int32_t upload_tables(const GcLayout &lay, const GcWorkspace &w, void *ws, cudaStream_t stream)
{
    std::vector<char> blob(w.table_bytes, 0);
    const size_t n = (size_t)lay.n_channels;
    if (n) {
        memcpy(blob.data() + w.off_pcm_off, lay.pcm_off.data(), n * 8);
        memcpy(blob.data() + w.off_adpcm_off, lay.adpcm_off.data(), n * 8);
        memcpy(blob.data() + w.off_rec_off, lay.rec_off.data(), n * 8);
        memcpy(blob.data() + w.off_n_samples, lay.n_samples.data(), n * 4);
        memcpy(blob.data() + w.off_enc_count, lay.enc_count.data(), n * 4);
        memcpy(blob.data() + w.off_hist, lay.hist.data(), n * 4);
    }
    // pageable source: the runtime stages it before returning, so `blob` may die at scope exit
    CUDA_TRY(cudaMemcpyAsync(ws, blob.data(), w.table_bytes, cudaMemcpyHostToDevice, stream));
    return VGB_OK;
}

// Validates lengths/params and fills everything in `lay` except pcm_off / adpcm_off.
// `decode`: n_samples is the decoded sample count and enc_count mirrors it.
int32_t layout_common(GcLayout &lay, const int32_t *n_samples, const vgb_gc_params *params, int32_t n_channels,
                      bool decode)
{
    if (n_channels < 0) return fail(VGB_E_ARG, "n_channels is negative (%d)", n_channels);
    if (n_channels > 0 && !n_samples) return fail(VGB_E_ARG, "n_samples is NULL");
    lay.n_channels = n_channels;
    lay.n_samples.resize(n_channels);
    lay.enc_count.resize(n_channels);
    lay.rec_off.resize(n_channels);
    lay.hist.assign((size_t)n_channels * 2, 0);
    int64_t rec = 0;
    for (int c = 0; c < n_channels; c++) {
        const int32_t n = n_samples[c];
        if (n < 0) return fail(VGB_E_ARG, "channel %d: negative sample count %d", c, n);
        int32_t enc = n;
        if (params) {
            if (!decode && params[c].sample_count != -1) {
                enc = params[c].sample_count;
                // GcAdpcmEncoder.Encode would run Array.Copy past pcm.Length and throw ArgumentException
                if (enc < 0 || enc > n)
                    return fail(VGB_E_ARG, "channel %d: sample_count %d outside the %d available samples", c, enc, n);
            }
            lay.hist[2 * c] = params[c].history1;
            lay.hist[2 * c + 1] = params[c].history2;
        }
        lay.n_samples[c] = n;
        lay.enc_count[c] = enc;
        const int32_t frames = div_round_up(n, kGcFrameSamples);
        lay.rec_off[c] = rec;
        rec += align_up((size_t)frames, 32);
        if (frames > lay.max_frames) lay.max_frames = frames;
        lay.total_frames += div_round_up(enc, kGcFrameSamples);
    }
    lay.rec_total = rec + 32;
    return VGB_OK;
}

void layout_pack_offsets(GcLayout &lay)
{
    lay.pcm_off.resize(lay.n_channels);
    lay.adpcm_off.resize(lay.n_channels);
    int64_t ps = 0, ab = 0;
    for (int c = 0; c < lay.n_channels; c++) {
        lay.pcm_off[c] = ps;
        lay.adpcm_off[c] = ab;
        ps += (int64_t)align_up((size_t)lay.n_samples[c], 8);
        ab += (int64_t)align_up((size_t)gc_sample_count_to_byte_count(lay.n_samples[c]), 16);
    }
    lay.pcm_total = ps + 8;
    lay.adpcm_total = ab + 16;
}

int max_encode_frames(const GcLayout &lay)
{
    int32_t m = 0;
    for (int c = 0; c < lay.n_channels; c++) m = std::max(m, div_round_up(lay.enc_count[c], kGcFrameSamples));
    return m;
}

// Kernel sequence of one encode call on `stream` (device pointers only).
int32_t run_gc_encode(const int16_t *d_pcm, const GcLayout &lay, const int16_t *d_coefs_in, int16_t *d_coefs_out,
                      uint8_t *d_adpcm, void *d_ws, const GcWorkspace &w, cudaStream_t stream, bool do_encode,
                      bool timed = true, bool tables_uploaded = false, cudaEvent_t after_coefs = nullptr)
{
    const bool was_timing = g_ctx.timing;
    if (!timed) g_ctx.timing = false;  // the kernel timers describe single-stream (_dev) calls only
    struct Restore { bool v; ~Restore() { g_ctx.timing = v; } } restore{was_timing};
    if (!tables_uploaded) VGB_TRY(upload_tables(lay, w, d_ws, stream));
    if (lay.n_channels == 0) return VGB_OK;
    GcChannelTable tab = table_view(d_ws, w, lay.n_channels);
    char *b = static_cast<char *>(d_ws);
    double2 *records = reinterpret_cast<double2 *>(b + w.off_records);
    uint32_t *mask = reinterpret_cast<uint32_t *>(b + w.off_mask);

    if (!d_coefs_in) {
        tick(0, true, stream);
        launch_gc_coef_frames(d_pcm, tab, records, mask, lay.max_frames, 0, INT_MAX, stream);
        tick(0, false, stream);
        tick(1, true, stream);
        launch_gc_coef_refine(tab, records, mask, d_coefs_out, stream);
        tick(1, false, stream);
        g_ctx.launches += (lay.max_frames > 0 ? 1 : 0) + 1;
    } else if (d_coefs_in != d_coefs_out) {
        CUDA_TRY(cudaMemcpyAsync(d_coefs_out, d_coefs_in, (size_t)lay.n_channels * 32, cudaMemcpyDeviceToDevice, stream));
    }
    if (after_coefs) CUDA_TRY(cudaEventRecord(after_coefs, stream));
    if (do_encode) {
        const int enc_frames = max_encode_frames(lay);
        int min_seg = 0;
        const int seg_count = gc_encode_pick_segments(lay.n_channels, enc_frames, &min_seg);
        GcSegArgs seg = seg_view(d_ws, w, seg_count);
        seg.min_seg_frames = min_seg;
        tick(2, true, stream);
        launch_gc_encode(d_pcm, tab, d_coefs_out, d_adpcm, lay.max_frames, 0, INT_MAX, seg, stream);
        tick(2, false, stream);
        g_ctx.launches += lay.max_frames > 0 ? (seg.seg_count > 1 ? 3 : 1) : 0;
        g_ctx.last_seg = seg;
    }
    CUDA_TRY(cudaGetLastError());
    return VGB_OK;
}

int32_t run_gc_decode(const uint8_t *d_adpcm, const GcLayout &lay, const int16_t *d_coefs, int16_t *d_pcm, void *d_ws,
                      const GcWorkspace &w, cudaStream_t stream)
{
    VGB_TRY(upload_tables(lay, w, d_ws, stream));
    if (lay.n_channels == 0) return VGB_OK;
    GcChannelTable tab = table_view(d_ws, w, lay.n_channels);
    CUDA_TRY(cudaMemsetAsync(tab.status, 0x7f, 4, stream));  // "no channel": any index is smaller
    tick(3, true, stream);
    launch_gc_decode(d_adpcm, tab, d_coefs, d_pcm, lay.max_frames, 0, INT_MAX, stream);
    tick(3, false, stream);
    g_ctx.launches += lay.max_frames > 0 ? 1 : 0;
    CUDA_TRY(cudaGetLastError());
    return VGB_OK;
}

// If ptr[c] == ptr[0] + c*stride for every c (the caller handed one slab), returns true and the stride in bytes.
template <typename T>
bool uniform_stride(T *const *ptr, int32_t n, int64_t &stride_bytes)
{
    if (n < 2) { stride_bytes = 0; return true; }
    const int64_t s = reinterpret_cast<const char *>(ptr[1]) - reinterpret_cast<const char *>(ptr[0]);
    if (s <= 0) return false;
    for (int c = 2; c < n; c++)
        if (reinterpret_cast<const char *>(ptr[c]) - reinterpret_cast<const char *>(ptr[c - 1]) != s) return false;
    stride_bytes = s;
    return true;
}


// Pageable caller buffers (a C# short[] pinned by the GC is still pageable for CUDA) move through the driver's staging
// buffers at a fraction of PCIe speed; page-locking the region for the duration of the call costs some ms per GiB and
// lets the copy engine read it directly at PCIe speed (tools/host_register_probe.py compares the two).  Inputs only: they are touched memory; registering a freshly allocated output would
// fault its pages in first and cost more than it saves.  Registrations live until the API call returns (PinScope).
thread_local std::vector<void *> t_pins;

struct PinScope {
    ~PinScope()
    {
        for (void *p : t_pins) cudaHostUnregister(p);
        t_pins.clear();
        (void)cudaGetLastError();
    }
};

void try_pin(const void *p, size_t bytes)
{
    if (!p || bytes < ((size_t)1 << 20)) return;
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { (void)cudaGetLastError(); return; }
    if (attr.type != cudaMemoryTypeUnregistered) return;  // already page-locked (vgb_host_alloc) or not host memory
    void *q = const_cast<void *>(p);
    if (cudaHostRegister(q, bytes, cudaHostRegisterDefault) == cudaSuccess ||
        ((void)cudaGetLastError(), cudaHostRegister(q, bytes, cudaHostRegisterReadOnly) == cudaSuccess))
        t_pins.push_back(q);
    else
        (void)cudaGetLastError();  // stay pageable
}

// Many small copies in one driver call (cudaMemcpyBatchAsync, CUDA 12.8+): a ragged batch of tens of thousands of short
// files otherwise spends more host time in cudaMemcpyAsync calls (~5 us each) than the copies take on the link.  Falls
// back to one call per copy when the batched call is refused.
int32_t copy_many(std::vector<void *> &dsts, std::vector<void *> &srcs, std::vector<size_t> &sizes, cudaMemcpyKind kind, cudaStream_t stream)
{
    const size_t n = sizes.size();
    if (n == 0) return VGB_OK;
    static bool batch_ok = std::getenv("VGB_NO_MEMCPY_BATCH") == nullptr;
    if (batch_ok && n >= 16) {
        cudaMemcpyAttributes attr{};
        attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;  // sources stay valid until the call returns (we synchronise)
        attr.flags = 0;
        size_t attr_idx = 0, fail_idx = 0;
        const cudaError_t e = cudaMemcpyBatchAsync(dsts.data(), srcs.data(), sizes.data(), n, &attr, &attr_idx, 1, &fail_idx, stream);
        if (e == cudaSuccess) return VGB_OK;
        (void)cudaGetLastError();
        batch_ok = false;  // e.g. an older driver: stay on the per-copy path for the rest of the process
    }
    for (size_t i = 0; i < n; i++) CUDA_TRY(cudaMemcpyAsync(dsts[i], srcs[i], sizes[i], kind, stream));
    return VGB_OK;
}

// Host -> device copy of every channel's bytes: one strided 2D copy when the caller's buffers form a slab,
// else one copy per channel.
template <typename T>
int32_t copy_channels_in(char *d_base, const std::vector<int64_t> &d_off_bytes, T *const *h_ptr,
                         const std::vector<int64_t> &bytes, cudaStream_t stream)
{
    const int32_t n = (int32_t)bytes.size();
    if (n == 0) return VGB_OK;
    bool same = true;
    for (int c = 1; c < n; c++) same = same && bytes[c] == bytes[0];
    int64_t hstride = 0;
    if (same && n > 1 && bytes[0] > 0 && uniform_stride(h_ptr, n, hstride) && hstride >= bytes[0]) {  // overlapping rows: per-channel copies
        const int64_t dstride = d_off_bytes[1] - d_off_bytes[0];
        bool dsame = true;
        for (int c = 2; c < n; c++) dsame = dsame && (d_off_bytes[c] - d_off_bytes[c - 1] == dstride);
        if (dsame) {
            try_pin(h_ptr[0], (size_t)(hstride * (n - 1) + bytes[0]));
            CUDA_TRY(cudaMemcpy2DAsync(d_base + d_off_bytes[0], (size_t)dstride, h_ptr[0], (size_t)hstride,
                                       (size_t)bytes[0], (size_t)n, cudaMemcpyHostToDevice, stream));
            return VGB_OK;
        }
    }
    std::vector<void *> dsts, srcs;
    std::vector<size_t> sizes;
    for (int c = 0; c < n; c++)
        if (bytes[c] > 0) {
            try_pin(h_ptr[c], (size_t)bytes[c]);
            dsts.push_back(d_base + d_off_bytes[c]);
            srcs.push_back(const_cast<void *>(static_cast<const void *>(h_ptr[c])));
            sizes.push_back((size_t)bytes[c]);
        }
    return copy_many(dsts, srcs, sizes, cudaMemcpyHostToDevice, stream);
}

template <typename T>
int32_t copy_channels_out(T *const *h_ptr, const char *d_base, const std::vector<int64_t> &d_off_bytes,
                          const std::vector<int64_t> &bytes, cudaStream_t stream)
{
    const int32_t n = (int32_t)bytes.size();
    if (n == 0) return VGB_OK;
    bool same = true;
    for (int c = 1; c < n; c++) same = same && bytes[c] == bytes[0];
    int64_t hstride = 0;
    if (same && n > 1 && bytes[0] > 0 && uniform_stride(h_ptr, n, hstride) && hstride >= bytes[0]) {
        const int64_t dstride = d_off_bytes[1] - d_off_bytes[0];
        bool dsame = true;
        for (int c = 2; c < n; c++) dsame = dsame && (d_off_bytes[c] - d_off_bytes[c - 1] == dstride);
        if (dsame) {
            CUDA_TRY(cudaMemcpy2DAsync(h_ptr[0], (size_t)hstride, d_base + d_off_bytes[0], (size_t)dstride,
                                       (size_t)bytes[0], (size_t)n, cudaMemcpyDeviceToHost, stream));
            return VGB_OK;
        }
    }
    std::vector<void *> dsts, srcs;
    std::vector<size_t> sizes;
    for (int c = 0; c < n; c++)
        if (bytes[c] > 0) {
            dsts.push_back(static_cast<void *>(h_ptr[c]));
            srcs.push_back(const_cast<char *>(d_base + d_off_bytes[c]));
            sizes.push_back((size_t)bytes[c]);
        }
    return copy_many(dsts, srcs, sizes, cudaMemcpyDeviceToHost, stream);
}

// Sub-batch of channels [c0, c1) of a validated full layout; offsets stay absolute into the shared slabs, the record
// slab of the group is its own.
GcLayout sub_layout(const GcLayout &full, int c0, int c1)
{
    GcLayout g;
    g.n_channels = c1 - c0;
    g.pcm_off.assign(full.pcm_off.begin() + c0, full.pcm_off.begin() + c1);
    g.adpcm_off.assign(full.adpcm_off.begin() + c0, full.adpcm_off.begin() + c1);
    g.n_samples.assign(full.n_samples.begin() + c0, full.n_samples.begin() + c1);
    g.enc_count.assign(full.enc_count.begin() + c0, full.enc_count.begin() + c1);
    g.hist.assign(full.hist.begin() + 2 * c0, full.hist.begin() + 2 * c1);
    g.rec_off.resize(g.n_channels);
    int64_t rec = 0;
    for (int c = 0; c < g.n_channels; c++) {
        const int32_t frames = div_round_up(g.n_samples[c], kGcFrameSamples);
        g.rec_off[c] = rec;
        rec += (int64_t)align_up((size_t)frames, 32);
        if (frames > g.max_frames) g.max_frames = frames;
        g.total_frames += div_round_up(g.enc_count[c], kGcFrameSamples);
    }
    g.rec_total = rec + 32;
    return g;
}

// ---- host-call pipeline over groups of independent units (channels / streams) ------------------------------------------
// Every host-pointer entry point moves bytes over PCIe on both sides of its kernels.  Units are independent, so the
// call is cut into groups: the H2D copy of group g+1, the kernels of group g and the D2H copy of group g-1 overlap on
// three kinds of streams.  `h2d(g)` enqueues on g_ctx.s_in, `kern(g, stream)` on one of the kernel streams,
// `d2h(g)` on g_ctx.s_out; the helper adds the events, the timeline taps and the final synchronisation.  Returns with
// nothing in flight, also on error (caller memory may be unpinned / freed right after).
struct PipelineDrain {
    ~PipelineDrain()
    {
        cudaStreamSynchronize(g_ctx.s_in);
        for (auto st : g_ctx.s_comp) cudaStreamSynchronize(st);
        cudaStreamSynchronize(g_ctx.s_out);
        (void)cudaGetLastError();
    }
};

// how many groups for `units` units carrying `bytes` bytes over PCIe in total (both directions)
int pipeline_group_count(int64_t units, int64_t bytes, int min_units_per_group)
{
    int64_t n = std::min<int64_t>(kMaxGroups / 2, std::min<int64_t>(bytes / (32 << 20), units / std::max(min_units_per_group, 1)));
    if (const char *env = std::getenv("VGB_PIPELINE_GROUPS")) {  // tuning knob: 1..kMaxGroups
        const int want = std::atoi(env);
        if (want >= 1 && want <= kMaxGroups && units >= want) n = want;
    }
    return (int)std::max<int64_t>(n, 1);
}

// group boundaries over units with the given weights (roughly equal weight per group, order preserved)
std::vector<int> pipeline_bounds(const std::vector<int64_t> &weight, int n_groups)
{
    const int n = (int)weight.size();
    std::vector<int> bound(n_groups + 1, n);
    bound[0] = 0;
    int64_t total = 0, run = 0;
    for (int64_t w : weight) total += w;
    int g = 1;
    for (int u = 0; u < n && g < n_groups; u++) {
        run += weight[u];
        if (run * n_groups >= total * g) bound[g++] = u + 1;
    }
    return bound;
}

template <class H2D, class Kern, class D2H, class Done>
int32_t run_group_pipeline(int n_groups, H2D h2d, Kern kern, D2H d2h, Done done)
{
    CUDA_TRY(cudaStreamSynchronize(g_ctx.stream));  // nothing of a previous call still uses the shared slabs
    PipelineDrain drain;
    CUDA_TRY(cudaEventRecord(g_ctx.ev_t0, g_ctx.s_in));
    g_ctx.last_groups = n_groups;
    for (int g = 0; g < n_groups; g++) {
        VGB_TRY(h2d(g));
        CUDA_TRY(cudaEventRecord(g_ctx.ev_in[g], g_ctx.s_in));
    }
    for (int g = 0; g < n_groups; g++) {
        cudaStream_t st = g_ctx.s_comp[g % kCompStreams];
        CUDA_TRY(cudaStreamWaitEvent(st, g_ctx.ev_in[g], 0));
        VGB_TRY(kern(g, st));
        CUDA_TRY(cudaEventRecord(g_ctx.ev_mid[g], st));
        CUDA_TRY(cudaEventRecord(g_ctx.ev_done[g], st));
    }
    for (int g = 0; g < n_groups; g++) {
        CUDA_TRY(cudaStreamWaitEvent(g_ctx.s_out, g_ctx.ev_done[g], 0));
        VGB_TRY(d2h(g));
        CUDA_TRY(cudaEventRecord(g_ctx.ev_out[g], g_ctx.s_out));
    }
    for (int g = 0; g < n_groups; g++) {
        CUDA_TRY(cudaEventSynchronize(g_ctx.ev_out[g]));
        VGB_TRY(done(g));
    }
    return VGB_OK;
}

// One host call, pipelined over three kinds of streams (input copies, kernels, output copies) in up to kMaxGroups
// channel groups: the H2D copy of group g+1, the kernels of group g and the D2H copy of group g-1 overlap (channels
// are independent; a channel's coefficients need all of its samples).
int32_t host_encode_impl(const int16_t *const *pcm, const int32_t *n_samples, const vgb_gc_params *params,
                         const int16_t *coefs_in, int32_t n_channels, int16_t *coefs_out, uint8_t *const *adpcm_out,
                         vgb_progress_cb cb, void *user, bool do_encode)
{
    PinScope pins;
    GcLayout lay;
    VGB_TRY(layout_common(lay, n_samples, params, n_channels, false));
    if (n_channels == 0) return VGB_OK;
    if (!pcm) return fail(VGB_E_ARG, "pcm is NULL");
    if (!coefs_out) return fail(VGB_E_ARG, "coefs_out is NULL");
    if (do_encode && !adpcm_out) return fail(VGB_E_ARG, "adpcm_out is NULL");
    for (int c = 0; c < n_channels; c++) {
        if (!pcm[c] && lay.n_samples[c] > 0) return fail(VGB_E_ARG, "pcm[%d] is NULL", c);
        if (do_encode && !adpcm_out[c] && lay.enc_count[c] > 0) return fail(VGB_E_ARG, "adpcm_out[%d] is NULL", c);
    }
    layout_pack_offsets(lay);

    // channel groups with roughly equal sample totals (boundaries on channel indices, order preserved).  The encoder is
    // throughput bound since it runs time-parallel (gc_encode.cu), so kernels of neighbouring groups share the SMs
    // without slowing each other: the PCIe copy of group g+1 hides the kernels of group g.
    int n_groups = 1;
    {
        int64_t total = 0;
        for (int c = 0; c < n_channels; c++) total += lay.n_samples[c];
        // a group should carry at least ~32 MB of PCM (a few ms of PCIe time) and 32 channels
        const int64_t by_bytes = total / (16 << 20), by_channels = n_channels / 32;
        n_groups = (int)std::min<int64_t>(kMaxGroups / 2, std::min<int64_t>(by_bytes, by_channels));
        if (n_groups < 1) n_groups = 1;
    }
    if (const char *env = std::getenv("VGB_ENCODE_GROUPS")) {  // tuning knob: 1..kMaxGroups
        const int want = std::atoi(env);
        if (want >= 1 && want <= kMaxGroups && n_channels >= want) n_groups = want;
    }
    std::vector<int> bound(n_groups + 1, n_channels);
    bound[0] = 0;
    {
        int64_t total = 0;
        for (int c = 0; c < n_channels; c++) total += lay.n_samples[c];
        int64_t run = 0;
        int g = 1;
        for (int c = 0; c < n_channels && g < n_groups; c++) {
            run += lay.n_samples[c];
            if (run * n_groups >= total * g) bound[g++] = c + 1;
        }
    }

    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    // every exit, including the error returns below, leaves no copy in flight on caller memory (pins are released
    // and the buffers may be freed as soon as this function returns)
    PipelineDrain drain;
    std::vector<GcLayout> glay(n_groups);
    std::vector<GcWorkspace> gws(n_groups);
    std::vector<size_t> ws_at(n_groups);
    size_t ws_total = 0;
    for (int g = 0; g < n_groups; g++) {
        glay[g] = sub_layout(lay, bound[g], bound[g + 1]);
        gws[g] = carve(glay[g].rec_total, glay[g].n_channels);
        ws_at[g] = ws_total;
        ws_total += align_up(gws[g].total, 256);
    }
    VGB_TRY(g_ctx.pcm.reserve((size_t)lay.pcm_total * 2));
    VGB_TRY(g_ctx.adpcm.reserve((size_t)lay.adpcm_total));
    VGB_TRY(g_ctx.coefs.reserve((size_t)n_channels * 32 * 2));
    VGB_TRY(g_ctx.ws.reserve(ws_total));
    // make sure nothing of a previous call is still using the buffers
    CUDA_TRY(cudaStreamSynchronize(g_ctx.stream));

    int16_t *d_coefs_out = static_cast<int16_t *>(g_ctx.coefs.p);
    int16_t *d_coefs_in = coefs_in ? d_coefs_out + (size_t)n_channels * 16 : nullptr;

    CUDA_TRY(cudaEventRecord(g_ctx.ev_t0, g_ctx.s_in));
    g_ctx.last_groups = n_groups;
    // stage 1: all H2D copies, in group order, on the input stream (the small tables first, while it is idle, so
    // that enqueuing the kernels below never has to wait for a pageable-memory copy behind a PCM transfer)
    for (int g = 0; g < n_groups; g++)
        VGB_TRY(upload_tables(glay[g], gws[g], static_cast<char *>(g_ctx.ws.p) + ws_at[g], g_ctx.s_in));
    for (int g = 0; g < n_groups; g++) {
        const int c0 = bound[g], n = bound[g + 1] - bound[g];
        std::vector<int64_t> off_b(n), len_b(n);
        for (int c = 0; c < n; c++) { off_b[c] = lay.pcm_off[c0 + c] * 2; len_b[c] = (int64_t)lay.n_samples[c0 + c] * 2; }
        VGB_TRY(copy_channels_in(static_cast<char *>(g_ctx.pcm.p), off_b, pcm + c0, len_b, g_ctx.s_in));
        if (coefs_in && n > 0)
            CUDA_TRY(cudaMemcpyAsync(d_coefs_in + (size_t)c0 * 16, coefs_in + (size_t)c0 * 16, (size_t)n * 32,
                                     cudaMemcpyHostToDevice, g_ctx.s_in));
        CUDA_TRY(cudaEventRecord(g_ctx.ev_in[g], g_ctx.s_in));
    }
    // stage 2: kernels of each group on its own stream, as soon as its PCM has landed
    for (int g = 0; g < n_groups; g++) {
        const int c0 = bound[g];
        cudaStream_t st = g_ctx.s_comp[g % kCompStreams];
        CUDA_TRY(cudaStreamWaitEvent(st, g_ctx.ev_in[g], 0));
        VGB_TRY(run_gc_encode(static_cast<const int16_t *>(g_ctx.pcm.p), glay[g],
                              d_coefs_in ? d_coefs_in + (size_t)c0 * 16 : nullptr, d_coefs_out + (size_t)c0 * 16,
                              static_cast<uint8_t *>(g_ctx.adpcm.p), static_cast<char *>(g_ctx.ws.p) + ws_at[g], gws[g],
                              st, do_encode, /*timed=*/false, /*tables_uploaded=*/true, g_ctx.ev_mid[g]));
        CUDA_TRY(cudaEventRecord(g_ctx.ev_done[g], st));
    }
    // stage 3: D2H of each group's results on the output stream
    for (int g = 0; g < n_groups; g++) {
        const int c0 = bound[g], n = bound[g + 1] - bound[g];
        CUDA_TRY(cudaStreamWaitEvent(g_ctx.s_out, g_ctx.ev_done[g], 0));
        if (n > 0)
            CUDA_TRY(cudaMemcpyAsync(coefs_out + (size_t)c0 * 16, d_coefs_out + (size_t)c0 * 16, (size_t)n * 32,
                                     cudaMemcpyDeviceToHost, g_ctx.s_out));
        if (do_encode) {
            std::vector<int64_t> off_b(n), len_b(n);
            for (int c = 0; c < n; c++) {
                off_b[c] = lay.adpcm_off[c0 + c];
                len_b[c] = gc_sample_count_to_byte_count(lay.enc_count[c0 + c]);
            }
            VGB_TRY(copy_channels_out(adpcm_out + c0, static_cast<const char *>(g_ctx.adpcm.p), off_b, len_b, g_ctx.s_out));
        }
        CUDA_TRY(cudaEventRecord(g_ctx.ev_out[g], g_ctx.s_out));
    }
    // the calling thread reports progress as the groups complete (IProgressReport.ReportAdd deltas sum to SetTotal)
    for (int g = 0; g < n_groups; g++) {
        CUDA_TRY(cudaEventSynchronize(g_ctx.ev_out[g]));
        if (cb && do_encode && glay[g].total_frames > 0) cb(user, glay[g].total_frames);
    }
    return VGB_OK;
}

// ---- several devices in one process (vgb_init_devices) ----------------------------------------------------------------
// The reference's counterpart is Parallel.ForEach over files (src/VGAudio.Cli/Batch.cs:24-25) on top of Parallel.For over
// channels: independent units.  A host-pointer batch call is sharded over the bound devices by greedy longest-first
// bin packing of the units' sample counts; every device gets a worker thread that runs the ordinary single-device call
// (its own H2D / kernels / D2H pipeline over its own PCIe link) on its share, results land directly in the caller's
// arrays.  No collective is involved: host data reaches each GPU fastest over that GPU's own link (SURVEY §8e); the NCCL
// scatterv / gatherv below serve data that is already resident on one device.
std::vector<Context *> bound_contexts()
{
    std::vector<Context *> v{&g_primary};
    for (auto &c : g_extra) v.push_back(c.get());
    return v;
}

// greedy LPT: heaviest unit first onto the least loaded device; a device's units keep ascending order
std::vector<std::vector<int>> shard_units(const std::vector<int64_t> &weight, int n_dev)
{
    const int n = (int)weight.size();
    std::vector<int> order(n);
    for (int i = 0; i < n; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return weight[a] > weight[b]; });
    std::vector<int64_t> load(n_dev, 0);
    std::vector<std::vector<int>> shards(n_dev);
    for (int u : order) {
        int best = 0;
        for (int d = 1; d < n_dev; d++) if (load[d] < load[best]) best = d;
        shards[best].push_back(u);
        load[best] += weight[u];
    }
    for (auto &sh : shards) std::sort(sh.begin(), sh.end());
    return shards;
}

bool sharding_active(int n_units) { return !g_extra.empty() && n_units >= 2 && t_ctx == &g_primary; }

struct SharedProgress {  // IProgressReport.ReportAdd from several worker threads, one at a time
    vgb_progress_cb cb;
    void *user;
    std::mutex mu;
    static void relay(void *self, int64_t delta)
    {
        auto *p = static_cast<SharedProgress *>(self);
        std::lock_guard<std::mutex> lock(p->mu);
        if (p->cb) p->cb(p->user, delta);
    }
};

// fn(device index, units) runs on a worker thread bound to that device's context; the first failure wins and its
// message is re-addressed from the shard-local unit index to the caller's.
template <class Fn>
int32_t run_sharded(const std::vector<std::vector<int>> &shards, Fn fn)
{
    const std::vector<Context *> ctxs = bound_contexts();
    const int n = (int)shards.size();
    std::vector<int32_t> rc(n, VGB_OK);
    std::vector<std::string> err(n);
    std::vector<std::thread> workers;
    for (int d = 0; d < n; d++) {
        if (shards[d].empty()) continue;
        workers.emplace_back([&, d]() {
            t_ctx = ctxs[d];
            rc[d] = fn(d, shards[d]);
            err[d] = g_err;
        });
    }
    for (auto &w : workers) w.join();
    for (int d = 0; d < n; d++)
        if (rc[d] != VGB_OK) {
            std::string m = err[d];
            for (const char *word : {"channel ", "stream "}) {
                const size_t len = std::strlen(word);
                if (m.compare(0, len, word) == 0) {
                    size_t end = len;
                    while (end < m.size() && m[end] >= '0' && m[end] <= '9') end++;
                    if (end > len) {
                        const int local = std::atoi(m.substr(len, end - len).c_str());
                        if (local >= 0 && local < (int)shards[d].size()) m = word + std::to_string(shards[d][local]) + m.substr(end);
                    }
                }
            }
            g_err = m + " (device " + std::to_string(ctxs[d]->device) + ")";
            return rc[d];
        }
    return VGB_OK;
}

template <class T>
std::vector<T> pick(const T *src, const std::vector<int> &units)
{
    std::vector<T> v(units.size());
    for (size_t i = 0; i < units.size(); i++) v[i] = src[units[i]];
    return v;
}

int32_t host_encode_sharded(const int16_t *const *pcm, const int32_t *n_samples, const vgb_gc_params *params,
                            const int16_t *coefs_in, int32_t n_channels, int16_t *coefs_out, uint8_t *const *adpcm_out,
                            vgb_progress_cb cb, void *user, bool do_encode)
{
    if (!sharding_active(n_channels) || !pcm || !n_samples || !coefs_out || (do_encode && !adpcm_out))
        return host_encode_impl(pcm, n_samples, params, coefs_in, n_channels, coefs_out, adpcm_out, cb, user, do_encode);
    std::vector<int64_t> weight(n_channels);
    for (int c = 0; c < n_channels; c++) weight[c] = (int64_t)std::max(n_samples[c], 0) + 64;
    const auto shards = shard_units(weight, 1 + (int)g_extra.size());
    SharedProgress prog{cb, user, {}};
    return run_sharded(shards, [&](int, const std::vector<int> &u) -> int32_t {
        const int m = (int)u.size();
        auto s_pcm = pick(pcm, u);
        auto s_n = pick(n_samples, u);
        std::vector<vgb_gc_params> s_par;
        if (params) s_par = pick(params, u);
        std::vector<int16_t> s_cin, s_cout((size_t)m * 16);
        if (coefs_in) {
            s_cin.resize((size_t)m * 16);
            for (int i = 0; i < m; i++) std::memcpy(&s_cin[(size_t)i * 16], coefs_in + (size_t)u[i] * 16, 32);
        }
        std::vector<uint8_t *> s_out;
        if (do_encode) s_out = pick(adpcm_out, u);
        VGB_TRY(host_encode_impl(s_pcm.data(), s_n.data(), params ? s_par.data() : nullptr, coefs_in ? s_cin.data() : nullptr, m,
                                 s_cout.data(), do_encode ? s_out.data() : nullptr, cb ? SharedProgress::relay : nullptr, &prog, do_encode));
        for (int i = 0; i < m; i++) std::memcpy(coefs_out + (size_t)u[i] * 16, &s_cout[(size_t)i * 16], 32);
        return VGB_OK;
    });
}

}  // namespace

// ==========================================================================================================
// extern "C"
// ==========================================================================================================
extern "C" {

int32_t vgb_abi_version(void) { return VGB_ABI_VERSION; }

const char *vgb_last_error(void) { return g_err.c_str(); }

int32_t vgb_init(int32_t device, uint32_t flags)
{
    (void)flags;
    if (device < 0) return fail(VGB_E_ARG, "device must be >= 0 (got %d)", device);
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    if (g_ctx.ready && g_ctx.device != device)
        return fail(VGB_E_STATE, "already bound to device %d; call vgb_shutdown first", g_ctx.device);
    g_ctx.device = device;
    return ensure_ready_locked();
}

static int32_t shutdown_current(void)  // releases the context this thread points at
{
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    if (!g_ctx.ready) return VGB_OK;
    cudaSetDevice(g_ctx.device);
    cudaStreamSynchronize(g_ctx.stream);
    cudaStreamSynchronize(g_ctx.s_in);
    for (auto st : g_ctx.s_comp) cudaStreamSynchronize(st);
    cudaStreamSynchronize(g_ctx.s_out);
    g_ctx.pcm.release();
    g_ctx.adpcm.release();
    g_ctx.coefs.release();
    g_ctx.ws.release();
    g_ctx.misc.release();
    for (auto &ev : g_ctx.ev) {
        if (ev) cudaEventDestroy(ev);
        ev = nullptr;
    }
    cudaStreamDestroy(g_ctx.stream);
    g_ctx.stream = nullptr;
    cudaStreamDestroy(g_ctx.s_in);
    cudaStreamDestroy(g_ctx.s_out);
    for (int g = 0; g < kCompStreams; g++) cudaStreamDestroy(g_ctx.s_comp[g]);
    for (int g = 0; g < kMaxGroups; g++) {
        cudaEventDestroy(g_ctx.ev_in[g]);
        cudaEventDestroy(g_ctx.ev_done[g]);
        cudaEventDestroy(g_ctx.ev_out[g]);
        cudaEventDestroy(g_ctx.ev_mid[g]);
    }
    if (g_ctx.ev_t0) cudaEventDestroy(g_ctx.ev_t0);
    g_ctx.ev_t0 = nullptr;
    hca_tables_release_locked();
    g_ctx.ready = false;
    return VGB_OK;
}

int32_t vgb_shutdown(void)
{
    vgb::containers_release();  // containers.cu keeps its own slabs and streams on the primary device
    for (auto &c : g_extra) {
        t_ctx = c.get();
        shutdown_current();
    }
    g_extra.clear();
    t_ctx = &g_primary;
    return shutdown_current();
}

}  // extern "C"

namespace vgb {  // hooks for containers.cu
int32_t abi_ensure_ready()
{
    Context &c = g_primary;
    std::lock_guard<std::mutex> lock(c.mu);
    Context *saved = t_ctx;
    t_ctx = &c;
    const int32_t s = ensure_ready_locked();
    t_ctx = saved;
    return s;
}
void abi_count_launches(int n) { g_primary.launches += n; }
}  // namespace vgb

extern "C" {

/* Bind several devices (SURVEY §8b: vgb_init(n_devices, flags)).  devices[0] becomes the primary device - the one the
 * *_dev entry points, the timers and the debug taps refer to; every host-pointer *_batch call is then sharded over all
 * of them (greedy longest-first over the units' sample counts, one worker thread and one H2D / kernel / D2H pipeline per
 * device, results written straight into the caller's arrays).  A device may be listed more than once (two pipelines on
 * one GPU; also how the sharding logic is tested on a single-GPU machine). */
int32_t vgb_init_devices(const int32_t *devices, int32_t n_devices, uint32_t flags)
{
    (void)flags;
    if (!devices || n_devices < 1) return fail(VGB_E_ARG, "at least one device is required");
    if (n_devices > 64) return fail(VGB_E_ARG, "too many devices (%d)", n_devices);
    for (int i = 0; i < n_devices; i++)
        if (devices[i] < 0) return fail(VGB_E_ARG, "device must be >= 0 (got %d)", devices[i]);
    if (t_ctx != &g_primary) return fail(VGB_E_STATE, "vgb_init_devices called from a worker thread");
    if (!g_extra.empty() || (g_primary.ready && g_primary.device != devices[0]))
        return fail(VGB_E_STATE, "already bound; call vgb_shutdown first");
    VGB_TRY(vgb_init(devices[0], flags));
    for (int i = 1; i < n_devices; i++) {
        g_extra.emplace_back(new Context());
        g_extra.back()->device = devices[i];
        t_ctx = g_extra.back().get();
        int32_t rc;
        {
            std::lock_guard<std::mutex> lock(g_ctx.mu);
            rc = ensure_ready_locked();
        }
        t_ctx = &g_primary;
        if (rc != VGB_OK) {
            const std::string keep = g_err;
            vgb_shutdown();
            g_err = keep;
            return rc;
        }
    }
    cudaSetDevice(g_primary.device);
    return VGB_OK;
}

int32_t vgb_device_count(void) { return g_primary.ready ? 1 + (int32_t)g_extra.size() : 0; }

int32_t vgb_host_alloc(void **ptr_out, uint64_t bytes)
{
    if (!ptr_out) return fail(VGB_E_ARG, "ptr_out is NULL");
    {
        std::lock_guard<std::mutex> lock(g_ctx.mu);
        VGB_TRY(ensure_ready_locked());
    }
    CUDA_TRY(cudaHostAlloc(ptr_out, bytes ? bytes : 1, cudaHostAllocDefault));
    return VGB_OK;
}

int32_t vgb_host_free(void *ptr)
{
    if (!ptr) return VGB_OK;
    CUDA_TRY(cudaFreeHost(ptr));
    return VGB_OK;
}

int64_t vgb_kernel_launch_count(void)
{
    int64_t n = g_primary.launches.load();
    for (auto &c : g_extra) n += c->launches.load();
    return n;
}

int32_t vgb_gcadpcm_sample_count_to_byte_count(int32_t n) { return gc_sample_count_to_byte_count(n); }
int32_t vgb_gcadpcm_byte_count_to_sample_count(int32_t b) { return gc_nibble_count_to_sample_count(b * 2); }
int32_t vgb_gcadpcm_sample_count_to_nibble_count(int32_t n) { return gc_sample_count_to_nibble_count(n); }
int32_t vgb_gcadpcm_nibble_count_to_sample_count(int32_t n) { return gc_nibble_count_to_sample_count(n); }
int32_t vgb_gcadpcm_sample_to_nibble(int32_t s)
{
    return kGcFrameNibbles * (s / kGcFrameSamples) + s % kGcFrameSamples + 2;
}
int32_t vgb_gcadpcm_nibble_to_sample(int32_t nib)
{
    return kGcFrameSamples * (nib / kGcFrameNibbles) + nib % kGcFrameNibbles - 2;
}

int32_t vgb_gcadpcm_coefs_batch(const int16_t *const *pcm, const int32_t *n_samples, int32_t n_channels,
                                int16_t *coefs_out)
{
    return host_encode_sharded(pcm, n_samples, nullptr, nullptr, n_channels, coefs_out, nullptr, nullptr, nullptr, false);
}

int32_t vgb_gcadpcm_encode_batch(const int16_t *const *pcm, const int32_t *n_samples, const vgb_gc_params *params,
                                 const int16_t *coefs_in, int32_t n_channels, int16_t *coefs_out,
                                 uint8_t *const *adpcm_out, vgb_progress_cb cb, void *user)
{
    return host_encode_sharded(pcm, n_samples, params, coefs_in, n_channels, coefs_out, adpcm_out, cb, user, true);
}

static int32_t gcadpcm_decode_one(const uint8_t *const *adpcm, const int32_t *n_bytes, const int16_t *coefs,
                                  const vgb_gc_params *params, int32_t n_channels, int16_t *const *pcm_out)
{
    PinScope pins;
    if (n_channels < 0) return fail(VGB_E_ARG, "n_channels is negative (%d)", n_channels);
    if (n_channels == 0) return VGB_OK;
    if (!adpcm || !n_bytes || !coefs || !pcm_out) return fail(VGB_E_ARG, "NULL argument");
    std::vector<int32_t> counts(n_channels);
    for (int c = 0; c < n_channels; c++) {
        if (n_bytes[c] < 0) return fail(VGB_E_ARG, "channel %d: negative byte count", c);
        int32_t want = (params && params[c].sample_count != -1) ? params[c].sample_count
                                                                : gc_nibble_count_to_sample_count(n_bytes[c] * 2);
        if (want < 0) return fail(VGB_E_ARG, "channel %d: negative sample count %d", c, want);
        // GcAdpcmChannel.cs:33-36: "Audio array length is too short for the specified number of samples."
        if (n_bytes[c] < gc_sample_count_to_byte_count(want))
            return fail(VGB_E_ARG, "channel %d: audio array length %d is too short for %d samples", c, n_bytes[c], want);
        if ((!adpcm[c] || !pcm_out[c]) && want > 0) return fail(VGB_E_ARG, "channel %d: NULL buffer", c);
        counts[c] = want;
    }
    GcLayout lay;
    VGB_TRY(layout_common(lay, counts.data(), params, n_channels, true));
    layout_pack_offsets(lay);

    // channel groups: H2D of the ADPCM of group g+1 || decode of group g || D2H of the PCM of group g-1
    std::vector<int64_t> weight(n_channels);
    int64_t pcie_bytes = 0;
    for (int c = 0; c < n_channels; c++) {
        weight[c] = (int64_t)counts[c] + 64;
        pcie_bytes += (int64_t)counts[c] * 2 + gc_sample_count_to_byte_count(counts[c]);
    }
    const int n_groups = pipeline_group_count(n_channels, pcie_bytes, 32);
    const std::vector<int> bound = pipeline_bounds(weight, n_groups);

    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    std::vector<GcLayout> glay(n_groups);
    std::vector<GcWorkspace> gws(n_groups);
    std::vector<size_t> ws_at(n_groups);
    size_t ws_total = 0;
    for (int g = 0; g < n_groups; g++) {
        glay[g] = sub_layout(lay, bound[g], bound[g + 1]);
        gws[g] = carve(32, glay[g].n_channels);
        ws_at[g] = ws_total;
        ws_total += align_up(gws[g].total, 256);
    }
    VGB_TRY(g_ctx.pcm.reserve((size_t)lay.pcm_total * 2));
    VGB_TRY(g_ctx.adpcm.reserve((size_t)lay.adpcm_total));
    VGB_TRY(g_ctx.coefs.reserve((size_t)n_channels * 32 * 2));
    VGB_TRY(g_ctx.ws.reserve(ws_total));
    char *ws_base = static_cast<char *>(g_ctx.ws.p);
    int16_t *d_coefs = static_cast<int16_t *>(g_ctx.coefs.p);
    std::vector<int32_t> bad(n_groups, INT_MAX);

    auto h2d = [&](int g) -> int32_t {
        const int c0 = bound[g], n = bound[g + 1] - c0;
        if (g == 0) {  // the small tables first, while the copy stream is idle
            for (int k = 0; k < n_groups; k++) VGB_TRY(upload_tables(glay[k], gws[k], ws_base + ws_at[k], g_ctx.s_in));
            CUDA_TRY(cudaMemcpyAsync(d_coefs, coefs, (size_t)n_channels * 32, cudaMemcpyHostToDevice, g_ctx.s_in));
        }
        std::vector<int64_t> off_b(n), len_b(n);
        for (int c = 0; c < n; c++) { off_b[c] = lay.adpcm_off[c0 + c]; len_b[c] = gc_sample_count_to_byte_count(counts[c0 + c]); }
        return copy_channels_in(static_cast<char *>(g_ctx.adpcm.p), off_b, adpcm + c0, len_b, g_ctx.s_in);
    };
    auto kern = [&](int g, cudaStream_t st) -> int32_t {
        if (glay[g].n_channels == 0) return VGB_OK;
        GcChannelTable tab = table_view(ws_base + ws_at[g], gws[g], glay[g].n_channels);
        CUDA_TRY(cudaMemsetAsync(tab.status, 0x7f, 4, st));  // "no channel": any index is smaller
        if (n_groups == 1) tick(3, true, st);  // the kernel timers describe unpipelined calls only
        launch_gc_decode(static_cast<const uint8_t *>(g_ctx.adpcm.p), tab, d_coefs + (size_t)bound[g] * 16,
                         static_cast<int16_t *>(g_ctx.pcm.p), glay[g].max_frames, 0, INT_MAX, st);
        if (n_groups == 1) tick(3, false, st);
        g_ctx.launches += glay[g].max_frames > 0 ? 1 : 0;
        CUDA_TRY(cudaGetLastError());
        return VGB_OK;
    };
    auto d2h = [&](int g) -> int32_t {
        const int c0 = bound[g], n = bound[g + 1] - c0;
        std::vector<int64_t> off_b(n), len_b(n);
        for (int c = 0; c < n; c++) { off_b[c] = lay.pcm_off[c0 + c] * 2; len_b[c] = (int64_t)counts[c0 + c] * 2; }
        VGB_TRY(copy_channels_out(pcm_out + c0, static_cast<const char *>(g_ctx.pcm.p), off_b, len_b, g_ctx.s_out));
        if (n > 0) CUDA_TRY(cudaMemcpyAsync(&bad[g], ws_base + ws_at[g] + gws[g].off_status, 4, cudaMemcpyDeviceToHost, g_ctx.s_out));
        return VGB_OK;
    };
    VGB_TRY(run_group_pipeline(n_groups, h2d, kern, d2h, [](int) { return VGB_OK; }));
    // coefs[predictor * 2] with predictor 8..15 is an IndexOutOfRangeException in GcAdpcmDecoder.Decode (:31-32)
    for (int g = 0; g < n_groups; g++)
        if (bad[g] >= 0 && bad[g] < glay[g].n_channels)
            return fail(VGB_E_DATA, "channel %d: a frame header selects a predictor outside 0..7", bound[g] + bad[g]);
    return VGB_OK;
}

int32_t vgb_gcadpcm_seek_entry_count(int32_t sample_count, int32_t samples_per_entry)
{
    if (samples_per_entry <= 0 || sample_count <= 0) return 0;
    return div_round_up(sample_count, samples_per_entry);
}

int32_t vgb_gcadpcm_seek_context_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int16_t *coefs,
                                       const vgb_gc_tap_params *params, int32_t n_channels,
                                       int16_t *const *seek_table_out, int16_t *loop_context_out)
{
    PinScope pins;
    if (n_channels < 0) return fail(VGB_E_ARG, "n_channels is negative (%d)", n_channels);
    if (n_channels == 0) return VGB_OK;
    if (!adpcm || !n_bytes || !coefs || !params) return fail(VGB_E_ARG, "NULL argument");
    std::vector<int32_t> counts(n_channels);
    std::vector<GcTapChannel> taps(n_channels);
    std::vector<int64_t> tap_off(n_channels), tap_len(n_channels);
    int64_t slab = 0;
    bool any_loop = false;
    for (int c = 0; c < n_channels; c++) {
        const vgb_gc_tap_params &p = params[c];
        if (p.sample_count < 0 || n_bytes[c] < 0) return fail(VGB_E_ARG, "channel %d: negative count", c);
        if (p.samples_per_seek_table_entry < 0) return fail(VGB_E_ARG, "channel %d: negative samples per seek table entry", c);
        if (n_bytes[c] < gc_sample_count_to_byte_count(p.sample_count))
            return fail(VGB_E_ARG, "channel %d: audio array length %d is too short for %d samples", c, n_bytes[c], p.sample_count);
        if (!adpcm[c] && p.sample_count > 0) return fail(VGB_E_ARG, "channel %d: NULL buffer", c);
        if (p.loop_start > p.sample_count) return fail(VGB_E_ARG, "channel %d: loop start %d past the end (%d samples)", c, p.loop_start, p.sample_count);
        counts[c] = p.sample_count;
        const int entries = vgb_gcadpcm_seek_entry_count(p.sample_count, p.samples_per_seek_table_entry);
        if (entries > 0 && (!seek_table_out || !seek_table_out[c])) return fail(VGB_E_ARG, "channel %d: seek_table_out is NULL", c);
        if (p.loop_start >= 0) any_loop = true;
        taps[c].out_off = slab;
        taps[c].samples_per_entry = p.sample_count > 0 ? p.samples_per_seek_table_entry : 0;
        taps[c].loop_start = p.loop_start;
        tap_off[c] = slab * 2;
        tap_len[c] = (int64_t)entries * 4;
        slab += (int64_t)align_up((size_t)entries * 2 + 2, 8);
    }
    if (any_loop && !loop_context_out) return fail(VGB_E_ARG, "loop_context_out is NULL");
    GcLayout lay;
    VGB_TRY(layout_common(lay, counts.data(), nullptr, n_channels, true));
    layout_pack_offsets(lay);

    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    cudaStream_t st = g_ctx.stream;
    const GcWorkspace w = carve(32, n_channels);
    const size_t o_taps = align_up((size_t)slab * 2 + 16, 256);
    VGB_TRY(g_ctx.adpcm.reserve((size_t)lay.adpcm_total));
    VGB_TRY(g_ctx.coefs.reserve((size_t)n_channels * 32 * 2));
    VGB_TRY(g_ctx.ws.reserve(w.total));
    VGB_TRY(g_ctx.misc.reserve(o_taps + taps.size() * sizeof(GcTapChannel)));
    char *misc = static_cast<char *>(g_ctx.misc.p);
    std::vector<int64_t> off_b(n_channels), len_b(n_channels);
    for (int c = 0; c < n_channels; c++) { off_b[c] = lay.adpcm_off[c]; len_b[c] = gc_sample_count_to_byte_count(counts[c]); }
    VGB_TRY(copy_channels_in(static_cast<char *>(g_ctx.adpcm.p), off_b, adpcm, len_b, st));
    CUDA_TRY(cudaMemcpyAsync(g_ctx.coefs.p, coefs, (size_t)n_channels * 32, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(misc + o_taps, taps.data(), taps.size() * sizeof(GcTapChannel), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(misc, 0, (size_t)slab * 2, st));  // entry 0 and absent history samples are zero
    VGB_TRY(upload_tables(lay, w, g_ctx.ws.p, st));
    GcChannelTable tab = table_view(g_ctx.ws.p, w, lay.n_channels);
    CUDA_TRY(cudaMemsetAsync(tab.status, 0x7f, 4, st));
    launch_gc_taps(static_cast<const uint8_t *>(g_ctx.adpcm.p), tab, static_cast<const int16_t *>(g_ctx.coefs.p),
                   reinterpret_cast<const GcTapChannel *>(misc + o_taps), reinterpret_cast<int16_t *>(misc), lay.max_frames, st);
    g_ctx.launches += lay.max_frames > 0 ? 1 : 0;
    CUDA_TRY(cudaGetLastError());
    if (seek_table_out) VGB_TRY(copy_channels_out(seek_table_out, misc, tap_off, tap_len, st));
    std::vector<int16_t> host_slab;
    if (any_loop) {
        host_slab.resize((size_t)slab);
        CUDA_TRY(cudaMemcpyAsync(host_slab.data(), misc, (size_t)slab * 2, cudaMemcpyDeviceToHost, st));
    }
    int32_t bad_channel = INT_MAX;
    CUDA_TRY(cudaMemcpyAsync(&bad_channel, tab.status, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (bad_channel >= 0 && bad_channel < n_channels)  // the reference's EnsurePcmDecoded would throw inside Decode
        return fail(VGB_E_DATA, "channel %d: a frame header selects a predictor outside 0..7", bad_channel);
    if (loop_context_out)
        for (int c = 0; c < n_channels; c++) {
            int16_t *ctx = loop_context_out + (size_t)c * 3;
            ctx[0] = ctx[1] = ctx[2] = 0;
            const int32_t ls = params[c].loop_start;
            if (ls < 0 || counts[c] == 0) continue;
            const int64_t frame_byte = (int64_t)(ls / kGcFrameSamples) * kGcFrameBytes;  // GcAdpcmDecoder.GetPredictorScale (:56-59)
            if (frame_byte >= n_bytes[c]) return fail(VGB_E_ARG, "channel %d: loop start %d has no frame header in %d bytes", c, ls, n_bytes[c]);
            ctx[0] = adpcm[c][frame_byte];
            const int entries = vgb_gcadpcm_seek_entry_count(counts[c], params[c].samples_per_seek_table_entry);
            ctx[1] = host_slab[(size_t)taps[c].out_off + 2 * entries];
            ctx[2] = host_slab[(size_t)taps[c].out_off + 2 * entries + 1];
        }
    return VGB_OK;
}

int32_t vgb_gcadpcm_encode_frames(int16_t *pcm_in_out, const int32_t *sample_count, const int16_t *coefs,
                                  int32_t n_frames, uint8_t *adpcm_out)
{
    if (n_frames < 0) return fail(VGB_E_ARG, "n_frames is negative");
    if (n_frames == 0) return VGB_OK;
    if (!pcm_in_out || !coefs || !adpcm_out) return fail(VGB_E_ARG, "NULL argument");
    if (sample_count)
        for (int f = 0; f < n_frames; f++)
            if (sample_count[f] < 0 || sample_count[f] > 14)
                return fail(VGB_E_ARG, "frame %d: sample_count %d outside 0..14", f, sample_count[f]);
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    cudaStream_t st = g_ctx.stream;
    const size_t n = (size_t)n_frames;
    const size_t o_pcm = 0, o_coef = align_up(n * 32, 256), o_cnt = o_coef + align_up(n * 32, 256),
                 o_out = o_cnt + align_up(n * 4, 256), total = o_out + align_up(n * 8, 256);
    VGB_TRY(g_ctx.misc.reserve(total));
    char *b = static_cast<char *>(g_ctx.misc.p);
    CUDA_TRY(cudaMemcpyAsync(b + o_pcm, pcm_in_out, n * 32, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(b + o_coef, coefs, n * 32, cudaMemcpyHostToDevice, st));
    if (sample_count) CUDA_TRY(cudaMemcpyAsync(b + o_cnt, sample_count, n * 4, cudaMemcpyHostToDevice, st));
    launch_gc_encode_frames(reinterpret_cast<int16_t *>(b + o_pcm),
                            sample_count ? reinterpret_cast<const int32_t *>(b + o_cnt) : nullptr,
                            reinterpret_cast<const int16_t *>(b + o_coef), n_frames,
                            reinterpret_cast<uint8_t *>(b + o_out), st);
    g_ctx.launches += 1;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(pcm_in_out, b + o_pcm, n * 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(adpcm_out, b + o_out, n * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return VGB_OK;
}

// ---- device-resident entry points --------------------------------------------------------------------------

uint64_t vgb_gcadpcm_workspace_bytes(int64_t total_frames, int32_t n_channels)
{
    if (total_frames < 0 || n_channels < 0) return 0;
    return carve(padded_rec_bound(total_frames, n_channels), n_channels).total;
}

static int32_t dev_layout(GcLayout &lay, const int64_t *pcm_offset, const int64_t *adpcm_offset,
                          const int32_t *n_samples, const vgb_gc_params *params, int32_t n_channels, bool decode,
                          bool need_adpcm)
{
    VGB_TRY(layout_common(lay, n_samples, params, n_channels, decode));
    if (n_channels == 0) return VGB_OK;
    if (!pcm_offset) return fail(VGB_E_ARG, "pcm_offset is NULL");
    if (need_adpcm && !adpcm_offset) return fail(VGB_E_ARG, "adpcm_offset is NULL");
    lay.pcm_off.assign(pcm_offset, pcm_offset + n_channels);
    lay.adpcm_off.assign(n_channels, 0);
    if (adpcm_offset) lay.adpcm_off.assign(adpcm_offset, adpcm_offset + n_channels);
    for (int c = 0; c < n_channels; c++) {
        if (lay.pcm_off[c] < 0 || (lay.pcm_off[c] & 7))
            return fail(VGB_E_ARG, "pcm_offset[%d]=%lld must be a non-negative multiple of 8 samples", c,
                        (long long)lay.pcm_off[c]);
        if (lay.adpcm_off[c] < 0 || (lay.adpcm_off[c] & 15))
            return fail(VGB_E_ARG, "adpcm_offset[%d]=%lld must be a non-negative multiple of 16 bytes", c,
                        (long long)lay.adpcm_off[c]);
    }
    return VGB_OK;
}

int32_t vgb_gcadpcm_encode_dev(const int16_t *d_pcm, const int64_t *pcm_offset, const int32_t *n_samples,
                               const vgb_gc_params *params, int32_t n_channels, const int16_t *d_coefs_in,
                               int16_t *d_coefs_out, uint8_t *d_adpcm, const int64_t *adpcm_offset, void *d_workspace,
                               uint64_t workspace_bytes, void *cuda_stream)
{
    GcLayout lay;
    VGB_TRY(dev_layout(lay, pcm_offset, adpcm_offset, n_samples, params, n_channels, false, true));
    if (n_channels == 0) return VGB_OK;
    if (!d_pcm || !d_coefs_out || !d_adpcm || !d_workspace) return fail(VGB_E_ARG, "NULL device pointer");
    const GcWorkspace w = carve(lay.rec_total, n_channels);
    if (w.total > workspace_bytes)
        return fail(VGB_E_ARG, "workspace too small: need %zu bytes, got %llu", w.total, (unsigned long long)workspace_bytes);
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    return run_gc_encode(d_pcm, lay, d_coefs_in, d_coefs_out, d_adpcm, d_workspace, w, static_cast<cudaStream_t>(cuda_stream), true);
}

int32_t vgb_gcadpcm_coefs_dev(const int16_t *d_pcm, const int64_t *pcm_offset, const int32_t *n_samples,
                              int32_t n_channels, int16_t *d_coefs_out, void *d_workspace, uint64_t workspace_bytes,
                              void *cuda_stream)
{
    GcLayout lay;
    VGB_TRY(dev_layout(lay, pcm_offset, nullptr, n_samples, nullptr, n_channels, false, false));
    if (n_channels == 0) return VGB_OK;
    if (!d_pcm || !d_coefs_out || !d_workspace) return fail(VGB_E_ARG, "NULL device pointer");
    const GcWorkspace w = carve(lay.rec_total, n_channels);
    if (w.total > workspace_bytes)
        return fail(VGB_E_ARG, "workspace too small: need %zu bytes, got %llu", w.total, (unsigned long long)workspace_bytes);
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    return run_gc_encode(d_pcm, lay, nullptr, d_coefs_out, nullptr, d_workspace, w, static_cast<cudaStream_t>(cuda_stream), false);
}

int32_t vgb_gcadpcm_decode_dev(const uint8_t *d_adpcm, const int64_t *adpcm_offset, const int16_t *d_coefs,
                               const vgb_gc_params *params, int32_t n_channels, int16_t *d_pcm,
                               const int64_t *pcm_offset, void *d_workspace, uint64_t workspace_bytes, void *cuda_stream)
{
    if (n_channels < 0) return fail(VGB_E_ARG, "n_channels is negative");
    if (n_channels == 0) return VGB_OK;
    if (!params) return fail(VGB_E_ARG, "params is NULL (sample counts are required)");
    std::vector<int32_t> counts(n_channels);
    for (int c = 0; c < n_channels; c++) {
        if (params[c].sample_count < 0) return fail(VGB_E_ARG, "channel %d: sample_count must be >= 0", c);
        counts[c] = params[c].sample_count;
    }
    GcLayout lay;
    VGB_TRY(dev_layout(lay, pcm_offset, adpcm_offset, counts.data(), params, n_channels, true, true));
    if (!d_pcm || !d_coefs || !d_adpcm || !d_workspace) return fail(VGB_E_ARG, "NULL device pointer");
    const GcWorkspace w = carve(32, n_channels);
    if (w.total > workspace_bytes)
        return fail(VGB_E_ARG, "workspace too small: need %zu bytes, got %llu", w.total, (unsigned long long)workspace_bytes);
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    return run_gc_decode(d_adpcm, lay, d_coefs, d_pcm, d_workspace, w, static_cast<cudaStream_t>(cuda_stream));
}

/* The decoder's status word of the most recent vgb_gcadpcm_decode_dev on this workspace (see the header). */
int32_t vgb_gcadpcm_decode_dev_status(const void *d_workspace, int32_t n_channels, void *cuda_stream)
{
    if (!d_workspace || n_channels < 0) return fail(VGB_E_ARG, "bad arguments");
    if (n_channels == 0) return VGB_OK;
    const GcWorkspace w = carve(32, n_channels);
    const GcChannelTable tab = table_view(const_cast<void *>(d_workspace), w, n_channels);
    int32_t bad_channel = INT_MAX;
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    CUDA_TRY(cudaMemcpyAsync(&bad_channel, tab.status, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (bad_channel >= 0 && bad_channel < n_channels)  // IndexOutOfRangeException at GcAdpcmDecoder.cs:31-32
        return fail(VGB_E_DATA, "channel %d: a frame header selects a predictor outside 0..7", bad_channel);
    return VGB_OK;
}

int32_t vgb_set_kernel_timing(int32_t enabled)
{
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    g_ctx.timing = enabled != 0;
    for (auto &u : g_ctx.ev_used) u = false;
    return VGB_OK;
}

int32_t vgb_last_kernel_ms(float *ms_out, int32_t n)
{
    if (!ms_out || n < 0) return fail(VGB_E_ARG, "bad arguments");
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    for (int i = 0; i < n; i++) ms_out[i] = 0.0f;
    if (!g_ctx.ready) return VGB_OK;
    for (int i = 0; i < n && i < kTimers; i++) {
        if (!g_ctx.ev_used[i]) continue;
        CUDA_TRY(cudaEventSynchronize(g_ctx.ev[2 * i + 1]));
        CUDA_TRY(cudaEventElapsedTime(&ms_out[i], g_ctx.ev[2 * i], g_ctx.ev[2 * i + 1]));
        g_ctx.ev_used[i] = false;
    }
    return VGB_OK;
}

/* Device timeline of the last host encode call (ms since its first copy was enqueued): for each channel group
 * [H2D landed, kernels finished, D2H finished].  bench.py prints it as evidence of the copy/compute overlap. */
int32_t vgb_debug_last_timeline(float *ms_out, int32_t n)
{
    if (!ms_out || n < 0) return fail(VGB_E_ARG, "bad arguments");
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    for (int i = 0; i < n; i++) ms_out[i] = -1.0f;
    if (!g_ctx.ready) return VGB_OK;
    for (int g = 0; g < g_ctx.last_groups && 3 * g + 2 < n; g++) {
        CUDA_TRY(cudaEventElapsedTime(&ms_out[3 * g], g_ctx.ev_t0, g_ctx.ev_in[g]));
        CUDA_TRY(cudaEventElapsedTime(&ms_out[3 * g + 1], g_ctx.ev_t0, g_ctx.ev_done[g]));
        CUDA_TRY(cudaEventElapsedTime(&ms_out[3 * g + 2], g_ctx.ev_t0, g_ctx.ev_out[g]));
    }
    return VGB_OK;
}

int32_t vgb_debug_last_coefs_done(float *ms_out, int32_t n)
{
    if (!ms_out || n < 0) return fail(VGB_E_ARG, "bad arguments");
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    for (int i = 0; i < n; i++) ms_out[i] = -1.0f;
    if (!g_ctx.ready) return VGB_OK;
    for (int g = 0; g < g_ctx.last_groups && g < n; g++)
        CUDA_TRY(cudaEventElapsedTime(&ms_out[g], g_ctx.ev_t0, g_ctx.ev_mid[g]));
    return VGB_OK;
}

/* Bookkeeping of the most recent time-parallel encode launch (see the header).  Synchronises the device. */
int32_t vgb_gcadpcm_debug_splice_stats(uint64_t *out, int32_t n)
{
    if (!out || n < 0) return fail(VGB_E_ARG, "bad arguments");
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    for (int i = 0; i < n; i++) out[i] = 0;
    if (!g_ctx.ready || !g_ctx.last_seg.stats) return VGB_OK;
    unsigned long long st[kGcStatWords] = {};
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(st, g_ctx.last_seg.stats, sizeof st, cudaMemcpyDeviceToHost));
    if (n > 0) out[0] = (uint64_t)g_ctx.last_seg.seg_count;
    for (int i = 1; i < n && i <= kGcStatWords; i++) out[i] = st[i - 1];
    return VGB_OK;
}

int32_t vgb_gcadpcm_debug_records(const int16_t *pcm, int32_t n_samples, double *dir_out, uint8_t *accepted_out)
{
    if (n_samples < 0 || (!pcm && n_samples > 0) || !dir_out || !accepted_out) return fail(VGB_E_ARG, "bad arguments");
    GcLayout lay;
    VGB_TRY(layout_common(lay, &n_samples, nullptr, 1, false));
    layout_pack_offsets(lay);
    const int frames = div_round_up(n_samples, kGcFrameSamples);
    if (frames == 0) return VGB_OK;
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    cudaStream_t st = g_ctx.stream;
    const GcWorkspace w = carve(lay.rec_total, 1);
    VGB_TRY(g_ctx.pcm.reserve((size_t)lay.pcm_total * 2));
    VGB_TRY(g_ctx.ws.reserve(w.total));
    CUDA_TRY(cudaMemcpyAsync(g_ctx.pcm.p, pcm, (size_t)n_samples * 2, cudaMemcpyHostToDevice, st));
    VGB_TRY(upload_tables(lay, w, g_ctx.ws.p, st));
    GcChannelTable tab = table_view(g_ctx.ws.p, w, 1);
    char *b = static_cast<char *>(g_ctx.ws.p);
    launch_gc_coef_frames(static_cast<const int16_t *>(g_ctx.pcm.p), tab, reinterpret_cast<double2 *>(b + w.off_records),
                          reinterpret_cast<uint32_t *>(b + w.off_mask), frames, 0, INT_MAX, st);
    g_ctx.launches += 1;
    CUDA_TRY(cudaGetLastError());
    std::vector<uint32_t> mask((size_t)frames / 32 + 1);
    CUDA_TRY(cudaMemcpyAsync(dir_out, b + w.off_records, (size_t)frames * 16, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(mask.data(), b + w.off_mask, mask.size() * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    for (int f = 0; f < frames; f++) accepted_out[f] = (mask[f >> 5] >> (f & 31)) & 1u;
    return VGB_OK;
}

// ---- CRI ADX --------------------------------------------------------------------------------------------------

int32_t vgb_adx_encoded_byte_count(int32_t pcm_length, int32_t padding, int32_t frame_size)
{
    if (pcm_length < 0 || padding < 0 || frame_size < 3) return 0;
    const int32_t spf = (frame_size - 2) * 2;
    return (int32_t)(((int64_t)pcm_length + padding + spf - 1) / spf) * frame_size;
}

}  // extern "C"

namespace {

// CriAdxCodec.CalculateCoefficients (CriAdxCodec.cs:173-184): host double math, once per distinct (freq, rate).
// (short)(double) goes through (int) truncation like the oracle.
void adx_calc_coefs(int highpass, int rate, int16_t &c0, int16_t &c1)
{
    const double sqrt2 = std::sqrt(2.0);
    const double a = sqrt2 - std::cos(2.0 * 3.14159265358979323846 * highpass / rate);
    const double b = sqrt2 - 1;
    const double c = (a - std::sqrt((a + b) * (a - b))) / b;
    c0 = (int16_t)(int32_t)(c * 8192);
    c1 = (int16_t)(int32_t)(c * c * -4096);
}

int32_t adx_validate(const vgb_adx_params &p, int c)
{
    if (p.frame_size < 3 || p.frame_size > 255) return fail(VGB_E_ARG, "channel %d: frame_size %d outside 3..255", c, p.frame_size);
    if (p.type != 2 && p.type != 3 && p.type != 4) return fail(VGB_E_ARG, "channel %d: unknown CriAdxType %d", c, p.type);
    if (p.type == 2 && (p.filter < 0 || p.filter > 3)) return fail(VGB_E_ARG, "channel %d: filter %d outside 0..3", c, p.filter);
    if (p.padding < 0) return fail(VGB_E_ARG, "channel %d: negative padding", c);
    if (p.sample_rate <= 0) return fail(VGB_E_ARG, "channel %d: sample_rate must be positive", c);
    return VGB_OK;
}

// Workspace of the time-parallel ADX encoder behind `base`: [trace: one word per whole standard-layout frame][used_start:
// n x kAdxMaxSegments][stats].  Fills trace_off of every row and returns the view; `bytes_out` = bytes needed.
AdxSegArgs adx_seg_carve(std::vector<AdxChannel> &tab, int first, int n, char *base, size_t &bytes_out)
{
    int64_t frames = 0;
    int max_whole = 0;
    for (int c = first; c < first + n; c++) {
        const bool standard = tab[c].frame_size == 18 && tab[c].padding == 0;
        const int whole = standard ? tab[c].n_samples / 32 : 0;
        tab[c].trace_off = frames;
        frames += whole;
        max_whole = std::max(max_whole, whole);
    }
    const size_t o_used = align_up((size_t)(frames + 1) * 4, 256);
    const size_t o_stats = o_used + align_up((size_t)std::max(n, 1) * kAdxMaxSegments * 4, 256);
    bytes_out = o_stats + 256;
    AdxSegArgs a{};
    a.trace = reinterpret_cast<uint32_t *>(base);
    a.used_start = reinterpret_cast<uint32_t *>(base + o_used);
    a.stats = reinterpret_cast<unsigned long long *>(base + o_stats);
    int min_seg = 0;
    a.seg_count = adx_encode_pick_segments(n, max_whole, &min_seg);
    a.min_seg_frames = min_seg;
    return a;
}

const int16_t kAdxFixed[4][2] = {{0, 0}, {0x0F00, 0}, {0x1CC0, (int16_t)0xF300}, {0x1880, (int16_t)0xF240}};

}  // namespace

extern "C" {

int32_t vgb_adx_calculate_coefficients(int32_t highpass_frequency, int32_t sample_rate, int16_t *coefs_out)
{
    if (!coefs_out) return fail(VGB_E_ARG, "coefs_out is NULL");
    if (sample_rate <= 0) return fail(VGB_E_ARG, "sample rate must be positive");
    adx_calc_coefs(highpass_frequency, sample_rate, coefs_out[0], coefs_out[1]);
    return VGB_OK;
}

static int32_t adx_encode_one(const int16_t *const *pcm, const int32_t *n_samples, const vgb_adx_params *params,
                              int32_t n_channels, int16_t *history_out, uint8_t *const *adpcm_out, vgb_progress_cb cb,
                              void *user)
{
    PinScope pins;
    if (n_channels < 0) return fail(VGB_E_ARG, "n_channels is negative");
    if (n_channels == 0) return VGB_OK;
    if (!pcm || !n_samples || !params || !adpcm_out) return fail(VGB_E_ARG, "NULL argument");
    std::vector<AdxChannel> tab(n_channels);
    std::vector<int64_t> in_off(n_channels), in_len(n_channels), out_off(n_channels), out_len(n_channels);
    int64_t ps = 0, ab = 0, frames_total = 0;
    for (int c = 0; c < n_channels; c++) {
        const vgb_adx_params &p = params[c];
        VGB_TRY(adx_validate(p, c));
        if (n_samples[c] < 0) return fail(VGB_E_ARG, "channel %d: negative sample count", c);
        // CriAdxCodec.cs:69-74 reads pcm[0]: an empty array throws IndexOutOfRangeException there
        if (p.version == 4 && p.padding == 0 && n_samples[c] == 0)
            return fail(VGB_E_ARG, "channel %d: version 4 without padding needs at least one sample", c);
        if (!pcm[c] && n_samples[c] > 0) return fail(VGB_E_ARG, "pcm[%d] is NULL", c);
        AdxChannel &t = tab[c];
        t.pcm_off = ps; t.adpcm_off = ab; t.n_samples = n_samples[c];
        t.frame_size = p.frame_size; t.version = p.version; t.padding = p.padding; t.type = p.type; t.filter = p.filter;
        t.history = 0;
        if (p.type == 2) { t.coef0 = kAdxFixed[p.filter][0]; t.coef1 = kAdxFixed[p.filter][1]; }
        else adx_calc_coefs(500, p.sample_rate, t.coef0, t.coef1);  // Encode hard-codes 500 (:63)
        const int32_t bytes = vgb_adx_encoded_byte_count(n_samples[c], p.padding, p.frame_size);
        if (!adpcm_out[c] && bytes > 0) return fail(VGB_E_ARG, "adpcm_out[%d] is NULL", c);
        in_off[c] = ps * 2; in_len[c] = (int64_t)n_samples[c] * 2; out_off[c] = ab; out_len[c] = bytes;
        ps += (int64_t)align_up((size_t)n_samples[c], 8);
        ab += (int64_t)align_up((size_t)bytes, 16);
        frames_total += bytes / p.frame_size;
    }
    // channel groups: H2D of group g+1 || encode of group g || D2H of group g-1
    std::vector<int64_t> weight(n_channels);
    int64_t pcie_bytes = 0;
    for (int c = 0; c < n_channels; c++) { weight[c] = in_len[c] + 64; pcie_bytes += in_len[c] + out_len[c]; }
    const int n_groups = pipeline_group_count(n_channels, pcie_bytes, 32);
    const std::vector<int> bound = pipeline_bounds(weight, n_groups);

    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    VGB_TRY(g_ctx.pcm.reserve((size_t)(ps + 8) * 2));
    VGB_TRY(g_ctx.adpcm.reserve((size_t)ab + 16));
    VGB_TRY(g_ctx.misc.reserve(tab.size() * sizeof(AdxChannel)));
    VGB_TRY(g_ctx.coefs.reserve((size_t)n_channels * 2));
    // bookkeeping of the time-parallel encoder, one region per group (trace offsets are group relative)
    std::vector<size_t> seg_at(n_groups), seg_bytes(n_groups);
    std::vector<AdxSegArgs> seg(n_groups);
    size_t seg_total = 0;
    for (int g = 0; g < n_groups; g++) {
        seg[g] = adx_seg_carve(tab, bound[g], bound[g + 1] - bound[g], nullptr, seg_bytes[g]);
        seg_at[g] = seg_total;
        seg_total += align_up(seg_bytes[g], 256);
    }
    VGB_TRY(g_ctx.ws.reserve(seg_total + 256));
    for (int g = 0; g < n_groups; g++) {
        char *base = static_cast<char *>(g_ctx.ws.p) + seg_at[g];
        const AdxSegArgs rel = seg[g];
        seg[g].trace = reinterpret_cast<uint32_t *>(base + (reinterpret_cast<char *>(rel.trace) - static_cast<char *>(nullptr)));
        seg[g].used_start = reinterpret_cast<uint32_t *>(base + (reinterpret_cast<char *>(rel.used_start) - static_cast<char *>(nullptr)));
        seg[g].stats = reinterpret_cast<unsigned long long *>(base + (reinterpret_cast<char *>(rel.stats) - static_cast<char *>(nullptr)));
    }
    const AdxChannel *d_tab = static_cast<const AdxChannel *>(g_ctx.misc.p);
    int16_t *d_hist = static_cast<int16_t *>(g_ctx.coefs.p);
    auto sub = [&](const std::vector<int64_t> &v, int g) { return std::vector<int64_t>(v.begin() + bound[g], v.begin() + bound[g + 1]); };
    auto h2d = [&](int g) -> int32_t {
        if (g == 0) CUDA_TRY(cudaMemcpyAsync(g_ctx.misc.p, tab.data(), tab.size() * sizeof(AdxChannel), cudaMemcpyHostToDevice, g_ctx.s_in));
        return copy_channels_in(static_cast<char *>(g_ctx.pcm.p), sub(in_off, g), pcm + bound[g], sub(in_len, g), g_ctx.s_in);
    };
    auto kern = [&](int g, cudaStream_t st) -> int32_t {
        const int c0 = bound[g], n = bound[g + 1] - c0;
        if (n == 0) return VGB_OK;
        if (n_groups == 1) tick(4, true, st);
        launch_adx_encode(static_cast<const int16_t *>(g_ctx.pcm.p), d_tab + c0, n, static_cast<uint8_t *>(g_ctx.adpcm.p), d_hist + c0, seg[g], st);
        if (n_groups == 1) tick(4, false, st);
        g_ctx.launches += seg[g].seg_count > 1 ? 3 : 1;
        CUDA_TRY(cudaGetLastError());
        return VGB_OK;
    };
    auto d2h = [&](int g) -> int32_t {
        const int c0 = bound[g], n = bound[g + 1] - c0;
        if (history_out && n > 0) CUDA_TRY(cudaMemcpyAsync(history_out + c0, d_hist + c0, (size_t)n * 2, cudaMemcpyDeviceToHost, g_ctx.s_out));
        return copy_channels_out(adpcm_out + c0, static_cast<const char *>(g_ctx.adpcm.p), sub(out_off, g), sub(out_len, g), g_ctx.s_out);
    };
    auto done = [&](int g) -> int32_t {  // IProgressReport: one delta per finished group, summing to the frame total
        int64_t frames = 0;
        for (int c = bound[g]; c < bound[g + 1]; c++) frames += out_len[c] / params[c].frame_size;
        if (cb && frames > 0) cb(user, frames);
        return VGB_OK;
    };
    (void)frames_total;
    return run_group_pipeline(n_groups, h2d, kern, d2h, done);
}

/* ---- device-resident ADX encode (see the header) ---- */
uint64_t vgb_adx_workspace_bytes(int64_t total_samples, int32_t n_channels)
{
    if (n_channels < 0 || total_samples < 0) return 0;
    const size_t n = (size_t)std::max(n_channels, 1);
    return align_up(n * sizeof(AdxChannel), 256) + align_up(n * 2, 256) + align_up((size_t)(total_samples / 32 + 1) * 4, 256) +
           align_up(n * kAdxMaxSegments * 4, 256) + 512;
}

int32_t vgb_adx_encode_dev(const int16_t *d_pcm, const int64_t *pcm_offset, const int32_t *n_samples, const vgb_adx_params *params,
                           int32_t n_channels, int16_t *d_history_out, uint8_t *d_adpcm, const int64_t *adpcm_offset,
                           void *d_workspace, uint64_t workspace_bytes, void *cuda_stream)
{
    if (n_channels < 0) return fail(VGB_E_ARG, "n_channels is negative");
    if (n_channels == 0) return VGB_OK;
    if (!d_pcm || !pcm_offset || !n_samples || !params || !d_adpcm || !adpcm_offset || !d_workspace) return fail(VGB_E_ARG, "NULL argument");
    {
        int64_t total = 0;
        for (int c = 0; c < n_channels; c++) total += n_samples[c] > 0 ? n_samples[c] : 0;
        if (vgb_adx_workspace_bytes(total, n_channels) > workspace_bytes)
            return fail(VGB_E_ARG, "workspace too small: need %llu bytes", (unsigned long long)vgb_adx_workspace_bytes(total, n_channels));
    }
    std::vector<AdxChannel> tab(n_channels);
    for (int c = 0; c < n_channels; c++) {
        const vgb_adx_params &p = params[c];
        VGB_TRY(adx_validate(p, c));
        if (n_samples[c] < 0) return fail(VGB_E_ARG, "channel %d: negative sample count", c);
        if (p.version == 4 && p.padding == 0 && n_samples[c] == 0)
            return fail(VGB_E_ARG, "channel %d: version 4 without padding needs at least one sample", c);
        if (pcm_offset[c] < 0 || (pcm_offset[c] & 7) || adpcm_offset[c] < 0 || (adpcm_offset[c] & 1))
            return fail(VGB_E_ARG, "channel %d: pcm_offset must be a multiple of 8 samples, adpcm_offset even", c);
        AdxChannel &t = tab[c];
        t.pcm_off = pcm_offset[c]; t.adpcm_off = adpcm_offset[c]; t.n_samples = n_samples[c];
        t.frame_size = p.frame_size; t.version = p.version; t.padding = p.padding; t.type = p.type; t.filter = p.filter;
        t.history = 0;
        if (p.type == 2) { t.coef0 = kAdxFixed[p.filter][0]; t.coef1 = kAdxFixed[p.filter][1]; }
        else adx_calc_coefs(500, p.sample_rate, t.coef0, t.coef1);  // Encode hard-codes 500 (:63)
    }
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    char *ws = static_cast<char *>(d_workspace);
    const size_t o_hist = align_up(tab.size() * sizeof(AdxChannel), 256), o_seg = o_hist + align_up(tab.size() * 2, 256);
    int16_t *d_hist = d_history_out ? d_history_out : reinterpret_cast<int16_t *>(ws + o_hist);
    size_t seg_bytes = 0;
    const AdxSegArgs seg = adx_seg_carve(tab, 0, n_channels, ws + o_seg, seg_bytes);
    CUDA_TRY(cudaMemcpyAsync(ws, tab.data(), tab.size() * sizeof(AdxChannel), cudaMemcpyHostToDevice, st));  // pageable: staged before return
    tick(4, true, st);
    launch_adx_encode(d_pcm, reinterpret_cast<const AdxChannel *>(ws), n_channels, d_adpcm, d_hist, seg, st);
    tick(4, false, st);
    g_ctx.launches += seg.seg_count > 1 ? 3 : 1;
    CUDA_TRY(cudaGetLastError());
    return VGB_OK;
}

static int32_t adx_decode_one(const uint8_t *const *adpcm, const int32_t *n_bytes, const int32_t *sample_count,
                              const vgb_adx_params *params, int32_t n_channels, int16_t *const *pcm_out)
{
    PinScope pins;
    if (n_channels < 0) return fail(VGB_E_ARG, "n_channels is negative");
    if (n_channels == 0) return VGB_OK;
    if (!adpcm || !n_bytes || !sample_count || !params || !pcm_out) return fail(VGB_E_ARG, "NULL argument");
    std::vector<AdxChannel> tab(n_channels);
    std::vector<int64_t> in_off(n_channels), in_len(n_channels), out_off(n_channels), out_len(n_channels);
    int64_t ps = 0, ab = 0;
    for (int c = 0; c < n_channels; c++) {
        const vgb_adx_params &p = params[c];
        VGB_TRY(adx_validate(p, c));
        if (sample_count[c] < 0 || n_bytes[c] < 0) return fail(VGB_E_ARG, "channel %d: negative length", c);
        const int32_t spf = (p.frame_size - 2) * 2;
        // the reference would index past the array (IndexOutOfRangeException) on a short buffer
        const int64_t frames = ((int64_t)sample_count[c] + spf - 1) / spf;
        const int64_t need = ((int64_t)(p.padding / spf) + frames) * p.frame_size;
        if (sample_count[c] > 0 && n_bytes[c] < need)
            return fail(VGB_E_ARG, "channel %d: %d bytes of ADX data, %lld needed for %d samples", c, n_bytes[c],
                        (long long)need, sample_count[c]);
        if ((!adpcm[c] || !pcm_out[c]) && sample_count[c] > 0) return fail(VGB_E_ARG, "channel %d: NULL buffer", c);
        AdxChannel &t = tab[c];
        t.pcm_off = ps; t.adpcm_off = ab; t.n_samples = sample_count[c];
        t.frame_size = p.frame_size; t.version = p.version; t.padding = p.padding; t.type = p.type; t.filter = p.filter;
        t.history = (int16_t)p.history;
        if (p.type == 2) { t.coef0 = 0; t.coef1 = 0; }
        else adx_calc_coefs(p.highpass_frequency, p.sample_rate, t.coef0, t.coef1);
        in_off[c] = ab; in_len[c] = sample_count[c] > 0 ? n_bytes[c] : 0; out_off[c] = ps * 2; out_len[c] = (int64_t)sample_count[c] * 2;
        ps += (int64_t)align_up((size_t)sample_count[c], 8);
        ab += (int64_t)align_up((size_t)n_bytes[c], 16);
    }
    std::vector<int64_t> weight(n_channels);
    int64_t pcie_bytes = 0;
    for (int c = 0; c < n_channels; c++) { weight[c] = out_len[c] + 64; pcie_bytes += in_len[c] + out_len[c]; }
    const int n_groups = pipeline_group_count(n_channels, pcie_bytes, 32);
    const std::vector<int> bound = pipeline_bounds(weight, n_groups);

    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    VGB_TRY(g_ctx.pcm.reserve((size_t)(ps + 8) * 2));
    VGB_TRY(g_ctx.adpcm.reserve((size_t)ab + 16));
    const size_t o_status = align_up(tab.size() * sizeof(AdxChannel), 256);
    VGB_TRY(g_ctx.misc.reserve(o_status + 16 * (size_t)n_groups));
    const AdxChannel *d_tab = static_cast<const AdxChannel *>(g_ctx.misc.p);
    int32_t *d_status = reinterpret_cast<int32_t *>(static_cast<char *>(g_ctx.misc.p) + o_status);  // [group * 4]
    std::vector<int32_t> bad(n_groups, INT_MAX);
    auto sub = [&](const std::vector<int64_t> &v, int g) { return std::vector<int64_t>(v.begin() + bound[g], v.begin() + bound[g + 1]); };
    auto h2d = [&](int g) -> int32_t {
        if (g == 0) {
            CUDA_TRY(cudaMemcpyAsync(g_ctx.misc.p, tab.data(), tab.size() * sizeof(AdxChannel), cudaMemcpyHostToDevice, g_ctx.s_in));
            CUDA_TRY(cudaMemsetAsync(d_status, 0x7f, 16 * (size_t)n_groups, g_ctx.s_in));
        }
        return copy_channels_in(static_cast<char *>(g_ctx.adpcm.p), sub(in_off, g), adpcm + bound[g], sub(in_len, g), g_ctx.s_in);
    };
    auto kern = [&](int g, cudaStream_t st) -> int32_t {
        const int c0 = bound[g], n = bound[g + 1] - c0;
        if (n == 0) return VGB_OK;
        if (n_groups == 1) tick(5, true, st);
        launch_adx_decode(static_cast<const uint8_t *>(g_ctx.adpcm.p), d_tab + c0, n, static_cast<int16_t *>(g_ctx.pcm.p), d_status + 4 * g, st);
        if (n_groups == 1) tick(5, false, st);
        g_ctx.launches += 1;
        CUDA_TRY(cudaGetLastError());
        return VGB_OK;
    };
    auto d2h = [&](int g) -> int32_t {
        VGB_TRY(copy_channels_out(pcm_out + bound[g], static_cast<const char *>(g_ctx.pcm.p), sub(out_off, g), sub(out_len, g), g_ctx.s_out));
        CUDA_TRY(cudaMemcpyAsync(&bad[g], d_status + 4 * g, 4, cudaMemcpyDeviceToHost, g_ctx.s_out));
        return VGB_OK;
    };
    VGB_TRY(run_group_pipeline(n_groups, h2d, kern, d2h, [](int) { return VGB_OK; }));
    // CriAdxCodec.Coefs[filterNum] (:186-191) has four rows: IndexOutOfRangeException in the reference
    for (int g = 0; g < n_groups; g++)
        if (bad[g] >= 0 && bad[g] < bound[g + 1] - bound[g])
            return fail(VGB_E_DATA, "channel %d: a Fixed-type frame selects a filter outside 0..3", bound[g] + bad[g]);
    return VGB_OK;
}

// ---- CRI HCA --------------------------------------------------------------------------------------------------

}  // extern "C"

namespace {

#include "hca_tables.inc"

// Extensions.DivideByRoundUp for non-negative ints
inline int hca_div_up(int a, int b) { return (int)std::ceil((double)a / b); }
inline int hca_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
inline int hca_next_multiple(int v, int m) { if (m <= 0) return v; if (v % m == 0) return v; return v + m - v % m; }

// CriHcaEncoder.Initialize (CriHcaEncoder.cs:61-114, non-looping) = CalculateBitrate :288-324,
// CalculateBandCounts :326-368, HcaInfo.CalculateHfrValues (HcaInfo.cs:50-56), SetChannelConfiguration :370-381,
// CalculateHeaderSize :400-418.  Integer/`Math.Round` logic only (half-to-even = nearbyint, SURVEY.md A.3).
// The encoder's input as ONE virtual sample stream (CriHcaEncoder.Encode :126-272 + the chunk loop of
// CriHcaFormat.EncodeFromPcm16 :53-81): frame k encodes virtual samples [1024 k, 1024 k + 1024).
struct HcaVirtual {
    int32_t pre_zero = 0;    // whole silent frames EncodePreAudio emits while BufferPreSamples > 1024 (:177-182)
    int32_t pre_fill = 0;    // then copies of the stream's first sample (:184-190)
    int32_t main_count = 0;  // Hca.SampleCount source samples
    int32_t post_count = 0;  // PostSamples taken from the loop start (SaveLoopAudio / EncodePostAudio); 0 when not looping
    int32_t loop_start = 0;  // source position of post sample 0
    int32_t src_count = 0;   // PCM length
    int32_t last_chunk = 0;  // index of the last 1024-sample chunk the format layer hands to Encode
};

int32_t hca_initialize(const vgb_hca_params &p, vgb_hca_info &h, HcaVirtual *virt = nullptr)
{
    if (p.channel_count > 8)
        return fail(VGB_E_ARG, "HCA channel count must be 8 or below");
    if (p.channel_count < 1) return fail(VGB_E_ARG, "HCA channel count must be at least 1");
    if (p.sample_rate <= 0 || p.sample_count < 0) return fail(VGB_E_ARG, "bad sample rate / sample count");
    if (p.looping && (p.loop_start < 0 || p.loop_end <= p.loop_start || p.loop_start >= p.sample_count))
        return fail(VGB_E_ARG, "loop points must satisfy 0 <= loop_start < loop_end and loop_start < sample_count");
    std::memset(&h, 0, sizeof h);
    const int cutoff0 = p.sample_rate / 2;
    h.channel_count = p.channel_count;
    h.track_count = 1;
    h.sample_count = p.sample_count;
    h.sample_rate = p.sample_rate;
    h.min_resolution = 1;
    h.max_resolution = 15;
    h.inserted_samples = 128;

    const int pcm_bitrate = h.sample_rate * h.channel_count * 16;
    {
        const int max_bitrate = pcm_bitrate / 4;
        int min_bitrate = 0, ratio = 6;
        switch (p.quality) {
        case 1: ratio = 4; break;
        case 2: ratio = 6; break;
        case 3: ratio = 8; break;
        case 4: ratio = h.channel_count == 1 ? 10 : 12; break;
        case 5: ratio = h.channel_count == 1 ? 12 : 16; break;
        default: break;
        }
        int bitrate = p.bitrate != 0 ? p.bitrate : pcm_bitrate / ratio;
        if (p.limit_bitrate) min_bitrate = std::min(h.channel_count == 1 ? 42666 : 32000 * h.channel_count, pcm_bitrate / 6);
        h.bitrate = hca_clampi(bitrate, min_bitrate, max_bitrate);
    }
    if (h.bitrate <= 0) return fail(VGB_E_ARG, "bitrate must be positive");
    {
        const int bitrate = h.bitrate;
        int cutoff = cutoff0;
        // `bitrate * 1024 / SampleRate / 8` in C# int arithmetic (CriHcaEncoder.cs:322): the product wraps above 2^31
        // (e.g. 6 channels x 96 kHz at Highest); the reference then ends with a negative frame size and fails
        h.frame_size = wmul(bitrate, 1024) / h.sample_rate / 8;
        int hfr_ratio, cutoff_ratio;
        if (h.channel_count <= 1 || pcm_bitrate / bitrate <= 6) { hfr_ratio = 6; cutoff_ratio = 12; }
        else { hfr_ratio = 8; cutoff_ratio = 16; }
        if (bitrate < pcm_bitrate / cutoff_ratio) cutoff = std::min(cutoff, cutoff_ratio * bitrate / (32 * h.channel_count));
        const int total = (int)std::nearbyint(cutoff * 256.0 / h.sample_rate);
        const double hs = std::nearbyint((hfr_ratio * (double)bitrate * 128.0) / pcm_bitrate);
        const int hfr_start = (int)std::min((double)total, hs);
        const int stereo_start = hfr_ratio == 6 ? hfr_start : (hfr_start + 1) / 2;
        const int hfr_bands = total - hfr_start;
        const int per_group = hca_div_up(hfr_bands, 8);
        int groups = 0;
        if (per_group > 0) groups = hca_div_up(hfr_bands, per_group);
        h.total_band_count = total;
        h.base_band_count = stereo_start;
        h.stereo_band_count = hfr_start - stereo_start;
        h.hfr_group_count = groups;
        h.bands_per_hfr_group = per_group;
    }
    if (h.frame_size < 8)
        return fail(VGB_E_DATA, h.frame_size < 0 ? "frame size overflows (bitrate * 1024 exceeds int32, as in the reference)" : "Bitrate is set too low.");
    if (h.bands_per_hfr_group > 0) {
        h.hfr_band_count = h.total_band_count - h.base_band_count - h.stereo_band_count;
        h.hfr_group_count = hca_div_up(h.hfr_band_count, h.bands_per_hfr_group);
    }
    {
        const int per_track = h.channel_count / h.track_count;
        const int config = kHcaDefaultChannelMapping[per_track];
        if (kHcaValidChannelMappings[per_track - 1][config] != 1) return fail(VGB_E_ARG, "Channel mapping is not valid.");
        h.channel_config = config;
    }
    int input_samples = h.sample_count, post_samples = 128;
    if (p.looping) {  // :89-99
        h.looping = 1;
        h.sample_count = std::min(p.loop_end, p.sample_count);
        h.inserted_samples += hca_next_multiple(p.loop_start, 1024) - p.loop_start;
        {  // CalculateLoopInfo (:383-398)
            const int ls = p.loop_start + h.inserted_samples, le = p.loop_end + h.inserted_samples;
            h.loop_start_frame = ls / 1024;
            h.pre_loop_samples = ls % 1024;
            h.loop_end_frame = le / 1024;
            h.post_loop_samples = 1024 - le % 1024;
            if (h.post_loop_samples == 1024) { h.loop_end_frame--; h.post_loop_samples = 0; }
        }
        input_samples = std::min(hca_next_multiple(h.sample_count, 128), p.sample_count) + 256;
        post_samples = input_samples - h.sample_count;
    }
    h.header_size = hca_next_multiple(96, 32);  // CalculateHeaderSize (:400-418), no comment
    if (h.looping) {  // whole padding frames so that the loop start frame lands on a 2048-byte boundary of the file
        const int loop_frame_offset = h.header_size + h.frame_size * h.loop_start_frame;
        const int padding_bytes = hca_next_multiple(loop_frame_offset, 2048) - loop_frame_offset;
        const int padding_frames = padding_bytes / h.frame_size;
        h.inserted_samples += padding_frames * 1024;
        h.loop_start_frame += padding_frames;
        h.loop_end_frame += padding_frames;
        h.header_size += padding_bytes % h.frame_size;
    }
    const int total_samples = input_samples + h.inserted_samples;
    h.frame_count = hca_div_up(total_samples, 1024);
    h.appended_samples = h.frame_count * 1024 - h.inserted_samples - input_samples;
    if (virt) {
        const int pre = h.inserted_samples - 128;  // BufferPreSamples (:113)
        const int zero_frames = pre > 1024 ? hca_div_up(pre, 1024) - 1 : 0;
        virt->pre_zero = zero_frames * 1024;
        virt->pre_fill = pre - virt->pre_zero;
        virt->main_count = h.sample_count;
        virt->post_count = h.looping ? post_samples : 0;  // a non-looping encoder's PostAudio is all zero
        virt->loop_start = p.loop_start;
        virt->src_count = p.sample_count;
        virt->last_chunk = h.sample_count > 0 ? (h.sample_count - 1) / 1024 : 0;
    }
    return VGB_OK;
}

// CriHcaFrame.GetChannelTypes (CriHcaFrame.cs:34-52)
// CriHcaFrame.cs:31 + ScaleAthCurve :60-84: the ATH curve (tabulated for 41856 Hz) resampled to the stream's rate; all
// zero unless HcaInfo.UseAthCurve (old files only; the encoder never sets it, so the encode entry points leave it zero).
void hca_fill_ath(const vgb_hca_info &h, uint8_t ath[128])
{
    std::memset(ath, 0, 128);
    if (!h.use_ath_curve) return;
    int acc = 0, i = 0;
    for (; i < 128; i++) {
        acc += h.sample_rate;
        const int index = acc >> 13;
        if (index >= (int)sizeof kHcaAthCurve) break;
        ath[i] = kHcaAthCurve[index];
    }
    for (; i < 128; i++) ath[i] = 0xff;
}

void hca_channel_types(const vgb_hca_info &h, int32_t types[8])
{
    static const int t2[] = {1, 2}, t3[] = {1, 2, 0}, t4a[] = {1, 2, 0, 0}, t4b[] = {1, 2, 1, 2}, t5a[] = {1, 2, 0, 0, 0},
                     t5b[] = {1, 2, 0, 1, 2}, t6[] = {1, 2, 0, 0, 1, 2}, t7[] = {1, 2, 0, 0, 1, 2, 0},
                     t8[] = {1, 2, 0, 0, 1, 2, 1, 2};
    for (int i = 0; i < 8; i++) types[i] = 0;
    const int per_track = h.channel_count / h.track_count;
    if (h.stereo_band_count == 0 || per_track == 1) return;
    const int *src = nullptr;
    switch (per_track) {
    case 2: src = t2; break;
    case 3: src = t3; break;
    case 4: src = h.channel_config != 0 ? t4a : t4b; break;
    case 5: src = h.channel_config > 2 ? t5a : t5b; break;
    case 6: src = t6; break;
    case 7: src = t7; break;
    case 8: src = t8; break;
    default: return;
    }
    for (int i = 0; i < per_track; i++) types[i] = src[i];
}

// One-time upload of the codec tables (per process/device).  Trig tables: Mdct.GenerateTrigTables (Mdct.cs:183-195)
// with the host libm, exactly as the oracle builds them; dead zones: CriHcaTables.QuantizerDeadZoneFunction (:68-78).
// (HcaTableStore is a member of the per-device Context: g_hca_tables below is the current device's store)

void hca_tables_release_locked()
{
    if (g_hca_tables.blob) cudaFree(g_hca_tables.blob);
    g_hca_tables.blob = nullptr;
    g_hca_tables.ready = false;
}

int32_t hca_tables_ready_locked()
{
    if (g_hca_tables.ready) return VGB_OK;
    std::vector<unsigned char> host;
    auto put = [&](const void *src, size_t bytes) { size_t at = align_up(host.size(), 16); host.resize(at + bytes); std::memcpy(host.data() + at, src, bytes); return at; };
    const size_t o_window = put(kHcaMdctWindow, sizeof kHcaMdctWindow);
    size_t o_sin[8], o_cos[8];
    for (int bits = 0; bits <= 7; bits++) {
        const int size = 1 << bits;
        std::vector<double> sn(size), cs(size);
        for (int i = 0; i < size; i++) {
            const double value = 3.14159265358979323846 * (4 * i + 1) / (4 * size);
            sn[i] = std::sin(value);
            cs[i] = std::cos(value);
        }
        o_sin[bits] = put(sn.data(), size * sizeof(double));
        o_cos[bits] = put(cs.data(), size * sizeof(double));
    }
    int32_t shuffle[128];
    for (int i = 0; i < 128; i++) {
        unsigned v = (unsigned)(i ^ (i / 2));
        v = ((v & 0xaaaaaaaau) >> 1) | ((v & 0x55555555u) << 1);
        v = ((v & 0xccccccccu) >> 2) | ((v & 0x33333333u) << 2);
        v = ((v & 0xf0f0f0f0u) >> 4) | ((v & 0x0f0f0f0fu) << 4);
        v = ((v & 0xff00ff00u) >> 8) | ((v & 0x00ff00ffu) << 8);
        v = (v >> 16) | (v << 16);
        shuffle[i] = (int32_t)(v >> (32 - 7));
    }
    const size_t o_shuffle = put(shuffle, sizeof shuffle);
    const size_t o_deq = put(kHcaDequantizerScaling, sizeof kHcaDequantizerScaling);
    const size_t o_qs = put(kHcaQuantizerScaling, sizeof kHcaQuantizerScaling);
    const size_t o_inv = put(kHcaQuantizerInverseStepSize, sizeof kHcaQuantizerInverseStepSize);
    double dead[16];
    for (int i = 0; i < 16; i++) {
        const int steps = (i < 8 ? i : (1 << (i - 4)) - 1) + 1;
        double boundary = kHcaQuantizerStepSize[i] / 2;
        int64_t bits;
        std::memcpy(&bits, &boundary, 8);
        bits -= steps;
        std::memcpy(&dead[i], &bits, 8);
    }
    const size_t o_dead = put(dead, sizeof dead);
    const size_t o_bounds = put(kHcaIntensityRatioBounds, sizeof kHcaIntensityRatioBounds);
    const size_t o_s2r = put(kHcaScaleToResolutionCurve, sizeof kHcaScaleToResolutionCurve);
    const size_t o_maxbits = put(kHcaQuantizedSpectrumMaxBits, sizeof kHcaQuantizedSpectrumMaxBits);
    const size_t o_qbits = put(kHcaQuantizeSpectrumBits, sizeof kHcaQuantizeSpectrumBits);
    const size_t o_qval = put(kHcaQuantizeSpectrumValue, sizeof kHcaQuantizeSpectrumValue);
    uint16_t crc[256];
    for (int i = 0; i < 256; i++) {
        uint16_t cur = (uint16_t)(i << 8);
        for (int j = 0; j < 8; j++) {
            const bool x = (cur & 0x8000) != 0;
            cur = (uint16_t)(cur << 1);
            if (x) cur ^= 0x8005;
        }
        crc[i] = cur;
    }
    const size_t o_crc = put(crc, sizeof crc);
    const size_t o_step = put(kHcaQuantizerStepSize, sizeof kHcaQuantizerStepSize);
    const size_t o_ratio = put(kHcaIntensityRatio, sizeof kHcaIntensityRatio);
    const size_t o_conv = put(kHcaScaleConversion, sizeof kHcaScaleConversion);
    const size_t o_dbits = put(kHcaQuantizedSpectrumBits, sizeof kHcaQuantizedSpectrumBits);
    const size_t o_dval = put(kHcaQuantizedSpectrumValue, sizeof kHcaQuantizedSpectrumValue);

    CUDA_TRY(cudaMalloc(&g_hca_tables.blob, host.size()));
    CUDA_TRY(cudaMemcpy(g_hca_tables.blob, host.data(), host.size(), cudaMemcpyHostToDevice));
    const char *b = static_cast<const char *>(g_hca_tables.blob);
    HcaTables &T = g_hca_tables.view;
    T.window = reinterpret_cast<const double *>(b + o_window);
    for (int bits = 0; bits <= 7; bits++) {
        T.sin_tab[bits] = reinterpret_cast<const double *>(b + o_sin[bits]);
        T.cos_tab[bits] = reinterpret_cast<const double *>(b + o_cos[bits]);
    }
    T.shuffle = reinterpret_cast<const int32_t *>(b + o_shuffle);
    T.mdct_scale = std::sqrt(2.0 / 128);
    T.sqrt2 = std::sqrt(2.0);
    T.dequantizer_scaling = reinterpret_cast<const double *>(b + o_deq);
    T.quantizer_scaling = reinterpret_cast<const double *>(b + o_qs);
    T.inv_step = reinterpret_cast<const double *>(b + o_inv);
    T.dead_zone = reinterpret_cast<const double *>(b + o_dead);
    T.intensity_bounds = reinterpret_cast<const double *>(b + o_bounds);
    T.scale_to_resolution = reinterpret_cast<const uint8_t *>(b + o_s2r);
    T.quantized_max_bits = reinterpret_cast<const uint8_t *>(b + o_maxbits);
    T.quantize_bits = reinterpret_cast<const uint8_t(*)[16]>(b + o_qbits);
    T.quantize_value = reinterpret_cast<const uint8_t(*)[16]>(b + o_qval);
    T.crc_table = reinterpret_cast<const uint16_t *>(b + o_crc);
    T.step_size = reinterpret_cast<const double *>(b + o_step);
    T.intensity_ratio = reinterpret_cast<const double *>(b + o_ratio);
    T.scale_conversion = reinterpret_cast<const double *>(b + o_conv);
    T.dequantize_bits = reinterpret_cast<const uint8_t(*)[16]>(b + o_dbits);
    T.dequantize_value = reinterpret_cast<const int8_t(*)[16]>(b + o_dval);
    g_hca_tables.ready = true;
    return VGB_OK;
}

}  // namespace

extern "C" {

int32_t vgb_hca_query(const vgb_hca_params *params, vgb_hca_info *info_out)
{
    if (!params || !info_out) return fail(VGB_E_ARG, "NULL argument");
    return hca_initialize(*params, *info_out);
}

static int32_t hca_encode_one(const int16_t *const *pcm, const vgb_hca_params *params, int32_t n_streams,
                              vgb_hca_info *info_out, uint8_t *const *frames_out, vgb_progress_cb cb, void *user)
{
    PinScope pins;
    if (n_streams < 0) return fail(VGB_E_ARG, "n_streams is negative");
    if (n_streams == 0) return VGB_OK;
    if (!pcm || !params || !frames_out) return fail(VGB_E_ARG, "NULL argument");
    std::vector<vgb_hca_info> infos(n_streams);
    std::vector<HcaVirtual> virt(n_streams);
    for (int s = 0; s < n_streams; s++) {
        VGB_TRY(hca_initialize(params[s], infos[s], &virt[s]));
        const vgb_hca_params &a = params[0], &b = params[s];
        if (a.channel_count != b.channel_count || a.sample_rate != b.sample_rate || a.quality != b.quality ||
            a.bitrate != b.bitrate || a.limit_bitrate != b.limit_bitrate)
            return fail(VGB_E_ARG, "stream %d: all streams of one call must share channel count, sample rate, quality and bitrate", s);
    }
    const vgb_hca_info &h0 = infos[0];
    const int nch = h0.channel_count;
    HcaConfig cfg{};
    cfg.channel_count = nch;
    cfg.frame_size = h0.frame_size;
    cfg.base_band_count = h0.base_band_count;
    cfg.stereo_band_count = h0.stereo_band_count;
    cfg.total_band_count = h0.total_band_count;
    cfg.hfr_band_count = h0.hfr_band_count;
    cfg.bands_per_hfr_group = h0.bands_per_hfr_group;
    cfg.hfr_group_count = h0.hfr_group_count;
    hca_channel_types(h0, cfg.channel_type);
    hca_fill_ath(h0, cfg.ath);

    std::vector<HcaStream> streams(n_streams);
    std::vector<int64_t> in_off((size_t)n_streams * nch), in_len((size_t)n_streams * nch), out_off(n_streams), out_len(n_streams);
    int64_t ps = 0, fb = 0, frames_total = 0;
    int max_frames = 0;
    for (int s = 0; s < n_streams; s++) {
        const int32_t n_src = params[s].sample_count;  // the PCM the caller holds (>= Hca.SampleCount when looping)
        const int64_t stride = (int64_t)align_up((size_t)n_src, 8);
        streams[s].pcm_off = ps;
        streams[s].channel_stride = stride;
        streams[s].frames_off = fb;
        streams[s].sample_count = infos[s].sample_count;
        streams[s].frame_count = infos[s].frame_count;
        streams[s].pre_zero = virt[s].pre_zero;
        streams[s].pre_fill = virt[s].pre_fill;
        streams[s].post_count = virt[s].post_count;
        streams[s].loop_start = virt[s].loop_start;
        streams[s].src_count = virt[s].src_count;
        streams[s].last_chunk = virt[s].last_chunk;
        for (int c = 0; c < nch; c++) {
            if (!pcm[(size_t)s * nch + c] && n_src > 0) return fail(VGB_E_ARG, "pcm[%d][%d] is NULL", s, c);
            in_off[(size_t)s * nch + c] = (ps + c * stride) * 2;
            in_len[(size_t)s * nch + c] = (int64_t)n_src * 2;
        }
        ps += stride * nch;
        out_off[s] = fb;
        out_len[s] = (int64_t)infos[s].frame_count * infos[s].frame_size;
        if (!frames_out[s] && out_len[s] > 0) return fail(VGB_E_ARG, "frames_out[%d] is NULL", s);
        fb += (int64_t)align_up((size_t)out_len[s], 16);
        max_frames = std::max(max_frames, infos[s].frame_count);
        frames_total += infos[s].frame_count;
    }

    // stream groups: H2D of group g+1 || encode of group g || D2H of group g-1
    std::vector<int64_t> weight(n_streams);
    int64_t pcie_bytes = 0;
    for (int s = 0; s < n_streams; s++) {
        weight[s] = (int64_t)infos[s].frame_count + 1;
        pcie_bytes += (int64_t)params[s].sample_count * 2 * nch + out_len[s];
    }
    const int n_groups = pipeline_group_count(n_streams, pcie_bytes, 16);
    const std::vector<int> bound = pipeline_bounds(weight, n_groups);

    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    VGB_TRY(hca_tables_ready_locked());
    const size_t o_status = align_up(streams.size() * sizeof(HcaStream), 256);
    VGB_TRY(g_ctx.pcm.reserve((size_t)(ps + 8) * 2));
    VGB_TRY(g_ctx.adpcm.reserve((size_t)fb + 16));
    VGB_TRY(g_ctx.misc.reserve(o_status + (size_t)n_streams * 4));
    char *misc = static_cast<char *>(g_ctx.misc.p);
    const HcaStream *d_streams = reinterpret_cast<const HcaStream *>(misc);
    int32_t *d_status = reinterpret_cast<int32_t *>(misc + o_status);
    std::vector<int32_t> status(n_streams, 0);
    auto h2d = [&](int g) -> int32_t {
        if (g == 0) {
            CUDA_TRY(cudaMemcpyAsync(misc, streams.data(), streams.size() * sizeof(HcaStream), cudaMemcpyHostToDevice, g_ctx.s_in));
            CUDA_TRY(cudaMemsetAsync(misc + o_status, 0, (size_t)n_streams * 4, g_ctx.s_in));
        }
        const size_t c0 = (size_t)bound[g] * nch, c1 = (size_t)bound[g + 1] * nch;
        return copy_channels_in(static_cast<char *>(g_ctx.pcm.p), std::vector<int64_t>(in_off.begin() + c0, in_off.begin() + c1), pcm + c0,
                                std::vector<int64_t>(in_len.begin() + c0, in_len.begin() + c1), g_ctx.s_in);
    };
    auto kern = [&](int g, cudaStream_t st) -> int32_t {
        const int s0 = bound[g], n = bound[g + 1] - s0;
        if (n == 0) return VGB_OK;
        int group_max = 0;
        for (int s = s0; s < s0 + n; s++) group_max = std::max(group_max, infos[s].frame_count);
        if (n_groups == 1) tick(6, true, st);
        CUDA_TRY(launch_hca_encode(static_cast<const int16_t *>(g_ctx.pcm.p), d_streams + s0, n, group_max, cfg, g_hca_tables.view,
                                   static_cast<uint8_t *>(g_ctx.adpcm.p), d_status + s0, st));
        if (n_groups == 1) tick(6, false, st);
        g_ctx.launches += 1;
        return VGB_OK;
    };
    auto d2h = [&](int g) -> int32_t {
        const int s0 = bound[g], n = bound[g + 1] - s0;
        if (n > 0) CUDA_TRY(cudaMemcpyAsync(status.data() + s0, d_status + s0, (size_t)n * 4, cudaMemcpyDeviceToHost, g_ctx.s_out));
        return copy_channels_out(frames_out + s0, static_cast<const char *>(g_ctx.adpcm.p), std::vector<int64_t>(out_off.begin() + s0, out_off.begin() + s0 + n),
                                 std::vector<int64_t>(out_len.begin() + s0, out_len.begin() + s0 + n), g_ctx.s_out);
    };
    (void)max_frames;
    VGB_TRY(run_group_pipeline(n_groups, h2d, kern, d2h, [](int) { return VGB_OK; }));
    for (int s = 0; s < n_streams; s++) {
        if (status[s] == VGB_HCA_BITRATE_TOO_LOW) return fail(VGB_E_DATA, "stream %d: Bitrate is set too low.", s);
        if (status[s] == VGB_HCA_NOT_IMPLEMENTED) return fail(VGB_E_STATE, "stream %d: evaluation boundary search failed (NotImplementedException in the reference)", s);
        if (status[s] == VGB_HCA_BIT_OVERFLOW) return fail(VGB_E_STATE, "stream %d: Not enough bits left in output buffer", s);
    }
    if (info_out) for (int s = 0; s < n_streams; s++) info_out[s] = infos[s];
    if (cb) cb(user, frames_total);
    return VGB_OK;
}

/* ---- device-resident HCA encode (see the header) ---- */
uint64_t vgb_hca_workspace_bytes(int32_t n_streams)
{
    if (n_streams < 0) return 0;
    return align_up((size_t)std::max(n_streams, 1) * sizeof(HcaStream), 256) + align_up((size_t)std::max(n_streams, 1) * 4, 256);
}

int32_t vgb_hca_encode_dev(const int16_t *d_pcm, const int64_t *pcm_offset, const int64_t *channel_stride, const vgb_hca_params *params,
                           int32_t n_streams, vgb_hca_info *info_out, uint8_t *d_frames, const int64_t *frames_offset,
                           void *d_workspace, uint64_t workspace_bytes, void *cuda_stream)
{
    if (n_streams < 0) return fail(VGB_E_ARG, "n_streams is negative");
    if (n_streams == 0) return VGB_OK;
    if (!d_pcm || !pcm_offset || !channel_stride || !params || !d_frames || !frames_offset || !d_workspace) return fail(VGB_E_ARG, "NULL argument");
    if (vgb_hca_workspace_bytes(n_streams) > workspace_bytes)
        return fail(VGB_E_ARG, "workspace too small: need %llu bytes", (unsigned long long)vgb_hca_workspace_bytes(n_streams));
    std::vector<vgb_hca_info> infos(n_streams);
    std::vector<HcaVirtual> virt(n_streams);
    for (int s = 0; s < n_streams; s++) {
        VGB_TRY(hca_initialize(params[s], infos[s], &virt[s]));
        const vgb_hca_params &a = params[0], &b = params[s];
        if (a.channel_count != b.channel_count || a.sample_rate != b.sample_rate || a.quality != b.quality ||
            a.bitrate != b.bitrate || a.limit_bitrate != b.limit_bitrate)
            return fail(VGB_E_ARG, "stream %d: all streams of one call must share channel count, sample rate, quality and bitrate", s);
    }
    const vgb_hca_info &h0 = infos[0];
    const int nch = h0.channel_count;
    HcaConfig cfg{};
    cfg.channel_count = nch;
    cfg.frame_size = h0.frame_size;
    cfg.base_band_count = h0.base_band_count;
    cfg.stereo_band_count = h0.stereo_band_count;
    cfg.total_band_count = h0.total_band_count;
    cfg.hfr_band_count = h0.hfr_band_count;
    cfg.bands_per_hfr_group = h0.bands_per_hfr_group;
    cfg.hfr_group_count = h0.hfr_group_count;
    hca_channel_types(h0, cfg.channel_type);
    std::vector<HcaStream> streams(n_streams);
    int max_frames = 0;
    for (int s = 0; s < n_streams; s++) {
        if (pcm_offset[s] < 0 || channel_stride[s] < params[s].sample_count || frames_offset[s] < 0)
            return fail(VGB_E_ARG, "stream %d: bad offsets (channel_stride must cover sample_count)", s);
        streams[s].pcm_off = pcm_offset[s];
        streams[s].channel_stride = channel_stride[s];
        streams[s].frames_off = frames_offset[s];
        streams[s].sample_count = infos[s].sample_count;
        streams[s].frame_count = infos[s].frame_count;
        streams[s].pre_zero = virt[s].pre_zero;
        streams[s].pre_fill = virt[s].pre_fill;
        streams[s].post_count = virt[s].post_count;
        streams[s].loop_start = virt[s].loop_start;
        streams[s].src_count = virt[s].src_count;
        streams[s].last_chunk = virt[s].last_chunk;
        max_frames = std::max(max_frames, infos[s].frame_count);
    }
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    VGB_TRY(hca_tables_ready_locked());
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    char *ws = static_cast<char *>(d_workspace);
    const size_t o_status = align_up(streams.size() * sizeof(HcaStream), 256);
    CUDA_TRY(cudaMemcpyAsync(ws, streams.data(), streams.size() * sizeof(HcaStream), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(ws + o_status, 0, (size_t)n_streams * 4, st));
    tick(6, true, st);
    CUDA_TRY(launch_hca_encode(d_pcm, reinterpret_cast<const HcaStream *>(ws), n_streams, max_frames, cfg, g_hca_tables.view, d_frames,
                               reinterpret_cast<int32_t *>(ws + o_status), st));
    tick(6, false, st);
    g_ctx.launches += 1;
    if (info_out) for (int s = 0; s < n_streams; s++) info_out[s] = infos[s];
    return VGB_OK;
}

/* Synchronises `cuda_stream` and maps the per-stream status words the last vgb_hca_encode_dev on this workspace left
 * (the reference's exceptions: Bitrate is set too low, ...). */
int32_t vgb_hca_encode_dev_status(const void *d_workspace, int32_t n_streams, void *cuda_stream)
{
    if (n_streams <= 0) return VGB_OK;
    if (!d_workspace) return fail(VGB_E_ARG, "NULL argument");
    std::vector<int32_t> status(n_streams, 0);
    const size_t o_status = align_up((size_t)n_streams * sizeof(HcaStream), 256);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    CUDA_TRY(cudaMemcpyAsync(status.data(), static_cast<const char *>(d_workspace) + o_status, (size_t)n_streams * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    for (int s = 0; s < n_streams; s++) {
        if (status[s] == VGB_HCA_BITRATE_TOO_LOW) return fail(VGB_E_DATA, "stream %d: Bitrate is set too low.", s);
        if (status[s] == VGB_HCA_NOT_IMPLEMENTED) return fail(VGB_E_STATE, "stream %d: evaluation boundary search failed (NotImplementedException in the reference)", s);
        if (status[s] == VGB_HCA_BIT_OVERFLOW) return fail(VGB_E_STATE, "stream %d: Not enough bits left in output buffer", s);
    }
    return VGB_OK;
}

/* Mdct.RunMdct / RunImdct (Utilities/Mdct.cs:63-119) of the codec's 128-point instance for n_sequences independent
 * sequences of n_blocks blocks (each sequence starts from a fresh Mdct object's all-zero state).  Host buffers
 * [sequence][block][128] doubles.  Unit-parity taps (SURVEY 8b); the codec kernels carry their own copy of the transform. */
static int32_t mdct128_impl(const double *in, int32_t n_sequences, int32_t n_blocks, double *out, bool inverse)
{
    if (n_sequences < 0 || n_blocks < 0) return fail(VGB_E_ARG, "negative count");
    if (n_sequences == 0 || n_blocks == 0) return VGB_OK;
    if (!in || !out) return fail(VGB_E_ARG, "NULL argument");
    const size_t bytes = (size_t)n_sequences * n_blocks * 128 * sizeof(double);
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    VGB_TRY(hca_tables_ready_locked());
    VGB_TRY(g_ctx.misc.reserve(2 * align_up(bytes, 256)));
    cudaStream_t st = g_ctx.stream;
    char *d_in = static_cast<char *>(g_ctx.misc.p), *d_out = d_in + align_up(bytes, 256);
    CUDA_TRY(cudaMemcpyAsync(d_in, in, bytes, cudaMemcpyHostToDevice, st));
    CUDA_TRY(launch_hca_mdct128(reinterpret_cast<const double *>(d_in), reinterpret_cast<double *>(d_out), n_sequences, n_blocks, inverse,
                                g_hca_tables.view, st));
    g_ctx.launches += 1;
    CUDA_TRY(cudaMemcpyAsync(out, d_out, bytes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return VGB_OK;
}
int32_t vgb_mdct128_batch(const double *in, int32_t n_sequences, int32_t n_blocks, double *out) { return mdct128_impl(in, n_sequences, n_blocks, out, false); }
int32_t vgb_imdct128_batch(const double *in, int32_t n_sequences, int32_t n_blocks, double *out) { return mdct128_impl(in, n_sequences, n_blocks, out, true); }

static int32_t hca_decode_one(const uint8_t *const *frames, const vgb_hca_info *info, int32_t n_streams,
                              int16_t *const *pcm_out)
{
    PinScope pins;
    if (n_streams < 0) return fail(VGB_E_ARG, "n_streams is negative");
    if (n_streams == 0) return VGB_OK;
    if (!frames || !info || !pcm_out) return fail(VGB_E_ARG, "NULL argument");
    const vgb_hca_info &h0 = info[0];
    const int nch = h0.channel_count;
    if (nch < 1 || nch > 8) return fail(VGB_E_ARG, "channel_count must be 1..8");
    for (int s = 0; s < n_streams; s++) {
        const vgb_hca_info &b = info[s];
        if (b.channel_count != nch || b.frame_size != h0.frame_size || b.base_band_count != h0.base_band_count ||
            b.stereo_band_count != h0.stereo_band_count || b.total_band_count != h0.total_band_count ||
            b.hfr_band_count != h0.hfr_band_count || b.bands_per_hfr_group != h0.bands_per_hfr_group ||
            b.hfr_group_count != h0.hfr_group_count || b.track_count != h0.track_count || b.channel_config != h0.channel_config)
            return fail(VGB_E_ARG, "stream %d: all streams of one call must share the band layout and frame size", s);
        if ((b.use_ath_curve != 0) != (h0.use_ath_curve != 0) || (b.use_ath_curve && b.sample_rate != h0.sample_rate))
            return fail(VGB_E_ARG, "stream %d: all streams of one call must share UseAthCurve (and then the sample rate)", s);
        if (b.sample_count < 0 || b.frame_count < 0 || b.inserted_samples < 0) return fail(VGB_E_ARG, "stream %d: negative count", s);
    }
    if (h0.frame_size < 8 || h0.frame_size > 0xffff) return fail(VGB_E_ARG, "frame_size out of range");
    if (h0.base_band_count < 0 || h0.stereo_band_count < 0 || h0.base_band_count + h0.stereo_band_count > 128 ||
        h0.total_band_count > 128 || h0.hfr_group_count < 0 || h0.hfr_group_count > 8 ||
        (h0.hfr_group_count > 0 && h0.bands_per_hfr_group <= 0))
        return fail(VGB_E_ARG, "band layout out of range");
    if (h0.hfr_group_count > 0) {  // ReconstructHighFrequency mirrors bands around base+stereo: keep both sides in 0..127
        const int start = h0.base_band_count + h0.stereo_band_count;
        const int hfr_bands = std::min(h0.hfr_band_count, std::min(h0.total_band_count, 127) - h0.hfr_band_count);
        if (hfr_bands > start || start + hfr_bands > 128) return fail(VGB_E_ARG, "high-frequency band layout out of range");
    }
    HcaConfig cfg{};
    cfg.channel_count = nch;
    cfg.frame_size = h0.frame_size;
    cfg.base_band_count = h0.base_band_count;
    cfg.stereo_band_count = h0.stereo_band_count;
    cfg.total_band_count = h0.total_band_count;
    cfg.hfr_band_count = h0.hfr_band_count;
    cfg.bands_per_hfr_group = h0.bands_per_hfr_group;
    cfg.hfr_group_count = h0.hfr_group_count;
    hca_channel_types(h0, cfg.channel_type);
    hca_fill_ath(h0, cfg.ath);

    std::vector<HcaStream> streams(n_streams);
    std::vector<int64_t> in_off(n_streams), in_len(n_streams), out_off((size_t)n_streams * nch), out_len((size_t)n_streams * nch);
    int64_t ps = 0, fb = 0, frames_total = 0;
    int max_frames = 0;
    for (int s = 0; s < n_streams; s++) {
        const int64_t stride = (int64_t)align_up((size_t)info[s].sample_count, 8);
        streams[s].pcm_off = ps;
        streams[s].channel_stride = stride;
        streams[s].frames_off = fb;
        streams[s].dct_off = frames_total;
        streams[s].sample_count = info[s].sample_count;
        streams[s].frame_count = info[s].frame_count;
        streams[s].inserted_samples = info[s].inserted_samples;
        for (int c = 0; c < nch; c++) {
            if (!pcm_out[(size_t)s * nch + c] && info[s].sample_count > 0) return fail(VGB_E_ARG, "pcm_out[%d][%d] is NULL", s, c);
            out_off[(size_t)s * nch + c] = (ps + c * stride) * 2;
            out_len[(size_t)s * nch + c] = (int64_t)info[s].sample_count * 2;
        }
        ps += stride * nch;
        in_off[s] = fb;
        in_len[s] = (int64_t)info[s].frame_count * info[s].frame_size;
        if (!frames[s] && in_len[s] > 0) return fail(VGB_E_ARG, "frames[%d] is NULL", s);
        fb += (int64_t)align_up((size_t)in_len[s], 16);
        max_frames = std::max(max_frames, info[s].frame_count);
        frames_total += info[s].frame_count;
    }

    // stream groups: H2D of the frames of group g+1 || decode of group g || D2H of the PCM of group g-1
    std::vector<int64_t> weight(n_streams);
    int64_t pcie_bytes = 0;
    for (int s = 0; s < n_streams; s++) {
        weight[s] = (int64_t)info[s].frame_count + 1;
        pcie_bytes += in_len[s] + (int64_t)info[s].sample_count * 2 * nch;
    }
    const int n_groups = pipeline_group_count(n_streams, pcie_bytes, 16);
    const std::vector<int> bound = pipeline_bounds(weight, n_groups);
    // per-group scratch: the seam addends (2 x 128 doubles per channel-frame) and the parse records; the kernels index
    // both by the group-relative frame number, so dct_off restarts at every group
    std::vector<int64_t> g_frames(n_groups, 0);
    std::vector<int> g_max(n_groups, 0);
    std::vector<size_t> edge_at(n_groups), parsed_at(n_groups);
    size_t edge_total = 0, parsed_total = 0;
    for (int g = 0; g < n_groups; g++) {
        for (int s = bound[g]; s < bound[g + 1]; s++) {
            streams[s].dct_off = g_frames[g];
            g_frames[g] += info[s].frame_count;
            g_max[g] = std::max(g_max[g], info[s].frame_count);
        }
        edge_at[g] = edge_total;
        edge_total += align_up((size_t)g_frames[g] * nch * 2 * 128 * sizeof(double), 256);
        parsed_at[g] = parsed_total;
        parsed_total += align_up(hca_decode_parsed_bytes(cfg, g_frames[g]), 256);
    }
    (void)max_frames;

    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    VGB_TRY(hca_tables_ready_locked());
    const size_t o_status = align_up(streams.size() * sizeof(HcaStream), 256);
    const size_t o_edge = align_up(o_status + (size_t)n_streams * 4, 256);
    const size_t o_parsed = align_up(o_edge + edge_total, 256);
    VGB_TRY(g_ctx.pcm.reserve((size_t)(ps + 8) * 2));
    VGB_TRY(g_ctx.adpcm.reserve((size_t)fb + 16));
    VGB_TRY(g_ctx.misc.reserve(o_parsed + parsed_total + 256));
    char *misc = static_cast<char *>(g_ctx.misc.p);
    const HcaStream *d_streams = reinterpret_cast<const HcaStream *>(misc);
    int32_t *d_status = reinterpret_cast<int32_t *>(misc + o_status);
    std::vector<int32_t> status(n_streams, 0);
    auto h2d = [&](int g) -> int32_t {
        if (g == 0) {
            CUDA_TRY(cudaMemcpyAsync(misc, streams.data(), streams.size() * sizeof(HcaStream), cudaMemcpyHostToDevice, g_ctx.s_in));
            CUDA_TRY(cudaMemsetAsync(misc + o_status, 0, (size_t)n_streams * 4, g_ctx.s_in));
            // samples past the last frame (sample_count > frame_count * 1024 - inserted) stay zero, like a fresh short[]
            CUDA_TRY(cudaMemsetAsync(g_ctx.pcm.p, 0, (size_t)ps * 2, g_ctx.s_in));
        }
        const int s0 = bound[g], n = bound[g + 1] - s0;
        return copy_channels_in(static_cast<char *>(g_ctx.adpcm.p), std::vector<int64_t>(in_off.begin() + s0, in_off.begin() + s0 + n), frames + s0,
                                std::vector<int64_t>(in_len.begin() + s0, in_len.begin() + s0 + n), g_ctx.s_in);
    };
    auto kern = [&](int g, cudaStream_t st) -> int32_t {
        const int s0 = bound[g], n = bound[g + 1] - s0;
        if (n == 0 || g_frames[g] == 0) return VGB_OK;
        if (n_groups == 1) tick(7, true, st);
        CUDA_TRY(launch_hca_decode(static_cast<const uint8_t *>(g_ctx.adpcm.p), d_streams + s0, n, g_max[g], g_frames[g], cfg, g_hca_tables.view,
                                   reinterpret_cast<uint8_t *>(misc + o_parsed + parsed_at[g]), reinterpret_cast<double *>(misc + o_edge + edge_at[g]),
                                   static_cast<int16_t *>(g_ctx.pcm.p), d_status + s0, st));
        if (n_groups == 1) tick(7, false, st);
        g_ctx.launches += 3;
        return VGB_OK;
    };
    auto d2h = [&](int g) -> int32_t {
        const int s0 = bound[g], n = bound[g + 1] - s0;
        if (n > 0) CUDA_TRY(cudaMemcpyAsync(status.data() + s0, d_status + s0, (size_t)n * 4, cudaMemcpyDeviceToHost, g_ctx.s_out));
        const size_t c0 = (size_t)s0 * nch, c1 = (size_t)(s0 + n) * nch;
        return copy_channels_out(pcm_out + c0, static_cast<const char *>(g_ctx.pcm.p), std::vector<int64_t>(out_off.begin() + c0, out_off.begin() + c1),
                                 std::vector<int64_t>(out_len.begin() + c0, out_len.begin() + c1), g_ctx.s_out);
    };
    VGB_TRY(run_group_pipeline(n_groups, h2d, kern, d2h, [](int) { return VGB_OK; }));
    for (int s = 0; s < n_streams; s++) {
        if (status[s] == VGB_HCA_BAD_SYNC) return fail(VGB_E_DATA, "stream %d: Invalid frame header", s);
        if (status[s] == VGB_HCA_BAD_DELTA) return fail(VGB_E_DATA, "stream %d: scale factor delta out of range", s);
        if (status[s] == VGB_HCA_BAD_INDEX) return fail(VGB_E_DATA, "stream %d: intensity index out of range", s);
    }
    return VGB_OK;
}

// ---- block (de)interleave (Utilities/Interleave.cs:9-166) ---------------------------------------------------------
namespace {
int32_t interleave_check(int32_t n_items, int32_t count, int64_t in_size, int32_t interleave_size, int64_t out_size)
{
    if (n_items < 0 || count <= 0) return fail(VGB_E_ARG, "bad item / channel count");
    if (interleave_size <= 0) return fail(VGB_E_ARG, "interleave size must be positive");
    if (in_size < 0 || out_size < 0) return fail(VGB_E_ARG, "negative size");
    return VGB_OK;
}
}  // namespace

// Launches with g_ctx.mu already held (shared by the *_dev entry points and the host-pointer wrappers, which keep the
// lock across staging, launch and read-back: every entry point may reserve() - free and reallocate - the shared slabs).
static int32_t interleave_locked(const void *d_in, int64_t in_channel_stride, int64_t in_item_stride, void *d_out, int64_t out_item_stride,
                                 int32_t n_items, int32_t count, int64_t in_size, int32_t interleave_size, int64_t out_size, cudaStream_t st)
{
    tick(8, true, st);
    CUDA_TRY(launch_interleave(d_in, in_channel_stride, in_item_stride, d_out, out_item_stride, n_items, count, in_size, interleave_size,
                               out_size, st));
    tick(8, false, st);
    g_ctx.launches += 1;
    return VGB_OK;
}

static int32_t deinterleave_locked(const void *d_in, int64_t in_item_stride, void *d_out, int64_t out_channel_stride, int64_t out_item_stride,
                                   int32_t n_items, int32_t count, int64_t in_size, int32_t interleave_size, int64_t out_size, cudaStream_t st)
{
    tick(9, true, st);
    CUDA_TRY(launch_deinterleave(d_in, in_item_stride, d_out, out_channel_stride, out_item_stride, n_items, count, in_size,
                                 interleave_size, out_size, st));
    tick(9, false, st);
    g_ctx.launches += 1;
    return VGB_OK;
}

int32_t vgb_interleave_dev(const void *d_in, int64_t in_channel_stride, int64_t in_item_stride, void *d_out, int64_t out_item_stride,
                           int32_t n_items, int32_t count, int64_t in_size, int32_t interleave_size, int64_t out_size, void *cuda_stream)
{
    if (out_size == -1) out_size = in_size;
    VGB_TRY(interleave_check(n_items, count, in_size, interleave_size, out_size));
    if (n_items == 0 || out_size == 0) return VGB_OK;
    if (!d_in || !d_out) return fail(VGB_E_ARG, "NULL argument");
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    return interleave_locked(d_in, in_channel_stride, in_item_stride, d_out, out_item_stride, n_items, count, in_size, interleave_size,
                             out_size, static_cast<cudaStream_t>(cuda_stream));
}

int32_t vgb_deinterleave_dev(const void *d_in, int64_t in_item_stride, void *d_out, int64_t out_channel_stride, int64_t out_item_stride,
                             int32_t n_items, int32_t count, int64_t in_size, int32_t interleave_size, int64_t out_size, void *cuda_stream)
{
    if (out_size == -1) out_size = in_size;
    VGB_TRY(interleave_check(n_items, count, in_size, interleave_size, out_size));
    if (n_items == 0 || out_size == 0) return VGB_OK;
    if (!d_in || !d_out) return fail(VGB_E_ARG, "NULL argument");
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    return deinterleave_locked(d_in, in_item_stride, d_out, out_channel_stride, out_item_stride, n_items, count, in_size, interleave_size,
                               out_size, static_cast<cudaStream_t>(cuda_stream));
}

int32_t vgb_interleave(const uint8_t *const *inputs, int32_t count, int32_t in_size, int32_t interleave_size, int32_t out_size,
                       uint8_t *output)
{
    if (out_size == -1) out_size = in_size;
    VGB_TRY(interleave_check(1, count, in_size, interleave_size, out_size));
    if (out_size == 0) return VGB_OK;
    if (!inputs || !output) return fail(VGB_E_ARG, "NULL argument");
    for (int c = 0; c < count; c++)
        if (!inputs[c] && in_size > 0) return fail(VGB_E_ARG, "inputs[%d] is NULL", c);
    const int64_t pitch = (int64_t)align_up((size_t)in_size, 16), out_bytes = (int64_t)out_size * count;
    std::lock_guard<std::mutex> lock(g_ctx.mu);  // one lock for staging, launch and read-back
    VGB_TRY(ensure_ready_locked());
    VGB_TRY(g_ctx.pcm.reserve((size_t)pitch * count + 16));
    VGB_TRY(g_ctx.adpcm.reserve((size_t)out_bytes + 16));
    for (int c = 0; c < count; c++)
        if (in_size > 0)
            CUDA_TRY(cudaMemcpyAsync(static_cast<char *>(g_ctx.pcm.p) + c * pitch, inputs[c], (size_t)in_size, cudaMemcpyHostToDevice, g_ctx.stream));
    VGB_TRY(interleave_locked(g_ctx.pcm.p, pitch, 0, g_ctx.adpcm.p, 0, 1, count, in_size, interleave_size, out_size, g_ctx.stream));
    CUDA_TRY(cudaMemcpyAsync(output, g_ctx.adpcm.p, (size_t)out_bytes, cudaMemcpyDeviceToHost, g_ctx.stream));
    CUDA_TRY(cudaStreamSynchronize(g_ctx.stream));
    return VGB_OK;
}

int32_t vgb_deinterleave(const uint8_t *input, int32_t length, int32_t interleave_size, int32_t count, int32_t out_size,
                         uint8_t *const *outputs)
{
    if (count <= 0) return fail(VGB_E_ARG, "bad channel count");
    if (length < 0 || length % count != 0)  // ArgumentOutOfRangeException (Interleave.cs:84-86)
        return fail(VGB_E_ARG, "The input array length (%d) must be divisible by the number of outputs.", length);
    const int32_t in_size = length / count;
    if (out_size == -1) out_size = in_size;
    VGB_TRY(interleave_check(1, count, in_size, interleave_size, out_size));
    if (out_size == 0) return VGB_OK;
    if ((!input && length > 0) || !outputs) return fail(VGB_E_ARG, "NULL argument");
    for (int c = 0; c < count; c++)
        if (!outputs[c]) return fail(VGB_E_ARG, "outputs[%d] is NULL", c);
    const int64_t pitch = (int64_t)align_up((size_t)out_size, 16);
    std::lock_guard<std::mutex> lock(g_ctx.mu);  // one lock for staging, launch and read-back
    VGB_TRY(ensure_ready_locked());
    VGB_TRY(g_ctx.adpcm.reserve((size_t)length + 16));
    VGB_TRY(g_ctx.pcm.reserve((size_t)pitch * count + 16));
    if (length > 0) CUDA_TRY(cudaMemcpyAsync(g_ctx.adpcm.p, input, (size_t)length, cudaMemcpyHostToDevice, g_ctx.stream));
    VGB_TRY(deinterleave_locked(g_ctx.adpcm.p, 0, g_ctx.pcm.p, pitch, 0, 1, count, in_size, interleave_size, out_size, g_ctx.stream));
    for (int c = 0; c < count; c++)
        CUDA_TRY(cudaMemcpyAsync(outputs[c], static_cast<char *>(g_ctx.pcm.p) + c * pitch, (size_t)out_size, cudaMemcpyDeviceToHost, g_ctx.stream));
    CUDA_TRY(cudaStreamSynchronize(g_ctx.stream));
    return VGB_OK;
}

}  // extern "C"

// ---- public host-pointer entry points: shard over the bound devices, or run on the one device --------------------------
extern "C" {

int32_t vgb_gcadpcm_decode_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int16_t *coefs,
                                 const vgb_gc_params *params, int32_t n_channels, int16_t *const *pcm_out)
{
    if (!sharding_active(n_channels) || !adpcm || !n_bytes || !coefs || !pcm_out)
        return gcadpcm_decode_one(adpcm, n_bytes, coefs, params, n_channels, pcm_out);
    std::vector<int64_t> weight(n_channels);
    for (int c = 0; c < n_channels; c++) weight[c] = (int64_t)std::max(n_bytes[c], 0) + 64;
    return run_sharded(shard_units(weight, 1 + (int)g_extra.size()), [&](int, const std::vector<int> &u) -> int32_t {
        const int m = (int)u.size();
        auto s_in = pick(adpcm, u);
        auto s_nb = pick(n_bytes, u);
        auto s_out = pick(pcm_out, u);
        std::vector<vgb_gc_params> s_par;
        if (params) s_par = pick(params, u);
        std::vector<int16_t> s_co((size_t)m * 16);
        for (int i = 0; i < m; i++) std::memcpy(&s_co[(size_t)i * 16], coefs + (size_t)u[i] * 16, 32);
        return gcadpcm_decode_one(s_in.data(), s_nb.data(), s_co.data(), params ? s_par.data() : nullptr, m, s_out.data());
    });
}

int32_t vgb_adx_encode_batch(const int16_t *const *pcm, const int32_t *n_samples, const vgb_adx_params *params,
                             int32_t n_channels, int16_t *history_out, uint8_t *const *adpcm_out, vgb_progress_cb cb, void *user)
{
    if (!sharding_active(n_channels) || !pcm || !n_samples || !params || !adpcm_out)
        return adx_encode_one(pcm, n_samples, params, n_channels, history_out, adpcm_out, cb, user);
    std::vector<int64_t> weight(n_channels);
    for (int c = 0; c < n_channels; c++) weight[c] = (int64_t)std::max(n_samples[c], 0) + 64;
    SharedProgress prog{cb, user, {}};
    return run_sharded(shard_units(weight, 1 + (int)g_extra.size()), [&](int, const std::vector<int> &u) -> int32_t {
        const int m = (int)u.size();
        auto s_pcm = pick(pcm, u);
        auto s_n = pick(n_samples, u);
        auto s_par = pick(params, u);
        auto s_out = pick(adpcm_out, u);
        std::vector<int16_t> s_hist(m);
        VGB_TRY(adx_encode_one(s_pcm.data(), s_n.data(), s_par.data(), m, s_hist.data(), s_out.data(), cb ? SharedProgress::relay : nullptr, &prog));
        if (history_out) for (int i = 0; i < m; i++) history_out[u[i]] = s_hist[i];
        return VGB_OK;
    });
}

int32_t vgb_adx_decode_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int32_t *sample_count,
                             const vgb_adx_params *params, int32_t n_channels, int16_t *const *pcm_out)
{
    if (!sharding_active(n_channels) || !adpcm || !n_bytes || !sample_count || !params || !pcm_out)
        return adx_decode_one(adpcm, n_bytes, sample_count, params, n_channels, pcm_out);
    std::vector<int64_t> weight(n_channels);
    for (int c = 0; c < n_channels; c++) weight[c] = (int64_t)std::max(sample_count[c], 0) + 64;
    return run_sharded(shard_units(weight, 1 + (int)g_extra.size()), [&](int, const std::vector<int> &u) -> int32_t {
        auto s_in = pick(adpcm, u);
        auto s_nb = pick(n_bytes, u);
        auto s_sc = pick(sample_count, u);
        auto s_par = pick(params, u);
        auto s_out = pick(pcm_out, u);
        return adx_decode_one(s_in.data(), s_nb.data(), s_sc.data(), s_par.data(), (int)u.size(), s_out.data());
    });
}

int32_t vgb_hca_encode_batch(const int16_t *const *pcm, const vgb_hca_params *params, int32_t n_streams,
                             vgb_hca_info *info_out, uint8_t *const *frames_out, vgb_progress_cb cb, void *user)
{
    if (!sharding_active(n_streams) || !pcm || !params || !frames_out)
        return hca_encode_one(pcm, params, n_streams, info_out, frames_out, cb, user);
    const int nch = params[0].channel_count;
    if (nch < 1 || nch > 8) return hca_encode_one(pcm, params, n_streams, info_out, frames_out, cb, user);
    std::vector<int64_t> weight(n_streams);
    for (int s = 0; s < n_streams; s++) weight[s] = (int64_t)std::max(params[s].sample_count, 0) + 1024;
    SharedProgress prog{cb, user, {}};
    return run_sharded(shard_units(weight, 1 + (int)g_extra.size()), [&](int, const std::vector<int> &u) -> int32_t {
        const int m = (int)u.size();
        std::vector<const int16_t *> s_pcm((size_t)m * nch);
        for (int i = 0; i < m; i++)
            for (int c = 0; c < nch; c++) s_pcm[(size_t)i * nch + c] = pcm[(size_t)u[i] * nch + c];
        auto s_par = pick(params, u);
        auto s_out = pick(frames_out, u);
        std::vector<vgb_hca_info> s_info(m);
        VGB_TRY(hca_encode_one(s_pcm.data(), s_par.data(), m, s_info.data(), s_out.data(), cb ? SharedProgress::relay : nullptr, &prog));
        if (info_out) for (int i = 0; i < m; i++) info_out[u[i]] = s_info[i];
        return VGB_OK;
    });
}

int32_t vgb_hca_decode_batch(const uint8_t *const *frames, const vgb_hca_info *info, int32_t n_streams, int16_t *const *pcm_out)
{
    if (!sharding_active(n_streams) || !frames || !info || !pcm_out) return hca_decode_one(frames, info, n_streams, pcm_out);
    const int nch = info[0].channel_count;
    if (nch < 1 || nch > 8) return hca_decode_one(frames, info, n_streams, pcm_out);
    std::vector<int64_t> weight(n_streams);
    for (int s = 0; s < n_streams; s++) weight[s] = (int64_t)std::max(info[s].frame_count, 0) + 1;
    return run_sharded(shard_units(weight, 1 + (int)g_extra.size()), [&](int, const std::vector<int> &u) -> int32_t {
        const int m = (int)u.size();
        auto s_in = pick(frames, u);
        auto s_info = pick(info, u);
        std::vector<int16_t *> s_out((size_t)m * nch);
        for (int i = 0; i < m; i++)
            for (int c = 0; c < nch; c++) s_out[(size_t)i * nch + c] = pcm_out[(size_t)u[i] * nch + c];
        return hca_decode_one(s_in.data(), s_info.data(), m, s_out.data());
    });
}

}  // extern "C"
