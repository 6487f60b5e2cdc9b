// abi.cuh — the host runtime shared by the translation units of the C ABI (c_abi.cu, abi_*.cu, containers.cu,
// collective.cu): error reporting, device buffers, the per-device context, pinning, copies, the grouped
// H2D / kernel / D2H pipeline of a host call and the sharding of a host call over several devices.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/vgaudio_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace vgb {

extern thread_local std::string g_err;               // vgb_last_error() of this thread
int32_t fail(int32_t code, const char *fmt, ...);    // sets g_err, returns `code`

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

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// VGB_E_ARG unless the caller's device pointer `p` (argument `name`) is `a`-byte aligned (a power of two; NULL passes).
// The _dev entry points check their base pointers with it before any device work: the kernels behind them read and
// write with vector loads, cp.async copies and 8-byte fields that would fault the context on a misaligned address.
inline int32_t check_aligned(const void *p, size_t a, const char *name)
{
    if (reinterpret_cast<uintptr_t>(p) & (a - 1)) return fail(VGB_E_ARG, "%s=%p must be %zu-byte aligned", name, p, a);
    return VGB_OK;
}

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
    char *c() const { return static_cast<char *>(p); }
};

constexpr int kTimers = 10;  // 0 coef phase 1, 1 coef refine, 2 gc encode, 3 gc decode, 4 adx encode, 5 adx decode, 6 hca encode, 7 hca decode, 8 interleave, 9 deinterleave
constexpr int kMaxGroups = 16;   // channel groups of one host call, pipelined: H2D(g+1) || kernels(g) || D2H(g-1)
constexpr int kCompStreams = 4;  // kernel streams the groups rotate over

struct ContainerState;  // containers.cu: the container layer's streams, events and working sets on one device

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
    AdxSegArgs last_adx_enc{};       // the same for the most recent ADX encode launch (vgb_adx_debug_encode_stats)
    AdxDecSegArgs last_adx_dec{};    // and time-parallel ADX decode (vgb_adx_debug_decode_stats)
    GcDecSegArgs last_gc_dec{};      // and GC-ADPCM decode (vgb_gcadpcm_debug_decode_stats)
    HcaTableStore hca_tables;
    std::atomic<ContainerState *> containers{nullptr};  // created on first use, released by containers_release
};

extern Context g_primary;                               // the device vgb_init / vgb_init_devices binds first
extern std::vector<std::unique_ptr<Context>> g_extra;   // further devices of vgb_init_devices
extern thread_local Context *t_ctx;                     // the context this thread works on
#define g_ctx (*t_ctx)

int32_t ensure_ready_locked();
void hca_tables_release_locked();  // abi_hca.cu
// abi_hca.cu, the HCA decoder's rules, shared by vgb_hca_decode_batch / _dev and the .hca -> WAVE converter:
HcaConfig hca_config(const vgb_hca_info &h0);  // the codec configuration of a call, from the HcaInfo its streams share
bool hca_same_config(const vgb_hca_info &a, const vgb_hca_info &b);  // one decode launch can take both streams
int32_t hca_decode_check(const vgb_hca_info *info, int32_t n_streams);  // VGB_E_ARG unless one launch can decode all (n >= 1)
int32_t hca_decode_fault(int32_t status, const char *what, int index);  // a decoder status word as the reference's exception
// synchronises `st` and copies the status words of the last vgb_hca_decode_dev on `d_workspace` to status[0..n)
int32_t hca_decode_words(const void *d_workspace, int32_t n_streams, int32_t *status, cudaStream_t st);
// the same for the encoder's status words of the last vgb_hca_encode_dev on `d_workspace`, and one such word as the
// reference's exception ("<what> <index>: Bitrate is set too low." ...)
int32_t hca_encode_words(const void *d_workspace, int32_t n_streams, int32_t *status, cudaStream_t st);
int32_t hca_encode_fault(int32_t status, const char *what, int index);
// abi_adx.cu: synchronises `st` and copies the per-channel status words of the last vgb_adx_decode_dev on `d_workspace`
// (bit 0: a Fixed-type frame selects a filter 4..7, bit 1: a frame of another type a filter 1..7) to status[0..n)
int32_t adx_decode_words(const void *d_workspace, int32_t n_channels, int32_t *status, cudaStream_t st);
// abi_gcadpcm.cu, the time-parallel GC-ADPCM decode of the NintendoWare -> WAVE converter: workspace bytes for
// n_channels channels holding full_frames full frames in all, the asynchronous decode (tab: host table; trace_off is
// filled here), and the per-channel status words (bit 0: a predictor 8..15), which synchronise `st`.  With d_coefs
// (16 coefficients per channel, channel-major, on the device) the table's coefficients are taken from there in stream
// order instead of from `tab`, so an encoder's output can be decoded without a round trip to the host.
uint64_t gc_decode_seg_workspace_bytes(int32_t n_channels, int64_t full_frames);
int32_t gc_decode_seg(const uint8_t *d_adpcm, std::vector<GcDecChannel> &tab, int16_t *d_pcm, void *d_workspace, cudaStream_t st,
                      const int16_t *d_coefs = nullptr);
int32_t gc_decode_seg_words(const void *d_workspace, int32_t n_channels, int32_t *status, cudaStream_t st);
// abi_gcadpcm.cu, GcAdpcmAlignment's tail (GcAdpcmAlignment.cs:44-57) on device rows, as vgb_gcadpcm_align_batch runs it:
// per channel the samples to re-encode from its first decode at d_src + src_off, encoded with its own coefficients
// (d_coefs, 16 per channel, in `chans` order) from the history in front of the kept frames.  dst_off is filled here;
// tail_adpcm_off receives each channel's encoded tail as a byte offset into d_workspace.  Asynchronous on `st`.
uint64_t gc_align_tails_workspace_bytes(const std::vector<GcAlignChannel> &chans);
int32_t gc_align_tails(const int16_t *d_src, std::vector<GcAlignChannel> &chans, const int16_t *d_coefs, void *d_workspace, cudaStream_t st,
                       std::vector<int64_t> &tail_adpcm_off);
void tick(int slot, bool begin, cudaStream_t stream);

// hooks of containers.cu, which keeps its own slabs and streams per context (Context::containers)
int32_t abi_ensure_ready();              // readies the calling thread's context and makes its device current
void abi_count_launches(int n);          // vgb_kernel_launch_count bookkeeping of the calling thread's context
void containers_release(Context &ctx);   // vgb_shutdown: drains and frees ctx's container state

// ---- pinning and copies ----------------------------------------------------------------------------------------
// Pageable caller buffers (a C# short[] pinned by the GC is still pageable for CUDA) move through the driver's staging
// buffers at a fraction of PCIe speed; page-locking the region for the duration of the call costs some ms per GiB and
// lets the copy engine read it directly at PCIe speed (tools/host_register_probe.py compares the two).  Inputs only: they are touched memory; registering a freshly allocated output would
// fault its pages in first and cost more than it saves.  Registrations live until the API call returns (PinScope).
struct PinScope {
    ~PinScope();
};
void try_pin(const void *p, size_t bytes);

// Many small copies in one driver call (cudaMemcpyBatchAsync, CUDA 12.8+): a ragged batch of tens of thousands of short
// files otherwise spends more host time in cudaMemcpyAsync calls (~5 us each) than the copies take on the link.  Falls
// back to one call per copy when the batched call is refused.  Zero-length copies are dropped.
struct CopyList {
    std::vector<void *> dst, src;
    std::vector<size_t> size;
    void add(void *d, const void *s, size_t n) { if (n) { dst.push_back(d); src.push_back(const_cast<void *>(s)); size.push_back(n); } }
    int32_t run(cudaMemcpyKind kind, cudaStream_t st);
};

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

// Copy of units [first, first + count) between the caller's buffers h_ptr[u] and the device slab (d_base + d_off[u],
// bytes[u] bytes each): one 2D copy when the host rows are one contiguous block and the device rows evenly spaced, else
// one copy per non-empty unit.  Host -> device copies pin their sources.
template <typename T>
int32_t copy_units(cudaMemcpyKind kind, char *d_base, const int64_t *d_off, T *const *h_ptr, const int64_t *bytes,
                   int first, int count, cudaStream_t stream)
{
    if (count <= 0) return VGB_OK;
    d_off += first;
    h_ptr += first;
    bytes += first;
    const bool in = kind == cudaMemcpyHostToDevice;
    auto host = [&](int c) { return const_cast<void *>(static_cast<const void *>(h_ptr[c])); };
    bool same = true;
    for (int c = 1; c < count; c++) same = same && bytes[c] == bytes[0];
    int64_t hstride = 0;
    // a strided copy takes pitches below 2 GiB (cudaDevAttrMaxPitch).  The host rows must touch end to end: separate
    // caller arrays can be evenly spaced as well, and a copy (or a page-lock) over the span between them covers memory
    // the caller never handed over - other buffers, one of them perhaps page-locked by this call, and a host range that
    // starts inside a registration and runs past its end is refused as an invalid argument.
    constexpr int64_t kMaxPitch = INT32_MAX;
    if (same && count > 1 && bytes[0] > 0 && uniform_stride(h_ptr, count, hstride) && hstride == bytes[0] &&
        hstride <= kMaxPitch) {
        const int64_t dstride = d_off[1] - d_off[0];
        bool dsame = dstride > 0 && dstride <= kMaxPitch;
        for (int c = 2; c < count; c++) dsame = dsame && (d_off[c] - d_off[c - 1] == dstride);
        if (dsame) {
            char *d = d_base + d_off[0];
            if (in) try_pin(host(0), (size_t)(hstride * (count - 1) + bytes[0]));
            CUDA_TRY(cudaMemcpy2DAsync(in ? d : host(0), (size_t)(in ? dstride : hstride), in ? (const void *)host(0) : d,
                                       (size_t)(in ? hstride : dstride), (size_t)bytes[0], (size_t)count, kind, stream));
            return VGB_OK;
        }
    }
    CopyList list;
    for (int c = 0; c < count; c++) {
        if (in && bytes[c] > 0) try_pin(host(c), (size_t)bytes[c]);
        if (in) list.add(d_base + d_off[c], host(c), (size_t)std::max<int64_t>(bytes[c], 0));
        else list.add(host(c), d_base + d_off[c], (size_t)std::max<int64_t>(bytes[c], 0));
    }
    return list.run(kind, stream);
}

// ---- host-call pipeline over groups of independent units (channels / streams) ------------------------------------------
// Every host-pointer entry point moves bytes over PCIe on both sides of its kernels.  Units are independent, so the
// call is cut into groups: the H2D copy of group g+1, the kernels of group g and the D2H copy of group g-1 overlap on
// three kinds of streams.  `h2d(g)` enqueues on g_ctx.s_in, `kern(g, stream, mid)` on one of the kernel streams and
// records `mid` there (vgb_debug_last_coefs_done), `d2h(g)` on g_ctx.s_out, and `done(g)` runs on the calling thread
// once group g's output has landed; the helper adds the events, the timeline taps and the final synchronisation.
// Returns with nothing in flight, also on error (caller memory may be unpinned / freed right after).
struct PipelineDrain {
    ~PipelineDrain();
};

// how many groups for `units` units carrying `bytes` bytes over PCIe in total (both directions); the environment
// variable `env` (1..kMaxGroups) overrides it
int pipeline_group_count(int64_t units, int64_t bytes, int min_units_per_group, const char *env = "VGB_PIPELINE_GROUPS");

// group boundaries over units with the given weights (roughly equal weight per group, order preserved)
std::vector<int> pipeline_bounds(const std::vector<int64_t> &weight, int n_groups);

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
        VGB_TRY(kern(g, st, g_ctx.ev_mid[g]));
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

// kern(g, stream) of a call whose kernels are one phase: `mid` is recorded when they finish
template <class Kern>
auto one_phase(Kern kern)
{
    return [kern](int g, cudaStream_t st, cudaEvent_t mid) -> int32_t {
        VGB_TRY(kern(g, st));
        CUDA_TRY(cudaEventRecord(mid, st));
        return VGB_OK;
    };
}

inline int32_t no_done(int) { return VGB_OK; }

// ---- several devices in one process (vgb_init_devices) ----------------------------------------------------------------
// The reference's counterpart is Parallel.ForEach over files (src/VGAudio.Cli/Batch.cs:24-25) on top of Parallel.For over
// channels: independent units.  A host-pointer batch call is sharded over the bound devices by greedy longest-first
// bin packing of the units' sample counts; every device gets a worker thread that runs the ordinary single-device call
// (its own H2D / kernels / D2H pipeline over its own PCIe link) on its share, results land directly in the caller's
// arrays.  No collective is involved: host data reaches each GPU fastest over that GPU's own link (SURVEY §8e); the NCCL
// scatterv / gatherv of collective.cu serve data that is already resident on one device.
// greedy LPT over the bound devices: heaviest unit first onto the least loaded device; a device's units keep ascending
// order.  Unit u of n weighs max(size(u), 0) + extra.
template <class Size>
std::vector<std::vector<int>> shard_units(int n, Size size, int64_t extra)
{
    std::vector<int> order(n);
    std::vector<int64_t> weight(n);
    for (int i = 0; i < n; i++) { order[i] = i; weight[i] = std::max<int64_t>(size(i), 0) + extra; }
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return weight[a] > weight[b]; });
    const int n_dev = 1 + (int)g_extra.size();
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

bool sharding_active(int n_units);

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
// message gets " (device N)" appended.  With `readdress`, a message that starts with "channel N" / "stream N" is also
// re-addressed from the shard-local unit index to the caller's; callers whose messages already name the caller's
// indices, or whose channel / stream numbers are not shard units, pass false.
template <class Fn>
int32_t run_sharded(const std::vector<std::vector<int>> &shards, Fn fn, bool readdress = true)
{
    std::vector<Context *> ctxs{&g_primary};
    for (auto &c : g_extra) ctxs.push_back(c.get());
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
                if (!readdress) break;
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

// gather: the `width` elements of row u of `src` for every u of `units`, in that order
template <class T>
std::vector<T> pick_rows(const T *src, const std::vector<int> &units, size_t width = 1)
{
    std::vector<T> v(units.size() * width);
    for (size_t i = 0; i < units.size(); i++) std::copy_n(src + units[i] * width, width, v.begin() + i * width);
    return v;
}

// scatter: the inverse of pick_rows
template <class T>
void put_rows(T *dst, const std::vector<int> &units, const std::vector<T> &rows, size_t width = 1)
{
    for (size_t i = 0; i < units.size(); i++) std::copy_n(rows.begin() + i * width, width, dst + units[i] * width);
}

}  // namespace vgb
