// c_abi.cu — the extern "C" boundary of libvgaudio_b200.so (declared in include/vgaudio_b200.h).
//
// Host-side responsibilities only: argument validation with the reference's error behaviour, HBM layout of a
// batch (channel slabs + tables), H2D/D2H movement, kernel sequencing on one stream, timing taps.
// No codec arithmetic happens on the CPU here; without a CUDA device every codec entry point fails (VGB_E_CUDA).
// This file holds the shared runtime declared in abi.cuh and the codec-independent entry points (devices, host memory,
// launch count, timers, debug taps, interleave); abi_gcadpcm.cu, abi_adx.cu and abi_hca.cu hold the codecs.
#include <cstdarg>
#include <cstdio>
#include <map>

#include "abi.cuh"

namespace vgb {

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

Context g_primary;
std::vector<std::unique_ptr<Context>> g_extra;
thread_local Context *t_ctx = &g_primary;

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

void tick(int slot, bool begin, cudaStream_t stream)
{
    if (!g_ctx.timing) return;
    cudaEventRecord(g_ctx.ev[2 * slot + (begin ? 0 : 1)], stream);
    if (!begin) g_ctx.ev_used[slot] = true;
}

thread_local std::vector<void *> t_pins;

PinScope::~PinScope()
{
    for (void *p : t_pins) cudaHostUnregister(p);
    t_pins.clear();
    (void)cudaGetLastError();
}

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

// Whether every host-side address of the list is page-locked (vgb_host_alloc, cudaHostRegister, pinned framework
// buffers).  With pageable caller memory, cudaMemcpyBatchAsync with stream-ordered source access faulted on the H100:
// a group of 3571 NintendoWare wave images of 3-260 KB crashed the calling thread inside the call, or left the context
// with an unspecified launch failure, with or without slack behind every image, before any kernel ran; one
// cudaMemcpyAsync per region copied the same group clean.  Pageable regions therefore take the per-copy path.
static bool host_side_locked(const std::vector<void *> &host)
{
    for (void *p : host) {
        cudaPointerAttributes attr;
        if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
        if (attr.type != cudaMemoryTypeHost) return false;
    }
    return true;
}

int32_t CopyList::run(cudaMemcpyKind kind, cudaStream_t st)
{
    const size_t n = size.size();
    if (n == 0) return VGB_OK;
    static bool batch_ok = std::getenv("VGB_NO_MEMCPY_BATCH") == nullptr;
    const bool locked = kind == cudaMemcpyHostToDevice ? host_side_locked(src) : kind == cudaMemcpyDeviceToHost ? host_side_locked(dst) : true;
    if (batch_ok && n >= 16 && locked) {
        cudaMemcpyAttributes attr{};
        attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;  // sources stay valid until the call returns (we synchronise)
        attr.flags = 0;
        size_t attr_idx = 0, fail_idx = 0;
        const cudaError_t e = cudaMemcpyBatchAsync(dst.data(), src.data(), size.data(), n, &attr, &attr_idx, 1, &fail_idx, st);
        if (e == cudaSuccess) return VGB_OK;
        (void)cudaGetLastError();
        batch_ok = false;  // e.g. an older driver: stay on the per-copy path for the rest of the process
    }
    for (size_t i = 0; i < n; i++) CUDA_TRY(cudaMemcpyAsync(dst[i], src[i], size[i], kind, st));
    return VGB_OK;
}

PipelineDrain::~PipelineDrain()
{
    cudaStreamSynchronize(g_ctx.s_in);
    for (auto st : g_ctx.s_comp) cudaStreamSynchronize(st);
    cudaStreamSynchronize(g_ctx.s_out);
    (void)cudaGetLastError();
}

int pipeline_group_count(int64_t units, int64_t bytes, int min_units_per_group, const char *env_name)
{
    int64_t n = std::min<int64_t>(kMaxGroups / 2, std::min<int64_t>(bytes / (32 << 20), units / std::max(min_units_per_group, 1)));
    if (const char *env = std::getenv(env_name)) {  // tuning knob: 1..kMaxGroups
        const int want = std::atoi(env);
        if (want >= 1 && want <= kMaxGroups && units >= want) n = want;
    }
    return (int)std::max<int64_t>(n, 1);
}

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

cudaError_t raise_dynamic_smem(const void *kernel, size_t bytes)
{
    static std::mutex mu;
    static std::map<std::pair<const void *, int>, size_t> raised;  // (kernel, device) -> the attribute's value
    int device = 0;
    cudaError_t e = cudaGetDevice(&device);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    size_t &now = raised[{kernel, device}];
    if (now >= bytes) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) now = bytes;
    return e;
}

bool sharding_active(int n_units) { return !g_extra.empty() && n_units >= 2 && t_ctx == &g_primary; }

}  // namespace vgb

using namespace vgb;

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
    // containers.cu keeps its own slabs and streams per context: those go first, while the context's device is bound
    vgb::containers_release(g_primary);
    for (auto &c : g_extra) vgb::containers_release(*c);
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
int32_t abi_ensure_ready()  // the primary's context on a caller thread, a worker's own in a sharded converter call
{
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    return ensure_ready_locked();
}
void abi_count_launches(int n) { g_ctx.launches += n; }
}  // namespace vgb

extern "C" {

/* Bind several devices (SURVEY §8b: vgb_init(n_devices, flags)).  devices[0] becomes the primary device - the one the
 * *_dev entry points, the timers and the debug taps refer to; every host-pointer codec *_batch call and both batch
 * converters are then sharded over all of them (greedy longest-first over the units' sample counts, one worker thread and
 * one H2D / kernel / D2H pipeline per device, results written straight into the caller's arrays).  The single-shot
 * container calls (vgb_*_read_batch, vgb_*_write_batch, vgb_*_crypt_batch) stay on the primary.  A device may be listed
 * more than once (two pipelines on one GPU; also how the sharding logic is tested on a single-GPU machine). */
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
