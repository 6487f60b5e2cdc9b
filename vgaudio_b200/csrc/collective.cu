// collective.cu — the one exchange step of the multi-GPU batch path: scatterv of PCM / gatherv of bitstreams between
// the ranks of a job, for data that is already resident in HBM (SURVEY §8e; the reference's counterpart is the file-level
// Parallel.ForEach of src/VGAudio.Cli/Batch.cs:24-25, which has no exchange at all because everything lives in one
// address space).  Variable sizes per rank, so both are grouped ncclSend / ncclRecv pairs - no padding to the longest
// shard, no host round trip; over NVLink 5 / NVSwitch every rank reaches the root at full link bandwidth.
//
// NCCL is bound at run time (dlopen "libnccl.so.2", preferring a copy the process has already loaded, e.g. the one
// PyTorch ships), so libvgaudio_b200.so has no link-time dependency on it and single-GPU users never touch it.  Every
// failure is VGB_E_NCCL with ncclGetErrorString / ncclGetLastError in vgb_last_error().
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "abi.cuh"

using vgb::fail;

namespace {

struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    const char *(*GetLastError)(ncclComm_t) = nullptr;
    ncclResult_t (*GetVersion)(int *) = nullptr;
};

std::mutex g_mu;
NcclApi g_api;
ncclComm_t g_comm = nullptr;
int g_ranks = 0, g_rank = -1;

int32_t load_api()
{
    if (g_api.handle) return VGB_OK;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);  // the copy this process already uses
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return fail(VGB_E_NCCL, "libnccl.so.2 not found (%s)", dlerror());
    NcclApi a;
    a.handle = h;
#define BIND(field, sym)                                                        \
    a.field = reinterpret_cast<decltype(a.field)>(dlsym(h, sym));              \
    if (!a.field) return fail(VGB_E_NCCL, "libnccl.so.2 lacks %s", sym);
    BIND(GetUniqueId, "ncclGetUniqueId")
    BIND(CommInitRank, "ncclCommInitRank")
    BIND(CommDestroy, "ncclCommDestroy")
    BIND(GroupStart, "ncclGroupStart")
    BIND(GroupEnd, "ncclGroupEnd")
    BIND(Send, "ncclSend")
    BIND(Recv, "ncclRecv")
    BIND(GetErrorString, "ncclGetErrorString")
    BIND(GetVersion, "ncclGetVersion")
#undef BIND
    a.GetLastError = reinterpret_cast<decltype(a.GetLastError)>(dlsym(h, "ncclGetLastError"));  // optional (>= 2.13)
    g_api = a;
    return VGB_OK;
}

int32_t nccl_fail(const char *what, ncclResult_t r)
{
    const char *last = (g_api.GetLastError && g_comm) ? g_api.GetLastError(g_comm) : "";
    return fail(VGB_E_NCCL, "%s failed: %s%s%s", what, g_api.GetErrorString ? g_api.GetErrorString(r) : "?", last && *last ? " - " : "",
                    last ? last : "");
}

#define NCCL_TRY(call)                                        \
    do {                                                      \
        ncclResult_t r_ = (call);                             \
        if (r_ != ncclSuccess) return nccl_fail(#call, r_);   \
    } while (0)

}  // namespace

extern "C" {

int32_t vgb_nccl_unique_id(uint8_t *id_out)
{
    if (!id_out) return fail(VGB_E_ARG, "id_out is NULL");
    std::lock_guard<std::mutex> lock(g_mu);
    if (int32_t rc = load_api()) return rc;
    static_assert(sizeof(ncclUniqueId) == VGB_NCCL_ID_BYTES, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    NCCL_TRY(g_api.GetUniqueId(&id));
    memcpy(id_out, &id, sizeof id);
    return VGB_OK;
}

int32_t vgb_nccl_init(const uint8_t *id, int32_t n_ranks, int32_t rank)
{
    if (!id || n_ranks < 1 || rank < 0 || rank >= n_ranks) return fail(VGB_E_ARG, "bad communicator arguments");
    std::lock_guard<std::mutex> lock(g_mu);
    if (g_comm) return fail(VGB_E_STATE, "a communicator already exists; call vgb_nccl_shutdown first");
    if (int32_t rc = load_api()) return rc;
    // The batch path's exchange is a one-to-many scatter / many-to-one gather of large blocks: the root's NVLink port is the
    // limit, and NCCL's default point-to-point channel count leaves most of it idle (32 channels per peer nearly halved
    // the exchange of a 4-GPU C5 run).  Only set when the user has not chosen a value.
    setenv("NCCL_MIN_P2P_NCHANNELS", "32", 0);
    setenv("NCCL_MAX_P2P_NCHANNELS", "32", 0);
    ncclUniqueId uid;
    memcpy(&uid, id, sizeof uid);
    NCCL_TRY(g_api.CommInitRank(&g_comm, n_ranks, uid, rank));  // on the calling thread's current device
    g_ranks = n_ranks;
    g_rank = rank;
    return VGB_OK;
}

int32_t vgb_nccl_shutdown(void)
{
    std::lock_guard<std::mutex> lock(g_mu);
    if (g_comm) g_api.CommDestroy(g_comm);
    g_comm = nullptr;
    g_ranks = 0;
    g_rank = -1;
    return VGB_OK;
}

int32_t vgb_nccl_version(void)
{
    std::lock_guard<std::mutex> lock(g_mu);
    if (load_api() != VGB_OK) return 0;
    int v = 0;
    return g_api.GetVersion(&v) == ncclSuccess ? v : 0;
}

int32_t vgb_scatterv_dev(const void *d_send, const int64_t *send_offset, const int64_t *counts, void *d_recv, int32_t root,
                         void *cuda_stream)
{
    std::lock_guard<std::mutex> lock(g_mu);
    if (!g_comm) return fail(VGB_E_STATE, "no communicator: call vgb_nccl_init on every rank first");
    if (!counts || root < 0 || root >= g_ranks) return fail(VGB_E_ARG, "bad arguments");
    if (g_rank == root && (!d_send || !send_offset)) return fail(VGB_E_ARG, "the root needs d_send and send_offset");
    for (int r = 0; r < g_ranks; r++)
        if (counts[r] < 0 || (g_rank == root && send_offset[r] < 0)) return fail(VGB_E_ARG, "rank %d: negative count / offset", r);
    if (counts[g_rank] > 0 && !d_recv) return fail(VGB_E_ARG, "d_recv is NULL");
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    NCCL_TRY(g_api.GroupStart());
    if (g_rank == root) {
        const char *src = static_cast<const char *>(d_send);
        for (int r = 0; r < g_ranks; r++) {
            if (counts[r] == 0) continue;
            if (r == root) {  // own share: a device copy on the same stream (skipped when it is already in place)
                if (src + send_offset[r] != d_recv &&
                    cudaMemcpyAsync(d_recv, src + send_offset[r], (size_t)counts[r], cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
                    g_api.GroupEnd();
                    return fail(VGB_E_CUDA, "device copy of the root's own share failed: %s", cudaGetErrorString(cudaGetLastError()));
                }
            } else {
                NCCL_TRY(g_api.Send(src + send_offset[r], (size_t)counts[r], ncclInt8, r, g_comm, st));
            }
        }
    } else if (counts[g_rank] > 0) {
        NCCL_TRY(g_api.Recv(d_recv, (size_t)counts[g_rank], ncclInt8, root, g_comm, st));
    }
    NCCL_TRY(g_api.GroupEnd());
    return VGB_OK;
}

int32_t vgb_gatherv_dev(const void *d_send, void *d_recv, const int64_t *recv_offset, const int64_t *counts, int32_t root,
                        void *cuda_stream)
{
    std::lock_guard<std::mutex> lock(g_mu);
    if (!g_comm) return fail(VGB_E_STATE, "no communicator: call vgb_nccl_init on every rank first");
    if (!counts || root < 0 || root >= g_ranks) return fail(VGB_E_ARG, "bad arguments");
    if (g_rank == root && (!d_recv || !recv_offset)) return fail(VGB_E_ARG, "the root needs d_recv and recv_offset");
    for (int r = 0; r < g_ranks; r++)
        if (counts[r] < 0 || (g_rank == root && recv_offset[r] < 0)) return fail(VGB_E_ARG, "rank %d: negative count / offset", r);
    if (counts[g_rank] > 0 && !d_send) return fail(VGB_E_ARG, "d_send is NULL");
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    NCCL_TRY(g_api.GroupStart());
    if (g_rank == root) {
        char *dst = static_cast<char *>(d_recv);
        for (int r = 0; r < g_ranks; r++) {
            if (counts[r] == 0) continue;
            if (r == root) {
                if (dst + recv_offset[r] != d_send &&
                    cudaMemcpyAsync(dst + recv_offset[r], d_send, (size_t)counts[r], cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
                    g_api.GroupEnd();
                    return fail(VGB_E_CUDA, "device copy of the root's own share failed: %s", cudaGetErrorString(cudaGetLastError()));
                }
            } else {
                NCCL_TRY(g_api.Recv(dst + recv_offset[r], (size_t)counts[r], ncclInt8, r, g_comm, st));
            }
        }
    } else if (counts[g_rank] > 0) {
        NCCL_TRY(g_api.Send(d_send, (size_t)counts[g_rank], ncclInt8, root, g_comm, st));
    }
    NCCL_TRY(g_api.GroupEnd());
    return VGB_OK;
}

int32_t vgb_sendrecv_dev(const void *const *send_ptr, const int64_t *send_bytes, const int32_t *send_peer, int32_t n_send,
                         void *const *recv_ptr, const int64_t *recv_bytes, const int32_t *recv_peer, int32_t n_recv, void *cuda_stream)
{
    std::lock_guard<std::mutex> lock(g_mu);
    if (!g_comm) return fail(VGB_E_STATE, "no communicator: call vgb_nccl_init on every rank first");
    if (n_send < 0 || n_recv < 0 || (n_send > 0 && (!send_ptr || !send_bytes || !send_peer)) || (n_recv > 0 && (!recv_ptr || !recv_bytes || !recv_peer)))
        return fail(VGB_E_ARG, "bad arguments");
    for (int i = 0; i < n_send; i++)
        if (send_bytes[i] < 0 || send_peer[i] < 0 || send_peer[i] >= g_ranks || send_peer[i] == g_rank || (send_bytes[i] > 0 && !send_ptr[i]))
            return fail(VGB_E_ARG, "send %d: bad peer / size / pointer", i);
    for (int i = 0; i < n_recv; i++)
        if (recv_bytes[i] < 0 || recv_peer[i] < 0 || recv_peer[i] >= g_ranks || recv_peer[i] == g_rank || (recv_bytes[i] > 0 && !recv_ptr[i]))
            return fail(VGB_E_ARG, "recv %d: bad peer / size / pointer", i);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    NCCL_TRY(g_api.GroupStart());
    for (int i = 0; i < n_send; i++)
        if (send_bytes[i] > 0) NCCL_TRY(g_api.Send(send_ptr[i], (size_t)send_bytes[i], ncclInt8, send_peer[i], g_comm, st));
    for (int i = 0; i < n_recv; i++)
        if (recv_bytes[i] > 0) NCCL_TRY(g_api.Recv(recv_ptr[i], (size_t)recv_bytes[i], ncclInt8, recv_peer[i], g_comm, st));
    NCCL_TRY(g_api.GroupEnd());
    return VGB_OK;
}

int32_t vgb_partition_lpt(const int64_t *weight, int32_t n_units, int32_t n_parts, int32_t *part_out, int64_t *load_out)
{
    if (n_units < 0 || n_parts < 1 || (n_units > 0 && (!weight || !part_out))) return fail(VGB_E_ARG, "bad arguments");
    std::vector<int32_t> order(n_units);
    for (int i = 0; i < n_units; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return weight[a] > weight[b]; });
    std::vector<int64_t> load(n_parts, 0);
    for (int u : order) {
        int best = 0;
        for (int p = 1; p < n_parts; p++) if (load[p] < load[best]) best = p;
        part_out[u] = best;
        load[best] += weight[u] > 0 ? weight[u] : 0;
    }
    if (load_out) for (int p = 0; p < n_parts; p++) load_out[p] = load[p];
    return VGB_OK;
}

}  // extern "C"
