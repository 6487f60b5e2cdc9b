// hca_keys.cu — the key search of HcaReader.FindKey for type-56 .hca files on sm_90a (H100).
//
// CriHcaEncryption.FindKey (Codecs/CriHca/CriHcaEncryption.cs:34-87) tries the keys in list order and keeps the first one
// TestKey accepts: from the first frame whose bytes [2, FrameSize - 2) are not all zero (on the encrypted frames), up to
// ten frames are decrypted with the key (CryptFrame: substitution of bytes [0, FrameSize - 2), then the CRC-16 of those
// bytes into the last two), and each must pass CriHcaPacking.UnpackFrame, whose last test is UnpackingWasSuccessful
// (CriHcaPacking.cs:207-229) on the bits left over.
//
// One CTA per file, one lane per key: the lanes of a CTA read the same encrypted window (the same byte at the same time
// while they are in step, so the loads broadcast) through their own key's table in shared memory, stored byte value
// major ([256][kLanes]) so that lanes reading one byte value hit 64 consecutive bytes.  A lane walks keys tid, tid +
// kLanes, ...  The walk is hca_unpack_walk, the decoder's parse, with a byte source that decrypts on the fly; the CRC of
// the decrypted bytes is computed only when the walk's reader reaches the frame's last two bytes, which a key that fails
// early never does.
//
// First-index search: a key is decisive when its walk passes every window frame or stops at a bad sync word (the sync
// word decrypts to 0xFFFF under every type-56 table exactly when the raw one is 0xFFFF, so that frame throws out of
// FindKey for the first key that passes the frames before it).  The file's result is the decisive key of lowest index.
// A lane stops at its first decisive key and atomicMin's its index into the CTA's word; a lane whose key index is above
// that word drops the key (also between frames).  Every lane's keys ascend, so the lane that found the lowest index
// holds its outcome.  The debug mode walks every key and writes every outcome.
#include <algorithm>

#include "common.cuh"
#include "hca_unpack.cuh"
#include "kernels.h"

namespace vgb {

namespace {

#include "hca_tables.inc"

constexpr int kLanes = 64;  // keys walked at once per file

struct HcaKeyParams {
    HcaKeySearch a;
    unsigned long long lens64[8], vals64[8];
    uint8_t maxbits[16], curve[64];
    uint16_t crc[256];  // Crc16 table, polynomial 0x8005 (Utilities/Crc16.cs)
};

// Crc16.Compute of the lane's decrypted bytes [0, fs - 2): CryptFrame's checksum (CriHcaEncryption.cs:29-31)
__device__ __noinline__ uint32_t hca_key_crc(const uint8_t *raw, int fs, const uint8_t *tab_lane, const uint16_t *crc_tab)
{
    uint32_t c = 0;
    for (int i = 0; i < fs - 2; i++) c = ((c << 8) ^ crc_tab[((c >> 8) ^ tab_lane[(int)__ldg(raw + i) * kLanes]) & 0xff]) & 0xffffu;
    return c;
}

__global__ void __launch_bounds__(kLanes) hca_key_search_kernel(const __grid_constant__ HcaKeyParams P)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ unsigned long long s_lens64[8], s_vals64[8], s_pairs, s_frames;
    __shared__ uint8_t s_maxbits[16], s_curve[64];
    __shared__ uint16_t s_crc[256];
    __shared__ HcaConfig s_cfg;
    __shared__ int s_decided;
    const HcaKeySearch &a = P.a;
    const int tid = threadIdx.x, f = blockIdx.x;
    uint8_t *tab_lane = smem_raw + tid;                      // [256][kLanes]: the lane's key's decryption table
    uint8_t *sres_lane = smem_raw + 256 * kLanes + tid;      // [channels][128][kLanes]: its frame's resolutions
    if (tid < 8) { s_lens64[tid] = P.lens64[tid]; s_vals64[tid] = P.vals64[tid]; }
    if (tid < 16) s_maxbits[tid] = P.maxbits[tid];
    s_curve[tid] = P.curve[tid];
    for (int i = tid; i < 256; i += kLanes) s_crc[i] = P.crc[i];
    const HcaKeyFileDev &fd = a.files[f];
    for (int i = tid; i < (int)(sizeof(HcaConfig) / 4); i += kLanes) reinterpret_cast<int32_t *>(&s_cfg)[i] = reinterpret_cast<const int32_t *>(&fd.cfg)[i];
    if (tid == 0) { s_decided = a.n_keys; s_pairs = 0; s_frames = 0; }
    const int64_t frames_off = fd.frames_off;
    const int window = fd.window;
    __syncthreads();

    const int fs = s_cfg.frame_size;
    const HcaUnpackSmem S{s_lens64, s_vals64, s_maxbits, s_curve, s_cfg.ath};
    volatile int *decided = &s_decided;
    unsigned long long pairs = 0, frames = 0;
    int mine = -1, mine_outcome = 0;  // this lane's decisive key and its outcome
    for (int k = tid; k < a.n_keys; k += kLanes) {
        if (!a.every && k > *decided) break;
        const uint4 *t = reinterpret_cast<const uint4 *>(a.tables + (size_t)k * 256);
        for (int q = 0; q < 16; q++) {
            const uint4 v = __ldg(t + q);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int i = 0; i < 16; i++) tab_lane[(16 * q + i) * kLanes] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
        }
        pairs++;
        int outcome = 0;
        bool dropped = false;
        for (int j = 0; j < window && !outcome; j++) {
            if (!a.every && k > *decided) { dropped = true; break; }
            const uint8_t *raw = a.frames + frames_off + (int64_t)j * fs;
            int crc = -1;
            // CryptFrame's output, bytes past the frame read as zero (BitReader.PeekInt)
            auto word = [&](int i) -> uint32_t {
                uint32_t v = 0;
#pragma unroll
                for (int b4 = 0; b4 < 4; b4++) {
                    const int b = 4 * i + b4;
                    uint32_t x = 0;
                    if (b < fs - 2) {
                        x = tab_lane[(int)__ldg(raw + b) * kLanes];
                    } else if (b < fs) {
                        if (crc < 0) crc = (int)hca_key_crc(raw, fs, tab_lane, s_crc);
                        x = b == fs - 2 ? (uint32_t)crc >> 8 : (uint32_t)crc & 0xffu;
                    }
                    v |= x << (24 - 8 * b4);
                }
                return v;
            };
            HcaUnpackEnd end{};
            const int st = hca_unpack_walk<true, kLanes>(word, s_cfg, S, sres_lane, HcaNoRecord{}, &end);
            frames++;
            if (st == VGB_HCA_BAD_SYNC) {
                outcome = 1 + 3 * j;
            } else if (st == VGB_HCA_BAD_DELTA) {
                outcome = 1 + 3 * j + 1;
            } else {  // UnpackingWasSuccessful (CriHcaPacking.cs:207-229), Remaining = LengthBits - Position
                const int remaining = fs * 8 - end.position;
                const bool empty = end.noise_level == 0 && !end.delta_any;  // FrameEmpty (:216-229)
                if (!((remaining >= 16 && remaining <= 128) || empty || (end.noise_level == 0 && remaining >= 16))) outcome = 1 + 3 * j + 2;
            }
        }
        if (dropped) break;
        if (a.every) {
            a.outcomes[(int64_t)f * a.n_keys + k] = outcome;
        } else if (outcome == 0 || (outcome - 1) % 3 == 0) {
            mine = k;
            mine_outcome = outcome;
            atomicMin(&s_decided, k);
            break;
        }
    }
    atomicAdd(&s_pairs, pairs);
    atomicAdd(&s_frames, frames);
    __syncthreads();
    if (!a.every && mine >= 0 && mine == s_decided) {
        a.first[2 * f] = mine;
        a.first[2 * f + 1] = mine_outcome;
    }
    if (!a.every && tid == 0 && s_decided == a.n_keys) {
        a.first[2 * f] = -1;
        a.first[2 * f + 1] = -1;
    }
    if (tid == 0) {
        atomicAdd(a.stats, s_pairs);
        atomicAdd(a.stats + 1, s_frames);
    }
}

}  // namespace

cudaError_t launch_hca_key_search(const HcaKeySearch &a, cudaStream_t stream)
{
    if (a.n_files <= 0) return cudaSuccess;
    HcaKeyParams P{};
    P.a = a;
    for (int r = 0; r < 8; r++)
        for (int code = 0; code < 16; code++) {
            P.lens64[r] |= (unsigned long long)(kHcaQuantizedSpectrumBits[r][code] & 15u) << (4 * code);
            P.vals64[r] |= (unsigned long long)((unsigned)kHcaQuantizedSpectrumValue[r][code] & 15u) << (4 * code);
        }
    std::copy(kHcaQuantizedSpectrumMaxBits, kHcaQuantizedSpectrumMaxBits + 16, P.maxbits);
    std::copy(kHcaScaleToResolutionCurve, kHcaScaleToResolutionCurve + 59, P.curve);
    for (int i = 0; i < 256; i++) {
        uint16_t v = (uint16_t)(i << 8);
        for (int k = 0; k < 8; k++) v = (uint16_t)((v & 0x8000) ? (v << 1) ^ 0x8005 : v << 1);
        P.crc[i] = v;
    }
    const size_t smem = 256 * kLanes + (size_t)std::max(a.max_channels, 1) * kHcaBands * kLanes;
    cudaError_t e = raise_dynamic_smem(hca_key_search_kernel, smem);
    if (e != cudaSuccess) return e;
    hca_key_search_kernel<<<(unsigned)a.n_files, kLanes, smem, stream>>>(P);
    return cudaGetLastError();
}

}  // namespace vgb
