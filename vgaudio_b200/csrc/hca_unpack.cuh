// hca_unpack.cuh — CriHcaPacking.UnpackFrame (Codecs/CriHca/CriHcaPacking.cs:10-229) for one frame on one thread: the
// walk behind the decoder's parse (hca_decode_parse_kernel, hca.cu) and the key search's frame test (hca_keys.cu).
#pragma once

#include "common.cuh"

namespace vgb {

constexpr int kHcaSubframes = 8, kHcaBands = 128;

// The per-band code descriptors and curves the walk reads, staged in shared memory by the calling kernel
struct HcaUnpackSmem {
    const unsigned long long *lens64, *vals64;  // [8]: QuantizedSpectrumBits / Value of resolutions 0..7, 4 bits per code
    const uint8_t *maxbits;                     // [16] QuantizedSpectrumMaxBits
    const uint8_t *curve;                       // [59] ScaleToResolutionCurve
    const uint8_t *ath;                         // [128] the frame's AthCurve
};

// What a walk reports besides its status: the bit position it reached (BitReader.Position) and what
// UnpackingWasSuccessful / FrameEmpty (:207-229) read
struct HcaUnpackEnd {
    int position, noise_level;
    bool delta_any;  // some channel's ScaleFactorDeltaBits > 0
};

// A sink that records nothing (the key search keeps only the walk's end)
struct HcaNoRecord {
    __device__ void band(int, int, int, int) const {}
    __device__ void clear_side(int) const {}
    __device__ void intensity(int, int, int) const {}
    __device__ void hfr(int, int, int) const {}
    __device__ void quant(int, int, int, int) const {}
    __device__ void quant_tail(int, int, int) const {}
    __device__ void fail() const {}
};

// UnpackFrameHeader + ReadSpectralCoefficients over the bytes word(i) gives (word i = bytes 4i..4i+3, big-endian; bytes
// past the frame must read as zero, as BitReader.PeekInt reads bits past the end).  The resolutions go to sres_lane
// [(c * 128 + b) * kStride] (the caller's shared memory, threads fastest), the fields to the sink `rec`.
//
// kKeyTest false (the decoder): a bad sync word, a scale-factor delta out of range or an intensity index 15 ends the
// frame with VGB_HCA_BAD_SYNC / BAD_DELTA / BAD_INDEX and rec.fail().  kKeyTest true (TestKey, CriHcaEncryption.cs:48-63):
// intensity 15 is read like any other value (the reference only fails on it later, in ApplyIntensityStereo), a bad delta
// ends the frame at once, and `end` gets the bit position reached.
template <bool kKeyTest, int kStride, class Word, class Rec>
__device__ __forceinline__ int hca_unpack_walk(Word word, const HcaConfig &cfg, const HcaUnpackSmem &S, uint8_t *sres_lane,
                                               const Rec &rec, HcaUnpackEnd *end)
{
    const int nch = cfg.channel_count;
    // BitReader.ReadInt / PeekInt (Utilities/BitReader.cs:51-99): a 64-bit window keeps the next bits left-aligned, so a
    // read is a shift; a refill happens once per 32 consumed bits from a word fetched at the previous refill
    uint64_t win = ((uint64_t)word(0) << 32) | word(1);
    int avail = 64, next = 2;
    uint32_t ahead = word(2);
    auto peek = [&](int count) -> uint32_t { return (uint32_t)((win >> 1) >> (63 - count)); };
    auto skip = [&](int count) {
        win <<= count;
        avail -= count;
        if (avail <= 32) {
            win |= (uint64_t)ahead << (32 - avail);
            avail += 32;
            ahead = word(++next);
        }
    };
    auto read = [&](int count) -> int { const uint32_t v = peek(count); skip(count); return (int)v; };

    int status = 0;
    bool delta_any = false;
    if (read(16) != 0xffff) {
        status = VGB_HCA_BAD_SYNC;
        if (kKeyTest) return status;
    }
    const int noise_level = read(9);
    const int eval_boundary = read(7);
    for (int c = 0; c < nch && !status; c++) {
        const int type = cfg.channel_type[c];
        const int coded = type == 2 ? cfg.base_band_count : cfg.base_band_count + cfg.stereo_band_count;
        const int delta_bits = read(3);  // ReadScaleFactors (:108-126)
        if (kKeyTest) delta_any |= delta_bits != 0;
        // DeltaDecode reads output[0] before its loop, so a channel without coded bands still consumes 6 bits (:183-186)
        if (coded == 0 && delta_bits != 0 && delta_bits < 6) skip(6);
        int prev = 0;
        for (int b = 0; b < kHcaBands; b++) {
            int sf = 0;
            if (b < coded && delta_bits != 0) {
                if (delta_bits >= 6 || b == 0) {
                    sf = read(6);
                } else {  // DeltaDecode (:183-208)
                    const int max_delta = 1 << (delta_bits - 1);
                    const int delta = read(delta_bits) - (max_delta - 1);  // ReadOffsetBinary, OffsetBias.Positive
                    if (delta < max_delta) {
                        sf = prev + delta;
                        if (sf < 0 || sf > 63) {
                            if (kKeyTest) return VGB_HCA_BAD_DELTA;
                            status = VGB_HCA_BAD_DELTA;
                            sf = 0;
                        }
                    } else {
                        sf = read(6);
                    }
                }
            }
            prev = sf;
            int res = 0;
            if (b < coded && sf != 0) {  // CalculateResolution (CriHcaPacking.cs:60-69) of athCurve[b] + noise (:86-94)
                int pos = S.ath[b] + (b < eval_boundary ? noise_level - 1 : noise_level) - 5 * sf / 2 + 2;
                pos = min(max(pos, 0), 58);
                res = S.curve[pos];
            }
            rec.band(c, b, sf, res);
            sres_lane[((size_t)c * kHcaBands + b) * kStride] = (uint8_t)res;
        }
        if (status) break;
        rec.clear_side(c);
        if (type == 2) {
            for (int i = 0; i < kHcaSubframes; i++) {
                int v = read(4);
                if (!kKeyTest && v > 14) { status = VGB_HCA_BAD_INDEX; v = 14; }
                rec.intensity(c, i, v);
            }
        } else if (cfg.hfr_group_count > 0) {
            for (int i = 0; i < cfg.hfr_group_count; i++) rec.hfr(c, i, read(6));
        }
    }
    if (!status) {
        for (int sf = 0; sf < kHcaSubframes; sf++)  // ReadSpectralCoefficients (:144-181)
            for (int c = 0; c < nch; c++) {
                const int type = cfg.channel_type[c];
                const int coded = type == 2 ? cfg.base_band_count : cfg.base_band_count + cfg.stereo_band_count;
                const uint8_t *rb = sres_lane + (size_t)c * kHcaBands * kStride;
                int res = coded > 0 ? rb[0] : 0;
                for (int b = 0; b < coded; b++) {
                    const int res_next = b + 1 < coded ? rb[(size_t)(b + 1) * kStride] : 0;
                    const int mbits = S.maxbits[res];
                    const unsigned long long lens = S.lens64[res], vals = S.vals64[res];
                    const int code = (int)peek(mbits);
                    // both code families, selected without a branch (lanes parse different frames)
                    const int bits_p = (int)((lens >> (4 * code)) & 15u);
                    const int v_p = (int)((unsigned)(vals >> (4 * code)) << 28) >> 28;
                    const int mag = code >> 1;
                    const int v_s = (code & 1) ? -mag : mag;
                    const int bits_s = mbits - (mag == 0 ? 1 : 0);
                    const bool prefix = mbits <= 4;
                    rec.quant(c, sf, b, prefix ? v_p : v_s);
                    skip(prefix ? bits_p : bits_s);
                    res = res_next;
                }
                rec.quant_tail(c, sf, coded);
            }
        if (kKeyTest) {
            end->position = 32 * next - avail;
            end->noise_level = noise_level;
            end->delta_any = delta_any;
        }
    } else {
        rec.fail();
    }
    return status;
}

}  // namespace vgb
