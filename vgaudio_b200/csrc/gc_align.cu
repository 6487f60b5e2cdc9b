// gc_align.cu — the tail of GcAdpcmAlignment (Formats/GcAdpcm/GcAdpcmAlignment.cs:44-55) on sm_90a (H100).
//
// The re-encoded part of an aligned loop is built from the channel's first decode only: the old samples on
// [samplesToKeep, loopEnd), then copies of [loopStart, loopStart + loopLength) until samplesToEncode samples are filled
// (:44-51).  Sample i of the tail is therefore old[keep + i] below loop_end and old[loop_start + (keep + i - loop_end) %
// loop_length] above it: pure index arithmetic over the decoded slab, one CTA per channel, 16-byte stores of 8 samples.
// The encoder's history pair (:53-55) goes to `hist_enc` and `hist_dec` alike: the encoder and the decoder of the tail
// both overwrite their table's pair at the end of a slice, so each keeps its own copy.
#include "common.cuh"
#include "kernels.h"

namespace vgb {

constexpr int kAlignThreads = 256;

__global__ void __launch_bounds__(kAlignThreads)
gc_align_tail_kernel(const int16_t *__restrict__ pcm, const GcAlignChannel *__restrict__ chans, int16_t *__restrict__ tail,
                     int16_t *__restrict__ hist_enc, int16_t *__restrict__ hist_dec)
{
    const GcAlignChannel a = chans[blockIdx.x];
    const int16_t *old = pcm + a.src_off;
    if (threadIdx.x == 0) {
        const int16_t h1 = a.keep < 1 ? 0 : old[a.keep - 1], h2 = a.keep < 2 ? 0 : old[a.keep - 2];
        hist_enc[2 * blockIdx.x] = h1;
        hist_enc[2 * blockIdx.x + 1] = h2;
        hist_dec[2 * blockIdx.x] = h1;
        hist_dec[2 * blockIdx.x + 1] = h2;
    }
    // loop_length > 0 whenever the tail runs past loop_end (the host rejects an empty loop that would have to repeat)
    const int32_t loop_length = a.loop_end - a.loop_start;
    uint4 *row = reinterpret_cast<uint4 *>(tail + a.dst_off);
    const int vectors = (a.count + 7) / 8;  // the row is padded to a multiple of 8 samples; the padding is zero
    for (int v = threadIdx.x; v < vectors; v += kAlignThreads) {
        uint32_t w[4];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int i = v * 8 + k;
            const int32_t j = a.keep + i;  // position in the aligned channel
            uint32_t s = 0;
            if (i < a.count) s = (uint16_t)old[j < a.loop_end ? j : a.loop_start + (j - a.loop_end) % loop_length];
            if (k & 1) w[k / 2] |= s << 16; else w[k / 2] = s;
        }
        row[v] = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

void launch_gc_align_tail(const int16_t *pcm, const GcAlignChannel *chans, int n_channels, int16_t *tail, int16_t *hist_enc,
                          int16_t *hist_dec, cudaStream_t stream)
{
    if (n_channels <= 0) return;
    gc_align_tail_kernel<<<n_channels, kAlignThreads, 0, stream>>>(pcm, chans, tail, hist_enc, hist_dec);
}

}  // namespace vgb
