// abi_hca.cu — the CRI HCA entry points of the C ABI: header maths (CriHcaEncoder.Initialize), the codec table store,
// host-pointer batch calls (pipelined over stream groups, sharded over the bound devices), device-resident encode and
// the MDCT taps.
#include <cmath>

#include "abi.cuh"

using namespace vgb;

#define g_hca_tables (g_ctx.hca_tables)

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

// Initialize of every stream of an encode call; the streams must share the codec configuration
int32_t hca_encode_infos(const vgb_hca_params *params, int32_t n_streams, std::vector<vgb_hca_info> &infos,
                         std::vector<HcaVirtual> &virt)
{
    infos.resize(n_streams);
    virt.resize(n_streams);
    for (int s = 0; s < n_streams; s++) {
        VGB_TRY(hca_initialize(params[s], infos[s], &virt[s]));
        const vgb_hca_params &a = params[0], &b = params[s];
        if (a.channel_count != b.channel_count || a.sample_rate != b.sample_rate || a.quality != b.quality ||
            a.bitrate != b.bitrate || a.limit_bitrate != b.limit_bitrate)
            return fail(VGB_E_ARG, "stream %d: all streams of one call must share channel count, sample rate, quality and bitrate", s);
    }
    return VGB_OK;
}

// The encoder's row of one stream: its place in the PCM and frame slabs and its virtual input stream
HcaStream hca_encode_stream(const vgb_hca_info &h, const HcaVirtual &v, int64_t pcm_off, int64_t channel_stride, int64_t frames_off)
{
    HcaStream t{};
    t.pcm_off = pcm_off;
    t.channel_stride = channel_stride;
    t.frames_off = frames_off;
    t.sample_count = h.sample_count;
    t.frame_count = h.frame_count;
    t.pre_zero = v.pre_zero;
    t.pre_fill = v.pre_fill;
    t.post_count = v.post_count;
    t.loop_start = v.loop_start;
    t.src_count = v.src_count;
    t.last_chunk = v.last_chunk;
    return t;
}

}  // namespace

// The codec configuration of a call, from the HcaInfo its streams share
HcaConfig vgb::hca_config(const vgb_hca_info &h0)
{
    HcaConfig cfg{};
    cfg.channel_count = h0.channel_count;
    cfg.frame_size = h0.frame_size;
    cfg.base_band_count = h0.base_band_count;
    cfg.stereo_band_count = h0.stereo_band_count;
    cfg.total_band_count = h0.total_band_count;
    cfg.hfr_band_count = h0.hfr_band_count;
    cfg.bands_per_hfr_group = h0.bands_per_hfr_group;
    cfg.hfr_group_count = h0.hfr_group_count;
    hca_channel_types(h0, cfg.channel_type);
    hca_fill_ath(h0, cfg.ath);
    return cfg;
}

int32_t vgb::hca_encode_fault(int32_t status, const char *what, int index)
{
    if (status == VGB_HCA_BITRATE_TOO_LOW) return fail(VGB_E_DATA, "%s %d: Bitrate is set too low.", what, index);
    if (status == VGB_HCA_NOT_IMPLEMENTED) return fail(VGB_E_STATE, "%s %d: evaluation boundary search failed (NotImplementedException in the reference)", what, index);
    if (status == VGB_HCA_BIT_OVERFLOW) return fail(VGB_E_STATE, "%s %d: Not enough bits left in output buffer", what, index);
    return VGB_OK;
}

namespace {

// The encoder's per-stream status words as the reference's exceptions
int32_t hca_encode_status(const std::vector<int32_t> &status)
{
    for (int s = 0; s < (int)status.size(); s++) VGB_TRY(hca_encode_fault(status[s], "stream", s));
    return VGB_OK;
}

}  // namespace

int32_t vgb::hca_encode_words(const void *d_workspace, int32_t n_streams, int32_t *status, cudaStream_t st)
{
    const size_t o_status = align_up((size_t)n_streams * sizeof(HcaStream), 256);
    CUDA_TRY(cudaMemcpyAsync(status, static_cast<const char *>(d_workspace) + o_status, (size_t)n_streams * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return VGB_OK;
}


// One-time upload of the codec tables (per process/device).  Trig tables: Mdct.GenerateTrigTables (Mdct.cs:183-195)
// with the host libm, exactly as the oracle builds them; dead zones: CriHcaTables.QuantizerDeadZoneFunction (:68-78).
// (HcaTableStore is a member of the per-device Context: g_hca_tables is the current device's store)

void vgb::hca_tables_release_locked()
{
    if (g_hca_tables.blob) cudaFree(g_hca_tables.blob);
    g_hca_tables.blob = nullptr;
    g_hca_tables.ready = false;
}

namespace {

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

// Byte offsets in a decode workspace (vgb_hca_decode_dev): stream table, status words, seam addends (2 x 128 doubles
// per channel-frame), parse records
struct HcaDecodeLayout {
    size_t o_status, o_edge, o_parsed, bytes;
    HcaDecodeLayout(const HcaConfig &cfg, int n_streams, int64_t total_frames)
    {
        const size_t n = (size_t)std::max(n_streams, 1);
        o_status = align_up(n * sizeof(HcaStream), 256);
        o_edge = align_up(o_status + n * 4, 256);
        o_parsed = align_up(o_edge + (size_t)total_frames * cfg.channel_count * 2 * 128 * sizeof(double), 256);
        bytes = align_up(o_parsed + hca_decode_parsed_bytes(cfg, total_frames), 256);
    }
};

}  // namespace

bool vgb::hca_same_config(const vgb_hca_info &a, const vgb_hca_info &b)
{
    return a.channel_count == b.channel_count && a.frame_size == b.frame_size && a.base_band_count == b.base_band_count &&
           a.stereo_band_count == b.stereo_band_count && a.total_band_count == b.total_band_count && a.hfr_band_count == b.hfr_band_count &&
           a.bands_per_hfr_group == b.bands_per_hfr_group && a.hfr_group_count == b.hfr_group_count && a.track_count == b.track_count &&
           a.channel_config == b.channel_config && (a.use_ath_curve != 0) == (b.use_ath_curve != 0) &&
           (!a.use_ath_curve || a.sample_rate == b.sample_rate);
}

int32_t vgb::hca_decode_check(const vgb_hca_info *info, int32_t n_streams)
{
    const vgb_hca_info &h0 = info[0];
    if (h0.channel_count < 1 || h0.channel_count > 8) return fail(VGB_E_ARG, "channel_count must be 1..8");
    for (int s = 0; s < n_streams; s++) {
        const vgb_hca_info &b = info[s];
        if (!hca_same_config(h0, b)) {
            vgb_hca_info c = b;  // b with h0's ATH fields: differs only when the band layout or frame size does
            c.use_ath_curve = h0.use_ath_curve;
            c.sample_rate = h0.sample_rate;
            if (!hca_same_config(h0, c)) return fail(VGB_E_ARG, "stream %d: all streams of one call must share the band layout and frame size", s);
            return fail(VGB_E_ARG, "stream %d: all streams of one call must share UseAthCurve (and then the sample rate)", s);
        }
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
    return VGB_OK;
}

int32_t vgb::hca_decode_fault(int32_t status, const char *what, int index)
{
    if (status == VGB_HCA_BAD_SYNC) return fail(VGB_E_DATA, "%s %d: Invalid frame header", what, index);
    if (status == VGB_HCA_BAD_DELTA) return fail(VGB_E_DATA, "%s %d: scale factor delta out of range", what, index);
    if (status == VGB_HCA_BAD_INDEX) return fail(VGB_E_DATA, "%s %d: intensity index out of range", what, index);
    return VGB_OK;
}

int32_t vgb::hca_decode_words(const void *d_workspace, int32_t n_streams, int32_t *status, cudaStream_t st)
{
    const size_t o_status = align_up((size_t)std::max(n_streams, 1) * sizeof(HcaStream), 256);
    CUDA_TRY(cudaMemcpyAsync(status, static_cast<const char *>(d_workspace) + o_status, (size_t)n_streams * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return VGB_OK;
}

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
    std::vector<vgb_hca_info> infos;
    std::vector<HcaVirtual> virt;
    VGB_TRY(hca_encode_infos(params, n_streams, infos, virt));
    const vgb_hca_info &h0 = infos[0];
    const int nch = h0.channel_count;
    const HcaConfig cfg = hca_config(h0);

    std::vector<HcaStream> streams(n_streams);
    std::vector<int64_t> in_off((size_t)n_streams * nch), in_len((size_t)n_streams * nch), out_off(n_streams), out_len(n_streams);
    int64_t ps = 0, fb = 0, frames_total = 0;
    for (int s = 0; s < n_streams; s++) {
        const int32_t n_src = params[s].sample_count;  // the PCM the caller holds (>= Hca.SampleCount when looping)
        const int64_t stride = (int64_t)align_up((size_t)n_src, 8);
        streams[s] = hca_encode_stream(infos[s], virt[s], ps, stride, fb);
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
        return copy_units(cudaMemcpyHostToDevice, g_ctx.pcm.c(), in_off.data(), pcm, in_len.data(), bound[g] * nch,
                          (bound[g + 1] - bound[g]) * nch, g_ctx.s_in);
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
        return copy_units(cudaMemcpyDeviceToHost, g_ctx.adpcm.c(), out_off.data(), frames_out, out_len.data(), s0, n, g_ctx.s_out);
    };
    VGB_TRY(run_group_pipeline(n_groups, h2d, one_phase(kern), d2h, no_done));
    VGB_TRY(hca_encode_status(status));
    if (info_out) for (int s = 0; s < n_streams; s++) info_out[s] = infos[s];
    if (cb) cb(user, frames_total);
    return VGB_OK;
}

int32_t vgb_hca_encode_batch(const int16_t *const *pcm, const vgb_hca_params *params, int32_t n_streams,
                             vgb_hca_info *info_out, uint8_t *const *frames_out, vgb_progress_cb cb, void *user)
{
    if (!sharding_active(n_streams) || !pcm || !params || !frames_out)
        return hca_encode_one(pcm, params, n_streams, info_out, frames_out, cb, user);
    const int nch = params[0].channel_count;
    if (nch < 1 || nch > 8) return hca_encode_one(pcm, params, n_streams, info_out, frames_out, cb, user);
    SharedProgress prog{cb, user, {}};
    return run_sharded(shard_units(n_streams, [&](int s) { return params[s].sample_count; }, 1024), [&](int, const std::vector<int> &u) -> int32_t {
        const int m = (int)u.size();
        auto s_pcm = pick_rows(pcm, u, nch);
        auto s_par = pick_rows(params, u);
        auto s_out = pick_rows(frames_out, u);
        std::vector<vgb_hca_info> s_info(m);
        VGB_TRY(hca_encode_one(s_pcm.data(), s_par.data(), m, s_info.data(), s_out.data(), cb ? SharedProgress::relay : nullptr, &prog));
        if (info_out) put_rows(info_out, u, s_info);
        return VGB_OK;
    });
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
    VGB_TRY(check_aligned(d_pcm, 2, "d_pcm"));
    VGB_TRY(check_aligned(d_workspace, 8, "d_workspace"));  // HcaStream's int64 fields
    if (vgb_hca_workspace_bytes(n_streams) > workspace_bytes)
        return fail(VGB_E_ARG, "workspace too small: need %llu bytes", (unsigned long long)vgb_hca_workspace_bytes(n_streams));
    std::vector<vgb_hca_info> infos;
    std::vector<HcaVirtual> virt;
    VGB_TRY(hca_encode_infos(params, n_streams, infos, virt));
    const HcaConfig cfg = hca_config(infos[0]);
    std::vector<HcaStream> streams(n_streams);
    int max_frames = 0;
    for (int s = 0; s < n_streams; s++) {
        if (pcm_offset[s] < 0 || channel_stride[s] < params[s].sample_count || frames_offset[s] < 0)
            return fail(VGB_E_ARG, "stream %d: bad offsets (channel_stride must cover sample_count)", s);
        streams[s] = hca_encode_stream(infos[s], virt[s], pcm_offset[s], channel_stride[s], frames_offset[s]);
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
    VGB_TRY(hca_encode_words(d_workspace, n_streams, status.data(), static_cast<cudaStream_t>(cuda_stream)));
    return hca_encode_status(status);
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
    VGB_TRY(hca_decode_check(info, n_streams));
    const vgb_hca_info &h0 = info[0];
    const int nch = h0.channel_count;
    const HcaConfig cfg = hca_config(h0);

    std::vector<HcaStream> streams(n_streams);
    std::vector<int64_t> in_off(n_streams), in_len(n_streams), out_off((size_t)n_streams * nch), out_len((size_t)n_streams * nch);
    int64_t ps = 0, fb = 0;
    for (int s = 0; s < n_streams; s++) {
        const int64_t stride = (int64_t)align_up((size_t)info[s].sample_count, 8);
        streams[s].pcm_off = ps;
        streams[s].channel_stride = stride;
        streams[s].frames_off = fb;
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
        return copy_units(cudaMemcpyHostToDevice, g_ctx.adpcm.c(), in_off.data(), frames, in_len.data(), s0, n, g_ctx.s_in);
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
        return copy_units(cudaMemcpyDeviceToHost, g_ctx.pcm.c(), out_off.data(), pcm_out, out_len.data(), s0 * nch, n * nch, g_ctx.s_out);
    };
    VGB_TRY(run_group_pipeline(n_groups, h2d, one_phase(kern), d2h, no_done));
    for (int s = 0; s < n_streams; s++) VGB_TRY(hca_decode_fault(status[s], "stream", s));
    return VGB_OK;
}

int32_t vgb_hca_decode_batch(const uint8_t *const *frames, const vgb_hca_info *info, int32_t n_streams, int16_t *const *pcm_out)
{
    if (!sharding_active(n_streams) || !frames || !info || !pcm_out) return hca_decode_one(frames, info, n_streams, pcm_out);
    const int nch = info[0].channel_count;
    if (nch < 1 || nch > 8) return hca_decode_one(frames, info, n_streams, pcm_out);
    return run_sharded(shard_units(n_streams, [&](int s) { return info[s].frame_count; }, 1), [&](int, const std::vector<int> &u) -> int32_t {
        auto s_in = pick_rows(frames, u);
        auto s_info = pick_rows(info, u);
        auto s_out = pick_rows(pcm_out, u, nch);
        return hca_decode_one(s_in.data(), s_info.data(), (int)u.size(), s_out.data());
    });
}

/* ---- device-resident HCA decode (see the header) ---- */
uint64_t vgb_hca_decode_workspace_bytes(const vgb_hca_info *info, int32_t n_streams)
{
    if (n_streams < 0 || (n_streams > 0 && !info)) return 0;
    int64_t frames = 0;
    for (int s = 0; s < n_streams; s++) frames += std::max(info[s].frame_count, 0);
    HcaConfig cfg{};
    cfg.channel_count = n_streams > 0 ? hca_clampi(info[0].channel_count, 1, 8) : 1;
    return HcaDecodeLayout(cfg, n_streams, frames).bytes;
}

int32_t vgb_hca_decode_dev(const uint8_t *d_frames, const int64_t *frames_offset, const vgb_hca_info *info, int32_t n_streams,
                           int16_t *d_pcm, const int64_t *pcm_offset, const int64_t *channel_stride,
                           void *d_workspace, uint64_t workspace_bytes, void *cuda_stream)
{
    if (n_streams < 0) return fail(VGB_E_ARG, "n_streams is negative");
    if (n_streams == 0) return VGB_OK;
    if (!d_frames || !frames_offset || !info || !d_pcm || !pcm_offset || !channel_stride || !d_workspace) return fail(VGB_E_ARG, "NULL argument");
    VGB_TRY(check_aligned(d_pcm, 2, "d_pcm"));
    VGB_TRY(check_aligned(d_workspace, 8, "d_workspace"));  // HcaStream's int64 fields, the fp64 seam addends
    if (n_streams > 65535) return fail(VGB_E_ARG, "n_streams %d: at most 65535 streams per call", n_streams);  // grid y / z of the frame kernels
    VGB_TRY(hca_decode_check(info, n_streams));
    const uint64_t need = vgb_hca_decode_workspace_bytes(info, n_streams);
    if (need > workspace_bytes) return fail(VGB_E_ARG, "workspace too small: need %llu bytes", (unsigned long long)need);
    const HcaConfig cfg = hca_config(info[0]);
    std::vector<HcaStream> streams(n_streams);
    int64_t total_frames = 0;
    int max_frames = 0;
    for (int s = 0; s < n_streams; s++) {
        const vgb_hca_info &h = info[s];
        if (frames_offset[s] < 0 || pcm_offset[s] < 0 || channel_stride[s] < h.sample_count)
            return fail(VGB_E_ARG, "stream %d: bad offsets (channel_stride must cover sample_count)", s);
        HcaStream &t = streams[s];
        t.pcm_off = pcm_offset[s];
        t.channel_stride = channel_stride[s];
        t.frames_off = frames_offset[s];
        t.dct_off = total_frames;  // the parse records and seam addends are indexed by the call-wide frame number
        t.sample_count = h.sample_count;
        t.frame_count = h.frame_count;
        t.inserted_samples = h.inserted_samples;
        total_frames += h.frame_count;
        max_frames = std::max(max_frames, h.frame_count);
    }
    const HcaDecodeLayout L(cfg, n_streams, total_frames);
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    VGB_TRY(hca_tables_ready_locked());
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    char *ws = static_cast<char *>(d_workspace);
    CUDA_TRY(cudaMemcpyAsync(ws, streams.data(), streams.size() * sizeof(HcaStream), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(ws + L.o_status, 0, (size_t)n_streams * 4, st));
    tick(7, true, st);
    CUDA_TRY(launch_hca_decode(d_frames, reinterpret_cast<const HcaStream *>(ws), n_streams, max_frames, total_frames, cfg, g_hca_tables.view,
                               reinterpret_cast<uint8_t *>(ws + L.o_parsed), reinterpret_cast<double *>(ws + L.o_edge), d_pcm,
                               reinterpret_cast<int32_t *>(ws + L.o_status), st));
    tick(7, false, st);
    g_ctx.launches += 3;
    return VGB_OK;
}

/* Synchronises `cuda_stream` and maps the per-stream status words the last vgb_hca_decode_dev on this workspace left
 * (the reference's InvalidDataException "Invalid frame header", ...). */
int32_t vgb_hca_decode_dev_status(const void *d_workspace, int32_t n_streams, void *cuda_stream)
{
    if (n_streams <= 0) return VGB_OK;
    if (!d_workspace) return fail(VGB_E_ARG, "NULL argument");
    std::vector<int32_t> status(n_streams, 0);
    VGB_TRY(hca_decode_words(d_workspace, n_streams, status.data(), static_cast<cudaStream_t>(cuda_stream)));
    for (int s = 0; s < n_streams; s++) VGB_TRY(hca_decode_fault(status[s], "stream", s));
    return VGB_OK;
}

}  // extern "C"
