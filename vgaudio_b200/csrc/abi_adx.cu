// abi_adx.cu — the CRI ADX entry points of the C ABI: host-pointer batch calls (pipelined over channel groups, sharded
// over the bound devices), the device-resident encode and the device-resident, time-parallel decode.
#include <climits>
#include <cmath>

#include "abi.cuh"

using namespace vgb;

extern "C" {

// ---- CRI ADX --------------------------------------------------------------------------------------------------

int32_t vgb_adx_encoded_byte_count(int32_t pcm_length, int32_t padding, int32_t frame_size)
{
    if (pcm_length < 0 || padding < 0 || frame_size < 3) return 0;
    const int32_t spf = (frame_size - 2) * 2;
    return (int32_t)(((int64_t)pcm_length + padding + spf - 1) / spf) * frame_size;
}

}  // extern "C"

namespace {

// (int)double on x64 (cvttsd2si): NaN and values outside int32 give int.MinValue
int32_t cast_double_to_int_x64(double v) { return (v > -2147483649.0 && v < 2147483648.0) ? (int32_t)v : INT32_MIN; }

// CriAdxCodec.CalculateCoefficients (CriAdxCodec.cs:173-184): host double math, once per distinct (freq, rate).
// (short)(double) goes through (int) truncation like the oracle; a rate of 0 makes the pair NaN, which C# casts to 0.
void adx_calc_coefs(int highpass, int rate, int16_t &c0, int16_t &c1)
{
    const double sqrt2 = std::sqrt(2.0);
    const double a = sqrt2 - std::cos(2.0 * 3.14159265358979323846 * highpass / rate);
    const double b = sqrt2 - 1;
    const double c = (a - std::sqrt((a + b) * (a - b))) / b;
    c0 = (int16_t)cast_double_to_int_x64(c * 8192);
    c1 = (int16_t)cast_double_to_int_x64(c * c * -4096);
}

// any_rate: the decode-side entry points take every sample rate the reference decodes (CalculateCoefficients is defined
// for all of them); the host batch calls keep their positive-rate rule
int32_t adx_validate(const vgb_adx_params &p, int c, bool any_rate = false)
{
    if (p.frame_size < 3 || p.frame_size > 255) return fail(VGB_E_ARG, "channel %d: frame_size %d outside 3..255", c, p.frame_size);
    if (p.type != 2 && p.type != 3 && p.type != 4) return fail(VGB_E_ARG, "channel %d: unknown CriAdxType %d", c, p.type);
    if (p.type == 2 && (p.filter < 0 || p.filter > 3)) return fail(VGB_E_ARG, "channel %d: filter %d outside 0..3", c, p.filter);
    if (p.padding < 0) return fail(VGB_E_ARG, "channel %d: negative padding", c);
    if (p.sample_rate <= 0 && !any_rate) return fail(VGB_E_ARG, "channel %d: sample_rate must be positive", c);
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

// Validates channel c of an encode call and fills its table row.
int32_t adx_encode_channel(const vgb_adx_params &p, int32_t n_samples, int c, int64_t pcm_off, int64_t adpcm_off, AdxChannel &t)
{
    VGB_TRY(adx_validate(p, c));
    if (n_samples < 0) return fail(VGB_E_ARG, "channel %d: negative sample count", c);
    // CriAdxCodec.cs:69-74 reads pcm[0]: an empty array throws IndexOutOfRangeException there
    if (p.version == 4 && p.padding == 0 && n_samples == 0)
        return fail(VGB_E_ARG, "channel %d: version 4 without padding needs at least one sample", c);
    t.pcm_off = pcm_off; t.adpcm_off = adpcm_off; t.n_samples = n_samples;
    t.frame_size = p.frame_size; t.version = p.version; t.padding = p.padding; t.type = p.type; t.filter = p.filter;
    t.history = 0;
    if (p.type == 2) { t.coef0 = kAdxFixed[p.filter][0]; t.coef1 = kAdxFixed[p.filter][1]; }
    else adx_calc_coefs(500, p.sample_rate, t.coef0, t.coef1);  // Encode hard-codes 500 (:63)
    return VGB_OK;
}

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
    int64_t ps = 0, ab = 0;
    for (int c = 0; c < n_channels; c++) {
        const vgb_adx_params &p = params[c];
        VGB_TRY(adx_encode_channel(p, n_samples[c], c, ps, ab, tab[c]));
        if (!pcm[c] && n_samples[c] > 0) return fail(VGB_E_ARG, "pcm[%d] is NULL", c);
        const int32_t bytes = vgb_adx_encoded_byte_count(n_samples[c], p.padding, p.frame_size);
        if (!adpcm_out[c] && bytes > 0) return fail(VGB_E_ARG, "adpcm_out[%d] is NULL", c);
        in_off[c] = ps * 2; in_len[c] = (int64_t)n_samples[c] * 2; out_off[c] = ab; out_len[c] = bytes;
        ps += (int64_t)align_up((size_t)n_samples[c], 8);
        ab += (int64_t)align_up((size_t)bytes, 16);
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
    auto h2d = [&](int g) -> int32_t {
        if (g == 0) CUDA_TRY(cudaMemcpyAsync(g_ctx.misc.p, tab.data(), tab.size() * sizeof(AdxChannel), cudaMemcpyHostToDevice, g_ctx.s_in));
        return copy_units(cudaMemcpyHostToDevice, g_ctx.pcm.c(), in_off.data(), pcm, in_len.data(), bound[g], bound[g + 1] - bound[g], g_ctx.s_in);
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
        return copy_units(cudaMemcpyDeviceToHost, g_ctx.adpcm.c(), out_off.data(), adpcm_out, out_len.data(), c0, n, g_ctx.s_out);
    };
    auto done = [&](int g) -> int32_t {  // IProgressReport: one delta per finished group, summing to the frame total
        int64_t frames = 0;
        for (int c = bound[g]; c < bound[g + 1]; c++) frames += out_len[c] / params[c].frame_size;
        if (cb && frames > 0) cb(user, frames);
        return VGB_OK;
    };
    return run_group_pipeline(n_groups, h2d, one_phase(kern), d2h, done);
}

int32_t vgb_adx_encode_batch(const int16_t *const *pcm, const int32_t *n_samples, const vgb_adx_params *params,
                             int32_t n_channels, int16_t *history_out, uint8_t *const *adpcm_out, vgb_progress_cb cb, void *user)
{
    if (!sharding_active(n_channels) || !pcm || !n_samples || !params || !adpcm_out)
        return adx_encode_one(pcm, n_samples, params, n_channels, history_out, adpcm_out, cb, user);
    SharedProgress prog{cb, user, {}};
    return run_sharded(shard_units(n_channels, [&](int c) { return n_samples[c]; }, 64), [&](int, const std::vector<int> &u) -> int32_t {
        const int m = (int)u.size();
        auto s_pcm = pick_rows(pcm, u);
        auto s_n = pick_rows(n_samples, u);
        auto s_par = pick_rows(params, u);
        auto s_out = pick_rows(adpcm_out, u);
        std::vector<int16_t> s_hist(m);
        VGB_TRY(adx_encode_one(s_pcm.data(), s_n.data(), s_par.data(), m, s_hist.data(), s_out.data(), cb ? SharedProgress::relay : nullptr, &prog));
        if (history_out) put_rows(history_out, u, s_hist);
        return VGB_OK;
    });
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
    VGB_TRY(check_aligned(d_pcm, 16, "d_pcm"));  // the encoder's cp.async
    VGB_TRY(check_aligned(d_history_out, 2, "d_history_out"));
    VGB_TRY(check_aligned(d_adpcm, 2, "d_adpcm"));  // uint16_t stores
    VGB_TRY(check_aligned(d_workspace, 8, "d_workspace"));  // AdxChannel's int64 fields
    {
        int64_t total = 0;
        for (int c = 0; c < n_channels; c++) total += n_samples[c] > 0 ? n_samples[c] : 0;
        if (vgb_adx_workspace_bytes(total, n_channels) > workspace_bytes)
            return fail(VGB_E_ARG, "workspace too small: need %llu bytes", (unsigned long long)vgb_adx_workspace_bytes(total, n_channels));
    }
    std::vector<AdxChannel> tab(n_channels);
    for (int c = 0; c < n_channels; c++) {
        VGB_TRY(adx_encode_channel(params[c], n_samples[c], c, pcm_offset[c], adpcm_offset[c], tab[c]));
        if (pcm_offset[c] < 0 || (pcm_offset[c] & 7) || adpcm_offset[c] < 0 || (adpcm_offset[c] & 1))
            return fail(VGB_E_ARG, "channel %d: pcm_offset must be a multiple of 8 samples, adpcm_offset even", c);
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
    auto h2d = [&](int g) -> int32_t {
        if (g == 0) {
            CUDA_TRY(cudaMemcpyAsync(g_ctx.misc.p, tab.data(), tab.size() * sizeof(AdxChannel), cudaMemcpyHostToDevice, g_ctx.s_in));
            CUDA_TRY(cudaMemsetAsync(d_status, 0x7f, 16 * (size_t)n_groups, g_ctx.s_in));
        }
        return copy_units(cudaMemcpyHostToDevice, g_ctx.adpcm.c(), in_off.data(), adpcm, in_len.data(), bound[g], bound[g + 1] - bound[g], g_ctx.s_in);
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
        VGB_TRY(copy_units(cudaMemcpyDeviceToHost, g_ctx.pcm.c(), out_off.data(), pcm_out, out_len.data(), bound[g], bound[g + 1] - bound[g], g_ctx.s_out));
        CUDA_TRY(cudaMemcpyAsync(&bad[g], d_status + 4 * g, 4, cudaMemcpyDeviceToHost, g_ctx.s_out));
        return VGB_OK;
    };
    VGB_TRY(run_group_pipeline(n_groups, h2d, one_phase(kern), d2h, no_done));
    // CriAdxCodec.Coefs[filterNum] (:186-191) has four rows: IndexOutOfRangeException in the reference
    for (int g = 0; g < n_groups; g++)
        if (bad[g] >= 0 && bad[g] < bound[g + 1] - bound[g])
            return fail(VGB_E_DATA, "channel %d: a Fixed-type frame selects a filter outside 0..3", bound[g] + bad[g]);
    return VGB_OK;
}

int32_t vgb_adx_decode_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int32_t *sample_count,
                             const vgb_adx_params *params, int32_t n_channels, int16_t *const *pcm_out)
{
    if (!sharding_active(n_channels) || !adpcm || !n_bytes || !sample_count || !params || !pcm_out)
        return adx_decode_one(adpcm, n_bytes, sample_count, params, n_channels, pcm_out);
    return run_sharded(shard_units(n_channels, [&](int c) { return sample_count[c]; }, 64), [&](int, const std::vector<int> &u) -> int32_t {
        auto s_in = pick_rows(adpcm, u);
        auto s_nb = pick_rows(n_bytes, u);
        auto s_sc = pick_rows(sample_count, u);
        auto s_par = pick_rows(params, u);
        auto s_out = pick_rows(pcm_out, u);
        return adx_decode_one(s_in.data(), s_nb.data(), s_sc.data(), s_par.data(), (int)u.size(), s_out.data());
    });
}

}  // extern "C"

namespace {

// Byte offsets in a workspace of the time-parallel decode (vgb_adx_decode_dev): channel table, status words, run-on
// start pairs, stats, the trace (one word per body frame)
struct AdxDecodeLayout {
    size_t o_status, o_used, o_stats, o_trace, bytes;
    AdxDecodeLayout(int n_channels, int64_t body_frames)
    {
        const size_t n = (size_t)std::max(n_channels, 1);
        o_status = align_up(n * sizeof(AdxDecChannel), 256);
        o_used = o_status + align_up(n * 4, 256);
        o_stats = o_used + align_up(n * kAdxDecMaxSegments * 4, 256);
        o_trace = o_stats + 256;
        bytes = o_trace + align_up((size_t)(body_frames + 1) * 4, 256);
    }
};

int64_t adx_body_frames(const int32_t *sample_count, const vgb_adx_params *params, int32_t n_channels)
{
    int64_t frames = 0;
    for (int c = 0; c < n_channels; c++) {
        const vgb_adx_params &p = params[c];
        if (p.frame_size < 3 || p.frame_size > 255 || p.padding < 0 || sample_count[c] < 0) continue;  // refused by the call
        frames += adx_dec_geom(sample_count[c], p.frame_size, p.padding).body;
    }
    return frames;
}

}  // namespace

int32_t vgb::adx_decode_words(const void *d_workspace, int32_t n_channels, int32_t *status, cudaStream_t st)
{
    const AdxDecodeLayout L(n_channels, 0);
    CUDA_TRY(cudaMemcpyAsync(status, static_cast<const char *>(d_workspace) + L.o_status, (size_t)n_channels * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return VGB_OK;
}

extern "C" {

/* ---- device-resident, time-parallel ADX decode (see the header) ---- */
uint64_t vgb_adx_decode_workspace_bytes(const int32_t *sample_count, const vgb_adx_params *params, int32_t n_channels)
{
    if (n_channels < 0 || (n_channels > 0 && (!sample_count || !params))) return 0;
    return AdxDecodeLayout(n_channels, adx_body_frames(sample_count, params, n_channels)).bytes;
}

int32_t vgb_adx_decode_dev(const uint8_t *d_adpcm, const int64_t *adpcm_offset, const int32_t *n_bytes, const int32_t *sample_count,
                           const vgb_adx_params *params, int32_t n_channels, int16_t *d_pcm, const int64_t *pcm_offset,
                           void *d_workspace, uint64_t workspace_bytes, void *cuda_stream)
{
    if (n_channels < 0) return fail(VGB_E_ARG, "n_channels is negative");
    if (n_channels == 0) return VGB_OK;
    if (!d_adpcm || !adpcm_offset || !n_bytes || !sample_count || !params || !d_pcm || !pcm_offset || !d_workspace)
        return fail(VGB_E_ARG, "NULL argument");
    if ((reinterpret_cast<uintptr_t>(d_pcm) & 1) || (reinterpret_cast<uintptr_t>(d_workspace) & 7))
        return fail(VGB_E_ARG, "d_pcm must be 2-byte and d_workspace 8-byte aligned");
    std::vector<AdxDecChannel> tab(n_channels);
    int64_t frames = 0;
    int max_body = 0;
    for (int c = 0; c < n_channels; c++) {
        const vgb_adx_params &p = params[c];
        VGB_TRY(adx_validate(p, c, /*any_rate=*/true));
        if (sample_count[c] < 0 || n_bytes[c] < 0) return fail(VGB_E_ARG, "channel %d: negative length", c);
        if (adpcm_offset[c] < 0 || pcm_offset[c] < 0) return fail(VGB_E_ARG, "channel %d: negative offset", c);
        const AdxDecGeom g = adx_dec_geom(sample_count[c], p.frame_size, p.padding);
        // the frames Decode walks must lie inside the row: the reference would index past its array
        const int64_t need = g.in0 + (int64_t)g.frames * p.frame_size;
        if (sample_count[c] > 0 && n_bytes[c] < need)
            return fail(VGB_E_ARG, "channel %d: %d bytes of ADX data, %lld needed for %d samples", c, n_bytes[c], (long long)need, sample_count[c]);
        AdxDecChannel &t = tab[c];
        t.pcm_off = pcm_offset[c]; t.adpcm_off = adpcm_offset[c]; t.trace_off = frames;
        t.n_samples = sample_count[c]; t.frame_size = p.frame_size; t.version = p.version; t.padding = p.padding; t.type = p.type;
        t.history = (int16_t)p.history;
        if (p.type == 2) { t.coef0 = 0; t.coef1 = 0; }
        else adx_calc_coefs(p.highpass_frequency, p.sample_rate, t.coef0, t.coef1);
        frames += g.body;
        max_body = std::max(max_body, g.body);
    }
    const AdxDecodeLayout L(n_channels, frames);
    if (L.bytes > workspace_bytes) return fail(VGB_E_ARG, "workspace too small: need %llu bytes", (unsigned long long)L.bytes);
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    char *ws = static_cast<char *>(d_workspace);
    AdxDecSegArgs sa{};
    sa.trace = reinterpret_cast<uint32_t *>(ws + L.o_trace);
    sa.used_start = reinterpret_cast<uint32_t *>(ws + L.o_used);
    sa.stats = reinterpret_cast<unsigned long long *>(ws + L.o_stats);
    sa.status = reinterpret_cast<int32_t *>(ws + L.o_status);
    sa.seg_count = adx_decode_pick_segments(n_channels, max_body, &sa.min_seg_frames);
    CUDA_TRY(cudaMemcpyAsync(ws, tab.data(), tab.size() * sizeof(AdxDecChannel), cudaMemcpyHostToDevice, st));  // pageable: staged before return
    CUDA_TRY(cudaMemsetAsync(ws + L.o_status, 0, (size_t)n_channels * 4, st));
    CUDA_TRY(cudaMemsetAsync(ws + L.o_stats, 0, kAdxDecStatWords * sizeof(unsigned long long), st));
    tick(5, true, st);
    launch_adx_decode_seg(d_adpcm, reinterpret_cast<const AdxDecChannel *>(ws), n_channels, d_pcm, sa, st);
    tick(5, false, st);
    g_ctx.launches += sa.seg_count > 1 ? 3 : 1;
    g_ctx.last_adx_dec = sa;
    CUDA_TRY(cudaGetLastError());
    return VGB_OK;
}

/* Synchronises `cuda_stream` and maps the status words the last vgb_adx_decode_dev on this workspace left: the lowest
 * channel whose Fixed-type frame selects a filter 4..7 (IndexOutOfRangeException at CriAdxCodec.Coefs, :186-191). */
int32_t vgb_adx_decode_dev_status(const void *d_workspace, int32_t n_channels, void *cuda_stream)
{
    if (n_channels <= 0) return VGB_OK;
    if (!d_workspace) return fail(VGB_E_ARG, "NULL argument");
    std::vector<int32_t> status(n_channels, 0);
    VGB_TRY(adx_decode_words(d_workspace, n_channels, status.data(), static_cast<cudaStream_t>(cuda_stream)));
    for (int c = 0; c < n_channels; c++)
        if (status[c] & 1) return fail(VGB_E_DATA, "channel %d: a Fixed-type frame selects a filter outside 0..3", c);
    return VGB_OK;
}

/* Bookkeeping of the most recent time-parallel ADX decode on this thread's context (see the header).  Synchronises
 * the device. */
int32_t vgb_adx_debug_decode_stats(uint64_t *out, int32_t n)
{
    if (!out || n < 0) return fail(VGB_E_ARG, "bad arguments");
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    for (int i = 0; i < n; i++) out[i] = 0;
    if (!g_ctx.ready || !g_ctx.last_adx_dec.stats) return VGB_OK;
    unsigned long long st[kAdxDecStatWords] = {};
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(st, g_ctx.last_adx_dec.stats, sizeof st, cudaMemcpyDeviceToHost));
    if (n > 0) out[0] = (uint64_t)g_ctx.last_adx_dec.seg_count;
    for (int i = 1; i < n && i <= kAdxDecStatWords; i++) out[i] = st[i - 1];
    return VGB_OK;
}

}  // extern "C"
