// abi_gcadpcm.cu — the GC-ADPCM (DSP) entry points of the C ABI: host-pointer batch calls (pipelined over channel groups,
// sharded over the bound devices), device-resident calls, seek tables and loop contexts, debug taps of the encoder.
#include <climits>

#include "abi.cuh"

using namespace vgb;

namespace {

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

// The record slab of a layout (rec_off, rec_total) and its frame counts, from n_samples and enc_count.
void layout_records(GcLayout &lay)
{
    lay.rec_off.resize(lay.n_channels);
    int64_t rec = 0;
    for (int c = 0; c < lay.n_channels; c++) {
        const int32_t frames = div_round_up(lay.n_samples[c], kGcFrameSamples);
        lay.rec_off[c] = rec;
        rec += (int64_t)align_up((size_t)frames, 32);
        if (frames > lay.max_frames) lay.max_frames = frames;
        lay.total_frames += div_round_up(lay.enc_count[c], kGcFrameSamples);
    }
    lay.rec_total = rec + 32;
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
    lay.hist.assign((size_t)n_channels * 2, 0);
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
    }
    layout_records(lay);
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
    layout_records(g);
    return g;
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
    std::vector<int64_t> weight(n_channels), pcm_b(n_channels), pcm_len(n_channels), adpcm_len(n_channels);
    int64_t total = 0;
    for (int c = 0; c < n_channels; c++) {
        weight[c] = lay.n_samples[c];
        total += lay.n_samples[c];
        pcm_b[c] = lay.pcm_off[c] * 2;
        pcm_len[c] = (int64_t)lay.n_samples[c] * 2;
        adpcm_len[c] = gc_sample_count_to_byte_count(lay.enc_count[c]);
    }

    // channel groups with roughly equal sample totals (boundaries on channel indices, order preserved).  The encoder is
    // throughput bound since it runs time-parallel (gc_encode.cu), so kernels of neighbouring groups share the SMs
    // without slowing each other: the PCIe copy of group g+1 hides the kernels of group g.  A group should carry at
    // least ~32 MB of PCM (a few ms of PCIe time) and 32 channels.
    const int n_groups = pipeline_group_count(n_channels, 2 * total, 32, "VGB_ENCODE_GROUPS");
    const std::vector<int> bound = pipeline_bounds(weight, n_groups);

    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
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
    int16_t *d_coefs_out = static_cast<int16_t *>(g_ctx.coefs.p);
    int16_t *d_coefs_in = coefs_in ? d_coefs_out + (size_t)n_channels * 16 : nullptr;

    auto h2d = [&](int g) -> int32_t {
        const int c0 = bound[g], n = bound[g + 1] - c0;
        if (g == 0)  // the small tables first, while the copy stream is idle
            for (int k = 0; k < n_groups; k++) VGB_TRY(upload_tables(glay[k], gws[k], g_ctx.ws.c() + ws_at[k], g_ctx.s_in));
        VGB_TRY(copy_units(cudaMemcpyHostToDevice, g_ctx.pcm.c(), pcm_b.data(), pcm, pcm_len.data(), c0, n, g_ctx.s_in));
        if (coefs_in && n > 0)
            CUDA_TRY(cudaMemcpyAsync(d_coefs_in + (size_t)c0 * 16, coefs_in + (size_t)c0 * 16, (size_t)n * 32,
                                     cudaMemcpyHostToDevice, g_ctx.s_in));
        return VGB_OK;
    };
    auto kern = [&](int g, cudaStream_t st, cudaEvent_t coefs_done) -> int32_t {
        const int c0 = bound[g];
        return run_gc_encode(static_cast<const int16_t *>(g_ctx.pcm.p), glay[g], d_coefs_in ? d_coefs_in + (size_t)c0 * 16 : nullptr,
                             d_coefs_out + (size_t)c0 * 16, static_cast<uint8_t *>(g_ctx.adpcm.p), g_ctx.ws.c() + ws_at[g], gws[g],
                             st, do_encode, /*timed=*/false, /*tables_uploaded=*/true, coefs_done);
    };
    auto d2h = [&](int g) -> int32_t {
        const int c0 = bound[g], n = bound[g + 1] - c0;
        if (n > 0)
            CUDA_TRY(cudaMemcpyAsync(coefs_out + (size_t)c0 * 16, d_coefs_out + (size_t)c0 * 16, (size_t)n * 32,
                                     cudaMemcpyDeviceToHost, g_ctx.s_out));
        if (!do_encode) return VGB_OK;
        return copy_units(cudaMemcpyDeviceToHost, g_ctx.adpcm.c(), lay.adpcm_off.data(), adpcm_out, adpcm_len.data(), c0, n, g_ctx.s_out);
    };
    auto done = [&](int g) -> int32_t {  // IProgressReport.ReportAdd: one delta per finished group, summing to SetTotal
        if (cb && do_encode && glay[g].total_frames > 0) cb(user, glay[g].total_frames);
        return VGB_OK;
    };
    return run_group_pipeline(n_groups, h2d, kern, d2h, done);
}

int32_t host_encode_sharded(const int16_t *const *pcm, const int32_t *n_samples, const vgb_gc_params *params,
                            const int16_t *coefs_in, int32_t n_channels, int16_t *coefs_out, uint8_t *const *adpcm_out,
                            vgb_progress_cb cb, void *user, bool do_encode)
{
    if (!sharding_active(n_channels) || !pcm || !n_samples || !coefs_out || (do_encode && !adpcm_out))
        return host_encode_impl(pcm, n_samples, params, coefs_in, n_channels, coefs_out, adpcm_out, cb, user, do_encode);
    SharedProgress prog{cb, user, {}};
    return run_sharded(shard_units(n_channels, [&](int c) { return n_samples[c]; }, 64), [&](int, const std::vector<int> &u) -> int32_t {
        const int m = (int)u.size();
        auto s_pcm = pick_rows(pcm, u);
        auto s_n = pick_rows(n_samples, u);
        std::vector<vgb_gc_params> s_par;
        if (params) s_par = pick_rows(params, u);
        std::vector<int16_t> s_cin, s_cout((size_t)m * 16);
        if (coefs_in) s_cin = pick_rows(coefs_in, u, 16);
        std::vector<uint8_t *> s_out;
        if (do_encode) s_out = pick_rows(adpcm_out, u);
        VGB_TRY(host_encode_impl(s_pcm.data(), s_n.data(), params ? s_par.data() : nullptr, coefs_in ? s_cin.data() : nullptr, m,
                                 s_cout.data(), do_encode ? s_out.data() : nullptr, cb ? SharedProgress::relay : nullptr, &prog, do_encode));
        put_rows(coefs_out, u, s_cout, 16);
        return VGB_OK;
    });
}

// ---- GcAdpcmAlignment (Formats/GcAdpcm/GcAdpcmAlignment.cs:20-63) --------------------------------------------------
struct AlignGeom {
    bool needed = false;
    int32_t loop_start_aligned = 0, sample_count_aligned = 0;
    int32_t keep = 0;        // samplesToKeep (:37-39): the whole frames below loop_end
    int32_t keep_bytes = 0;  // bytesToKeep
    int32_t count = 0;       // samplesToEncode
};

// SampleCountToNibbleCount without int32 wrap-around: where the reference's wraps, new byte[...] throws
int64_t gc_nibble_count64(int64_t n) { return 16 * (n / kGcFrameSamples) + (n % kGcFrameSamples ? n % kGcFrameSamples + 2 : 0); }

// The constructor's arithmetic (:22-39).  Returns why the loop points are unusable (the reference throws, or never
// returns), or nullptr.
const char *align_geometry(const vgb_gc_align_params &p, AlignGeom &g)
{
    g = AlignGeom{};
    const int32_t m = p.multiple, ls = p.loop_start, le = p.loop_end;
    if (m == -1 && ls == INT_MIN) return "loop_start % multiple overflows";  // int.MinValue % -1: OverflowException
    g.needed = m != 0 && (m == -1 ? 0 : ls % m) != 0;                        // !Helpers.LoopPointsAreAligned
    if (!g.needed) return nullptr;
    if (ls < 0 || le < 0) return "negative loop point";
    if (le < ls) return "loop_end is before loop_start";
    const int64_t lsa = (m <= 0 || ls % m == 0) ? ls : (int64_t)ls + m - ls % m;  // Helpers.GetNextMultiple
    const int64_t sca = (int64_t)le + (lsa - ls);
    if (sca > INT32_MAX || gc_nibble_count64(sca) > INT32_MAX) return "the aligned sample count overflows int32";
    // the reference's tail loop (:48) would step by loopLength == 0 forever
    if (le == ls && lsa != ls) return "loop_start == loop_end: an empty loop cannot fill the shift of the loop start";
    g.loop_start_aligned = (int32_t)lsa;
    g.sample_count_aligned = (int32_t)sca;
    g.keep = le / kGcFrameSamples * kGcFrameSamples;
    g.keep_bytes = le / kGcFrameSamples * kGcFrameBytes;
    g.count = g.sample_count_aligned - g.keep;
    return nullptr;
}

// Validation of a whole batch (host only): the channels that need alignment and their geometry.
int32_t align_plan(const uint8_t *const *adpcm, const int32_t *n_bytes, const vgb_gc_align_params *params, int32_t n_channels,
                   uint8_t *const *adpcm_out, int16_t *const *pcm_out, std::vector<int> &idx, std::vector<AlignGeom> &geo)
{
    if (n_channels < 0) return fail(VGB_E_ARG, "n_channels is negative (%d)", n_channels);
    if (n_channels > 0 && (!adpcm || !n_bytes || !params)) return fail(VGB_E_ARG, "NULL argument");
    for (int c = 0; c < n_channels; c++) {
        AlignGeom g;
        if (const char *why = align_geometry(params[c], g)) return fail(VGB_E_ARG, "channel %d: %s", c, why);
        if (!g.needed) continue;
        const int32_t le = params[c].loop_end;
        // GcAdpcmDecoder.Decode reads SampleCountToByteCount(loop_end) bytes (GcAdpcmChannel.cs:33-36's message)
        if (n_bytes[c] < gc_sample_count_to_byte_count(le))  // le <= sample_count_aligned: no wrap-around
            return fail(VGB_E_ARG, "channel %d: audio array length %d is too short for %d samples", c, n_bytes[c], le);
        if (!adpcm[c]) return fail(VGB_E_ARG, "channel %d: NULL buffer", c);
        if (!adpcm_out || !adpcm_out[c]) return fail(VGB_E_ARG, "channel %d: adpcm_aligned_out is NULL", c);
        if (pcm_out && !pcm_out[c]) return fail(VGB_E_ARG, "channel %d: pcm_aligned_out is NULL", c);
        idx.push_back(c);
        geo.push_back(g);
    }
    return VGB_OK;
}

// GcAdpcmAlignment.cs:44-62 on device rows, after the first decode: the tails from that decode (d_src, gc_align_tail_kernel,
// :44-55), their encode with each channel's own coefficients from the history the tail kernel leaves in the encoder's
// table (:57), and, with `dec`, their decode (:61).  enc / dec lay the tails out in d_pcm / d_adpcm; their tables go to
// ws_enc / ws_dec here.  The caller holds g_ctx.mu.
int32_t align_tails(const int16_t *d_src, const GcAlignChannel *d_chans, const GcLayout &enc, const GcLayout *dec, const int16_t *d_coefs,
                    int16_t *d_pcm, uint8_t *d_adpcm, char *ws_enc, const GcWorkspace &w_enc, char *ws_dec, const GcWorkspace &w_dec,
                    cudaStream_t st)
{
    const int m = enc.n_channels;
    if (m == 0) return VGB_OK;
    VGB_TRY(upload_tables(enc, w_enc, ws_enc, st));
    if (dec) VGB_TRY(upload_tables(*dec, w_dec, ws_dec, st));
    const GcChannelTable t_enc = table_view(ws_enc, w_enc, m);
    const GcChannelTable t_dec = dec ? table_view(ws_dec, w_dec, m) : t_enc;
    launch_gc_align_tail(d_src, d_chans, m, d_pcm, t_enc.hist, t_dec.hist, st);
    g_ctx.launches += 1;
    CUDA_TRY(cudaGetLastError());
    VGB_TRY(run_gc_encode(d_pcm, enc, d_coefs, const_cast<int16_t *>(d_coefs), d_adpcm, ws_enc, w_enc, st,
                          /*do_encode=*/true, /*timed=*/false, /*tables_uploaded=*/true));
    if (dec) {
        launch_gc_decode(d_adpcm, t_dec, d_coefs, d_pcm, dec->max_frames, 0, INT_MAX, st);
        g_ctx.launches += dec->max_frames > 0 ? 1 : 0;
        CUDA_TRY(cudaGetLastError());
    }
    return VGB_OK;
}

// The workspace of vgb::gc_align_tails: [channel table | tail PCM rows | tail ADPCM rows | encoder workspace]
struct TailWs {
    GcLayout enc;
    GcWorkspace w{};
    size_t o_pcm = 0, o_adpcm = 0, o_enc = 0, total = 0;
    int32_t build(const std::vector<GcAlignChannel> &chans)
    {
        std::vector<int32_t> n(chans.size());
        for (size_t i = 0; i < chans.size(); i++) n[i] = chans[i].count;
        VGB_TRY(layout_common(enc, n.data(), nullptr, (int32_t)n.size(), true));
        layout_pack_offsets(enc);
        w = carve(enc.rec_total, enc.n_channels);
        o_pcm = align_up(std::max<size_t>(chans.size(), 1) * sizeof(GcAlignChannel), 256);
        o_adpcm = o_pcm + align_up((size_t)enc.pcm_total * 2, 256);
        o_enc = o_adpcm + align_up((size_t)enc.adpcm_total, 256);
        total = o_enc + w.total;
        return VGB_OK;
    }
};

// One device: H2D of the prefixes, then decode -> tail -> encode (-> decode) on one stream, D2H into the caller's rows
// and one synchronisation.  A predictor 8..15 below loop_end leaves the lowest such channel in *bad and returns
// VGB_E_DATA.
int32_t align_one(const uint8_t *const *adpcm, const int32_t *n_bytes, const int16_t *coefs, const vgb_gc_align_params *params,
                  int32_t n_channels, uint8_t *const *adpcm_out, int16_t *const *pcm_out, int32_t *bad)
{
    PinScope pins;
    std::vector<int> idx;
    std::vector<AlignGeom> geo;
    VGB_TRY(align_plan(adpcm, n_bytes, params, n_channels, adpcm_out, pcm_out, idx, geo));
    const int m = (int)idx.size();
    if (m == 0) return VGB_OK;
    if (!coefs) return fail(VGB_E_ARG, "coefs is NULL");

    // slabs: adpcm = [prefixes | tails], pcm = [decoded prefixes | tails | decoded tails]; workspaces of the three kernels
    std::vector<int32_t> n_pre(m), n_tail(m);
    for (int i = 0; i < m; i++) {
        n_pre[i] = params[idx[i]].loop_end;
        n_tail[i] = geo[i].count;
    }
    GcLayout pre, enc;
    VGB_TRY(layout_common(pre, n_pre.data(), nullptr, m, true));
    VGB_TRY(layout_common(enc, n_tail.data(), nullptr, m, true));
    layout_pack_offsets(pre);
    layout_pack_offsets(enc);
    for (int i = 0; i < m; i++) {
        enc.pcm_off[i] += pre.pcm_total;
        enc.adpcm_off[i] += pre.adpcm_total;
    }
    GcLayout dec = enc;
    for (int i = 0; i < m; i++) dec.pcm_off[i] += enc.pcm_total;
    const GcWorkspace w_pre = carve(32, m), w_enc = carve(enc.rec_total, m), w_dec = carve(32, m);
    const size_t at_enc = align_up(w_pre.total, 256), at_dec = at_enc + align_up(w_enc.total, 256);

    std::vector<GcAlignChannel> chans(m);
    std::vector<int16_t> co((size_t)m * 16);
    std::vector<const uint8_t *> src(m);
    std::vector<uint8_t *> tail_dst(m);
    std::vector<int16_t *> pcm_pre_dst(m), pcm_tail_dst(m);
    std::vector<int64_t> pre_bytes(m), tail_bytes(m), pre_pcm_b(m), pre_pcm_len(m), dec_pcm_b(m), dec_pcm_len(m);
    for (int i = 0; i < m; i++) {
        const int c = idx[i];
        const AlignGeom &g = geo[i];
        chans[i] = GcAlignChannel{pre.pcm_off[i], enc.pcm_off[i], params[c].loop_start, params[c].loop_end, g.keep, g.count};
        std::copy_n(coefs + (size_t)c * 16, 16, co.begin() + (size_t)i * 16);
        src[i] = adpcm[c];
        pre_bytes[i] = gc_sample_count_to_byte_count(n_pre[i]);
        tail_dst[i] = adpcm_out[c] + g.keep_bytes;
        tail_bytes[i] = gc_sample_count_to_byte_count(g.count);
        if (pcm_out) {
            pcm_pre_dst[i] = pcm_out[c];
            pcm_tail_dst[i] = pcm_out[c] + g.keep;
        }
        pre_pcm_b[i] = pre.pcm_off[i] * 2;
        pre_pcm_len[i] = (int64_t)g.keep * 2;
        dec_pcm_b[i] = dec.pcm_off[i] * 2;
        dec_pcm_len[i] = (int64_t)g.count * 2;
    }

    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    cudaStream_t st = g_ctx.stream;
    VGB_TRY(g_ctx.adpcm.reserve((size_t)(pre.adpcm_total + enc.adpcm_total)));
    VGB_TRY(g_ctx.pcm.reserve((size_t)(pre.pcm_total + 2 * enc.pcm_total) * 2));
    VGB_TRY(g_ctx.coefs.reserve(co.size() * 2));
    VGB_TRY(g_ctx.ws.reserve(at_dec + w_dec.total));
    VGB_TRY(g_ctx.misc.reserve(chans.size() * sizeof(GcAlignChannel)));
    int16_t *d_pcm = static_cast<int16_t *>(g_ctx.pcm.p);
    uint8_t *d_adpcm = static_cast<uint8_t *>(g_ctx.adpcm.p);
    const int16_t *d_coefs = static_cast<const int16_t *>(g_ctx.coefs.p);
    const GcAlignChannel *d_chans = static_cast<const GcAlignChannel *>(g_ctx.misc.p);

    VGB_TRY(copy_units(cudaMemcpyHostToDevice, g_ctx.adpcm.c(), pre.adpcm_off.data(), src.data(), pre_bytes.data(), 0, m, st));
    // pageable sources: the runtime stages them before returning
    CUDA_TRY(cudaMemcpyAsync(g_ctx.coefs.p, co.data(), co.size() * 2, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(g_ctx.misc.p, chans.data(), chans.size() * sizeof(GcAlignChannel), cudaMemcpyHostToDevice, st));
    VGB_TRY(upload_tables(pre, w_pre, g_ctx.ws.p, st));
    const GcChannelTable t_pre = table_view(g_ctx.ws.p, w_pre, m);

    CUDA_TRY(cudaMemsetAsync(t_pre.status, 0x7f, 4, st));  // "no channel": any index is smaller
    launch_gc_decode(d_adpcm, t_pre, d_coefs, d_pcm, pre.max_frames, 0, INT_MAX, st);           // :41-42
    g_ctx.launches += pre.max_frames > 0 ? 1 : 0;
    CUDA_TRY(cudaGetLastError());
    VGB_TRY(align_tails(d_pcm, d_chans, enc, pcm_out ? &dec : nullptr, d_coefs, d_pcm, d_adpcm, g_ctx.ws.c() + at_enc, w_enc,
                        g_ctx.ws.c() + at_dec, w_dec, st));                                    // :44-61
    VGB_TRY(copy_units(cudaMemcpyDeviceToHost, g_ctx.adpcm.c(), enc.adpcm_off.data(), tail_dst.data(), tail_bytes.data(), 0, m, st));
    if (pcm_out) {  // PcmAligned = first decode on [0, keep), the tail's decode on [keep, sample_count_aligned) (:43, :62)
        VGB_TRY(copy_units(cudaMemcpyDeviceToHost, g_ctx.pcm.c(), pre_pcm_b.data(), pcm_pre_dst.data(), pre_pcm_len.data(), 0, m, st));
        VGB_TRY(copy_units(cudaMemcpyDeviceToHost, g_ctx.pcm.c(), dec_pcm_b.data(), pcm_tail_dst.data(), dec_pcm_len.data(), 0, m, st));
    }
    int32_t bad_channel = INT_MAX;
    CUDA_TRY(cudaMemcpyAsync(&bad_channel, t_pre.status, 4, cudaMemcpyDeviceToHost, st));
    // the kept frames are the caller's own bytes (:58): copied here while the device works
    for (int i = 0; i < m; i++) memcpy(adpcm_out[idx[i]], adpcm[idx[i]], (size_t)geo[i].keep_bytes);
    CUDA_TRY(cudaStreamSynchronize(st));
    if (bad_channel >= 0 && bad_channel < m) {  // IndexOutOfRangeException in the first Decode (GcAdpcmDecoder.cs:31-32)
        if (bad) *bad = idx[bad_channel];
        return fail(VGB_E_DATA, "channel %d: a frame header selects a predictor outside 0..7", idx[bad_channel]);
    }
    return VGB_OK;
}

// Byte offsets in a workspace of the time-parallel decode: channel table, status words, run-on start pairs, stats, the
// trace (one word per full frame)
struct GcSegDecodeLayout {
    size_t o_status, o_used, o_stats, o_trace, bytes;
    GcSegDecodeLayout(int n_channels, int64_t full_frames)
    {
        const size_t n = (size_t)std::max(n_channels, 1);
        o_status = align_up(n * sizeof(GcDecChannel), 256);
        o_used = o_status + align_up(n * 4, 256);
        o_stats = o_used + align_up(n * kGcDecMaxSegments * 4, 256);
        o_trace = o_stats + 256;
        bytes = o_trace + align_up((size_t)(full_frames + 1) * 4, 256);
    }
};

}  // namespace

uint64_t vgb::gc_decode_seg_workspace_bytes(int32_t n_channels, int64_t full_frames)
{
    return GcSegDecodeLayout(n_channels, full_frames).bytes;
}

int32_t vgb::gc_decode_seg(const uint8_t *d_adpcm, std::vector<GcDecChannel> &tab, int16_t *d_pcm, void *d_workspace, cudaStream_t st,
                           const int16_t *d_coefs)
{
    const int n_channels = (int)tab.size();
    if (n_channels == 0) return VGB_OK;
    int64_t frames = 0;
    int max_full = 0;
    for (GcDecChannel &c : tab) {
        const int full = c.n_samples / kGcFrameSamples;
        c.trace_off = frames;
        frames += full;
        max_full = std::max(max_full, full);
    }
    const GcSegDecodeLayout L(n_channels, frames);
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    char *ws = static_cast<char *>(d_workspace);
    GcDecSegArgs sa{};
    sa.trace = reinterpret_cast<uint32_t *>(ws + L.o_trace);
    sa.used_start = reinterpret_cast<uint32_t *>(ws + L.o_used);
    sa.stats = reinterpret_cast<unsigned long long *>(ws + L.o_stats);
    sa.status = reinterpret_cast<int32_t *>(ws + L.o_status);
    sa.seg_count = gc_decode_pick_segments(n_channels, max_full, &sa.min_seg_frames);
    CUDA_TRY(cudaMemcpyAsync(ws, tab.data(), tab.size() * sizeof(GcDecChannel), cudaMemcpyHostToDevice, st));  // pageable: staged before return
    if (d_coefs)
        CUDA_TRY(cudaMemcpy2DAsync(ws + offsetof(GcDecChannel, coefs), sizeof(GcDecChannel), d_coefs, 32, 32, (size_t)n_channels,
                                   cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaMemsetAsync(ws + L.o_status, 0, (size_t)n_channels * 4, st));
    CUDA_TRY(cudaMemsetAsync(ws + L.o_stats, 0, kGcDecStatWords * sizeof(unsigned long long), st));
    tick(3, true, st);
    launch_gc_decode_seg(d_adpcm, reinterpret_cast<const GcDecChannel *>(ws), n_channels, d_pcm, sa, st);
    tick(3, false, st);
    g_ctx.launches += sa.seg_count > 1 ? 3 : 1;
    g_ctx.last_gc_dec = sa;
    CUDA_TRY(cudaGetLastError());
    return VGB_OK;
}

int32_t vgb::gc_decode_seg_words(const void *d_workspace, int32_t n_channels, int32_t *status, cudaStream_t st)
{
    const GcSegDecodeLayout L(n_channels, 0);
    CUDA_TRY(cudaMemcpyAsync(status, static_cast<const char *>(d_workspace) + L.o_status, (size_t)n_channels * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return VGB_OK;
}

uint64_t vgb::gc_align_tails_workspace_bytes(const std::vector<GcAlignChannel> &chans)
{
    TailWs t;
    return t.build(chans) == VGB_OK ? t.total : 0;
}

int32_t vgb::gc_align_tails(const int16_t *d_src, std::vector<GcAlignChannel> &chans, const int16_t *d_coefs, void *d_workspace,
                            cudaStream_t st, std::vector<int64_t> &tail_adpcm_off)
{
    TailWs t;
    VGB_TRY(t.build(chans));
    for (size_t i = 0; i < chans.size(); i++) chans[i].dst_off = t.enc.pcm_off[i];
    tail_adpcm_off.resize(chans.size());
    for (size_t i = 0; i < chans.size(); i++) tail_adpcm_off[i] = (int64_t)t.o_adpcm + t.enc.adpcm_off[i];
    if (chans.empty()) return VGB_OK;
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    char *ws = static_cast<char *>(d_workspace);
    CUDA_TRY(cudaMemcpyAsync(ws, chans.data(), chans.size() * sizeof(GcAlignChannel), cudaMemcpyHostToDevice, st));  // pageable: staged before return
    return align_tails(d_src, reinterpret_cast<const GcAlignChannel *>(ws), t.enc, nullptr, d_coefs, reinterpret_cast<int16_t *>(ws + t.o_pcm),
                       reinterpret_cast<uint8_t *>(ws + t.o_adpcm), ws + t.o_enc, t.w, nullptr, t.w, st);
}

extern "C" {

/* Bookkeeping of the most recent time-parallel GC-ADPCM decode on this thread's context (see the header).
 * Synchronises the device. */
int32_t vgb_gcadpcm_debug_decode_stats(uint64_t *out, int32_t n)
{
    if (!out || n < 0) return fail(VGB_E_ARG, "bad arguments");
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    for (int i = 0; i < n; i++) out[i] = 0;
    if (!g_ctx.ready || !g_ctx.last_gc_dec.stats) return VGB_OK;
    unsigned long long st[kGcDecStatWords] = {};
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(st, g_ctx.last_gc_dec.stats, sizeof st, cudaMemcpyDeviceToHost));
    if (n > 0) out[0] = (uint64_t)g_ctx.last_gc_dec.seg_count;
    for (int i = 1; i < n && i <= kGcDecStatWords; i++) out[i] = st[i - 1];
    return VGB_OK;
}

int32_t vgb_gcadpcm_alignment(const vgb_gc_align_params *p, vgb_gc_alignment *out)
{
    if (!p || !out) return fail(VGB_E_ARG, "NULL argument");
    *out = vgb_gc_alignment{0, 0, 0};
    AlignGeom g;
    if (const char *why = align_geometry(*p, g)) return fail(VGB_E_ARG, "%s", why);
    if (g.needed) *out = vgb_gc_alignment{1, g.loop_start_aligned, g.sample_count_aligned};
    return VGB_OK;
}

int32_t vgb_gcadpcm_align_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int16_t *coefs,
                                const vgb_gc_align_params *params, int32_t n_channels,
                                uint8_t *const *adpcm_aligned_out, int16_t *const *pcm_aligned_out)
{
    if (!sharding_active(n_channels) || !adpcm || !n_bytes || !coefs || !params)
        return align_one(adpcm, n_bytes, coefs, params, n_channels, adpcm_aligned_out, pcm_aligned_out, nullptr);
    {  // every argument error before any device works
        std::vector<int> idx;
        std::vector<AlignGeom> geo;
        VGB_TRY(align_plan(adpcm, n_bytes, params, n_channels, adpcm_aligned_out, pcm_aligned_out, idx, geo));
        if (idx.empty()) return VGB_OK;
    }
    // a shard that meets a bad predictor reports its lowest channel; the call names the lowest of all shards
    std::mutex mu;
    int32_t lowest_bad = INT_MAX;
    auto needed = [&](int c) { AlignGeom g; align_geometry(params[c], g); return g.needed ? params[c].loop_end : 0; };
    VGB_TRY(run_sharded(shard_units(n_channels, needed, 64), [&](int, const std::vector<int> &u) -> int32_t {
        auto s_in = pick_rows(adpcm, u);
        auto s_nb = pick_rows(n_bytes, u);
        auto s_co = pick_rows(coefs, u, 16);
        auto s_par = pick_rows(params, u);
        std::vector<uint8_t *> s_out;
        std::vector<int16_t *> s_pcm;
        if (adpcm_aligned_out) s_out = pick_rows(adpcm_aligned_out, u);
        if (pcm_aligned_out) s_pcm = pick_rows(pcm_aligned_out, u);
        int32_t bad = -1;
        const int32_t rc = align_one(s_in.data(), s_nb.data(), s_co.data(), s_par.data(), (int32_t)u.size(),
                                     adpcm_aligned_out ? s_out.data() : nullptr, pcm_aligned_out ? s_pcm.data() : nullptr, &bad);
        if (rc == VGB_E_DATA && bad >= 0) {
            std::lock_guard<std::mutex> lock(mu);
            lowest_bad = std::min(lowest_bad, (int32_t)u[bad]);
            return VGB_OK;
        }
        return rc;
    }));
    if (lowest_bad != INT_MAX) return fail(VGB_E_DATA, "channel %d: a frame header selects a predictor outside 0..7", lowest_bad);
    return VGB_OK;
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
    std::vector<int64_t> weight(n_channels), adpcm_len(n_channels), pcm_b(n_channels), pcm_len(n_channels);
    int64_t pcie_bytes = 0;
    for (int c = 0; c < n_channels; c++) {
        weight[c] = (int64_t)counts[c] + 64;
        pcie_bytes += (int64_t)counts[c] * 2 + gc_sample_count_to_byte_count(counts[c]);
        adpcm_len[c] = gc_sample_count_to_byte_count(counts[c]);
        pcm_b[c] = lay.pcm_off[c] * 2;
        pcm_len[c] = (int64_t)counts[c] * 2;
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
        return copy_units(cudaMemcpyHostToDevice, g_ctx.adpcm.c(), lay.adpcm_off.data(), adpcm, adpcm_len.data(), c0, n, g_ctx.s_in);
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
        VGB_TRY(copy_units(cudaMemcpyDeviceToHost, g_ctx.pcm.c(), pcm_b.data(), pcm_out, pcm_len.data(), c0, n, g_ctx.s_out));
        if (n > 0) CUDA_TRY(cudaMemcpyAsync(&bad[g], ws_base + ws_at[g] + gws[g].off_status, 4, cudaMemcpyDeviceToHost, g_ctx.s_out));
        return VGB_OK;
    };
    VGB_TRY(run_group_pipeline(n_groups, h2d, one_phase(kern), d2h, no_done));
    // coefs[predictor * 2] with predictor 8..15 is an IndexOutOfRangeException in GcAdpcmDecoder.Decode (:31-32)
    for (int g = 0; g < n_groups; g++)
        if (bad[g] >= 0 && bad[g] < glay[g].n_channels)
            return fail(VGB_E_DATA, "channel %d: a frame header selects a predictor outside 0..7", bound[g] + bad[g]);
    return VGB_OK;
}

int32_t vgb_gcadpcm_decode_batch(const uint8_t *const *adpcm, const int32_t *n_bytes, const int16_t *coefs,
                                 const vgb_gc_params *params, int32_t n_channels, int16_t *const *pcm_out)
{
    if (!sharding_active(n_channels) || !adpcm || !n_bytes || !coefs || !pcm_out)
        return gcadpcm_decode_one(adpcm, n_bytes, coefs, params, n_channels, pcm_out);
    return run_sharded(shard_units(n_channels, [&](int c) { return n_bytes[c]; }, 64), [&](int, const std::vector<int> &u) -> int32_t {
        const int m = (int)u.size();
        auto s_in = pick_rows(adpcm, u);
        auto s_nb = pick_rows(n_bytes, u);
        auto s_out = pick_rows(pcm_out, u);
        std::vector<vgb_gc_params> s_par;
        if (params) s_par = pick_rows(params, u);
        auto s_co = pick_rows(coefs, u, 16);
        return gcadpcm_decode_one(s_in.data(), s_nb.data(), s_co.data(), params ? s_par.data() : nullptr, m, s_out.data());
    });
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
    std::vector<int64_t> len_b(n_channels);
    for (int c = 0; c < n_channels; c++) len_b[c] = gc_sample_count_to_byte_count(counts[c]);
    VGB_TRY(copy_units(cudaMemcpyHostToDevice, g_ctx.adpcm.c(), lay.adpcm_off.data(), adpcm, len_b.data(), 0, n_channels, st));
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
    if (seek_table_out) VGB_TRY(copy_units(cudaMemcpyDeviceToHost, misc, tap_off.data(), seek_table_out, tap_len.data(), 0, n_channels, st));
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
    VGB_TRY(check_aligned(d_pcm, 16, "d_pcm"));  // gc_coef_frames_kernel's uint4 loads, the encoder's cp.async
    VGB_TRY(check_aligned(d_coefs_in, 2, "d_coefs_in"));
    VGB_TRY(check_aligned(d_coefs_out, 2, "d_coefs_out"));
    VGB_TRY(check_aligned(d_adpcm, 16, "d_adpcm"));  // the encoder's uint4 stores
    VGB_TRY(check_aligned(d_workspace, 16, "d_workspace"));  // double2 records
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
    VGB_TRY(check_aligned(d_pcm, 16, "d_pcm"));
    VGB_TRY(check_aligned(d_coefs_out, 2, "d_coefs_out"));
    VGB_TRY(check_aligned(d_workspace, 16, "d_workspace"));
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
    VGB_TRY(check_aligned(d_adpcm, 16, "d_adpcm"));  // gc_decode_kernel's cp.async
    VGB_TRY(check_aligned(d_coefs, 2, "d_coefs"));
    VGB_TRY(check_aligned(d_pcm, 16, "d_pcm"));  // its uint4 stores
    VGB_TRY(check_aligned(d_workspace, 16, "d_workspace"));
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

int32_t vgb_gcadpcm_debug_refine_trace(const int16_t *const *pcm, const int32_t *n_samples, int32_t n_channels, int32_t warps,
                                       double *cent_out, int32_t *hits_out, int16_t *coefs_out)
{
    if (n_channels < 0 || (warps != 4 && warps != 8) || !cent_out || !hits_out || !coefs_out)
        return fail(VGB_E_ARG, "bad arguments");
    if (n_channels == 0) return VGB_OK;
    if (!pcm) return fail(VGB_E_ARG, "pcm is NULL");
    GcLayout lay;
    VGB_TRY(layout_common(lay, n_samples, nullptr, n_channels, false));
    for (int c = 0; c < n_channels; c++)
        if (!pcm[c] && lay.n_samples[c] > 0) return fail(VGB_E_ARG, "pcm[%d] is NULL", c);
    layout_pack_offsets(lay);
    std::vector<int64_t> pcm_b(n_channels), pcm_len(n_channels);
    for (int c = 0; c < n_channels; c++) {
        pcm_b[c] = lay.pcm_off[c] * 2;
        pcm_len[c] = (int64_t)lay.n_samples[c] * 2;
    }
    std::lock_guard<std::mutex> lock(g_ctx.mu);
    VGB_TRY(ensure_ready_locked());
    cudaStream_t st = g_ctx.stream;
    const GcWorkspace w = carve(lay.rec_total, n_channels);
    const size_t n = (size_t)n_channels, cent_bytes = n * 7 * 8 * 2 * 8, hits_bytes = n * 7 * 8 * 4;
    VGB_TRY(g_ctx.pcm.reserve((size_t)lay.pcm_total * 2));
    VGB_TRY(g_ctx.ws.reserve(w.total));
    VGB_TRY(g_ctx.coefs.reserve(n * 32));
    VGB_TRY(g_ctx.misc.reserve(align_up(cent_bytes, 256) + hits_bytes));
    double *d_cent = reinterpret_cast<double *>(g_ctx.misc.p);
    int32_t *d_hits = reinterpret_cast<int32_t *>(g_ctx.misc.c() + align_up(cent_bytes, 256));
    VGB_TRY(copy_units(cudaMemcpyHostToDevice, g_ctx.pcm.c(), pcm_b.data(), pcm, pcm_len.data(), 0, n_channels, st));
    VGB_TRY(upload_tables(lay, w, g_ctx.ws.p, st));
    GcChannelTable tab = table_view(g_ctx.ws.p, w, n_channels);
    double2 *records = reinterpret_cast<double2 *>(g_ctx.ws.c() + w.off_records);
    uint32_t *mask = reinterpret_cast<uint32_t *>(g_ctx.ws.c() + w.off_mask);
    launch_gc_coef_frames(static_cast<const int16_t *>(g_ctx.pcm.p), tab, records, mask, lay.max_frames, 0, INT_MAX, st);
    launch_gc_coef_refine_tap(tab, records, mask, static_cast<int16_t *>(g_ctx.coefs.p), warps, d_cent, d_hits, st);
    g_ctx.launches += (lay.max_frames > 0 ? 1 : 0) + 1;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(cent_out, d_cent, cent_bytes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(hits_out, d_hits, hits_bytes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(coefs_out, g_ctx.coefs.p, n * 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return VGB_OK;
}

}  // extern "C"
