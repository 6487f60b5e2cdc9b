// vgaudio_batch — batch conversion of a directory of audio files on the GPU: WAVE, .dsp, .adx and .hca files to
// .dsp / .adx / .hca, and .dsp, .adx and .hca files to WAVE.
//
// The counterpart of `VGAudioCli -b` (src/VGAudio.Cli/Batch.cs:11-51): the reference enumerates the input files and runs
// Convert.ConvertFile on each from a Parallel.ForEach; here the host only reads and writes files, and every
// reader -> encoder -> writer chain of a chunk of files runs as ONE coalesced call on the device per kind of input
// (vgb_convert_wave_batch for WAVE files, vgb_transcode_batch for coded files, vgb_convert_*_to_wave_batch for
// --out-format wav).  A file that fails is reported and skipped, like the reference's try/catch (:39-43).
//
//   vgaudio_batch -i <indir> -o <outdir> --out-format dsp|adx|hca|wav [-r]   (wav: .dsp, .hca and .adx inputs are decoded) [--no-trim] [--hcaquality Highest|High|Middle|Low|Lowest]
//                 [--bitrate N] [--limit-bitrate] [--keycode N] [--keystring S] [--in-keycode N] [--in-keystring S]
//                 [--adxtype Linear|Fixed|Exp|ExpEnc...] [--framesize N] [--version 3|4] [--chunk-mb N] [--devices LIST]
//
// With --out-format dsp|adx|hca the inputs are the .wav / .wave files and the .dsp, .adx and .hca files in another codec
// than the output's (a file already in the output's codec is not listed: the same codec would be a rewrite).
// --keycode / --keystring are the output's key; --in-keycode N is the key of type-56 .hca inputs, and --in-keystring S,
// or else --in-keycode N, the CriAdxKey of type-8 / type-9 .adx inputs.
// With --out-format wav, --keycode N is the key of type-56 .hca files (HcaReader.FindKey), and --keystring S, or else
// --keycode N, the CriAdxKey of type-8 / type-9 .adx files; there is no list of known keys.
// --devices 0,1,2,3 binds those CUDA devices (vgb_init_devices): every chunk of files is then sharded over them, one
// worker and one copy / kernel pipeline per device.  A device may be listed more than once.  The default is device 0.
#include <sys/stat.h>

#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <string>
#include <vector>

#include "../../include/vgaudio_b200.h"

namespace fs = std::filesystem;

static bool read_file(const fs::path &p, std::vector<uint8_t> &out)
{
    std::ifstream f(p, std::ios::binary | std::ios::ate);
    if (!f) return false;
    const std::streamsize n = f.tellg();
    f.seekg(0);
    out.resize((size_t)n);
    return n == 0 || (bool)f.read(reinterpret_cast<char *>(out.data()), n);
}

// the kind of an input file: 0 .dsp, 1 .hca, 2 .adx, 3 WAVE, -1 none of them
static int kind_of(const fs::path &p)
{
    std::string ext = p.extension().string();
    std::transform(ext.begin(), ext.end(), ext.begin(), ::tolower);
    return ext == ".dsp" ? 0 : ext == ".hca" ? 1 : ext == ".adx" ? 2 : (ext == ".wav" || ext == ".wave") ? 3 : -1;
}
static const int32_t kContainerOfKind[3] = {VGB_CONTAINER_DSP, VGB_CONTAINER_HCA, VGB_CONTAINER_ADX};

static int usage()
{
    std::fprintf(stderr, "usage: vgaudio_batch -i <indir> -o <outdir> --out-format dsp|adx|hca|wav [-r] [--no-trim] [--hcaquality Q] [--bitrate N]\n"
                         "                     [--limit-bitrate] [--keycode N] [--keystring S] [--in-keycode N] [--in-keystring S]\n"
                         "                     [--adxtype linear|fixed|exp] [--framesize N] [--version 3|4] [--chunk-mb N] [--devices LIST]\n");
    return 2;
}

// "0,1,3": comma-separated CUDA ordinals, at least one, repeats allowed
static bool parse_devices(const std::string &list, std::vector<int32_t> &out)
{
    out.clear();
    size_t at = 0;
    while (true) {
        const size_t end = std::min(list.find(',', at), list.size());
        const std::string item = list.substr(at, end - at);
        if (item.empty() || item.size() > 4 || item.find_first_not_of("0123456789") != std::string::npos) return false;
        out.push_back((int32_t)std::atoi(item.c_str()));
        if (end == list.size()) break;
        at = end + 1;
    }
    return out.size() <= 64;  // vgb_init_devices' limit
}

int main(int argc, char **argv)
{
    std::string in_dir, out_dir, fmt, key_string, in_key_string;
    bool recurse = false, have_code = false, have_in_code = false;
    uint64_t key_code = 0, in_key_code = 0;
    size_t chunk_mb = 1024;
    std::vector<int32_t> devices;  // empty: device 0 through vgb_init
    vgb_convert_options opt{};
    opt.hca_key_type = -1;
    for (int i = 1; i < argc; i++) {
        const std::string a = argv[i];
        auto next = [&]() -> const char * { return i + 1 < argc ? argv[++i] : ""; };
        if (a == "-i") in_dir = next();
        else if (a == "-o") out_dir = next();
        else if (a == "--out-format") fmt = next();
        else if (a == "-r") recurse = true;
        else if (a == "--no-trim") opt.no_trim = 1;
        else if (a == "--bitrate") opt.hca_bitrate = std::atoi(next());
        else if (a == "--limit-bitrate") opt.hca_limit_bitrate = 1;
        else if (a == "--keycode") { key_code = std::strtoull(next(), nullptr, 0); have_code = true; }
        else if (a == "--keystring") key_string = next();
        else if (a == "--in-keycode") { in_key_code = std::strtoull(next(), nullptr, 0); have_in_code = true; }
        else if (a == "--in-keystring") in_key_string = next();
        else if (a == "--framesize") opt.adx_frame_size = std::atoi(next());
        else if (a == "--version") opt.adx_version = std::atoi(next());
        else if (a == "--chunk-mb") chunk_mb = (size_t)std::atoll(next());
        else if (a == "--devices") { if (!parse_devices(next(), devices)) return usage(); }
        else if (a == "--hcaquality") {
            const std::string q = next();
            const char *names[] = {"", "highest", "high", "middle", "low", "lowest"};
            for (int k = 1; k <= 5; k++) if (strcasecmp(q.c_str(), names[k]) == 0) opt.hca_quality = k;
            if (!opt.hca_quality) return usage();
        } else if (a == "--adxtype") {
            const std::string t = next();
            opt.adx_type = strcasecmp(t.c_str(), "fixed") == 0 ? 2 : strcasecmp(t.c_str(), "exp") == 0 ? 4 : 3;
        } else return usage();
    }
    if (in_dir.empty() || out_dir.empty()) return usage();
    const bool to_wave = fmt == "wav";  // the decode direction: .dsp, .hca and .adx files in, 16-bit WAVE files out
    if (fmt == "dsp") opt.out_type = VGB_CONTAINER_DSP;
    else if (fmt == "adx") opt.out_type = VGB_CONTAINER_ADX;
    else if (fmt == "hca") opt.out_type = VGB_CONTAINER_HCA;
    else if (!to_wave) return usage();
    vgb_adx_key adx_key{};  // the CriAdxKey of --keystring / --keycode, for writing .adx files or reading keyed ones
    const bool have_adx_key = have_code || !key_string.empty();
    if ((opt.out_type == VGB_CONTAINER_ADX || to_wave) && have_adx_key) {
        const int32_t s = !key_string.empty() ? vgb_adx_key_from_string(key_string.c_str(), &adx_key) : vgb_adx_key_from_code(key_code, &adx_key);
        if (s != VGB_OK) { std::fprintf(stderr, "%s\n", vgb_last_error()); return 1; }
    }
    if (opt.out_type == VGB_CONTAINER_ADX && have_adx_key) {
        opt.adx_has_key = 1; opt.adx_key_seed = adx_key.seed; opt.adx_key_mult = adx_key.mult; opt.adx_key_inc = adx_key.inc;
        opt.adx_encryption_type = !key_string.empty() ? 8 : 9;  // CreateConfiguration.cs:126-135: key strings are type 8, key codes type 9
    }
    if (opt.out_type == VGB_CONTAINER_HCA && have_code) { opt.hca_key_type = 56; opt.hca_key_code = key_code; }
    // the keys of coded inputs that are transcoded: --in-keystring, or else --in-keycode, for .adx; --in-keycode for .hca
    vgb_adx_key in_adx_key{};
    const bool have_in_adx_key = !to_wave && (have_in_code || !in_key_string.empty());
    if (have_in_adx_key) {
        const int32_t s = !in_key_string.empty() ? vgb_adx_key_from_string(in_key_string.c_str(), &in_adx_key) : vgb_adx_key_from_code(in_key_code, &in_adx_key);
        if (s != VGB_OK) { std::fprintf(stderr, "%s\n", vgb_last_error()); return 1; }
    }

    // Batch.cs:16-19: the files of the input directory (here: the .dsp, .hca and .adx ones when decoding; else the WAVE
    // ones and the coded ones in another codec than the output's)
    std::vector<fs::path> files;
    std::error_code ec;
    auto take = [&](const fs::directory_entry &e) {
        if (!e.is_regular_file()) return;
        const int kind = kind_of(e.path());
        if (kind < 0) return;
        if (to_wave ? kind < 3 : (kind == 3 || kContainerOfKind[kind] != opt.out_type)) files.push_back(e.path());
    };
    if (recurse) for (auto &e : fs::recursive_directory_iterator(in_dir, ec)) take(e);
    else for (auto &e : fs::directory_iterator(in_dir, ec)) take(e);
    if (ec) { std::fprintf(stderr, "cannot read %s: %s\n", in_dir.c_str(), ec.message().c_str()); return 1; }
    std::sort(files.begin(), files.end());
    const int32_t bound = devices.empty() ? vgb_init(0, 0) : vgb_init_devices(devices.data(), (int32_t)devices.size(), 0);
    if (bound != VGB_OK) { std::fprintf(stderr, "%s\n", vgb_last_error()); return 1; }

    const auto t0 = std::chrono::steady_clock::now();
    size_t done = 0, failed = 0;
    uint64_t bytes_in = 0, bytes_out = 0;
    for (size_t first = 0; first < files.size();) {
        // a chunk of files that fits the host budget
        std::vector<std::vector<uint8_t>> in;
        size_t last = first, held = 0;
        while (last < files.size() && (last == first || held < (chunk_mb << 20))) {
            in.emplace_back();
            if (!read_file(files[last], in.back())) { std::fprintf(stderr, "Error reading %s\n", files[last].c_str()); in.back().clear(); }
            held += in.back().size();
            last++;
        }
        const int n = (int)(last - first);
        std::vector<const uint8_t *> ptr(n);
        std::vector<int64_t> len(n), out_size(n);
        std::vector<int32_t> status(n);
        for (int k = 0; k < n; k++) { ptr[k] = in[k].data(); len[k] = (int64_t)in[k].size(); bytes_in += in[k].size(); }
        // every kind of input goes to its own call, each on its rows of the chunk's tables: decoding, one converter per
        // codec; encoding, the WAVE converter for WAVE files and one transcode call for the coded ones
        std::vector<int32_t> rows[4];
        for (int k = 0; k < n; k++) {
            const int kind = kind_of(files[first + k]);
            rows[to_wave ? kind : (kind == 3 ? 3 : 0)].push_back(k);
        }
        auto convert = [&](uint8_t *const *outs) -> int32_t {
            for (int h = 0; h < 4; h++) {
                const std::vector<int32_t> &r = rows[h];
                if (r.empty()) continue;
                std::vector<const uint8_t *> p;
                std::vector<int64_t> l, sz(r.size());
                std::vector<uint8_t *> o;
                std::vector<int32_t> st(r.size()), types;
                for (int32_t k : r) {
                    p.push_back(ptr[k]); l.push_back(len[k]); o.push_back(outs ? outs[k] : nullptr);
                    const int kind = kind_of(files[first + k]);
                    if (kind < 3) types.push_back(kContainerOfKind[kind]);
                }
                const int32_t m = (int32_t)r.size();
                uint8_t *const *ot = outs ? o.data() : nullptr;
                int32_t s;
                if (h == 3) s = vgb_convert_wave_batch(p.data(), l.data(), m, &opt, sz.data(), ot, st.data(), nullptr, nullptr);
                else if (!to_wave) s = vgb_transcode_batch(p.data(), l.data(), types.data(), m, &opt, have_in_adx_key ? &in_adx_key : nullptr,
                                                           have_in_code ? &in_key_code : nullptr, sz.data(), ot, st.data(), nullptr, nullptr);
                else s = h == 2 ? vgb_convert_adx_to_wave_batch(p.data(), l.data(), m, have_adx_key ? &adx_key : nullptr, sz.data(), ot, st.data())
                       : h == 1 ? vgb_convert_hca_to_wave_batch(p.data(), l.data(), m, have_code ? &key_code : nullptr, sz.data(), ot, st.data())
                                : vgb_convert_dsp_to_wave_batch(p.data(), l.data(), m, sz.data(), ot, st.data());
                if (s != VGB_OK) return s;
                for (int32_t j = 0; j < m; j++) { out_size[r[j]] = sz[j]; status[r[j]] = st[j]; }
            }
            return VGB_OK;
        };
        if (convert(nullptr) != VGB_OK) {
            std::fprintf(stderr, "%s\n", vgb_last_error());
            return 1;
        }
        std::vector<std::vector<uint8_t>> out(n);
        std::vector<uint8_t *> optr(n, nullptr);
        for (int k = 0; k < n; k++) if (status[k] == VGB_OK) { out[k].resize((size_t)out_size[k]); optr[k] = out[k].data(); }
        if (convert(optr.data()) != VGB_OK) {
            std::fprintf(stderr, "%s\n", vgb_last_error());
            return 1;
        }
        for (int k = 0; k < n; k++) {
            const fs::path &src = files[first + k];
            if (status[k] != VGB_OK) { std::fprintf(stderr, "Error converting %s\n", src.filename().c_str()); failed++; continue; }
            fs::path rel = fs::relative(src, in_dir, ec);
            fs::path dst = fs::path(out_dir) / rel;
            dst.replace_extension(fmt);                         // Path.ChangeExtension (Batch.cs:29)
            fs::create_directories(dst.parent_path(), ec);
            std::ofstream f(dst, std::ios::binary);
            f.write(reinterpret_cast<const char *>(out[k].data()), (std::streamsize)out[k].size());
            bytes_out += out[k].size();
            done++;
        }
        first = last;
    }
    const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    std::printf("%zu files converted, %zu failed, %.1f MB in, %.1f MB out, %.3f s\n", done, failed, bytes_in / 1e6, bytes_out / 1e6, s);
    vgb_shutdown();
    return failed ? 3 : 0;
}
