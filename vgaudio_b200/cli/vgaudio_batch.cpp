// vgaudio_batch — batch conversion of a directory of audio files on the GPU: WAVE, .dsp, .adx and .hca files to
// .dsp / .adx / .hca, WAVE files (with --coded also .adx, .hca and .dsp files) to .brstm / .bcstm / .bfstm / .idsp / .hps, and .dsp, .adx, .hca, .brstm, .bcstm, .bfstm,
// .idsp and .hps files, the NintendoWare wave files (.brwav / .rwav, .bcwav / .cwav / .bms, .bfwav) and prefetch
// streams (.bcstp, .bfstp) to WAVE; with --nw-inputs also the NintendoWare, IDSP and HPS files to any other codec.
//
// The counterpart of `VGAudioCli -b` (src/VGAudio.Cli/Batch.cs:11-51): the reference enumerates the input files and runs
// Convert.ConvertFile on each from a Parallel.ForEach; here the host only reads and writes files, and every
// reader -> encoder -> writer chain of a chunk of files runs as ONE coalesced call on the device per kind of input
// (vgb_convert_wave_batch for WAVE files, vgb_transcode_batch / vgb_transcode_nw_batch / vgb_transcode_from_nw_batch for coded files, vgb_convert_*_to_wave_batch for
// --out-format wav).  A file that fails is reported and skipped, like the reference's try/catch (:39-43).
//
//   vgaudio_batch -i <indir> -o <outdir> --out-format dsp|adx|hca|brstm|bcstm|bfstm|idsp|hps|wav [-r]   (wav: .dsp, .hca, .adx, .brstm, .bcstm, .bfstm, .idsp, .hps, .brwav, .rwav, .bcwav, .cwav, .bms, .bfwav, .bcstp and .bfstp inputs are decoded) [--no-trim] [--hcaquality Highest|High|Middle|Low|Lowest]
//                 [--bitrate N] [--limit-bitrate] [--keycode N] [--keystring S] [--in-keycode N] [--in-keystring S]
//                 [--adxtype Linear|Fixed|Exp|ExpEnc...] [--framesize N] [--version 3|4] [--chunk-mb N] [--devices LIST] [--rewrite]
//                 [-l <start>-<end> | --no-loop] [--loop-align N] [--coded] [--nw-inputs] [--keep-codec]
//
// -l <start>-<end> sets the loop of every file, --no-loop removes it (AudioData.SetLoop on each file as read, before any
// encode or write, Convert.cs:82-90), in every direction: WAVE to any target, transcodes, --rewrite and --out-format wav
// (vgb_convert_to_wave_batch).  A file whose format refuses the points fails alone with the reference's message: points
// outside 0..sample count or an end below the start, and for .hca sources any points but the file's own or a loop the file
// does not have (no re-encode can add one).  The key searches ignore them.  --loop-align N sets the loop point alignment
// of the NintendoWare targets and, when N > 0, of .dsp output (CreateConfiguration.Dsp).
// With --out-format dsp|adx|hca the inputs are the .wav / .wave files and the .dsp, .adx and .hca files in another codec
// than the output's (a file already in the output's codec is not listed: the same codec would be a rewrite).
// --rewrite, with --out-format adx|hca only, also lists the .adx (respectively .hca) inputs and rewrites them in their own
// codec without re-encoding (vgb_rewrite_batch): decrypted with their input key and written in the clear, or re-keyed
// with the output key; the encoder's options do not apply to them.
// --coded, with --out-format brstm|bcstm|bfstm|idsp|hps only, also lists the .adx and .hca inputs, and with -f pcm16|pcm8
// into brstm|bcstm|bfstm the .dsp inputs, and transcodes them on the device (vgb_transcode_nw_batch) with the same input
// keys as the other transcodes.  Without it those targets take WAVE inputs only.  (A .dsp file into GC-ADPCM would be a
// rewrite in its own codec, which is not performed.)
// --nw-inputs, with any --out-format but wav, also lists the NintendoWare inputs (.brstm, .bcstm, .bfstm, .brwav, .rwav,
// .bcwav, .cwav, .bms, .bfwav, .bcstp, .bfstp), and the .idsp and .hps inputs when the output is not GC-ADPCM (adx, hca,
// or brstm|bcstm|bfstm with -f pcm16|pcm8), and transcodes them on the device (vgb_transcode_from_nw_batch).  A file
// already in the output's codec (a GC-ADPCM stream into dsp, idsp, hps or GC-ADPCM NintendoWare, a PCM16 one into
// -f pcm16, a PCM8 one into -f pcm8) is a rewrite, which is not performed: it is reported as a failed file.
// --keep-codec, with --out-format brstm|bcstm|bfstm|idsp|hps into GC-ADPCM only, also lists the .dsp inputs and rewrites
// them into the output's container without re-encoding (vgb_rewrite_gc_batch): the source's ADPCM is copied, only a loop
// tail that the target's alignment moves is re-encoded.
// --keycode / --keystring are the output's key; --in-keycode N is the key of type-56 .hca inputs, and --in-keystring S,
// or else --in-keycode N, the CriAdxKey of type-8 / type-9 .adx inputs.
// With --out-format wav, --keycode N is the key of type-56 .hca files (HcaReader.FindKey), and --keystring S, or else
// --keycode N, the CriAdxKey of type-8 / type-9 .adx files.  There is no list of known keys; instead
// --find-adx-key, when no key option names the .adx inputs' key (--keystring / --keycode with wav, --in-keystring /
// --in-keycode otherwise), recovers it from the files first (vgb_adx_find_keys, GuessAdx): for each of revisions 8 and 9,
// over that revision's .adx inputs, every key is printed as GuessAdx prints it and the files are decoded with the one of
// highest full confidence (then short confidence, then the lowest key).  Without a key found they fail as without a key.
// --hca-keys FILE, when no key option names the type-56 .hca inputs' key (--keycode with wav, --in-keycode otherwise: a
// given key wins untested, as HcaReader's EncryptionKey ?? FindKey does), is a list of key codes, one per line, decimal or
// 0x hex; blank lines and lines starting with # are skipped.  Per chunk of files the type-56 .hca files are searched
// (vgb_hca_find_keys, HcaReader.FindKey over the list in order) and converted with one call per key found; each key is
// printed with its number of files.  A file no listed key decrypts fails as without a key.
// --devices 0,1,2,3 binds those CUDA devices (vgb_init_devices): every chunk of files is then sharded over them, one
// worker and one copy / kernel pipeline per device.  A device may be listed more than once.  The default is device 0.
#include <sys/stat.h>

#include <algorithm>
#include <chrono>
#include <cerrno>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <map>
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

// the kind of an input file: 0 .dsp, 1 .hca, 2 .adx, 3 WAVE, 4 .brstm, 5 .bcstm, 6 .bfstm, 7 .idsp, 8 .hps, 9 .brwav /
// .rwav, 10 .bcwav / .cwav / .bms, 11 .bfwav, 12 .bcstp, 13 .bfstp, -1 none of them (from 4 on, the kind is the
// VGB_CONTAINER_* of its reader).  The extension picks the reader, as in the reference (src/VGAudio.Cli/ContainerTypes.cs).
// The NintendoWare, IDSP and HPS streams are decoded to WAVE with --out-format wav, and written from WAVE inputs (with
// --coded also from .adx, .hca and PCM-bound .dsp inputs) with --out-format brstm|bcstm|bfstm|idsp|hps; the wave and
// prefetch files are decoded to WAVE.  With --nw-inputs every coded --out-format also takes them as inputs.
static int kind_of(const fs::path &p)
{
    std::string ext = p.extension().string();
    std::transform(ext.begin(), ext.end(), ext.begin(), ::tolower);
    return ext == ".dsp" ? 0 : ext == ".hca" ? 1 : ext == ".adx" ? 2 : (ext == ".wav" || ext == ".wave") ? 3
         : ext == ".brstm" ? 4 : ext == ".bcstm" ? 5 : ext == ".bfstm" ? 6 : ext == ".idsp" ? 7 : ext == ".hps" ? 8
         : (ext == ".brwav" || ext == ".rwav") ? 9 : (ext == ".bcwav" || ext == ".cwav" || ext == ".bms") ? 10
         : ext == ".bfwav" ? 11 : ext == ".bcstp" ? 12 : ext == ".bfstp" ? 13 : -1;
}
static_assert(VGB_CONTAINER_BRSTM == 4 && VGB_CONTAINER_HPS == 8 && VGB_CONTAINER_BRWAV == 9 && VGB_CONTAINER_BFSTP == 13,
              "kinds 4..13 are their readers' container types");
static const int32_t kContainerOfKind[3] = {VGB_CONTAINER_DSP, VGB_CONTAINER_HCA, VGB_CONTAINER_ADX};

static int usage()
{
    std::fprintf(stderr, "usage: vgaudio_batch -i <indir> -o <outdir> --out-format dsp|adx|hca|brstm|bcstm|bfstm|idsp|hps|wav [-r] [--no-trim] [--hcaquality Q] [--bitrate N]\n"
                         "                     [--limit-bitrate] [--keycode N] [--keystring S] [--in-keycode N] [--in-keystring S] [--rewrite]\n"
                         "                     [--adxtype linear|fixed|exp] [--framesize N] [--version 3|4] [--chunk-mb N] [--devices LIST]\n"
                         "                     [-f gcadpcm|pcm16|pcm8] [--loop-align N] [--little-endian|--big-endian] [--find-adx-key] [--hca-keys FILE]\n"
                         "                     [-l <start-end>] [--no-loop] [--coded] [--nw-inputs] [--keep-codec]\n"
                         "       -l <start-end>   Set the start and end loop points (zero-indexed samples) of every file\n"
                         "       --no-loop        Sets the audio to not loop\n"
                         "       wav decodes .dsp, .hca, .adx, .brstm, .bcstm, .bfstm, .idsp, .hps, .brwav, .rwav, .bcwav, .cwav, .bms,\n"
                         "       .bfwav, .bcstp and .bfstp inputs\n"
                         "       --nw-inputs      Also transcode the .brstm, .bcstm, .bfstm, .brwav, .rwav, .bcwav, .cwav, .bms, .bfwav,\n"
                         "                        .bcstp, .bfstp (and, into a codec other than GC-ADPCM, .idsp and .hps) inputs\n"
                         "       --keep-codec     Also rewrite the .dsp inputs into brstm, bcstm, bfstm, idsp or hps without re-encoding\n");
    return 2;
}

// the reference's messages for a bad command line (CliArguments.cs: PrintWithUsage)
static int usage(const char *why)
{
    std::fprintf(stderr, "%s\n", why);
    return usage();
}

// int.TryParse with the default NumberStyles.Integer: white space around an optional sign and decimal digits, in range
static bool parse_int(const std::string &t, int32_t &out)
{
    const char *ws = " \t\n\v\f\r";
    const size_t a = t.find_first_not_of(ws), b = t.find_last_not_of(ws);
    if (a == std::string::npos) return false;
    std::string d = t.substr(a, b - a + 1);
    bool neg = false;
    if (d[0] == '+' || d[0] == '-') { neg = d[0] == '-'; d.erase(0, 1); }
    if (d.empty() || d.find_first_not_of("0123456789") != std::string::npos) return false;
    int64_t v = 0;
    for (char c : d) {
        v = v * 10 + (c - '0');
        if (v > (int64_t)INT32_MAX + 1) return false;
    }
    if (neg) v = -v;
    if (v < INT32_MIN || v > INT32_MAX) return false;
    out = (int32_t)v;
    return true;
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

// the revision of an .adx image (0 when its header cannot be read)
// --hca-keys: one key code per line, decimal or 0x hex; blank lines and lines starting with # are skipped
static bool read_hca_keys(const std::string &path, std::vector<uint64_t> &codes)
{
    std::ifstream f(path);
    if (!f) { std::fprintf(stderr, "cannot read %s\n", path.c_str()); return false; }
    std::string line;
    for (int n = 1; std::getline(f, line); n++) {
        const size_t a = line.find_first_not_of(" \t\r"), b = line.find_last_not_of(" \t\r");
        if (a == std::string::npos || line[a] == '#') continue;
        const std::string t = line.substr(a, b - a + 1);
        const bool hex = t.size() > 2 && t[0] == '0' && (t[1] == 'x' || t[1] == 'X');
        const size_t digits = hex ? t.find_first_not_of("0123456789abcdefABCDEF", 2) : t.find_first_not_of("0123456789");
        errno = 0;
        char *end = nullptr;
        const unsigned long long v = std::strtoull(t.c_str(), &end, hex ? 16 : 10);
        if (digits != std::string::npos || errno == ERANGE || t[0] == '-' || *end) {
            std::fprintf(stderr, "%s:%d: not a key code: %s\n", path.c_str(), n, t.c_str());
            return false;
        }
        codes.push_back((uint64_t)v);
    }
    return true;
}

static int adx_revision(const std::vector<uint8_t> &img)
{
    int32_t rev = 0, n = 0, start = 0;
    return vgb_adx_key_load(img.data(), (int64_t)img.size(), &rev, nullptr, 0, &n, &start) == VGB_OK ? rev : 0;
}

// GuessAdx over the .adx inputs of one revision: prints every key as AddKey does (GuessAdx.cs:146-155) and picks the
// one of highest full confidence, then short confidence, then the lowest (the keys come sorted)
static bool find_adx_key(const std::vector<fs::path> &paths, int revision, vgb_adx_key &out)
{
    std::vector<std::vector<uint8_t>> imgs;
    for (const fs::path &p : paths) {
        std::vector<uint8_t> img;
        if (read_file(p, img) && adx_revision(img) == revision) imgs.push_back(std::move(img));
    }
    if (imgs.empty()) return false;
    std::vector<const uint8_t *> ptr;
    std::vector<int64_t> len;
    for (const auto &img : imgs) { ptr.push_back(img.data()); len.push_back((int64_t)img.size()); }
    std::vector<vgb_adx_found_key> keys(256);
    int32_t n = 0;
    if (vgb_adx_find_keys(ptr.data(), len.data(), (int32_t)imgs.size(), keys.data(), (int32_t)keys.size(), &n, nullptr, nullptr) != VGB_OK) {
        std::fprintf(stderr, "ADX key search (revision %d): %s\n", revision, vgb_last_error());
        return false;
    }
    const vgb_adx_found_key *best = nullptr;
    for (int i = 0; i < n; i++) {
        const vgb_adx_found_key &k = keys[(size_t)i];
        std::printf("----------------------------------------\nSeed - %04x Multiplier - %04x Increment - %04x\n", k.key.seed, k.key.mult, k.key.inc);
        std::printf("Confidence Short - %.3f %% Full - %.3f %%\n", 100.0 * k.confidence_short, 100.0 * k.confidence_full);
        if (revision == 9) std::printf("Key code: %llu\n", (unsigned long long)k.key_code);
        std::printf("----------------------------------------\n");
        if (k.status != VGB_OK) continue;
        if (!best || k.confidence_full > best->confidence_full ||
            (k.confidence_full == best->confidence_full && k.confidence_short > best->confidence_short)) best = &k;
    }
    if (best) out = best->key;
    return best != nullptr;
}

int main(int argc, char **argv)
{
    std::string in_dir, out_dir, fmt, key_string, in_key_string, hca_keys_path;
    bool recurse = false, have_code = false, have_in_code = false, find_key = false, rewrite = false, coded = false, nw_inputs = false,
         keep_codec = false;
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
        else if (a == "--loop-align") opt.nw_loop_point_alignment = std::atoi(next());
        else if (a == "-l") {  // CliArguments.cs:95-124
            if (opt.loop_mode == VGB_LOOP_CLEAR) return usage("Can't set loop points while using --no-loop.");
            if (i + 1 >= argc) return usage("No argument after -l switch.");
            const std::string arg = argv[++i];
            const size_t dash = arg.find('-');
            if (dash == std::string::npos || arg.find('-', dash + 1) != std::string::npos)
                return usage("-l switch requires two loop points in the format <start>-<end>.");
            if (!parse_int(arg.substr(0, dash), opt.loop_start) || !parse_int(arg.substr(dash + 1), opt.loop_end))
                return usage("Error parsing loop points.");
            opt.loop_mode = VGB_LOOP_SET;
        } else if (a == "--no-loop") {  // :125-134
            if (opt.loop_mode == VGB_LOOP_SET) return usage("Can't set loop points while using --no-loop.");
            opt.loop_mode = VGB_LOOP_CLEAR;
        }
        else if (a == "--find-adx-key") find_key = true;
        else if (a == "--rewrite") rewrite = true;
        else if (a == "--coded") coded = true;
        else if (a == "--nw-inputs") nw_inputs = true;
        else if (a == "--keep-codec") keep_codec = true;
        else if (a == "--hca-keys") hca_keys_path = next();
        else if (a == "--little-endian") opt.nw_endianness = 1;
        else if (a == "--big-endian") opt.nw_endianness = 2;
        else if (a == "-f") {  // NwCodec + 1
            const std::string c = next();
            opt.nw_codec_plus1 = strcasecmp(c.c_str(), "pcm8") == 0 ? 1 : strcasecmp(c.c_str(), "pcm16") == 0 ? 2 : strcasecmp(c.c_str(), "gcadpcm") == 0 ? 3 : 0;
            if (!opt.nw_codec_plus1) return usage();
        }
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
    else if (fmt == "brstm") opt.out_type = VGB_CONTAINER_BRSTM;
    else if (fmt == "bcstm") opt.out_type = VGB_CONTAINER_BCSTM;
    else if (fmt == "bfstm") opt.out_type = VGB_CONTAINER_BFSTM;
    else if (fmt == "idsp") opt.out_type = VGB_CONTAINER_IDSP;
    else if (fmt == "hps") opt.out_type = VGB_CONTAINER_HPS;
    else if (fmt == "hca") opt.out_type = VGB_CONTAINER_HCA;
    else if (!to_wave) return usage();
    // CreateConfiguration.Dsp (src/VGAudio.Cli/CreateConfiguration.cs:49-52): a positive --loop-align aligns .dsp loops too
    if (opt.out_type == VGB_CONTAINER_DSP && opt.nw_loop_point_alignment > 0) opt.dsp_loop_point_alignment = opt.nw_loop_point_alignment;
    if (rewrite && opt.out_type != VGB_CONTAINER_ADX && opt.out_type != VGB_CONTAINER_HCA) {
        std::fprintf(stderr, "--rewrite takes --out-format adx or hca\n");
        return 2;
    }
    const bool nw_out = opt.out_type >= VGB_CONTAINER_BRSTM;  // NintendoWare, IDSP and HPS targets
    if (coded && !nw_out) {
        std::fprintf(stderr, "--coded takes --out-format brstm, bcstm, bfstm, idsp or hps\n");
        return 2;
    }
    if (nw_inputs && to_wave) {
        std::fprintf(stderr, "--nw-inputs takes --out-format dsp, adx, hca, brstm, bcstm, bfstm, idsp or hps\n");
        return 2;
    }
    if ((opt.out_type == VGB_CONTAINER_IDSP || opt.out_type == VGB_CONTAINER_HPS) && (opt.nw_codec_plus1 == 1 || opt.nw_codec_plus1 == 2)) {
        // CreateConfiguration.Idsp / .Hps (src/VGAudio.Cli/CreateConfiguration.cs:57-75, 103-115): GC-ADPCM only
        std::fprintf(stderr, "Can't use format %s with %s files\n", opt.nw_codec_plus1 == 2 ? "PCM16" : "PCM8",
                     opt.out_type == VGB_CONTAINER_IDSP ? "IDSP" : "HPS");
        return 1;
    }
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
    // --hca-keys: the list is searched only when no key option names the .hca inputs' key
    std::vector<uint64_t> hca_codes;
    if (!hca_keys_path.empty() && !read_hca_keys(hca_keys_path, hca_codes)) return 1;
    const bool search_hca = !hca_keys_path.empty() && !(to_wave ? have_code : have_in_code) && (to_wave || opt.out_type != VGB_CONTAINER_HCA || rewrite);
    std::map<int32_t, size_t> hca_key_files;  // key index -> files it decrypted

    // Batch.cs:16-19: the files of the input directory (here: the .dsp, .hca, .adx, NintendoWare, IDSP and HPS ones when decoding; else the WAVE
    // ones and the coded ones in another codec than the output's, and with --rewrite those in the output's codec too;
    // the NintendoWare, IDSP and HPS targets take WAVE inputs, and with --coded .adx and .hca ones, and .dsp ones into PCM;
    // with --nw-inputs every target also takes the NintendoWare inputs, and the IDSP and HPS ones into another codec than
    // GC-ADPCM, the only codec they hold)
    const bool nw_pcm = opt.out_type <= VGB_CONTAINER_BFSTM && (opt.nw_codec_plus1 == 1 || opt.nw_codec_plus1 == 2);
    const bool gc_out = opt.out_type == VGB_CONTAINER_DSP || opt.out_type >= VGB_CONTAINER_IDSP || (nw_out && !nw_pcm);
    if (keep_codec && (!nw_out || nw_pcm)) {
        std::fprintf(stderr, "--keep-codec takes --out-format brstm, bcstm, bfstm, idsp or hps in GC-ADPCM\n");
        return 2;
    }
    std::vector<fs::path> files;
    std::error_code ec;
    auto take = [&](const fs::directory_entry &e) {
        if (!e.is_regular_file()) return;
        const int kind = kind_of(e.path());
        if (kind < 0) return;
        const bool coded_in = kind < 3 && (nw_out ? (coded && (kind != 0 || nw_pcm)) || (keep_codec && kind == 0)
                                                  : rewrite || kContainerOfKind[kind] != opt.out_type);
        const bool nw_in = nw_inputs && kind > 3 && ((kind != VGB_CONTAINER_IDSP && kind != VGB_CONTAINER_HPS) || !gc_out);
        if (to_wave ? kind != 3 : (kind == 3 || coded_in || nw_in)) files.push_back(e.path());
    };
    if (recurse) for (auto &e : fs::recursive_directory_iterator(in_dir, ec)) take(e);
    else for (auto &e : fs::directory_iterator(in_dir, ec)) take(e);
    if (ec) { std::fprintf(stderr, "cannot read %s: %s\n", in_dir.c_str(), ec.message().c_str()); return 1; }
    std::sort(files.begin(), files.end());
    const int32_t bound = devices.empty() ? vgb_init(0, 0) : vgb_init_devices(devices.data(), (int32_t)devices.size(), 0);
    if (bound != VGB_OK) { std::fprintf(stderr, "%s\n", vgb_last_error()); return 1; }

    // --find-adx-key: the keys of the keyed .adx inputs, per revision, when no key option gives them
    const bool adx_key_given = to_wave ? have_adx_key : have_in_adx_key;
    vgb_adx_key found[2]{};
    bool have_found[2] = {false, false};
    if (find_key && !adx_key_given && (to_wave || opt.out_type != VGB_CONTAINER_ADX || rewrite)) {
        std::vector<fs::path> adx;
        for (const fs::path &p : files) if (kind_of(p) == 2) adx.push_back(p);
        for (int r = 0; r < 2; r++) have_found[r] = find_adx_key(adx, 8 + r, found[r]);
    }

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
        // codec (one for every NintendoWare reader, one for IDSP and HPS); encoding, the WAVE converter for WAVE files
        // and one transcode call for the coded ones (vgb_transcode_nw_batch for the NintendoWare, IDSP and HPS targets; with
        // --rewrite, one rewrite call for those in the output's codec), and row 4 for the NintendoWare, IDSP and HPS inputs
        // (vgb_transcode_from_nw_batch)
        // rows 6 and 7: .adx files of revision 8 / 9 whose key --find-adx-key found, each revision with its own key
        // rows 8 and up: type-56 .hca files whose key --hca-keys found, one row per key (hca_row_key)
        std::vector<int32_t> hca_index(n, -1);
        if (search_hca) {
            std::vector<int32_t> hk;
            for (int k = 0; k < n; k++) if (kind_of(files[first + k]) == 1) hk.push_back(k);
            std::vector<const uint8_t *> hp;
            std::vector<int64_t> hl;
            for (int32_t k : hk) { hp.push_back(ptr[k]); hl.push_back(len[k]); }
            std::vector<int32_t> idx(hk.size()), st(hk.size());
            if (!hk.empty() && vgb_hca_find_keys(hp.data(), hl.data(), (int32_t)hk.size(), hca_codes.data(), (int32_t)hca_codes.size(), idx.data(), st.data()) != VGB_OK) {
                std::fprintf(stderr, "%s\n", vgb_last_error());
                return 1;
            }
            for (size_t j = 0; j < hk.size(); j++) if (st[j] == VGB_OK) hca_index[hk[j]] = idx[j];
        }
        std::vector<std::vector<int32_t>> rows(8);
        std::vector<int32_t> hca_row_key(8, -1);
        for (int k = 0; k < n; k++) {
            const int kind = kind_of(files[first + k]);
            const int rev = kind == 2 && (have_found[0] || have_found[1]) ? adx_revision(in[k]) : 0;
            if (hca_index[k] >= 0) {
                const size_t row = std::find(hca_row_key.begin(), hca_row_key.end(), hca_index[k]) - hca_row_key.begin();
                if (row == rows.size()) { rows.emplace_back(); hca_row_key.push_back(hca_index[k]); }
                rows[row].push_back(k);
                hca_key_files[hca_index[k]]++;
            } else if ((rev == 8 || rev == 9) && have_found[rev - 8]) rows[rev - 2].push_back(k);
            else rows[to_wave ? ((kind == 7 || kind == 8) ? 5 : std::min(kind, 4)) : kind > 3 ? 4 : (kind == 3 ? 3 : 0)].push_back(k);
        }
        auto convert = [&](uint8_t *const *outs) -> int32_t {
            for (int part = 0; part < (int)rows.size() * 2; part++) {
                // every row splits into the files in another codec than the output's (part even) and, transcoding, the
                // ones in the output's own codec (part odd), which only --rewrite (.adx, .hca) and --keep-codec (.dsp) list
                const int h = part / 2;
                std::vector<int32_t> r;
                for (int32_t k : rows[h]) {
                    const int kind = kind_of(files[first + k]);
                    const bool same = !to_wave && h != 3 && kind < 3 && (kContainerOfKind[kind] == opt.out_type || (keep_codec && kind == 0));
                    if (same == (part % 2 == 1)) r.push_back(k);
                }
                if (r.empty()) continue;
                std::vector<const uint8_t *> p;
                std::vector<int64_t> l, sz(r.size());
                std::vector<uint8_t *> o;
                std::vector<int32_t> st(r.size()), types;
                for (int32_t k : r) {
                    p.push_back(ptr[k]); l.push_back(len[k]); o.push_back(outs ? outs[k] : nullptr);
                    const int kind = kind_of(files[first + k]);
                    if (kind < 3) types.push_back(kContainerOfKind[kind]);
                    else if (kind > 3) types.push_back(kind);  // BRSTM .. BFSTM, IDSP, HPS, BRWAV .. BFSTP
                }
                const int32_t m = (int32_t)r.size();
                uint8_t *const *ot = outs ? o.data() : nullptr;
                int32_t s;
                const bool adx_found = h == 6 || h == 7;
                const vgb_adx_key *wave_adx_key = adx_found ? &found[h - 6] : have_adx_key ? &adx_key : nullptr;
                const vgb_adx_key *tx_adx_key = adx_found ? &found[h - 6] : have_in_adx_key ? &in_adx_key : nullptr;
                const uint64_t *hca_found = h >= 8 ? &hca_codes[(size_t)hca_row_key[h]] : nullptr;
                const uint64_t *tx_hca_key = hca_found ? hca_found : have_in_code ? &in_key_code : nullptr;
                if (part % 2 && keep_codec) s = vgb_rewrite_gc_batch(p.data(), l.data(), types.data(), m, &opt, sz.data(), ot, st.data());
                else if (part % 2) s = vgb_rewrite_batch(p.data(), l.data(), m, &opt, tx_adx_key, tx_hca_key, sz.data(), ot, st.data(), nullptr, nullptr);
                else if (to_wave) {  // one reader per row; only the loop fields of opt are read
                    const uint64_t *wave_hca_key = hca_found ? hca_found : have_code ? &key_code : nullptr;
                    s = vgb_convert_to_wave_batch(p.data(), l.data(), types.data(), m, &opt, wave_adx_key, wave_hca_key, sz.data(), ot, st.data());
                } else if (h == 3) s = vgb_convert_wave_batch(p.data(), l.data(), m, &opt, sz.data(), ot, st.data(), nullptr, nullptr);
                else if (h == 4) s = vgb_transcode_from_nw_batch(p.data(), l.data(), types.data(), m, &opt, sz.data(), ot, st.data(), nullptr, nullptr);
                else s = (nw_out ? vgb_transcode_nw_batch : vgb_transcode_batch)(p.data(), l.data(), types.data(), m, &opt, tx_adx_key,
                                                                               tx_hca_key, sz.data(), ot, st.data(), nullptr, nullptr);
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
    for (const auto &kv : hca_key_files)
        std::printf("HCA key %llu (0x%016llX, list entry %d): %zu files\n", (unsigned long long)hca_codes[(size_t)kv.first],
                    (unsigned long long)hca_codes[(size_t)kv.first], kv.first, kv.second);
    std::printf("%zu files converted, %zu failed, %.1f MB in, %.1f MB out, %.3f s\n", done, failed, bytes_in / 1e6, bytes_out / 1e6, s);
    vgb_shutdown();
    return failed ? 3 : 0;
}
