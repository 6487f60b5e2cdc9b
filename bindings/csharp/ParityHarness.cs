// bindings/csharp/ParityHarness.cs — closes the "parity unpinned" gap of DESIGN.md §3 on a machine that has .NET.
//
// Two modes, both against the UNMODIFIED managed VGAudio (reference src/VGAudio/VGAudio.csproj):
//   ParityHarness live            encodes / decodes the built-in inputs with the managed code AND with libvgaudio_b200.so
//                                 (needs a CUDA device) and compares byte for byte - GC-ADPCM, CRI ADX (all types, versions,
//                                 padding), CRI HCA (qualities, 1..8 channels, looping), GC-ADPCM loop alignment.  Modelled on the reference's own
//                                 differential tool (src/VGAudio.Tools/GcAdpcm/Encode.cs:44-150).
//   ParityHarness vectors <dir>   no GPU, no native library: reads the vector files tools/dump_vectors.py wrote on the GPU
//                                 box (inputs + this repository's outputs), re-encodes every input with the managed
//                                 code only and diffs.  This is the cheap way to turn "unpinned" into "pinned".
// File format of <dir>/manifest.tsv (one case per line, tab separated):
//   codec  name  params(key=value,...)  input files(comma separated, one per channel, raw little-endian int16)  output file
// Build: console project referencing src/VGAudio/VGAudio.csproj, plus bindings/csharp/*.cs for `live`.  NOT compiled here.
using System;
using System.Collections.Generic;
using System.IO;
using System.Linq;
using VGAudio.Codecs.CriAdx;
using VGAudio.Codecs.CriHca;
using VGAudio.Codecs.GcAdpcm;
using VGAudio.Formats;
using VGAudio.Formats.CriHca;
using VGAudio.Formats.GcAdpcm;
using VGAudio.Formats.Pcm16;
using VGAudio.Native;

internal static unsafe class ParityHarness
{
    private static short[] Sine(int n, double f, int rate) =>
        Enumerable.Range(0, n).Select(i => (short)(short.MaxValue * Math.Sin(2 * Math.PI * f / rate * i))).ToArray();

    private static short[] ReadPcm(string path)
    {
        byte[] raw = File.ReadAllBytes(path);
        var pcm = new short[raw.Length / 2];
        Buffer.BlockCopy(raw, 0, pcm, 0, pcm.Length * 2);
        return pcm;
    }

    private static Dictionary<string, string> Params(string s) =>
        s.Split(new[] { ',' }, StringSplitOptions.RemoveEmptyEntries).Select(kv => kv.Split('=')).ToDictionary(kv => kv[0], kv => kv[1]);

    private static bool Report(string name, byte[] managed, byte[] ours)
    {
        bool same = managed.SequenceEqual(ours);
        int first = same ? -1 : Enumerable.Range(0, Math.Min(managed.Length, ours.Length)).FirstOrDefault(i => managed[i] != ours[i]);
        Console.WriteLine($"{name,-48} {(same ? "identical" : $"DIFFERENT (lengths {managed.Length}/{ours.Length}, first at {first})")}");
        return same;
    }

    // ---- managed reference paths -------------------------------------------------------------------------------------
    private static byte[] ManagedGc(short[] pcm, out short[] coefs)
    {
        coefs = GcAdpcmCoefficients.CalculateCoefficients(pcm);                       // GcAdpcmCoefficients.cs:9
        return GcAdpcmEncoder.Encode(pcm, coefs);                                      // GcAdpcmEncoder.cs:14
    }

    private static byte[] ManagedAdx(short[] pcm, Dictionary<string, string> p) =>
        CriAdxCodec.Encode(pcm, new CriAdxParameters                                   // CriAdxCodec.cs:56
        {
            SampleRate = int.Parse(p["sample_rate"]), FrameSize = int.Parse(p["frame_size"]), Version = int.Parse(p["version"]),
            Padding = int.Parse(p["padding"]), Type = (CriAdxType)int.Parse(p["type"]), Filter = int.Parse(p["filter"])
        });

    private static byte[] ManagedHca(short[][] pcm, Dictionary<string, string> p)
    {
        var cfg = new CriHcaParameters
        {
            Quality = (CriHcaQuality)int.Parse(p["quality"]), Bitrate = int.Parse(p["bitrate"]), LimitBitrate = p["limit_bitrate"] == "1",
            ChannelCount = pcm.Length, SampleRate = int.Parse(p["sample_rate"]), SampleCount = pcm[0].Length,
            Looping = p["looping"] == "1", LoopStart = int.Parse(p["loop_start"]), LoopEnd = int.Parse(p["loop_end"])
        };
        var format = new Pcm16Format(pcm, cfg.SampleRate);
        if (cfg.Looping) format = format.WithLoop(true, cfg.LoopStart, cfg.LoopEnd);
        CriHcaFormat hca = new CriHcaFormat().EncodeFromPcm16(format, cfg);            // CriHcaFormat.cs:34-84
        return hca.AudioData.SelectMany(f => f).ToArray();
    }

    // ---- the same calls through the C ABI (one channel / one stream per call; the drop-in bodies batch them) ---------------
    private static byte[] NativeAdx(short[] pcm, CriAdxParameters cfg)
    {
        var prm = new VgbAdxParams { SampleRate = cfg.SampleRate, HighpassFrequency = 500, FrameSize = cfg.FrameSize, Version = cfg.Version,
                                     Padding = cfg.Padding, Type = (int)cfg.Type, Filter = cfg.Filter };
        var outBytes = new byte[VgAudioB200Cri.vgb_adx_encoded_byte_count(pcm.Length, cfg.Padding, cfg.FrameSize)];
        int n = pcm.Length;
        short history;
        fixed (short* p0 = pcm) fixed (byte* o0 = outBytes)
        {
            short* pp = p0; byte* oo = o0;
            VgAudioB200.Check(VgAudioB200Cri.vgb_adx_encode_batch(&pp, &n, &prm, 1, &history, &oo, null, IntPtr.Zero));
        }
        return outBytes;
    }

    private static byte[] NativeHca(short[][] pcm, Dictionary<string, string> p)
    {
        var prm = new VgbHcaParams { Quality = int.Parse(p["quality"]), Bitrate = int.Parse(p["bitrate"]), LimitBitrate = int.Parse(p["limit_bitrate"]),
                                     ChannelCount = pcm.Length, SampleRate = int.Parse(p["sample_rate"]), SampleCount = pcm[0].Length,
                                     Looping = int.Parse(p["looping"]), LoopStart = int.Parse(p["loop_start"]), LoopEnd = int.Parse(p["loop_end"]) };
        VgbHcaInfo h;
        VgAudioB200.Check(VgAudioB200Cri.vgb_hca_query(&prm, &h));
        var slab = new byte[h.FrameCount * h.FrameSize];
        var pins = pcm.Select(c => System.Runtime.InteropServices.GCHandle.Alloc(c, System.Runtime.InteropServices.GCHandleType.Pinned)).ToArray();
        try
        {
            short** tab = stackalloc short*[pcm.Length];
            for (int c = 0; c < pcm.Length; c++) tab[c] = (short*)pins[c].AddrOfPinnedObject();
            fixed (byte* o0 = slab)
            {
                byte* oo = o0;
                VgAudioB200.Check(VgAudioB200Cri.vgb_hca_encode_batch(tab, &prm, 1, &h, &oo, null, IntPtr.Zero));
            }
        }
        finally { foreach (var g in pins) g.Free(); }
        return slab;
    }

    // WaveReader -> GetFormat<T> (encode) -> writer, as Convert.ConvertFile runs it (src/VGAudio.Cli/Convert.cs:18-36), with the
    // writer configuration the params column names (CreateConfiguration.cs:118-150: keystring -> ADX type 8, keycode -> HCA key)
    private static byte[] ManagedConvert(byte[] wave, string kind, Dictionary<string, string> p)
    {
        AudioData audio = new VGAudio.Containers.Wave.WaveReader().Read(wave);
        switch (kind)
        {
            case "wave_to_dsp":
                return new VGAudio.Containers.Dsp.DspWriter().GetFile(audio);
            case "wave_to_adx":
                var adx = new VGAudio.Containers.Adx.AdxConfiguration();
                if (p.TryGetValue("keystring", out string ks)) { adx.EncryptionKey = new CriAdxKey(ks); adx.EncryptionType = 8; }
                return new VGAudio.Containers.Adx.AdxWriter().GetFile(audio, adx);
            default:
                var hca = new VGAudio.Containers.Hca.HcaConfiguration();
                if (p.TryGetValue("quality", out string q)) hca.Quality = (CriHcaQuality)int.Parse(q);
                if (p.TryGetValue("keycode", out string kc)) hca.EncryptionKey = new CriHcaKey(ulong.Parse(kc));
                return new VGAudio.Containers.Hca.HcaWriter().GetFile(audio, hca);
        }
    }

    // ---- vectors mode --------------------------------------------------------------------------------------------------
    private static int Vectors(string dir)
    {
        int bad = 0, n = 0;
        foreach (string line in File.ReadLines(Path.Combine(dir, "manifest.tsv")))
        {
            if (line.StartsWith("#") || line.Trim().Length == 0) continue;
            string[] f = line.Split('\t');
            var p = Params(f[2]);
            short[][] pcm = f[0].StartsWith("wave_to_") ? null : f[3].Split(',').Select(x => ReadPcm(Path.Combine(dir, x))).ToArray();
            byte[] ours = File.ReadAllBytes(Path.Combine(dir, f[4]));
            byte[] managed;
            switch (f[0])
            {
                case "gcadpcm":   // output file = 32 bytes of coefficients (16 x int16 LE) followed by the ADPCM bytes
                    byte[] adpcm = ManagedGc(pcm[0], out short[] coefs);
                    managed = new byte[32 + adpcm.Length];
                    Buffer.BlockCopy(coefs, 0, managed, 0, 32);
                    Buffer.BlockCopy(adpcm, 0, managed, 32, adpcm.Length);
                    break;
                case "gcadpcm_decode":   // input file 0 = coefficients + ADPCM as above, output = PCM16
                    byte[] blob = File.ReadAllBytes(Path.Combine(dir, f[3]));
                    var c2 = new short[16];
                    Buffer.BlockCopy(blob, 0, c2, 0, 32);
                    short[] dec = GcAdpcmDecoder.Decode(blob.Skip(32).ToArray(), c2, new GcAdpcmParameters { SampleCount = int.Parse(p["sample_count"]) });
                    managed = new byte[dec.Length * 2];
                    Buffer.BlockCopy(dec, 0, managed, 0, managed.Length);
                    break;
                case "criadx": managed = ManagedAdx(pcm[0], p); break;
                case "crihca": managed = ManagedHca(pcm, p); break;
                case "wave_to_dsp":   // input = a WAVE file; the finished file against WaveReader -> DspWriter.GetFile
                case "wave_to_adx":
                case "wave_to_hca":
                    managed = ManagedConvert(File.ReadAllBytes(Path.Combine(dir, f[3])), f[0], p);
                    break;
                default: Console.WriteLine($"unknown codec {f[0]}"); bad++; continue;
            }
            n++;
            if (!Report($"{f[0]}/{f[1]}", managed, ours)) bad++;
        }
        Console.WriteLine($"{n - bad} of {n} cases identical");
        return bad;
    }

    // ---- GcAdpcmAlignment: the managed GcAdpcmFormat.WithAlignment path (GcAdpcmChannelBuilder.GetAlignment -> new
    // GcAdpcmAlignment, GcAdpcmAlignment.cs:20-63) against vgb_gcadpcm_alignment + vgb_gcadpcm_align_batch ------------------
    private static bool AlignmentCase(string name, byte[] adpcm, short[] coefs, int sampleCount, int multiple, int loopStart, int loopEnd)
    {
        GcAdpcmChannel managed = new GcAdpcmFormatBuilder(new[] { new GcAdpcmChannel(adpcm, coefs, sampleCount) }, 48000)
            .WithLoop(true, loopStart, loopEnd).WithAlignment(multiple).Build().Channels[0];
        var prm = new VgAudioB200.VgbGcAlignParams { Multiple = multiple, LoopStart = loopStart, LoopEnd = loopEnd };
        var geo = new VgAudioB200.VgbGcAlignment();
        VgAudioB200.Check(VgAudioB200.vgb_gcadpcm_alignment(&prm, &geo));
        if (geo.AlignmentNeeded == 0)
            return Report($"gcadpcm align {name} (not needed)", managed.GetAdpcmAudio(), adpcm) && managed.SampleCount == sampleCount;
        var adpcmOurs = new byte[GcAdpcmMath.SampleCountToByteCount(geo.SampleCountAligned)];
        var pcmOurs = new short[geo.SampleCountAligned];
        int len = adpcm.Length;
        fixed (byte* a0 = adpcm) fixed (short* c = coefs) fixed (byte* o0 = adpcmOurs) fixed (short* p0 = pcmOurs)
        {
            byte* a = a0; byte* o = o0; short* pp = p0;
            VgAudioB200.Check(VgAudioB200.vgb_gcadpcm_align_batch(&a, &len, c, &prm, 1, &o, &pp));
        }
        byte[] pcmManagedBytes = managed.GetPcmAudio().SelectMany(BitConverter.GetBytes).ToArray();
        byte[] pcmOursBytes = pcmOurs.SelectMany(BitConverter.GetBytes).ToArray();
        bool same = Report($"gcadpcm align {name} AdpcmAligned", managed.GetAdpcmAudio(), adpcmOurs);
        same &= Report($"gcadpcm align {name} PcmAligned", pcmManagedBytes, pcmOursBytes);
        return same && managed.SampleCount == geo.SampleCountAligned;
    }

    private static int AlignmentCases()
    {
        int bad = 0;
        // GcAdpcmAlignmentTests.cs:13-61: ADPCM of 0x40 zero bytes, zero coefficients
        foreach (var (m, ls, le) in new[] { (0, 0, 10), (0, 5, 10), (1, 7, 10), (3, 12, 13), (5, 10, 13),     // AlignmentNotNeeded
                                            (2, 3, 10), (4, 2, 10), (3, 31, 50), (16, 24, 50), (16, 31, 50) }) // AlignmentNeeded, AlignedLoopPoints
            if (!AlignmentCase($"{m}/{ls}/{le}", new byte[0x40], new short[16], 112, m, ls, le)) bad++;
        // GcAdpcmAlignmentTests.cs:64-108 (AlignedAdpcmIsCorrect / AlignedPcmIsCorrect): a sine of period 56
        foreach (var (m, ls, cycles) in new[] { (1000, 4524, 100), (1000, 2012, 1), (1000, 60, 1), (1000, 60, 20) })
        {
            int le = cycles * 4 * 14 + ls;
            short[] pcm = Sine((le + 13) / 14 * 14, 1, 14 * 4);
            byte[] adpcm = ManagedGc(pcm, out short[] coefs);
            if (!AlignmentCase($"sine {m}/{ls}/{le}", adpcm, coefs, pcm.Length, m, ls, le)) bad++;
        }
        // seeded: BRSTM's default multiple 0x3800 and others, loop points anywhere, sines at random pitches
        var rng = new Random(0x414C49);
        int[] multiples = { 0x3800, 0x3800, 14, 8, 1000, -3, 4096 };
        for (int i = 0; i < 24; i++)
        {
            int n = rng.Next(20, 200000);
            short[] pcm = Sine(n, 40 + rng.Next(8000), 48000);
            byte[] adpcm = ManagedGc(pcm, out short[] coefs);
            int le = rng.Next(1, n + 1), ls = rng.Next(0, le);
            if (!AlignmentCase($"seeded {i}", adpcm, coefs, n, multiples[i % multiples.Length], ls, le)) bad++;
        }
        return bad;
    }

    // ---- live mode -----------------------------------------------------------------------------------------------------
    private static int Live()
    {
        VgAudioB200.Check(VgAudioB200.vgb_init(0, 0));
        double[] freqs = { 261.63, 329.63, 392, 523.25, 659.25, 783.99, 1046.50, 130.81 };   // GenerateAudio.cs:14
        int bad = 0;
        foreach (double fq in freqs)
        {
            short[] pcm = Sine(48000, fq, 48000);
            byte[] adpcmManaged = ManagedGc(pcm, out short[] coefsManaged);
            var coefsNative = new short[16];
            var adpcmNative = new byte[adpcmManaged.Length];
            int len = pcm.Length;
            fixed (short* pp0 = pcm) fixed (short* c = coefsNative) fixed (byte* a = adpcmNative)
            {
                short* pp = pp0; byte* aa = a;
                VgAudioB200.Check(VgAudioB200.vgb_gcadpcm_encode_batch(&pp, &len, null, null, 1, c, &aa, null, IntPtr.Zero));
            }
            if (!coefsManaged.SequenceEqual(coefsNative)) { Console.WriteLine($"gcadpcm {fq} Hz: coefficients DIFFERENT"); bad++; }
            if (!Report($"gcadpcm sine {fq:F2} Hz", adpcmManaged, adpcmNative)) bad++;

            // CRI ADX: every type and version, two paddings (CriCodecs.B200.cs holds the drop-in body used here)
            foreach (int type in new[] { 2, 3, 4 })
            foreach (int version in new[] { 3, 4 })
            foreach (int padding in new[] { 0, 45 })
            {
                var cfg = new CriAdxParameters { SampleRate = 48000, Version = version, Type = (CriAdxType)type, Padding = padding, Filter = 2 };
                byte[] managed = CriAdxCodec.Encode((short[])pcm.Clone(), cfg);
                byte[] ours = NativeAdx(pcm, cfg);
                if (!Report($"criadx {fq:F0} Hz type {type} v{version} pad {padding}", managed, ours)) bad++;
            }
        }
        // CRI HCA: qualities x channel counts, one looping case
        foreach (int quality in new[] { 1, 2, 3, 4, 5 })
        foreach (int channels in new[] { 1, 2, 3, 4, 5, 6, 7, 8 })
        {
            short[][] pcm = Enumerable.Range(0, channels).Select(c => Sine(30000, freqs[c], 48000)).ToArray();
            var p = new Dictionary<string, string> { ["quality"] = quality.ToString(), ["bitrate"] = "0", ["limit_bitrate"] = "0",
                ["sample_rate"] = "48000", ["looping"] = channels == 2 ? "1" : "0", ["loop_start"] = "5000", ["loop_end"] = "25000" };
            byte[] managed = ManagedHca(pcm, p);
            byte[] ours = NativeHca(pcm, p);
            if (!Report($"crihca quality {quality} x {channels} ch", managed, ours)) bad++;
        }
        return bad + AlignmentCases();
    }

    private static int Main(string[] args)
    {
        if (args.Length >= 2 && args[0] == "vectors") return Vectors(args[1]);
        if (args.Length >= 1 && args[0] == "live") return Live();
        Console.WriteLine("usage: ParityHarness live | ParityHarness vectors <dir written by tools/dump_vectors.py>");
        return 2;
    }
}
