// bindings/csharp/Containers.B200.cs — P/Invoke declarations and replacement bodies for the container layer either side of
// the codec path (include/vgaudio_b200.h, "Containers either side of the codec path"): WaveReader, DspWriter / DspReader,
// AdxWriter / AdxReader (+ CriAdxEncryption), HcaWriter / HcaReader (+ CriHcaEncryption) and the CLI's batch job.
// NOT compiled in this repository (no .NET toolchain in the build image); this is the file a VGAudio maintainer adds.
using System;
using System.Collections.Generic;
using System.IO;
using System.Linq;
using System.Runtime.InteropServices;

namespace VGAudio.Native
{
    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbWaveInfo
    {
        public int ChannelCount, SampleRate, BitsPerSample, SampleCount, Looping, LoopStart, LoopEnd, Reserved;
        public long DataOffset, DataSize;
    }

    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbDspDesc   // what DspWriter reads from GcAdpcmFormat + DspConfiguration (DspWriter.cs:17-36)
    {
        public int ChannelCount, SampleRate, SampleCount, Looping, LoopStart, LoopEnd;
        public int SamplesPerInterleave, LoopPointAlignment, NoTrim;   // 0 = 0x3800, 1, TrimFile = true
    }

    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbAdxDesc   // what AdxWriter reads from CriAdxFormat + AdxConfiguration (AdxWriter.cs:18-55)
    {
        public int ChannelCount, SampleRate, SampleCount, Looping, LoopStart, LoopEnd, AlignmentSamples;
        public int FrameSize, Version, Type, HighpassFrequency, EncryptionType, NoTrim;
    }

    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbAdxKey { public int Seed, Mult, Inc; }

    [StructLayout(LayoutKind.Sequential)]
    internal unsafe struct VgbAdxFileInfo   // AdxStructure (Containers/Adx/AdxStructure.cs) + where the audio sits
    {
        public int HeaderSize, Type, FrameSize, BitDepth, ChannelCount, SampleRate, SampleCount, HighpassFrequency;
        public int Version, Revision, InsertedSamples, LoopCount, Looping, LoopType;
        public int LoopStartSample, LoopStartByte, LoopEndSample, LoopEndByte;
        public int SamplesPerFrame, Reserved;
        public long AudioOffset, AudioSize;
        public fixed short History[255 * 2];
    }

    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbConvertOptions
    {
        public int OutType;                 // 1 .dsp, 2 .adx, 3 .hca
        public int NoTrim;
        public int DspSamplesPerInterleave, DspLoopPointAlignment;
        public int AdxVersion, AdxFrameSize, AdxType, AdxFilterPlus1;
        public int AdxEncryptionType, AdxHasKey, AdxKeySeed, AdxKeyMult, AdxKeyInc;
        public int HcaQuality, HcaBitrate, HcaLimitBitrate;
        public int HcaKeyType;              // -1 = none (0 IS a key type)
        public int Reserved;
        public ulong HcaKeyCode;
        public long GroupBytes;
    }

    internal static unsafe class VgAudioB200Containers
    {
        private const string Lib = "vgaudio_b200";

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_wave_parse(byte* file, long length, VgbWaveInfo* info);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_wave_read_batch(byte** files, long* lengths, VgbWaveInfo* info, int nFiles, short** pcmOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern long vgb_dsp_file_size(VgbDspDesc* desc);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_dsp_write_batch(VgbDspDesc* files, int nFiles, byte** adpcm, short* coefs, short* gain, short* startHist,
            short* loopContext, byte** filesOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern long vgb_adx_file_size(VgbAdxDesc* desc);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_adx_key_from_code(ulong keyCode, VgbAdxKey* key);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_adx_key_from_string([MarshalAs(UnmanagedType.LPStr)] string s, VgbAdxKey* key);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_write_batch(VgbAdxDesc* files, int nFiles, byte** audio, int* audioLen, short* history, VgbAdxKey* key, byte** filesOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_crypt_batch(byte** audio, int nChannels, int length, VgbAdxKey* key, int encryptionType, int frameSize);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_hca_key_tables(int keyType, ulong keyCode, byte* decrypt, byte* encrypt);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_hca_crypt_batch(byte** frames, int* frameCount, int nStreams, int frameSize, int keyType, ulong keyCode, int decrypt);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_hca_write_batch(VgbHcaInfo* info, int nFiles, byte** frames, int keyType, ulong keyCode, byte** comment, float* volume, byte** filesOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_convert_dsp_to_wave_batch(byte** files, long* lengths, int nFiles, long* outSizes, byte** filesOut, int* statusOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_hca_parse(byte* file, long length, VgbHcaInfo* info, int* encryptionType);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_adx_parse(byte* file, long length, VgbAdxFileInfo* info);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_convert_adx_to_wave_batch(byte** files, long* lengths, int nFiles, VgbAdxKey* key, long* outSizes, byte** filesOut, int* statusOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_convert_hca_to_wave_batch(byte** files, long* lengths, int nFiles, ulong* keyCode, long* outSizes, byte** filesOut, int* statusOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_convert_wave_batch(byte** files, long* lengths, int nFiles, VgbConvertOptions* options, long* outSizes,
            byte** filesOut, int* statusOut, VgbProgress progress, IntPtr user);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_transcode_batch(byte** files, long* lengths, int* inType, int nFiles, VgbConvertOptions* options,
            VgbAdxKey* inAdxKey, ulong* inHcaKeyCode, long* outSizes, byte** filesOut, int* statusOut, VgbProgress progress, IntPtr user);
    }
}

namespace VGAudio.Containers.Dsp
{
    using VGAudio.Native;

    // Replacement body for DspWriter.WriteStream (Containers/Dsp/DspWriter.cs:42-52): the header fields and the
    // block interleave of WriteHeader / WriteData (:54-99) become one native call that returns the finished file.
    public partial class DspWriterB200
    {
        internal static unsafe byte[] GetFile(VGAudio.Formats.GcAdpcm.GcAdpcmFormat adpcm, DspConfiguration config)
        {
            var desc = new VgbDspDesc
            {
                ChannelCount = adpcm.ChannelCount, SampleRate = adpcm.SampleRate, SampleCount = adpcm.SampleCount,
                Looping = adpcm.Looping ? 1 : 0, LoopStart = adpcm.LoopStart, LoopEnd = adpcm.LoopEnd,
                SamplesPerInterleave = config.SamplesPerInterleave, LoopPointAlignment = config.LoopPointAlignment, NoTrim = config.TrimFile ? 0 : 1
            };
            long size = VgAudioB200Containers.vgb_dsp_file_size(&desc);
            if (size < 0) VgAudioB200.Check((int)size);
            var file = new byte[size];
            int n = adpcm.ChannelCount;
            byte[][] audio = adpcm.Channels.Select(c => c.GetAdpcmAudio()).ToArray();
            short[] coefs = adpcm.Channels.SelectMany(c => c.Coefs).ToArray();
            short[] gain = adpcm.Channels.Select(c => c.Gain).ToArray();
            short[] hist = adpcm.Channels.SelectMany(c => new[] { c.StartContext.Hist1, c.StartContext.Hist2 }).ToArray();
            short[] loop = adpcm.Channels.SelectMany(c => new[] { c.LoopContext.PredScale, c.LoopContext.Hist1, c.LoopContext.Hist2 }).ToArray();
            var pins = audio.Select(a => GCHandle.Alloc(a, GCHandleType.Pinned)).ToArray();
            try
            {
                byte** rows = stackalloc byte*[n];
                for (int i = 0; i < n; i++) rows[i] = (byte*)pins[i].AddrOfPinnedObject();
                fixed (byte* pf = file)
                fixed (short* pc = coefs, pg = gain, ph = hist, pl = loop)
                {
                    byte* outPtr = pf;
                    VgAudioB200.Check(VgAudioB200Containers.vgb_dsp_write_batch(&desc, 1, rows, pc, pg, ph, adpcm.Looping ? pl : null, &outPtr));
                }
            }
            finally { foreach (var h in pins) h.Free(); }
            return file;
        }
    }
}

namespace VGAudio.Cli
{
    using VGAudio.Native;

    // Replacement for the Parallel.ForEach of Batch.BatchConvert (src/VGAudio.Cli/Batch.cs:24-46) when every input is a
    // WAVE file and the output is .dsp / .adx / .hca: the managed side still enumerates, reads and writes files; a chunk of
    // file images goes through ONE native call (sizing pass, then the filling pass).
    internal static class BatchB200
    {
        public static unsafe void ConvertChunk(string[] inPaths, string[] outPaths, VgbConvertOptions options, Action<string> log, Action<int> reportAdd)
        {
            int n = inPaths.Length;
            byte[][] images = inPaths.Select(File.ReadAllBytes).ToArray();
            var inPins = images.Select(a => GCHandle.Alloc(a, GCHandleType.Pinned)).ToArray();
            var outPins = new List<GCHandle>();
            try
            {
                byte** inPtr = stackalloc byte*[n];
                byte** outPtr = stackalloc byte*[n];
                long* len = stackalloc long[n];
                long* outSize = stackalloc long[n];
                int* status = stackalloc int[n];
                for (int i = 0; i < n; i++) { inPtr[i] = (byte*)inPins[i].AddrOfPinnedObject(); len[i] = images[i].Length; }
                VgAudioB200.Check(VgAudioB200Containers.vgb_convert_wave_batch(inPtr, len, n, &options, outSize, null, status, null, IntPtr.Zero));
                var outputs = new byte[n][];
                for (int i = 0; i < n; i++)
                {
                    outPtr[i] = null;
                    if (status[i] != VgAudioB200.Ok) continue;
                    outputs[i] = new byte[outSize[i]];
                    outPins.Add(GCHandle.Alloc(outputs[i], GCHandleType.Pinned));
                    outPtr[i] = (byte*)outPins[outPins.Count - 1].AddrOfPinnedObject();
                }
                VgbProgress cb = (user, delta) => reportAdd((int)delta);   // progress.ReportAdd(1) per file (Batch.cs:45)
                VgAudioB200.Check(VgAudioB200Containers.vgb_convert_wave_batch(inPtr, len, n, &options, outSize, outPtr, status, cb, IntPtr.Zero));
                for (int i = 0; i < n; i++)
                {
                    if (status[i] != VgAudioB200.Ok) { log($"Error converting {Path.GetFileName(inPaths[i])}"); continue; }   // Batch.cs:39-43
                    Directory.CreateDirectory(Path.GetDirectoryName(outPaths[i]));
                    File.WriteAllBytes(outPaths[i], outputs[i]);
                }
            }
            finally
            {
                foreach (var h in inPins) h.Free();
                foreach (var h in outPins) h.Free();
            }
        }

        // The decode direction for a chunk of .hca files (`-b --out-format wav`): HcaReader -> ToPcm16 -> WaveWriter per file
        // in one native call per pass.  keyCode is the type-56 key (CriHcaKey(ulong)); the native library carries no list of
        // known keys, so a caller that wants HcaReader.FindKey's search runs CriHcaEncryption.FindKey on the file and passes
        // the code it finds.  A file whose frames the decoder refuses (a wrong key, a bad frame) fails in the second pass alone.
        public static unsafe void ConvertHcaToWave(string[] inPaths, string[] outPaths, ulong? keyCode, Action<string> log, Action<int> reportAdd)
        {
            int n = inPaths.Length;
            byte[][] images = inPaths.Select(File.ReadAllBytes).ToArray();
            var inPins = images.Select(a => GCHandle.Alloc(a, GCHandleType.Pinned)).ToArray();
            var outPins = new List<GCHandle>();
            try
            {
                byte** inPtr = stackalloc byte*[n];
                byte** outPtr = stackalloc byte*[n];
                long* len = stackalloc long[n];
                long* outSize = stackalloc long[n];
                int* status = stackalloc int[n];
                ulong code = keyCode ?? 0;
                ulong* codePtr = keyCode.HasValue ? &code : null;
                for (int i = 0; i < n; i++) { inPtr[i] = (byte*)inPins[i].AddrOfPinnedObject(); len[i] = images[i].Length; }
                VgAudioB200.Check(VgAudioB200Containers.vgb_convert_hca_to_wave_batch(inPtr, len, n, codePtr, outSize, null, status));
                var outputs = new byte[n][];
                for (int i = 0; i < n; i++)
                {
                    outPtr[i] = null;
                    if (status[i] != VgAudioB200.Ok) continue;
                    outputs[i] = new byte[outSize[i]];
                    outPins.Add(GCHandle.Alloc(outputs[i], GCHandleType.Pinned));
                    outPtr[i] = (byte*)outPins[outPins.Count - 1].AddrOfPinnedObject();
                }
                VgAudioB200.Check(VgAudioB200Containers.vgb_convert_hca_to_wave_batch(inPtr, len, n, codePtr, outSize, outPtr, status));
                for (int i = 0; i < n; i++)
                {
                    if (status[i] != VgAudioB200.Ok) { log($"Error converting {Path.GetFileName(inPaths[i])}"); }   // Batch.cs:39-43
                    else
                    {
                        Directory.CreateDirectory(Path.GetDirectoryName(outPaths[i]));
                        File.WriteAllBytes(outPaths[i], outputs[i]);
                    }
                    reportAdd(1);
                }
            }
            finally
            {
                foreach (var h in inPins) h.Free();
                foreach (var h in outPins) h.Free();
            }
        }

        // The decode direction for a chunk of .adx files (`-b --out-format wav`): AdxReader -> ToPcm16 -> WaveWriter per file
        // in one native call per pass.  key (CriAdxKey from --keystring / --keycode, as vgb_adx_key_from_string / _code make it)
        // decrypts files of revision 8 and 9; the native library carries no list of known keys, so a caller that wants
        // CriAdxEncryption.FindKey's search runs it on the file and passes the key it finds.  A file whose frames select a
        // filter the reference cannot index fails in the second pass alone.
        public static unsafe void ConvertAdxToWave(string[] inPaths, string[] outPaths, VgbAdxKey? key, Action<string> log, Action<int> reportAdd)
        {
            int n = inPaths.Length;
            byte[][] images = inPaths.Select(File.ReadAllBytes).ToArray();
            var inPins = images.Select(a => GCHandle.Alloc(a, GCHandleType.Pinned)).ToArray();
            var outPins = new List<GCHandle>();
            try
            {
                byte** inPtr = stackalloc byte*[n];
                byte** outPtr = stackalloc byte*[n];
                long* len = stackalloc long[n];
                long* outSize = stackalloc long[n];
                int* status = stackalloc int[n];
                VgbAdxKey k = key ?? default;
                VgbAdxKey* keyPtr = key.HasValue ? &k : null;
                for (int i = 0; i < n; i++) { inPtr[i] = (byte*)inPins[i].AddrOfPinnedObject(); len[i] = images[i].Length; }
                VgAudioB200.Check(VgAudioB200Containers.vgb_convert_adx_to_wave_batch(inPtr, len, n, keyPtr, outSize, null, status));
                var outputs = new byte[n][];
                for (int i = 0; i < n; i++)
                {
                    outPtr[i] = null;
                    if (status[i] != VgAudioB200.Ok) continue;
                    outputs[i] = new byte[outSize[i]];
                    outPins.Add(GCHandle.Alloc(outputs[i], GCHandleType.Pinned));
                    outPtr[i] = (byte*)outPins[outPins.Count - 1].AddrOfPinnedObject();
                }
                VgAudioB200.Check(VgAudioB200Containers.vgb_convert_adx_to_wave_batch(inPtr, len, n, keyPtr, outSize, outPtr, status));
                for (int i = 0; i < n; i++)
                {
                    if (status[i] != VgAudioB200.Ok) { log($"Error converting {Path.GetFileName(inPaths[i])}"); }   // Batch.cs:39-43
                    else
                    {
                        Directory.CreateDirectory(Path.GetDirectoryName(outPaths[i]));
                        File.WriteAllBytes(outPaths[i], outputs[i]);
                    }
                    reportAdd(1);
                }
            }
            finally
            {
                foreach (var h in inPins) h.Free();
                foreach (var h in outPins) h.Free();
            }
        }

        // Coded files in, another codec out (`-b -i adx/ --out-format hca` and the like): per file the source's reader,
        // ToPcm16 and the target's encoder and writer from the options (Convert.ConvertFile with KeepConfiguration false),
        // decoded and re-encoded on the device in one native call per pass.  inTypes[i] is VGB_CONTAINER_DSP / _ADX / _HCA
        // (1 / 2 / 3) for file i; a file already in options.OutType's codec fails alone (no rewrite is performed).
        // inAdxKey decrypts revision 8 / 9 .adx sources and inHcaKeyCode "ciph" 56 .hca sources; the output's key is in
        // options.  A file whose frames the decoder refuses fails in the second pass alone.
        public static unsafe void Transcode(string[] inPaths, int[] inTypes, string[] outPaths, VgbConvertOptions options, VgbAdxKey? inAdxKey,
            ulong? inHcaKeyCode, Action<string> log, Action<int> reportAdd)
        {
            int n = inPaths.Length;
            byte[][] images = inPaths.Select(File.ReadAllBytes).ToArray();
            var inPins = images.Select(a => GCHandle.Alloc(a, GCHandleType.Pinned)).ToArray();
            var outPins = new List<GCHandle>();
            try
            {
                byte** inPtr = stackalloc byte*[n];
                byte** outPtr = stackalloc byte*[n];
                long* len = stackalloc long[n];
                long* outSize = stackalloc long[n];
                int* status = stackalloc int[n];
                VgbAdxKey k = inAdxKey ?? default;
                VgbAdxKey* keyPtr = inAdxKey.HasValue ? &k : null;
                ulong code = inHcaKeyCode ?? 0;
                ulong* codePtr = inHcaKeyCode.HasValue ? &code : null;
                for (int i = 0; i < n; i++) { inPtr[i] = (byte*)inPins[i].AddrOfPinnedObject(); len[i] = images[i].Length; }
                fixed (int* types = inTypes)
                {
                    VgAudioB200.Check(VgAudioB200Containers.vgb_transcode_batch(inPtr, len, types, n, &options, keyPtr, codePtr, outSize, null, status, null, IntPtr.Zero));
                    var outputs = new byte[n][];
                    for (int i = 0; i < n; i++)
                    {
                        outPtr[i] = null;
                        if (status[i] != VgAudioB200.Ok) continue;
                        outputs[i] = new byte[outSize[i]];
                        outPins.Add(GCHandle.Alloc(outputs[i], GCHandleType.Pinned));
                        outPtr[i] = (byte*)outPins[outPins.Count - 1].AddrOfPinnedObject();
                    }
                    VgbProgress cb = (user, delta) => reportAdd((int)delta);   // progress.ReportAdd(1) per file (Batch.cs:45)
                    VgAudioB200.Check(VgAudioB200Containers.vgb_transcode_batch(inPtr, len, types, n, &options, keyPtr, codePtr, outSize, outPtr, status, cb, IntPtr.Zero));
                    GC.KeepAlive(cb);
                    for (int i = 0; i < n; i++)
                    {
                        if (status[i] != VgAudioB200.Ok) { log($"Error converting {Path.GetFileName(inPaths[i])}"); continue; }   // Batch.cs:39-43
                        Directory.CreateDirectory(Path.GetDirectoryName(outPaths[i]));
                        File.WriteAllBytes(outPaths[i], outputs[i]);
                    }
                }
            }
            finally
            {
                foreach (var h in inPins) h.Free();
                foreach (var h in outPins) h.Free();
            }
        }
    }
}
