// bindings/csharp/Containers.B200.cs — P/Invoke declarations and replacement bodies for the container layer either side of
// the codec path (include/vgaudio_b200.h, "Containers either side of the codec path"): WaveReader, DspWriter / DspReader,
// AdxWriter / AdxReader (+ CriAdxEncryption), HcaWriter / HcaReader (+ CriHcaEncryption), BrstmReader / BCFstmReader and the
// CLI's batch job.
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
    internal struct VgbAdxFoundKey   // one key of vgb_adx_find_keys (GuessAdx.AddKey)
    {
        public VgbAdxKey Key;
        public int Status;                     // Ok, or the confidence pass's error (confidences NaN)
        public ulong KeyCode;                  // CriAdxKey.KeyCode
        public long DiffShort, TotalShort, DiffFull, TotalFull;
        public double ConfidenceShort, ConfidenceFull;
    }

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
    internal unsafe struct VgbNwInfo   // BxstmStructure (Containers/NintendoWare/BxstmStructure.cs), what decoding needs
    {
        public int Codec, Looping, ChannelCount, SampleRate, LoopStart, SampleCount;
        public int InterleaveSize, BigEndian;
        public uint Version;
        public int SeekTable, RegionCount, TrackCount, AdpcmChannelCount, SamplesPerSeekEntry;
        public int LoopStartUnaligned, LoopEndUnaligned, OutputSize, Reserved;
        public long AudioOffset, AudioLength;
        public fixed short Coefs[255 * 16];
        public fixed short Gain[255];
        public fixed short StartContext[255 * 3], LoopContext[255 * 3];
    }

    [StructLayout(LayoutKind.Sequential)]
    internal unsafe struct VgbIdspInfo   // IdspStructure (Containers/Idsp/IdspStructure.cs) with the region DeInterleave reads
    {
        public int ChannelCount, SampleRate, SampleCount, LoopStart, LoopEnd, InterleaveSize;
        public int HeaderSize, ChannelInfoSize, AudioDataOffset, AudioDataLength;
        public int Looping, Interleave, OutputSize, Reserved;
        public long AudioOffset, AudioLength;
        public fixed int ChSampleCount[255], ChNibbleCount[255], ChSampleRate[255];
        public fixed int ChLooping[255], StartAddress[255], EndAddress[255];
        public fixed int CurrentAddress[255];
        public fixed short Coefs[255 * 16];
        public fixed short Gain[255];
        public fixed short StartContext[255 * 3], LoopContext[255 * 3];
    }

    [StructLayout(LayoutKind.Sequential)]
    internal unsafe struct VgbHpsInfo   // HpsStructure (Containers/Hps/HpsStructure.cs)
    {
        public int SampleRate, ChannelCount, SampleCount, Looping, LoopStart, BlockCount;
        public int FirstBlock, LoopBlock;
        public fixed int MaxBlockSize[255], EndAddress[255];
        public fixed long ChannelAudioBytes[255];
        public fixed short Coefs[255 * 16];
        public fixed short Gain[255];
        public fixed short StartContext[255 * 3], LoopContext[255 * 3];
    }

    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbHpsBlock   // HpsBlock (Containers/Hps/HpsBlock.cs)
    {
        public int Offset, Size, FinalNibble, NextOffset;
    }

    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbConvertOptions
    {
        public int OutType;                 // 1 .dsp, 2 .adx, 3 .hca, 4 .brstm, 5 .bcstm, 6 .bfstm, 7 .idsp, 8 .hps
        public int NoTrim;
        public int DspSamplesPerInterleave, DspLoopPointAlignment;
        public int AdxVersion, AdxFrameSize, AdxType, AdxFilterPlus1;
        public int AdxEncryptionType, AdxHasKey, AdxKeySeed, AdxKeyMult, AdxKeyInc;
        public int HcaQuality, HcaBitrate, HcaLimitBitrate;
        public int HcaKeyType;              // -1 = none (0 IS a key type)
        public int Reserved;
        public ulong HcaKeyCode;
        public long GroupBytes;
        public int NwCodecPlus1;            // 0 = GC-ADPCM; else NwCodec + 1
        public int NwEndianness;            // 0 = the target's, 1 = little, 2 = big (BRSTM is always big)
        public int NwLoopPointAlignment;    // 0 = BytesToSamples(0x2000, codec)
        public int NwPad;
        // AudioData.SetLoop on every source before any encode or write (Convert.cs:82-90): 0 keeps each file's loop,
        // 1 (VGB_LOOP_SET, -l) loops every file over [LoopStart, LoopEnd), 2 (VGB_LOOP_CLEAR, --no-loop) clears it
        public int LoopMode, LoopStart, LoopEnd;
        public int LoopPad;
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
        // GuessAdx (VGAudio.Tools/CrackAdx/GuessAdx.cs) on the GPU: fileStatus may be null, revision may be null
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_find_keys(byte** files, long* lengths, int nFiles, VgbAdxFoundKey* keysOut, int maxKeys, int* nKeysOut,
            int* fileStatusOut, int* revisionOut);
        // HcaReader.FindKey over a caller's list of type-56 key codes: per file the first index and VgAudioB200.Ok, or -1 and
        // VGB_E_DATA (a bad sync word), HcaKeySkipped, HcaKeyNotFound or the read error
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_hca_find_keys(byte** files, long* lengths, int nFiles, ulong* keyCodes, int nKeys, int* keyIndexOut, int* fileStatusOut);
        public const int HcaKeySkipped = 1, HcaKeyNotFound = 2;
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_convert_hca_to_wave_batch(byte** files, long* lengths, int nFiles, ulong* keyCode, long* outSizes, byte** filesOut, int* statusOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_brstm_parse(byte* file, long length, VgbNwInfo* info);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_bcfstm_parse(byte* file, long length, VgbNwInfo* info);
        // NintendoWare wave files and prefetch streams (read only), named by the reader the extension picks (ContainerTypes.cs)
        public const int VGB_CONTAINER_BRWAV = 9;    // BrwavReader: .brwav .rwav
        public const int VGB_CONTAINER_BCWAV = 10;   // BCFstmReader: .bcwav .cwav .bms
        public const int VGB_CONTAINER_BFWAV = 11;   // BCFstmReader: .bfwav
        public const int VGB_CONTAINER_BCSTP = 12;   // BCFstmReader: .bcstp
        public const int VGB_CONTAINER_BFSTP = 13;   // BCFstmReader: .bfstp
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_nw_file_parse(byte* file, long length, int inType, VgbNwInfo* info, long* channelOffsets);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_convert_nw_to_wave_batch(byte** files, long* lengths, int* inType, int nFiles, long* outSizes, byte** filesOut, int* statusOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_idsp_parse(byte* file, long length, VgbIdspInfo* info);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_hps_parse(byte* file, long length, VgbHpsInfo* info, VgbHpsBlock* blocks, int blockCapacity);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_convert_idsp_hps_to_wave_batch(byte** files, long* lengths, int* inType, int nFiles, long* outSizes, byte** filesOut, int* statusOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_convert_to_wave_batch(byte** files, long* lengths, int* inType, int nFiles, VgbConvertOptions* options,
            VgbAdxKey* adxKey, ulong* hcaKeyCode, long* outSizes, byte** filesOut, int* statusOut);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_gcadpcm_debug_decode_stats(ulong* output, int n);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_convert_wave_batch(byte** files, long* lengths, int nFiles, VgbConvertOptions* options, long* outSizes,
            byte** filesOut, int* statusOut, VgbProgress progress, IntPtr user);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_transcode_batch(byte** files, long* lengths, int* inType, int nFiles, VgbConvertOptions* options,
            VgbAdxKey* inAdxKey, ulong* inHcaKeyCode, long* outSizes, byte** filesOut, int* statusOut, VgbProgress progress, IntPtr user);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_transcode_nw_batch(byte** files, long* lengths, int* inType, int nFiles, VgbConvertOptions* options,
            VgbAdxKey* inAdxKey, ulong* inHcaKeyCode, long* outSizes, byte** filesOut, int* statusOut, VgbProgress progress, IntPtr user);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_transcode_from_nw_batch(byte** files, long* lengths, int* inType, int nFiles, VgbConvertOptions* options,
            long* outSizes, byte** filesOut, int* statusOut, VgbProgress progress, IntPtr user);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_rewrite_batch(byte** files, long* lengths, int nFiles, VgbConvertOptions* options, VgbAdxKey* inAdxKey,
            ulong* inHcaKeyCode, long* outSizes, byte** filesOut, int* statusOut, VgbProgress progress, IntPtr user);
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
        // in one native call per pass.  keyCode is the type-56 key (CriHcaKey(ulong)), used untested as HcaReader's
        // EncryptionKey is; the native library carries no list of known keys, so a caller with a list of codes runs
        // FindHcaKeys (HcaReader.FindKey on the GPU) first and converts each key's files with it.  A file whose frames the
        // decoder refuses (a wrong key, a bad frame) fails in the second pass alone.
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

        // HcaReader.FindKey over the keys in list order for each file: (index of the first key that decrypts it or -1, status:
        // VgAudioB200.Ok, VGB_E_DATA for a bad sync word in the test window, HcaKeySkipped when "ciph" is not 56,
        // HcaKeyNotFound, or the file's read error)
        public static unsafe (int[] Index, int[] Status) FindHcaKeys(byte[][] files, ulong[] keys)
        {
            int n = files.Length;
            var pins = files.Select(a => GCHandle.Alloc(a, GCHandleType.Pinned)).ToArray();
            try
            {
                byte** inPtr = stackalloc byte*[Math.Max(n, 1)];
                long* len = stackalloc long[Math.Max(n, 1)];
                for (int i = 0; i < n; i++) { inPtr[i] = (byte*)pins[i].AddrOfPinnedObject(); len[i] = files[i].Length; }
                var index = new int[Math.Max(n, 1)];
                var status = new int[Math.Max(n, 1)];
                fixed (ulong* k = keys.Length > 0 ? keys : new ulong[1])
                fixed (int* ix = index)
                fixed (int* st = status)
                    VgAudioB200.Check(VgAudioB200Containers.vgb_hca_find_keys(inPtr, len, n, k, keys.Length, ix, st));
                return (index.Take(n).ToArray(), status.Take(n).ToArray());
            }
            finally
            {
                foreach (var h in pins) h.Free();
            }
        }

        // GuessAdx.Run over .adx files of one revision (the first file's; others are skipped): every key valid on every file,
        // ascending by (seed, mult, inc), with AddKey's confidences.  More than maxKeys keys throw, with no partial list.
        public static unsafe VgbAdxFoundKey[] FindAdxKeys(string[] inPaths, int maxKeys = 256)
        {
            int n = inPaths.Length;
            byte[][] images = inPaths.Select(File.ReadAllBytes).ToArray();
            var inPins = images.Select(a => GCHandle.Alloc(a, GCHandleType.Pinned)).ToArray();
            try
            {
                byte** inPtr = stackalloc byte*[Math.Max(n, 1)];
                long* len = stackalloc long[Math.Max(n, 1)];
                for (int i = 0; i < n; i++) { inPtr[i] = (byte*)inPins[i].AddrOfPinnedObject(); len[i] = images[i].Length; }
                var keys = new VgbAdxFoundKey[Math.Max(maxKeys, 1)];
                int found = 0;
                fixed (VgbAdxFoundKey* k = keys)
                    VgAudioB200.Check(VgAudioB200Containers.vgb_adx_find_keys(inPtr, len, n, k, maxKeys, &found, null, null));
                return keys.Take(found).ToArray();
            }
            finally
            {
                foreach (var h in inPins) h.Free();
            }
        }

        // The decode direction for a chunk of .adx files (`-b --out-format wav`): AdxReader -> ToPcm16 -> WaveWriter per file
        // in one native call per pass.  key (CriAdxKey from --keystring / --keycode, as vgb_adx_key_from_string / _code make it)
        // decrypts files of revision 8 and 9; the native library carries no list of known keys, so a caller passes the key
        // CriAdxEncryption.FindKey or FindAdxKeys (GuessAdx) finds.  A file whose frames select a
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

        // The decode direction for a chunk of NintendoWare files (`-b --out-format wav` over .brstm / .bcstm / .bfstm, the
        // wave files .brwav / .rwav / .bcwav / .cwav / .bms / .bfwav and the prefetch streams .bcstp / .bfstp): the reader
        // the extension names (ContainerTypes.cs: BrstmReader, BrwavReader, BCFstmReader for the others) -> ToPcm16 ->
        // WaveWriter per file in one native call per pass.  inTypes[i] is VGB_CONTAINER_BRSTM / _BCSTM / _BFSTM (4 / 5 / 6)
        // or VGB_CONTAINER_BRWAV / _BCWAV / _BFWAV / _BCSTP / _BFSTP (9 .. 13).  A file whose GC-ADPCM frames select a
        // predictor outside 0..7 fails in the second pass alone.
        public static unsafe void ConvertNwToWave(string[] inPaths, int[] inTypes, string[] outPaths, Action<string> log, Action<int> reportAdd)
        {
            ConvertTypedToWave(inPaths, inTypes, outPaths, log, reportAdd, VgAudioB200Containers.vgb_convert_nw_to_wave_batch);
        }

        // The decode direction for a chunk of IDSP and HPS streams (`-b --out-format wav` over .idsp / .hps): IdspReader or
        // HpsReader as the extension names it (ContainerTypes.cs) -> ToPcm16 -> WaveWriter per file in one native call per
        // pass.  inTypes[i] is VGB_CONTAINER_IDSP / _HPS (7 / 8).  A file whose frames select a predictor outside 0..7 fails
        // in the second pass alone.
        public static unsafe void ConvertIdspHpsToWave(string[] inPaths, int[] inTypes, string[] outPaths, Action<string> log, Action<int> reportAdd)
        {
            ConvertTypedToWave(inPaths, inTypes, outPaths, log, reportAdd, VgAudioB200Containers.vgb_convert_idsp_hps_to_wave_batch);
        }

        // The decode direction for a chunk of files of any readable container in one native call per pass, with the batch's
        // -l / --no-loop: inTypes[i] names file i's reader (VGB_CONTAINER_DSP / _ADX / _HCA / _BRSTM .. _BFSTP / _IDSP /
        // _HPS), options carries only the loop (LoopMode, LoopStart, LoopEnd; null keeps every file's loop), adxKey decrypts
        // .adx files of revision 8 and 9 and hcaKeyCode "ciph" 56 .hca files.  A file whose loop its format's WithLoop
        // refuses fails alone with the reference's message, as does a file the decoder refuses in the second pass.
        // Like the rest of this file, ConvertToWave and the Loop* fields of VgbConvertOptions are not compiled or run by
        // this repository's build or tests (no .NET toolchain); the struct layout follows vgb_convert_options field by field.
        public static unsafe void ConvertToWave(string[] inPaths, int[] inTypes, string[] outPaths, VgbConvertOptions? options, VgbAdxKey? adxKey,
                                                ulong? hcaKeyCode, Action<string> log, Action<int> reportAdd)
        {
            ConvertTypedToWave(inPaths, inTypes, outPaths, log, reportAdd, (files, lengths, types, nFiles, outSizes, filesOut, statusOut) =>
            {
                VgbConvertOptions o = options ?? default;   // locals of the lambda: their addresses may be taken
                VgbAdxKey k = adxKey ?? default;
                ulong code = hcaKeyCode ?? 0;
                return VgAudioB200Containers.vgb_convert_to_wave_batch(files, lengths, types, nFiles, options.HasValue ? &o : null,
                    adxKey.HasValue ? &k : null, hcaKeyCode.HasValue ? &code : null, outSizes, filesOut, statusOut);
            });
        }

        private unsafe delegate int TypedToWave(byte** files, long* lengths, int* inType, int nFiles, long* outSizes, byte** filesOut, int* statusOut);

        // The two passes of a converter whose files carry an in_type each (the reader), with per-file status
        private static unsafe void ConvertTypedToWave(string[] inPaths, int[] inTypes, string[] outPaths, Action<string> log, Action<int> reportAdd,
                                                      TypedToWave convert)
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
                fixed (int* types = inTypes)
                {
                    VgAudioB200.Check(convert(inPtr, len, types, n, outSize, null, status));
                    var outputs = new byte[n][];
                    for (int i = 0; i < n; i++)
                    {
                        outPtr[i] = null;
                        if (status[i] != VgAudioB200.Ok) continue;
                        outputs[i] = new byte[outSize[i]];
                        outPins.Add(GCHandle.Alloc(outputs[i], GCHandleType.Pinned));
                        outPtr[i] = (byte*)outPins[outPins.Count - 1].AddrOfPinnedObject();
                    }
                    VgAudioB200.Check(convert(inPtr, len, types, n, outSize, outPtr, status));
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
        public static void Transcode(string[] inPaths, int[] inTypes, string[] outPaths, VgbConvertOptions options, VgbAdxKey? inAdxKey,
            ulong? inHcaKeyCode, Action<string> log, Action<int> reportAdd) =>
            Transcode(TxCall.Coded, inPaths, inTypes, outPaths, options, inAdxKey, inHcaKeyCode, log, reportAdd);

        // Coded files into a NintendoWare stream, IDSP or HPS file (`-b -i hca/ --out-format bfstm` and the like):
        // options.OutType is VGB_CONTAINER_BRSTM / _BCSTM / _BFSTM / _IDSP / _HPS (4..8), inTypes and keys as in
        // Transcode, the target's options (NwCodecPlus1, NwEndianness, NwLoopPointAlignment, NoTrim) as in ConvertWave.
        // .adx and .hca sources are re-encoded; a .dsp source is taken into PCM16 / PCM8 only, and fails alone for a
        // GC-ADPCM target (no rewrite is performed).
        public static void TranscodeNw(string[] inPaths, int[] inTypes, string[] outPaths, VgbConvertOptions options, VgbAdxKey? inAdxKey,
            ulong? inHcaKeyCode, Action<string> log, Action<int> reportAdd) =>
            Transcode(TxCall.IntoNw, inPaths, inTypes, outPaths, options, inAdxKey, inHcaKeyCode, log, reportAdd);

        // NintendoWare streams, wave and prefetch files, IDSP and HPS files into any coded target (`-b -i brstm/
        // --out-format hca --nw-inputs` and the like): inTypes[i] is VGB_CONTAINER_BRSTM .. _BFSTP (4..13), options.OutType
        // any of .dsp, .adx, .hca, .brstm, .bcstm, .bfstm, .idsp, .hps (1..8) with the target's options as in ConvertWave.
        // None of these containers is encrypted, so there are no input keys.  A file already in the target's codec fails
        // alone (no rewrite is performed); a file whose GC-ADPCM frames select a predictor outside 0..7 fails in the
        // second pass alone.
        public static void TranscodeFromNw(string[] inPaths, int[] inTypes, string[] outPaths, VgbConvertOptions options, Action<string> log,
            Action<int> reportAdd) =>
            Transcode(TxCall.FromNw, inPaths, inTypes, outPaths, options, null, null, log, reportAdd);

        // vgb_transcode_batch, vgb_transcode_nw_batch or vgb_transcode_from_nw_batch
        enum TxCall { Coded, IntoNw, FromNw }

        static unsafe int TranscodeCall(TxCall call, byte** files, long* lengths, int* types, int n, VgbConvertOptions* options, VgbAdxKey* key,
            ulong* code, long* outSizes, byte** filesOut, int* status, VgbProgress cb) =>
            call == TxCall.FromNw ? VgAudioB200Containers.vgb_transcode_from_nw_batch(files, lengths, types, n, options, outSizes, filesOut, status, cb, IntPtr.Zero)
            : call == TxCall.IntoNw ? VgAudioB200Containers.vgb_transcode_nw_batch(files, lengths, types, n, options, key, code, outSizes, filesOut, status, cb, IntPtr.Zero)
            : VgAudioB200Containers.vgb_transcode_batch(files, lengths, types, n, options, key, code, outSizes, filesOut, status, cb, IntPtr.Zero);

        static unsafe void Transcode(TxCall call, string[] inPaths, int[] inTypes, string[] outPaths, VgbConvertOptions options, VgbAdxKey? inAdxKey,
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
                    VgAudioB200.Check(TranscodeCall(call, inPtr, len, types, n, &options, keyPtr, codePtr, outSize, null, status, null));
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
                    VgAudioB200.Check(TranscodeCall(call, inPtr, len, types, n, &options, keyPtr, codePtr, outSize, outPtr, status, cb));
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

        // Convert.ConvertFile with the same container on both sides (.adx -> .adx or .hca -> .hca): the frames are
        // decrypted with inAdxKey (revision 8 / 9 .adx files) or inHcaKeyCode ("ciph" 56 .hca files; "ciph" 1 uses the
        // built-in table) and encrypted with the output key in options, or written in the clear - never re-encoded, so
        // the encoder's options do not apply.  options.OutType (VGB_CONTAINER_ADX or _HCA) names the reader and the writer.
        public static unsafe void Rewrite(string[] inPaths, string[] outPaths, VgbConvertOptions options, VgbAdxKey? inAdxKey,
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
                VgAudioB200.Check(VgAudioB200Containers.vgb_rewrite_batch(inPtr, len, n, &options, keyPtr, codePtr, outSize, null, status, null, IntPtr.Zero));
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
                VgAudioB200.Check(VgAudioB200Containers.vgb_rewrite_batch(inPtr, len, n, &options, keyPtr, codePtr, outSize, outPtr, status, cb, IntPtr.Zero));
                GC.KeepAlive(cb);
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
    }
}
