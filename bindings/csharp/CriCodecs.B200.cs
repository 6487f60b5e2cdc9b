// bindings/csharp/CriCodecs.B200.cs — P/Invoke declarations and drop-in bodies for the CRI ADX and CRI HCA paths.
// NOT compiled in this repository (no .NET toolchain in the build image).
using System;
using System.Runtime.InteropServices;
using VGAudio.Codecs.CriAdx;
using VGAudio.Codecs.CriHca;
using VGAudio.Formats.Pcm16;

namespace VGAudio.Native
{
    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbAdxParams   // CriAdxParameters (Codecs/CriAdx/CriAdxParameters.cs:3-13)
    {
        public int SampleRate, HighpassFrequency, FrameSize, Version, History, Padding, Type, Filter;
    }

    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbHcaParams   // CriHcaParameters (Codecs/CriHca/CriHcaParameters.cs:3-15)
    {
        public int Quality, Bitrate, LimitBitrate, ChannelCount, SampleRate, SampleCount, Looping, LoopStart, LoopEnd;
    }

    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbHcaInfo     // HcaInfo (Codecs/CriHca/HcaInfo.cs:5-48)
    {
        public int ChannelCount, SampleRate, SampleCount, FrameCount, InsertedSamples, AppendedSamples;
        public int HeaderSize, FrameSize, MinResolution, MaxResolution, TrackCount, ChannelConfig;
        public int TotalBandCount, BaseBandCount, StereoBandCount, HfrBandCount, BandsPerHfrGroup, HfrGroupCount;
        public int Bitrate;
        public int Looping, LoopStartFrame, LoopEndFrame, PreLoopSamples, PostLoopSamples;  // HcaInfo.cs:29-33
        public int UseAthCurve;  // HcaInfo.cs:38 (old files: the decoder adds the ATH curve to the noise level)
    }

    internal static unsafe class VgAudioB200Cri
    {
        private const string Lib = "vgaudio_b200";

        // InterleaveExtensions.Interleave / DeInterleave for byte payloads (Utilities/Interleave.cs:9-41, :81-117)
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_interleave(byte** inputs, int count, int inSize, int interleaveSize, int outSize, byte* output);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_deinterleave(byte* input, int length, int interleaveSize, int count, int outSize, byte** outputs);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_calculate_coefficients(int highpassFrequency, int sampleRate, short* coefsOut);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_encoded_byte_count(int pcmLength, int padding, int frameSize);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_encode_batch(short** pcm, int* nSamples, VgbAdxParams* parameters, int nChannels,
            short* historyOut, byte** adpcmOut, VgbProgress progress, IntPtr user);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_decode_batch(byte** adpcm, int* nBytes, int* sampleCount, VgbAdxParams* parameters,
            int nChannels, short** pcmOut);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern ulong vgb_adx_decode_workspace_bytes(int* sampleCount, VgbAdxParams* parameters, int nChannels);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_decode_dev(byte* dAdpcm, long* adpcmOffset, int* nBytes, int* sampleCount, VgbAdxParams* parameters,
            int nChannels, short* dPcm, long* pcmOffset, void* dWorkspace, ulong workspaceBytes, IntPtr cudaStream);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_decode_dev_status(void* dWorkspace, int nChannels, IntPtr cudaStream);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_adx_debug_decode_stats(ulong* output, int n);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_hca_query(VgbHcaParams* parameters, VgbHcaInfo* infoOut);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_hca_encode_batch(short** pcm, VgbHcaParams* parameters, int nStreams, VgbHcaInfo* infoOut,
            byte** framesOut, VgbProgress progress, IntPtr user);
    }
}

namespace VGAudio.Formats.CriAdx
{
    public partial class CriAdxFormat
    {
        // replaces the Parallel.For of CriAdxFormat.EncodeFromPcm16 (Formats/CriAdx/CriAdxFormat.cs:67-81):
        // channelConfig is built per channel exactly as at :69-78; the History each CriAdxCodec.Encode writes back into
        // its config (CriAdxCodec.cs:73, read at CriAdxFormat.cs:80) comes back in historyOut.
        private static unsafe CriAdxChannel[] EncodeChannelsB200(Pcm16Format pcm16, CriAdxParameters config, int alignmentSamples)
        {
            int n = pcm16.ChannelCount;
            var adpcm = new byte[n][];
            var history = new short[n];
            var pins = new GCHandle[2 * n];
            var inPtr = stackalloc short*[n];
            var outPtr = stackalloc byte*[n];
            var lens = stackalloc int[n];
            var prm = stackalloc Native.VgbAdxParams[n];
            Native.VgbProgress cb = config.Progress == null ? null : (u, d) => config.Progress.ReportAdd((int)d);
            try
            {
                for (int i = 0; i < n; i++)
                {
                    short[] pcm = pcm16.Channels[i];
                    adpcm[i] = new byte[Native.VgAudioB200Cri.vgb_adx_encoded_byte_count(pcm.Length, alignmentSamples, config.FrameSize)];
                    pins[2 * i] = GCHandle.Alloc(pcm, GCHandleType.Pinned);
                    pins[2 * i + 1] = GCHandle.Alloc(adpcm[i], GCHandleType.Pinned);
                    inPtr[i] = (short*)pins[2 * i].AddrOfPinnedObject();
                    outPtr[i] = (byte*)pins[2 * i + 1].AddrOfPinnedObject();
                    lens[i] = pcm.Length;
                    prm[i] = new Native.VgbAdxParams
                    {
                        SampleRate = pcm16.SampleRate, HighpassFrequency = 500, FrameSize = config.FrameSize, Version = config.Version,
                        Padding = alignmentSamples, Type = (int)config.Type, Filter = config.Filter
                    };
                }
                fixed (short* h = history)
                    Native.VgAudioB200.Check(Native.VgAudioB200Cri.vgb_adx_encode_batch(inPtr, lens, prm, n, h, outPtr, cb, IntPtr.Zero));
            }
            finally { foreach (var h in pins) if (h.IsAllocated) h.Free(); }
            GC.KeepAlive(cb);
            var channels = new CriAdxChannel[n];
            for (int i = 0; i < n; i++) channels[i] = new CriAdxChannel(adpcm[i], history[i], config.Version);   // :80
            return channels;
        }
    }
}

namespace VGAudio.Formats.CriHca
{
    public partial class CriHcaFormat
    {
        // replaces the frame loop of CriHcaFormat.EncodeFromPcm16 (Formats/CriHca/CriHcaFormat.cs:43-81), looping
        // streams included: returns byte[FrameCount][FrameSize] and the HcaInfo CriHcaEncoder.Initialize computes.
        private static unsafe byte[][] EncodeFramesB200(Pcm16Format pcm16, CriHcaParameters config, out Native.VgbHcaInfo info)
        {
            int nch = pcm16.ChannelCount;
            var prm = new Native.VgbHcaParams
            {
                Quality = (int)config.Quality, Bitrate = config.Bitrate, LimitBitrate = config.LimitBitrate ? 1 : 0,
                ChannelCount = nch, SampleRate = pcm16.SampleRate, SampleCount = pcm16.SampleCount,
                Looping = pcm16.Looping ? 1 : 0, LoopStart = pcm16.LoopStart, LoopEnd = pcm16.LoopEnd
            };
            Native.VgbHcaInfo h;
            Native.VgAudioB200.Check(Native.VgAudioB200Cri.vgb_hca_query(&prm, &h));
            var slab = new byte[h.FrameCount * h.FrameSize];
            var pins = new GCHandle[nch];
            var inPtr = stackalloc short*[nch];
            try
            {
                for (int c = 0; c < nch; c++)
                {
                    pins[c] = GCHandle.Alloc(pcm16.Channels[c], GCHandleType.Pinned);
                    inPtr[c] = (short*)pins[c].AddrOfPinnedObject();
                }
                fixed (byte* o = slab)
                {
                    byte* op = o;
                    Native.VgAudioB200.Check(Native.VgAudioB200Cri.vgb_hca_encode_batch(inPtr, &prm, 1, &h, &op, null, IntPtr.Zero));
                }
            }
            finally { foreach (var p in pins) if (p.IsAllocated) p.Free(); }
            var audio = new byte[h.FrameCount][];
            for (int f = 0; f < h.FrameCount; f++)
            {
                audio[f] = new byte[h.FrameSize];
                Buffer.BlockCopy(slab, f * h.FrameSize, audio[f], 0, h.FrameSize);
            }
            info = h;
            return audio;
        }
    }
}
