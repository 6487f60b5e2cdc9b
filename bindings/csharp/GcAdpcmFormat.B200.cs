// bindings/csharp/GcAdpcmFormat.B200.cs — drop-in bodies for the hot paths of
// src/VGAudio/Formats/GcAdpcm/GcAdpcmFormat.cs.  Everything around them (builders, loop handling, containers) is
// untouched: the Parallel.For over channels (GcAdpcmFormat.cs:65-68, :45-48 and :31-38) becomes ONE batched native call.
// GcAdpcmAlignment and GcAdpcmChannelBuilder gain `partial` and the internal members below, and GetAlignment's
// `new GcAdpcmAlignment(LoopAlignmentMultiple, LoopStart, LoopEnd, Adpcm, Coefs)` (GcAdpcmChannelBuilder.cs:153) becomes
// `BatchAlignment ?? new GcAdpcmAlignment(...)`: the fresh-alignment path then runs as before, including the
// AlignedAdpcm / AlignedPcm / AlignedLoopStart assignments (:155-160) that the loop context and seek table read.  (Handing
// the result over as PreviousAlignment would skip those assignments and change the loop context.)
// NOT compiled here (no .NET toolchain in the build image).
using System;
using System.Collections.Generic;
using System.Runtime.InteropServices;
using System.Threading.Tasks;
using VGAudio.Codecs.GcAdpcm;
using VGAudio.Formats.Pcm16;
using VGAudio.Native;
using static VGAudio.Codecs.GcAdpcm.GcAdpcmMath;

namespace VGAudio.Formats.GcAdpcm
{
    internal partial class GcAdpcmAlignment
    {
        // The result of vgb_gcadpcm_align_batch for one channel: what the public constructor (:20-63) computes
        internal GcAdpcmAlignment(int multiple, int loopStart, int loopEnd, int loopStartAligned, int sampleCountAligned,
            byte[] adpcmAligned, short[] pcmAligned)
        {
            AlignmentMultiple = multiple;
            LoopStart = loopStart;
            LoopEnd = loopEnd;
            AlignmentNeeded = true;
            LoopStartAligned = loopStartAligned;
            SampleCountAligned = sampleCountAligned;
            AdpcmAligned = adpcmAligned;
            PcmAligned = pcmAligned;
        }
    }

    public partial class GcAdpcmChannelBuilder
    {
        // set by the GcAdpcmFormat constructor below for a channel whose alignment one batched native call computed
        internal GcAdpcmAlignment BatchAlignment { get; set; }
    }

    public partial class GcAdpcmFormat
    {
        // replaces the body of internal GcAdpcmFormat(GcAdpcmFormatBuilder b)  (GcAdpcmFormat.cs:27-40).  Every channel
        // whose builder would run new GcAdpcmAlignment in GetAlignment (GcAdpcmChannelBuilder.cs:148-163: looping, no
        // reusable PreviousAlignment, loop start not on the multiple) gets it from one batched call instead, through
        // BatchAlignment; the builder's own flow (loop context, seek table, PreviousAlignment reuse) stays managed.
        internal unsafe GcAdpcmFormat(GcAdpcmFormatBuilder b) : base(b)
        {
            Channels = b.Channels;
            AlignmentMultiple = b.AlignmentMultiple;

            int n = Channels.Length;
            var builders = new GcAdpcmChannelBuilder[n];
            var todo = new List<int>();
            for (int i = 0; i < n; i++)
            {
                builders[i] = Channels[i]
                    .GetCloneBuilder()
                    .WithLoop(Looping, UnalignedLoopStart, UnalignedLoopEnd)
                    .WithLoopAlignment(b.AlignmentMultiple);
                GcAdpcmChannelBuilder cb = builders[i];
                if (cb.Looping && !cb.PreviousAlignmentIsValid() && !Utilities.Helpers.LoopPointsAreAligned(cb.LoopStart, cb.LoopAlignmentMultiple))
                    todo.Add(i);
            }

            int m = todo.Count;
            if (m > 0)
            {
                var prm = new VgAudioB200.VgbGcAlignParams[m];
                var geo = new VgAudioB200.VgbGcAlignment[m];
                var coefs = new short[m * 16];
                var adpcmOut = new byte[m][];
                var pcmOut = new short[m][];
                var pins = new GCHandle[3 * m];
                var inPtr = new IntPtr[m];
                var adpcmPtr = new IntPtr[m];
                var pcmPtr = new IntPtr[m];
                var lens = new int[m];
                try
                {
                    for (int k = 0; k < m; k++)
                    {
                        GcAdpcmChannelBuilder cb = builders[todo[k]];
                        prm[k] = new VgAudioB200.VgbGcAlignParams { Multiple = cb.LoopAlignmentMultiple, LoopStart = cb.LoopStart, LoopEnd = cb.LoopEnd };
                        fixed (VgAudioB200.VgbGcAlignParams* p = &prm[k])
                        fixed (VgAudioB200.VgbGcAlignment* g = &geo[k])
                            VgAudioB200.Check(VgAudioB200.vgb_gcadpcm_alignment(p, g));
                        adpcmOut[k] = new byte[SampleCountToByteCount(geo[k].SampleCountAligned)];   // :33-34
                        pcmOut[k] = new short[geo[k].SampleCountAligned];
                        Array.Copy(cb.Coefs, 0, coefs, k * 16, 16);
                        pins[3 * k] = GCHandle.Alloc(cb.Adpcm, GCHandleType.Pinned);
                        pins[3 * k + 1] = GCHandle.Alloc(adpcmOut[k], GCHandleType.Pinned);
                        pins[3 * k + 2] = GCHandle.Alloc(pcmOut[k], GCHandleType.Pinned);
                        inPtr[k] = pins[3 * k].AddrOfPinnedObject();
                        adpcmPtr[k] = pins[3 * k + 1].AddrOfPinnedObject();
                        pcmPtr[k] = pins[3 * k + 2].AddrOfPinnedObject();
                        lens[k] = cb.Adpcm.Length;
                    }
                    fixed (IntPtr* ip = inPtr) fixed (IntPtr* ap = adpcmPtr) fixed (IntPtr* pp = pcmPtr)
                    fixed (int* l = lens) fixed (short* c = coefs) fixed (VgAudioB200.VgbGcAlignParams* p = prm)
                        VgAudioB200.Check(VgAudioB200.vgb_gcadpcm_align_batch((byte**)ip, l, c, p, m, (byte**)ap, (short**)pp));
                }
                finally { foreach (var h in pins) if (h.IsAllocated) h.Free(); }

                for (int k = 0; k < m; k++)
                {
                    builders[todo[k]].BatchAlignment = new GcAdpcmAlignment(prm[k].Multiple, prm[k].LoopStart, prm[k].LoopEnd,
                        geo[k].LoopStartAligned, geo[k].SampleCountAligned, adpcmOut[k], pcmOut[k]);
                }
            }

            Parallel.For(0, n, i => { Channels[i] = builders[i].Build(); });                  // :31-38, minus the re-encodes
        }

        // replaces GcAdpcmFormat.EncodeFromPcm16(Pcm16Format, GcAdpcmParameters)  (GcAdpcmFormat.cs:58-74)
        public override unsafe GcAdpcmFormat EncodeFromPcm16(Pcm16Format pcm16, GcAdpcmParameters config)
        {
            int n = pcm16.ChannelCount;
            var channels = new GcAdpcmChannel[n];
            int frameCount = pcm16.SampleCount.DivideByRoundUp(14) * n;
            config?.Progress?.SetTotal(frameCount);                                  // :62-63

            int sampleCount = config == null || config.SampleCount == -1 ? pcm16.SampleCount : config.SampleCount;
            var coefs = new short[n * 16];
            var adpcm = new byte[n][];
            var pins = new GCHandle[2 * n];                                           // short[][] / byte[][] are not blittable
            var pcmPtr = stackalloc short*[n];
            var outPtr = stackalloc byte*[n];
            var lens = stackalloc int[n];
            var prm = stackalloc VgbGcParams[n];
            VgbProgress cb = config?.Progress == null ? null : (u, d) => config.Progress.ReportAdd((int)d);
            try
            {
                for (int i = 0; i < n; i++)
                {
                    adpcm[i] = new byte[SampleCountToByteCount(sampleCount)];         // GcAdpcmEncoder.cs:18
                    pins[2 * i] = GCHandle.Alloc(pcm16.Channels[i], GCHandleType.Pinned);
                    pins[2 * i + 1] = GCHandle.Alloc(adpcm[i], GCHandleType.Pinned);
                    pcmPtr[i] = (short*)pins[2 * i].AddrOfPinnedObject();
                    outPtr[i] = (byte*)pins[2 * i + 1].AddrOfPinnedObject();
                    lens[i] = pcm16.Channels[i].Length;
                    prm[i] = new VgbGcParams { SampleCount = config?.SampleCount ?? -1, History1 = config?.History1 ?? 0, History2 = config?.History2 ?? 0 };
                }
                fixed (short* c = coefs)
                    VgAudioB200.Check(VgAudioB200.vgb_gcadpcm_encode_batch(pcmPtr, lens, prm, null, n, c, outPtr, cb, IntPtr.Zero));
            }
            finally { foreach (var h in pins) if (h.IsAllocated) h.Free(); }
            GC.KeepAlive(cb);

            for (int i = 0; i < n; i++)
            {
                var c = new short[16];
                Array.Copy(coefs, i * 16, c, 0, 16);
                channels[i] = new GcAdpcmChannel(adpcm[i], c, pcm16.SampleCount);     // EncodeChannel :134
            }
            return new GcAdpcmFormatBuilder(channels, pcm16.SampleRate)
                .WithLoop(pcm16.Looping, pcm16.LoopStart, pcm16.LoopEnd)
                .WithTracks(pcm16.Tracks)
                .Build();                                                             // :70-73 unchanged
        }

        // replaces GcAdpcmFormat.ToPcm16()  (GcAdpcmFormat.cs:42-54) for channels that need decoding
        public override unsafe Pcm16Format ToPcm16()
        {
            int n = Channels.Length;
            var pcm = new short[n][];
            var coefs = new short[n * 16];
            var pins = new GCHandle[2 * n];
            var inPtr = stackalloc byte*[n];
            var outPtr = stackalloc short*[n];
            var lens = stackalloc int[n];
            var prm = stackalloc VgbGcParams[n];
            try
            {
                for (int i = 0; i < n; i++)
                {
                    byte[] a = Channels[i].GetAdpcmAudio();
                    pcm[i] = new short[Channels[i].SampleCount];
                    Array.Copy(Channels[i].Coefs, 0, coefs, i * 16, 16);
                    pins[2 * i] = GCHandle.Alloc(a, GCHandleType.Pinned);
                    pins[2 * i + 1] = GCHandle.Alloc(pcm[i], GCHandleType.Pinned);
                    inPtr[i] = (byte*)pins[2 * i].AddrOfPinnedObject();
                    outPtr[i] = (short*)pins[2 * i + 1].AddrOfPinnedObject();
                    lens[i] = a.Length;
                    prm[i] = new VgbGcParams { SampleCount = Channels[i].SampleCount, History1 = Channels[i].StartContext.Hist1, History2 = Channels[i].StartContext.Hist2 };
                }
                fixed (short* c = coefs)
                    VgAudioB200.Check(VgAudioB200.vgb_gcadpcm_decode_batch(inPtr, lens, c, prm, n, outPtr));
            }
            finally { foreach (var h in pins) if (h.IsAllocated) h.Free(); }
            return new Pcm16FormatBuilder(pcm, SampleRate).WithLoop(Looping, LoopStart, LoopEnd).WithTracks(Tracks).Build();
        }
    }
}
