// bindings/csharp/VgAudioB200Native.cs — P/Invoke declarations for libvgaudio_b200.so (include/vgaudio_b200.h).
// NOT compiled in this repository (no .NET toolchain in the build image); this is the file a VGAudio maintainer adds.
using System;
using System.Runtime.InteropServices;

namespace VGAudio.Native
{
    [StructLayout(LayoutKind.Sequential)]
    internal struct VgbGcParams
    {
        public int SampleCount;   // GcAdpcmParameters.SampleCount (-1 = whole input)
        public short History1;
        public short History2;
    }

    [UnmanagedFunctionPointer(CallingConvention.Cdecl)]
    internal delegate void VgbProgress(IntPtr user, long framesDoneDelta);

    internal static unsafe class VgAudioB200
    {
        private const string Lib = "vgaudio_b200";   // libvgaudio_b200.so / vgaudio_b200.dll

        public const int Ok = 0, EArg = -1, EData = -2, EState = -3, ECuda = -4, ENccl = -5, ENoMem = -6;

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_abi_version();
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_init(int device, uint flags);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_shutdown();
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern IntPtr vgb_last_error();
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_host_alloc(out IntPtr ptr, ulong bytes);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_host_free(IntPtr ptr);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_gcadpcm_sample_count_to_byte_count(int sampleCount);
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)] public static extern int vgb_gcadpcm_byte_count_to_sample_count(int byteCount);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_gcadpcm_coefs_batch(short** pcm, int* nSamples, int nChannels, short* coefsOut);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_gcadpcm_encode_batch(short** pcm, int* nSamples, VgbGcParams* parameters, short* coefsIn,
            int nChannels, short* coefsOut, byte** adpcmOut, VgbProgress progress, IntPtr user);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_gcadpcm_decode_batch(byte** adpcm, int* nBytes, short* coefs, VgbGcParams* parameters,
            int nChannels, short** pcmOut);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_gcadpcm_encode_frames(short* pcmInOut, int* sampleCount, short* coefs, int nFrames, byte* adpcmOut);

        /// <summary>Maps a VGB_E_* status back to the exception type the managed code path throws.</summary>
        [StructLayout(LayoutKind.Sequential)]
        internal struct VgbGcTapParams { public int SampleCount, SamplesPerSeekTableEntry, LoopStart; }

        // GcAdpcmSeekTable.CreateSeekTable + GcAdpcmLoopContext(adpcm, pcm, loopStart) without the CPU decode
        // (GcAdpcmChannelBuilder.cs:176-202)
        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern int vgb_gcadpcm_seek_entry_count(int sampleCount, int samplesPerEntry);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        public static extern unsafe int vgb_gcadpcm_seek_context_batch(byte** adpcm, int* nBytes, short* coefs, VgbGcTapParams* parameters,
            int nChannels, short** seekTableOut, short* loopContextOut);

        // GcAdpcmAlignment (GcAdpcmAlignment.cs:20-63): the loop-alignment re-encode of a batch of channels
        [StructLayout(LayoutKind.Sequential)]
        internal struct VgbGcAlignParams { public int Multiple, LoopStart, LoopEnd; }

        [StructLayout(LayoutKind.Sequential)]
        internal struct VgbGcAlignment { public int AlignmentNeeded, LoopStartAligned, SampleCountAligned; }

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        internal static extern int vgb_gcadpcm_alignment(VgbGcAlignParams* parameters, VgbGcAlignment* alignmentOut);

        [DllImport(Lib, CallingConvention = CallingConvention.Cdecl)]
        internal static extern int vgb_gcadpcm_align_batch(byte** adpcm, int* nBytes, short* coefs, VgbGcAlignParams* parameters,
            int nChannels, byte** adpcmAlignedOut, short** pcmAlignedOut);

        public static void Check(int status)
        {
            if (status == Ok) return;
            string msg = Marshal.PtrToStringAnsi(vgb_last_error()) ?? "vgaudio_b200 error";
            switch (status)
            {
                case EArg: throw new ArgumentException(msg);
                case EData: throw new System.IO.InvalidDataException(msg);
                case EState: throw new InvalidOperationException(msg);
                case ENoMem: throw new OutOfMemoryException(msg);
                default: throw new InvalidOperationException(msg);   // VGB_E_CUDA / VGB_E_NCCL: no CPU fallback
            }
        }
    }
}
