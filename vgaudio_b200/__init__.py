"""vgaudio_b200 — B200-native batch engine for VGAudio's per-channel codec hot path.

Host-side mirror of the reference's interface for that path (names follow the reference):
  codecs.gcadpcm : GcAdpcmMath helpers, GcAdpcmCoefficients, GcAdpcmEncoder, GcAdpcmDecoder, GcAdpcmParameters
  formats        : Pcm16Format, GcAdpcmChannel, GcAdpcmFormat (.encode_from_pcm16 / .to_pcm16), align_loops
  criadx, crihca : CriAdxParameters / CriHcaParameters, encode / decode (+ _batch)
  interleave     : InterleaveExtensions.Interleave / DeInterleave for byte payloads
All arithmetic runs in libvgaudio_b200.so (CUDA, sm_90a) through the C ABI in include/vgaudio_b200.h.
"""
from ._native import VgbError, lib  # noqa: F401  (fails loudly when the native library is missing)
from . import gcadpcm, criadx, crihca, formats, interleave  # noqa: F401
