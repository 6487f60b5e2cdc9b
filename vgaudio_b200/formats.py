"""Host-side mirror of the reference's format layer for the GC-ADPCM path (the drop-in boundary).

  Pcm16Format      Formats/Pcm16/Pcm16Format.cs:12-50        short[][] Channels + SampleRate
  GcAdpcmChannel   Formats/GcAdpcm/GcAdpcmChannel.cs:6-29    Adpcm, Coefs, SampleCount
  GcAdpcmFormat    Formats/GcAdpcm/GcAdpcmFormat.cs:14-74    EncodeFromPcm16 (:58-74), ToPcm16 (:42-54)

The reference runs `Parallel.For(0, ChannelCount, i => EncodeChannel(...))`; here the whole loop is ONE batched
call into libvgaudio_b200.so.  The post-encode channel rebuild of GcAdpcmChannelBuilder (SURVEY.md §8f rank 1) is
`align_loops` below (GcAdpcmAlignment) and `gcadpcm.seek_table_and_loop_context`.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from . import gcadpcm
from .gcadpcm import GcAdpcmParameters


@dataclass
class Pcm16Format:
    channels: List[np.ndarray]
    sample_rate: int = 48000

    def __post_init__(self):
        if isinstance(self.channels, np.ndarray) and self.channels.ndim == 2:
            base = np.ascontiguousarray(self.channels, dtype=np.int16)
            self.channels = [base[i] for i in range(base.shape[0])]
        else:
            self.channels = [np.ascontiguousarray(c, dtype=np.int16) for c in self.channels]
        lengths = {len(c) for c in self.channels}
        if len(lengths) > 1:  # Pcm16FormatBuilder.cs:14-28 throws InvalidDataException
            raise ValueError("All channels must have the same sample count")

    @property
    def channel_count(self) -> int:
        return len(self.channels)

    @property
    def sample_count(self) -> int:
        return len(self.channels[0]) if self.channels else 0


@dataclass
class GcAdpcmChannel:
    adpcm: np.ndarray
    coefs: np.ndarray
    sample_count: int
    history1: int = 0  # StartContext.Hist1
    history2: int = 0

    def __post_init__(self):
        # GcAdpcmChannel.cs:33-36
        if len(self.adpcm) < gcadpcm.sample_count_to_byte_count(self.sample_count):
            raise ValueError("Audio array length is too short for the specified number of samples.")


@dataclass
class GcAdpcmFormat:
    channels: List[GcAdpcmChannel] = field(default_factory=list)
    sample_rate: int = 48000

    @property
    def channel_count(self) -> int:
        return len(self.channels)

    @property
    def sample_count(self) -> int:
        return self.channels[0].sample_count if self.channels else 0

    def encode_from_pcm16(self, pcm16: Pcm16Format, config: Optional[GcAdpcmParameters] = None) -> "GcAdpcmFormat":
        """GcAdpcmFormat.EncodeFromPcm16(Pcm16Format, GcAdpcmParameters) (GcAdpcmFormat.cs:58-74)."""
        config = config or GcAdpcmParameters()
        if config.progress:
            pass  # SetTotal(frameCount * channels) is implied: the deltas reported sum to it (GcAdpcmFormat.cs:62-63)
        coefs, adpcm = gcadpcm.encode_batch(pcm16.channels, configs=[config] * pcm16.channel_count,
                                            progress=config.progress)
        chans = [GcAdpcmChannel(adpcm[i], coefs[i].copy(), pcm16.sample_count) for i in range(pcm16.channel_count)]
        return GcAdpcmFormat(chans, pcm16.sample_rate)

    def to_pcm16(self) -> Pcm16Format:
        """GcAdpcmFormat.ToPcm16() (GcAdpcmFormat.cs:42-54 -> GcAdpcmChannel.GetPcmAudio :57-60)."""
        if not self.channels:
            return Pcm16Format([], self.sample_rate)
        cfg = [GcAdpcmParameters(c.sample_count, c.history1, c.history2) for c in self.channels]
        pcm = gcadpcm.decode_batch([c.adpcm for c in self.channels], np.stack([c.coefs for c in self.channels]), cfg)
        return Pcm16Format(pcm, self.sample_rate)


# ---- GcAdpcmAlignment (Formats/GcAdpcm/GcAdpcmAlignment.cs:20-63) -------------------------------------------------
@dataclass
class GcAdpcmAlignment:
    alignment_needed: bool
    loop_start: int
    loop_end: int
    loop_start_aligned: int = 0
    sample_count_aligned: int = 0
    adpcm_aligned: Optional[np.ndarray] = None
    pcm_aligned: Optional[np.ndarray] = None


def align_loops(adpcm_channels, coefs, multiple: int, loop_start: int, loop_end: int) -> List[GcAdpcmAlignment]:
    """GcAdpcmAlignment(multiple, loopStart, loopEnd, adpcm, coefs) for every channel of a format (the channels of one
    stream share the loop points): one native call, vgb_gcadpcm_align_batch."""
    n = len(adpcm_channels)
    needed, loop_start_aligned, sample_count_aligned = gcadpcm.alignment(multiple, loop_start, loop_end)
    if not needed or n == 0:
        return [GcAdpcmAlignment(False, loop_start, loop_end) for _ in range(n)]
    adpcm_aligned, pcm_aligned = gcadpcm.align_batch(adpcm_channels, coefs, (multiple, loop_start, loop_end))
    return [GcAdpcmAlignment(True, loop_start, loop_end, loop_start_aligned, sample_count_aligned, adpcm_aligned[c],
                             pcm_aligned[c]) for c in range(n)]
