"""CPU restatement of AdxReader.ReadFile / ReadHeader / ReadData (Containers/Adx/AdxReader.cs:14-124, geometry of
AdxStructure.cs and the stream DeInterleave of Utilities/Interleave.cs:118-166), written apart from the product's C++
parser so that the tests can compare the two, plus the reader chain AdxReader -> ToAudioStream -> CriAdxFormat.ToPcm16
-> WaveWriter on top of the oracle's codec, encryption and WAVE writer.

Status: 0, or E_PAST (a read past the image - EndOfStreamException), E_SIGNATURE, E_DIV0 (frame size or channel count 0),
E_OFFSET (negative audio offset), E_SHORT (the audio region is shorter than AudioDataLength), E_LENGTH (a negative or
indivisible audio length), E_PURPOSE (frame sizes 1 and 2, InsertedSamples <= -samples per frame: refused on purpose)."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from oracle import pyoracle as O

E_PAST, E_SIGNATURE, E_DIV0, E_OFFSET, E_SHORT, E_LENGTH, E_PURPOSE = -20, -21, -22, -23, -24, -25, -26


def _i32(v: int) -> int:
    """C# int arithmetic: wrap to 32 bits."""
    return (v + (1 << 31)) % (1 << 32) - (1 << 31)


@dataclass
class AdxInfo:
    header_size: int = 0
    type: int = 0
    frame_size: int = 0
    bit_depth: int = 0
    channel_count: int = 0
    sample_rate: int = 0
    sample_count: int = 0
    highpass_frequency: int = 0
    version: int = 0
    revision: int = 0
    inserted_samples: int = 0
    loop_count: int = 0
    looping: int = 0
    loop_type: int = 0
    loop_start_sample: int = 0
    loop_start_byte: int = 0
    loop_end_sample: int = 0
    loop_end_byte: int = 0
    samples_per_frame: int = 0
    audio_offset: int = 0
    audio_size: int = 0
    history: List[tuple] = field(default_factory=list)


class _Past(Exception):
    pass


def adx_parse(image):
    """(status, AdxInfo) for one .adx image."""
    data = np.ascontiguousarray(image, dtype=np.uint8).tobytes()
    h = AdxInfo()
    pos = 0

    def take(n: int, signed: bool = False) -> int:
        nonlocal pos
        if pos < 0 or pos + n > len(data):
            raise _Past
        pos += n
        return int.from_bytes(data[pos - n: pos], "big", signed=signed)

    try:
        if take(2) != 0x8000:
            return E_SIGNATURE, h
        h.header_size = take(2, True)
        h.type, h.frame_size, h.bit_depth, h.channel_count = take(1), take(1), take(1), take(1)
        h.sample_rate, h.sample_count = take(4, True), take(4, True)
        h.highpass_frequency = take(2, True)
        h.version, h.revision = take(1), take(1)
        if h.version >= 4:
            pos += 4
            h.history = [(take(2, True), take(2, True)) for _ in range(h.channel_count)]
            if h.channel_count == 1:
                pos += 4
        if pos + 24 <= h.header_size:
            h.inserted_samples = take(2, True)
            h.loop_count = take(2, True)
            if h.loop_count > 0:
                h.looping = 1
                h.loop_type, h.loop_start_sample, h.loop_start_byte, h.loop_end_sample, h.loop_end_byte = (take(4, True) for _ in range(5))
    except _Past:
        return E_PAST, h
    if h.frame_size == 0:
        return E_DIV0, h
    # NibbleCountToSampleCount(2 * FrameSize, FrameSize): one frame of 2 * FrameSize nibbles, 4 of them header
    h.samples_per_frame = 2 * h.frame_size - 4
    # DivideByRoundUp: (int)Math.Ceiling((double)value / divisor); x / 0.0 is +-inf or NaN, which (int) makes int.MinValue
    frames = -(1 << 31) if h.samples_per_frame == 0 else math.ceil(h.sample_count / h.samples_per_frame)
    h.audio_size = _i32(_i32(h.frame_size * frames) * h.channel_count)
    h.audio_offset = h.header_size + 4
    if h.audio_offset < 0:
        return E_OFFSET, h
    if len(data) - h.audio_offset < h.audio_size:
        return E_SHORT, h
    if h.channel_count == 0:
        return E_DIV0, h
    if math.fmod(h.audio_size, h.channel_count) != 0 or h.audio_size < 0:  # C#'s % keeps the dividend's sign
        return E_LENGTH, h
    if h.frame_size < 3 or h.inserted_samples <= -h.samples_per_frame:
        return E_PURPOSE, h
    return 0, h


def audio_rows(image, h: AdxInfo) -> List[np.ndarray]:
    """Stream.DeInterleave(AudioDataLength, FrameSize, ChannelCount): frame-interleaved audio -> one row per channel."""
    data = np.ascontiguousarray(image, dtype=np.uint8)[h.audio_offset: h.audio_offset + h.audio_size]
    return [np.ascontiguousarray(r) for r in O.deinterleave(data, h.frame_size, h.channel_count)] if h.audio_size else \
        [np.zeros(0, np.uint8) for _ in range(h.channel_count)]


def expected_wave(image, key=None) -> Optional[np.ndarray]:
    """The reader chain on the CPU: the WAVE image the reference writes for one .adx image (None where it fails)."""
    st, h = adx_parse(image)
    if st != 0:
        return None
    rows = audio_rows(image, h)
    if h.revision in (8, 9):
        if key is None:
            return None
        rows = O.adx_crypt(rows, key, h.revision, h.frame_size)
    samples = _i32(h.sample_count - h.inserted_samples)
    loop = None
    if h.looping:
        loop = (_i32(h.loop_start_sample - h.inserted_samples), _i32(h.loop_end_sample - h.inserted_samples))
        if not (0 <= loop[0] <= samples and 0 <= loop[1] <= samples and loop[0] <= loop[1]):
            return None
    if samples < 0:
        return None
    spf, pad = h.samples_per_frame, max(h.inserted_samples, 0)
    if samples > 0 and (pad // spf + -(-samples // spf)) * h.frame_size > h.audio_size // h.channel_count:
        return None  # IndexOutOfRangeException
    # coefs[filterNum] (CriAdxCodec.cs:12,26): four rows for Fixed, one for every other type; every frame Decode walks
    # ... but only inside the sample loop: the head frame yields nothing when samples <= pad % spf, and is never checked
    first = 0 if min(spf, samples) > pad % spf else 1
    heads = int(pad / spf) * h.frame_size + np.arange(first, -(-samples // spf)) * h.frame_size
    if any(heads.size and int((r[heads] >> 5).max()) > (3 if h.type == 2 else 0) for r in rows):
        return None
    pcm = [O.adx_decode(r, samples, h.sample_rate, h.highpass_frequency, h.frame_size, h.version, 0, h.inserted_samples, h.type)
           for r in rows]
    return O.wave_write16(pcm, h.sample_rate, loop)
