"""CPU restatement of HcaReader.ReadHcaHeader (Containers/Hca/HcaReader.cs:59-121) plus the frame region ReadFile /
ReadHcaData read behind the header (:27-31, :123-138), written apart from the product's C++ parser so that the tests can
compare the two.  Returns the oracle's HcaInfo, so its output feeds oracle.hca_decode directly.

Status: 0, or E_TRUNCATED (a read past the image - EndOfStreamException - or fewer than frame_count * frame_size bytes
behind the header), E_NOT_HCA (signature), E_CHUNK (an id the reader does not know - NotSupportedException), E_HEADER
(negative header size or frame count, a frame size below 2 bytes)."""
from __future__ import annotations

import numpy as np

from oracle import pyoracle as O

E_TRUNCATED, E_NOT_HCA, E_CHUNK, E_HEADER = -2, -13, -14, -15


class _Past(Exception):
    """A BinaryReader read past the end of the stream."""


def _i32(v: int) -> int:
    """C# int arithmetic: wrap to 32 bits."""
    return (v + (1 << 31)) % (1 << 32) - (1 << 31)


def hca_parse(image):
    """(status, O.HcaInfo, ciph) for one .hca image; ciph is the "ciph" chunk's value (0 without one)."""
    data = np.ascontiguousarray(image, dtype=np.uint8).tobytes()
    info, ciph = O.HcaInfo(), 0
    pos = 0

    def take(n: int) -> bytes:
        nonlocal pos
        if pos + n > len(data):
            raise _Past
        pos += n
        return data[pos - n: pos]

    def u(n: int) -> int:
        return int.from_bytes(take(n), "big")

    def s(n: int) -> int:
        return int.from_bytes(take(n), "big", signed=True)

    def chunk_id() -> bytes:  # ReadChunkId (:226-236): every byte masked with 0x7f
        return bytes(b & 0x7F for b in take(4))

    try:
        sig = chunk_id()
        version = s(2)
        info.header_size = s(2)
        if sig != b"HCA\0":
            return E_NOT_HCA, info, ciph
        has_ath = False
        while pos < info.header_size:
            cid = chunk_id()
            if cid == b"fmt\0":  # :140-149
                info.channel_count = u(1)
                info.sample_rate = u(1) << 16 | u(2)
                info.frame_count = s(4)
                info.inserted_samples = s(2)
                info.appended_samples = s(2)
                info.sample_count = _i32(info.frame_count * 1024 - info.inserted_samples - info.appended_samples)
            elif cid == b"comp":  # :151-164
                info.frame_size = s(2)
                (info.min_resolution, info.max_resolution, info.track_count, info.channel_config, info.total_band_count,
                 info.base_band_count, info.stereo_band_count, info.bands_per_hfr_group) = take(8)
                take(2)  # Reserved1, Reserved2
            elif cid == b"dec\0":  # :166-187
                info.frame_size = s(2)
                info.min_resolution, info.max_resolution = take(2)
                info.total_band_count = u(1) + 1
                info.base_band_count = u(1) + 1
                packed = u(1)
                info.track_count, info.channel_config = packed >> 4, packed & 0xF
                if u(1) == 0:  # DecStereoType
                    info.base_band_count = info.total_band_count
                else:
                    info.stereo_band_count = info.total_band_count - info.base_band_count
            elif cid == b"loop":  # :189-197, HcaInfo.LoopEndSample (HcaInfo.cs:36)
                info.looping = 1
                info.loop_start_frame, info.loop_end_frame = s(4), s(4)
                info.pre_loop_samples, info.post_loop_samples = s(2), s(2)
                loop_end = _i32((info.loop_end_frame + 1) * 1024 - info.post_loop_samples - info.inserted_samples)
                info.sample_count = min(info.sample_count, loop_end)
            elif cid == b"ath\0":  # :199-202
                info.use_ath_curve = int(s(2) == 1)
                has_ath = True
            elif cid == b"ciph":
                ciph = s(2)
            elif cid == b"rva\0":  # a float32 volume
                take(4)
            elif cid == b"vbr\0":
                take(4)
            elif cid == b"comm":  # :220-224: Position++, then ReadUTF8Z, which fails when it starts at the end of the stream
                pos += 1
                if pos >= len(data):
                    raise _Past
                pos = info.header_size
            elif cid == b"pad\0":
                pos = info.header_size
            else:
                return E_CHUNK, info, ciph
    except _Past:
        return E_TRUNCATED, info, ciph
    if version < 0x0200 and not has_ath:
        info.use_ath_curve = 1
    if info.track_count < 1:
        info.track_count = 1
    if info.bands_per_hfr_group > 0:  # HcaInfo.CalculateHfrValues (HcaInfo.cs:50-56), DivideByRoundUp
        info.hfr_band_count = info.total_band_count - info.base_band_count - info.stereo_band_count
        info.hfr_group_count = -(-info.hfr_band_count // info.bands_per_hfr_group)
    if info.header_size < 0 or info.frame_count < 0 or (info.frame_count > 0 and info.frame_size < 2):
        return E_HEADER, info, ciph
    if info.frame_count * max(info.frame_size, 0) > len(data) - info.header_size:
        return E_TRUNCATED, info, ciph
    return 0, info, ciph
