"""CPU restatement of the NintendoWare wave and prefetch readers, written apart from the product's C++ so that the
tests can compare the two: BrwavReader (Containers/NintendoWare/BrwavReader.cs, Structures/RwavWaveInfo.cs,
RwavChannelInfo.cs, BrstmHeader.ReadBrwav), the whole BCFstmReader.ReadFile (BCFstmReader.cs:14-288: wave info block,
wave data block, prefetch data block) and Common.ToAudioStream (Common.cs:45-116) with the checks of the format
builders it calls (GcAdpcmChannel, Pcm16FormatBuilder, Pcm8FormatBuilder, WithLoop), then ToPcm16 -> WaveWriter on the
oracle's GC-ADPCM decoder, de-interleave and WAVE writer.

It sits on nw_reader_oracle's binary reader and primitives.  For the stream types (4..6) it is nw_reader_oracle.

parse() returns (0, info) or (E_DATA, message); info.rows is None for interleaved audio, else [(offset, length)] per
channel, what ReadBytes returned."""
from __future__ import annotations

from typing import List, Optional

import numpy as np

import nw_reader_oracle as R
from nw_reader_oracle import E_ARG, E_DATA, _Fail, _R, _i32, _is
from oracle import pyoracle as O

BRWAV, BCWAV, BFWAV, BCSTP, BFSTP = 9, 10, 11, 12, 13
STREAMS = (R.BRSTM, R.BCSTM, R.BFSTM)
TYPES = STREAMS + (BRWAV, BCWAV, BFWAV, BCSTP, BFSTP)


def _cs_trunc_div(a: int, b: int) -> int:
    return R._cs_div(a, b)


def nibble_to_sample(n: int) -> int:
    q = _cs_trunc_div(n, 16)
    return _i32(14 * q + (n - 16 * q) - 2)


def _nibble_count_to_samples(n: int) -> int:
    q = _cs_trunc_div(n, 16)
    extra = n - 16 * q
    return _i32(14 * q + (0 if extra < 2 else extra - 2))


def bytes_to_samples(n: int, codec: int) -> int:
    if codec == 2:
        return _nibble_count_to_samples(_i32(n * 2))
    return _cs_trunc_div(n, 2) if codec == 1 else (n if codec == 0 else 0)


class Info(R.NwInfo):
    rows: Optional[list] = None


def _new_info() -> Info:
    h = Info()
    h.rows = None
    return h


def _wave_rows(r: _R, h: Info, offsets: Optional[List[int]]):
    """ReadDataBlock's wave path: every channel is ReadBytes(SamplesToBytes(SampleCount)) at the payload + its offset."""
    h.output_size = R.samples_to_bytes(h.sample_count, h.codec)
    if h.channel_count > 0 and h.output_size < 0:
        raise _Fail("Non-negative number required.")
    base = r.pos
    h.rows = []
    for c in range(h.channel_count):
        if offsets is None:
            raise _Fail("Object reference not set to an instance of an object.")
        if c >= len(offsets):
            raise _Fail("Index was out of range.")
        r.seek(_i32(base + offsets[c]))
        at = r.pos
        h.rows.append((at, r.read_bytes(h.output_size)))
    h.interleave_size = 0
    held = [(a, g) for a, g in h.rows if g > 0]
    h.audio_offset = min(a for a, _ in held) if held else 0
    h.audio_length = (max(a + g for a, g in held) - h.audio_offset) if held else 0


def _channel_table(r: _R, h: Info, wave_offsets: List[int]):
    """ChannelInfo.ReadBfstm."""
    base = r.pos
    count = r.take(4, True)
    refs = [r.ref(base) for _ in range(max(count, 0))]
    for c in refs:
        r.seek(c["abs"])
        if _is(c, 0x7100):
            wave_offsets.append(r.ref(0)["offset"])
        a = r.ref(c["abs"])
        if _is(a, 0x0300):
            r.seek(a["abs"])
            h.channels.append(R._channel(r, False))


def _brwav(r: _R, h: Info):
    if r.magic() != b"RWAV":
        raise _Fail("File has no RWAV header")
    bom = r.take(2)
    if bom != 0xFEFF:
        raise _Fail(f"Expected 65279, but got {bom} at offset 0x4")
    h.version = (r.take(1) << 24) | (r.take(1) << 16)
    if len(r.d) < r.take(4, True):
        raise _Fail("Actual file length is less than stated length")
    r.take(2, True), r.take(2, True)
    head_off, head_size, data_off, data_size = (r.take(4, True) for _ in range(4))
    r.seek(head_off)
    if r.magic() != b"INFO":
        raise _Fail("Unknown or invalid INFO block")
    if r.take(4, True) != head_size:
        raise _Fail("HEAD block size in RWAV header doesn't match size in HEAD header")
    base = r.pos
    h.codec, h.looping, h.channel_count = r.take(1), int(r.take(1) != 0), r.take(1)
    r.pos += 1
    h.sample_rate = r.take(2)
    r.pos += 2
    h.loop_start = nibble_to_sample(r.take(4, True))
    h.sample_count = nibble_to_sample(r.take(4, True))
    table = r.take(4, True)
    r.take(4, True)
    r.seek(_i32(base + table))
    info_offsets = [r.take(4, True) for _ in range(h.channel_count)]
    audio = []
    for off in info_offsets:
        r.seek(_i32(base + off))
        audio.append(r.take(4, True))
        adpcm = r.take(4, True)
        for _ in range(4):
            r.take(4, True)
        r.seek(_i32(base + adpcm))
        h.channels.append(R._channel(r, True))
    r.seek(data_off)
    if r.magic() != b"DATA":
        raise _Fail("Unknown or invalid DATA block")
    if r.take(4, True) != data_size:
        raise _Fail("DATA block size in main header doesn't match size in DATA header")
    _wave_rows(r, h, audio)
    h.big_endian = 1


def _bcfstm(r: _R, h: Info):
    """BCFstmReader.ReadFile, every path."""
    if r.magic() not in (b"CSTM", b"FSTM", b"CWAV", b"FWAV", b"CSTP", b"FSTP"):
        raise _Fail("File has no CSTM or FSTM header")
    bom = r.take(2, be=False)
    if bom not in (0xFEFF, 0xFFFE):
        raise _Fail("File has no byte order mark")
    r.be = bom == 0xFFFE
    r.pos -= 2
    h.big_endian = int(r.be)
    r.take(2), r.take(2, True)
    h.version = v = r.take(4)
    if len(r.d) < r.take(4, True):
        raise _Fail("Actual file length is less than stated length")
    count = r.take(2, True)
    r.pos += 2
    blocks = [r.ref(0, True) for _ in range(count)]

    def first(*types):
        return next((b for b in blocks if b["type"] in types), None)

    info = first(0x4000, 0x7000)
    if info is None:
        raise _Fail("File has no INFO block")
    r.seek(info["abs"])
    if r.magic() != b"INFO":
        raise _Fail("Unknown or invalid INFO block")
    if r.take(4, True) != info["size"]:
        raise _Fail("INFO block size in main header doesn't match size in INFO header")
    major = v >> 24
    wave_offsets, have_channels, audio_ref, region_ref, region_info_size, region_count = [], False, None, None, 0, 0
    if info["type"] == 0x7000:  # StreamInfo.ReadBfwav, ChannelInfo.ReadBfstm
        h.codec, h.looping = r.take(1), int(r.take(1) != 0)
        r.pos += 2
        h.sample_rate, h.loop_start, h.sample_count = r.take(4, True), r.take(4, True), r.take(4, True)
        if (major == 0 and v >= 0x00010200) or (major >= 2 and v >= 0x02010100):
            h.loop_start_unaligned = r.take(4, True)
        else:
            r.pos += 4
        h.channel_count = r.take(4, True)
        r.pos -= 4
        if not 0 <= h.channel_count <= 255:
            raise _Fail("this reader takes 0..255")
        _channel_table(r, h, wave_offsets)
        have_channels = True
    else:
        base = r.pos
        sref, tref, cref = r.ref(base), r.ref(base), r.ref(base)
        if not _is(sref, 0x4100):
            raise _Fail("Could not read stream info.")
        r.seek(sref["abs"])
        h.codec, h.looping, h.channel_count, region_count = r.take(1), int(r.take(1) != 0), r.take(1), r.take(1)
        h.sample_rate, h.loop_start, h.sample_count = r.take(4, True), r.take(4, True), r.take(4, True)
        r.take(4, True)
        h.interleave_size = r.take(4, True)
        for _ in range(5):
            r.take(4, True)
        h.samples_per_seek_entry = r.take(4, True)
        audio_ref = r.ref(0)
        if (major >= 2 and v >= 0x02010000) or major == 0:
            region_info_size = r.take(2, True)
            r.pos += 2
            region_ref = r.ref(0)
        if (major == 0 and v >= 0x00040000) or (major >= 2 and v >= 0x02030000):
            h.loop_start_unaligned, h.loop_end_unaligned = r.take(4, True), r.take(4, True)
        if major == 0 and v >= 0x00050000:
            r.take(4)
        if _is(tref, 0x0101):
            r.seek(tref["abs"])
            tb = r.pos
            for t in [r.ref(tb) for _ in range(max(r.take(4, True), 0))]:
                r.seek(t["abs"])
                for _ in range(4):
                    r.take(1)
                r.seek(r.ref(t["abs"])["abs"])
                r.take(4, True), r.take(1), r.take(1)
                h.track_count += 1
        if _is(cref, 0x0101):
            r.seek(cref["abs"])
            _channel_table(r, h, wave_offsets)
            have_channels = True
    seek = first(0x4001)
    if seek is not None:
        r.seek(seek["abs"])
        if r.magic() != b"SEEK":
            raise _Fail("Unknown or invalid SEEK block")
        if r.take(4, True) != seek["size"]:
            raise _Fail("SEEK block size in main header doesn't match size in SEEK header")
        entries = R._div_round_up(h.sample_count, h.samples_per_seek_entry)
        R._seek_split(r.read_bytes(_i32(4 * h.channel_count * entries)), h.channel_count, False)
        h.seek_table = 1
    regn = first(0x4003)
    if regn is not None:
        r.seek(regn["abs"])
        if r.magic() != b"REGN":
            raise _Fail("Unknown or invalid REGN block")
        if r.take(4, True) != regn["size"]:
            raise _Fail("REGN block size in main header doesn't match size in REGN header")
        if region_ref is None:
            raise _Fail("Object reference not set to an instance of an object.")
        start = _i32(_i32(regn["abs"] + 8) + region_ref["offset"])
        for i in range(region_count):
            r.seek(_i32(start + _i32(region_info_size * i)))
            r.take(4, True), r.take(4, True)
            for _ in range(h.channel_count * 3):
                r.take(2, True)
            h.region_count += 1
    data = first(0x4002, 0x4004, 0x7001)
    if data is None:
        raise _Fail("File has no DATA block")
    r.seek(data["abs"])
    if r.magic() not in (b"DATA", b"PDAT"):
        raise _Fail("Unknown or invalid DATA block")
    if r.take(4, True) != data["size"]:
        raise _Fail("DATA block size in main header doesn't match size in DATA header")
    if data["type"] == 0x7001:
        _wave_rows(r, h, wave_offsets if have_channels else None)
        return
    if data["type"] == 0x4004:  # PrefetchData.ReadPrefetchData; only PrefetchData[0] is read
        count = r.take(4, True)
        pdat = []
        for _ in range(max(count, 0)):
            base = r.pos
            r.take(4, True)
            size = r.take(4, True)
            samples = bytes_to_samples(R._cs_div(size, h.channel_count), h.codec)
            r.take(4, True)
            pdat.append((size, samples, r.ref(base)))
        if not pdat:
            raise _Fail("Index was out of range.")
        size, samples, ref = pdat[0]
        r.seek(ref["abs"])
        h.output_size = R._deinterleave_checks(r, size, h.channel_count, size)
        h.audio_offset, h.audio_length = r.pos, size
        h.looping, h.sample_count = 0, samples  # Common.ToAudioStream
        return
    if audio_ref is None:
        raise _Fail("Object reference not set to an instance of an object.")
    audio_offset = _i32(_i32(data["abs"] + audio_ref["offset"]) + 8)
    r.seek(audio_offset)
    length = _i32(data["size"] - _i32(audio_offset - data["abs"]))
    h.output_size = R._deinterleave_checks(r, length, h.channel_count, R.samples_to_bytes(h.sample_count, h.codec))
    h.audio_offset, h.audio_length = r.pos, length


def parse(image, kind: int):
    """(0, info) or (E_DATA, message) for one image read by the reader `kind` names."""
    if kind in STREAMS:
        st, h = R.parse(image, kind)
        if st == 0:
            h.rows = None
        return st, h
    data = np.ascontiguousarray(image, dtype=np.uint8).tobytes()
    h = _new_info()
    r = _R(data, kind == BRWAV)
    try:
        (_brwav if kind == BRWAV else _bcfstm)(r, h)
        if h.codec == 3:
            raise _Fail("IMA ADPCM is not decoded")
        if h.codec > 3:
            raise _Fail("is not decoded")
        if h.codec == 2 and len(h.channels) < h.channel_count:
            raise _Fail("GC-ADPCM stream of")
    except _Fail as e:
        return E_DATA, str(e)
    return 0, h


def row_lengths(h: Info) -> List[int]:
    return [g for _, g in h.rows] if h.rows is not None else [h.output_size] * h.channel_count


def plan(image, kind: int):
    """The sizing pass: (status, message, samples, WAVE loop or None, info)."""
    if kind not in TYPES:
        return E_ARG, "in_type", None, None, None
    st, h = parse(image, kind)
    if st:
        return st, h, None, None, None
    if kind in STREAMS:
        st, loop, h = R.plan(image, kind)
        return st, "", (h.sample_count if st == 0 else None), loop, h
    if h.sample_count < 0:
        return E_DATA, "negative sample count", None, None, h
    ch, rows, n = h.channel_count, row_lengths(h), h.sample_count
    loop_end = n
    if h.codec == 2:
        if any(rl < R._gc_bytes(n) for rl in rows):
            return E_ARG, "Audio array length is too short for the specified number of samples.", None, None, h
        if ch == 0:
            return E_DATA, "Channels parameter cannot be empty or null", None, None, h
        if h.looping and not 0 <= h.loop_start <= n:
            return E_ARG, "Loop points must be less than the number of samples and non-negative.", None, None, h
        samples = n
    else:
        if h.codec == 1 and h.big_endian and any(rl % 2 for rl in rows):
            return E_DATA, "Index was outside the bounds of the array.", None, None, h
        if ch == 0:
            return E_DATA, "Channels parameter cannot be empty or null", None, None, h
        counts = [(rl + 1) // 2 if h.codec == 1 else rl for rl in rows]
        samples = counts[0]
        if any(c != samples for c in counts):
            return E_DATA, "All channels must have the same sample count", None, None, h
        if h.looping:
            if not (0 <= h.loop_start <= samples and 0 <= loop_end <= samples):
                return E_ARG, "Loop points must be less than the number of samples and non-negative.", None, None, h
            if loop_end < h.loop_start:
                return E_ARG, "The loop end must be greater than the loop start", None, None, h
    if samples * ch * 2 >= 1 << 31:
        return E_ARG, "more than 2 GiB of PCM", None, None, h
    return 0, "", samples, ((h.loop_start, loop_end) if h.looping else None), h


def rows(image, h: Info) -> List[np.ndarray]:
    """The channel rows ToAudioStream hands the format builders."""
    if h.rows is None:
        return R.rows(image, h)
    data = np.ascontiguousarray(image, dtype=np.uint8)
    return [data[a: a + g].copy() for a, g in h.rows]


def decoded_pcm(image, kind: int):
    """(status, [int16 channels], loop) of the reader chain; a bad predictor is E_DATA."""
    if kind in STREAMS:
        return R.decoded_pcm(image, kind)
    st, _, samples, loop, h = plan(image, kind)
    if st:
        return st, None, None
    rs = rows(image, h)
    if h.codec == 2:
        out = []
        for c, r in enumerate(rs):
            ch = h.channels[c]
            heads = r[0: 8 * (-(-samples // 14)): 8]
            if heads.size and int(heads.max()) >= 0x80:
                return E_DATA, None, None
            out.append(O.decode(r, np.asarray(ch["coefs"], np.int16), samples, ch["start"][1], ch["start"][2]))
        return 0, out, loop
    if h.codec == 1:
        padded = [np.concatenate([r, np.zeros(len(r) % 2, np.uint8)]) for r in rs]  # ToShortArray rounds up
        return 0, [np.frombuffer(r.tobytes(), dtype=">i2" if h.big_endian else "<i2").astype(np.int16) for r in padded], loop
    return 0, [(r.astype(np.int16) << 8).astype(np.int16) for r in rs], loop


def expected_wave(image, kind: int) -> Optional[np.ndarray]:
    """The WAVE image the reference writes for one image (None where it fails)."""
    st, pcm, loop = decoded_pcm(image, kind)
    if st:
        return None
    return O.wave_write16(pcm, parse(image, kind)[1].sample_rate, loop)


def wave_size(image, kind: int) -> int:
    st, _, samples, loop, h = plan(image, kind)
    if st:
        return 0
    return int(O.wave_write16([np.zeros(samples, np.int16)] * h.channel_count, h.sample_rate, loop).size)
