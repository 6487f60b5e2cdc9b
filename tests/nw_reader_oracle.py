"""CPU restatement of BrstmReader.ReadFile (Containers/NintendoWare/BrstmReader.cs:12-185), BCFstmReader.ReadFile
(BCFstmReader.cs:14-288) and Common.ToAudioStream (Common.cs:45-116), written apart from the product's C++ readers so
that the tests can compare the two, plus the reader chain reader -> ToAudioStream -> ToPcm16 -> WaveWriter on top of the
oracle's GC-ADPCM decoder, de-interleave and WAVE writer.

parse() returns (0, info) or (E_DATA, message): every exception the reference raises while reading, and the refusals
the product makes on purpose (codec 3 and above, GC-ADPCM without channel info for every channel, wave / prefetch
files and blocks), in the reference's order."""
from __future__ import annotations

import math
import struct
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from oracle import pyoracle as O

E_DATA, E_ARG = -2, -1
BRSTM, BCSTM, BFSTM = 4, 5, 6
I32_MIN = -(1 << 31)


def _i32(v: int) -> int:
    return (v + (1 << 31)) % (1 << 32) - (1 << 31)


def _cs_div(a: int, b: int) -> int:
    if b == 0:
        raise _Fail("Attempted to divide by zero.")
    if a == I32_MIN and b == -1:
        raise _Fail("Arithmetic operation resulted in an overflow.")
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def _cs_rem(a: int, b: int) -> int:
    return a - _cs_div(a, b) * b


def _div_round_up(v: int, d: int) -> int:
    """Extensions.DivideByRoundUp through a double; NaN and out-of-range results are int.MinValue (x64 conversion)."""
    if d == 0:
        q = math.nan if v == 0 else math.inf
    else:
        q = math.ceil(v / d)
    return I32_MIN if (isinstance(q, float) and (math.isnan(q) or math.isinf(q))) or q >= 2 ** 31 or q < -2 ** 31 else int(q)


def _next_multiple(v: int, m: int) -> int:
    if m <= 0 or math.fmod(v, m) == 0:
        return v
    return _i32(v + m - int(math.fmod(v, m)))


def _gc_bytes(n: int) -> int:
    whole, rest = int(n / 14), int(math.fmod(n, 14))
    nib = _i32(16 * whole + (0 if rest == 0 else rest + 2))
    return _i32(int(nib / 2) + (int(math.fmod(nib, 2)) if math.fmod(nib, 2) != 0 else 0))


def samples_to_bytes(n: int, codec: int) -> int:
    return _gc_bytes(n) if codec == 2 else (_i32(n * 2) if codec == 1 else (n if codec == 0 else 0))


class _Fail(Exception):
    pass


@dataclass
class NwInfo:
    codec: int = 0
    looping: int = 0
    channel_count: int = 0
    sample_rate: int = 0
    loop_start: int = 0
    sample_count: int = 0
    interleave_size: int = 0
    big_endian: int = 0
    version: int = 0
    seek_table: int = 0
    region_count: int = 0
    track_count: int = 0
    samples_per_seek_entry: int = 0
    loop_start_unaligned: int = 0
    loop_end_unaligned: int = 0
    output_size: int = 0
    audio_offset: int = 0
    audio_length: int = 0
    channels: List[dict] = field(default_factory=list)   # per channel info: coefs, gain, start, loop

    @property
    def adpcm_channel_count(self):
        return len(self.channels)


class _R:
    def __init__(self, data: bytes, be: bool):
        self.d, self.pos, self.be = data, 0, be

    def seek(self, p):
        if p < 0:
            raise _Fail("Non-negative number required.")
        self.pos = p

    def take(self, n, signed=False, be=None):
        if self.pos + n > len(self.d):
            raise _Fail("Unable to read beyond the end of the stream.")
        v = int.from_bytes(self.d[self.pos: self.pos + n], "big" if (self.be if be is None else be) else "little", signed=signed)
        self.pos += n
        return v

    def magic(self) -> bytes:
        if self.pos + 4 > len(self.d):
            raise _Fail("Index and count must refer to a location within the buffer.")
        self.pos += 4
        return self.d[self.pos - 4: self.pos]

    def read_bytes(self, n) -> int:
        if n < 0:
            raise _Fail("Non-negative number required.")
        got = max(0, min(n, len(self.d) - self.pos))
        self.pos += got
        return got

    def ref(self, base=0, sized=False):
        t = self.take(2, True)
        self.pos += 2
        off = self.take(4, True)
        size = self.take(4, True) if sized else 0
        return dict(type=t, offset=off, base=base, abs=_i32(base + off), size=size)


def _is(ref, t):
    return ref["type"] == t and ref["offset"] > 0


def _channel(r: _R, gain: bool) -> dict:
    coefs = [r.take(2, True) for _ in range(16)]
    g = r.take(2, True) if gain else 0
    start = tuple(r.take(2, True) for _ in range(3))
    loop = tuple(r.take(2, True) for _ in range(3))
    return dict(coefs=coefs, gain=g, start=start, loop=loop)


def _deinterleave_checks(r: _R, length: int, ch: int, out: int) -> int:
    if len(r.d) - r.pos < length:
        raise _Fail("Specified length is greater than the number of bytes remaining in the Stream")
    if ch == 0:
        raise _Fail("Attempted to divide by zero.")
    if math.fmod(length, ch) != 0:
        raise _Fail("must be divisible by the number of outputs.")
    if out == -1:
        out = int(length / ch)
    if out < 0:
        raise _Fail("Arithmetic operation resulted in an overflow.")
    return out


def _seek_split(got: int, ch: int, be_shorts: bool):
    if be_shorts and got % 2:
        raise _Fail("Index was outside the bounds of the array.")
    shorts = (got + 1) // 2
    if ch == 0:
        raise _Fail("Attempted to divide by zero.")
    if shorts % ch:
        raise _Fail("must be divisible by the number of outputs.")


def _brstm(r: _R, h: NwInfo):
    if r.magic() != b"RSTM":
        raise _Fail("File has no RSTM header")
    bom = r.take(2)
    if bom != 0xFEFF:
        raise _Fail(f"Expected 65279, but got {bom} at offset 0x4")
    h.version = (r.take(1) << 24) | (r.take(1) << 16)
    file_size = r.take(4, True)
    if len(r.d) < file_size:
        raise _Fail("Actual file length is less than stated length")
    r.take(2, True), r.take(2, True)
    head_off, head_size, seek_off, seek_size, data_off, data_size = (r.take(4, True) for _ in range(6))
    r.seek(head_off)
    if r.magic() != b"HEAD":
        raise _Fail("Unknown or invalid HEAD block")
    if r.take(4, True) != head_size:
        raise _Fail("HEAD block size in RSTM header doesn't match size in HEAD header")
    base = r.pos
    sref, tref, cref = r.ref(base), r.ref(base), r.ref(base)
    if not _is(sref, 0x0100):
        raise _Fail("Could not read stream info.")
    r.seek(sref["abs"])
    h.codec, h.looping, h.channel_count = r.take(1), int(r.take(1) != 0), r.take(1)
    r.pos += 1
    h.sample_rate = r.take(2)
    r.pos += 2
    h.loop_start, h.sample_count = r.take(4, True), r.take(4, True)
    audio_data_offset = r.take(4, True)
    r.take(4, True)
    h.interleave_size = r.take(4, True)
    for _ in range(4):
        r.take(4, True)
    h.samples_per_seek_entry = r.take(4, True)
    if not _is(tref, 0x0100):
        raise _Fail("Could not read track info.")
    r.seek(tref["abs"])
    count = r.take(1)
    r.take(1)
    r.pos += 2
    refs = [r.ref(tref["base"]) for _ in range(count)]
    for t in refs:
        r.seek(t["abs"])
        if t["type"] & 0xFF == 1:
            r.take(1), r.take(1)
            r.pos += 6
        r.take(1), r.take(1), r.take(1)
        h.track_count += 1
    if not _is(cref, 0x0100):
        raise _Fail("Could not read channel info.")
    r.seek(cref["abs"])
    count = r.take(1)
    r.pos += 3
    refs = [r.ref(cref["base"]) for _ in range(count)]
    for c in refs:
        r.seek(c["abs"])
        a = r.ref(cref["base"])
        if a["offset"] > 0:
            r.seek(a["abs"])
            h.channels.append(_channel(r, True))
    if seek_off != 0:
        r.seek(seek_off)
        if r.magic() != b"ADPC":
            raise _Fail("Unknown or invalid ADPC block")
        if r.take(4, True) != seek_size:
            raise _Fail("ADPC block size in RSTM header doesn't match size in ADPC header")
        sc, spe = h.sample_count, h.samples_per_seek_entry
        full_last = _cs_rem(sc, spe) == 0 and sc > 0
        bpe = 4 * h.channel_count
        n_short = _i32(_cs_div(_gc_bytes(sc), spe) + 1)
        n_std = _i32(_cs_div(sc, spe) + (0 if full_last else 1))
        size_short = _next_multiple(_i32(8 + _i32(n_short * bpe)), 0x20)
        size_std = _next_multiple(_i32(8 + _i32(n_std * bpe)), 0x20)
        table = None
        if seek_size == size_std:
            table, h.seek_table = _i32(bpe * n_std), 1
        elif seek_size == size_short:
            table, h.seek_table = _i32(bpe * n_short), 2
        if table is not None:
            _seek_split(r.read_bytes(table), h.channel_count, True)
    r.seek(data_off)
    if r.magic() != b"DATA":
        raise _Fail("Unknown or invalid DATA block")
    if r.take(4, True) != data_size:
        raise _Fail("DATA block size in main header doesn't match size in DATA header")
    r.seek(audio_data_offset)
    length = _i32(data_size - _i32(audio_data_offset - data_off))
    h.output_size = _deinterleave_checks(r, length, h.channel_count, samples_to_bytes(h.sample_count, h.codec))
    h.audio_offset, h.audio_length, h.big_endian = r.pos, length, 1


def _bcfstm(r: _R, h: NwInfo):
    mg = r.magic()
    if mg not in (b"CSTM", b"FSTM", b"CWAV", b"FWAV", b"CSTP", b"FSTP"):
        raise _Fail("File has no CSTM or FSTM header")
    bom = r.take(2, be=False)
    if bom == 0xFEFF:
        r.be = False
    elif bom == 0xFFFE:
        r.be = True
    else:
        raise _Fail("File has no byte order mark")
    r.pos -= 2
    if mg not in (b"CSTM", b"FSTM"):
        raise _Fail("files are not read")
    h.big_endian = int(r.be)
    r.take(2), r.take(2, True)
    h.version = r.take(4)
    file_size = r.take(4, True)
    if len(r.d) < file_size:
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
    if info["type"] == 0x7000:
        raise _Fail("a wave info block is not read")
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
    v, major = h.version, h.version >> 24
    region_ref, region_info_size = None, 0
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
        refs = [r.ref(tb) for _ in range(max(r.take(4, True), 0))]
        for t in refs:
            r.seek(t["abs"])
            for _ in range(4):
                r.take(1)
            tr = r.ref(t["abs"])
            r.seek(tr["abs"])
            r.take(4, True), r.take(1), r.take(1)
            h.track_count += 1
    if _is(cref, 0x0101):
        r.seek(cref["abs"])
        cb = r.pos
        refs = [r.ref(cb) for _ in range(max(r.take(4, True), 0))]
        for c in refs:
            r.seek(c["abs"])
            if _is(c, 0x7100):
                r.ref(0)
            a = r.ref(c["abs"])
            if _is(a, 0x0300):
                r.seek(a["abs"])
                h.channels.append(_channel(r, False))
    seek = first(0x4001)
    if seek is not None:
        r.seek(seek["abs"])
        if r.magic() != b"SEEK":
            raise _Fail("Unknown or invalid SEEK block")
        if r.take(4, True) != seek["size"]:
            raise _Fail("SEEK block size in main header doesn't match size in SEEK header")
        entries = _div_round_up(h.sample_count, h.samples_per_seek_entry)
        _seek_split(r.read_bytes(_i32(4 * h.channel_count * entries)), h.channel_count, False)
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
    bid = r.magic()
    if bid not in (b"DATA", b"PDAT"):
        raise _Fail("Unknown or invalid DATA block")
    if r.take(4, True) != data["size"]:
        raise _Fail("DATA block size in main header doesn't match size in DATA header")
    if data["type"] != 0x4002:
        raise _Fail("prefetch and wave data blocks are not read")
    audio_offset = _i32(_i32(data["abs"] + audio_ref["offset"]) + 8)
    r.seek(audio_offset)
    length = _i32(data["size"] - _i32(audio_offset - data["abs"]))
    h.output_size = _deinterleave_checks(r, length, h.channel_count, samples_to_bytes(h.sample_count, h.codec))
    h.audio_offset, h.audio_length = r.pos, length


def parse(image, kind: int):
    """(0, NwInfo) or (E_DATA, message) for one image read by the reader `kind` names."""
    data = np.ascontiguousarray(image, dtype=np.uint8).tobytes()
    h = NwInfo()
    r = _R(data, kind == BRSTM)
    try:
        (_brstm if kind == BRSTM else _bcfstm)(r, h)
        if h.codec == 3:
            raise _Fail("IMA ADPCM is not decoded")
        if h.codec > 3:
            raise _Fail("is not decoded")
        if h.codec == 2 and len(h.channels) < h.channel_count:
            raise _Fail("GC-ADPCM stream of")
    except _Fail as e:
        return E_DATA, str(e)
    return 0, h


def plan(image, kind: int):
    """The sizing pass: (status, WAVE loop or None, NwInfo) - status 0, E_DATA or E_ARG as the converter's plan."""
    if kind not in (BRSTM, BCSTM, BFSTM):
        return E_ARG, None, None
    st, h = parse(image, kind)
    if st:
        return st, None, None
    if h.sample_count < 0:
        return E_DATA, None, h
    if h.looping and not (0 <= h.loop_start <= h.sample_count):
        return E_ARG, None, h
    if h.sample_count * h.channel_count * 2 >= 1 << 31:
        return E_ARG, None, h
    return 0, ((h.loop_start, h.sample_count) if h.looping else None), h


def rows(image, h: NwInfo) -> List[np.ndarray]:
    """Stream.DeInterleave(AudioDataLength, InterleaveSize, ChannelCount, SamplesToBytes(SampleCount))."""
    data = np.ascontiguousarray(image, dtype=np.uint8)[h.audio_offset: h.audio_offset + h.audio_length]
    in_size = h.audio_length // h.channel_count
    if h.interleave_size <= 0 or in_size == 0:
        return [np.zeros(h.output_size, np.uint8) for _ in range(h.channel_count)]
    return O.deinterleave(data, h.interleave_size, h.channel_count, h.output_size)


def decoded_pcm(image, kind: int):
    """(status, [int16 channels], loop) of the reader chain; a bad predictor is E_DATA."""
    st, loop, h = plan(image, kind)
    if st:
        return st, None, None
    rs = rows(image, h)
    n = h.sample_count
    if h.codec == 2:
        out = []
        for c, r in enumerate(rs):
            ch = h.channels[c]
            heads = r[0: 8 * (-(-n // 14)): 8]
            if heads.size and int(heads.max()) >= 0x80:
                return E_DATA, None, None
            out.append(O.decode(r, np.asarray(ch["coefs"], np.int16), n, ch["start"][1], ch["start"][2]))
        return 0, out, loop
    if h.codec == 1:
        return 0, [np.frombuffer(r.tobytes(), dtype=">i2" if h.big_endian else "<i2").astype(np.int16) for r in rs], loop
    return 0, [(r.astype(np.int16) << 8).astype(np.int16) for r in rs], loop


def expected_wave(image, kind: int) -> Optional[np.ndarray]:
    """The WAVE image the reference writes for one stream image (None where it fails)."""
    st, pcm, loop = decoded_pcm(image, kind)
    if st:
        return None
    h = parse(image, kind)[1]
    return O.wave_write16(pcm, h.sample_rate, loop)


def wave_size(image, kind: int) -> int:
    st, loop, h = plan(image, kind)
    if st:
        return 0
    return int(O.wave_write16([np.zeros(h.sample_count, np.int16)] * h.channel_count, h.sample_rate, loop).size)
