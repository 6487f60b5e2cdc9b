"""CPU restatement of IdspReader.ReadFile (Containers/Idsp/IdspReader.cs:13-112) and HpsReader.ReadFile (Containers/Hps/
HpsReader.cs:14-163) with the checks of ToAudioStream -> GcAdpcmFormat.ToPcm16, written apart from the product's C++
readers so that the tests can compare the two, plus the reader chain reader -> ToAudioStream -> ToPcm16 -> WaveWriter on
top of the oracle's GC-ADPCM decoder, de-interleave and WAVE writer.  It reads any image, hostile ones included; the
writer oracle's parse_idsp / parse_hps assume writer-made files and are not used here.

parse_idsp() / parse_hps() return (0, info) or (E_DATA, message): every exception the reference raises while reading,
and the refusals the product makes on purpose (IDSP: fewer than 0 or more than 255 channels; HPS: more than 255), in
the reference's order.  Messages are substrings of the product's."""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from oracle import pyoracle as O

E_DATA, E_ARG = -2, -1
IDSP, HPS = 7, 8


def _i32(v: int) -> int:
    return (v + (1 << 31)) % (1 << 32) - (1 << 31)


def _tdiv(a: int, b: int) -> int:  # C# int division (truncating)
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def _trem(a: int, b: int) -> int:
    return a - _tdiv(a, b) * b


def _next_multiple(v: int, m: int) -> int:  # Helpers.GetNextMultiple
    if m <= 0 or _trem(v, m) == 0:
        return v
    return _i32(v + m - _trem(v, m))


def gc_bytes(n: int) -> int:  # GcAdpcmMath.SampleCountToByteCount, wrapping
    whole, rest = _tdiv(n, 14), _trem(n, 14)
    nib = _i32(16 * whole + (0 if rest == 0 else rest + 2))
    return _i32(_tdiv(nib, 2) + _trem(nib, 2))


def nibble_to_sample(nb: int) -> int:
    return _i32(_i32(14 * _tdiv(nb, 16)) + _trem(nb, 16) - 2)


def nibble_count_to_samples(nb: int) -> int:
    extra = _trem(nb, 16)
    return _i32(14 * _tdiv(nb, 16) + (0 if extra < 2 else extra - 2))


class _Fail(Exception):
    pass


class _R:
    """BigEndian BinaryReader over the image: reads past the end throw, ReadBytes returns what is left."""

    def __init__(self, data: bytes):
        self.d, self.pos = data, 0

    def seek(self, p):
        if p < 0:
            raise _Fail("Non-negative number required.")
        self.pos = p

    def take(self, n, signed=True):
        if self.pos + n > len(self.d):
            raise _Fail("Unable to read beyond the end of the stream.")
        v = int.from_bytes(self.d[self.pos: self.pos + n], "big", signed=signed)
        self.pos += n
        return v

    def i32(self):
        return self.take(4)

    def i16(self):
        return self.take(2)

    def read_bytes(self, n) -> int:
        if n < 0:
            raise _Fail("Non-negative number required.")
        got = max(0, min(n, len(self.d) - self.pos))
        self.pos += got
        return got


@dataclass
class IdspInfo:
    channel_count: int = 0
    sample_rate: int = 0
    sample_count: int = 0
    loop_start: int = 0
    loop_end: int = 0
    interleave_size: int = 0
    header_size: int = 0
    channel_info_size: int = 0
    audio_data_offset: int = 0
    audio_data_length: int = 0
    looping: int = 0
    interleave: int = 0
    output_size: int = 0
    audio_offset: int = 0
    audio_length: int = 0
    channels: List[dict] = field(default_factory=list)


def parse_idsp(image):
    """(0, IdspInfo) or (E_DATA, message)"""
    d = np.ascontiguousarray(image, dtype=np.uint8).tobytes()
    r, h = _R(d), IdspInfo()
    try:
        if len(d) < 4:
            raise _Fail("Index and count must refer to a location within the buffer.")
        r.pos = 4
        if d[:4] != b"IDSP":
            raise _Fail("File has no IDSP header")
        r.pos += 4
        (h.channel_count, h.sample_rate, h.sample_count, h.loop_start, h.loop_end, h.interleave_size, h.header_size,
         h.channel_info_size, h.audio_data_offset, h.audio_data_length) = (r.i32() for _ in range(10))
        if not 0 <= h.channel_count <= 255:
            raise _Fail("channels (this reader takes 0..255)")
        for i in range(h.channel_count):
            r.seek(_i32(h.header_size + _i32(i * h.channel_info_size)))
            c = dict(sample_count=r.i32(), nibble_count=r.i32(), sample_rate=r.i32(), looping=int(r.i16() == 1))
            r.pos += 2
            c.update(start_address=r.i32(), end_address=r.i32(), current_address=r.i32())
            c["coefs"] = [r.i16() for _ in range(16)]
            c["gain"] = r.i16()
            c["start"] = tuple(r.i16() for _ in range(3))
            c["loop"] = tuple(r.i16() for _ in range(3))
            h.channels.append(c)
        h.looping = int(any(c["looping"] for c in h.channels))
        r.seek(h.audio_data_offset)
        h.interleave = h.audio_data_length if h.interleave_size == 0 else h.interleave_size
        length = _i32(h.channel_count * h.audio_data_length)
        h.output_size = gc_bytes(h.sample_count)
        if len(d) - r.pos < length:
            raise _Fail("Specified length is greater than the number of bytes remaining in the Stream")
        if h.channel_count == 0:
            raise _Fail("Attempted to divide by zero.")
        if _trem(length, h.channel_count) != 0:
            raise _Fail("must be divisible by the number of outputs.")
        if h.output_size < 0:
            raise _Fail("Arithmetic operation resulted in an overflow.")
        h.audio_offset, h.audio_length = r.pos, length
    except _Fail as e:
        return E_DATA, str(e)
    return 0, h


@dataclass
class HpsInfo:
    sample_rate: int = 0
    channel_count: int = 0
    sample_count: int = 0
    looping: int = 0
    loop_start: int = 0
    first_block: int = 0
    loop_block: int = -1
    channels: List[dict] = field(default_factory=list)
    blocks: List[dict] = field(default_factory=list)      # offset, size, final_nibble, next_offset, ctx
    pieces: List[List[tuple]] = field(default_factory=list)  # per channel: (file offset, bytes) of each block's piece

    @property
    def block_count(self):
        return len(self.blocks)


def parse_hps(image):
    """(0, HpsInfo) or (E_DATA, message)"""
    d = np.ascontiguousarray(image, dtype=np.uint8).tobytes()
    r, h = _R(d), HpsInfo()
    try:
        if len(d) < 8:
            raise _Fail("Index and count must refer to a location within the buffer.")
        r.pos = 8
        if d[:8] != b" HALPST\0":
            raise _Fail("File has no HALPST header")
        h.sample_rate, h.channel_count = r.i32(), r.i32()
        ch = h.channel_count
        if ch > 255:
            raise _Fail("channels (this reader takes at most 255)")
        for _ in range(ch):
            c = dict(max_block_size=r.i32())
            r.i32()
            c["end_address"] = r.i32()
            r.i32()
            c["coefs"] = [r.i16() for _ in range(16)]
            c["gain"] = r.i16()
            c["start"] = tuple(r.i16() for _ in range(3))
            h.channels.append(c)
        r.seek(_next_multiple(max(0x80, r.pos), 0x20))
        h.first_block = r.pos
        h.pieces = [[] for _ in range(max(ch, 0))]
        current, nxt = 0, r.pos
        while nxt > current:
            r.seek(nxt)
            current = nxt
            b = dict(offset=current, size=r.i32(), final_nibble=r.i32(), next_offset=r.i32(), ctx=[])
            for _ in range(ch):
                b["ctx"].append(tuple(r.i16() for _ in range(3)))
                r.pos += 2
            r.seek(_next_multiple(_i32(r.pos), 0x20))
            start = r.pos
            v = _i32(b["final_nibble"] + 1)
            size_bytes = _tdiv(v, 2) + (v & 1)
            for i in range(ch):
                r.seek(_i32(start + _i32(_tdiv(b["size"], ch) * i)))
                at = r.pos
                h.pieces[i].append((at, r.read_bytes(size_bytes)))
            h.blocks.append(b)
            nxt = b["next_offset"]
        if ch <= 0:
            raise _Fail("Sequence contains no elements.")
        h.sample_count = _i32(nibble_to_sample(h.channels[0]["end_address"]) + 1)
        if any(_i32(nibble_to_sample(c["end_address"]) + 1) != h.sample_count for c in h.channels):
            raise _Fail("Channels have differing sample counts")
        start_offset = h.blocks[-1]["next_offset"]
        if start_offset != -1:
            nib = 0
            for k, b in enumerate(h.blocks):
                if b["offset"] == start_offset:
                    h.looping, h.loop_start, h.loop_block = 1, nibble_count_to_samples(nib), k
                    for i, c in enumerate(h.channels):
                        c["loop"] = b["ctx"][i]
                nib = _i32(nib + _i32(b["final_nibble"] + 1))
    except _Fail as e:
        return E_DATA, str(e)
    return 0, h


def parse(image, kind):
    return parse_idsp(image) if kind == IDSP else parse_hps(image)


def plan(image, kind: int):
    """The sizing pass: (status, WAVE loop or None, info) - status 0, E_DATA or E_ARG as the converter's plan."""
    if kind not in (IDSP, HPS):
        return E_ARG, None, None
    st, h = parse(image, kind)
    if st:
        return st, None, None
    n = h.sample_count
    if n < 0:
        return E_DATA, None, h
    if kind == HPS:
        need = gc_bytes(n)
        for c in range(h.channel_count):
            total = sum(g for _, g in h.pieces[c])
            if total > 2 ** 31 - 1:
                return E_DATA, None, h
            if total < need:
                return E_ARG, None, h
        loop = (h.loop_start, n)
    else:
        loop = (h.loop_start, h.loop_end)
    if h.looping and not (0 <= loop[0] <= n and 0 <= loop[1] <= n and loop[1] >= loop[0]):
        return E_ARG, None, h
    if n * h.channel_count * 2 >= 1 << 31:
        return E_ARG, None, h
    return 0, (loop if h.looping else None), h


def rows(image, kind, h) -> List[np.ndarray]:
    """The channels' ADPCM arrays the decoder reads (at least SampleCountToByteCount(sample_count) bytes each)."""
    data = np.ascontiguousarray(image, dtype=np.uint8)
    if kind == IDSP:
        region = data[h.audio_offset: h.audio_offset + max(h.audio_length, 0)]
        in_size = _tdiv(h.audio_length, h.channel_count)
        if h.interleave <= 0 or in_size <= 0:
            return [np.zeros(h.output_size, np.uint8) for _ in range(h.channel_count)]
        return O.deinterleave(region, h.interleave, h.channel_count, h.output_size)
    return [np.concatenate([data[a: a + g] for a, g in ps] + [np.zeros(0, np.uint8)]) for ps in h.pieces]


def decoded_pcm(image, kind: int):
    """(status, [int16 channels], loop) of the reader chain; a bad predictor is E_DATA."""
    st, loop, h = plan(image, kind)
    if st:
        return st, None, None
    n = h.sample_count
    out = []
    for c, r in enumerate(rows(image, kind, h)):
        ch = h.channels[c]
        heads = r[0: 8 * (-(-n // 14)): 8]
        if heads.size and int(heads.max()) >= 0x80:
            return E_DATA, None, None
        out.append(O.decode(np.ascontiguousarray(r[:gc_bytes(n)]), np.asarray(ch["coefs"], np.int16), n, ch["start"][1], ch["start"][2]))
    return 0, out, loop


def expected_wave(image, kind: int) -> Optional[np.ndarray]:
    """The WAVE image the reference writes for one IDSP / HPS image (None where it fails)."""
    st, pcm, loop = decoded_pcm(image, kind)
    if st:
        return None
    return O.wave_write16(pcm, parse(image, kind)[1].sample_rate, loop)


def wave_size(image, kind: int) -> int:
    st, loop, h = plan(image, kind)
    if st:
        return 0
    return int(O.wave_write16([np.zeros(h.sample_count, np.int16)] * h.channel_count, h.sample_rate, loop).size)


# ---- hand-built images ------------------------------------------------------------------------------------------------
def hps_header(rate: int, chans: List[dict]) -> bytearray:
    """The HALPST header: chans[c] = dict(coefs, end_address, start=(ps, h1, h2), max_block=0x10000)"""
    out = bytearray(_next_multiple(max(0x80, 0x10 + 0x38 * len(chans)), 0x20))
    struct.pack_into(">8sii", out, 0, b" HALPST\0", rate, len(chans))
    for c, ch in enumerate(chans):
        struct.pack_into(">iiii16hh3h", out, 0x10 + 0x38 * c, ch.get("max_block", 0x10000), 2, ch["end_address"], 2,
                         *[int(v) for v in ch["coefs"]], 0, *[int(v) for v in ch["start"]])
    return out


def put(out: bytearray, at: int, data: bytes) -> None:
    if len(out) < at + len(data):
        out.extend(bytes(at + len(data) - len(out)))
    out[at: at + len(data)] = data


def hps_block(out: bytearray, offset: int, size: int, final: int, nxt: int, pieces: List[bytes], ctx=None) -> int:
    """Writes one block header at `offset` and channel c's bytes at the audio start + size / ch * c; returns the audio
    start."""
    ch = len(pieces)
    put(out, offset, struct.pack(">iii", size, final, nxt))
    for c in range(ch):
        put(out, offset + 12 + 8 * c, struct.pack(">hhhh", *(ctx[c] if ctx else (0, 0, 0)), 0))
    start = _next_multiple(offset + 12 + 8 * ch, 0x20)
    for c, p in enumerate(pieces):
        put(out, start + _tdiv(size, ch) * c, p)
    return start


def sample_to_nibble(s: int) -> int:
    return s // 14 * 16 + s % 14 + 2


def hps_chain(rate: int, channels: List[tuple], piece_bytes: List[int], stride=lambda n: n, gap: int = 0,
              loop_block: Optional[int] = None, odd_final: bool = False, n_samples: Optional[int] = None) -> np.ndarray:
    """A valid HPS image from encoded channels [(adpcm row, coefs, start context)]: block j carries piece_bytes[j] bytes of
    every channel at a per-channel stride of stride(piece) bytes (so sources need not be aligned), blocks `gap` bytes
    apart; odd_final writes FinalNibble = 2 * bytes - 2 (the same byte count); loop_block: the last block's NextOffset."""
    ch = len(channels)
    n = n_samples if n_samples is not None else sum(piece_bytes) * 2 // 16 * 14
    chans = [dict(coefs=co, end_address=sample_to_nibble(n - 1), start=st) for _, co, st in channels]
    out = hps_header(rate, chans)
    offsets, at = [], len(out)
    for pb in piece_bytes:
        offsets.append(at)
        start = _next_multiple(at + 12 + 8 * ch, 0x20)
        at = start + stride(pb) * ch + gap
    pos = 0
    for j, pb in enumerate(piece_bytes):
        nxt = offsets[j + 1] if j + 1 < len(piece_bytes) else (offsets[loop_block] if loop_block is not None else -1)
        pieces = [bytes(np.asarray(row, np.uint8)[pos: pos + pb]) for row, _, _ in channels]
        hps_block(out, offsets[j], stride(pb) * ch, 2 * pb - (2 if odd_final else 1), nxt, pieces)
        pos += pb
    return np.frombuffer(bytes(out), np.uint8).copy()


def idsp_image(rate: int, channels: List[tuple], n: int, loop=None, interleave: int = 16, header_size: int = 0x40,
               info_size: int = 0x60, audio_len: Optional[int] = None, loop_flags=None) -> np.ndarray:
    """An IDSP image from encoded channels [(adpcm row, coefs, start context)] interleaved in `interleave`-byte blocks
    (0: one block per channel)."""
    ch = len(channels)
    ads = audio_len if audio_len is not None else gc_bytes(n)
    head = _next_multiple(header_size + info_size * ch, 0x20)
    ls, le = loop if loop else (0, 0)
    out = bytearray(head)
    struct.pack_into(">4s11i", out, 0, b"IDSP", 0, ch, rate, n, ls, le, interleave, header_size, info_size, head, ads)
    for c, (_, co, st) in enumerate(channels):
        flag = (loop_flags[c] if loop_flags else (1 if loop else 0))
        struct.pack_into(">iiihhiii16hh3h3h", out, header_size + info_size * c, n, 0, rate, flag, 0, 2, 0, 2,
                         *[int(v) for v in co], 0, *[int(v) for v in st], 0, 0, 0)
    arrays = [np.concatenate([np.asarray(row, np.uint8)[:ads], np.zeros(max(0, ads - len(row)), np.uint8)]) for row, _, _ in channels]
    if interleave == 0:
        region = b"".join(bytes(a) for a in arrays)
    else:
        region = bytes(O.interleave([np.ascontiguousarray(a) for a in arrays], interleave, ads))
    put(out, head, region)
    return np.frombuffer(bytes(out), np.uint8).copy()


def encoded(pcm: np.ndarray, start_hist=(0, 0)):
    """(adpcm row, coefs, start context) of one channel through the oracle's encoder, with a start history"""
    co = O.calculate_coefficients(pcm)
    ad = O.encode(pcm, co)
    return ad, co, (int(ad[0]) if len(ad) else 0, start_hist[0], start_hist[1])
