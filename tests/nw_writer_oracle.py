"""CPU restatement of BrstmWriter (Containers/NintendoWare/BrstmWriter.cs) and BCFstmWriter (BCFstmWriter.cs) with
BxstmConfiguration's defaults, written apart from the product's C++ sizing pass and assembly kernel so that the tests can
compare the two.  The GC-ADPCM channels come from the C oracle (CalculateCoefficients, Encode, Decode, the seek table
and the loop context), the data region from its InterleaveExtensions.Interleave.

A GC-ADPCM loop start that is not a multiple of the loop point alignment goes through GcAdpcmFormat.WithAlignment
(the oracle's GcAdpcmAlignment, oracle/gcalign.c) and the writer's channel rebuild as the reference chains them: the data
is AdpcmAligned and the header carries the moved loop, while the loop context (taken at the unaligned loop start) and
the seek table (from the full decode) are the ones the first encode's build left behind.

write() returns (0, file bytes) or (E_ARG / E_DATA, None) for the per-file refusals: more than 255 channels, a file
of 2 GiB or more, GC-ADPCM without samples (GcAdpcmChannel reads Adpcm[0]) and loop points the alignment cannot
handle."""
from __future__ import annotations

import struct
from typing import List, Optional, Tuple

import numpy as np

from oracle import pyoracle as O
from oracle import pygcalign

E_DATA, E_ARG = -2, -1
BRSTM, BCSTM, BFSTM = 4, 5, 6
PCM8, PCM16, GCADPCM = 0, 1, 2


def _ceil(a: int, b: int) -> int:
    return -(-a // b)


def _next_multiple(v: int, m: int) -> int:
    return v if v % m == 0 else v + m - v % m


def samples_to_bytes(n: int, codec: int) -> int:
    return O.sample_count_to_byte_count(n) if codec == GCADPCM else n * 2 if codec == PCM16 else n


def samples_per_block(codec: int) -> int:  # BytesToSamples(0x2000, codec)
    return 14336 if codec == GCADPCM else 0x1000 if codec == PCM16 else 0x2000


def file_big_endian(kind: int, endianness: int = 0) -> bool:
    if kind == BRSTM:
        return True
    return endianness == 2 if endianness else kind == BFSTM


class _W:
    def __init__(self, size: int, be: bool):
        self.b = bytearray(size)
        self.e = ">" if be else "<"
        self.at = 0

    def put(self, fmt: str, *v):
        s = struct.pack(self.e + fmt, *v)
        self.b[self.at:self.at + len(s)] = s
        self.at += len(s)

    def raw(self, s: bytes):
        self.b[self.at:self.at + len(s)] = s
        self.at += len(s)


def _tracks(ch: int):
    out = []
    for t in range(_ceil(ch, 2)):
        cc = min(ch - 2 * t, 2)
        out.append((cc, 2 * t, 2 * t + 1 if cc >= 2 else 0))
    return out


def _gc_channels(pcm: List[np.ndarray], loop_start: Optional[int], spe: int):
    """GetFormat<GcAdpcmFormat> and the writer's channel rebuild for channels that need no alignment: (adpcm, coefs,
    start context, loop context, seek table) per channel."""
    out = []
    for p in pcm:
        n = len(p)
        co = O.calculate_coefficients(p)
        ad = O.encode(p, co)
        dec = O.decode(ad, co, n)
        start = (int(ad[0]), 0, 0)
        loop = tuple(int(v) for v in O.gc_loop_context(ad, dec, loop_start)) if loop_start is not None else start
        out.append((ad, co, start, loop, np.asarray(O.gc_seek_table(dec, spe), dtype=np.int16)))
    return out


def geometry(kind: int, codec: int, ch: int, n: int, loop: Optional[Tuple[int, int]]):
    sc = loop[1] if loop else n
    spi = samples_per_block(codec)
    g = dict(sc=sc, spi=spi, bpi=samples_to_bytes(spi, codec), ads=_next_multiple(samples_to_bytes(sc, codec), 0x20),
             icount=_ceil(sc, spi))
    g["last_samples"] = sc - (g["icount"] - 1) * spi
    g["last_np"] = samples_to_bytes(g["last_samples"], codec)
    g["last"] = _next_multiple(g["last_np"], 0x20)
    g["entries"] = _ceil(sc, spi) if codec == GCADPCM else 0
    T = _ceil(ch, 2)
    adpcm = codec == GCADPCM
    if kind == BRSTM:
        g["h2"] = 4 + 8 * T + 0x0c * T
        h3 = 4 + 8 * ch + (0x38 if adpcm else 8) * ch
        g["head"] = _next_multiple(8 + 24 + 0x34 + g["h2"] + h3, 0x20)
    else:
        g["i1"] = 0x38 + 0xc
        g["i2"] = 4 + 8 * T if kind == BCSTM else 0
        g["i3"] = 4 + 8 * ch + (0x14 * T if kind == BCSTM else 0) + 8 * ch + (0x2e if adpcm else 0) * ch
        g["head"] = _next_multiple(8 + 24 + g["i1"] + g["i2"] + g["i3"], 0x20)
    g["seek_off"] = 0x40 + g["head"] if adpcm else 0
    g["seek_size"] = _next_multiple(8 + g["entries"] * ch * 4, 0x20) if adpcm else 0
    g["data_off"] = 0x40 + g["head"] + g["seek_size"]
    g["data_size"] = 0x20 + g["ads"] * ch
    g["file_size"] = g["data_off"] + g["data_size"]
    return g


def file_size(kind: int, codec: int, ch: int, n: int, loop: Optional[Tuple[int, int]], alignment: int = 0) -> int:
    return geometry(kind, codec, ch, n, aligned_loop(codec, loop, alignment)[1])["file_size"]


def aligned_loop(codec: int, loop: Optional[Tuple[int, int]], alignment: int = 0):
    """(status, the format's loop after GcAdpcmFormat.WithAlignment, needed)"""
    if codec != GCADPCM or not loop:
        return 0, loop, False
    rc, (needed, lsa, sca), _, _ = pygcalign.gc_align(alignment or 14336, loop[0], loop[1])
    if rc:
        return E_ARG, None, False
    return 0, ((lsa, sca) if needed else loop), bool(needed)


def check(kind: int, codec: int, ch: int, n: int, loop: Optional[Tuple[int, int]], alignment: int = 0) -> int:
    if ch > 255:
        return E_ARG
    if codec == GCADPCM and n == 0:
        return E_DATA
    st, floop, _ = aligned_loop(codec, loop, alignment)
    if st:
        return st
    if geometry(kind, codec, ch, n, floop)["file_size"] >= 1 << 31:
        return E_ARG
    return 0


def write(kind: int, codec: int, pcm: List[np.ndarray], rate: int, loop: Optional[Tuple[int, int]] = None, endianness: int = 0,
          alignment: int = 0):
    """The file BrstmWriter (kind BRSTM) or BCFstmWriter (BCSTM: version 2.1, BFSTM: version 0.3) writes for channels
    `pcm` (int16, equal lengths) at `rate`, looping over loop = (start, end) or not."""
    ch, n = len(pcm), len(pcm[0])
    s = check(kind, codec, ch, n, loop, alignment)
    if s:
        return s, None
    _, floop, needed = aligned_loop(codec, loop, alignment)
    g = geometry(kind, codec, ch, n, floop)
    be = file_big_endian(kind, endianness)
    adpcm = codec == GCADPCM
    looping = 1 if loop else 0
    ls = floop[0] if loop else 0
    tracks = _tracks(ch)
    T = len(tracks)
    gc = _gc_channels(pcm, loop[0] if loop else None, g["spi"]) if adpcm else None
    w = _W(g["file_size"], be)

    def ctx(c):
        return struct.pack(w.e + "3h", *c)

    if kind == BRSTM:
        marker = 0x01000000
        w.raw(b"RSTM"); w.put("HhIhh", 0xfeff, 0x0100, g["file_size"], 0x40, 2)
        w.put("6I", 0x40, g["head"], g["seek_off"], g["seek_size"], g["data_off"], g["data_size"])
        w.at = 0x40
        h2 = g["h2"]
        w.raw(b"HEAD"); w.put("7I", g["head"], marker, 24, marker, 24 + 0x34, marker, 24 + 0x34 + h2)
        w.put("BBBBHh", codec, looping, ch, 0, rate & 0xffff, 0)
        w.put("11i", ls, g["sc"], g["data_off"] + 0x20, g["icount"], g["bpi"], g["spi"], g["last_np"], g["last_samples"], g["last"],
              g["spi"] if adpcm else 0, 4 if adpcm else 0)
        w.put("BBh", T, 1, 0)
        for t in range(T):
            w.put("II", 0x01010000, 24 + 0x34 + 4 + 8 * T + 0x0c * t)
        for cc, left, right in tracks:
            w.put("BBhiBBBB", 0x7f, 0x40, 0, 0, cc, left, right, 0)
        w.put("BBh", ch, 0, 0)
        base = 24 + 0x34 + h2 + 4
        cis = 0x38 if adpcm else 8
        for c in range(ch):
            w.put("II", marker, base + 8 * ch + cis * c)
        for c in range(ch):
            w.put("I", marker)
            if not adpcm:
                w.put("i", 0)
                continue
            ad, co, start, lc, _ = gc[c]
            w.put("i", base + 8 * ch + cis * c + 8)
            w.put("16h", *[int(v) for v in co]); w.put("h", 0); w.raw(ctx(start)); w.raw(ctx(lc)); w.put("h", 0)
        if adpcm:
            w.at = g["seek_off"]
            w.raw(b"ADPC"); w.put("I", g["seek_size"])
        w.at = g["data_off"]
        w.raw(b"DATA"); w.put("Ii", g["data_size"], 0x18)
        seek_e = ">"
    else:
        track_info = kind == BCSTM
        w.raw(b"CSTM" if kind == BCSTM else b"FSTM"); w.put("Hh", 0xfeff, 0x40)
        w.put("Ii", (0x201 if track_info else 3) << 16, g["file_size"])
        w.put("hh", 3 if adpcm else 2, 0)
        w.put("hhiI", 0x4000, 0, 0x40, g["head"])
        if adpcm:
            w.put("hhiI", 0x4001, 0, g["seek_off"], g["seek_size"])
        w.put("hhiI", 0x4002, 0, g["data_off"], g["data_size"])
        w.at = 0x40
        i1, i2 = g["i1"], g["i2"]
        w.raw(b"INFO"); w.put("I", g["head"])
        w.put("hhi", 0x4100, 0, 24)
        if track_info:
            w.put("hhi", 0x0101, 0, 24 + i1)
        else:
            w.put("ii", 0, -1)
        w.put("hhi", 0x0101, 0, 24 + i1 + i2)
        w.put("BBBBi", codec, looping, ch, 0, rate)
        w.put("10i", ls, g["sc"], g["icount"], g["bpi"], g["spi"], g["last_np"], g["last_samples"], g["last"], 4, g["spi"])
        w.put("hhi", 0x1F00, 0, 0x18)
        w.put("hhii", 0x0100, 0, 0, -1)
        if track_info:
            w.put("i", T)
            for t in range(T):
                w.put("hhi", 0x4101, 0, (4 + 8 * T) + (4 + 8 * ch) + 0x14 * t)
        w.put("i", ch)
        for c in range(ch):
            w.put("hhi", 0x4102, 0, (4 + 8 * ch) + (0x14 * T if track_info else 0) + 8 * c)
        if track_info:
            for cc, left, right in tracks:
                w.put("BBhhhiiBBh", 0x7f, 0x40, 0, 0x0100, 0, 0xc, cc, left, right, 0)
        for c in range(ch):
            if adpcm:
                w.put("hhi", 0x0300, 0, 8 * ch - 8 * c + 0x2e * c)
            else:
                w.put("ii", 0, -1)
        if adpcm:
            for ad, co, start, lc, _ in gc:
                w.put("16h", *[int(v) for v in co]); w.raw(ctx(start)); w.raw(ctx(lc)); w.put("h", 0)
            w.at = g["seek_off"]
            w.raw(b"SEEK"); w.put("I", g["seek_size"])
        w.at = g["data_off"]
        w.raw(b"DATA"); w.put("I", g["data_size"])
        seek_e = "<"  # BCFstmWriter.WriteSeekBlock: BuildSeekTable(..., Endianness.LittleEndian) in either byte order
    if adpcm:
        # GcAdpcmFormat.BuildSeekTable: tables.Interleave(2), Array.Resize to entries * 2 * channels
        tabs = [t for *_, t in gc]
        inter = np.stack([t.reshape(-1, 2) for t in tabs], axis=1).reshape(-1)
        want = g["entries"] * 2 * ch
        table = np.zeros(want, dtype=np.int16)
        m = min(want, len(inter))
        table[:m] = inter[:m]
        w.at = g["seek_off"] + 8
        w.raw(table.astype(seek_e + "i2").tobytes())
        arrays = [np.asarray(ad, dtype=np.uint8) for ad, *_ in gc]
        if needed:  # GcAdpcmChannel.GetAdpcmAudio: AdpcmAligned
            arrays = [pygcalign.gc_align(alignment or 14336, loop[0], loop[1], ad, co)[2] for ad, co, *_ in gc]
    elif codec == PCM16:
        arrays = [np.asarray(p, dtype=np.int16).astype((">" if be else "<") + "i2").view(np.uint8) for p in pcm]
    else:
        arrays = [(np.asarray(p, dtype=np.int16) >> 8).astype(np.uint8) for p in pcm]  # Pcm8Codec.EncodeSigned
    data_at = g["data_off"] + 0x20
    if g["ads"] and arrays[0].size:
        region = O.interleave([np.ascontiguousarray(a) for a in arrays], g["bpi"], g["ads"])
        w.b[data_at:data_at + len(region)] = bytes(region)
    return 0, np.frombuffer(bytes(w.b), dtype=np.uint8).copy()


def wave_write8(channels: List[np.ndarray], sample_rate: int, loop: Optional[Tuple[int, int]] = None) -> np.ndarray:
    """An 8-bit PCM WAVE image (unsigned samples), with a smpl loop when loop is given."""
    ch, n = len(channels), len(channels[0])
    data = np.stack([np.asarray(c, dtype=np.uint8) for c in channels], axis=1).reshape(-1).tobytes()
    fmt = struct.pack("<HHIIHH", 1, ch, sample_rate, sample_rate * ch, ch, 8)
    chunks = b"fmt " + struct.pack("<I", len(fmt)) + fmt
    if loop:
        smpl = bytearray(0x3c)
        struct.pack_into("<I", smpl, 28, 1)
        struct.pack_into("<II", smpl, 44, loop[0], loop[1])
        chunks += b"smpl" + struct.pack("<I", len(smpl)) + bytes(smpl)
    chunks += b"data" + struct.pack("<I", len(data)) + data + (b"\0" if len(data) & 1 else b"")
    return np.frombuffer(b"RIFF" + struct.pack("<I", 4 + len(chunks)) + b"WAVE" + chunks, dtype=np.uint8).copy()
