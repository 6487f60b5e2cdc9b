"""CPU restatement of IdspWriter (Containers/Idsp/IdspWriter.cs, IdspConfiguration's block size of 16 bytes) and
HpsWriter (Containers/Hps/HpsWriter.cs), written apart from the product's C++ sizing pass and assembly kernels so that
the tests can compare the two.  The GC-ADPCM channels come from the C oracle (CalculateCoefficients, Encode, Decode, the
loop context, GcAdpcmAlignment and InterleaveExtensions.Interleave).

The channel rules follow GcAdpcmChannelBuilder (PrepareForBuild, GetAlignment, GetLoopContext), GcAdpcmChannel's
constructor and GetCloneBuilder as the two writers chain them:

- IDSP (SetupWriter: WithAlignment(ByteCountToSampleCount(16)) = 28 samples).  The rebuild reuses the loop context of the
  first encode, taken at the UNALIGNED loop start (GetAlignment sets AlignedLoopStart = alignment.LoopStart, the unaligned
  one).  With loop start 0, or without a loop, the first build takes CurrentLoopContextIsValid(0) without a decode, so the
  loop context is (0, 0, 0).
- HPS: each block's predictor/scale comes from GetAdpcmAudio() (AdpcmAligned when the loop moved), but Hist1 / Hist2
  come from the channel's Pcm, which is the first encode's full decode in every case: AlignmentNeeded keeps Pcm = b.Pcm,
  and the per-channel rebuild reuses PreviousAlignment without touching AlignedPcm.  That decode is only sample_count
  long, so in a file whose loop moved, a block with StartSample - 1 >= sample_count makes GcAdpcmLoopContext.GetHist1
  index past it: the reference throws IndexOutOfRangeException, and write() refuses the file.

write_*() return (0, file bytes) or (E_ARG / E_DATA, None) for the per-file refusals."""
from __future__ import annotations

import struct
from typing import List, Optional, Tuple

import numpy as np

from oracle import pyoracle as O
from oracle import pygcalign

E_DATA, E_ARG = -2, -1
IDSP, HPS = 7, 8
IDSP_BLOCK = 16
IDSP_ALIGNMENT = 28  # ByteCountToSampleCount(16)


def _next_multiple(v: int, m: int) -> int:
    return v if v % m == 0 else v + m - v % m


def nibble_count(n: int) -> int:  # SampleCountToNibbleCount
    return n // 14 * 16 + (n % 14 + 2 if n % 14 else 0)


def sample_to_nibble(s: int) -> int:
    return s // 14 * 16 + s % 14 + 2


def nibble_to_sample(nb: int) -> int:
    return nb // 16 * 14 + nb % 16 - 2


def byte_count_to_sample_count(b: int) -> int:  # NibbleCountToSampleCount(b * 2)
    nb = b * 2
    return nb // 16 * 14 + (nb % 16 - 2 if nb % 16 else 0)


def _alignment(multiple: int, loop):
    """(status, the format's (sample_count, loop_start, loop_end) after WithAlignment, needed, sca)"""
    if not loop:
        return 0, None, False
    rc, (needed, lsa, sca), _, _ = pygcalign.gc_align(multiple, loop[0], loop[1])
    if rc:
        return E_ARG, None, False
    return 0, ((lsa, sca) if needed else loop), bool(needed)


# ---- IDSP -------------------------------------------------------------------------------------------------------------
def idsp_geometry(ch: int, n: int, loop, trim: bool = True):
    st, floop, needed = _alignment(IDSP_ALIGNMENT, loop)
    if st:
        return st, None
    fsc = floop[1] if needed else n                                    # GcAdpcmFormat.SampleCount
    ls, le = floop if loop else (0, 0)
    sc = le if trim and loop else max(fsc, le)                         # IdspWriter.SampleCount
    ads = _next_multiple(O.sample_count_to_byte_count(sc), IDSP_BLOCK)
    head = 0x40 + 0x60 * ch
    return 0, dict(sc=sc, ls=ls, le=le, ads=ads, head=head, file_size=head + ads * ch, needed=needed,
                   chan_sc=floop[1] if needed else n)


def idsp_check(ch: int, n: int, loop, trim: bool = True) -> int:
    if ch > 255:
        return E_ARG
    if n == 0:
        return E_DATA
    st, g = idsp_geometry(ch, n, loop, trim)
    if st:
        return st
    return E_ARG if g["file_size"] >= 1 << 31 else 0


def write_idsp(pcm: List[np.ndarray], rate: int, loop: Optional[Tuple[int, int]] = None, trim: bool = True):
    ch, n = len(pcm), len(pcm[0])
    st = idsp_check(ch, n, loop, trim)
    if st:
        return st, None
    _, g = idsp_geometry(ch, n, loop, trim)
    out = bytearray(g["file_size"])
    struct.pack_into(">4s11i", out, 0, b"IDSP", 0, ch, rate, g["sc"], g["ls"], g["le"], IDSP_BLOCK, 0x40, 0x60, g["head"], g["ads"])
    arrays = []
    for c, p in enumerate(pcm):
        co = O.calculate_coefficients(p)
        ad = O.encode(p, co)
        ctx = (0, 0, 0)
        if loop and loop[0] > 0:  # the first build's decode at the unaligned loop start
            ctx = O.gc_loop_context(ad, O.decode(ad, co, n), loop[0])
        start_addr = sample_to_nibble(g["ls"] if loop else 0)
        end_addr = sample_to_nibble(g["le"] if loop else g["sc"] - 1)
        struct.pack_into(">iiihhiii16hh3h3h", out, 0x40 + 0x60 * c, g["chan_sc"], nibble_count(g["chan_sc"]), rate, 1 if loop else 0, 0,
                         start_addr, end_addr, 2, *[int(v) for v in co], 0, int(ad[0]), 0, 0, *ctx)
        arrays.append(pygcalign.gc_align(IDSP_ALIGNMENT, loop[0], loop[1], ad, co)[2] if g["needed"] else np.asarray(ad, dtype=np.uint8))
    region = O.interleave([np.ascontiguousarray(a) for a in arrays], IDSP_BLOCK, g["ads"])
    out[g["head"]:g["head"] + len(region)] = bytes(region)
    return 0, np.frombuffer(bytes(out), dtype=np.uint8).copy()


# ---- HPS --------------------------------------------------------------------------------------------------------------
def hps_channel_size(ch: int) -> int:
    return _next_multiple(0x10000 // ch, 0x20)


def hps_geometry(ch: int, n: int, loop):
    """(status, geometry with the block map) as SetupWriter and CreateBlockMap build it"""
    cs = hps_channel_size(ch)
    alignment = byte_count_to_sample_count(cs)
    st, floop, needed = _alignment(alignment, loop)
    if st:
        return st, None
    sc = floop[1] if needed else n                                     # GcAdpcmFormat.SampleCount
    ls = floop[0] if loop else 0
    head = _next_multiple(max(0x80, 0x10 + 0x38 * ch), 0x20)
    nibbles = nibble_count(sc)
    M = cs * ch // ch * 2
    count = -(-nibbles // M)
    loop_block = sample_to_nibble(ls) // M if loop else count - 1
    blocks, cur = [], 0
    while len(blocks) < loop_block:
        blocks.append((cur, M))
        cur += M
    while cur < nibbles:
        left, rem = count - len(blocks), nibbles - cur
        size = min(rem, _next_multiple(-(-rem // left), 0x40))
        blocks.append((cur, size))
        cur += size
    if len(blocks) != count:  # CreateBlockMap would leave a null block behind
        return E_ARG, None
    hdr = _next_multiple(4 + 8 * ch, 0x20)
    out, at = [], head
    for nib, size in blocks:
        cs_b = -(-size // 2)
        written = _next_multiple(cs_b, 0x20) * ch
        out.append(dict(offset=at, start=nibble_to_sample(nib + 2), byte_in=nib // 2, end_nibble=size - 1, chan_size=cs_b,
                        written=written))
        at += hdr + written
    for i, b in enumerate(out):
        b["next"] = out[i + 1]["offset"] if i + 1 < len(out) else (out[loop_block]["offset"] if loop else -1)
    return 0, dict(sc=sc, ls=ls, head=head, hdr=hdr, blocks=out, file_size=at, needed=needed, loop_block=loop_block)


def hps_check(ch: int, n: int, loop) -> int:
    if ch > 255:
        return E_ARG
    if n == 0:
        return E_DATA
    if ch % 4 == 3:  # WriteBlock writes 12 + 8 * ch header bytes where the block map leaves GetNextMultiple(4 + 8 * ch, 0x20)
        return E_ARG
    st, g = hps_geometry(ch, n, loop)
    if st:
        return st
    if g["file_size"] >= 1 << 31:
        return E_ARG
    if g["needed"] and any(b["start"] - 1 >= n for b in g["blocks"]):  # GetHist1 past the first decode
        return E_ARG
    return 0


def write_hps(pcm: List[np.ndarray], rate: int, loop: Optional[Tuple[int, int]] = None):
    ch, n = len(pcm), len(pcm[0])
    st = hps_check(ch, n, loop)
    if st:
        return st, None
    _, g = hps_geometry(ch, n, loop)
    out = bytearray(g["file_size"])
    struct.pack_into(">8sii", out, 0, b" HALPST\0", rate, ch)
    arrays, decs = [], []
    for c, p in enumerate(pcm):
        co = O.calculate_coefficients(p)
        ad = O.encode(p, co)
        decs.append(O.decode(ad, co, n))
        struct.pack_into(">iiii16hh3h", out, 0x10 + 0x38 * c, 0x10000, 2, sample_to_nibble(g["sc"] - 1), 2, *[int(v) for v in co], 0,
                         int(ad[0]), 0, 0)
        arrays.append(pygcalign.gc_align(byte_count_to_sample_count(hps_channel_size(ch)), loop[0], loop[1], ad, co)[2]
                      if g["needed"] else np.asarray(ad, dtype=np.uint8))
    for b in g["blocks"]:
        at = b["offset"]
        struct.pack_into(">iii", out, at, b["written"], b["end_nibble"], b["next"])
        s = b["start"]
        for c in range(ch):
            h1 = int(decs[c][s - 1]) if s >= 1 else 0
            h2 = int(decs[c][s - 2]) if s >= 2 else 0
            struct.pack_into(">hhhh", out, at + 12 + 8 * c, int(arrays[c][s // 14 * 8]), h1, h2, 0)
        at += g["hdr"]
        for c in range(ch):
            out[at:at + b["chan_size"]] = bytes(arrays[c][b["byte_in"]:b["byte_in"] + b["chan_size"]])
            at += _next_multiple(b["chan_size"], 0x20)
    return 0, np.frombuffer(bytes(out), dtype=np.uint8).copy()


# ---- test-side readers (IdspReader.cs, HpsReader.cs) ------------------------------------------------------------------
def parse_idsp(f) -> dict:
    b = bytes(f)
    assert b[:4] == b"IDSP"
    _, ch, rate, sc, ls, le, block, si, ci, head, ads = struct.unpack_from(">11i", b, 4)
    chans = []
    for c in range(ch):
        v = struct.unpack_from(">iiihhiii16hh3h3h", b, si + ci * c)
        chans.append(dict(sample_count=v[0], nibble_count=v[1], looping=v[3], start_addr=v[5], end_addr=v[6], coefs=list(v[8:24]),
                          start=v[25:28], loop=v[28:31]))
    data = np.frombuffer(b, dtype=np.uint8, offset=head, count=ads * ch)
    arrays = data.reshape(-1, ch, block).transpose(1, 0, 2).reshape(ch, -1)  # every block is full: ads is a multiple of 16
    return dict(channels=ch, rate=rate, sample_count=sc, loop_start=ls, loop_end=le, block=block, header_size=head,
                audio_data_size=ads, chans=chans, arrays=arrays)


def parse_hps(f) -> dict:
    b = bytes(f)
    assert b[:8] == b" HALPST\0"
    rate, ch = struct.unpack_from(">ii", b, 8)
    chans = []
    for c in range(ch):
        v = struct.unpack_from(">iiii16hh3h", b, 0x10 + 0x38 * c)
        chans.append(dict(max_block=v[0], end_address=v[2], coefs=list(v[4:20]), start=v[21:24]))
    pos = _next_multiple(max(0x80, 0x10 + 0x38 * ch), 0x20)
    blocks, cur, audio = [], 0, [bytearray() for _ in range(ch)]
    while pos > cur:
        cur = pos
        size, final, nxt = struct.unpack_from(">iii", b, cur)
        ctx = [struct.unpack_from(">hhh", b, cur + 12 + 8 * c) for c in range(ch)]
        start = _next_multiple(cur + 12 + 8 * ch, 0x20)
        n_bytes = -(-(final + 1) // 2)
        for c in range(ch):
            at = start + size // ch * c
            audio[c] += b[at:at + n_bytes]
        blocks.append(dict(offset=cur, size=size, final_nibble=final, next=nxt, ctx=ctx))
        pos = nxt
    loop_start, looping = 0, blocks[-1]["next"] != -1
    if looping:
        nib = 0
        for blk in blocks:
            if blk["offset"] == blocks[-1]["next"]:
                break
            nib += blk["final_nibble"] + 1
        loop_start = nibble_to_sample(nib + 2)
    return dict(channels=ch, rate=rate, chans=chans, blocks=blocks, looping=looping, loop_start=loop_start,
                sample_count=nibble_to_sample(chans[0]["end_address"]) + 1, arrays=[np.frombuffer(bytes(a), dtype=np.uint8) for a in audio])
