"""Builders of NintendoWare wave and prefetch images for the tests, hand-assembled in the layout the reference readers
walk: .brwav (RWAV, big-endian: file header, INFO with the wave info, its channel table and per-channel ADPCM info, DATA
with every channel as its own run), .bcwav / .bfwav (CWAV / FWAV in either byte order: block references, a wave info
block whose channel table carries each channel's audio offset, a wave data block) and .bcstp / .bfstp (a stream image of
nw_files whose DATA block is replaced by a PDAT block of one or more prefetch regions).

Channel offsets are given per channel (relative to the DATA payload), so tests can put the runs in order, reversed,
overlapping, with gaps or past the image's end."""
from __future__ import annotations

import struct
from typing import List, Optional, Sequence

import numpy as np

import nw_files as F
from nw_files import Channel, GCADPCM, PCM16, PCM8, samples_to_bytes  # noqa: F401  (re-exported)

BRWAV, BCWAV, BFWAV, BCSTP, BFSTP = 9, 10, 11, 12, 13
BCWAV_VERSIONS = (0x02010000, 0x02010100)   # without / with the unaligned loop start (BCWAV 2.1.1)
BFWAV_VERSIONS = (0x00010100, 0x00010200)   # without / with the unaligned loop start (BFWAV 0.1.2)


def sample_to_nibble(n: int) -> int:
    """GcAdpcmMath.SampleToNibble: NibbleToSample of it gives n back."""
    return 16 * (n // 14) + n % 14 + 2


def layout(kind: str, sizes: Sequence[int]) -> List[int]:
    """Channel offsets into the DATA payload for runs of the given sizes: "ordered", "reversed", "overlap" (every channel
    shares channel 0's run from its middle on), "gaps" (0x60 spare bytes between runs)."""
    step = [-(-s // 0x20) * 0x20 for s in sizes]
    if kind == "ordered":
        return [sum(step[:c]) for c in range(len(sizes))]
    if kind == "gaps":
        return [sum(step[:c]) + 0x60 * (c + 1) for c in range(len(sizes))]
    if kind == "reversed":
        return [sum(step[c + 1:]) for c in range(len(sizes))]
    if kind == "overlap":
        return [(c * sizes[0] // (2 * len(sizes))) & ~0x7 for c in range(len(sizes))]
    raise ValueError(kind)


def _payload(chans: Sequence[Channel], offsets: Sequence[int], length: int, cut: int) -> bytes:
    """The DATA payload: each channel's bytes (cut or zero-padded to `length`) at its offset; `cut` bytes dropped from the
    end so that the last run reaches past the image."""
    end = max([o + length for o in offsets] + [0])
    out = bytearray(end)
    for k, o in zip(chans, offsets):
        d = bytes(k.data[:length]).ljust(length, b"\0")
        out[o: o + length] = d
    return bytes(out[: max(0, len(out) - cut)])


def rwav(codec: int, chans: Sequence[Channel], sample_count: int, rate: int = 32000, loop: Optional[int] = None,
         offsets: Optional[Sequence[int]] = None, cut: int = 0, nibble_fields: bool = True, magic: bytes = b"RWAV",
         file_size_delta: int = 0, channel_count: Optional[int] = None) -> np.ndarray:
    """An RWAV image.  The loop start and sample count fields are written as nibbles (nibble_fields) so that the reader's
    NibbleToSample gives them back; with nibble_fields=False they are written raw, as a PCM file may hold them."""
    E = ">"
    ch = len(chans) if channel_count is None else channel_count
    length = samples_to_bytes(sample_count, codec)
    if offsets is None:
        offsets = layout("ordered", [length] * len(chans))
    enc = sample_to_nibble if nibble_fields else (lambda v: v)
    info = bytearray(b"INFO\0\0\0\0")
    base = len(info)
    body = bytearray(struct.pack(E + "BBBxHxx", codec, int(loop is not None), ch, rate & 0xFFFF))
    body += struct.pack(E + "ii", enc(loop or 0), enc(sample_count))
    table_at = len(body) + 8
    body += struct.pack(E + "ii", table_at, 0)
    body += b"\0" * (4 * ch)
    for c in range(ch):
        struct.pack_into(E + "i", body, table_at + 4 * c, len(body))
        k = chans[c] if c < len(chans) else Channel(b"")
        adpcm_at = len(body) + 24
        body += struct.pack(E + "6i", offsets[c] if c < len(offsets) else 0, adpcm_at, 0x7F, 0x7F, 0, 0)
        body += struct.pack(E + "16h", *[int(v) for v in k.coefs]) + struct.pack(E + "h", k.gain)
        body += struct.pack(E + "3h3hxx", *k.start, *k.loop)
    struct.pack_into(E + "i", body, 20, len(body))
    info += body
    F._pad(info)
    struct.pack_into(E + "i", info, 4, len(info))
    head_off = 0x20
    data_off = head_off + len(info)
    data = bytearray(b"DATA\0\0\0\0") + _payload(chans, offsets, length, cut)
    struct.pack_into(E + "i", data, 4, len(data))
    img = bytearray(0x20) + info + data
    struct.pack_into(E + "4sHBBihh4i", img, 0, magic, 0xFEFF, 1, 2, len(img) + file_size_delta, 0x20, 2,
                     head_off, len(info), data_off, len(data))
    return np.frombuffer(bytes(img), dtype=np.uint8).copy()


def _header(E, mg, v, blocks):
    header = bytearray(0x14 + 12 * len(blocks))
    F._pad(header)
    off = len(header)
    out = bytearray(header)
    for i, (t, b) in enumerate(blocks):
        struct.pack_into(E + "hHii", out, 0x14 + 12 * i, t, 0, off, len(b))
        out += b
        off += len(b)
    struct.pack_into(E + "4sHHIihH", out, 0, mg, 0xFEFF, 0x40, v, len(out), len(blocks), 0)
    out[0:4] = mg
    return out


def cwav(kind: int, codec: int, chans: Sequence[Channel], sample_count: int, rate: int = 32000, loop: Optional[int] = None,
         big_endian: Optional[bool] = None, version: Optional[int] = None, offsets: Optional[Sequence[int]] = None, cut: int = 0,
         magic: Optional[bytes] = None, wave_refs: Optional[Sequence[bool]] = None, adpcm_info: bool = True,
         channel_count: Optional[int] = None) -> np.ndarray:
    """A CWAV (kind BCWAV, little-endian by default) or FWAV (BFWAV, big-endian by default) image.  wave_refs[c] False
    writes channel c's reference as a plain (non-wave) channel info, with no audio offset; adpcm_info False leaves the
    GC-ADPCM info references out."""
    be = (kind == BFWAV) if big_endian is None else big_endian
    E = ">" if be else "<"
    v = version if version is not None else (BCWAV_VERSIONS[1] if kind == BCWAV else BFWAV_VERSIONS[1])
    ch = len(chans) if channel_count is None else channel_count
    length = samples_to_bytes(sample_count, codec)
    if offsets is None:
        offsets = layout("ordered", [length] * len(chans))
    refs = [True] * ch if wave_refs is None else list(wave_refs)
    info = bytearray(b"INFO\0\0\0\0")
    body = bytearray(struct.pack(E + "BBxx", codec, int(loop is not None)))
    body += struct.pack(E + "iiii", rate, loop or 0, sample_count, loop or 0)  # the last: unaligned loop start or padding
    tbase = len(body)
    body += struct.pack(E + "i", ch) + b"\0" * (8 * ch)
    for c in range(ch):
        entry = len(body)
        struct.pack_into(E + "hHi", body, tbase + 4 + 8 * c, 0x7100 if refs[c] else 0x0100, 0, entry - tbase)
        if refs[c]:
            body += struct.pack(E + "hHi", 0x1F00, 0, offsets[c] if c < len(offsets) else 0)
        adpcm_ref = len(body)
        body += b"\0" * 8 + b"\0" * 8  # the ADPCM info reference, then the (unused) reserved reference
        if adpcm_info:
            struct.pack_into(E + "hHi", body, adpcm_ref, 0x0300, 0, len(body) - entry)
            k = chans[c] if c < len(chans) else Channel(b"")
            body += struct.pack(E + "16h", *[int(x) for x in k.coefs]) + struct.pack(E + "3h3hxx", *k.start, *k.loop)
    info += body
    F._pad(info)
    struct.pack_into(E + "i", info, 4, len(info))
    data = bytearray(b"DATA\0\0\0\0") + _payload(chans, offsets, length, cut)
    struct.pack_into(E + "i", data, 4, len(data))
    mg = magic or (b"CWAV" if kind == BCWAV else b"FWAV")
    out = _header(E, mg, v, [(0x7000, info), (0x7001, data)])
    return np.frombuffer(bytes(out), dtype=np.uint8).copy()


def cstp(kind: int, codec: int, chans: Sequence[Channel], sample_count: int, prefetch: Sequence[int], interleave: int = 0x400,
         big_endian: Optional[bool] = None, loop: Optional[int] = None, magic: Optional[bytes] = None, count: Optional[int] = None,
         **kw) -> np.ndarray:
    """A CSTP (kind BCSTP) or FSTP (BFSTP) image: the stream image nw_files builds with its DATA block replaced by a PDAT
    block of len(prefetch) entries.  Entry i holds prefetch[i] bytes per channel, interleaved; entry 0 starts at the
    track's start, the others follow it.  count overrides the stated entry count."""
    be = (kind == BFSTP) if big_endian is None else big_endian
    E = ">" if be else "<"
    stream_kind = F.BCSTM if kind == BCSTP else F.BFSTM
    img = bytearray(F.build(stream_kind, codec, list(chans), sample_count, loop=loop, interleave=interleave, big_endian=be,
                            seek="none", **kw).tobytes())
    n_blocks = struct.unpack_from(E + "h", img, 0x10)[0]
    at = next(0x14 + 12 * i for i in range(n_blocks) if struct.unpack_from(E + "h", img, 0x14 + 12 * i)[0] == 0x4002)
    data_off = struct.unpack_from(E + "i", img, at + 4)[0]
    ch = len(chans)
    n = len(prefetch)
    pdat = bytearray(b"PDAT\0\0\0\0") + struct.pack(E + "i", n if count is None else count) + b"\0" * (20 * n)
    F._pad(pdat)
    pos = 0
    for i, per in enumerate(prefetch):
        region = F._interleave([bytes(k.data[pos: pos + per]) for k in chans], per, interleave)
        entry = 12 + 20 * i  # StartSample, Size, padding, the audio reference
        struct.pack_into(E + "iiihHi", pdat, entry, 0, per * ch, 0, 0x1F00, 0, len(pdat) - entry)
        pdat += region
        F._pad(pdat)
        pos += per
    struct.pack_into(E + "i", pdat, 4, len(pdat))
    out = img[:data_off] + pdat
    struct.pack_into(E + "hHii", out, at, 0x4004, 0, data_off, len(pdat))
    struct.pack_into(E + "i", out, 0x0C, len(out))
    out[0:4] = magic or (b"CSTP" if kind == BCSTP else b"FSTP")
    return np.frombuffer(bytes(out), dtype=np.uint8).copy()


def channels(oracle, codec: int, n_ch: int, n: int, seed: int, big_endian: bool, loop: Optional[int] = None) -> List[Channel]:
    pcm = F.pcm_channels(n_ch, n, seed)
    if codec == GCADPCM:
        return F.gc_channels(oracle, pcm, loop or 0, (seed * 37 % 900, -seed * 11 % 700))
    if codec == PCM16:
        return F.pcm16_channels(pcm, big_endian)
    return F.pcm8_channels(pcm)


def encoded(oracle, kind: int, codec: int, n_ch: int, n: int, loop: Optional[int] = None, seed: int = 0,
            big_endian: Optional[bool] = None, layout_kind: str = "ordered", prefetch: Optional[Sequence[int]] = None,
            **kw) -> np.ndarray:
    """An image of `kind` with n_ch seeded channels of n samples in `codec`."""
    be = True if kind == BRWAV else (kind in (BFWAV, BFSTP) if big_endian is None else big_endian)
    chans = channels(oracle, codec, n_ch, n, seed, be, loop)
    if kind in (BCSTP, BFSTP):
        per = samples_to_bytes(n, codec)
        return cstp(kind, codec, chans, n, prefetch if prefetch is not None else [per], big_endian=be, loop=loop, **kw)
    offsets = layout(layout_kind, [samples_to_bytes(n, codec)] * n_ch)
    if kind == BRWAV:
        return rwav(codec, chans, n, loop=loop, offsets=offsets, **kw)
    return cwav(kind, codec, chans, n, loop=loop, big_endian=be, offsets=offsets, **kw)
