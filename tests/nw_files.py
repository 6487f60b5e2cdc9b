"""Builders of NintendoWare stream images for the tests: .brstm (big-endian), .bcstm (little-endian) and .bfstm (either
byte order, several versions), written field by field from the formats' block structure (file header with block
references, HEAD / INFO with stream, track and channel info, ADPC / SEEK seek tables, REGN, DATA with the audio
interleaved in blocks).  Audio: GC-ADPCM from the oracle's encoder, PCM16 / PCM8 from seeded PCM.

Every field a test may want to break is a keyword of `build`; the defaults describe a well-formed file."""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from vgaudio_b200 import synth

BRSTM, BCSTM, BFSTM = 4, 5, 6
PCM8, PCM16, GCADPCM = 0, 1, 2
BCSTM_VERSIONS = (0x02000000, 0x02010000, 0x02030000)       # no region info / region info / + unaligned loop
BFSTM_VERSIONS = (0x00030000, 0x00040000, 0x00050000)       # region info / + unaligned loop / + checksum


def gc_bytes(n: int) -> int:
    """GcAdpcmMath.SampleCountToByteCount for n >= 0."""
    whole, rest = divmod(n, 14)
    nib = 16 * whole + (rest + 2 if rest else 0)
    return nib // 2 + nib % 2


def samples_to_bytes(n: int, codec: int) -> int:
    return gc_bytes(n) if codec == GCADPCM else (2 * n if codec == PCM16 else (n if codec == PCM8 else 0))


@dataclass
class Channel:
    data: bytes                      # the channel's audio bytes in file order
    coefs: np.ndarray = field(default_factory=lambda: np.zeros(16, np.int16))
    gain: int = 0
    start: tuple = (0, 0, 0)         # PredScale, Hist1, Hist2
    loop: tuple = (0, 0, 0)


def pcm_channels(channels: int, n: int, seed: int, silent: Optional[tuple] = None) -> List[np.ndarray]:
    out = []
    for c in range(channels):
        x = synth.channel(1000 * seed + c + 4, n, 48000, degenerate=False)
        if silent:
            x = x.copy()
            x[silent[0]:silent[1]] = 0
        out.append(x)
    return out


def gc_channels(oracle, pcm: List[np.ndarray], loop_start: int = 0, start_hist=(0, 0)) -> List[Channel]:
    """Encodes each channel with the oracle (start history as given); the loop context from the oracle's decode."""
    out = []
    for p in pcm:
        co = oracle.calculate_coefficients(p)
        ad = oracle.encode(p, co, -1, start_hist[0], start_hist[1])
        dec = oracle.decode(ad, co, len(p), start_hist[0], start_hist[1])
        ctx = oracle.gc_loop_context(ad, dec, loop_start) if len(p) else (0, 0, 0)
        out.append(Channel(ad.tobytes(), co, 0, (int(ad[0]) if ad.size else 0, start_hist[0], start_hist[1]), tuple(int(v) for v in ctx)))
    return out


def pcm16_channels(pcm: List[np.ndarray], big_endian: bool) -> List[Channel]:
    return [Channel(np.asarray(p, dtype=">i2" if big_endian else "<i2").tobytes()) for p in pcm]


def pcm8_channels(pcm: List[np.ndarray]) -> List[Channel]:
    return [Channel((np.asarray(p, np.int16) >> 8).astype(np.int8).tobytes()) for p in pcm]


def _interleave(rows: List[bytes], in_size: int, interleave: int) -> bytes:
    """The audio region Stream.DeInterleave reads back: rows cut or zero-padded to in_size bytes, blocks of `interleave`
    bytes per channel, the last block shorter."""
    ch = len(rows)
    padded = [bytes(r[:in_size]).ljust(in_size, b"\0") for r in rows]
    if in_size == 0 or ch == 0:
        return b""
    if interleave <= 0:
        return b"".join(padded)
    out = bytearray()
    for b in range(0, in_size, interleave):
        for r in padded:
            out += r[b: b + interleave]
    return bytes(out)


def _pad(b: bytearray, m: int = 0x20) -> None:
    b += b"\0" * (-len(b) % m)


def build(kind: int, codec: int, chans: List[Channel], sample_count: int, rate: int = 32000, loop: Optional[int] = None,
          interleave: int = 0x2000, in_size: Optional[int] = None, big_endian: Optional[bool] = None,
          version: Optional[int] = None, seek: str = "standard", regions: int = 0, tracks: int = 1, track_type: int = 1,
          spe: int = 0x3800, magic: Optional[bytes] = None, file_size_delta: int = 0, channel_count: Optional[int] = None,
          adpcm_info: Optional[int] = None, audio_skew: int = 0) -> np.ndarray:
    """One stream image.  loop: loop start (None: not looping).  in_size: bytes per channel in the DATA region (default
    SamplesToBytes(sample_count)); seek: "standard", "short" (BRSTM), "unknown" (a size matching neither), "none";
    regions: REGN entries (BCFSTM; 0 = no block); adpcm_info: channel infos written (default: all); audio_skew: bytes
    added to the audio offset (and the DATA size), shifting where the region starts."""
    be = True if kind == BRSTM else bool(big_endian)
    E = ">" if be else "<"
    ch = len(chans) if channel_count is None else channel_count
    if in_size is None:
        in_size = samples_to_bytes(sample_count, codec)
    audio = _interleave([c.data for c in chans], in_size, interleave)
    n_info = len(chans) if adpcm_info is None else adpcm_info
    looping = loop is not None
    loop_start = loop or 0
    blocks_n = -(-in_size // interleave) if interleave > 0 and in_size else 0
    last = in_size - (blocks_n - 1) * interleave if blocks_n else 0
    spi = interleave * 14 // 8 if codec == GCADPCM else interleave // max(1, 2 if codec == PCM16 else 1)
    if kind == BRSTM:
        return _brstm(codec, chans, ch, sample_count, rate, looping, loop_start, interleave, blocks_n, last, spi, spe, audio,
                      seek, tracks, track_type, n_info, magic, file_size_delta, audio_skew)
    v = version if version is not None else (BCSTM_VERSIONS[2] if kind == BCSTM else BFSTM_VERSIONS[2])
    return _bcfstm(kind, E, codec, chans, ch, sample_count, rate, looping, loop_start, interleave, blocks_n, last, spi, spe, audio,
                   v, seek, regions, tracks, n_info, magic, file_size_delta, audio_skew)


def _seek_table(E, chans, entries):
    out = bytearray()
    for e in range(entries):
        for c in range(len(chans)):
            out += struct.pack(E + "hh", (e * 7 + c) % 3000, -(e * 5 + c) % 2000)
    return bytes(out)


def _brstm(codec, chans, ch, n, rate, looping, loop_start, ilv, blocks_n, last, spi, spe, audio, seek, tracks, track_type,
           n_info, magic, file_size_delta, audio_skew):
    E = ">"
    # HEAD: three references, stream info, track info, channel info
    head = bytearray(b"HEAD\0\0\0\0")
    base = 8
    body = bytearray(24)  # the three references
    stream_off = len(body)
    body += b"\0" * 52
    track_off = len(body)
    body += struct.pack(E + "BBH", tracks, track_type, 0)
    trefs = len(body)
    body += b"\0" * (8 * tracks)
    for t in range(tracks):
        struct.pack_into(E + "hHi", body, trefs + 8 * t, 0x0100 | track_type, 0, len(body))
        if track_type == 1:
            body += struct.pack(E + "BB6x", 0x7F, 0x40)
        body += struct.pack(E + "BBBx", min(ch, 2), 2 * t, 2 * t + 1)
    chan_off = len(body)
    body += struct.pack(E + "B3x", n_info)
    crefs = len(body)
    body += b"\0" * (8 * n_info)
    for c in range(n_info):
        struct.pack_into(E + "hHi", body, crefs + 8 * c, 0x0100, 0, len(body))
        inner = len(body)
        body += b"\0" * 8
        struct.pack_into(E + "hHi", body, inner, 0x0100, 0, len(body))
        k = chans[c] if c < len(chans) else Channel(b"")
        body += struct.pack(E + "16h", *[int(v) for v in k.coefs]) + struct.pack(E + "h", k.gain)
        body += struct.pack(E + "3h3hxx", *k.start, *k.loop)
    for i, off in enumerate((stream_off, track_off, chan_off)):
        struct.pack_into(E + "hHi", body, 8 * i, 0x0100, 0, off)
    head += body
    _pad(head)
    head_off = 0x40
    seek_off = head_off + len(head)
    # ADPC
    adpc = bytearray()
    if seek != "none":
        bpe = 4 * ch
        full_last = spe > 0 and n % spe == 0 and n > 0
        n_std = n // spe + (0 if full_last else 1) if spe > 0 else 1   # (spe 0: a file the reader must refuse)
        n_short = gc_bytes(n) // spe + 1 if spe > 0 else 1
        entries = {"standard": n_std, "short": n_short, "unknown": n_std + 3}[seek]
        size = -(-(8 + entries * bpe) // 0x20) * 0x20
        if seek == "unknown" and size in (-(-(8 + n_std * bpe) // 0x20) * 0x20, -(-(8 + n_short * bpe) // 0x20) * 0x20):
            size += 0x40
        adpc = bytearray(b"ADPC" + struct.pack(E + "i", size)) + _seek_table(E, chans, entries)
        adpc = bytearray(bytes(adpc).ljust(size, b"\0"))
    data_off = seek_off + len(adpc)
    audio_off = data_off + 0x20 + audio_skew
    data = bytearray(b"DATA" + struct.pack(E + "i", 0x18 + audio_skew + len(audio)) + b"\0" * (0x18 + audio_skew)) + audio
    data_size = len(data)
    struct.pack_into(E + "i", data, 4, data_size)
    stream = struct.pack(E + "BBBxHH", codec, int(looping), ch, rate & 0xFFFF, 0) + struct.pack(
        E + "11i", loop_start, n, audio_off, blocks_n, ilv, spi, last, n % spi if spi else 0, last, spe, 0)[:44]
    img = bytearray(0x40)
    img[head_off - 0x40: head_off - 0x40] = b""
    img += head
    struct.pack_into(E + "52s", img, head_off + 8 + stream_off, stream)
    struct.pack_into(E + "i", img, head_off + 4, len(head))
    img += adpc + data
    file_size = len(img) + file_size_delta
    struct.pack_into(E + "4sHBBihh6i", img, 0, magic or b"RSTM", 0xFEFF, 1, 0, file_size, 0x40, 3 if adpc else 2,
                     head_off, len(head), seek_off if adpc else 0, len(adpc), data_off, data_size)
    return np.frombuffer(bytes(img), dtype=np.uint8).copy()


def _bcfstm(kind, E, codec, chans, ch, n, rate, looping, loop_start, ilv, blocks_n, last, spi, spe, audio, v, seek, regions, tracks,
            n_info, magic, file_size_delta, audio_skew):
    major = v >> 24
    has_region = (major >= 2 and v >= 0x02010000) or major == 0
    has_unaligned = (major == 0 and v >= 0x00040000) or (major >= 2 and v >= 0x02030000)
    has_checksum = major == 0 and v >= 0x00050000
    info = bytearray(b"INFO\0\0\0\0")
    body = bytearray(24)
    stream_off = len(body)
    body += struct.pack(E + "BBBB", codec, int(looping), ch, regions)
    body += struct.pack(E + "11i", rate, loop_start, n, blocks_n, ilv, spi, last, n % spi if spi else 0, last, 4 * ch, spe)
    body += struct.pack(E + "hHi", 0x1F00, 0, 0x18 + audio_skew)        # audio reference: behind the DATA header
    if has_region:
        body += struct.pack(E + "hH", 0x100, 0) + struct.pack(E + "hHi", 0x0000, 0, 0x18)
    if has_unaligned:
        body += struct.pack(E + "ii", loop_start, n)
    if has_checksum:
        body += struct.pack(E + "I", 0x12345678)
    track_off = len(body)
    tbase = len(body)
    body += struct.pack(E + "i", tracks) + b"\0" * (8 * tracks)
    for t in range(tracks):
        struct.pack_into(E + "hHi", body, tbase + 4 + 8 * t, 0x4101, 0, len(body) - tbase)
        entry = len(body)
        body += struct.pack(E + "BBBB", 0x7F, 0x40, 0, 0) + b"\0" * 8
        struct.pack_into(E + "hHi", body, entry + 4, 0x0100, 0, len(body) - entry)
        body += struct.pack(E + "iBBxx", 2, 2 * t, 2 * t + 1)
    chan_off = len(body)
    cbase = len(body)
    body += struct.pack(E + "i", n_info) + b"\0" * (8 * n_info)
    for c in range(n_info):
        struct.pack_into(E + "hHi", body, cbase + 4 + 8 * c, 0x4102, 0, len(body) - cbase)
        entry = len(body)
        body += b"\0" * 8
        struct.pack_into(E + "hHi", body, entry, 0x0300, 0, len(body) - entry)
        k = chans[c] if c < len(chans) else Channel(b"")
        body += struct.pack(E + "16h", *[int(x) for x in k.coefs]) + struct.pack(E + "3h3hxx", *k.start, *k.loop)
    refs = ((0x4100, stream_off), (0x0101, track_off) if tracks else (0, 0), (0x0101, chan_off))
    for i, (t, off) in enumerate(refs):
        struct.pack_into(E + "hHi", body, 8 * i, t, 0, off)
    info += body
    _pad(info)
    struct.pack_into(E + "i", info, 4, len(info))
    blocks = [(0x4000, info)]
    if seek != "none":
        entries = -(-n // spe) if spe else 0
        seek_b = bytearray(b"SEEK\0\0\0\0") + _seek_table(E, chans, entries + (3 if seek == "unknown" else 0))
        _pad(seek_b)
        struct.pack_into(E + "i", seek_b, 4, len(seek_b))
        blocks.append((0x4001, seek_b))
    if regions:
        regn = bytearray(b"REGN\0\0\0\0") + b"\0" * 0x18
        for r in range(regions):
            entry = struct.pack(E + "ii", r * 100, r * 100 + 50) + b"".join(struct.pack(E + "hhh", r, c, -c) for c in range(ch))
            regn += entry.ljust(0x100, b"\0")
        _pad(regn)
        struct.pack_into(E + "i", regn, 4, len(regn))
        blocks.append((0x4003, regn))
    data = bytearray(b"DATA\0\0\0\0" + b"\0" * (0x18 + audio_skew)) + audio  # last block, unpadded: its size sets the region
    struct.pack_into(E + "i", data, 4, len(data))
    blocks.append((0x4002, data))
    header = bytearray(0x14 + 12 * len(blocks))
    _pad(header)
    off = len(header)
    out = bytearray(header)
    for i, (t, b) in enumerate(blocks):
        struct.pack_into(E + "hHii", out, 0x14 + 12 * i, t, 0, off, len(b))
        out += b
        off += len(b)
    mg = magic or (b"CSTM" if kind == BCSTM else b"FSTM")
    struct.pack_into(E + "4sHHIihH", out, 0, mg, 0xFEFF, 0x40, v, len(out) + file_size_delta, len(blocks), 0)
    out[0:4] = mg
    return np.frombuffer(bytes(out), dtype=np.uint8).copy()


def encoded(oracle, kind: int, codec: int, channels: int, n: int, loop: Optional[int] = None, seed: int = 0, big_endian=None,
            silent: Optional[tuple] = None, start_hist=(0, 0), **kw) -> np.ndarray:
    """A stream image of `channels` seeded channels of n samples in `codec`."""
    pcm = pcm_channels(channels, n, seed, silent)
    be = True if kind == BRSTM else bool(big_endian)
    if codec == GCADPCM:
        chans = gc_channels(oracle, pcm, loop or 0, start_hist)
    elif codec == PCM16:
        chans = pcm16_channels(pcm, be)
    else:
        chans = pcm8_channels(pcm)
    return build(kind, codec, chans, n, loop=loop, big_endian=big_endian, **kw)
