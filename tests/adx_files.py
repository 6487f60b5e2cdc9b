"""Builders of .adx test images on the oracle: encoded files of every type, version and frame size (with the alignment
padding of looping files and both key kinds), and hand-assembled headers."""
from __future__ import annotations

import struct

import numpy as np

from vgaudio_b200 import synth

KEY_CODE = 0x0123456789ABCDEF
KEY_STRING = "vgaudio-b200"


def alignment(loop_start: int, channels: int, frame_size: int) -> int:
    """CriAdxFormat.EncodeFromPcm16's alignment samples (CriAdxFormat.cs:61-63)."""
    spf = (frame_size - 2) * 2
    mult = spf * 2 if channels == 1 else spf
    return -(-loop_start // mult) * mult - loop_start


def encoded(oracle, channels, n, rate=48000, frame_size=18, version=4, type=3, loop=None, key=None, enc_type=0, seed=0,
            filter=2, pcm=None):
    """An .adx image the way the reference's encoder and AdxWriter make it."""
    align = alignment(loop[0], channels, frame_size) if loop else 0
    if pcm is None:
        pcm = [synth.channel(seed + c, n, rate, degenerate=False) for c in range(channels)]
    enc = [oracle.adx_encode(p, rate, frame_size, version, align, type, filter) for p in pcm]
    return oracle.adx_write([e[0] for e in enc], [e[1] for e in enc], rate, n, loop, align, frame_size, version, type, 500,
                            enc_type, key)


def header(channels=2, rate=48000, samples=100, frame_size=18, version=4, type=3, revision=0, highpass=500, header_size=None,
           inserted=None, loop_count=None, loop=(0, 0, 0, 0, 0), history=None, audio=None, tail=b""):
    """A hand-assembled image: fields in AdxReader's order, then zero audio (or `audio`) behind header_size + 4."""
    h = struct.pack(">HhBBBBiihBB", 0x8000, 0, type, frame_size, 4, channels, rate, samples, highpass, version, revision)
    if version >= 4:
        h += b"\0" * 4
        for c in range(channels):
            a, b = history[c] if history else (c, -c)
            h += struct.pack(">hh", a, b)
        if channels == 1:
            h += b"\0" * 4
    if inserted is not None:
        h += struct.pack(">hh", inserted, loop_count or 0)
        if loop_count and loop_count > 0:
            h += struct.pack(">iiiii", *loop)
    if header_size is None:
        header_size = max(len(h) - 4, 32)
    h = bytearray(h.ljust(header_size + 4, b"\0"))
    h[2:4] = struct.pack(">h", header_size)
    if audio is None:
        spf = (frame_size - 2) * 2
        audio = bytes(-(-samples // spf) * frame_size * channels) if spf > 0 and samples > 0 else b""
    head = bytes(h[: max(header_size + 4, 20)])  # a negative header size still leaves the fixed fields in the image
    return np.frombuffer(head + bytes(audio) + tail, dtype=np.uint8).copy()
