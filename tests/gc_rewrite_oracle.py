"""The oracle chain of a .dsp file rewritten into a BRSTM / BCSTM / BFSTM / IDSP / HPS file without re-encoding
(Convert.ConvertFile with a .dsp source and a GC-ADPCM writer: DspReader, AudioData.SetLoop for -l / --no-loop, then
GetFormat<GcAdpcmFormat> hands the writer the source's own channels, which GcAdpcmChannelBuilder rebuilds).  It composes
the existing restatements: the .dsp reader and SetLoop (loop_override_oracle.source / set_loop), the C oracle's
decode, loop context, seek table and GcAdpcmAlignment, and the writers (nw_writer_oracle.write,
gc_container_writer_oracle.write_idsp / write_hps) fed the source's ADPCM and coefficients instead of an encode.

The builder's reuse rules (GcAdpcmChannelBuilder.cs:118-202) as the rebuilds chain them for a .dsp source:
- DspReader builds each channel with the header's loop context at the header's loop start (the start address, also when
  the file does not loop).  Every rebuild after it (the format's, SetLoop's, WithAlignment's, which leaves
  AlignedLoopStart at the UNALIGNED loop start) keeps a context taken at its own loop start and decodes one otherwise,
  from history 0.  So the header's context reaches the writer (`keep`) iff the loop start the reader built with and the
  one the writer sees are both the header's.
- NintendoWare (RecalculateLoopContext) and HPS (EnsureLoopContextIsSelfCalculated) never take a context they did not
  calculate: theirs is the decode's at the unaligned loop start.  The NintendoWare seek table comes from the same
  decode (EnsurePcmDecoded: the unaligned ADPCM, history 0).  IDSP writes the header's context when `keep` holds.
- GcAdpcmChannel keeps the header's gain and start history; its start predictor/scale is Adpcm[0].
- HpsWriter reads each block's history from the channel's Pcm.  With `keep` no rebuild ever decoded, and when the loop
  moved the channel keeps that unset Pcm: every block's history is 0 and nothing is read past the decode.

A frame header with a predictor outside 0..7 in the decoded frames fails the file (MSG_PREDICTOR)."""
from __future__ import annotations

import contextlib
import struct
from typing import List, Optional

import numpy as np

import gc_container_writer_oracle as GW
import loop_override_oracle as LO
import nw_writer_oracle as NW
import transcode_nw_oracle as TN
from oracle import pyoracle as O

DSP = TN.DSP
BRSTM, BCSTM, BFSTM, IDSP, HPS = TN.BRSTM, TN.BCSTM, TN.BFSTM, TN.IDSP, TN.HPS
TARGETS = TN.TARGETS
E_DATA, E_ARG = TN.E_DATA, TN.E_ARG
MSG_PREDICTOR = "a frame header selects a predictor outside 0..7"
MSG_IN_TYPE = "only .dsp sources are rewritten"


class Source:
    """One .dsp file as DspReader and SetLoop leave it."""

    def __init__(self, info, rows, loop, rate):
        self.n = info.sample_count
        self.rate = rate
        self.loop = loop
        ch = info.channel_count
        self.adpcm = [np.asarray(r, dtype=np.uint8) for r in rows]
        self.coefs = [np.array(info.coefs[c][:], dtype=np.int16) for c in range(ch)]
        self.gain = [int(info.gain[c]) for c in range(ch)]
        self.start_hist = [(int(info.start_ctx[c][1]), int(info.start_ctx[c][2])) for c in range(ch)]
        self.header_ctx = [tuple(int(v) for v in info.loop_ctx[c][:]) for c in range(ch)]
        read_ls = info.loop_start if info.looping else 0
        ls = loop[0] if loop else 0
        self.keep = read_ls == info.loop_start and ls == info.loop_start
        # history 0; not for frames the decoder refuses (the C oracle would index past the coefficients)
        self.decoded = None if self.bad_predictor() else [O.decode(a, co, self.n) for a, co in zip(self.adpcm, self.coefs)]

    @property
    def channels(self) -> int:
        return len(self.adpcm)

    def bad_predictor(self) -> bool:
        frames = -(-self.n // 14)
        return any(int(a[f * 8]) >> 4 >= 8 for a in self.adpcm for f in range(frames))

    def decoded_ctx(self, c: int, loop_start: int):
        return tuple(int(v) for v in O.gc_loop_context(self.adpcm[c], self.decoded[c], loop_start))


def read(img, mode: int = LO.KEEP, start: int = 0, end: int = 0):
    """(Source, None), or (None, SetLoop's message), or (None, None) where the reader fails."""
    src = LO.source(img, LO.DSP_T)
    if src is None:
        return None, None
    _, n, loop, rate, kind, points = src
    loop, msg = LO.set_loop(kind, n, loop, mode, start, end, points)
    if msg:
        return None, msg
    st, info = O.dsp_parse(img)
    return Source(info, O.dsp_read_data(img, info), loop, rate), None


def _hps_no_hist(s: Source) -> bool:
    st, g = GW.hps_geometry(s.channels, s.n, s.loop)
    return s.keep and st == 0 and g["needed"]


def _hps_n(s: Source) -> int:
    """The length the HPS restatement checks the block histories against: past every block when they are not read."""
    if not _hps_no_hist(s):
        return s.n
    return max([s.n] + [b["start"] + 1 for b in GW.hps_geometry(s.channels, s.n, s.loop)[1]["blocks"]])


def check(s: Source, out_type: int, alignment: int = 0, trim: bool = True) -> int:
    if out_type == HPS:
        return GW.hps_check(s.channels, _hps_n(s), s.loop)
    return TN.target_check(s.channels, s.n, s.loop, out_type, TN.GCADPCM, alignment, trim)


def expected_size(img, out_type: int, alignment: int = 0, trim: bool = True, mode: int = LO.KEEP, start: int = 0, end: int = 0):
    """(size, None) or (None, message / writer status / None where the reader fails) of the sizing pass."""
    s, why = read(img, mode, start, end)
    if s is None:
        return None, why
    st = check(s, out_type, alignment, trim)
    if st:
        return None, st
    return TN.target_size(s.channels, s.n, s.loop, out_type, TN.GCADPCM, alignment, trim), None


@contextlib.contextmanager
def _patched(module, name, value):
    old = getattr(module, name)
    setattr(module, name, value)
    try:
        yield
    finally:
        setattr(module, name, old)


class _SourceCodec:
    """The C oracle with CalculateCoefficients / Encode / Decode handing back the source's channels: channel c is named
    by the placeholder row tokens[c] the writer restatement is given instead of its PCM."""

    def __init__(self, s: Source, tokens: List[np.ndarray], hist: bool):
        self._c = {id(t): c for c, t in enumerate(tokens)}
        self._a = {id(a): c for c, a in enumerate(s.adpcm)}
        self._s = s
        self._hist = hist
        self._len = len(tokens[0])

    def __getattr__(self, name):
        return getattr(O, name)

    def calculate_coefficients(self, p):
        return self._s.coefs[self._c[id(p)]]

    def encode(self, p, coefs):
        return self._s.adpcm[self._c[id(p)]]

    def decode(self, adpcm, coefs, n, h1=0, h2=0):
        return self._s.decoded[self._a[id(adpcm)]] if self._hist else np.zeros(self._len, np.int16)


def _nw_file(s: Source, out_type: int, endianness: int, alignment: int):
    def channels(pcm, loop_start, spe):
        out = []
        for c in range(s.channels):
            start = (int(s.adpcm[c][0]),) + s.start_hist[c]
            lc = s.decoded_ctx(c, loop_start) if loop_start is not None else start
            out.append((s.adpcm[c], s.coefs[c], start, lc, np.asarray(O.gc_seek_table(s.decoded[c], spe), dtype=np.int16)))
        return out

    tokens = [np.zeros(s.n, np.int16) for _ in range(s.channels)]
    with _patched(NW, "_gc_channels", channels):
        st, f = NW.write(out_type, NW.GCADPCM, tokens, s.rate, s.loop, endianness, alignment)
    if st == 0 and out_type == BRSTM:  # BrstmWriter writes channel.Gain in front of the start context
        ch = s.channels
        g = NW.geometry(out_type, NW.GCADPCM, ch, s.n, NW.aligned_loop(NW.GCADPCM, s.loop, alignment)[1])
        base = 24 + 0x34 + g["h2"] + 4
        for c in range(ch):
            struct.pack_into(">h", f, 0x48 + base + 8 * ch + 0x38 * c + 8 + 32, s.gain[c])
    return st, f


def _gc_file(s: Source, out_type: int, trim: bool):
    idsp = out_type == IDSP
    hist = idsp or not _hps_no_hist(s)
    tokens = [np.zeros(s.n if idsp else _hps_n(s), np.int16) for _ in range(s.channels)]
    with _patched(GW, "O", _SourceCodec(s, tokens, hist)):
        st, f = GW.write_idsp(tokens, s.rate, s.loop, trim) if idsp else GW.write_hps(tokens, s.rate, s.loop)
    if st:
        return st, None
    info0, stride = (0x40 + 0x3c, 0x60) if idsp else (0x10 + 0x30, 0x38)
    for c in range(s.channels):
        at = info0 + stride * c
        struct.pack_into(">h", f, at, s.gain[c])
        struct.pack_into(">2h", f, at + 4, *s.start_hist[c])
        if idsp:
            ctx = s.header_ctx[c] if s.keep else s.decoded_ctx(c, s.loop[0] if s.loop else 0)
            struct.pack_into(">3h", f, at + 8, *ctx)
    return 0, f


def expected(img, out_type: int, endianness: int = 0, alignment: int = 0, trim: bool = True, mode: int = LO.KEEP, start: int = 0,
             end: int = 0):
    """The whole chain for one file: (file, None), or (None, message / writer status / None where the reader fails)."""
    s, why = read(img, mode, start, end)
    if s is None:
        return None, why
    st = check(s, out_type, alignment, trim)
    if st:
        return None, st
    if s.bad_predictor():
        return None, MSG_PREDICTOR
    st, f = _nw_file(s, out_type, endianness, alignment) if out_type in TN.NW_TARGETS else _gc_file(s, out_type, trim)
    return (f, None) if st == 0 else (None, st)


def dsp_image(ch: int, n: int, rate: int, loop=None, seed: int = 0, gain=None, loop_ctx=None, pcm=None):
    """A .dsp image the way the reference's encoder and DspWriter make it, with a start history and gain in the header;
    loop_ctx (one (ps, h1, h2) per channel) replaces the header's loop context, right or wrong."""
    from vgaudio_b200 import synth

    if pcm is None:
        pcm = [synth.channel(seed + c, max(n, 1), rate, degenerate=False)[:n] for c in range(ch)]
    coefs = np.stack([O.calculate_coefficients(p) for p in pcm])
    adpcm = [O.encode(p, co) for p, co in zip(pcm, coefs)]
    ctx = loop_ctx
    if loop and ctx is None:
        ctx = [O.gc_loop_context(a, O.decode(a, co, n), loop[0]) for a, co in zip(adpcm, coefs)]
    ctx = np.array(ctx, dtype=np.int16).reshape(ch, 3) if ctx is not None else None
    hist = np.array([[3 * c + seed % 7 + 1, -c - 2] for c in range(ch)], dtype=np.int16)
    g = np.array(gain if gain is not None else [100 * c - 7 for c in range(ch)], dtype=np.int16)
    return O.dsp_write(adpcm, coefs, rate, n, loop, ctx, g, hist)


def options(ct, out_type: int, endianness: int = 0, alignment: int = 0, trim: bool = True, **kw):
    """The vgb_convert_options of a rewrite target (kw: loop=, no_loop=, group_bytes= ...)."""
    return ct.convert_options(out_type, nw_endianness=endianness, nw_loop_point_alignment=alignment, no_trim=0 if trim else 1, **kw)
