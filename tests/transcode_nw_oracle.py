"""The oracle chain of a transcode into a NintendoWare stream, IDSP or HPS file (Convert.ConvertFile with a .dsp, .adx
or .hca source and a BRSTM / BCSTM / BFSTM / IDSP / HPS writer): the source's reader restatement and the oracle's
decoder give what ToPcm16 yields (transcode_oracle.source_pcm, through loop_override_oracle.source for the loop kind),
AudioData.SetLoop applies -l / --no-loop (loop_override_oracle.set_loop), then the target's writer restatement
(nw_writer_oracle.write, gc_container_writer_oracle.write_idsp / write_hps) configured from the options alone gives the
file.  A .dsp source into GC-ADPCM is a rewrite in its own codec (GetFormat<GcAdpcmFormat> hands back the source's
format), which is not performed."""
from __future__ import annotations

import gc_container_writer_oracle as GW
import loop_override_oracle as LO
import nw_writer_oracle as NW

DSP, ADX, HCA = 1, 2, 3
BRSTM, BCSTM, BFSTM, IDSP, HPS = 4, 5, 6, 7, 8
NW_TARGETS = (BRSTM, BCSTM, BFSTM)
TARGETS = (BRSTM, BCSTM, BFSTM, IDSP, HPS)
PCM8, PCM16, GCADPCM = NW.PCM8, NW.PCM16, NW.GCADPCM
E_DATA, E_ARG = NW.E_DATA, NW.E_ARG
MSG_REWRITE = "the source is already in the target's codec; rewriting a container in its own codec is not performed"


def codec_plus1(codec: int) -> int:
    """vgb_convert_options.nw_codec_plus1 of a codec (GC-ADPCM is also the default, 0)."""
    return codec + 1


def is_rewrite(in_type: int, out_type: int, codec: int = GCADPCM) -> bool:
    return in_type == DSP and (out_type in (IDSP, HPS) or codec == GCADPCM)


def planned(img, in_type: int, out_type: int, codec: int = GCADPCM, mode: int = LO.KEEP, start: int = 0, end: int = 0,
            adx_key=None, hca_key=None):
    """(pcm, sample count, loop after SetLoop, rate) of one source, or (None, message) where SetLoop refuses it, or
    (None, None) where the reader chain fails, or (None, MSG_REWRITE)."""
    if is_rewrite(in_type, out_type, codec):
        return None, MSG_REWRITE
    src = LO.source(img, in_type, adx_key, hca_key)
    if src is None:
        return None, None
    pcm, n, loop, rate, kind, points = src
    loop, msg = LO.set_loop(kind, n, loop, mode, start, end, points)
    if msg:
        return None, msg
    return (pcm, n, loop, rate), None


def target_check(ch: int, n: int, loop, out_type: int, codec: int = GCADPCM, alignment: int = 0, trim: bool = True) -> int:
    """The target writer's per-file refusal for this PCM (0: none)."""
    if out_type in NW_TARGETS:
        return NW.check(out_type, codec, ch, n, loop, alignment)
    if out_type == IDSP:
        return GW.idsp_check(ch, n, loop, trim)
    return GW.hps_check(ch, n, loop)


def target_size(ch: int, n: int, loop, out_type: int, codec: int = GCADPCM, alignment: int = 0, trim: bool = True) -> int:
    """The target file's size from the geometry alone (the file must pass target_check)."""
    if out_type in NW_TARGETS:
        return NW.file_size(out_type, codec, ch, n, loop, alignment)
    if out_type == IDSP:
        return GW.idsp_geometry(ch, n, loop, trim)[1]["file_size"]
    return GW.hps_geometry(ch, n, loop)[1]["file_size"]


def target_file(pcm, n, loop, rate, out_type: int, codec: int = GCADPCM, endianness: int = 0, alignment: int = 0, trim: bool = True):
    """(status, file) of the target writer."""
    if out_type in NW_TARGETS:
        return NW.write(out_type, codec, pcm, rate, loop, endianness, alignment)
    if out_type == IDSP:
        return GW.write_idsp(pcm, rate, loop, trim)
    return GW.write_hps(pcm, rate, loop)


def expected_size(img, in_type: int, out_type: int, codec: int = GCADPCM, alignment: int = 0, trim: bool = True, mode: int = LO.KEEP,
                  start: int = 0, end: int = 0, adx_key=None, hca_key=None):
    """(size, None) or (None, message / writer status / None where the reader fails) of the sizing pass."""
    p, why = planned(img, in_type, out_type, codec, mode, start, end, adx_key, hca_key)
    if p is None:
        return None, why
    pcm, n, loop, rate = p
    st = target_check(len(pcm), n, loop, out_type, codec, alignment, trim)
    if st:
        return None, st
    return target_size(len(pcm), n, loop, out_type, codec, alignment, trim), None


def expected(img, in_type: int, out_type: int, codec: int = GCADPCM, endianness: int = 0, alignment: int = 0, trim: bool = True,
             mode: int = LO.KEEP, start: int = 0, end: int = 0, adx_key=None, hca_key=None):
    """The whole chain for one file: (file, None), or (None, message / writer status / None where the reader fails)."""
    p, why = planned(img, in_type, out_type, codec, mode, start, end, adx_key, hca_key)
    if p is None:
        return None, why
    pcm, n, loop, rate = p
    st, f = target_file(pcm, n, loop, rate, out_type, codec, endianness, alignment, trim)
    return (f, None) if st == 0 else (None, st)


def options(ct, out_type: int, codec: int = GCADPCM, endianness: int = 0, alignment: int = 0, trim: bool = True, **kw):
    """The vgb_convert_options of a target configuration (kw: loop=, no_loop=, group_bytes= ...)."""
    return ct.convert_options(out_type, nw_codec_plus1=codec_plus1(codec), nw_endianness=endianness, nw_loop_point_alignment=alignment,
                              no_trim=0 if trim else 1, **kw)
