"""The oracle chain of a transcode from a NintendoWare stream, wave or prefetch file, IDSP or HPS file into any coded
target (Convert.ConvertFile with a BRSTM / BCSTM / BFSTM / BRWAV / BCWAV / BFWAV / BCSTP / BFSTP / IDSP / HPS source):
the source's reader restatement gives what ToPcm16 yields (loop_override_oracle.source), AudioData.SetLoop applies -l /
--no-loop (loop_override_oracle.set_loop), then the target's writer restatement configured from the options alone gives
the file (transcode_oracle for .dsp / .adx / .hca, transcode_nw_oracle for the NintendoWare streams, IDSP and HPS).

AudioData.GetFormat<T> hands a source in the target's codec its own format back: a rewrite, which is not performed.  An
IDSP or HPS source is refused for a GC-ADPCM target before it is read (the container fixes its codec); a NintendoWare
source only once its header is parsed and SetLoop has run."""
from __future__ import annotations

import loop_override_oracle as LO
import nw_wave_reader_oracle as RNW
import transcode_nw_oracle as W
import transcode_oracle as T

DSP, ADX, HCA = 1, 2, 3
BRSTM, BCSTM, BFSTM, IDSP, HPS = 4, 5, 6, 7, 8
BRWAV, BCWAV, BFWAV, BCSTP, BFSTP = 9, 10, 11, 12, 13
NW_SOURCES = (BRSTM, BCSTM, BFSTM, BRWAV, BCWAV, BFWAV, BCSTP, BFSTP)
SOURCES = NW_SOURCES + (IDSP, HPS)
TARGETS = (DSP, ADX, HCA, BRSTM, BCSTM, BFSTM, IDSP, HPS)
NW_TARGETS = W.NW_TARGETS
PCM8, PCM16, GCADPCM = W.PCM8, W.PCM16, W.GCADPCM
CODEC_ADX, CODEC_HCA = 3, 4                     # past the NintendoWare codec numbers
MSG_REWRITE = W.MSG_REWRITE
MSG_IN_TYPE = "is not BRSTM, BCSTM, BFSTM, BRWAV, BCWAV, BFWAV, BCSTP, BFSTP, IDSP or HPS"


def target_codec(out_type: int, codec: int = GCADPCM) -> int:
    """The format type GetFormat<T> asks for: `codec` (the -f option) for a NintendoWare stream, GC-ADPCM for .dsp, IDSP
    and HPS."""
    if out_type == ADX:
        return CODEC_ADX
    if out_type == HCA:
        return CODEC_HCA
    return codec if out_type in NW_TARGETS else GCADPCM


def source_codec(img, in_type: int):
    """The source's format type: GC-ADPCM for IDSP / HPS, the header's codec for NintendoWare (None: unreadable)."""
    if in_type in (IDSP, HPS):
        return GCADPCM
    st, _, _, _, h = RNW.plan(img, in_type)
    return None if st else h.codec


def planned(img, in_type: int, out_type: int, codec: int = GCADPCM, mode: int = LO.KEEP, start: int = 0, end: int = 0):
    """(pcm, sample count, loop after SetLoop, rate) of one source, or (None, MSG_REWRITE), (None, a SetLoop message), or
    (None, None) where the reader chain fails; in the product's order."""
    if in_type in (IDSP, HPS) and target_codec(out_type, codec) == GCADPCM:
        return None, MSG_REWRITE
    src = LO.source(img, in_type)
    if src is None:
        return None, None
    pcm, n, loop, rate, kind, points = src
    loop, msg = LO.set_loop(kind, n, loop, mode, start, end, points)
    if msg:
        return None, msg
    if in_type in NW_SOURCES and source_codec(img, in_type) == target_codec(out_type, codec):
        return None, MSG_REWRITE
    return (pcm, n, loop, rate), None


def is_rewrite(img, in_type: int, out_type: int, codec: int = GCADPCM) -> bool:
    return source_codec(img, in_type) == target_codec(out_type, codec)


def expected_size(img, in_type: int, out_type: int, codec: int = GCADPCM, alignment: int = 0, trim: bool = True, mode: int = LO.KEEP,
                  start: int = 0, end: int = 0):
    """(size, None) or (None, message / writer status / None where the reader fails) of the sizing pass."""
    p, why = planned(img, in_type, out_type, codec, mode, start, end)
    if p is None:
        return None, why
    pcm, n, loop, rate = p
    if out_type in (DSP, ADX, HCA):
        if out_type == HCA and LO.hca_target_refuses(loop):
            return None, -1
        return T.target_size(len(pcm), n, loop, rate, out_type), None
    st = W.target_check(len(pcm), n, loop, out_type, codec, alignment, trim)
    if st:
        return None, st
    return W.target_size(len(pcm), n, loop, out_type, codec, alignment, trim), None


def expected(img, in_type: int, out_type: int, codec: int = GCADPCM, endianness: int = 0, alignment: int = 0, trim: bool = True,
             mode: int = LO.KEEP, start: int = 0, end: int = 0):
    """The whole chain for one file: (file, None), or (None, message / writer status / None where the reader fails)."""
    p, why = planned(img, in_type, out_type, codec, mode, start, end)
    if p is None:
        return None, why
    pcm, n, loop, rate = p
    if out_type in (DSP, ADX, HCA):
        if out_type == HCA and LO.hca_target_refuses(loop):
            return None, -1
        return T.target_file(pcm, n, loop, rate, out_type), None
    st, f = W.target_file(pcm, n, loop, rate, out_type, codec, endianness, alignment, trim)
    return (f, None) if st == 0 else (None, st)


def options(ct, out_type: int, codec: int = GCADPCM, endianness: int = 0, alignment: int = 0, trim: bool = True, **kw):
    """The vgb_convert_options of a target configuration (HCA quality High, the oracle's; kw: loop=, no_loop=,
    group_bytes= ...)."""
    return W.options(ct, out_type, codec, endianness, alignment, trim, hca_quality=2, **kw)


# ---- stimuli ------------------------------------------------------------------------------------------------------------
def _gc_rows(pcm, seed: int):
    """(adpcm row, coefs, start context) per channel, with a start history, for the IDSP and HPS builders."""
    import idsp_hps_reader_oracle as RI

    return [RI.encoded(p, (seed * 31 % 500, -seed * 7 % 300)) for p in pcm]


def idsp(channels: int, n: int, seed: int, loop=None):
    import idsp_hps_reader_oracle as RI
    import nw_files as NF

    return RI.idsp_image(32000, _gc_rows(NF.pcm_channels(channels, n, seed), seed), n, loop=loop)


def hps(channels: int, n: int, seed: int):
    """An HPS chain of three blocks of whole frames."""
    import idsp_hps_reader_oracle as RI
    import nw_files as NF

    frames = -(-n // 14)
    pieces = [8 * (frames // 3), 8 * (frames // 3), 8 * (frames - 2 * (frames // 3))]
    return RI.hps_chain(32000, _gc_rows(NF.pcm_channels(channels, n, seed), seed), pieces, n_samples=n)


def sources(oracle, scale: int = 1):
    """(in_type, image, note) of every reader in every codec it holds, both byte orders, looping and not; sample counts
    that are no multiple of 14 or 1024 (scale multiplies the stream lengths)."""
    import nw_files as NF
    import nw_wave_files as NWF

    s = scale
    out = [(BRSTM, NF.encoded(oracle, NF.BRSTM, GCADPCM, 2, 3001 * s, loop=500, seed=1), "brstm gc-adpcm loop"),
           (BRSTM, NF.encoded(oracle, NF.BRSTM, PCM16, 1, 2503 * s, seed=2), "brstm pcm16"),
           (BRSTM, NF.encoded(oracle, NF.BRSTM, PCM8, 2, 2011 * s, loop=101, seed=3), "brstm pcm8 loop"),
           (BCSTM, NF.encoded(oracle, NF.BCSTM, GCADPCM, 1, 3003 * s, seed=4), "bcstm gc-adpcm"),
           (BCSTM, NF.encoded(oracle, NF.BCSTM, PCM16, 2, 2501 * s, loop=333, seed=5, big_endian=True), "bcstm pcm16 be loop"),
           (BCSTM, NF.encoded(oracle, NF.BCSTM, PCM8, 1, 1999 * s, seed=6), "bcstm pcm8"),
           (BFSTM, NF.encoded(oracle, NF.BFSTM, GCADPCM, 2, 4001 * s, loop=1001, seed=7), "bfstm gc-adpcm loop"),
           (BFSTM, NF.encoded(oracle, NF.BFSTM, PCM16, 1, 2207 * s, seed=8, big_endian=False), "bfstm pcm16 le"),
           (BFSTM, NF.encoded(oracle, NF.BFSTM, PCM8, 2, 2305 * s, seed=9), "bfstm pcm8"),
           (BRWAV, NWF.encoded(oracle, NWF.BRWAV, GCADPCM, 2, 3001 * s, loop=300, seed=10), "brwav gc-adpcm loop"),
           (BRWAV, NWF.encoded(oracle, NWF.BRWAV, PCM16, 1, 2500 * s, seed=11), "brwav pcm16"),
           (BCWAV, NWF.encoded(oracle, NWF.BCWAV, PCM8, 1, 2003 * s, seed=12), "bcwav pcm8"),
           (BCWAV, NWF.encoded(oracle, NWF.BCWAV, GCADPCM, 2, 3007 * s, loop=700, seed=13), "bcwav gc-adpcm loop"),
           (BFWAV, NWF.encoded(oracle, NWF.BFWAV, PCM16, 2, 2509 * s, loop=9, seed=14), "bfwav pcm16 loop"),
           (BFWAV, NWF.encoded(oracle, NWF.BFWAV, GCADPCM, 1, 2999 * s, seed=15), "bfwav gc-adpcm"),
           (BCSTP, NWF.encoded(oracle, NWF.BCSTP, GCADPCM, 1, 3001 * s, loop=200, seed=16), "bcstp gc-adpcm loop"),
           (BCSTP, NWF.encoded(oracle, NWF.BCSTP, PCM8, 2, 1801 * s, seed=17), "bcstp pcm8"),
           (BFSTP, NWF.encoded(oracle, NWF.BFSTP, PCM16, 2, 2001 * s, seed=18), "bfstp pcm16"),
           (IDSP, idsp(2, 3001 * s, 19, loop=(100, 2000 * s)), "idsp loop"),
           (IDSP, idsp(1, 2777 * s, 20), "idsp"),
           (HPS, hps(2, 5003 * s, 21), "hps"),
           (HPS, hps(2, 4097, 22), "hps short")]
    for in_type, img, note in out:  # every stimulus is readable, so every case reaches SetLoop
        assert LO.source(img, in_type) is not None, note
    return out
