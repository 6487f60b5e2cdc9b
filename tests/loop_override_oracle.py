"""The batch's loop setting (VGAudioCli's -l <start>-<end> and --no-loop) restated: Convert.ConvertFile calls
AudioData.SetLoop on the audio it has just read, before any encode or write (Convert.cs:82-90, Formats/AudioData.cs:39-52),
and each format's WithLoop decides (AudioFormatBaseBuilder.cs:23-58, CriHcaFormatBuilder.cs:27-56).  set_loop is that
rule; the chains below put it between the existing oracle pieces: a source's reader restatement (what ToPcm16 yields),
then the target's writer restatement."""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np

import adx_reader_oracle as RA
import cri_rewrite_oracle as RW
import gc_container_writer_oracle as GW
import idsp_hps_reader_oracle as RI
import nw_wave_reader_oracle as RNW
import nw_writer_oracle as NW
import transcode_oracle as T
from oracle import pyoracle as O

KEEP, SET, CLEAR = 0, 1, 2                      # vgb_convert_options.loop_mode
PCM, GCADPCM, ADX, HCA = "pcm", "gcadpcm", "adx", "hca"
MSG_RANGE = "Loop points must be less than the number of samples and non-negative."
MSG_ORDER = "The loop end must be greater than the loop start"
MSG_HCA_CHANGE = "Changing the loop points on HCA audio without re-encoding is not supported."
MSG_HCA_ADD = "Adding a loop to HCA audio without re-encoding is not supported."

# the container types of the C ABI
DSP_T, ADX_T, HCA_T, BRSTM_T, BCSTM_T, BFSTM_T, IDSP_T, HPS_T = 1, 2, 3, 4, 5, 6, 7, 8
BRWAV_T, BCWAV_T, BFWAV_T, BCSTP_T, BFSTP_T = 9, 10, 11, 12, 13
NW_T = (BRSTM_T, BCSTM_T, BFSTM_T, BRWAV_T, BCWAV_T, BFWAV_T, BCSTP_T, BFSTP_T)


def set_loop(kind: str, sample_count: int, loop: Optional[Tuple[int, int]], mode: int, start: int = 0, end: int = 0,
             hca_points: Optional[Tuple[int, int]] = None):
    """(the loop afterwards or None, None) or (None, the reference's message).  kind: PCM (WAVE, PCM NintendoWare),
    GCADPCM (.dsp, NintendoWare, IDSP, HPS), ADX (points unaligned: ToPcm16 hands them on) or HCA; sample_count is the
    format builder's own count (channel 0's length, the unaligned count, or an HCA file's count as HcaReader cut it);
    hca_points is the HCA file's (LoopStartSample, LoopEndSample), defined whether or not it loops."""
    if mode == KEEP:
        return loop, None
    if mode == CLEAR:                                   # WithLoop(false): no loop, both points 0
        return None, None
    if start < 0 or start > sample_count or end < 0 or end > sample_count:
        return None, MSG_RANGE
    if end < start:
        return None, MSG_ORDER
    if kind == HCA:                                     # base checks first, then the two NotSupportedExceptions in order
        if (start, end) != tuple(hca_points):
            return None, MSG_HCA_CHANGE
        if loop is None:
            return None, MSG_HCA_ADD
    return (start, end), None


def adx_header_loop(loop: Optional[Tuple[int, int]], alignment_samples: int):
    """CriAdxFormat's LoopStart / LoopEnd: what a rewrite writes in the header (the unaligned points + AlignmentSamples)."""
    return None if loop is None else (loop[0] + alignment_samples, loop[1] + alignment_samples)


def hca_points(info) -> Tuple[int, int]:
    """HcaInfo.LoopStartSample / LoopEndSample (HcaInfo.cs:35-36) of an O.HcaInfo, in C#'s int arithmetic."""
    i32 = RA._i32
    return (i32(info.loop_start_frame * 1024 + info.pre_loop_samples - info.inserted_samples),
            i32((info.loop_end_frame + 1) * 1024 - info.post_loop_samples - info.inserted_samples))


def hca_target_refuses(loop) -> bool:
    """A difference on purpose: the .hca encoder refuses an empty loop (start == end), where CriHcaEncoder would write a
    file whose loop chunk ends a frame before it starts."""
    return loop is not None and loop[1] <= loop[0]


# ---- the sources: what ToPcm16 yields, and the kind whose WithLoop applies -----------------------------------------------
def source(img, in_type: int, adx_key=None, hca_key=None):
    """(pcm channels, sample count, loop, rate, kind, hca points) of one image, or None where the reader chain fails."""
    if in_type in (DSP_T, ADX_T, HCA_T):
        src = T.source_pcm(img, in_type, adx_key, hca_key)
        if src is None:
            return None
        pcm, n, loop, rate = src
        points = None
        if in_type == HCA_T:
            points = hca_points(RW.hca_parse(img)[1])
        return pcm, n, loop, rate, {DSP_T: GCADPCM, ADX_T: ADX, HCA_T: HCA}[in_type], points
    if in_type in NW_T:  # streams, wave files and prefetch streams: a PCM wave file's count is channel 0's row
        st, _, samples, _, h = RNW.plan(img, in_type)
        if st:
            return None
        st, pcm, loop = RNW.decoded_pcm(img, in_type)
        if st:
            return None
        return pcm, samples, loop, h.sample_rate, GCADPCM if h.codec == 2 else PCM, None
    st, pcm, loop = RI.decoded_pcm(img, in_type)
    if st:
        return None
    h = RI.parse(img, in_type)[1]
    return pcm, h.sample_count, loop, h.sample_rate, GCADPCM, None


def expected_wave(img, in_type: int, mode: int, start: int = 0, end: int = 0, adx_key=None, hca_key=None):
    """reader -> SetLoop -> ToPcm16 -> WaveWriter: (WAVE image, None), (None, message) or (None, None) where the reader
    chain itself fails."""
    src = source(img, in_type, adx_key, hca_key)
    if src is None:
        return None, None
    pcm, n, loop, rate, kind, points = src
    loop, msg = set_loop(kind, n, loop, mode, start, end, points)
    if msg:
        return None, msg
    return O.wave_write16(pcm, rate, loop), None


def expected_transcode(img, in_type: int, out_type: int, mode: int, start: int = 0, end: int = 0, adx_key=None, hca_key=None, **target):
    """transcode_oracle.source_pcm -> set_loop -> transcode_oracle.target_file."""
    src = source(img, in_type, adx_key, hca_key)
    if src is None:
        return None, None
    pcm, n, loop, rate, kind, points = src
    loop, msg = set_loop(kind, n, loop, mode, start, end, points)
    if msg:
        return None, msg
    if out_type == HCA_T and hca_target_refuses(loop):
        return None, -1
    return T.target_file(pcm, n, loop, rate, out_type, **target), None


# ---- WAVE sources into every target -------------------------------------------------------------------------------------
def expected_from_wave(pcm: List[np.ndarray], rate: int, loop, out_type: int, mode: int, start: int = 0, end: int = 0,
                       loop_align: int = 0):
    """A WAVE file of `pcm` with smpl loop `loop` through SetLoop into out_type (loop_align: the CLI's --loop-align):
    (file, None), (None, message) for a SetLoop refusal, or (None, status) for a writer refusal."""
    loop, msg = set_loop(PCM, len(pcm[0]), loop, mode, start, end)
    if msg:
        return None, msg
    n = len(pcm[0])
    if out_type == DSP_T:
        if loop_align <= 0:
            return T.target_file(pcm, n, loop, rate, DSP_T), None
        coefs = np.stack([O.calculate_coefficients(p) for p in pcm])
        adpcm = [O.encode(p, c) for p, c in zip(pcm, coefs)]
        ctx = None
        if loop:
            if len(pcm) == 1 and O.sample_count_to_byte_count(loop[1] + (-loop[0]) % loop_align) > O.sample_count_to_byte_count(n):
                return None, -1  # the aligned loop end lies past the mono audio (DspWriter's Stream.Write throws)
            ctx = np.stack([np.array(O.gc_loop_context(a, O.decode(a, c, n), loop[0]), dtype=np.int16) for a, c in zip(adpcm, coefs)])
        return O.dsp_write(adpcm, coefs, rate, n, loop, ctx, None, None, 0x3800, loop_align, True), None
    if out_type == HCA_T and hca_target_refuses(loop):
        return None, -1
    if out_type in (ADX_T, HCA_T):
        return T.target_file(pcm, n, loop, rate, out_type), None
    if out_type in (BRSTM_T, BCSTM_T, BFSTM_T):
        st, f = NW.write(out_type, NW.GCADPCM, pcm, rate, loop, 0, loop_align)
    elif out_type == IDSP_T:
        st, f = GW.write_idsp(pcm, rate, loop)
    else:
        st, f = GW.write_hps(pcm, rate, loop)
    return (f, None) if st == 0 else (None, st)


# ---- rewrites -------------------------------------------------------------------------------------------------------------
def expected_adx_rewrite(image, mode: int, start: int = 0, end: int = 0, no_trim: bool = False, in_key=None):
    """cri_rewrite_oracle.expected_adx with SetLoop on the reader's CriAdxFormat: the new unaligned points go to the
    writer, which writes them plus AlignmentSamples and trims a looping file at the new loop end."""
    st, h = RA.adx_parse(image)
    if st != 0:
        return None, None
    rows = RA.audio_rows(image, h)
    if h.revision in (8, 9):
        if in_key is None:
            return None, None
        rows = O.adx_crypt(rows, in_key, h.revision, h.frame_size)
    samples = RA._i32(h.sample_count - h.inserted_samples)
    loop = None
    if h.looping:
        loop = (RA._i32(h.loop_start_sample - h.inserted_samples), RA._i32(h.loop_end_sample - h.inserted_samples))
        if not (0 <= loop[0] <= samples and 0 <= loop[1] <= samples and loop[0] <= loop[1]):
            return None, None
    loop, msg = set_loop(ADX, samples, loop, mode, start, end)
    if msg:
        return None, msg
    if samples < 0 or h.inserted_samples < 0:
        return None, None
    history = [hh[0] for hh in h.history] if h.history else [0] * h.channel_count
    return O.adx_write(rows, history, h.sample_rate, samples, loop, h.inserted_samples, h.frame_size, h.version, h.type,
                       h.highpass_frequency, 0, None, not no_trim), None


def expected_hca_rewrite(image, mode: int, start: int = 0, end: int = 0):
    """cri_rewrite_oracle.expected_hca with SetLoop on the reader's CriHcaFormat: --no-loop drops the loop chunk (the
    frames and the header size stay), -l passes only with the file's own points."""
    st, info, ciph, comment, rva = RW.hca_parse(image)
    if st != 0:
        return None, None
    loop = hca_points(info) if info.looping else None
    loop, msg = set_loop(HCA, info.sample_count, loop, mode, start, end, hca_points(info))
    if msg:
        return None, msg
    if loop is not None or not info.looping:
        return RW.expected_hca(image), None
    # rebuild the header without the loop chunk, the source's frames as they are ("ciph" 0 sources, no keys)
    assert ciph == 0
    info.looping = 0
    chunks = RW.hca_chunks(info, False, ciph, comment, rva)
    img = np.ascontiguousarray(image, np.uint8)
    total = info.header_size + info.frame_size * info.frame_count
    out = np.zeros(total, np.uint8)
    out[:len(chunks)] = np.frombuffer(chunks, np.uint8)
    crc = O.crc16(out[:info.header_size - 2].tobytes())
    out[info.header_size - 2: info.header_size] = (crc >> 8, crc & 0xFF)
    out[info.header_size:] = img[info.header_size: total]
    return out, None
