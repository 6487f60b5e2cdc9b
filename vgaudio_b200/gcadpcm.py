"""Host-side mirror of VGAudio.Codecs.GcAdpcm over the C ABI (no arithmetic here).

Reference interface (paths under VGAudio's src/VGAudio/):
  GcAdpcmMath                          Codecs/GcAdpcm/GcAdpcmMath.cs:7-47
  GcAdpcmCoefficients.CalculateCoefficients(short[])            GcAdpcmCoefficients.cs:9
  GcAdpcmEncoder.Encode(short[], short[], GcAdpcmParameters)     GcAdpcmEncoder.cs:14
  GcAdpcmEncoder.DspEncodeFrame(short[], int, byte[], short[])   GcAdpcmEncoder.cs:48
  GcAdpcmDecoder.Decode(byte[], short[], GcAdpcmParameters)      GcAdpcmDecoder.cs:10
The *_batch functions are what one Parallel.For over channels (Formats/GcAdpcm/GcAdpcmFormat.cs:45,65) becomes.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Callable, Optional, Sequence

import numpy as np

from . import _native as N

BYTES_PER_FRAME = 8
SAMPLES_PER_FRAME = 14
NIBBLES_PER_FRAME = 16


# ---- GcAdpcmMath -----------------------------------------------------------------------------------------
def nibble_count_to_sample_count(n: int) -> int:
    return N.lib.vgb_gcadpcm_nibble_count_to_sample_count(n)


def sample_count_to_nibble_count(n: int) -> int:
    return N.lib.vgb_gcadpcm_sample_count_to_nibble_count(n)


def nibble_to_sample(n: int) -> int:
    return N.lib.vgb_gcadpcm_nibble_to_sample(n)


def sample_to_nibble(n: int) -> int:
    return N.lib.vgb_gcadpcm_sample_to_nibble(n)


def sample_count_to_byte_count(n: int) -> int:
    return N.lib.vgb_gcadpcm_sample_count_to_byte_count(n)


def byte_count_to_sample_count(n: int) -> int:
    return N.lib.vgb_gcadpcm_byte_count_to_sample_count(n)


@dataclass
class GcAdpcmParameters:
    """GcAdpcmParameters : CodecParameters (GcAdpcmParameters.cs:3-7, CodecParameters.cs:3-17)."""

    sample_count: int = -1
    history1: int = 0
    history2: int = 0
    progress: Optional[Callable[[int], None]] = None  # IProgressReport.ReportAdd


def _as_i16(a) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.int16)
    if a.ndim != 1:
        raise ValueError("expected a 1-D int16 array")
    return a


def _as_u8(a) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.uint8)
    if a.ndim != 1:
        raise ValueError("expected a 1-D uint8 array")
    return a


def _channel_list(channels, conv) -> list:
    if isinstance(channels, np.ndarray) and channels.ndim == 2:
        base = np.ascontiguousarray(channels, dtype=conv(np.zeros(0)).dtype)
        return [base[i] for i in range(base.shape[0])]  # views of one slab: uniform stride
    return [conv(c) for c in channels]


def _ptr_table(arrays: Sequence[np.ndarray]):
    tab = (C.c_void_p * max(len(arrays), 1))()
    for i, a in enumerate(arrays):
        tab[i] = a.ctypes.data
    return tab


def _params_array(configs, n: int):
    if configs is None:
        return None
    if isinstance(configs, GcAdpcmParameters):
        configs = [configs] * n
    if len(configs) != n:
        raise ValueError("one GcAdpcmParameters per channel expected")
    arr = (N.VgbGcParams * max(n, 1))()
    for i, p in enumerate(configs):
        p = p or GcAdpcmParameters()
        arr[i].sample_count, arr[i].history1, arr[i].history2 = p.sample_count, p.history1, p.history2
    return arr


# ---- GcAdpcmCoefficients ---------------------------------------------------------------------------------
def calculate_coefficients_batch(channels) -> np.ndarray:
    chans = _channel_list(channels, _as_i16)
    n = len(chans)
    coefs = np.zeros((n, 16), dtype=np.int16)
    lens = np.array([len(c) for c in chans], dtype=np.int32)
    N.check(N.lib.vgb_gcadpcm_coefs_batch(_ptr_table(chans), lens.ctypes.data, n, coefs.ctypes.data))
    return coefs


def calculate_coefficients(source) -> np.ndarray:
    """GcAdpcmCoefficients.CalculateCoefficients(short[] source) -> short[16]."""
    return calculate_coefficients_batch([source])[0]


# ---- GcAdpcmEncoder --------------------------------------------------------------------------------------
def encode_batch(channels, coefs=None, configs=None, progress: Optional[Callable[[int], None]] = None):
    """EncodeChannel (GcAdpcmFormat.cs:129-135) for every channel: returns (coefs[n,16], [adpcm bytes per channel]).
    With `coefs` given only GcAdpcmEncoder.Encode runs."""
    chans = _channel_list(channels, _as_i16)
    n = len(chans)
    lens = np.array([len(c) for c in chans], dtype=np.int32)
    params = _params_array(configs, n)
    coefs_out = np.zeros((n, 16), dtype=np.int16)
    coefs_in = None
    if coefs is not None:
        coefs_in = np.ascontiguousarray(coefs, dtype=np.int16).reshape(n, 16)
    counts = []
    for i in range(n):
        sc = lens[i] if params is None or params[i].sample_count == -1 else params[i].sample_count
        counts.append(int(sc))
    sizes = [sample_count_to_byte_count(max(c, 0)) for c in counts]
    if n and len(set(sizes)) == 1:
        slab = np.zeros((n, sizes[0]), dtype=np.uint8)
        outs = [slab[i] for i in range(n)]
    else:
        outs = [np.zeros(s, dtype=np.uint8) for s in sizes]
    cb = N.PROGRESS_CB(lambda user, delta: progress(delta)) if progress else None
    N.check(
        N.lib.vgb_gcadpcm_encode_batch(
            _ptr_table(chans), lens.ctypes.data, C.cast(params, C.c_void_p) if params is not None else None,
            coefs_in.ctypes.data if coefs_in is not None else None, n, coefs_out.ctypes.data, _ptr_table(outs),
            C.cast(cb, C.c_void_p) if cb else None, None,
        )
    )
    return coefs_out, outs


def encode(pcm, coefs, config: Optional[GcAdpcmParameters] = None) -> np.ndarray:
    """GcAdpcmEncoder.Encode(short[] pcm, short[] coefs, GcAdpcmParameters config = null) -> byte[]."""
    config = config or GcAdpcmParameters()
    _, outs = encode_batch([pcm], coefs=np.asarray(coefs, dtype=np.int16).reshape(1, 16), configs=[config],
                           progress=config.progress)
    return outs[0]


def dsp_encode_frames(pcm_in_out: np.ndarray, coefs: np.ndarray, sample_count=None) -> np.ndarray:
    """DspEncodeFrame for n independent frames. pcm_in_out [n,16] int16 is rewritten in place; returns [n,8]."""
    if not (isinstance(pcm_in_out, np.ndarray) and pcm_in_out.dtype == np.int16 and pcm_in_out.flags.c_contiguous):
        raise ValueError("pcm_in_out must be a C-contiguous int16 array [n,16] (it is rewritten in place)")
    io = pcm_in_out.reshape(-1, 16)
    n = io.shape[0]
    co = np.ascontiguousarray(coefs, dtype=np.int16).reshape(n, 16)
    out = np.zeros((n, 8), dtype=np.uint8)
    cnt = None
    if sample_count is not None:
        cnt = np.ascontiguousarray(np.broadcast_to(np.asarray(sample_count, dtype=np.int32), (n,)))
    N.check(N.lib.vgb_gcadpcm_encode_frames(io.ctypes.data, cnt.ctypes.data if cnt is not None else None,
                                            co.ctypes.data, n, out.ctypes.data))
    return out


def dsp_encode_frame(pcm_in_out: np.ndarray, sample_count: int, coefs) -> np.ndarray:
    """GcAdpcmEncoder.DspEncodeFrame(short[] pcmInOut, int sampleCount, byte[] adpcmOut, short[] coefsIn)."""
    return dsp_encode_frames(pcm_in_out, np.asarray(coefs, dtype=np.int16), sample_count)[0]


# ---- GcAdpcmDecoder --------------------------------------------------------------------------------------
def decode_batch(adpcm, coefs, configs=None) -> list:
    chans = _channel_list(adpcm, _as_u8)
    n = len(chans)
    lens = np.array([len(c) for c in chans], dtype=np.int32)
    params = _params_array(configs, n)
    co = np.ascontiguousarray(coefs, dtype=np.int16).reshape(n, 16)
    counts = []
    for i in range(n):
        sc = byte_count_to_sample_count(int(lens[i])) if params is None or params[i].sample_count == -1 \
            else params[i].sample_count
        counts.append(int(sc))
    if n and len(set(counts)) == 1 and counts[0] >= 0:
        slab = np.zeros((n, counts[0]), dtype=np.int16)
        outs = [slab[i] for i in range(n)]
    else:
        outs = [np.zeros(max(c, 0), dtype=np.int16) for c in counts]
    N.check(N.lib.vgb_gcadpcm_decode_batch(_ptr_table(chans), lens.ctypes.data, co.ctypes.data,
                                           C.cast(params, C.c_void_p) if params is not None else None, n,
                                           _ptr_table(outs)))
    return outs


def decode(adpcm, coefficients, config: Optional[GcAdpcmParameters] = None) -> np.ndarray:
    """GcAdpcmDecoder.Decode(byte[] adpcm, short[] coefficients, GcAdpcmParameters config = null) -> short[]."""
    return decode_batch([adpcm], np.asarray(coefficients, dtype=np.int16).reshape(1, 16),
                        [config] if config else None)[0]


# ---- post-encode channel rebuild (GcAdpcmChannelBuilder.GetSeekTable / GetLoopContext) ------------------------------
def seek_table_and_loop_context(adpcm, coefs, sample_counts, samples_per_seek_table_entry: int = 0, loop_starts=None):
    """For every channel: GcAdpcmSeekTable.CreateSeekTable(decoded pcm, samplesPerEntry) (GcAdpcmSeekTable.cs:25-38)
    and GcAdpcmLoopContext(adpcm, decoded pcm, loopStart) (GcAdpcmLoopContext.cs:17-26), without keeping the decoded
    PCM.  Returns (seek_tables: list of int16[entries*2] or None, loop_contexts: list of (pred_scale, hist1, hist2) or
    None per channel).  loop_starts: None, or one entry per channel (None / negative = no loop)."""
    chans = _channel_list(adpcm, _as_u8)
    n = len(chans)
    lens = np.array([len(c) for c in chans], dtype=np.int32)
    co = np.ascontiguousarray(coefs, dtype=np.int16).reshape(n, 16)
    counts = [int(sample_counts)] * n if np.isscalar(sample_counts) else [int(v) for v in sample_counts]
    loops = [-1] * n if loop_starts is None else [(-1 if v is None else int(v)) for v in loop_starts]
    params = (N.VgbGcTapParams * max(n, 1))()
    tables = []
    for i in range(n):
        params[i] = N.VgbGcTapParams(counts[i], samples_per_seek_table_entry, loops[i])
        entries = N.lib.vgb_gcadpcm_seek_entry_count(counts[i], samples_per_seek_table_entry)
        tables.append(np.zeros(entries * 2, dtype=np.int16))
    ctx = np.zeros((max(n, 1), 3), dtype=np.int16)
    ttab = (C.c_void_p * max(n, 1))(*[t.ctypes.data if t.size else None for t in tables])
    N.check(N.lib.vgb_gcadpcm_seek_context_batch(_ptr_table(chans), lens.ctypes.data, co.ctypes.data,
                                                 C.cast(params, C.c_void_p), n, ttab, ctx.ctypes.data))
    seek = [t if samples_per_seek_table_entry > 0 else None for t in tables]
    contexts = [(int(ctx[i, 0]) & 0xFF, int(ctx[i, 1]), int(ctx[i, 2])) if loops[i] >= 0 else None for i in range(n)]
    return seek, contexts


def alignment(multiple: int, loop_start: int, loop_end: int):
    """GcAdpcmAlignment's geometry (GcAdpcmAlignment.cs:22-31), host only: (alignment_needed, loop_start_aligned,
    sample_count_aligned), all zero when no alignment is needed."""
    out = N.VgbGcAlignment()
    N.check(N.lib.vgb_gcadpcm_alignment(C.byref(N.VgbGcAlignParams(multiple, loop_start, loop_end)), C.byref(out)))
    return bool(out.alignment_needed), out.loop_start_aligned, out.sample_count_aligned


def align_batch(adpcm, coefs, params, pcm: bool = True):
    """new GcAdpcmAlignment(multiple, loopStart, loopEnd, adpcm, coefs) (GcAdpcmAlignment.cs:20-63) for every channel in
    one call.  params: one (multiple, loop_start, loop_end) per channel, or one for all.  Returns (adpcm_aligned,
    pcm_aligned): per channel the AdpcmAligned bytes / PcmAligned samples, None where no alignment is needed (and for
    every PcmAligned when pcm is False)."""
    chans = _channel_list(adpcm, _as_u8)
    n = len(chans)
    lens = np.array([len(c) for c in chans], dtype=np.int32)
    co = np.ascontiguousarray(coefs, dtype=np.int16).reshape(n, 16)
    if n and np.ndim(params) == 1:
        params = [params] * n
    if len(params) != n:
        raise ValueError("one (multiple, loop_start, loop_end) per channel expected")
    par = (N.VgbGcAlignParams * max(n, 1))(*[N.VgbGcAlignParams(*map(int, p)) for p in params])
    out_a, out_p = [None] * n, [None] * n
    for i, p in enumerate(params):
        needed, _, count = alignment(*map(int, p))
        if needed:
            out_a[i] = np.zeros(sample_count_to_byte_count(count), dtype=np.uint8)
            out_p[i] = np.zeros(count, dtype=np.int16) if pcm else None
    ptab = (C.c_void_p * max(n, 1))(*[a.ctypes.data if a is not None else None for a in out_p])
    N.check(N.lib.vgb_gcadpcm_align_batch(_ptr_table(chans), lens.ctypes.data, co.ctypes.data, C.cast(par, C.c_void_p), n,
                                          (C.c_void_p * max(n, 1))(*[a.ctypes.data if a is not None else None for a in out_a]),
                                          ptab if pcm else None))
    return out_a, out_p


def get_predictor_scale(adpcm, sample: int) -> int:
    """GcAdpcmDecoder.GetPredictorScale (GcAdpcmDecoder.cs:56-59): metadata lookup, no arithmetic."""
    return int(adpcm[sample // SAMPLES_PER_FRAME * BYTES_PER_FRAME])
