"""Host-side mirror of VGAudio.Codecs.CriHca's encoder entry over the C ABI (no arithmetic here).

Reference interface (paths under VGAudio's src/VGAudio/):
  CriHcaParameters / CriHcaQuality                    Codecs/CriHca/CriHcaParameters.cs:3-15, CriHcaQuality.cs:3-10
  CriHcaEncoder.InitializeNew(config) -> .Hca (HcaInfo)  Codecs/CriHca/CriHcaEncoder.cs:49-114
  CriHcaFormat.EncodeFromPcm16(pcm16, config)          Formats/CriHca/CriHcaFormat.cs:34-84  (-> byte[FrameCount][FrameSize])
  CriHcaDecoder.Decode(hca, audio, config) -> short[][] Codecs/CriHca/CriHcaDecoder.cs:11-25
Looping streams (Pcm16Format.Looping / LoopStart / LoopEnd -> CriHcaParameters) are encoded like the reference's
streaming front end does (pre-roll, loop-start audio appended after the loop end, loop frame aligned to 2048 bytes).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _native as N

NOT_SET, HIGHEST, HIGH, MIDDLE, LOW, LOWEST = range(6)  # CriHcaQuality


@dataclass
class CriHcaParameters:
    quality: int = HIGH
    bitrate: int = 0
    limit_bitrate: bool = False
    channel_count: int = 0
    sample_rate: int = 0
    sample_count: int = -1
    looping: bool = False
    loop_start: int = 0
    loop_end: int = 0
    progress: Optional[Callable[[int], None]] = None

    def _native(self) -> N.VgbHcaParams:
        return N.VgbHcaParams(self.quality, self.bitrate, int(self.limit_bitrate), self.channel_count, self.sample_rate,
                              self.sample_count, int(self.looping), self.loop_start, self.loop_end)


def query(config: CriHcaParameters) -> N.VgbHcaInfo:
    """CriHcaEncoder.InitializeNew(config).Hca"""
    info = N.VgbHcaInfo()
    p = config._native()
    N.check(N.lib.vgb_hca_query(C.byref(p), C.byref(info)))
    return info


def encode_batch(streams: Sequence[Sequence[np.ndarray]], sample_rate: int, config: Optional[CriHcaParameters] = None,
                 progress: Optional[Callable[[int], None]] = None):
    """CriHcaFormat.EncodeFromPcm16 for a batch of streams (each a list of equally long int16 channels) that share the
    configuration.  Returns ([HcaInfo], [frames uint8[frame_count, frame_size]])."""
    config = config or CriHcaParameters()
    n = len(streams)
    if n == 0:
        return [], []
    nch = len(streams[0])
    chans = []
    params = (N.VgbHcaParams * n)()
    for s, st in enumerate(streams):
        if len(st) != nch:
            raise ValueError("all streams of a batch must have the same channel count")
        arrs = [np.ascontiguousarray(c, dtype=np.int16) for c in st]
        if len({len(a) for a in arrs}) > 1:
            raise ValueError("All channels must have the same sample count")
        chans.extend(arrs)
        params[s] = N.VgbHcaParams(config.quality, config.bitrate, int(config.limit_bitrate), nch, sample_rate,
                                   len(arrs[0]) if arrs else 0, int(config.looping), config.loop_start, config.loop_end)
    infos = (N.VgbHcaInfo * n)()
    for s in range(n):
        N.check(N.lib.vgb_hca_query(C.byref(params[s]), C.byref(infos[s])))
    outs = [np.zeros((infos[s].frame_count, infos[s].frame_size), dtype=np.uint8) for s in range(n)]
    ptab = (C.c_void_p * max(len(chans), 1))(*[a.ctypes.data for a in chans])
    otab = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    cb = N.PROGRESS_CB(lambda user, delta: progress(delta)) if progress else None
    N.check(N.lib.vgb_hca_encode_batch(ptab, C.cast(params, C.c_void_p), n, C.cast(infos, C.c_void_p), otab,
                                       C.cast(cb, C.c_void_p) if cb else None, None))
    return [infos[s] for s in range(n)], outs


def encode(channels: Sequence[np.ndarray], sample_rate: int, config: Optional[CriHcaParameters] = None):
    """One stream: (HcaInfo, frames[frame_count, frame_size])."""
    config = config or CriHcaParameters()
    infos, outs = encode_batch([channels], sample_rate, config, config.progress)
    return infos[0], outs[0]


def decode_batch(infos: Sequence[N.VgbHcaInfo], frames: Sequence[np.ndarray]) -> List[List[np.ndarray]]:
    """CriHcaDecoder.Decode for a batch of streams that share the band layout: frames[s] is uint8[frame_count,
    frame_size] (the reference's byte[][] audio); returns per stream a list of int16[sample_count] channels."""
    n = len(infos)
    if n == 0:
        return []
    if len(frames) != n:
        raise ValueError("one frame array per stream")
    nch = infos[0].channel_count
    info_arr = (N.VgbHcaInfo * n)(*infos)
    ins = []
    for s in range(n):
        f = np.ascontiguousarray(frames[s], dtype=np.uint8).reshape(-1)
        if f.size < infos[s].frame_count * infos[s].frame_size:
            raise ValueError(f"stream {s}: {f.size} bytes of frames, HcaInfo needs {infos[s].frame_count * infos[s].frame_size}")
        ins.append(f)
    outs = [[np.zeros(max(infos[s].sample_count, 0), dtype=np.int16) for _ in range(nch)] for s in range(n)]
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in ins])
    flat = [a for st in outs for a in st]
    otab = (C.c_void_p * max(len(flat), 1))(*[a.ctypes.data for a in flat])
    N.check(N.lib.vgb_hca_decode_batch(ftab, C.cast(info_arr, C.c_void_p), n, otab))
    return outs


def decode(info: N.VgbHcaInfo, frames: np.ndarray) -> List[np.ndarray]:
    """One stream: list of int16[sample_count] channels."""
    return decode_batch([info], [frames])[0]


def mdct_run(blocks: np.ndarray, inverse: bool = False) -> np.ndarray:
    """Mdct.RunMdct / RunImdct (Utilities/Mdct.cs:63-119) of the codec's 128-point instance over sequences of blocks:
    blocks is float64[..., n_blocks, 128]; every leading index is an independent sequence starting from zero state."""
    a = np.ascontiguousarray(blocks, dtype=np.float64)
    if a.ndim < 2 or a.shape[-1] != 128:
        raise ValueError("expected float64[..., n_blocks, 128]")
    n_blocks = a.shape[-2]
    n_seq = int(np.prod(a.shape[:-2])) if a.ndim > 2 else 1
    out = np.empty_like(a)
    fn = N.lib.vgb_imdct128_batch if inverse else N.lib.vgb_mdct128_batch
    N.check(fn(a.ctypes.data, n_seq, n_blocks, out.ctypes.data))
    return out
