"""Host-side mirror of VGAudio.Codecs.CriAdx over the C ABI (no arithmetic here).

Reference interface (paths under VGAudio's src/VGAudio/):
  CriAdxCodec.Encode(short[] pcm, CriAdxParameters config) -> byte[]     Codecs/CriAdx/CriAdxCodec.cs:56  (mutates config.History)
  CriAdxCodec.Decode(byte[] adpcm, int sampleCount, CriAdxParameters)    Codecs/CriAdx/CriAdxCodec.cs:9
  CriAdxParameters                                                         Codecs/CriAdx/CriAdxParameters.cs:3-13
  CriAdxFormat.EncodeFromPcm16 / ToPcm16 loop bodies                       Formats/CriAdx/CriAdxFormat.cs:67-81 / :37-49
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, replace
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _native as N
from .gcadpcm import _as_i16, _as_u8, _channel_list, _ptr_table

FIXED, LINEAR, EXPONENTIAL = 2, 3, 4  # CriAdxType.cs:3-8


@dataclass
class CriAdxParameters:
    sample_rate: int = 48000
    highpass_frequency: int = 500
    frame_size: int = 18
    version: int = 4
    history: int = 0
    padding: int = 0
    type: int = LINEAR
    filter: int = 0
    progress: Optional[Callable[[int], None]] = None


def _params_array(configs: Sequence[CriAdxParameters]):
    arr = (N.VgbAdxParams * max(len(configs), 1))()
    for i, p in enumerate(configs):
        arr[i].sample_rate, arr[i].highpass_frequency, arr[i].frame_size = p.sample_rate, p.highpass_frequency, p.frame_size
        arr[i].version, arr[i].history, arr[i].padding, arr[i].type, arr[i].filter = p.version, p.history, p.padding, p.type, p.filter
    return arr


def encoded_byte_count(pcm_length: int, padding: int, frame_size: int) -> int:
    return N.lib.vgb_adx_encoded_byte_count(pcm_length, padding, frame_size)


def encode_batch(channels, configs, progress: Optional[Callable[[int], None]] = None):
    """One CriAdxCodec.Encode per channel in a single call: returns ([adpcm bytes], history[n])."""
    chans = _channel_list(channels, _as_i16)
    n = len(chans)
    if isinstance(configs, CriAdxParameters):
        configs = [configs] * n
    lens = np.array([len(c) for c in chans], dtype=np.int32)
    params = _params_array(configs)
    sizes = [encoded_byte_count(int(lens[i]), configs[i].padding, configs[i].frame_size) for i in range(n)]
    if n and len(set(sizes)) == 1:
        slab = np.zeros((n, sizes[0]), dtype=np.uint8)
        outs = [slab[i] for i in range(n)]
    else:
        outs = [np.zeros(s, dtype=np.uint8) for s in sizes]
    hist = np.zeros(n, dtype=np.int16)
    cb = N.PROGRESS_CB(lambda user, delta: progress(delta)) if progress else None
    N.check(N.lib.vgb_adx_encode_batch(_ptr_table(chans), lens.ctypes.data, C.cast(params, C.c_void_p), n,
                                       hist.ctypes.data, _ptr_table(outs), C.cast(cb, C.c_void_p) if cb else None, None))
    return outs, hist


def encode(pcm, config: CriAdxParameters) -> np.ndarray:
    """CriAdxCodec.Encode: like the reference it writes the seeded history back into `config.history`."""
    outs, hist = encode_batch([pcm], [config], config.progress)
    if config.version == 4 and config.padding == 0:
        config.history = int(hist[0])  # CriAdxCodec.cs:73
    return outs[0]


def decode_batch(adpcm, sample_counts, configs) -> List[np.ndarray]:
    chans = _channel_list(adpcm, _as_u8)
    n = len(chans)
    if isinstance(configs, CriAdxParameters):
        configs = [configs] * n
    if np.isscalar(sample_counts):
        sample_counts = [int(sample_counts)] * n
    lens = np.array([len(c) for c in chans], dtype=np.int32)
    counts = np.array(sample_counts, dtype=np.int32)
    params = _params_array(configs)
    if n and len(set(counts.tolist())) == 1 and counts[0] >= 0:
        slab = np.zeros((n, int(counts[0])), dtype=np.int16)
        outs = [slab[i] for i in range(n)]
    else:
        outs = [np.zeros(max(int(c), 0), dtype=np.int16) for c in counts]
    N.check(N.lib.vgb_adx_decode_batch(_ptr_table(chans), lens.ctypes.data, counts.ctypes.data,
                                       C.cast(params, C.c_void_p), n, _ptr_table(outs)))
    return outs


def decode(adpcm, sample_count: int, config: Optional[CriAdxParameters] = None) -> np.ndarray:
    """CriAdxCodec.Decode(byte[] adpcm, int sampleCount, CriAdxParameters config = null)."""
    return decode_batch([adpcm], [sample_count], [config or CriAdxParameters()])[0]
