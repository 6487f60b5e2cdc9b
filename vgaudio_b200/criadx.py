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


def decode_dev(d_adpcm, adpcm_offset, n_bytes, sample_counts, configs, d_pcm, pcm_offset, stream=None, workspace=None):
    """CriAdxCodec.Decode for every channel on device buffers (vgb_adx_decode_dev, the time-parallel decoder): d_adpcm is
    a uint8 and d_pcm an int16 CUDA tensor (views at any element offset are fine); channel c reads n_bytes[c] bytes at
    adpcm_offset[c] and writes sample_counts[c] samples at pcm_offset[c].  Runs on `stream` (a torch.cuda.Stream, default
    the current one) and waits for it; raises VgbError(VGB_E_DATA) for a Fixed-type frame with a filter outside 0..3.
    `workspace` (a uint8 CUDA tensor of at least vgb_adx_decode_workspace_bytes) is allocated when None.  Returns the
    workspace: vgb_adx_debug_decode_stats reads the last decode's bookkeeping from it, so keep it while the tap is read."""
    import torch

    n = len(sample_counts)
    if isinstance(configs, CriAdxParameters):
        configs = [configs] * n
    counts = np.ascontiguousarray(sample_counts, dtype=np.int32)
    nb = np.ascontiguousarray(n_bytes, dtype=np.int32)
    a_off = np.ascontiguousarray(adpcm_offset, dtype=np.int64)
    p_off = np.ascontiguousarray(pcm_offset, dtype=np.int64)
    params = _params_array(configs)
    ws_bytes = N.lib.vgb_adx_decode_workspace_bytes(counts.ctypes.data, C.cast(params, C.c_void_p), n)
    if workspace is None:
        workspace = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=d_pcm.device)
    st = (stream or torch.cuda.current_stream(d_pcm.device)).cuda_stream
    N.check(N.lib.vgb_adx_decode_dev(d_adpcm.data_ptr(), a_off.ctypes.data, nb.ctypes.data, counts.ctypes.data, C.cast(params, C.c_void_p), n,
                                     d_pcm.data_ptr(), p_off.ctypes.data, workspace.data_ptr(), workspace.numel(), st))
    N.check(N.lib.vgb_adx_decode_dev_status(workspace.data_ptr(), n, st))
    return workspace
