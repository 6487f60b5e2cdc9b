"""ctypes wrapper of oracle/libvgoracle.so — TEST INFRASTRUCTURE (see oracle/vgoracle.h).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VGORACLE_LIB") or os.path.join(_HERE, "libvgoracle.so")  # VGORACLE_LIB: e.g. the `make asan` build


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h")) or f == "Makefile"]
    stale = not os.path.exists(LIB_PATH) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs)
    if force or stale:
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        L = C.CDLL(LIB_PATH)
        i32, i64, vp = C.c_int, C.c_int64, C.c_void_p
        for name in ("vgo_gc_nibble_count_to_sample_count", "vgo_gc_sample_count_to_nibble_count",
                     "vgo_gc_nibble_to_sample", "vgo_gc_sample_to_nibble", "vgo_gc_sample_count_to_byte_count",
                     "vgo_gc_byte_count_to_sample_count"):
            getattr(L, name).argtypes = [i32]
            getattr(L, name).restype = i32
        L.vgo_divide_by_round_up.argtypes = [i32, i32]
        L.vgo_gc_calculate_coefficients.argtypes = [vp, i32, vp]
        L.vgo_gc_calculate_coefficients.restype = None
        L.vgo_gc_coef_records.argtypes = [vp, i32, vp, vp, vp]
        L.vgo_gc_encode.argtypes = [vp, i32, vp, i32, C.c_int16, C.c_int16, vp]
        L.vgo_gc_encode.restype = None
        L.vgo_gc_dsp_encode_frame.argtypes = [vp, i32, vp, vp]
        L.vgo_gc_dsp_encode_frame.restype = None
        L.vgo_gc_decode.argtypes = [vp, vp, i32, C.c_int16, C.c_int16, vp]
        L.vgo_gc_decode.restype = None
        L.vgo_gc_seek_table.argtypes = [vp, i32, i32, vp]
        L.vgo_gc_seek_table.restype = i32
        L.vgo_gc_loop_context.argtypes = [vp, vp, i32, vp]
        L.vgo_gc_loop_context.restype = None
        L.vgo_gc_encode_batch.argtypes = [vp, i64, i32, i32, vp, vp, i64, i32]
        L.vgo_gc_decode_batch.argtypes = [vp, i64, vp, i32, i32, vp, i64, i32]
        L.vgo_adx_calculate_coefficients.argtypes = [i32, i32, vp]
        L.vgo_adx_calculate_coefficients.restype = None
        L.vgo_adx_encoded_byte_count.argtypes = [i32, i32, i32]
        L.vgo_adx_encode_frame.argtypes = [vp, vp, vp, i32, i32, i32]
        L.vgo_adx_encode_frame.restype = None
        L.vgo_adx_encode.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, vp]
        L.vgo_adx_decode.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, i32, vp]
        L.vgo_adx_decode.restype = None
        L.vgo_hca_init.argtypes = [vp, vp]
        L.vgo_hca_encode.argtypes = [vp, vp, vp, vp]
        L.vgo_hca_encode_ath.argtypes = [vp, vp, vp, vp]
        L.vgo_hca_spectra.argtypes = [vp, vp, vp]
        L.vgo_hca_decode.argtypes = [vp, vp, vp]
        L.vgo_hca_unpack_ok.argtypes = [vp, vp]
        L.vgo_hca_unpack_ok.restype = C.c_int
        L.vgo_hca_mdct_run.argtypes = [vp, i32, vp]
        L.vgo_hca_mdct_run.restype = None
        L.vgo_hca_imdct_run.argtypes = [vp, i32, vp]
        L.vgo_hca_imdct_run.restype = None
        L.vgo_hca_mdct_tables.argtypes = [vp, vp, vp, i32]
        L.vgo_hca_mdct_tables.restype = None
        L.vgo_crc16.argtypes = [vp, i32]
        L.vgo_crc16.restype = C.c_uint16
        _lib = L
    return _lib


def sample_count_to_byte_count(n: int) -> int:
    return lib().vgo_gc_sample_count_to_byte_count(n)


def calculate_coefficients(pcm) -> np.ndarray:
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    co = np.zeros(16, dtype=np.int16)
    lib().vgo_gc_calculate_coefficients(pcm.ctypes.data, len(pcm), co.ctypes.data)
    return co


def coef_records(pcm):
    """(accepted[frames] uint8, records[frames,2], direct[frames,2]) of coefficient phase 1."""
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    frames = (len(pcm) + 13) // 14
    rec = np.zeros((frames, 2)); dire = np.zeros((frames, 2)); acc = np.zeros(frames, dtype=np.uint8)
    lib().vgo_gc_coef_records(pcm.ctypes.data, len(pcm), rec.ctypes.data, dire.ctypes.data, acc.ctypes.data)
    return acc, rec, dire


GC_COEF_PASSES = 7
# phase-1 outcome of a frame (vgoracle.h VGO_GC_ACCEPTED / VGO_GC_REJ_*)
GC_ACCEPTED, GC_REJ_QUIET, GC_REJ_BIG, GC_REJ_RANGE, GC_REJ_DEN, GC_REJ_K1 = range(6)
GC_COEF_PASS = np.dtype([("cent", np.float64, (8, 2)), ("hits", np.int32, 8), ("count", np.int32), ("empty", np.int32),
                         ("ties_same", np.int32), ("ties_distinct", np.int32), ("tie_record", np.int32),
                         ("tie_lo", np.int32), ("tie_hi", np.int32), ("pad", np.int32)], align=True)
GC_COEF_TRACE = np.dtype([("pass", GC_COEF_PASS, GC_COEF_PASSES), ("n_frames", np.int32), ("n_records", np.int32)],
                         align=True)


def gc_coef_trace(pcm):
    """calculate_coefficients() plus the trace of every refinement pass and every frame's phase-1 outcome:
    (coefs[16] int16, GC_COEF_TRACE record, outcome[frames] uint8)."""
    L = lib()
    if not getattr(L, "_coef_trace_ready", False):
        L.vgo_gc_coef_trace.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.vgo_gc_coef_trace.restype = None
        if L.vgo_gc_refine_trace_size() != GC_COEF_TRACE.itemsize:
            raise RuntimeError("vgo_gc_refine_trace layout differs from GC_COEF_TRACE")
        L._coef_trace_ready = True
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    co = np.zeros(16, dtype=np.int16)
    trace = np.zeros((), dtype=GC_COEF_TRACE)
    outcome = np.zeros((len(pcm) + 13) // 14, dtype=np.uint8)
    L.vgo_gc_coef_trace(pcm.ctypes.data, len(pcm), trace.ctypes.data, outcome.ctypes.data, co.ctypes.data)
    return co, trace, outcome


def encode(pcm, coefs, sample_count: int = -1, history1: int = 0, history2: int = 0) -> np.ndarray:
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    coefs = np.ascontiguousarray(coefs, dtype=np.int16)
    n = len(pcm) if sample_count == -1 else sample_count
    out = np.zeros(sample_count_to_byte_count(n), dtype=np.uint8)
    lib().vgo_gc_encode(pcm.ctypes.data, len(pcm), coefs.ctypes.data, sample_count, history1, history2, out.ctypes.data)
    return out


GC_PRED_TRACE = np.dtype([("error", np.uint64), ("max_abs_diff", np.uint32), ("over", np.int32, 13),
                          ("first_sp", np.int8), ("n_passes", np.int8), ("final_sp", np.int8), ("bumped", np.uint8),
                          ("final12", np.uint8), ("wrapped", np.uint8), ("pad", np.uint8, 2)], align=True)
GC_FRAME_TRACE = np.dtype([("pred", GC_PRED_TRACE, 8), ("winner", np.int8), ("tie", np.uint8), ("pad", np.uint8, 6)],
                          align=True)


def gc_encode_trace(pcm, coefs, sample_count: int = -1, h1: int = 0, h2: int = 0):
    """encode() plus one vgo_gc_frame_trace record per frame: (adpcm bytes, structured array of GC_FRAME_TRACE)."""
    L = lib()
    if not getattr(L, "_trace_ready", False):
        L.vgo_gc_encode_trace.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int16, C.c_int16, C.c_void_p,
                                          C.c_void_p]
        L.vgo_gc_encode_trace.restype = None
        if L.vgo_gc_frame_trace_size() != GC_FRAME_TRACE.itemsize:
            raise RuntimeError("vgo_gc_frame_trace layout differs from GC_FRAME_TRACE")
        L._trace_ready = True
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    coefs = np.ascontiguousarray(coefs, dtype=np.int16)
    n = len(pcm) if sample_count == -1 else sample_count
    out = np.zeros(sample_count_to_byte_count(n), dtype=np.uint8)
    trace = np.zeros((n + 13) // 14, dtype=GC_FRAME_TRACE)
    L.vgo_gc_encode_trace(pcm.ctypes.data, len(pcm), coefs.ctypes.data, sample_count, h1, h2, out.ctypes.data,
                          trace.ctypes.data)
    return out, trace


def dsp_encode_frame(pcm_in_out: np.ndarray, sample_count: int, coefs) -> np.ndarray:
    assert pcm_in_out.dtype == np.int16 and pcm_in_out.flags.c_contiguous and pcm_in_out.size == 16
    coefs = np.ascontiguousarray(coefs, dtype=np.int16)
    out = np.zeros(8, dtype=np.uint8)
    lib().vgo_gc_dsp_encode_frame(pcm_in_out.ctypes.data, sample_count, out.ctypes.data, coefs.ctypes.data)
    return out


def decode(adpcm, coefs, sample_count: int, history1: int = 0, history2: int = 0) -> np.ndarray:
    adpcm = np.ascontiguousarray(adpcm, dtype=np.uint8)
    coefs = np.ascontiguousarray(coefs, dtype=np.int16)
    out = np.zeros(sample_count, dtype=np.int16)
    lib().vgo_gc_decode(adpcm.ctypes.data, coefs.ctypes.data, sample_count, history1, history2, out.ctypes.data)
    return out


def encode_batch(pcm2d: np.ndarray, n_threads: int = 0):
    """Reference Parallel.For path: (coefs[n,16], adpcm[n,bytes], threads_used)."""
    pcm2d = np.ascontiguousarray(pcm2d, dtype=np.int16)
    n_ch, n = pcm2d.shape
    nb = sample_count_to_byte_count(n)
    coefs = np.zeros((n_ch, 16), dtype=np.int16)
    out = np.zeros((n_ch, nb), dtype=np.uint8)
    used = lib().vgo_gc_encode_batch(pcm2d.ctypes.data, n, n_ch, n, coefs.ctypes.data, out.ctypes.data, nb, n_threads)
    return coefs, out, used


def decode_batch(adpcm2d: np.ndarray, coefs: np.ndarray, sample_count: int, n_threads: int = 0):
    adpcm2d = np.ascontiguousarray(adpcm2d, dtype=np.uint8)
    coefs = np.ascontiguousarray(coefs, dtype=np.int16)
    n_ch, nb = adpcm2d.shape
    out = np.zeros((n_ch, sample_count), dtype=np.int16)
    used = lib().vgo_gc_decode_batch(adpcm2d.ctypes.data, nb, coefs.ctypes.data, n_ch, sample_count, out.ctypes.data,
                                     sample_count, n_threads)
    return out, used


# ---- CRI ADX (oracle/criadx.c; parity unpinned, see vgoracle.h) ----------------------------------------------------
ADX_FIXED, ADX_LINEAR, ADX_EXPONENTIAL = 2, 3, 4


def adx_coefficients(highpass_freq: int, sample_rate: int) -> np.ndarray:
    co = np.zeros(2, dtype=np.int16)
    lib().vgo_adx_calculate_coefficients(highpass_freq, sample_rate, co.ctypes.data)
    return co


def adx_encode(pcm, sample_rate=48000, frame_size=18, version=4, padding=0, type=ADX_LINEAR, filter=0):
    """CriAdxCodec.Encode -> (adpcm bytes, History written back into the config)."""
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    out = np.zeros(lib().vgo_adx_encoded_byte_count(len(pcm), padding, frame_size), dtype=np.uint8)
    hist = lib().vgo_adx_encode(pcm.ctypes.data, len(pcm), sample_rate, frame_size, version, padding, type, filter,
                                out.ctypes.data)
    return out, hist


def adx_decode(adpcm, sample_count, sample_rate=48000, highpass_freq=500, frame_size=18, version=4, history=0,
               padding=0, type=ADX_LINEAR):
    adpcm = np.ascontiguousarray(adpcm, dtype=np.uint8)
    out = np.zeros(sample_count, dtype=np.int16)
    lib().vgo_adx_decode(adpcm.ctypes.data, sample_count, sample_rate, highpass_freq, frame_size, version, history,
                         padding, type, out.ctypes.data)
    return out


def adx_encode_frame(pcm_in_out: np.ndarray, coefs, samples_per_frame=32, type=ADX_LINEAR, version=4) -> np.ndarray:
    assert pcm_in_out.dtype == np.int16 and pcm_in_out.flags.c_contiguous and pcm_in_out.size == samples_per_frame + 2
    coefs = np.ascontiguousarray(coefs, dtype=np.int16)
    out = np.zeros(samples_per_frame // 2 + 2, dtype=np.uint8)
    lib().vgo_adx_encode_frame(pcm_in_out.ctypes.data, out.ctypes.data, coefs.ctypes.data, samples_per_frame, type,
                               version)
    return out


# ---- CRI HCA (oracle/crihca.c; tables pinned, frame bytes parity unpinned, non-looping only) -----------------------
class HcaParams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("quality", "bitrate", "limit_bitrate", "channel_count", "sample_rate",
                                         "sample_count", "looping", "loop_start", "loop_end")]


class HcaInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "channel_count", "sample_rate", "sample_count", "frame_count", "inserted_samples", "appended_samples",
        "header_size", "frame_size", "min_resolution", "max_resolution", "track_count", "channel_config",
        "total_band_count", "base_band_count", "stereo_band_count", "hfr_band_count", "bands_per_hfr_group",
        "hfr_group_count", "bitrate", "looping", "loop_start_frame", "loop_end_frame", "pre_loop_samples",
        "post_loop_samples", "use_ath_curve")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


def _chan_table(channels):
    arrs = [np.ascontiguousarray(c, dtype=np.int16) for c in channels]
    tab = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    return arrs, tab


def gc_seek_table(pcm, samples_per_entry) -> np.ndarray:
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    entries = -(-len(pcm) // samples_per_entry) if samples_per_entry > 0 else 0
    out = np.zeros(entries * 2, dtype=np.int16)
    if entries:
        lib().vgo_gc_seek_table(C.c_void_p(pcm.ctypes.data), len(pcm), samples_per_entry, C.c_void_p(out.ctypes.data))
    return out


def gc_loop_context(adpcm, pcm, loop_start):
    adpcm = np.ascontiguousarray(adpcm, dtype=np.uint8)
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    out = np.zeros(3, dtype=np.int16)
    lib().vgo_gc_loop_context(C.c_void_p(adpcm.ctypes.data), C.c_void_p(pcm.ctypes.data), int(loop_start), C.c_void_p(out.ctypes.data))
    return int(out[0]) & 0xFF, int(out[1]), int(out[2])


def interleave(inputs, interleave_size, output_size=-1) -> np.ndarray:
    arrs = [np.ascontiguousarray(a, dtype=np.uint8).ravel() for a in inputs]
    count, in_size = len(arrs), arrs[0].size
    out_size = in_size if output_size == -1 else output_size
    out = np.zeros(out_size * count, dtype=np.uint8)
    tab = (C.c_void_p * count)(*[a.ctypes.data for a in arrs])
    L = lib()
    L.vgo_interleave.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.vgo_interleave(tab, count, in_size, interleave_size, out_size, out.ctypes.data)
    return out


def deinterleave(data, interleave_size, output_count, output_size=-1):
    data = np.ascontiguousarray(data, dtype=np.uint8).ravel()
    in_size = data.size // output_count
    out_size = in_size if output_size == -1 else output_size
    outs = [np.zeros(out_size, dtype=np.uint8) for _ in range(output_count)]
    tab = (C.c_void_p * output_count)(*[o.ctypes.data for o in outs])
    L = lib()
    L.vgo_deinterleave.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.vgo_deinterleave.restype = C.c_int
    if L.vgo_deinterleave(data.ctypes.data, data.size, interleave_size, output_count, out_size, tab) != 0:
        raise ValueError("The input array length must be divisible by the number of outputs.")
    return outs


def hca_params(channels, sample_rate=48000, quality=2, bitrate=0, limit_bitrate=False, loop=None) -> HcaParams:
    """loop = (loop_start, loop_end) in samples or None (Pcm16Format.Looping / LoopStart / LoopEnd)."""
    looping, ls, le = (1, int(loop[0]), int(loop[1])) if loop else (0, 0, 0)
    return HcaParams(quality, bitrate, int(limit_bitrate), len(channels), sample_rate, len(channels[0]), looping, ls, le)


def hca_init(params: HcaParams) -> HcaInfo:
    info = HcaInfo()
    rc = lib().vgo_hca_init(C.byref(params), C.byref(info))
    if rc:
        raise ValueError(f"vgo_hca_init failed: {rc}")
    return info


def hca_encode(channels, sample_rate=48000, quality=2, bitrate=0, limit_bitrate=False, loop=None, ath=False):
    """CriHcaFormat.EncodeFromPcm16 for one stream -> (HcaInfo, frames[frame_count, frame_size]).
    ath=True: the test helper vgo_hca_encode_ath (a stream for the decoder's UseAthCurve path)."""
    arrs, tab = _chan_table(channels)
    p = hca_params(arrs, sample_rate, quality, bitrate, limit_bitrate, loop)
    info = hca_init(p)
    frames = np.zeros((info.frame_count, info.frame_size), dtype=np.uint8)
    fn = lib().vgo_hca_encode_ath if ath else lib().vgo_hca_encode
    rc = fn(tab, C.byref(p), C.byref(info), frames.ctypes.data)
    if rc:
        raise ValueError(f"vgo_hca_encode failed: {rc}")
    return info, frames


def hca_spectra(channels, sample_rate=48000, quality=2, bitrate=0):
    arrs, tab = _chan_table(channels)
    p = hca_params(arrs, sample_rate, quality, bitrate)
    info = hca_init(p)
    out = np.zeros((info.frame_count, info.channel_count, 8, 128))
    lib().vgo_hca_spectra(tab, C.byref(p), out.ctypes.data)
    return out


def hca_decode(info: HcaInfo, frames) -> np.ndarray:
    frames = np.ascontiguousarray(frames, dtype=np.uint8)
    out = np.zeros((info.channel_count, info.sample_count), dtype=np.int16)
    tab = (C.c_void_p * info.channel_count)(*[out[c].ctypes.data for c in range(info.channel_count)])
    lib().vgo_hca_decode(C.byref(info), frames.ctypes.data, tab)
    return out


def hca_unpack_ok(info, frames) -> bool:
    frames = np.ascontiguousarray(frames, dtype=np.uint8)
    return bool(lib().vgo_hca_unpack_ok(C.byref(info), frames.ctypes.data))


def hca_mdct(blocks: np.ndarray) -> np.ndarray:
    blocks = np.ascontiguousarray(blocks, dtype=np.float64).reshape(-1, 128)
    out = np.zeros_like(blocks)
    lib().vgo_hca_mdct_run(blocks.ctypes.data, len(blocks), out.ctypes.data)
    return out


def hca_imdct(spectra: np.ndarray) -> np.ndarray:
    spectra = np.ascontiguousarray(spectra, dtype=np.float64).reshape(-1, 128)
    out = np.zeros_like(spectra)
    lib().vgo_hca_imdct_run(spectra.ctypes.data, len(spectra), out.ctypes.data)
    return out


def hca_mdct_tables(bits: int):
    n = 1 << bits
    s, c, sh = np.zeros(n), np.zeros(n), np.zeros(n, dtype=np.int32)
    lib().vgo_hca_mdct_tables(s.ctypes.data, c.ctypes.data, sh.ctypes.data, bits)
    return s, c, sh


def crc16(data: bytes) -> int:
    buf = np.frombuffer(data, dtype=np.uint8)
    return int(lib().vgo_crc16(buf.ctypes.data, len(buf)))


# ---- container layer (oracle/containers.c; SURVEY.md 8f rank 2-4) -------------------------------------------------------
class WaveInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("channel_count", "sample_rate", "bits_per_sample", "sample_count", "looping",
                                         "loop_start", "loop_end", "reserved")] + [("data_offset", C.c_int64), ("data_size", C.c_int64)]


class DspDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("channel_count", "sample_rate", "sample_count", "looping", "loop_start", "loop_end",
                                         "samples_per_interleave", "loop_point_alignment", "trim_file")]


class DspInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("sample_count", "nibble_count", "sample_rate", "looping", "format", "start_address",
                                         "end_address", "current_address", "channel_count", "frames_per_interleave",
                                         "loop_start", "loop_end")] + [
        ("coefs", (C.c_int16 * 16) * 64), ("gain", C.c_int16 * 64), ("start_ctx", (C.c_int16 * 3) * 64), ("loop_ctx", (C.c_int16 * 3) * 64)]


class AdxDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("channel_count", "sample_rate", "sample_count", "looping", "loop_start", "loop_end",
                                         "alignment_samples", "frame_size", "version", "type", "highpass_frequency",
                                         "encryption_type", "trim_file")]


def _u8(b) -> np.ndarray:
    return np.frombuffer(bytes(b), dtype=np.uint8) if not isinstance(b, np.ndarray) else np.ascontiguousarray(b, dtype=np.uint8).ravel()


def _ptrs(rows):
    return (C.c_void_p * max(len(rows), 1))(*[r.ctypes.data for r in rows])


def wave_parse(file):
    """(status, WaveInfo): status 0 or a VGO_E_* code."""
    L = lib()
    f = _u8(file)
    info = WaveInfo()
    L.vgo_wave_parse.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    return int(L.vgo_wave_parse(f.ctypes.data, f.size, C.byref(info))), info


def wave_read(file, info: WaveInfo):
    L = lib()
    f = _u8(file)
    rows = [np.zeros(info.sample_count, dtype=np.int16) for _ in range(info.channel_count)]
    fn = L.vgo_wave_read16 if info.bits_per_sample == 16 else L.vgo_wave_read8_as16
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    fn.restype = None
    fn(f.ctypes.data, C.byref(info), _ptrs(rows))
    return rows


def wave_write16(channels, sample_rate=48000, loop=None) -> np.ndarray:
    """WaveWriter (16-bit codec): the reference's own way to make the files its reader test parses."""
    L = lib()
    rows = [np.ascontiguousarray(c, dtype=np.int16) for c in channels]
    n = rows[0].size
    L.vgo_wave_file_size.restype = C.c_int64
    L.vgo_wave_file_size.argtypes = [C.c_int, C.c_int, C.c_int]
    out = np.zeros(L.vgo_wave_file_size(len(rows), n, int(loop is not None)), dtype=np.uint8)
    L.vgo_wave_write16.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.vgo_wave_write16.restype = None
    L.vgo_wave_write16(_ptrs(rows), len(rows), n, sample_rate, int(loop is not None), loop[0] if loop else 0, loop[1] if loop else 0,
                       out.ctypes.data)
    return out


def dsp_write(adpcm, coefs, sample_rate, sample_count, loop=None, loop_ctx=None, gain=None, start_hist=None,
              samples_per_interleave=0x3800, loop_point_alignment=1, trim_file=True) -> np.ndarray:
    L = lib()
    rows = [_u8(a) for a in adpcm]
    d = DspDesc(len(rows), sample_rate, sample_count, int(loop is not None), loop[0] if loop else 0, loop[1] if loop else 0,
                samples_per_interleave, loop_point_alignment, int(trim_file))
    L.vgo_dsp_file_size.restype = C.c_int64
    L.vgo_dsp_file_size.argtypes = [C.c_void_p]
    out = np.zeros(L.vgo_dsp_file_size(C.byref(d)), dtype=np.uint8)
    co = np.ascontiguousarray(coefs, dtype=np.int16)
    g = np.ascontiguousarray(gain, dtype=np.int16) if gain is not None else None
    sh = np.ascontiguousarray(start_hist, dtype=np.int16) if start_hist is not None else None
    lc = np.ascontiguousarray(loop_ctx, dtype=np.int16) if loop_ctx is not None else None
    L.vgo_dsp_write.argtypes = [C.c_void_p] * 7
    st = L.vgo_dsp_write(C.byref(d), _ptrs(rows), co.ctypes.data, g.ctypes.data if g is not None else None,
                         sh.ctypes.data if sh is not None else None, lc.ctypes.data if lc is not None else None, out.ctypes.data)
    if st != 0:
        raise ValueError(f"vgo_dsp_write: {st}")
    return out


def dsp_parse(file):
    L = lib()
    f = _u8(file)
    info = DspInfo()
    L.vgo_dsp_parse.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    return int(L.vgo_dsp_parse(f.ctypes.data, f.size, C.byref(info))), info


def dsp_read_data(file, info: DspInfo):
    L = lib()
    f = _u8(file)
    rows = [np.zeros(sample_count_to_byte_count(info.sample_count), dtype=np.uint8) for _ in range(info.channel_count)]
    L.vgo_dsp_read_data.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    st = L.vgo_dsp_read_data(f.ctypes.data, f.size, C.byref(info), _ptrs(rows))
    if st != 0:
        raise ValueError(f"vgo_dsp_read_data: {st}")
    return rows


def adx_key(key_code=None, key_string=None):
    L = lib()
    k = (C.c_int32 * 3)()
    if key_string is not None:
        L.vgo_adx_key_from_string.argtypes = [C.c_char_p, C.c_void_p]
        L.vgo_adx_key_from_string.restype = None
        L.vgo_adx_key_from_string(key_string.encode("ascii"), k)
    else:
        L.vgo_adx_key_from_code.argtypes = [C.c_uint64, C.c_void_p]
        L.vgo_adx_key_from_code.restype = None
        L.vgo_adx_key_from_code(int(key_code), k)
    return (int(k[0]), int(k[1]), int(k[2]))


def adx_crypt(audio, key, encryption_type, frame_size):
    L = lib()
    rows = [np.array(a, dtype=np.uint8, copy=True) for a in audio]
    k = (C.c_int32 * 3)(*key)
    L.vgo_adx_crypt_channel.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    L.vgo_adx_crypt_channel.restype = None
    for c, r in enumerate(rows):
        L.vgo_adx_crypt_channel(r.ctypes.data, r.size, k, encryption_type, frame_size, c, len(rows))
    return rows


def adx_write(audio, history, sample_rate, sample_count, loop=None, alignment_samples=0, frame_size=18, version=4, type=ADX_LINEAR,
              highpass_frequency=500, encryption_type=0, key=None, trim_file=True) -> np.ndarray:
    L = lib()
    rows = [_u8(a) for a in audio]
    d = AdxDesc(len(rows), sample_rate, sample_count, int(loop is not None), loop[0] if loop else 0, loop[1] if loop else 0,
                alignment_samples, frame_size, version, type, highpass_frequency, encryption_type, int(trim_file))
    L.vgo_adx_file_size.restype = C.c_int64
    L.vgo_adx_file_size.argtypes = [C.c_void_p]
    out = np.zeros(L.vgo_adx_file_size(C.byref(d)), dtype=np.uint8)
    h = np.ascontiguousarray(history, dtype=np.int16)
    k = (C.c_int32 * 3)(*key) if key is not None else None
    L.vgo_adx_write.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    st = L.vgo_adx_write(C.byref(d), _ptrs(rows), rows[0].size, h.ctypes.data, k, out.ctypes.data)
    if st != 0:
        raise ValueError(f"vgo_adx_write: {st}")
    return out


def hca_key_tables(key_type, key_code=0):
    L = lib()
    dec, enc = np.zeros(256, np.uint8), np.zeros(256, np.uint8)
    L.vgo_hca_key_tables.argtypes = [C.c_int, C.c_uint64, C.c_void_p, C.c_void_p]
    st = L.vgo_hca_key_tables(key_type, key_code, dec.ctypes.data, enc.ctypes.data)
    if st != 0:
        raise ValueError(f"vgo_hca_key_tables: {st}")
    return dec, enc


def hca_crypt_frames(frames, frame_size, table) -> np.ndarray:
    L = lib()
    out = np.array(frames, dtype=np.uint8, copy=True).ravel()
    t = np.ascontiguousarray(table, dtype=np.uint8)
    L.vgo_hca_crypt_frame.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.vgo_hca_crypt_frame.restype = None
    for f in range(out.size // frame_size):
        L.vgo_hca_crypt_frame(out.ctypes.data + f * frame_size, frame_size, t.ctypes.data)
    return out


def hca_write(info: HcaInfo, frames, encrypt_table=None, key_type=0, comment=None, volume=1.0) -> np.ndarray:
    L = lib()
    fr = _u8(frames)
    out = np.zeros(info.header_size + info.frame_size * info.frame_count, dtype=np.uint8)
    t = np.ascontiguousarray(encrypt_table, dtype=np.uint8) if encrypt_table is not None else None
    vbits = int(np.array([volume], dtype=np.float32).view(np.uint32)[0])
    L.vgo_hca_write.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_char_p, C.c_uint32, C.c_void_p]
    st = L.vgo_hca_write(C.byref(info), fr.ctypes.data, t.ctypes.data if t is not None else None, key_type,
                         comment.encode("utf-8") if comment is not None else None, vbits, out.ctypes.data)
    if st != 0:
        raise ValueError(f"vgo_hca_write: {st}")
    return out
