"""Host-side mirror of the reference's container layer either side of the codec path (SURVEY.md 8f rank 2-4) over the
C ABI: WaveReader, DspWriter / DspReader, AdxWriter (+ CriAdxEncryption / CriAdxKey), HcaWriter (+ CriHcaEncryption /
CriHcaKey) and the CLI's batch conversion (src/VGAudio.Cli/Batch.cs).  No arithmetic here: parsing, byte movement and
key streams run in libvgaudio_b200.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _native as N

CONTAINER_DSP, CONTAINER_ADX, CONTAINER_HCA = 1, 2, 3


def _bytes_arr(b) -> np.ndarray:
    return np.frombuffer(bytes(b), dtype=np.uint8) if not isinstance(b, np.ndarray) else np.ascontiguousarray(b, dtype=np.uint8).ravel()


# ---- WAVE front end (Containers/Wave/WaveReader.cs:13-51) -------------------------------------------------------------
def wave_parse(file) -> N.VgbWaveInfo:
    """RiffParser.ParseRiff + WaveReader validation on a file image; raises VgbError(VGB_E_DATA) with the reference's
    InvalidDataException message."""
    f = _bytes_arr(file)
    info = N.VgbWaveInfo()
    N.check(N.lib.vgb_wave_parse(f.ctypes.data, f.size, C.byref(info)))
    return info


def wave_read_batch(files: Sequence) -> List[Tuple[N.VgbWaveInfo, List[np.ndarray]]]:
    """WaveReader.Read for a batch of file images: [(info, [channel int16 arrays])]."""
    arrs = [_bytes_arr(f) for f in files]
    infos = (N.VgbWaveInfo * len(arrs))()
    for i, a in enumerate(arrs):
        N.check(N.lib.vgb_wave_parse(a.ctypes.data, a.size, C.byref(infos[i])))
    rows = [np.zeros(infos[i].sample_count, dtype=np.int16) for i in range(len(arrs)) for _ in range(infos[i].channel_count)]
    ftab = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    rtab = (C.c_void_p * max(len(rows), 1))(*[r.ctypes.data for r in rows])
    lens = (C.c_int64 * max(len(arrs), 1))(*[a.size for a in arrs])
    N.check(N.lib.vgb_wave_read_batch(ftab, lens, infos, len(arrs), rtab))
    return _rows_per_file(infos, rows)


def _rows_per_file(infos, rows) -> list:
    """[(info, the info's channel_count rows)] for file-major channel rows."""
    out, r = [], 0
    for info in infos:
        out.append((info, rows[r:r + info.channel_count]))
        r += info.channel_count
    return out


# ---- DSP (Containers/Dsp/DspWriter.cs, DspReader.cs) ------------------------------------------------------------------
@dataclass
class DspFile:
    """One GcAdpcmFormat as DspWriter sees it: per channel the ADPCM bytes, 16 coefficients and, when looping, the loop
    context (PredScale, Hist1, Hist2)."""
    adpcm: Sequence[np.ndarray]
    coefs: np.ndarray            # [channels][16] int16
    sample_rate: int
    sample_count: int
    looping: bool = False
    loop_start: int = 0
    loop_end: int = 0
    loop_context: Optional[np.ndarray] = None   # [channels][3]
    gain: Optional[np.ndarray] = None
    start_hist: Optional[np.ndarray] = None     # [channels][2]
    samples_per_interleave: int = 0
    loop_point_alignment: int = 0
    trim_file: bool = True

    def desc(self) -> N.VgbDspDesc:
        return N.VgbDspDesc(len(self.adpcm), self.sample_rate, self.sample_count, int(self.looping), self.loop_start, self.loop_end,
                            self.samples_per_interleave, self.loop_point_alignment, int(not self.trim_file))


def dsp_file_size(f: DspFile) -> int:
    d = f.desc()
    size = N.lib.vgb_dsp_file_size(C.byref(d))
    if size < 0:
        N.check(int(size))
    return int(size)


def dsp_write_batch(files: Sequence[DspFile]) -> List[np.ndarray]:
    """DspWriter.GetFile for a batch."""
    n = len(files)
    descs = (N.VgbDspDesc * n)(*[f.desc() for f in files])
    rows = [np.ascontiguousarray(a, dtype=np.uint8) for f in files for a in f.adpcm]
    total = len(rows)
    coefs = np.ascontiguousarray(np.concatenate([np.asarray(f.coefs, dtype=np.int16).reshape(-1, 16) for f in files]))
    gain = np.concatenate([np.asarray(f.gain, np.int16).ravel() if f.gain is not None else np.zeros(len(f.adpcm), np.int16) for f in files])
    hist = np.concatenate([np.asarray(f.start_hist, np.int16).reshape(-1, 2) if f.start_hist is not None else np.zeros((len(f.adpcm), 2), np.int16)
                           for f in files])
    any_loop = any(f.looping for f in files)
    ctx = np.concatenate([np.asarray(f.loop_context, np.int16).reshape(-1, 3) if f.loop_context is not None else np.zeros((len(f.adpcm), 3), np.int16)
                          for f in files])
    outs = [np.zeros(dsp_file_size(f), dtype=np.uint8) for f in files]
    atab = (C.c_void_p * max(total, 1))(*[r.ctypes.data for r in rows])
    otab = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    gain, hist, ctx = np.ascontiguousarray(gain), np.ascontiguousarray(hist), np.ascontiguousarray(ctx)
    N.check(N.lib.vgb_dsp_write_batch(descs, n, atab, coefs.ctypes.data, gain.ctypes.data, hist.ctypes.data,
                                      ctx.ctypes.data if any_loop else None, otab))
    return outs


def dsp_parse(file) -> N.VgbDspInfo:
    f = _bytes_arr(file)
    info = N.VgbDspInfo()
    N.check(N.lib.vgb_dsp_parse(f.ctypes.data, f.size, C.byref(info)))
    return info


def dsp_read_batch(files: Sequence) -> List[Tuple[N.VgbDspInfo, List[np.ndarray]]]:
    """DspReader.Read for a batch: [(structure, [channel ADPCM byte arrays])]."""
    arrs = [_bytes_arr(f) for f in files]
    n = len(arrs)
    infos = (N.VgbDspInfo * n)()
    for i, a in enumerate(arrs):
        N.check(N.lib.vgb_dsp_parse(a.ctypes.data, a.size, C.byref(infos[i])))
    rows = [np.zeros(N.lib.vgb_gcadpcm_sample_count_to_byte_count(infos[i].sample_count), dtype=np.uint8)
            for i in range(n) for _ in range(infos[i].channel_count)]
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
    lens = (C.c_int64 * n)(*[a.size for a in arrs])
    rtab = (C.c_void_p * max(len(rows), 1))(*[r.ctypes.data for r in rows])
    N.check(N.lib.vgb_dsp_read_batch(ftab, lens, infos, n, rtab))
    return _rows_per_file(infos, rows)


# ---- CRI ADX (Containers/Adx/AdxWriter.cs, Codecs/CriAdx/CriAdxEncryption.cs, CriAdxKey.cs) ----------------------------
def adx_key(key_code: Optional[int] = None, key_string: Optional[str] = None) -> N.VgbAdxKey:
    k = N.VgbAdxKey()
    if key_string is not None:
        N.check(N.lib.vgb_adx_key_from_string(key_string.encode("ascii"), C.byref(k)))
    else:
        N.check(N.lib.vgb_adx_key_from_code(int(key_code), C.byref(k)))
    return k


@dataclass
class AdxFile:
    """One CriAdxFormat as AdxWriter sees it; sample_count / loop points are the unaligned PCM values."""
    audio: Sequence[np.ndarray]
    history: Sequence[int]
    sample_rate: int
    sample_count: int
    looping: bool = False
    loop_start: int = 0
    loop_end: int = 0
    alignment_samples: int = 0
    frame_size: int = 18
    version: int = 4
    type: int = 3
    highpass_frequency: int = 500
    encryption_type: int = 0
    trim_file: bool = True

    def desc(self) -> N.VgbAdxDesc:
        return N.VgbAdxDesc(len(self.audio), self.sample_rate, self.sample_count, int(self.looping), self.loop_start, self.loop_end,
                            self.alignment_samples, self.frame_size, self.version, self.type, self.highpass_frequency,
                            self.encryption_type, int(not self.trim_file))


def adx_file_size(f: AdxFile) -> int:
    d = f.desc()
    size = N.lib.vgb_adx_file_size(C.byref(d))
    if size < 0:
        N.check(int(size))
    return int(size)


def adx_write_batch(files: Sequence[AdxFile], key: Optional[N.VgbAdxKey] = None) -> List[np.ndarray]:
    n = len(files)
    descs = (N.VgbAdxDesc * n)(*[f.desc() for f in files])
    rows = [np.ascontiguousarray(a, dtype=np.uint8) for f in files for a in f.audio]
    lens = (C.c_int32 * max(len(rows), 1))(*[r.size for r in rows])
    hist = np.ascontiguousarray(np.concatenate([np.asarray(f.history, np.int16).ravel() for f in files]))
    outs = [np.zeros(adx_file_size(f), dtype=np.uint8) for f in files]
    atab = (C.c_void_p * max(len(rows), 1))(*[r.ctypes.data for r in rows])
    otab = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    N.check(N.lib.vgb_adx_write_batch(descs, n, atab, lens, hist.ctypes.data, C.byref(key) if key is not None else None, otab))
    return outs


def adx_crypt(audio: Sequence[np.ndarray], key: N.VgbAdxKey, encryption_type: int, frame_size: int) -> List[np.ndarray]:
    """CriAdxEncryption.EncryptDecrypt on copies of one file's channels."""
    rows = [np.array(a, dtype=np.uint8, copy=True) for a in audio]
    tab = (C.c_void_p * max(len(rows), 1))(*[r.ctypes.data for r in rows])
    N.check(N.lib.vgb_adx_crypt_batch(tab, len(rows), rows[0].size if rows else 0, C.byref(key), encryption_type, frame_size))
    return rows


# ---- CRI HCA (Containers/Hca/HcaWriter.cs, Codecs/CriHca/CriHcaEncryption.cs, CriHcaKey.cs) -----------------------------
def adx_parse(file) -> N.VgbAdxFileInfo:
    """AdxReader.ReadFile's header and data reads on a file image; raises VgbError(VGB_E_DATA)."""
    f = _bytes_arr(file)
    info = N.VgbAdxFileInfo()
    N.check(N.lib.vgb_adx_parse(f.ctypes.data, f.size, C.byref(info)))
    return info


def hca_key_tables(key_type: int, key_code: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    dec, enc = np.zeros(256, np.uint8), np.zeros(256, np.uint8)
    N.check(N.lib.vgb_hca_key_tables(key_type, key_code, dec.ctypes.data, enc.ctypes.data))
    return dec, enc


def hca_crypt_batch(frames: Sequence[np.ndarray], frame_size: int, key_type: int, key_code: int = 0, decrypt: bool = False) -> List[np.ndarray]:
    rows = [np.array(f, dtype=np.uint8, copy=True).ravel() for f in frames]
    counts = (C.c_int32 * max(len(rows), 1))(*[r.size // frame_size for r in rows])
    tab = (C.c_void_p * max(len(rows), 1))(*[r.ctypes.data for r in rows])
    N.check(N.lib.vgb_hca_crypt_batch(tab, counts, len(rows), frame_size, key_type, key_code, int(decrypt)))
    return rows


def hca_parse(file) -> Tuple[N.VgbHcaInfo, int]:
    """HcaReader.ReadHcaHeader on a file image: (HcaInfo, the "ciph" encryption type); raises VgbError(VGB_E_DATA)."""
    f = _bytes_arr(file)
    info, ciph = N.VgbHcaInfo(), C.c_int32(0)
    N.check(N.lib.vgb_hca_parse(f.ctypes.data, f.size, C.byref(info), C.byref(ciph)))
    return info, int(ciph.value)


def hca_write_batch(infos: Sequence[N.VgbHcaInfo], frames: Sequence[np.ndarray], key_type: int = -1, key_code: int = 0,
                    comments: Optional[Sequence[Optional[str]]] = None, volumes: Optional[Sequence[float]] = None) -> List[np.ndarray]:
    n = len(infos)
    arr = (N.VgbHcaInfo * n)(*infos)
    rows = [np.ascontiguousarray(f, dtype=np.uint8).ravel() for f in frames]
    outs = [np.zeros(infos[i].header_size + infos[i].frame_size * infos[i].frame_count, dtype=np.uint8) for i in range(n)]
    ftab = (C.c_void_p * n)(*[r.ctypes.data for r in rows])
    otab = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    ctab = None
    if comments is not None:
        ctab = (C.c_char_p * n)(*[c.encode("utf-8") if c is not None else None for c in comments])
    vol = (C.c_float * n)(*volumes) if volumes is not None else None
    N.check(N.lib.vgb_hca_write_batch(arr, n, ftab, key_type, key_code, ctab, vol, otab))
    return outs


# ---- batch conversion (src/VGAudio.Cli/Batch.cs:11-51) -----------------------------------------------------------------
def convert_options(out_type: int, **kw) -> N.VgbConvertOptions:
    o = N.VgbConvertOptions()
    o.out_type = out_type
    o.hca_key_type = -1
    for k, v in kw.items():
        if not hasattr(o, k):
            raise TypeError(f"unknown option {k}")
        setattr(o, k, v)
    return o


def _convert(call, files) -> Tuple[List[Optional[np.ndarray]], List[int]]:
    """The two passes of a batch converter call: call(ftab, lens, n, sizes, files_out, status) sizes every file with
    files_out NULL, then writes the files that are good into buffers of those sizes."""
    arrs = [_bytes_arr(f) for f in files]
    n = len(arrs)
    ftab = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in arrs])
    lens = (C.c_int64 * max(n, 1))(*[a.size for a in arrs])
    sizes = (C.c_int64 * max(n, 1))()
    status = (C.c_int32 * max(n, 1))()
    N.check(call(ftab, lens, n, sizes, None, status))
    outs = [np.zeros(sizes[i], dtype=np.uint8) if status[i] == 0 else None for i in range(n)]
    otab = (C.c_void_p * max(n, 1))(*[o.ctypes.data if o is not None else None for o in outs])
    N.check(call(ftab, lens, n, sizes, otab, status))
    return outs, [int(status[i]) for i in range(n)]


def convert_wave_batch(files: Sequence, options: N.VgbConvertOptions, progress=None) -> Tuple[List[Optional[np.ndarray]], List[int]]:
    """BatchConvert for WAVE inputs held in memory: ([output file bytes or None], [per-file status])."""
    cb = N.PROGRESS_CB(lambda user, delta: progress(delta)) if progress else None
    return _convert(lambda ftab, lens, n, sizes, otab, status: N.lib.vgb_convert_wave_batch(
        ftab, lens, n, C.byref(options), sizes, otab, status, cb if otab is not None else None, None), files)


def convert_dsp_to_wave_batch(files: Sequence) -> Tuple[List[Optional[np.ndarray]], List[int]]:
    """The decode direction of the batch job: .dsp images in, 16-bit WAVE images out (DspReader -> ToPcm16 -> WaveWriter)."""
    return _convert(N.lib.vgb_convert_dsp_to_wave_batch, files)


def convert_hca_to_wave_batch(files: Sequence, key_code: Optional[int] = None) -> Tuple[List[Optional[np.ndarray]], List[int]]:
    """The decode direction of the batch job for .hca images: HcaReader -> decrypt -> ToPcm16 -> WaveWriter.  key_code is
    the type-56 key of keyed files (None: such files fail); a file whose frames the decoder refuses fails alone."""
    code = C.c_uint64(key_code) if key_code is not None else None
    outs, status = _convert(lambda ftab, lens, n, sizes, otab, st: N.lib.vgb_convert_hca_to_wave_batch(
        ftab, lens, n, C.byref(code) if code is not None else None, sizes, otab, st), files)
    return [o if s == 0 else None for o, s in zip(outs, status)], status  # the fill pass may refuse a file's frames


def convert_adx_to_wave_batch(files: Sequence, key: Optional[N.VgbAdxKey] = None) -> Tuple[List[Optional[np.ndarray]], List[int]]:
    """The decode direction of the batch job for .adx images: AdxReader -> decrypt -> ToPcm16 -> WaveWriter.  key (from
    adx_key) decrypts files of revision 8 and 9 (None: such files fail); a file with a bad Fixed-type filter fails alone."""
    outs, status = _convert(lambda ftab, lens, n, sizes, otab, st: N.lib.vgb_convert_adx_to_wave_batch(
        ftab, lens, n, C.byref(key) if key is not None else None, sizes, otab, st), files)
    return [o if s == 0 else None for o, s in zip(outs, status)], status  # the fill pass may refuse a file's frames


def transcode_batch(files: Sequence, in_types: Sequence[int], options: N.VgbConvertOptions, adx_key: Optional[N.VgbAdxKey] = None,
                    hca_key_code: Optional[int] = None, progress=None) -> Tuple[List[Optional[np.ndarray]], List[int]]:
    """.dsp / .adx / .hca images in (in_types: CONTAINER_* per file), options.out_type out, decoded and re-encoded on the
    device: ([output file bytes or None], [per-file status]).  adx_key (from adx_key) decrypts revision 8 / 9 .adx
    sources, hca_key_code "ciph" 56 .hca sources; the output's key is in options."""
    types = (C.c_int32 * max(len(in_types), 1))(*in_types)
    code = C.c_uint64(hca_key_code) if hca_key_code is not None else None
    cb = N.PROGRESS_CB(lambda user, delta: progress(delta)) if progress else None
    outs, status = _convert(lambda ftab, lens, n, sizes, otab, st: N.lib.vgb_transcode_batch(
        ftab, lens, types, n, C.byref(options), C.byref(adx_key) if adx_key is not None else None,
        C.byref(code) if code is not None else None, sizes, otab, st, cb if otab is not None else None, None), files)
    return [o if s == 0 else None for o, s in zip(outs, status)], status  # the fill pass may refuse a file's frames
