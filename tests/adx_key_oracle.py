"""ctypes bindings of oracle/adxkeys.c, the C restatement of VGAudio.Tools/CrackAdx/GuessAdx.cs - TEST INFRASTRUCTURE:
LoadFiles / AdxFile, the candidate lists, KeyIsValid, Run over a box and GetReencodeConfidence, in oracle/libvgoracle.so."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle


def lib() -> C.CDLL:
    return pyoracle.lib()


def _u8(b) -> np.ndarray:
    return np.frombuffer(bytes(b), dtype=np.uint8) if not isinstance(b, np.ndarray) else np.ascontiguousarray(b, dtype=np.uint8).ravel()


def adx_key_load(image, type_so_far=0):
    """LoadFiles + AdxFile on one image: (status, type, scales, start_frame, frame_size); status 0 loaded, 1 another
    revision, negative where the reference throws."""
    L = lib()
    f = _u8(image)
    t, fs, start, n = C.c_int(type_so_far), C.c_int(0), C.c_int(0), C.c_int(0)
    L.vgo_adx_key_load.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    L.vgo_adx_key_load.restype = C.c_int
    st = L.vgo_adx_key_load(f.ctypes.data, f.size, C.byref(t), C.byref(fs), C.byref(start), None, 0, C.byref(n))
    scales = np.zeros(max(n.value, 1), dtype=np.uint16)
    if st == 0:
        t2 = C.c_int(type_so_far)
        L.vgo_adx_key_load(f.ctypes.data, f.size, C.byref(t2), C.byref(fs), C.byref(start), scales.ctypes.data, scales.size, C.byref(n))
    return st, t.value, scales[:n.value] if st == 0 else None, start.value, fs.value


def adx_key_list(revision, which):
    """GuessAdx's lists: which 0 seeds, 1 multipliers, 2 increments."""
    L = lib()
    L.vgo_adx_key_list.argtypes = [C.c_int, C.c_int, C.c_void_p]
    L.vgo_adx_key_list.restype = C.c_int
    out = np.zeros(0x2000, dtype=np.int32)
    return out[:L.vgo_adx_key_list(revision, which, out.ctypes.data)].copy()


def adx_key_is_valid(revision, key, scales):
    L = lib()
    s = np.ascontiguousarray(scales, dtype=np.uint16)
    L.vgo_adx_key_is_valid.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    L.vgo_adx_key_is_valid.restype = C.c_int
    return bool(L.vgo_adx_key_is_valid(revision, (C.c_int32 * 3)(*key), s.ctypes.data, s.size))


def adx_guess_box(revision, files, box):
    """Run() over box = (i0, i1, m0, m1, c0, c1) for loaded files [(scales, start_frame)]: (sorted keys, (tried, steps,
    matches))."""
    L = lib()
    sc = [np.ascontiguousarray(s if s is not None and s.size else np.zeros(1, np.uint16), dtype=np.uint16) for s, _ in files]
    n = len(files)
    tab = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in sc])
    nf = (C.c_int * max(n, 1))(*[0 if s is None else int(s.size) for s, _ in files])
    st = (C.c_int * max(n, 1))(*[int(b) for _, b in files])
    stats = (C.c_uint64 * 3)()
    L.vgo_adx_guess_box.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int] * 6 + [C.c_void_p, C.c_int, C.c_void_p]
    L.vgo_adx_guess_box.restype = C.c_int
    cap = 4096
    while True:
        out = np.zeros(3 * cap, dtype=np.int32)
        k = L.vgo_adx_guess_box(revision, n, tab, nf, st, *box, out.ctypes.data, cap, stats)
        if k <= cap:
            break
        cap = k
    return [tuple(int(v) for v in out[3 * i:3 * i + 3]) for i in range(k)], (int(stats[0]), int(stats[1]), int(stats[2]))


def adx_key_confidence(image, key):
    """GetReencodeConfidence for one image: (status, [diff short, total short, diff full, total full])."""
    L = lib()
    f = _u8(image)
    out = (C.c_int32 * 4)()
    L.vgo_adx_key_confidence.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    L.vgo_adx_key_confidence.restype = C.c_int
    st = L.vgo_adx_key_confidence(f.ctypes.data, f.size, (C.c_int32 * 3)(*key), out)
    return st, [int(v) for v in out]
