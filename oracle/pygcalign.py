"""ctypes wrapper of vgo_gc_align (oracle/gcalign.c, inside oracle/libvgoracle.so) — TEST INFRASTRUCTURE.

Only tests/ and tools/align_bench.py's oracle arm may import this.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import pyoracle


def _lib() -> C.CDLL:
    L = pyoracle.lib()
    if not getattr(L, "_align_ready", False):
        L.vgo_gc_align.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]
        L.vgo_gc_align.restype = C.c_int
        L._align_ready = True
    return L


def gc_align(multiple, loop_start, loop_end, adpcm=None, coefs=None):
    """GcAdpcmAlignment(multiple, loopStart, loopEnd, adpcm, coefs): (status, (needed, loop_start_aligned,
    sample_count_aligned), adpcm_aligned or None, pcm_aligned or None).  status 0, -1 (argument / overflow / endless tail
    loop) or -2 (a predictor 8..15 below loop_end); without adpcm only the geometry is computed."""
    L = _lib()
    geom = np.zeros(3, dtype=np.int32)
    rc = L.vgo_gc_align(multiple, loop_start, loop_end, None, -1, None, geom.ctypes.data, None, None)
    if adpcm is None or rc != 0 or not geom[0]:
        return rc, tuple(int(v) for v in geom), None, None
    adpcm = np.ascontiguousarray(adpcm, dtype=np.uint8)
    coefs = np.ascontiguousarray(coefs, dtype=np.int16)
    out_a = np.zeros(pyoracle.sample_count_to_byte_count(int(geom[2])), dtype=np.uint8)
    out_p = np.zeros(int(geom[2]), dtype=np.int16)
    rc = L.vgo_gc_align(multiple, loop_start, loop_end, adpcm.ctypes.data, len(adpcm), coefs.ctypes.data, geom.ctypes.data,
                        out_a.ctypes.data, out_p.ctypes.data)
    if rc != 0:
        return rc, tuple(int(v) for v in geom), None, None
    return rc, tuple(int(v) for v in geom), out_a, out_p
