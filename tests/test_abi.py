"""CPU tests of the C-ABI library: it loads, exports every symbol include/vgaudio_b200.h declares, the pure-integer
size helpers match the reference's KAT tables, and codec calls FAIL LOUDLY (VGB_E_CUDA) when there is no GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "vgaudio_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vgb_[a-z0-9_]+)\s*\(", text)) - {"vgb_progress_cb"})


def test_library_exports_every_declared_symbol(vg):
    from vgaudio_b200 import _native

    raw = C.CDLL(_native.LIB_PATH)
    names = declared_symbols()
    assert len(names) >= 20
    for name in names:
        assert hasattr(raw, name), f"{name} declared in the header but not exported"
        assert name in _native.SIGNATURES, f"{name} has no ctypes signature"
    assert set(_native.SIGNATURES) == set(names)


def test_abi_version(vg):
    assert vg.lib.vgb_abi_version() == 1


# GcAdpcmHelpersTests.cs:8-100 through the product's helpers (host-side integer math, no device needed)
@pytest.mark.parametrize("fn,arg,expected", [
    ("nibble_to_sample", 2, 0), ("nibble_to_sample", 19, 15), ("nibble_to_sample", 100010, 87508),
    ("sample_to_nibble", 0, 2), ("sample_to_nibble", 14, 18), ("sample_to_nibble", 87508, 100010),
    ("nibble_count_to_sample_count", 17, 14), ("nibble_count_to_sample_count", 100000, 87500),
    ("sample_count_to_nibble_count", 1, 3), ("sample_count_to_nibble_count", 87500, 100000),
    ("sample_count_to_byte_count", 1, 2), ("sample_count_to_byte_count", 15, 10),
    ("sample_count_to_byte_count", 87500, 50000), ("byte_count_to_sample_count", 8, 14),
])
def test_size_helpers(vg, fn, arg, expected):
    assert getattr(vg.gcadpcm, fn)(arg) == expected


def test_argument_errors_do_not_need_a_device(vg):
    from vgaudio_b200 import _native as N

    lens = np.array([-5], dtype=np.int32)
    tab = (C.c_void_p * 1)()
    co = np.zeros(16, dtype=np.int16)
    assert vg.lib.vgb_gcadpcm_coefs_batch(tab, lens.ctypes.data, 1, co.ctypes.data) == N.VGB_E_ARG
    assert b"negative" in vg.lib.vgb_last_error()
    assert vg.lib.vgb_gcadpcm_coefs_batch(tab, lens.ctypes.data, -1, co.ctypes.data) == N.VGB_E_ARG
    assert vg.lib.vgb_init(-1, 0) == N.VGB_E_ARG


def test_no_cpu_fallback_without_gpu(vg):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is for GPU-less hosts")
    with pytest.raises(vg.VgbError) as info:
        vg.gcadpcm.calculate_coefficients(np.zeros(100, dtype=np.int16))
    assert info.value.code == -4  # VGB_E_CUDA
    with pytest.raises(vg.VgbError):
        vg.gcadpcm.decode(np.zeros(8, dtype=np.uint8), np.zeros(16, dtype=np.int16))


def test_product_does_not_import_the_oracle():
    """Nothing under vgaudio_b200/ may reference oracle/ (the oracle is test infrastructure)."""
    pkg = os.path.join(ROOT, "vgaudio_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".hpp")):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                assert "pyoracle" not in text and "vgoracle" not in text and "libvgoracle" not in text, f


# ---- host logic that needs no device: CriHcaEncoder.Initialize (CriHcaEncoder.cs:61-114) in the library vs the oracle --------

@pytest.mark.parametrize("nch", [1, 2, 3, 4, 5, 6, 7, 8])
def test_hca_query_matches_the_oracle_over_a_parameter_grid(vg, oracle, nch):
    import ctypes as C
    from vgaudio_b200 import _native as N
    checked = 0
    for rate in (8000, 22050, 32000, 44100, 48000, 96000):
        for quality in (0, 1, 2, 3, 4, 5):
            for bitrate, limit in ((0, False), (0, True), (64000 * nch, False), (24000, True)):
                for n, loop in ((48000, None), (100000, (5000, 90000)), (2049, (2048, 2049)), (30000, (0, 30000)), (1, None)):
                    p = N.VgbHcaParams(quality, bitrate, int(limit), nch, rate, n, 1 if loop else 0, loop[0] if loop else 0,
                                       loop[1] if loop else 0)
                    info = N.VgbHcaInfo()
                    rc = vg.lib.vgb_hca_query(C.byref(p), C.byref(info))
                    op = oracle.HcaParams(quality, bitrate, int(limit), nch, rate, n, 1 if loop else 0, loop[0] if loop else 0,
                                          loop[1] if loop else 0)
                    try:
                        want = oracle.hca_init(op)
                    except ValueError:
                        assert rc != 0
                        continue
                    if want.frame_size < 8:  # "Bitrate is set too low." is raised by the library at query time
                        assert rc != 0
                        continue
                    assert rc == 0, (rate, quality, bitrate, limit, n, loop)
                    assert info.as_dict() == want.as_dict(), (rate, quality, bitrate, limit, n, loop)
                    checked += 1
    assert checked > 300


def test_seek_entry_count_helper(vg):
    f = vg.lib.vgb_gcadpcm_seek_entry_count
    assert [f(n, spe) for n, spe in ((0, 100), (1, 100), (100, 100), (101, 100), (14336 * 3 + 1, 14336), (50, 0))] == [0, 1, 1, 2, 4, 0]


def test_adx_host_helpers_match_the_oracle(vg, oracle):
    """CriAdxCodec.CalculateCoefficients and the encoded size formula: host arithmetic, no device needed."""
    import numpy as np
    out = np.zeros(2, dtype=np.int16)
    for rate in list(range(4000, 200001, 997)) + [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 192000]:
        for hp in (0, 1, 100, 500, 1000, rate // 4):
            assert vg.lib.vgb_adx_calculate_coefficients(hp, rate, out.ctypes.data) == 0
            assert out.tolist() == oracle.adx_coefficients(hp, rate).tolist(), (hp, rate)
    # the encoder's own pair (500 Hz) at every rate 1..4000: below 1000 Hz cos(2 pi 500 / rate) stops looking like a
    # high-pass filter, and at every divisor of 500 the pair is (8192, -4096)
    for rate in range(1, 4001):
        for hp in (500, rate // 2, rate):
            assert vg.lib.vgb_adx_calculate_coefficients(hp, rate, out.ctypes.data) == 0
            assert out.tolist() == oracle.adx_coefficients(hp, rate).tolist(), (hp, rate)
    L = oracle.lib()
    for n in (0, 1, 31, 32, 33, 1000, 123457):
        for padding in (0, 1, 31, 32, 100):
            for fs in (18, 34, 6):
                assert vg.lib.vgb_adx_encoded_byte_count(n, padding, fs) == L.vgo_adx_encoded_byte_count(n, padding, fs), (n, padding, fs)


def test_gc_math_helpers_equal_the_oracle_on_a_dense_range(vg, oracle):
    """GcAdpcmMath (GcAdpcmMath.cs:7-47): the library's host helpers against the oracle's restatement for every argument in a
    dense range (the oracle itself is pinned to the reference's KAT tables in test_oracle_gcadpcm.py)."""
    L = oracle.lib()
    pairs = [("vgb_gcadpcm_sample_count_to_byte_count", "vgo_gc_sample_count_to_byte_count"),
             ("vgb_gcadpcm_byte_count_to_sample_count", "vgo_gc_byte_count_to_sample_count"),
             ("vgb_gcadpcm_sample_count_to_nibble_count", "vgo_gc_sample_count_to_nibble_count"),
             ("vgb_gcadpcm_nibble_count_to_sample_count", "vgo_gc_nibble_count_to_sample_count"),
             ("vgb_gcadpcm_sample_to_nibble", "vgo_gc_sample_to_nibble"),
             ("vgb_gcadpcm_nibble_to_sample", "vgo_gc_nibble_to_sample")]
    values = list(range(0, 3000)) + [10 ** 6 + k for k in range(40)] + [2 ** 30 + k for k in range(20)]
    for ours, theirs in pairs:
        f, g = getattr(vg.lib, ours), getattr(L, theirs)
        for v in values:
            assert f(v) == g(v), (ours, v)


def test_partition_lpt_and_collective_errors_without_a_communicator(vg):
    """vgb_partition_lpt is host logic (greedy longest-first, the file -> GPU assignment of the multi-GPU batch path);
    the collectives refuse to run before vgb_nccl_init (VGB_E_STATE), and a missing NCCL is VGB_E_NCCL, never a crash."""
    import ctypes as C

    from vgaudio_b200 import _native as N

    w = np.array([10, 1, 9, 2, 8, 3, 7, 4, 6, 5, 0, 11], dtype=np.int64)
    part = np.zeros(len(w), dtype=np.int32)
    load = np.zeros(3, dtype=np.int64)
    N.check(vg.lib.vgb_partition_lpt(w.ctypes.data, len(w), 3, part.ctypes.data, load.ctypes.data))
    assert load.sum() == w.sum() and load.max() - load.min() <= 1          # 66 over 3 parts: 22 each
    assert [int(w[part == p].sum()) for p in range(3)] == load.tolist()
    N.check(vg.lib.vgb_partition_lpt(w.ctypes.data, 0, 4, None, None))
    assert vg.lib.vgb_partition_lpt(w.ctypes.data, 3, 0, part.ctypes.data, None) == N.VGB_E_ARG
    counts = np.zeros(8, dtype=np.int64)
    assert vg.lib.vgb_scatterv_dev(None, counts.ctypes.data, counts.ctypes.data, None, 0, None) == N.VGB_E_STATE
    assert vg.lib.vgb_gatherv_dev(None, None, counts.ctypes.data, counts.ctypes.data, 0, None) == N.VGB_E_STATE
    assert vg.lib.vgb_nccl_version() >= 0
    assert vg.lib.vgb_device_count() in (0, 1)  # nothing bound on a CPU box, one device after another test's vgb_init
