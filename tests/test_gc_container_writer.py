"""IDSP and HPS writers on the host: the oracle's files read back through the test-side readers, the sizing pass of
vgb_convert_wave_batch against the oracle's file sizes, and every per-file refusal with its message."""
import ctypes as C
import itertools

import numpy as np
import pytest

import vgaudio_b200 as vg
from oracle import pyoracle as O
from vgaudio_b200 import _native as N
from vgaudio_b200 import containers as ct

import gc_container_writer_oracle as W

CHANNELS = (1, 2, 3, 5, 6, 7)  # 3, 5, 6, 7: 0x10000 / ch is not a multiple of 0x20


def _pcm(ch, n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return [(np.sin(t * (0.01 + 0.003 * c)) * 9000 + rng.normal(0, 300, n)).clip(-32768, 32767).astype(np.int16) for c in range(ch)]


def hps_shift_loop(ch, n):
    """A loop whose move makes HpsWriter read a block's history past the first decode: a loop start just past a block
    boundary (the largest shift), the loop end at the last sample and more than one block behind the loop block."""
    a = W.byte_count_to_sample_count(W.hps_channel_size(ch))
    return (a + 1, n) if n > 3 * a else None


def loops(n, ch=1):
    """no loop; start 0; aligned for both writers (a multiple of 28 and of the HPS alignment); unaligned; an end before
    the last sample; and, where the file is long enough, the HPS history case"""
    a = W.byte_count_to_sample_count(W.hps_channel_size(ch))
    out = [None, (0, n)]
    if n > 200:
        out += [(101, n - 7), (n // 3, n), (0, n - 20)]
    if n > a + 50:
        out.append((a, n - 3))
    h = hps_shift_loop(ch, n)
    if h:
        out.append(h)
    return out


def size_pass(files, opts):
    n = len(files)
    arrs = [np.ascontiguousarray(f, dtype=np.uint8) for f in files]
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
    lens = (C.c_int64 * n)(*[a.size for a in arrs])
    sizes = (C.c_int64 * n)()
    status = (C.c_int32 * n)()
    N.check(N.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(opts), sizes, None, status, None, None))
    return list(sizes), list(status)


def oracle_size(kind, ch, n, loop, trim=True):
    if kind == W.IDSP:
        st = W.idsp_check(ch, n, loop, trim)
        return (0, st) if st else (W.idsp_geometry(ch, n, loop, trim)[1]["file_size"], 0)
    st = W.hps_check(ch, n, loop)
    return (0, st) if st else (W.hps_geometry(ch, n, loop)[1]["file_size"], 0)


def test_oracle_files_parse_back():
    for ch, n in ((1, 300000), (2, 100), (2, 60000), (5, 20000), (6, 14336)):
        for loop in loops(n, ch):
            pcm = _pcm(ch, n, ch)
            st, f = W.write_idsp(pcm, 32000, loop)
            assert st == 0
            info = W.parse_idsp(f)
            floop = W._alignment(W.IDSP_ALIGNMENT, loop)[1]
            assert (info["channels"], info["rate"], info["block"]) == (ch, 32000, 16)
            assert (info["loop_start"], info["loop_end"]) == (floop if loop else (0, 0))
            assert info["sample_count"] == (floop[1] if loop else n)
            for c in range(ch):
                assert info["chans"][c]["coefs"] == [int(v) for v in O.calculate_coefficients(pcm[c])]
                assert info["chans"][c]["looping"] == (1 if loop else 0)
                if not loop or loop[0] == 0:
                    assert info["chans"][c]["loop"] == (0, 0, 0)  # rule 1: no decode for loop start 0
            st, f = W.write_hps(pcm, 32000, loop)
            if st:  # only the history case refuses these
                g = W.hps_geometry(ch, n, loop)[1]
                assert st == W.E_ARG and g["needed"] and any(b["start"] - 1 >= n for b in g["blocks"])
                continue
            h = W.parse_hps(f)
            g = W.hps_geometry(ch, n, loop)[1]
            assert [b["offset"] for b in h["blocks"]] == [b["offset"] for b in g["blocks"]]
            assert [b["next"] for b in h["blocks"]] == [b["next"] for b in g["blocks"]]
            assert h["looping"] == bool(loop)
            assert h["sample_count"] == g["sc"]
            if loop:
                assert h["loop_start"] == W._alignment(W.byte_count_to_sample_count(W.hps_channel_size(ch)), loop)[1][0]
                assert h["blocks"][-1]["next"] == h["blocks"][g["loop_block"]]["offset"]
            else:
                assert h["blocks"][-1]["next"] == -1
            # the block contexts' predictor/scale is the frame header at each block's start
            for b in h["blocks"]:
                for c in range(ch):
                    assert b["ctx"][c][0] & 0xFF == b["ctx"][c][0]


def test_hps_history_case_is_real():
    """the shift case: the loop moves, and a block behind the loop block starts past the unaligned sample count"""
    ch, n = 2, 200000
    loop = hps_shift_loop(ch, n)
    g = W.hps_geometry(ch, n, loop)[1]
    assert g["needed"] and len(g["blocks"]) > g["loop_block"] + 1
    assert any(b["start"] - 1 >= n for b in g["blocks"])
    assert W.hps_check(ch, n, loop) == W.E_ARG
    # the same loop without the moved end past n: a loop start on the boundary keeps the file
    assert W.hps_check(ch, n, (loop[0] - 1, n)) == 0


@pytest.mark.parametrize("kind", (W.IDSP, W.HPS))
def test_sizing_pass_matches_the_oracle(kind):
    for trim in (True, False):
        files, want = [], []
        for ch in CHANNELS:
            for n in (1, 13, 14336, 14336 * 2 + 77, 70000 if ch > 1 else 200000):
                for loop in loops(n, ch):
                    files.append(O.wave_write16(_pcm(ch, n, n), 48000, loop))
                    want.append(oracle_size(kind, ch, n, loop, trim))
        sizes, status = size_pass(files, ct.convert_options(kind, no_trim=0 if trim else 1))
        assert sizes == [w[0] for w in want]
        assert status == [w[1] for w in want]
        assert any(s == 0 for s in sizes) == (kind == W.HPS)


def _refusal(kind, wave, **kw):
    sizes, status = size_pass([wave], ct.convert_options(kind, **kw))
    return sizes[0], status[0], vg.lib.vgb_last_error().decode()


def _empty_wave():
    b = bytearray(O.wave_write16([np.zeros(0, np.int16)], 32000).tobytes()) + b"junk" + bytes(8)
    b[4:8] = (len(b) - 8).to_bytes(4, "little")
    return np.frombuffer(bytes(b), dtype=np.uint8)


def test_per_file_refusals_name_their_cause():
    for kind in (W.IDSP, W.HPS):
        assert _refusal(kind, _empty_wave())[1:] == (N.VGB_E_DATA, "file 0: no samples to encode")
        size, status, err = _refusal(kind, O.wave_write16([np.zeros(4, np.int16)] * 256, 32000))
        assert (size, status) == (0, N.VGB_E_ARG) and "256 channels (at most 255" in err
        # the nw_* options are ignored
        pcm = _pcm(2, 20000, 3)
        assert _refusal(kind, O.wave_write16(pcm, 32000, (100, 19000)), nw_codec_plus1=1, nw_loop_point_alignment=7)[:2] == \
            oracle_size(kind, 2, 20000, (100, 19000))
    size, status, err = _refusal(W.HPS, O.wave_write16(_pcm(3, 100, 1), 32000))
    assert (size, status) == (0, N.VGB_E_ARG) and "4k + 3 channels" in err
    n = 200000
    size, status, err = _refusal(W.HPS, O.wave_write16(_pcm(2, n, 1), 32000, hps_shift_loop(2, n)))
    assert (size, status) == (0, N.VGB_E_ARG) and "IndexOutOfRangeException" in err
    assert W.idsp_check(2, n, hps_shift_loop(2, n)) == 0  # IDSP reads no block history


def test_out_type_range():
    wave = O.wave_write16(_pcm(1, 100, 1), 32000)
    for bad in (0, 9):
        with pytest.raises(Exception):
            size_pass([wave], ct.convert_options(bad))
        assert "_IDSP / _HPS" in vg.lib.vgb_last_error().decode()


def test_transcode_still_refuses_idsp_and_hps():
    p = _pcm(1, 100, 1)[0]
    co = O.calculate_coefficients(p)
    dsp = O.dsp_write([O.encode(p, co)], np.stack([co]), 32000, 100)
    for kind in (W.IDSP, W.HPS):
        with pytest.raises(Exception):
            ct.transcode_batch([dsp], [ct.CONTAINER_DSP], ct.convert_options(kind))
        assert "out_type" in vg.lib.vgb_last_error().decode()
