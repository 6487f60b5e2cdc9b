"""vgb_rewrite_gc_batch's sizing pass, on the host without a device: .dsp files into BRSTM, BCSTM, BFSTM, IDSP and HPS
with every byte order, loop point alignment, trim setting and loop setting give the oracle chain's size; every per-file
refusal fails its own file with its message, in the reference's order; the call's own refusals fail the call."""
import ctypes as C

import numpy as np
import pytest

import gc_rewrite_oracle as R
import loop_override_oracle as LO


def _sizing(vg, files, opt, in_types=None):
    """(sizes, statuses, messages): the sizing pass file by file, so that each message belongs to its file."""
    sizes, status, msgs = [], [], []
    for k, f in enumerate(files):
        f = np.ascontiguousarray(f, np.uint8)
        ftab = (C.c_void_p * 1)(f.ctypes.data)
        lens = (C.c_int64 * 1)(f.size)
        types = (C.c_int32 * 1)(in_types[k] if in_types else R.DSP)
        sz, st = (C.c_int64 * 1)(), (C.c_int32 * 1)()
        assert vg.lib.vgb_rewrite_gc_batch(ftab, lens, types, 1, C.byref(opt), sz, None, st) == 0
        sizes.append(int(sz[0]))
        status.append(int(st[0]))
        msgs.append((vg.lib.vgb_last_error() or b"").decode() if st[0] else "")
    return sizes, status, msgs


def _sources():
    """Short .dsp files: 1, 2, 3 and 4 channels; looping with loop starts on and off every target's alignment, from 0,
    and not looping."""
    return [R.dsp_image(1, 5001, 44100, seed=1),
            R.dsp_image(2, 9007, 48000, (1001, 8000), seed=2),
            R.dsp_image(3, 3001, 22050, (28 * 20, 3001), seed=3),
            R.dsp_image(4, 4100, 32000, (0, 4100), seed=4),
            R.dsp_image(2, 20000, 32000, (14336, 19000), seed=5),
            R.dsp_image(1, 13, 32000, seed=6)]


CONFIGS = {R.BRSTM: [(0, 0), (0, 28)], R.BCSTM: [(0, 0), (2, 1000)], R.BFSTM: [(0, 0), (1, 14)], R.IDSP: [(0, 0)], R.HPS: [(0, 0)]}
LOOPS = [(LO.KEEP, 0, 0), (LO.SET, 700, 2000), (LO.SET, 1001, 3001), (LO.CLEAR, 0, 0)]


def _loop_kw(mode, s, e):
    return dict(loop=(s, e)) if mode == LO.SET else dict(no_loop=True) if mode == LO.CLEAR else {}


@pytest.mark.parametrize("dst", R.TARGETS)
def test_sizing_pass_matches_the_oracle_chain(vg, oracle, dst):
    from vgaudio_b200 import containers as ct

    files = _sources()
    checked = refused = 0
    for endianness, alignment in CONFIGS[dst]:
        for trim in ((True, False) if dst == R.IDSP else (True,)):
            for mode, s, e in LOOPS:
                opt = R.options(ct, dst, endianness, alignment, trim, **_loop_kw(mode, s, e))
                sizes, status, msgs = _sizing(vg, files, opt)
                for k, f in enumerate(files):
                    size, why = R.expected_size(f, dst, alignment, trim, mode, s, e)
                    if size is None:
                        assert status[k] != 0 and sizes[k] == 0, (k, dst, mode, why)
                        if isinstance(why, str):
                            assert why in msgs[k], (msgs[k], why)
                        else:
                            assert status[k] == why, (k, status[k], why, msgs[k])
                        refused += 1
                    else:
                        assert status[k] == 0 and sizes[k] == size, (k, dst, endianness, alignment, trim, mode, sizes[k], size, msgs[k])
                        checked += 1
    assert checked >= 8 * len(CONFIGS[dst]) and refused >= 1


def test_per_file_refusals_in_order(vg, oracle):
    """in_type, then the reader, then the loop setting, then the target: each file fails alone with its own message."""
    from vgaudio_b200 import containers as ct

    good = R.dsp_image(2, 3000, 32000, (500, 2500), seed=7)
    short = np.ascontiguousarray(good[:0x60 * 2 + 10])
    three = R.dsp_image(3, 3000, 32000, seed=8)
    empty = R.dsp_image(1, 0, 32000, seed=9)
    files = [good, good, short, good, three, empty]
    types = [R.DSP, 2, R.DSP, R.DSP, R.DSP, R.DSP]
    opt = R.options(ct, R.HPS)
    sizes, status, msgs = _sizing(vg, files[:3] + files[4:], opt, types[:3] + types[4:])
    assert status[0] == 0 and sizes[0] == R.expected_size(good, R.HPS)[0]
    assert status[1] == -1 and "in_type 2" in msgs[1] and R.MSG_IN_TYPE in msgs[1]
    assert status[2] == -2 and "enough data" in msgs[2]
    assert status[3] == -1 and "4k + 3 channels" in msgs[3]
    assert status[4] == -2 and "no samples" in msgs[4]
    # the loop setting before the target: a loop end past the samples fails even a 3-channel HPS file with SetLoop's message
    sizes, status, msgs = _sizing(vg, [three, good], R.options(ct, R.HPS, loop=(0, 5000)))
    assert status == [-1, -1] and all(LO.MSG_RANGE in m for m in msgs)
    sizes, status, msgs = _sizing(vg, [good], R.options(ct, R.BRSTM, loop=(2000, 1000)))
    assert status == [-1] and LO.MSG_ORDER in msgs[0]


def test_hps_history_refusal_follows_the_channels_decode(vg, oracle):
    """A moved HPS loop with a block past the unaligned samples: refused when the writer's channels hold a decode (-l
    moved the loop away from the header's), written with history 0 when the header's context survived."""
    from vgaudio_b200 import containers as ct

    looping = R.dsp_image(2, 60000, 32000, (1000, 60000), seed=10)
    plain = R.dsp_image(2, 60000, 32000, seed=11)
    sizes, status, msgs = _sizing(vg, [looping], R.options(ct, R.HPS))
    assert status == [0] and sizes[0] == R.expected_size(looping, R.HPS)[0]
    sizes, status, msgs = _sizing(vg, [looping, plain], R.options(ct, R.HPS, loop=(1000, 60000)))
    assert status[0] == 0 and sizes[0] == R.expected_size(looping, R.HPS, mode=LO.SET, start=1000, end=60000)[0]
    assert status[1] == -1 and "reads its history past" in msgs[1]
    assert R.expected_size(plain, R.HPS, mode=LO.SET, start=1000, end=60000) == (None, R.E_ARG)


@pytest.mark.parametrize("out_type", [0, R.DSP, 2, 3, 9, 100])
def test_bad_out_type_fails_the_call(vg, oracle, out_type):
    from vgaudio_b200 import containers as ct

    with pytest.raises(vg._native.VgbError) as e:
        ct.rewrite_gc_batch([R.dsp_image(1, 100, 32000)], [R.DSP], R.options(ct, out_type))
    assert e.value.code == -1 and "out_type" in str(e.value)


@pytest.mark.parametrize("codec", [1, 2, 4])
def test_a_codec_other_than_gcadpcm_fails_the_call(vg, oracle, codec):
    from vgaudio_b200 import containers as ct

    with pytest.raises(vg._native.VgbError) as e:
        ct.rewrite_gc_batch([R.dsp_image(1, 100, 32000)], [R.DSP], ct.convert_options(R.BFSTM, nw_codec_plus1=codec))
    assert e.value.code == -1 and "nw_codec_plus1" in str(e.value)
    # GC-ADPCM named explicitly is the default
    sizes, status, _ = _sizing(vg, [R.dsp_image(1, 100, 32000)], ct.convert_options(R.BFSTM, nw_codec_plus1=3))
    assert status == [0] and sizes[0] == R.expected_size(R.dsp_image(1, 100, 32000), R.BFSTM)[0]


def test_loop_setting_refusals_fail_the_call(vg, oracle):
    from vgaudio_b200 import containers as ct

    opt = R.options(ct, R.IDSP)
    opt.loop_mode = 7
    with pytest.raises(vg._native.VgbError):
        ct.rewrite_gc_batch([R.dsp_image(1, 100, 32000)], [R.DSP], opt)


def test_null_arguments_and_empty_calls(vg, oracle):
    from vgaudio_b200 import containers as ct

    opt = R.options(ct, R.BCSTM)
    assert vg.lib.vgb_rewrite_gc_batch(None, None, None, 0, C.byref(opt), None, None, None) == 0
    assert vg.lib.vgb_rewrite_gc_batch(None, None, None, -1, C.byref(opt), None, None, None) == -1
    f = np.ascontiguousarray(R.dsp_image(1, 100, 32000), np.uint8)
    ftab = (C.c_void_p * 1)(f.ctypes.data)
    lens = (C.c_int64 * 1)(f.size)
    sz = (C.c_int64 * 1)()
    assert vg.lib.vgb_rewrite_gc_batch(ftab, lens, None, 1, C.byref(opt), sz, None, None) == -1
