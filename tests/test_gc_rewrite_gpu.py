""".dsp files rewritten into BRSTM, BCSTM, BFSTM, IDSP and HPS on the device (vgb_rewrite_gc_batch) against the oracle
chain (the .dsp reader, the builder's reuse rules, the writers fed the source's ADPCM), byte for byte: every channel
count the targets take, loops already aligned and moved, a header loop context that is wrong on purpose, -l / --no-loop,
--loop-align, both byte orders, files shorter than one frame, a bad predictor, two bound devices, and the CLI's
--keep-codec.  Without an oracle: a .dsp file the converter made from WAVE rewrites into the bytes the WAVE file
converts into, because both carry the same encoder's ADPCM."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gc_rewrite_oracle as R
import loop_override_oracle as LO
from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")


def _wrong_ctx(ch):
    return [(0x17, 1234 + c, -4321 - c) for c in range(ch)]


def _files():
    """(name, image): mono, stereo and 3-channel; no loop; loops that no target moves (start 0, and a multiple of every
    alignment: 14336 * 4 = 57344 = HPS's stereo and 4-channel alignment, a multiple of 28); loops every target moves; a
    header loop context that is wrong; files shorter than one frame."""
    out = [("mono plain", R.dsp_image(1, 20011, 32000, seed=1)),
           ("stereo plain", R.dsp_image(2, 15000, 48000, seed=2)),
           ("3ch plain", R.dsp_image(3, 9001, 22050, seed=3)),
           ("stereo loop 0", R.dsp_image(2, 12000, 32000, (0, 12000), seed=4)),
           ("stereo aligned", R.dsp_image(2, 70000, 32000, (57344, 69000), seed=5)),
           ("mono moved", R.dsp_image(1, 30000, 44100, (1001, 29000), seed=6)),
           ("stereo moved", R.dsp_image(2, 40000, 32000, (5003, 40000), seed=7)),
           ("3ch moved", R.dsp_image(3, 8000, 32000, (333, 7000), seed=8)),
           ("stereo wrong ctx", R.dsp_image(2, 20000, 32000, (2002, 19000), seed=9, loop_ctx=_wrong_ctx(2))),
           ("mono wrong ctx at 0", R.dsp_image(1, 5000, 32000, (0, 5000), seed=10, loop_ctx=_wrong_ctx(1))),
           ("plain wrong ctx", R.dsp_image(2, 6000, 32000, seed=11, loop_ctx=_wrong_ctx(2))),
           ("short", R.dsp_image(1, 9, 32000, seed=12)),
           ("short stereo loop", R.dsp_image(2, 13, 32000, (2, 13), seed=13)),
           ("4ch moved", R.dsp_image(4, 9000, 32000, (100, 9000), seed=14))]
    return out


def _compare(ct, files, opt, dst, endianness=0, alignment=0, trim=True, mode=LO.KEEP, s=0, e=0):
    outs, status = ct.rewrite_gc_batch([f for _, f in files], [R.DSP] * len(files), opt)
    good = 0
    for k, (name, f) in enumerate(files):
        want, why = R.expected(f, dst, endianness, alignment, trim, mode, s, e)
        if want is None:
            assert status[k] != 0 and outs[k] is None, (name, dst, why)
            continue
        assert status[k] == 0, (name, dst, status[k])
        diff = int(np.flatnonzero(outs[k] != want)[0]) if outs[k].size == want.size and (outs[k] != want).any() else (outs[k].size, want.size)
        assert outs[k].tobytes() == want.tobytes(), (name, dst, endianness, alignment, trim, mode, s, e, diff)
        good += 1
    return good


CONFIGS = [(R.BRSTM, 0, 0, True), (R.BRSTM, 0, 28, True), (R.BCSTM, 0, 0, True), (R.BCSTM, 2, 1000, True), (R.BFSTM, 0, 0, True),
           (R.BFSTM, 1, 14, True), (R.IDSP, 0, 0, True), (R.IDSP, 0, 0, False), (R.HPS, 0, 0, True)]
LOOPS = [(LO.KEEP, 0, 0), (LO.SET, 2002, 5000), (LO.SET, 0, 3000), (LO.CLEAR, 0, 0)]


@pytest.mark.parametrize("dst,endianness,alignment,trim", CONFIGS)
def test_rewrite_matches_the_oracle(vg, oracle, dst, endianness, alignment, trim):
    from vgaudio_b200 import containers as ct

    files = _files()
    good = 0
    for mode, s, e in LOOPS:
        loop = dict(loop=(s, e)) if mode == LO.SET else dict(no_loop=True) if mode == LO.CLEAR else {}
        good += _compare(ct, files, R.options(ct, dst, endianness, alignment, trim, **loop), dst, endianness, alignment, trim, mode, s, e)
    assert good >= 2 * len(files)


def test_bad_predictor_fails_its_own_file(vg, oracle):
    from vgaudio_b200 import containers as ct

    good = R.dsp_image(2, 5000, 32000, (100, 5000), seed=20)
    bad = R.dsp_image(1, 5000, 32000, seed=21)
    bad[0x60 + 8 * 100] = 0x95  # frame 100's header: predictor 9
    for dst in R.TARGETS:
        outs, status = ct.rewrite_gc_batch([good, bad, good], [R.DSP] * 3, R.options(ct, dst))
        assert R.expected(bad, dst) == (None, R.MSG_PREDICTOR)
        assert status[1] == -2 and outs[1] is None
        assert status[0] == status[2] == 0 and outs[0].tobytes() == outs[2].tobytes() == R.expected(good, dst)[0].tobytes()
    with pytest.raises(vg._native.VgbError) as e:  # without status_out the call fails
        files = [np.ascontiguousarray(f, np.uint8) for f in (good, bad)]
        ftab = (C.c_void_p * 2)(*[f.ctypes.data for f in files])
        lens = (C.c_int64 * 2)(*[f.size for f in files])
        types = (C.c_int32 * 2)(R.DSP, R.DSP)
        sizes = (C.c_int64 * 2)()
        opt = R.options(ct, R.BFSTM)
        vg._native.check(vg.lib.vgb_rewrite_gc_batch(ftab, lens, types, 2, C.byref(opt), sizes, None, None))
        outs = [np.zeros(sizes[i], np.uint8) for i in range(2)]
        otab = (C.c_void_p * 2)(*[o.ctypes.data for o in outs])
        vg._native.check(vg.lib.vgb_rewrite_gc_batch(ftab, lens, types, 2, C.byref(opt), sizes, otab, None))
    assert "predictors outside 0..7" in str(e.value)


def test_many_groups_and_two_bound_devices(vg, oracle):
    """A mixed call of many small groups, on one context and sharded over two bound contexts of device 0."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = [f for _, f in _files()] * 3
    bad = R.dsp_image(2, 3000, 32000, seed=22)
    bad[0x60 * 2 + 8 * 5] = 0xC1
    files.insert(7, bad)
    for dst in (R.BFSTM, R.IDSP, R.HPS):
        opt = R.options(ct, dst, group_bytes=1 << 16)
        one, st_one = ct.rewrite_gc_batch(files, [R.DSP] * len(files), opt)
        for k, f in enumerate(files):
            want, why = R.expected(f, dst)
            assert (st_one[k] == 0) == (want is not None), (dst, k, why)
            if want is not None:
                assert one[k].tobytes() == want.tobytes(), (dst, k)
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
        try:
            two, st_two = ct.rewrite_gc_batch(files, [R.DSP] * len(files), opt)
        finally:
            N.check(vg.lib.vgb_shutdown())
            N.check(vg.lib.vgb_init(0, 0))
        assert st_two == st_one
        assert all((a is None and b is None) or a.tobytes() == b.tobytes() for a, b in zip(one, two)), dst


def test_rewrite_of_a_converted_dsp_equals_the_wave_conversion(vg, oracle):
    """A .dsp file the converter made from a WAVE file carries the encoder's ADPCM, history-0 start contexts and gain 0,
    so where no target moves its loop its rewrite is the WAVE file's conversion.  Left out: IDSP files that loop from 0,
    whose .dsp header holds the context DspWriter recalculated there, (Adpcm[0], 0, 0), which IDSP keeps where the WAVE
    conversion writes (0, 0, 0)."""
    import gc_container_writer_oracle as GW
    from vgaudio_b200 import containers as ct

    specs = [(1, 20000, None), (2, 30000, None), (2, 70000, (57344, 70000)), (1, 30000, (28672, 30000)), (2, 8000, (0, 8000))]
    waves = []
    for k, (ch, n, loop) in enumerate(specs):
        rows = [synth.channel(300 + 2 * k + c, n) for c in range(ch)]
        waves.append(oracle.wave_write16(rows, 32000, loop))
    dsps, st = ct.convert_wave_batch(waves, ct.convert_options(R.DSP))
    assert st == [0] * len(waves)
    compared = 0
    for dst in R.TARGETS:
        def taken(ch, loop):
            if loop is None:
                return True
            if dst == R.IDSP:
                return loop[0] > 0 and loop[0] % GW.IDSP_ALIGNMENT == 0
            if dst == R.HPS:
                return loop[0] % GW.byte_count_to_sample_count(GW.hps_channel_size(ch)) == 0
            return loop[0] % 14336 == 0

        keep = [k for k, (ch, _, loop) in enumerate(specs) if taken(ch, loop)]
        opt = R.options(ct, dst)
        via_wave, st_w = ct.convert_wave_batch([waves[k] for k in keep], opt)
        rewritten, st_r = ct.rewrite_gc_batch([dsps[k] for k in keep], [R.DSP] * len(keep), opt)
        assert st_w == st_r == [0] * len(keep)
        for j, k in enumerate(keep):
            assert rewritten[j].tobytes() == via_wave[j].tobytes(), (dst, k)
            compared += 1
    assert compared >= 15


# ---- the CLI ------------------------------------------------------------------------------------------------------------
def _cli(*args):
    return subprocess.run([CLI, *[str(a) for a in args]], capture_output=True, text=True, timeout=300)


def test_cli_keep_codec(tmp_path, oracle):
    src = tmp_path / "dsps"
    src.mkdir()
    images = {"a.dsp": R.dsp_image(2, 40000, 32000, (5003, 40000), seed=30), "b.dsp": R.dsp_image(1, 9000, 32000, seed=31),
              "c.dsp": R.dsp_image(2, 6000, 32000, (0, 6000), seed=32, loop_ctx=_wrong_ctx(2))}
    for name, img in images.items():
        (src / name).write_bytes(img.tobytes())
    for fmt, dst in (("bfstm", R.BFSTM), ("idsp", R.IDSP), ("hps", R.HPS)):
        out = tmp_path / fmt
        r = _cli("-i", src, "-o", out, "--out-format", fmt, "--keep-codec")
        assert r.returncode == 0, r.stderr
        assert f"{len(images)} files converted, 0 failed" in r.stdout
        for name, img in images.items():
            want, why = R.expected(img, dst)
            assert (out / name).with_suffix("." + fmt).read_bytes() == want.tobytes(), (fmt, name)
    # -l and --loop-align reach the rewrite as they reach every other call
    out = tmp_path / "brstm"
    r = _cli("-i", src, "-o", out, "--out-format", "brstm", "--keep-codec", "-l", "28-5000", "--loop-align", "56")
    assert r.returncode == 0, r.stderr
    for name, img in images.items():
        want, _ = R.expected(img, R.BRSTM, alignment=56, mode=LO.SET, start=28, end=5000)
        assert (out / name).with_suffix(".brstm").read_bytes() == want.tobytes(), name
    # without the flag a folder of .dsp files is not taken, as before; the flag takes GC-ADPCM NintendoWare, IDSP and HPS only
    out = tmp_path / "none"
    r = _cli("-i", src, "-o", out, "--out-format", "bfstm")
    assert r.returncode == 0 and "0 files converted, 0 failed" in r.stdout and not out.exists(), (r.stdout, r.stderr)
    r = _cli("-i", src, "-o", out, "--out-format", "bfstm", "--coded")
    assert r.returncode == 0 and "0 files converted, 0 failed" in r.stdout, (r.stdout, r.stderr)
    for bad in (["--out-format", "dsp"], ["--out-format", "bfstm", "-f", "pcm16"], ["--out-format", "wav"]):
        r = _cli("-i", src, "-o", out, *bad, "--keep-codec")
        assert r.returncode == 2 and "--keep-codec takes" in r.stderr, bad
