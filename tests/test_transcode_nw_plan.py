"""vgb_transcode_nw_batch's sizing pass, on the host without a device: for .adx, .hca and .dsp sources into BRSTM,
BCSTM, BFSTM, IDSP and HPS, with every codec, byte order, loop point alignment and loop setting, the size equals the
oracle chain's (the source's reader restatement, SetLoop, then the target writer's geometry); every per-file refusal
fails its own file with its message, and the call's own refusals fail the call."""
import ctypes as C

import numpy as np
import pytest

import adx_files as F
import loop_override_oracle as LO
import transcode_nw_oracle as W
import transcode_oracle as T

ADX_KEY_STRING = "transcode nw"


def _sizing(vg, files, in_types, opt, adx_key=None, hca_key=None):
    """(sizes, statuses, messages): the sizing pass file by file, so that each message belongs to its file."""
    sizes, status, msgs = [], [], []
    for f, t in zip(files, in_types):
        f = np.ascontiguousarray(f, np.uint8)
        ftab = (C.c_void_p * 1)(f.ctypes.data)
        lens = (C.c_int64 * 1)(f.size)
        types = (C.c_int32 * 1)(t)
        sz, st = (C.c_int64 * 1)(), (C.c_int32 * 1)()
        code = C.c_uint64(hca_key) if hca_key is not None else None
        assert vg.lib.vgb_transcode_nw_batch(ftab, lens, types, 1, C.byref(opt), C.byref(adx_key) if adx_key is not None else None,
                                             C.byref(code) if code is not None else None, sz, None, st, None, None) == 0
        sizes.append(int(sz[0]))
        status.append(int(st[0]))
        msgs.append((vg.lib.vgb_last_error() or b"").decode() if st[0] else "")
    return sizes, status, msgs


def _sources(oracle, kind):
    """Short sources of one codec: 1, 2, 4 and 8 channels, looping (loop starts on and off every alignment) and not,
    sample counts that are no multiple of an ADX frame or of 1024."""
    if kind == T.ADX:
        key = oracle.adx_key(key_string=ADX_KEY_STRING)
        return [T.adx_file(oracle, 1, 5001, 44100, 18, 4, 3, seed=1),
                T.adx_file(oracle, 2, 9007, 48000, 18, 4, 3, (1001, 8000), seed=2),
                T.adx_file(oracle, 2, 7003, 32000, 18, 3, 2, (28, 7000), seed=3),
                T.adx_file(oracle, 4, 3333, 22050, 18, 3, 4, seed=4),
                T.adx_file(oracle, 8, 2011, 32000, 33, 4, 4, (0, 2011), seed=5),
                T.adx_file(oracle, 2, 6001, 48000, 18, 4, 3, (300, 5999), key, 9, seed=6)]
    if kind == T.HCA:
        return [T.hca_file(1, 44100, 5001, 9), T.hca_file(2, 48000, 9007, 10, loop=(1001, 8000)), T.hca_file(4, 22050, 3001, 11),
                T.hca_file(8, 32000, 2047, 12, key_type=1), T.hca_file(2, 48000, 4001, 13, loop=(0, 4001), key_type=56)]
    return [T.dsp_file(1, 5001, 44100, seed=14), T.dsp_file(2, 9007, 48000, (1001, 8000), seed=15), T.dsp_file(4, 3001, 22050, seed=16)]


def _keys(ct):
    return dict(adx_key=ct.adx_key(key_string=ADX_KEY_STRING), hca_key=T.HCA_KEY)


# (codec, endianness, loop point alignment) per target
CONFIGS = {W.BRSTM: [(W.GCADPCM, 0, 0), (W.GCADPCM, 0, 28), (W.PCM16, 0, 0), (W.PCM8, 0, 0)],
           W.BCSTM: [(W.GCADPCM, 0, 0), (W.GCADPCM, 2, 1000), (W.PCM16, 1, 0), (W.PCM8, 2, 0)],
           W.BFSTM: [(W.GCADPCM, 0, 0), (W.GCADPCM, 1, 14), (W.PCM16, 0, 0), (W.PCM8, 1, 0)],
           W.IDSP: [(W.GCADPCM, 0, 0)],
           W.HPS: [(W.GCADPCM, 0, 0)]}
LOOPS = [(LO.KEEP, 0, 0), (LO.SET, 700, 2000), (LO.CLEAR, 0, 0)]


@pytest.mark.parametrize("dst", W.TARGETS)
@pytest.mark.parametrize("src", [T.ADX, T.HCA, T.DSP])
def test_sizing_pass_matches_the_oracle_chain(vg, oracle, src, dst):
    from vgaudio_b200 import containers as ct

    files = _sources(oracle, src)
    keys = _keys(ct)
    checked = 0
    for codec, endianness, alignment in CONFIGS[dst]:
        for trim in ((True, False) if dst == W.IDSP else (True,)):
            for mode, s, e in LOOPS:
                loop = dict(loop=(s, e)) if mode == LO.SET else dict(no_loop=True) if mode == LO.CLEAR else {}
                opt = W.options(ct, dst, codec, endianness, alignment, trim, **loop)
                sizes, status, msgs = _sizing(vg, files, [src] * len(files), opt, keys["adx_key"], keys["hca_key"])
                for k, f in enumerate(files):
                    want, why = W.expected_size(f, src, dst, codec, alignment, trim, mode, s, e, oracle.adx_key(key_string=ADX_KEY_STRING),
                                                T.HCA_KEY)
                    ctx = (codec, endianness, alignment, trim, mode, k, status[k], msgs[k], why)
                    if want is not None:
                        assert status[k] == 0 and sizes[k] == want, ctx
                        checked += 1
                    else:
                        assert status[k] != 0 and sizes[k] == 0, ctx
                        if isinstance(why, str):
                            assert why in msgs[k], ctx
                        else:
                            assert status[k] == why, ctx
    if src != T.DSP or dst in W.NW_TARGETS:
        assert checked > 0


def test_dsp_into_gcadpcm_is_a_rewrite(vg, oracle):
    """GetFormat<GcAdpcmFormat> hands a .dsp source its own format: refused per file with the rewrite message for every
    GC-ADPCM target (IDSP and HPS whatever nw_codec_plus1 says); a PCM NintendoWare target decodes it."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    dsp = T.dsp_file(2, 5000, 48000, (100, 4000), seed=20)
    for dst, plus1 in [(W.BRSTM, 0), (W.BRSTM, 3), (W.BCSTM, 0), (W.BFSTM, 3), (W.IDSP, 0), (W.IDSP, 2), (W.HPS, 0), (W.HPS, 1)]:
        sizes, status, msgs = _sizing(vg, [dsp], [T.DSP], ct.convert_options(dst, nw_codec_plus1=plus1))
        assert status == [N.VGB_E_ARG] and sizes == [0], (dst, plus1, status)
        assert W.MSG_REWRITE in msgs[0] and msgs[0].startswith("file 0: "), msgs
    for dst in W.NW_TARGETS:
        for codec in (W.PCM16, W.PCM8):
            sizes, status, msgs = _sizing(vg, [dsp], [T.DSP], W.options(ct, dst, codec))
            assert status == [0] and sizes == [W.expected_size(dsp, T.DSP, dst, codec)[0]], msgs


def _bad_adx_loop():
    return F.header(samples=64, inserted=8, loop_count=1, loop=(1, 4, 0, 100, 0), header_size=80)


def test_per_file_rejections_carry_their_messages(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    key = oracle.adx_key(key_code=F.KEY_CODE)
    keyed_adx = T.adx_file(oracle, 2, 5000, 48000, key=key, enc_type=9, seed=30)
    keyed_hca = T.hca_file(2, 48000, 4000, 31, key_type=56)
    looping_hca = T.hca_file(2, 48000, 9000, 32, loop=(1000, 8000))
    empty_adx = F.header(samples=0, inserted=0, loop_count=0, header_size=60)
    hps_msg = "HpsWriter writes the block headers of 4k + 3 channels"
    cases = [  # (image, in_type, options, status, message fragment)
        (T.adx_file(oracle, 1, 3000, 48000), 0, ct.convert_options(W.BRSTM), N.VGB_E_ARG, "in_type 0 (VGB_CONTAINER_DSP / _ADX / _HCA)"),
        (T.adx_file(oracle, 1, 3000, 48000), 4, ct.convert_options(W.BFSTM), N.VGB_E_ARG, "in_type 4 (VGB_CONTAINER_DSP / _ADX / _HCA)"),
        (T.adx_file(oracle, 1, 3000, 48000), 7, ct.convert_options(W.HPS), N.VGB_E_ARG, "in_type 7 (VGB_CONTAINER_DSP / _ADX / _HCA)"),
        (keyed_adx, T.ADX, ct.convert_options(W.BCSTM), N.VGB_E_DATA, "encrypted ADX file (type 9) and no key"),
        (keyed_hca, T.HCA, ct.convert_options(W.IDSP), N.VGB_E_DATA, "Cannot find key to decrypt HCA file."),
        (looping_hca, T.HCA, ct.convert_options(W.BFSTM, loop=(1000, 7000)), N.VGB_E_ARG, LO.MSG_HCA_CHANGE),
        (T.hca_file(1, 48000, 3000, 33), T.HCA, ct.convert_options(W.BRSTM, loop=(0, 3000)), N.VGB_E_ARG, LO.MSG_HCA_CHANGE),
        (_bad_adx_loop(), T.ADX, ct.convert_options(W.HPS), N.VGB_E_ARG, LO.MSG_RANGE),
        (T.adx_file(oracle, 3, 3000, 48000, seed=34), T.ADX, ct.convert_options(W.HPS), N.VGB_E_ARG, hps_msg),
        (T.hca_file(7, 48000, 3000, 35), T.HCA, ct.convert_options(W.HPS), N.VGB_E_ARG, hps_msg),
        # GcAdpcmAlignment: an empty loop whose start has to move
        (T.adx_file(oracle, 2, 6000, 48000, seed=36), T.ADX, ct.convert_options(W.BRSTM, loop=(1001, 1001)), N.VGB_E_ARG,
         "an empty loop cannot fill the shift of the loop start"),
        (T.adx_file(oracle, 2, 6000, 48000, seed=36), T.ADX, ct.convert_options(W.IDSP, loop=(1001, 1001)), N.VGB_E_ARG,
         "an empty loop cannot fill the shift of the loop start"),
        (empty_adx, T.ADX, ct.convert_options(W.BFSTM), N.VGB_E_DATA, "no samples to encode"),
        (empty_adx, T.ADX, ct.convert_options(W.IDSP), N.VGB_E_DATA, "no samples to encode"),
        (empty_adx, T.ADX, ct.convert_options(W.HPS), N.VGB_E_DATA, "no samples to encode"),
        (T.adx_file(oracle, 1, 3000, 48000), T.ADX, ct.convert_options(W.BRSTM, nw_codec_plus1=5), N.VGB_E_ARG, "nw_codec_plus1 5"),
    ]
    for k, (img, t, opt, want, frag) in enumerate(cases):
        sizes, status, msgs = _sizing(vg, [img], [t], opt)
        assert status == [want] and sizes == [0], (k, status, msgs)
        assert frag in msgs[0], (k, msgs[0])
        assert msgs[0].startswith("file 0") or frag.startswith("nw_codec_plus1"), (k, msgs[0])   # an option's message names no file
    # the keyed sources with their keys, the HCA file with its own points and the empty file into PCM plan without error
    sizes, status, msgs = _sizing(vg, [keyed_adx], [T.ADX], ct.convert_options(W.BCSTM), adx_key=ct.adx_key(key_code=F.KEY_CODE))
    assert status == [0], msgs
    sizes, status, msgs = _sizing(vg, [keyed_hca], [T.HCA], ct.convert_options(W.IDSP), hca_key=T.HCA_KEY)
    assert status == [0], msgs
    sizes, status, msgs = _sizing(vg, [looping_hca], [T.HCA], ct.convert_options(W.BFSTM, loop=(1000, 8000)))
    assert status == [0] and sizes[0] == W.expected_size(looping_hca, T.HCA, W.BFSTM)[0], msgs
    sizes, status, msgs = _sizing(vg, [empty_adx], [T.ADX], W.options(ct, W.BFSTM, W.PCM16))
    assert status == [0] and sizes[0] == W.expected_size(empty_adx, T.ADX, W.BFSTM, W.PCM16)[0], (sizes, msgs)


@pytest.mark.parametrize("out_type", [0, T.DSP, T.ADX, T.HCA, 9, 13, -1])
def test_call_refuses_other_targets(vg, oracle, out_type):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    f = T.adx_file(oracle, 1, 3000, 48000)
    ftab = (C.c_void_p * 1)(f.ctypes.data)
    lens = (C.c_int64 * 1)(f.size)
    types = (C.c_int32 * 1)(T.ADX)
    sizes, st = (C.c_int64 * 1)(-7), (C.c_int32 * 1)(-7)
    opt = ct.convert_options(out_type)
    assert vg.lib.vgb_transcode_nw_batch(ftab, lens, types, 1, C.byref(opt), None, None, sizes, None, st, None, None) == N.VGB_E_ARG
    msg = vg.lib.vgb_last_error().decode()
    assert f"out_type {out_type} (VGB_CONTAINER_BRSTM / _BCSTM / _BFSTM / _IDSP / _HPS)" in msg, msg
    assert sizes[0] == -7 and st[0] == -7   # refused before any file is read
    with pytest.raises(N.VgbError):
        ct.transcode_nw_batch([f], [T.ADX], opt)


def test_null_arguments_and_bad_loop_mode(vg):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    sizes = (C.c_int64 * 1)()
    f = np.zeros(16, np.uint8)
    ftab = (C.c_void_p * 1)(f.ctypes.data)
    lens = (C.c_int64 * 1)(16)
    types = (C.c_int32 * 1)(T.ADX)
    opt = ct.convert_options(W.BFSTM)
    lib = vg.lib
    assert lib.vgb_transcode_nw_batch(ftab, lens, None, 1, C.byref(opt), None, None, sizes, None, None, None, None) == N.VGB_E_ARG
    assert lib.vgb_transcode_nw_batch(None, lens, types, 1, C.byref(opt), None, None, sizes, None, None, None, None) == N.VGB_E_ARG
    assert lib.vgb_transcode_nw_batch(ftab, None, types, 1, C.byref(opt), None, None, sizes, None, None, None, None) == N.VGB_E_ARG
    assert lib.vgb_transcode_nw_batch(ftab, lens, types, 1, None, None, None, sizes, None, None, None, None) == N.VGB_E_ARG
    assert lib.vgb_transcode_nw_batch(ftab, lens, types, 1, C.byref(opt), None, None, None, None, None, None, None) == N.VGB_E_ARG
    assert "NULL argument" in lib.vgb_last_error().decode()
    assert lib.vgb_transcode_nw_batch(ftab, lens, types, -1, C.byref(opt), None, None, sizes, None, None, None, None) == N.VGB_E_ARG
    assert lib.vgb_transcode_nw_batch(None, None, None, 0, None, None, None, None, None, None, None, None) == 0
    bad = ct.convert_options(W.BFSTM)
    bad.loop_mode = 3
    assert lib.vgb_transcode_nw_batch(ftab, lens, types, 1, C.byref(bad), None, None, sizes, None, None, None, None) == N.VGB_E_ARG
    assert "loop_mode 3" in lib.vgb_last_error().decode()


def test_sizing_pass_batch_mixes_sources(vg, oracle):
    """One call over mixed sources gives each file the size and status of its own call."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = _sources(oracle, T.ADX)[:3] + _sources(oracle, T.HCA)[:3] + _sources(oracle, T.DSP)[:2]
    types = [T.ADX] * 3 + [T.HCA] * 3 + [T.DSP] * 2
    n = len(files)
    ftab = (C.c_void_p * n)(*[f.ctypes.data for f in files])
    lens = (C.c_int64 * n)(*[f.size for f in files])
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    opt = ct.convert_options(W.BFSTM)
    assert vg.lib.vgb_transcode_nw_batch(ftab, lens, (C.c_int32 * n)(*types), n, C.byref(opt), None, None, sizes, None, status, None, None) == 0
    assert list(status)[6:] == [N.VGB_E_ARG] * 2 and list(sizes)[6:] == [0, 0]   # .dsp into GC-ADPCM
    one, st_one, _ = _sizing(vg, files[:6], types[:6], opt)
    assert list(sizes)[:6] == one and list(status)[:6] == st_one


def test_fill_pass_with_no_file_left_returns_without_a_device(vg, oracle):
    """When every file fails its sizing pass, the fill pass has nothing to transcode: it returns VGB_OK with the per-file
    statuses and touches no device."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = [T.adx_file(oracle, 2, 5000, 48000, key=oracle.adx_key(key_code=F.KEY_CODE), enc_type=9, seed=40),
             T.dsp_file(2, 5000, 48000, seed=41), T.hca_file(3, 48000, 3000, 42)]
    types = [T.ADX, T.DSP, T.HCA]
    outs, status = ct.transcode_nw_batch(files, types, ct.convert_options(W.HPS))
    assert status == [N.VGB_E_DATA, N.VGB_E_ARG, N.VGB_E_ARG] and outs == [None] * 3
    n = len(files)
    ftab = (C.c_void_p * n)(*[f.ctypes.data for f in files])
    lens = (C.c_int64 * n)(*[f.size for f in files])
    sizes, otab = (C.c_int64 * n)(), (C.c_void_p * n)()
    opt = ct.convert_options(W.HPS)
    assert vg.lib.vgb_transcode_nw_batch(ftab, lens, (C.c_int32 * n)(*types), n, C.byref(opt), None, None, sizes, otab, None, None, None) == 0
    assert list(sizes) == [0] * n


def test_cli_coded_flag_parse_errors(vg, tmp_path):
    """--coded takes a NintendoWare, IDSP or HPS --out-format only."""
    import os
    import subprocess

    cli = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vgaudio_b200", "cli", "vgaudio_batch")
    (tmp_path / "in").mkdir()
    for fmt in ("dsp", "adx", "hca", "wav"):
        r = subprocess.run([cli, "-i", str(tmp_path / "in"), "-o", str(tmp_path / "out"), "--out-format", fmt, "--coded"],
                           capture_output=True, text=True)
        assert r.returncode == 2 and "--coded takes --out-format brstm, bcstm, bfstm, idsp or hps" in r.stderr, (fmt, r.stderr)
