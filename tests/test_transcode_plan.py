"""vgb_transcode_batch's sizing pass, on the host without a device: for every direction between .dsp, .adx and .hca the
size equals the oracle chain's output (the source's reader restatement, then the target writer's geometry), and every
per-file rejection fails its own file with its message."""
import ctypes as C
import struct

import numpy as np
import pytest

import adx_files as F
import transcode_oracle as T

DIRECTIONS = [(T.DSP, T.ADX), (T.DSP, T.HCA), (T.ADX, T.DSP), (T.ADX, T.HCA), (T.HCA, T.DSP), (T.HCA, T.ADX)]


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
        assert vg.lib.vgb_transcode_batch(ftab, lens, types, 1, C.byref(opt), C.byref(adx_key) if adx_key is not None else None,
                                          C.byref(code) if code is not None else None, sz, None, st, None, None) == 0
        sizes.append(int(sz[0]))
        status.append(int(st[0]))
        msgs.append((vg.lib.vgb_last_error() or b"").decode() if st[0] else "")
    return sizes, status, msgs


def _sources(oracle, kind):
    """Short source images of one codec: mono, stereo, 3 and 8 channels, looping and not."""
    if kind == T.DSP:
        return [T.dsp_file(1, 5000, 44100, seed=1), T.dsp_file(2, 9000, 48000, (1001, 8000), seed=2),
                T.dsp_file(3, 3000, 22050, seed=3), T.dsp_file(8, 2000, 32000, (7, 1999), seed=4)]
    if kind == T.ADX:
        return [T.adx_file(oracle, 1, 5000, 44100, seed=5), T.adx_file(oracle, 2, 9000, 48000, loop=(1001, 8000), seed=6),
                T.adx_file(oracle, 3, 3000, 22050, 18, 3, 4, seed=7), T.adx_file(oracle, 8, 2000, 32000, 33, 4, 2, loop=(7, 1999), seed=8)]
    return [T.hca_file(1, 44100, 5000, 9), T.hca_file(2, 48000, 9000, 10, loop=(1001, 8000)), T.hca_file(3, 22050, 3000, 11),
            T.hca_file(8, 32000, 2000, 12, key_type=1)]


@pytest.mark.parametrize("src,dst", DIRECTIONS)
def test_sizing_pass_matches_the_oracle_chain(vg, oracle, src, dst):
    from vgaudio_b200 import containers as ct

    files = _sources(oracle, src)
    sizes, status, msgs = _sizing(vg, files, [src] * len(files), ct.convert_options(dst, hca_quality=2))
    for k, f in enumerate(files):
        pcm, n, loop, rate = T.source_pcm(f, src)
        assert status[k] == 0, (k, msgs[k])
        assert sizes[k] == T.target_size(len(pcm), n, loop, rate, dst), k


def test_sizing_pass_batch_mixes_sources_and_needs_no_device(vg, oracle):
    from vgaudio_b200 import containers as ct

    files = _sources(oracle, T.DSP)[:2] + _sources(oracle, T.ADX)[:2] + _sources(oracle, T.HCA)[:2]
    types = [T.DSP] * 2 + [T.ADX] * 2 + [T.HCA] * 2
    n = len(files)
    ftab = (C.c_void_p * n)(*[f.ctypes.data for f in files])
    lens = (C.c_int64 * n)(*[f.size for f in files])
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    opt = ct.convert_options(ct.CONTAINER_HCA, hca_quality=2)
    assert vg.lib.vgb_transcode_batch(ftab, lens, (C.c_int32 * n)(*types), n, C.byref(opt), None, None, sizes, None, status, None, None) == 0
    from vgaudio_b200 import _native as N

    assert list(status) == [0, 0, 0, 0, N.VGB_E_ARG, N.VGB_E_ARG]   # the last two are HCA already
    assert sizes[4] == sizes[5] == 0
    one, _, _ = _sizing(vg, files[:4], types[:4], opt)
    assert list(sizes)[:4] == one


def _bad_adx_loop():
    return F.header(samples=64, inserted=8, loop_count=1, loop=(1, 4, 0, 100, 0), header_size=80)


def test_per_file_rejections_carry_their_messages(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    key = oracle.adx_key(key_code=F.KEY_CODE)
    keyed_adx = T.adx_file(oracle, 2, 5000, 48000, key=key, enc_type=9, seed=20)
    keyed_hca = T.hca_file(2, 48000, 4000, 21, key_type=56)
    short_dsp = T.dsp_file(2, 5000, 48000, seed=22)[:-100].copy()
    nine = T.adx_file(oracle, 9, 3000, 48000, seed=23)
    empty_dsp = T.dsp_file(1, 0, 48000, seed=24)
    cases = [  # (image, in_type, out_type, status, message fragment)
        (T.dsp_file(1, 3000, 48000), T.DSP, T.DSP, N.VGB_E_ARG, "rewriting a container in its own codec is not performed"),
        (keyed_hca, T.HCA, T.HCA, N.VGB_E_ARG, "rewriting a container in its own codec is not performed"),
        (T.dsp_file(1, 3000, 48000), 0, T.ADX, N.VGB_E_ARG, "in_type 0"),
        (T.dsp_file(1, 3000, 48000), 4, T.ADX, N.VGB_E_ARG, "in_type 4"),
        (keyed_adx, T.ADX, T.DSP, N.VGB_E_DATA, "encrypted ADX file (type 9) and no key"),
        (keyed_hca, T.HCA, T.ADX, N.VGB_E_DATA, "Cannot find key to decrypt HCA file."),
        (_bad_adx_loop(), T.ADX, T.HCA, N.VGB_E_ARG, "Loop points must be less than the number of samples and non-negative."),
        (short_dsp, T.DSP, T.HCA, N.VGB_E_DATA, "Specified length is greater than the number of bytes remaining"),
        (np.frombuffer(b"\x80\x01junk", np.uint8).copy(), T.ADX, T.DSP, N.VGB_E_DATA, "File doesn't have ADX signature"),
        (np.frombuffer(b"HCA\x00\x02\x00", np.uint8).copy(), T.HCA, T.DSP, N.VGB_E_DATA, "not enough data for an HCA header"),
        (nine, T.ADX, T.HCA, N.VGB_E_ARG, "HCA channel count must be 8 or below"),  # vgb_hca_query's message, as for WAVE
        (empty_dsp, T.DSP, T.ADX, N.VGB_E_DATA, "no samples"),  # version 4 reads pcm[0]
    ]
    for k, (img, t, out, want, frag) in enumerate(cases):
        opt = ct.convert_options(out, hca_quality=2)
        sizes, status, msgs = _sizing(vg, [img], [t], opt)
        assert status == [want] and sizes == [0], (k, status, msgs)
        assert frag in msgs[0], (k, msgs[0])
    # the same keyed sources with their keys plan without error
    sizes, status, msgs = _sizing(vg, [keyed_adx], [T.ADX], ct.convert_options(T.DSP), adx_key=ct.adx_key(key_code=F.KEY_CODE))
    assert status == [0], msgs
    sizes, status, msgs = _sizing(vg, [keyed_hca], [T.HCA], ct.convert_options(T.DSP), hca_key=T.HCA_KEY)
    assert status == [0], msgs
    # a version-3 target takes the empty .dsp file (AdxWriter writes a header and one footer frame)
    sizes, status, msgs = _sizing(vg, [empty_dsp], [T.DSP], ct.convert_options(T.ADX, adx_version=3))
    assert status == [0] and sizes[0] == 32 + 4 + 18, (sizes, msgs)


def test_adx_rate_zero_or_below_follows_the_direct_path(vg, oracle):
    """An .adx file with a sample rate <= 0 decodes in the reference; its PCM goes on to the target with that rate, where
    a WAVE round trip would store it in a RIFF header first.  GC-ADPCM takes any rate; HCA's encoder refuses it."""
    from vgaudio_b200 import containers as ct

    for rate in (0, -44100):
        img = T.adx_file(oracle, 2, 4000, 48000, seed=30)
        img[8:12] = np.frombuffer(struct.pack(">i", rate), np.uint8)
        pcm, n, loop, r = T.source_pcm(img, T.ADX)
        assert r == rate
        sizes, status, msgs = _sizing(vg, [img], [T.ADX], ct.convert_options(T.DSP))
        assert status == [0] and sizes[0] == T.target_size(2, n, loop, rate, T.DSP), msgs
        sizes, status, msgs = _sizing(vg, [img], [T.ADX], ct.convert_options(T.HCA, hca_quality=2))
        assert status[0] != 0 and sizes == [0]


def test_null_arguments_and_bad_out_type(vg):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    sizes = (C.c_int64 * 1)()
    f = np.zeros(16, np.uint8)
    ftab = (C.c_void_p * 1)(f.ctypes.data)
    lens = (C.c_int64 * 1)(16)
    types = (C.c_int32 * 1)(T.DSP)
    opt = ct.convert_options(T.ADX)
    assert vg.lib.vgb_transcode_batch(ftab, lens, None, 1, C.byref(opt), None, None, sizes, None, None, None, None) == N.VGB_E_ARG
    assert vg.lib.vgb_transcode_batch(None, None, None, 0, None, None, None, None, None, None, None, None) == 0
    bad = ct.convert_options(7)
    assert vg.lib.vgb_transcode_batch(ftab, lens, types, 1, C.byref(bad), None, None, sizes, None, None, None, None) == N.VGB_E_ARG


def test_fill_pass_with_no_file_left_returns_without_a_device(vg, oracle):
    """When every file fails its sizing pass, the fill pass has nothing to transcode: it returns VGB_OK with the per-file
    statuses and touches no device."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = [T.adx_file(oracle, 2, 5000, 48000, key=oracle.adx_key(key_code=F.KEY_CODE), enc_type=9, seed=40),
             T.dsp_file(2, 5000, 48000, seed=41)[:-100].copy(), T.hca_file(1, 48000, 3000, 42)]
    outs, status = ct.transcode_batch(files, [T.ADX, T.DSP, T.HCA], ct.convert_options(T.HCA, hca_quality=2))
    assert status == [N.VGB_E_DATA, N.VGB_E_DATA, N.VGB_E_ARG] and outs == [None] * 3
    n = len(files)
    ftab = (C.c_void_p * n)(*[f.ctypes.data for f in files])
    lens = (C.c_int64 * n)(*[f.size for f in files])
    types = (C.c_int32 * n)(T.ADX, T.DSP, T.HCA)
    sizes, otab = (C.c_int64 * n)(), (C.c_void_p * n)()
    opt = ct.convert_options(T.HCA, hca_quality=2)
    assert vg.lib.vgb_transcode_batch(ftab, lens, types, n, C.byref(opt), None, None, sizes, otab, None, None, None) == 0
    assert list(sizes) == [0] * n
