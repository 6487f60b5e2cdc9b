"""vgb_transcode_batch on the GPU: every direction between .dsp, .adx and .hca byte-identical to the oracle chain (the
source's reader restatement and oracle decode, then the oracle's encoder and writer from a fresh configuration), the
same bytes as the two-call composition through the WAVE converters, per-file failures found on the device, many groups
in flight with mixed sources, two bound devices and the CLI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import adx_files as F
import adx_reader_oracle as RA
import hca_reader_oracle as RH
import transcode_oracle as T

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")
DIRECTIONS = [(T.DSP, T.ADX), (T.DSP, T.HCA), (T.ADX, T.DSP), (T.ADX, T.HCA), (T.HCA, T.DSP), (T.HCA, T.ADX)]
ADX_KEY_STRING = "transcode"


# ---- source jobs ------------------------------------------------------------------------------------------------------
def _dsp_job(oracle):
    """1, 2, 3 and 8 channels, looping and not; loop starts whose ADX Linear alignment is and is not a multiple of 8
    (the .adx target's `lead` rows and its padding)."""
    return [T.dsp_file(1, 20000, 44100, seed=1), T.dsp_file(2, 33000, 48000, (1001, 30000), seed=2),
            T.dsp_file(3, 7000, 22050, seed=3), T.dsp_file(8, 5000, 32000, (7, 4999), seed=4),
            T.dsp_file(2, 16000, 48000, (3000, 15000), seed=5),   # alignment 8: the lead path
            T.dsp_file(1, 12345, 24000, (64, 12000), seed=6),     # alignment 0: version 4 writes pcm[0] as History
            T.dsp_file(2, 1, 48000, seed=7)]


def _adx_job(oracle, key):
    """Every type, versions 3 and 4, frame sizes 9 / 18 / 33, looping sources with inserted samples, keyed sources of
    both revisions (one key), an empty file and a head frame that yields no sample."""
    files = []
    for i, (ch, fs, version, type) in enumerate([(1, 18, 4, 3), (2, 18, 4, 2), (2, 18, 3, 4), (3, 18, 3, 3), (4, 9, 4, 3),
                                                 (5, 33, 4, 4), (8, 18, 4, 4)]):
        files.append(T.adx_file(oracle, ch, 3000 + 1700 * i, 48000 if i % 2 else 44100, fs, version, type, seed=10 * i))
    for i, (ch, fs, version) in enumerate([(1, 18, 4), (2, 18, 4), (2, 18, 3), (3, 11, 4)]):
        files.append(T.adx_file(oracle, ch, 40000, 32000, fs, version, 3, (3001 + 7 * i, 35000), seed=50 + i))
    files.append(T.adx_file(oracle, 2, 20000, 48000, 18, 4, 3, (1234, 18000), key, 9, seed=60))
    files.append(T.adx_file(oracle, 1, 15000, 44100, 18, 4, 3, None, key, 8, seed=61))
    files.append(F.header(samples=0, inserted=0, loop_count=0, header_size=60))  # empty
    return files


def _hca_job(oracle):
    """1, 2, 3 and 8 channels, qualities, a looping file (trimmed at its loop end), keys of type 1 and 56, an ATH curve."""
    return [T.hca_file(1, 48000, 9000, 20, quality=1), T.hca_file(2, 44100, 30000, 21, loop=(4000, 21000)),
            T.hca_file(3, 48000, 8000, 22, quality=3), T.hca_file(8, 48000, 6000, 23, quality=5),
            T.hca_file(1, 32000, 12000, 24, loop=(0, 12000), key_type=1), T.hca_file(2, 48000, 15000, 25, key_type=56),
            T.hca_file(2, 22050, 9000, 26, ath=True)]


def _job(oracle, kind):
    if kind == T.DSP:
        return _dsp_job(oracle)
    if kind == T.ADX:
        return _adx_job(oracle, oracle.adx_key(key_string=ADX_KEY_STRING))
    return _hca_job(oracle)


def _transcode(ct, files, types, opt, **kw):
    return ct.transcode_batch(files, types, opt, adx_key=ct.adx_key(key_string=ADX_KEY_STRING), hca_key_code=T.HCA_KEY, **kw)


def _check(files, src, outs, status, dst, **target):
    """Every file the product converted is the oracle chain's; every file it refused, the oracle chain cannot write."""
    for k, f in enumerate(files):
        pcm = T.source_pcm(f, src, adx_key=T.O.adx_key(key_string=ADX_KEY_STRING), hca_key=T.HCA_KEY)
        assert pcm is not None, k
        if status[k] != 0:
            with pytest.raises(Exception):
                T.target_file(*pcm, dst, **target)
            continue
        want = T.target_file(*pcm, dst, **target)
        assert outs[k].tobytes() == want.tobytes(), (k, int(np.flatnonzero(outs[k][:min(want.size, outs[k].size)] != want[:outs[k].size])[0])
                                                     if outs[k].size == want.size else (outs[k].size, want.size))


@pytest.mark.parametrize("src,dst", DIRECTIONS)
def test_every_direction_matches_the_oracle_chain(vg, oracle, src, dst):
    from vgaudio_b200 import containers as ct

    files = _job(oracle, src)
    outs, status = _transcode(ct, files, [src] * len(files), ct.convert_options(dst, hca_quality=2))
    good = [k for k, s in enumerate(status) if s == 0]
    assert len(good) >= len(files) - 1, status   # only an empty source may be refused by its target
    _check(files, src, outs, status, dst)


def test_keyed_and_configured_outputs_match_the_oracle_chain(vg, oracle):
    """ADX type 8 / 9 keys, version 3, Fixed type and 33-byte frames; HCA type-56 and type-0 keys."""
    from vgaudio_b200 import containers as ct

    kc = oracle.adx_key(key_code=0x123456789A)
    dsp, hca, adx = _dsp_job(oracle)[:5], _hca_job(oracle)[:5], _adx_job(oracle, oracle.adx_key(key_string=ADX_KEY_STRING))[:9]
    adx_cases = [
        (dict(adx_has_key=1, adx_key_seed=kc[0], adx_key_mult=kc[1], adx_key_inc=kc[2], adx_encryption_type=9), dict(enc_type=9, adx_key=kc)),
        (dict(adx_has_key=1, adx_key_seed=kc[0], adx_key_mult=kc[1], adx_key_inc=kc[2], adx_encryption_type=8), dict(enc_type=8, adx_key=kc)),
        (dict(adx_version=3, adx_frame_size=34, adx_type=2), dict(version=3, frame_size=34, type=2)),
        (dict(adx_type=4, adx_filter_plus1=1), dict(type=4, filter=0)),
    ]
    for opts, target in adx_cases:
        for files, src in ((dsp, T.DSP), (hca, T.HCA)):
            outs, status = _transcode(ct, files, [src] * len(files), ct.convert_options(T.ADX, **opts))
            assert status == [0] * len(files), (opts, status)
            _check(files, src, outs, status, T.ADX, **target)
    for key_type in (56, 0):
        opt = ct.convert_options(T.HCA, hca_quality=2, hca_key_type=key_type, hca_key_code=0xCC55463930DBE1AB)
        for files, src in ((dsp, T.DSP), (adx, T.ADX)):
            outs, status = _transcode(ct, files, [src] * len(files), opt)
            assert status == [0] * len(files), (key_type, status)
            _check(files, src, outs, status, T.HCA, hca_key_type=key_type, hca_key_code=0xCC55463930DBE1AB)


def _composition(ct, files, src, opt):
    """The two-call composition through the existing converters: source -> .wav, then .wav -> target."""
    if src == T.DSP:
        waves, st = ct.convert_dsp_to_wave_batch(files)
    elif src == T.ADX:
        waves, st = ct.convert_adx_to_wave_batch(files, ct.adx_key(key_string=ADX_KEY_STRING))
    else:
        waves, st = ct.convert_hca_to_wave_batch(files, key_code=T.HCA_KEY)
    assert st == [0] * len(files), st
    return ct.convert_wave_batch(waves, opt)


@pytest.mark.parametrize("dst", [T.DSP, T.ADX, T.HCA])
def test_same_bytes_as_the_two_call_composition(vg, oracle, dst):
    from vgaudio_b200 import containers as ct

    opts = [ct.convert_options(dst, hca_quality=2)]
    if dst == T.ADX:
        opts.append(ct.convert_options(dst, adx_version=3, adx_frame_size=20, adx_type=4))
    if dst == T.DSP:
        opts.append(ct.convert_options(dst, dsp_samples_per_interleave=14 * 100, dsp_loop_point_alignment=28, no_trim=1))
    for opt in opts:
        for src in (T.DSP, T.ADX, T.HCA):
            if src == dst:
                continue
            files = [f for f in _job(oracle, src) if T.source_pcm(f, src, T.O.adx_key(key_string=ADX_KEY_STRING), T.HCA_KEY)[1] > 0]
            want, wst = _composition(ct, files, src, opt)
            outs, status = _transcode(ct, files, [src] * len(files), opt)
            assert status == wst, (src, status, wst)
            for k in range(len(files)):
                if wst[k] == 0:
                    assert outs[k].tobytes() == want[k].tobytes(), (src, k)


def _raw(vg, files, types, opt, status=True, fill=0xAB):
    """vgb_transcode_batch by hand: (return code, sizes, statuses, buffers) with buffers pre-filled with `fill`."""
    n = len(files)
    files = [np.ascontiguousarray(f, np.uint8) for f in files]
    ftab = (C.c_void_p * n)(*[f.ctypes.data for f in files])
    lens = (C.c_int64 * n)(*[f.size for f in files])
    tys = (C.c_int32 * n)(*types)
    sizes, st = (C.c_int64 * n)(), (C.c_int32 * n)()
    assert vg.lib.vgb_transcode_batch(ftab, lens, tys, n, C.byref(opt), None, None, sizes, None, st, None, None) == 0
    bufs = [np.full(max(sizes[k], 1), fill, np.uint8) for k in range(n)]
    otab = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    rc = vg.lib.vgb_transcode_batch(ftab, lens, tys, n, C.byref(opt), None, None, sizes, otab, st if status else None, None, None)
    return rc, list(sizes), list(st), bufs


def test_device_side_failures(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    good_adx = T.adx_file(oracle, 2, 8000, 48000, seed=30)
    bad_filter = T.adx_file(oracle, 2, 6000, 48000, 18, 4, 2, seed=31)
    _, h = RA.adx_parse(bad_filter)
    bad_filter[h.audio_offset + 18 * 2 * 100 + 18] |= 0x80       # Fixed type: filter 4 in frame 100 of channel 1
    good_hca = T.hca_file(2, 48000, 8000, 32)
    bad_sync = T.hca_file(2, 48000, 8000, 33)
    _, info, _ = RH.hca_parse(bad_sync)
    bad_sync[info.header_size + info.frame_size] ^= 0xff          # frame 1's sync word
    files = [good_adx, bad_filter, good_hca, bad_sync]
    types = [T.ADX, T.ADX, T.HCA, T.HCA]
    opt = ct.convert_options(T.DSP)
    rc, sizes, st, bufs = _raw(vg, files, types, opt)
    assert rc == 0 and st[0] == st[2] == 0 and st[1] == st[3] == N.VGB_E_DATA, st
    assert sizes[1] == sizes[3] == 0
    assert (bufs[1] == 0xAB).all() and (bufs[3] == 0xAB).all()   # a refused file's buffer is not written
    assert bufs[0].tobytes() == T.expected(good_adx, T.ADX, T.DSP).tobytes()
    assert bufs[2].tobytes() == T.expected(good_hca, T.HCA, T.DSP).tobytes()
    # HCA target: the encoder's status of a refused file's garbage is not an error of the call
    rc, sizes, st, bufs = _raw(vg, [bad_filter, good_adx], [T.ADX, T.ADX], ct.convert_options(T.HCA, hca_quality=1))
    assert rc == 0 and st == [N.VGB_E_DATA, 0], st
    # without status_out a refused file fails the call after the others were written
    rc, sizes, st, bufs = _raw(vg, [good_adx, bad_filter], [T.ADX, T.ADX], opt, status=False)
    assert rc == N.VGB_E_DATA and sizes[1] == 0
    assert bufs[0].tobytes() == T.expected(good_adx, T.ADX, T.DSP).tobytes()
    # a GC-ADPCM predictor 8..15 fails the call
    dsp = T.dsp_file(1, 6000, 48000, seed=34)
    dsp[0x60] = 0x80 | (dsp[0x60] & 0x0F)
    rc, _, _, _ = _raw(vg, [T.dsp_file(2, 5000, 48000, seed=35), dsp], [T.DSP, T.DSP], ct.convert_options(T.HCA, hca_quality=2))
    assert rc == N.VGB_E_DATA
    # the library is usable again
    outs, status = _transcode(ct, [good_adx], [T.ADX], opt)
    assert status == [0] and outs[0].tobytes() == T.expected(good_adx, T.ADX, T.DSP).tobytes()


def _mixed(oracle):
    files = _dsp_job(oracle)[:5] + _adx_job(oracle, oracle.adx_key(key_string=ADX_KEY_STRING))[:11] + _hca_job(oracle)
    types = [T.DSP] * 5 + [T.ADX] * 11 + [T.HCA] * len(_hca_job(oracle))
    order = np.random.default_rng(5).permutation(len(files))   # sources interleaved in the call
    return [files[i] for i in order], [types[i] for i in order]


@pytest.mark.parametrize("dst", [T.DSP, T.ADX, T.HCA])
def test_many_groups_with_mixed_sources_give_the_bytes_of_one_group(vg, oracle, dst):
    from vgaudio_b200 import containers as ct

    files, types = _mixed(oracle)
    opt = ct.convert_options(dst, hca_quality=2, group_bytes=1 << 40)
    one, st_one = _transcode(ct, files, types, opt)
    small = ct.convert_options(dst, hca_quality=2, group_bytes=40000)   # every file a group of its own: more groups than ways
    deltas = []
    many, st_many = _transcode(ct, files, types, small, progress=deltas.append)
    assert st_one == st_many
    assert sum(deltas) == sum(1 for t in types if t != dst)   # one per file planned without error
    for k in range(len(files)):
        if types[k] == dst:
            assert st_one[k] != 0
            continue
        assert st_one[k] == 0, (k, st_one[k])
        assert one[k].tobytes() == many[k].tobytes(), k
    # VGB_CONVERT_SERIAL: one way, each group finished before the next starts
    os.environ["VGB_CONVERT_SERIAL"] = "1"
    try:
        serial, st_serial = _transcode(ct, files, types, small)
    finally:
        del os.environ["VGB_CONVERT_SERIAL"]
    assert st_serial == st_one and all(a is None and b is None or a.tobytes() == b.tobytes() for a, b in zip(serial, one))


def test_two_bound_devices_give_the_same_bytes(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files, types = _mixed(oracle)
    opt = ct.convert_options(T.ADX, group_bytes=1 << 20)
    one, st_one = _transcode(ct, files, types, opt)
    N.check(vg.lib.vgb_shutdown())
    N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
    try:
        two, st_two = _transcode(ct, files, types, opt)
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    assert st_one == st_two
    assert all(a is None and b is None or a.tobytes() == b.tobytes() for a, b in zip(one, two))


def test_cli_transcodes_a_mixed_directory(tmp_path, vg, oracle):
    """--out-format hca with --keycode (the output's key) and --in-keystring (the .adx sources' key): .wav files go
    through the WAVE converter, .dsp and .adx files are transcoded, .hca files are not listed."""
    src, dst = tmp_path / "in", tmp_path / "out"
    src.mkdir()
    key = oracle.adx_key(key_string=ADX_KEY_STRING)
    pcm = [T.synth.channel(80 + c, 9000, 48000, degenerate=False) for c in range(2)]
    (src / "a.wav").write_bytes(oracle.wave_write16(pcm, 48000, (100, 8000)).tobytes())
    dsp = T.dsp_file(2, 12000, 44100, (500, 11000), seed=81)
    (src / "b.dsp").write_bytes(dsp.tobytes())
    adx = T.adx_file(oracle, 2, 10000, 48000, 18, 4, 3, None, key, 9, seed=82)
    (src / "c.adx").write_bytes(adx.tobytes())
    (src / "d.hca").write_bytes(T.hca_file(1, 48000, 5000, 83).tobytes())
    code = 0xCC55463930DBE1AB
    r = subprocess.run([CLI, "-i", str(src), "-o", str(dst), "--out-format", "hca", "--keycode", str(code),
                        "--in-keystring", ADX_KEY_STRING], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert sorted(os.listdir(dst)) == ["a.hca", "b.hca", "c.hca"]
    target = dict(hca_key_type=56, hca_key_code=code)
    assert (dst / "a.hca").read_bytes() == T.target_file(pcm, 9000, (100, 8000), 48000, T.HCA, **target).tobytes()
    assert (dst / "b.hca").read_bytes() == T.expected(dsp, T.DSP, T.HCA, **target).tobytes()
    assert (dst / "c.hca").read_bytes() == T.expected(adx, T.ADX, T.HCA, adx_key=key, **target).tobytes()


def _all_failing(oracle):
    """Coded files that all fail the sizing pass: a keyed .adx file without its key, a truncated .dsp file, and a .hca
    file given for an .hca output."""
    keyed = T.adx_file(oracle, 2, 5000, 48000, key=oracle.adx_key(key_string=ADX_KEY_STRING), enc_type=8, seed=90)
    short = T.dsp_file(2, 5000, 48000, seed=91)[:-100].copy()
    return [keyed, short, T.hca_file(1, 48000, 3000, 92)], [T.ADX, T.DSP, T.HCA]


def test_a_fill_pass_where_every_file_failed_sizing(vg, oracle, tmp_path):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files, types = _all_failing(oracle)
    opt = ct.convert_options(T.HCA, hca_quality=2)
    outs, status = ct.transcode_batch(files, types, opt)   # both passes, with no key for the .adx file
    assert status == [N.VGB_E_DATA, N.VGB_E_DATA, N.VGB_E_ARG] and outs == [None] * 3
    rc, sizes, st, _ = _raw(vg, files, types, opt, status=False)   # without status_out too
    assert rc == 0 and sizes == [0, 0, 0]
    # the CLI reports the files and goes on
    src, dst = tmp_path / "in", tmp_path / "out"
    src.mkdir()
    for name, f in zip(("a.adx", "b.dsp"), files):
        (src / name).write_bytes(f.tobytes())
    r = subprocess.run([CLI, "-i", str(src), "-o", str(dst), "--out-format", "hca"], capture_output=True, text=True)
    assert r.returncode == 3, r.stdout + r.stderr   # some files failed
    assert "0 files converted, 2 failed" in r.stdout and "Error converting a.adx" in r.stderr and "Error converting b.dsp" in r.stderr
    assert not dst.exists() or os.listdir(dst) == []


def test_more_files_than_one_hca_decode_launch_takes(vg, oracle):
    """65 600 short .hca files in one group's worth of bytes: groups hold at most 4096 files, so no HCA decode launch gets
    more streams than it takes (65535)."""
    from vgaudio_b200 import containers as ct

    one = T.hca_file(1, 48000, 1500, 93)
    want = T.expected(one, T.HCA, T.DSP)
    files = [one] * 65600
    outs, status = ct.transcode_batch(files, [T.HCA] * len(files), ct.convert_options(T.DSP, group_bytes=1 << 40))
    assert status == [0] * len(files)
    assert all(o.tobytes() == want.tobytes() for o in outs)
