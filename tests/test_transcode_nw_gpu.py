"""vgb_transcode_nw_batch on the GPU: .adx and .hca sources (and .dsp sources into PCM) into BRSTM, BCSTM, BFSTM, IDSP
and HPS byte-identical to the oracle chain (the source's reader restatement and oracle decode, SetLoop, then the target
writer's restatement from a fresh configuration), the same bytes as the two-call composition through the WAVE
converters, per-file failures found on the device, many groups in flight with mixed sources, two bound devices and the
CLI's --coded."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import adx_reader_oracle as RA
import hca_reader_oracle as RH
import loop_override_oracle as LO
import transcode_nw_oracle as W
import transcode_oracle as T

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")
ADX_KEY_STRING = "transcode nw"


# ---- source jobs ------------------------------------------------------------------------------------------------------
def _adx_job(oracle):
    """Every type, versions 3 and 4, frame sizes 9 / 18 / 33, sample counts off the 32-sample frame, loops whose start
    needs alignment and loops that do not (0 and multiples of 14336 / 28), keyed sources of both revisions."""
    key = oracle.adx_key(key_string=ADX_KEY_STRING)
    return [T.adx_file(oracle, 1, 20001, 44100, 18, 4, 3, seed=1),
            T.adx_file(oracle, 2, 33007, 48000, 18, 4, 3, (1001, 30000), seed=2),
            T.adx_file(oracle, 2, 17011, 32000, 18, 3, 2, (28 * 100, 17000), seed=3),
            T.adx_file(oracle, 4, 9013, 22050, 9, 4, 4, seed=4),
            T.adx_file(oracle, 8, 5003, 32000, 33, 4, 4, (0, 5003), seed=5),
            T.adx_file(oracle, 2, 40001, 48000, 18, 4, 3, (14336, 39999), key, 9, seed=6),
            T.adx_file(oracle, 1, 15009, 44100, 18, 4, 3, (3001, 15000), key, 8, seed=7)]


def _hca_job():
    """1, 2, 4 and 8 channels, counts off the 1024-sample frame, looping files (trimmed at their loop end) with loop
    starts on and off the alignments, keys of type 1 and 56."""
    return [T.hca_file(1, 48000, 9007, 20, quality=1), T.hca_file(2, 44100, 30011, 21, loop=(4000, 21000)),
            T.hca_file(4, 48000, 8003, 22, quality=3), T.hca_file(8, 48000, 6001, 23, quality=5),
            T.hca_file(1, 32000, 12007, 24, loop=(0, 12007), key_type=1), T.hca_file(2, 48000, 15001, 25, key_type=56),
            T.hca_file(2, 48000, 20003, 26, loop=(14336, 20000), key_type=56)]


def _dsp_job():
    return [T.dsp_file(1, 20001, 44100, seed=30), T.dsp_file(2, 9007, 48000, (1001, 8000), seed=31), T.dsp_file(3, 5003, 22050, seed=32)]


def _job(oracle, kind):
    return _adx_job(oracle) if kind == T.ADX else _hca_job() if kind == T.HCA else _dsp_job()


def _transcode(ct, files, types, opt, **kw):
    return ct.transcode_nw_batch(files, types, opt, adx_key=ct.adx_key(key_string=ADX_KEY_STRING), hca_key_code=T.HCA_KEY, **kw)


def _want(oracle, f, src, dst, codec=W.GCADPCM, endianness=0, alignment=0, trim=True, mode=LO.KEEP, s=0, e=0):
    return W.expected(f, src, dst, codec, endianness, alignment, trim, mode, s, e, oracle.adx_key(key_string=ADX_KEY_STRING), T.HCA_KEY)


def _check(oracle, files, src, outs, status, dst, **cfg):
    """Every file the product wrote is the oracle chain's; every file it refused, the oracle chain refuses.  Returns the
    number of files compared."""
    same = 0
    for k, f in enumerate(files):
        want, why = _want(oracle, f, src, dst, **cfg)
        if want is None:
            assert status[k] != 0 and outs[k] is None, (k, status[k], why)
            continue
        assert status[k] == 0, (k, status[k])
        got = outs[k]
        diff = int(np.flatnonzero(got != want)[0]) if got.size == want.size and (got != want).any() else (got.size, want.size)
        assert got.tobytes() == want.tobytes(), (k, diff)
        same += 1
    return same


DIRECTIONS = [(src, dst) for src in (T.ADX, T.HCA) for dst in W.TARGETS]


@pytest.mark.parametrize("src,dst", DIRECTIONS)
def test_every_direction_matches_the_oracle_chain(vg, oracle, src, dst):
    from vgaudio_b200 import containers as ct

    files = _job(oracle, src)
    outs, status = _transcode(ct, files, [src] * len(files), ct.convert_options(dst))
    # HPS refuses most looping files whose loop start moves (their blocks read history past the first decode)
    assert _check(oracle, files, src, outs, status, dst) >= (3 if dst == W.HPS else len(files) - 2), status


@pytest.mark.parametrize("src,dst,codec,endianness", [(T.HCA, W.BCSTM, W.PCM16, 0), (T.ADX, W.BFSTM, W.PCM8, 0), (T.DSP, W.BRSTM, W.PCM16, 0),
                                                      (T.DSP, W.BCSTM, W.PCM8, 2), (T.DSP, W.BFSTM, W.PCM16, 1), (T.HCA, W.BRSTM, W.PCM8, 0)])
def test_pcm_targets_match_the_oracle_chain(vg, oracle, src, dst, codec, endianness):
    from vgaudio_b200 import containers as ct

    files = _job(oracle, src)
    outs, status = _transcode(ct, files, [src] * len(files), W.options(ct, dst, codec, endianness))
    assert _check(oracle, files, src, outs, status, dst, codec=codec, endianness=endianness) == len(files), status


def test_configured_targets_match_the_oracle_chain(vg, oracle):
    """--loop-align, byte order and IDSP's no_trim."""
    from vgaudio_b200 import containers as ct

    adx, hca = _adx_job(oracle), _hca_job()
    for dst, cfg in [(W.BRSTM, dict(alignment=28)), (W.BCSTM, dict(alignment=1000, endianness=2)), (W.BFSTM, dict(endianness=1, alignment=14)),
                     (W.IDSP, dict(trim=False))]:
        for files, src in ((adx, T.ADX), (hca, T.HCA)):
            opt = W.options(ct, dst, **cfg)
            outs, status = _transcode(ct, files, [src] * len(files), opt)
            assert _check(oracle, files, src, outs, status, dst, **cfg) >= len(files) - 2, (dst, cfg, status)


@pytest.mark.parametrize("dst", [W.BRSTM, W.BFSTM, W.IDSP, W.HPS])
def test_loop_set_and_clear_match_the_oracle_chain(vg, oracle, dst):
    """-l on .adx sources (a start that needs alignment and one that does not), --no-loop on both sources, and -l with an
    .hca file's own points."""
    from vgaudio_b200 import containers as ct

    adx, hca = _adx_job(oracle), _hca_job()
    for files, src in ((adx, T.ADX), (hca, T.HCA)):
        converted = {}
        for mode, s, e in ((LO.SET, 1234, 5000), (LO.SET, 0, 5003), (LO.CLEAR, 0, 0)):
            loop = dict(loop=(s, e)) if mode == LO.SET else dict(no_loop=True)
            outs, status = _transcode(ct, files, [src] * len(files), ct.convert_options(dst, **loop))
            converted[(mode, s)] = _check(oracle, files, src, outs, status, dst, mode=mode, s=s, e=e)
        assert converted[(LO.CLEAR, 0)] == len(files), converted
        # an .hca source refuses points other than its own; the .adx sources take them (HPS: a start that needs no alignment)
        assert converted[(LO.SET, 1234)] + converted[(LO.SET, 0)] == 0 if src == T.HCA else converted[(LO.SET, 0)] >= 3, (src, converted)
    for own, points in ((hca[1], (4000, 21000)), (hca[4], (0, 12007))):
        outs, status = _transcode(ct, [own], [T.HCA], ct.convert_options(dst, loop=points))
        want, why = _want(oracle, own, T.HCA, dst, mode=LO.SET, s=points[0], e=points[1])
        assert (status == [0] and outs[0].tobytes() == want.tobytes()) if want is not None else status[0] != 0, (points, status, why)


def _composition(ct, files, src, opt):
    """The two-call composition through the existing converters: source -> .wav, then .wav -> target (the WAVE
    converter takes the loop setting on the WAVE side)."""
    waves, st = ct.convert_to_wave_batch(files, [src] * len(files), adx_key=ct.adx_key(key_string=ADX_KEY_STRING), hca_key_code=T.HCA_KEY)
    assert st == [0] * len(files), st
    return ct.convert_wave_batch(waves, opt)


@pytest.mark.parametrize("dst", W.TARGETS)
def test_same_bytes_as_the_two_call_composition(vg, oracle, dst):
    from vgaudio_b200 import containers as ct

    opts = [ct.convert_options(dst)]
    if dst in W.NW_TARGETS:
        opts += [W.options(ct, dst, W.PCM16, alignment=28), W.options(ct, dst, W.GCADPCM, 2, 1000)]
    for opt in opts:
        for src in (T.ADX, T.HCA, T.DSP):
            if W.is_rewrite(src, dst, opt.nw_codec_plus1 - 1 if opt.nw_codec_plus1 else W.GCADPCM):
                continue
            files = _job(oracle, src)
            want, wst = _composition(ct, files, src, opt)
            outs, status = _transcode(ct, files, [src] * len(files), opt)
            assert status == wst, (src, status, wst)
            for k in range(len(files)):
                if wst[k] == 0:
                    assert outs[k].tobytes() == want[k].tobytes(), (src, k)


def _raw(vg, files, types, opt, status=True, fill=0xAB):
    """vgb_transcode_nw_batch by hand: (return code, sizes, statuses, buffers) with buffers pre-filled with `fill`."""
    n = len(files)
    files = [np.ascontiguousarray(f, np.uint8) for f in files]
    ftab = (C.c_void_p * n)(*[f.ctypes.data for f in files])
    lens = (C.c_int64 * n)(*[f.size for f in files])
    tys = (C.c_int32 * n)(*types)
    sizes, st = (C.c_int64 * n)(), (C.c_int32 * n)()
    assert vg.lib.vgb_transcode_nw_batch(ftab, lens, tys, n, C.byref(opt), None, None, sizes, None, st, None, None) == 0
    bufs = [np.full(max(sizes[k], 1), fill, np.uint8) for k in range(n)]
    otab = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    rc = vg.lib.vgb_transcode_nw_batch(ftab, lens, tys, n, C.byref(opt), None, None, sizes, otab, st if status else None, None, None)
    return rc, list(sizes), list(st), bufs


@pytest.mark.parametrize("dst", [W.BFSTM, W.HPS])
def test_device_side_failures(vg, oracle, dst):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    good_adx = T.adx_file(oracle, 2, 8003, 48000, seed=40)
    bad_filter = T.adx_file(oracle, 2, 6001, 48000, 18, 4, 2, seed=41)
    _, h = RA.adx_parse(bad_filter)
    bad_filter[h.audio_offset + 18 * 2 * 100 + 18] |= 0x80       # Fixed type: filter 4 in frame 100 of channel 1
    good_hca = T.hca_file(2, 48000, 8003, 42)
    bad_sync = T.hca_file(2, 48000, 8003, 43)
    _, info, _ = RH.hca_parse(bad_sync)
    bad_sync[info.header_size + info.frame_size] ^= 0xff          # frame 1's sync word
    files = [good_adx, bad_filter, good_hca, bad_sync]
    types = [T.ADX, T.ADX, T.HCA, T.HCA]
    opt = ct.convert_options(dst)
    rc, sizes, st, bufs = _raw(vg, files, types, opt)
    assert rc == 0 and st[0] == st[2] == 0 and st[1] == st[3] == N.VGB_E_DATA, st
    assert sizes[1] == sizes[3] == 0
    assert (bufs[1] == 0xAB).all() and (bufs[3] == 0xAB).all()   # a refused file's buffer is not written
    assert bufs[0].tobytes() == _want(oracle, good_adx, T.ADX, dst)[0].tobytes()
    assert bufs[2].tobytes() == _want(oracle, good_hca, T.HCA, dst)[0].tobytes()
    # without status_out a refused file fails the call after the others were written
    rc, sizes, st, bufs = _raw(vg, [good_hca, bad_sync, good_adx], [T.HCA, T.HCA, T.ADX], opt, status=False)
    assert rc == N.VGB_E_DATA and sizes[1] == 0
    assert bufs[0].tobytes() == _want(oracle, good_hca, T.HCA, dst)[0].tobytes()
    assert bufs[2].tobytes() == _want(oracle, good_adx, T.ADX, dst)[0].tobytes()
    # the library is usable again
    outs, status = _transcode(ct, [good_adx], [T.ADX], opt)
    assert status == [0] and outs[0].tobytes() == _want(oracle, good_adx, T.ADX, dst)[0].tobytes()


def test_dsp_predictor_out_of_range_fails_the_call(vg, oracle):
    """A .dsp frame header with a predictor 8..15 fails the call, as in .dsp -> WAVE."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    dsp = T.dsp_file(1, 6000, 48000, seed=44)
    dsp[0x60] = 0x80 | (dsp[0x60] & 0x0F)
    rc, _, _, _ = _raw(vg, [T.dsp_file(2, 5000, 48000, seed=45), dsp], [T.DSP, T.DSP], W.options(ct, W.BRSTM, W.PCM16))
    assert rc == N.VGB_E_DATA


def _mixed(oracle):
    files = _adx_job(oracle) + _hca_job() + _dsp_job()
    types = [T.ADX] * 7 + [T.HCA] * 7 + [T.DSP] * 3
    order = np.random.default_rng(7).permutation(len(files))   # sources interleaved in the call
    return [files[i] for i in order], [types[i] for i in order]


@pytest.mark.parametrize("dst,codec", [(W.BRSTM, W.GCADPCM), (W.HPS, W.GCADPCM), (W.BCSTM, W.PCM16)])
def test_many_groups_with_mixed_sources_give_the_bytes_of_one_group(vg, oracle, dst, codec):
    from vgaudio_b200 import containers as ct

    files, types = _mixed(oracle)
    one, st_one = _transcode(ct, files, types, W.options(ct, dst, codec, group_bytes=1 << 40))
    deltas = []
    small = W.options(ct, dst, codec, group_bytes=60000)   # every file a group of its own: more groups than ways
    many, st_many = _transcode(ct, files, types, small, progress=deltas.append)
    assert st_one == st_many
    assert sum(deltas) == sum(1 for s in st_one if s == 0)   # one per file planned without error
    for k in range(len(files)):
        want, why = _want(oracle, files[k], types[k], dst, codec)
        if want is None:   # .dsp into GC-ADPCM, or an HPS file the writer refuses
            assert st_one[k] != 0, (k, why)
            continue
        assert st_one[k] == 0, (k, st_one[k])
        assert one[k].tobytes() == many[k].tobytes(), k
        assert one[k].tobytes() == want.tobytes(), k
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
    for opt in (ct.convert_options(W.BFSTM, group_bytes=1 << 20), W.options(ct, W.BRSTM, W.PCM8, group_bytes=1 << 20)):
        one, st_one = _transcode(ct, files, types, opt)
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
        try:
            two, st_two = _transcode(ct, files, types, opt)
        finally:
            N.check(vg.lib.vgb_shutdown())
            N.check(vg.lib.vgb_init(0, 0))
        assert st_one == st_two
        for k, (x, y) in enumerate(zip(one, two)):
            if x is None or y is None:
                assert x is None and y is None, k
                continue
            diff = int(np.flatnonzero(x != y)[0]) if x.size == y.size and (x != y).any() else (x.size, y.size)
            assert x.tobytes() == y.tobytes(), (opt.out_type, opt.nw_codec_plus1, k, types[k], diff)


# ---- the CLI ------------------------------------------------------------------------------------------------------------
def _cli(*args):
    return subprocess.run([CLI, *[str(a) for a in args]], capture_output=True, text=True)


def _mixed_dir(oracle, src):
    """a.wav, b.adx (revision 9, keyed), c.hca (type 56), d.dsp and e.hca; the looping ones start their loops at 0, which
    no target moves (HPS refuses most moved loops of short files)."""
    src.mkdir()
    pcm = [T.synth.channel(80 + c, 9001, 48000, degenerate=False) for c in range(2)]
    (src / "a.wav").write_bytes(oracle.wave_write16(pcm, 48000, (0, 8000)).tobytes())
    key = oracle.adx_key(key_string=ADX_KEY_STRING)
    files = dict(b=T.adx_file(oracle, 2, 10007, 48000, 18, 4, 3, (0, 10000), key, 9, seed=82),
                 c=T.hca_file(2, 48000, 7001, 83, key_type=56), d=T.dsp_file(2, 12001, 44100, (500, 11000), seed=84),
                 e=T.hca_file(1, 44100, 9003, 85, loop=(0, 9000)))
    (src / "b.adx").write_bytes(files["b"].tobytes())
    (src / "c.hca").write_bytes(files["c"].tobytes())
    (src / "d.dsp").write_bytes(files["d"].tobytes())
    (src / "e.hca").write_bytes(files["e"].tobytes())
    return pcm, key, files


@pytest.mark.parametrize("fmt,dst", [("bfstm", W.BFSTM), ("hps", W.HPS)])
def test_cli_coded_mixed_directory(tmp_path, vg, oracle, fmt, dst):
    """--coded with the input keys given: .wav through the WAVE converter, .adx and .hca transcoded, .dsp not listed
    (GC-ADPCM); without --coded exactly today's output set (the .wav file alone)."""
    src = tmp_path / "in"
    pcm, key, files = _mixed_dir(oracle, src)
    out = tmp_path / "out"
    r = _cli("-i", src, "-o", out, "--out-format", fmt, "--coded", "--in-keystring", ADX_KEY_STRING, "--in-keycode", T.HCA_KEY)
    assert r.returncode == 0, r.stdout + r.stderr
    assert sorted(os.listdir(out)) == [f"{n}.{fmt}" for n in "abce"]
    want = LO.expected_from_wave(pcm, 48000, (0, 8000), dst, LO.KEEP)[0]
    assert (out / f"a.{fmt}").read_bytes() == want.tobytes()
    for n, t in (("b", T.ADX), ("c", T.HCA), ("e", T.HCA)):
        assert (out / f"{n}.{fmt}").read_bytes() == _want(oracle, files[n], t, dst)[0].tobytes(), n
    plain = tmp_path / "plain"
    r = _cli("-i", src, "-o", plain, "--out-format", fmt, "--in-keystring", ADX_KEY_STRING, "--in-keycode", T.HCA_KEY)
    assert r.returncode == 0, r.stdout + r.stderr
    assert sorted(os.listdir(plain)) == [f"a.{fmt}"] and (plain / f"a.{fmt}").read_bytes() == want.tobytes()


def test_cli_coded_with_key_searches_and_pcm(tmp_path, vg, oracle):
    """--hca-keys finds the type-56 key (rows 8+) and --find-adx-key the revision-8 key (row 6); with -f pcm16 the .dsp
    file is listed too; -l reaches the coded inputs, and a looping .hca file refuses new points alone."""
    import adx_files as F

    src = tmp_path / "in"
    pcm, key, files = _mixed_dir(oracle, src)
    (src / "b.adx").unlink()
    planted = oracle.adx_key(key_string=F.KEY_STRING)
    adx8 = {f"t{i}": T.adx_file(oracle, ch, n, 48000, key=planted, enc_type=8, seed=90 + i) for i, (ch, n) in enumerate([(2, 20000), (1, 12000), (2, 9000)])}
    for name, img in adx8.items():
        (src / f"{name}.adx").write_bytes(img.tobytes())
    (tmp_path / "keys.txt").write_text(f"# keys\n12345\n{hex(T.HCA_KEY)}\n")
    out = tmp_path / "out"
    r = _cli("-i", src, "-o", out, "--out-format", "bcstm", "--coded", "-f", "pcm16", "--find-adx-key", "--hca-keys", tmp_path / "keys.txt")
    assert r.returncode == 0, r.stdout + r.stderr
    assert "list entry 1): 1 files" in r.stdout and "Seed - " in r.stdout, r.stdout
    assert sorted(os.listdir(out)) == ["a.bcstm", "c.bcstm", "d.bcstm", "e.bcstm", "t0.bcstm", "t1.bcstm", "t2.bcstm"]
    for n, t in (("c", T.HCA), ("d", T.DSP), ("e", T.HCA)):
        assert (out / f"{n}.bcstm").read_bytes() == _want(oracle, files[n], t, W.BCSTM, W.PCM16)[0].tobytes(), n
    given = tmp_path / "given"
    r = _cli("-i", src, "-o", given, "--out-format", "bcstm", "--coded", "-f", "pcm16", "--in-keystring", F.KEY_STRING, "--in-keycode", T.HCA_KEY)
    assert r.returncode == 0, r.stdout + r.stderr
    for name, img in adx8.items():
        want = W.expected(img, T.ADX, W.BCSTM, W.PCM16, adx_key=planted)[0].tobytes()
        assert (out / f"{name}.bcstm").read_bytes() == (given / f"{name}.bcstm").read_bytes() == want, name
    # a loop setting reaches the coded inputs; the .hca files refuse new points and fail alone
    lo = tmp_path / "lo"
    r = _cli("-i", src, "-o", lo, "--out-format", "brstm", "--coded", "--in-keystring", F.KEY_STRING, "--in-keycode", T.HCA_KEY, "-l", "1000-7000")
    assert r.returncode == 3 and "Error converting c.hca" in r.stderr and "Error converting e.hca" in r.stderr, r.stdout + r.stderr
    assert sorted(os.listdir(lo)) == ["a.brstm", "t0.brstm", "t1.brstm", "t2.brstm"]
    assert (lo / "t1.brstm").read_bytes() == W.expected(adx8["t1"], T.ADX, W.BRSTM, mode=LO.SET, start=1000, end=7000, adx_key=planted)[0].tobytes()
