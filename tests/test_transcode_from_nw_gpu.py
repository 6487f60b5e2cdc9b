"""vgb_transcode_from_nw_batch on the GPU: every NintendoWare stream, wave and prefetch reader, IDSP and HPS into every
coded target byte-identical to the oracle chain (the reader restatement, SetLoop, then the target writer's restatement
from a fresh configuration) and to the two-call composition through WAVE; looping files into Linear .adx whose lead is
0, a multiple of 8 and not, for GC-ADPCM and PCM rows in one group; predictor faults that fail their own file; many
small groups; two bound devices; and the CLI's --nw-inputs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import adx_files as F
import loop_override_oracle as LO
import nw_files as NF
import nw_wave_files as NWF
import transcode_from_nw_oracle as X

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")

# every cell of the codec table: (target, codec of a NintendoWare target)
CELLS = [(X.DSP, X.GCADPCM), (X.ADX, X.GCADPCM), (X.HCA, X.GCADPCM), (X.BRSTM, X.GCADPCM), (X.BCSTM, X.PCM16), (X.BFSTM, X.PCM8),
         (X.BCSTM, X.GCADPCM), (X.BRSTM, X.PCM8), (X.BFSTM, X.PCM16), (X.IDSP, X.GCADPCM), (X.HPS, X.GCADPCM)]


def _sources(oracle):
    return X.sources(oracle, scale=3)


def _check(files, types, outs, status, dst, codec=X.GCADPCM, **cfg):
    """Every file the product wrote is the oracle chain's; every file it refused, the chain refuses.  Returns the
    (source codec, in_type) of every file compared."""
    done = set()
    for k, (f, t) in enumerate(zip(files, types)):
        want, why = X.expected(f, t, dst, codec, **cfg)
        if want is None:
            assert status[k] != 0 and outs[k] is None, (k, t, status[k], why)
            continue
        assert status[k] == 0, (k, t, status[k])
        got = outs[k]
        diff = int(np.flatnonzero(got != want)[0]) if got.size == want.size and (got != want).any() else (got.size, want.size)
        assert got.tobytes() == want.tobytes(), (k, t, diff)
        done.add((X.source_codec(f, t), t))
    return done


@pytest.mark.parametrize("dst,codec", CELLS)
def test_every_cell_matches_the_oracle_chain(vg, oracle, dst, codec):
    from vgaudio_b200 import containers as ct

    srcs = _sources(oracle)
    files, types = [f for _, f, _ in srcs], [t for t, _, _ in srcs]
    outs, status = ct.transcode_from_nw_batch(files, types, X.options(ct, dst, codec))
    done = _check(files, types, outs, status, dst, codec)
    # every source codec that is not the target's, from every reader that holds it
    want = {(X.source_codec(f, t), t) for f, t in zip(files, types) if not X.is_rewrite(f, t, dst, codec)}
    if dst == X.HPS:   # HPS refuses looping files whose loop start moves past their first decode
        assert len(done) >= len(want) - 4, (want - done)
    else:
        assert done == want, (want - done)


def test_configured_targets_match_the_oracle_chain(vg, oracle):
    """Byte order, --loop-align, IDSP's no_trim, and -l / --no-loop."""
    from vgaudio_b200 import containers as ct

    srcs = _sources(oracle)
    files, types = [f for _, f, _ in srcs], [t for t, _, _ in srcs]
    for dst, codec, cfg, loop in [(X.BCSTM, X.PCM16, dict(endianness=2, alignment=1000), {}), (X.BFSTM, X.GCADPCM, dict(endianness=1, alignment=14), {}),
                                  (X.IDSP, X.GCADPCM, dict(trim=False), {}), (X.BRSTM, X.PCM16, {}, dict(loop=(700, 5000))),
                                  (X.HCA, X.GCADPCM, {}, dict(no_loop=True)), (X.DSP, X.GCADPCM, {}, dict(loop=(1234, 5000)))]:
        mode, s, e = (LO.SET, *loop["loop"]) if "loop" in loop else (LO.CLEAR, 0, 0) if loop else (LO.KEEP, 0, 0)
        outs, status = ct.transcode_from_nw_batch(files, types, X.options(ct, dst, codec, **cfg, **loop))
        assert len(_check(files, types, outs, status, dst, codec, mode=mode, start=s, end=e, **cfg)) >= 8, (dst, codec, cfg, loop)


def _lead_job(oracle):
    """Looping files whose Linear .adx lead (alignment_samples: the loop start up to a multiple of 32 samples, 64 for mono)
    is 0, 8 and 16, and 3, 5, 21 - GC-ADPCM and PCM rows alike - beside non-looping files, in one call."""
    n = 9001
    return [(X.BRSTM, NF.encoded(oracle, NF.BRSTM, X.GCADPCM, 2, n, loop=3200, seed=50)),     # 0
            (X.BCSTM, NF.encoded(oracle, NF.BCSTM, X.GCADPCM, 2, n, loop=3192, seed=51)),     # 8
            (X.BFSTM, NF.encoded(oracle, NF.BFSTM, X.GCADPCM, 1, n, loop=3197, seed=52)),     # 3
            (X.BCSTM, NF.encoded(oracle, NF.BCSTM, X.PCM16, 2, n, loop=1003, seed=53)),       # 21
            (X.BFSTM, NF.encoded(oracle, NF.BFSTM, X.PCM8, 1, n, loop=1008, seed=54)),        # 16
            (X.BCWAV, NWF.encoded(oracle, NWF.BCWAV, X.PCM16, 2, n, loop=3195, seed=55)),     # 5
            (X.BRWAV, NWF.encoded(oracle, NWF.BRWAV, X.GCADPCM, 2, n, loop=2019, seed=56)),   # 29
            (X.BCSTP, NWF.encoded(oracle, NWF.BCSTP, X.GCADPCM, 1, n, seed=57)),              # no loop
            (X.IDSP, X.idsp(2, n, 58, loop=(1021, n))),                                        # 3
            (X.IDSP, X.idsp(1, n, 59, loop=(1016, 8000))),                                     # 8
            (X.BRSTM, NF.encoded(oracle, NF.BRSTM, X.PCM16, 2, 7003, seed=60)),                # no loop
            (X.HPS, X.hps(2, 8001, 61)),                                                       # no loop
            (X.BFWAV, NWF.encoded(oracle, NWF.BFWAV, X.GCADPCM, 1, 5005, seed=62))]           # no loop


@pytest.mark.parametrize("loop", [None, (1003, 5000), (1016, 5000), (1024, 5000)])
def test_looping_files_into_linear_adx(vg, oracle, loop):
    """The hazard of the lead: rows of an aligned-vector decoder start behind `lead` zeros; a lead that is no multiple of
    8 decodes past the slab and is moved behind its lead.  All in one group with non-looping files."""
    from vgaudio_b200 import containers as ct

    job = _lead_job(oracle)
    files, types = [f for _, f in job], [t for t, _ in job]
    kw = dict(loop=loop) if loop else {}
    opt = X.options(ct, X.ADX, group_bytes=1 << 40, **kw)
    mode, s, e = (LO.SET, *loop) if loop else (LO.KEEP, 0, 0)
    leads = set()
    for t, f in job:
        p, _ = X.planned(f, t, X.ADX, mode=mode, start=s, end=e)
        if p and p[2]:
            leads.add(F.alignment(p[2][0], len(p[0]), 18) % 8 != 0)
    assert leads == {False, True} or loop is not None
    outs, status = ct.transcode_from_nw_batch(files, types, opt)
    assert len(_check(files, types, outs, status, X.ADX, mode=mode, start=s, end=e)) >= 10
    assert status == [0] * len(files), status
    # the composition through WAVE gives the same bytes
    waves, wst = ct.convert_to_wave_batch(files, types)
    assert wst == [0] * len(files)
    want, st = ct.convert_wave_batch(waves, opt)
    assert st == status and all(a.tobytes() == b.tobytes() for a, b in zip(outs, want))


@pytest.mark.parametrize("dst,codec", CELLS)
def test_same_bytes_as_the_two_call_composition(vg, oracle, dst, codec):
    from vgaudio_b200 import containers as ct

    srcs = _sources(oracle)
    keep = [(t, f) for t, f, _ in srcs if not X.is_rewrite(f, t, dst, codec)]
    files, types = [f for _, f in keep], [t for t, _ in keep]
    opt = X.options(ct, dst, codec, loop=(600, 5000)) if dst == X.IDSP else X.options(ct, dst, codec)
    waves, wst = ct.convert_to_wave_batch(files, types, opt)
    assert wst == [0] * len(files), wst
    want, st_want = ct.convert_wave_batch(waves, opt)
    outs, status = ct.transcode_from_nw_batch(files, types, opt)
    assert status == st_want, (status, st_want)
    for k in range(len(files)):
        if status[k] == 0:
            assert outs[k].tobytes() == want[k].tobytes(), (types[k], k)


def _bad_predictor(oracle, kind, predictor=8):
    """A stereo GC-ADPCM file whose channel 1 selects `predictor` on frame 100."""
    if kind in (X.IDSP, X.HPS):
        import idsp_hps_reader_oracle as RI

        n = 14 * 400
        enc = X._gc_rows(NF.pcm_channels(2, n, 71), 71)
        ad = np.array(enc[1][0], np.uint8)
        ad[800] = (predictor << 4) | (ad[800] & 0x0F)
        enc[1] = (ad, enc[1][1], enc[1][2])
        return RI.idsp_image(32000, enc, n) if kind == X.IDSP else RI.hps_chain(32000, enc, [0x400, 0x400, 0x480], n_samples=n)
    chans = NF.gc_channels(oracle, NF.pcm_channels(2, 14 * 400, 71))
    d = bytearray(chans[1].data)
    d[800] = (predictor << 4) | (d[800] & 0x0F)
    chans[1].data = bytes(d)
    return NF.build(kind, X.GCADPCM, chans, 14 * 400)


def _raw(vg, files, types, opt, status=True, fill=0xAB):
    """vgb_transcode_from_nw_batch by hand: (return code, sizes, statuses, buffers) with buffers pre-filled with `fill`."""
    n = len(files)
    files = [np.ascontiguousarray(f, np.uint8) for f in files]
    ftab = (C.c_void_p * n)(*[f.ctypes.data for f in files])
    lens = (C.c_int64 * n)(*[f.size for f in files])
    tys = (C.c_int32 * n)(*types)
    sizes, st = (C.c_int64 * n)(), (C.c_int32 * n)()
    assert vg.lib.vgb_transcode_from_nw_batch(ftab, lens, tys, n, C.byref(opt), sizes, None, st, None, None) == 0
    bufs = [np.full(max(sizes[k], 1), fill, np.uint8) for k in range(n)]
    otab = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    rc = vg.lib.vgb_transcode_from_nw_batch(ftab, lens, tys, n, C.byref(opt), sizes, otab, st if status else None, None, None)
    return rc, list(sizes), list(st), bufs


@pytest.mark.parametrize("dst,codec", [(X.HCA, X.GCADPCM), (X.BRSTM, X.PCM16)])
def test_predictor_fault_fails_its_own_file(vg, oracle, dst, codec):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    srcs = _sources(oracle)
    good = [(t, f) for t, f, _ in srcs if not X.is_rewrite(f, t, dst, codec)][:8]
    bad = [(X.BRSTM, _bad_predictor(oracle, X.BRSTM)), (X.BFSTM, _bad_predictor(oracle, X.BFSTM, 15)),
           (X.IDSP, _bad_predictor(oracle, X.IDSP)), (X.HPS, _bad_predictor(oracle, X.HPS, 9))]
    job = good[:3] + bad[:2] + good[3:6] + bad[2:] + good[6:]
    files, types = [f for _, f in job], [t for t, _ in job]
    opt = X.options(ct, dst, codec, group_bytes=1 << 40)   # one group
    rc, sizes, st, bufs = _raw(vg, files, types, opt)
    assert rc == 0
    for k, (t, f) in enumerate(job):
        if any(f is b for _, b in bad):
            assert st[k] == N.VGB_E_DATA and sizes[k] == 0 and (bufs[k] == 0xAB).all(), (k, st[k])
        else:
            assert st[k] == 0 and bufs[k].tobytes() == X.expected(f, t, dst, codec)[0].tobytes(), (k, t, st[k])
    # without status_out the call fails once the others are written
    rc, sizes, _, bufs = _raw(vg, files[:4], types[:4], opt, status=False)
    assert rc == N.VGB_E_DATA and b"pass status_out" in vg.lib.vgb_last_error()
    assert bufs[0].tobytes() == X.expected(files[0], types[0], dst, codec)[0].tobytes()
    outs, status = ct.transcode_from_nw_batch(files[:1], types[:1], opt)   # the library is usable again
    assert status == [0] and outs[0].tobytes() == bufs[0].tobytes()


def _mixed(oracle):
    srcs = _sources(oracle)
    order = np.random.default_rng(7).permutation(len(srcs))   # streams, wave, prefetch, IDSP and HPS files interleaved
    return [srcs[i][1] for i in order], [srcs[i][0] for i in order]


@pytest.mark.parametrize("dst,codec", [(X.HCA, X.GCADPCM), (X.BCSTM, X.PCM16), (X.ADX, X.GCADPCM)])
def test_many_groups_give_the_bytes_of_one_group(vg, oracle, dst, codec):
    from vgaudio_b200 import containers as ct

    files, types = _mixed(oracle)
    one, st_one = ct.transcode_from_nw_batch(files, types, X.options(ct, dst, codec, group_bytes=1 << 40, loop=(1001, 5000)))
    deltas = []
    small = X.options(ct, dst, codec, group_bytes=30000, loop=(1001, 5000))   # a group or two per file: more groups than ways
    many, st_many = ct.transcode_from_nw_batch(files, types, small, progress=deltas.append)
    assert st_one == st_many
    assert sum(deltas) == sum(1 for s in st_one if s == 0)
    assert sum(1 for s in st_one if s == 0) >= 10
    for k in range(len(files)):
        assert (one[k] is None and many[k] is None) or one[k].tobytes() == many[k].tobytes(), k
        want, _ = X.expected(files[k], types[k], dst, codec, mode=LO.SET, start=1001, end=5000)
        assert (want is None) == (one[k] is None) and (want is None or one[k].tobytes() == want.tobytes()), (k, types[k])


def test_two_bound_devices_give_the_same_bytes(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files, types = _mixed(oracle)
    for opt in (X.options(ct, X.HCA, group_bytes=1 << 20), X.options(ct, X.BRSTM, X.PCM8, group_bytes=1 << 20)):
        one, st_one = ct.transcode_from_nw_batch(files, types, opt)
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
        try:
            two, st_two = ct.transcode_from_nw_batch(files, types, opt)
        finally:
            N.check(vg.lib.vgb_shutdown())
            N.check(vg.lib.vgb_init(0, 0))
        assert st_one == st_two
        for k, (x, y) in enumerate(zip(one, two)):
            assert (x is None and y is None) or x.tobytes() == y.tobytes(), (opt.out_type, k, types[k])


# ---- the CLI ------------------------------------------------------------------------------------------------------------
def _cli(*args):
    return subprocess.run([CLI, *[str(a) for a in args]], capture_output=True, text=True)


def _mixed_dir(oracle, src):
    """a.wav, and one file of each kind --nw-inputs lists: GC-ADPCM, PCM16 and PCM8 streams, wave and prefetch files,
    IDSP and HPS."""
    src.mkdir()
    pcm = NF.pcm_channels(2, 6001, 80)
    (src / "a.wav").write_bytes(oracle.wave_write16(pcm, 32000, None).tobytes())
    files = {"b.brstm": (X.BRSTM, NF.encoded(oracle, NF.BRSTM, X.GCADPCM, 2, 6001, loop=1000, seed=81)),
             "c.bcstm": (X.BCSTM, NF.encoded(oracle, NF.BCSTM, X.PCM16, 2, 5003, seed=82)),
             "d.bfwav": (X.BFWAV, NWF.encoded(oracle, NWF.BFWAV, X.PCM8, 1, 4001, seed=83)),
             "e.bcstp": (X.BCSTP, NWF.encoded(oracle, NWF.BCSTP, X.GCADPCM, 1, 4003, seed=84)),
             "f.idsp": (X.IDSP, X.idsp(2, 5001, 85)),
             "g.hps": (X.HPS, X.hps(2, 7001, 86)),
             "h.rwav": (X.BRWAV, NWF.encoded(oracle, NWF.BRWAV, X.PCM16, 1, 3001, seed=87))}
    for name, (_, img) in files.items():
        (src / name).write_bytes(img.tobytes())
    return pcm, files


@pytest.mark.parametrize("fmt,dst,codec,extra", [("hca", X.HCA, X.GCADPCM, []), ("dsp", X.DSP, X.GCADPCM, []),
                                                 ("bcstm", X.BCSTM, X.PCM16, ["-f", "pcm16"])])
def test_cli_nw_inputs_mixed_directory(tmp_path, vg, oracle, fmt, dst, codec, extra):
    src = tmp_path / "in"
    pcm, files = _mixed_dir(oracle, src)
    out = tmp_path / "out"
    opt_args = ["--hcaquality", "high"] if dst == X.HCA else []
    r = _cli("-i", src, "-o", out, "--out-format", fmt, "--nw-inputs", *extra, *opt_args)
    listed = {n: v for n, v in files.items() if v[0] not in (X.IDSP, X.HPS) or X.target_codec(dst, codec) != X.GCADPCM}
    rewrites = {n for n, (t, img) in listed.items() if X.is_rewrite(img, t, dst, codec)}
    assert r.returncode == (3 if rewrites else 0), r.stdout + r.stderr
    for n in rewrites:
        assert f"Error converting {n}" in r.stderr, (n, r.stderr)
    converted = sorted(["a"] + [n.split(".")[0] for n in listed if n not in rewrites])
    assert sorted(os.listdir(out)) == [f"{n}.{fmt}" for n in converted]
    for n, (t, img) in listed.items():
        if n not in rewrites:
            assert (out / f"{n.split('.')[0]}.{fmt}").read_bytes() == X.expected(img, t, dst, codec)[0].tobytes(), n
    # without the flag: exactly today's output set
    plain = tmp_path / "plain"
    r = _cli("-i", src, "-o", plain, "--out-format", fmt, *extra, *opt_args)
    assert r.returncode == 0, r.stdout + r.stderr
    assert sorted(os.listdir(plain)) == [f"a.{fmt}"]
    assert (plain / f"a.{fmt}").read_bytes() == (out / f"a.{fmt}").read_bytes()


def test_cli_nw_inputs_with_loop_and_devices(tmp_path, vg, oracle):
    """--nw-inputs combines with -l, --no-loop and --devices."""
    src = tmp_path / "in"
    _, files = _mixed_dir(oracle, src)
    for args, mode, s, e in ((["-l", "500-3000"], LO.SET, 500, 3000), (["--no-loop", "--devices", "0,0"], LO.CLEAR, 0, 0)):
        out = tmp_path / f"out{mode}"
        r = _cli("-i", src, "-o", out, "--out-format", "adx", "--nw-inputs", *args)
        assert r.returncode == 0, r.stdout + r.stderr
        for n, (t, img) in files.items():
            want = X.expected(img, t, X.ADX, mode=mode, start=s, end=e)[0]
            assert (out / f"{n.split('.')[0]}.adx").read_bytes() == want.tobytes(), (n, args)
