"""The batch's loop setting (-l / --no-loop, vgb_convert_options.loop_*) in the host-only sizing passes: for every
source kind and {keep, set, clear}, vgb_convert_wave_batch, vgb_transcode_batch, vgb_rewrite_batch and
vgb_convert_to_wave_batch size each file as the oracle chain (loop_override_oracle) writes it, and refuse it with the
reference's message where SetLoop throws.  No device is needed; also the CLI's parse errors, which come before any device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import adx_files as F
import cri_rewrite_oracle as RW
import gc_container_writer_oracle as GW
import loop_override_oracle as L
import nw_files as NF
import nw_wave_files as NWF
import transcode_oracle as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = [(L.KEEP, 0, 0), (L.SET, 100, 900), (L.CLEAR, 0, 0)]


def _opts(out_type, mode, s, e, **kw):
    from vgaudio_b200 import containers as ct

    o = ct.convert_options(out_type, **kw)
    o.loop_mode, o.loop_start, o.loop_end = mode, s, e
    return o


def _one(call, img):
    """(size, status, message) of one file's sizing pass; call(ftab, lens, sizes, status) makes it."""
    f = np.ascontiguousarray(img, np.uint8)
    ftab, lens = (C.c_void_p * 1)(f.ctypes.data), (C.c_int64 * 1)(f.size)
    sz, st = (C.c_int64 * 1)(), (C.c_int32 * 1)()
    assert call(ftab, lens, sz, st) == 0
    from vgaudio_b200 import _native as N

    return int(sz[0]), int(st[0]), (N.lib.vgb_last_error() or b"").decode() if st[0] else ""


def _to_wave(vg, img, in_type, opt, adx_key=None, hca_key=None):
    types = (C.c_int32 * 1)(in_type)
    code = C.c_uint64(hca_key) if hca_key is not None else None
    return _one(lambda ftab, lens, sz, st: vg.lib.vgb_convert_to_wave_batch(
        ftab, lens, types, 1, C.byref(opt) if opt is not None else None, C.byref(adx_key) if adx_key is not None else None,
        C.byref(code) if code is not None else None, sz, None, st), img)


def _wave(vg, img, opt):
    return _one(lambda ftab, lens, sz, st: vg.lib.vgb_convert_wave_batch(ftab, lens, 1, C.byref(opt), sz, None, st, None, None), img)


def _transcode(vg, img, in_type, opt):
    types = (C.c_int32 * 1)(in_type)
    return _one(lambda ftab, lens, sz, st: vg.lib.vgb_transcode_batch(ftab, lens, types, 1, C.byref(opt), None, None, sz, None, st, None, None), img)


def _rewrite(vg, img, opt):
    return _one(lambda ftab, lens, sz, st: vg.lib.vgb_rewrite_batch(ftab, lens, 1, C.byref(opt), None, None, sz, None, st, None, None), img)


def _check(got, want, msg):
    """got: (size, status, message); want: the oracle's (file or None, message or status)."""
    size, status, message = got
    if want[0] is not None:
        assert status == 0 and size == want[0].size, (got, msg)
    elif isinstance(want[1], str):
        assert status == -1 and message.endswith(want[1]) and size == 0, (got, want[1], msg)
    else:
        assert status != 0 and size == 0, (got, msg)


def _pcm(ch, n, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return [(np.sin(t * (0.01 + 0.003 * c)) * 9000 + rng.normal(0, 400, n)).clip(-32768, 32767).astype(np.int16) for c in range(ch)]


def _sources(oracle):
    """(in_type, image, note) of every readable source kind, looping and not."""
    out = [(L.DSP_T, T.dsp_file(2, 3000, 32000, seed=1), "dsp"), (L.DSP_T, T.dsp_file(1, 2000, 32000, (50, 1500), seed=2), "dsp loop"),
           (L.ADX_T, F.encoded(oracle, 2, 3000, 32000, seed=3), "adx"),
           (L.ADX_T, F.encoded(oracle, 1, 2000, 32000, loop=(100, 1900), seed=4), "adx loop, inserted samples"),
           (L.HCA_T, T.hca_file(1, 32000, 3000, 5), "hca"), (L.HCA_T, T.hca_file(2, 32000, 5000, 6, loop=(1024, 4000)), "hca loop"),
           (L.BRSTM_T, NF.encoded(oracle, NF.BRSTM, NF.GCADPCM, 2, 3000, loop=500, seed=7), "brstm"),
           (L.BCSTM_T, NF.encoded(oracle, NF.BCSTM, NF.PCM16, 1, 2000, seed=8), "bcstm pcm16"),
           (L.IDSP_T, GW.write_idsp(_pcm(2, 3000, 9), 32000, (100, 2000))[1], "idsp loop"),
           (L.HPS_T, GW.write_hps(_pcm(1, 3000, 10), 32000)[1], "hps"),
           (L.BRWAV_T, NWF.encoded(oracle, NWF.BRWAV, NWF.PCM16, 2, 2500, loop=300, seed=11), "brwav pcm16 loop"),
           (L.BCWAV_T, NWF.encoded(oracle, NWF.BCWAV, NWF.GCADPCM, 2, 3000, loop=700, seed=12), "bcwav gc-adpcm loop"),
           (L.BFWAV_T, NWF.encoded(oracle, NWF.BFWAV, NWF.PCM8, 1, 2000, seed=13), "bfwav pcm8"),
           (L.BCSTP_T, NWF.encoded(oracle, NWF.BCSTP, NWF.GCADPCM, 1, 3000, loop=200, seed=14), "bcstp gc-adpcm loop"),
           (L.BFSTP_T, NWF.encoded(oracle, NWF.BFSTP, NWF.PCM16, 2, 2000, seed=15), "bfstp pcm16")]
    for in_type, img, note in out:  # every stimulus is readable, so every case below reaches SetLoop
        assert L.source(img, in_type) is not None, note
    return out


def test_set_loop_rules():
    assert L.set_loop(L.PCM, 1000, None, L.SET, 0, 0) == ((0, 0), None)
    assert L.set_loop(L.PCM, 1000, None, L.SET, 0, 1000) == ((0, 1000), None)
    assert L.set_loop(L.PCM, 1000, None, L.SET, 5, 5) == ((5, 5), None)
    assert L.set_loop(L.PCM, 1000, None, L.SET, 0, 1001)[1] == L.MSG_RANGE
    assert L.set_loop(L.PCM, 1000, None, L.SET, -1, 10)[1] == L.MSG_RANGE
    assert L.set_loop(L.PCM, 1000, None, L.SET, 10, 9)[1] == L.MSG_ORDER
    assert L.set_loop(L.GCADPCM, 1000, (1, 2), L.CLEAR) == (None, None)
    # HCA: the base checks first, then a change, then an add
    assert L.set_loop(L.HCA, 1000, None, L.SET, 0, 2000, (0, 1024))[1] == L.MSG_RANGE
    assert L.set_loop(L.HCA, 1000, (10, 900), L.SET, 10, 800, (10, 900))[1] == L.MSG_HCA_CHANGE
    assert L.set_loop(L.HCA, 2000, None, L.SET, 0, 1024, (0, 1024))[1] == L.MSG_HCA_ADD
    assert L.set_loop(L.HCA, 1000, (10, 900), L.SET, 10, 900, (10, 900)) == ((10, 900), None)
    assert L.adx_header_loop((10, 20), 7) == (17, 27)


@pytest.mark.parametrize("mode,s,e", MODES + [(L.SET, 0, 0), (L.SET, 300, 300), (L.SET, 10, 5), (L.SET, 0, 10 ** 6), (L.SET, -1, 5)])
def test_decode_direction_sizes_and_messages(vg, oracle, mode, s, e):
    for in_type, img, note in _sources(oracle):
        got = _to_wave(vg, img, in_type, _opts(0, mode, s, e))
        _check(got, L.expected_wave(img, in_type, mode, s, e), (note, mode, s, e))


def test_decode_direction_hca_own_points_and_whole_file(vg, oracle):
    img = T.hca_file(2, 32000, 5000, 6, loop=(1024, 4000))
    st, info, _ = T.RH.hca_parse(img)
    s, e = L.hca_points(info)
    for mode, a, b in [(L.SET, s, e), (L.SET, 0, info.sample_count), (L.SET, s, e - 1), (L.CLEAR, 0, 0)]:
        _check(_to_wave(vg, img, L.HCA_T, _opts(0, mode, a, b)), L.expected_wave(img, L.HCA_T, mode, a, b), (mode, a, b))
    # a file without a loop: its own points are (-InsertedSamples, 1024 - InsertedSamples), so -l meets the base check,
    # then "Changing", and "Adding" only when it has no inserted samples
    plain = T.hca_file(1, 32000, 3000, 5)
    p0 = L.hca_points(T.RH.hca_parse(plain)[1])
    for a, b, msg in [(0, 1000, L.MSG_HCA_CHANGE), (max(p0[0], 0), max(p0[1], 0), L.MSG_HCA_CHANGE if p0[0] < 0 else L.MSG_HCA_ADD)]:
        got = _to_wave(vg, plain, L.HCA_T, _opts(0, L.SET, a, b))
        assert got[1] == -1 and got[2].endswith(msg), got
        assert L.expected_wave(plain, L.HCA_T, L.SET, a, b) == (None, msg)
    info = RW.hca_info(channels=1, looping=False)
    info.inserted_samples = 0
    bare = RW.hca_source(info, RW.hca_frames(info, 4))
    assert L.hca_points(RW.hca_parse(bare)[1]) == (0, 1024)
    for op in (_to_wave, _rewrite):
        got = op(vg, bare, L.HCA_T, _opts(L.HCA_T, L.SET, 0, 1024)) if op is _to_wave else op(vg, bare, _opts(L.HCA_T, L.SET, 0, 1024))
        assert got[1] == -1 and got[2].endswith(L.MSG_HCA_ADD), got


def test_decode_direction_null_options_equal_the_five_calls(vg, oracle):
    for in_type, img, note in _sources(oracle):
        want = _to_wave(vg, img, in_type, None)
        assert want == _to_wave(vg, img, in_type, _opts(0, 0, 0, 0)), note
        types = (C.c_int32 * 1)(in_type)
        if in_type == L.DSP_T:
            old = _one(lambda f, l, sz, st: vg.lib.vgb_convert_dsp_to_wave_batch(f, l, 1, sz, None, st), img)
        elif in_type == L.ADX_T:
            old = _one(lambda f, l, sz, st: vg.lib.vgb_convert_adx_to_wave_batch(f, l, 1, None, sz, None, st), img)
        elif in_type == L.HCA_T:
            old = _one(lambda f, l, sz, st: vg.lib.vgb_convert_hca_to_wave_batch(f, l, 1, None, sz, None, st), img)
        elif in_type in (L.IDSP_T, L.HPS_T):
            old = _one(lambda f, l, sz, st: vg.lib.vgb_convert_idsp_hps_to_wave_batch(f, l, types, 1, sz, None, st), img)
        else:
            old = _one(lambda f, l, sz, st: vg.lib.vgb_convert_nw_to_wave_batch(f, l, types, 1, sz, None, st), img)
        assert want == old, note
    got = _to_wave(vg, np.zeros(16, np.uint8), 99, None)
    assert got[1] == -1 and "in_type 99" in got[2]


@pytest.mark.parametrize("kind", [L.BRWAV_T, L.BCWAV_T, L.BFWAV_T])
def test_pcm_nintendoware_row_sets_the_count(vg, oracle, kind):
    """A PCM16 wave file whose channel run ends 1000 bytes early (at the image's end): its header says 2000 samples,
    but Pcm16FormatBuilder's SampleCount is channel 0's row, 1500 samples, and -l is checked against that."""
    chans = NWF.channels(oracle, NWF.PCM16, 1, 2000, 21, kind != L.BCWAV_T)
    img = NWF.rwav(NWF.PCM16, chans, 2000, cut=1000) if kind == L.BRWAV_T else NWF.cwav(kind, NWF.PCM16, chans, 2000, cut=1000)
    src = L.source(img, kind)
    assert src is not None and src[1] == 1500 and len(src[0][0]) == 1500
    for mode, s, e in [(L.SET, 0, 1500), (L.SET, 100, 1400), (L.SET, 1500, 1500), (L.CLEAR, 0, 0), (L.KEEP, 0, 0)]:
        got = _to_wave(vg, img, kind, _opts(0, mode, s, e))
        want = L.expected_wave(img, kind, mode, s, e)
        assert want[0] is not None, (mode, s, e)
        _check(got, want, (kind, mode, s, e))
    for s, e in [(0, 1501), (0, 2000), (1501, 1501)]:
        got = _to_wave(vg, img, kind, _opts(0, L.SET, s, e))
        assert got[1] == -1 and got[2].endswith(L.MSG_RANGE) and got[0] == 0, (kind, s, e, got)
        assert L.expected_wave(img, kind, L.SET, s, e) == (None, L.MSG_RANGE)


@pytest.mark.parametrize("out_type", [L.DSP_T, L.ADX_T, L.HCA_T, L.BRSTM_T, L.BCSTM_T, L.BFSTM_T, L.IDSP_T, L.HPS_T])
def test_wave_sources_into_every_target(vg, oracle, out_type):
    pcm = _pcm(2, 40000, 3)
    for loop in (None, (1000, 39000)):
        img = oracle.wave_write16(pcm, 32000, loop)
        for mode, s, e in MODES + [(L.SET, 0, 0), (L.SET, 0, 40000), (L.SET, 5000, 5000), (L.SET, 10, 40001), (L.SET, 9, 8), (L.SET, -3, 8)]:
            got = _wave(vg, img, _opts(out_type, mode, s, e))
            _check(got, L.expected_from_wave(pcm, 32000, loop, out_type, mode, s, e), (out_type, loop, mode, s, e))


@pytest.mark.parametrize("src,dst", [(L.DSP_T, L.ADX_T), (L.DSP_T, L.HCA_T), (L.ADX_T, L.DSP_T), (L.ADX_T, L.HCA_T), (L.HCA_T, L.DSP_T), (L.HCA_T, L.ADX_T)])
def test_transcode_sizes_and_messages(vg, oracle, src, dst):
    for in_type, img, note in _sources(oracle):
        if in_type != src:
            continue
        for mode, s, e in MODES + [(L.SET, 0, 0), (L.SET, 10, 5), (L.SET, 0, 10 ** 6)]:
            got = _transcode(vg, img, src, _opts(dst, mode, s, e, hca_quality=2))
            want = L.expected_transcode(img, src, dst, mode, s, e)
            _check(got, want, (note, dst, mode, s, e))


def test_rewrite_sizes_and_messages(vg, oracle):
    adx = RW.adx_source(2, 40, loop=(100, 900), inserted=20, seed=1)
    plain = RW.adx_source(1, 40, seed=2)
    for img in (adx, plain):
        for mode, s, e in MODES + [(L.SET, 0, 1100), (L.SET, 0, 100), (L.SET, 5, 4), (L.SET, 0, 5000)]:
            _check(_rewrite(vg, img, _opts(L.ADX_T, mode, s, e)), L.expected_adx_rewrite(img, mode, s, e), (mode, s, e))
    info = RW.hca_info(looping=True)
    hca = RW.hca_source(info, RW.hca_frames(info, 3))
    st, parsed, *_ = RW.hca_parse(hca)
    s0, e0 = L.hca_points(parsed)
    for mode, s, e in [(L.KEEP, 0, 0), (L.CLEAR, 0, 0), (L.SET, s0, e0), (L.SET, s0, e0 - 1), (L.SET, 0, 10 ** 6)]:
        _check(_rewrite(vg, hca, _opts(L.HCA_T, mode, s, e)), L.expected_hca_rewrite(hca, mode, s, e), (mode, s, e))


def test_bad_loop_mode_fails_the_call(vg, oracle):
    """An unknown loop_mode is a bad argument of the call in every call that takes options: VGB_E_ARG before any file."""
    from vgaudio_b200 import _native as N

    wav = np.ascontiguousarray(oracle.wave_write16(_pcm(1, 1000), 32000), np.uint8)
    dsp = np.ascontiguousarray(T.dsp_file(1, 1000, 32000, seed=3), np.uint8)
    adx = np.ascontiguousarray(RW.adx_source(1, 10, seed=4), np.uint8)

    def call(fn, img, *a):
        ftab, lens = (C.c_void_p * 1)(img.ctypes.data), (C.c_int64 * 1)(img.size)
        sz, st = (C.c_int64 * 1)(-5), (C.c_int32 * 1)(-5)
        code = fn(ftab, lens, *a, sz, st)
        return code, int(sz[0]), int(st[0]), (N.lib.vgb_last_error() or b"").decode()

    one = (C.c_int32 * 1)
    for got in [
        call(lambda f, l, sz, st: vg.lib.vgb_convert_wave_batch(f, l, 1, C.byref(_opts(L.DSP_T, 7, 0, 0)), sz, None, st, None, None), wav),
        call(lambda f, l, sz, st: vg.lib.vgb_transcode_batch(f, l, one(L.DSP_T), 1, C.byref(_opts(L.ADX_T, 3, 0, 0)), None, None, sz, None, st,
                                                             None, None), dsp),
        call(lambda f, l, sz, st: vg.lib.vgb_rewrite_batch(f, l, 1, C.byref(_opts(L.ADX_T, -1, 0, 0)), None, None, sz, None, st, None, None), adx),
        call(lambda f, l, sz, st: vg.lib.vgb_convert_to_wave_batch(f, l, one(L.DSP_T), 1, C.byref(_opts(0, 9, 0, 0)), None, None, sz, None, st), dsp),
    ]:
        code, size, status, message = got
        assert code == N.VGB_E_ARG and "loop_mode" in message and not message.startswith("file"), got
        assert size == -5 and status == -5, got  # no file was read


def test_python_loop_keywords():
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    o = ct.convert_options(ct.CONTAINER_BRSTM, loop=(12, 3456))
    assert (o.loop_mode, o.loop_start, o.loop_end, o.out_type) == (N.VGB_LOOP_SET, 12, 3456, ct.CONTAINER_BRSTM)
    o = ct.convert_options(ct.CONTAINER_DSP, no_loop=True)
    assert (o.loop_mode, o.loop_start, o.loop_end) == (N.VGB_LOOP_CLEAR, 0, 0)
    o = ct.convert_options(ct.CONTAINER_ADX)
    assert (o.loop_mode, o.loop_start, o.loop_end) == (0, 0, 0)
    with pytest.raises(ValueError, match="Can't set loop points while using --no-loop."):
        ct.convert_options(ct.CONTAINER_HCA, loop=(0, 1), no_loop=True)


@pytest.mark.parametrize("args,message", [
    (["-l"], "No argument after -l switch."),
    (["-l", "5"], "-l switch requires two loop points in the format <start>-<end>."),
    (["-l", "1-2-3"], "-l switch requires two loop points in the format <start>-<end>."),
    (["-l", "x-2"], "Error parsing loop points."),
    (["-l", "5-"], "Error parsing loop points."),
    (["-l", "1-99999999999"], "Error parsing loop points."),
    (["--no-loop", "-l", "1-2"], "Can't set loop points while using --no-loop."),
    (["-l", "1-2", "--no-loop"], "Can't set loop points while using --no-loop."),
])
def test_cli_parse_errors(vg, tmp_path, args, message):
    cli = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")
    if not os.path.exists(cli):
        pytest.skip("the CLI is not built")
    r = subprocess.run([cli, "-i", str(tmp_path), "-o", str(tmp_path / "o"), "--out-format", "dsp"] + args, capture_output=True, text=True)
    assert r.returncode == 2 and r.stderr.splitlines()[0] == message, r.stderr
