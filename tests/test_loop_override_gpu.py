"""The batch's loop setting (-l / --no-loop) on the GPU: every output byte-identical to the oracle chain of
loop_override_oracle (a reader restatement, SetLoop, the writer restatement), refusals with the reference's messages,
in every direction: WAVE into each target (loop starts that do and do not need realignment, .dsp with and without
--loop-align, ADX loop starts on and off the lead path), the six transcodes, .adx / .hca rewrites (trimmed shorter and
longer than the source), every reader to WAVE, a mixed batch over several groups, two bound devices, and the CLI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import vgaudio_b200 as vg
from vgaudio_b200 import _native as N
from vgaudio_b200 import containers as ct

import adx_files as F
import cri_rewrite_oracle as RW
import gc_container_writer_oracle as GW
import loop_override_oracle as L
import nw_files as NF
import nw_wave_files as NWF
import transcode_oracle as T

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")


@pytest.fixture(scope="module", autouse=True)
def _device():
    N.check(vg.lib.vgb_init(0, 0))


def _pcm(ch, n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return [(np.sin(t * (0.011 + 0.002 * c)) * 8000 + rng.normal(0, 500, n)).clip(-32768, 32767).astype(np.int16) for c in range(ch)]


def _opts(out_type, mode, s=0, e=0, **kw):
    o = ct.convert_options(out_type, **kw)
    o.loop_mode, o.loop_start, o.loop_end = mode, s, e
    return o


def _same(out, status, want, note):
    """out/status: one converted file; want: the oracle's (file or None, message or status)."""
    if want[0] is not None:
        assert status == 0 and out is not None and out.tobytes() == want[0].tobytes(), note
    else:
        assert status != 0 and out is None, (note, status, want[1])


# loops per target: (mode, start, end) with starts that need realignment and starts that do not
N_SAMPLES = 70000
SETS = {
    L.DSP_T: [(L.SET, 1000, 60000), (L.SET, 0, N_SAMPLES), (L.SET, 300, 300)],
    L.ADX_T: [(L.SET, 1000, 60000), (L.SET, 1024, 60000), (L.SET, 0, 0)],       # stereo: alignment 24 (lead) and 0
    L.HCA_T: [(L.SET, 1000, 60000), (L.SET, 2048, N_SAMPLES), (L.SET, 5, 5)],
    L.BRSTM_T: [(L.SET, 1000, 60000), (L.SET, 14336, 60000)],
    L.BCSTM_T: [(L.SET, 1000, 60000), (L.SET, 14336, 60001)],
    L.BFSTM_T: [(L.SET, 20000, 50000), (L.SET, 0, 1)],
    L.IDSP_T: [(L.SET, 1000, 60000), (L.SET, 1120, 60000), (L.SET, 7, 7)],
    L.HPS_T: [(L.SET, 1000, 60000), (L.SET, 0, 60000), (L.SET, 57344, 65000)],
}


@pytest.mark.parametrize("out_type", sorted(SETS))
def test_wave_into_every_target(oracle, out_type):
    pcms = [_pcm(2, N_SAMPLES, 1), _pcm(1, N_SAMPLES, 2)]
    loops = [(3000, 66000), None]
    files = [oracle.wave_write16(p, 32000, lp) for p, lp in zip(pcms, loops)]
    for mode, s, e in [(L.KEEP, 0, 0), (L.CLEAR, 0, 0)] + SETS[out_type] + [(L.SET, 10, 9), (L.SET, 0, N_SAMPLES + 1)]:
        outs, status = ct.convert_wave_batch(files, _opts(out_type, mode, s, e))
        for k, (p, lp) in enumerate(zip(pcms, loops)):
            _same(outs[k], status[k], L.expected_from_wave(p, 32000, lp, out_type, mode, s, e), (out_type, k, mode, s, e))


@pytest.mark.parametrize("align", [28, 14 * 3])
def test_dsp_loop_alignment(oracle, align):
    pcms = [_pcm(2, 30000, 3), _pcm(1, 30000, 4)]
    files = [oracle.wave_write16(p, 32000) for p in pcms]
    for mode, s, e in [(L.SET, 1001, 29000), (L.SET, 28 * 42, 29000), (L.CLEAR, 0, 0)]:
        outs, status = ct.convert_wave_batch(files, _opts(L.DSP_T, mode, s, e, dsp_loop_point_alignment=align))
        for k, p in enumerate(pcms):
            _same(outs[k], status[k], L.expected_from_wave(p, 32000, None, L.DSP_T, mode, s, e, loop_align=align), (align, k, mode, s, e))


def test_smpl_loop_equals_the_same_loop_set(oracle):
    """WAVE with smpl (a, b), a < b, kept == the same file without smpl plus -l a-b; --no-loop == no smpl at all."""
    pcm = _pcm(2, 40000, 5)
    with_smpl, plain = oracle.wave_write16(pcm, 32000, (1234, 38000)), oracle.wave_write16(pcm, 32000)
    for out_type in sorted(SETS):
        a = ct.convert_wave_batch([with_smpl], _opts(out_type, L.KEEP))
        b = ct.convert_wave_batch([plain], _opts(out_type, L.SET, 1234, 38000))
        c = ct.convert_wave_batch([with_smpl], _opts(out_type, L.CLEAR))
        d = ct.convert_wave_batch([plain], _opts(out_type, L.KEEP))
        assert a[1] == b[1] and [o.tobytes() for o in a[0] if o is not None] == [o.tobytes() for o in b[0] if o is not None], out_type
        assert c[1] == d[1] == [0] and c[0][0].tobytes() == d[0][0].tobytes(), out_type


DIRECTIONS = [(L.DSP_T, L.ADX_T), (L.DSP_T, L.HCA_T), (L.ADX_T, L.DSP_T), (L.ADX_T, L.HCA_T), (L.HCA_T, L.DSP_T), (L.HCA_T, L.ADX_T)]


def _coded(oracle, kind):
    if kind == L.DSP_T:
        return [T.dsp_file(2, 20000, 32000, seed=11), T.dsp_file(1, 15000, 32000, (100, 14000), seed=12)]
    if kind == L.ADX_T:
        return [F.encoded(oracle, 2, 20000, 32000, seed=13), F.encoded(oracle, 1, 15000, 32000, loop=(100, 14000), seed=14)]
    return [T.hca_file(2, 32000, 20000, 15), T.hca_file(1, 32000, 15000, 16, loop=(2048, 14000))]


@pytest.mark.parametrize("src,dst", DIRECTIONS)
def test_transcodes(oracle, src, dst):
    files = _coded(oracle, src)
    cases = [(L.KEEP, 0, 0), (L.CLEAR, 0, 0), (L.SET, 1000, 12000), (L.SET, 0, 0)]
    if src == L.HCA_T:  # the file's own points pass
        cases.append((L.SET, *L.hca_points(T.RH.hca_parse(files[1])[1])))
    for mode, s, e in cases:
        outs, status = ct.transcode_batch(files, [src] * len(files), _opts(dst, mode, s, e, hca_quality=2))
        for k, f in enumerate(files):
            _same(outs[k], status[k], L.expected_transcode(f, src, dst, mode, s, e), (src, dst, k, mode, s, e))


def test_adx_rewrites_trimmed_shorter_and_longer(oracle):
    files = [RW.adx_source(2, 60, loop=(100, 900), inserted=20, seed=1), RW.adx_source(1, 60, seed=2),
             RW.adx_source(2, 40, version=3, loop=(64, 1000), seed=3)]
    spf = 32
    for mode, s, e in [(L.KEEP, 0, 0), (L.CLEAR, 0, 0), (L.SET, 10, 200), (L.SET, 100, 40 * spf - 20), (L.SET, 0, 0), (L.SET, 5, 4)]:
        for no_trim in (False, True):
            outs, status = ct.rewrite_batch(files, _opts(L.ADX_T, mode, s, e, no_trim=int(no_trim)))
            for k, f in enumerate(files):
                want = L.expected_adx_rewrite(f, mode, s, e, no_trim)
                _same(outs[k], status[k], want, (k, mode, s, e, no_trim))
    # the cut follows the new loop end: shorter than the source, and longer (zero frames past it) with the loop at the end
    short = ct.rewrite_batch(files[:1], _opts(L.ADX_T, L.SET, 10, 200))[0][0]
    long_ = ct.rewrite_batch(files[:1], _opts(L.ADX_T, L.SET, 100, 60 * spf - 20))[0][0]
    counts = [L.RA.adx_parse(f)[1].sample_count for f in (short, files[0], long_)]
    assert counts[0] < counts[1] < counts[2], counts
    assert long_.tobytes() == L.expected_adx_rewrite(files[0], L.SET, 100, 60 * spf - 20)[0].tobytes()


def test_hca_rewrites(oracle):
    info = RW.hca_info(looping=True)
    img = RW.hca_source(info, RW.hca_frames(info, 7))
    s0, e0 = L.hca_points(RW.hca_parse(img)[1])
    for mode, s, e in [(L.KEEP, 0, 0), (L.CLEAR, 0, 0), (L.SET, s0, e0), (L.SET, s0 + 1, e0)]:
        outs, status = ct.rewrite_batch([img], _opts(L.HCA_T, mode, s, e))
        _same(outs[0], status[0], L.expected_hca_rewrite(img, mode, s, e), (mode, s, e))


def _readers(oracle):
    """(image, in_type) of every reader kind, looping and not."""
    return [(T.dsp_file(2, 9000, 32000, (100, 8000), seed=21), L.DSP_T), (T.dsp_file(1, 7000, 32000, seed=22), L.DSP_T),
            (F.encoded(oracle, 2, 9000, 32000, loop=(100, 8000), seed=23), L.ADX_T), (F.encoded(oracle, 1, 7000, 32000, seed=24), L.ADX_T),
            (T.hca_file(2, 32000, 9000, 25, loop=(1024, 8000)), L.HCA_T), (T.hca_file(1, 32000, 7000, 26), L.HCA_T),
            (NF.encoded(oracle, NF.BRSTM, NF.GCADPCM, 2, 9000, loop=500, seed=27), L.BRSTM_T),
            (NF.encoded(oracle, NF.BCSTM, NF.PCM16, 1, 7000, seed=28), L.BCSTM_T),
            (NF.encoded(oracle, NF.BFSTM, NF.GCADPCM, 1, 7000, seed=29), L.BFSTM_T),
            (GW.write_idsp(_pcm(2, 9000, 30), 32000, (100, 8000))[1], L.IDSP_T), (GW.write_hps(_pcm(1, 7000, 31), 32000)[1], L.HPS_T),
            (NWF.encoded(oracle, NWF.BRWAV, NWF.GCADPCM, 2, 9000, loop=400, seed=32), L.BRWAV_T),
            (NWF.encoded(oracle, NWF.BCWAV, NWF.PCM16, 1, 7000, seed=33), L.BCWAV_T),
            (NWF.cwav(NWF.BFWAV, NWF.PCM16, NWF.channels(oracle, NWF.PCM16, 1, 7000, 34, True), 7000, cut=2000), L.BFWAV_T),  # row: 6000
            (NWF.encoded(oracle, NWF.BCSTP, NWF.GCADPCM, 2, 9000, loop=300, seed=35), L.BCSTP_T),
            (NWF.encoded(oracle, NWF.BFSTP, NWF.PCM8, 1, 7000, seed=36), L.BFSTP_T)]


@pytest.mark.parametrize("mode,s,e", [(L.KEEP, 0, 0), (L.CLEAR, 0, 0), (L.SET, 500, 6000), (L.SET, 0, 7000), (L.SET, 0, 0), (L.SET, 0, 8500)])
def test_every_reader_to_wave_in_one_mixed_call(oracle, mode, s, e):
    imgs, types = zip(*_readers(oracle))
    outs, status = ct.convert_to_wave_batch(list(imgs), list(types), _opts(0, mode, s, e))
    for k, (img, t) in enumerate(zip(imgs, types)):
        _same(outs[k], status[k], L.expected_wave(img, t, mode, s, e), (k, t, mode, s, e))


def test_null_options_equal_the_five_calls(oracle):
    pairs = _readers(oracle)
    imgs, types = zip(*pairs)
    got = ct.convert_to_wave_batch(list(imgs), list(types), None)
    for k, (img, t) in enumerate(pairs):
        if t == L.DSP_T:
            old = ct.convert_dsp_to_wave_batch([img])
        elif t == L.ADX_T:
            old = ct.convert_adx_to_wave_batch([img])
        elif t == L.HCA_T:
            old = ct.convert_hca_to_wave_batch([img])
        elif t in (L.IDSP_T, L.HPS_T):
            old = ct.convert_idsp_hps_to_wave_batch([img], [t])
        else:
            old = ct.convert_nw_to_wave_batch([img], [t])
        assert got[1][k] == old[1][0] == 0 and got[0][k].tobytes() == old[0][0].tobytes(), k


def test_mixed_batch_over_groups_and_two_devices(oracle):
    """Many WAVE files, half of them looping, over several groups (group_bytes), every file realigned for BRSTM; then the
    same job on one device bound twice gives the same bytes."""
    pcms = [_pcm(1 + k % 3, 20000 + 997 * k, 40 + k) for k in range(12)]
    files = [oracle.wave_write16(p, 32000, (500, len(p[0]) - 7) if k % 2 else None) for k, p in enumerate(pcms)]
    opt = _opts(L.BRSTM_T, L.SET, 1001, 19000, group_bytes=1 << 17)
    one = ct.convert_wave_batch(files, opt)
    for k, p in enumerate(pcms):
        _same(one[0][k], one[1][k], L.expected_from_wave(p, 32000, None, L.BRSTM_T, L.SET, 1001, 19000), k)
    imgs, types = zip(*_readers(oracle))
    dec_one = ct.convert_to_wave_batch(list(imgs), list(types), _opts(0, L.CLEAR))
    N.check(vg.lib.vgb_shutdown())
    N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
    try:
        assert vg.lib.vgb_device_count() == 2
        two = ct.convert_wave_batch(files, opt)
        dec_two = ct.convert_to_wave_batch(list(imgs), list(types), _opts(0, L.CLEAR))
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    for a, b in ((one, two), (dec_one, dec_two)):
        assert a[1] == b[1]
        assert [o.tobytes() if o is not None else None for o in a[0]] == [o.tobytes() if o is not None else None for o in b[0]]


def _run(*args):
    return subprocess.run([CLI, *map(str, args)], capture_output=True, text=True, timeout=600)


def test_cli_end_to_end(tmp_path, oracle):
    src = tmp_path / "in"
    src.mkdir()
    pcm = _pcm(2, 30000, 50)
    (src / "a.wav").write_bytes(oracle.wave_write16(pcm, 32000, (100, 29000)).tobytes())
    dsp = T.dsp_file(1, 9000, 32000, (100, 8000), seed=51)
    (src / "b.dsp").write_bytes(dsp.tobytes())
    hca = T.hca_file(1, 32000, 7000, 52)
    (src / "c.hca").write_bytes(hca.tobytes())
    # WAVE -> .dsp with -l and --loop-align; the coded files transcode (.hca refuses -l: it has no loop)
    r = _run("-i", src, "-o", tmp_path / "dsp", "--out-format", "dsp", "-l", "1001-8000", "--loop-align", "28")
    assert r.returncode == 3, r.stderr  # c.hca failed
    got = (tmp_path / "dsp" / "a.dsp").read_bytes()
    assert got == L.expected_from_wave(pcm, 32000, (100, 29000), L.DSP_T, L.SET, 1001, 8000, loop_align=28)[0].tobytes()
    assert not (tmp_path / "dsp" / "c.dsp").exists()
    # --no-loop to WAVE from every source
    r = _run("-i", src, "-o", tmp_path / "wav", "--out-format", "wav", "--no-loop")
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "wav" / "b.wav").read_bytes() == L.expected_wave(dsp, L.DSP_T, L.CLEAR)[0].tobytes()
    assert (tmp_path / "wav" / "c.wav").read_bytes() == L.expected_wave(hca, L.HCA_T, L.CLEAR)[0].tobytes()
    # -l into a NintendoWare target
    r = _run("-i", src, "-o", tmp_path / "nw", "--out-format", "bcstm", "-l", "2000-20000")
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "nw" / "a.bcstm").read_bytes() == L.expected_from_wave(pcm, 32000, (100, 29000), L.BCSTM_T, L.SET, 2000, 20000)[0].tobytes()
