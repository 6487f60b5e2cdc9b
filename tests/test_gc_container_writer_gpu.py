"""WAVE -> .idsp / .hps on the GPU: every file byte-identical to the oracle's writer (refused files refused alike),
HPS files of one block and one frame either side of it, long tracks with forced decode segments, per-file refusals in
the middle of a batch, many groups in flight, two bound devices and the CLI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import vgaudio_b200 as vg
from oracle import pyoracle as O
from vgaudio_b200 import containers as ct

import gc_container_writer_oracle as W
import nw_writer_oracle as NW
from test_gc_container_writer import CHANNELS, hps_shift_loop, loops

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _device():
    vg._native.check(vg.lib.vgb_init(0, 0))


def _pcm(ch, n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return [(np.sin(t * (0.013 + 0.002 * c)) * 8000 + rng.normal(0, 500, n)).clip(-32768, 32767).astype(np.int16) for c in range(ch)]


def _write(kind, pcm, rate, loop, trim=True):
    return W.write_idsp(pcm, rate, loop, trim) if kind == W.IDSP else W.write_hps(pcm, rate, loop)


def _check(kind, jobs, pcms, outs, status, rate=lambda i: 32000 + i, trim=True):
    for i, (p, (ch, n, loop)) in enumerate(zip(pcms, jobs)):
        st, want = _write(kind, p, rate(i), loop, trim)
        assert status[i] == st, f"job {i}: {ch} channels, {n} samples, loop {loop}"
        if st == 0:
            assert outs[i].tobytes() == want.tobytes(), f"job {i}: {ch} channels, {n} samples, loop {loop}"
        else:
            assert outs[i] is None


def _jobs():
    out = []
    for ch in CHANNELS:
        for n in (100, 4096, 14336 * 5 + 9, 70000 if ch > 1 else 150000):
            out += [(ch, n, loop) for loop in loops(n, ch)]
    return out


@pytest.mark.parametrize("kind", (W.IDSP, W.HPS))
@pytest.mark.parametrize("trim", (True, False))
def test_files_are_byte_identical_to_the_oracle(kind, trim):
    if kind == W.HPS and not trim:
        pytest.skip("HpsWriter does not read TrimFile")
    jobs = _jobs()
    pcms = [_pcm(ch, n, i) for i, (ch, n, _) in enumerate(jobs)]
    waves = [O.wave_write16(p, 32000 + i, loop) for i, (p, (_, _, loop)) in enumerate(zip(pcms, jobs))]
    outs, status = ct.convert_wave_batch(waves, ct.convert_options(kind, no_trim=0 if trim else 1))
    _check(kind, jobs, pcms, outs, status, trim=trim)
    if kind == W.HPS:
        assert any(s != 0 for s in status) and any(s == 0 for s in status)


@pytest.mark.parametrize("kind", (W.IDSP, W.HPS))
def test_8bit_wave_inputs(kind):
    rng = np.random.default_rng(5)
    chans = [rng.integers(0, 256, 30000, dtype=np.uint8) for _ in range(2)]
    pcm = [((c.astype(np.int16) - 0x80) << 8).astype(np.int16) for c in chans]
    jobs = [(2, 30000, loop) for loop in (None, (0, 29000), (57344 // 4, 29000), (101, 29000))]
    waves = [NW.wave_write8(chans, 22050, loop) for _, _, loop in jobs]
    outs, status = ct.convert_wave_batch(waves, ct.convert_options(kind))
    _check(kind, jobs, [pcm] * len(jobs), outs, status, rate=lambda i: 22050)
    assert status[:2] == [0, 0]


def test_hps_block_boundaries():
    """files of exactly one block and one frame either side of it, looping or not"""
    jobs = []
    for ch in (1, 2, 4):
        a = W.byte_count_to_sample_count(W.hps_channel_size(ch))  # samples of one full block
        for n in (a - 14, a, a + 14, 2 * a - 14, 2 * a, 2 * a + 14):
            jobs += [(ch, n, None), (ch, n, (0, n)), (ch, n, (a, n)) if n > a else (ch, n, (14, n))]
            if n > a - 14:
                jobs.append((ch, n, (a - 14, n)))
    pcms = [_pcm(ch, n, i) for i, (ch, n, _) in enumerate(jobs)]
    waves = [O.wave_write16(p, 32000 + i, loop) for i, (p, (_, _, loop)) in enumerate(zip(pcms, jobs))]
    outs, status = ct.convert_wave_batch(waves, ct.convert_options(W.HPS))
    _check(W.HPS, jobs, pcms, outs, status)
    one_block = [i for i, (ch, n, loop) in enumerate(jobs) if status[i] == 0 and len(W.parse_hps(outs[i])["blocks"]) == 1]
    assert one_block


@pytest.mark.parametrize("kind", (W.IDSP, W.HPS))
def test_long_tracks_with_forced_segments(kind, monkeypatch):
    monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", "7")
    n = 48000 * 180
    # an unaligned loop whose end sits near a decode-segment boundary (seven segments of about 88 000 frames), an HPS
    # loop start just behind a block boundary and an aligned one
    jobs = [(2, n, (100003, 88163 * 14 + 9)), (2, n, None), (2, n, (57344 * 3 + 1, 57344 * 40 + 5)), (2, n, (57344 * 10, n - 1))]
    pcms = [_pcm(2, n, 40 + i) for i in range(len(jobs))]
    waves = [O.wave_write16(p, 48000, j[2]) for p, j in zip(pcms, jobs)]
    outs, status = ct.convert_wave_batch(waves, ct.convert_options(kind))
    _check(kind, jobs, pcms, outs, status, rate=lambda i: 48000)
    assert status == [0] * len(jobs)


@pytest.mark.parametrize("kind", (W.IDSP, W.HPS))
@pytest.mark.parametrize("with_status", (True, False))
def test_a_bad_file_fails_alone_in_many_groups(kind, with_status):
    pcms = [_pcm(2, 3000 + 997 * i, i) for i in range(24)]
    loops_ = [(101 * i if kind == W.IDSP or i % 2 else 0, len(p[0]) - 1) for i, p in enumerate(pcms)]
    waves = [O.wave_write16(p, 32000, l) for p, l in zip(pcms, loops_)]
    waves[11] = waves[11][:30]  # a truncated RIFF header: refused
    o = ct.convert_options(kind, group_bytes=20000)
    if with_status:
        outs, status = ct.convert_wave_batch(waves, o)
        assert status[11] == vg._native.VGB_E_DATA and outs[11] is None
    else:
        arrs = [np.ascontiguousarray(w) for w in waves]
        n = len(arrs)
        ftab = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
        lens = (C.c_int64 * n)(*[a.size for a in arrs])
        sizes = (C.c_int64 * n)()
        vg._native.check(vg.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(o), sizes, None, None, None, None))
        assert sizes[11] == 0
        outs = [np.zeros(sizes[i], np.uint8) for i in range(n)]
        otab = (C.c_void_p * n)(*[x.ctypes.data if x.size else None for x in outs])
        vg._native.check(vg.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(o), sizes, otab, None, None, None))
    for i in range(24):
        if i == 11:
            continue
        st, want = _write(kind, pcms[i], 32000, loops_[i])
        if st == 0:
            assert outs[i].tobytes() == want.tobytes()
        elif with_status:
            assert status[i] == st and outs[i] is None
        else:
            assert outs[i].size == 0
    assert sum(_write(kind, pcms[i], 32000, loops_[i])[0] == 0 for i in range(24) if i != 11) >= 12


def test_two_bound_devices():
    import torch
    ids = (C.c_int32 * 2)(0, 1 if torch.cuda.device_count() > 1 else 0)  # device 0 twice when only one is visible
    vg._native.check(vg.lib.vgb_init_devices(ids, 2, 0))
    try:
        pcms = [_pcm(1 + i % 2 * 3, 20000 + 311 * i, i) for i in range(12)]  # 1 and 4 channels
        jobs = [(len(p), len(p[0]), (1000 + i if i % 3 else 0, len(p[0]))) for i, p in enumerate(pcms)]
        waves = [O.wave_write16(p, 44100, j[2]) for p, j in zip(pcms, jobs)]
        for kind in (W.IDSP, W.HPS):
            outs, status = ct.convert_wave_batch(waves, ct.convert_options(kind))
            _check(kind, jobs, pcms, outs, status, rate=lambda i: 44100)
            assert status[::3] == [0] * 4
    finally:
        vg._native.check(vg.lib.vgb_init(0, 0))


def test_cli_writes_both_extensions(tmp_path):
    exe = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")
    src = tmp_path / "in"
    src.mkdir()
    pcms = [_pcm(2, 30000 + 100 * i, i) for i in range(3)]
    for i, p in enumerate(pcms):
        (src / f"t{i}.wav").write_bytes(O.wave_write16(p, 32000, (0, 29000)).tobytes())
    for ext, kind in (("idsp", W.IDSP), ("hps", W.HPS)):
        dst = tmp_path / ext
        r = subprocess.run([exe, "-i", str(src), "-o", str(dst), "--out-format", ext], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        for i, p in enumerate(pcms):
            assert (dst / f"t{i}.{ext}").read_bytes() == _write(kind, p, 32000, (0, 29000))[1].tobytes()
        for fmt, name in (("pcm16", "PCM16"), ("pcm8", "PCM8")):
            r = subprocess.run([exe, "-i", str(src), "-o", str(tmp_path / "x"), "--out-format", ext, "-f", fmt], capture_output=True,
                               text=True, timeout=300)
            assert r.returncode != 0 and f"Can't use format {name} with {ext.upper()} files" in r.stderr
