"""WAVE -> .brstm / .bcstm / .bfstm on the GPU: every file byte-identical to the oracle's writer, per-file refusals in
the middle of a batch, many groups in flight, two bound devices, and the written files decoded back by the
repository's NintendoWare reader."""
import itertools
import os
import subprocess

import numpy as np
import pytest

import vgaudio_b200 as vg
from oracle import pyoracle as O
from vgaudio_b200 import containers as ct

import nw_writer_oracle as W

pytestmark = pytest.mark.gpu

KINDS = (W.BRSTM, W.BCSTM, W.BFSTM)
CODECS = (W.PCM8, W.PCM16, W.GCADPCM)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _device():
    vg._native.check(vg.lib.vgb_init(0, 0))


def _pcm(ch, n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return [(np.sin(t * (0.013 + 0.002 * c)) * 8000 + rng.normal(0, 500, n)).clip(-32768, 32767).astype(np.int16) for c in range(ch)]


def _jobs():
    """(channels, samples, loop): shorter than one block, exactly one block, many blocks; no loop, loop start 0, loop
    start on the alignment, loop end inside the last frame"""
    out = []
    for ch in (1, 2, 3, 8):
        for n in (100, 14336, 4096, 8192, 14336 * 5 + 9):
            out.append((ch, n, None))
            out.append((ch, n, (0, n)))
            if n > 30:
                out.append((ch, n, (0, n - 5)))
            if n > 14336 + 20:
                out.append((ch, n, (14336, n - 13)))
            if n > 200:  # unaligned: GcAdpcmAlignment moves the loop and re-encodes the tail
                out.append((ch, n, (100, n - 7)))
                out.append((ch, n, (n // 3 + 1, n)))
    return out


def _convert(kind, codec, waves, **kw):
    return ct.convert_wave_batch(waves, ct.convert_options(kind, nw_codec_plus1=codec + 1, **kw))


@pytest.mark.parametrize("kind,codec", list(itertools.product(KINDS, CODECS)))
@pytest.mark.parametrize("endianness", (0, 1, 2))
def test_files_are_byte_identical_to_the_oracle(kind, codec, endianness):
    if kind == W.BRSTM and endianness:
        pytest.skip("BRSTM is always big-endian")
    jobs = _jobs()
    pcms = [_pcm(ch, n, i) for i, (ch, n, _) in enumerate(jobs)]
    waves = [O.wave_write16(p, 32000 + i, loop) for i, (p, (_, _, loop)) in enumerate(zip(pcms, jobs))]
    outs, status = _convert(kind, codec, waves, nw_endianness=endianness)
    assert status == [0] * len(jobs)
    for i, (p, (ch, n, loop)) in enumerate(zip(pcms, jobs)):
        st, want = W.write(kind, codec, p, 32000 + i, loop, endianness)
        assert st == 0
        assert outs[i].tobytes() == want.tobytes(), f"job {i}: {ch} channels, {n} samples, loop {loop}"


@pytest.mark.parametrize("kind", KINDS)
def test_8bit_wave_inputs(kind):
    rng = np.random.default_rng(5)
    for codec in CODECS:
        chans = [rng.integers(0, 256, 30000, dtype=np.uint8) for _ in range(2)]
        wave = W.wave_write8(chans, 22050, (14336, 29000))
        pcm = [((c.astype(np.int16) - 0x80) << 8).astype(np.int16) for c in chans]
        outs, status = _convert(kind, codec, [wave])
        st, want = W.write(kind, codec, pcm, 22050, (14336, 29000))
        assert status == [0] and st == 0 and outs[0].tobytes() == want.tobytes()


def test_long_tracks_with_forced_segments(monkeypatch):
    monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", "7")
    n = 48000 * 180
    pcms = [_pcm(2, n, 40 + i) for i in range(2)]
    # an unaligned loop whose end sits near a decode-segment boundary (seven segments of about 88 000 frames): the tail is
    # built from samples on both sides of it
    loops = [(100003, 88163 * 14 + 9), None, (14336 * 100, n - 1)]
    pcms.append(_pcm(2, n, 42))
    waves = [O.wave_write16(p, 48000, l) for p, l in zip(pcms, loops)]
    for kind in (W.BRSTM, W.BFSTM):
        outs, status = _convert(kind, W.GCADPCM, waves)
        assert status == [0, 0, 0]
        for o, p, l in zip(outs, pcms, loops):
            assert o.tobytes() == W.write(kind, W.GCADPCM, p, 48000, l)[1].tobytes()


@pytest.mark.parametrize("with_status", (True, False))
def test_a_bad_file_fails_alone_in_many_groups(with_status):
    pcms = [_pcm(2, 3000 + 997 * i, i) for i in range(24)]
    waves = [O.wave_write16(p, 32000, (101 * i, len(p[0]) - 1)) for i, p in enumerate(pcms)]
    waves[11] = waves[11][:30]  # a truncated RIFF header: refused
    o = ct.convert_options(W.BFSTM, group_bytes=20000)
    if with_status:
        outs, status = ct.convert_wave_batch(waves, o)
        assert status[11] == vg._native.VGB_E_DATA and outs[11] is None
        good = [i for i in range(24) if i != 11]
    else:
        import ctypes as C
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
        good = [i for i in range(24) if i != 11]
    for i in good:
        assert outs[i].tobytes() == W.write(W.BFSTM, W.GCADPCM, pcms[i], 32000, (101 * i, len(pcms[i][0]) - 1))[1].tobytes()


def test_two_bound_devices():
    import ctypes as C
    import torch
    ids = (C.c_int32 * 2)(0, 1 if torch.cuda.device_count() > 1 else 0)  # device 0 twice when only one is visible
    vg._native.check(vg.lib.vgb_init_devices(ids, 2, 0))
    try:
        pcms = [_pcm(1 + i % 3, 20000 + 311 * i, i) for i in range(12)]
        waves = [O.wave_write16(p, 44100, (1000 + i, len(p[0]))) for i, p in enumerate(pcms)]
        outs, status = _convert(W.BCSTM, W.GCADPCM, waves)
        assert status == [0] * 12
        for i, (o, p) in enumerate(zip(outs, pcms)):
            assert o.tobytes() == W.write(W.BCSTM, W.GCADPCM, p, 44100, (1000 + i, len(p[0])))[1].tobytes()
    finally:
        vg._native.check(vg.lib.vgb_init(0, 0))


@pytest.mark.parametrize("kind", KINDS)
def test_written_files_decode_back(kind):
    pcms = [_pcm(2, 40000, 9), _pcm(1, 20000, 10), _pcm(2, 30000, 11)]
    loops = [(14336, 39000), None, (100, 29000)]
    waves = [O.wave_write16(p, 32000, l) for p, l in zip(pcms, loops)]
    outs, status = _convert(kind, W.GCADPCM, waves)
    assert status == [0, 0, 0]
    back, st = ct.convert_nw_to_wave_batch(outs, [kind] * 3)
    assert st == [0, 0, 0]
    from oracle import pygcalign
    for b, p, l in zip(back, pcms, loops):
        fl = W.aligned_loop(W.GCADPCM, l)[1]
        dec = []
        for c in p:
            co = O.calculate_coefficients(c)
            ad = O.encode(c, co)
            rc, (needed, _, _), _, pa = pygcalign.gc_align(14336, l[0], l[1], ad, co) if l else (0, (0, 0, 0), None, None)
            dec.append(pa if needed else O.decode(ad, co, len(c))[:fl[1] if l else len(c)])  # the aligned channel's PCM
        assert b.tobytes() == O.wave_write16(dec, 32000, fl).tobytes()


def test_cli_writes_every_extension(tmp_path):
    exe = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")
    src = tmp_path / "in"
    src.mkdir()
    pcms = [_pcm(2, 30000 + 100 * i, i) for i in range(3)]
    for i, p in enumerate(pcms):
        (src / f"t{i}.wav").write_bytes(O.wave_write16(p, 32000, (1234, 29000)).tobytes())
    for ext, kind in (("brstm", W.BRSTM), ("bcstm", W.BCSTM), ("bfstm", W.BFSTM)):
        dst = tmp_path / ext
        r = subprocess.run([exe, "-i", str(src), "-o", str(dst), "--out-format", ext], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        for i, p in enumerate(pcms):
            assert (dst / f"t{i}.{ext}").read_bytes() == W.write(kind, W.GCADPCM, p, 32000, (1234, 29000))[1].tobytes()
