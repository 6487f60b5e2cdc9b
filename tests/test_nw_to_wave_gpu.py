""".brstm / .bcstm / .bfstm -> WAVE on the GPU: vgb_convert_nw_to_wave_batch against the oracle chain (nw_reader_oracle:
the reader restatement -> the oracle's de-interleave -> the oracle's GC-ADPCM decode or the PCM conversion -> the oracle's
WAVE writer) for every format x codec x channel count x loop case, per-file failures in a mixed batch, the time-parallel
decoder under forced small segments (the stats tap proving that run-ons lock and that the cascade repairs a held
silence), the serial arm against the segmented one, a three-minute stereo track, two bound devices and the CLI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gc_relock as G
import nw_files as F
import nw_reader_oracle as R
from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")
FORMATS = [(F.BRSTM, None), (F.BCSTM, False), (F.BFSTM, False), (F.BFSTM, True)]
EXT = {F.BRSTM: "brstm", F.BCSTM: "bcstm", F.BFSTM: "bfstm"}


def _matrix(oracle):
    """(kind, image): every format x codec x channel count x loop case, plus the region and interleave variants."""
    files = []
    i = 0
    for kind, be in FORMATS:
        for codec in (F.PCM8, F.PCM16, F.GCADPCM):
            for ch in (1, 2, 8):
                for loop in (None, 777):
                    n = 2000 + 997 * (i % 7)
                    files.append((kind, F.encoded(oracle, kind, codec, ch, n, loop=loop, seed=i, big_endian=be,
                                                  interleave=0x200 * (1 + i % 3), start_hist=(i * 37 % 900, -i * 11 % 700))))
                    i += 1
    for kind, be in FORMATS:
        n = 4321
        full = F.samples_to_bytes(n, F.GCADPCM)
        for in_size in (full - 333, full + 101):  # zero-filled / truncated rows
            files.append((kind, F.encoded(oracle, kind, F.GCADPCM, 2, n, seed=500 + in_size, big_endian=be, interleave=0x100, in_size=in_size)))
        files.append((kind, F.encoded(oracle, kind, F.PCM16, 2, 999, seed=7, big_endian=be, interleave=0)))  # interleave 0: zeros
        files.append((kind, F.encoded(oracle, kind, F.GCADPCM, 1, 0, seed=8, big_endian=be)))             # empty
        files.append((kind, F.encoded(oracle, kind, F.GCADPCM, 3, 13, seed=9, big_endian=be)))            # one partial frame
    for v in F.BCSTM_VERSIONS:
        files.append((F.BCSTM, F.encoded(oracle, F.BCSTM, F.GCADPCM, 2, 3000, loop=3000, seed=11, version=v)))
    for v in F.BFSTM_VERSIONS:
        files.append((F.BFSTM, F.encoded(oracle, F.BFSTM, F.PCM8, 2, 3000, seed=12, version=v, regions=1, big_endian=True)))
    files.append((F.BFSTM, F.encoded(oracle, F.BCSTM, F.PCM16, 2, 1000, seed=13)))   # BCFstmReader takes either magic
    return files


def _check(ct, files):
    outs, status = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert status == [0] * len(files), status
    for i, (kind, img) in enumerate(files):
        want = R.expected_wave(img, kind)
        assert want is not None and outs[i].tobytes() == want.tobytes(), i
    return outs


def _stats(vg):
    out = (C.c_uint64 * 5)()
    assert vg.lib.vgb_gcadpcm_debug_decode_stats(out, 5) == 0
    return list(out)


@pytest.mark.parametrize("segments", [None, "1", "7"])
def test_converter_matches_the_oracle_chain(vg, oracle, monkeypatch, segments):
    from vgaudio_b200 import containers as ct

    if segments:  # the plain serial loop, and many short segments with their splices
        monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", segments)
        monkeypatch.setenv("VGB_GC_DEC_MIN_SEG_FRAMES", "16")
    _check(ct, _matrix(oracle))


def _bad_predictor(oracle, kind, frame=100):
    """Stereo GC-ADPCM file whose channel 1 selects predictor 9 on one frame."""
    pcm = F.pcm_channels(2, 14 * 400, 71)
    chans = F.gc_channels(oracle, pcm)
    d = bytearray(chans[1].data)
    d[8 * frame] = 0x90 | (d[8 * frame] & 0x0F)
    chans[1].data = bytes(d)
    return F.build(kind, F.GCADPCM, chans, 14 * 400)


def test_bad_files_fail_alone(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    good = [(F.BRSTM, F.encoded(oracle, F.BRSTM, F.GCADPCM, 2, 9000, loop=100, seed=30)),
            (F.BCSTM, F.encoded(oracle, F.BCSTM, F.PCM16, 1, 6000, seed=31)),
            (F.BFSTM, F.encoded(oracle, F.BFSTM, F.GCADPCM, 8, 5000, seed=32, big_endian=True))]
    ima = F.encoded(oracle, F.BRSTM, F.PCM16, 2, 500, seed=33)
    ima[0x48 + 24] = 3
    files = [good[0], (F.BRSTM, _bad_predictor(oracle, F.BRSTM)), (F.BRSTM, F.encoded(oracle, F.BCSTM, F.PCM8, 1, 100, seed=34)),
             good[1], (F.BCSTM, F.encoded(oracle, F.BCSTM, F.PCM8, 1, 100, loop=101, seed=35)), (F.BRSTM, ima),
             (F.BFSTM, _bad_predictor(oracle, F.BFSTM, 399)), good[2]]
    outs, status = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert status == [0, N.VGB_E_DATA, N.VGB_E_DATA, 0, N.VGB_E_ARG, N.VGB_E_DATA, N.VGB_E_DATA, 0], status
    for i in (0, 3, 7):
        assert outs[i].tobytes() == R.expected_wave(files[i][1], files[i][0]).tobytes(), i
    assert R.expected_wave(files[1][1], F.BRSTM) is None and R.expected_wave(files[6][1], F.BFSTM) is None
    # without status_out: the good files are written, the call fails with the decoder's error
    pick = [files[i] for i in (0, 1, 3, 7)]
    n = len(pick)
    imgs = [f for _, f in pick]
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in imgs])
    lens = (C.c_int64 * n)(*[a.size for a in imgs])
    types = (C.c_int32 * n)(*[k for k, _ in pick])
    sizes = (C.c_int64 * n)()
    assert vg.lib.vgb_convert_nw_to_wave_batch(ftab, lens, types, n, sizes, None, None) == 0
    bufs = [np.full(sizes[i], 0xEE, np.uint8) for i in range(n)]
    otab = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    assert vg.lib.vgb_convert_nw_to_wave_batch(ftab, lens, types, n, sizes, otab, None) == N.VGB_E_DATA
    assert b"predictor" in vg.lib.vgb_last_error()
    assert sizes[1] == 0 and np.all(bufs[1] == 0xEE)
    for j, i in ((0, 0), (2, 3), (3, 7)):
        assert bufs[j].tobytes() == outs[i].tobytes()


def _silence_file(oracle, frames, lo, hi, hist=(1000, -1000)):
    """Stereo GC-ADPCM .bcstm whose channels start from `hist` and hold a digital silence over frames [lo, hi)."""
    pcm = F.pcm_channels(2, 14 * frames, 91)
    chans = F.gc_channels(oracle, pcm)
    for k in chans:
        ad, co = G.silence_stimulus(np.frombuffer(k.data, np.uint8), k.coefs, lo, hi)
        k.data, k.coefs, k.start = ad.tobytes(), co, (0, hist[0], hist[1])
    return F.build(F.BCSTM, F.GCADPCM, chans, 14 * frames)


def test_forced_segments_lock_and_the_cascade_repairs(vg, oracle, monkeypatch):
    from vgaudio_b200 import containers as ct

    monkeypatch.setenv("VGB_GC_DEC_MIN_SEG_FRAMES", "16")
    loud = (F.BRSTM, F.encoded(oracle, F.BRSTM, F.GCADPCM, 2, 14 * 6000 + 5, seed=80))
    for seg in ("8", "64", "256"):
        monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", seg)
        _check(ct, [loud])
        st = _stats(vg)
        seg_len = (-(-6000 // int(seg)) + 3) // 4 * 4  # gc_dec_seg_len: ceil(full / segments) on a 4-frame grid
        assert st[0] == int(seg) and st[1] > 0 and 0 < st[4] <= seg_len, st   # run-ons ran inside their segments ...
        assert st[1] < 2 * (int(seg) - 1) * seg_len // 2, st                  # ... and most stopped early: they locked
    # a held silence over segments 0..5 of 8: a run-on cannot lock inside it, the cascade carries the true pair across
    monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", "8")
    silent = (F.BCSTM, _silence_file(oracle, 4000, 0, 2600))
    _check(ct, [silent])
    st = _stats(vg)
    assert st[0] == 8 and st[3] >= 1 and st[2] > 0, st
    # silence in the middle of the track, entered with the true (nonzero) pair
    mid = (F.BCSTM, _silence_file(oracle, 4000, 1200, 3300))
    _check(ct, [mid])
    st = _stats(vg)
    assert st[3] >= 1 and st[2] > 0, st


def test_serial_and_segmented_arms_give_the_same_bytes(vg, oracle, monkeypatch):
    from vgaudio_b200 import containers as ct

    files = [(k, f) for k, f in _matrix(oracle) if R.parse(f, k)[1].codec == F.GCADPCM]
    files += [(F.BCSTM, _silence_file(oracle, 3000, 100, 2000)), (F.BRSTM, F.encoded(oracle, F.BRSTM, F.GCADPCM, 2, 14 * 9000 + 3, seed=81))]
    # the reference suite's full-scale sine: a wrong pair never re-locks on it, so the cascade decodes the channel serially
    sine = F.gc_channels(oracle, [synth.reference_sine(14 * 5000 + 9, 261.63, 48000)])
    files.append((F.BFSTM, F.build(F.BFSTM, F.GCADPCM, sine, 14 * 5000 + 9, big_endian=True)))
    monkeypatch.setenv("VGB_GC_DEC_MIN_SEG_FRAMES", "16")
    seg, _ = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert _stats(vg)[0] > 1
    monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", "1")
    ser, _ = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert _stats(vg)[0] == 1
    assert all(a is not None and a.tobytes() == b.tobytes() for a, b in zip(seg, ser))


def test_three_minute_stereo_track(vg, oracle):
    from vgaudio_b200 import containers as ct

    n = 180 * 32000 + 11
    img = F.encoded(oracle, F.BRSTM, F.GCADPCM, 2, n, loop=32000 * 7, seed=90, interleave=0x2000)
    out = _check(ct, [(F.BRSTM, img)])[0]
    assert out.size > 4 * n
    assert _stats(vg)[0] > 1  # the default pick cuts a lone long track into segments


def test_two_devices_give_the_same_bytes(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = _matrix(oracle)
    one, s1 = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    N.check(vg.lib.vgb_shutdown())
    try:
        N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
        two, s2 = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    assert s1 == s2 == [0] * len(files)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(one, two))


def test_cli_converts_a_mixed_directory(tmp_path, vg, oracle):
    """A directory of .brstm, .bcstm and .bfstm files (and a .dsp) -> WAV; every output is the oracle's."""
    src, out = tmp_path / "nw", tmp_path / "out"
    src.mkdir()
    files = {}
    for i, (kind, be) in enumerate(FORMATS):
        for codec in (F.PCM8, F.PCM16, F.GCADPCM):
            name = f"f{i}_{codec}.{EXT[kind]}"
            img = F.encoded(oracle, kind, codec, 1 + i, 5000 + 100 * i, loop=300 if codec == F.GCADPCM else None, seed=10 * i + codec,
                            big_endian=be)
            (src / name).write_bytes(img.tobytes())
            files[name] = (kind, img)
    bad = _bad_predictor(oracle, F.BRSTM)
    (src / "bad.brstm").write_bytes(bad.tobytes())
    pcm = [F.pcm_channels(1, 5000, 3)[0]]
    coefs = np.stack([oracle.calculate_coefficients(p) for p in pcm])
    (src / "c.dsp").write_bytes(oracle.dsp_write([oracle.encode(p, c) for p, c in zip(pcm, coefs)], coefs, 32000, 5000).tobytes())
    r = subprocess.run([CLI, "-i", str(src), "-o", str(out), "--out-format", "wav"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 3, r.stderr  # one file failed
    assert r.stdout.startswith(f"{len(files) + 1} files converted, 1 failed"), r.stdout
    assert "bad.brstm" in r.stderr
    for name, (kind, img) in files.items():
        assert (out / (name.rsplit(".", 1)[0] + ".wav")).read_bytes() == R.expected_wave(img, kind).tobytes(), name
    assert (out / "c.wav").stat().st_size == 44 + 5000 * 2 and not (out / "bad.wav").exists()
