""".idsp / .hps -> WAVE on the GPU: vgb_convert_idsp_hps_to_wave_batch against the oracle chain (idsp_hps_reader_oracle:
the reader restatement -> the oracle's de-interleave or the concatenation of block pieces -> the oracle's GC-ADPCM
decode -> the oracle's WAVE writer) over the writer oracle's files, a round trip through the product's own writers,
hand-built HPS chains that drive every path of hps_gather_kernel, per-file failures, the time-parallel decoder under
forced short segments, the serial arm against the segmented one, a three-minute stereo track, two bound devices and
the CLI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gc_container_writer_oracle as W
import idsp_hps_reader_oracle as R
from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")


def _pcm(ch, n, seed):
    return list(synth.batch(ch, n, 32000, first_index=seed * 8, degenerate=False))


def _enc(n, seed, ch):
    return [R.encoded(p, (seed * 31 % 500, -seed * 7 % 300)) for p in _pcm(ch, n, seed)]


LOOPS = [None, "zero", "aligned", "unaligned"]


def _loop(kind, n):
    return {None: None, "zero": (0, n), "aligned": (28 * 300, n - 5), "unaligned": (4321, n - 17)}[kind]


def _matrix():
    files, i = [], 0
    for ch in (1, 2, 3, 5, 6, 7):
        for lp in LOOPS:
            for trim in (True, False):
                n = 9000 + 997 * (i % 5)
                st, img = W.write_idsp(_pcm(ch, n, i), 32000, _loop(lp, n), trim)
                assert st == 0
                files.append((R.IDSP, img))
                i += 1
    for ch in (1, 2, 5, 6):
        for lp in LOOPS:
            n = 70000 + 997 * (i % 5)
            st, img = W.write_hps(_pcm(ch, n, i), 32000, _loop(lp, n))
            if st == 0:
                files.append((R.HPS, img))
            i += 1
    return files


def _check(ct, files):
    outs, status = ct.convert_idsp_hps_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert status == [0] * len(files), status
    for i, (kind, img) in enumerate(files):
        want = R.expected_wave(img, kind)
        assert want is not None and outs[i].tobytes() == want.tobytes(), i
    return outs


def _stats(vg):
    out = (C.c_uint64 * 5)()
    assert vg.lib.vgb_gcadpcm_debug_decode_stats(out, 5) == 0
    return list(out)


def test_converter_matches_the_oracle_chain(vg, oracle):
    from vgaudio_b200 import containers as ct

    _check(ct, _matrix())


def test_round_trip_through_the_writers(vg, oracle):
    """WAVE -> the product's IDSP / HPS writer -> this converter: equal to the oracle decode of the oracle writer's file."""
    from vgaudio_b200 import containers as ct

    for kind, ch, n, loop in ((R.IDSP, 2, 30011, (1000, 29000)), (R.HPS, 2, 100003, None), (R.IDSP, 1, 5000, None),
                              (R.HPS, 1, 70000, (0, 70000))):
        pcm = _pcm(ch, n, kind + ch)
        wave = oracle.wave_write16(pcm, 32000, loop)
        written, st = ct.convert_wave_batch([wave], ct.convert_options(kind))
        assert st == [0]
        st, ref = (W.write_idsp if kind == R.IDSP else W.write_hps)(pcm, 32000, loop)
        assert st == 0 and written[0].tobytes() == ref.tobytes()
        outs, st = ct.convert_idsp_hps_to_wave_batch(written, [kind])
        assert st == [0] and outs[0].tobytes() == R.expected_wave(ref, kind).tobytes()


def _gather_files():
    """Hand-built HPS chains for every path of hps_gather_kernel."""
    files = []
    n = 0x3000 * 2 // 16 * 14
    enc2, enc3 = _enc(n, 40, 2), _enc(n, 41, 3)
    # whole frames at 0x20 multiples on both sides: the 16-byte path
    files.append(R.hps_chain(32000, enc2, [0x1000, 0x1000, 0x1000]))
    # odd piece lengths with an exact stride: odd sources and destinations, byte-wise copies
    files.append(R.hps_chain(32000, enc3, [0x333, 0x101, 0x7, 0x1, 0x15f1, 0x80f], stride=lambda b: b, n_samples=(0x333 + 0x101 + 0x7 + 0x1 + 0x15f1) * 2 // 16 * 14))
    # strides of 4 and 8 bytes off the 16-byte grid: the 4- and 8-byte paths
    files.append(R.hps_chain(32000, enc2, [0x104, 0x208, 0x40c, 0x800], stride=lambda b: b + 4))
    files.append(R.hps_chain(32000, enc2, [0x108, 0x218, 0x408, 0x800], stride=lambda b: b + 8, odd_final=True, loop_block=1))
    # one long piece per channel: several tiles per piece
    files.append(R.hps_chain(32000, enc2, [0x2a00, 0x600]))
    # empty pieces: FinalNibble -1 gives AudioSizeBytes 0
    img = R.hps_chain(32000, enc2, [0x800, 0x400, 0x800, 0x800], n_samples=0x800 * 3 * 2 // 16 * 14)
    _, h = R.parse_hps(img)
    b = bytearray(img.tobytes())
    b[h.blocks[1]["offset"] + 4: h.blocks[1]["offset"] + 8] = (-1).to_bytes(4, "big", signed=True)
    files.append(np.frombuffer(bytes(b), np.uint8).copy())
    # the last piece of the second channel cut short by the end of the image, the sample count within what is left
    img = R.hps_chain(32000, enc2, [0x800, 0x800], n_samples=(0x800 + 0x700) * 2 // 16 * 14)
    files.append(img[: img.size - 0x100].copy())
    return files


def test_gather_paths(vg, oracle):
    from vgaudio_b200 import containers as ct

    files = _gather_files()
    for f in files:
        assert R.plan(f, R.HPS)[0] == 0
    _check(ct, [(R.HPS, f) for f in files])
    # every file alone too (a group of one: the piece table starts at tile 0)
    for f in files:
        _check(ct, [(R.HPS, f)])


def _bad_predictor(kind, frame=100):
    n = 14 * 400
    enc = _enc(n, 71, 2)
    ad = np.array(enc[1][0], np.uint8)
    ad[8 * frame] = 0x90 | (ad[8 * frame] & 0x0F)
    enc[1] = (ad, enc[1][1], enc[1][2])
    if kind == R.IDSP:
        return R.idsp_image(32000, enc, n)
    return R.hps_chain(32000, enc, [0x400, 0x400, 0x480], n_samples=n)


def test_bad_files_fail_alone(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    good = _matrix()[:3] + [(R.HPS, _gather_files()[1])]
    files = [good[0], (R.IDSP, _bad_predictor(R.IDSP)), good[1], (R.HPS, _bad_predictor(R.HPS)), (R.IDSP, good[3][1]), good[2], good[3]]
    outs, status = ct.convert_idsp_hps_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert status == [0, N.VGB_E_DATA, 0, N.VGB_E_DATA, N.VGB_E_DATA, 0, 0], status
    for i in (0, 2, 5, 6):
        assert outs[i].tobytes() == R.expected_wave(files[i][1], files[i][0]).tobytes(), i
    pick = [files[i] for i in (0, 1, 2, 6)]
    n = len(pick)
    imgs = [f for _, f in pick]
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in imgs])
    lens = (C.c_int64 * n)(*[a.size for a in imgs])
    types = (C.c_int32 * n)(*[k for k, _ in pick])
    sizes = (C.c_int64 * n)()
    assert vg.lib.vgb_convert_idsp_hps_to_wave_batch(ftab, lens, types, n, sizes, None, None) == 0
    bufs = [np.full(sizes[i], 0xEE, np.uint8) for i in range(n)]
    otab = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    assert vg.lib.vgb_convert_idsp_hps_to_wave_batch(ftab, lens, types, n, sizes, otab, None) == N.VGB_E_DATA
    assert b"predictor" in vg.lib.vgb_last_error()
    assert sizes[1] == 0 and np.all(bufs[1] == 0xEE)
    for j, i in ((0, 0), (2, 2), (3, 6)):
        assert bufs[j].tobytes() == outs[i].tobytes()


def _long_hps(seconds, seed, loop=None):
    n = seconds * 32000 + 11
    st, img = W.write_hps(_pcm(2, n, seed), 32000, loop(n) if loop else None)
    assert st == 0
    return img


def test_forced_segments_run_on_and_repair(vg, oracle, monkeypatch):
    from vgaudio_b200 import containers as ct

    monkeypatch.setenv("VGB_GC_DEC_MIN_SEG_FRAMES", "16")
    img = _long_hps(3, 90)
    for seg in ("8", "64"):
        monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", seg)
        _check(ct, [(R.HPS, img)])
        st = _stats(vg)
        assert st[0] == int(seg) and st[1] > 0, st  # run-ons ran
    # a held digital silence over most of an IDSP file: no run-on locks inside it, the cascade repairs the boundaries
    import gc_relock as G

    n = 14 * 4000
    enc = _enc(n, 91, 2)
    held = []
    for ad, co, _ in enc:
        ad2, co2 = G.silence_stimulus(np.asarray(ad, np.uint8), co, 0, 2600)
        held.append((ad2, co2, (int(ad2[0]), 1000, -1000)))
    monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", "8")
    _check(ct, [(R.IDSP, R.idsp_image(32000, held, n))])
    st = _stats(vg)
    assert st[0] == 8 and st[3] >= 1 and st[2] > 0, st


def test_serial_and_segmented_arms_give_the_same_bytes(vg, oracle, monkeypatch):
    from vgaudio_b200 import containers as ct

    files = _matrix() + [(R.HPS, f) for f in _gather_files()] + [(R.HPS, _long_hps(4, 92))]
    monkeypatch.setenv("VGB_GC_DEC_MIN_SEG_FRAMES", "16")
    seg, _ = ct.convert_idsp_hps_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert _stats(vg)[0] > 1
    monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", "1")
    ser, _ = ct.convert_idsp_hps_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert _stats(vg)[0] == 1
    assert all(a is not None and a.tobytes() == b.tobytes() for a, b in zip(seg, ser))


def test_three_minute_stereo_track(vg, oracle):
    from vgaudio_b200 import containers as ct

    img = _long_hps(180, 93, loop=lambda n: (0, n))
    out = _check(ct, [(R.HPS, img)])[0]
    assert out.size > 4 * 180 * 32000
    assert _stats(vg)[0] > 1  # the default pick cuts a lone long track into segments


def test_two_devices_give_the_same_bytes(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = _matrix() + [(R.HPS, f) for f in _gather_files()]
    one, s1 = ct.convert_idsp_hps_to_wave_batch([f for _, f in files], [k for k, _ in files])
    N.check(vg.lib.vgb_shutdown())
    try:
        N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
        two, s2 = ct.convert_idsp_hps_to_wave_batch([f for _, f in files], [k for k, _ in files])
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    assert s1 == s2 == [0] * len(files)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(one, two))


def test_cli_converts_a_mixed_directory(tmp_path, vg, oracle):
    """A directory of .idsp, .hps, .brstm and .dsp files -> WAV; every IDSP / HPS output is the oracle's.  With
    --out-format dsp the .idsp / .hps files are not taken."""
    src, out, out2 = tmp_path / "in", tmp_path / "out", tmp_path / "out2"
    src.mkdir()
    files = {}
    for i, (kind, img) in enumerate(_matrix()[::5]):
        name = f"f{i}.{'idsp' if kind == R.IDSP else 'hps'}"
        (src / name).write_bytes(img.tobytes())
        files[name] = (kind, img)
    (src / "bad.hps").write_bytes(_bad_predictor(R.HPS).tobytes())
    pcm = _pcm(1, 5000, 3)
    coefs = np.stack([oracle.calculate_coefficients(p) for p in pcm])
    (src / "c.dsp").write_bytes(oracle.dsp_write([oracle.encode(p, c) for p, c in zip(pcm, coefs)], coefs, 32000, 5000).tobytes())
    import nw_files as F

    (src / "d.brstm").write_bytes(F.encoded(oracle, F.BRSTM, F.GCADPCM, 2, 3000, seed=5).tobytes())
    r = subprocess.run([CLI, "-i", str(src), "-o", str(out), "--out-format", "wav"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 3, r.stderr  # one file failed
    assert r.stdout.startswith(f"{len(files) + 2} files converted, 1 failed"), r.stdout
    assert "bad.hps" in r.stderr
    for name, (kind, img) in files.items():
        assert (out / (name.rsplit(".", 1)[0] + ".wav")).read_bytes() == R.expected_wave(img, kind).tobytes(), name
    assert (out / "c.wav").stat().st_size == 44 + 5000 * 2 and (out / "d.wav").exists() and not (out / "bad.wav").exists()
    r = subprocess.run([CLI, "-i", str(src), "-o", str(out2), "--out-format", "dsp"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.startswith("0 files converted"), r.stdout
