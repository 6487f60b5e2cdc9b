"""NintendoWare wave files (.brwav, .bcwav, .bfwav) and prefetch streams (.bcstp, .bfstp) -> WAVE on the GPU:
vgb_convert_nw_to_wave_batch against the oracle chain (nw_wave_reader_oracle: the reader restatement -> the channel rows
ReadBytes or the de-interleave gives -> the oracle's GC-ADPCM decode or the PCM conversion -> the oracle's WAVE writer)
over the builder matrix, a mixed call where every bad file fails alone, the serial and forced-segment decode arms, a
job of thousands of sound effects over several groups, two pipelines and the CLI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import nw_files as NF
import nw_wave_files as F
import nw_wave_reader_oracle as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")
WAVE_KINDS = [(F.BRWAV, None), (F.BCWAV, False), (F.BCWAV, True), (F.BFWAV, True), (F.BFWAV, False)]
PREFETCH_KINDS = [(F.BCSTP, False), (F.BFSTP, True), (F.BFSTP, False)]


def _matrix(oracle):
    """(kind, image): wave files of every kind x codec x 1/2/3/8 channels x loop x channel layout, short final channels,
    prefetch files with one and two PDAT entries."""
    files = []
    i = 0
    for kind, be in WAVE_KINDS:
        for codec in (F.PCM8, F.PCM16, F.GCADPCM):
            for ch in (1, 2, 3, 8):
                for loop in (None, 555):
                    lay = ("ordered", "reversed", "overlap", "gaps")[i % 4]
                    files.append((kind, F.encoded(oracle, kind, codec, ch, 1500 + 1013 * (i % 6), loop=loop, seed=i, big_endian=be,
                                                  layout_kind=lay)))
                    i += 1
        for codec in (F.PCM8, F.PCM16):  # mono, its run cut short by the image's end: a shorter WAVE
            chans = F.channels(oracle, codec, 1, 3000, 40 + i, kind == F.BRWAV or bool(be))
            files.append((kind, F.rwav(codec, chans, 3000, cut=1000) if kind == F.BRWAV else
                          F.cwav(kind, codec, chans, 3000, big_endian=be, cut=1000)))
            i += 1
    for kind, be in PREFETCH_KINDS:
        for codec in (F.PCM8, F.PCM16, F.GCADPCM):
            for ch in (1, 2, 3):
                n = 9000 + 7 * i
                per = F.samples_to_bytes(n, codec)
                pre = [per] if ch == 1 else [per // 3 // 8 * 8, per - per // 3 // 8 * 8]
                files.append((kind, F.encoded(oracle, kind, codec, ch, n, seed=i, big_endian=be, prefetch=pre, interleave=0x100 * (1 + i % 3))))
                i += 1
    files.append((F.BCWAV, NF.encoded(oracle, NF.BCSTM, F.GCADPCM, 2, 4000, seed=99)))  # a CSTM read as BCWAV
    return files


def _check(ct, files):
    outs, status = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert status == [0] * len(files), status
    for i, (kind, img) in enumerate(files):
        want = R.expected_wave(img, kind)
        assert want is not None and outs[i].tobytes() == want.tobytes(), i
    return outs


@pytest.mark.parametrize("segments", [None, "1", "7"])
def test_matrix_matches_the_oracle_chain(vg, oracle, monkeypatch, segments):
    from vgaudio_b200 import containers as ct

    if segments:  # the plain serial loop, and many short segments with their splices
        monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", segments)
        monkeypatch.setenv("VGB_GC_DEC_MIN_SEG_FRAMES", "16")
    _check(ct, _matrix(oracle))


def test_serial_and_segmented_arms_give_the_same_bytes(vg, oracle, monkeypatch):
    from vgaudio_b200 import containers as ct

    files = [(k, f) for k, f in _matrix(oracle) if R.parse(f, k)[1].codec == F.GCADPCM]
    files.append((F.BFWAV, F.encoded(oracle, F.BFWAV, F.GCADPCM, 2, 14 * 9000 + 3, seed=81)))
    monkeypatch.setenv("VGB_GC_DEC_MIN_SEG_FRAMES", "16")
    seg, _ = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    monkeypatch.setenv("VGB_GC_DEC_SEGMENTS", "1")
    ser, _ = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert all(a is not None and a.tobytes() == b.tobytes() for a, b in zip(seg, ser))


def _bad_predictor(oracle, kind):
    chans = F.channels(oracle, F.GCADPCM, 2, 14 * 300, 71, kind == F.BRWAV)
    d = bytearray(chans[1].data)
    d[8 * 120] = 0xA0 | (d[8 * 120] & 0x0F)
    chans[1].data = bytes(d)
    return F.rwav(F.GCADPCM, chans, 14 * 300) if kind == F.BRWAV else F.cwav(kind, F.GCADPCM, chans, 14 * 300)


def test_bad_files_fail_alone(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    good = [(NF.BRSTM, NF.encoded(oracle, NF.BRSTM, F.GCADPCM, 2, 9000, loop=100, seed=30)),
            (F.BCWAV, F.encoded(oracle, F.BCWAV, F.GCADPCM, 2, 7000, loop=50, seed=31)),
            (F.BFSTP, F.encoded(oracle, F.BFSTP, F.PCM16, 2, 6000, seed=32)),
            (F.BRWAV, F.encoded(oracle, F.BRWAV, F.PCM8, 1, 5000, seed=33))]
    short_gc = F.cwav(F.BFWAV, F.GCADPCM, F.channels(oracle, F.GCADPCM, 2, 5000, 34, True), 5000, cut=50)
    uneven = F.cwav(F.BCWAV, F.PCM16, F.channels(oracle, F.PCM16, 2, 5000, 35, False), 5000, cut=60)
    files = [good[0], (F.BCWAV, F.encoded(oracle, F.BCWAV, F.PCM8, 1, 100, seed=36, magic=b"XXXX")), good[1],
             (F.BFWAV, short_gc), (F.BCWAV, uneven), good[2], (F.BRWAV, _bad_predictor(oracle, F.BRWAV)),
             (F.BFWAV, _bad_predictor(oracle, F.BFWAV)), good[3], (7, good[0][1])]
    outs, status = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert status == [0, N.VGB_E_DATA, 0, N.VGB_E_ARG, N.VGB_E_DATA, 0, N.VGB_E_DATA, N.VGB_E_DATA, 0, N.VGB_E_ARG], status
    for i in (0, 2, 5, 8):
        assert outs[i].tobytes() == R.expected_wave(files[i][1], files[i][0]).tobytes(), i
    assert R.expected_wave(files[6][1], F.BRWAV) is None and R.expected_wave(files[7][1], F.BFWAV) is None


def _effects(oracle, count, seed):
    """`count` sound effects of 0.05-2 s at 32 kHz, mono and stereo, GC-ADPCM and PCM16, as .bcwav / .bfwav / .brwav.
    The GC-ADPCM channels are prefixes of a few long encodings: a prefix of whole bytes decodes to the prefix."""
    rng = np.random.default_rng(seed)
    long_n = 2 * 32000
    pcm = NF.pcm_channels(4, long_n, seed)
    gc = NF.gc_channels(oracle, pcm)
    files = []
    for i in range(count):
        n = int(rng.integers(1600, long_n + 1))
        ch = 1 + i % 2
        kind = (F.BCWAV, F.BFWAV, F.BRWAV)[i % 3]
        codec = F.GCADPCM if i % 4 < 3 else F.PCM16
        be = kind != F.BCWAV
        pick = [(i + c) % 4 for c in range(ch)]
        if codec == F.GCADPCM:
            chans = [NF.Channel(gc[p].data[: NF.gc_bytes(n)], gc[p].coefs, 0, gc[p].start) for p in pick]
        else:
            chans = NF.pcm16_channels([pcm[p][:n] for p in pick], be)
        loop = int(rng.integers(0, n)) if i % 5 == 0 else None
        files.append((kind, F.rwav(codec, chans, n, loop=loop) if kind == F.BRWAV else F.cwav(kind, codec, chans, n, loop=loop)))
    return files


def test_thousands_of_sound_effects_in_one_call(vg, oracle):
    from vgaudio_b200 import containers as ct

    files = _effects(oracle, 6000, 5)
    # what a file takes of a group's 1 GiB: PCM + WAVE + its runs + its rows
    group = sum(2 * R.wave_size(f, k) + h.audio_length + h.output_size * h.channel_count for k, f in files for h in [R.parse(f, k)[1]])
    assert group > 1.2 * (1 << 30)
    outs, status = ct.convert_nw_to_wave_batch([f for _, f in files], [k for k, _ in files])
    assert status == [0] * len(files)
    for i in range(0, len(files), 7):
        assert outs[i].tobytes() == R.expected_wave(files[i][1], files[i][0]).tobytes(), i


def test_two_pipelines_give_the_same_bytes(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = _matrix(oracle) + _effects(oracle, 300, 6)
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


def test_cli_converts_every_new_extension(tmp_path, vg, oracle):
    """A directory of every new extension next to a .brstm, a .dsp and a .wav -> WAV; every output is the oracle's, a
    bad file is reported by name; with --out-format dsp none of the new extensions is listed."""
    src, out, out2 = tmp_path / "nw", tmp_path / "out", tmp_path / "out2"
    src.mkdir()
    exts = {F.BRWAV: ("brwav", "rwav"), F.BCWAV: ("bcwav", "cwav", "bms"), F.BFWAV: ("bfwav",), F.BCSTP: ("bcstp",), F.BFSTP: ("bfstp",)}
    files = {}
    i = 0
    for kind, names in exts.items():
        for ext in names:
            codec = (F.PCM8, F.PCM16, F.GCADPCM)[i % 3]
            img = F.encoded(oracle, kind, codec, 1 + i % 2, 4000 + 100 * i, loop=200 if codec == F.GCADPCM and kind < F.BCSTP else None, seed=i)
            name = f"f{i}.{ext}"
            (src / name).write_bytes(img.tobytes())
            files[name] = (kind, img)
            i += 1
    brstm = NF.encoded(oracle, NF.BRSTM, F.GCADPCM, 2, 5000, seed=50)
    (src / "s.brstm").write_bytes(brstm.tobytes())
    files["s.brstm"] = (NF.BRSTM, brstm)
    (src / "bad.bfwav").write_bytes(_bad_predictor(oracle, F.BFWAV).tobytes())
    pcm = [NF.pcm_channels(1, 5000, 3)[0]]
    coefs = np.stack([oracle.calculate_coefficients(p) for p in pcm])
    (src / "c.dsp").write_bytes(oracle.dsp_write([oracle.encode(p, c) for p, c in zip(pcm, coefs)], coefs, 32000, 5000).tobytes())
    (src / "w.wav").write_bytes(oracle.wave_write16(pcm, 32000, None).tobytes())
    r = subprocess.run([CLI, "-i", str(src), "-o", str(out), "--out-format", "wav"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 3, r.stderr  # one file failed
    assert r.stdout.startswith(f"{len(files) + 1} files converted, 1 failed"), r.stdout
    assert "bad.bfwav" in r.stderr
    for name, (kind, img) in files.items():
        assert (out / (name.rsplit(".", 1)[0] + ".wav")).read_bytes() == R.expected_wave(img, kind).tobytes(), name
    assert (out / "c.wav").stat().st_size == 44 + 5000 * 2 and not (out / "bad.wav").exists()
    r = subprocess.run([CLI, "-i", str(src), "-o", str(out2), "--out-format", "dsp"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith("1 files converted, 0 failed"), (r.stdout, r.stderr)
    assert sorted(p.name for p in out2.iterdir()) == ["w.dsp"]
