""".adx -> WAVE on the GPU: vgb_convert_adx_to_wave_batch against the oracle chain (adx_reader_oracle: the parse ->
oracle.adx_crypt -> oracle.adx_decode -> oracle.wave_write16), per-file failures, the time-parallel decode
vgb_adx_decode_dev against vgb_adx_decode_batch and the oracle (with forced small segments, the stats tap proving that
run-ons lock and the cascade repairs), two bound devices and a WAV -> ADX -> WAV round trip through the CLI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import adx_files as F
import adx_reader_oracle as R
from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")


def _keys(oracle):
    return oracle.adx_key(key_code=F.KEY_CODE), oracle.adx_key(key_string=F.KEY_STRING)


def _job(oracle):
    """(image, oracle key or None) over types, versions, frame sizes, looping, keys, empty files and 1..8 channels."""
    code, string = _keys(oracle)
    files = []
    for i, (ch, fs, version, type) in enumerate([(1, 18, 4, 3), (2, 18, 4, 2), (2, 18, 3, 4), (3, 18, 3, 3), (4, 9, 4, 3), (5, 33, 4, 4),
                                                 (6, 3, 3, 2), (7, 130, 4, 3), (8, 18, 4, 4), (2, 18, 4, 3)]):
        files.append((F.encoded(oracle, ch, 3000 + 1700 * i, 48000 if i % 2 else 44100, fs, version, type, seed=10 * i), None))
    for i, (ch, fs, version) in enumerate([(1, 18, 4), (2, 18, 4), (2, 18, 3), (3, 11, 4)]):  # looping: alignment padding
        files.append((F.encoded(oracle, ch, 40000, 32000, fs, version, 3, (3001 + 7 * i, 35000), seed=50 + i), None))
    files.append((F.encoded(oracle, 2, 20000, 48000, 18, 4, 3, (1234, 18000), code, 9, seed=60), code))
    files.append((F.encoded(oracle, 1, 15000, 44100, 18, 4, 3, None, string, 8, seed=61), string))
    files.append((F.encoded(oracle, 2, 9000, 48000, 18, 3, 4, None, code, 9, seed=62), code))
    files.append((F.header(samples=0, inserted=0, loop_count=0, header_size=60), None))  # empty
    files.append((F.header(samples=70, inserted=-5, loop_count=0, header_size=60,
                           audio=np.random.default_rng(3).integers(0, 32, 6 * 18, np.uint8).tobytes()), None))  # negative padding
    for rate in (0, -44100):  # CalculateCoefficients of a rate <= 0: (0, 0) from NaN for 0, ordinary doubles below
        pcm = [synth.channel(70 + c, 4000, 48000, degenerate=False) for c in range(2)]
        enc = [oracle.adx_encode(p, 48000, 18, 4, 0, 3, 0) for p in pcm]
        img = oracle.adx_write([e[0] for e in enc], [e[1] for e in enc], 48000, 4000)
        img[8:12] = np.frombuffer(int(rate).to_bytes(4, "big", signed=True), np.uint8)
        files.append((img, None))
    files.append((_silent_head(np.random.default_rng(4)), None))
    return files


def _silent_head(rng):
    """Stereo Linear file whose unaligned count (10) is below InsertedSamples % 32 (20): the head frame yields no sample, so
    CriAdxCodec.Decode never indexes the coefficient table with its filter number, which selects filter 2 here."""
    audio = rng.integers(0, 32, 2 * 18, np.uint8)
    audio[0] |= 0x40
    return F.header(samples=30, inserted=20, loop_count=0, header_size=60, audio=audio.tobytes())


def _check_job(ct, oracle, files, key):
    outs, status = ct.convert_adx_to_wave_batch([f for f, _ in files], key)
    assert status == [0] * len(files), status
    for i, (img, k) in enumerate(files):
        want = R.expected_wave(img, k)
        assert want is not None and outs[i].tobytes() == want.tobytes(), i
    return outs


@pytest.mark.parametrize("segments", [None, "1", "7"])
def test_converter_matches_the_oracle_chain(vg, oracle, monkeypatch, segments):
    from vgaudio_b200 import containers as ct

    if segments:  # the plain serial loop, and many short segments with their splices
        monkeypatch.setenv("VGB_ADX_DEC_SEGMENTS", segments)
        monkeypatch.setenv("VGB_ADX_DEC_MIN_SEG_FRAMES", "16")
    code, string = _keys(oracle)
    files = _job(oracle)
    _check_job(ct, oracle, [f for f in files if f[1] != string], ct.adx_key(key_code=F.KEY_CODE))
    _check_job(ct, oracle, [f for f in files if f[1] != code], ct.adx_key(key_string=F.KEY_STRING))


def _bad_filter(oracle, type):
    img = F.encoded(oracle, 2, 6000, 48000, 18, 4, type, seed=71)
    _, h = R.adx_parse(img)
    img[h.audio_offset + 18 * 2 * 100 + 18] |= 0x80 if type == 2 else 0x40  # frame 100 of channel 1
    return img


def test_bad_files_fail_alone(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    good = [F.encoded(oracle, 2, 8000, 48000, seed=30), F.encoded(oracle, 1, 6000, 44100, 18, 4, 2, (100, 5000), seed=31)]
    keyed = F.encoded(oracle, 2, 5000, 48000, 18, 4, 3, None, oracle.adx_key(key_code=F.KEY_CODE), 9, seed=32)
    short = F.encoded(oracle, 1, 6000, 48000, seed=33)
    _, h = R.adx_parse(short)
    short = short[: h.audio_offset + h.audio_size - 1].copy()
    bad_loop = F.header(samples=64, inserted=8, loop_count=1, loop=(1, 4, 0, 100, 0), header_size=80)
    negative = F.header(samples=100, inserted=200, loop_count=0, header_size=60)
    files = [good[0], _bad_filter(oracle, 2), keyed, short, good[1], bad_loop, negative, _bad_filter(oracle, 3)]
    outs, status = ct.convert_adx_to_wave_batch(files)  # no key: the type-9 file cannot be decrypted
    assert status[0] == 0 and status[4] == 0
    assert [status[i] for i in (1, 2, 3, 6, 7)] == [N.VGB_E_DATA] * 5 and status[5] == N.VGB_E_ARG
    assert all(outs[i] is None for i in (1, 2, 3, 5, 6, 7))
    assert outs[0].tobytes() == R.expected_wave(good[0]).tobytes()
    assert outs[4].tobytes() == R.expected_wave(good[1]).tobytes()
    # without status_out a filter found on the device fails the call after the good files were written
    n = 2
    arrs = [good[0], files[1]]
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
    lens = (C.c_int64 * n)(*[a.size for a in arrs])
    sizes = (C.c_int64 * n)()
    assert vg.lib.vgb_convert_adx_to_wave_batch(ftab, lens, n, None, sizes, None, None) == 0
    bufs = [np.zeros(sizes[i], np.uint8) for i in range(n)]
    otab = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    assert vg.lib.vgb_convert_adx_to_wave_batch(ftab, lens, n, None, sizes, otab, None) == N.VGB_E_DATA
    assert bufs[0].tobytes() == R.expected_wave(good[0]).tobytes() and sizes[1] == 0


# ---- the device-resident, time-parallel decode ----------------------------------------------------------------------
def _decode_dev(vg, rows, counts, configs):
    """vgb_adx_decode_dev on torch buffers with odd offsets (every store width and the per-byte input path);
    returns (status, [pcm rows], stats)."""
    import torch

    from vgaudio_b200 import criadx

    a_off = np.cumsum([0] + [r.size + 16 + (7 if i % 3 == 1 else 0) for i, r in enumerate(rows)])[:-1].astype(np.int64)
    a_off = [o if i % 3 == 1 else (o + 15) // 16 * 16 for i, o in enumerate(a_off)]
    d_adpcm = torch.zeros(int(a_off[-1] + rows[-1].size + 32), dtype=torch.uint8, device="cuda")
    for o, r in zip(a_off, rows):
        d_adpcm[int(o): int(o) + r.size] = torch.from_numpy(r).cuda()
    p_off = np.cumsum([0] + [c + 5 for c in counts])[:-1].astype(np.int64) + 3
    d_pcm = torch.full((int(p_off[-1] + counts[-1] + 8),), 0x5555, dtype=torch.int16, device="cuda")
    st = 0
    c32 = np.array(counts, np.int32)
    ws = torch.empty(vg.lib.vgb_adx_decode_workspace_bytes(c32.ctypes.data, C.cast(criadx._params_array(configs), C.c_void_p), len(rows)),
                     dtype=torch.uint8, device="cuda")
    try:
        criadx.decode_dev(d_adpcm, a_off, [r.size for r in rows], counts, configs, d_pcm, p_off, workspace=ws)
    except vg._native.VgbError as e:
        st = e.code
    stats = (C.c_uint64 * 5)()
    vg._native.check(vg.lib.vgb_adx_debug_decode_stats(stats, 5))  # ws is still allocated
    pcm = d_pcm.cpu().numpy()
    return st, [pcm[p_off[i]: p_off[i] + counts[i]] for i in range(len(rows))], list(stats)


def _burst_then_silence(rng, frames, loud):
    """Linear-type 18-byte frames: `loud` frames of random nibbles at large scales, then all-zero frames (digital silence)."""
    a = rng.integers(0, 256, (frames, 18), dtype=np.uint8)
    a[:, 0] &= 0x0f  # filter 0, scale < 0x1000
    a[loud:] = 0
    return a.ravel()


@pytest.mark.parametrize("segments,min_seg", [(None, None), ("5", "8"), ("64", "1")])
def test_decode_dev_matches_batch_and_oracle(vg, oracle, monkeypatch, segments, min_seg):
    from vgaudio_b200 import criadx

    if segments:
        monkeypatch.setenv("VGB_ADX_DEC_SEGMENTS", segments)
        monkeypatch.setenv("VGB_ADX_DEC_MIN_SEG_FRAMES", min_seg)
    rng = np.random.default_rng(11)
    rows, counts, configs = [], [], []
    for i, (fs, version, type, padding, history) in enumerate([
            (18, 4, 3, 0, 0), (18, 3, 4, 0, 1234), (18, 4, 2, 37, -20000), (18, 4, 3, 1000, 0), (9, 4, 3, 3, 5), (255, 3, 4, 600, 0),
            (18, 4, 3, 31, 0), (3, 4, 2, 1, 7), (18, 3, 3, 0, 0), (18, 4, 4, 64, 0)]):
        spf = (fs - 2) * 2
        n = int(rng.integers(1, 3000)) * 32 + int(rng.integers(0, 40))
        pcm = synth.channel(90 + i, n + padding, 48000, degenerate=False)
        if fs <= 130:
            data, _ = oracle.adx_encode(pcm[:n], 48000, fs, version, padding, type, 1)
        else:  # beyond the oracle encoder's frame: random frames of the right type
            frames = -(-(n + padding) // spf)
            data = rng.integers(0, 256, (frames, fs), dtype=np.uint8)
            data[:, 0] &= 0x0f
            data = data.ravel()
        rows.append(np.ascontiguousarray(data, np.uint8))
        counts.append(n)
        configs.append(criadx.CriAdxParameters(48000, 500, fs, version, history, padding, type))
    rows.append(_burst_then_silence(rng, 4000, 300))  # a pair stuck under the >> 12: boundaries in the silence never re-lock
    counts.append(4000 * 32)
    configs.append(criadx.CriAdxParameters(48000, 500, 18, 4, 0, 0, 3))
    st, dev, stats = _decode_dev(vg, rows, counts, configs)
    assert st == 0
    host = criadx.decode_batch(rows, counts, configs)
    for i, (r, n, c) in enumerate(zip(rows, counts, configs)):
        want = oracle.adx_decode(r, n, c.sample_rate, c.highpass_frequency, c.frame_size, c.version, c.history, c.padding, c.type)
        assert np.array_equal(dev[i], want) and np.array_equal(host[i], want), i
    silent = dev[-1][300 * 32:]
    assert silent[-1] != 0  # the stimulus: the true pair stays nonzero to the end, a start from (0, 0) decodes zeros
    if segments:
        assert stats[0] == int(segments) and stats[1] > 0  # segments, frames decoded by run-ons
        assert stats[2] > 0 and stats[3] >= 1             # the cascade repaired the boundaries in the silence
        assert stats[4] <= 64 * 32                         # run-ons that locked stayed inside their segments


def test_bad_fixed_filter_names_its_channel(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import criadx

    rows, counts, configs = [], [], []
    for i in range(5):
        pcm = synth.channel(i, 5000, 48000, degenerate=False)
        rows.append(oracle.adx_encode(pcm, 48000, 18, 4, 0, 2, 1)[0])
        counts.append(5000)
        configs.append(criadx.CriAdxParameters(48000, 500, 18, 4, 0, 0, 2, 1))
    rows[3][18 * 77] |= 0x80
    rows[4][18 * 3] |= 0x80
    st, _, _ = _decode_dev(vg, rows, counts, configs)
    assert st == N.VGB_E_DATA and b"channel 3:" in vg.lib.vgb_last_error()
    with pytest.raises(N.VgbError) as e:
        criadx.decode_batch(rows, counts, configs)
    assert e.value.code == N.VGB_E_DATA and b"channel 3:" in vg.lib.vgb_last_error()


def test_two_devices_give_the_same_bytes(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = [f for f, k in _job(oracle) if k is None]
    one, s1 = ct.convert_adx_to_wave_batch(files)
    N.check(vg.lib.vgb_shutdown())
    try:
        N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
        two, s2 = ct.convert_adx_to_wave_batch(files)
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    assert s1 == s2 == [0] * len(files)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(one, two))


def test_cli_round_trip_on_a_mixed_directory(tmp_path, vg, oracle):
    """WAV -> ADX (keyed, looping) with the CLI, then a directory of .dsp, .hca and .adx files -> WAV."""
    from vgaudio_b200 import containers as ct

    wav_in, adx_dir, out = tmp_path / "wav", tmp_path / "adx", tmp_path / "out"
    wav_in.mkdir()
    waves = {"a.wav": oracle.wave_write16([synth.channel(40 + c, 20000, 48000, degenerate=False) for c in range(2)], 48000, (1000, 18000)),
             "b.wav": oracle.wave_write16([synth.channel(44, 15000, 44100, degenerate=False)], 44100)}
    for name, data in waves.items():
        (wav_in / name).write_bytes(data.tobytes())
    r = subprocess.run([CLI, "-i", str(wav_in), "-o", str(adx_dir), "--out-format", "adx", "--keystring", F.KEY_STRING],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    pcm = [synth.channel(60, 5000, 32000, degenerate=False)]
    coefs = np.stack([oracle.calculate_coefficients(p) for p in pcm])
    (adx_dir / "c.dsp").write_bytes(oracle.dsp_write([oracle.encode(p, c) for p, c in zip(pcm, coefs)], coefs, 32000, 5000).tobytes())
    hca_info, frames = oracle.hca_encode([synth.channel(61, 9000, 48000, degenerate=False)], 48000, 2)
    (adx_dir / "d.hca").write_bytes(oracle.hca_write(hca_info, frames).tobytes())
    r = subprocess.run([CLI, "-i", str(adx_dir), "-o", str(out), "--out-format", "wav", "--keystring", F.KEY_STRING],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.startswith("4 files converted, 0 failed"), r.stdout
    key = oracle.adx_key(key_string=F.KEY_STRING)
    for name in ("a", "b"):
        img = np.frombuffer((adx_dir / f"{name}.adx").read_bytes(), np.uint8)
        assert R.adx_parse(img)[1].revision == 8
        assert (out / f"{name}.wav").read_bytes() == R.expected_wave(img, key).tobytes()
    assert (out / "c.wav").stat().st_size == 44 + 5000 * 2 and (out / "d.wav").exists()
    # the library call gives the same bytes as the CLI
    outs, st = ct.convert_adx_to_wave_batch([np.frombuffer((adx_dir / "a.adx").read_bytes(), np.uint8)], ct.adx_key(key_string=F.KEY_STRING))
    assert st == [0] and outs[0].tobytes() == (out / "a.wav").read_bytes()


@pytest.mark.parametrize("shift_in,shift_out", [(1, 0), (0, 1), (3, 5), (8, 4)])
def test_decode_dev_on_offset_tensor_views(vg, oracle, shift_in, shift_out):
    """Base pointers that are not 16-byte aligned (tensor views at an element offset) pick the per-byte input path and a
    narrower store from the absolute addresses and decode bit-exactly."""
    import torch

    from vgaudio_b200 import criadx

    rows, counts, configs = [], [], []
    for i, padding in enumerate((0, 13, 45)):
        n = 3000 + 97 * i
        data, _ = oracle.adx_encode(synth.channel(80 + i, n + padding, 48000, degenerate=False)[:n], 48000, 18, 4, padding, 3, 0)
        rows.append(np.ascontiguousarray(data, np.uint8))
        counts.append(n)
        configs.append(criadx.CriAdxParameters(48000, 500, 18, 4, 0, padding, 3))
    a_off = np.cumsum([0] + [(r.size + 15) // 16 * 16 for r in rows])[:-1].astype(np.int64)
    p_off = np.cumsum([0] + [(c + 7) // 8 * 8 for c in counts])[:-1].astype(np.int64)
    base_in = torch.zeros(int(a_off[-1] + rows[-1].size + 32), dtype=torch.uint8, device="cuda")
    d_adpcm = base_in[shift_in:]
    for o, r in zip(a_off, rows):
        d_adpcm[int(o): int(o) + r.size] = torch.from_numpy(r).cuda()
    base_out = torch.full((int(p_off[-1] + counts[-1] + 16),), 0x5555, dtype=torch.int16, device="cuda")
    d_pcm = base_out[shift_out:]
    ws = criadx.decode_dev(d_adpcm, a_off, [r.size for r in rows], counts, configs, d_pcm, p_off)
    assert ws.numel() > 0
    pcm = d_pcm.cpu().numpy()
    for r, n, c, o in zip(rows, counts, configs, p_off):
        want = oracle.adx_decode(r, n, 48000, 500, 18, 4, 0, c.padding, 3)
        assert np.array_equal(pcm[o: o + n], want)


def test_misaligned_pcm_or_workspace_is_refused(vg):
    """An int16 output at an odd address or a workspace off an 8-byte boundary is VGB_E_ARG, before any launch."""
    import torch

    from vgaudio_b200 import _native as N
    from vgaudio_b200 import criadx

    rows = np.zeros(18 * 4, np.uint8)
    cfg = criadx.CriAdxParameters(48000, 500, 18, 4, 0, 0, 3)
    params = C.cast(criadx._params_array([cfg]), C.c_void_p)
    counts, nb, off = np.array([100], np.int32), np.array([rows.size], np.int32), np.zeros(1, np.int64)
    d_adpcm = torch.from_numpy(rows).cuda()
    raw = torch.zeros(512, dtype=torch.uint8, device="cuda")
    ws = torch.zeros(vg.lib.vgb_adx_decode_workspace_bytes(counts.ctypes.data, params, 1) + 16, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    call = lambda pcm_ptr, ws_ptr: vg.lib.vgb_adx_decode_dev(d_adpcm.data_ptr(), off.ctypes.data, nb.ctypes.data, counts.ctypes.data, params, 1,
                                                             pcm_ptr, off.ctypes.data, ws_ptr, ws.numel() - 16, stream)
    assert call(raw.data_ptr() + 1, ws.data_ptr()) == N.VGB_E_ARG
    assert call(raw.data_ptr(), ws.data_ptr() + 4) == N.VGB_E_ARG
    assert call(raw.data_ptr(), ws.data_ptr()) == N.VGB_OK
    N.check(vg.lib.vgb_adx_decode_dev_status(ws.data_ptr(), 1, stream))


def test_frame_that_yields_no_sample_never_checks_its_filter(vg, oracle):
    """The head frame of a channel whose count is below padding % spf is read but yields nothing: a filter number the
    table cannot index there is no error, in the converter and in vgb_adx_decode_dev, as in CriAdxCodec.Decode."""
    from vgaudio_b200 import containers as ct
    from vgaudio_b200 import criadx

    img = _silent_head(np.random.default_rng(5))
    want = R.expected_wave(img)
    assert want is not None
    outs, st = ct.convert_adx_to_wave_batch([img])
    assert st == [0] and outs[0].tobytes() == want.tobytes()
    row = np.ascontiguousarray(img[64: 64 + 18])  # channel 0's only frame: filter bits 2 in a Linear-type header
    cfg = criadx.CriAdxParameters(48000, 500, 18, 4, 0, 20, 3)
    st, dev, _ = _decode_dev(vg, [row], [10], [cfg])
    assert st == 0 and np.array_equal(dev[0], np.zeros(10, np.int16))
