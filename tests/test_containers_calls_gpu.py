"""The single-shot container calls (WAVE read, DSP write / read, ADX write / crypt, HCA write / crypt) on wide batches
(at least 20 caller rows, which the library copies with one batched driver call) and narrow ones (fewer than 16), with
zero-length rows and empty channels, against the CPU oracle: their kernel launch counts, an error in the last file or
row (the call fails with its message and the next good call is right), and container calls interleaved with a codec
host call and the batch converter."""
import ctypes as C

import numpy as np
import pytest

from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu


def _pcm(n_ch, n, first):
    return [synth.channel(first + c, max(n, 1))[:n] for c in range(n_ch)]


def _launches(vg):
    return int(vg.lib.vgb_kernel_launch_count())


def _raises(vg, code, message, fn, *args):
    with pytest.raises(vg.VgbError) as e:
        fn(*args)
    assert e.value.code == code and str(e.value).endswith(": " + message), str(e.value)


def _null_last(monkeypatch, name, arg):
    """Make the C call `name` see NULL in the last entry of its pointer-table argument `arg`."""
    from vgaudio_b200 import _native as N

    real = getattr(N.lib, name)

    def call(*args):
        tab = args[arg]
        tab[len(tab) - 1] = None
        return real(*args)

    monkeypatch.setattr(N.lib, name, call)


# ---- WAVE ---------------------------------------------------------------------------------------------------------------
def _wave_files(oracle, n_files, first):
    rng = np.random.default_rng(first)
    files = []
    for k in range(n_files):
        ch = int(rng.integers(1, 9))
        n = int(rng.choice([1, 7, 300, 2048, 5001, 12345]))
        loop = (3, n) if k % 5 == 0 and n > 3 else None
        files.append(oracle.wave_write16(_pcm(ch, n, first + 8 * k), 44100, loop))
    return files


def _wave_read_raw(vg, files, infos, rows):
    """vgb_wave_read_batch on explicit descriptions: files / rows may hold None."""
    from vgaudio_b200 import _native as N

    n = len(files)
    ftab = (C.c_void_p * n)(*[f.ctypes.data if f is not None else None for f in files])
    lens = (C.c_int64 * n)(*[f.size if f is not None else 0 for f in files])
    rtab = (C.c_void_p * max(len(rows), 1))(*[r.ctypes.data if r is not None else None for r in rows])
    arr = (N.VgbWaveInfo * n)(*infos)
    N.check(N.lib.vgb_wave_read_batch(ftab, lens, arr, n, rtab))


def _check_wave_read(vg, oracle, files):
    from vgaudio_b200 import containers as ct

    before = _launches(vg)
    got = ct.wave_read_batch(files)
    assert _launches(vg) - before == 1
    for f, (info, rows) in zip(files, got):
        want = oracle.wave_read(f, oracle.wave_parse(f)[1])
        assert len(rows) == len(want) and all(np.array_equal(a, b) for a, b in zip(rows, want))


@pytest.mark.parametrize("n_files", [40, 5])
def test_wave_read_wide_and_narrow(vg, oracle, n_files):
    from vgaudio_b200 import containers as ct

    files = _wave_files(oracle, n_files, 1000 + n_files)
    _check_wave_read(vg, oracle, files)
    # a file described with no samples: its rows are empty, and neither it nor they need a pointer
    infos = [ct.wave_parse(f) for f in files]
    empty = type(infos[0]).from_buffer_copy(infos[1])
    empty.sample_count = empty.data_offset = 0
    files2 = [files[0], None, *files[2:]]
    infos2 = [infos[0], empty, *infos[2:]]
    rows = []
    for k, info in enumerate(infos2):
        rows += [np.zeros(info.sample_count, np.int16) if k != 1 else None for _ in range(info.channel_count)]
    _wave_read_raw(vg, files2, infos2, rows)
    r = 0
    for k, (f, info) in enumerate(zip(files2, infos2)):
        if k != 1:
            want = oracle.wave_read(f, oracle.wave_parse(f)[1])
            assert all(np.array_equal(a, b) for a, b in zip(rows[r:r + info.channel_count], want))
        r += info.channel_count


def test_wave_read_error_in_last_row_or_file(vg, oracle, monkeypatch):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = _wave_files(oracle, 24, 77)
    infos = [ct.wave_parse(f) for f in files]
    n_rows = sum(i.channel_count for i in infos)
    with monkeypatch.context() as m:
        _null_last(m, "vgb_wave_read_batch", 4)
        _raises(vg, N.VGB_E_ARG, f"pcm_out[{n_rows - 1}] is NULL", ct.wave_read_batch, files)
    bad = type(infos[0]).from_buffer_copy(infos[-1])
    bad.data_offset = files[-1].size
    rows = [np.zeros(i.sample_count, np.int16) for i in infos for _ in range(i.channel_count)]
    _raises(vg, N.VGB_E_ARG, f"file {len(files) - 1}: the description does not fit an image of {files[-1].size} bytes",
            _wave_read_raw, vg, files, infos[:-1] + [bad], rows)
    _check_wave_read(vg, oracle, files)


# ---- DSP ----------------------------------------------------------------------------------------------------------------
def _dsp_cases(oracle, n_files, first):
    """(DspFile for the writer, the oracle's file) for n_files files of 1-3 channels; file 1 has no samples."""
    from vgaudio_b200 import containers as ct

    out = []
    for k in range(n_files):
        ch = 1 + k % 3
        n = 0 if k == 1 else 14 * (20 + 37 * k) + k % 14
        pcm = _pcm(ch, n, first + 4 * k)
        if n:
            coefs = np.stack([oracle.calculate_coefficients(p) for p in pcm])
            adpcm = [oracle.encode(p, c) for p, c in zip(pcm, coefs)]
        else:
            coefs, adpcm = np.zeros((ch, 16), np.int16), [np.zeros(0, np.uint8) for _ in range(ch)]
        spi = 14 * 8 if k % 4 == 2 else 0
        loop = (14, n) if k % 6 == 3 else None
        ctx = np.stack([np.array(oracle.gc_loop_context(a, oracle.decode(a, c, n), loop[0]), dtype=np.int16)
                        for a, c in zip(adpcm, coefs)]) if loop else None
        f = ct.DspFile(adpcm, coefs, 32000, n, loop is not None, loop[0] if loop else 0, loop[1] if loop else 0, ctx,
                       samples_per_interleave=spi)
        out.append((f, oracle.dsp_write(adpcm, coefs, 32000, n, loop, ctx, None, None, spi or 0x3800)))
    return out


def _check_dsp_write(vg, cases):
    from vgaudio_b200 import containers as ct

    before = _launches(vg)
    got = ct.dsp_write_batch([c[0] for c in cases])
    assert _launches(vg) - before == 1
    for k, (g, (_, w)) in enumerate(zip(got, cases)):
        assert g.tobytes() == w.tobytes(), k


def _check_dsp_read(vg, oracle, images):
    from vgaudio_b200 import containers as ct

    multi = sum(1 for f in images if ct.dsp_parse(f).channel_count > 1 and ct.dsp_parse(f).sample_count > 0)
    before = _launches(vg)
    got = ct.dsp_read_batch(images)
    assert _launches(vg) - before == multi
    for k, (f, (_, rows)) in enumerate(zip(images, got)):
        want = oracle.dsp_read_data(f, oracle.dsp_parse(f)[1])
        assert len(rows) == len(want) and all(a.tobytes() == b.tobytes() for a, b in zip(rows, want)), k


@pytest.mark.parametrize("n_files", [24, 4])
def test_dsp_write_and_read_wide_and_narrow(vg, oracle, n_files):
    cases = _dsp_cases(oracle, n_files, 2000 + n_files)
    _check_dsp_write(vg, cases)
    _check_dsp_read(vg, oracle, [c[1] for c in cases])


def test_dsp_errors_in_last_file(vg, oracle, monkeypatch):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    cases = _dsp_cases(oracle, 24, 3000)
    images = [c[1] for c in cases]
    with monkeypatch.context() as m:
        _null_last(m, "vgb_dsp_write_batch", 7)
        _raises(vg, N.VGB_E_ARG, f"files_out[{len(cases) - 1}] is NULL", ct.dsp_write_batch, [c[0] for c in cases])
    _check_dsp_write(vg, cases)
    # frames per interleave 0 in the last (three-channel) file
    last = len(images) - 1
    assert ct.dsp_parse(images[last]).channel_count == 3
    real = N.lib.vgb_dsp_read_batch

    def zero_interleave(ftab, lens, infos, n, rtab):
        infos[n - 1].frames_per_interleave = 0
        return real(ftab, lens, infos, n, rtab)

    with monkeypatch.context() as m:
        m.setattr(N.lib, "vgb_dsp_read_batch", zero_interleave)
        _raises(vg, N.VGB_E_DATA, f"file {last}: frames per interleave is 0", ct.dsp_read_batch, images)
    with monkeypatch.context() as m:
        _null_last(m, "vgb_dsp_read_batch", 4)
        n_rows = sum(ct.dsp_parse(f).channel_count for f in images)
        _raises(vg, N.VGB_E_ARG, f"adpcm_out[{n_rows - 1}] is NULL", ct.dsp_read_batch, images)
    _check_dsp_read(vg, oracle, images)


# ---- CRI ADX ------------------------------------------------------------------------------------------------------------
def _adx_cases(oracle, n_files, first):
    from vgaudio_b200 import containers as ct

    out = []
    for k in range(n_files):
        ch = 1 + k % 2
        n = 1 if k == 2 else 500 + 211 * k
        enc = [oracle.adx_encode(p) for p in _pcm(ch, n, first + 2 * k)]
        audio, hist = [e[0] for e in enc], [e[1] for e in enc]
        out.append((ct.AdxFile(audio, hist, 48000, n), oracle.adx_write(audio, hist, 48000, n)))
    return out


def _check_adx_write(vg, cases):
    from vgaudio_b200 import containers as ct

    before = _launches(vg)
    got = ct.adx_write_batch([c[0] for c in cases])
    assert _launches(vg) - before == 1
    for k, (g, (_, w)) in enumerate(zip(got, cases)):
        assert g.tobytes() == w.tobytes(), k


def _check_adx_crypt(vg, oracle, audio, key):
    from vgaudio_b200 import containers as ct

    before = _launches(vg)
    got = ct.adx_crypt(audio, key, 8, 18)
    assert _launches(vg) - before == 1
    want = oracle.adx_crypt(audio, (key.seed, key.mult, key.inc), 8, 18)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))


@pytest.mark.parametrize("n_files", [20, 3])
def test_adx_write_and_crypt_wide_and_narrow(vg, oracle, n_files):
    from vgaudio_b200 import containers as ct

    _check_adx_write(vg, _adx_cases(oracle, n_files, 4000 + n_files))
    audio = [oracle.adx_encode(p)[0] for p in _pcm(n_files, 6000, 4100)]
    audio[-1][:] = 0  # an empty channel: the key stream skips its frames
    _check_adx_crypt(vg, oracle, audio, ct.adx_key(key_string="karaage"))


def test_adx_errors_in_last_file_or_row(vg, oracle, monkeypatch):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    cases = _adx_cases(oracle, 20, 5000)
    with monkeypatch.context() as m:
        _null_last(m, "vgb_adx_write_batch", 6)
        _raises(vg, N.VGB_E_ARG, f"files_out[{len(cases) - 1}] is NULL", ct.adx_write_batch, [c[0] for c in cases])
    _check_adx_write(vg, cases)
    audio = [oracle.adx_encode(p)[0] for p in _pcm(20, 3000, 5100)]
    key = ct.adx_key(key_code=123456789012)
    with monkeypatch.context() as m:
        _null_last(m, "vgb_adx_crypt_batch", 0)
        _raises(vg, N.VGB_E_ARG, "audio[19] is NULL", ct.adx_crypt, audio, key, 8, 18)
    _check_adx_crypt(vg, oracle, audio, key)


# ---- CRI HCA ------------------------------------------------------------------------------------------------------------
def _hca_streams(oracle):
    """Two encoded mono streams of one frame size: (oracle info, frames[frame_count, frame_size]) each."""
    return [oracle.hca_encode(_pcm(1, 40000, 6000 + k), 48000) for k in range(2)]


def _hca_cut(oracle, streams, counts):
    """Streams of the given frame counts cut from the encoded ones: (oracle info, frames) each."""
    out = []
    for k, n in enumerate(counts):
        oi, fr = streams[k % len(streams)]
        info = type(oi).from_buffer_copy(oi)
        info.frame_count = n
        out.append((info, np.ascontiguousarray(fr[:n])))
    return out


def _native_info(oi):
    from vgaudio_b200 import _native as N

    p = N.VgbHcaInfo()
    for name, _ in N.VgbHcaInfo._fields_:
        setattr(p, name, getattr(oi, name))
    return p


def _check_hca_crypt(vg, oracle, cut):
    from vgaudio_b200 import containers as ct

    fs = cut[0][0].frame_size
    before = _launches(vg)
    got = ct.hca_crypt_batch([c[1] for c in cut], fs, 56, 0xCC55463930DBE1AB)
    assert _launches(vg) - before == 1
    table = oracle.hca_key_tables(56, 0xCC55463930DBE1AB)[1]
    for k, (g, (_, fr)) in enumerate(zip(got, cut)):
        assert g.tobytes() == oracle.hca_crypt_frames(fr, fs, table).tobytes(), k


def _check_hca_write(vg, oracle, cut):
    from vgaudio_b200 import containers as ct

    before = _launches(vg)
    got = ct.hca_write_batch([_native_info(c[0]) for c in cut], [c[1] for c in cut], 1)
    assert _launches(vg) - before == 1
    table = oracle.hca_key_tables(1)[1]
    for k, (g, (oi, fr)) in enumerate(zip(got, cut)):
        assert g.tobytes() == oracle.hca_write(oi, fr, table, 1).tobytes(), k


@pytest.mark.parametrize("n_streams", [32, 6])
def test_hca_crypt_and_write_wide_and_narrow(vg, oracle, n_streams):
    streams = _hca_streams(oracle)
    counts = [0 if k % 7 == 3 else 1 + (k * 5) % 30 for k in range(n_streams)]
    cut = _hca_cut(oracle, streams, counts)
    _check_hca_crypt(vg, oracle, cut)
    _check_hca_write(vg, oracle, cut[:20])


def test_hca_errors_in_last_stream_or_file(vg, oracle, monkeypatch):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    cut = _hca_cut(oracle, _hca_streams(oracle), [1 + k % 9 for k in range(32)])
    fs = cut[0][0].frame_size
    with monkeypatch.context() as m:
        _null_last(m, "vgb_hca_crypt_batch", 0)
        _raises(vg, N.VGB_E_ARG, "frames[31] is NULL", ct.hca_crypt_batch, [c[1] for c in cut], fs, 56, 0xCC55463930DBE1AB)
    _check_hca_crypt(vg, oracle, cut)
    with monkeypatch.context() as m:
        _null_last(m, "vgb_hca_write_batch", 7)
        _raises(vg, N.VGB_E_ARG, "files_out[19] is NULL", ct.hca_write_batch, [_native_info(c[0]) for c in cut[:20]],
                [c[1] for c in cut[:20]], 1)
    _check_hca_write(vg, oracle, cut[:20])


# ---- container calls between a codec host call and the batch converter ------------------------------------------------------
def test_container_calls_interleaved_with_codec_and_converter(vg, oracle):
    from vgaudio_b200 import containers as ct

    waves = _wave_files(oracle, 20, 7000)
    dsp = _dsp_cases(oracle, 20, 7100)
    pcm = synth.batch(24, 14 * 300 + 5)
    conv_in = [oracle.wave_write16(_pcm(2, 9000, 7200), 48000, (100, 8000)), oracle.wave_write16(_pcm(1, 5000, 7210), 32000, None)]

    def encode():
        coefs, adpcm = vg.gcadpcm.encode_batch(pcm)
        for c in (0, 11, 23):
            co = oracle.calculate_coefficients(pcm[c])
            assert np.array_equal(coefs[c], co) and adpcm[c].tobytes() == oracle.encode(pcm[c], co).tobytes()

    def convert():
        outs, status = ct.convert_wave_batch(conv_in, ct.convert_options(ct.CONTAINER_DSP))
        assert status == [0, 0]
        for out, (ch, n, first, rate, loop) in zip(outs, [(2, 9000, 7200, 48000, (100, 8000)), (1, 5000, 7210, 32000, None)]):
            p = _pcm(ch, n, first)
            coefs = np.stack([oracle.calculate_coefficients(x) for x in p])
            adpcm = [oracle.encode(x, c) for x, c in zip(p, coefs)]
            ctx = np.stack([np.array(oracle.gc_loop_context(a, oracle.decode(a, c, n), loop[0]), dtype=np.int16)
                            for a, c in zip(adpcm, coefs)]) if loop else None
            assert out.tobytes() == oracle.dsp_write(adpcm, coefs, rate, n, loop, ctx).tobytes()

    for step in (encode, lambda: _check_wave_read(vg, oracle, waves), convert, lambda: _check_dsp_write(vg, dsp), encode,
                 lambda: _check_dsp_read(vg, oracle, [c[1] for c in dsp]), convert, lambda: _check_wave_read(vg, oracle, waves)):
        step()
