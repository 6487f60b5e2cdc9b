"""Every CRI ADX decode path against the throwing restatement of CriAdxCodec.Decode (adx_decode_ref): the serial decoder
behind vgb_adx_decode_batch, the time-parallel decoder behind vgb_adx_decode_dev / vgb_adx_decode_dev_status, the
.adx -> WAVE batch converter and the .adx -> .dsp transcode.  Where the reference returns, every path gives its PCM bit
for bit; where it throws (coefs[filterNum] past the four Fixed rows or the one row of the other types, in a frame that
yields a sample), the channel calls fail with VGB_E_DATA naming the lowest faulting channel with the message of its
kind, the file calls fail that file alone, and the next clean call is exact.

The streams (adx_decode_ref.clean_streams / fault_streams) cover every type and version, frame sizes 18, 3, 9 and 255,
padding 0, odd, past a frame and past the sample count (the silent head frame), counts on and off the serial decoder's
8-frame groups, and a fault frame with each filter number at the head, in a serial group, in a remainder frame, at a
forced segment boundary, inside a run-on, in the partial tail and past frameCount."""
import ctypes as C

import numpy as np
import pytest

import adx_decode_ref as D
import transcode_oracle as T

pytestmark = pytest.mark.gpu

E_DATA = -2


@pytest.fixture(scope="module")
def matrix():
    """(clean, faults, silent): every stream with the reference's verdict attached as .pcm / .err."""
    out = (D.clean_streams(), D.fault_streams(), D.fault_streams(silent=True))
    for s in out[0] + out[1] + out[2]:
        pcm, s.err = D.verdict(s.data, s.n, **s.params())
        s.pcm = None if pcm is None else np.array(pcm, np.int16)
    assert all(s.err is None for s in out[0])
    return out


def _env(monkeypatch, groups="1", segments="1"):
    monkeypatch.setenv("VGB_PIPELINE_GROUPS", groups)
    monkeypatch.setenv("VGB_ADX_DEC_SEGMENTS", segments)
    monkeypatch.setenv("VGB_ADX_DEC_MIN_SEG_FRAMES", "8")


def _cfg(s: D.Stream):
    from vgaudio_b200 import criadx

    return criadx.CriAdxParameters(48000, 500, s.frame_size, s.version, s.history, s.padding, s.type)


def _message(ch, type, unit="channel"):
    """The converter's message for each kind of fault (containers_abi.inc, AdxFront::faults)."""
    if type == D.FIXED:
        return f"{unit} {ch}: a Fixed-type frame selects a filter outside 0..3"
    return f"{unit} {ch}: a frame of type {type} selects a filter other than 0"


def _host(streams):
    """vgb_adx_decode_batch: (status, message, [pcm rows])."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import criadx

    try:
        return 0, "", criadx.decode_batch([s.data for s in streams], [s.n for s in streams], [_cfg(s) for s in streams])
    except N.VgbError as e:
        return e.code, str(e), None


def _k0(s: D.Stream) -> int:
    spf = (s.frame_size - 2) * 2
    start = s.padding % spf if s.padding > 0 else 0
    return max(min(s.n, spf) - start, 0)


def _dev(vg, streams):
    """vgb_adx_decode_dev + vgb_adx_decode_dev_status on one slab per direction: rows at 16-byte aligned offsets and at
    odd ones, outputs whose body frames start at addresses that select the 16-, 4- and 2-byte stores in turn, guard
    samples between them.  Returns (status, message, [pcm rows], stats, store widths)."""
    import torch

    from vgaudio_b200 import _native as N
    from vgaudio_b200 import criadx

    a_off, p_off, widths = [], [], []
    ia = ip = 0
    for i, s in enumerate(streams):
        a = (ia + 15) // 16 * 16 + (5 if i % 4 == 3 else 0)
        a_off.append(a)
        ia = a + s.data.size + 8
        want = (0, 2, 1)[i % 3]  # (pcm_off + k0) % 8: 0 -> 16-byte stores, 2 -> 4-byte, 1 -> 2-byte
        p = ip + 8
        while (p + _k0(s)) % 8 != want:
            p += 1
        p_off.append(p)
        widths.append((16, 4, 2)[i % 3])
        ip = p + s.n
    d_adpcm = torch.zeros(ia + 16, dtype=torch.uint8)
    for a, s in zip(a_off, streams):
        d_adpcm[a: a + s.data.size] = torch.from_numpy(s.data)
    d_adpcm = d_adpcm.cuda()
    d_pcm = torch.full((ip + 16,), 0x5555, dtype=torch.int16, device="cuda")
    assert d_pcm.data_ptr() % 16 == 0 and d_adpcm.data_ptr() % 16 == 0
    st, msg = 0, ""
    c32 = np.array([s.n for s in streams], np.int32)
    params = criadx._params_array([_cfg(s) for s in streams])
    ws = torch.empty(vg.lib.vgb_adx_decode_workspace_bytes(c32.ctypes.data, C.cast(params, C.c_void_p), len(streams)),
                     dtype=torch.uint8, device="cuda")
    try:
        criadx.decode_dev(d_adpcm, a_off, [s.data.size for s in streams], c32, [_cfg(s) for s in streams], d_pcm, p_off, workspace=ws)
    except N.VgbError as e:
        st, msg = e.code, str(e)
    stats = (C.c_uint64 * 5)()
    N.check(vg.lib.vgb_adx_debug_decode_stats(stats, 5))  # ws is still allocated
    pcm = d_pcm.cpu().numpy()
    written = np.zeros(pcm.size, bool)
    for p, s in zip(p_off, streams):
        written[p: p + s.n] = True
    assert (pcm[~written] == 0x5555).all(), "a decode wrote outside its channel's samples"
    return st, msg, [pcm[p: p + s.n] for p, s in zip(p_off, streams)], list(stats), widths


def _companions(cases, clean):
    """For each case: a clean stream in front of it and, behind it, a later throwing case of the matrix (so that the
    channel named is the lowest faulting one, across the pipeline's groups)."""
    throwing = [s for s in cases if s.err is not None]
    for i, s in enumerate(cases):
        yield s, clean[(7 * i) % (len(clean) - 1)], clean[(7 * i + 3) % (len(clean) - 1)], throwing[(i * 5 + 1) % len(throwing)]


def _check_fault_calls(call, cases, clean):
    """Each case as channel 1 of [clean, case, clean, throwing case]: a throwing case is named with its kind's
    message, else channel 3 is; then the case alone (or the clean channel when it throws) decodes exactly."""
    for s, a, b, later in _companions(cases, clean):
        st, msg = call([a, s, b, later])[:2]
        named, kind = (1, s.type) if s.err is not None else (3, later.type)
        assert st == E_DATA and _message(named, kind) in msg, (s, st, msg)
        follow = a if s.err is not None else s
        st, msg, pcm = call([follow])[:3]
        assert st == 0 and np.array_equal(pcm[0], follow.pcm), (s, st, msg)


# ---- vgb_adx_decode_batch: the serial decoder -------------------------------------------------------------------------
@pytest.mark.parametrize("groups", ["1", "3"])
def test_host_batch_clean_matrix(vg, matrix, monkeypatch, groups):
    _env(monkeypatch, groups=groups)
    clean = matrix[0]
    st, msg, pcm = _host(clean)
    assert st == 0, msg
    for s, p in zip(clean, pcm):
        assert np.array_equal(p, s.pcm), s


@pytest.mark.parametrize("groups", ["1", "3"])
@pytest.mark.parametrize("type", [D.FIXED, D.LINEAR, D.EXPONENTIAL])
def test_host_batch_filter_faults(vg, matrix, monkeypatch, type, groups):
    _env(monkeypatch, groups=groups)
    _check_fault_calls(_host, [s for s in matrix[1] if s.type == type], matrix[0])


@pytest.mark.parametrize("groups", ["1", "3"])
@pytest.mark.parametrize("type", [D.FIXED, D.LINEAR, D.EXPONENTIAL])
def test_host_batch_silent_head(vg, matrix, monkeypatch, type, groups):
    """The head frame of a count <= padding % spf yields nothing and is never checked; one more sample and it is."""
    _env(monkeypatch, groups=groups)
    cases = [s for s in matrix[2] if s.type == type]
    assert {s.placement for s in cases if s.err is None and s.filter > 3} == {"silent_head"}
    _check_fault_calls(_host, cases, matrix[0])


# ---- vgb_adx_decode_dev: the time-parallel decoder ---------------------------------------------------------------------
@pytest.mark.parametrize("segments", ["1", "8"])
def test_device_clean_matrix(vg, matrix, monkeypatch, segments):
    _env(monkeypatch, segments=segments)
    clean = matrix[0]
    st, msg, pcm, stats, widths = _dev(vg, clean)
    assert st == 0, msg
    for s, p in zip(clean, pcm):
        assert np.array_equal(p, s.pcm), s
    assert {w for s, w in zip(clean, widths) if s.frame_size == 18 and s.n > 32 * 16} == {16, 4, 2}
    assert stats[0] == int(segments)
    if segments == "8":
        assert stats[1] > 0   # frames decoded by the boundary run-ons
        assert stats[3] >= 1  # boundaries the cascade repaired (the silence stream)


@pytest.mark.parametrize("segments", ["1", "8"])
@pytest.mark.parametrize("type", [D.FIXED, D.LINEAR, D.EXPONENTIAL])
def test_device_filter_faults(vg, matrix, monkeypatch, type, segments):
    _env(monkeypatch, segments=segments)
    _check_fault_calls(lambda streams: _dev(vg, streams), [s for s in matrix[1] if s.type == type], matrix[0])


@pytest.mark.parametrize("segments", ["1", "8"])
@pytest.mark.parametrize("type", [D.FIXED, D.LINEAR, D.EXPONENTIAL])
def test_device_silent_head(vg, matrix, monkeypatch, type, segments):
    _env(monkeypatch, segments=segments)
    _check_fault_calls(lambda streams: _dev(vg, streams), [s for s in matrix[2] if s.type == type], matrix[0])


# ---- the batch converter and the transcode: one file per clean row, one stereo file per case --------------------------
def _files(matrix):
    """(image, [streams of its channels]): every clean row alone, every case beside a clean row of its geometry."""
    rng = np.random.default_rng(5)
    files = [([s], D.adx_image([s])) for s in matrix[0]]
    for s in matrix[1] + matrix[2]:
        mate = D.Stream(D.clean_row(rng, s.type, s.frame_size, s.padding, s.n), s.n, s.frame_size, s.version, s.padding, s.type)
        files.append(([mate, s], D.adx_image([mate, s])))
    return files


def _file_pcm(chans):
    """The reference over a file's channels (history 0, as ToPcm16 decodes them): [pcm] or None where one throws."""
    got = [D.verdict(c.data, c.n, **c.params(history=0)) for c in chans]
    return None if any(e is not None for _, e in got) else [np.array(p, np.int16) for p, _ in got]


@pytest.mark.parametrize("groups,segments", [("1", "1"), ("3", "8")])
def test_converter_fails_each_throwing_file_alone(vg, oracle, matrix, monkeypatch, groups, segments):
    from vgaudio_b200 import containers as ct

    _env(monkeypatch, groups, segments)
    files = _files(matrix)
    outs, status = ct.convert_adx_to_wave_batch([img for _, img in files])
    failed = 0
    for (chans, img), out, st in zip(files, outs, status):
        pcm = _file_pcm(chans)
        if pcm is None:
            assert st == E_DATA and out is None, chans[-1]
            failed += 1
        else:
            assert st == 0 and out.tobytes() == oracle.wave_write16(pcm, 48000).tobytes(), chans[-1]
    assert failed > 500
    chans, img = files[1]
    outs, status = ct.convert_adx_to_wave_batch([img])
    assert status == [0] and outs[0].tobytes() == oracle.wave_write16(_file_pcm(chans), 48000).tobytes()


@pytest.mark.parametrize("groups,segments", [("1", "1"), ("3", "8")])
def test_transcode_to_dsp_fails_each_throwing_file_alone(vg, oracle, matrix, monkeypatch, groups, segments):
    from vgaudio_b200 import containers as ct

    _env(monkeypatch, groups, segments)
    files = _files(matrix)[::3]
    outs, status = ct.transcode_batch([img for _, img in files], [T.ADX] * len(files), ct.convert_options(T.DSP))
    failed = 0
    for (chans, img), out, st in zip(files, outs, status):
        if _file_pcm(chans) is None:
            assert st == E_DATA and out is None, chans[-1]
            failed += 1
        else:
            assert st == 0 and out.tobytes() == T.expected(img, T.ADX, T.DSP).tobytes(), chans[-1]
    assert failed > 100
    chans, img = files[1]
    outs, status = ct.transcode_batch([img], [T.ADX], ct.convert_options(T.DSP))
    assert status == [0] and outs[0].tobytes() == T.expected(img, T.ADX, T.DSP).tobytes()
