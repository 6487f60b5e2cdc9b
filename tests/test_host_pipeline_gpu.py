"""The host-pointer batch calls of GC-ADPCM decode, ADX encode/decode and HCA encode/decode cut their units into groups
and pipeline them (H2D of group g+1 under the kernels of group g and the D2H of group g-1).  VGB_PIPELINE_GROUPS
forces the group count.  On a seeded ragged batch with empty units, every group count gives the oracle's bytes, encode
progress deltas sum to the frame total, and a hostile unit in the last group is named by the caller's index."""
import numpy as np
import pytest

from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu

GROUPS = (1, 3, 7)
N_UNITS = 30
EMPTY = (0, 9, 17)  # unit indices with no samples; the last unit is never empty


@pytest.fixture
def pipeline_groups(monkeypatch):
    """Calls `fn` once per forced group count and returns the results in GROUPS order."""

    def run(fn):
        out = []
        for g in GROUPS:
            monkeypatch.setenv("VGB_PIPELINE_GROUPS", str(g))
            out.append(fn())
        monkeypatch.delenv("VGB_PIPELINE_GROUPS")
        return out

    return run


def _lengths(seed, lo=1, hi=9000):
    n = np.random.default_rng(seed).integers(lo, hi, N_UNITS)
    n[list(EMPTY)] = 0
    return [int(x) for x in n]


def _channels(seed):
    return [synth.channel(seed + c, max(n, 1), degenerate=False)[:n] for c, n in enumerate(_lengths(seed))]


def _same(results):
    first = results[0]
    for r in results[1:]:
        assert len(r) == len(first)
        for a, b in zip(first, r):
            assert np.array_equal(np.asarray(a), np.asarray(b))


def _gc_inputs(oracle):
    pcm = _channels(700)
    coefs = np.zeros((N_UNITS, 16), dtype=np.int16)
    adpcm = []
    for c, x in enumerate(pcm):
        if len(x):
            coefs[c] = oracle.calculate_coefficients(x)
            adpcm.append(oracle.encode(x, coefs[c]))
        else:
            adpcm.append(np.zeros(0, dtype=np.uint8))
    return pcm, coefs, adpcm


def test_gcadpcm_decode(vg, oracle, pipeline_groups):
    pcm, coefs, adpcm = _gc_inputs(oracle)
    cfgs = [vg.gcadpcm.GcAdpcmParameters(sample_count=len(x)) for x in pcm]
    results = pipeline_groups(lambda: vg.gcadpcm.decode_batch(adpcm, coefs, cfgs))
    _same(results)
    for c, x in enumerate(pcm):
        want = oracle.decode(adpcm[c], coefs[c], len(x)) if len(x) else np.zeros(0, dtype=np.int16)
        assert np.array_equal(results[0][c], want), c


def test_gcadpcm_decode_error_names_the_callers_channel(vg, oracle, pipeline_groups):
    pcm, coefs, adpcm = _gc_inputs(oracle)
    last = N_UNITS - 1
    adpcm[last] = adpcm[last].copy()
    adpcm[last][0] = 0x80 | (adpcm[last][0] & 0x0F)  # frame header: predictor 8
    cfgs = [vg.gcadpcm.GcAdpcmParameters(sample_count=len(x)) for x in pcm]

    def call():
        with pytest.raises(vg.VgbError) as e:
            vg.gcadpcm.decode_batch(adpcm, coefs, cfgs)
        return str(e.value)

    for msg in pipeline_groups(call):
        assert f"channel {last}: a frame header selects a predictor outside 0..7" in msg, msg


def _adx_cfgs(vg, pcm, **kw):
    # version 3 for the empty units: version 4 without padding needs a sample (CriAdxCodec.cs:69-74)
    return [vg.criadx.CriAdxParameters(sample_rate=48000, type=2 + c % 3, filter=c % 4, version=4 if len(x) else 3, **kw)
            for c, x in enumerate(pcm)]


def test_adx_encode_and_decode(vg, oracle, pipeline_groups):
    pcm = _channels(800)
    cfgs = _adx_cfgs(vg, pcm)
    progress = []

    def encode():
        seen = []
        out = vg.criadx.encode_batch(pcm, cfgs, progress=seen.append)
        progress.append(seen)
        return list(out[0]) + [out[1]]

    enc = pipeline_groups(encode)
    _same(enc)
    adpcm, hist = enc[0][:-1], enc[0][-1]
    frames = sum(len(a) // 18 for a in adpcm)
    for seen in progress:
        assert sum(seen) == frames
    for c, x in enumerate(pcm):
        want, want_hist = oracle.adx_encode(x, 48000, 18, cfgs[c].version, 0, cfgs[c].type, cfgs[c].filter)
        assert adpcm[c].tobytes() == want.tobytes(), c
        assert int(hist[c]) == want_hist, c

    dcfgs = _adx_cfgs(vg, pcm)
    for c in range(N_UNITS):
        dcfgs[c].history = int(hist[c])
    counts = [len(x) for x in pcm]
    dec = pipeline_groups(lambda: vg.criadx.decode_batch(adpcm, counts, dcfgs))
    _same(dec)
    for c, x in enumerate(pcm):
        want = oracle.adx_decode(adpcm[c], len(x), 48000, 500, 18, cfgs[c].version, int(hist[c]), 0, cfgs[c].type)
        assert np.array_equal(dec[0][c], want), c


def test_adx_decode_error_names_the_callers_channel(vg, pipeline_groups):
    pcm = _channels(800)
    cfgs = _adx_cfgs(vg, pcm)
    last = N_UNITS - 1
    cfgs[last].type = 2  # Fixed
    adpcm, hist = vg.criadx.encode_batch(pcm, cfgs)
    adpcm = [a.copy() for a in adpcm]
    adpcm[last][0] |= 0x80  # frame header: filter number 4 or more
    for c in range(N_UNITS):
        cfgs[c].history = int(hist[c])

    def call():
        with pytest.raises(vg.VgbError) as e:
            vg.criadx.decode_batch(adpcm, [len(x) for x in pcm], cfgs)
        return str(e.value)

    for msg in pipeline_groups(call):
        assert f"channel {last}: a Fixed-type frame selects a filter outside 0..3" in msg, msg


def test_hca_encode_and_decode(vg, oracle, pipeline_groups):
    lengths = _lengths(900, hi=6000)
    streams = [[synth.channel(900 + 2 * s + c, max(n, 1), degenerate=False)[:n] for c in range(2)]
               for s, n in enumerate(lengths)]
    progress = []

    def encode():
        seen = []
        infos, frames = vg.crihca.encode_batch(streams, 48000, progress=seen.append)
        progress.append(seen)
        return infos, frames

    enc = pipeline_groups(encode)
    infos, frames = enc[0]
    for other_infos, other_frames in enc[1:]:
        assert [i.as_dict() for i in other_infos] == [i.as_dict() for i in infos]
        _same([frames, other_frames])
    for seen in progress:
        assert sum(seen) == sum(i.frame_count for i in infos)
    for s in range(N_UNITS):
        o_info, o_frames = oracle.hca_encode(streams[s], 48000)
        assert infos[s].as_dict() == o_info.as_dict(), s
        assert np.array_equal(frames[s], o_frames), s

    dec = pipeline_groups(lambda: [np.stack(p) for p in vg.crihca.decode_batch(infos, frames)])
    _same(dec)
    for s in range(N_UNITS):
        assert np.array_equal(dec[0][s], oracle.hca_decode(infos[s], frames[s])), s


def test_hca_rows_of_separate_buffers_far_apart(vg, oracle):
    """Caller buffers that are evenly spaced but not one block: the inputs of two streams 2 MiB apart, the output of the
    first stream between them and that of the second far behind.  The call copies each buffer on its own, so it neither
    page-locks the memory between the inputs nor copies over a span that runs from there into unregistered memory."""
    import ctypes as C

    MiB = 1 << 20
    buf = np.zeros(16 * MiB, dtype=np.uint8)
    pcm = [[synth.channel(930 + s, 4000, degenerate=False)] for s in range(2)]
    o = [oracle.hca_encode(st, 48000) for st in pcm]
    info0 = o[0][0]
    size = info0.frame_count * info0.frame_size
    infos = (vg._native.VgbHcaInfo * 2)()
    for s in range(2):
        for k, v in o[s][0].as_dict().items():
            setattr(infos[s], k, v)

    # decode: frames at 0 and 2 MiB, PCM at 1 MiB and 8 MiB
    for s, at in enumerate((0, 2 * MiB)):
        buf[at:at + size] = o[s][1].ravel()
    ftab = (C.c_void_p * 2)(buf.ctypes.data, buf.ctypes.data + 2 * MiB)
    otab = (C.c_void_p * 2)(buf.ctypes.data + MiB, buf.ctypes.data + 8 * MiB)
    vg._native.check(vg.lib.vgb_hca_decode_batch(ftab, C.cast(infos, C.c_void_p), 2, otab))
    for s, at in enumerate((MiB, 8 * MiB)):
        got = buf[at:at + 2 * 4000].view(np.int16)
        assert np.array_equal(got, oracle.hca_decode(infos[s], o[s][1])[0]), s

    # encode: PCM at 0 and 2 MiB, frames at 1 MiB and 8 MiB
    buf[:] = 0
    for s, at in enumerate((0, 2 * MiB)):
        buf[at:at + 8000] = pcm[s][0].view(np.uint8)
    params = (vg._native.VgbHcaParams * 2)(*[vg._native.VgbHcaParams(2, 0, 0, 1, 48000, 4000, 0, 0, 0) for _ in range(2)])
    vg._native.check(vg.lib.vgb_hca_encode_batch(ftab, C.cast(params, C.c_void_p), 2, C.cast(infos, C.c_void_p), otab,
                                                 None, None))
    for s, at in enumerate((MiB, 8 * MiB)):
        assert np.array_equal(buf[at:at + size], o[s][1].ravel()), s
