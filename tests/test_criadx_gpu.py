"""GPU parity tests for CRI ADX: the CUDA path through the C ABI against the CPU oracle, bit-exact (integer codec)."""
import numpy as np
import pytest

from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu


def _cfg(vg, **kw):
    return vg.criadx.CriAdxParameters(**kw)


@pytest.mark.parametrize("typ", [2, 3, 4])
@pytest.mark.parametrize("version", [3, 4])
def test_encode_decode_match_oracle(vg, oracle, typ, version):
    pcm = synth.batch(20, 9000)
    pcm = pcm[[1, 2, 3] + list(range(4, 20))]  # drop the all-zero channel? keep square/sine/ramp + mixes
    cfgs = [_cfg(vg, sample_rate=48000, version=version, type=typ, filter=(c % 4)) for c in range(len(pcm))]
    adpcm, hist = vg.criadx.encode_batch(pcm, cfgs)
    for c in range(len(pcm)):
        want, want_hist = oracle.adx_encode(pcm[c], 48000, 18, version, 0, typ, c % 4)
        assert adpcm[c].tobytes() == want.tobytes(), (typ, version, c)
        assert int(hist[c]) == want_hist
    dcfgs = [_cfg(vg, version=version, type=typ, history=int(hist[c])) for c in range(len(pcm))]
    dec = vg.criadx.decode_batch(adpcm, 9000, dcfgs)
    for c in range(len(pcm)):
        want = oracle.adx_decode(adpcm[c], 9000, 48000, 500, 18, version, int(hist[c]), 0, typ)
        assert np.array_equal(dec[c], want), (typ, version, c)


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 63, 64, 65, 1000, 4097])
@pytest.mark.parametrize("padding", [0, 1, 13, 32, 45, 64])
def test_edge_lengths_and_padding(vg, oracle, n, padding):
    chans = [synth.channel(30 + i, max(n, 1))[:n] for i in range(4)]
    cfgs = [_cfg(vg, padding=padding, sample_rate=44100) for _ in chans]
    adpcm, hist = vg.criadx.encode_batch(chans, cfgs)
    for c, pcm in enumerate(chans):
        want, want_hist = oracle.adx_encode(pcm, 44100, 18, 4, padding, 3, 0)
        assert adpcm[c].tobytes() == want.tobytes(), (n, padding, c)
        assert int(hist[c]) == want_hist
    dcfgs = [_cfg(vg, padding=padding, sample_rate=44100, history=int(hist[c])) for c in range(len(chans))]
    dec = vg.criadx.decode_batch(adpcm, n, dcfgs)
    for c in range(len(chans)):
        want = oracle.adx_decode(adpcm[c], n, 44100, 500, 18, 4, int(hist[c]), padding, 3)
        assert np.array_equal(dec[c], want), (n, padding, c)


def test_other_frame_sizes_and_ragged_batch(vg, oracle):
    lens = [100, 777, 5000, 64, 4096, 33]
    sizes = [18, 10, 34, 18, 66, 4]
    chans = [synth.channel(50 + i, L) for i, L in enumerate(lens)]
    cfgs = [_cfg(vg, frame_size=fs, type=3 + (i % 2)) for i, fs in enumerate(sizes)]
    adpcm, hist = vg.criadx.encode_batch(chans, cfgs)
    for c in range(len(chans)):
        want, wh = oracle.adx_encode(chans[c], 48000, sizes[c], 4, 0, 3 + (c % 2), 0)
        assert adpcm[c].tobytes() == want.tobytes(), c
        dec = vg.criadx.decode(adpcm[c], lens[c], _cfg(vg, frame_size=sizes[c], type=3 + (c % 2), history=int(hist[c])))
        assert np.array_equal(dec, oracle.adx_decode(want, lens[c], 48000, 500, sizes[c], 4, wh, 0, 3 + (c % 2))), c


def test_decode_hostile_streams(vg, oracle):
    rng = np.random.default_rng(17)
    n_ch, frames = 70, 150
    adpcm = rng.integers(0, 256, (n_ch, frames * 18), dtype=np.uint8)
    adpcm[:, 0::18] &= 0x1F   # filter bits zero: the reference indexes a one-entry table for Linear/Exponential
    for typ in (3, 4):
        cfgs = [_cfg(vg, type=typ, history=int(rng.integers(-32768, 32768)), version=3 + (c % 2)) for c in range(n_ch)]
        dec = vg.criadx.decode_batch(adpcm, frames * 32 - 5, cfgs)
        for c in range(n_ch):
            want = oracle.adx_decode(adpcm[c], frames * 32 - 5, 48000, 500, 18, cfgs[c].version, cfgs[c].history, 0, typ)
            assert np.array_equal(dec[c], want), (typ, c)


def test_fixed_type_rejects_filter_numbers_past_the_table(vg, oracle):
    """Fixed-type frames carry their filter number in the top three bits; CriAdxCodec.Coefs has four rows (:186-191), so
    4..7 is an IndexOutOfRangeException in the reference: VGB_E_DATA here.  0..3 decode like the oracle."""
    rng = np.random.default_rng(19)
    n_ch, frames = 12, 40
    adpcm = rng.integers(0, 256, (n_ch, frames * 18), dtype=np.uint8)
    adpcm[:, 0::18] &= 0x7F   # filter numbers 0..3
    cfgs = [_cfg(vg, type=2, history=0, version=3 + (c % 2)) for c in range(n_ch)]
    dec = vg.criadx.decode_batch(adpcm, frames * 32, cfgs)
    for c in range(n_ch):
        assert np.array_equal(dec[c], oracle.adx_decode(adpcm[c], frames * 32, 48000, 500, 18, cfgs[c].version, 0, 0, 2)), c
    for ch, frame in [(0, 0), (11, 39), (6, 20)]:
        bad = adpcm.copy()
        bad[ch, frame * 18] |= 0x80
        with pytest.raises(vg.VgbError) as e:
            vg.criadx.decode_batch(bad, frames * 32, cfgs)
        assert e.value.code == -2 and f"channel {ch}:" in str(e.value)


def test_errors(vg):
    with pytest.raises(vg.VgbError):   # empty v4 channel: the reference throws IndexOutOfRangeException (CriAdxCodec.cs:71)
        vg.criadx.encode_batch([np.zeros(0, dtype=np.int16)], [_cfg(vg)])
    with pytest.raises(vg.VgbError):   # too few bytes for the requested sample count
        vg.criadx.decode(np.zeros(18, dtype=np.uint8), 100, _cfg(vg))
    with pytest.raises(vg.VgbError):
        vg.criadx.encode_batch([np.zeros(10, dtype=np.int16)], [_cfg(vg, type=7)])


@pytest.mark.parametrize("seg", [1, 2, 7, 64, None])
def test_time_parallel_encode_is_bit_exact(vg, oracle, seg):
    """The ADX encoder cuts a channel's whole frames into segments encoded concurrently from raw history and splices them
    at the boundaries (adx.cu); VGB_ADX_SEGMENTS forces the count.  Mixed batch: every type / version, ragged lengths with
    partial last frames, full-scale noise and squares (slow to re-lock), 500 Hz noise (never re-locks), and channels the segmentation must leave to the
    serial loop (another frame size, padding)."""
    import os

    rng = np.random.default_rng(31)
    lens = [32 * 2000, 32 * 2000 + 17, 32 * 3000 + 1, 32 * 700, 32 * 256 * 3, 32 * 5000 + 31, 40, 32 * 2500, 32 * 2200 + 9, 32 * 2100]
    chans = [synth.channel(40 + i, L) for i, L in enumerate(lens)]
    chans[3] = rng.integers(-32768, 32768, lens[3]).astype(np.int16)                       # white, full scale
    chans[7] = np.where((np.arange(lens[7]) // 2) % 2 == 0, 32767, -32768).astype(np.int16)  # Nyquist/2 square
    cfgs = [_cfg(vg, sample_rate=48000, version=4 - (i % 2), type=2 + (i % 3), filter=i % 4) for i in range(len(chans))]
    cfgs[8] = _cfg(vg, sample_rate=44100, frame_size=34, version=4, type=3)   # not the standard layout
    cfgs[9] = _cfg(vg, sample_rate=48000, padding=45, version=4, type=3)      # padded stream
    chans.append(rng.integers(-6000, 6000, 32 * 2400 + 5).astype(np.int16))   # never re-locks at 500 Hz: the cascade
    cfgs.append(_cfg(vg, sample_rate=500, version=4, type=3))
    saved = {k: os.environ.get(k) for k in ("VGB_ADX_SEGMENTS", "VGB_ADX_MIN_SEG_FRAMES")}
    os.environ["VGB_ADX_MIN_SEG_FRAMES"] = "256"  # the default (4096) is sized for the run-on tail; short inputs must still be cut
    if seg is None:
        os.environ.pop("VGB_ADX_SEGMENTS", None)
    else:
        os.environ["VGB_ADX_SEGMENTS"] = str(seg)
    try:
        adpcm, hist = vg.criadx.encode_batch(chans, cfgs)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    for c, pcm in enumerate(chans):
        p = cfgs[c]
        want, want_hist = oracle.adx_encode(pcm, p.sample_rate, p.frame_size, p.version, p.padding, p.type, p.filter)
        got = np.frombuffer(adpcm[c].tobytes(), np.uint8)
        first = np.flatnonzero(got != want)
        assert first.size == 0, f"seg {seg} channel {c}: first differing byte {first[0]} (frame {first[0] // p.frame_size})"
        assert int(hist[c]) == want_hist, c
