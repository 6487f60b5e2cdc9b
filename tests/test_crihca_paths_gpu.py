"""GPU tests of the CRI HCA kernels on the stimuli of tests/hca_stimuli.py, whose reach into the rare paths of the encoder
and decoder tests/test_oracle_hca_trace.py proves with the oracle's frame traces.

Encoder: vgb_hca_encode_batch against the oracle, infos equal and frames byte-identical, streams in ragged batches.
Decoder: vgb_hca_decode_batch on structured frames the encoder never writes, PCM bit-identical to the oracle's on every
channel layout; malformed streams rejected with VGB_E_DATA naming the stream, and the next call still exact."""
import numpy as np
import pytest

import hca_stimuli as H

pytestmark = pytest.mark.gpu

ENC = {s.name: s for s in H.encoder_stimuli()}
DEC = {d.name: d for d in H.decoder_stimuli()}


def _vg_info(vg, info):
    out = vg._native.VgbHcaInfo()
    for k, v in info.as_dict().items():
        setattr(out, k, v)
    return out


def _encode(vg, s, streams=None):
    cfg = vg.crihca.CriHcaParameters(quality=s.quality, bitrate=s.bitrate)
    return vg.crihca.encode_batch(s.streams if streams is None else streams, s.rate, cfg)


@pytest.mark.parametrize("name", [n for n, s in ENC.items() if not s.fails])
def test_encoder_paths_byte_identical_to_oracle(vg, oracle, name):
    s = ENC[name]
    infos, frames = _encode(vg, s)
    for i, st in enumerate(s.streams):
        o_info, o_frames = oracle.hca_encode(st, s.rate, s.quality, s.bitrate)
        assert infos[i].as_dict() == o_info.as_dict(), (name, i)
        same = (frames[i] == o_frames).all(axis=1)
        assert same.all(), f"{name} stream {i}: frames {np.flatnonzero(~same)[:8]} of {len(same)} differ"


def test_encoder_bitrate_too_low_inside_the_frame_loop(vg, oracle):
    """The frame loop runs out of bands to drop: VGB_E_DATA naming the stream; a silent stream of the same
    configuration needs no bits and encodes."""
    s = H.bitrate_too_low()
    silent = [np.zeros(3000, np.int16)]
    with pytest.raises(vg.VgbError) as e:
        _encode(vg, s, [silent, s.streams[0]])
    assert e.value.code == vg._native.VGB_E_DATA
    assert "stream 1:" in str(e.value) and "too low" in str(e.value)
    good = ENC["hfr_empty_groups_8500"]
    infos, frames = _encode(vg, good)
    for i, st in enumerate(good.streams):
        assert np.array_equal(frames[i], oracle.hca_encode(st, good.rate, good.quality, good.bitrate)[1]), i


@pytest.mark.parametrize("name", list(DEC))
def test_decoder_structured_frames_bit_identical_to_oracle(vg, oracle, name):
    d = DEC[name]
    info = _vg_info(vg, d.info)
    if d.info.base_band_count > 0:  # the layouts the encoder's Initialize gives: vgb_hca_query agrees
        q = vg.crihca.query(vg.crihca.CriHcaParameters(quality=0, channel_count=d.info.channel_count,
                                                       sample_rate=d.info.sample_rate, sample_count=d.info.sample_count,
                                                       bitrate=d.info.bitrate))
        assert q.as_dict() == d.info.as_dict()
    pcm = vg.crihca.decode_batch([info] * len(d.streams), d.streams)
    for i, frames in enumerate(d.streams):
        want = oracle.hca_decode(d.info, frames)
        got = np.stack(pcm[i])
        assert np.array_equal(got, want), f"{name} stream {i}: {int((got != want).sum())} samples differ"


@pytest.mark.parametrize("case", range(len(H.fault_cases())))
def test_decoder_rejects_malformed_streams(vg, oracle, case):
    name, o_info, bad, fault = H.fault_cases()[case]
    streams = H.fault_streams(o_info, bad, fault, seed=2000 + case)
    info = _vg_info(vg, o_info)
    with pytest.raises(vg.VgbError) as e:
        vg.crihca.decode_batch([info] * len(streams), streams)
    assert e.value.code == vg._native.VGB_E_DATA, name
    assert f"stream {bad}:" in str(e.value), (name, str(e.value))
    assert ("intensity" if fault.kind == "intensity15" else "delta") in str(e.value), name
    good = [f for s, f in enumerate(streams) if s != bad]
    pcm = vg.crihca.decode_batch([info] * len(good), good)
    for i, frames in enumerate(good):
        assert np.array_equal(np.stack(pcm[i]), oracle.hca_decode(o_info, frames)), (name, i)


def test_secondary_channel_without_coded_bands_reads_the_leading_scale_factor(vg, oracle):
    """DeltaDecode reads its first value before the loop (CriHcaPacking.cs:183-186), so a stereo-secondary channel with
    base_band_count == 0 and delta_bits 1..5 consumes 6 bits; every field behind it depends on that."""
    d = DEC["2ch_base0"]
    _, tr = oracle.hca_decode_trace(d.info, d.streams[0])
    assert np.isin(tr["delta_bits"][:, 1], [1, 2, 3, 4, 5]).any()
    got = np.stack(vg.crihca.decode(_vg_info(vg, d.info), d.streams[0]))
    assert np.array_equal(got, oracle.hca_decode(d.info, d.streams[0]))


def test_no_call_is_left_broken(vg, oracle):
    """After every rejection above the device context still encodes byte-exact."""
    s = ENC["raw_scale_factors"]
    infos, frames = _encode(vg, s)
    for i, st in enumerate(s.streams):
        assert np.array_equal(frames[i], oracle.hca_encode(st, s.rate, s.quality, s.bitrate)[1]), i
