"""CPU tests of the oracle's CRI HCA frame traces (vgo_hca_encode_trace, vgo_hca_decode_trace) and of the coverage of
the stimulus set (tests/hca_stimuli.py) that tests/test_crihca_paths_gpu.py runs on the GPU."""
import numpy as np
import pytest

import hca_stimuli as H


@pytest.fixture(scope="module")
def enc(oracle):
    """[(stim, [(status, info, frames, trace) per stream])]"""
    return [(s, [oracle.hca_encode_trace(st, s.rate, s.quality, s.bitrate) for st in s.streams]) for s in H.encoder_stimuli()]


@pytest.fixture(scope="module")
def dec(oracle):
    return H.decoder_stimuli()


def test_trace_frames_equal_encode_frames(oracle, enc):
    for s, runs in enc:
        for st, (rc, info, frames, trace) in zip(s.streams, runs):
            if s.fails:
                assert rc == -2, s.name
                with pytest.raises(ValueError):
                    oracle.hca_encode(st, s.rate, s.quality, s.bitrate)
                continue
            assert rc == 0, s.name
            o_info, o_frames = oracle.hca_encode(st, s.rate, s.quality, s.bitrate)
            assert info.as_dict() == o_info.as_dict(), s.name
            assert np.array_equal(frames, o_frames), s.name
            # the record describes the frame that was written: noise level, boundary and every channel's delta_bits
            head = frames[:, 2].astype(np.int32) << 8 | frames[:, 3]
            assert np.array_equal(head >> 7, trace["noise_level"]), s.name
            assert np.array_equal(head & 127, trace["eval_boundary"]), s.name
            assert np.array_equal(frames[:, 4] >> 5, trace["delta_bits"][:, 0]), s.name
            assert (trace["res_hist"].sum(axis=1) == trace["coded"].sum(axis=1)).all(), s.name


def _frames_of(enc, prefix):
    tr = [t for s, runs in enc if s.name.startswith(prefix) for (_, _, _, t) in runs]
    assert tr, prefix
    return np.concatenate(tr)


def test_each_encoder_stimulus_reaches_its_path(enc):
    assert (_frames_of(enc, "band_dropping")["drop_rounds"] > 0).sum() >= 50
    for s, runs in enc:
        if s.name.startswith("band_dropping"):
            assert all((t["drop_rounds"] > 0).any() for *_, t in runs), s.name
    nan = _frames_of(enc, "hfr_empty_groups")["hfr_flags"] & H.O.HCA_HFR_AVG_NAN
    assert nan.any(axis=(1, 2)).all()                          # every frame of those configurations
    failing = _frames_of(enc, "bitrate_too_low")
    assert (failing["status"] == -2).sum() == 1 and failing["drop_rounds"].max() > 0
    anti = _frames_of(enc, "anti_phase_et_zero")
    assert (anti["is_flags"][:, 1] & H.O.HCA_IS_ET_ZERO).any() and (anti["is_flags"][:, 1] & H.O.HCA_IS_CLAMP_HIGH).any()
    assert (_frames_of(enc, "pair_high_bands_silent")["is_flags"][:, 1] & H.O.HCA_IS_SILENT).any()
    assert (_frames_of(enc, "pair_one_silent")["delta_bits"][:, :2] == 0).any()
    assert (_frames_of(enc, "raw_scale_factors")["delta_bits"][:, :2] == 6).sum() >= 3
    assert (_frames_of(enc, "delta_bits_5")["delta_bits"][:, :2] == 5).sum() >= 5
    clamp = _frames_of(enc, "clamped")
    assert clamp["clamped"].sum() > 0 and clamp["sf_max"].sum() > 0


def test_encoder_coverage_of_the_whole_set(enc):
    tr = np.concatenate([t for _, runs in enc for (*_, t) in runs])
    ok = tr[tr["status"] == 0]
    written = np.concatenate([t["delta_bits"][:, :i.channel_count].ravel() for _, runs in enc for (_, i, _, t) in runs])
    assert set(range(7)) <= set(np.unique(written).tolist())   # every delta_bits the encoder writes
    assert (ok["escapes"] > 0).any() and ok["sf_zero"].any() and ok["sf_max"].any() and ok["clamped"].any()
    assert (ok["res_hist"].sum(axis=0) > 0).all()              # every resolution 0..15
    flags = ok["is_flags"]
    for f in (H.O.HCA_IS_SILENT, H.O.HCA_IS_ET_ZERO, H.O.HCA_IS_CLAMP_HIGH):
        assert (flags & f).any(), f
    # the lower clamp never acts: et = 2 * sum |l + r| <= 2 * (el + er), so the ratio (el + er) / et is at least 0.5
    assert not (flags & H.O.HCA_IS_CLAMP_LOW).any()
    idx = ok["intensity"][ok["intensity"] >= 0]
    assert 0 in idx and idx.max() >= 10
    assert (ok["hfr_flags"] & H.O.HCA_HFR_AVG_NAN).any() and (ok["hfr_scale"] >= 0).any()
    assert (tr["status"] == -2).any()
    sizes = {info.frame_size for _, runs in enc for (_, info, _, _) in runs}
    assert {22, 28, 33, 4096} <= sizes


def test_structured_decoder_frames_are_valid(oracle, dec):
    for d in dec:
        for frames in d.streams:
            assert oracle.hca_unpack_ok(d.info, frames), d.name
            pcm, tr = oracle.hca_decode_trace(d.info, frames)
            assert (tr["unpack"] == H.O.HCA_UNPACK_OK).all(), d.name
            assert np.array_equal(pcm, oracle.hca_decode(d.info, frames)), d.name


def test_decoder_coverage(oracle, dec):
    traces = []
    for d in dec:
        for frames in d.streams:
            traces.append((d, oracle.hca_decode_trace(d.info, frames)[1]))
    tr = np.concatenate([t for _, t in traces])
    read = np.concatenate([t["delta_bits"][:, :d.info.channel_count].ravel() for d, t in traces])
    assert set(range(8)) <= set(np.unique(read).tolist())
    hfr = tr[tr["hfr_index_max"] >= 0]
    assert hfr["hfr_index_min"].min() == 1 and hfr["hfr_index_max"].max() == 127
    assert (hfr["hfr_index_max"] == 126).any() and (hfr["hfr_index_min"] == 2).any()
    assert tr["pcm_clip_high"].sum() > 0 and tr["pcm_clip_low"].sum() > 0 and tr["pcm_in_range"].sum() > 0
    # PcmFloatToShort's int32 guard cannot fire on a frame: a coefficient is at most sqrt(128) (scale factor 63, or an
    # HFR copy, whose gain is sqrt(128) * 2^(53/128 * (hfr_scale - 63))) times 2 (intensity ratio), the DCT-IV scales
    # by sqrt(2/128) over 128 bins and the overlap adds two of those: |v| < 2 * 0.125 * 128 * 2 * 11.32 * 32768 < 2^25
    assert tr["pcm_out_of_int32"].sum() == 0
    # the secondary channel without coded bands reads DeltaDecode's leading 6 bits for delta_bits 1..5
    base0 = np.concatenate([t for d, t in traces if d.info.base_band_count == 0])
    assert np.isin(base0["delta_bits"][:, 1], [1, 2, 3, 4, 5]).sum() >= 3
    names = {d.name for d in dec}
    assert {f"{n}ch_q5_48000" for n in range(1, 9)} <= names
    infos = [d.info for d in dec]
    assert any(i.stereo_band_count and i.hfr_group_count for i in infos)
    assert any(not i.stereo_band_count and not i.hfr_group_count for i in infos)


def test_fault_cases_are_rejected_by_the_oracle(oracle):
    cases = H.fault_cases()
    assert {c[1].channel_count for c in cases if c[3].kind == "intensity15"} == {2, 4, 6, 8}
    for i, (name, info, bad, fault) in enumerate(cases):
        streams = H.fault_streams(info, bad, fault, seed=2000 + i)
        for s, frames in enumerate(streams):
            assert oracle.hca_unpack_ok(info, frames) == (s != bad), name
        _, tr = oracle.hca_decode_trace(info, streams[bad])
        want = H.O.HCA_UNPACK_INTENSITY_15 if fault.kind == "intensity15" else H.O.HCA_UNPACK_BAD_DELTA
        assert tr["unpack"][fault.frame] == want, name
        assert (np.delete(tr["unpack"], fault.frame) == H.O.HCA_UNPACK_OK).all(), name
