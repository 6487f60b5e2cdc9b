"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle, bit-exact (integer codec)."""
import hashlib
import json
import os

import numpy as np
import pytest

from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def test_phase1_records_match_oracle(vg, oracle):
    import ctypes as C

    for idx, n in [(1, 5000), (2, 14 * 700), (3, 4001), (5, 48000), (8, 14 * 256 + 3), (0, 600)]:
        pcm = synth.channel(idx, n)
        frames = (n + 13) // 14
        direct = np.zeros((frames, 2))
        acc = np.zeros(frames, dtype=np.uint8)
        from vgaudio_b200 import _native as N

        N.check(vg.lib.vgb_gcadpcm_debug_records(pcm.ctypes.data, n, direct.ctypes.data, acc.ctypes.data))
        o_acc, _, o_dir = oracle.coef_records(pcm)
        assert np.array_equal(acc, o_acc), (idx, n)
        sel = o_acc.astype(bool)
        # bit-exact doubles (compare the raw 64-bit patterns)
        assert np.array_equal(direct[sel].view(np.uint64), o_dir[sel].view(np.uint64)), (idx, n)


@pytest.mark.parametrize("n", [0, 1, 2, 13, 14, 15, 27, 28, 29, 223, 224, 225, 447, 448, 449, 3583, 3584, 3585, 10007])
def test_edge_lengths_coefs_encode_decode(vg, oracle, n):
    chans = [synth.channel(i, max(n, 1))[:n] for i in range(6)]
    coefs, adpcm = vg.gcadpcm.encode_batch(chans)
    for c, pcm in enumerate(chans):
        o_co = oracle.calculate_coefficients(pcm)
        assert np.array_equal(coefs[c], o_co), (n, c)
        o_ad = oracle.encode(pcm, o_co)
        assert adpcm[c].tobytes() == o_ad.tobytes(), (n, c)
    dec = vg.gcadpcm.decode_batch(adpcm, coefs, [vg.gcadpcm.GcAdpcmParameters(n)] * len(chans))
    for c, pcm in enumerate(chans):
        assert np.array_equal(dec[c], oracle.decode(adpcm[c], coefs[c], n)), (n, c)
    # default sample count = ByteCountToSampleCount(len) (GcAdpcmDecoder.cs:12)
    dflt = vg.gcadpcm.decode_batch(adpcm, coefs)
    for c in range(len(chans)):
        m = vg.gcadpcm.byte_count_to_sample_count(len(adpcm[c]))
        assert np.array_equal(dflt[c], oracle.decode(adpcm[c], coefs[c], m)), (n, c)


def test_every_residue_mod_14_and_mod_32(vg, oracle):
    lens = list(range(1000, 1000 + 14 * 32 + 1, 7)) + list(range(5000, 5033))
    chans = [synth.channel(10 + i, L) for i, L in enumerate(lens)]
    coefs, adpcm = vg.gcadpcm.encode_batch(chans)  # ragged batch in ONE call
    for c, pcm in enumerate(chans):
        o_co = oracle.calculate_coefficients(pcm)
        assert np.array_equal(coefs[c], o_co), lens[c]
        assert adpcm[c].tobytes() == oracle.encode(pcm, o_co).tobytes(), lens[c]


def test_batch_matches_oracle_seeded_set(vg, oracle):
    pcm = synth.batch(48, 48000)  # includes the four degenerate channels
    coefs, adpcm = vg.gcadpcm.encode_batch(pcm)
    o_coefs, o_adpcm, _ = oracle.encode_batch(pcm)
    assert np.array_equal(coefs, o_coefs)
    assert np.array_equal(np.stack(adpcm), o_adpcm)
    dec = vg.gcadpcm.decode_batch(np.stack(adpcm), coefs, [vg.gcadpcm.GcAdpcmParameters(48000)] * 48)
    o_dec, _ = oracle.decode_batch(o_adpcm, o_coefs, 48000)
    assert np.array_equal(np.stack(dec), o_dec)


def test_committed_golden_vectors(vg):
    with open(os.path.join(GOLDEN, "gcadpcm_golden.json")) as fh:
        gold = json.load(fh)
    chans = [synth.channel(c["index"], c["n"], degenerate=c["degenerate"]) for c in gold["cases"]]
    coefs, adpcm = vg.gcadpcm.encode_batch(chans)
    for i, case in enumerate(gold["cases"]):
        assert hashlib.sha256(chans[i].tobytes()).hexdigest() == case["pcm_sha256"], case["name"]
        assert coefs[i].tolist() == case["coefs"], case["name"]
        assert hashlib.sha256(adpcm[i].tobytes()).hexdigest() == case["adpcm_sha256"], case["name"]


def test_reference_test_properties_on_gpu(vg):
    """The reference's own assertions, run against the CUDA path (GcAdpcmFormatTests.cs:87-157,
    GcAdpcmAlignmentTests.cs:64-90)."""
    for start in (0, 50, 200, 100):
        pcm = synth.reference_ramp(start, 112)
        coefs = vg.gcadpcm.calculate_coefficients(pcm)
        dec = vg.gcadpcm.decode(vg.gcadpcm.encode(pcm, coefs), coefs, vg.gcadpcm.GcAdpcmParameters(112))
        assert [int(dec[49]), int(dec[48]), int(dec[99]), int(dec[98])] == [50 + start, 49 + start, 100 + start, 99 + start]
    n = 100 * 56 + 112
    pcm = synth.reference_sine(n, 1, 56)
    coefs = vg.gcadpcm.calculate_coefficients(pcm)
    dec = vg.gcadpcm.decode(vg.gcadpcm.encode(pcm, coefs), coefs, vg.gcadpcm.GcAdpcmParameters(n))
    assert np.abs(dec[56: n - 14].astype(np.int32) - pcm[56: n - 14]).max() <= 2


def test_encode_with_given_coefs_history_and_sample_count(vg, oracle):
    rng = np.random.default_rng(5)
    pcm = synth.channel(21, 3000)
    coefs = rng.integers(-4096, 4096, 16).astype(np.int16)
    for sc, h1, h2 in [(-1, 0, 0), (3000, 1234, -4321), (2999, -32768, 32767), (1401, 5, 6), (14, 1, 2), (0, 9, 9)]:
        cfg = vg.gcadpcm.GcAdpcmParameters(sc, h1, h2)
        got = vg.gcadpcm.encode(pcm, coefs, cfg)
        want = oracle.encode(pcm, coefs, sc, h1, h2)
        assert got.tobytes() == want.tobytes(), (sc, h1, h2)


def test_extreme_coefficients_wrap_like_int32(vg, oracle):
    """Hostile coefficient sets overflow int32 in the predictor sum (SURVEY.md A.7) and hit scale 12 / bump paths."""
    rng = np.random.default_rng(11)
    pcm = np.where(rng.random(14 * 400) < 0.5, -32768, 32767).astype(np.int16)
    pcm[::3] = rng.integers(-32768, 32768, len(pcm[::3]))
    all_coefs, wants = [], []
    for trial in range(6):
        coefs = rng.choice(np.array([-32768, 32767, -20000, 20000, 0, 2048], dtype=np.int16), 16)
        got = vg.gcadpcm.encode(pcm, coefs)
        want = oracle.encode(pcm, coefs)
        assert got.tobytes() == want.tobytes(), trial
        dec = vg.gcadpcm.decode(got, coefs, vg.gcadpcm.GcAdpcmParameters(len(pcm)))
        assert np.array_equal(dec, oracle.decode(want, coefs, len(pcm)))
        all_coefs.append(coefs)
        wants.append(want)
    # the same six trials as one batch: the hostile frames also run in quarters 1..3 of a warp
    _, got = vg.gcadpcm.encode_batch([pcm] * 6, coefs=np.stack(all_coefs))
    for trial in range(6):
        assert got[trial].tobytes() == wants[trial].tobytes(), ("batch", trial)


def test_decode_hostile_streams(vg, oracle):
    rng = np.random.default_rng(3)
    n_ch, frames = 70, 333   # 70 channels: more than two warps of 32
    adpcm = rng.integers(0, 256, (n_ch, frames * 8), dtype=np.uint8)
    adpcm[:, ::8] &= 0x7F  # predictor index 0..7 (8..15 would throw in the reference)
    coefs = rng.integers(-32768, 32768, (n_ch, 16)).astype(np.int16)
    cfgs = [vg.gcadpcm.GcAdpcmParameters(frames * 14 - (c % 14), int(rng.integers(-32768, 32768)),
                                         int(rng.integers(-32768, 32768))) for c in range(n_ch)]
    dec = vg.gcadpcm.decode_batch(adpcm, coefs, cfgs)
    for c in range(n_ch):
        want = oracle.decode(adpcm[c], coefs[c], cfgs[c].sample_count, cfgs[c].history1, cfgs[c].history2)
        assert np.array_equal(dec[c], want), c


def test_decode_rejects_predictor_indices_past_the_table(vg):
    """coefs[predictor * 2] with predictor 8..15 is an IndexOutOfRangeException in GcAdpcmDecoder.Decode (:31-32): the
    batch call reports VGB_E_DATA (and names the lowest such channel) instead of decoding garbage."""
    rng = np.random.default_rng(4)
    adpcm = rng.integers(0, 256, (40, 64 * 8), dtype=np.uint8)
    adpcm[:, ::8] &= 0x7F
    coefs = rng.integers(-2048, 2048, (40, 16)).astype(np.int16)
    cfgs = [vg.gcadpcm.GcAdpcmParameters(64 * 14)] * 40
    vg.gcadpcm.decode_batch(adpcm, coefs, cfgs)  # clean
    for ch, frame in [(33, 63), (7, 0), (39, 17)]:
        bad = adpcm.copy()
        bad[ch, frame * 8] |= 0x80
        with pytest.raises(vg.VgbError) as e:
            vg.gcadpcm.decode_batch(bad, coefs, cfgs)
        assert e.value.code == -2 and f"channel {ch}:" in str(e.value)
    bad = adpcm.copy()
    bad[5, 8] |= 0x80
    with pytest.raises(vg.VgbError) as e:  # the seek-table rebuild decodes the same stream
        vg.gcadpcm.seek_table_and_loop_context(list(bad), coefs, [64 * 14] * 40, 100, [10] * 40)
    assert e.value.code == -2


def test_dsp_encode_frame_independent_frames(vg, oracle):
    rng = np.random.default_rng(9)
    n = 300
    io = rng.integers(-32768, 32768, (n, 16)).astype(np.int16)
    io[: n // 2] //= 16
    coefs = rng.integers(-3000, 5000, (n, 16)).astype(np.int16)
    counts = rng.integers(0, 15, n).astype(np.int32)
    counts[:40] = 14
    want_io = io.copy()
    want_out = np.zeros((n, 8), dtype=np.uint8)
    for f in range(n):
        want_out[f] = oracle.dsp_encode_frame(want_io[f], int(counts[f]), coefs[f])
    got_out = vg.gcadpcm.dsp_encode_frames(io, coefs, counts)
    assert np.array_equal(got_out, want_out)
    assert np.array_equal(io, want_io)


def test_format_level_drop_in(vg, oracle):
    """GcAdpcmFormat.EncodeFromPcm16 -> ToPcm16 through the mirrored format classes."""
    from vgaudio_b200.formats import GcAdpcmFormat, Pcm16Format

    pcm = Pcm16Format(synth.batch(8, 20000), 48000)
    seen = []
    cfg = vg.gcadpcm.GcAdpcmParameters(progress=seen.append)
    fmt = GcAdpcmFormat().encode_from_pcm16(pcm, cfg)
    assert sum(seen) == ((20000 + 13) // 14) * 8  # Progress.SetTotal value (GcAdpcmFormat.cs:62)
    back = fmt.to_pcm16()
    for c in range(8):
        co = oracle.calculate_coefficients(pcm.channels[c])
        assert np.array_equal(fmt.channels[c].coefs, co)
        ad = oracle.encode(pcm.channels[c], co)
        assert fmt.channels[c].adpcm.tobytes() == ad.tobytes()
        assert np.array_equal(back.channels[c], oracle.decode(ad, co, 20000))


def test_large_batch_property_round_trip(vg):
    """Size-independent property at a larger shape: decode(encode(x)) stays close to x for benign signals and the
    decoder agrees with the encoder's own reconstruction (checked via a second encode of the decoded signal being
    stable in length and header validity)."""
    pcm = synth.batch(256, 14 * 2048, degenerate=False, first_index=100)
    coefs, adpcm = vg.gcadpcm.encode_batch(pcm)
    ad = np.stack(adpcm)
    assert ad.shape == (256, 8 * 2048)
    assert ((ad[:, ::8] >> 4) < 8).all() and ((ad[:, ::8] & 15) <= 12).all()
    dec = np.stack(vg.gcadpcm.decode_batch(ad, coefs))
    err = dec.astype(np.int64) - pcm
    # the bursts are full-scale noise (unpredictable); outside them the codec tracks closely
    assert np.median(np.abs(err)) < 200


def test_loud_signals_exercise_float32_rounding_regime(vg, oracle):
    """Residuals above 2^24/2048 = 8192 make (float)distance inexact in the reference's quantiser
    (GcAdpcmEncoder.cs:142-144); the integer fast path must still agree bit for bit (gc_attempt_fast exit test)."""
    rng = np.random.default_rng(2024)
    n = 14 * 1500
    chans = []
    for i in range(24):
        kind = (i + i // 4) % 4  # channel i runs in quarter i % 4: every kind visits every quarter
        if kind == 0:
            x = rng.integers(-32768, 32768, n)                       # white, full scale
        elif kind == 1:
            x = 30000 * np.sign(np.sin(np.arange(n) * rng.uniform(0.2, 3.0))) + rng.integers(-2000, 2000, n)
        elif kind == 2:
            x = 32000 * np.sin(np.arange(n) * rng.uniform(2.0, 3.1)) + rng.normal(0, 500, n)  # near Nyquist
        else:
            x = np.cumsum(rng.integers(-9000, 9001, n)) % 65536 - 32768                      # sawtooth-like wraps
        chans.append(np.clip(x, -32768, 32767).astype(np.int16))
    pcm = np.stack(chans)
    coefs, adpcm = vg.gcadpcm.encode_batch(pcm)
    o_coefs, o_adpcm, _ = oracle.encode_batch(pcm)
    assert np.array_equal(coefs, o_coefs)
    assert np.array_equal(np.stack(adpcm), o_adpcm)
    # same signals against arbitrary (not analysed) coefficient sets of natural magnitude
    rand_coefs = rng.integers(-6000, 6001, (24, 16)).astype(np.int16)
    _, adpcm2 = vg.gcadpcm.encode_batch(pcm, coefs=rand_coefs)
    for c in range(24):
        assert adpcm2[c].tobytes() == oracle.encode(pcm[c], rand_coefs[c]).tobytes(), c


# ---- post-encode channel rebuild (SURVEY 8f rank 1): seek table + loop context without keeping the decoded PCM --------

@pytest.mark.parametrize("spe", [0x3800, 1000, 14, 56, 57, 3, 1])
def test_seek_table_and_loop_context_match_the_oracle(vg, oracle, spe):
    lens = [30000, 14 * 500, 14 * 500 + 5, 57, 56, 13, 1, 100001]
    loops = [12345, 0, 1, 56, None, 12, 0, 99999]
    pcm = [synth.channel(700 + i, n, degenerate=False) for i, n in enumerate(lens)]
    coefs, adpcm = [], []
    for x in pcm:
        c = oracle.calculate_coefficients(x)
        coefs.append(c)
        adpcm.append(oracle.encode(x, c))
    seek, ctx = vg.gcadpcm.seek_table_and_loop_context(adpcm, np.stack(coefs), lens, spe, loops)
    for i, x in enumerate(pcm):
        dec = oracle.decode(adpcm[i], coefs[i], lens[i])
        assert np.array_equal(seek[i], oracle.gc_seek_table(dec, spe)), (i, spe)
        if loops[i] is None:
            assert ctx[i] is None
        else:
            assert ctx[i] == oracle.gc_loop_context(adpcm[i], dec, loops[i]), (i, loops[i])


def test_seek_context_without_table_and_errors(vg, oracle):
    x = synth.channel(9, 5000)
    c = oracle.calculate_coefficients(x)
    a = oracle.encode(x, c)
    seek, ctx = vg.gcadpcm.seek_table_and_loop_context([a], c.reshape(1, 16), [5000], 0, [2500])
    assert seek[0] is None
    dec = oracle.decode(a, c, 5000)
    assert ctx[0] == oracle.gc_loop_context(a, dec, 2500)
    with pytest.raises(vg.VgbError):  # loop start past the end of the channel
        vg.gcadpcm.seek_table_and_loop_context([a], c.reshape(1, 16), [5000], 0, [5001])


@pytest.mark.parametrize("groups", [1, 3, 16])
def test_host_pipeline_over_channel_groups(vg, oracle, groups):
    """The host call pipelines channel groups (H2D of group g+1 under the kernels of group g, D2H of group g-1): same
    bytes as the oracle for any group count, progress deltas (one per group) summing to the frame total
    (GcAdpcmFormat.cs:62).  VGB_ENCODE_GROUPS forces the group count."""
    n_ch, n = 72, 14 * 1100 + 9  # 1101 frames, partial last frame
    pcm = np.stack([synth.channel(800 + c, n, degenerate=False) for c in range(n_ch)])
    seen = []
    saved = os.environ.get("VGB_ENCODE_GROUPS")
    os.environ["VGB_ENCODE_GROUPS"] = str(groups)
    try:
        coefs, adpcm = vg.gcadpcm.encode_batch(pcm, progress=seen.append)
    finally:
        if saved is None:
            os.environ.pop("VGB_ENCODE_GROUPS", None)
        else:
            os.environ["VGB_ENCODE_GROUPS"] = saved
    assert sum(seen) == n_ch * 1101 and len(seen) == groups
    for c in range(0, n_ch, 7):
        co = oracle.calculate_coefficients(pcm[c])
        assert np.array_equal(coefs[c], co), c
        assert np.array_equal(adpcm[c], oracle.encode(pcm[c], co)), c


@pytest.mark.parametrize("multiple,loop_start,loop_end", [(0x3800, 5000, 40000), (14336, 14336, 30000), (8, 1001, 9000),
                                                           (100, 33, 50), (1024, 5, 70000)])
def test_loop_alignment_matches_the_reference_composition(vg, oracle, multiple, loop_start, loop_end):
    """GcAdpcmAlignment (GcAdpcmAlignment.cs:20-63): decode, rebuild the tail so that the loop start lands on a multiple,
    re-encode it from the reconstructed history, decode again - checked against the same steps done with the oracle."""
    n = 72000
    pcm = [synth.channel(900 + c, n, degenerate=False) for c in range(3)]
    coefs = [oracle.calculate_coefficients(x) for x in pcm]
    adpcm = [oracle.encode(x, c) for x, c in zip(pcm, coefs)]
    got = vg.formats.align_loops(adpcm, np.stack(coefs), multiple, loop_start, loop_end)
    for c in range(3):
        if loop_start % multiple == 0:
            assert not got[c].alignment_needed
            continue
        aligned_start = loop_start + (multiple - loop_start % multiple)
        count = loop_end + aligned_start - loop_start
        keep_frames = loop_end // 14
        keep = keep_frames * 14
        to_encode = count - keep
        old = oracle.decode(adpcm[c], coefs[c], loop_end)
        want_pcm = np.zeros(count, np.int16)
        want_pcm[:loop_end] = old
        tail = np.zeros(to_encode, np.int16)
        tail[:loop_end - keep] = old[keep:loop_end]
        cur = loop_end - keep
        while cur < to_encode:
            k = min(loop_end - loop_start, to_encode - cur)
            tail[cur:cur + k] = want_pcm[loop_start:loop_start + k]
            cur += loop_end - loop_start
        h1 = int(old[keep - 1]) if keep >= 1 else 0
        h2 = int(old[keep - 2]) if keep >= 2 else 0
        new_adpcm = oracle.encode(tail, coefs[c], to_encode, h1, h2)
        want_adpcm = np.concatenate([adpcm[c][:keep_frames * 8], new_adpcm])
        want_pcm[keep:keep + to_encode] = oracle.decode(new_adpcm, coefs[c], to_encode, h1, h2)
        assert got[c].alignment_needed and got[c].loop_start_aligned == aligned_start and got[c].sample_count_aligned == count
        assert np.array_equal(got[c].adpcm_aligned, want_adpcm), c
        assert np.array_equal(got[c].pcm_aligned, want_pcm), c


def test_shutdown_releases_everything_and_the_next_call_reinitialises(vg, oracle):
    """vgb_shutdown frees the device slabs, streams, events and the HCA table blob; the next call brings all of it back."""
    x = synth.channel(21, 5000)
    co = oracle.calculate_coefficients(x)
    want = oracle.encode(x, co)
    info0, frames0 = vg.crihca.encode([x], 48000)
    for _ in range(2):
        assert vg.lib.vgb_shutdown() == 0
        coefs, adpcm = vg.gcadpcm.encode_batch([x])
        assert np.array_equal(coefs[0], co) and np.array_equal(adpcm[0], want)
        info1, frames1 = vg.crihca.encode([x], 48000)
        assert np.array_equal(frames0, frames1)
