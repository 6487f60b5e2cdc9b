"""CPU tests: pin the oracle (oracle/gcadpcm.c) against everything the reference's own tests hold for GC-ADPCM.

The reference has no golden bitstream for this codec (SURVEY.md §4/§8c), so the pins are its KAT tables for the
nibble/sample math and its round-trip properties.  Sources are cited per test (paths under
VGAudio's src/VGAudio.Tests/).
"""
import json
import os

import numpy as np
import pytest

from vgaudio_b200 import synth

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


# ---- Formats/GcAdpcm/GcAdpcmHelpersTests.cs:8-100 (exact tables) ----------------------------------------------
@pytest.mark.parametrize("nibble,expected", [(2, 0), (3, 1), (15, 13), (18, 14), (19, 15), (100010, 87508)])
def test_nibble_to_sample(oracle, nibble, expected):
    assert oracle.lib().vgo_gc_nibble_to_sample(nibble) == expected


@pytest.mark.parametrize("sample,expected", [(0, 2), (1, 3), (13, 15), (14, 18), (15, 19), (87508, 100010)])
def test_sample_to_nibble(oracle, sample, expected):
    assert oracle.lib().vgo_gc_sample_to_nibble(sample) == expected


@pytest.mark.parametrize("nibbles,expected", [(0, 0), (1, 0), (2, 0), (3, 1), (15, 13), (16, 14), (17, 14), (18, 14),
                                               (19, 15), (100000, 87500)])
def test_nibble_count_to_sample_count(oracle, nibbles, expected):
    assert oracle.lib().vgo_gc_nibble_count_to_sample_count(nibbles) == expected


@pytest.mark.parametrize("samples,expected", [(0, 0), (1, 3), (2, 4), (13, 15), (14, 16), (15, 19), (87500, 100000)])
def test_sample_count_to_nibble_count(oracle, samples, expected):
    assert oracle.lib().vgo_gc_sample_count_to_nibble_count(samples) == expected


@pytest.mark.parametrize("samples,expected", [(0, 0), (1, 2), (2, 2), (3, 3), (13, 8), (14, 8), (15, 10), (87500, 50000)])
def test_sample_count_to_byte_count(oracle, samples, expected):
    assert oracle.lib().vgo_gc_sample_count_to_byte_count(samples) == expected


def test_conversions_are_reversible(oracle):  # GcAdpcmHelpersTests.cs:80-100
    L = oracle.lib()
    for i in range(1, 10000):
        assert L.vgo_gc_nibble_to_sample(L.vgo_gc_sample_to_nibble(i)) == i
        assert L.vgo_gc_nibble_count_to_sample_count(L.vgo_gc_sample_count_to_nibble_count(i)) == i


# ---- Formats/GcAdpcmFormatTests.cs:87-157: ramps survive encode -> decode exactly at the seek-table positions ----
@pytest.mark.parametrize("start", [0, 50, 200, 100])
def test_ramp_seek_table_samples_exact(oracle, start):
    pcm = synth.reference_ramp(start, 112)
    coefs = oracle.calculate_coefficients(pcm)
    dec = oracle.decode(oracle.encode(pcm, coefs), coefs, 112)
    # BuildSeekTable(samplesPerEntry=50): entry i = (decoded[50i-1], decoded[50i-2]) == expected {50,49,100,99}+start
    assert [int(dec[49]), int(dec[48]), int(dec[99]), int(dec[98])] == [50 + start, 49 + start, 100 + start, 99 + start]


# ---- Formats/GcAdpcm/GcAdpcmAlignmentTests.cs:64-90: sine of period 56 decodes within 2 LSB past the first cycle --
@pytest.mark.parametrize("cycles", [1, 20, 100])
def test_sine_round_trip_within_two_lsb(oracle, cycles):
    n = cycles * 56 + 56 * 2
    pcm = synth.reference_sine(n, 1, 56)
    coefs = oracle.calculate_coefficients(pcm)
    dec = oracle.decode(oracle.encode(pcm, coefs), coefs, n)
    err = np.abs(dec[56: n - 14].astype(np.int32) - pcm[56: n - 14].astype(np.int32))
    assert err.max() <= 2


# ---- GcAdpcmAlignmentTests.cs:92-108: the encoder's embedded reconstruction IS the decoder ---------------------
def test_encoder_reconstruction_equals_decoder(oracle):
    pcm = synth.channel(7, 14 * 300)
    coefs = oracle.calculate_coefficients(pcm)
    adpcm = oracle.encode(pcm, coefs)
    dec = oracle.decode(adpcm, coefs, len(pcm))
    window = np.zeros(16, dtype=np.int16)
    for f in range(300):
        window[2:] = pcm[14 * f: 14 * f + 14]
        frame = oracle.dsp_encode_frame(window, 14, coefs)
        assert frame.tobytes() == adpcm[8 * f: 8 * f + 8].tobytes()
        assert np.array_equal(window[2:], dec[14 * f: 14 * f + 14])
        window[0], window[1] = window[14], window[15]


def test_silent_channel_gives_zero_coefficients(oracle):  # SURVEY.md A.19 (NaN path)
    assert not oracle.calculate_coefficients(np.zeros(1000, dtype=np.int16)).any()
    assert not oracle.calculate_coefficients(np.zeros(0, dtype=np.int16)).any()


def test_partial_last_frame_and_empty(oracle):
    for n in (0, 1, 2, 13, 14, 15, 27, 28, 29):
        pcm = synth.channel(9, 64)[:n]
        coefs = oracle.calculate_coefficients(pcm)
        adpcm = oracle.encode(pcm, coefs)
        assert len(adpcm) == oracle.sample_count_to_byte_count(n)
        assert len(oracle.decode(adpcm, coefs, n)) == n


def test_batch_driver_matches_single_channel(oracle):
    pcm = synth.batch(6, 5000)
    coefs, adpcm, used = oracle.encode_batch(pcm, 3)
    assert used >= 1
    for c in range(6):
        co = oracle.calculate_coefficients(pcm[c])
        assert np.array_equal(co, coefs[c])
        assert np.array_equal(oracle.encode(pcm[c], co), adpcm[c])
    dec, _ = oracle.decode_batch(adpcm, coefs, 5000, 2)
    for c in range(6):
        assert np.array_equal(dec[c], oracle.decode(adpcm[c], coefs[c], 5000))


# ---- committed golden vectors (tests/golden/gcadpcm_golden.json, made by tests/golden/make_golden.py) ----------
def test_oracle_matches_committed_golden(oracle):
    with open(os.path.join(GOLDEN, "gcadpcm_golden.json")) as fh:
        gold = json.load(fh)
    for case in gold["cases"]:
        pcm = synth.channel(case["index"], case["n"], degenerate=case["degenerate"])
        coefs = oracle.calculate_coefficients(pcm)
        adpcm = oracle.encode(pcm, coefs)
        assert coefs.tolist() == case["coefs"], case["name"]
        import hashlib

        assert hashlib.sha256(adpcm.tobytes()).hexdigest() == case["adpcm_sha256"], case["name"]
        assert hashlib.sha256(pcm.tobytes()).hexdigest() == case["pcm_sha256"], case["name"]
