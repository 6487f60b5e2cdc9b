"""GcAdpcmAlignment's pins (src/VGAudio.Tests/Formats/GcAdpcm/GcAdpcmAlignmentTests.cs:13-108), rows restated as literals.

The geometry theories run through the oracle's vgo_gc_align and the product's host-only vgb_gcadpcm_alignment (no
device needed); the re-encode theories run through the oracle, which the GPU tests then compare the product with."""
import numpy as np
import pytest

from oracle.pygcalign import gc_align
from vgaudio_b200 import synth

# (multiple, loopStart, loopEnd); every row of the reference passes an ADPCM array of 0x40 bytes and zero coefficients
NOT_NEEDED = [(0, 0, 10), (0, 5, 10), (1, 7, 10), (3, 12, 13), (5, 10, 13)]
NEEDED = [(2, 3, 10), (4, 2, 10), (3, 31, 50), (16, 24, 50), (16, 31, 50)]
# AlignedLoopPointsAreCorrect: (multiple, loopStart, loopEnd, LoopStartAligned, SampleCountAligned)
ALIGNED_POINTS = [(2, 3, 10, 4, 11), (4, 2, 10, 4, 12), (3, 31, 50, 33, 52), (16, 24, 50, 32, 58), (16, 31, 50, 32, 51)]
# AlignedAdpcmIsCorrect / AlignedPcmIsCorrect: (multiple, loopStart, sineCycles)
SINE_ROWS = [(1000, 4524, 100), (1000, 2012, 1), (1000, 60, 1), (1000, 60, 20)]


def _oracle_alignment(oracle, multiple, loop_start, loop_end):
    rc, geom, adpcm, pcm = gc_align(multiple, loop_start, loop_end, np.zeros(0x40, np.uint8), np.zeros(16, np.int16))
    assert rc == 0
    return geom, adpcm, pcm


@pytest.mark.parametrize("multiple,loop_start,loop_end", NOT_NEEDED)
def test_alignment_not_needed(vg, oracle, multiple, loop_start, loop_end):
    geom, adpcm, pcm = _oracle_alignment(oracle, multiple, loop_start, loop_end)
    assert geom == (0, 0, 0) and adpcm is None and pcm is None
    assert vg.gcadpcm.alignment(multiple, loop_start, loop_end) == (False, 0, 0)


@pytest.mark.parametrize("multiple,loop_start,loop_end", NEEDED)
def test_alignment_needed(vg, oracle, multiple, loop_start, loop_end):
    geom, _, _ = _oracle_alignment(oracle, multiple, loop_start, loop_end)
    assert geom[0] == 1
    assert vg.gcadpcm.alignment(multiple, loop_start, loop_end)[0] is True


@pytest.mark.parametrize("multiple,loop_start,loop_end,want_start,want_count", ALIGNED_POINTS)
def test_aligned_loop_points_are_correct(vg, oracle, multiple, loop_start, loop_end, want_start, want_count):
    geom, adpcm, pcm = _oracle_alignment(oracle, multiple, loop_start, loop_end)
    assert geom[1:] == (want_start, want_count)
    assert len(adpcm) == oracle.sample_count_to_byte_count(want_count) and len(pcm) == want_count
    assert vg.gcadpcm.alignment(multiple, loop_start, loop_end) == (True, want_start, want_count)


def sine_case(oracle, loop_start, cycles):
    """The reference theories' input: a sine of period 56 up to the frame after loopEnd, its own coefficients."""
    loop_end = cycles * 4 * 14 + loop_start
    pcm = synth.reference_sine(-(-loop_end // 14) * 14, 1, 14 * 4)
    coefs = oracle.calculate_coefficients(pcm)
    return loop_end, coefs, oracle.encode(pcm, coefs)


@pytest.mark.parametrize("multiple,loop_start,cycles", SINE_ROWS)
def test_aligned_adpcm_is_correct(oracle, multiple, loop_start, cycles):
    loop_end, coefs, adpcm = sine_case(oracle, loop_start, cycles)
    rc, (_, _, count), adpcm_aligned, _ = gc_align(multiple, loop_start, loop_end, adpcm, coefs)
    assert rc == 0
    got = oracle.decode(adpcm_aligned, coefs, count).astype(np.int32)
    want = synth.reference_sine(count, 1, 14 * 4).astype(np.int32)
    end = -(-count // 14) * 14 - 14  # skip the first sine cycle and the last ADPCM frame (history samples)
    assert np.abs(want[56:end] - got[56:end]).max(initial=0) <= 2


@pytest.mark.parametrize("multiple,loop_start,cycles", SINE_ROWS)
def test_aligned_pcm_is_correct(oracle, multiple, loop_start, cycles):
    loop_end, coefs, adpcm = sine_case(oracle, loop_start, cycles)
    rc, (_, _, count), adpcm_aligned, pcm_aligned = gc_align(multiple, loop_start, loop_end, adpcm, coefs)
    assert rc == 0
    assert np.array_equal(pcm_aligned, oracle.decode(adpcm_aligned, coefs, count))


@pytest.mark.parametrize("multiple,loop_start,loop_end", [(5, 7, 7), (-1, -2**31, 10), (4, -5, 10), (4, 5, -1), (4, 9, 8),
                                                          (2**30, 2**30 + 1, 2**30 + 2)])
def test_unusable_loop_points_are_argument_errors(vg, oracle, multiple, loop_start, loop_end):
    """Where the reference throws (or, for an empty loop whose start moves, never returns) the oracle says -1 and the
    product's geometry call VGB_E_ARG."""
    from vgaudio_b200 import _native as N

    assert gc_align(multiple, loop_start, loop_end)[0] == -1
    with pytest.raises(N.VgbError) as e:
        vg.gcadpcm.alignment(multiple, loop_start, loop_end)
    assert e.value.code == N.VGB_E_ARG


@pytest.mark.parametrize("multiple,loop_start,loop_end,want", [(-3, 4, 10, (1, 4, 10)), (-3, 4, 4, (1, 4, 4)),
                                                               (5, 5, 5, (0, 0, 0)), (-7, -14, -20, (0, 0, 0))])
def test_multiples_that_move_nothing(vg, oracle, multiple, loop_start, loop_end, want):
    """GetNextMultiple leaves the start alone for a multiple <= 0, but a negative multiple that does not divide it still
    asks for alignment (C# `%` truncates toward zero); a multiple that divides it asks for none, whatever the loop
    points."""
    assert gc_align(multiple, loop_start, loop_end)[:2] == (0, want)
    assert vg.gcadpcm.alignment(multiple, loop_start, loop_end) == (bool(want[0]), want[1], want[2])


def test_a_bad_predictor_below_loop_end_is_a_data_error(oracle):
    loop_end, coefs, adpcm = sine_case(oracle, 60, 1)
    bad = adpcm.copy()
    bad[8 * ((loop_end - 1) // 14)] |= 0x80  # the frame holding sample loop_end - 1
    assert gc_align(1000, 60, loop_end, bad, coefs)[0] == -2
    after = np.concatenate([adpcm, np.array([0xF0, 0, 0, 0, 0, 0, 0, 0], np.uint8)])  # a bad frame past loop_end
    assert gc_align(1000, 60, loop_end, after, coefs)[0] == 0
