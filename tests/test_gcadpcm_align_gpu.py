"""vgb_gcadpcm_align_batch (GcAdpcmAlignment, Formats/GcAdpcm/GcAdpcmAlignment.cs:20-63) against the oracle's literal
restatement vgo_gc_align: AdpcmAligned and PcmAligned byte-identical on the reference's pin theories, at the BRSTM
default multiple 0x3800, on ragged batches and on the edges of the tail arithmetic; errors with the reference's outcome;
no device work when nothing needs alignment; the same bytes on three bound devices."""
import ctypes as C

import numpy as np
import pytest

from oracle.pygcalign import gc_align
from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu

# AlignedAdpcmIsCorrect / AlignedPcmIsCorrect rows (GcAdpcmAlignmentTests.cs:64-108): (multiple, loopStart, sineCycles)
SINE_ROWS = [(1000, 4524, 100), (1000, 2012, 1), (1000, 60, 1), (1000, 60, 20)]


def encoded(oracle, seed, n):
    pcm = synth.channel(seed, n, degenerate=False)
    co = oracle.calculate_coefficients(pcm)
    return oracle.encode(pcm, co), co


def sine_case(oracle, loop_start, cycles):
    loop_end = cycles * 4 * 14 + loop_start
    pcm = synth.reference_sine(-(-loop_end // 14) * 14, 1, 14 * 4)
    co = oracle.calculate_coefficients(pcm)
    return loop_end, co, oracle.encode(pcm, co)


def check_against_oracle(vg, oracle, adpcm, coefs, params, pcm=True):
    got_a, got_p = vg.gcadpcm.align_batch(adpcm, coefs, params, pcm=pcm)
    for c, p in enumerate(params):
        rc, geom, want_a, want_p = gc_align(*p, adpcm[c], coefs[c])
        assert rc == 0, (c, p)
        if not geom[0]:
            assert got_a[c] is None and got_p[c] is None, c
            continue
        assert got_a[c].tobytes() == want_a.tobytes(), (c, p)
        if pcm:
            assert np.array_equal(got_p[c], want_p), (c, p)
        else:
            assert got_p[c] is None
    return got_a, got_p


@pytest.mark.parametrize("multiple,loop_start,cycles", SINE_ROWS)
def test_pin_theories_match_the_oracle(vg, oracle, multiple, loop_start, cycles):
    loop_end, co, adpcm = sine_case(oracle, loop_start, cycles)
    check_against_oracle(vg, oracle, [adpcm], co.reshape(1, 16), [(multiple, loop_start, loop_end)])


def test_brstm_default_multiple_on_a_stereo_minute(vg, oracle):
    n = 48000 * 60
    chans = [encoded(oracle, 40 + c, n) for c in range(2)]
    params = [(0x3800, 1234567, n - 5)] * 2
    got_a, got_p = check_against_oracle(vg, oracle, [a for a, _ in chans], np.stack([c for _, c in chans]), params)
    # identity: PcmAligned is the decode of AdpcmAligned from history (0, 0)
    count = len(got_p[0])
    dec = vg.gcadpcm.decode_batch(got_a, np.stack([c for _, c in chans]), [vg.gcadpcm.GcAdpcmParameters(count)] * 2)
    for c in range(2):
        assert np.array_equal(dec[c], got_p[c])


def ragged(oracle, seed=0):
    """Channels of different lengths and loop points, some needing no alignment."""
    rng = np.random.default_rng([0x414C49, seed])
    adpcm, coefs, params = [], [], []
    for c in range(37):
        n = int(rng.integers(20, 90000))
        a, co = encoded(oracle, 300 + 37 * seed + c, n)
        loop_end = int(rng.integers(1, n + 1))
        loop_start = int(rng.integers(0, loop_end))
        multiple = [0x3800, 14, 8, 1000, 0, 1, loop_start or 1, 3][c % 8]
        adpcm.append(a)
        coefs.append(co)
        params.append((multiple, loop_start, loop_end))
    return adpcm, np.stack(coefs), params


@pytest.mark.parametrize("seed", [0, 1])
def test_ragged_batch_matches_the_oracle(vg, oracle, seed):
    adpcm, coefs, params = ragged(oracle, seed)
    assert any(not vg.gcadpcm.alignment(*p)[0] for p in params) and any(vg.gcadpcm.alignment(*p)[0] for p in params)
    check_against_oracle(vg, oracle, adpcm, coefs, params)


@pytest.mark.parametrize("name,n,params", [
    ("loop_end below one frame (keep 0)", 200, (16, 3, 11)),
    ("loop_end a multiple of 14", 3000, (0x3800, 100, 14 * 150)),
    ("loop inside one frame", 3000, (1000, 141, 146)),
    ("loop of one sample", 3000, (4096, 1000, 1001)),
    ("partial last tail frame", 5000, (100, 1001, 4000)),
    ("loop_end == sample_count", 14 * 300 + 5, (0x3800, 77, 14 * 300 + 5)),
    ("negative multiple", 3000, (-3, 1000, 2500)),
    ("negative multiple, loop_end a multiple of 14", 3000, (-3, 1000, 14 * 150)),
])
@pytest.mark.parametrize("pcm", [True, False])
def test_edges_of_the_tail(vg, oracle, name, n, params, pcm):
    a, co = encoded(oracle, 77, n)
    assert vg.gcadpcm.alignment(*params)[0], name
    check_against_oracle(vg, oracle, [a, a], np.stack([co, co]), [params, params], pcm=pcm)


def raw_call(vg, adpcm, coefs, params, out_a, out_p):
    from vgaudio_b200 import _native as N

    n = len(adpcm)
    lens = np.array([len(a) for a in adpcm], dtype=np.int32)
    par = (N.VgbGcAlignParams * max(n, 1))(*[N.VgbGcAlignParams(*p) for p in params])
    ptr = lambda rows: (C.c_void_p * max(n, 1))(*[r.ctypes.data if r is not None else None for r in rows])  # noqa: E731
    co = np.ascontiguousarray(coefs, dtype=np.int16)
    rc = vg.lib.vgb_gcadpcm_align_batch(ptr(adpcm), lens.ctypes.data, co.ctypes.data, C.cast(par, C.c_void_p), n, ptr(out_a),
                                        ptr(out_p) if out_p is not None else None)
    return rc, (vg.lib.vgb_last_error() or b"").decode()


def test_rows_of_channels_without_alignment_are_not_written(vg, oracle):
    a, co = encoded(oracle, 5, 9000)
    params = [(8, 16, 5000), (8, 17, 5000), (0, 3, 9000), (8, 19, 5000)]
    out_a = [np.full(vg.gcadpcm.sample_count_to_byte_count(8000), 0xA5, np.uint8) for _ in params]
    out_p = [np.full(8000, 0x5A5A, np.int16) for _ in params]
    rc, msg = raw_call(vg, [a] * 4, np.stack([co] * 4), params, out_a, out_p)
    assert rc == 0, msg
    for c in (0, 2):
        assert (out_a[c] == 0xA5).all() and (out_p[c] == 0x5A5A).all(), c
    for c in (1, 3):
        _, (_, _, count), want_a, want_p = gc_align(*params[c], a, co)
        assert out_a[c][:len(want_a)].tobytes() == want_a.tobytes() and (out_a[c][len(want_a):] == 0xA5).all()
        assert np.array_equal(out_p[c][:count], want_p) and (out_p[c][count:] == 0x5A5A).all()


def test_nothing_to_align_launches_nothing(vg, oracle):
    a, co = encoded(oracle, 6, 4000)
    before = vg.lib.vgb_kernel_launch_count()
    got_a, got_p = vg.gcadpcm.align_batch([a, a, a], np.stack([co] * 3), [(0, 5, 100), (5, 10, 3000), (-7, -14, 99)])
    assert got_a == [None] * 3 and got_p == [None] * 3
    assert vg.lib.vgb_kernel_launch_count() == before
    assert vg.formats.align_loops([a], co.reshape(1, 16), 0x3800, 0x3800 * 2, 3000 * 14)[0].alignment_needed is False


@pytest.mark.parametrize("params,short,want", [
    ((4, -5, 100), False, "negative loop point"),
    ((4, 5, -1), False, "negative loop point"),
    ((4, 90, 80), False, "before loop_start"),
    ((4, 1001, 1001), False, "empty loop"),
    ((2**30, 2**30 + 1, 2**30 + 2), False, "overflows"),
    ((4, 5, 3000), True, "too short"),
])
def test_argument_errors_name_the_channel(vg, oracle, params, short, want):
    from vgaudio_b200 import _native as N

    a, co = encoded(oracle, 8, 3000)
    rows = [a, a, a[:100] if short else a]
    plist = [(8, 16, 500), (8, 17, 500), params]
    outs = [np.zeros(vg.gcadpcm.sample_count_to_byte_count(600), np.uint8), np.zeros(600, np.uint8), None]
    before = vg.lib.vgb_kernel_launch_count()
    rc, msg = raw_call(vg, rows, np.stack([co] * 3), plist, outs, None)
    assert rc == N.VGB_E_ARG and msg.startswith("channel 2:") and want in msg, msg
    assert vg.lib.vgb_kernel_launch_count() == before  # checked before any device work
    check_against_oracle(vg, oracle, [a, a], np.stack([co, co]), plist[:2])  # the next good call is exact


def test_bad_predictor_below_loop_end_is_a_data_error_and_after_it_is_not(vg, oracle):
    from vgaudio_b200 import _native as N

    a, co = encoded(oracle, 9, 6000)
    params = (1000, 60, 4000)
    bad_hi = a.copy()
    bad_hi[8 * (3999 // 14)] |= 0x80   # the frame holding sample loop_end - 1
    bad_lo = a.copy()
    bad_lo[8 * 3] = 0x90
    after = a.copy()
    after[8 * (4000 // 14 + 2)] = 0xF0  # past loop_end: never decoded, not reported
    assert gc_align(*params, bad_hi, co)[0] == -2 and gc_align(*params, after, co)[0] == 0
    rows = [a, after, bad_hi, a, bad_lo]
    outs = [np.zeros(vg.gcadpcm.sample_count_to_byte_count(5000), np.uint8) for _ in rows]
    rc, msg = raw_call(vg, rows, np.stack([co] * 5), [params] * 5, outs, None)
    assert rc == N.VGB_E_DATA and msg.startswith("channel 2:"), msg
    check_against_oracle(vg, oracle, [a, after], np.stack([co, co]), [params] * 2)


def test_three_bound_devices_give_the_same_bytes(vg, oracle):
    import torch

    from vgaudio_b200 import _native as N

    adpcm, coefs, params = ragged(oracle, 2)
    one_a, one_p = vg.gcadpcm.align_batch(adpcm, coefs, params)
    n = torch.cuda.device_count()
    devs = [0, 1 % n, 2 % n] if n > 1 else [0, 0, 0]
    N.check(vg.lib.vgb_shutdown())
    N.check(vg.lib.vgb_init_devices((C.c_int32 * 3)(*devs), 3, 0))
    try:
        assert vg.lib.vgb_device_count() == 3
        three_a, three_p = vg.gcadpcm.align_batch(adpcm, coefs, params)
        # a bad predictor on two shards: the lowest channel is named
        a, co = encoded(oracle, 9, 6000)
        bad = a.copy()
        bad[8 * 10] = 0xA0
        rows = [a, a, a, bad, a, bad, a]
        outs = [np.zeros(vg.gcadpcm.sample_count_to_byte_count(5000), np.uint8) for _ in rows]
        rc, msg = raw_call(vg, rows, np.stack([co] * 7), [(1000, 60, 4000)] * 7, outs, None)
        assert rc == N.VGB_E_DATA and msg.startswith("channel 3:"), msg
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    for c in range(len(adpcm)):
        assert (one_a[c] is None) == (three_a[c] is None), c
        if one_a[c] is not None:
            assert one_a[c].tobytes() == three_a[c].tobytes() and np.array_equal(one_p[c], three_p[c]), c
