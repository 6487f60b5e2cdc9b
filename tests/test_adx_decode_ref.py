"""The throwing restatement of CriAdxCodec.Decode (adx_decode_ref) pinned on the CPU: its PCM against the oracle's
vgo_adx_decode on every stream of the decode-path matrix that the reference accepts, its verdicts against the reader
chain's filter rule (adx_reader_oracle.expected_wave) on .adx images built from the same rows, and the placements of the
matrix against the decoders' geometry."""
import numpy as np
import pytest

import adx_decode_ref as D
import adx_reader_oracle as R


def _matrix():
    return D.clean_streams() + D.fault_streams() + D.fault_streams(silent=True)


def _throws(s: D.Stream) -> bool:
    """What the rule says without decoding: the fault frame is read, yields a sample and selects a row the table lacks."""
    if s.fault is None or s.fault >= D.frame_count(s.n, s.frame_size):
        return False
    if s.fault == 0 and not D.head_yields(s.n, s.frame_size, s.padding):
        return False
    return s.filter > (3 if s.type == D.FIXED else 0)


def test_pcm_matches_the_oracle_where_the_reference_returns(oracle):
    returned = 0
    for s in _matrix():
        pcm, err = D.verdict(s.data, s.n, **s.params())
        if err is not None:
            continue
        want = oracle.adx_decode(s.data, s.n, 48000, 500, s.frame_size, s.version, s.history, s.padding, s.type)
        assert np.array_equal(np.array(pcm, np.int16), want), s
        returned += 1
    assert returned > 600


def test_throws_exactly_at_the_fault_frame():
    thrown = {D.FIXED: 0, D.LINEAR: 0, D.EXPONENTIAL: 0}
    for s in _matrix():
        _, err = D.verdict(s.data, s.n, **s.params())
        assert (err is not None) == _throws(s), s
        if err is not None:
            assert (err.frame, err.filter_num, err.rows) == (s.fault, s.filter, 4 if s.type == D.FIXED else 1), s
            thrown[s.type] += 1
    assert min(thrown.values()) > 100, thrown


@pytest.mark.parametrize("scale,want", [(13, 0), (28, 0), (29, -32768), (12, 1), (0, 4096)])
def test_exponential_scale_takes_the_masked_shift_and_the_short_cast(scale, want):
    """(short)(1 << (12 - scale)) with C#'s shift count masked to 5 bits: counts 31 and 16 leave 0, 15 leaves -32768."""
    row = np.zeros(18, np.uint8)
    row[0], row[1] = scale >> 8, scale & 0xFF
    row[2] = 0x10  # first nibble 1: the first sample is scale * 1
    assert D.decode(row, 1, version=4, type=D.EXPONENTIAL)[0] == max(-32768, min(32767, want))


def test_version_rounding_orders_differ_where_the_reference_says():
    """Version 4 shifts the sum of both products, version 3 each product: a stream where they part ways."""
    row = np.zeros(18, np.uint8)
    row[0] = 2 << 5  # Fixed filter 2: (0x1CC0, -0x0D00)
    pcm3 = D.decode(row, 32, version=3, history=1001, type=D.FIXED)
    pcm4 = D.decode(row, 32, version=4, history=1001, type=D.FIXED)
    assert pcm3[0] == (1001 * 0x1CC0 >> 12) + (1001 * -0x0D00 >> 12) and pcm4[0] == (1001 * (0x1CC0 - 0x0D00)) >> 12
    assert pcm3 != pcm4


def test_verdicts_match_the_reader_chain_on_adx_images():
    """Each fault row beside a clean row of the same geometry in a stereo file, each clean row alone: the file fails in
    the reader chain exactly where a channel throws, and otherwise holds the restatement's PCM."""
    rng = np.random.default_rng(3)
    checked = failed = 0
    for s in D.fault_streams() + D.fault_streams(silent=True) + D.clean_streams()[:-1]:
        if s.fault is None:
            chans = [s]
        else:
            chans = [D.Stream(D.clean_row(rng, s.type, s.frame_size, s.padding, s.n), s.n, s.frame_size, s.version, s.padding, s.type), s]
        img = D.adx_image(chans)
        got = [D.verdict(c.data, c.n, **c.params(history=0)) for c in chans]
        want = R.expected_wave(img)
        if any(e is not None for _, e in got):
            assert want is None, s
            failed += 1
        else:
            assert want is not None, s
            st, h = R.adx_parse(img)
            pcm = np.frombuffer(want.tobytes()[-2 * s.n * len(chans):], "<i2").reshape(s.n, len(chans)) if s.n else None
            for k, (p, _) in enumerate(got):
                assert pcm is None or np.array_equal(pcm[:, k], np.array(p, np.int16)), (s, k)
        checked += 1
    assert failed > 400 and checked - failed > 400


def test_placements_reach_their_paths():
    """Every placement lands where its name says, by the serial decoder's fast-path predicate (18-byte frames, no
    padding, whole 8-frame groups) and the time-parallel decoder's segment boundaries (8 segments of at least 8 frames)."""
    seen = set()
    for s in D.fault_streams():
        fc = D.frame_count(s.n, s.frame_size)
        fast = D.serial_fast_frames(s.n, s.frame_size, s.padding)
        bounds = D.seg_boundaries(s.n, s.frame_size, s.padding, 8, 8)
        p = s.placement
        seen.add(p)
        if p == "head":
            assert s.fault == 0
        elif p in ("group_first", "group_last"):
            assert s.frame_size == 18 and s.padding == 0 and s.fault < fast and s.fault % 8 == (0 if p == "group_first" else 7)
        elif p == "remainder":
            assert fast <= s.fault < fc - 1 and fast % 8 == 0 and fast > 0
        elif p in ("boundary", "boundary_last"):
            assert s.fault in bounds and len(bounds) >= 2
        elif p == "run_on":
            assert any(b < s.fault < b2 for b, b2 in zip(bounds, bounds[1:]))
        elif p == "tail":
            assert s.fault == fc - 1 and s.fault > 0
        elif p == "past":
            assert s.fault == fc and (D.head_row_frame(s.frame_size, s.padding) + fc + 1) * s.frame_size <= s.data.size
    assert seen == {"head", "group_first", "group_last", "remainder", "boundary", "boundary_last", "run_on", "tail", "past"}
    # the partial tail: at least one layout whose last frame yields fewer than spf samples, both kernels' slow path
    assert any((s.n + (s.padding % ((s.frame_size - 2) * 2))) % ((s.frame_size - 2) * 2) for s in D.fault_streams() if s.placement == "tail")
    silent = D.fault_streams(silent=True)
    assert {s.placement for s in silent} == {"silent_head", "yielding_head"}
