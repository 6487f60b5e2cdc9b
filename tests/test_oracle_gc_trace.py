"""CPU tests of the oracle's GC-ADPCM frame trace (vgo_gc_encode_trace) and of the coverage of the encoder stimulus set
(tests/gc_stimuli.py) that tests/test_gcadpcm_layout_gpu.py runs on the GPU."""
import numpy as np
import pytest

import gc_stimuli as G
from vgaudio_b200 import synth


@pytest.fixture(scope="module")
def stims(oracle):
    return G.build()


def test_trace_bytes_equal_encode_bytes_on_the_stimulus_set(oracle, stims):
    for s in stims:
        got, trace = oracle.gc_encode_trace(s.pcm, s.coefs, s.sample_count, s.h1, s.h2)
        assert got.tobytes() == oracle.encode(s.pcm, s.coefs, s.sample_count, s.h1, s.h2).tobytes(), s.name
        assert len(trace) == s.frames, s.name
        # the header the trace names is the header that was written
        if s.frames:
            heads = got[::8][: s.frames]
            assert np.array_equal(heads >> 4, trace["winner"]), s.name
            assert np.array_equal(heads & 15, trace["pred"]["final_sp"][np.arange(s.frames), trace["winner"]]), s.name


def test_trace_bytes_equal_encode_bytes_on_the_oracle_corpora(oracle):
    """The inputs test_oracle_gcadpcm.py pins the oracle with."""
    cases = [(synth.reference_ramp(start, 112), -1) for start in (0, 50, 200, 100)]
    cases += [(synth.reference_sine(c * 56 + 112, 1, 56), -1) for c in (1, 20, 100)]
    cases += [(synth.channel(7, 14 * 300), -1)] + [(synth.channel(9, 64)[:n], -1) for n in (0, 1, 2, 13, 14, 15, 27, 28, 29)]
    cases += [(x, -1) for x in synth.batch(6, 5000)] + [(synth.channel(21, 3000), 1401)]
    for i, (pcm, sc) in enumerate(cases):
        co = oracle.calculate_coefficients(pcm)
        got, trace = oracle.gc_encode_trace(pcm, co, sc, 3, -4)
        assert got.tobytes() == oracle.encode(pcm, co, sc, 3, -4).tobytes(), i


def test_trace_agrees_with_a_plain_restatement(oracle, stims):
    """Checks the instrumentation, not the arithmetic: every recorded fact of a few hundred frames (natural, loud and
    hostile coefficient sets) against the pure-Python restatement of DspEncodeCoef in gc_stimuli."""
    rng = np.random.default_rng(31)
    picked = [s for s in stims if s.frames > 100]
    checked = 0
    for s in picked:
        _, trace = oracle.gc_encode_trace(s.pcm, s.coefs, s.sample_count, s.h1, s.h2)
        win = G.frame_windows(s.pcm, s.coefs, s.sample_count, s.h1, s.h2)
        cats = G.frame_categories(trace)
        rare = np.flatnonzero(cats["C3"] | cats["C1"] | cats["C7"] | cats["C6b"])
        frames = np.concatenate([rng.choice(s.frames, 12, replace=False), rare[:4]])
        for f in frames:
            recs = [G.py_try_predictor(win[f], int(s.coefs[2 * p]), int(s.coefs[2 * p + 1])) for p in range(8)]
            for p, r in enumerate(recs):
                t = trace[f]["pred"][p]
                where = (s.name, int(f), p)
                assert int(t["error"]) == r["error"], where
                assert int(t["max_abs_diff"]) == r["max_abs_diff"], where
                assert int(t["n_passes"]) == r["n_passes"], where
                assert list(t["over"][: r["n_passes"]]) == r["over"], where
                assert not t["over"][r["n_passes"]:].any(), where
                assert (int(t["first_sp"]), int(t["final_sp"])) == (r["first_sp"], r["final_sp"]), where
                assert (bool(t["bumped"]), bool(t["final12"]), bool(t["wrapped"])) == \
                       (r["bumped"], r["final12"], r["wrapped"]), where
            errs = [r["error"] for r in recs]
            assert trace[f]["winner"] == errs.index(min(errs)), (s.name, f)
            assert bool(trace[f]["tie"]) == (errs.count(min(errs)) > 1), (s.name, f)
            checked += 1
    assert checked >= 200


def test_pass_powers_follow_the_bump_rule():
    assert G.pass_powers(3, [5, 0]) == [3, 4]
    assert G.pass_powers(3, [249, 0]) == [3, 5]           # one bump: a power skipped
    assert G.pass_powers(3, [248, 0]) == [3, 4]           # the near miss
    assert G.pass_powers(2, [1000, 5, 0]) == [2, 5, 6]    # 1008 > 256, 504 > 256: two bumps
    assert G.pass_powers(10, [100000, 3]) == [10, 12]     # bumps stop at 11, the next pass is 12


# Categories the encoder test must place in every quarter slot, both ways round.  C2 (a chain of >= 5 passes won by
# its predictor) is not in the list: the bounded search over these materials finds no such frame (a predictor whose
# chain is that long loses the frame); the matrix prints its row so that a change that makes it reachable shows.
REQUIRED = ("C1", "C1hi", "C3", "C3hi", "C3_248", "C3_249", "C4", "C5", "C6", "C6b", "C7", "C7loud", "C8", "C6_alone")


def test_coverage_matrix_has_no_empty_cell(stims):
    """Each category in each quarter slot with a warp mate that lacks it at the same frame, and the reverse; C1, C3,
    C5 and C6 also at chunk positions 15 and 0 and on a segment's first frame for 3 and 8 segments.  Laid out as the
    GPU test encodes the set (four rotations by one channel)."""
    cats = [G.categories_of(s) for s in stims]
    cov = G.coverage(stims, cats)
    empty = [(k, c) for k in REQUIRED for c in G.required_cells(k) if cov[k].get(c, 0) == 0]
    assert not empty, "empty cells " + repr(empty) + "\n" + G.format_matrix(cov)


def test_stimulus_set_shapes(stims):
    assert len(stims) % 8 == 0
    frames = sorted(s.frames for s in stims)
    assert 0 in frames and {15, 16, 17, 31, 32, 33} <= set(frames)
    assert any(s.n_enc % 14 for s in stims if s.n_enc)            # partial last frames
    assert any(s.h1 or s.h2 for s in stims) and any(s.sample_count != -1 for s in stims)
    assert sum(s.natural for s in stims) >= 4
