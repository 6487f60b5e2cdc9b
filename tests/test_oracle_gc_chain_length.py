"""CPU tests of where the encoder's speculative window ends, by chain length of the winning predictor.

The GC-ADPCM encoder (gc_encode.cu) evaluates the scale powers sp_first and sp_first + 1 in its first round and only
sp_first + 2 in its second; a predictor whose chain needs a fourth power is handed to gc_slow_frame as unresolved.
Category C1 of tests/gc_stimuli.py lumps chains of 3 and 4 passes together, so the coverage matrix of
tests/test_oracle_gc_trace.py cannot say which of the two it placed.  Here the two are told apart on the same stimulus
set that tests/test_gcadpcm_layout_gpu.py encodes: a 3-pass chain (the longest the fast path finishes) must sit in
every quarter slot next to a warp mate without one, and the reverse; a 4-pass chain is searched for with the same
seeded, bounded search the set is built with."""
import numpy as np
import pytest

import gc_stimuli as G


def winner_passes(trace) -> np.ndarray:
    """Pass count of the winning predictor's chain, per frame."""
    if len(trace) == 0:
        return np.zeros(0, np.int64)
    w = trace["winner"].astype(np.int64)
    return trace["pred"][np.arange(len(trace)), w]["n_passes"].astype(np.int64)


def coverage_of(stims, traces, passes: int) -> dict:
    """G.coverage cells of "the winner's chain has exactly `passes` passes" (in the C1 row) and of the same with the
    winner among predictors 4..7 (in the C1hi row)."""
    cats = []
    for s, tr in zip(stims, traces):
        c = G.frame_categories(tr)
        n = winner_passes(tr)
        c["C1"] = n == passes
        c["C1hi"] = c["C1"] & (tr["winner"] >= 4) if len(tr) else np.zeros(0, bool)
        cats.append(c)
    return G.coverage(stims, cats)


@pytest.fixture(scope="module")
def stims_traces(oracle):
    stims = G.build()
    return stims, [G.trace_of(s)[1] for s in stims]


def test_three_pass_chains_fill_every_cell(stims_traces):
    stims, traces = stims_traces
    cov = coverage_of(stims, traces, 3)
    empty = [(k, c) for k in ("C1", "C1hi") for c in G.required_cells(k) if cov[k].get(c, 0) == 0]
    assert not empty, "empty cells " + repr(empty) + "\n" + G.format_matrix(cov, ("C1", "C1hi"))


def test_four_pass_chains(stims_traces):
    """A 4-pass winner in the set must fill every quarter cell; the set has none, so the bounded search over the
    materials the set draws from is run, and the test is skipped when it finds no predictor (winning or not) that
    needs four passes."""
    stims, traces = stims_traces
    if any((winner_passes(tr) == 4).any() for tr in traces):
        cov = coverage_of(stims, traces, 4)
        empty = [c for c in G.required_cells("C1") if c[0] in ("has", "lacks") and cov["C1"].get(c, 0) == 0]
        assert not empty, "empty cells " + repr(empty)
        return
    kinds = ("unstable", "ramp_unstable", "hostile", "square", "split", "white_random")
    frames = 0
    for t in range(G.SEARCH_TRIES):
        kind = kinds[t % len(kinds)]
        pcm, co, _ = G.material(kind, 20000 + t, G.SEARCH_FRAMES * G.FRAME)
        tr = G.trace_of(G.Stim(f"four:{kind}:{t}", pcm, co))[1]
        frames += len(tr)
        assert not (tr["pred"]["n_passes"] == 4).any(), \
            f"{kind} seed {20000 + t} has a 4-pass chain: add it to the stimulus set and to this coverage check"
    pytest.skip(f"no predictor needs four passes in {frames} searched frames; the path that sends a fourth power to "
                f"gc_slow_frame is not placed by the stimulus set")
