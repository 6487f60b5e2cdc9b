"""CPU tests of the oracle's coefficient trace (vgo_gc_coef_trace) and of the coverage of the coefficient stimulus set
(tests/gc_coef_stimuli.py) that tests/test_gcadpcm_coefs_gpu.py runs through the refinement kernel pass by pass."""
import numpy as np
import pytest

import gc_coef_stimuli as G
from vgaudio_b200 import synth


@pytest.fixture(scope="module")
def stims(oracle):
    return G.build()


@pytest.fixture(scope="module")
def infos(stims):
    return [G.analyse(s) for s in stims]


def corpora():
    """The channels test_gcadpcm_gpu.py's coefficient tests encode: edge lengths, every residue mod 14 and 32, the
    seeded batch with its degenerate channels."""
    out = [synth.channel(i, max(n, 1))[:n] for n in (0, 1, 2, 13, 14, 15, 27, 28, 29, 223, 224, 225, 447, 448, 449, 3583,
                                                      3584, 3585, 10007) for i in range(6)]
    out += [synth.channel(10 + i, L) for i, L in enumerate(list(range(1000, 1000 + 14 * 32 + 1, 7)) + list(range(5000, 5033)))]
    return out + list(synth.batch(48, 48000))


def test_trace_quantises_to_calculate_coefficients(oracle, stims):
    for pcm in [s.pcm for s in stims] + corpora():
        co, trace, outcome = oracle.gc_coef_trace(pcm)
        want = oracle.calculate_coefficients(pcm)
        assert np.array_equal(co, want), len(pcm)
        last = trace["pass"]["cent"][-1]
        assert [G.quantise(v) for v in last.ravel()] == want.tolist(), len(pcm)
        acc, _, _ = oracle.coef_records(pcm)
        assert np.array_equal(outcome == oracle.GC_ACCEPTED, acc.astype(bool)), len(pcm)
        assert int(trace["n_records"]) == int(acc.sum()) and int(trace["n_frames"]) == len(acc)


def test_restatement_reproduces_every_traced_value(oracle, stims, infos):
    """A plain-Python CalculateCoefficients / FilterRecords from the direct-form records gives every traced centroid (raw
    bits), bucket count, empty-bucket and tie fact, on the stimuli and on the corpora of the older GPU tests."""
    pairs = [(s.name, i["trace"], i["ref"]) for s, i in zip(stims, infos)]
    for k, pcm in enumerate(corpora()):
        pairs.append((f"corpus {k} ({len(pcm)} samples)", oracle.gc_coef_trace(pcm)[1], G.refine(G.direct_records(pcm))))
    for name, trace, ref in pairs:
        assert not G.trace_fields_equal(trace, ref), (name, G.trace_fields_equal(trace, ref))
        assert list(trace["pass"]["count"]) == list(G.PASS_BUCKETS), name
    assert len(pairs) > 250


def test_coverage_matrix(stims, infos):
    """Every category is reached somewhere in the set (the searched tie categories are checked, or skipped with the
    search's result, by test_searched_ties), and the set's launch shapes cover both CTA widths' producer pipelines."""
    cov = G.coverage(infos)
    print("\ncoefficient stimulus coverage (occurrences over the set)\n" + G.format_coverage(cov))
    unplaced = {f"rej_{r}_at_{f}" for r, f in G.UNPLACED}
    empty = [k for k in G.CATEGORIES if cov[k] == 0 and k not in G.TIES and k not in unplaced]
    assert not empty, f"categories not reached: {empty}\n" + G.format_coverage(cov)
    facts = G.shape_facts(stims)
    print("launch shapes", facts)
    assert {1, 2, 3, 4, 6, 7, 8, 15} <= facts["n_blocks"]
    for P in G.PRODUCERS:
        chunks = facts["chunks"][P]
        assert any(c % 2 for c in chunks) and any(c % 2 == 0 for c in chunks), P
        assert max(chunks) > G.K_DEPTH, P  # the producers' fetch ring wraps
    assert facts["n_mod_8"] == set(range(8))
    assert {0, 1, 31} <= facts["frames_mod_32"]
    assert facts["partial_last_frame"]


@pytest.mark.parametrize("category", G.TIES)
def test_searched_ties(infos, category):
    n = sum(i["cats"][category] for i in infos)
    if n == 0:
        pytest.skip(f"{category}: the bounded search over {G.TIE_TRIES} seeded candidates found none")
    assert n > 0


def test_sensitivity_self_check(stims, infos):
    """The set can see the errors the trace is for: a pairwise (tree) sum of the buckets changes the trace of channels
    whose coefficients it leaves as they are, and so does a last-minimum tie rule on the consequential-tie channel."""
    tree_only = 0
    for s, i in zip(stims, infos):
        tree = G.refine(G.direct_records(s.pcm), "tree")
        if G.trace_fields_equal(i["trace"], tree) and np.array_equal(tree["coefs"], i["coefs"]):
            tree_only += 1
    assert tree_only >= 10, tree_only
    conseq = [i for i in infos if i["cats"]["tie_consequential"]]
    if not conseq:
        pytest.skip("no consequential tie in the set: the last-minimum rule cannot be told apart")
    for i in conseq:
        assert G.trace_fields_equal(i["trace"], i["last"])
