"""GPU tests of the GC-ADPCM coefficient kernels pass by pass.  vgb_gcadpcm_debug_refine_trace runs phase 1 and
gc_coef_refine_kernel with its tap on, at both CTA widths, and every pass's centroids (raw 64-bit patterns) and bucket
counts are compared with the oracle's trace (pyoracle.gc_coef_trace) over the stimulus set of tests/gc_coef_stimuli.py,
whose coverage tests/test_oracle_gc_coef_trace.py proves.  An order change of the per-bucket sums or a different tie rule
shows here even when the int16 coefficients do not move."""
import ctypes as C

import numpy as np
import pytest

import gc_coef_stimuli as G
from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def stims(oracle):
    return G.build()


@pytest.fixture(scope="module")
def infos(stims):
    return [G.analyse(s) for s in stims]


def tap(vg, pcms, warps):
    """(cent [n, 7, 8, 2], hits [n, 7, 8], coefs [n, 16]) of the refinement tap."""
    from vgaudio_b200 import _native as N

    arrs = [np.ascontiguousarray(p, dtype=np.int16) for p in pcms]
    n = len(arrs)
    ptrs = (C.c_void_p * n)(*[a.ctypes.data if a.size else None for a in arrs])
    lens = np.array([a.size for a in arrs], np.int32)
    cent = np.zeros((n, G.PASSES, 8, 2))
    hits = np.zeros((n, G.PASSES, 8), np.int32)
    coefs = np.zeros((n, 16), np.int16)
    N.check(vg.lib.vgb_gcadpcm_debug_refine_trace(ptrs, lens.ctypes.data, n, warps, cent.ctypes.data, hits.ctypes.data,
                                                  coefs.ctypes.data))
    return cent, hits, coefs


def mismatches(names, infos, cats, cent, hits, coefs, warps, limit=8):
    """One line per channel that differs from its oracle trace: the first pass and bucket that differ, and the
    channel's categories."""
    bad = []
    for c, (name, info) in enumerate(zip(names, infos)):
        P = info["trace"]["pass"]
        ok_c = G.same_bits(cent[c], P["cent"]).all(axis=2)             # [7, 8]
        ok_h = hits[c] == P["hits"]
        wrong = np.argwhere(~(ok_c & ok_h))
        if wrong.size == 0 and np.array_equal(coefs[c], info["coefs"]):
            continue
        where = "coefficients only" if wrong.size == 0 else (
            f"pass {wrong[0][0]} bucket {wrong[0][1]}: centroid {cent[c][tuple(wrong[0])].tolist()} hits "
            f"{int(hits[c][tuple(wrong[0])])}, want {P['cent'][tuple(wrong[0])].tolist()} hits "
            f"{int(P['hits'][tuple(wrong[0])])} ({len(wrong)} cells differ)")
        here = [k for k, v in cats[c].items() if v] if cats else []
        bad.append(f"{name} ({warps} warps): {where}; categories {here}")
        if len(bad) >= limit:
            break
    return bad


@pytest.mark.parametrize("warps", [4, 8])
def test_every_pass_matches_the_oracle_trace(vg, stims, infos, warps):
    """Every stimulus in one ragged batch, at both CTA widths (3 and 7 producer warps)."""
    cent, hits, coefs = tap(vg, [s.pcm for s in stims], warps)
    bad = mismatches([s.name for s in stims], infos, [i["cats"] for i in infos], cent, hits, coefs, warps)
    assert not bad, "\n".join(bad)


def test_second_wave_of_the_narrow_cta(vg, oracle):
    """1,100 short channels: more than the 8 x 132 CTAs of the 4-warp kernel that are resident at once on an H100."""
    pcms = [synth.channel(3000 + i, 14 * (20 + i % 53) - i % 14) for i in range(1100)]
    infos = []
    for p in pcms:
        co, trace, _ = oracle.gc_coef_trace(p)
        infos.append({"coefs": co, "trace": trace})
    cent, hits, coefs = tap(vg, pcms, 4)
    bad = mismatches([f"short {i}" for i in range(len(pcms))], infos, None, cent, hits, coefs, 4)
    assert not bad, "\n".join(bad)


def test_phase1_records_and_mask(vg, oracle, stims):
    """Phase 1 on its own: the accept mask (every rejection reason, at the tile edges) and the direct-form records."""
    from vgaudio_b200 import _native as N

    for s in stims:
        frames = s.frames
        direct = np.zeros((max(frames, 1), 2))
        acc = np.zeros(max(frames, 1), np.uint8)
        pcm = np.ascontiguousarray(s.pcm)
        N.check(vg.lib.vgb_gcadpcm_debug_records(pcm.ctypes.data if pcm.size else None, len(pcm), direct.ctypes.data,
                                                 acc.ctypes.data))
        o_acc, _, o_dir = oracle.coef_records(pcm)
        assert np.array_equal(acc[:frames], o_acc), s.name
        sel = o_acc.astype(bool)
        assert np.array_equal(direct[:frames][sel].view(np.uint64), o_dir[sel].view(np.uint64)), s.name


def test_encode_path_agrees_with_the_tap(vg, oracle, stims, infos):
    """The production path (encode_batch: phase 1, the refinement without its tap, the encoder) gives the oracle's
    coefficients and bytes on the same stimuli."""
    coefs, adpcm = vg.gcadpcm.encode_batch([s.pcm for s in stims])
    for c, (s, i) in enumerate(zip(stims, infos)):
        assert np.array_equal(coefs[c], i["coefs"]), s.name
        assert adpcm[c].tobytes() == oracle.encode(s.pcm, i["coefs"]).tobytes(), s.name
