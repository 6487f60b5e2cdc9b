"""GPU tests of the GC-ADPCM encoder's warp layout (four channels per warp, gc_encode.cu) over the stimulus set of
tests/gc_stimuli.py, whose rare frames tests/test_oracle_gc_trace.py proves reach every exactness device in every
quarter slot.  Every channel is compared bit for bit with pyoracle.encode under its own coefficients and history, in
layouts that move it through every slot, next to different warp mates, across segment counts and host groups."""
import ctypes as C
import os

import numpy as np
import pytest

import gc_stimuli as G

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def stims(oracle):
    return G.build()


@pytest.fixture(scope="module")
def wanted(oracle, stims):
    return [oracle.encode(s.pcm, s.coefs, s.sample_count, s.h1, s.h2) for s in stims]


@pytest.fixture(scope="module")
def cats(stims):
    return [G.categories_of(s) for s in stims]


@pytest.fixture
def env():
    """set(name, value) for VGB_* knobs of the encode call; None removes one.  Restored after the test."""
    names = ("VGB_GC_SEGMENTS", "VGB_GC_MIN_SEG_FRAMES", "VGB_ENCODE_GROUPS")
    saved = {k: os.environ.get(k) for k in names}

    def set_(name, value):
        if value is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = str(value)

    yield set_
    for k, v in saved.items():
        set_(k, v)


def splice_stats(vg):
    from vgaudio_b200 import _native as N

    out = (C.c_uint64 * 4)()
    N.check(vg.lib.vgb_gcadpcm_debug_splice_stats(out, 4))
    return {"segments": int(out[0]), "runon_frames": int(out[1]), "cascade_frames": int(out[2])}


def encode_layout(vg, stims, order, with_coefs=True):
    P = vg.gcadpcm.GcAdpcmParameters
    chans = [stims[i].pcm for i in order]
    coefs = np.stack([stims[i].coefs for i in order]) if with_coefs else None
    configs = [P(stims[i].sample_count, stims[i].h1, stims[i].h2) for i in order]
    return vg.gcadpcm.encode_batch(chans, coefs, configs)


def check_layout(stims, wanted, cats, order, adpcm, what):
    bad = []
    for pos, i in enumerate(order):
        got = np.asarray(adpcm[pos], np.uint8)
        want = wanted[i]
        if got.tobytes() == want.tobytes():
            continue
        if got.size != want.size:
            bad.append(f"{stims[i].name} (slot {pos % 4}, position {pos}): {got.size} bytes, want {want.size}")
            continue
        f = int(np.flatnonzero(got != want)[0]) // 8
        here = [k for k in G.CATEGORIES if cats[i][k][f]]
        bad.append(f"{stims[i].name} (slot {pos % 4}, position {pos}): first differing frame {f} "
                   f"(chunk position {f % 16}), categories {here or 'none'}")
    assert not bad, f"{what}: " + "; ".join(bad)


@pytest.mark.parametrize("seg", [1, 3, 8, None])
def test_rotations_and_segment_counts(vg, stims, wanted, cats, env, seg):
    """Four rotations by one channel (every channel visits every quarter slot with different mates) and one by four
    (warp 0 and warp 1 of a CTA swapped), cut into 1, 3 and 8 segments of >= 256 frames and by the library's own
    choice."""
    env("VGB_GC_MIN_SEG_FRAMES", G.MIN_SEG_FRAMES)
    env("VGB_GC_SEGMENTS", seg)
    n = len(stims)
    for r in (0, 1, 2, 3, 4):
        order = G.rotation(n, r)
        _, adpcm = encode_layout(vg, stims, order)
        check_layout(stims, wanted, cats, order, adpcm, f"rotation {r}, segments {seg}")
        if seg is not None:
            assert splice_stats(vg)["segments"] == seg


def test_segmented_runs_reach_run_on_and_cascade(vg, stims, wanted, cats, env):
    """The splice machinery is exercised on this set: run-on frames and cascade frames both occur."""
    env("VGB_GC_MIN_SEG_FRAMES", G.MIN_SEG_FRAMES)
    seen = []
    for seg in (3, 8):
        env("VGB_GC_SEGMENTS", seg)
        order = G.rotation(len(stims), 0)
        _, adpcm = encode_layout(vg, stims, order)
        check_layout(stims, wanted, cats, order, adpcm, f"segments {seg}")
        seen.append(splice_stats(vg))
    assert max(s["runon_frames"] for s in seen) > 0, seen
    assert max(s["cascade_frames"] for s in seen) > 0, seen


@pytest.mark.parametrize("count", [1, 2, 3, 4, 5, 6, 7, 8, 9, 17])
def test_channel_counts_mod_8(vg, stims, wanted, cats, count):
    """The first N channels: every pattern of idle quarters and idle warps of a 2-warp CTA."""
    for r in (0, 1):
        order = G.rotation(len(stims), r)[:count]
        _, adpcm = encode_layout(vg, stims, order)
        check_layout(stims, wanted, cats, order, adpcm, f"{count} channels, rotation {r}")


def test_host_groups_cut_through_warps(vg, stims, wanted, cats, env):
    env("VGB_ENCODE_GROUPS", 3)
    for r in (0, 1):
        order = G.rotation(len(stims), r)
        _, adpcm = encode_layout(vg, stims, order)
        check_layout(stims, wanted, cats, order, adpcm, f"3 host groups, rotation {r}")


def test_computed_coefficients_feed_every_slot(vg, oracle, stims):
    """The natural channels without coefficients: the coefficient kernels feed the encoder in every quarter slot."""
    nat = [i for i, s in enumerate(stims) if s.natural]
    assert len(nat) >= 4
    for r in range(4):
        order = nat[r:] + nat[:r]
        coefs, adpcm = encode_layout(vg, stims, order, with_coefs=False)
        for pos, i in enumerate(order):
            s = stims[i]
            co = oracle.calculate_coefficients(s.pcm)
            assert np.array_equal(coefs[pos], co), (s.name, pos % 4)
            assert adpcm[pos].tobytes() == oracle.encode(s.pcm, co).tobytes(), (s.name, pos % 4)
