"""CPU tests of the oracle's CRI ADX frame trace (vgo_adx_encode_trace), of the coverage of the encoder stimulus set
(tests/adx_stimuli.py) that tests/test_criadx_paths_gpu.py runs on the GPU, and of the two integer identities the
encoders rest on (tools/adx_quantiser_check.c, tools/quantiser_check.c)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import adx_relock as R
import adx_stimuli as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def stims(oracle):
    return A.build()


@pytest.fixture(scope="module")
def traced(oracle, stims):
    return [oracle.adx_encode_trace(s.pcm, *s.args) for s in stims]


def test_trace_bytes_and_history_equal_encode(oracle, stims, traced):
    for s, (got, hist, trace) in zip(stims, traced):
        want, want_hist = oracle.adx_encode(s.pcm, *s.args)
        assert got.tobytes() == want.tobytes(), s.name
        assert hist == want_hist, s.name
        assert len(trace) == want.size // s.frame_size, s.name
        assert (trace["frame"] == np.arange(len(trace))).all(), s.name


def test_traced_facts_agree_with_the_bytes(stims, traced):
    """Header scale and filter bits, the nibble histogram and the history hand-over, recomputed from what was written."""
    for s, (got, _, tr) in zip(stims, traced):
        if not len(tr):
            continue
        fr = got.reshape(-1, s.frame_size).astype(np.int64)
        live = (tr["layout"] & A.O.ADX_FRAME_SKIPPED) == 0
        assert not fr[~live].any(), s.name                                   # `continue` leaves the frame zero
        assert np.array_equal(((fr[:, 0] & 0x1F) << 8 | fr[:, 1])[live], tr["scale_out"][live]), s.name
        assert np.array_equal((fr[:, 0] >> 5)[live], np.full(live.sum(), s.filter if s.type == 2 else 0)), s.name
        body = fr[:, 2:]
        nib = np.stack([body >> 4, body & 15], axis=2).reshape(len(fr), -1)
        hist = np.stack([np.bincount(row, minlength=16) for row in nib])
        assert np.array_equal(hist[live], tr["nibbles"][live]), s.name
        if s.type == 4:
            assert np.array_equal(tr["scale_out"][live], 12 - tr["power"][live]), s.name
            assert np.array_equal(tr["md_gain"][live], (8 << tr["power"][live]) - 1), s.name
        else:
            assert (tr["power"] == -1).all() and np.array_equal(tr["scale_out"][live], tr["scale_lin"][live]), s.name
            assert np.array_equal(tr["md_gain"][live], tr["max_distance"][live]), s.name
        assert np.array_equal(np.minimum(tr["scale_raw"], 0x1000) - 1, tr["scale_lin"]) or not live.all(), s.name
        idx = np.flatnonzero(live)
        assert np.array_equal(tr["hist_out"][idx[:-1]], tr["hist_in"][idx[1:]]), s.name


def test_coverage_matrix(stims, traced):
    """Every category on the 18-byte path and on the general path (the layout categories on the general path only)."""
    cov = A.coverage(stims, [t for _, _, t in traced])
    print("\n" + A.format_matrix(cov))
    empty = [(k, p) for k in A.CATEGORIES if k not in A.UNREACHED for p in ("std", "gen")
             if cov[k][p] == 0 and not (k in A.LAYOUT_ONLY and p == "std")]
    assert not empty, f"empty cells {empty}\n" + A.format_matrix(cov)
    assert all(cov[k]["std"] == 0 for k in A.LAYOUT_ONLY)
    assert all(cov[k]["std"] == cov[k]["gen"] == 0 for k in A.UNREACHED)


def test_layouts_and_types_of_the_set(stims):
    sizes = {s.frame_size for s in stims}
    assert {3, 10, 18, 34, 255} <= sizes
    assert {1, 31, 32, 45} <= {s.padding for s in stims}
    assert {(2, f) for f in range(4)} <= {(s.type, s.filter) for s in stims if s.type == 2}
    assert {3, 4} <= {s.type for s in stims} and {3, 4} == {s.version for s in stims}
    for std in (True, False):  # partial last frames on both paths' channels, and channels without one
        tails = {len(s.pcm) % ((s.frame_size - 2) * 2) == 0 for s in stims if s.std == std and s.role == "frame"}
        assert tails == {True, False}, std
    splice = [s for s in stims if s.role in ("fast", "slow", "never")]
    assert {len(s.pcm) % 32 for s in splice} == {0, 1, 31}
    assert any(s.whole == 0 and len(s.pcm) > 0 for s in stims if s.std)


def test_splice_material_relocks_as_labelled(oracle, stims):
    """Fast material re-locks within a few frames of a raw-history start, slow material takes tens to hundreds of
    frames, and the 500 Hz material (predictor 2 h1 - h2) never re-locks, so the cascade must carry its boundaries."""
    for s in stims:
        if s.role not in ("fast", "slow", "never"):
            continue
        r = R.census(oracle, s, cap=s.whole)
        if s.role == "fast":
            assert (r > 0).all() and r.max() <= 8, (s.name, r)
        elif s.role == "slow":
            assert np.median(r[r > 0]) >= 20, (s.name, r)
        else:
            assert (r == -1).all(), (s.name, r)


def test_cast_overflow_is_unreachable(oracle):
    """(int)(raw * gain) leaves int32 only when |raw| * 32767 >= 2^31 * maxDistance, i.e. |raw| >= 65538 * maxDistance.
    A pass-2 raw is an int16 sample minus a prediction of at most (|c0| + |c1|) * 32768 / 4096 <= 3 * 32768 (the
    computed pair is (2c, -c^2) in Q12 with 0 < c <= 1, the Fixed pairs are smaller), so |raw| <= 131072: Exponential
    frames (maxDistance >= 7) and maxDistance >= 2 cannot overflow.  maxDistance == 1 is left; this bounded search over
    rates (every divisor of 500 among them), types, versions and signals, with crafted maxDistance-1 frames, finds none."""
    rng = np.random.default_rng(41)
    rates = [1, 2, 4, 5, 10, 20, 25, 50, 100, 125, 250, 500, 600, 750, 1000, 1500, 2000, 4000, 8000, 48000]
    n = 32 * 24
    signals = [np.zeros(n, np.int16), rng.integers(-3, 4, n).astype(np.int16), rng.integers(-32768, 32768, n).astype(np.int16),
               np.repeat(rng.integers(-32768, 32768, n // 32), 32).astype(np.int16),
               np.cumsum(rng.integers(-2, 3, n)).astype(np.int16)]
    frames = small = 0
    for rate in rates:
        for typ, filt in ((2, 0), (2, 1), (2, 2), (2, 3), (3, 0), (4, 0)):
            for version in (3, 4):
                b = A.Builder(rng, rate, 18, version, 0, typ, filt)
                for _ in range(24):
                    b.craft(int(rng.choice([-1, 1])), int(rng.choice([-1, 0, 1])))
                for pcm in signals + [b.build("md1", 0).pcm]:
                    _, _, tr = oracle.adx_encode_trace(pcm, rate, 18, version, 0, typ, filt)
                    assert tr["cast_ovf"].sum() == 0, (rate, typ, filt, version)
                    frames += len(tr)
                    small += int((tr["md_gain"] == 1).sum())
    assert frames > 20000 and small > 2000, (frames, small)


def _cc():
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    return cc


@pytest.mark.parametrize("tool", ["adx_quantiser_check", "quantiser_check"])
def test_integer_quantiser_identity(tmp_path, tool):
    """The enumerations behind the encoders' integer quantisers: adx.cu's threshold count (every maxDistance 0..32768
    around every threshold, the full raw range for small maxDistance) and gc_encode.cu's rounding (every scale shift;
    about 20 s).  Exit code 0 means no mismatch."""
    exe = tmp_path / tool
    subprocess.run([_cc(), "-O2", "-ffp-contract=off", "-o", str(exe), os.path.join(ROOT, "tools", tool + ".c")], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
    assert "mismatch" not in r.stdout.replace("mismatches 0", ""), r.stdout[-2000:]
