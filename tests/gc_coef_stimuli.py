"""Seeded GC-ADPCM coefficient stimuli that reach every rare path of phase 1 and of the refinement.  Data generation only.

gc_coef_refine_kernel (DESIGN.md §5.2) promises that every bucket's fp64 sum is added in record order, exactly like
FilterRecords.  A change of that order almost never moves the final int16 coefficients, so the tests compare every
pass's centroids and bucket counts instead: the oracle's coefficient trace (pyoracle.gc_coef_trace) records them, with
each pass's empty buckets and tied minima and each frame's phase-1 outcome.  refine() below restates
CalculateCoefficients / FilterRecords (GcAdpcmCoefficients.cs:63-108, :344-396) from the direct-form records in plain
Python; it reproduces the trace bit for bit, and its `mode` switches on the mutants the sensitivity self-check uses.

categories() names, per channel, what the kernel's rare paths see:
  no_frames / no_records / records_K     a channel without frames, with frames but no record (the NaN mean), K records
  mask_hole                              a 32-frame block with a rejected frame between two accepted ones
  rej_<reason>_at_<f>                    phase 1 rejects frame f (0, 255 or 256: the edges of a 256-frame tile of
                                         gc_coef_frames_kernel, frame 256 taking its history from the previous tile)
  one_bucket_nb<NB>                      a block of 32 records that all land in one bucket, in a pass with NB buckets
  queue_steps_nb<NB> / queue_pad_nb<NB>  a bucket's queue in a block that is / is not a whole number of consumer steps
  empty_bucket                           a pass 1..6 leaves a bucket without a record (the (1, 0, 0) reset)
  tie_same / tie_distinct                a record's minimum distance is shared by bit-identical / by distinct centroids
  tie_consequential                      a channel with a bit-identical tie, where handing tied records to the LAST
                                         minimum changes the trace
build() makes the set; the tie channels come from a bounded search over seeded candidates, driven by the trace.
"""
from __future__ import annotations

import dataclasses

import numpy as np

from vgaudio_b200 import synth

FRAME = 14
TILE = 256                    # frames per CTA tile of gc_coef_frames_kernel
PASSES = 7
PASS_BUCKETS = (1, 2, 2, 4, 4, 8, 8)
PRODUCERS = (3, 7)            # producer warps of the 4- and 8-warp refinement CTAs
K_DEPTH = 4                   # chunks a producer fetches ahead (gc_refine_pass)
REASONS = ("quiet", "big", "range", "den", "k1")  # pyoracle.GC_REJ_QUIET .. GC_REJ_K1
REJECT_AT = (0, 255, 256)


def step_of(nb: int) -> int:
    """refine_step of gc_coefs.cu: queue entries the consumer adds per iteration."""
    return 4 if nb >= 4 else (8 if nb == 2 else 16)


@dataclasses.dataclass
class Stim:
    name: str
    pcm: np.ndarray

    @property
    def frames(self) -> int:
        return (len(self.pcm) + FRAME - 1) // FRAME


# ---- a plain restatement of the refinement (GcAdpcmCoefficients.cs:63-108, :307-396) ---------------------------------
def _finish(k1, k2):
    if k1 >= 1.0:
        k1 = 0.9999999999
    elif k1 <= -1.0:
        k1 = -0.9999999999
    if k2 >= 1.0:
        k2 = 0.9999999999
    elif k2 <= -1.0:
        k2 = -0.9999999999
    return (1.0, (k2 * k1) + k1, k2)


def _from_mean(s0, s1, s2):
    """MergeFinishRecord (:307-333) of the mean vector (s0, s1, s2)."""
    err = s0
    t1 = (-(0.0 + s1) / err) if err > 0.0 else 0.0
    err *= 1.0 - (t1 * t1)
    acc = 0.0 + t1 * s1
    t2 = (-(acc + s2) / err) if err > 0.0 else 0.0
    return _finish(t1, t2)


def _ordered(xs):
    a = 0.0
    for x in xs:
        a += x
    return a


def _pairwise(xs):
    xs = list(xs)
    while len(xs) > 1:
        xs = [xs[i] + xs[i + 1] if i + 1 < len(xs) else xs[i] for i in range(0, len(xs), 2)]
    return 0.0 + xs[0] if xs else 0.0


def quantise(v) -> int:
    d = -v * 2048.0
    if d > 0.0:
        return 32767 if d > 32767.0 else int(np.rint(d))
    if d < -32768.0:
        return -32768
    if d != d:
        return 0
    return int(np.rint(d))


def direct_records(pcm) -> np.ndarray:
    """[records, 2] the accepted frames' direct-form pairs (MatrixFilter, :285-305), in record order."""
    from oracle import pyoracle

    acc, _, d = pyoracle.coef_records(pcm)
    return d[acc.astype(bool)]


def refine(recs: np.ndarray, mode: str | None = None) -> dict:
    """The refinement from the direct-form records.  mode None is the reference; "tree" sums each bucket pairwise,
    "lasttie" gives a tied record to the last minimum.  Returns the trace fields of pyoracle.GC_COEF_PASS per pass
    (cent [7, 8, 2], hits [7, 8], empty, ties_same, ties_distinct, tie_record, tie_lo, tie_hi), the bucket of every
    record in every pass (picks [7, records]) and the coefficients."""
    add = _pairwise if mode == "tree" else _ordered
    n = len(recs)
    r1, r2 = recs[:, 0].tolist(), recs[:, 1].tolist()
    out = {"cent": np.zeros((PASSES, 8, 2)), "hits": np.zeros((PASSES, 8), np.int32), "picks": [np.zeros(n, np.int64)],
           "empty": [int(n == 0)], "ties_same": [0], "ties_distinct": [0], "tie_record": [-1], "tie_lo": [-1],
           "tie_hi": [-1]}
    nan = float("nan")
    best = [_from_mean(1.0, _ordered(r1) / n if n else nan, _ordered(r2) / n if n else nan)] + [(1.0, 0.0, 0.0)] * 7
    out["hits"][0, 0] = n
    out["cent"][0] = [c[1:] for c in best]
    ta, tb = 2.0 * recs[:, 0], 2.0 * recs[:, 1]
    count, p = 1, 1
    for _ in range(3):
        for i in range(count):
            b = best[i]
            best[count + i] = ((0.01 * 0.0) + b[0], (0.01 * -1.0) + b[1], (0.01 * 0.0) + b[2])
        count *= 2
        for _ in range(2):
            dist = np.empty((n, count))
            for c in range(count):
                a0, a1, a2 = best[c]
                dist[:, c] = ((a0 * a0) + (a1 * a1) + (a2 * a2)) + (ta * ((a0 * a1) + (a1 * a2))) + (tb * (a0 * a2))
            dist = np.where(dist < 1.0e30, dist, np.inf)  # ContrastVectors' scan starts at 1e30; NaN never wins
            least = dist.min(axis=1) if n else np.zeros(0)
            if mode == "lasttie":
                pick = count - 1 - np.argmin(dist[:, ::-1], axis=1)
            else:
                pick = np.argmin(dist, axis=1)
            pick[~np.isfinite(least)] = 0
            tied = (dist == least[:, None]) & np.isfinite(least)[:, None]
            same = distinct = 0
            first = (-1, -1, -1)
            key = [np.array(c, np.float64).tobytes() for c in best]
            for z in np.flatnonzero(tied.sum(axis=1) > 1):
                idx = np.flatnonzero(tied[z])
                if len({key[c] for c in idx}) == 1:
                    same += 1
                else:
                    distinct += 1
                if first[0] < 0:
                    first = (int(z), int(idx[0]), int(idx[-1]))
            for c in range(count):
                sel = np.flatnonzero(pick == c)
                h = len(sel)
                s1, s2 = add(r1[z] for z in sel), add(r2[z] for z in sel)
                best[c] = _from_mean(1.0, s1 / h, s2 / h) if h else _from_mean(0.0, s1, s2)
                out["hits"][p, c] = h
            out["cent"][p] = [c[1:] for c in best]
            out["picks"].append(pick)
            out["empty"].append(int((out["hits"][p, :count] == 0).sum()))
            out["ties_same"].append(same)
            out["ties_distinct"].append(distinct)
            for k, v in zip(("tie_record", "tie_lo", "tie_hi"), first):
                out[k].append(v)
            p += 1
    out["coefs"] = np.array([quantise(best[z][k]) for z in range(8) for k in (1, 2)], np.int16)
    return out


def same_bits(a, b) -> np.ndarray:
    """Elementwise: the doubles have the same 64-bit pattern, or both are NaN (a NaN's payload is the platform's)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


def trace_fields_equal(trace, ref) -> list:
    """Names of the pyoracle.gc_coef_trace fields that differ from a refine() result (centroids as raw bits)."""
    P = trace["pass"]
    bad = []
    if not same_bits(P["cent"], ref["cent"]).all():
        bad.append("cent")
    if not np.array_equal(P["hits"], ref["hits"]):
        bad.append("hits")
    for k in ("empty", "ties_same", "ties_distinct", "tie_record", "tie_lo", "tie_hi"):
        if not np.array_equal(P[k], np.asarray(ref[k])):
            bad.append(k)
    return bad


# ---- categories ------------------------------------------------------------------------------------------------------
CATEGORIES = (("no_frames", "no_records") + tuple(f"records_{k}" for k in (1, 2, 7, 8, 9)) + ("mask_hole",)
              + tuple(f"rej_{r}_at_{f}" for r in REASONS for f in REJECT_AT)
              + tuple(f"one_bucket_nb{nb}" for nb in (1, 2, 4, 8))
              + tuple(f"queue_{k}_nb{nb}" for nb in (1, 2, 4, 8) for k in ("steps", "pad"))
              + ("empty_bucket", "tie_same", "tie_distinct", "tie_consequential"))
TIES = ("tie_same", "tie_consequential", "tie_distinct")  # found by search, or skipped with a reason


def analyse(s: Stim) -> dict:
    """The oracle trace of a stimulus and what the restatement adds: {coefs, trace, outcome, ref, last, cats}."""
    from oracle import pyoracle

    coefs, trace, outcome = pyoracle.gc_coef_trace(s.pcm)
    recs = direct_records(s.pcm)
    ref = refine(recs)
    P = trace["pass"]
    c = dict.fromkeys(CATEGORIES, 0)
    n_rec = int(trace["n_records"])
    c["no_frames"] = int(s.frames == 0)
    c["no_records"] = int(s.frames > 0 and n_rec == 0)
    for k in (1, 2, 7, 8, 9):
        c[f"records_{k}"] = int(n_rec == k)
    ok = outcome == pyoracle.GC_ACCEPTED
    for b in range(0, s.frames, 32):
        blk = ok[b:b + 32]
        acc = np.flatnonzero(blk)
        if acc.size >= 2 and not blk[acc[0]:acc[-1] + 1].all():
            c["mask_hole"] += 1
    for i, r in enumerate(REASONS):
        for f in REJECT_AT:
            c[f"rej_{r}_at_{f}"] = int(f < s.frames and outcome[f] == i + 1)
    block = np.flatnonzero(ok) // 32
    for p, nb in enumerate(PASS_BUCKETS):
        if n_rec == 0:
            break
        q = np.bincount(block * 8 + ref["picks"][p], minlength=8 * (block[-1] + 1)).reshape(-1, 8)[:, :nb]
        c[f"one_bucket_nb{nb}"] += int((q.max(axis=1) == 32).sum())
        c[f"queue_steps_nb{nb}"] += int(((q > 0) & (q % step_of(nb) == 0)).sum())
        c[f"queue_pad_nb{nb}"] += int((q % step_of(nb) != 0).sum())
    c["empty_bucket"] = int(P["empty"][1:].sum())
    c["tie_same"] = int(P["ties_same"].sum())
    c["tie_distinct"] = int(P["ties_distinct"].sum())
    last = None
    if c["tie_same"] + c["tie_distinct"]:
        last = refine(recs, "lasttie")
        c["tie_consequential"] = int(c["tie_same"] > 0 and bool(trace_fields_equal(trace, last)))
    return {"coefs": coefs, "trace": trace, "outcome": outcome, "ref": ref, "last": last, "cats": c}


def coverage(infos) -> dict:
    return {k: sum(i["cats"][k] for i in infos) for k in CATEGORIES}


def format_coverage(cov: dict) -> str:
    return "\n".join(f"{k:<22} {cov[k]:>7}" for k in CATEGORIES)


def shape_facts(stims) -> dict:
    """Launch shapes of the set: block counts, chunk counts per producer count, n mod 8, frames mod 32."""
    blocks = {(s.frames + 31) // 32 for s in stims if s.frames}
    return {
        "n_blocks": blocks,
        "chunks": {P: {(b + P - 1) // P for b in blocks} for P in PRODUCERS},
        "n_mod_8": {len(s.pcm) % 8 for s in stims if len(s.pcm)},
        "frames_mod_32": {s.frames % 32 for s in stims if s.frames},
        "partial_last_frame": any(len(s.pcm) % FRAME for s in stims),
    }


# ---- materials -------------------------------------------------------------------------------------------------------
def _put(pcm, f, win):
    """Writes the 16-sample window (two history samples, then frame f) into pcm; frame 0 takes zero history."""
    if f == 0:
        assert not win[:2].any()
        pcm[:FRAME] = win[2:]
    else:
        pcm[FRAME * f - 2: FRAME * f + FRAME] = win


def _outcome_of(win) -> int:
    from oracle import pyoracle

    return int(pyoracle.gc_coef_trace(np.concatenate([np.zeros(12, np.int16), win]))[2][1])


def reject_window(reason: str, rng, zero_history: bool, phase: int = 0) -> np.ndarray:
    """A window (two history samples + one frame) that phase 1 rejects for `reason`."""
    w = np.zeros(16, np.int16)
    if reason == "big":          # only the frame's last sample is non-zero: the covariance's first row is all zero
        w[15] = 3000
    elif reason == "range":      # a constant stretch: the 2x2 covariance is singular, lo / hi = 0
        w[:] = 1200
    elif reason == "den":        # A, 0, -A, 0, ...: x[t] = -x[t-2] exactly, so k2 = 1 and 1 - k2^2 == 0
        w[:] = np.array([2500, 0, -2500, 0], np.int16)[(np.arange(16) + phase) % 4]
    elif reason == "k1":         # searched: |k1| > 1 is common in white noise, and in random walks after zero history
        for t in range(1000):
            w = rng.integers(-3000, 3001, 16)
            w = (w if t % 2 == 0 else np.cumsum(w) // 4).astype(np.int16)
            if zero_history:
                w[:2] = 0
            if _outcome_of(w) == REASONS.index("k1") + 1:
                break
    if zero_history:
        w[:2] = 0
    assert _outcome_of(w) == REASONS.index(reason) + 1, reason
    return w


# A range rejection needs the lag-1 and lag-2 windows (x1..x14, x0..x13) nearly parallel.  Frame 0's history is zero,
# so x2 sits in the lag-1 window where the lag-2 window holds a zero: the constant and geometric windows tried keep
# lo / hi far above 1e-10 there, and the set does not place one.
UNPLACED = {("range", 0)}


def rejection_channels(rng) -> list:
    """Per reason two channels: rejected frames 0 and 255 in one, 256 (history from frame 255) in the other.  The lengths
    run through every residue mod 8 and end in partial frames."""
    out = []
    for i, reason in enumerate(REASONS):
        for j, at in enumerate(((0, 255), (256,))):
            n = 4200 + 17 * (2 * i + j)
            pcm = synth.channel(200 + 2 * i + j, n).copy()
            for f in at:
                if (reason, f) not in UNPLACED:
                    _put(pcm, f, reject_window(reason, rng, f == 0, phase=2))
            out.append(Stim(f"reject:{reason}:{'+'.join(map(str, at))}", pcm))
    return out


def sparse_records(k: int, rng, frames: int = 70) -> Stim:
    """Silence with exactly k accepted noise frames (the frame after each is silent and rejected as quiet)."""
    pcm = np.zeros(frames * FRAME - 5, np.int16)
    for f in range(1, 1 + 7 * k, 7):
        while True:
            w = np.zeros(16, np.int16)
            w[2:] = rng.integers(-2000, 2001, 14)
            if _outcome_of(w) == 0:
                break
        _put(pcm, f, w)
    return Stim(f"records:{k}", pcm)


def holes(rng) -> Stim:
    """Natural audio with a silent gap and clicks inside 32-frame blocks: the accept mask has holes."""
    pcm = synth.channel(300, FRAME * 200 + 9).copy()
    pcm[FRAME * 40: FRAME * 43] = 0                 # silent gap: frames 40-42 rejected as quiet
    _put(pcm, 50, reject_window("big", rng, False))  # a click on the frame's last sample
    pcm[FRAME * 70: FRAME * 72] = 0
    pcm[FRAME * 70 + 6] = 4000                      # a click mid-frame: accepted, record (0, 0)
    return Stim("holes", pcm)


# frames of the block-count channels: n_blocks 1, 1, 2, 3, 4, 6, 7, 8, 15, 40, 66 with frames mod 32 of 31, 0 and 1;
# 40 and 66 blocks give more than K_DEPTH chunks for both producer counts
BLOCK_FRAMES = (31, 32, 33, 95, 128, 161, 224, 255, 463, 1280, 2100)


def segments(seed: int, seg_frames: int = 96) -> np.ndarray:
    """Stationary segments of different character (tones, coloured noise, a near-silent hiss), each three blocks long:
    each segment's records cluster, so whole blocks land in one bucket."""
    rng = np.random.default_rng([0x636F, seed])
    n = seg_frames * FRAME
    t = np.arange(n)
    parts = []
    for kind in rng.permutation(6):
        if kind < 3:
            x = 9000 * np.sin(2 * np.pi * (150 + 900 * kind + rng.integers(0, 80)) / 48000 * t)
        elif kind == 3:
            x = np.cumsum(rng.normal(0, 300, n))
            x -= np.convolve(x, np.ones(64) / 64, "same")
        elif kind == 4:
            x = rng.normal(0, 40, n)
        else:
            x = np.diff(rng.normal(0, 3000, n + 1))
        parts.append(np.clip(np.round(x), -32768, 32767).astype(np.int16))
    return np.concatenate(parts)


def tie_candidate(seed: int) -> np.ndarray:
    """Natural audio or a tone, with white-noise frames and sparse clicks (frames whose records are exactly (0, 0)).  Every
    finite record is at distance exactly 1 from a centroid reset to (1, 0, 0), a (0, 0) record at 1 + c1^2 + c2^2 from
    every centroid: when two buckets are empty at once, such records tie between them."""
    rng = np.random.default_rng([0x7469, seed])
    frames = int(rng.integers(40, 200))
    if seed % 2:
        pcm = synth.reference_sine(frames * FRAME, float(rng.integers(100, 3000)), 48000)
        spots = rng.choice(frames, int(rng.integers(2, 8)), replace=False)
    else:
        pcm = synth.channel(400 + seed, frames * FRAME).copy()
        spots = rng.choice(frames, int(rng.integers(3, frames // 2)), replace=False)
    for f in spots:
        kind = rng.integers(0, 3)
        seg = pcm[FRAME * f: FRAME * f + FRAME]
        if kind == 0:    # clicks at least three samples apart: lag-1 and lag-2 correlations vanish
            seg[:] = 0
            seg[rng.integers(0, 3)::int(rng.integers(3, 6))] = rng.integers(-5000, 5001)
        elif kind == 1:
            seg[:] = rng.integers(-30000, 30001, FRAME)
        else:
            seg[:] = 0
    return pcm


TIE_TRIES = 60


def search_tie(category: str):
    """The first seeded candidate whose trace has the tie category; None if the bounded search finds none."""
    for t in range(TIE_TRIES):
        s = Stim(f"{category}:{t}", tie_candidate(1000 * TIES.index(category) + t))
        info = analyse(s)
        if info["cats"][category]:
            return s
    return None


def build() -> list:
    """The stimulus channels."""
    rng = np.random.default_rng(0x636F6566)
    out = [Stim("empty", np.zeros(0, np.int16)), Stim("silent", np.zeros(FRAME * 40 + 5, np.int16))]
    out += [sparse_records(k, rng) for k in (1, 2, 7, 8, 9)]
    out += rejection_channels(rng)
    out.append(holes(rng))
    for i, f in enumerate(BLOCK_FRAMES):
        out.append(Stim(f"blocks:{f}", synth.channel(500 + i, FRAME * f - (3 * i) % FRAME)))
    out += [Stim(f"segments:{k}", segments(k)) for k in range(2)]
    for cat in TIES:
        s = search_tie(cat)
        if s is not None:
            out.append(s)
    return out
