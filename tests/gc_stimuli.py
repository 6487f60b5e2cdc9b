"""Seeded GC-ADPCM encoder stimuli that reach every rare path of the scale chain and the argmin.  Data generation only.

The encoder's exactness devices (DESIGN.md §5.3) only matter on rare frames.  The oracle's frame trace
(pyoracle.gc_encode_trace) records, per frame and predictor, what the reference's DspEncodeCoef did; frame_categories()
turns that into the categories below, each evaluated on the WINNING predictor's chain (a device that misfires on a
losing predictor cannot change the bytes):

  C1  the winner's chain needs 3 or 4 passes                   C5  a pass of the winner has |diff| >= 2^24
  C2  the winner's chain needs >= 5 passes                     C6  the minimum error is >= 2^27 - 1
  C3  the winner's chain bumps (over + 8 > 256 below 12)       C6b some error >= 2^27 - 1, the minimum below it
  C4  the winner's chain ends on a pass at 12 with over > 1    C7  another predictor ties the winner's error
  C8  a prediction sum or difference of the winner's chain     (quiet: min < 2^27 - 1; loud: C6 as well)
      wraps int32

`*hi` variants ask for the winner among predictors 4..7; C3_248 / C3_249 are the near miss and the exact edge of the
bump.  The `*_alone` flags mark frames where the rare path is the only unusual thing in the channel's frame (the other
predictors "calm": at most 4 passes, no bump, every |diff| < 2^24), so that a wrong decision there shows in the bytes:
C3hi_alone (the winner 4..7 bumps, predictors 0..3 calm), C6_alone (a loud frame won by a predictor other than 0, every
chain plain and below 2^29), C2hi_alone and C3_249_alone (the winner bumps at exactly 249 and the pass the bump skips
would have ended its chain).  The bounded search finds no C2, C2hi_alone or C3_249_alone frame: a predictor whose
chain is that long or that unstable does not win its frame on these materials.

build() makes the channel set.  Threshold cases are not crafted: a seeded search over candidate channels keeps the
first candidate whose trace has the case (history is serial, so a crafted frame could not be spliced into a channel).
"""
from __future__ import annotations

import dataclasses

import numpy as np

from vgaudio_b200 import synth

ERR_SAT = (1 << 27) - 1
BIG = 1 << 24
HUGE = 1 << 29
FRAME = 14

CATEGORIES = ("C1", "C1hi", "C2", "C2hi", "C3", "C3hi", "C3_248", "C3_249", "C4", "C5", "C6", "C6b", "C7", "C7loud",
              "C8", "C2hi_alone", "C3hi_alone", "C3_249_alone", "C6_alone")
# categories the matrix also places at chunk position 0 and 15 and at the first frame of a segment
PLACED = ("C1", "C3", "C5", "C6")
SEGMENT_COUNTS = (1, 3, 8)
MIN_SEG_FRAMES = 256
CHUNK_FRAMES = 16


@dataclasses.dataclass
class Stim:
    name: str
    pcm: np.ndarray
    coefs: np.ndarray
    sample_count: int = -1
    h1: int = 0
    h2: int = 0
    natural: bool = False  # coefficients are CalculateCoefficients' (the set the coefficient kernels reproduce)

    @property
    def n_enc(self) -> int:
        return len(self.pcm) if self.sample_count == -1 else self.sample_count

    @property
    def frames(self) -> int:
        return (self.n_enc + FRAME - 1) // FRAME


# ---- a plain restatement of DspEncodeCoef (GcAdpcmEncoder.cs:96-171), used to look at one pass in isolation ----------
def _wrap(v: int) -> int:
    return ((v + 0x80000000) & 0xFFFFFFFF) - 0x80000000


def _sat(v: int, lo: int, hi: int) -> int:
    return lo if v < lo else (hi if v > hi else v)


def _trunc_div(a: int, b: int) -> int:
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def py_pass(win, c0: int, c1: int, sp: int):
    """One do/while pass at scalePower sp from the window win[0..15] (history older first): (over, error, recon,
    max |diff|, wrapped)."""
    recon = [int(win[0]), int(win[1])]
    scale = (1 << sp) * 2048
    over, err, peak, wrapped = 0, 0, 0, False
    for s in range(14):
        want = int(win[s + 2]) * 2048
        wide = recon[s] * c1 + recon[s + 1] * c0
        guess = _wrap(wide)
        diff = _wrap(want - guess)
        wrapped |= wide != guess or diff != want - guess
        peak = max(peak, abs(diff))
        ratio = np.float32(diff) / np.float32(scale)
        half = float(np.float32(0.4999999))
        raw = int(float(ratio) + half) if diff > 0 else int(float(ratio) - half)
        q = _sat(raw, -8, 7)
        if q != raw:
            over = max(over, abs(raw - q))
        out = _sat(_wrap(guess + q * scale + 1024) >> 11, -32768, 32767)
        recon.append(out)
        err += (int(win[s + 2]) - out) ** 2
    return over, err, recon, peak, wrapped


def py_try_predictor(win, c0: int, c1: int):
    """The whole chain, with the facts vgo_gc_encode_trace records for one predictor."""
    peak, wrapped = 0, False
    for s in range(14):
        wide = int(win[s]) * c1 + int(win[s + 1]) * c0
        wrapped |= wide != _wrap(wide)
        diff = _sat(_wrap(int(win[s + 2]) - _trunc_div(_wrap(wide), 2048)), -32768, 32767)
        if abs(diff) > abs(peak):
            peak = diff
    sp = 0
    while sp <= 12 and (peak > 7 or peak < -8):
        peak = _trunc_div(peak, 2)
        sp += 1
    sp = -1 if sp <= 1 else sp - 2
    rec = dict(first_sp=sp + 1, over=[], bumped=False, final12=False, wrapped=wrapped, max_abs_diff=0)
    while True:
        sp += 1
        over, err, recon, mad, wr = py_pass(win, c0, c1, sp)
        rec["over"].append(over)
        rec["wrapped"] |= wr
        rec["max_abs_diff"] = max(rec["max_abs_diff"], mad)
        pass_power = sp
        if over + 8 > 256 and pass_power < 12:
            rec["bumped"] = True
        if pass_power >= 12 and over > 1:
            rec["final12"] = True
        x = over + 8
        while x > 256:
            sp += 1
            if sp >= 12:
                sp = 11
            x >>= 1
        if pass_power >= 12:
            sp = 12
            break
        if not (sp < 12 and over > 1):
            break
    rec.update(final_sp=sp, error=err, n_passes=len(rec["over"]), recon=recon)
    return rec


def pass_powers(first_sp: int, overs) -> list:
    """The scalePower of each pass of a chain, from its first power and the over of each pass (:118-170)."""
    out, sp = [], first_sp
    for o in overs:
        out.append(sp)
        x = o + 8
        while x > 256:
            sp = min(sp + 1, 11)
            x >>= 1
        sp += 1
    return out


# ---- categories ------------------------------------------------------------------------------------------------------
def frame_categories(trace, pcm=None, coefs=None, sample_count=-1, h1=0, h2=0) -> dict:
    """{category: bool[frames]} from a pyoracle.gc_encode_trace record array.  C3_249_alone needs the channel itself
    (pcm, coefs, history) to look at the pass the bump skips; without it that flag is all False."""
    pred = trace["pred"]
    nf = len(trace)
    w = trace["winner"].astype(np.int64)
    idx = np.arange(nf)
    W = pred[idx, w]
    err = pred["error"]
    emin = err.min(axis=1) if nf else np.zeros(0, np.uint64)
    hi = w >= 4
    npass = W["n_passes"].astype(np.int64)
    over = W["over"]
    col = np.arange(13)[None, :]
    not_last = col < (npass[:, None] - 1)  # a pass with over > 248 below 12 is never the last one
    c = {}
    c["C1"] = (npass == 3) | (npass == 4)
    c["C2"] = npass >= 5
    c["C3"] = W["bumped"].astype(bool)
    c["C3_248"] = ((over == 248) & not_last).any(axis=1)
    c["C3_249"] = ((over == 249) & not_last).any(axis=1)
    c["C4"] = W["final12"].astype(bool)
    c["C5"] = W["max_abs_diff"] >= BIG
    c["C6"] = emin >= ERR_SAT
    c["C6b"] = (emin < ERR_SAT) & (err >= ERR_SAT).any(axis=1)
    c["C7"] = trace["tie"].astype(bool) & (emin < ERR_SAT)
    c["C7loud"] = trace["tie"].astype(bool) & c["C6"]
    c["C8"] = W["wrapped"].astype(bool)
    for k in ("C1", "C2", "C3"):
        c[k + "hi"] = c[k] & hi
    plain = (pred["n_passes"] <= 4) & (pred["bumped"] == 0)            # [frames, 8]
    calm = plain & (pred["max_abs_diff"] < BIG)
    # the winner (4..7) needs >= 5 passes or bumps, and predictors 0..3 are all calm
    c["C2hi_alone"] = c["C2hi"] & calm[:, :4].all(axis=1)
    c["C3hi_alone"] = c["C3hi"] & calm[:, :4].all(axis=1)
    # a loud frame whose winner is not predictor 0, every chain plain and below 2^29 (a loud frame cannot be calm:
    # it needs |diff| >= 2^24)
    c["C6_alone"] = c["C6"] & (w != 0) & (plain & (pred["max_abs_diff"] < HUGE)).all(axis=1)
    c["C3_249_alone"] = np.zeros(nf, bool)
    if pcm is not None:
        others_calm = calm.sum(axis=1) - calm[idx, w] == 7
        cand = np.flatnonzero(c["C3_249"] & others_calm & (W["max_abs_diff"] < BIG))
        if cand.size:
            recon = frame_windows(pcm, coefs, sample_count, h1, h2)
            for f in cand:
                c["C3_249_alone"][f] = _bump_249_skips_an_ending_pass(W[f], recon[f], int(coefs[2 * w[f]]),
                                                                      int(coefs[2 * w[f] + 1]))
    return c


def _bump_249_skips_an_ending_pass(rec, win, c0, c1) -> bool:
    """The winner bumps at over == 249 at power p <= 10 among its first three passes, and the pass at p + 1 that the
    bump skips would have ended the chain (over <= 1): a bump missed at exactly 249 changes the bytes."""
    overs = [int(v) for v in rec["over"][: int(rec["n_passes"])]]
    powers = pass_powers(int(rec["first_sp"]), overs)
    for k, (o, p) in enumerate(zip(overs, powers)):
        if o > 248:
            if o == 249 and k <= 2 and p <= 10 and k < len(overs) - 1:
                return py_pass(win, c0, c1, p + 1)[0] <= 1
            return False
    return False


def frame_windows(pcm, coefs, sample_count=-1, h1=0, h2=0) -> np.ndarray:
    """[frames, 16] int16: the window each frame of the encode starts from (two reconstructed history samples, older
    first, then the 14 input samples zero-padded) - what DspEncodeFrame sees (:30-41).  The encoder's reconstruction
    is the decoder's output (GcAdpcmAlignmentTests.cs:92-108, test_encoder_reconstruction_equals_decoder)."""
    from oracle import pyoracle

    n = len(pcm) if sample_count == -1 else sample_count
    nf = (n + FRAME - 1) // FRAME
    ad = pyoracle.encode(pcm, coefs, sample_count, h1, h2)
    dec = pyoracle.decode(ad, coefs, n, h1, h2) if n else np.zeros(0, np.int16)
    src = np.zeros(nf * FRAME, np.int64)
    src[:n] = np.asarray(pcm[:n], np.int64)
    win = np.zeros((nf, 16), np.int16)
    hist = np.concatenate([[h2, h1], dec.astype(np.int64)])
    for f in range(nf):
        win[f, 0], win[f, 1] = hist[14 * f], hist[14 * f + 1]
        win[f, 2:] = src[14 * f: 14 * f + 14]
    return win


# ---- materials -------------------------------------------------------------------------------------------------------
UNSTABLE = np.array([4095, -2047, 4000, -1900, 3800, -2000, 2048, -1024], dtype=np.int16)
HOSTILE = np.array([-32768, 32767, -20000, 20000, 0, 2048], dtype=np.int16)


def white(rng, n, amp=32768):
    return rng.integers(-amp, amp, n).astype(np.int16)


def nyquist_square(n, period=2):
    return np.where((np.arange(n) // (period // 2)) % 2 == 0, 32767, -32768).astype(np.int16)


def hostile_pcm(rng, n):
    x = np.where(rng.random(n) < 0.5, -32768, 32767).astype(np.int16)
    x[::3] = rng.integers(-32768, 32768, len(x[::3]))
    return x


def material(kind: str, seed: int, n: int):
    """(pcm, coefs, natural) for one candidate channel of the given kind."""
    from oracle import pyoracle

    rng = np.random.default_rng([0x6743, seed])
    if kind == "synth":
        x = synth.channel(40 + seed, n)
        return x, pyoracle.calculate_coefficients(x), True
    if kind == "sine":  # the reference suite's 261.63 Hz sine: its own coefficients bump, some at exactly 249
        x = synth.reference_sine(n, 261.63, 48000)
        return x, pyoracle.calculate_coefficients(x), True
    if kind == "white":
        x = white(rng, n)
        return x, pyoracle.calculate_coefficients(x), True
    if kind == "white_random":
        return white(rng, n, int(rng.choice([4096, 16384, 32768]))), rng.integers(-6000, 6001, 16).astype(np.int16), False
    if kind == "square":
        return nyquist_square(n, int(rng.choice([2, 4, 8]))), rng.choice(UNSTABLE, 16), False
    if kind == "unstable":
        x = white(rng, n, int(rng.choice([256, 2048, 8192, 32768])))
        if rng.random() < 0.5:
            x = np.clip(np.cumsum(x.astype(np.int64) // 64), -32768, 32767).astype(np.int16)  # slow, drifting material
        return x, rng.choice(UNSTABLE, 16), False
    if kind == "ramp_unstable":  # steps and ramps through a first-order pole just outside the unit circle
        steps = rng.integers(-300, 301, n // 64 + 1).repeat(64)[:n]
        x = np.clip(np.cumsum(steps), -32768, 32767).astype(np.int16)
        pole = rng.integers(2100, 3300, 8)
        co = np.zeros(16, np.int16)
        co[0::2] = pole
        co[1::2] = rng.integers(-600, 300, 8)
        return x, co, False
    if kind == "split":  # predictors 0..3 plain first-order sets, 4..7 resonant / unstable ones, on smooth material
        x = np.clip(np.cumsum(rng.integers(-64, 65, n)), -8000, 8000).astype(np.int16)
        co = rng.choice(UNSTABLE, 16)
        co[:8] = rng.integers(-1024, 2048, 8)
        co[1:8:2] = 0
        return x, co, False
    if kind == "hostile":
        return hostile_pcm(rng, n), rng.choice(HOSTILE, 16), False
    raise ValueError(kind)


def trace_of(s: Stim):
    from oracle import pyoracle

    return pyoracle.gc_encode_trace(s.pcm, s.coefs, s.sample_count, s.h1, s.h2)


def categories_of(s: Stim, trace=None) -> dict:
    if trace is None:
        trace = trace_of(s)[1]
    return frame_categories(trace, s.pcm, s.coefs, s.sample_count, s.h1, s.h2)


# searched cases: (category the candidate must contain, material kinds tried in turn)
SEARCHES = (
    ("C3hi_alone", ("split",)),
    ("C3_248", ("unstable", "ramp_unstable", "hostile")),
    ("C3_249", ("hostile", "unstable", "ramp_unstable")),
    ("C6_alone", ("white_random", "white", "unstable")),
    ("C7loud", ("hostile", "square", "unstable")),
    ("C6b", ("white_random", "unstable", "hostile")),
    ("C4", ("hostile", "unstable")),
    ("C8", ("hostile",)),
    ("C1hi", ("synth", "unstable")),
    ("C3hi", ("unstable", "hostile")),
    ("C3_249_alone", ("hostile", "ramp_unstable", "unstable")),
)
SEARCH_FRAMES = 600
SEARCH_TRIES = 24


def search(k: int, frames: int = SEARCH_FRAMES, tries: int = SEARCH_TRIES):
    """The first candidate of search k (seeded, bounded) whose trace has the case in at least three frames; None if
    none does."""
    case, kinds = SEARCHES[k]
    for t in range(tries):
        kind = kinds[t % len(kinds)]
        pcm, co, natural = material(kind, 1000 * (1 + k) + t, frames * FRAME)
        s = Stim(f"{case}:{kind}:{t}", pcm, co, natural=natural)
        if categories_of(s)[case].sum() >= 3:
            return s
    return None


# lengths (frames) of the short channels: warp mates end at frames 15, 16, 17, 31, 32 and 33; some last frames partial
SHORT = ((15, 0), (16, 3), (17, 0), (31, 13), (32, 0), (33, 7))
LONG_FRAMES = 2100


def build(long_frames: int = LONG_FRAMES) -> list:
    """The stimulus channels, a multiple of 8 of them (two warps of a CTA)."""
    from oracle import pyoracle

    out = [s for s in (search(k) for k in range(len(SEARCHES))) if s is not None]
    found = len(out)
    rng = np.random.default_rng(0x57494D)
    n = long_frames * FRAME
    # long channels of every material, with odd sample counts, histories and a partial last frame
    for i, kind in enumerate(("synth", "white", "hostile", "unstable", "square", "ramp_unstable", "white_random",
                              "synth", "sine")):
        pcm, co, natural = material(kind, 50 + i, n - 5 * i)
        sc, h1, h2 = -1, 0, 0
        if i % 2:
            sc, h1, h2 = len(pcm) - 11 * i, int(rng.integers(-32768, 32768)), int(rng.integers(-32768, 32768))
        out.append(Stim(f"long:{kind}:{i}", pcm, co, sc, h1, h2, natural=natural and sc == -1 and h1 == 0 and h2 == 0))
    # C1 is sparse: search long candidates that have it on a segment's first frame for every segment count
    # (a C1 frame at a multiple of 16 becomes a segment start when the channel is cut to S times that many frames;
    # cutting a channel leaves its earlier frames as they are)
    for S in SEGMENT_COUNTS[1:]:
        for t in range(SEARCH_TRIES):
            kind = ("ramp_unstable", "unstable")[t % 2]
            pcm, co, _ = material(kind, 9000 + 100 * S + t, n)
            c1 = categories_of(Stim("", pcm, co))["C1"]
            at = [f for f in range(MIN_SEG_FRAMES, long_frames // S + 1, CHUNK_FRAMES) if c1[f]]
            if at:
                out.append(Stim(f"C1_at_segment_start_{S}:{kind}:{t}", pcm[: at[-1] * S * FRAME - 3], co))
                break
    # the searched channels are short: stretch them to the long length so that every segment count cuts them
    for k, s in enumerate(out[:found]):
        if len(s.pcm) < n:
            kind = s.name.split(":")[1]
            tail, _, _ = material(kind, 7000 + k, n - len(s.pcm))
            out[k] = Stim(s.name, np.concatenate([s.pcm, tail]), s.coefs)  # the searched frames stay as found
    kinds = ("hostile", "unstable", "synth", "white_random", "square", "synth")
    for i, (frames, short_by) in enumerate(SHORT):
        pcm, co, natural = material(kinds[i], 80 + i, frames * FRAME - short_by)
        out.append(Stim(f"short:{frames}:{kinds[i]}", pcm, co, natural=natural))
    out.append(Stim("empty", np.zeros(0, np.int16), rng.integers(-4096, 4096, 16).astype(np.int16)))
    pad = 0
    while len(out) % 8:
        pcm, co, natural = material("synth", 90 + pad, 14 * 700 + 3)
        out.append(Stim(f"fill:synth:{pad}", pcm, co, natural=natural))
        pad += 1
    # spread the short channels out: every warp of every rotation keeps long warp mates
    longs = [s for s in out if s.frames > 2 * max(f for f, _ in SHORT)]
    shorts = [s for s in out if s.frames <= 2 * max(f for f, _ in SHORT)]
    step = max(len(out) // max(len(shorts), 1), 1)
    order = []
    for i in range(len(out)):
        order.append(shorts.pop(0) if i % step == step - 1 and shorts else (longs.pop(0) if longs else shorts.pop(0)))
    return order


# ---- layouts ---------------------------------------------------------------------------------------------------------
def rotation(n: int, r: int) -> list:
    """Channel order of layout r: the stimulus list rotated left by r (position p holds channel (p + r) % n)."""
    return [(p + r) % n for p in range(n)]


def segment_starts(frames: int, seg_count: int, min_seg: int = MIN_SEG_FRAMES) -> list:
    """First frames of a channel's segments: gc_seg_len of gc_encode.cu with frame_begin = 0."""
    if frames <= 0:
        return []
    per = (-(-frames // max(seg_count, 1)) + CHUNK_FRAMES - 1) // CHUNK_FRAMES * CHUNK_FRAMES
    seg_len = max(per, min_seg)
    return [j * seg_len for j in range(seg_count) if j * seg_len < frames]


def coverage(stims, cats, rotations=range(4)) -> dict:
    """Where the categories land when the stimulus list is encoded in the given rotations (four channels per warp,
    quarter slot = position % 4).  Returns {category: {cell: count}} with the cells
      ("has", q)   the channel in slot q has the category at frame f and a live warp mate at frame f does not
      ("lacks", q) the channel in slot q lacks it at frame f (but encodes f) and a live warp mate has it
      ("pos15",) / ("pos0",)          "has" at chunk position 15 / 0, any slot
      ("seg", S)                     "has" at the first frame of a segment other than frame 0, S segments
    cats: the frame_categories() of every stimulus."""
    n = len(stims)
    frames = np.array([s.frames for s in stims])
    cell = {k: {} for k in CATEGORIES}
    seg_first = [{S: set(segment_starts(int(frames[i]), S)[1:]) for S in SEGMENT_COUNTS} for i in range(n)]
    for r in rotations:
        order = rotation(n, r)
        for w0 in range(0, n, 4):
            mates = order[w0: w0 + 4]
            top = max(frames[m] for m in mates)
            for k in CATEGORIES:
                # [4, top]: 1 has, 0 lacks, -1 the channel has no frame there
                grid = np.full((len(mates), top), -1, np.int8)
                for j, m in enumerate(mates):
                    grid[j, : frames[m]] = cats[m][k]
                has = grid == 1
                lacks = grid == 0
                for j, m in enumerate(mates):
                    others_lack = np.zeros(top, bool)
                    others_have = np.zeros(top, bool)
                    for jj in range(len(mates)):
                        if jj != j:
                            others_lack |= lacks[jj]
                            others_have |= has[jj]
                    fwd = has[j] & others_lack
                    rev = lacks[j] & others_have
                    q = j  # positions w0..w0+3 are slots 0..3
                    c = cell[k]
                    c[("has", q)] = c.get(("has", q), 0) + int(fwd.sum())
                    c[("lacks", q)] = c.get(("lacks", q), 0) + int(rev.sum())
                    f = np.flatnonzero(fwd)
                    c[("pos15",)] = c.get(("pos15",), 0) + int((f % CHUNK_FRAMES == 15).sum())
                    c[("pos0",)] = c.get(("pos0",), 0) + int((f % CHUNK_FRAMES == 0).sum())
                    for S in SEGMENT_COUNTS:
                        c[("seg", S)] = c.get(("seg", S), 0) + sum(1 for x in f if x in seg_first[m][S])
    return cell


def required_cells(k: str) -> list:
    cells = [(d, q) for q in range(4) for d in ("has", "lacks")]
    if k in PLACED:
        cells += [("pos15",), ("pos0",)] + [("seg", S) for S in SEGMENT_COUNTS if S > 1]
    return cells


def format_matrix(cell, keys=CATEGORIES) -> str:
    cols = [(d, q) for q in range(4) for d in ("has", "lacks")] + [("pos15",), ("pos0",)] + \
           [("seg", S) for S in SEGMENT_COUNTS if S > 1]
    head = "category      " + " ".join(f"{'/'.join(map(str, c)):>9}" for c in cols)
    rows = [head] + [f"{k:<13} " + " ".join(f"{cell[k].get(c, 0):>9}" for c in cols) for k in keys]
    return "\n".join(rows)
