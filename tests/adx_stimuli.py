"""Seeded CRI ADX encoder stimuli that reach every rare path of EncodeFrame (CriAdxCodec.cs:107-171) on the 18-byte
path and on the general path of adx.cu, and the splice paths of the time-parallel encoder.  Data generation only.

The oracle's frame trace (pyoracle.adx_encode_trace) records what the reference's EncodeFrame did; frame_categories()
turns it into the categories below.  tests/test_oracle_adx_trace.py proves the set reaches each of them, and
tests/test_criadx_paths_gpu.py encodes the set on the GPU.

  clip1_hi / clip1_lo   a pass-1 distance Clamp16 clips at +32767 / -32768        md_32768   maxDistance == 32768
  md_0                  maxDistance == 0 (gain 0, every nibble 0)                  scale_clamp  the 0x1000 clamp acts
  pow_<p>               the Exponential power p = 0..12                            so_<s>     scaleOut s = 2^m - 1, 2^m, 2^m + 1
  exp_so_pow2           an Exponential frame whose Linear scaleOut is a power of two (the edge of Helpers.Log2)
  tie_k<k>_md32767      |raw| * 32767 == T_k * 32767 (gain exactly 1.0), k = 1..7
  tie_k6_j<j>           |raw| * 32767 == T_6 * 4681 j, j = 1..6 (gain 7 / j; j = 3, 5, 6 are inexact in fp64)
  cast_ovf              raw * gain leaves int32 (the (int) cast gives INT_MIN)
  clip2_hi / clip2_lo   Clamp16 of the scaled distance clips                        recon_hi / recon_lo  the reconstruction clips
  v4_differs            a version-4 frame whose prediction differs from version 3's on some sample
  skipped / padded / partial   the frame's layout: all padding (`continue`), leading padding, zero-filled tail

Threshold frames are crafted: the builder tracks the reconstructed history (h1, h2) the oracle's encoder hands on, and a
crafted frame puts the residual r0 on its first sample and the distance d1 on its last, and keeps every distance between
within max(|r0|, |d1|), so pass 1 sees maxDistance = max(|r0|, |d1|) and pass 2 quantises r0 exactly.
"""
from __future__ import annotations

import dataclasses
from typing import List, Optional

import numpy as np

from oracle import pyoracle as O
from vgaudio_b200 import synth

T = [0] + [4681 * k - 2340 for k in range(1, 8)]                 # ScaleShortToNibble's thresholds T_1..T_7
FIXED_COEFS = [(0, 0), (0x0F00, 0), (0x1CC0, -3328), (0x1880, -3520)]
MIN_SEG_FRAMES = 4                                               # VGB_ADX_MIN_SEG_FRAMES for the forced-segment runs
SCALE_EDGES = sorted({0, 1, 2, 3, 4095} | {v for m in range(2, 12) for v in (2 ** m - 1, 2 ** m, 2 ** m + 1)})


@dataclasses.dataclass
class Stim:
    name: str
    pcm: np.ndarray
    rate: int = 48000
    frame_size: int = 18
    version: int = 4
    padding: int = 0
    type: int = 3
    filter: int = 0
    role: str = "frame"   # "frame": crafted paths; "fast", "slow", "never": splice material; "short": tiny channels

    @property
    def std(self) -> bool:
        """The 18-byte path of adx.cu (no padding); its partial last frame still takes the general loop."""
        return self.frame_size == 18 and self.padding == 0

    @property
    def whole(self) -> int:
        return len(self.pcm) // 32 if self.std else 0

    @property
    def args(self):
        return (self.rate, self.frame_size, self.version, self.padding, self.type, self.filter)

    def coefs(self):
        return FIXED_COEFS[self.filter] if self.type == 2 else tuple(int(c) for c in O.adx_coefficients(500, self.rate))


def _pred(a: int, b: int, c0: int, c1: int) -> int:
    return ((a * c0) >> 12) + ((b * c1) >> 12)


def shaped(h1, h2, c0, c1, spf, r0, d1) -> Optional[np.ndarray]:
    """A frame with residual r0 on its first sample and pass-1 distance d1 on its last; the samples between follow the
    raw-neighbour prediction pulled toward zero by at most m = max(|r0|, |d1|), so no distance exceeds m.  None when a
    sample leaves int16 (d1 = -32768 stands for a distance Clamp16 clips to 32768)."""
    m = max(abs(r0), abs(d1))
    x = [_pred(h1, h2, c0, c1) + r0]
    for i in range(1, spf):
        p = _pred(x[-1], x[-2] if i > 1 else h1, c0, c1)
        x.append(p + d1 if i == spf - 1 else p - min(max(p, -m), m))
    if min(x) < -32768 or max(x) > 32767:
        return None
    return np.array(x, np.int16)


class Builder:
    """One channel of a given layout, frame by frame, tracking the history the oracle's encoder hands on."""

    def __init__(self, rng, rate, frame_size, version, padding, type, filter=0):
        self.rng = rng
        self.layout = dict(rate=rate, frame_size=frame_size, version=version, padding=padding, type=type, filter=filter)
        self.spf = (frame_size - 2) * 2
        self.c0, self.c1 = FIXED_COEFS[filter] if type == 2 else tuple(int(c) for c in O.adx_coefficients(500, rate))
        # head: whatever real samples the padding leaves in its last frame, or one frame; quiet noise
        lead = padding % self.spf
        head = (rng.integers(-300, 300, self.spf - lead)).astype(np.int16)
        self.parts = [head]
        _, _, tr = O.adx_encode_trace(head, rate, frame_size, version, padding, type, filter)
        self.h1, self.h2 = (int(v) for v in tr[-1]["hist_out"])
        self.win = np.zeros(self.spf + 2, np.int16)

    def frame(self, x: np.ndarray):
        self.win[0], self.win[1] = self.h2, self.h1
        self.win[2:] = x
        O.adx_encode_frame(self.win, np.array([self.c0, self.c1], np.int16), self.spf, self.layout["type"],
                           self.layout["version"])
        self.h2, self.h1 = int(self.win[self.spf]), int(self.win[self.spf + 1])
        self.parts.append(np.asarray(x, np.int16))

    def craft(self, r0: int, d1: int, flips=True):
        """Appends shaped(r0, d1), trying sign flips, then quiet frames that settle the history, until it fits."""
        signs = [(1, 1), (-1, -1), (1, -1), (-1, 1)] if flips else [(1, 1)]
        for _ in range(8):
            for a, b in signs:
                x = shaped(self.h1, self.h2, self.c0, self.c1, self.spf, a * r0, b * d1)
                if x is not None:
                    self.frame(x)
                    return
            self.frame(np.zeros(self.spf, np.int16))
        raise RuntimeError(f"no room for a frame with r0={r0}, d1={d1} in {self.layout}")

    def build(self, name, tail: int) -> Stim:
        pcm = np.concatenate(self.parts + [self.rng.integers(-2000, 2000, tail).astype(np.int16)])
        return Stim(name, pcm, **self.layout)


def _frame_recipes(b: Builder):
    """Every crafted frame path, in one channel."""
    rng = b.rng
    typ = b.layout["type"]
    loud = 20000 if typ == 4 else 32767      # an Exponential maxDistance of power 12 gains exactly 1.0
    for k in range(1, 8):                    # ties at gain 1.0
        b.craft(T[k], loud)
    for j in range(1, 7):                    # T_6 = 7 * 3678 ties at maxDistance 4681 j
        b.craft(3678 * j, 4681 * j)
    for s in SCALE_EDGES:                    # Linear scaleOut s: maxDistance 7 s + 1
        b.craft(7 * s + 1, (7 * s + 1) // 2)
    b.craft(30000, 1000)                     # scale 4286: the 0x1000 clamp
    b.craft(0, 0)                            # maxDistance 0 from any history
    b.craft(12000, -32768, flips=False)      # a distance clipped at -32768: maxDistance 32768
    b.frame(np.resize(np.array([32767, 32767, -32768, -32768], np.int16), b.spf))   # full-scale square
    for _ in range(2):
        b.frame(rng.integers(-32768, 32768, b.spf).astype(np.int16))                # full-scale noise
    b.craft(0, 0)


# crafted channels: (rate, frame_size, version, padding, type, filter); the first ten take the 18-byte path
FRAME_LAYOUTS = [
    (48000, 18, 4, 0, 3, 0), (48000, 18, 3, 0, 3, 0), (44100, 18, 4, 0, 4, 0), (48000, 18, 3, 0, 4, 0),
    (48000, 18, 4, 0, 2, 0), (48000, 18, 3, 0, 2, 1), (48000, 18, 4, 0, 2, 2), (44100, 18, 3, 0, 2, 3),
    (8000, 18, 4, 0, 3, 0), (1000, 18, 3, 0, 4, 0),
    (48000, 3, 4, 1, 3, 0), (48000, 10, 3, 31, 4, 0), (44100, 34, 4, 32, 2, 2), (48000, 255, 4, 45, 4, 0),
    (48000, 10, 4, 0, 3, 0), (32000, 34, 3, 0, 2, 3), (48000, 18, 4, 1, 3, 0), (48000, 18, 3, 45, 4, 0),
    (22050, 255, 3, 0, 3, 0), (48000, 3, 3, 0, 2, 0), (48000, 18, 4, 32, 2, 1), (8000, 10, 4, 0, 4, 0),
]


def frame_stimuli(seed: int = 5) -> List[Stim]:
    rng = np.random.default_rng(seed)
    out = []
    for i, (rate, fs, v, pad, typ, filt) in enumerate(FRAME_LAYOUTS):
        b = Builder(rng, rate, fs, v, pad, typ, filt)
        _frame_recipes(b)
        spf = (fs - 2) * 2
        tail = (1, spf - 1, spf // 2, 0)[i % 4]   # partial last frames of several lengths, and none
        out.append(b.build(f"frames_t{typ}f{filt}_v{v}_fs{fs}_pad{pad}_{rate}", tail))
    return out


def splice_stimuli(seed: int = 9) -> List[Stim]:
    """18-byte material for the time-parallel encoder: re-locking fast (8000 Hz), slowly (48 kHz) and never (500 Hz,
    predictor (8192, -4096) = 2 h1 - h2, a double pole at z = 1), lengths 0, 1 and 31 (mod 32)."""
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate((32 * 1500, 32 * 1400 + 1, 32 * 1300 + 31)):
        noise = rng.integers(-6000, 6000, n).astype(np.int16)
        out.append(Stim(f"fast_8000_noise_{n % 32}", noise, 8000, version=4 - i % 2, type=3 + i % 2, role="fast"))
        out.append(Stim(f"fast_8000_synth_{n % 32}", synth.channel(60 + i, n, 8000, degenerate=False), 8000,
                        version=3 + i % 2, type=3, role="fast"))
        quiet = (synth.channel(70 + i, n, 8000, degenerate=False) // 64).astype(np.int16)
        out.append(Stim(f"fast_8000_quiet_{n % 32}", quiet, 8000, version=4, type=4 - i % 2, role="fast"))
        out.append(Stim(f"slow_48000_synth_{n % 32}", synth.channel(80 + i, n, 48000, degenerate=False), 48000,
                        version=4 - i % 2, type=3, role="slow"))
        out.append(Stim(f"never_500_noise_{n % 32}", rng.integers(-6000, 6000, n).astype(np.int16), 500,
                        version=4 - i % 2, type=3 + i % 2, role="never"))
    return out


def short_stimuli(seed: int = 13) -> List[Stim]:
    """18-byte channels with no or few whole frames: whole == 0 beside more segments, more segments than whole frames."""
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate((0, 1, 17, 31, 32, 33, 63, 64 + 31, 32 * 5 + 1, 32 * 9)):
        v = 3 if n == 0 else 4 - i % 2
        out.append(Stim(f"short_{n}", rng.integers(-20000, 20000, n).astype(np.int16), 48000, version=v,
                        type=2 + i % 3, filter=i % 4, role="short"))
    return out


def build() -> List[Stim]:
    return frame_stimuli() + splice_stimuli() + short_stimuli()


# ---- categories of the oracle's trace ---------------------------------------------------------------------------------
def _pow2(v: np.ndarray) -> np.ndarray:
    return (v > 0) & ((v & (v - 1)) == 0)


def frame_categories(trace: np.ndarray, version: int) -> dict:
    """{category: bool[frames]} of one channel's trace."""
    t = trace
    live = (t["layout"] & O.ADX_FRAME_SKIPPED) == 0
    c = {
        "clip1_hi": t["clip1_hi"] > 0, "clip1_lo": t["clip1_lo"] > 0,
        "md_32768": t["max_distance"] == 32768, "md_0": live & (t["max_distance"] == 0),
        "scale_clamp": t["scale_raw"] > 0x1000,
        "exp_so_pow2": (t["power"] >= 0) & _pow2(t["scale_lin"]),
        "cast_ovf": t["cast_ovf"] > 0, "clip2_hi": t["clip2_hi"] > 0, "clip2_lo": t["clip2_lo"] > 0,
        "recon_hi": t["recon_hi"] > 0, "recon_lo": t["recon_lo"] > 0,
        "v4_differs": (t["v4_differs"] > 0) & (version == 4),
        "skipped": ~live, "padded": (t["layout"] & O.ADX_FRAME_PADDED) != 0,
        "partial": (t["layout"] & O.ADX_FRAME_PARTIAL) != 0,
    }
    for p in range(13):
        c[f"pow_{p}"] = t["power"] == p
    for s in SCALE_EDGES:
        c[f"so_{s}"] = live & (t["scale_lin"] == s)
    for k in range(1, 8):
        c[f"tie_k{k}_md32767"] = (t["md_gain"] == 32767) & (t["ties"][:, k] > 0)
    for j in range(1, 7):
        c[f"tie_k6_j{j}"] = (t["md_gain"] == 4681 * j) & (t["ties"][:, 6] > 0)
    return c


CATEGORIES = tuple(frame_categories(np.zeros(0, O.ADX_FRAME_TRACE), 4))
LAYOUT_ONLY = ("skipped", "padded", "partial")   # general path by definition
# no stimulus reaches it, and none can: see test_oracle_adx_trace.test_cast_overflow_is_unreachable
UNREACHED = ("cast_ovf",)


def paths(s: Stim, n_frames: int) -> np.ndarray:
    """bool[frames]: True where adx.cu takes the 18-byte path (whole frames of a standard channel)."""
    return np.arange(n_frames) < s.whole


def coverage(stims, traces) -> dict:
    """{category: {"std": frames, "gen": frames}}"""
    cov = {k: {"std": 0, "gen": 0} for k in CATEGORIES}
    for s, tr in zip(stims, traces):
        cats = frame_categories(tr, s.version)
        std = paths(s, len(tr))
        for k, m in cats.items():
            cov[k]["std"] += int((m & std).sum())
            cov[k]["gen"] += int((m & ~std).sum())
    return cov


def format_matrix(cov) -> str:
    rows = [f"{'category':<20}{'18-byte':>10}{'general':>10}"]
    rows += [f"{k:<20}{v['std']:>10}{v['gen']:>10}" for k, v in cov.items()]
    return "\n".join(rows)


def categories_at(s: Stim, trace: np.ndarray, frame: int) -> List[str]:
    cats = frame_categories(trace, s.version)
    return [k for k in CATEGORIES if frame < len(trace) and cats[k][frame]]
