"""Re-lock census of the GC-ADPCM decoder (GcAdpcmDecoder.cs:10-54) on the CPU: started at frame k from a wrong
(hist1, hist2), after how many frames does the decoder's frame-end pair equal the true one?  From there its output is
the true output, which is what the run-on phase of the time-parallel decoder (gc_decode_seg_kernel) relies on.

The decoder is restated here with numpy over many (channel, start) trials at once; the truth is the oracle's decode."""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np


def _wrap32(v: np.ndarray) -> np.ndarray:
    return ((v + (1 << 31)) % (1 << 32)) - (1 << 31)


def relock_frames(adpcm: np.ndarray, coefs: np.ndarray, truth: np.ndarray, starts: Sequence[int], pairs: Sequence[Tuple[int, int]],
                  cap: int) -> np.ndarray:
    """For each trial t: decode the full frames of one channel from frame starts[t] with history pairs[t]; the number of
    frames decoded until (and including) the first whose end pair equals the truth's, or -1 when none does within `cap`
    frames or before the channel's full frames end."""
    adpcm = np.asarray(adpcm, np.uint8)
    co = np.asarray(coefs, np.int64).reshape(8, 2)
    truth = np.asarray(truth, np.int64)
    full = truth.size // 14
    starts = np.asarray(starts, np.int64)
    h1 = np.array([p[0] for p in pairs], np.int64)
    h2 = np.array([p[1] for p in pairs], np.int64)
    out = np.full(starts.size, -1, np.int64)
    live = np.ones(starts.size, bool)
    for t in range(cap):
        f = starts + t
        live &= f < full
        if not live.any():
            break
        idx = np.nonzero(live)[0]
        fi = f[idx]
        head = adpcm[fi * 8].astype(np.int64)
        pred, sp = (head >> 4) & 7, head & 0xF
        c1, c2 = co[pred, 0], co[pred, 1]
        scale = (1 << sp) * 2048
        a, b = h1[idx], h2[idx]
        for s in range(14):
            byte = adpcm[fi * 8 + 1 + s // 2].astype(np.int64)
            nib = (byte >> 4) if s % 2 == 0 else (byte & 0xF)
            nib = np.where(nib >= 8, nib - 16, nib)
            v = _wrap32(nib * scale + 1024 + c1 * a + c2 * b) >> 11
            v = np.clip(v, -32768, 32767)
            b, a = a, v
        h1[idx], h2[idx] = a, b
        hit = (a == truth[fi * 14 + 13]) & (b == truth[fi * 14 + 12])
        done = idx[hit]
        out[done] = t + 1
        live[done] = False
    return out


def census(oracle, channels: List[np.ndarray], every: int = 64, cap: int = 4096, seed: int = 1) -> dict:
    """Frames to re-lock over `channels` (PCM, encoded by the oracle), a start every `every` full frames, each from (0, 0)
    (the chain's guess) and from a random pair: median, p99, max and the trials that never re-locked within `cap`."""
    rng = np.random.default_rng(seed)
    res = []
    for pcm in channels:
        co = oracle.calculate_coefficients(pcm)
        ad = oracle.encode(pcm, co)
        truth = oracle.decode(ad, co, len(pcm))
        full = len(pcm) // 14
        starts = list(range(1, full, every))
        pairs = [(0, 0)] * len(starts) + [tuple(int(x) for x in rng.integers(-32768, 32768, 2)) for _ in starts]
        r = relock_frames(ad, co, truth, starts + starts, pairs, cap)
        # trials that ran off the end of the channel without a verdict are not counted
        ends = np.array(starts + starts) + cap > full
        res.append(r[~((r < 0) & ends)])
    allr = np.concatenate(res)
    ok = allr[allr > 0]
    if ok.size == 0:
        return dict(trials=int(allr.size), never=int((allr < 0).sum()), median=None, p99=None, max=None)
    return dict(trials=int(allr.size), never=int((allr < 0).sum()), median=float(np.median(ok)), p99=float(np.percentile(ok, 99)),
                max=int(ok.max()))


def silence_stimulus(adpcm: np.ndarray, coefs: np.ndarray, lo: int, hi: int) -> Tuple[np.ndarray, np.ndarray]:
    """Frames [lo, hi) of a channel made digital silence that HOLDS the history: header 0x00 (predictor 0, scale 0), zero
    nibbles, and coefficient pair 0 = (2048, 0), so every sample repeats hist1 ((2048 * h1 + 1024) >> 11 = h1).  A wrong
    pair entering the stretch stays wrong to its end."""
    ad = np.array(adpcm, np.uint8, copy=True)
    ad[lo * 8: hi * 8] = 0
    co = np.array(coefs, np.int16, copy=True)
    co[0], co[1] = 2048, 0
    return ad, co
