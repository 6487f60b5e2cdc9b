"""Re-lock census of the CRI ADX encoder (CriAdxCodec.cs:56-147) on the CPU: a chain started at whole frame k from the
raw samples in front of it (what adx_encode_kernel's chain phase guesses for segment s > 0), after how many frames does
the pair it hands on equal the true one?  From there its bytes are the true bytes, which is what the run-on phase
relies on; a start that never re-locks leaves its boundary to the cascade.  The truth is the oracle's frame trace."""
from __future__ import annotations

from typing import Sequence

import numpy as np


def relock_frames(oracle, stim, starts: Sequence[int], cap: int) -> np.ndarray:
    """For each start k (1 <= k < stim.whole): frames encoded until (and including) the first whose end pair equals the
    truth's, or -1 when none does within `cap` frames or before the channel's whole frames end."""
    assert stim.std
    _, _, trace = oracle.adx_encode_trace(stim.pcm, *stim.args)
    truth = trace["hist_out"]
    co = np.array(stim.coefs(), np.int16)
    pcm = stim.pcm
    win = np.zeros(34, np.int16)
    out = np.full(len(starts), -1, np.int64)
    for i, k in enumerate(starts):
        h1, h2 = int(pcm[32 * k - 1]), int(pcm[32 * k - 2])
        for t in range(min(cap, stim.whole - k)):
            f = k + t
            win[0], win[1] = h2, h1
            win[2:] = pcm[32 * f: 32 * f + 32]
            oracle.adx_encode_frame(win, co, 32, stim.type, stim.version)
            h2, h1 = int(win[32]), int(win[33])
            if h1 == truth[f][0] and h2 == truth[f][1]:
                out[i] = t + 1
                break
    return out


def census(oracle, stim, n_starts: int = 7, cap: int = 400) -> np.ndarray:
    """relock_frames at n_starts starts spread over the channel."""
    starts = np.linspace(1, stim.whole - 1, n_starts + 2)[1:-1].astype(int)
    return relock_frames(oracle, stim, starts, cap)
