"""The GC-ADPCM encoder's squared error (gc_encode.cu: a 32-bit sum modulo 2^32 plus a float32 sum that gives the
multiple of 2^32) on frames whose errors are set exactly: winning errors in every range k * 2^32 the encoder's fast
path can produce (k = 0..13), exactly on 2^27 - 1, 2^31 and 2^32 * k, and pairs that straddle a multiple of 2^32 so
that comparing the low 32 bits alone would pick the loser.

Construction (every frame starts from history -32768): a predictor (8192, 0) predicts -131072, beyond what a nibble
can reach, so it reconstructs -32768 for every sample and its error is sum (x + 32768)^2; a predictor (-8192, 0)
reconstructs 32767, -32768, 32767, ... and its error differs in the even samples.  Both chains end on their pass at
scalePower 12 and every difference stays below 2^29, so these frames run the fast path.  The CPU test proves with the
oracle's frame trace that each frame has the designed errors and winner; the GPU test compares the encoder's bytes."""
import math

import numpy as np
import pytest

A, B = (8192, 0), (-8192, 0)   # coefficients (c0, c1) of the two predictor kinds
FULL = 65535 ** 2
SAT = (1 << 27) - 1


def _odd_even(x):
    return x[1::2], x[0::2]


def _usable(v: int) -> bool:
    # off the quantiser's rounding thresholds at scalePower 11 and 12 (no exactness fallback)
    return 0 <= v <= 65535 and v % 2048 not in (1024, 1028) and v % 4096 not in (2048, 2052)


def _squares(target: int, n: int):
    """n usable values whose squares sum to target (greedy, the last four searched), or None."""
    if n == 1:
        v = math.isqrt(max(target, 0))
        return [v] if target >= 0 and v * v == target and _usable(v) else None
    if target < 0 or target > n * FULL:
        return None
    top = min(65535, math.isqrt(target))
    tries = {4: 16, 3: 64, 2: 4096}.get(n, 1)  # four squares make every number; three do not (4^a (8b + 7))
    for v in range(top, max(-1, top - tries), -1):
        if _usable(v):
            rest = _squares(target - v * v, n - 1)
            if rest is not None:
                return [v] + rest
    return None


def _frame(err_a: int, even_a):
    """14 biased samples a = x + 32768 with the given even samples and sum a^2 == err_a."""
    odd = _squares(err_a - sum(v * v for v in even_a), 7)
    assert odd is not None, f"no frame with error {err_a}"
    a = np.zeros(14, np.int64)
    a[0::2] = even_a
    a[1::2] = odd
    return a


def _err_b(a):
    odd, even = _odd_even(a)
    return int((odd ** 2).sum() + ((65535 - even) ** 2).sum())


def _frames():
    """(biased samples, predictor kinds, expected winner, expected winning error) per frame."""
    out = []
    balanced = [32767] * 7                 # A - B = -65535
    for k in range(2, 9):
        for base in ((k << 32) - 1, k << 32, (k << 32) + 1, (k << 32) + (1 << 31)):
            # A wins by 65535, and the pair straddles k * 2^32 for the first two bases
            a = _frame(base, balanced)
            out.append((a, "AB", 0, base))
            # B wins: even samples four higher make A - B = +65535
            even = balanced[:6] + [32771]
            a = _frame(base + 65535, even)
            out.append((a, "AB", 1, base))
    # low ranges and the key's saturation: the winner far below the other kind (no even sample is balanced)
    for err in (SAT - 1, SAT, SAT + 1, 1 << 30, (1 << 31) - 1, 1 << 31, (1 << 31) + 1, (1 << 32) - 1, 1 << 32,
                (1 << 32) + 1, 3 << 31):
        a = _frame(err, [1] * 7)
        out.append((a, "AB", 0, err))
        out.append((a, "BA", 1, err))
    # the top ranges: every predictor the same kind, the first of eight equal errors wins
    for k in range(9, 14):
        for err in (k << 32, (k << 32) + (1 << 31)):
            if err <= 14 * FULL:
                out.append((_frame(err, [65535 - 1] * 6 + [65535 - 3]), "AA", 0, err))
    return out


def _channel(frames, kinds):
    pcm = np.concatenate([a - 32768 for a, _, _, _ in frames]).astype(np.int16)
    co = np.array([v for i in range(8) for v in (A if kinds[i % 2] == "A" else B)], np.int16)
    return pcm, co


@pytest.fixture(scope="module")
def channels():
    fr = _frames()
    by_kinds = {}
    for f in fr:
        by_kinds.setdefault(f[1], []).append(f)
    return [(kinds, fs) + _channel(fs, kinds) for kinds, fs in sorted(by_kinds.items())]


def test_frames_have_the_designed_errors(oracle, channels):
    ranges = set()
    for kinds, fs, pcm, co in channels:
        _, trace = oracle.gc_encode_trace(pcm, co, -1, -32768, -32768)
        assert len(trace) == len(fs)
        for f, (a, _, winner, err) in enumerate(fs):
            t = trace[f]
            assert int(t["winner"]) == winner, (kinds, f)
            assert int(t["pred"][winner]["error"]) == err, (kinds, f)
            assert all(int(p["final_sp"]) == 12 and not p["bumped"] and int(p["max_abs_diff"]) < (1 << 29) for p in t["pred"])
            errs = [int(p["error"]) for p in t["pred"]]
            if kinds != "AA":
                loser = errs[1 - winner]
                assert loser > err
                if (loser >> 32) != (err >> 32) and (loser & 0xFFFFFFFF) < (err & 0xFFFFFFFF):
                    ranges.add("straddle")
            ranges.add(err >> 32)
    assert ranges >= set(range(14)) | {"straddle"}, ranges


@pytest.mark.gpu
def test_encoder_matches_oracle(vg, oracle, channels):
    P = vg.gcadpcm.GcAdpcmParameters
    for rot in range(4):  # every channel in every quarter slot of a warp
        chans = [c[2] for c in channels]
        order = [(i + rot) % len(chans) for i in range(len(chans))]
        pcm = [chans[i] for i in order]
        co = np.stack([channels[i][3] for i in order])
        _, adpcm = vg.gcadpcm.encode_batch(pcm, co, [P(len(p), -32768, -32768) for p in pcm])
        for pos, i in enumerate(order):
            want = oracle.encode(chans[i], channels[i][3], -1, -32768, -32768)
            assert np.asarray(adpcm[pos], np.uint8).tobytes() == want.tobytes(), (channels[i][0], rot)
