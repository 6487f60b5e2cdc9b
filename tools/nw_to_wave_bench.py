#!/usr/bin/env python
"""tools/nw_to_wave_bench.py — the fill pass of vgb_convert_nw_to_wave_batch, time-parallel GC-ADPCM decode against the
serial one.

  python tools/nw_to_wave_bench.py [--files 2048] [--tracks 32] [--runs 3] [--warmup 1] [--check 16]

Two jobs, GC-ADPCM encoded by the product itself (vgaudio_b200.gcadpcm.encode_batch) from synth PCM at 32 kHz and
wrapped into stream files by tests/nw_files.py:
  tracks  `tracks` stereo .brstm files of 3 minutes, looping - the BGM case one thread per channel serves worst;
  short   `files` files of 1-10 s, 2/3 mono and 1/3 stereo, cycling .brstm / .bcstm / .bfstm (big-endian every other
          .bfstm), every eighth looping and every eighth PCM16 instead of GC-ADPCM.
Each job's fill pass runs with the segmented decode and with VGB_GC_DEC_SEGMENTS=1 (the plain serial loop inside the
same kernels), alternating, `warmup` + `runs` times each under a host clock around the synchronous call; medians, minima
and maxima are reported.  The decode kernel time is the sum of the gc_decode_seg_kernel launches of one more fill pass
per arm under torch.profiler (CUDA activity), medians of `runs` such passes.  `check` files of each job are compared with
the oracle chain (tests/nw_reader_oracle.py) and the two arms with each other.  One JSON line per job with the GPU's name
and power limit.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _job(np, F, synth, gc, specs):
    """specs: (kind, channels, samples, loop or None, codec, big_endian) -> images."""
    base = [synth.channel(700 + c, 32000 * 12, 32000, degenerate=False) for c in range(8)]
    pcm, owner = [], []
    for i, (kind, ch, n, loop, codec, be) in enumerate(specs):
        for c in range(ch):
            src = base[(i + c) % len(base)]
            reps = -(-n // src.size)
            x = np.roll(np.tile(src, reps)[:n], 9973 * i + 31 * c)
            pcm.append(np.ascontiguousarray(x, np.int16))
            owner.append(i)
    want = [k for k, (_, _, _, _, codec, _) in enumerate(specs) if codec == F.GCADPCM]
    rows = [p for p, o in zip(pcm, owner) if o in set(want)]
    coefs, adpcm = gc.encode_batch(rows) if rows else (None, [])
    out, r, j = [], 0, 0
    for i, (kind, ch, n, loop, codec, be) in enumerate(specs):
        mine = pcm[j: j + ch]
        j += ch
        if codec == F.GCADPCM:
            chans = [F.Channel(adpcm[r + c].tobytes(), coefs[r + c], 0, (int(adpcm[r + c][0]), 0, 0)) for c in range(ch)]
            r += ch
        else:
            chans = F.pcm16_channels(mine, kind == F.BRSTM or bool(be))
        out.append(F.build(kind, codec, chans, n, rate=32000, loop=loop, big_endian=be))
    return out


def _decode_ms(torch, call):
    """Device time of the gc_decode_seg_kernel launches of one call, from torch.profiler's CUDA activity."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.events():
        if "gc_decode_seg_kernel" in e.name:
            us += getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0) or 0.0
    return us / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--tracks", type=int, default=32)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=16)
    a = ap.parse_args()

    import numpy as np
    import torch

    import bench
    import nw_files as F
    import nw_reader_oracle as R
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import gcadpcm, synth

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    O.build()
    N.check(N.lib.vgb_init(0, 0))
    rng = np.random.default_rng(2026)
    kinds = (F.BRSTM, F.BCSTM, F.BFSTM)
    short = []
    for i in range(a.files):
        n = int(rng.integers(32000, 320001))
        short.append((kinds[i % 3], 2 if i % 3 == 2 else 1, n, n // 5 if i % 8 == 0 else None,
                      F.PCM16 if i % 8 == 5 else F.GCADPCM, (i // 3) % 2 == 1))
    tracks = [(F.BRSTM, 2, 180 * 32000, 32000 * 7 + 11, F.GCADPCM, None) for _ in range(a.tracks)]
    ident = bench.gpu_identity(0, torch)
    ok_all = True
    for name, specs in (("tracks", tracks), ("short", short)):
        imgs = _job(np, F, synth, gcadpcm, specs)
        types = [s[0] for s in specs]
        n = len(imgs)
        ftab = (C.c_void_p * n)(*[h.ctypes.data for h in imgs])
        lens = (C.c_int64 * n)(*[h.size for h in imgs])
        ttab = (C.c_int32 * n)(*types)
        sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
        N.check(N.lib.vgb_convert_nw_to_wave_batch(ftab, lens, ttab, n, sizes, None, status))
        assert all(status[i] == 0 for i in range(n))
        outs = [torch.empty(sizes[i], dtype=torch.uint8).pin_memory() for i in range(n)]
        otab = (C.c_void_p * n)(*[o.data_ptr() for o in outs])

        def fill():
            N.check(N.lib.vgb_convert_nw_to_wave_batch(ftab, lens, ttab, n, sizes, otab, status))

        times = {"segmented": [], "serial": []}
        kern = {"segmented": [], "serial": []}
        stats = None
        for r in range(a.warmup + a.runs):
            for arm in ("segmented", "serial"):
                if arm == "serial":
                    os.environ["VGB_GC_DEC_SEGMENTS"] = "1"
                t0 = time.perf_counter()
                fill()
                dt = time.perf_counter() - t0
                assert all(status[i] == 0 for i in range(n))
                if r >= a.warmup:
                    times[arm].append(dt)
                    kern[arm].append(_decode_ms(torch, fill))
                if arm == "segmented" and stats is None:
                    st = (C.c_uint64 * 5)()
                    N.check(N.lib.vgb_gcadpcm_debug_decode_stats(st, 5))
                    stats = list(st)
                if arm == "serial" and r == a.warmup + a.runs - 1:
                    serial_bytes = [outs[i].numpy().tobytes() for i in range(n)]
                os.environ.pop("VGB_GC_DEC_SEGMENTS", None)
        fill()
        same_arms = all(outs[i].numpy().tobytes() == serial_bytes[i] for i in range(n))
        checked = sorted(set(np.linspace(0, n - 1, min(a.check, n)).astype(int).tolist()))
        identical = all(outs[i].numpy().tobytes() == R.expected_wave(imgs[i], types[i]).tobytes() for i in checked)
        ok_all &= identical and same_arms
        row = {"tool": "nw_to_wave_bench", "job": name, "files": n, "stream_bytes": int(sum(h.size for h in imgs)),
               "wave_bytes": int(sum(int(sizes[i]) for i in range(n))), "runs": a.runs, "gpu": ident["name"],
               "power_limit_w": ident["power_limit_w"],
               "decode_kernel_ms": {arm: round(statistics.median(v), 3) for arm, v in kern.items()},
               "segments_last_group": stats[0], "runon_frames": stats[1], "cascade_frames": stats[2], "boundaries_repaired": stats[3],
               "longest_runon": stats[4], "oracle_checked": len(checked), "oracle_identical": identical, "arms_identical": same_arms}
        for arm, ts in times.items():
            row[f"{arm}_fill_ms"] = {"median": round(statistics.median(ts) * 1e3, 2), "min": round(min(ts) * 1e3, 2), "max": round(max(ts) * 1e3, 2)}
        print(json.dumps(row), flush=True)
    N.check(N.lib.vgb_shutdown())
    if not ok_all:
        raise SystemExit("converted files differ from the oracle chain or between the arms")


if __name__ == "__main__":
    main()
