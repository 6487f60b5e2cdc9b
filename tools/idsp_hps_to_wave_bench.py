#!/usr/bin/env python
"""tools/idsp_hps_to_wave_bench.py — the fill pass of vgb_convert_idsp_hps_to_wave_batch, time-parallel GC-ADPCM decode
against the serial one, and the device time of the HPS block gather.

  python tools/idsp_hps_to_wave_bench.py [--files 2048] [--tracks 32] [--runs 3] [--warmup 1] [--check 16]

Two jobs, written by the product itself (vgb_convert_wave_batch with the IDSP and HPS targets) from synth PCM at 32 kHz:
  tracks  `tracks` stereo .hps files of 3 minutes, looping - the BGM case one thread per channel serves worst;
  short   `files` files of 1-10 s, alternating .idsp / .hps, mono and stereo, every eighth looping (.hps from the start:
          HpsWriter moves other loop starts to a block boundary).
Each job's fill pass runs with the segmented decode and with VGB_GC_DEC_SEGMENTS=1 (the plain serial loop inside the
same kernels), alternating, `warmup` + `runs` times each under a host clock around the synchronous call; medians, minima
and maxima are reported.  The hps_gather_kernel and gc_decode_seg_kernel device times are sums over one more fill pass
per arm under torch.profiler (CUDA activity), medians of `runs` such passes; the bytes the gather reads and writes over
its kernel time are set against the H100's 3.35 TB/s.  `check` files of each job are compared with the oracle chain
(tests/idsp_hps_reader_oracle.py) and the two arms with each other.  One JSON line per job with the GPU's name and
power limit.
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

HBM_TBPS = 3.35  # H100 SXM5 80 GB HBM3 peak


def _job(np, O, ct, synth, specs):
    """specs: (kind, channels, samples, loop or None) -> file images written by the product's IDSP / HPS writers."""
    base = [synth.channel(700 + c, 32000 * 12, 32000, degenerate=False) for c in range(8)]
    out = [None] * len(specs)
    for kind in (7, 8):
        mine = [i for i, s in enumerate(specs) if s[0] == kind]
        waves = []
        for i in mine:
            _, ch, n, loop = specs[i]
            pcm = []
            for c in range(ch):
                src = base[(i + c) % len(base)]
                pcm.append(np.ascontiguousarray(np.roll(np.tile(src, -(-n // src.size))[:n], 9973 * i + 31 * c), np.int16))
            waves.append(O.wave_write16(pcm, 32000, loop))
        files, status = ct.convert_wave_batch(waves, ct.convert_options(kind))
        assert status == [0] * len(mine), status
        for i, f in zip(mine, files):
            out[i] = f
    return out


def _kernel_ms(torch, call, names):
    """Device time per kernel name of one call, from torch.profiler's CUDA activity."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    us = {k: 0.0 for k in names}
    for e in prof.events():
        for k in names:
            if k in e.name:
                us[k] += getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0) or 0.0
    return {k: v / 1e3 for k, v in us.items()}


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
    import idsp_hps_reader_oracle as R
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct
    from vgaudio_b200 import synth

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    O.build()
    N.check(N.lib.vgb_init(0, 0))
    rng = np.random.default_rng(2026)
    short = []
    for i in range(a.files):
        n = int(rng.integers(32000, 320001))
        short.append((R.IDSP if i % 2 == 0 else R.HPS, 1 + (i // 2) % 2, n, ((n // 5 if i % 2 == 0 else 0), n) if i % 8 == 0 else None))
    tracks = [(R.HPS, 2, 180 * 32000, (0, 180 * 32000)) for _ in range(a.tracks)]
    ident = bench.gpu_identity(0, torch)
    names = ("hps_gather_kernel", "gc_decode_seg_kernel")
    ok_all = True
    for name, specs in (("tracks", tracks), ("short", short)):
        imgs = _job(np, O, ct, synth, specs)
        types = [s[0] for s in specs]
        n = len(imgs)
        ftab = (C.c_void_p * n)(*[h.ctypes.data for h in imgs])
        lens = (C.c_int64 * n)(*[h.size for h in imgs])
        ttab = (C.c_int32 * n)(*types)
        sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
        N.check(N.lib.vgb_convert_idsp_hps_to_wave_batch(ftab, lens, ttab, n, sizes, None, status))
        assert all(status[i] == 0 for i in range(n))
        outs = [torch.empty(sizes[i], dtype=torch.uint8).pin_memory() for i in range(n)]
        otab = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
        # the bytes the gather moves: every HPS channel row, SampleCountToByteCount(sample_count)
        gather_bytes = 0
        for i in range(n):
            if types[i] == R.HPS:
                _, h = R.parse_hps(imgs[i])
                gather_bytes += R.gc_bytes(h.sample_count) * h.channel_count

        def fill():
            N.check(N.lib.vgb_convert_idsp_hps_to_wave_batch(ftab, lens, ttab, n, sizes, otab, status))

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
                    kern[arm].append(_kernel_ms(torch, fill, names))
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
        gather_ms = statistics.median([k["hps_gather_kernel"] for k in kern["segmented"] + kern["serial"]])
        row = {"tool": "idsp_hps_to_wave_bench", "job": name, "files": n, "hps_files": types.count(R.HPS),
               "stream_bytes": int(sum(h.size for h in imgs)), "wave_bytes": int(sum(int(sizes[i]) for i in range(n))),
               "runs": a.runs, "gpu": ident["name"], "power_limit_w": ident["power_limit_w"],
               "decode_kernel_ms": {arm: round(statistics.median([k["gc_decode_seg_kernel"] for k in v]), 3) for arm, v in kern.items()},
               "gather_kernel_ms": round(gather_ms, 4), "gather_bytes": gather_bytes,
               "gather_tb_per_s": round(2 * gather_bytes / (gather_ms * 1e-3) / 1e12, 3) if gather_ms > 0 else None,
               "gather_fraction_of_hbm": round(2 * gather_bytes / (gather_ms * 1e-3) / 1e12 / HBM_TBPS, 3) if gather_ms > 0 else None,
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
