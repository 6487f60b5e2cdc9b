#!/usr/bin/env python
"""tools/gc_rewrite_bench.py — the fill pass of vgb_rewrite_gc_batch against the two-call composition through WAVE.

  python tools/gc_rewrite_bench.py [--files 2048] [--tracks 32] [--runs 3] [--warmup 1] [--check 3] [--check-tracks 1]

Two jobs of WAVE images: `short`, the 2048-file job of `bench.py --config batch` (mono / stereo, 1-6 s at 48 kHz, every
eighth file looping), and `tracks`, `tracks` stereo files of 3 minutes at 48 kHz, looping from 7 s + 11 samples, a loop
start no target's alignment divides, so every target moves it and re-encodes the tail.  As set-up each job is encoded
once to .dsp by vgb_convert_wave_batch.  Then for each direction .dsp -> .brstm / .bcstm / .bfstm / .idsp / .hps,
alternating, `warmup` + `runs` times each under a host clock (both calls return after their last copy has landed; every
buffer is pinned, and the sizing passes, host-only, are outside the timed region):
  direct       one vgb_rewrite_gc_batch fill pass, .dsp images in, target images out (the source's ADPCM is kept);
  composition  vgb_convert_to_wave_batch's fill pass, then vgb_convert_wave_batch's fill pass on those WAVE images (the
               coefficient search and the full encode run again).
The arms' bytes differ by design (the composition re-encodes).  `check` files of each direction (`check-tracks` of the
tracks) are compared with the oracle chain (tests/gc_rewrite_oracle.py), statuses and bytes.  One JSON line per job and
direction, with the GPU's name and power limit.
"""
import argparse
import ctypes as C
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

NAMES = {4: "brstm", 5: "bcstm", 6: "bfstm", 7: "idsp", 8: "hps"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--tracks", type=int, default=32)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=3, help="files per direction of the short job compared with the oracle chain")
    ap.add_argument("--check-tracks", type=int, default=1, help="the same for the tracks job")
    a = ap.parse_args()

    import numpy as np
    import torch

    import bench
    import bench_configs
    import gc_rewrite_oracle as R
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct
    from vgaudio_b200 import synth

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    O.build()
    N.check(N.lib.vgb_init(0, 0))
    ident = bench.gpu_identity(0, torch)

    def pinned(arr):
        t = torch.empty(int(arr.size), dtype=torch.uint8, pin_memory=True)
        t.numpy()[:] = arr
        return t

    def tab(ts):
        return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts]), (C.c_int64 * len(ts))(*[int(t.numel()) for t in ts])

    def sized(call, n, all_ok=True):
        """The sizing pass of `call`, then pinned buffers of those sizes: (buffers, their table, sizes, status array)."""
        sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
        N.check(call(sizes, None, status))
        if all_ok:
            assert all(status[i] == 0 for i in range(n)), [status[i] for i in range(n) if status[i]][:4]
        outs = [torch.empty(max(int(sizes[i]), 1), dtype=torch.uint8, pin_memory=True) for i in range(n)]
        return outs, (C.c_void_p * n)(*[o.data_ptr() for o in outs]), sizes, status

    jobs = []
    waves, _ = bench_configs._batch_files(torch, bench, a.files, torch.device("cuda", 0))
    jobs.append(("short", waves, a.check))
    tracks = []
    for i in range(a.tracks):
        n = 180 * 48000
        pcm = [synth.channel(900 + 2 * i + c, n, 48000, degenerate=False) for c in range(2)]
        tracks.append(pinned(O.wave_write16(pcm, 48000, (48000 * 7 + 11, n - 5))))
    jobs.append(("tracks", tracks, a.check_tracks))

    ok_all = True
    for job, waves, n_check in jobs:
        n = len(waves)
        wtab, wlens = tab(waves)
        opt_dsp = ct.convert_options(R.DSP)
        outs, otab, sizes, status = sized(lambda s, o, st: N.lib.vgb_convert_wave_batch(wtab, wlens, n, C.byref(opt_dsp), s, o, st, None, None), n)
        N.check(N.lib.vgb_convert_wave_batch(wtab, wlens, n, C.byref(opt_dsp), sizes, otab, status, None, None))
        dsps = [o[: int(sizes[i])].clone().pin_memory() for i, o in enumerate(outs)]
        del outs
        ftab, lens = tab(dsps)
        types = (C.c_int32 * n)(*([R.DSP] * n))
        for dst in R.TARGETS:
            opt = ct.convert_options(dst)
            direct = lambda s, o, st: N.lib.vgb_rewrite_gc_batch(ftab, lens, types, n, C.byref(opt), s, o, st)
            to_wave = lambda s, o, st: N.lib.vgb_convert_to_wave_batch(ftab, lens, types, n, None, None, None, s, o, st)
            d_outs, d_tab, d_sizes, d_status = sized(direct, n, all_ok=False)  # HPS refuses some moved loops
            w_outs, w_tab, w_sizes, w_status = sized(to_wave, n)
            N.check(to_wave(w_sizes, w_tab, w_status))  # the WAVE images, so the second call can be sized
            wt2 = [w[: int(w_sizes[i])] for i, w in enumerate(w_outs)]
            wtab2, wlens2 = tab(wt2)
            c_outs, c_tab, c_sizes, c_status = sized(
                lambda s, o, st: N.lib.vgb_convert_wave_batch(wtab2, wlens2, n, C.byref(opt), s, o, st, None, None), n, all_ok=False)
            times = {"direct": [], "composition": []}
            for r in range(a.warmup + a.runs):
                for arm in ("direct", "composition"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if arm == "direct":
                        N.check(direct(d_sizes, d_tab, d_status))
                    else:
                        N.check(to_wave(w_sizes, w_tab, w_status))
                        N.check(N.lib.vgb_convert_wave_batch(wtab2, wlens2, n, C.byref(opt), c_sizes, c_tab, c_status, None, None))
                    dt = time.perf_counter() - t0
                    if r >= a.warmup:
                        times[arm].append(dt)
            good = [i for i in range(n) if d_status[i] == 0]
            picks = sorted(set(np.linspace(0, n - 1, min(n_check, n)).astype(int).tolist())) if n_check > 0 else []
            oracle_ok = True
            for i in picks:
                want, _ = R.expected(dsps[i].numpy(), dst)
                if want is None:
                    oracle_ok &= d_status[i] != 0
                else:
                    oracle_ok &= d_status[i] == 0 and d_outs[i][: int(d_sizes[i])].numpy().tobytes() == want.tobytes()
            ok_all &= oracle_ok
            row = {"tool": "gc_rewrite_bench", "job": job, "direction": f"dsp->{NAMES[dst]}", "files": n, "refused": n - len(good),
                   "composition_refused": sum(1 for i in range(n) if c_status[i] != 0),
                   "in_bytes": int(sum(int(t.numel()) for t in dsps)), "out_bytes": int(sum(int(d_sizes[i]) for i in range(n))),
                   "runs": a.runs, "gpu": ident["name"], "power_limit_w": ident["power_limit_w"],
                   "oracle_checked": len(picks), "oracle_identical": oracle_ok}
            for arm, ts in times.items():
                row[f"{arm}_ms"] = {"median": round(statistics.median(ts) * 1e3, 2), "min": round(min(ts) * 1e3, 2), "max": round(max(ts) * 1e3, 2)}
            row["speedup_median"] = round(statistics.median(times["composition"]) / statistics.median(times["direct"]), 3)
            print(json.dumps(row), flush=True)
            del d_outs, w_outs, c_outs
    N.check(N.lib.vgb_shutdown())
    if not ok_all:
        raise SystemExit("rewritten files differ from the oracle chain")


if __name__ == "__main__":
    main()
