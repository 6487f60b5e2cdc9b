#!/usr/bin/env python
"""tools/loop_override_bench.py — what the converter's loop stages cost when every file loops.

  python tools/loop_override_bench.py [--files 2048] [--runs 3] [--warmup 1] [--check 8] [--formats dsp,adx,hca,brstm,hps]

The flagship batch job (bench_configs' 2048 synthetic WAVE files, mono / stereo, 1-6 s at 48 kHz, one in eight with a
smpl loop) goes into each target three ways:
  keep     the files' own loops (1/8 of them loop);
  set      -l 1001-47000 on every file: a loop start that no target's multiple divides, so every NintendoWare / HPS file
           is realigned and every .adx file takes the lead path;
  clear    --no-loop: no file loops.
Per target the three arms alternate within one call, `warmup` + `runs` fill passes each under a host clock (pinned
buffers; the sizing pass is outside the timed region); the median is reported.  One more pass per arm with one group in
flight (VGB_CONVERT_SERIAL) gives vgb_convert_debug_stage_ms.  `check` files per arm are compared byte for byte with the
oracle chain (tests/loop_override_oracle.py).  One JSON line per target and arm, with the GPU's name and power limit read
in the same process.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

LOOP = (1001, 47000)  # every file holds at least 48000 samples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=8)
    ap.add_argument("--formats", default="dsp,adx,hca,brstm,hps")
    a = ap.parse_args()

    import numpy as np
    import torch

    import bench
    import bench_configs
    import loop_override_oracle as L
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    O.build()
    N.check(N.lib.vgb_init(0, 0))
    ident = bench.gpu_identity(0, torch)
    device = torch.device("cuda", 0)
    files, meta = bench_configs._batch_files(torch, bench, a.files, device)
    n = len(files)
    ftab = (C.c_void_p * n)(*[f.data_ptr() for f in files])
    lens = (C.c_int64 * n)(*[int(f.numel()) for f in files])
    samples = sum(len(m[0]) * m[1] for m in meta)
    types = {"dsp": L.DSP_T, "adx": L.ADX_T, "hca": L.HCA_T, "brstm": L.BRSTM_T, "hps": L.HPS_T}
    arms = [("keep", L.KEEP), ("set", L.SET), ("clear", L.CLEAR)]
    for fmt in a.formats.split(","):
        out_type = types[fmt]
        plans = {}
        for name, mode in arms:
            opt = ct.convert_options(out_type, hca_quality=2)
            opt.loop_mode = mode
            opt.loop_start, opt.loop_end = LOOP if mode == L.SET else (0, 0)
            sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
            N.check(N.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(opt), sizes, None, status, None, None))
            outs = [torch.empty(max(int(sizes[i]), 1), dtype=torch.uint8, pin_memory=True) for i in range(n)]
            otab = (C.c_void_p * n)(*[o.data_ptr() if status[i] == 0 else None for i, o in enumerate(outs)])
            plans[name] = (opt, sizes, status, outs, otab, [])

        def fill(name):
            opt, sizes, status, outs, otab, _ = plans[name]
            N.check(N.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(opt), sizes, otab, status, None, None))

        for _ in range(a.warmup):
            for name, _m in arms:
                fill(name)
        torch.cuda.synchronize()
        for _ in range(a.runs):  # the arms alternate
            for name, _m in arms:
                t0 = time.perf_counter()
                fill(name)
                torch.cuda.synchronize()
                plans[name][5].append((time.perf_counter() - t0) * 1e3)
        for name, mode in arms:
            opt, sizes, status, outs, otab, times = plans[name]
            os.environ["VGB_CONVERT_SERIAL"] = "1"
            fill(name)
            del os.environ["VGB_CONVERT_SERIAL"]
            buf = (C.c_float * 4)()
            N.lib.vgb_convert_debug_stage_ms(buf, 4)
            checked = mismatched = 0
            for i in np.linspace(0, n - 1, a.check).astype(int):
                rows, ns, loop = meta[i]
                want = L.expected_from_wave(rows, bench_configs.SAMPLE_RATE, loop, out_type, mode, *(LOOP if mode == L.SET else (0, 0)))
                got = outs[i].numpy()[: int(sizes[i])].tobytes() if status[i] == 0 else None
                checked += 1
                mismatched += int((want[0].tobytes() if want[0] is not None else None) != got)
            looping = sum(1 for i in range(n) if status[i] == 0 and (mode == L.SET or (mode == L.KEEP and meta[i][2] is not None)))
            print(json.dumps({"target": fmt, "arm": name, "files": n, "looping_files": looping, "failed": sum(1 for i in range(n) if status[i]),
                              "fill_ms_median": round(statistics.median(times), 2), "fill_ms": [round(t, 2) for t in times],
                              "msamples_per_s": round(samples / (statistics.median(times) / 1e3) / 1e6, 1),
                              "stage_ms_serial": {"split": round(buf[0], 2), "encode": round(buf[1], 2), "loop_context": round(buf[2], 2),
                                                  "assembly": round(buf[3], 2)},
                              "oracle_checked": checked, "oracle_mismatched": mismatched, **ident}), flush=True)
    N.check(N.lib.vgb_shutdown())


if __name__ == "__main__":
    main()
