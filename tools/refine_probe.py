#!/usr/bin/env python
"""How the GC-ADPCM coefficient refinement's time grows with the number of CTAs that share an SM.

gc_coef_refine_kernel runs one CTA per channel, up to eight per SM.  This probe times it alone (vgb_gcadpcm_coefs_dev
with the kernel timers on, index 1 of vgb_last_kernel_ms) on the first C first channels of bench.py's C2 signal, at
channel counts that are whole multiples of the SM count, so every run is one wave with the same number of resident CTAs
on every SM.  If a CTA's time barely grows from one to eight CTAs per SM, the SMs are not what limits the kernel; if it
grows in proportion, CTAs on one SM compete for its pipes.  Tuning tool, not a bench value.

  python tools/refine_probe.py [--seconds S] [--per-sm 1,2,4,6,8] [--reps R]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import vgaudio_b200 as vg  # noqa: E402
from vgaudio_b200 import _native as N  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=30.0, help="audio seconds per channel")
    ap.add_argument("--per-sm", default="1,2,4,6,8", help="resident CTAs per SM to sweep")
    ap.add_argument("--reps", type=int, default=5, help="timed calls per point (the median is reported)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("refine_probe.py needs a CUDA device")

    dev = torch.device("cuda", 0)
    N.check(vg.lib.vgb_init(0, 0))
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    per_sm = [int(v) for v in args.per_sm.split(",")]
    n = int(round(args.seconds * bench.SAMPLE_RATE))
    frames = (n + 13) // 14
    records = (frames + 31) // 32 * 32  # per channel, as the kernel walks them (whole blocks of 32)
    max_ch = n_sm * max(per_sm)
    # the C2 generator with the same seed: the first 1024 channels are bench.py's C2 batch
    pcm = bench.make_batch_gpu(torch, max_ch, n, 0, dev)
    stride = (n + 7) // 8 * 8
    if stride != n:
        padded = torch.zeros((max_ch, stride), dtype=torch.int16, device=dev)
        padded[:, :n] = pcm
        pcm = padded
    stream = torch.cuda.current_stream()
    N.check(vg.lib.vgb_set_kernel_timing(1))

    sampler = bench.ClockSampler(0)
    sampler.start()
    rows = []
    for k in per_sm:
        n_ch = n_sm * k
        ws_bytes = int(vg.lib.vgb_gcadpcm_workspace_bytes(frames * n_ch, n_ch))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        coefs = torch.zeros((n_ch, 16), dtype=torch.int16, device=dev)
        off = np.arange(n_ch, dtype=np.int64) * stride
        lens = np.full(n_ch, n, dtype=np.int32)

        def call():
            N.check(vg.lib.vgb_gcadpcm_coefs_dev(pcm.data_ptr(), off.ctypes.data, lens.ctypes.data, n_ch, coefs.data_ptr(),
                                                 ws.data_ptr(), ws_bytes, stream.cuda_stream))
            buf = (C.c_float * 2)()
            N.check(vg.lib.vgb_last_kernel_ms(buf, 2))  # synchronises on the kernel events
            return float(buf[1])

        call()
        call()
        ms = statistics.median(call() for _ in range(args.reps))
        rows.append({"ctas_per_sm": k, "channels": n_ch, "refine_ms": round(ms, 3),
                     "ns_per_record_per_channel": round(ms * 1e6 / records, 2)})
        del ws, coefs
    clocks = sampler.stop()
    base = rows[0]["refine_ms"]
    for r in rows:
        r["vs_first"] = round(r["refine_ms"] / base, 2)
    print(json.dumps({"probe": "gc_coef_refine CTAs-per-SM sweep", "gpu": bench.gpu_identity(0, torch), "sms": n_sm,
                      "clocks": clocks, "seconds": args.seconds, "records_per_channel": records, "reps": args.reps,
                      "sweep": rows}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
