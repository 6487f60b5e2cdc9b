#!/usr/bin/env python
"""tools/convert_devices_bench.py — the fill pass of vgb_convert_wave_batch over one or more device lists.

  python tools/convert_devices_bench.py [--out-format dsp|adx|hca] [--files 2048] [--runs 5] [--warmup 1] 0 0,0 0,1,2,3

The job is bench.py --config batch's (bench_configs._batch_files: 2048 WAVE files in pinned host memory, 2/3 mono, 1/3
stereo, 1-6 s at 48 kHz, every eighth file looping).  For every device list the library is bound with vgb_init_devices
(vgb_init for a single device), the fill pass runs `warmup` times, then `runs` times under a host clock; the call
returns only after its last copy has landed, so each timing ends in the call's own synchronisation.  Every list must
produce byte-identical files.  One JSON line per list, with the GPU's name, its power limit and the visible GPU count.

Listing one card several times (0,0) measures the cost of the sharding path on a shared device, not scaling.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def parse_list(text):
    devs = [int(x) for x in text.split(",")]
    if not devs or any(d < 0 for d in devs):
        raise argparse.ArgumentTypeError(f"not a device list: {text!r}")
    return devs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lists", nargs="+", type=parse_list, help="comma-separated CUDA ordinals, one list per measurement")
    ap.add_argument("--out-format", default="dsp", choices=["dsp", "adx", "hca"])
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()

    import torch

    import bench
    import bench_configs
    import vgaudio_b200 as vg
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    visible = torch.cuda.device_count()
    for devs in a.lists:
        if max(devs) >= visible:
            raise SystemExit(f"device list {devs}: only {visible} GPU(s) visible")
    files, meta = bench_configs._batch_files(torch, bench, a.files, torch.device("cuda", 0))
    total_samples = sum(len(m[0]) * m[1] for m in meta)
    out_type = {"dsp": ct.CONTAINER_DSP, "adx": ct.CONTAINER_ADX, "hca": ct.CONTAINER_HCA}[a.out_format]
    opt = ct.convert_options(out_type, hca_quality=2)
    n = len(files)
    ftab = (C.c_void_p * n)(*[f.data_ptr() for f in files])
    lens = (C.c_int64 * n)(*[int(f.numel()) for f in files])
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    N.check(vg.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(opt), sizes, None, status, None, None))
    outs = [torch.empty(int(sizes[i]), dtype=torch.uint8, pin_memory=True) for i in range(n)]
    otab = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
    ident = bench.gpu_identity(0, torch)
    first_digest, same = None, True
    for devs in a.lists:
        N.check(vg.lib.vgb_shutdown())
        if len(devs) == 1:
            N.check(vg.lib.vgb_init(devs[0], 0))
        else:
            N.check(vg.lib.vgb_init_devices((C.c_int32 * len(devs))(*devs), len(devs), 0))
        for o in outs:
            o.zero_()

        def fill():
            N.check(vg.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(opt), sizes, otab, status, None, None))

        for _ in range(max(a.warmup, 1)):
            fill()
        ms = []
        for _ in range(a.runs):
            t0 = time.perf_counter()
            fill()
            ms.append((time.perf_counter() - t0) * 1e3)
        h = hashlib.sha256()
        for o in outs:
            h.update(o.numpy().tobytes())
        digest = h.hexdigest()
        first_digest = first_digest or digest
        print(json.dumps({"devices": devs, "out_format": a.out_format, "files": n, "total_samples": int(total_samples),
                          "runs": a.runs, "ms_median": round(statistics.median(ms), 3), "ms_min": round(min(ms), 3),
                          "ms_all": [round(x, 3) for x in ms], "msamples_per_s": round(total_samples / (statistics.median(ms) / 1e3) / 1e6, 1),
                          "bytes_equal_first_list": digest == first_digest, "all_status_ok": all(status[i] == 0 for i in range(n)),
                          "gpu": ident["name"], "power_limit_w": ident["power_limit_w"], "visible_gpus": visible}), flush=True)
        same = same and digest == first_digest
    N.check(vg.lib.vgb_shutdown())
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
