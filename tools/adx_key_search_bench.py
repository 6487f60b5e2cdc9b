#!/usr/bin/env python
"""tools/adx_key_search_bench.py — the CRI ADX key search (vgb_adx_find_keys) on keyed .adx files.

  python tools/adx_key_search_bench.py [--jobs 1,16,256] [--runs 2] [--warmup 1] [--out results.json]

Jobs of 1, 16 and 256 stereo files of 1-10 s at 48 kHz, encoded by the product (WAVE -> .adx through
vgb_convert_wave_batch: Linear, 18-byte frames, version 4) and keyed with a key string (revision 8) or a key code
(revision 9).  Per job and revision, `warmup` + `runs` calls; reported per call (median, min, max):
  call_ms     the whole call under a host clock: loading, the search, dedup and every key's confidence pass;
  kernel_ms   the search kernels alone, CUDA events around their launches (vgb_adx_debug_key_search_stats slot 3);
  cand_per_s  candidates tried over kernel_ms.
Every run must return the planted key (revision 9: its 13-bit equivalent).  The oracle's single-thread rate
(oracle/adxkeys.c on the first file over a sub-box of the search) is reported beside it, labelled as a CPU rate.  One
JSON line per job and revision, with the GPU's name and power limit, printed and, with --out, also written there as a
list.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KEY_STRING = "vgaudio-b200"
KEY_CODE = 0x0123456789ABCDEF


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [v.strip() for v in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_job(ct, O, synth, np, n_files, revision, seed):
    rng = np.random.default_rng(seed)
    waves = []
    for i in range(n_files):
        n = int(rng.integers(48000, 480001))
        waves.append(O.wave_write16([synth.channel(seed * 1000 + 2 * i + c, n, 48000, degenerate=False) for c in range(2)], 48000, None))
    k = ct.adx_key(key_string=KEY_STRING) if revision == 8 else ct.adx_key(key_code=KEY_CODE)
    opt = ct.convert_options(ct.CONTAINER_ADX, adx_encryption_type=revision, adx_has_key=1, adx_key_seed=k.seed,
                             adx_key_mult=k.mult, adx_key_inc=k.inc)
    outs, st = ct.convert_wave_batch(waves, opt)
    assert all(s == 0 for s in st)
    want = (k.seed, k.mult, k.inc) if revision == 8 else (k.seed & 0x1FFF, k.mult & 0x1FFF, k.inc & 0x1FFF)
    return outs, want


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", default="1,16,256")
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the lines to this JSON file")
    a = ap.parse_args()

    import numpy as np

    import vgaudio_b200 as vg
    import adx_key_oracle as K
    from oracle import pyoracle as O
    from vgaudio_b200 import containers as ct
    from vgaudio_b200 import synth

    vg._native.check(vg.lib.vgb_init(0, 0))
    info = gpu_info()
    lines = []
    for revision in (8, 9):
        for n_files in [int(x) for x in a.jobs.split(",")]:
            files, want = make_job(ct, O, synth, np, n_files, revision, seed=n_files * 10 + revision)
            calls, kernels, tried = [], [], 0
            keys = []
            for r in range(a.warmup + a.runs):
                t = time.perf_counter()
                res = ct.adx_find_keys(files)
                dt = (time.perf_counter() - t) * 1e3
                stats = ct.adx_key_search_stats(with_time=True)
                keys = [(k.key.seed, k.key.mult, k.key.inc) for k in res.keys]
                assert want in keys, (want, keys)
                if r >= a.warmup:
                    calls.append(dt)
                    kernels.append(stats[3] / 1e3)
                    tried = stats[0]
            # the oracle, one CPU thread, on the first file over a sub-box of the search
            st, _, scales, start = ct.adx_key_load(files[0])
            box = (0, 256, 0, 16, 0, 64)
            t = time.perf_counter()
            _, ostats = K.adx_guess_box(revision, [(scales, start)], box)
            ot = time.perf_counter() - t
            km = statistics.median(kernels)
            line = dict(info, job=f"rev{revision}_{n_files}_stereo_1to10s", revision=revision, files=n_files,
                        seconds_of_audio=round(sum(int(f[12:16].view(">i4")[0]) for f in files) / 48000, 1),
                        keys=len(keys), candidates=tried,
                        call_ms={"median": round(statistics.median(calls), 2), "min": round(min(calls), 2), "max": round(max(calls), 2)},
                        kernel_ms={"median": round(km, 3), "min": round(min(kernels), 3), "max": round(max(kernels), 3)},
                        cand_per_s=float(f"{tried / (km / 1e3):.4g}") if km > 0 else None,
                        cpu_oracle_single_thread_cand_per_s=float(f"{ostats[0] / ot:.4g}") if ot > 0 else None)
            print(json.dumps(line), flush=True)
            lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
