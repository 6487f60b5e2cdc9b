#!/usr/bin/env python
"""tools/hca_key_search_bench.py — the CRI HCA key search (vgb_hca_find_keys, HcaReader.FindKey over a key list).

  python tools/hca_key_search_bench.py [--files 2048] [--lists 256,4096] [--runs 5] [--warmup 1] [--out results.json]

The job: `files` type-56 .hca files of 1-10 s at 48 kHz, mono and stereo, encoded and keyed by the product
(WAVE -> .hca through vgb_convert_wave_batch), under 4 distinct keys.  Each list holds random codes with the 4 true keys
at its end, the worst case for the first-index search.  Per list, `warmup` + `runs` calls; reported:
  call_ms          the whole call under a host clock (it returns after the device is done): median, min, max;
  kernel_ms        the search kernel alone, CUDA events around its launch (vgb_hca_debug_key_search_stats slot 3),
                   of the median call;
  pairs, frames    (file, key) walks started and frames unpacked in that call;
  frames_per_s     frames over kernel_ms.
A file that comes back with another code (a random code TestKey accepts first) or a status is counted, and the first
eight such files are checked against the restatement.  In the same run the found indices are checked against the C
restatement (oracle/hcakeys.c, FindKey) on a 64-file sample, and that restatement's single-thread time on the sample is
reported as "cpu_c_restatement_ms" (a C restatement on one host thread, not .NET).  One JSON line per list, with the
GPU's name and power limit read in the same run, printed and, with --out, also written there as a list.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KEYS = [0x00D7E1B6C2A94F03, 0x0000000000001234, 0x0123456789ABCDEF, 0x00005EED0000C0DE]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [v.strip() for v in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_job(ct, O, synth, np, n_files, seed):
    rng = np.random.default_rng(seed)
    waves, owner = [], []
    for i in range(n_files):
        n = int(rng.integers(48000, 480001))
        ch = 1 + i % 2
        waves.append(O.wave_write16([synth.channel(seed * 1000 + 2 * i + c, n, 48000, degenerate=False) for c in range(ch)], 48000, None))
        owner.append(i % len(KEYS))
    files = [None] * n_files
    for k, code in enumerate(KEYS):
        idx = [i for i in range(n_files) if owner[i] == k]
        outs, st = ct.convert_wave_batch([waves[i] for i in idx], ct.convert_options(ct.CONTAINER_HCA, hca_key_type=56, hca_key_code=code))
        assert all(s == 0 for s in st)
        for i, o in zip(idx, outs):
            files[i] = o
    return files, owner


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--lists", default="256,4096")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the lines to this JSON file")
    args = ap.parse_args()

    import numpy as np

    import hca_key_oracle as K
    from oracle import pyoracle as O
    from vgaudio_b200 import containers as ct
    from vgaudio_b200 import synth

    O.build()
    info = gpu_info()
    files, owner = make_job(ct, O, synth, np, args.files, 17)
    lines = []
    for n_keys in [int(v) for v in args.lists.split(",")]:
        rng = np.random.default_rng(n_keys)
        keys = [int(v) for v in rng.integers(1, 1 << 63, size=n_keys - len(KEYS), dtype=np.int64)] + KEYS
        for _ in range(args.warmup):
            ct.hca_find_keys(files, keys)
        runs = []
        for _ in range(args.runs):
            t0 = time.perf_counter()
            idx, status = ct.hca_find_keys(files, keys)
            ms = (time.perf_counter() - t0) * 1e3
            runs.append((ms, ct.hca_key_search_stats()))
        # a random code that TestKey accepts before the true key is FindKey's answer too: checked against the oracle
        odd = [f for f in range(args.files) if status[f] != 0 or keys[idx[f]] != KEYS[owner[f]]]
        odd_check = [(f, idx[f], status[f], K.image_find_key(files[f], keys)) for f in odd[:8]]
        runs.sort(key=lambda r: r[0])
        med_ms, (pairs, frames, searched, kernel_us) = runs[len(runs) // 2]
        sample = list(range(0, args.files, max(1, args.files // 64)))[:64]
        t0 = time.perf_counter()
        ref = [K.image_find_key(files[i], keys) for i in sample]
        cpu_ms = (time.perf_counter() - t0) * 1e3
        parity = all(ref[j] == (idx[i], status[i]) for j, i in enumerate(sample))
        line = dict(info, files=args.files, keys=n_keys, true_keys_at="end",
                    call_ms={"median": round(med_ms, 3), "min": round(runs[0][0], 3), "max": round(runs[-1][0], 3)},
                    kernel_ms=round(kernel_us / 1e3, 3), pairs=pairs, frames=frames, files_searched=searched,
                    frames_per_s=round(frames / (kernel_us / 1e6), 1) if kernel_us else None,
                    parity_64_file_sample=parity, files_not_on_their_true_key=len(odd),
                    those_vs_oracle=[[int(v) for v in (f, i, st, *ref_)] for f, i, st, ref_ in odd_check], cpu_c_restatement_ms_64_files=round(cpu_ms, 1),
                    cpu_c_restatement_label="C restatement, not .NET, one host thread")
        print(json.dumps(line), flush=True)
        lines.append(line)
        assert parity and all((i, st) == tuple(ref_) for _, i, st, ref_ in odd_check)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
