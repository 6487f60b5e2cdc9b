#!/usr/bin/env python
"""What the GC-ADPCM coefficient refinement's CTAs wait for when eight of them share an SM.

Builds diagnostic copies of libvgaudio_b200.so in a temporary directory, each with gc_coefs.cu compiled under one
VGB_REFINE_DIAG value (gc_coefs.cu), and times gc_coef_refine_kernel<4> in each at 1, 2, 4, 6 and 8 CTAs per SM on
bench.py's C2 signal, the way tools/refine_probe.py does:

  a  the kernel as it ships (VGB_REFINE_DIAG=0)
  b  the producers only: the consumer warp keeps the chunk barriers but adds nothing (=1)
  c  the consumer only: the producers queue record i of every block in bucket i % NB without the nearest-centroid
     search, so every chunk's chain is known from the sizes alone (=2)
  d  the producers with the fp64 distances and compares replaced by integer stand-ins (=3)

Beside (c) it prints that variant's chain: the consumer's DADD steps per pass and their floor at the dependent-DADD
latency given by --dadd-cycles (`tools/microbench d` measures it).  The CPU-side parts (arguments, sizes, the chain
census of (c)) run without a GPU with --dry-run.  Tuning tool, not a bench value; the shipped kernels do not depend on
the flag (VGB_REFINE_DIAG defaults to 0).

  python tools/refine_contention.py [--variants a,b,c,d] [--per-sm 1,2,4,6,8] [--seconds S] [--reps R] [--dry-run]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = {"a": 0, "b": 1, "c": 2, "d": 3}
SAMPLE_RATE = 48000  # bench.SAMPLE_RATE, checked in main() when bench can be imported
PRODUCERS = 3        # producer warps of gc_coef_refine_kernel<4>: one chunk = 3 blocks of 32 records
PASS_BUCKETS = (1, 2, 2, 4, 4, 8, 8)


def refine_step(nb: int) -> int:
    return 4 if nb >= 4 else (8 if nb == 2 else 16)


def sizes(seconds: float) -> dict:
    n = int(round(seconds * SAMPLE_RATE))
    frames = (n + 13) // 14
    blocks = (frames + 31) // 32
    chunks = (blocks + PRODUCERS - 1) // PRODUCERS
    return {"samples": n, "frames": frames, "records": blocks * 32, "blocks": blocks, "chunks": chunks}


def fixed_pattern_chain(seconds: float, dadd_cycles: float, sm_mhz: float) -> dict:
    """Chain of variant (c) with every record accepted: a full chunk queues 96 / NB records per bucket, padded to the
    consumer's step; the lanes walk in lockstep, so a chunk costs its longest queue.  The tail chunk is ignored."""
    s = sizes(seconds)
    per_pass = []
    for nb in PASS_BUCKETS:
        per_bucket = 32 * PRODUCERS // nb
        step = refine_step(nb)
        per_pass.append((per_bucket + step - 1) // step * step * s["chunks"])
    total = sum(per_pass)
    return {"dadd_steps_per_pass": per_pass, "dadd_steps": total, "dadd_cycles": dadd_cycles,
            "floor_ms": round(total * dadd_cycles / (sm_mhz * 1e3), 3)}


def build_variant(tmp: str, diag: int) -> str:
    """A copy of vgaudio_b200/ with gc_coefs.cu rebuilt under -DVGB_REFINE_DIAG=diag; the other objects are reused
    from the tree's build when present."""
    dst = os.path.join(tmp, f"diag{diag}")
    shutil.copytree(os.path.join(ROOT, "vgaudio_b200"), os.path.join(dst, "vgaudio_b200"),
                    ignore=shutil.ignore_patterns("__pycache__", "gc_coefs.o", "*.so", "vgaudio_batch"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(dst, "include"))
    csrc = os.path.join(dst, "vgaudio_b200", "csrc")
    subprocess.run(["make", "-C", csrc, "-j8", "../libvgaudio_b200.so", f"EXTRA=-DVGB_REFINE_DIAG={diag}"], check=True,
                   stdout=subprocess.DEVNULL)
    return os.path.join(dst, "vgaudio_b200", "libvgaudio_b200.so")


def load(path: str):
    from vgaudio_b200 import _native as N

    lib = C.CDLL(path)
    for name in ("vgb_init", "vgb_set_kernel_timing", "vgb_gcadpcm_workspace_bytes", "vgb_gcadpcm_coefs_dev",
                 "vgb_last_kernel_ms"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = N.SIGNATURES[name]
    return lib


def sweep(lib, torch, bench, per_sm, seconds, reps):
    import numpy as np
    from vgaudio_b200 import _native as N

    dev = torch.device("cuda", 0)
    N.check(lib.vgb_init(0, 0))
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    n = int(round(seconds * bench.SAMPLE_RATE))
    frames = (n + 13) // 14
    max_ch = n_sm * max(per_sm)
    pcm = bench.make_batch_gpu(torch, max_ch, n, 0, dev)
    stride = (n + 7) // 8 * 8
    if stride != n:
        padded = torch.zeros((max_ch, stride), dtype=torch.int16, device=dev)
        padded[:, :n] = pcm
        pcm = padded
    stream = torch.cuda.current_stream()
    N.check(lib.vgb_set_kernel_timing(1))
    rows = []
    for k in per_sm:
        n_ch = n_sm * k
        ws_bytes = int(lib.vgb_gcadpcm_workspace_bytes(frames * n_ch, n_ch))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        coefs = torch.zeros((n_ch, 16), dtype=torch.int16, device=dev)
        off = np.arange(n_ch, dtype=np.int64) * stride
        lens = np.full(n_ch, n, dtype=np.int32)

        def call():
            N.check(lib.vgb_gcadpcm_coefs_dev(pcm.data_ptr(), off.ctypes.data, lens.ctypes.data, n_ch, coefs.data_ptr(),
                                              ws.data_ptr(), ws_bytes, stream.cuda_stream))
            buf = (C.c_float * 2)()
            N.check(lib.vgb_last_kernel_ms(buf, 2))  # synchronises on the kernel events
            return float(buf[1])

        call()
        call()
        rows.append({"ctas_per_sm": k, "refine_ms": round(statistics.median(call() for _ in range(reps)), 3)})
        del ws, coefs
    for r in rows:
        r["vs_first"] = round(r["refine_ms"] / rows[0]["refine_ms"], 2)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", default="a,b,c,d", help="diagnostic builds to time (a b c d, see the module doc)")
    ap.add_argument("--per-sm", default="1,2,4,6,8", help="resident CTAs per SM to sweep")
    ap.add_argument("--seconds", type=float, default=30.0, help="audio seconds per channel")
    ap.add_argument("--reps", type=int, default=5, help="timed calls per point (the median is reported)")
    ap.add_argument("--dadd-cycles", type=float, default=8.0, help="dependent DADD latency for the chain floor")
    ap.add_argument("--sm-mhz", type=float, default=1980.0, help="SM clock for the chain floor when not measured")
    ap.add_argument("--dry-run", action="store_true", help="sizes and the chain census only (no GPU, no build)")
    args = ap.parse_args()
    variants = [v.strip() for v in args.variants.split(",") if v.strip()]
    bad = [v for v in variants if v not in VARIANTS]
    if bad:
        ap.error(f"unknown variants {bad}; choose from {sorted(VARIANTS)}")
    per_sm = [int(v) for v in args.per_sm.split(",")]
    out = {"probe": "gc_coef_refine diagnostic variants, CTAs-per-SM sweep", "sizes": sizes(args.seconds),
           "chain_c": fixed_pattern_chain(args.seconds, args.dadd_cycles, args.sm_mhz)}
    if args.dry_run:
        print(json.dumps(out))
        return 0

    import torch

    import bench

    if not torch.cuda.is_available():
        raise SystemExit("refine_contention.py needs a CUDA device (or --dry-run)")
    assert bench.SAMPLE_RATE == SAMPLE_RATE
    sampler = bench.ClockSampler(0)
    sampler.start()
    results = {}
    with tempfile.TemporaryDirectory(prefix="vgb_refine_diag_") as tmp:
        for v in variants:
            lib = load(build_variant(tmp, VARIANTS[v]))
            results[v] = sweep(lib, torch, bench, per_sm, args.seconds, args.reps)
    out["clocks"] = sampler.stop()
    out["gpu"] = bench.gpu_identity(0, torch)
    if isinstance(out["clocks"].get("sm_mhz"), (int, float)):
        out["chain_c"] = fixed_pattern_chain(args.seconds, args.dadd_cycles, float(out["clocks"]["sm_mhz"]))
    out["sweep"] = results
    print(json.dumps(out))
    print("variant  " + "  ".join(f"{k:>6}/SM" for k in per_sm) + "   8/1")
    for v, rows in results.items():
        print(f"{v:>7}  " + "  ".join(f"{r['refine_ms']:9.3f}" for r in rows) + f"  {rows[-1]['refine_ms'] / rows[0]['refine_ms']:5.2f}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
