#!/usr/bin/env python
"""tools/cri_rewrite_bench.py — vgb_rewrite_batch's fill pass against its copy floor.

  python tools/cri_rewrite_bench.py [--files 2048] [--tracks 32] [--runs 5] [--warmup 1] [--check 64] [--profile DIR]

Four seeded jobs, built once with the product's own writers (vgb_convert_wave_batch from WAVE images of stereo noise
and tones at 44.1 kHz, every fourth file looping):
  hca_short   `files` .hca files of 1-10 s, keyed with a type-56 key, rewritten in the clear;
  adx_short   `files` .adx files of 1-10 s, keyed with a type-9 key code, re-keyed with a type-8 key string;
  hca_tracks / adx_tracks   `tracks` stereo files of 3 minutes, the same rewrites.
Per job, alternating with the copy floor, `warmup` + `runs` fill passes under a host clock (every buffer is pinned; the
sizing pass, host only, is outside the timed region), and the floor: one pinned H2D of the job's input bytes plus one
D2H of its output bytes, CUDA events around each.  `check` files per job (every track) are compared byte for byte with
the oracle chain (tests/cri_rewrite_oracle.py), whose one-thread time is reported for scale, extrapolated by bytes from
those files.  One JSON line per job with the GPU's name and power limit.  --profile DIR traces one fill pass of each job
with torch.profiler (CUDA activities) into DIR, in a run of its own.
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

HCA_KEY = 0x00D7E1B6C2A94F03
ADX_KEY_CODE = 0x0123456789ABCDEF
ADX_KEY_STRING = "vgaudio-b200"
RATE = 44100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--tracks", type=int, default=32)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=64)
    ap.add_argument("--profile", default="")
    a = ap.parse_args()

    import numpy as np
    import torch

    import bench
    import cri_rewrite_oracle as R
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    O.build()
    N.check(N.lib.vgb_init(0, 0))
    ident = bench.gpu_identity(0, torch)
    in_adx = ct.adx_key(key_code=ADX_KEY_CODE)
    out_adx = ct.adx_key(key_string=ADX_KEY_STRING)
    hca_code = C.c_uint64(HCA_KEY)

    def tab(ts):
        return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts]), (C.c_int64 * len(ts))(*[int(t.numel()) for t in ts])

    def pinned(arr):
        t = torch.empty(max(int(arr.size), 1), dtype=torch.uint8, pin_memory=True)
        t.numpy()[: arr.size] = arr
        return t[: arr.size]

    def wave(rng, seconds, looping):
        n = int(seconds * RATE)
        t = np.arange(n) / RATE
        pcm = [np.clip(3000 * np.sin(2 * np.pi * rng.uniform(80, 4000) * t) + rng.normal(0, 800, n), -32768, 32767).astype(np.int16)
               for _ in range(2)]
        return O.wave_write16(pcm, RATE, (n // 5, n - 7) if looping else None)

    def encode(lengths, out_type, seed):
        """The job's files in out_type, keyed, from WAVE images made 256 at a time."""
        rng = np.random.default_rng(seed)
        opt = ct.convert_options(out_type, hca_key_type=56 if out_type == R.HCA else -1, hca_key_code=HCA_KEY,
                                 adx_has_key=int(out_type == R.ADX), adx_encryption_type=9 if out_type == R.ADX else 0,
                                 adx_key_seed=in_adx.seed, adx_key_mult=in_adx.mult, adx_key_inc=in_adx.inc)
        files = []
        for g in range(0, len(lengths), 256):
            waves = [wave(rng, s, (g + k) % 4 == 0) for k, s in enumerate(lengths[g:g + 256])]
            outs, status = ct.convert_wave_batch(waves, opt)
            assert all(s == 0 for s in status)
            files += [pinned(o) for o in outs]
        return files

    rng = np.random.default_rng(1)
    short = rng.uniform(1.0, 10.0, a.files).tolist()
    jobs = [("hca_short", R.HCA, encode(short, R.HCA, 2)), ("adx_short", R.ADX, encode(short, R.ADX, 3)),
            ("hca_tracks", R.HCA, encode([180.0] * a.tracks, R.HCA, 4)), ("adx_tracks", R.ADX, encode([180.0] * a.tracks, R.ADX, 5))]

    ok_all = True
    for job, fmt, files in jobs:
        n = len(files)
        ftab, lens = tab(files)
        opt = ct.convert_options(fmt) if fmt == R.HCA else ct.convert_options(
            fmt, adx_has_key=1, adx_encryption_type=8, adx_key_seed=out_adx.seed, adx_key_mult=out_adx.mult, adx_key_inc=out_adx.inc)
        call = lambda s, o, st: N.lib.vgb_rewrite_batch(ftab, lens, n, C.byref(opt), C.byref(in_adx), C.byref(hca_code), s, o, st, None, None)  # noqa: E731
        sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
        N.check(call(sizes, None, status))
        assert all(status[i] == 0 for i in range(n))
        outs = [torch.empty(int(sizes[i]), dtype=torch.uint8, pin_memory=True) for i in range(n)]
        otab = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
        in_bytes, out_bytes = sum(int(f.numel()) for f in files), sum(int(sizes[i]) for i in range(n))
        h_in = torch.empty(in_bytes, dtype=torch.uint8, pin_memory=True)
        h_out = torch.empty(out_bytes, dtype=torch.uint8, pin_memory=True)
        d_in = torch.empty(in_bytes, dtype=torch.uint8, device="cuda")
        d_out = torch.empty(out_bytes, dtype=torch.uint8, device="cuda")
        fill, floor_h2d, floor_d2h = [], [], []
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        for r in range(a.warmup + a.runs):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            N.check(call(sizes, otab, status))
            dt = time.perf_counter() - t0
            e0.record()
            d_in.copy_(h_in, non_blocking=True)
            e1.record()
            h_out.copy_(d_out, non_blocking=True)
            e2.record()
            torch.cuda.synchronize()
            if r >= a.warmup:
                fill.append(dt)
                floor_h2d.append(e0.elapsed_time(e1) / 1e3)
                floor_d2h.append(e1.elapsed_time(e2) / 1e3)
        # a sample against the oracle chain, and its one-thread time
        checked = sorted(set(np.linspace(0, n - 1, min(a.check, n)).astype(int).tolist()))
        same, t_oracle, b_oracle = True, 0.0, 0
        for i in checked:
            img = files[i].numpy()
            t0 = time.perf_counter()
            want = R.expected_hca(img, in_key_code=HCA_KEY) if fmt == R.HCA else R.expected_adx(img, 8, O.adx_key(key_string=ADX_KEY_STRING), False,
                                                                                               O.adx_key(key_code=ADX_KEY_CODE))
            t_oracle += time.perf_counter() - t0
            b_oracle += img.size
            same &= want is not None and outs[i].numpy().tobytes() == want.tobytes()
        ok_all &= same
        fill_med = statistics.median(fill)
        floor = statistics.median(floor_h2d) + statistics.median(floor_d2h)
        row = {"tool": "cri_rewrite_bench", "job": job, "files": n, "in_bytes": in_bytes, "out_bytes": out_bytes, "runs": a.runs,
               "gpu": ident["name"], "power_limit_w": ident["power_limit_w"],
               "fill_ms": {"median": round(fill_med * 1e3, 2), "min": round(min(fill) * 1e3, 2), "max": round(max(fill) * 1e3, 2)},
               "floor_ms": {"h2d": round(statistics.median(floor_h2d) * 1e3, 2), "d2h": round(statistics.median(floor_d2h) * 1e3, 2),
                            "sum": round(floor * 1e3, 2)},
               "fill_over_floor": round(fill_med / floor, 3), "fill_gb_per_s": round((in_bytes + out_bytes) / fill_med / 1e9, 2),
               "oracle_one_thread_s": round(t_oracle * in_bytes / max(b_oracle, 1), 2), "oracle_checked": len(checked), "oracle_identical": same}
        print(json.dumps(row), flush=True)
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                N.check(call(sizes, otab, status))
                torch.cuda.synchronize()
            out = Path(a.profile)
            out.mkdir(parents=True, exist_ok=True)
            (out / f"{job}.txt").write_text(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
        del outs, h_in, h_out, d_in, d_out
    N.check(N.lib.vgb_shutdown())
    if not ok_all:
        raise SystemExit("rewritten files differ from the oracle chain")


if __name__ == "__main__":
    main()
