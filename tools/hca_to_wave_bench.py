#!/usr/bin/env python
"""tools/hca_to_wave_bench.py — the fill pass of vgb_convert_hca_to_wave_batch on a job of .hca files.

  python tools/hca_to_wave_bench.py [--files 2048] [--runs 5] [--warmup 1] [--check 24]

The job is made by the product itself, so it needs nothing outside the tree: synth PCM (2/3 mono, 1/3 stereo, 1-10 s at
48 kHz, every eighth file looping) becomes WAVE images, vgb_convert_wave_batch encodes them to .hca at quality High,
every fourth file with the type-56 key.  The fill pass then runs `warmup` times and `runs` times under a host clock (the
call returns after its last copy has landed); the median is reported.  `check` files spread over the job are compared
with the oracle chain (tests/hca_reader_oracle.py's hca_parse -> hca_crypt_frames -> hca_decode -> wave_write16).  One
JSON line with the GPU's name and power limit.
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

KEY = 0x00D7E1B6C2A94F03


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=24)
    a = ap.parse_args()

    import numpy as np
    import torch

    import bench
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct
    from vgaudio_b200 import synth
    from test_hca_to_wave_gpu import _expected

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    N.check(N.lib.vgb_init(0, 0))
    rng = np.random.default_rng(2026)
    waves = []
    for i in range(a.files):
        ch = 2 if i % 3 == 2 else 1
        n = int(rng.integers(48000, 480001))
        pcm = [synth.channel(4 * i + c, n, 48000, degenerate=False) for c in range(ch)]
        loop = (n // 5, n - n // 7) if i % 8 == 0 else None
        waves.append(O.wave_write16(pcm, 48000, loop))
    hcas = [None] * a.files
    for keyed in (0, 1):
        pick = [i for i in range(a.files) if (i % 4 == 3) == bool(keyed)]
        opt = ct.convert_options(ct.CONTAINER_HCA, hca_quality=2, hca_key_type=56 if keyed else -1, hca_key_code=KEY)
        outs, st = ct.convert_wave_batch([waves[i] for i in pick], opt)
        assert all(s == 0 for s in st)
        for i, o in zip(pick, outs):
            hcas[i] = o
    del waves
    n = a.files
    ftab = (C.c_void_p * n)(*[h.ctypes.data for h in hcas])
    lens = (C.c_int64 * n)(*[h.size for h in hcas])
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    code = C.c_uint64(KEY)
    N.check(N.lib.vgb_convert_hca_to_wave_batch(ftab, lens, n, C.byref(code), sizes, None, status))
    assert all(status[i] == 0 for i in range(n))
    outs = [torch.empty(sizes[i], dtype=torch.uint8).pin_memory() for i in range(n)]
    otab = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
    times = []
    for r in range(a.warmup + a.runs):
        t0 = time.perf_counter()
        N.check(N.lib.vgb_convert_hca_to_wave_batch(ftab, lens, n, C.byref(code), sizes, otab, status))
        if r >= a.warmup:
            times.append(time.perf_counter() - t0)
    assert all(status[i] == 0 for i in range(n))
    checked = sorted(set(np.linspace(0, n - 1, min(a.check, n)).astype(int).tolist()))
    identical = all(outs[i].numpy().tobytes() == _expected(O, hcas[i], KEY).tobytes() for i in checked)
    frames = sum(int(h[16]) << 24 | int(h[17]) << 16 | int(h[18]) << 8 | int(h[19]) for h in hcas)
    pcm_bytes = sum(int(sizes[i]) for i in range(n))
    ident = bench.gpu_identity(0, torch)
    med = statistics.median(times)
    print(json.dumps({"tool": "hca_to_wave_bench", "files": n, "hca_bytes": int(sum(h.size for h in hcas)), "frames": frames,
                      "wave_bytes": pcm_bytes, "runs": a.runs, "median_ms": round(med * 1e3, 3),
                      "min_ms": round(min(times) * 1e3, 3), "max_ms": round(max(times) * 1e3, 3),
                      "wave_gb_per_s": round(pcm_bytes / med / 1e9, 3), "oracle_checked": len(checked), "oracle_identical": identical,
                      "gpu": ident["name"], "power_limit_w": ident["power_limit_w"]}), flush=True)
    N.check(N.lib.vgb_shutdown())
    if not identical:
        raise SystemExit("converted files differ from the oracle chain")


if __name__ == "__main__":
    main()
