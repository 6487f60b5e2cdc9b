#!/usr/bin/env python
"""tools/align_bench.py — GcAdpcmAlignment (loop alignment) of GC-ADPCM channels: vgb_gcadpcm_align_batch against the
composition it replaced and against the CPU oracle.

  python tools/align_bench.py [--channels 512] [--seconds 60] [--runs 3] [--warmup 1]

Workloads: seeded looping channels of `seconds` at 48 kHz, aligned to the BRSTM default multiple 0x3800
(BxstmConfiguration's LoopPointAlignment): a batch of `channels` channels, each with its own loop points, and one stereo
file (two channels sharing theirs).  The input ADPCM is encoded once by the library.  Arms:
  align_batch   the one native call (H2D of the prefixes, decode, tail, encode, decode, D2H, one synchronisation)
  composition   what formats.align_loops did before that call existed: decode_batch of [0, loop_end) to the host, the
                tails built on the host, encode_batch from the reconstructed history, decode_batch of the tails
  oracle        oracle/gcalign.c's vgo_gc_align per channel on every host core (a thread per core; ctypes releases the GIL)
Each timing is the wall time of the synchronous call(s), after `warmup` untimed calls (the oracle runs once).  Every
arm's AdpcmAligned and PcmAligned bytes must equal align_batch's.  One JSON line per (workload, arm), with the card's
name and power limit read in the same run.
"""
import argparse
import concurrent.futures as cf
import ctypes as C
import hashlib
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MULTIPLE = 0x3800
RATE = 48000


def make_channels(torch, n_channels, n, seed):
    """Seeded PCM on the GPU (three sines and noise per channel), encoded by the library: (adpcm rows, coefs)."""
    import vgaudio_b200 as vg

    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.arange(n, device="cuda", dtype=torch.float64) / RATE
    pcm = torch.empty((n_channels, n), dtype=torch.int16)
    for c in range(n_channels):
        f = torch.exp(torch.empty(3, device="cuda", dtype=torch.float64).uniform_(np.log(60.0), np.log(12000.0), generator=g))
        a = torch.empty(3, device="cuda", dtype=torch.float64).uniform_(500.0, 9000.0, generator=g)
        x = (a[:, None] * torch.sin(2 * np.pi * f[:, None] * t[None, :])).sum(0)
        x += torch.randn(n, device="cuda", dtype=torch.float64, generator=g) * 300.0
        pcm[c].copy_(x.round().clamp(-32768, 32767).to(torch.int16))
    coefs, adpcm = vg.gcadpcm.encode_batch(pcm.numpy())
    return adpcm, coefs


def loop_points(n_channels, n, seed, shared):
    rng = np.random.default_rng([0x414C49474E, seed])
    out = []
    for c in range(n_channels):
        if shared and c:
            out.append(out[0])
            continue
        loop_start = int(rng.integers(1, n // 2))
        loop_start += loop_start % MULTIPLE == 0  # every channel needs alignment
        out.append((MULTIPLE, loop_start, n - int(rng.integers(0, 14 * 64))))
    return out


def digest(adpcm_rows, pcm_rows):
    h = hashlib.sha256()
    for a, p in zip(adpcm_rows, pcm_rows):
        h.update(np.ascontiguousarray(a).tobytes())
        h.update(np.ascontiguousarray(p).tobytes())
    return h.hexdigest()


def arm_align_batch(vg, N, adpcm, coefs, params):
    n = len(adpcm)
    geo = [vg.gcadpcm.alignment(*p) for p in params]
    out_a = [np.zeros(vg.gcadpcm.sample_count_to_byte_count(g[2]), np.uint8) for g in geo]
    out_p = [np.zeros(g[2], np.int16) for g in geo]
    lens = np.array([len(a) for a in adpcm], dtype=np.int32)
    par = (N.VgbGcAlignParams * n)(*[N.VgbGcAlignParams(*p) for p in params])
    tab = lambda rows: (C.c_void_p * n)(*[r.ctypes.data for r in rows])  # noqa: E731
    co = np.ascontiguousarray(coefs)
    args = (tab(adpcm), lens.ctypes.data, co.ctypes.data, C.cast(par, C.c_void_p), n, tab(out_a), tab(out_p))

    def run():
        assert lens.size == co.shape[0] == n  # keeps the arrays behind the raw addresses in `args` alive
        N.check(vg.lib.vgb_gcadpcm_align_batch(*args))
        return out_a, out_p
    return run


def arm_composition(vg, adpcm, coefs, params):
    """The three-call composition formats.align_loops ran before vgb_gcadpcm_align_batch (GcAdpcmAlignment.cs:41-62)."""
    P = vg.gcadpcm.GcAdpcmParameters

    def run():
        n = len(adpcm)
        old = vg.gcadpcm.decode_batch(adpcm, coefs, [P(sample_count=p[2]) for p in params])
        tails, configs, pcm_aligned, geo = [], [], [], []
        for c, (multiple, loop_start, loop_end) in enumerate(params):
            count = vg.gcadpcm.alignment(multiple, loop_start, loop_end)[2]
            keep = loop_end // 14 * 14
            aligned = np.zeros(count, dtype=np.int16)
            aligned[:loop_end] = old[c][:loop_end]
            tail = np.zeros(count - keep, dtype=np.int16)
            tail[:loop_end - keep] = old[c][keep:loop_end]
            cur = loop_end - keep
            while cur < count - keep:
                k = min(loop_end - loop_start, count - keep - cur)
                tail[cur:cur + k] = aligned[loop_start:loop_start + k]
                cur += loop_end - loop_start
            tails.append(tail)
            pcm_aligned.append(aligned)
            geo.append((keep, count))
            configs.append(P(sample_count=count - keep, history1=int(old[c][keep - 1]) if keep >= 1 else 0,
                             history2=int(old[c][keep - 2]) if keep >= 2 else 0))
        _, new_adpcm = vg.gcadpcm.encode_batch(tails, coefs=coefs, configs=configs)
        decoded = vg.gcadpcm.decode_batch(new_adpcm, coefs, configs)
        out_a = []
        for c in range(n):
            keep, count = geo[c]
            a = np.zeros(vg.gcadpcm.sample_count_to_byte_count(count), dtype=np.uint8)
            a[:keep // 14 * 8] = adpcm[c][:keep // 14 * 8]
            a[keep // 14 * 8:] = new_adpcm[c]
            pcm_aligned[c][keep:] = decoded[c][:count - keep]
            out_a.append(a)
        return out_a, pcm_aligned
    return run


def arm_oracle(gc_align, adpcm, coefs, params):
    def one(c):
        rc, _, a, p = gc_align(*params[c], adpcm[c], coefs[c])
        assert rc == 0
        return a, p

    def run():
        with cf.ThreadPoolExecutor(os.cpu_count()) as ex:
            res = list(ex.map(one, range(len(adpcm))))
        return [r[0] for r in res], [r[1] for r in res]
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=512)
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()

    import torch

    import bench
    import vgaudio_b200 as vg
    from oracle.pygcalign import gc_align
    from vgaudio_b200 import _native as N

    if not torch.cuda.is_available():
        raise SystemExit("align_bench measures the GPU path: no CUDA device")
    N.check(vg.lib.vgb_init(0, 0))
    ident = bench.gpu_identity(0, torch)
    n = int(a.seconds * RATE)
    ok = True
    for workload, n_ch, shared in (("batch", a.channels, False), ("stereo", 2, True)):
        adpcm, coefs = make_channels(torch, n_ch, n, seed=n_ch)
        params = loop_points(n_ch, n, n_ch, shared)
        want = None
        arms = (("align_batch", lambda: arm_align_batch(vg, N, adpcm, coefs, params), a.warmup, a.runs),
                ("composition", lambda: arm_composition(vg, adpcm, coefs, params), a.warmup, a.runs),
                ("oracle", lambda: arm_oracle(gc_align, adpcm, coefs, params), 0, 1))
        for arm, make, warmup, runs in arms:  # one arm's buffers at a time: the batch holds gigabytes per arm
            run = make()
            for _ in range(warmup):
                run()
            ms = []
            for _ in range(runs):
                t0 = time.perf_counter()
                out_a, out_p = run()
                ms.append((time.perf_counter() - t0) * 1e3)
            d = digest(out_a, out_p)
            want = want or d
            ok = ok and d == want
            print(json.dumps({"workload": workload, "arm": arm, "channels": n_ch, "seconds": a.seconds, "multiple": MULTIPLE,
                              "aligned_samples": int(sum(len(p) for p in out_p)), "runs": runs,
                              "ms_median": round(statistics.median(ms), 3), "ms_all": [round(x, 3) for x in ms],
                              "bytes_equal_align_batch": d == want, "host_cores": os.cpu_count(),
                              "gpu": ident["name"], "power_limit_w": ident["power_limit_w"]}), flush=True)
            del run, out_a, out_p
    N.check(vg.lib.vgb_shutdown())
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
