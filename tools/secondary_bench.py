#!/usr/bin/env python
"""tools/secondary_bench.py — the host entry points of the non-headline codecs at full size on one GPU, PINNED host
buffers: CRI ADX encode / decode (1024 channels x 30 s) and CRI HCA decode (512 mono streams x 30 s, quality High).
(GC-ADPCM decode and HCA encode at full size are `bench.py --config c3 / c4`.)

Per entry:
  kernel_ms        CUDA events around the kernels of an UNPIPELINED call (VGB_PIPELINE_GROUPS=1)
  wall_ms          the synchronous host call, pipelined over unit groups (H2D || kernels || D2H), copies included
  pcie_floor_ms    max(H2D bytes, D2H bytes) / 55 GB/s (the links are full duplex)
  wall_over_floor  wall_ms / max(pcie_floor_ms, kernel_ms): 1.0 = perfectly hidden
  roofline         algorithmic bytes / kernel_ms against MEASURED_PEAKS.json's HBM copy bandwidth
  cpu_baseline     the oracle port on all host cores (one channel / stream per task), bounded sample
  parity           outputs of a sample of units compared with the oracle, bit-exact
Usage: python tools/secondary_bench.py [--scale 1.0] > secondary_bench.json
"""
import argparse
import ctypes as C
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import vgaudio_b200 as vg  # noqa: E402
from oracle import pyoracle  # noqa: E402  (checker and CPU baseline only)
from vgaudio_b200 import _native as N  # noqa: E402

SLOT = {"adx_encode": 4, "adx_decode": 5, "hca_encode": 6, "hca_decode": 7}
RATE = 48000
CORES = os.cpu_count() or 1


def peak_gbs():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return 3350.0, "H100 SXM data sheet (3.35 TB/s), not measured"


def measure(call, slot, reps=3):
    """(wall_ms pipelined, kernel_ms unpipelined)."""
    os.environ["VGB_PIPELINE_GROUPS"] = "1"
    call()
    kms = None
    buf = (C.c_float * 10)()
    for _ in range(2):
        call()
        N.check(vg.lib.vgb_last_kernel_ms(buf, 10))
        kms = float(buf[slot]) if kms is None else min(kms, float(buf[slot]))
    os.environ.pop("VGB_PIPELINE_GROUPS", None)
    call()
    best = None
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        dt = (time.perf_counter() - t0) * 1e3
        best = dt if best is None else min(best, dt)
    return best, kms


def entry(name, samples, wall, kms, h2d, d2h, alg_bytes, cpu, parity, extra):
    peak, src = peak_gbs()
    floor = max(h2d, d2h) / 55e9 * 1e3
    out = {"path": name}
    out.update(extra)
    out.update({"Msamples_per_s_e2e": round(samples / wall / 1e3, 1), "wall_ms": round(wall, 2), "kernel_ms": round(kms, 3),
                "kernel_Msamples_per_s": round(samples / kms / 1e3, 1), "h2d_bytes": int(h2d), "d2h_bytes": int(d2h),
                "pcie_floor_ms": round(floor, 2), "wall_over_floor": round(wall / max(floor, kms), 3),
                "roofline": {"bound": "hbm", "achieved": round(alg_bytes / kms / 1e6, 1), "peak": peak, "unit": "GB/s",
                             "frac": round(alg_bytes / kms / 1e6 / peak, 4), "algorithmic_bytes": int(alg_bytes), "peak_source": src},
                "cpu_baseline": cpu, "parity": parity})
    return out


def cpu_rate(fn, units, samples_per_unit, what):
    k = min(len(units), CORES)
    t0 = time.perf_counter()
    with ThreadPoolExecutor(max_workers=k) as pool:
        res = list(pool.map(fn, units[:k]))
    dt = time.perf_counter() - t0
    return res, {"value": round(k * samples_per_unit / dt / 1e6, 2), "unit": "Msamples/s", "cores": k, "kind": "port",
                 "sample": f"{k} units x {samples_per_unit} samples ({dt:.2f} s wall), {what}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    N.check(vg.lib.vgb_init(0, 0))
    N.check(vg.lib.vgb_set_kernel_timing(1))
    n = int(30 * RATE)
    results = []

    # ---------------- CRI ADX: 1024 channels, Linear, version 4, 18-byte frames ----------------
    n_ch = max(32, int(1024 * args.scale))
    pcm = bench.make_batch_gpu(torch, n_ch, n, 11, dev)
    h_pcm = torch.empty((n_ch, n), dtype=torch.int16, pin_memory=True)
    h_pcm.copy_(pcm)
    nb = int(vg.lib.vgb_adx_encoded_byte_count(n, 0, 18))
    h_adx = torch.empty((n_ch, nb), dtype=torch.uint8, pin_memory=True)
    h_dec = torch.empty((n_ch, n), dtype=torch.int16, pin_memory=True)
    params = (N.VgbAdxParams * n_ch)(*[N.VgbAdxParams(RATE, 500, 18, 4, 0, 0, 3, 0) for _ in range(n_ch)])
    lens = np.full(n_ch, n, dtype=np.int32)
    nbs = np.full(n_ch, nb, dtype=np.int32)
    hist = np.zeros(n_ch, dtype=np.int16)
    in_tab = (C.c_void_p * n_ch)(*[h_pcm.data_ptr() + 2 * n * c for c in range(n_ch)])
    adx_tab = (C.c_void_p * n_ch)(*[h_adx.data_ptr() + nb * c for c in range(n_ch)])
    dec_tab = (C.c_void_p * n_ch)(*[h_dec.data_ptr() + 2 * n * c for c in range(n_ch)])

    def adx_enc():
        N.check(vg.lib.vgb_adx_encode_batch(in_tab, lens.ctypes.data, params, n_ch, hist.ctypes.data, adx_tab, None, None))

    wall, kms = measure(adx_enc, SLOT["adx_encode"])
    host = h_pcm.numpy()
    res, cpu = cpu_rate(lambda c: pyoracle.adx_encode(host[c], RATE, 18, 4, 0, 3, 0), list(range(n_ch)), n,
                        "C restatement of CriAdxCodec.Encode, one channel per task")
    ok = all(np.array_equal(h_adx[c].numpy(), res[c][0]) and int(hist[c]) == res[c][1] for c in range(len(res)))
    results.append(entry("CRI ADX encode (vgb_adx_encode_batch)", n_ch * n, wall, kms, n_ch * n * 2, n_ch * nb, n_ch * (n * 2 + nb), cpu,
                         {"channels_checked": len(res), "bytes_equal_oracle": bool(ok)}, {"channels": n_ch, "samples_per_channel": n}))

    for c in range(n_ch):
        params[c].history = int(hist[c])

    def adx_dec():
        counts = np.full(n_ch, n, dtype=np.int32)
        N.check(vg.lib.vgb_adx_decode_batch(adx_tab, nbs.ctypes.data, counts.ctypes.data, params, n_ch, dec_tab))

    wall, kms = measure(adx_dec, SLOT["adx_decode"])
    enc_host = h_adx.numpy()
    res, cpu = cpu_rate(lambda c: pyoracle.adx_decode(enc_host[c], n, RATE, 500, 18, 4, int(hist[c]), 0, 3), list(range(n_ch)), n,
                        "C restatement of CriAdxCodec.Decode, one channel per task")
    ok = all(np.array_equal(h_dec[c].numpy(), res[c]) for c in range(len(res)))
    results.append(entry("CRI ADX decode (vgb_adx_decode_batch)", n_ch * n, wall, kms, n_ch * nb, n_ch * n * 2, n_ch * (n * 2 + nb), cpu,
                         {"channels_checked": len(res), "pcm_equal_oracle": bool(ok)}, {"channels": n_ch, "samples_per_channel": n}))
    del pcm

    # ---------------- CRI HCA decode: 512 mono streams, quality High ----------------
    n_st = max(16, int(512 * args.scale))
    pcm = bench.make_batch_gpu(torch, n_st, n, 12, dev, degenerate=False)
    h_in = torch.empty((n_st, n), dtype=torch.int16, pin_memory=True)
    h_in.copy_(pcm)
    hp = (N.VgbHcaParams * n_st)(*[N.VgbHcaParams(2, 0, 0, 1, RATE, n, 0, 0, 0) for _ in range(n_st)])
    infos = (N.VgbHcaInfo * n_st)()
    N.check(vg.lib.vgb_hca_query(C.byref(hp[0]), C.byref(infos[0])))
    fbytes = infos[0].frame_count * infos[0].frame_size
    h_frames = torch.empty((n_st, fbytes), dtype=torch.uint8, pin_memory=True)
    h_out = torch.empty((n_st, n), dtype=torch.int16, pin_memory=True)
    pin = (C.c_void_p * n_st)(*[h_in.data_ptr() + 2 * n * s for s in range(n_st)])
    ftab = (C.c_void_p * n_st)(*[h_frames.data_ptr() + fbytes * s for s in range(n_st)])
    otab = (C.c_void_p * n_st)(*[h_out.data_ptr() + 2 * n * s for s in range(n_st)])
    N.check(vg.lib.vgb_hca_encode_batch(pin, hp, n_st, infos, ftab, None, None))

    def hca_dec():
        N.check(vg.lib.vgb_hca_decode_batch(ftab, infos, n_st, otab))

    wall, kms = measure(hca_dec, SLOT["hca_decode"])
    fr_host = h_frames.numpy()
    o_info = pyoracle.HcaInfo()
    C.memmove(C.byref(o_info), C.byref(infos[0]), C.sizeof(o_info))
    res, cpu = cpu_rate(lambda s: pyoracle.hca_decode(o_info, fr_host[s].reshape(infos[0].frame_count, infos[0].frame_size)), list(range(n_st)), n,
                        "C restatement of CriHcaDecoder.Decode, one stream per task")
    ok = all(np.array_equal(h_out[s].numpy(), res[s][0]) for s in range(len(res)))
    results.append(entry("CRI HCA decode (vgb_hca_decode_batch)", n_st * n, wall, kms, n_st * fbytes, n_st * n * 2, n_st * (n * 2 + fbytes), cpu,
                         {"streams_checked": len(res), "pcm_equal_oracle": bool(ok)}, {"streams": n_st, "samples_per_stream": n, "frame_size": int(infos[0].frame_size)}))
    print(json.dumps({"device": torch.cuda.get_device_name(0), "host_cores": CORES, "entries": results}, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
