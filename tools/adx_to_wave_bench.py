#!/usr/bin/env python
"""tools/adx_to_wave_bench.py — the fill pass of vgb_convert_adx_to_wave_batch, time-parallel decode against the serial one.

  python tools/adx_to_wave_bench.py [--files 2048] [--tracks 32] [--runs 3] [--warmup 1] [--check 16]

Two jobs, made by the product itself from synth PCM (WAVE images encoded to .adx by vgb_convert_wave_batch, Linear, 18-byte
frames, version 4):
  short  `files` files of 1-10 s at 48 kHz, 2/3 mono and 1/3 stereo, every eighth looping (so padded), every fourth
         keyed (type 9), as tools/hca_to_wave_bench.py builds its job;
  tracks `tracks` stereo files of 3 minutes at 48 kHz, looping - the BGM case one thread per channel serves worst.
Each job's fill pass runs with the segmented decode and with VGB_ADX_DEC_SEGMENTS=1 (the plain serial loop inside the
same kernels), alternating, `warmup` + `runs` times each under a host clock (the call returns after its last copy has
landed); medians, minima and maxima are reported.  The ADX-decode kernel time is the decoder alone on the job's channel
rows, already on the device: vgb_adx_decode_dev with kernel timing on (CUDA events, slot 5 of vgb_last_kernel_ms).
`check` files of each job are compared with the oracle chain (tests/adx_reader_oracle.py).  One JSON line per job with
the GPU's name and power limit.
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


def _adx_job(ct, O, synth, np, specs):
    """specs: (channels, samples, loop or None, keyed) -> .adx images (product encoder)."""
    out = [None] * len(specs)
    for keyed in (False, True):
        pick = [i for i, s in enumerate(specs) if s[3] == keyed]
        if not pick:
            continue
        waves = []
        for i in pick:
            ch, n, loop, _ = specs[i]
            waves.append(O.wave_write16([synth.channel(4 * i + c, n, 48000, degenerate=False) for c in range(ch)], 48000, loop))
        k = ct.adx_key(key_code=KEY)
        opt = ct.convert_options(ct.CONTAINER_ADX, adx_encryption_type=9 if keyed else 0, adx_has_key=int(keyed),
                                 adx_key_seed=k.seed, adx_key_mult=k.mult, adx_key_inc=k.inc)
        outs, st = ct.convert_wave_batch(waves, opt)
        assert all(s == 0 for s in st)
        for i, o in zip(pick, outs):
            out[i] = o
    return out


def _kernel_ms(N, ct, criadx, np, torch, adxs, key, segments):
    """The decoder alone on every channel row of the job, rows already de-interleaved and decrypted on the device."""
    rows, counts, configs = [], [], []
    for img in adxs:
        h = ct.adx_parse(img)
        audio = np.asarray(img[h.audio_offset: h.audio_offset + h.audio_size]).reshape(-1, h.channel_count, h.frame_size)
        chans = [np.ascontiguousarray(audio[:, c, :]).ravel() for c in range(h.channel_count)]
        if h.revision in (8, 9):
            chans = ct.adx_crypt(chans, key, h.revision, h.frame_size)
        for r in chans:
            rows.append(r)
            counts.append(h.sample_count - h.inserted_samples)
            configs.append(criadx.CriAdxParameters(h.sample_rate, h.highpass_frequency, h.frame_size, h.version, 0, max(h.inserted_samples, 0), h.type))
    a_off = np.cumsum([0] + [(r.size + 15) // 16 * 16 for r in rows])[:-1].astype(np.int64)
    d_adpcm = torch.from_numpy(np.concatenate([np.pad(r, (0, (r.size + 15) // 16 * 16 - r.size)) for r in rows])).cuda()
    p_off = np.cumsum([0] + [(c + 7) // 8 * 8 for c in counts])[:-1].astype(np.int64)
    d_pcm = torch.empty(int(p_off[-1] + counts[-1] + 8), dtype=torch.int16, device="cuda")
    if segments:
        os.environ["VGB_ADX_DEC_SEGMENTS"] = segments
    try:
        N.check(N.lib.vgb_set_kernel_timing(1))
        ms = []
        ws = None
        for _ in range(3):
            ws = criadx.decode_dev(d_adpcm, a_off, [r.size for r in rows], counts, configs, d_pcm, p_off, workspace=ws)
            t = (C.c_float * 10)()
            N.lib.vgb_last_kernel_ms(t, 10)
            ms.append(t[5])
        N.check(N.lib.vgb_set_kernel_timing(0))
    finally:
        os.environ.pop("VGB_ADX_DEC_SEGMENTS", None)
    stats = (C.c_uint64 * 5)()
    N.check(N.lib.vgb_adx_debug_decode_stats(stats, 5))  # reads the bookkeeping from ws, still allocated here
    del ws
    return statistics.median(ms), list(stats)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--tracks", type=int, default=32)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=16)
    a = ap.parse_args()

    import numpy as np
    import torch

    import adx_reader_oracle as R
    import bench
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct
    from vgaudio_b200 import criadx, synth

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    O.build()
    N.check(N.lib.vgb_init(0, 0))
    rng = np.random.default_rng(2026)
    short = []
    for i in range(a.files):
        n = int(rng.integers(48000, 480001))
        short.append((2 if i % 3 == 2 else 1, n, (n // 5, n - n // 7) if i % 8 == 0 else None, i % 4 == 3))
    tracks = [(2, 180 * 48000, (48000 * 7 + 11, 180 * 48000 - 5), False) for _ in range(a.tracks)]
    ident = bench.gpu_identity(0, torch)
    key = ct.adx_key(key_code=KEY)
    okey = O.adx_key(key_code=KEY)
    ok_all = True
    for name, specs in (("short", short), ("tracks", tracks)):
        adxs = _adx_job(ct, O, synth, np, specs)
        n = len(adxs)
        ftab = (C.c_void_p * n)(*[h.ctypes.data for h in adxs])
        lens = (C.c_int64 * n)(*[h.size for h in adxs])
        sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
        N.check(N.lib.vgb_convert_adx_to_wave_batch(ftab, lens, n, C.byref(key), sizes, None, status))
        assert all(status[i] == 0 for i in range(n))
        outs = [torch.empty(sizes[i], dtype=torch.uint8).pin_memory() for i in range(n)]
        otab = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
        times = {"segmented": [], "serial": []}
        for r in range(a.warmup + a.runs):
            for arm in ("segmented", "serial"):
                if arm == "serial":
                    os.environ["VGB_ADX_DEC_SEGMENTS"] = "1"
                t0 = time.perf_counter()
                N.check(N.lib.vgb_convert_adx_to_wave_batch(ftab, lens, n, C.byref(key), sizes, otab, status))
                dt = time.perf_counter() - t0
                os.environ.pop("VGB_ADX_DEC_SEGMENTS", None)
                assert all(status[i] == 0 for i in range(n))
                if r >= a.warmup:
                    times[arm].append(dt)
                if arm == "serial" and r == a.warmup + a.runs - 1:  # the last fill pass: the serial arm's bytes
                    serial_bytes = [outs[i].numpy().tobytes() for i in range(n)]
        checked = sorted(set(np.linspace(0, n - 1, min(a.check, n)).astype(int).tolist()))
        identical = all(outs[i].numpy().tobytes() == R.expected_wave(adxs[i], okey).tobytes() for i in checked)
        seg_ms, stats = _kernel_ms(N, ct, criadx, np, torch, adxs, key, None)
        ser_ms, _ = _kernel_ms(N, ct, criadx, np, torch, adxs, key, "1")
        N.check(N.lib.vgb_convert_adx_to_wave_batch(ftab, lens, n, C.byref(key), sizes, otab, status))
        same_arms = all(outs[i].numpy().tobytes() == serial_bytes[i] for i in range(n))
        ok_all &= identical and same_arms
        wave_bytes = sum(int(sizes[i]) for i in range(n))
        row = {"tool": "adx_to_wave_bench", "job": name, "files": n, "adx_bytes": int(sum(h.size for h in adxs)), "wave_bytes": wave_bytes,
               "runs": a.runs, "gpu": ident["name"], "power_limit_w": ident["power_limit_w"],
               "decode_kernel_ms": {"segmented": round(seg_ms, 3), "serial": round(ser_ms, 3)},
               "segments": stats[0], "runon_frames": stats[1], "cascade_frames": stats[2], "boundaries_repaired": stats[3],
               "longest_runon": stats[4], "oracle_checked": len(checked), "oracle_identical": identical, "arms_identical": same_arms}
        for arm, ts in times.items():
            row[f"{arm}_ms"] = {"median": round(statistics.median(ts) * 1e3, 2), "min": round(min(ts) * 1e3, 2), "max": round(max(ts) * 1e3, 2)}
        print(json.dumps(row), flush=True)
    N.check(N.lib.vgb_shutdown())
    if not ok_all:
        raise SystemExit("converted files differ from the oracle chain or between the arms")


if __name__ == "__main__":
    main()
