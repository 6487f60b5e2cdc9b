#!/usr/bin/env python
"""tools/transcode_nw_bench.py — the fill pass of vgb_transcode_nw_batch against the two-call composition through WAVE.

  python tools/transcode_nw_bench.py [--files 2048] [--tracks 32] [--runs 3] [--warmup 1] [--check 3] [--check-tracks 0]

Two jobs of WAVE images: `short`, the 2048-file job of `bench.py --config batch` (mono / stereo, 1-6 s at 48 kHz, every
eighth file looping), and `tracks`, `tracks` stereo files of 3 minutes at 48 kHz, looping.  As set-up each job is encoded
once to keyed .adx and .hca by vgb_convert_wave_batch (default options, HCA quality High).  Then for each direction
.adx / .hca -> .brstm / .bfstm / .idsp / .hps (GC-ADPCM) and .hca -> .bcstm (-f pcm16), alternating, `warmup` + `runs`
times each under a host clock (both calls return after their last copy has landed; every buffer is pinned, and the
sizing passes, host-only, are outside the timed region):
  direct       one vgb_transcode_nw_batch fill pass, coded images in, target images out;
  composition  vgb_convert_to_wave_batch's fill pass, then vgb_convert_wave_batch's fill pass on those WAVE images.
Both arms must give identical bytes and statuses, and `check` files of each direction (`check-tracks` of the tracks) are
compared with the oracle chain (tests/transcode_nw_oracle.py).  One JSON line per job and direction, with the GPU's name
and power limit.
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

ADX_KEY_CODE = 0x0123456789ABCDEF
HCA_KEY = 0x00D7E1B6C2A94F03
NAMES = {2: "adx", 3: "hca", 4: "brstm", 5: "bcstm", 6: "bfstm", 7: "idsp", 8: "hps"}
# (source, target, nw_codec_plus1): GC-ADPCM into every container but BCSTM, PCM16 into BCSTM
DIRECTIONS = [(s, d, 0) for s in (2, 3) for d in (4, 6, 7, 8)] + [(3, 5, 2)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--tracks", type=int, default=32)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=3, help="files per direction of the short job compared with the oracle chain")
    ap.add_argument("--check-tracks", type=int, default=0, help="the same for the tracks job (the CPU oracle takes minutes per track)")
    a = ap.parse_args()

    import numpy as np
    import torch

    import bench
    import bench_configs
    import transcode_nw_oracle as W
    import transcode_oracle as T
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct
    from vgaudio_b200 import synth

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    O.build()
    N.check(N.lib.vgb_init(0, 0))
    ident = bench.gpu_identity(0, torch)
    adx_key = ct.adx_key(key_code=ADX_KEY_CODE)
    hca_code = C.c_uint64(HCA_KEY)

    def pinned(arr):
        t = torch.empty(int(arr.size), dtype=torch.uint8, pin_memory=True)
        t.numpy()[:] = arr
        return t

    def tab(ts):
        return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts]), (C.c_int64 * len(ts))(*[int(t.numel()) for t in ts])

    def to_wave(types, ftab, lens, n, sizes, otab, status):
        return N.lib.vgb_convert_to_wave_batch(ftab, lens, types, n, None, C.byref(adx_key), C.byref(hca_code), sizes, otab, status)

    def sized(call, n, all_ok=True):
        """The sizing pass of `call`, then pinned buffers of those sizes: (buffers, their table, status array)."""
        sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
        N.check(call(sizes, None, status))
        if all_ok:
            assert all(status[i] == 0 for i in range(n)), [status[i] for i in range(n) if status[i]][:4]
        outs = [torch.empty(max(int(sizes[i]), 1), dtype=torch.uint8, pin_memory=True) for i in range(n)]
        return outs, (C.c_void_p * n)(*[o.data_ptr() for o in outs]), sizes, status

    # ---- the jobs: WAVE images ----
    jobs = []
    waves, _ = bench_configs._batch_files(torch, bench, a.files, torch.device("cuda", 0))
    jobs.append(("short", waves, a.check))
    tracks = []
    for i in range(a.tracks):
        n = 180 * 48000
        pcm = [synth.channel(900 + 2 * i + c, n, 48000, degenerate=False) for c in range(2)]
        tracks.append(pinned(O.wave_write16(pcm, 48000, (48000 * 7 + 11, n - 5))))
    jobs.append(("tracks", tracks, a.check_tracks))

    ok_all = True
    for job, waves, n_check in jobs:
        n = len(waves)
        wtab, wlens = tab(waves)
        coded = {}
        for dst in (T.ADX, T.HCA):  # set-up: the job once in both codecs (keyed .adx and .hca, so decryption runs too)
            opt = ct.convert_options(dst, hca_quality=2, hca_key_type=56 if dst == T.HCA else -1, hca_key_code=HCA_KEY,
                                     adx_has_key=int(dst == T.ADX), adx_encryption_type=9 if dst == T.ADX else 0,
                                     adx_key_seed=adx_key.seed, adx_key_mult=adx_key.mult, adx_key_inc=adx_key.inc)
            outs, otab, sizes, status = sized(lambda s, o, st: N.lib.vgb_convert_wave_batch(wtab, wlens, n, C.byref(opt), s, o, st, None, None), n)
            N.check(N.lib.vgb_convert_wave_batch(wtab, wlens, n, C.byref(opt), sizes, otab, status, None, None))
            coded[dst] = [o[: int(sizes[i])].clone().pin_memory() for i, o in enumerate(outs)]
        for src, dst, plus1 in DIRECTIONS:
            ftab, lens = tab(coded[src])
            types = (C.c_int32 * n)(*([src] * n))
            opt = ct.convert_options(dst, nw_codec_plus1=plus1)
            direct = lambda s, o, st: N.lib.vgb_transcode_nw_batch(ftab, lens, types, n, C.byref(opt), C.byref(adx_key), C.byref(hca_code),
                                                                    s, o, st, None, None)
            d_outs, d_tab, d_sizes, d_status = sized(direct, n, all_ok=False)  # HPS may refuse a file whose loop moved
            w_outs, w_tab, w_sizes, w_status = sized(lambda s, o, st: to_wave(types, ftab, lens, n, s, o, st), n)
            N.check(to_wave(types, ftab, lens, n, w_sizes, w_tab, w_status))  # the WAVE images, so the second call can be sized
            wt2 = [w[: int(w_sizes[i])] for i, w in enumerate(w_outs)]
            wtab2, wlens2 = tab(wt2)
            c_outs, c_tab, c_sizes, c_status = sized(
                lambda s, o, st: N.lib.vgb_convert_wave_batch(wtab2, wlens2, n, C.byref(opt), s, o, st, None, None), n, all_ok=False)
            times = {"direct": [], "composition": []}
            for r in range(a.warmup + a.runs):
                for arm in ("direct", "composition"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if arm == "direct":
                        N.check(direct(d_sizes, d_tab, d_status))
                    else:
                        N.check(to_wave(types, ftab, lens, n, w_sizes, w_tab, w_status))
                        N.check(N.lib.vgb_convert_wave_batch(wtab2, wlens2, n, C.byref(opt), c_sizes, c_tab, c_status, None, None))
                    dt = time.perf_counter() - t0
                    if r >= a.warmup:
                        times[arm].append(dt)
            good = [i for i in range(n) if d_status[i] == 0]
            same = all(d_status[i] == c_status[i] for i in range(n)) and all(
                d_sizes[i] == c_sizes[i] and d_outs[i][: int(d_sizes[i])].numpy().tobytes() == c_outs[i][: int(c_sizes[i])].numpy().tobytes()
                for i in good)
            checked = [good[j] for j in sorted(set(np.linspace(0, len(good) - 1, min(n_check, len(good))).astype(int).tolist()))] if n_check > 0 and good else []
            oracle_ok = True
            for i in checked:
                want, _ = W.expected(coded[src][i].numpy(), src, dst, plus1 - 1 if plus1 else W.GCADPCM, adx_key=O.adx_key(key_code=ADX_KEY_CODE),
                                     hca_key=HCA_KEY)
                oracle_ok &= want is not None and d_outs[i][: int(d_sizes[i])].numpy().tobytes() == want.tobytes()
            ok_all &= same and oracle_ok
            row = {"tool": "transcode_nw_bench", "job": job, "direction": f"{NAMES[src]}->{NAMES[dst]}" + ("(pcm16)" if plus1 == 2 else ""),
                   "files": n, "refused": n - len(good),
                   "in_bytes": int(sum(int(t.numel()) for t in coded[src])), "out_bytes": int(sum(int(d_sizes[i]) for i in range(n))),
                   "wave_bytes": int(sum(int(w_sizes[i]) for i in range(n))), "runs": a.runs,
                   "gpu": ident["name"], "power_limit_w": ident["power_limit_w"],
                   "arms_identical": same, "oracle_checked": len(checked), "oracle_identical": oracle_ok}
            for arm, ts in times.items():
                row[f"{arm}_ms"] = {"median": round(statistics.median(ts) * 1e3, 2), "min": round(min(ts) * 1e3, 2), "max": round(max(ts) * 1e3, 2)}
            row["speedup_median"] = round(statistics.median(times["composition"]) / statistics.median(times["direct"]), 3)
            print(json.dumps(row), flush=True)
            del d_outs, w_outs, c_outs
    N.check(N.lib.vgb_shutdown())
    if not ok_all:
        raise SystemExit("transcoded files differ from the composition or from the oracle chain")


if __name__ == "__main__":
    main()
