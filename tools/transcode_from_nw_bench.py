#!/usr/bin/env python
"""tools/transcode_from_nw_bench.py — the fill pass of vgb_transcode_from_nw_batch against the two-call composition
through WAVE.

  python tools/transcode_from_nw_bench.py [--files 2048] [--tracks 32] [--runs 3] [--warmup 1] [--check 3] [--check-tracks 0]

Two jobs of WAVE images: `short`, the 2048-file job of `bench.py --config batch` (mono / stereo, 1-6 s at 48 kHz, every
eighth file looping), and `tracks`, `tracks` stereo files of 3 minutes at 48 kHz, looping.  As set-up each job is written
once as GC-ADPCM .brstm, .bfstm, .idsp and .hps and as PCM16 .bcstm by vgb_convert_wave_batch (a file the HPS writer
refuses is left out of the .hps job), and as PCM16 .bfwav by the test builder (tests/nw_wave_files.py).  Then for each
direction, alternating, `warmup` + `runs` times each under a host clock (both calls return after their last copy has
landed; every buffer is pinned, and the sizing passes, host-only, are outside the timed region):
  direct       one vgb_transcode_from_nw_batch fill pass, source images in, target images out;
  composition  vgb_convert_to_wave_batch's fill pass, then vgb_convert_wave_batch's fill pass on those WAVE images.
Both arms must give identical bytes and statuses, and `check` files of each direction (`check-tracks` of the tracks) are
compared with the oracle chain (tests/transcode_from_nw_oracle.py).  One JSON line per job and direction, with the GPU's
name and power limit.
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

NAMES = {1: "dsp", 2: "adx", 3: "hca", 4: "brstm", 5: "bcstm", 6: "bfstm", 7: "idsp", 8: "hps", 11: "bfwav"}
# the sources, each from the WAVE job: (in_type, nw_codec_plus1 of the set-up write; 11 is built on the host)
SOURCES = [(4, 0), (6, 0), (7, 0), (8, 0), (5, 2), (11, 2)]
# (source, target, nw_codec_plus1 of the target)
DIRECTIONS = [(4, 2, 0), (6, 3, 0), (7, 2, 0), (8, 3, 0), (5, 1, 0), (5, 4, 0), (6, 5, 2), (11, 3, 0)]


def _name(in_type, plus1):
    return NAMES[in_type] + ("(pcm16)" if plus1 == 2 else "(pcm8)" if plus1 == 1 else "")


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
    import nw_files as NF
    import nw_wave_files as NWF
    import transcode_from_nw_oracle as X
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct
    from vgaudio_b200 import synth

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    O.build()
    N.check(N.lib.vgb_init(0, 0))
    ident = bench.gpu_identity(0, torch)

    def pinned(arr):
        t = torch.empty(int(arr.size), dtype=torch.uint8, pin_memory=True)
        t.numpy()[:] = arr
        return t

    def tab(ts):
        return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts]), (C.c_int64 * len(ts))(*[int(t.numel()) for t in ts])

    def to_wave(types, ftab, lens, n, sizes, otab, status):
        return N.lib.vgb_convert_to_wave_batch(ftab, lens, types, n, None, None, None, sizes, otab, status)

    def sized(call, n, all_ok=True):
        """The sizing pass of `call`, then pinned buffers of those sizes: (buffers, their table, sizes, status array)."""
        sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
        N.check(call(sizes, None, status))
        if all_ok:
            assert all(status[i] == 0 for i in range(n)), [status[i] for i in range(n) if status[i]][:4]
        outs = [torch.empty(max(int(sizes[i]), 1), dtype=torch.uint8, pin_memory=True) for i in range(n)]
        return outs, (C.c_void_p * n)(*[o.data_ptr() for o in outs]), sizes, status

    def bfwav(rows, n, rate):
        chans = NF.pcm16_channels([np.asarray(r, np.int16) for r in rows], True)
        return NWF.cwav(NWF.BFWAV, X.PCM16, chans, n, rate=rate, big_endian=True,
                        offsets=NWF.layout("ordered", [NWF.samples_to_bytes(n, X.PCM16)] * len(rows)))

    # ---- the jobs: WAVE images, and the PCM16 .bfwav images of the same audio ----
    jobs = []
    waves, meta = bench_configs._batch_files(torch, bench, a.files, torch.device("cuda", 0))
    jobs.append(("short", waves, [pinned(bfwav(rows, n, 48000)) for rows, n, _ in meta], a.check))
    tracks, tracks_wav = [], []
    for i in range(a.tracks):
        n = 180 * 48000
        pcm = [synth.channel(900 + 2 * i + c, n, 48000, degenerate=False) for c in range(2)]
        tracks.append(pinned(O.wave_write16(pcm, 48000, (48000 * 7 + 11, n - 5))))
        tracks_wav.append(pinned(bfwav(pcm, n, 48000)))
    jobs.append(("tracks", tracks, tracks_wav, a.check_tracks))

    ok_all = True
    for job, waves, bfwavs, n_check in jobs:
        n = len(waves)
        wtab, wlens = tab(waves)
        srcs = {11: bfwavs}
        for in_type, plus1 in SOURCES:  # set-up: the job once in every source container
            if in_type == 11:
                continue
            opt = ct.convert_options(in_type, nw_codec_plus1=plus1)
            outs, otab, sizes, status = sized(lambda s, o, st: N.lib.vgb_convert_wave_batch(wtab, wlens, n, C.byref(opt), s, o, st, None, None), n,
                                              all_ok=in_type != 8)
            N.check(N.lib.vgb_convert_wave_batch(wtab, wlens, n, C.byref(opt), sizes, otab, status, None, None))
            srcs[in_type] = [o[: int(sizes[i])].clone().pin_memory() for i, o in enumerate(outs) if status[i] == 0]
        for src, dst, plus1 in DIRECTIONS:
            files = srcs[src]
            m = len(files)
            ftab, lens = tab(files)
            types = (C.c_int32 * m)(*([src] * m))
            opt = ct.convert_options(dst, nw_codec_plus1=plus1, hca_quality=2)
            direct = lambda s, o, st: N.lib.vgb_transcode_from_nw_batch(ftab, lens, types, m, C.byref(opt), s, o, st, None, None)
            d_outs, d_tab, d_sizes, d_status = sized(direct, m, all_ok=False)
            w_outs, w_tab, w_sizes, w_status = sized(lambda s, o, st: to_wave(types, ftab, lens, m, s, o, st), m)
            N.check(to_wave(types, ftab, lens, m, w_sizes, w_tab, w_status))  # the WAVE images, so the second call can be sized
            wt2 = [w[: int(w_sizes[i])] for i, w in enumerate(w_outs)]
            wtab2, wlens2 = tab(wt2)
            c_outs, c_tab, c_sizes, c_status = sized(
                lambda s, o, st: N.lib.vgb_convert_wave_batch(wtab2, wlens2, m, C.byref(opt), s, o, st, None, None), m, all_ok=False)
            times = {"direct": [], "composition": []}
            for r in range(a.warmup + a.runs):
                for arm in ("direct", "composition"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if arm == "direct":
                        N.check(direct(d_sizes, d_tab, d_status))
                    else:
                        N.check(to_wave(types, ftab, lens, m, w_sizes, w_tab, w_status))
                        N.check(N.lib.vgb_convert_wave_batch(wtab2, wlens2, m, C.byref(opt), c_sizes, c_tab, c_status, None, None))
                    dt = time.perf_counter() - t0
                    if r >= a.warmup:
                        times[arm].append(dt)
            good = [i for i in range(m) if d_status[i] == 0]
            same = all(d_status[i] == c_status[i] for i in range(m)) and all(
                d_sizes[i] == c_sizes[i] and d_outs[i][: int(d_sizes[i])].numpy().tobytes() == c_outs[i][: int(c_sizes[i])].numpy().tobytes()
                for i in good)
            checked = [good[j] for j in sorted(set(np.linspace(0, len(good) - 1, min(n_check, len(good))).astype(int).tolist()))] if n_check > 0 and good else []
            oracle_ok = True
            for i in checked:
                want, _ = X.expected(files[i].numpy(), src, dst, plus1 - 1 if plus1 else X.GCADPCM)
                oracle_ok &= want is not None and d_outs[i][: int(d_sizes[i])].numpy().tobytes() == want.tobytes()
            ok_all &= same and oracle_ok
            row = {"tool": "transcode_from_nw_bench", "job": job,
                   "direction": f"{_name(src, dict(SOURCES)[src])}->{_name(dst, plus1)}", "files": m, "refused": m - len(good),
                   "looping": sum(1 for i in range(m) if b"smpl" in wt2[i][:64].numpy().tobytes()),
                   "in_bytes": int(sum(int(t.numel()) for t in files)), "out_bytes": int(sum(int(d_sizes[i]) for i in range(m))),
                   "wave_bytes": int(sum(int(w_sizes[i]) for i in range(m))), "runs": a.runs,
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
