#!/usr/bin/env python
"""tools/nw_wave_to_wave_bench.py — the fill pass of vgb_convert_nw_to_wave_batch on NintendoWare wave and prefetch
files, against the same audio as .bcstm streams.

  python tools/nw_wave_to_wave_bench.py [--files 8192] [--prefetch 64] [--runs 3] [--warmup 1] [--check 16]

Two jobs, GC-ADPCM encoded by the product itself (vgaudio_b200.gcadpcm.encode_batch) from synth PCM at 32 kHz:
  effects   `files` sound effects of 0.05-2 s, mono and stereo, 3/4 GC-ADPCM and 1/4 PCM16, cycling .bcwav / .bfwav /
            .brwav (tests/nw_wave_files.py) - a sound archive's shape;
  prefetch  `prefetch` stereo GC-ADPCM .bfstp files whose one PDAT region holds 5 s per channel.
Each job also runs as "stream": the same channels wrapped into .bcstm files (tests/nw_files.py, interleave 0x2000; for
the prefetch job, the region's samples).  The only device difference is one gather launch per group for the wave files
in place of one de-interleave launch per stream file.  The two arms alternate, `warmup` + `runs` times each, under a
host clock around the synchronous fill pass; medians, minima and maxima are reported.  `check` files of each arm are
compared with the oracle chain (tests/nw_wave_reader_oracle.py), and the two arms' WAVE files with each other.  One
JSON line per job with the GPU's name and power limit.
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


def _channels(np, NF, synth, gc, specs):
    """specs: (channels, samples, codec, big_endian) -> per file its nw_files.Channel list."""
    base = [synth.channel(900 + c, 32000 * 6, 32000, degenerate=False) for c in range(8)]
    pcm, owner = [], []
    for i, (ch, n, codec, be) in enumerate(specs):
        for c in range(ch):
            src = base[(i + c) % len(base)]
            x = np.roll(np.tile(src, -(-n // src.size))[:n], 7919 * i + 31 * c)
            pcm.append(np.ascontiguousarray(x, np.int16))
            owner.append(i)
    gc_files = {i for i, s in enumerate(specs) if s[2] == NF.GCADPCM}
    rows = [p for p, o in zip(pcm, owner) if o in gc_files]
    coefs, adpcm = gc.encode_batch(rows) if rows else (None, [])
    out, r, j = [], 0, 0
    for i, (ch, n, codec, be) in enumerate(specs):
        mine = pcm[j: j + ch]
        j += ch
        if codec == NF.GCADPCM:
            out.append([NF.Channel(adpcm[r + c].tobytes(), coefs[r + c], 0, (int(adpcm[r + c][0]), 0, 0)) for c in range(ch)])
            r += ch
        else:
            out.append(NF.pcm16_channels(mine, be))
    return out


def _arm(N, imgs, types):
    n = len(imgs)
    ftab = (C.c_void_p * n)(*[h.ctypes.data for h in imgs])
    lens = (C.c_int64 * n)(*[h.size for h in imgs])
    ttab = (C.c_int32 * n)(*types)
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    N.check(N.lib.vgb_convert_nw_to_wave_batch(ftab, lens, ttab, n, sizes, None, status))
    assert all(status[i] == 0 for i in range(n))
    return dict(ftab=ftab, lens=lens, ttab=ttab, n=n, sizes=sizes, status=status, imgs=imgs, types=types)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=8192)
    ap.add_argument("--prefetch", type=int, default=64)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=16)
    a = ap.parse_args()

    import numpy as np
    import torch

    import bench
    import nw_files as NF
    import nw_wave_files as F
    import nw_wave_reader_oracle as R
    from oracle import pyoracle as O
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import gcadpcm, synth

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    O.build()
    N.check(N.lib.vgb_init(0, 0))
    ident = bench.gpu_identity(0, torch)
    rng = np.random.default_rng(2026)
    ok_all = True

    # effects: wave files and the same channels as .bcstm streams
    kinds = (F.BCWAV, F.BFWAV, F.BRWAV)
    specs = []
    for i in range(a.files):
        kind = kinds[i % 3]
        specs.append((1 + i % 2, int(rng.integers(1600, 64001)), NF.GCADPCM if i % 4 < 3 else NF.PCM16, kind != F.BCWAV))
    chans = _channels(np, NF, synth, gcadpcm, specs)
    wave = [F.rwav(s[2], ch, s[1]) if kinds[i % 3] == F.BRWAV else F.cwav(kinds[i % 3], s[2], ch, s[1], big_endian=s[3])
            for i, (s, ch) in enumerate(zip(specs, chans))]
    # the stream arm: BCSTM is little-endian, so PCM16 channels are re-encoded in its byte order
    stream_chans = [ch if s[2] == NF.GCADPCM else [NF.Channel(np.frombuffer(c.data, ">i2" if s[3] else "<i2").astype("<i2").tobytes()) for c in ch]
                    for s, ch in zip(specs, chans)]
    stream = [NF.build(NF.BCSTM, s[2], ch, s[1], seek="none") for s, ch in zip(specs, stream_chans)]
    jobs = [("effects", _arm(N, wave, [kinds[i % 3] for i in range(a.files)]), _arm(N, stream, [NF.BCSTM] * a.files))]

    # prefetch: one 5 s region per stereo file, and the region's samples as a .bcstm stream
    pn = 5 * 32000
    per = NF.gc_bytes(pn)
    pspecs = [(2, pn, NF.GCADPCM, True) for _ in range(a.prefetch)]
    pchans = _channels(np, NF, synth, gcadpcm, pspecs)
    pre = [F.cstp(F.BFSTP, NF.GCADPCM, ch, pn, [per], interleave=0x2000) for ch in pchans]
    samples = R.bytes_to_samples(per, NF.GCADPCM)
    pstream = [NF.build(NF.BCSTM, NF.GCADPCM, ch, samples, seek="none") for ch in pchans]
    jobs.append(("prefetch", _arm(N, pre, [F.BFSTP] * a.prefetch), _arm(N, pstream, [NF.BCSTM] * a.prefetch)))

    for name, file_arm, stream_arm in jobs:
        arms = {"files": file_arm, "stream": stream_arm}
        for arm in arms.values():
            arm["outs"] = [torch.empty(arm["sizes"][i], dtype=torch.uint8).pin_memory() for i in range(arm["n"])]
            arm["otab"] = (C.c_void_p * arm["n"])(*[o.data_ptr() for o in arm["outs"]])
        times = {k: [] for k in arms}
        for r in range(a.warmup + a.runs):
            for k, arm in arms.items():
                t0 = time.perf_counter()
                N.check(N.lib.vgb_convert_nw_to_wave_batch(arm["ftab"], arm["lens"], arm["ttab"], arm["n"], arm["sizes"], arm["otab"], arm["status"]))
                dt = time.perf_counter() - t0
                assert all(arm["status"][i] == 0 for i in range(arm["n"]))
                if r >= a.warmup:
                    times[k].append(dt)
        n = file_arm["n"]
        same = all(file_arm["outs"][i].numpy().tobytes() == stream_arm["outs"][i].numpy().tobytes() for i in range(n))
        checked = sorted(set(np.linspace(0, n - 1, min(a.check, n)).astype(int).tolist()))
        identical = all(arm["outs"][i].numpy().tobytes() == R.expected_wave(arm["imgs"][i], arm["types"][i]).tobytes()
                        for arm in arms.values() for i in checked)
        ok_all &= identical and same
        row = {"tool": "nw_wave_to_wave_bench", "job": name, "files": n, "runs": a.runs, "gpu": ident["name"],
               "power_limit_w": ident["power_limit_w"],
               "input_bytes": {k: int(sum(h.size for h in arm["imgs"])) for k, arm in arms.items()},
               "wave_bytes": int(sum(int(file_arm["sizes"][i]) for i in range(n))),
               "oracle_checked": len(checked), "oracle_identical": identical, "arms_identical": same}
        for k, ts in times.items():
            row[f"{k}_fill_ms"] = {"median": round(statistics.median(ts) * 1e3, 2), "min": round(min(ts) * 1e3, 2), "max": round(max(ts) * 1e3, 2)}
        print(json.dumps(row), flush=True)
    N.check(N.lib.vgb_shutdown())
    if not ok_all:
        raise SystemExit("converted files differ from the oracle chain or between the arms")


if __name__ == "__main__":
    main()
