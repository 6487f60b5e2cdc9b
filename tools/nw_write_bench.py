"""WAVE -> .brstm / .bfstm against WAVE -> .dsp through vgb_convert_wave_batch on one GPU: the fill pass (sizes known,
output buffers allocated and page-locked beforehand) timed per arm, arms alternated in one process, median of 3.  Jobs:
2048 stereo WAVE files of 1-10 s at 32 kHz, and 32 stereo three-minute looping tracks (unaligned loop starts, so every
GC-ADPCM channel takes GcAdpcmAlignment's tail).  Sampled files are checked byte for byte against
tests/nw_writer_oracle.py.  Prints one JSON line with the card's name and power limit.

    python tools/nw_write_bench.py [--files 2048] [--tracks 32] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import vgaudio_b200 as vg  # noqa: E402
from oracle import pyoracle as O  # noqa: E402
from vgaudio_b200 import _native as N  # noqa: E402
from vgaudio_b200 import containers as ct  # noqa: E402

import nw_writer_oracle as W  # noqa: E402


def job_files(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        s = int(rng.integers(32000, 320000))
        pcm = [(rng.normal(0, 3000, s)).astype(np.int16) for _ in range(2)]
        out.append((pcm, 32000, (int(rng.integers(1, s // 2)), s) if i % 2 else None))
    return out


def job_tracks(n, seed):
    rng = np.random.default_rng(seed)
    s = 32000 * 180
    t = np.arange(s)
    return [([(np.sin(t * (0.01 + 0.001 * k + c * 0.0003)) * 8000 + rng.normal(0, 200, s)).astype(np.int16) for c in range(2)],
             32000, (1000 + 977 * k, s - 5)) for k in range(n)]


class Arm:
    def __init__(self, waves, opts):
        self.opts = opts
        self.arrs = [np.ascontiguousarray(w) for w in waves]
        n = len(self.arrs)
        self.ftab = (C.c_void_p * n)(*[a.ctypes.data for a in self.arrs])
        self.lens = (C.c_int64 * n)(*[a.size for a in self.arrs])
        self.sizes = (C.c_int64 * n)()
        self.status = (C.c_int32 * n)()
        N.check(N.lib.vgb_convert_wave_batch(self.ftab, self.lens, n, C.byref(opts), self.sizes, None, self.status, None, None))
        assert all(s == 0 for s in self.status)
        self.outs = [torch.empty(int(self.sizes[i]), dtype=torch.uint8, pin_memory=True) for i in range(n)]
        self.otab = (C.c_void_p * n)(*[o.data_ptr() for o in self.outs])

    def fill(self):
        t0 = time.perf_counter()
        N.check(N.lib.vgb_convert_wave_batch(self.ftab, self.lens, len(self.arrs), C.byref(self.opts), self.sizes, self.otab,
                                             self.status, None, None))
        return (time.perf_counter() - t0) * 1e3

    def file(self, i):
        return self.outs[i].numpy().tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--tracks", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    N.check(vg.lib.vgb_init(0, 0))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    result = {"gpu": gpu, "jobs": {}}
    for name, job in (("files", job_files(a.files, 1)), ("tracks", job_tracks(a.tracks, 2))):
        waves = [O.wave_write16(p, r, l) for p, r, l in job]
        arms = {"dsp": Arm(waves, ct.convert_options(ct.CONTAINER_DSP)),
                "brstm": Arm(waves, ct.convert_options(ct.CONTAINER_BRSTM)),
                "bfstm": Arm(waves, ct.convert_options(ct.CONTAINER_BFSTM))}
        times = {k: [] for k in arms}
        for _ in range(1 + a.reps):  # the first round warms up
            for k, arm in arms.items():
                times[k].append(arm.fill())
        for k, kind in (("brstm", W.BRSTM), ("bfstm", W.BFSTM)):  # sampled byte checks against the oracle
            for i in (0, len(job) // 2, len(job) - 1):
                p, r, l = job[i]
                assert arms[k].file(i) == W.write(kind, W.GCADPCM, p, r, l)[1].tobytes(), f"{name} {k} file {i} differs"
        result["jobs"][name] = {"n": len(job), "wave_gb": round(sum(w.size for w in waves) / 1e9, 3),
                                "fill_ms_median": {k: round(float(np.median(v[1:])), 2) for k, v in times.items()},
                                "fill_ms_all": {k: [round(x, 2) for x in v[1:]] for k, v in times.items()}}
        del arms
    print(json.dumps(result))


if __name__ == "__main__":
    main()
