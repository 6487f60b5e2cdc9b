"""WAVE -> .idsp / .hps against WAVE -> .dsp and .bfstm through vgb_convert_wave_batch on one GPU: the fill pass (sizes
known, output buffers allocated and page-locked beforehand) timed per arm, arms alternated in one process, median of 3.
The jobs of tools/nw_write_bench.py: 2048 stereo WAVE files of 1-10 s at 32 kHz, and 32 stereo three-minute looping
tracks with unaligned loop starts.  HPS refuses the files whose moved loop makes HpsWriter read a block's history past
the first decode; "refused" counts them per arm.  Sampled files are checked byte for byte against
tests/gc_container_writer_oracle.py.  Prints one JSON line with the card's name and power limit.

    python tools/idsp_hps_write_bench.py [--files 2048] [--tracks 32] [--reps 3]
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

import gc_container_writer_oracle as W  # noqa: E402
from nw_write_bench import job_files, job_tracks  # noqa: E402


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
        self.refused = sum(1 for s in self.status if s != 0)
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
                "idsp": Arm(waves, ct.convert_options(ct.CONTAINER_IDSP)),
                "hps": Arm(waves, ct.convert_options(ct.CONTAINER_HPS)),
                "bfstm": Arm(waves, ct.convert_options(ct.CONTAINER_BFSTM))}
        times = {k: [] for k in arms}
        for _ in range(1 + a.reps):  # the first round warms up
            for k, arm in arms.items():
                times[k].append(arm.fill())
        checked = 0
        for k, write in (("idsp", W.write_idsp), ("hps", W.write_hps)):  # sampled byte checks against the oracle
            for i in (0, 1, len(job) // 2, len(job) - 1):
                p, r, l = job[i]
                st, want = write(p, r, l)
                assert st == arms[k].status[i], f"{name} {k} file {i}: status {arms[k].status[i]}, oracle {st}"
                if st == 0:
                    assert arms[k].file(i) == want.tobytes(), f"{name} {k} file {i} differs"
                    checked += 1
        result["jobs"][name] = {"n": len(job), "wave_gb": round(sum(w.size for w in waves) / 1e9, 3),
                                "fill_ms_median": {k: round(float(np.median(v[1:])), 2) for k, v in times.items()},
                                "fill_ms_all": {k: [round(x, 2) for x in v[1:]] for k, v in times.items()},
                                "refused": {k: arm.refused for k, arm in arms.items()}, "oracle_checked_files": checked}
        del arms
    print(json.dumps(result))


if __name__ == "__main__":
    main()
