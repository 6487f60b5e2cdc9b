#!/usr/bin/env python
"""tools/interleave_bench.py — the block (de)interleave kernels, vector-load variant against the TMA bulk-copy variant
(VGB_INTERLEAVE_TMA=1), device resident: 2048 two-channel payloads of 822 864 bytes in 0x2000-byte blocks (the .dsp layout
of a C2-sized batch).  Prints one JSON object; outputs of both variants must be identical."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import vgaudio_b200 as vg  # noqa: E402
from vgaudio_b200 import _native as N  # noqa: E402


def main():
    dev = torch.device("cuda", 0)
    N.check(vg.lib.vgb_init(0, 0))
    items, count, size, ilv = 2048, 2, 822864, 0x2000
    src = torch.randint(0, 256, (items, count, size), dtype=torch.uint8, device=dev)
    out = {k: torch.zeros((items, count * size), dtype=torch.uint8, device=dev) for k in ("vector", "tma")}
    back = {k: torch.zeros((items, count, size), dtype=torch.uint8, device=dev) for k in ("vector", "tma")}
    stream = torch.cuda.current_stream()
    peak = 3350.0  # H100 SXM data sheet, unless MEASURED_PEAKS.json holds a measured copy bandwidth
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    res = {"shape": {"items": items, "channels": count, "bytes_per_channel": size, "block": ilv}, "bytes_moved_per_call": 2 * items * count * size}
    for name in ("vector", "tma"):
        if name == "tma":
            os.environ["VGB_INTERLEAVE_TMA"] = "1"
        else:
            os.environ.pop("VGB_INTERLEAVE_TMA", None)

        def fwd():
            N.check(vg.lib.vgb_interleave_dev(src.data_ptr(), size, count * size, out[name].data_ptr(), count * size, items, count, size, ilv, size,
                                              stream.cuda_stream))

        def bwd():
            N.check(vg.lib.vgb_deinterleave_dev(out[name].data_ptr(), count * size, back[name].data_ptr(), size, count * size, items, count, size,
                                                ilv, size, stream.cuda_stream))

        for fn, key in ((fwd, "interleave"), (bwd, "deinterleave")):
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(10):
                fn()
            e1.record(stream)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            gbs = res["bytes_moved_per_call"] / ms / 1e6
            res[f"{name}_{key}"] = {"ms": round(ms, 4), "GB_per_s": round(gbs, 1), "frac_of_measured_copy_peak": round(gbs / peak, 3)}
    os.environ.pop("VGB_INTERLEAVE_TMA", None)
    res["outputs_identical"] = bool((out["vector"] == out["tma"]).all().item()) and bool((back["vector"] == back["tma"]).all().item()) and \
        bool((back["vector"] == src).all().item())
    print(json.dumps(res, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
