#!/usr/bin/env python
"""tools/gc_relock_census.py — how many frames the GC-ADPCM decoder needs to re-lock from a wrong history pair, on the
CPU with the oracle (tests/gc_relock.py).  The time-parallel decoder's shortest segment (kGcDecMinSegFrames,
common.cuh) is chosen from these numbers: a boundary's run-on costs about this many frames, so a segment should be
longer than nearly all of them.

  python tools/gc_relock_census.py [--channels 96] [--seconds 10] [--every 61] [--cap 8192]

Channel sets, each reported on its own JSON line: vgaudio_b200.synth material (three sines, noise and a full-scale burst
per second, peaks 2000..32767) at 48 kHz, and the reference test suite's 261.63 Hz full-scale sine and its ramp; a start
every `every` full frames, each from (0, 0) - the chain's guess - and from a random pair."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=96)
    ap.add_argument("--seconds", type=int, default=10)
    ap.add_argument("--every", type=int, default=61)
    ap.add_argument("--cap", type=int, default=8192)
    a = ap.parse_args()

    import gc_relock as G
    from oracle import pyoracle as O
    from vgaudio_b200 import synth

    O.build()
    n = 48000 * a.seconds
    sets = {"synth": [synth.channel(100 + i, n, 48000, degenerate=False) for i in range(a.channels)],
            "reference_sine": [synth.reference_sine(n, 261.63, 48000)], "reference_ramp": [synth.reference_ramp(0, n)]}
    for name, chans in sets.items():
        row = G.census(O, chans, every=a.every, cap=a.cap)
        row.update(tool="gc_relock_census", set=name, channels=len(chans), seconds=a.seconds, every=a.every, cap=a.cap)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
