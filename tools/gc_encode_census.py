"""Static instruction census of gc_encode_kernel's frame loop (sm_90a SASS), split by block and by pipe.

    python tools/gc_encode_census.py [vgaudio_b200/csrc/gc_encode.o] [--mode 0|1|2]

Reads `cuobjdump -sass` of gc_encode_kernel<mode> (0 chain, 1 run-on, 2 cascade) and finds the frame loop from its
control flow: the loop head is the target of the backward branch that closes it, round 0 runs from the head to the
round-1 vote's branch (the first predicate VOTE.ANY), round 1 from there to that branch's target, and the tail from the
target to the backward branch.  The `i == 15` block at the loop head (wait for and widen the next chunk, once per 16
frames) is left out.  Opcodes are binned by the pipe that issues them on Hopper: the IMAD family (multiply-add pipe),
the integer ALU (adds, shifts, logic, min/max, compares, selects) and everything else (shared memory, shuffles,
votes, control).
"""
import argparse
import os
import re
import subprocess
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "_ZN3vgb16gc_encode_kernelILi{}EEEvPKsNS_14GcChannelTableES2_PhiiNS_9GcSegArgsE"
LINE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P[0-9T]\s+)?([A-Z0-9_.]+)\s*([^;]*);")
ALU = ("IADD3", "VIADD", "LEA", "SHF", "LOP3", "VIMNMX", "VIMNMX3", "VIADDMNMX", "SEL", "ISETP", "PRMT", "IABS", "FLO", "PLOP3",
       "MOV", "BMSK", "UIADD3", "ULOP3", "USHF", "UMOV", "P2R", "R2P", "VABSDIFF", "IMNMX")


def pipe(op: str) -> str:
    root = op.split(".")[0]
    if root in ("IMAD", "IMUL"):
        return "imad"
    if root in ALU:
        return "alu"
    return "other"


def sass(obj: str, mode: int):
    out = subprocess.run(["cuobjdump", "-sass", "-fun", KERNEL.format(mode), obj], check=True, capture_output=True,
                         text=True).stdout
    return [(int(m.group(1), 16), m.group(3), m.group(4)) for m in LINE.finditer(out)]


def census(ins):
    addr = [a for a, _, _ in ins]
    at = {a: i for i, a in enumerate(addr)}
    vote = next(i for i, (_, op, args) in enumerate(ins) if op == "VOTE.ANY" and args.startswith("P"))
    br0 = next(i for i in range(vote, len(ins)) if ins[i][1] == "BRA")
    tail0 = at[int(ins[br0][2].split(",")[-1].strip(), 16)]
    # the backward branch after the tail that jumps above the vote closes the frame loop
    back = next(i for i in range(tail0, len(ins)) if ins[i][1] == "BRA" and int(ins[i][2].split(",")[-1].strip(), 16) < addr[vote])
    head = at[int(ins[back][2].split(",")[-1].strip(), 16)]
    skip = set()
    first_bssy = next(i for i in range(head, vote) if ins[i][1] == "BSSY")
    if first_bssy - head <= 2:  # the i == 15 block opens the loop body
        end = at[int(ins[first_bssy][2].split(",")[-1].strip(), 16)]
        skip = set(range(first_bssy, end))
    blocks = {"round 0": [i for i in range(head, br0 + 1) if i not in skip],
              "round 1": list(range(br0 + 1, tail0)),
              "tail": list(range(tail0, back + 1))}
    res = {}
    for name, idx in blocks.items():
        ops = [ins[i][1] for i in idx if ins[i][1] != "NOP"]
        by_pipe = Counter(pipe(op) for op in ops)
        res[name] = (len(ops), by_pipe, Counter(ops))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("obj", nargs="?", default=os.path.join(ROOT, "vgaudio_b200", "csrc", "gc_encode.o"))
    ap.add_argument("--mode", type=int, default=0)
    ap.add_argument("--opcodes", action="store_true", help="also list the opcodes of each block")
    args = ap.parse_args()
    for name, (n, by_pipe, ops) in census(sass(args.obj, args.mode)).items():
        wide = sum(c for op, c in ops.items() if op.startswith("IMAD.WIDE"))
        print(f"{name:8s} {n:5d} instructions: IMAD pipe {by_pipe['imad']:4d} (IMAD.WIDE {wide:3d}), "
              f"ALU {by_pipe['alu']:4d}, other {by_pipe['other']:4d}")
        if args.opcodes:
            for op, c in ops.most_common():
                print(f"    {c:5d} {op}")


if __name__ == "__main__":
    main()
