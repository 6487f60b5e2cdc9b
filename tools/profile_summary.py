"""Turn raw ncu artefacts (a launch list, a kernel capture) into short summaries.

  python tools/profile_summary.py launches <launches.csv> <out.md> "<command line that was profiled>"
  python tools/profile_summary.py kernel   <capture.ncu-rep> <out.json> <kernel name> "<workload>" <frames>

`launches` reads the CSV written by `ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file ...` and
groups the library's own kernels (namespace vgb::) by name.  `kernel` reads one `ncu --set full` capture through
`ncu -i ... --page raw --csv` and keeps the numbers bench.py's roofline object and DESIGN.md quote.
"""
import csv
import io
import json
import subprocess
import sys
from collections import OrderedDict


def launches(path, out_md, command):
    rows = []
    with open(path) as f:
        lines = [ln for ln in f if ln.startswith('"')]
    for r in csv.DictReader(io.StringIO("".join(lines))):
        if r["Metric Name"] != "gpu__time_duration.sum":
            continue
        v = float(r["Metric Value"].replace(",", ""))
        unit = r["Metric Unit"]
        ms = v / 1e6 if unit in ("ns", "nsecond") else v / 1e3 if unit in ("us", "usecond") else v if unit in ("ms", "msecond") else v * 1e3
        rows.append((r["Kernel Name"], ms, r["Grid Size"]))
    ours = OrderedDict()
    other = 0.0
    for name, ms, grid in rows:
        head = name.replace("<unnamed>::", "").replace("(anonymous namespace)::", "").split("(")[0]
        if head.startswith("void "):  # templated kernels are printed with their return type
            head = head[5:]
        if "vgb::" in head or head.startswith(("gc_", "adx_", "hca_", "wave_", "dsp_", "interleave", "deinterleave")):
            short = head.split("vgb::")[1] if "vgb::" in head else head  # keep the template argument: <0> chain, <1> run-on, <2> cascade
            ours.setdefault((short, grid), []).append(ms)
        else:
            other += ms
    total = sum(sum(v) for v in ours.values())
    with open(out_md, "w") as f:
        f.write(f"# ncu launch list of `{command}`\n\n")
        f.write("`ncu --metrics gpu__time_duration.sum --clock-control none` (cold-cache, serialised: compare SHARES, not "
                "absolute times). Library kernels only; torch data-generation kernels "
                f"({other:.1f} ms in total) omitted.\n\n")
        f.write("| kernel | grid | launches | total ms | ms / launch | share of library GPU time |\n|---|---|---|---|---|---|\n")
        for (k, g), v in sorted(ours.items(), key=lambda kv: -sum(kv[1])):
            f.write(f"| `{k}` | {g} | {len(v)} | {sum(v):.3f} | {sum(v) / len(v):.3f} | {100 * sum(v) / total:.1f} % |\n")
    print(open(out_md).read())


def kernel(rep, out_json, name, workload, frames):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rd = list(csv.reader(io.StringIO(raw)))
    header, units, vals = rd[0], rd[1], rd[2]
    m = {h: (u, v) for h, u, v in zip(header, units, vals)}

    def num(key):
        u, v = m[key]
        x = float(v.replace(",", ""))
        scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "ms": 1.0, "msecond": 1.0, "us": 1e-3, "usecond": 1e-3,
                 "ns": 1e-6, "nsecond": 1e-6, "s": 1e3, "second": 1e3}.get(u, 1.0)
        return x * scale

    rd_b, wr_b = num("dram__bytes_read.sum"), num("dram__bytes_write.sum")
    inst = num("smsp__inst_executed.sum")
    out = {
        "kernel": name, "workload": workload,
        "source": f"ncu --set full --clock-control none, 1 launch ({rep})",
        "gpu__time_duration_ms": num("gpu__time_duration.sum"),
        "dram_bytes_read": rd_b, "dram_bytes_write": wr_b, "dram_bytes_total": rd_b + wr_b,
        "dram_throughput_pct_of_peak": num("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
        "warp_instructions": inst, "warp_instructions_per_frame": inst / float(frames) if float(frames) else None,
        "issue_active_pct": num("smsp__issue_active.avg.pct_of_peak_sustained_active"),
        "warps_per_smsp": num("smsp__warps_active.avg.per_cycle_active"),
        "registers_per_thread": int(num("launch__registers_per_thread")),
        "grid": int(num("launch__grid_size")), "block": int(num("launch__block_size")),
    }
    json.dump(out, open(out_json, "w"), indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    if sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3], sys.argv[4])
    else:
        kernel(*sys.argv[2:7])
