#!/usr/bin/env python
"""bench.py — GC-ADPCM batch encode throughput on H100 (BASELINE.json metric), one JSON line on rank 0.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--channels C] [--seconds S] [--dump-outputs DIR]

A "step" = one pass of the hot path (coefficient analysis + exhaustive encode, GcAdpcmFormat.EncodeFromPcm16's loop)
over one synthetic batch.  Default workload = BASELINE.json configs[1]: 1024 channels x 30 s x 48 kHz PCM16 per GPU
(weak scaling: every rank encodes its own 1024 channels; no data-path collective — the channels are independent).

  value      device-resident: PCM already in HBM, ADPCM left in HBM; CUDA events on the launching stream.
  e2e        the same batch through the host C-ABI call (vgb_gcadpcm_encode_batch) with PINNED HOST buffers:
             H2D of the PCM, kernels, D2H of coefficients + ADPCM all inside the timed region.
  roofline   the dominant kernel (gc_encode_kernel): algorithmic bytes (2 B read + 8/14 B written per sample) over its
             measured launch time, against the measured HBM copy bandwidth in MEASURED_PEAKS.json (else the H100 SXM
             data-sheet figure, named as such).
  cpu_baseline  the CPU oracle port of the reference (oracle/, C, one task per channel on all host cores) on a bounded
             sample of the same batch.
--impl reference times that CPU port alone (the reference itself is C#/.NET and cannot run in this image).
--dump-outputs DIR writes what the last timed step computed (see dump_outputs) as DIR/<name>.npy.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SAMPLE_RATE = 48000
ALG_BYTES_PER_SAMPLE = 2.0 + 8.0 / 14.0  # SURVEY.md §8(d): 2 B PCM read + 8/14 B ADPCM written


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--channels", type=int, default=1024, help="channels per GPU")
    ap.add_argument("--seconds", type=float, default=30.0, help="audio seconds per channel")
    ap.add_argument("--cpu-seconds", type=float, default=15.0, help="target wall time of the CPU baseline sample")
    ap.add_argument("--config", default="c2", choices=["c2", "c3", "c4", "c5", "batch"],
                    help="BASELINE.json configuration: c2 GC-ADPCM encode (default, the headline), c3 GC-ADPCM decode of 8192 channels, "
                         "c4 HCA encode of 512 streams, c5 65 536-file mixed batch with NCCL scatter/gather (strong scaling), "
                         "batch WAVE files -> .dsp/.adx/.hca files through the batch converter (--files, default 2048)")
    ap.add_argument("--files", type=int, default=65536, help="c5: number of files in the whole job")
    ap.add_argument("--c5-chunks", type=int, default=2, help="c5: chunks per rank of the scatter / encode / gather pipeline (1: no overlap; "
                    "2 measured best at 4 GPUs: 115.5 ms against 122.8 with 1 and 118.2 with 4 - a chunk's encode is latency bound, so more, smaller chunks cost more than they hide)")
    ap.add_argument("--out-format", default="dsp", choices=["dsp", "adx", "hca"], help="batch: container to write")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="c2: write the last timed step's coefficients and a seeded sample of its ADPCM rows as DIR/<name>.npy")
    args = ap.parse_args()
    if args.dump_outputs and (args.impl != "ours" or args.config != "c2"):
        ap.error("--dump-outputs is implemented for --impl ours --config c2")
    return args


def env_rank():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))


# ------------------------------------------------------------------------------------------------------------
# synthetic data (same recipe as vgaudio_b200/synth.py, generated on the GPU because the batch is 1.5e9 samples)
# ------------------------------------------------------------------------------------------------------------
def make_batch_gpu(torch, n_channels: int, n: int, rank: int, device, degenerate: bool = True):
    g = torch.Generator(device=device)
    g.manual_seed(0x5647415544494F + 7919 * rank)
    out = torch.empty((n_channels, n), dtype=torch.int16, device=device)
    t = torch.arange(n, device=device, dtype=torch.float32) / SAMPLE_RATE
    peaks = torch.tensor([2000.0, 8000.0, 20000.0, 32767.0], device=device)
    chunk = 64
    for c0 in range(0, n_channels, chunk):
        m = min(chunk, n_channels - c0)
        peak = peaks[torch.randint(0, 4, (m,), generator=g, device=device)]
        w = torch.rand((m, 3), generator=g, device=device) + 0.05
        amps = w / w.sum(1, keepdim=True) * peak[:, None]
        freq = torch.exp(torch.rand((m, 3), generator=g, device=device) * (np.log(12000.0) - np.log(60.0)) + np.log(60.0))
        phase = torch.rand((m, 3), generator=g, device=device) * (2 * np.pi)
        x = torch.zeros((m, n), device=device, dtype=torch.float32)
        for k in range(3):
            x += amps[:, k, None] * torch.sin(2 * np.pi * freq[:, k, None] * t[None, :] + phase[:, k, None])
        x += torch.randn((m, n), generator=g, device=device) * (peak[:, None] * 10 ** (-30 / 20))
        # one 50 ms full-scale burst per second
        burst = int(0.05 * SAMPLE_RATE)
        secs = max(n // SAMPLE_RATE, 1)
        starts = torch.randint(0, max(SAMPLE_RATE - burst, 1), (m, secs), generator=g, device=device)
        idx = torch.arange(n, device=device)
        sec_of = torch.clamp(idx // SAMPLE_RATE, max=secs - 1)
        within = idx[None, :] - (sec_of[None, :] * SAMPLE_RATE + starts[:, sec_of])
        in_burst = (within >= 0) & (within < burst)
        sign = torch.randint(0, 2, (m, n), generator=g, device=device, dtype=torch.int8).bool()
        full = torch.where(sign, torch.tensor(32767.0, device=device), torch.tensor(-32768.0, device=device))
        x = torch.where(in_burst, full, x)
        out[c0:c0 + m] = torch.clamp(torch.round(x), -32768, 32767).to(torch.int16)
        del x, in_burst, sign, full, within
    # degenerate channels (all-zero, Nyquist/4 square) as in the test generator
    if n_channels >= 4 and degenerate:
        out[0].zero_()
        out[1] = torch.where((torch.arange(n, device=device) // 4) % 2 == 0, 32767, -32768).to(torch.int16)
    return out


# ------------------------------------------------------------------------------------------------------------
# clocks sampler
# ------------------------------------------------------------------------------------------------------------
class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.gpu = gpu_index
        self.lines = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100", "-i", str(self.gpu)],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._pump, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        for ln in self.lines:
            f = [s.strip() for s in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def gpu_identity(gpu_index: int, torch) -> dict:
    """The card a number was measured on and its power limit (part of every absolute number)."""
    out = {"name": torch.cuda.get_device_name(gpu_index), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(gpu_index)],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


DUMP_BYTES = 48 << 20  # budget of the sampled ADPCM rows (float32); the whole dump stays under 64 MB


def dump_outputs(out_dir: str, coefs_dev, adpcm_dev, n_bytes: int) -> None:
    """What a caller of vgb_gcadpcm_encode_dev receives, from the last timed step: the coefficient table of every channel
    and the ADPCM bytes of a fixed, seeded sample of whole channel rows (all rows when they fit the budget)."""
    n_ch = coefs_dev.shape[0]
    rows = min(n_ch, max(1, DUMP_BYTES // (4 * max(n_bytes, 1))))
    pick = np.sort(np.random.default_rng(0x5647).choice(n_ch, rows, replace=False))
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "coefs.npy"), coefs_dev.cpu().numpy().astype(np.float32))
    np.save(os.path.join(out_dir, "adpcm_rows.npy"), pick.astype(np.float64))
    np.save(os.path.join(out_dir, "adpcm.npy"), adpcm_dev[pick, :n_bytes].cpu().numpy().astype(np.float32))


# ------------------------------------------------------------------------------------------------------------
# CPU baseline (oracle port of the reference's Parallel.For path)
# ------------------------------------------------------------------------------------------------------------
def cpu_baseline(pcm_host: np.ndarray, target_seconds: float):
    from oracle import pyoracle

    cores = os.cpu_count() or 1
    n_ch, n = pcm_host.shape
    # calibrate on one channel per core, then size the sample to ~target_seconds
    probe = min(n_ch, cores)
    t0 = time.perf_counter()
    _, _, used = pyoracle.encode_batch(pcm_host[:probe], 0)
    dt = time.perf_counter() - t0
    rate = probe * n / dt
    want = int(max(probe, min(n_ch, rate * target_seconds / n)))
    want = max(used, want // used * used)
    want = min(want, n_ch)
    t0 = time.perf_counter()
    coefs, adpcm, used = pyoracle.encode_batch(pcm_host[:want], 0)
    dt = time.perf_counter() - t0
    value = want * n / dt / 1e6
    # one channel on one thread, so the reader can see how far the box's `cores` threads really scale
    t0 = time.perf_counter()
    pyoracle.encode_batch(pcm_host[4:5] if n_ch > 4 else pcm_host[:1], 1)
    one = n / (time.perf_counter() - t0) / 1e6
    return {"value": round(value, 3), "unit": "Msamples/s", "cores": used, "kind": "port", "one_thread_msamples_s": round(one, 3),
            "parallel_speedup": round(value / one, 1) if one > 0 else None,
            "sample": f"{want} of {n_ch} channels x {n} samples ({dt:.1f} s wall), C restatement of the reference "
                      f"(oracle/gcadpcm.c) one task per channel; the C#/.NET reference cannot run in this image"}, coefs, adpcm, want


def main():
    args = parse_args()
    rank, local_rank, world = env_rank()
    n = int(round(args.seconds * SAMPLE_RATE))
    n_ch = args.channels
    workload = f"{n_ch} ch x {args.seconds:g} s x 48 kHz PCM16 -> GC-ADPCM (coefs + encode), per GPU"

    if args.impl == "reference":
        if rank != 0:
            return 0
        # the data generator only: loaded by path so that this process never maps the product library
        import importlib.util

        spec = importlib.util.spec_from_file_location("vgb_synth", os.path.join(ROOT, "vgaudio_b200", "synth.py"))
        synth = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(synth)

        cores = os.cpu_count() or 1
        sample_ch = min(n_ch, max(cores, 8))
        pcm = np.stack([synth.channel(4 + i, n) for i in range(min(sample_ch, 16))])
        pcm = np.concatenate([pcm] * ((sample_ch + len(pcm) - 1) // len(pcm)))[:sample_ch]
        from oracle import pyoracle

        times = []
        used = 1
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            _, _, used = pyoracle.encode_batch(pcm, 0)
            if i >= args.warmup:
                times.append(time.perf_counter() - t0)
        ms = 1e3 * sum(times) / len(times)
        value = sample_ch * n / (ms / 1e3) / 1e6
        line = {
            "impl": "reference", "metric": "GC-ADPCM encode Msamples/sec (batch)", "value": round(value, 3),
            "unit": "Msamples/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": round(ms, 3), "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "int32", "data": "synthetic",
            "config": {"workload": workload, "sample": f"{sample_ch} channels x {n} samples per step"},
            "cpu_baseline": {"value": round(value, 3), "unit": "Msamples/s", "cores": used, "kind": "port",
                             "sample": f"{sample_ch} channels x {n} samples per step; C restatement of the reference "
                                       f"(no .NET toolchain in the image), pthread pool over all host cores"},
            "e2e": {"value": round(value, 3), "unit": "Msamples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        }
        print(json.dumps(line))
        return 0

    import torch
    import torch.distributed as dist

    import vgaudio_b200 as vg
    from vgaudio_b200 import _native as N

    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: vgaudio_b200 has no CPU fallback")
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    N.check(vg.lib.vgb_init(local_rank, 0))

    if args.config != "c2":
        import bench_configs

        ctx = {"torch": torch, "dist": dist, "vg": vg, "N": N, "bench": sys.modules[__name__]}
        line = getattr(bench_configs, "run_" + args.config)(args, (rank, local_rank, world), ctx)
        if rank == 0 and line is not None:
            print(json.dumps(line))
        if world > 1:
            dist.destroy_process_group()
        return 0

    # ---- data + HBM layout -----------------------------------------------------------------------------------
    pcm = make_batch_gpu(torch, n_ch, n, rank, device)
    stride = (n + 7) // 8 * 8
    if stride != n:
        padded = torch.zeros((n_ch, stride), dtype=torch.int16, device=device)
        padded[:, :n] = pcm
        pcm_dev = padded
    else:
        pcm_dev = pcm
    n_bytes = vg.gcadpcm.sample_count_to_byte_count(n)
    a_stride = (n_bytes + 15) // 16 * 16
    adpcm_dev = torch.zeros((n_ch, a_stride), dtype=torch.uint8, device=device)
    coefs_dev = torch.zeros((n_ch, 16), dtype=torch.int16, device=device)
    frames = (n + 13) // 14
    ws_bytes = int(vg.lib.vgb_gcadpcm_workspace_bytes(frames * n_ch, n_ch))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    pcm_off = (np.arange(n_ch, dtype=np.int64) * stride)
    ad_off = (np.arange(n_ch, dtype=np.int64) * a_stride)
    lens = np.full(n_ch, n, dtype=np.int32)
    stream = torch.cuda.current_stream()

    def step_dev():
        N.check(vg.lib.vgb_gcadpcm_encode_dev(pcm_dev.data_ptr(), pcm_off.ctypes.data, lens.ctypes.data, None, n_ch,
                                              None, coefs_dev.data_ptr(), adpcm_dev.data_ptr(), ad_off.ctypes.data,
                                              ws.data_ptr(), ws_bytes, stream.cuda_stream))

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    samples_per_step = n_ch * n
    N.check(vg.lib.vgb_set_kernel_timing(1))
    for _ in range(args.warmup):
        step_dev()
    barrier()

    sampler = ClockSampler(local_rank)
    sampler.start()
    launches0 = vg.lib.vgb_kernel_launch_count()
    kernel_ms = np.zeros(4)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(args.steps):
        step_dev()
        buf = (C.c_float * 4)()
        # reading the per-kernel events synchronises on them; they sit on the same stream, inside the timed region
        N.check(vg.lib.vgb_last_kernel_ms(buf, 4))
        kernel_ms += np.array(list(buf))
    ev1.record(stream)
    torch.cuda.synchronize()
    elapsed_ms = ev0.elapsed_time(ev1)
    st4 = (C.c_uint64 * 4)()
    N.check(vg.lib.vgb_gcadpcm_debug_splice_stats(st4, 4))
    splice = {"segments_per_channel": int(st4[0]), "runon_frames": int(st4[1]), "cascade_frames": int(st4[2]),
              "cascade_boundaries": int(st4[3]),
              "fallback_frames_frac": round((int(st4[1]) + int(st4[2])) / max(n_ch * ((n + 13) // 14), 1), 6)}
    launches = vg.lib.vgb_kernel_launch_count() - launches0
    clocks = sampler.stop()
    if world > 1:
        tmax = torch.tensor([elapsed_ms], device=device, dtype=torch.float64)
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        elapsed_ms = float(tmax.item())
    barrier()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, coefs_dev, adpcm_dev, n_bytes)
    kernel_ms /= args.steps
    ms_per_step = elapsed_ms / args.steps
    value = world * samples_per_step / (ms_per_step / 1e3) / 1e6

    # ---- end-to-end through the host C-ABI call (pinned host buffers, copies inside the timed region) -----------
    e2e = None
    pcm_host = None
    if not args.no_e2e:
        pcm_host_t = torch.empty((n_ch, n), dtype=torch.int16, pin_memory=True)
        pcm_host_t.copy_(pcm)
        adpcm_host_t = torch.empty((n_ch, n_bytes), dtype=torch.uint8, pin_memory=True)
        coefs_host = np.zeros((n_ch, 16), dtype=np.int16)
        pcm_host = pcm_host_t.numpy()
        adpcm_host = adpcm_host_t.numpy()
        in_tab = (C.c_void_p * n_ch)(*[pcm_host_t.data_ptr() + 2 * n * c for c in range(n_ch)])
        out_tab = (C.c_void_p * n_ch)(*[adpcm_host_t.data_ptr() + n_bytes * c for c in range(n_ch)])

        def step_e2e():
            N.check(vg.lib.vgb_gcadpcm_encode_batch(in_tab, lens.ctypes.data, None, None, n_ch, coefs_host.ctypes.data,
                                                    out_tab, None, None))

        e2e_steps = args.steps
        step_e2e()  # warm-up (allocates the library's own device buffers)
        barrier()
        t0 = time.perf_counter()
        for _ in range(e2e_steps):
            step_e2e()
        torch.cuda.synchronize()
        e2e_ms = (time.perf_counter() - t0) * 1e3 / e2e_steps
        if world > 1:
            tmax = torch.tensor([e2e_ms], device=device, dtype=torch.float64)
            dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
            e2e_ms = float(tmax.item())
        tl = (C.c_float * 48)()
        N.check(vg.lib.vgb_debug_last_timeline(tl, 48))
        tc = (C.c_float * 16)()
        N.check(vg.lib.vgb_debug_last_coefs_done(tc, 16))
        e2e = {"value": round(world * samples_per_step / (e2e_ms / 1e3) / 1e6, 3), "unit": "Msamples/s",
               "timeline_ms": {"note": "ms since the first copy was enqueued, per channel group: [H2D landed, kernels done, D2H done]; the copy of group g+1 runs under the kernels of group g",
                               "groups": [[round(tl[3 * g + k], 1) for k in range(3)] for g in range(16) if tl[3 * g] >= 0],
                               "coefs_done": [round(tc[g], 1) for g in range(16) if tl[3 * g] >= 0]},
               "h2d_bytes_per_step": int(n_ch * n * 2), "d2h_bytes_per_step": int(n_ch * n_bytes + n_ch * 32),
               "ms_per_step": round(e2e_ms, 3), "steps": e2e_steps,
               "api": "vgb_gcadpcm_encode_batch (host pointers, pinned), wall clock around the synchronous call"}
        # cross-check: device-resident and host paths produced the same bytes
        same = bool((adpcm_dev[:, :n_bytes].cpu() == adpcm_host_t).all().item()) and \
            bool((coefs_dev.cpu().numpy() == coefs_host).all())
        e2e["matches_device_resident"] = same

    # ---- CPU baseline + parity spot check (rank 0) -------------------------------------------------------------
    cpu = None
    parity = None
    if rank == 0 and not args.no_cpu:
        if pcm_host is None:
            pcm_host = pcm.cpu().numpy()
        cpu, o_coefs, o_adpcm, want = cpu_baseline(pcm_host, args.cpu_seconds)
        g_coefs = coefs_dev[:want].cpu().numpy()
        g_adpcm = adpcm_dev[:want, :n_bytes].cpu().numpy()
        parity = {"channels_checked": int(want), "coefs_equal": bool((g_coefs == o_coefs).all()),
                  "adpcm_bytes_equal": bool((g_adpcm == o_adpcm).all())}

    if rank == 0:
        gpu = gpu_identity(local_rank, torch)
        peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
        if os.path.exists(peaks_path):
            peak = float(json.load(open(peaks_path))["hbm_gbs"]); peak_src = "measured (MEASURED_PEAKS.json hbm_gbs, burst copy)"
        else:
            peak = 3350.0; peak_src = "H100 SXM data sheet (3.35 TB/s), not measured"
        enc_ms = float(kernel_ms[2])
        achieved = samples_per_step * ALG_BYTES_PER_SAMPLE / (enc_ms / 1e3) / 1e9 if enc_ms > 0 else None
        line = {
            "metric": "GC-ADPCM encode Msamples/sec (batch)", "value": round(value, 3), "unit": "Msamples/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(ms_per_step, 3),
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "int32", "data": "synthetic",
            "config": {"workload": workload, "global_channels": world * n_ch, "samples_per_channel": n,
                       "l2": "inputs (2.9 GB/GPU) larger than L2, no flush needed", "parallelism": f"dp{world} (channels sharded)"},
            "e2e": e2e,
            "gpu_launches": int(launches),
            "gpu": gpu,
            "clocks": clocks,
            "roofline": {"bound": "hbm", "kernel": "gc_encode_kernel", "achieved": round(achieved, 2) if achieved else None,
                         "peak": peak, "unit": "GB/s", "frac": round(achieved / peak, 5) if achieved else None,
                         "peak_source": peak_src,
                         "algorithmic_bytes_per_launch": int(samples_per_step * ALG_BYTES_PER_SAMPLE),
                         "note": "instruction-issue bound (exhaustive 8-predictor x scale search), not HBM (DESIGN.md 5.3)"},
            "kernel_ms": {"gc_coef_frames": round(float(kernel_ms[0]), 3), "gc_coef_refine": round(float(kernel_ms[1]), 3),
                          "gc_encode": round(float(kernel_ms[2]), 3)},
            "time_parallel": splice,
            "cpu_baseline": cpu,
            "parity": parity,
        }
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
