"""bench.py --config c3 | c4 | c5: the other BASELINE.json configurations, each at full size with distinct synthetic
channels, a bit-exact spot check against the CPU oracle inside the run, `roofline`, `cpu_baseline` and `e2e` objects.

  c3  8192-channel GC-ADPCM decode (.dsp payloads -> PCM16) on one H100, bit-exact check       (BASELINE configs[2])
  c4  512-stream CRI HCA encode (128-point MDCT, quality High, mono 48 kHz) on one H100          (BASELINE configs[3])
  c5  65 536-file mixed GC-ADPCM + ADX batch encode, STRONG scaling over N GPUs: the root rank holds the PCM in HBM,
      one NCCL scatterv hands every rank its files, every rank encodes, one NCCL gatherv returns the bitstreams
      (BASELINE configs[4]; launched under torchrun for N > 1)

Timing rules as in bench.py: CUDA events on the launching stream, W warm-up steps, max over ranks, inputs far larger than
L2.  The oracle (oracle/) is used as the checker and as the CPU baseline only.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

SAMPLE_RATE = 48000
ROOT = os.path.dirname(os.path.abspath(__file__))


def _peak():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        return float(json.load(open(path))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs, burst copy)"
    return 3350.0, "H100 SXM data sheet (3.35 TB/s), not measured"


def _barrier(torch, dist, world):
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()


def _max_over_ranks(torch, dist, world, device, value):
    if world == 1:
        return float(value)
    t = torch.tensor([value], device=device, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def _base_line(metric, value, world, args, ms, scaling, dtype, config):
    return {"metric": metric, "value": round(value, 3), "unit": "Msamples/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": round(ms, 3), "higher_is_better": True, "scaling": scaling,
            "vs_baseline": None, "dtype": dtype, "data": "synthetic", "config": config}


# ======================================================================================================================
# c3: GC-ADPCM decode
# ======================================================================================================================
def run_c3(args, env, ctx):
    torch, dist, vg, N, bench = ctx["torch"], ctx["dist"], ctx["vg"], ctx["N"], ctx["bench"]
    rank, local_rank, world = env
    device = torch.device("cuda", local_rank)
    n_ch = args.channels if args.channels != 1024 else 8192
    n = int(round(args.seconds * SAMPLE_RATE))
    stream = torch.cuda.current_stream()
    stride = (n + 7) // 8 * 8
    n_bytes = vg.gcadpcm.sample_count_to_byte_count(n)
    a_stride = (n_bytes + 15) // 16 * 16
    frames = (n + 13) // 14

    # ---- the input of the decoder = the encoder's output for n_ch DISTINCT synthetic channels (encoded 1024 at a time)
    adpcm = torch.zeros((n_ch, a_stride), dtype=torch.uint8, device=device)
    coefs = torch.zeros((n_ch, 16), dtype=torch.int16, device=device)
    chunk = min(1024, n_ch)
    ws_bytes = int(vg.lib.vgb_gcadpcm_workspace_bytes(frames * chunk, chunk))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    lens_c = np.full(chunk, n, dtype=np.int32)
    keep_pcm = []  # the first 512 channels' PCM stays for the round-trip property
    for c0 in range(0, n_ch, chunk):
        m = min(chunk, n_ch - c0)
        pcm = bench.make_batch_gpu(torch, m, n, rank * 64 + c0 // chunk, device, degenerate=(c0 == 0))
        pad = torch.zeros((m, stride), dtype=torch.int16, device=device)
        pad[:, :n] = pcm
        off_p = np.arange(m, dtype=np.int64) * stride
        off_a = (np.arange(m, dtype=np.int64) + c0) * a_stride
        N.check(vg.lib.vgb_gcadpcm_encode_dev(pad.data_ptr(), off_p.ctypes.data, lens_c.ctypes.data, None, m, None,
                                              coefs[c0:].data_ptr(), adpcm.data_ptr(), off_a.ctypes.data, ws.data_ptr(), ws_bytes,
                                              stream.cuda_stream))
        torch.cuda.synchronize()
        if c0 == 0:
            keep_pcm = pcm[:512].clone()
        del pcm, pad
    del ws
    pcm_out = torch.zeros((n_ch, stride), dtype=torch.int16, device=device)
    dws_bytes = int(vg.lib.vgb_gcadpcm_workspace_bytes(32, n_ch))
    dws = torch.empty(dws_bytes, dtype=torch.uint8, device=device)
    off_a = np.arange(n_ch, dtype=np.int64) * a_stride
    off_p = np.arange(n_ch, dtype=np.int64) * stride
    params = (N.VgbGcParams * n_ch)()
    for c in range(n_ch):
        params[c].sample_count, params[c].history1, params[c].history2 = n, 0, 0

    def step():
        N.check(vg.lib.vgb_gcadpcm_decode_dev(adpcm.data_ptr(), off_a.ctypes.data, coefs.data_ptr(), params, n_ch, pcm_out.data_ptr(),
                                              off_p.ctypes.data, dws.data_ptr(), dws_bytes, stream.cuda_stream))

    N.check(vg.lib.vgb_set_kernel_timing(1))
    for _ in range(args.warmup):
        step()
    _barrier(torch, dist, world)
    sampler = bench.ClockSampler(local_rank)
    sampler.start()
    launches0 = vg.lib.vgb_kernel_launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kms = 0.0
    ev0.record(stream)
    for _ in range(args.steps):
        step()
        buf = (C.c_float * 4)()
        N.check(vg.lib.vgb_last_kernel_ms(buf, 4))
        kms += buf[3]
    ev1.record(stream)
    torch.cuda.synchronize()
    ms = _max_over_ranks(torch, dist, world, device, ev0.elapsed_time(ev1) / args.steps)
    launches = vg.lib.vgb_kernel_launch_count() - launches0
    clocks = sampler.stop()
    kms /= args.steps
    samples = n_ch * n
    value = world * samples / (ms / 1e3) / 1e6

    # ---- e2e: host API with pinned buffers, 2048 channels per call (SURVEY §8d: chunk when host RAM is short)
    e2e = None
    if not args.no_e2e:
        per = min(2048, n_ch)
        h_in = torch.empty((per, n_bytes), dtype=torch.uint8, pin_memory=True)
        h_out = torch.empty((per, n), dtype=torch.int16, pin_memory=True)
        h_coefs = np.zeros((per, 16), dtype=np.int16)
        in_tab = (C.c_void_p * per)(*[h_in.data_ptr() + n_bytes * c for c in range(per)])
        out_tab = (C.c_void_p * per)(*[h_out.data_ptr() + 2 * n * c for c in range(per)])
        nb = np.full(per, n_bytes, dtype=np.int32)
        pr = (N.VgbGcParams * per)()
        for c in range(per):
            pr[c].sample_count, pr[c].history1, pr[c].history2 = n, 0, 0
        total_ms, same = 0.0, True
        for rep in range(2):  # first pass warms the library's slabs
            total_ms = 0.0
            for c0 in range(0, n_ch, per):
                h_in.copy_(adpcm[c0:c0 + per, :n_bytes])
                h_coefs[:] = coefs[c0:c0 + per].cpu().numpy()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                N.check(vg.lib.vgb_gcadpcm_decode_batch(in_tab, nb.ctypes.data, h_coefs.ctypes.data, pr, per, out_tab))
                total_ms += (time.perf_counter() - t0) * 1e3
                if rep == 1 and c0 == 0:
                    same = bool((h_out[:64].to(device) == pcm_out[:64, :n]).all().item())
        total_ms = _max_over_ranks(torch, dist, world, device, total_ms)
        tl = (C.c_float * 48)()
        N.check(vg.lib.vgb_debug_last_timeline(tl, 48))
        h2d, d2h = n_ch * (n_bytes + 32), n_ch * n * 2
        e2e = {"value": round(world * samples / (total_ms / 1e3) / 1e6, 3), "unit": "Msamples/s", "ms_per_step": round(total_ms, 3),
               "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h),
               "pcie_floor_ms": round(d2h / 55e9 * 1e3, 1),
               "api": f"vgb_gcadpcm_decode_batch, pinned host buffers, {n_ch // per} calls of {per} channels",
               "timeline_ms_last_call": [[round(tl[3 * g + k], 1) for k in range(3)] for g in range(16) if tl[3 * g] >= 0],
               "matches_device_resident": same}

    # ---- parity: >= 512 channels decoded by the oracle from the same bytes, bit-exact; round trip against the input
    parity = cpu = None
    if rank == 0 and not args.no_cpu:
        from oracle import pyoracle

        k = min(512, n_ch)
        a_host = adpcm[:k, :n_bytes].cpu().numpy()
        c_host = coefs[:k].cpu().numpy()
        t0 = time.perf_counter()
        o_dec, used = pyoracle.decode_batch(a_host, c_host, n)
        dt = time.perf_counter() - t0
        g_dec = pcm_out[:k, :n].cpu().numpy()
        err = np.abs(g_dec[:min(k, len(keep_pcm))].astype(np.int32) - keep_pcm[:k].cpu().numpy().astype(np.int32))
        parity = {"channels_checked": int(k), "pcm_equal_oracle": bool(np.array_equal(g_dec, o_dec)),
                  "round_trip_rms_lsb": round(float(np.sqrt((err.astype(np.float64) ** 2).mean())), 2)}
        # CPU baseline: the same oracle decode over all host cores on a bounded sample, timed again warm
        t0 = time.perf_counter()
        pyoracle.decode_batch(a_host, c_host, n)
        dt = min(dt, time.perf_counter() - t0)
        cpu = {"value": round(k * n / dt / 1e6, 3), "unit": "Msamples/s", "cores": int(used), "kind": "port",
               "sample": f"{k} of {n_ch} channels x {n} samples ({dt:.2f} s wall), C restatement of GcAdpcmDecoder.Decode, one task per channel"}

    if rank != 0:
        return None
    peak, peak_src = _peak()
    alg = samples * (2.0 + 8.0 / 14.0)
    achieved = alg / (kms / 1e3) / 1e9 if kms > 0 else None
    line = _base_line("GC-ADPCM decode Msamples/sec (batch)", value, world, args, ms, "weak", "int32",
                      {"workload": f"{n_ch} ch x {args.seconds:g} s x 48 kHz GC-ADPCM (.dsp payload) -> PCM16, per GPU",
                       "global_channels": world * n_ch, "samples_per_channel": n, "distinct_channels": True,
                       "l2": "inputs + outputs (30 GB/GPU) larger than L2, no flush needed", "parallelism": f"dp{world} (channels sharded)"})
    line.update({"e2e": e2e, "gpu_launches": int(launches), "clocks": clocks,
                 "roofline": {"bound": "hbm", "kernel": "gc_decode_kernel", "achieved": round(achieved, 2) if achieved else None, "peak": peak,
                              "unit": "GB/s", "frac": round(achieved / peak, 5) if achieved else None, "traffic": None, "peak_source": peak_src,
                              "algorithmic_bytes_per_launch": int(alg), "note": "8/14 B read + 2 B written per sample; one thread per channel, chain latency bound below ~30k channels"},
                 "kernel_ms": {"gc_decode": round(kms, 3)}, "cpu_baseline": cpu, "parity": parity})
    return line


# ======================================================================================================================
# c4: CRI HCA encode
# ======================================================================================================================
def run_c4(args, env, ctx):
    torch, dist, vg, N, bench = ctx["torch"], ctx["dist"], ctx["vg"], ctx["N"], ctx["bench"]
    rank, local_rank, world = env
    device = torch.device("cuda", local_rank)
    n_st = args.channels if args.channels != 1024 else 512
    n = int(round(args.seconds * SAMPLE_RATE))
    stream = torch.cuda.current_stream()
    stride = (n + 7) // 8 * 8
    pcm = bench.make_batch_gpu(torch, n_st, n, rank, device, degenerate=False)
    pcm_dev = torch.zeros((n_st, stride), dtype=torch.int16, device=device)
    pcm_dev[:, :n] = pcm
    params = (N.VgbHcaParams * n_st)()
    for s in range(n_st):
        params[s] = N.VgbHcaParams(2, 0, 0, 1, SAMPLE_RATE, n, 0, 0, 0)  # quality High, mono
    info0 = N.VgbHcaInfo()
    N.check(vg.lib.vgb_hca_query(C.byref(params[0]), C.byref(info0)))
    fbytes = info0.frame_count * info0.frame_size
    f_stride = (fbytes + 15) // 16 * 16
    frames_dev = torch.zeros((n_st, f_stride), dtype=torch.uint8, device=device)
    ws_bytes = int(vg.lib.vgb_hca_workspace_bytes(n_st))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    off_p = np.arange(n_st, dtype=np.int64) * stride
    ch_stride = np.full(n_st, stride, dtype=np.int64)
    off_f = np.arange(n_st, dtype=np.int64) * f_stride

    def step():
        N.check(vg.lib.vgb_hca_encode_dev(pcm_dev.data_ptr(), off_p.ctypes.data, ch_stride.ctypes.data, params, n_st, None,
                                          frames_dev.data_ptr(), off_f.ctypes.data, ws.data_ptr(), ws_bytes, stream.cuda_stream))

    N.check(vg.lib.vgb_set_kernel_timing(1))
    for _ in range(args.warmup):
        step()
    N.check(vg.lib.vgb_hca_encode_dev_status(ws.data_ptr(), n_st, stream.cuda_stream))
    _barrier(torch, dist, world)
    sampler = bench.ClockSampler(local_rank)
    sampler.start()
    launches0 = vg.lib.vgb_kernel_launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kms = 0.0
    ev0.record(stream)
    for _ in range(args.steps):
        step()
        buf = (C.c_float * 8)()
        N.check(vg.lib.vgb_last_kernel_ms(buf, 8))
        kms += buf[6]
    ev1.record(stream)
    torch.cuda.synchronize()
    ms = _max_over_ranks(torch, dist, world, device, ev0.elapsed_time(ev1) / args.steps)
    launches = vg.lib.vgb_kernel_launch_count() - launches0
    clocks = sampler.stop()
    kms /= args.steps
    samples = n_st * n
    value = world * samples / (ms / 1e3) / 1e6

    e2e = None
    if not args.no_e2e:
        h_in = torch.empty((n_st, n), dtype=torch.int16, pin_memory=True)
        h_in.copy_(pcm)
        h_out = torch.empty((n_st, fbytes), dtype=torch.uint8, pin_memory=True)
        in_tab = (C.c_void_p * n_st)(*[h_in.data_ptr() + 2 * n * s for s in range(n_st)])
        out_tab = (C.c_void_p * n_st)(*[h_out.data_ptr() + fbytes * s for s in range(n_st)])
        infos = (N.VgbHcaInfo * n_st)()

        def step_e2e():
            N.check(vg.lib.vgb_hca_encode_batch(in_tab, params, n_st, infos, out_tab, None, None))

        step_e2e()
        _barrier(torch, dist, world)
        reps = max(1, min(args.steps, 3))
        t0 = time.perf_counter()
        for _ in range(reps):
            step_e2e()
        e_ms = _max_over_ranks(torch, dist, world, device, (time.perf_counter() - t0) * 1e3 / reps)
        tl = (C.c_float * 48)()
        N.check(vg.lib.vgb_debug_last_timeline(tl, 48))
        same = bool((h_out.to(device) == frames_dev[:, :fbytes]).all().item())
        e2e = {"value": round(world * samples / (e_ms / 1e3) / 1e6, 3), "unit": "Msamples/s", "ms_per_step": round(e_ms, 3),
               "h2d_bytes_per_step": int(n_st * n * 2), "d2h_bytes_per_step": int(n_st * fbytes),
               "pcie_floor_ms": round(n_st * n * 2 / 55e9 * 1e3, 1), "api": "vgb_hca_encode_batch, pinned host buffers",
               "timeline_ms": [[round(tl[3 * g + k], 1) for k in range(3)] for g in range(16) if tl[3 * g] >= 0],
               "matches_device_resident": same}

    parity = cpu = None
    if rank == 0 and not args.no_cpu:
        from oracle import pyoracle

        k = min(64, n_st)
        host = pcm[:k].cpu().numpy()
        got = frames_dev[:k, :fbytes].cpu().numpy()
        cores = os.cpu_count() or 1

        def one(s):
            _, fr = pyoracle.hca_encode([host[s]], SAMPLE_RATE, 2)
            return fr.reshape(-1)

        t0 = time.perf_counter()
        with ThreadPoolExecutor(max_workers=min(cores, k)) as pool:  # ctypes releases the GIL: one stream per core
            want = list(pool.map(one, range(k)))
        dt = time.perf_counter() - t0
        equal = all(np.array_equal(got[s], want[s]) for s in range(k))
        # decoded-domain check demanded by north_star: RMS between the decodes of both frame sets (0 when bytes are equal)
        parity = {"streams_checked": int(k), "frames_byte_identical": bool(equal), "rms_vs_reference_path": 0.0 if equal else None}
        cpu = {"value": round(k * n / dt / 1e6, 3), "unit": "Msamples/s", "cores": int(min(cores, k)), "kind": "port",
               "sample": f"{k} of {n_st} streams x {n} samples ({dt:.1f} s wall), C restatement of CriHcaEncoder, one stream per core "
                         "(the reference's CriHcaFormat.EncodeFromPcm16 is single-threaded per stream; its batch level is Parallel.ForEach over files)"}

    if rank != 0:
        return None
    peak, peak_src = _peak()
    alg = samples * 2.0 + n_st * fbytes
    achieved = alg / (kms / 1e3) / 1e9 if kms > 0 else None
    line = _base_line("CRI HCA encode Msamples/sec (batch)", value, world, args, ms, "weak", "f64",
                      {"workload": f"{n_st} mono streams x {args.seconds:g} s x 48 kHz PCM16 -> CRI HCA, quality High ({info0.frame_size} B frames), per GPU",
                       "global_streams": world * n_st, "samples_per_stream": n, "frames_per_stream": int(info0.frame_count), "distinct_streams": True,
                       "l2": "inputs (1.5 GB/GPU) larger than L2, no flush needed", "parallelism": f"dp{world} (streams sharded)"})
    line.update({"e2e": e2e, "gpu_launches": int(launches), "clocks": clocks,
                 "roofline": {"bound": "hbm", "kernel": "hca_encode_kernel", "achieved": round(achieved, 2) if achieved else None, "peak": peak,
                              "unit": "GB/s", "frac": round(achieved / peak, 5) if achieved else None, "traffic": None, "peak_source": peak_src,
                              "algorithmic_bytes_per_launch": int(alg), "note": "fp64 MDCT + bit allocation search, ALU bound (~135 ops/sample, SURVEY 8d)"},
                 "kernel_ms": {"hca_encode": round(kms, 3)}, "cpu_baseline": cpu, "parity": parity})
    return line


# ======================================================================================================================
# c5: mixed GC-ADPCM + ADX batch, strong scaling with NCCL scatterv / gatherv
# ======================================================================================================================
def _c5_lengths(n_files):
    rng = np.random.default_rng([0x5647415544494F, 5])
    return rng.integers(1 * SAMPLE_RATE, 10 * SAMPLE_RATE + 1, n_files).astype(np.int64)


def _c5_fill(torch, slab, offs, lens, file_ids, device):
    """Synthetic audio straight into the slab: per file three sines + noise at -30 dB of a peak from {2000 .. 32767}."""
    g = torch.Generator(device=device)
    g.manual_seed(0x5647415544494F + 99)
    nf = len(file_ids)
    peaks = torch.tensor([2000.0, 8000.0, 20000.0, 32767.0], device=device)[torch.randint(0, 4, (nf,), generator=g, device=device)]
    w = torch.rand((nf, 3), generator=g, device=device) + 0.05
    amps = w / w.sum(1, keepdim=True) * peaks[:, None]
    freq = torch.exp(torch.rand((nf, 3), generator=g, device=device) * (np.log(12000.0) - np.log(60.0)) + np.log(60.0))
    phase = torch.rand((nf, 3), generator=g, device=device) * (2 * np.pi)
    offs_t = torch.as_tensor(offs, device=device)
    ends_t = offs_t + torch.as_tensor(lens, device=device)
    total = int(slab.numel())
    step = 1 << 27
    for s0 in range(0, total, step):
        idx = torch.arange(s0, min(s0 + step, total), device=device)
        f = torch.clamp(torch.searchsorted(offs_t, idx, right=True) - 1, min=0)
        inside = idx < ends_t[f]
        t = (idx - offs_t[f]).to(torch.float32) / SAMPLE_RATE
        x = torch.zeros(idx.numel(), device=device)
        for k in range(3):
            x += amps[f, k] * torch.sin(2 * np.pi * freq[f, k] * t + phase[f, k])
        x += torch.randn(idx.numel(), generator=g, device=device) * (peaks[f] * 10 ** (-30 / 20))
        slab[s0:s0 + idx.numel()] = torch.where(inside, torch.clamp(torch.round(x), -32768, 32767), torch.zeros_like(x)).to(torch.int16)
        del idx, f, inside, t, x


class _Chunk:
    """One (rank, chunk) work unit of c5: its files (GC-ADPCM first, then ADX, longest first), where its PCM lies in the
    root's slab and in the owner's receive buffer, and the layout of its output block
    [GC payloads (16-aligned) | coefficient table | ADX payloads]."""

    def __init__(self, vg, lens, is_gc, slab_sample_off):
        self.n = len(lens)
        self.lens = lens.astype(np.int64)
        self.n_gc = int(is_gc.sum())
        self.n_adx = self.n - self.n_gc
        pad = (self.lens + 7) // 8 * 8
        self.file_off = np.concatenate(([0], np.cumsum(pad)[:-1])).astype(np.int64) if self.n else np.zeros(0, np.int64)  # samples, chunk relative
        self.samples_padded = int(pad.sum())
        self.slab_off = int(slab_sample_off)                                                                               # samples in the root slab
        self.gc_lens = self.lens[:self.n_gc].astype(np.int32)
        self.adx_lens = self.lens[self.n_gc:].astype(np.int32)
        self.gc_bytes = np.array([vg.gcadpcm.sample_count_to_byte_count(int(v)) for v in self.gc_lens], dtype=np.int64)
        self.adx_bytes = np.array([vg.lib.vgb_adx_encoded_byte_count(int(v), 0, 18) for v in self.adx_lens], dtype=np.int64)
        g16, a16 = (self.gc_bytes + 15) // 16 * 16, (self.adx_bytes + 15) // 16 * 16
        self.gc_out = np.concatenate(([0], np.cumsum(g16)[:-1])).astype(np.int64) if self.n_gc else np.zeros(0, np.int64)
        self.coef_at = int(g16.sum())
        self.adx_at = (self.coef_at + self.n_gc * 32 + 15) // 16 * 16
        self.adx_out = (self.adx_at + np.concatenate(([0], np.cumsum(a16)[:-1]))).astype(np.int64) if self.n_adx else np.zeros(0, np.int64)
        self.out_bytes = (self.adx_at + int(a16.sum()) + 255) // 256 * 256
        self.gc_frames = int(((self.gc_lens.astype(np.int64) + 13) // 14).sum())


def run_c5(args, env, ctx):
    torch, dist, vg, N, bench = ctx["torch"], ctx["dist"], ctx["vg"], ctx["N"], ctx["bench"]
    rank, local_rank, world = env
    device = torch.device("cuda", local_rank)
    compute = torch.cuda.current_stream()
    comm = torch.cuda.Stream(device=device)
    n_files = args.files
    K = max(1, args.c5_chunks) if world > 1 else 1   # a single rank has nothing to overlap
    lens = _c5_lengths(n_files)
    is_gc = (np.arange(n_files) % 2) == 0                       # even index -> GC-ADPCM, odd -> ADX (Linear, v4, 18-byte frames)
    # ---- plan (identical on every rank): files -> ranks by greedy longest-first, a rank's files dealt round-robin (longest
    # first) into K chunks, inside a chunk GC-ADPCM first and longest first (neighbouring channels of a warp are alike)
    part = np.zeros(n_files, dtype=np.int32)
    load = np.zeros(world, dtype=np.int64)
    N.check(vg.lib.vgb_partition_lpt(lens.ctypes.data, n_files, world, part.ctypes.data, load.ctypes.data))
    chunks = [[None] * K for _ in range(world)]
    slab_cursor = 0
    file_order = []                                              # slab order of the original file indices
    for r in range(world):
        mine = np.flatnonzero(part == r)
        mine = mine[np.argsort(-lens[mine], kind="stable")]
        for k in range(K):
            sel = mine[k::K]
            sel = sel[np.lexsort((-lens[sel], ~is_gc[sel]))]
            ch = _Chunk(vg, lens[sel], is_gc[sel], slab_cursor)
            ch.files = sel
            chunks[r][k] = ch
            slab_cursor += ch.samples_padded
            file_order.append(sel)
    total_padded = slab_cursor
    file_order = np.concatenate(file_order)
    slab_file_off = np.concatenate([chunks[r][k].slab_off + chunks[r][k].file_off for r in range(world) for k in range(K)])
    my = chunks[rank]
    my_pcm_off = np.concatenate(([0], np.cumsum([c.samples_padded for c in my])[:-1])).astype(np.int64)       # samples in my receive buffer
    my_out_off = np.concatenate(([0], np.cumsum([c.out_bytes for c in my])[:-1])).astype(np.int64)
    gathered_off = {}                                            # root: where (rank, chunk) lands in the gathered buffer
    cur = 0
    for r in range(world):
        for k in range(K):
            gathered_off[(r, k)] = cur
            cur += chunks[r][k].out_bytes
    gathered_bytes = cur

    # ---- buffers.  Root: the whole PCM slab (its own chunks are encoded in place, their outputs written straight into the
    # gathered buffer); others: a receive buffer for their PCM and an output buffer.
    if rank == 0:
        slab = torch.zeros(total_padded + 8, dtype=torch.int16, device=device)
        _c5_fill(torch, slab, slab_file_off, lens[file_order], file_order, device)
        gathered = torch.zeros(gathered_bytes + 256, dtype=torch.uint8, device=device)
        pcm_base = [slab.data_ptr() + 2 * c.slab_off for c in my]
        out_base = [gathered.data_ptr() + gathered_off[(0, k)] for k in range(K)]
        my_pcm = my_out = None
    else:
        slab = gathered = None
        my_pcm = torch.zeros(int(sum(c.samples_padded for c in my)) + 8, dtype=torch.int16, device=device)
        my_out = torch.zeros(int(sum(c.out_bytes for c in my)) + 256, dtype=torch.uint8, device=device)
        pcm_base = [my_pcm.data_ptr() + 2 * int(o) for o in my_pcm_off]
        out_base = [my_out.data_ptr() + int(o) for o in my_out_off]
    # the two codecs of a chunk, and consecutive chunks, run on separate streams: every encode ends in a thin tail (the
    # boundary run-ons, the cascade) that another stream's kernels fill; two chunks in flight -> two workspaces each (one
    # chunk, one lane: a single rank keeps 14 GB of workspace for the second lane out of an 80 GB card)
    LANES = min(2, K)
    gc_streams = [torch.cuda.Stream(device=device) for _ in range(LANES)]
    adx_streams = [torch.cuda.Stream(device=device) for _ in range(LANES)]
    gws_bytes = int(vg.lib.vgb_gcadpcm_workspace_bytes(max(c.gc_frames for c in my), max(max(c.n_gc for c in my), 1)))
    gws = [torch.empty(gws_bytes, dtype=torch.uint8, device=device) for _ in range(LANES)]
    aws_bytes = int(vg.lib.vgb_adx_workspace_bytes(max(int(c.adx_lens.astype(np.int64).sum()) for c in my), max(max(c.n_adx for c in my), 1)))
    aws = [torch.empty(aws_bytes, dtype=torch.uint8, device=device) for _ in range(LANES)]
    adx_params = (N.VgbAdxParams * max(max(c.n_adx for c in my), 1))()
    for i in range(len(adx_params)):
        adx_params[i] = N.VgbAdxParams(SAMPLE_RATE, 500, 18, 4, 0, 0, 3, 0)

    # ---- communicator inside the library (the id travels over torch.distributed)
    if world > 1:
        idbuf = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            raw = (C.c_uint8 * 128)()
            N.check(vg.lib.vgb_nccl_unique_id(raw))
            idbuf = torch.tensor(list(raw), dtype=torch.uint8)
        idbuf = idbuf.to(device)
        dist.broadcast(idbuf, 0)
        raw = (C.c_uint8 * 128)(*idbuf.cpu().tolist())
        N.check(vg.lib.vgb_nccl_init(raw, world, rank))

    def exchange(scatter_k, gather_k):
        """One NCCL group on the comm stream: the root sends every peer its PCM chunk `scatter_k` and receives the output
        blocks of chunk `gather_k`; a peer does the opposite.  Full duplex: both directions move at once."""
        sp, sb, speer, rp, rb, rpeer = [], [], [], [], [], []
        if rank == 0:
            for r in range(1, world):
                if scatter_k is not None:
                    c = chunks[r][scatter_k]
                    sp.append(slab.data_ptr() + 2 * c.slab_off); sb.append(2 * c.samples_padded); speer.append(r)
                if gather_k is not None:
                    rp.append(gathered.data_ptr() + gathered_off[(r, gather_k)]); rb.append(chunks[r][gather_k].out_bytes); rpeer.append(r)
        else:
            if scatter_k is not None:
                rp.append(pcm_base[scatter_k]); rb.append(2 * my[scatter_k].samples_padded); rpeer.append(0)
            if gather_k is not None:
                sp.append(out_base[gather_k]); sb.append(my[gather_k].out_bytes); speer.append(0)
        if not sp and not rp:
            return
        arr = lambda v, t: (t * max(len(v), 1))(*v)
        N.check(vg.lib.vgb_sendrecv_dev(arr(sp, C.c_void_p), arr(sb, C.c_int64), arr(speer, C.c_int32), len(sp),
                                        arr(rp, C.c_void_p), arr(rb, C.c_int64), arr(rpeer, C.c_int32), len(rp), comm.cuda_stream))

    def encode(k, ready, done):
        """Chunk k on its lane's two streams, after event `ready`; `done` (a list) receives one event per stream."""
        c = my[k]
        lane = k % LANES
        for st in (gc_streams[lane], adx_streams[lane]):
            st.wait_event(ready)
        if c.n_gc:
            off = c.file_off[:c.n_gc].copy()
            N.check(vg.lib.vgb_gcadpcm_encode_dev(pcm_base[k], off.ctypes.data, c.gc_lens.ctypes.data, None, c.n_gc, None,
                                                  out_base[k] + c.coef_at, out_base[k], c.gc_out.ctypes.data, gws[lane].data_ptr(), gws_bytes,
                                                  gc_streams[lane].cuda_stream))
        if c.n_adx:
            off = c.file_off[c.n_gc:].copy()
            N.check(vg.lib.vgb_adx_encode_dev(pcm_base[k], off.ctypes.data, c.adx_lens.ctypes.data, adx_params, c.n_adx, None,
                                              out_base[k], c.adx_out.ctypes.data, aws[lane].data_ptr(), aws_bytes, adx_streams[lane].cuda_stream))
        for st in (gc_streams[lane], adx_streams[lane]):
            ev = torch.cuda.Event()
            ev.record(st)
            done.append(ev)

    def step(phases=None):
        """Pipeline over the K chunks: comm step t = {scatter chunk t, gather chunk t-2}; encode chunk t follows comm step t."""
        enc_done = [[] for _ in range(K)]
        start = torch.cuda.Event()
        start.record(compute)
        comm.wait_event(start)
        arrived = start
        for t in range(K + 2):
            sk = t if t < K else None
            gk = t - 2 if t - 2 >= 0 else None
            if world > 1 and (sk is not None or gk is not None):
                if gk is not None:
                    for ev in enc_done[gk]:
                        comm.wait_event(ev)
                if phases is not None:
                    phases.append(("comm", t, torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
                    phases[-1][2].record(comm)
                exchange(sk, gk)
                if phases is not None:
                    phases[-1][3].record(comm)
                arrived = torch.cuda.Event()
                arrived.record(comm)
            if sk is not None:
                if phases is not None:
                    phases.append(("enc", t, torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
                    gc_streams[sk % LANES].wait_event(arrived)
                    phases[-1][2].record(gc_streams[sk % LANES])
                encode(sk, arrived, enc_done[sk])
                if phases is not None:
                    phases[-1][3].record(gc_streams[sk % LANES])
        compute.wait_stream(comm)
        for evs in enc_done:
            for ev in evs:
                compute.wait_event(ev)

    N.check(vg.lib.vgb_set_kernel_timing(0))
    for _ in range(args.warmup):
        step()
    _barrier(torch, dist, world)
    sampler = bench.ClockSampler(local_rank)
    sampler.start()
    launches0 = vg.lib.vgb_kernel_launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(compute)
    for _ in range(args.steps):
        step()
    ev1.record(compute)
    torch.cuda.synchronize()
    ms = _max_over_ranks(torch, dist, world, device, ev0.elapsed_time(ev1) / args.steps)
    launches = vg.lib.vgb_kernel_launch_count() - launches0
    clocks = sampler.stop()
    # one more, instrumented step (untimed) for the phase breakdown
    phases = []
    _barrier(torch, dist, world)
    step(phases)
    torch.cuda.synchronize()
    comm_ms = sum(p[2].elapsed_time(p[3]) for p in phases if p[0] == "comm")
    enc_ms = sum(p[2].elapsed_time(p[3]) for p in phases if p[0] == "enc")
    enc_all = np.zeros(world)
    enc_all[rank] = enc_ms
    comm_all = _max_over_ranks(torch, dist, world, device, comm_ms)
    if world > 1:
        t = torch.as_tensor(enc_all, device=device)
        dist.all_reduce(t)
        enc_all = t.cpu().numpy()
    total = int(lens.sum())
    value = total / (ms / 1e3) / 1e6
    scatter_bytes = int(sum(2 * chunks[r][k].samples_padded for r in range(1, world) for k in range(K)))
    gather_bytes = int(sum(chunks[r][k].out_bytes for r in range(1, world) for k in range(K)))

    # ---- e2e: every rank's files from ITS OWN pinned host memory through the host API (one H2D link per GPU)
    e2e = None
    if not args.no_e2e:
        torch.cuda.synchronize()
        n_samp = int(sum(c.samples_padded for c in my))
        h_pcm = torch.empty(n_samp + 8, dtype=torch.int16, pin_memory=True)
        if rank == 0:
            for k, c in enumerate(my):
                h_pcm[int(my_pcm_off[k]):int(my_pcm_off[k]) + c.samples_padded].copy_(slab[c.slab_off:c.slab_off + c.samples_padded])
        else:
            h_pcm[:n_samp].copy_(my_pcm[:n_samp])
        # the host-pointer calls allocate their own device buffers: release the timed leg's workspaces and, on a single
        # rank, the device copy of the PCM (the parity check then reads the pinned copy, same offsets) - on one 80 GB card
        # the timed leg's buffers alone take ~58 GB
        del gws, aws
        if world == 1:
            slab = h_pcm
        torch.cuda.empty_cache()
        h_out =torch.empty(int(sum(c.out_bytes for c in my)) + 256, dtype=torch.uint8, pin_memory=True)
        gc_in, gc_tab, ad_in, ad_tab, gl, al = [], [], [], [], [], []
        for k, c in enumerate(my):
            gc_in += [h_pcm.data_ptr() + 2 * int(my_pcm_off[k] + o) for o in c.file_off[:c.n_gc]]
            gc_tab += [h_out.data_ptr() + int(my_out_off[k] + o) for o in c.gc_out]
            ad_in += [h_pcm.data_ptr() + 2 * int(my_pcm_off[k] + o) for o in c.file_off[c.n_gc:]]
            ad_tab += [h_out.data_ptr() + int(my_out_off[k] + o) for o in c.adx_out]
            gl += list(c.gc_lens); al += list(c.adx_lens)
        n_gc, n_adx = len(gl), len(al)
        gl, al = np.array(gl, dtype=np.int32), np.array(al, dtype=np.int32)
        gc_in, gc_tab = (C.c_void_p * max(n_gc, 1))(*gc_in), (C.c_void_p * max(n_gc, 1))(*gc_tab)
        ad_in, ad_tab = (C.c_void_p * max(n_adx, 1))(*ad_in), (C.c_void_p * max(n_adx, 1))(*ad_tab)
        h_coefs = np.zeros((max(n_gc, 1), 16), dtype=np.int16)
        ap = (N.VgbAdxParams * max(n_adx, 1))(*[N.VgbAdxParams(SAMPLE_RATE, 500, 18, 4, 0, 0, 3, 0) for _ in range(max(n_adx, 1))])

        def step_e2e():
            if n_gc:
                N.check(vg.lib.vgb_gcadpcm_encode_batch(gc_in, gl.ctypes.data, None, None, n_gc, h_coefs.ctypes.data, gc_tab, None, None))
            if n_adx:
                N.check(vg.lib.vgb_adx_encode_batch(ad_in, al.ctypes.data, ap, n_adx, None, ad_tab, None, None))

        step_e2e()
        _barrier(torch, dist, world)
        t0 = time.perf_counter()
        step_e2e()
        e_ms = _max_over_ranks(torch, dist, world, device, (time.perf_counter() - t0) * 1e3)
        dev_out = gathered if rank == 0 else my_out
        same = True
        for k, c in enumerate(my):
            base = gathered_off[(0, k)] if rank == 0 else int(my_out_off[k])
            if c.n_gc:
                same = same and bool((h_out[int(my_out_off[k]):int(my_out_off[k]) + c.coef_at].to(device) == dev_out[base:base + c.coef_at]).all().item())
            if c.n_adx:
                lo, hi = c.adx_at, int(c.adx_out[-1] + c.adx_bytes[-1])
                same = same and bool((h_out[int(my_out_off[k]) + lo:int(my_out_off[k]) + hi].to(device) == dev_out[base + lo:base + hi]).all().item())
        e2e = {"value": round(total / (e_ms / 1e3) / 1e6, 3), "unit": "Msamples/s", "ms_per_step": round(e_ms, 3),
               "h2d_bytes_per_step": int(total * 2), "d2h_bytes_per_step": int(gathered_bytes),
               "pcie_floor_ms": round(total * 2 / world / 55e9 * 1e3, 1),
               "api": "vgb_gcadpcm_encode_batch + vgb_adx_encode_batch per rank on its own files from pinned host memory (one PCIe link per GPU)",
               "matches_device_resident": same}

    # ---- parity on the root: >= 128 GC + 128 ADX files drawn across every rank's blocks of the gathered buffer
    parity = cpu = None
    if rank == 0 and not args.no_cpu:
        from oracle import pyoracle

        rng = np.random.default_rng(7)
        checked_gc = checked_adx = 0
        ok = True
        cpu_samples, cpu_t = 0, 0.0
        want_each = max(1, -(-128 // (world * K)))
        for r in range(world):
            for k in range(K):
                c = chunks[r][k]
                base = gathered_off[(r, k)]
                for i in (rng.choice(c.n_gc, min(want_each, c.n_gc), replace=False) if c.n_gc else []):
                    L, o = int(c.gc_lens[i]), c.slab_off + int(c.file_off[i])
                    x = slab[o:o + L].cpu().numpy()
                    t0 = time.perf_counter()
                    co = pyoracle.calculate_coefficients(x)
                    want = pyoracle.encode(x, co)
                    cpu_t += time.perf_counter() - t0
                    cpu_samples += L
                    got = gathered[base + int(c.gc_out[i]):base + int(c.gc_out[i]) + int(c.gc_bytes[i])].cpu().numpy()
                    gco = gathered[base + c.coef_at + 32 * int(i):base + c.coef_at + 32 * int(i) + 32].cpu().numpy().view(np.int16)
                    ok = ok and np.array_equal(got, want) and np.array_equal(gco, co)
                    checked_gc += 1
                for i in (rng.choice(c.n_adx, min(want_each, c.n_adx), replace=False) if c.n_adx else []):
                    L, o = int(c.adx_lens[i]), c.slab_off + int(c.file_off[c.n_gc + i])
                    x = slab[o:o + L].cpu().numpy()
                    want, _ = pyoracle.adx_encode(x, SAMPLE_RATE, 18, 4, 0, 3, 0)
                    got = gathered[base + int(c.adx_out[i]):base + int(c.adx_out[i]) + int(c.adx_bytes[i])].cpu().numpy()
                    ok = ok and np.array_equal(got, want)
                    checked_adx += 1
        parity = {"gc_files_checked": checked_gc, "adx_files_checked": checked_adx, "bytes_equal_oracle": bool(ok)}
        cores = os.cpu_count() or 1
        if cpu_t > 0:
            cpu = {"value": round(cpu_samples / cpu_t / 1e6 * cores, 3), "unit": "Msamples/s", "cores": cores, "kind": "port",
                   "sample": f"{checked_gc} GC-ADPCM files ({cpu_samples} samples) timed on ONE core ({cpu_samples / cpu_t / 1e6:.2f} Msamples/s) "
                             f"x {cores} cores: the reference's Parallel.ForEach over files is embarrassingly parallel"}

    if world > 1:
        N.check(vg.lib.vgb_nccl_shutdown())
    if rank != 0:
        return None
    mean_enc = float(enc_all.mean()) if world > 0 else 0.0
    peak, peak_src = _peak()
    per_gpu = total * 2.567 / (float(enc_all.max()) / 1e3) / 1e9 / world if enc_all.max() > 0 else None
    line = _base_line("mixed GC-ADPCM + ADX batch encode Msamples/sec", value, world, args, ms, "strong", "int32",
                      {"workload": f"{n_files} mono files, 1-10 s x 48 kHz, even -> GC-ADPCM (coefs + encode), odd -> CRI ADX (Linear, v4, 18 B frames); whole job",
                       "total_samples": total, "files_per_rank": [int((part == r).sum()) for r in range(world)], "chunks_per_rank": K,
                       "l2": "inputs (34.6 GB) larger than L2, no flush needed",
                       "parallelism": f"{world} ranks, files partitioned longest-first; the root holds the PCM, per chunk one NCCL group scatters chunk t and gathers chunk t-2 while chunk t-1 encodes"})
    line.update({"e2e": e2e, "gpu_launches": int(launches), "clocks": clocks,
                 "collective": {"comm_busy_ms": round(comm_all, 3), "scatter_bytes": scatter_bytes, "gather_bytes": gather_bytes,
                                "nccl_version": int(vg.lib.vgb_nccl_version()), "encode_ms_per_rank": [round(float(v), 3) for v in enc_all],
                                "imbalance": round(float(enc_all.max() / mean_enc), 4) if mean_enc > 0 else None,
                                "exposed_ms": round(ms - float(enc_all.max()), 3),
                                "note": "comm_busy_ms = summed duration of the NCCL groups of one step on the busiest rank; exposed_ms = step time minus the slowest rank's encode time; run with --c5-chunks 1 for separate scatter / gather times"},
                 "roofline": {"bound": "hbm", "kernel": "gc_encode_kernel + adx_encode_kernel", "achieved": round(per_gpu, 2) if per_gpu else None,
                              "peak": peak, "unit": "GB/s", "frac": round(per_gpu / peak, 5) if per_gpu else None, "traffic": None, "peak_source": peak_src,
                              "note": "per-GPU algorithmic bytes (2 B in + ~0.57 B out per sample) over the slowest rank's encode time"},
                 "cpu_baseline": cpu, "parity": parity})
    return line


# ======================================================================================================================
# batch: WAVE files in -> .dsp / .adx / .hca files out through vgb_convert_wave_batch (SURVEY 8f rank 2-4; the CLI's
# Batch.cs job).  One GPU; the whole chain (RIFF parse, H2D of the data chunks, de-interleave, encode, loop context, file
# assembly, D2H) is inside the timed region - there is no device-resident variant of a file converter.
# ======================================================================================================================
def _batch_files(torch, bench, n_files, device, seed=0):
    """Synthetic WAVE images in pinned host memory: mono / stereo, 1-6 s at 48 kHz, every eighth file looping."""
    rng = np.random.default_rng(1234 + seed)
    lens = rng.integers(1 * SAMPLE_RATE, 6 * SAMPLE_RATE + 1, n_files)
    chans = np.where(np.arange(n_files) % 3 == 2, 2, 1)
    files, meta = [], []
    n_max = int(lens.max())
    pool = bench.make_batch_gpu(torch, 64, n_max, 7 + seed, device, degenerate=False).cpu().numpy()  # 64 distinct signals
    for i in range(n_files):
        n, ch = int(lens[i]), int(chans[i])
        # distinct content per file: a signal of the pool from a file-specific offset, second channel from another signal
        rows = [np.roll(pool[(i * 2 + c) % 64], -(i * 37 + c * 101) % n_max)[:n] for c in range(ch)]
        loop = (int(n // 5), int(n - n // 7)) if i % 8 == 5 else None
        data = np.stack(rows, axis=1).astype("<i2").tobytes()
        fmt = np.array([1, ch], dtype="<u2").tobytes() + np.array([SAMPLE_RATE, SAMPLE_RATE * 2 * ch], dtype="<u4").tobytes() + \
            np.array([2 * ch, 16], dtype="<u2").tobytes()
        smpl = b""
        if loop:
            body = np.zeros(15, dtype="<i4")
            body[7] = 1
            body[11], body[12] = loop
            smpl = b"smpl" + np.array([0x3c], dtype="<u4").tobytes() + body.tobytes()
        body = b"WAVE" + b"fmt " + np.array([16], dtype="<u4").tobytes() + fmt + smpl + b"data" + np.array([len(data)], dtype="<u4").tobytes() + data
        img = b"RIFF" + np.array([len(body)], dtype="<u4").tobytes() + body
        t = torch.empty(len(img), dtype=torch.uint8, pin_memory=True)
        t.numpy()[:] = np.frombuffer(img, dtype=np.uint8)
        files.append(t)
        meta.append((rows, n, loop))
    return files, meta


def run_batch(args, env, ctx):
    torch, vg, N, bench = ctx["torch"], ctx["vg"], ctx["N"], ctx["bench"]
    rank, local_rank, world = env
    if world != 1:
        raise SystemExit("--config batch runs on one GPU (files of a job are independent: run one process per GPU on disjoint file lists)")
    from vgaudio_b200 import containers as ct

    device = torch.device("cuda", local_rank)
    n_files = args.files if args.files != 65536 else 2048
    out_type = {"dsp": ct.CONTAINER_DSP, "adx": ct.CONTAINER_ADX, "hca": ct.CONTAINER_HCA}[args.out_format]
    files, meta = _batch_files(torch, bench, n_files, device)
    total_samples = sum(len(m[0]) * m[1] for m in meta)
    in_bytes = sum(int(f.numel()) for f in files)
    opt = ct.convert_options(out_type, hca_quality=2)
    n = len(files)
    ftab = (C.c_void_p * n)(*[f.data_ptr() for f in files])
    lens = (C.c_int64 * n)(*[int(f.numel()) for f in files])
    sizes = (C.c_int64 * n)()
    status = (C.c_int32 * n)()
    N.check(vg.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(opt), sizes, None, status, None, None))
    outs = [torch.empty(int(sizes[i]), dtype=torch.uint8, pin_memory=True) for i in range(n)]
    otab = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
    out_bytes = sum(int(sizes[i]) for i in range(n))

    def step():
        N.check(vg.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(opt), sizes, otab, status, None, None))

    for _ in range(max(args.warmup, 1)):
        step()
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(local_rank)
    sampler.start()
    launches0 = vg.lib.vgb_kernel_launch_count()
    stage = np.zeros(4)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / args.steps
    launches = vg.lib.vgb_kernel_launch_count() - launches0
    clocks = sampler.stop()
    # the stage timers of overlapping groups overlap too: one more, untimed, pass with one group in flight gives clean ones
    os.environ["VGB_CONVERT_SERIAL"] = "1"
    stage[:] = 0
    for _ in range(args.steps):
        step()
        buf = (C.c_float * 4)()
        vg.lib.vgb_convert_debug_stage_ms(buf, 4)
        stage += np.array(list(buf))
    del os.environ["VGB_CONVERT_SERIAL"]
    stage /= args.steps
    value = total_samples / (ms / 1e3) / 1e6
    peak, peak_src = _peak()
    pcm_bytes = 2 * total_samples
    # byte movers: the split kernel reads the data chunks and writes the channel rows (2 x PCM bytes); the assembly kernel
    # reads the encoded payload and writes the files (2 x output bytes)
    split_gbs = 2 * pcm_bytes / (stage[0] / 1e3) / 1e9 if stage[0] > 0 else None
    asm_gbs = 2 * out_bytes / (stage[3] / 1e3) / 1e9 if stage[3] > 0 else None

    # ---- parity + CPU baseline: the oracle's WaveReader -> encoder -> writer chain, one file per task ---------------------
    cpu = parity = None
    if not args.no_cpu:
        from oracle import pyoracle as o

        def one(i):
            img = files[i].numpy()
            st, info = o.wave_parse(img)
            rows = o.wave_read(img, info)
            loop = (info.loop_start, info.loop_end) if info.looping else None
            if out_type == ct.CONTAINER_DSP:
                coefs = np.stack([o.calculate_coefficients(p) for p in rows])
                adpcm = [o.encode(p, c) for p, c in zip(rows, coefs)]
                ctxs = None
                if loop:
                    ctxs = np.stack([np.array(o.gc_loop_context(a, o.decode(a, c, info.sample_count), loop[0]), dtype=np.int16)
                                     for a, c in zip(adpcm, coefs)])
                return o.dsp_write(adpcm, coefs, info.sample_rate, info.sample_count, loop, ctxs)
            if out_type == ct.CONTAINER_ADX:
                ch = info.channel_count
                align = (-loop[0]) % (64 if ch == 1 else 32) if loop else 0
                enc = [o.adx_encode(p, info.sample_rate, 18, 4, align, 3, 0) for p in rows]
                return o.adx_write([e[0] for e in enc], [e[1] for e in enc], info.sample_rate, info.sample_count, loop, align)
            hinfo, frames = o.hca_encode(rows, info.sample_rate, quality=2, loop=loop)
            return o.hca_write(hinfo, frames)

        cores = os.cpu_count() or 1
        sample = list(range(min(n, max(cores, 64))))
        t0 = time.perf_counter()
        with ThreadPoolExecutor(max_workers=cores) as ex:
            want = list(ex.map(one, sample))
        cpu_s = time.perf_counter() - t0
        cpu_samples = sum(len(meta[i][0]) * meta[i][1] for i in sample)
        cpu = {"value": round(cpu_samples / cpu_s / 1e6, 3), "unit": "Msamples/s", "cores": min(cores, len(sample)), "kind": "port",
               "sample": f"{len(sample)} of {n} files ({cpu_samples} samples, {cpu_s:.1f} s wall): the oracle's WaveReader -> encoder -> "
                         f"writer chain, one file per task (ctypes releases the GIL), as Batch.cs runs Convert.ConvertFile per file"}
        equal = all(outs[i].numpy().tobytes() == want[k].tobytes() for k, i in enumerate(sample))
        parity = {"files_checked": len(sample), "file_bytes_equal_oracle": bool(equal)}

    line = _base_line(f"batch WAVE -> .{args.out_format} conversion Msamples/sec", value, world, args, ms, "weak", "int32" if out_type != ct.CONTAINER_HCA else "f64",
                      {"workload": f"{n} WAVE files (2/3 mono, 1/3 stereo, 1-6 s x 48 kHz, 1/8 looping) -> .{args.out_format} through vgb_convert_wave_batch",
                       "total_samples": int(total_samples), "files_per_s": round(n / (ms / 1e3), 1),
                       "l2": f"inputs ({in_bytes / 1e9:.2f} GB) larger than L2, no flush needed", "parallelism": "one GPU, files coalesced into 256 MiB batches"})
    line["e2e"] = {"value": round(value, 3), "unit": "Msamples/s", "ms_per_step": round(ms, 3), "h2d_bytes_per_step": int(in_bytes),
                   "d2h_bytes_per_step": int(out_bytes), "pcie_floor_ms": round((in_bytes / 55.6e9 + 0) * 1e3, 1),
                   "api": "vgb_convert_wave_batch: pinned host file images in, pinned host files out (value IS the end-to-end figure: a file "
                          "converter has no device-resident variant)"}
    line["gpu_launches"] = int(launches)
    line["clocks"] = clocks
    line["stage_ms"] = {"wave_split": round(float(stage[0]), 3), "encode": round(float(stage[1]), 3), "loop_context_decode": round(float(stage[2]), 3),
                        "file_assembly": round(float(stage[3]), 3)}
    dom = "wave_split_kernel" if stage[0] >= stage[3] else f"{args.out_format}_assemble_kernel"
    ach = split_gbs if stage[0] >= stage[3] else asm_gbs
    line["roofline"] = {"bound": "hbm", "kernel": dom + " (the byte movers; the encode kernels have their own lines under --config c2/c4)",
                        "achieved": round(ach, 1) if ach else None, "peak": peak, "unit": "GB/s", "frac": round(ach / peak, 4) if ach else None,
                        "traffic": None, "peak_source": peak_src,
                        "byte_movers_gbs": {"wave_split": round(split_gbs, 1) if split_gbs else None, "file_assembly": round(asm_gbs, 1) if asm_gbs else None},
                        "note": "algorithmic bytes = bytes read + bytes written once each; stage times are CUDA events around the launches of a batch "
                                "(table uploads included), summed over the batches of a separate pass with one batch in flight (VGB_CONVERT_SERIAL)"}
    line["cpu_baseline"] = cpu
    line["parity"] = parity
    return line
