"""Both batch converters sharded over several bound devices (vgb_init_devices).  The live files of a call are spread over
the devices by longest-first bin packing; every device runs the single-device group loop on its own files with its own
streams and working sets.  Outputs, sizes and per-file statuses must equal the single-device call of the same job byte
for byte, and the oracle chain.  A single-GPU box binds device 0 three times - the same code path (per-device container
state, worker threads, shared progress, error addressing); on a multi-GPU box distinct devices are used."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")
FILE_WEIGHT = 1024   # the per-file constant of the converters' bin packing (include/vgaudio_b200.h)


def _bind(vg, devs):
    from vgaudio_b200 import _native as N

    N.check(vg.lib.vgb_shutdown())
    if devs == [0]:
        N.check(vg.lib.vgb_init(0, 0))
    else:
        N.check(vg.lib.vgb_init_devices((C.c_int32 * len(devs))(*devs), len(devs), 0))
    assert vg.lib.vgb_device_count() == len(devs)


@pytest.fixture
def three_devices(vg):
    import torch

    from vgaudio_b200 import _native as N

    n = torch.cuda.device_count()
    devs = [0, 1 % n, 2 % n] if n > 1 else [0, 0, 0]
    _bind(vg, devs)
    yield devs
    N.check(vg.lib.vgb_shutdown())
    N.check(vg.lib.vgb_init(0, 0))
    assert vg.lib.vgb_device_count() == 1


def _on_one_device(vg, devs, fn):
    """fn() with only device 0 bound, then the devices `devs` bound again."""
    _bind(vg, [0])
    try:
        return fn()
    finally:
        _bind(vg, devs)


def _lpt(weights, n_dev=3):
    """shard_units (vgaudio_b200/csrc/abi.cuh): heaviest first onto the least loaded device, ascending inside a shard."""
    order = sorted(range(len(weights)), key=lambda u: -weights[u])   # sorted() is stable, as std::stable_sort
    load, shards = [0] * n_dev, [[] for _ in range(n_dev)]
    for u in order:
        best = min(range(n_dev), key=lambda d: (load[d], d))
        shards[best].append(u)
        load[best] += weights[u]
    return [sorted(s) for s in shards]


def _pcm(n_ch, n, first):
    return [synth.channel(first + c, max(n, 1))[:n] for c in range(n_ch)]


def _wave8(channels, rate):
    ch = len(channels)
    data = np.stack(channels, axis=1).astype(np.uint8).tobytes()
    fmt = struct.pack("<HHIIHH", 1, ch, rate, rate * ch, ch, 8)
    body = b"WAVE" + b"fmt " + struct.pack("<I", 16) + fmt + b"data" + struct.pack("<I", len(data)) + data
    return np.frombuffer(b"RIFF" + struct.pack("<I", len(body)) + body, dtype=np.uint8)


def _wave_job(oracle):
    """A seeded job of 46 good WAVE files (mono / stereo / 3 / 6 channels, 16- and 8-bit, 1 sample to 6 s, looping at odd
    points) and two malformed ones, placed in front of files of two different shards.  Returns (files, meta, shards of the
    good files, indices of the malformed ones)."""
    rng = np.random.default_rng(2024)
    files, meta = [], []
    for k in range(46):
        ch = [1, 2, 3, 6][k % 4]
        rate = [16000, 22050, 32000][k % 3]
        kind = k % 5
        n = 1 if k in (3, 21) else int(rng.integers(40, 3000)) if kind == 1 else int(rng.integers(1 * rate, 6 * rate + 1))
        if kind == 4 and k not in (3, 21):   # 8-bit
            raw = [rng.integers(0, 256, n) for _ in range(ch)]
            files.append(_wave8(raw, rate))
            meta.append(([((r.astype(np.int32) - 0x80) << 8).astype(np.int16) for r in raw], n, None, rate, True))
            continue
        loop = None
        if kind in (0, 2) and n > 4096:
            ls = int(rng.integers(1, n // 3)) | 1
            loop = (ls, int(rng.integers(ls + 2048, n + 1)))
        pcm = _pcm(ch, n, first=600 + 7 * k)
        files.append(oracle.wave_write16(pcm, rate, loop))
        meta.append((pcm, n, loop, rate, False))
    shards = _lpt([m[1] * len(m[0]) + FILE_WEIGHT for m in meta])
    assert sum(1 for s in shards if s) >= 2
    # truncated RIFF in front of the first file of shard 1, bad block align in front of the first file of shard 2
    truncated = files[5][:30].copy()
    bad_align = files[6].copy()
    bad_align[32] ^= 0x01
    at1, at2 = shards[1][0], shards[2][0]
    assert at1 != at2
    for at, f in sorted([(at1, truncated), (at2, bad_align)], key=lambda p: -p[0]):
        files.insert(at, f)
        meta.insert(at, None)
    bad = [k for k, m in enumerate(meta) if m is None]
    return files, meta, shards, bad


def _encode_gc(oracle, pcm):
    coefs = np.stack([oracle.calculate_coefficients(p) for p in pcm])
    return coefs, [oracle.encode(p, c) for p, c in zip(pcm, coefs)]


def _oracle_dsp(oracle, pcm, n, loop, rate):
    coefs, adpcm = _encode_gc(oracle, pcm)
    ctx = None
    if loop:
        ctx = np.stack([np.array(oracle.gc_loop_context(a, oracle.decode(a, c, n), loop[0]), dtype=np.int16) for a, c in zip(adpcm, coefs)])
    return oracle.dsp_write(adpcm, coefs, rate, n, loop, ctx)


def _oracle_adx(oracle, pcm, n, loop, rate):
    align = (-loop[0]) % (64 if len(pcm) == 1 else 32) if loop else 0
    enc = [oracle.adx_encode(p, rate, 18, 4, align, 3, 0) for p in pcm]
    return oracle.adx_write([e[0] for e in enc], [e[1] for e in enc], rate, n, loop, align, 18, 4, 3, 500, 0, None)


def _oracle_hca(oracle, pcm, n, loop, rate):
    info, frames = oracle.hca_encode(pcm, rate, quality=2, loop=loop)
    return oracle.hca_write(info, frames)


def _wave_cases(oracle, ct):
    kc = oracle.adx_key(key_code=0x123456789A)
    ks = oracle.adx_key(key_string="karaage")
    mb = 1 << 20
    return [
        ("dsp", ct.convert_options(ct.CONTAINER_DSP, group_bytes=mb), _oracle_dsp),
        ("dsp-1c00-28-notrim", ct.convert_options(ct.CONTAINER_DSP, group_bytes=mb, dsp_samples_per_interleave=0x1c00,
                                                  dsp_loop_point_alignment=28, no_trim=1), None),
        ("adx", ct.convert_options(ct.CONTAINER_ADX, group_bytes=mb), _oracle_adx),
        ("adx-fixed-v3-34", ct.convert_options(ct.CONTAINER_ADX, group_bytes=mb, adx_version=3, adx_frame_size=34, adx_type=2), None),
        ("adx-type9", ct.convert_options(ct.CONTAINER_ADX, group_bytes=mb, adx_has_key=1, adx_key_seed=kc[0], adx_key_mult=kc[1],
                                         adx_key_inc=kc[2], adx_encryption_type=9), None),
        ("adx-type8", ct.convert_options(ct.CONTAINER_ADX, group_bytes=mb, adx_has_key=1, adx_key_seed=ks[0], adx_key_mult=ks[1],
                                         adx_key_inc=ks[2], adx_encryption_type=8), None),
        ("hca", ct.convert_options(ct.CONTAINER_HCA, group_bytes=mb, hca_quality=2), _oracle_hca),
        ("hca-key56", ct.convert_options(ct.CONTAINER_HCA, group_bytes=mb, hca_quality=2, hca_key_type=56, hca_key_code=0xCC55463930DBE1AB), None),
        ("hca-key0", ct.convert_options(ct.CONTAINER_HCA, group_bytes=mb, hca_quality=2, hca_key_type=0), None),
    ]


def test_wave_to_every_target_equals_one_device_and_oracle(vg, oracle, three_devices):
    from vgaudio_b200 import containers as ct

    files, meta, shards, bad = _wave_job(oracle)
    for name, opt, chain in _wave_cases(oracle, ct):
        job, job_meta = files, meta
        if name.startswith("hca"):   # HCA wants a frame's worth of signal, not white noise: short and 8-bit files stay out
            keep = [k for k, m in enumerate(meta) if m is None or (m[1] >= 1024 and not m[4])]
            job, job_meta = [files[k] for k in keep], [meta[k] for k in keep]
        outs, status = ct.convert_wave_batch(job, opt)
        one_outs, one_status = _on_one_device(vg, three_devices, lambda: ct.convert_wave_batch(job, opt))
        assert status == one_status, name
        for k, m in enumerate(job_meta):
            if m is None:
                assert status[k] != 0 and outs[k] is None, (name, k)
                continue
            if one_outs[k] is None:
                assert outs[k] is None, (name, k)
                continue
            assert outs[k].tobytes() == one_outs[k].tobytes(), (name, k)
            if chain is not None:
                assert status[k] == 0, (name, k)
                want = chain(oracle, *m[:4])
                assert outs[k].tobytes() == want.tobytes(), (name, k, int(np.flatnonzero(outs[k][:want.size] != want[:outs[k].size])[0])
                                                             if outs[k].size and want.size else -1)
    # a sharded call times the groups of every device that had files: several groups each with 1 MiB groups
    ct.convert_wave_batch(files, _wave_cases(oracle, ct)[0][1])
    buf = (C.c_float * 4)()
    assert vg.lib.vgb_convert_debug_stage_ms(buf, 4) >= 2 * sum(1 for s in shards if s)
    assert buf[0] > 0 and buf[1] > 0 and buf[3] > 0


def _dsp_job(oracle):
    rng = np.random.default_rng(77)
    files, want = [], []
    for k, (ch, loop) in enumerate([(1, None), (2, (1001, 20000)), (1, (33, 9000)), (3, None), (6, (5, 7000)), (2, None), (1, None),
                                    (4, None), (2, (0, 14000)), (1, (777, 12000)), (8, None), (2, None), (1, (9, 30001))]):
        n = int(rng.integers(loop[1] if loop else 1000, 32000)) if k != 6 else 1
        if loop and loop[1] > n:
            n = loop[1]
        pcm = _pcm(ch, n, first=900 + 9 * k)
        coefs, adpcm = _encode_gc(oracle, pcm)
        ctx = np.stack([np.array(oracle.gc_loop_context(a, oracle.decode(a, c, n), loop[0]), dtype=np.int16) for a, c in zip(adpcm, coefs)]) if loop else None
        hist = np.array([[5 * c + k, -2 * c] for c in range(ch)], dtype=np.int16)
        spi = [0x3800, 14 * 16, 14 * 100][k % 3]
        files.append(oracle.dsp_write(adpcm, coefs, 22050 + k, n, loop, ctx, None, hist, spi, 1, False))
        dec = [oracle.decode(a, c, n, int(h[0]), int(h[1])) for a, c, h in zip(adpcm, coefs, hist)]
        want.append(oracle.wave_write16(dec, 22050 + k, loop))
    return files, want


def test_dsp_to_wave_equals_one_device_and_oracle(vg, oracle, three_devices):
    from vgaudio_b200 import containers as ct

    files, want = _dsp_job(oracle)
    outs, status = ct.convert_dsp_to_wave_batch(files)
    one_outs, one_status = _on_one_device(vg, three_devices, lambda: ct.convert_dsp_to_wave_batch(files))
    assert status == one_status == [0] * len(files)
    for k, w in enumerate(want):
        assert outs[k].tobytes() == one_outs[k].tobytes() == w.tobytes(), k
    # a frame header that selects predictor 8: the whole call fails, naming the device that met it
    broken = [f.copy() for f in files]
    broken[0][0x60] = 0x80 | (broken[0][0x60] & 0x0F)    # file 0 is mono: its payload starts right behind the header
    with pytest.raises(vg.VgbError) as e:
        ct.convert_dsp_to_wave_batch(broken)
    assert e.value.code == -2, str(e.value)
    assert any(str(e.value).endswith(f"(device {d})") for d in set(three_devices)), str(e.value)
    again, st = ct.convert_dsp_to_wave_batch(files)
    assert st == status and all(a.tobytes() == w.tobytes() for a, w in zip(again, want))


def test_progress_sums_to_the_live_files(vg, oracle, three_devices):
    from vgaudio_b200 import containers as ct

    files, meta, _, bad = _wave_job(oracle)
    for opt in (ct.convert_options(ct.CONTAINER_DSP, group_bytes=1 << 20), ct.convert_options(ct.CONTAINER_ADX, group_bytes=300000)):
        seen = []
        _, status = ct.convert_wave_batch(files, opt, progress=seen.append)
        live = sum(1 for s in status if s == 0)
        assert live == len(files) - len(bad)
        assert all(d > 0 for d in seen) and sum(seen) == live, seen


def test_sizing_pass_is_host_only_and_unchanged(vg, oracle, three_devices):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files, meta, _, bad = _wave_job(oracle)
    arrs = [np.ascontiguousarray(f, dtype=np.uint8) for f in files]
    n = len(arrs)
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
    lens = (C.c_int64 * n)(*[a.size for a in arrs])

    def sizing(opt, call="wave"):
        sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
        before = vg.lib.vgb_kernel_launch_count()
        if call == "wave":
            N.check(vg.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(opt), sizes, None, status, None, None))
        else:
            N.check(vg.lib.vgb_convert_dsp_to_wave_batch(ftab, lens, n, sizes, None, status))
        assert vg.lib.vgb_kernel_launch_count() == before
        return list(sizes), list(status)

    for opt in (ct.convert_options(ct.CONTAINER_DSP), ct.convert_options(ct.CONTAINER_ADX), ct.convert_options(ct.CONTAINER_HCA, hca_quality=2)):
        three = sizing(opt)
        assert three == _on_one_device(vg, three_devices, lambda: sizing(opt))  # noqa: B023 (called right here)
        assert all(three[1][k] != 0 and three[0][k] == 0 for k in bad)
    three = sizing(None, "dsp")   # WAVE images are not .dsp files: every one fails alone, on the host
    assert three == _on_one_device(vg, three_devices, lambda: sizing(None, "dsp")) and all(s != 0 for s in three[1])


def test_lifetime_bind_convert_shutdown_rebind(vg, oracle, three_devices):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files, meta, _, _ = _wave_job(oracle)
    opt = ct.convert_options(ct.CONTAINER_DSP, group_bytes=1 << 20)
    dsp_files, _ = _dsp_job(oracle)

    def sequence():
        _bind(vg, three_devices)
        a = ct.convert_wave_batch(files, opt)
        b = ct.convert_dsp_to_wave_batch(dsp_files)
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
        c = ct.convert_wave_batch(files, opt)
        return [x.tobytes() if x is not None else None for r in (a, b, c) for x in r[0]] + [r[1] for r in (a, b, c)]

    first = sequence()
    second = sequence()
    assert first == second
    # the single-shot calls stay on the primary, after all of it
    pcm = _pcm(2, 5000, first=1000)
    coefs, adpcm = _encode_gc(oracle, pcm)
    got = ct.dsp_write_batch([ct.DspFile(adpcm, coefs, 32000, 5000)])
    assert got[0].tobytes() == oracle.dsp_write(adpcm, coefs, 32000, 5000).tobytes()
    _bind(vg, three_devices)
    got = ct.dsp_write_batch([ct.DspFile(adpcm, coefs, 32000, 5000)])
    assert got[0].tobytes() == oracle.dsp_write(adpcm, coefs, 32000, 5000).tobytes()


def test_cli_devices_flag(tmp_path, oracle):
    src = tmp_path / "in"
    src.mkdir()
    for k in range(7):
        ch, n = [1, 2, 3][k % 3], 4000 + 3001 * k
        loop = (101, n - 7) if k % 2 else None
        (src / f"f{k}.wav").write_bytes(oracle.wave_write16(_pcm(ch, n, first=1100 + 5 * k), 16000, loop).tobytes())
    runs = {}
    for name, extra in (("plain", []), ("devices", ["--devices", "0,0"])):
        out = tmp_path / name
        r = subprocess.run([CLI, "-i", str(src), "-o", str(out), "--out-format", "dsp"] + extra, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "7 files converted, 0 failed" in r.stdout, (r.stdout, r.stderr)
        runs[name] = {p.name: p.read_bytes() for p in sorted(out.iterdir())}
    assert len(runs["plain"]) == 7 and runs["plain"] == runs["devices"]
    for bad in ("x", "0,", ""):
        r = subprocess.run([CLI, "--devices", bad, "-i", str(src), "-o", str(tmp_path / "never"), "--out-format", "dsp"], capture_output=True,
                           text=True, timeout=60)
        assert r.returncode != 0 and "usage: vgaudio_batch" in r.stderr and "--devices LIST" in r.stderr, bad
        assert not (tmp_path / "never").exists()
