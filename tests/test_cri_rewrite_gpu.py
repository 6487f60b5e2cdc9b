"""vgb_rewrite_batch on the device: every .adx and .hca stimulus rewritten byte for byte as the oracle chain writes it
(the reader's restatement, decryption, the writer's restatement, encryption), in mixed batches over several groups, on
two bound devices, and through vgaudio_batch --rewrite."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import adx_files as F
import cri_rewrite_oracle as R
from vgaudio_b200 import _native as N
from vgaudio_b200 import containers as ct
from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")


def _adx_expected(img, opts, key):
    out_key = (opts["adx_key_seed"], opts["adx_key_mult"], opts["adx_key_inc"]) if opts.get("adx_has_key") else None
    return R.expected_adx(img, opts.get("adx_encryption_type", 0), out_key, bool(opts.get("no_trim")), key)


def _adx_key(key):
    return N.VgbAdxKey(*key) if key is not None else None


@pytest.mark.parametrize("case", R.adx_cases(), ids=lambda c: c[0])
def test_adx_bytes(vg, oracle, case):
    name, img, opts, key, _ = case
    want = _adx_expected(img, opts, key)
    outs, status = ct.rewrite_batch([img], ct.convert_options(R.ADX, **opts), adx_key=_adx_key(key))
    assert status == [0], vg.lib.vgb_last_error()
    assert outs[0].tobytes() == want.tobytes()


@pytest.mark.parametrize("case", R.hca_cases(), ids=lambda c: c[0])
def test_hca_bytes(vg, oracle, case):
    name, img, opts, _ = case
    want = R.expected_hca(img, opts["hca_key_type"], opts["hca_key_code"], R.HCA_KEY)
    outs, status = ct.rewrite_batch([img], ct.convert_options(R.HCA, **opts), hca_key_code=R.HCA_KEY)
    assert status == [0], vg.lib.vgb_last_error()
    assert outs[0].tobytes() == want.tobytes()


def _mixed(fmt):
    """Every stimulus of one option set, with refused files between them."""
    k8, k9, k9b = R.adx_keys()
    if fmt == R.ADX:
        opts = R.adx_out(9, k9b)
        imgs = [c[1] for c in R.adx_cases() if c[3] in (None, k9)]
        bad = [c[2] for c in R.refused_cases() if c[1] == R.ADX]
        want = lambda img: _adx_expected(img, opts, k9)  # noqa: E731
    else:
        opts = R.hca_out(56)
        imgs = [c[1] for c in R.hca_cases()]
        bad = [c[2] for c in R.refused_cases() if c[1] == R.HCA and "without key" not in c[0]]
        want = lambda img: R.expected_hca(img, 56, R.HCA_KEY_OUT, R.HCA_KEY)  # noqa: E731
    files = []
    for i, img in enumerate(imgs):
        files.append(img)
        if i < len(bad):
            files.append(bad[i])
    return files, opts, want


@pytest.mark.parametrize("fmt", [R.ADX, R.HCA], ids=["adx", "hca"])
def test_mixed_batch_in_several_groups(vg, oracle, fmt):
    files, opts, want = _mixed(fmt)
    k9 = R.adx_keys()[1]
    expect = [want(f) for f in files]
    assert sum(e is None for e in expect) >= 4
    for group_bytes in (0, 1):  # 1 input byte per group: every file is a group of its own
        seen = []
        o = ct.convert_options(fmt, group_bytes=group_bytes, **opts)
        outs, status = ct.rewrite_batch(files, o, adx_key=_adx_key(k9), hca_key_code=R.HCA_KEY, progress=seen.append)
        for e, out, st in zip(expect, outs, status):
            assert (st == 0) == (e is not None)
            if e is not None:
                assert out.tobytes() == e.tobytes()
        assert sum(seen) == sum(e is not None for e in expect) and all(d > 0 for d in seen)
        if group_bytes:
            assert seen == [1] * sum(e is not None for e in expect)


def test_two_devices_same_bytes(vg, oracle):
    files, opts, _ = _mixed(R.HCA)
    adx_files, adx_opts, _ = _mixed(R.ADX)
    k9 = R.adx_keys()[1]
    one = [ct.rewrite_batch(files, ct.convert_options(R.HCA, **opts), hca_key_code=R.HCA_KEY),
           ct.rewrite_batch(adx_files, ct.convert_options(R.ADX, **adx_opts), adx_key=_adx_key(k9))]
    N.check(vg.lib.vgb_shutdown())
    N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
    try:
        assert vg.lib.vgb_device_count() == 2
        two = [ct.rewrite_batch(files, ct.convert_options(R.HCA, **opts), hca_key_code=R.HCA_KEY),
               ct.rewrite_batch(adx_files, ct.convert_options(R.ADX, **adx_opts), adx_key=_adx_key(k9))]
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    for (o1, s1), (o2, s2) in zip(one, two):
        assert s1 == s2
        assert [o.tobytes() if o is not None else None for o in o1] == [o.tobytes() if o is not None else None for o in o2]


def _run(*args):
    r = subprocess.run([CLI, *map(str, args)], capture_output=True, text=True, timeout=600)
    return r


def test_cli_rewrite_hca(tmp_path, oracle):
    src = tmp_path / "in"
    src.mkdir()
    imgs = {}
    for i in range(3):  # encoded frames: the key search unpacks them
        pcm = [synth.channel(50 + 2 * i + c, 20000 + 7000 * i, 44100, degenerate=False) for c in range(2)]
        info, frames = oracle.hca_encode(pcm, 44100, loop=(3000, 18000) if i == 1 else None)
        imgs[f"k{i}.hca"] = R.hca_source(info, frames, ciph=56, comment=b"cli")
    info = R.hca_info(frame_count=4)
    imgs["plain.hca"] = R.hca_source(info, R.hca_frames(info, 60), ciph=1)
    for name, img in imgs.items():
        (src / name).write_bytes(img.tobytes())
    (src / "x.wav").write_bytes(oracle.wave_write16([np.zeros(100, np.int16)], 32000).tobytes())
    keys = tmp_path / "keys.txt"
    keys.write_text(f"# keys\n12345\n0x{R.HCA_KEY:016X}\n999\n")
    # decrypted with the key found in the list; a .wav input still goes through the encoder
    out = tmp_path / "plain"
    r = _run("-i", src, "-o", out, "--out-format", "hca", "--rewrite", "--hca-keys", keys)
    assert r.returncode == 0 and "5 files converted, 0 failed" in r.stdout and "list entry 1): 3 files" in r.stdout, r.stdout + r.stderr
    for name, img in imgs.items():
        assert (out / name).read_bytes() == R.expected_hca(img, in_key_code=R.HCA_KEY).tobytes(), name
    # the same with the input key given, re-keyed with --keycode
    out2 = tmp_path / "rekeyed"
    r = _run("-i", src, "-o", out2, "--out-format", "hca", "--rewrite", "--in-keycode", R.HCA_KEY, "--keycode", R.HCA_KEY_OUT)
    assert r.returncode == 0, r.stdout + r.stderr
    for name, img in imgs.items():
        assert (out2 / name).read_bytes() == R.expected_hca(img, 56, R.HCA_KEY_OUT, R.HCA_KEY).tobytes(), name
    # without --rewrite the .hca files are not listed
    r = _run("-i", src, "-o", tmp_path / "none", "--out-format", "hca", "--hca-keys", keys)
    assert r.returncode == 0 and "1 files converted" in r.stdout and not (tmp_path / "none" / "k0.hca").exists(), r.stdout
    assert _run("-i", src, "-o", tmp_path / "bad", "--out-format", "dsp", "--rewrite").returncode == 2


def test_cli_rewrite_adx_found_key(tmp_path, oracle, vg):
    k8, k9, _ = R.adx_keys()
    src = tmp_path / "in"
    src.mkdir()
    imgs = {f"t{i}.adx": F.encoded(oracle, ch, n, key=k9, enc_type=9, seed=70 + i, loop=(300, n - 50) if i == 1 else None)
            for i, (ch, n) in enumerate([(2, 20000), (1, 12000), (2, 9000)])}
    for name, img in imgs.items():
        (src / name).write_bytes(img.tobytes())
    # the key the CLI picks: highest full confidence, then short, then the lowest (the search returns them sorted)
    search = ct.adx_find_keys(list(imgs.values()))
    ok = [k for k in search.keys if k.status == 0]
    best = max(ok, key=lambda k: (k.confidence_full, k.confidence_short, -ok.index(k)))
    found = (best.key.seed, best.key.mult, best.key.inc)
    out = tmp_path / "rekeyed"
    r = _run("-i", src, "-o", out, "--out-format", "adx", "--rewrite", "--find-adx-key", "--keystring", R.ADX_KEY_STRING)
    assert r.returncode == 0 and "3 files converted, 0 failed" in r.stdout and "Key code: " in r.stdout, r.stdout + r.stderr
    for name, img in imgs.items():
        assert (out / name).read_bytes() == R.expected_adx(img, 8, k8, False, found).tobytes(), name
    # --in-keycode names the key; the output in the clear
    out2 = tmp_path / "plain"
    r = _run("-i", src, "-o", out2, "--out-format", "adx", "--rewrite", "--in-keycode", R.ADX_KEY_CODE)
    assert r.returncode == 0, r.stdout + r.stderr
    for name, img in imgs.items():
        assert (out2 / name).read_bytes() == R.expected_adx(img, in_key=k9).tobytes(), name
    # without --rewrite the .adx files are not listed
    r = _run("-i", src, "-o", tmp_path / "none", "--out-format", "adx", "--in-keycode", R.ADX_KEY_CODE)
    assert r.returncode == 0 and "0 files converted" in r.stdout, r.stdout
