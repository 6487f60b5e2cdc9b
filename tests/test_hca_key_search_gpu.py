"""CRI HCA key search on the GPU (vgb_hca_find_keys, vgb_hca_debug_key_outcomes): every (file, key) outcome and each
file's first index against the C restatement of HcaReader.FindKey (oracle/hcakeys.c, bound by hca_key_oracle.py), on
type-56 images of 1..8 channels with intensity-stereo and HFR layouts, silent lead-ins, short files, a window that ends
at the end of the file, a bad sync word, all-empty and frameless files, equivalent codes and random decoys."""
import ctypes as C
import os

import numpy as np
import pytest

import hca_key_oracle as K

pytestmark = pytest.mark.gpu
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vgaudio_b200", "cli", "vgaudio_batch")


@pytest.fixture(scope="module")
def files(oracle):
    return K.key_files(oracle)


def _oracle_matrix(imgs, keys):
    return np.stack([K.image_outcomes(img, keys) for img in imgs])


@pytest.mark.parametrize("at,n", [("start", 64), ("middle", 160), ("end", 256)])
def test_outcome_matrix_matches_oracle(vg, oracle, files, at, n):
    from vgaudio_b200 import containers as ct

    imgs = [img for _, img in files]
    keys = K.key_list(n, 100 + n, planted=(K.KEY, K.KEY2), at=at)
    got = ct.hca_key_outcomes(imgs, keys)
    want = _oracle_matrix(imgs, keys)
    bad = np.argwhere(got != want)
    assert bad.size == 0, [(files[f][0], k, int(got[f, k]), int(want[f, k])) for f, k in bad[:10]]
    pairs, frames, searched, _ = ct.hca_key_search_stats()
    assert searched == sum(1 for img in imgs if K.split(img)[1] == 56)
    assert pairs == searched * len(keys)
    # every outcome kind is on the matrix
    kinds = {int(v) if v <= 0 else (int(v) - 1) % 3 + 1 for v in want.ravel()}
    assert {-1, 0, 1, 2, 3} <= kinds, kinds


@pytest.mark.parametrize("at,n", [("start", 64), ("middle", 160), ("end", 256)])
def test_first_index_matches_oracle(vg, oracle, files, at, n):
    from vgaudio_b200 import containers as ct

    imgs = [img for _, img in files] + [np.frombuffer(b"not an hca file at all", np.uint8)]
    keys = K.key_list(n, 200 + n, planted=(K.KEY, K.KEY2), at=at)
    idx, status = ct.hca_find_keys(imgs, keys)
    for i, img in enumerate(imgs[:-1]):
        assert (idx[i], status[i]) == K.image_find_key(img, keys), files[i][0]
    assert idx[-1] == -1 and status[-1] < 0
    names = [name for name, _ in files]
    # the first of KEY and its equivalent code wins; the bad sync is an error; the all-empty and frameless files take key 0
    first = min(keys.index(K.KEY), keys.index(K.equivalent(K.KEY)))
    assert idx[names.index("enc_2ch_q3_44100")] == first
    assert status[names.index("bad_sync_4")] == -2
    assert idx[names.index("all_empty")] == 0 and idx[names.index("no_frames")] == 0
    assert status[names.index("plain")] == 1


def test_no_keys_and_unlisted_key(vg, oracle, files):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    imgs = [img for _, img in files]
    idx, status = ct.hca_find_keys(imgs, [])
    for i, img in enumerate(imgs):
        assert idx[i] == -1
        assert status[i] == (N.VGB_HCA_KEY_NOT_FOUND if K.split(img)[1] == 56 else N.VGB_HCA_KEY_SKIPPED)
    keys = K.key_list(64, 7, planted=(K.KEY,))
    idx, status = ct.hca_find_keys(imgs, keys)
    names = [name for name, _ in files]
    assert status[names.index("key2")] == N.VGB_HCA_KEY_NOT_FOUND
    assert (idx[names.index("key2")], status[names.index("key2")]) == K.image_find_key(files[names.index("key2")][1], keys)


def test_shuffled_keys_permute_the_matrix(vg, oracle, files):
    from vgaudio_b200 import containers as ct

    imgs = [img for _, img in files]
    keys = K.key_list(200, 31, planted=(K.KEY, K.KEY2))
    perm = np.random.default_rng(5).permutation(len(keys))
    a = ct.hca_key_outcomes(imgs, keys)
    b = ct.hca_key_outcomes(imgs, [keys[p] for p in perm])
    assert np.array_equal(a[:, perm], b)


def test_large_job_matches_oracle(vg, oracle):
    """256 files x 1024 keys, four distinct planted keys at different places in the list."""
    from vgaudio_b200 import containers as ct

    rng = np.random.default_rng(77)
    planted = [K.KEY, K.KEY2, 0x0123456789ABCDEF, 0x0000BEEF00C0FFEE]
    keys = K.key_list(1024, 78, planted=tuple(planted), at="end")
    for p, pos in zip(planted, (10, 300, 700)):
        keys.remove(p)
        keys.insert(pos, p)
    bases = []
    for i in range(8):
        ch = 1 + i % 2
        info, frames = oracle.hca_encode(K._pcm(ch, 6000 + 3000 * i, 48000, 300 + i), 48000, 1 + i % 5)
        bases.append((info, frames))
    imgs = []
    for f in range(256):
        info, frames = bases[f % 8]
        imgs.append(K.keyed(oracle, info, frames, planted[int(rng.integers(0, 4))]))
    idx, status = ct.hca_find_keys(imgs, keys)
    sample = list(range(0, 256, 8))
    for f in sample:
        assert (idx[f], status[f]) == K.image_find_key(imgs[f], keys), f
    assert all(s == 0 for s in status)
    for f in range(256):
        assert keys[idx[f]] in planted or K.equivalent(keys[idx[f]]) in planted


def test_device_bound_twice_gives_the_same_result(vg, oracle, files):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    imgs = [img for _, img in files]
    keys = K.key_list(128, 41, planted=(K.KEY, K.KEY2), at="middle")
    one = ct.hca_find_keys(imgs, keys)
    one_m = ct.hca_key_outcomes(imgs, keys)
    N.check(vg.lib.vgb_shutdown())
    try:
        N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
        two = ct.hca_find_keys(imgs, keys)
        two_m = ct.hca_key_outcomes(imgs, keys)
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    assert one == two
    assert np.array_equal(one_m, two_m)


def _expected_wave(oracle, img, key_code):
    """The reader chain on the CPU for one .hca image: decrypt with key_code when it is type 56, decode, WaveWriter."""
    info, ciph, frames = K.split(img)
    if ciph == 56:
        frames = oracle.hca_crypt_frames(frames, info.frame_size, oracle.hca_key_tables(56, key_code)[0]).reshape(frames.shape)
    pcm = oracle.hca_decode(info, frames)
    return oracle.wave_write16(list(pcm), info.sample_rate, None)


def _cli_dir(oracle, tmp_path):
    src = tmp_path / "in"
    src.mkdir()
    made = {}
    for name, ch, n, seed, key in (("a", 2, 20000, 1, K.KEY), ("b", 1, 15000, 2, K.KEY2), ("c", 2, 9000, 3, K.KEY),
                                   ("d", 1, 8000, 4, 0x0000777700007777), ("e", 1, 7000, 5, None)):
        info, frames = oracle.hca_encode(K._pcm(ch, n, 48000, 40 + seed), 48000, 2)
        img = K.keyed(oracle, info, frames, key) if key else oracle.hca_write(info, frames)
        (src / f"{name}.hca").write_bytes(img.tobytes())
        made[name] = (img, key)
    keys = tmp_path / "keys.txt"
    keys.write_text("# two of the three keys\n\n" + "\n".join(str(v) for v in K.key_list(40, 9, planted=(K.KEY,), at="middle")[:-1])
                    + f"\n0x{K.KEY:X}\n{K.KEY2}\n")
    return src, keys, made


def test_cli_hca_keys_to_wave(vg, oracle, tmp_path):
    import subprocess

    src, keys, made = _cli_dir(oracle, tmp_path)
    out = tmp_path / "out"
    r = subprocess.run([CLI, "-i", str(src), "-o", str(out), "--out-format", "wav", "--hca-keys", str(keys)], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 3, (r.stdout, r.stderr)      # one file failed
    assert "Error converting d.hca" in r.stderr
    assert "4 files converted, 1 failed" in r.stdout
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("HCA key")]
    assert len(lines) == 2 and any(ln.endswith(": 2 files") for ln in lines) and any(ln.endswith(": 1 files") for ln in lines)
    for name in "abce":
        img, key = made[name]
        assert (out / f"{name}.wav").read_bytes() == _expected_wave(oracle, img, key).tobytes(), name
    assert not (out / "d.wav").exists()


def test_cli_hca_keys_transcode(vg, oracle, tmp_path):
    """.hca -> .adx with the list gives the files a given --in-keycode gives."""
    import subprocess

    src, keys, made = _cli_dir(oracle, tmp_path)
    found, given = tmp_path / "found", tmp_path / "given"
    r = subprocess.run([CLI, "-i", str(src), "-o", str(found), "--out-format", "adx", "--hca-keys", str(keys)], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 3 and "Error converting d.hca" in r.stderr, (r.stdout, r.stderr)
    for key, names in ((K.KEY, "ac"), (K.KEY2, "b")):
        one = tmp_path / f"one_{key}"
        one.mkdir()
        for nm in names:
            (one / f"{nm}.hca").write_bytes(made[nm][0].tobytes())
        r2 = subprocess.run([CLI, "-i", str(one), "-o", str(given), "--out-format", "adx", "--in-keycode", str(key)], capture_output=True,
                            text=True, timeout=300)
        assert r2.returncode == 0, r2.stderr
        for nm in names:
            assert (found / f"{nm}.adx").read_bytes() == (given / f"{nm}.adx").read_bytes(), nm
