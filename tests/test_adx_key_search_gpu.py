"""CRI ADX key search on the GPU (vgb_adx_find_keys, vgb_adx_debug_find_keys_box): key sets, search counts and every
confidence field against the C restatement of GuessAdx (oracle/adxkeys.c, bound by adx_key_oracle.py), on images with planted keys - key strings
for revision 8, key codes for revision 9 - of 1, 2 and 6 channels, frame sizes 18 and 12, silent lead-ins
(StartFrame > 0), zero-scale frames inside the audio and short files that many keys fit."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import adx_files as AF
import adx_key_oracle as K
from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")


def planted_key(oracle, revision):
    return oracle.adx_key(key_string=AF.KEY_STRING) if revision == 8 else oracle.adx_key(key_code=AF.KEY_CODE)


def equivalent(key, revision):
    """What the search reports for a planted key: revision 9 reads only the low 13 bits."""
    return key if revision == 8 else tuple(v & 0x1FFF for v in key)


def pcm_with(n, seed, lead=0, gap=None):
    x = synth.channel(seed, n, 48000, degenerate=False).copy()
    x[:lead] = 0
    if gap:
        x[gap[0]:gap[1]] = 0
    return x


def image(oracle, revision, channels, n, frame_size=18, seed=0, lead=0, gap=None):
    pcm = [pcm_with(n, seed + c, lead, gap) for c in range(channels)]
    return AF.encoded(oracle, channels, n, frame_size=frame_size, key=planted_key(oracle, revision), enc_type=revision, pcm=pcm)


def loaded(ct, imgs):
    out = []
    for img in imgs:
        st, _, scales, start = ct.adx_key_load(img)
        assert st == 0
        out.append((scales, start))
    return out


def state_after(key, steps):
    x = key[0]
    for _ in range(steps):
        x = (x * key[1] + key[2]) & 0x7FFF
    return x


def box_around(oracle, revision, files, key, di=(3, 5), dm=(1, 2), dc=(12, 12)):
    """A box that holds the planted key's candidate in file 0's scan."""
    scales, start = files[0]
    k = equivalent(key, revision)
    index = (int(scales[start]) ^ state_after(k, start)) & 0xFFF
    m = int(np.nonzero(K.adx_key_list(revision, 1) == k[1])[0][0])
    c = int(np.nonzero(K.adx_key_list(revision, 2) == k[2])[0][0])
    n_m, n_c = K.adx_key_list(revision, 1).size, K.adx_key_list(revision, 2).size
    return (max(index - di[0], 0), min(index + di[1], 0x1000), max(m - dm[0], 0), min(m + dm[1], n_m), max(c - dc[0], 0), min(c + dc[1], n_c))


def oracle_confidence(oracle, imgs, key):
    """AddKey's sums and confidences (GuessAdx.cs:141-144) from the oracle's GetReencodeConfidence per file."""
    sums = [0, 0, 0, 0]
    for img in imgs:
        st, q = K.adx_key_confidence(img, key)
        if st != 0:
            return None
        sums = [a + b for a, b in zip(sums, q)]
    return sums, 1.0 - sums[0] / sums[1], 1.0 - sums[2] / sums[3]


def bits(x):
    return struct.pack("<d", x)


def check_against_oracle(oracle, ct, revision, imgs, box, max_keys=4096):
    got = ct.adx_find_keys(imgs, box=box, max_keys=max_keys)
    stats = ct.adx_key_search_stats()
    want_keys, want_stats = K.adx_guess_box(revision, loaded(ct, imgs), box)
    assert got.revision == revision and got.file_status == [0] * len(imgs)
    assert [(k.key.seed, k.key.mult, k.key.inc) for k in got.keys] == want_keys
    assert stats == want_stats
    for k in got.keys:
        key = (k.key.seed, k.key.mult, k.key.inc)
        assert k.key_code == ((key[0] << 27) | ((key[1] & 0xFFFC) << 12) | (key[2] >> 1)) + 1
        want = oracle_confidence(oracle, imgs, key)
        assert want is not None and k.status == 0, key
        (ds, ts, df, tf), cs, cf = want
        assert (k.diff_short, k.total_short, k.diff_full, k.total_full) == (ds, ts, df, tf), key
        assert bits(k.confidence_short) == bits(cs) and bits(k.confidence_full) == bits(cf), key
    return got, want_stats


@pytest.mark.parametrize("revision", [8, 9])
def test_box_matches_oracle(vg, oracle, revision):
    from vgaudio_b200 import containers as ct

    imgs = [image(oracle, revision, 2, 3000, seed=1, gap=(900, 1400)),   # zero-scale frames inside the audio
            image(oracle, revision, 1, 2000, seed=5, lead=300),          # a silent lead-in: StartFrame > 0
            image(oracle, revision, 6, 700, frame_size=12, seed=9)]
    files = loaded(ct, imgs)
    assert files[1][1] > 0 and any(int(s) == 0 for s in files[0][0][files[0][1]:])
    key = planted_key(oracle, revision)
    box = box_around(oracle, revision, files, key)
    got, stats = check_against_oracle(oracle, ct, revision, imgs, box)
    assert equivalent(key, revision) in [(k.key.seed, k.key.mult, k.key.inc) for k in got.keys]
    assert stats[0] > 0 and stats[2] >= 1
    # a lead-in file scanned first: FindStartingKey winds the key back
    box = box_around(oracle, revision, files[1:], key)
    got, _ = check_against_oracle(oracle, ct, revision, imgs[1:], box)
    assert equivalent(key, revision) in [(k.key.seed, k.key.mult, k.key.inc) for k in got.keys]


@pytest.mark.parametrize("revision", [8, 9])
def test_short_file_many_keys(vg, oracle, revision):
    """Three frames hold many keys; each gets its own confidence pass.  Past max_keys the call fails and writes nothing."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    img = image(oracle, revision, 1, 90, seed=3)
    files = loaded(ct, [img])
    assert files[0][0].size == 3
    # revision 8 with StartFrame 0 takes only the indices whose seed is a listed prime
    box = (0, 0x1000, 0, 1, 0, 4) if revision == 8 else (0, 8, 0, 4, 0, 24)
    got, _ = check_against_oracle(oracle, ct, revision, [img], box)
    n = len(got.keys)
    assert n > 4
    with pytest.raises(N.VgbError) as e:
        ct.adx_find_keys([img], box=box, max_keys=n - 1)
    assert e.value.code == N.VGB_E_ARG
    # no partial list, whatever the size of the caller's buffer
    f = np.ascontiguousarray(img)
    ftab = (C.c_void_p * 1)(f.ctypes.data)
    lens = (C.c_int64 * 1)(f.size)
    keys = (N.VgbAdxFoundKey * 4)()
    for k in keys:
        k.status = 77
    n_keys = C.c_int32(-1)
    rc = vg.lib.vgb_adx_debug_find_keys_box(ftab, lens, 1, *box, 0, keys, 4, C.byref(n_keys), None, None)
    assert rc == N.VGB_E_ARG and all(k.status == 77 for k in keys)
    assert ct.adx_find_keys([img], box=box, max_keys=n).keys[-1].key.seed == got.keys[-1].key.seed


def test_no_whole_frame_and_failing_reencode(vg, oracle):
    """A file without a frame adds nothing and validates every key; a key whose re-read fails on a file gets that
    status and NaN confidences."""
    from vgaudio_b200 import containers as ct

    good = image(oracle, 9, 2, 1500, seed=2)
    empty = AF.header(samples=0, revision=9)
    files = loaded(ct, [good])
    box = box_around(oracle, 9, files, planted_key(oracle, 9))
    a = ct.adx_find_keys([good], box=box)
    b = ct.adx_find_keys([good, empty], box=box)
    assert [(k.key.seed, k.key.mult, k.key.inc) for k in a.keys] == [(k.key.seed, k.key.mult, k.key.inc) for k in b.keys]
    assert b.file_status == [0, 0]
    # the empty file has no samples: its re-encode reads pcm[0] (CriAdxCodec.cs:69-74) and throws for every key
    assert all(k.status != 0 and np.isnan(k.confidence_full) and np.isnan(k.confidence_short) for k in b.keys)


def test_one_file_scan_gives_the_same_set(vg, oracle):
    """Revision 9 over every scale index: scanning one file finds what every file's scan finds."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    imgs = [image(oracle, 9, 1, 60, seed=4), image(oracle, 9, 2, 500, seed=6, lead=100), image(oracle, 9, 1, 400, seed=8)]
    files = loaded(ct, imgs)
    box = box_around(oracle, 9, files, planted_key(oracle, 9), dm=(2, 2), dc=(6, 6))
    box = (0, 0x1000) + box[2:]
    every, _ = check_against_oracle(oracle, ct, 9, imgs, box)
    one = ct.adx_find_keys(imgs, box=box, flags=N.VGB_ADX_KEYS_ONE_FILE)
    assert [(k.key.seed, k.key.mult, k.key.inc) for k in one.keys] == [(k.key.seed, k.key.mult, k.key.inc) for k in every.keys]
    assert ct.adx_key_search_stats()[0] < K.adx_guess_box(9, files, box)[1][0]


def test_full_revision_8_search_matches_oracle(vg, oracle):
    from vgaudio_b200 import containers as ct

    imgs = [image(oracle, 8, 2, 4000, seed=1), image(oracle, 8, 1, 3000, seed=2)]
    got = ct.adx_find_keys(imgs)
    want, stats = K.adx_guess_box(8, loaded(ct, imgs), (0, 0x1000, 0, 0x400, 0, 0x400))
    assert [(k.key.seed, k.key.mult, k.key.inc) for k in got.keys] == want
    assert ct.adx_key_search_stats() == stats
    assert planted_key(oracle, 8) in want


def test_full_revision_9_search_and_decode(vg, oracle):
    from vgaudio_b200 import containers as ct

    imgs = [image(oracle, 9, 2, 48000, seed=11), image(oracle, 9, 1, 30000, seed=12, lead=2000)]
    got = ct.adx_find_keys(imgs)
    keys = [(k.key.seed, k.key.mult, k.key.inc) for k in got.keys]
    planted = planted_key(oracle, 9)
    assert equivalent(planted, 9) in keys
    for key in keys:
        for scales, _ in loaded(ct, imgs):
            assert K.adx_key_is_valid(9, key, scales)
    # the 13-bit equivalent of the planted 15-bit key decrypts the files byte for byte the same.  (Confidence does not
    # single it out: the key (seed + 1, mult, inc + 1 - mult) keeps the key stream one ahead, so bit 12 agrees on
    # almost every frame, and its re-encode can score as high.)
    found = next(k for k in got.keys if (k.key.seed, k.key.mult, k.key.inc) == equivalent(planted, 9))
    with_found, st1 = ct.convert_adx_to_wave_batch(imgs, found.key)
    with_planted, st2 = ct.convert_adx_to_wave_batch(imgs, ct.adx_key(key_code=AF.KEY_CODE))
    assert st1 == st2 == [0, 0]
    assert all(a.tobytes() == b.tobytes() for a, b in zip(with_found, with_planted))


def test_device_bound_twice_gives_the_same_result(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    imgs = [image(oracle, 8, 2, 4000, seed=1), image(oracle, 8, 1, 3000, seed=2), image(oracle, 8, 1, 64, seed=3)]
    box = (0, 0x1000) + box_around(oracle, 8, loaded(ct, imgs), planted_key(oracle, 8), dm=(8, 8), dc=(8, 8))[2:]
    one = ct.adx_find_keys(imgs, box=box)
    one_stats = ct.adx_key_search_stats()
    N.check(vg.lib.vgb_shutdown())
    try:
        N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
        two = ct.adx_find_keys(imgs, box=box)
        two_stats = ct.adx_key_search_stats()
        full = ct.adx_find_keys(imgs[:2])
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    fields = lambda r: [(k.key.seed, k.key.mult, k.key.inc, k.status, k.key_code, k.diff_short, k.total_short, k.diff_full,
                         k.total_full, bits(k.confidence_short), bits(k.confidence_full)) for k in r.keys]
    assert fields(one) == fields(two) and one_stats == two_stats
    assert planted_key(oracle, 8) in [(k.key.seed, k.key.mult, k.key.inc) for k in full.keys]


@pytest.mark.parametrize("revision", [8, 9])
def test_cli_find_adx_key(vg, oracle, tmp_path, revision):
    src, a, b = tmp_path / "in", tmp_path / "found", tmp_path / "given"
    src.mkdir()
    for i, (ch, n) in enumerate([(2, 20000), (1, 12000), (2, 9000)]):
        (src / f"t{i}.adx").write_bytes(image(oracle, revision, ch, n, seed=20 + i).tobytes())
    key_opt = ["--keystring", AF.KEY_STRING] if revision == 8 else ["--keycode", str(AF.KEY_CODE)]
    r1 = subprocess.run([CLI, "-i", str(src), "-o", str(a), "--out-format", "wav", "--find-adx-key"], capture_output=True, text=True, timeout=600)
    r2 = subprocess.run([CLI, "-i", str(src), "-o", str(b), "--out-format", "wav"] + key_opt, capture_output=True, text=True, timeout=600)
    assert r1.returncode == 0 and r2.returncode == 0, r1.stderr + r2.stderr
    assert "Seed - " in r1.stdout and ("Key code: " in r1.stdout) == (revision == 9)
    assert sorted(p.name for p in a.iterdir()) == sorted(p.name for p in b.iterdir()) == [f"t{i}.wav" for i in range(3)]
    if revision == 8:  # revision 9 decodes with the most confident key, which need not be the planted one's equivalent
        for i in range(3):
            assert (a / f"t{i}.wav").read_bytes() == (b / f"t{i}.wav").read_bytes()
    # without the flag a keyed file still fails
    r3 = subprocess.run([CLI, "-i", str(src), "-o", str(tmp_path / "none"), "--out-format", "wav"], capture_output=True, text=True, timeout=600)
    assert r3.returncode == 3
