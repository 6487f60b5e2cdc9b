"""CRI ADX key search (GuessAdx.cs), CPU side: the C oracle against a plain-Python restatement on tiny boxes, the
candidate lists, KeyCode, the host-side file loading of vgb_adx_key_load against the oracle's LoadFiles, and the
deliberate differences the call decides before it touches a device."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import adx_files as AF
import adx_key_oracle as K
from oracle import pyoracle as O
from vgaudio_b200 import _native as N
from vgaudio_b200 import containers as ct

MASK = {8: 0xE000, 9: 0x1000}
MAX_SEED = {8: 0x8000, 9: 0x2000}


def py_lists(revision):
    """GuessAdx.cs:48-71, from a sieve of its own."""
    if revision == 8:
        sieve = np.ones(0x8000, dtype=bool)
        sieve[:2] = False
        for i in range(2, 0xB6):
            if sieve[i]:
                sieve[i * i::i] = False
        primes = [int(p) for p in np.nonzero(sieve)[0] if p >= 0x4000][:0x400]
        return primes, primes, primes
    return list(range(0x2000)), [x for x in range(0x2000) if x & 3 == 1], [x for x in range(0x2000) if x & 1]


def py_guess(revision, files, box):
    """Run / TryScale / FindStartingKey / AddKey over a box, restated from the C#."""
    seeds, mults, incs = py_lists(revision)
    seed_set = set(seeds)
    mask, smask = MASK[revision], MAX_SEED[revision] - 1
    i0, i1, m0, m1, c0, c1 = box
    tried, keys, stats = set(), [], [0, 0, 0]

    def valid(key, scales):
        x = key[0]
        for s in scales:
            if ((s ^ x) & mask) != 0 and s != 0:
                return False
            x = (x * key[1] + key[2]) & 0x7FFF
        return True

    for index in range(i0, i1):
        for scales, start in files:
            if len(scales) == 0:
                continue
            seed = (int(scales[start]) ^ index) & smask
            if start == 0 and seed not in seed_set:
                continue
            for mult in mults[m0:m1]:
                for inc in incs[c0:c1]:
                    x, ok = seed, True
                    stats[0] += 1
                    for s in scales[start:]:
                        stats[1] += 1
                        if ((int(s) ^ x) & mask) != 0 and s != 0:
                            ok = False
                            break
                        x = (x * mult + inc) & 0x7FFF
                    if not ok:
                        continue
                    stats[2] += 1
                    real = seed if start == 0 else None
                    if start > 0:
                        for r in seeds:
                            y = r
                            for _ in range(start):
                                y = (y * mult + inc) & 0x7FFF
                            if (y & smask) == seed:
                                real = r
                                break
                    if real is None:
                        continue
                    key = (real, mult, inc)
                    if key in tried:
                        continue
                    tried.add(key)
                    if all(valid(key, [int(v) for v in s]) for s, _ in files):
                        keys.append(key)
    return sorted(keys), tuple(stats)


def key_code(key):
    """CriAdxKey.KeyCode (CriAdxKey.cs:48-57)."""
    return ((key[0] << 27) | ((key[1] & 0xFFFC) << 12) | (key[2] >> 1)) + 1


def keyed(channels, n, revision, frame_size=18, seed=0, pcm=None):
    key = O.adx_key(key_string=AF.KEY_STRING) if revision == 8 else O.adx_key(key_code=AF.KEY_CODE)
    return AF.encoded(O, channels, n, frame_size=frame_size, key=key, enc_type=revision, seed=seed, pcm=pcm), key


def test_lists():
    for rev in (8, 9):
        for which, want in enumerate(py_lists(rev)):
            got = K.adx_key_list(rev, which)
            assert got.tolist() == want
    primes = K.adx_key_list(8, 1)
    assert primes.size == 0x400 and primes[0] == 16411 and primes[-1] == 26681
    assert K.adx_key_list(9, 0).size == 0x2000 and K.adx_key_list(9, 1).size == 0x800 and K.adx_key_list(9, 2).size == 0x1000


def test_key_code_round_trip():
    rng = np.random.default_rng(5)
    for _ in range(200):
        key = (int(rng.integers(0, 0x2000)), int(rng.integers(0, 0x800)) * 4 + 1, int(rng.integers(0, 0x1000)) * 2 + 1)
        k = ct.adx_key(key_code=key_code(key))
        assert (k.seed, k.mult, k.inc) == key
    # the 15-bit key of a code keeps its KeyCode through vgb_adx_key_from_code
    k = ct.adx_key(key_code=AF.KEY_CODE)
    k2 = ct.adx_key(key_code=key_code((k.seed, k.mult, k.inc)))
    assert (k2.seed, k2.mult, k2.inc) == (k.seed, k.mult, k.inc)


@pytest.mark.parametrize("revision", [8, 9])
def test_oracle_against_restatement(revision):
    """Short files (a few frames) match many candidates; a silent lead-in makes StartFrame > 0."""
    seeds, mults, incs = py_lists(revision)
    rng = np.random.default_rng(revision)
    for trial in range(4):
        pcm = [np.concatenate([np.zeros(64 * (trial % 2), np.int16), (rng.normal(0, 3000, 64 + 32 * trial)).astype(np.int16)])]
        img, key = keyed(1, pcm[0].size, revision, pcm=pcm)
        st, rev, scales, start = ct.adx_key_load(img)
        assert st == 0 and rev == revision and (start > 0) == (trial % 2 == 1)
        files = [(scales, start)]
        m = mults.index(key[1]) if key[1] in mults else 0
        c = incs.index(key[2]) if key[2] in incs else 0
        box = (0, 24, max(m - 2, 0), m + 2, max(c - 8, 0), c + 8)
        want = py_guess(revision, files, box)
        got = K.adx_guess_box(revision, files, box)
        assert got == want


def test_loading_against_oracle():
    imgs = []
    for rev in (8, 9):
        imgs.append(keyed(2, 700, rev)[0])
        imgs.append(keyed(1, 300, rev, frame_size=12, pcm=[np.concatenate([np.zeros(200, np.int16), np.full(100, 900, np.int16)])])[0])
    imgs.append(AF.header(samples=0, revision=8))                    # no audio: no frame
    imgs.append(AF.header(samples=500, revision=9)[:60])             # short image: the rest reads as zeros
    imgs.append(AF.header(samples=100, revision=9))                  # all-zero audio: StartFrame 0
    imgs.append(np.zeros(3, np.uint8))                               # not an ADX file
    imgs.append(AF.header(frame_size=0, revision=9))                 # frame size 0
    for img in imgs:
        for rev in (0, 8, 9):
            st, r, scales, start = ct.adx_key_load(img, rev)
            ost, otype, oscales, ostart, _ = K.adx_key_load(img, rev)
            assert (st == 0) == (ost == 0) and (st == N.VGB_ADX_KEY_SKIPPED) == (ost == 1), (st, ost)
            assert r == otype
            if st == 0:
                assert scales.tolist() == oscales.tolist() and start == ostart


def test_mixed_revisions_and_unreadable_files():
    """Without a device: unreadable files get their status and are left out; the revision comes from the first file
    read, and while it is 0 the next file sets it (a revision-0 file read first is kept, as in LoadFiles); files of
    another revision are skipped; a first revision other than 8 / 9 fails the call with VGB_E_ARG."""
    bad = np.frombuffer(b"RIFF....", np.uint8).copy()
    plain = AF.encoded(O, 1, 200)
    rev3 = AF.header(samples=64, revision=3)
    good8, good9 = keyed(1, 200, 8)[0], keyed(1, 200, 9)[0]
    for files, want_status, want_rev in [([bad, plain], [N.VGB_E_DATA, 0], 0),
                                         ([rev3, good8, bad], [0, N.VGB_ADX_KEY_SKIPPED, N.VGB_E_DATA], 3),
                                         ([], [], 0)]:
        n = len(files)
        ftab = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in files])
        lens = (C.c_int64 * max(n, 1))(*[a.size for a in files])
        status = (C.c_int32 * max(n, 1))()
        n_keys, rev = C.c_int32(-1), C.c_int32(-1)
        rc = N.lib.vgb_adx_find_keys(ftab, lens, n, None, 0, C.byref(n_keys), status, C.byref(rev))
        assert rc == N.VGB_E_ARG and rev.value == want_rev and n_keys.value == 0
        assert [status[i] for i in range(n)] == want_status
    # LoadFiles' rule, file after file
    st, rev, _, _ = ct.adx_key_load(plain, 0)
    assert st == 0 and rev == 0
    st, rev, _, _ = ct.adx_key_load(good8, rev)
    assert st == 0 and rev == 8
    st, rev, _, _ = ct.adx_key_load(good9, rev)
    assert st == N.VGB_ADX_KEY_SKIPPED and rev == 8


def test_box_out_of_range_is_refused():
    img = keyed(1, 100, 9)[0]
    for box in [(0, 0x1001, 0, 1, 0, 1), (5, 4, 0, 1, 0, 1), (0, 1, 0, 0x801, 0, 1), (0, 1, 0, 1, 0, 0x1001), (-1, 1, 0, 1, 0, 1)]:
        with pytest.raises(N.VgbError) as e:
            ct.adx_find_keys([img], box=box)
        assert e.value.code == N.VGB_E_ARG


def test_key_is_valid_matches_restatement():
    img, key = keyed(2, 900, 8)
    _, _, scales, _ = ct.adx_key_load(img)
    assert K.adx_key_is_valid(8, key, scales)
    other = next(p for p in K.adx_key_list(8, 2) if p != key[2])
    assert K.adx_key_is_valid(8, (key[0], key[1], int(other)), scales) == py_guess_valid(8, (key[0], key[1], int(other)), scales)


def py_guess_valid(revision, key, scales):
    x = key[0]
    for s in scales:
        if ((int(s) ^ x) & MASK[revision]) != 0 and s != 0:
            return False
        x = (x * key[1] + key[2]) & 0x7FFF
    return True
