"""CRI HCA key search (HcaReader.FindKey), CPU side: the C oracle (oracle/hcakeys.c) against a plain-Python restatement
of TestKey and UnpackFrame on keyed images, structured frames with faults and random bytes; the coverage of every way a
key test ends, proven from the oracle's Remaining values; FindFirstNonEmptyFrame's window; and what vgb_hca_find_keys
decides before it touches a device (files that are not searched, n_keys == 0)."""
from __future__ import annotations

import json
import os

import numpy as np
import pytest

import hca_key_oracle as K
import hca_stimuli as H
from oracle import pyoracle as O
from vgaudio_b200 import _native as N
from vgaudio_b200 import containers as ct

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "hca_tables.json")))["unpacked"]
MAX_BITS = GOLD["QuantizedSpectrumMaxBits"]
SPEC_BITS = GOLD["QuantizedSpectrumBits"]
CURVE = GOLD["ScaleToResolutionCurve"]
ATH = GOLD["AthCurve"]


def crc16(data) -> int:
    """Crc16 (Utilities/Crc16.cs), polynomial 0x8005, initial value 0."""
    crc = 0
    for b in data:
        crc ^= int(b) << 8
        for _ in range(8):
            crc = ((crc << 1) ^ 0x8005) & 0xFFFF if crc & 0x8000 else (crc << 1) & 0xFFFF
    return crc


def ath_curve(info):
    """CriHcaFrame.AthCurve (CriHcaFrame.cs:31, ScaleAthCurve :60-84)."""
    if not info.use_ath_curve:
        return [0] * 128
    out, acc = [], 0
    for _ in range(128):
        acc += info.sample_rate
        i = acc >> 13
        if i >= len(ATH):
            break
        out.append(ATH[i])
    return out + [0xFF] * (128 - len(out))


def unpack(info, buf):
    """CriHcaPacking.UnpackFrame (CriHcaPacking.cs:10-229) on one decrypted frame: ("sync" | "delta" | "ok", remaining,
    noise level, FrameEmpty).  Bits past the end read as zero (BitReader.PeekInt)."""
    bits = np.unpackbits(np.asarray(buf, dtype=np.uint8))
    n = bits.size
    pos = 0

    def peek(count):
        v = 0
        for i in range(count):
            v = (v << 1) | (int(bits[pos + i]) if pos + i < n else 0)
        return v

    def read(count):
        nonlocal pos
        v = peek(count)
        pos += count
        return v

    if read(16) != 0xFFFF:
        return "sync", None, None, None
    noise, boundary = read(9), read(7)
    ath = ath_curve(info)
    types = H.channel_types(info)
    res_all, deltas = [], []
    for t in types:
        coded = H.coded_count(info, t)
        db = read(3)
        deltas.append(db)
        sfs = [0] * 128
        if db >= 6:
            for i in range(coded):
                sfs[i] = read(6)
        elif db > 0:
            sfs[0] = read(6)
            max_delta = 1 << (db - 1)
            for i in range(1, coded):
                d = read(db) - (max_delta - 1)
                if d < max_delta:
                    v = sfs[i - 1] + d
                    if v < 0 or v > 63:
                        return "delta", None, None, None
                    sfs[i] = v
                else:
                    sfs[i] = read(6)
        res = []
        for i in range(coded):
            if sfs[i] == 0:
                res.append(0)
            else:
                p = ath[i] + noise - (1 if i < boundary else 0) - 5 * sfs[i] // 2 + 2
                res.append(CURVE[min(max(p, 0), 58)])
        res_all.append(res)
        if t == 2:
            pos += 4 * 8
        elif info.hfr_group_count > 0:
            pos += 6 * info.hfr_group_count
    for _ in range(8):
        for res in res_all:
            for r in res:
                b = MAX_BITS[r]
                code = peek(b)
                if r < 8:
                    b = SPEC_BITS[r][code]
                elif code // 2 == 0:
                    b -= 1
                pos += b
    empty = noise == 0 and all(d == 0 for d in deltas)
    return "ok", n - pos, noise, empty


def py_test_key(info, frames, table, no_crc=False):
    """TestKey (CriHcaEncryption.cs:48-63) with FindFirstNonEmptyFrame: (outcome, [(remaining, noise, empty)])."""
    start = next((i for i, f in enumerate(frames) if f[2:-2].any()), 0)
    end = min(len(frames), start + 10)
    seen = []
    for i in range(start, end):
        j = i - start
        buf = np.array(frames[i], dtype=np.uint8)
        buf[:-2] = table[buf[:-2]]
        if not no_crc:
            c = crc16(buf[:-2])
            buf[-2], buf[-1] = c >> 8, c & 0xFF
        kind, rem, noise, empty = unpack(info, buf)
        if kind == "sync":
            return 1 + 3 * j, seen
        if kind == "delta":
            return 2 + 3 * j, seen
        seen.append((rem, noise, empty))
        if not ((16 <= rem <= 128) or empty or (noise == 0 and rem >= 16)):
            return 3 + 3 * j, seen
    return 0, seen


def cpu_stimuli():
    """(name, info, encrypted frames): the key-search images, structured frames with faults and random bytes, encrypted
    with KEY the way HcaWriter does."""
    out = []
    for name, img in K.key_files(O):
        info, ciph, frames = K.split(img)
        if ciph == 56:
            out.append((name, info, frames))
    enc = O.hca_key_tables(56, K.KEY)[1]
    for name, info, stream, fault in H.fault_cases():
        for s, fr in enumerate(H.fault_streams(info, stream, fault, seed=900 + len(out))):
            out.append((f"{name}_{s}", info, O.hca_crypt_frames(fr, info.frame_size, enc).reshape(fr.shape)))
    rng = np.random.default_rng(4)
    for name, info in H.decoder_layouts()[::4]:
        fr = rng.integers(0, 256, size=(6, info.frame_size), dtype=np.uint8)
        fr[:, :2] = 0xFF
        out.append((f"random_{name}", info, fr))
    return out


@pytest.fixture(scope="module")
def stimuli():
    return cpu_stimuli()


def keys_for(i):
    return [K.KEY, K.equivalent(K.KEY), K.KEY + 1] + [int(v) for v in np.random.default_rng(50 + i).integers(1, 1 << 62, size=5)]


def test_oracle_matches_python_restatement(stimuli):
    for i, (name, info, frames) in enumerate(stimuli[::3]):
        keys = keys_for(i)
        got, rem = K.outcomes(info, frames, keys)
        for k, code in enumerate(keys):
            want, seen = py_test_key(info, frames, O.hca_key_tables(56, code)[0])
            assert got[k] == want, (name, k)
            assert [r for r in rem[k] if r != K.NO_REMAINING] == [s[0] for s in seen], (name, k)


def test_every_way_a_key_test_ends_is_covered(stimuli):
    """From the oracle's Remaining values (and the restatement's noise level, which agrees with the oracle above)."""
    seen = set()
    crc_flips = 0
    for i, (name, info, frames) in enumerate(stimuli):
        keys = keys_for(i) + [int(v) for v in np.random.default_rng(70 + i).integers(1, 1 << 62, size=24)]
        out, rem = K.outcomes(info, frames, keys)
        raw, _ = K.outcomes(info, frames, keys, no_crc=True)
        crc_flips += int(np.sum(out != raw))
        for k in range(len(keys)):
            r = out[k] if out[k] <= 0 else (out[k] - 1) % 3 + 1
            seen.add({0: "pass", 1: "sync", 2: "delta", 3: "unsuccessful"}[int(r)])
            for j in np.nonzero(rem[k] != K.NO_REMAINING)[0]:
                v = int(rem[k][j])
                if 16 <= v <= 128:
                    seen.add("remaining 16..128")
                if v < 16:
                    seen.add("remaining < 16")
        # the noise-level cases need the frames' fields: the restatement on this file's first keys
        for code in keys[:3]:
            _, frames_seen = py_test_key(info, frames, O.hca_key_tables(56, code)[0])
            for v, noise, empty in frames_seen:
                if empty:
                    seen.add("pass through FrameEmpty")
                elif noise == 0 and v > 128:
                    seen.add("noise 0, remaining > 128")
                elif noise > 0 and v > 128:
                    seen.add("noise > 0, remaining > 128")
    assert crc_flips > 0
    assert {"pass", "sync", "delta", "unsuccessful", "remaining 16..128", "remaining < 16", "pass through FrameEmpty",
            "noise 0, remaining > 128", "noise > 0, remaining > 128"} <= seen, seen


def test_window_selection():
    fs = 64
    frames = np.zeros((14, fs), dtype=np.uint8)
    frames[:, :2] = 0xFF
    frames[:, -2:] = 0x55          # the CRC bytes do not count
    assert K.window(frames) == (0, 10)  # every frame empty: frame 0
    frames[3, 2] = 1
    assert K.window(frames) == (3, 13)
    frames[3, 2] = 0
    frames[6, fs - 3] = 9
    assert K.window(frames) == (6, 14)  # the window ends at the end of the file
    assert K.window(frames[:0]) == (0, 0)


def test_statuses_decided_on_the_host():
    """Without keys every type-56 file is NOT_FOUND; other types are SKIPPED; unreadable files keep their error.  None
    of this reaches a device."""
    imgs = [img for _, img in K.key_files(O)] + [np.frombuffer(b"HCA\0 short", np.uint8)]
    idx, status = ct.hca_find_keys(imgs, [])
    for i, img in enumerate(imgs[:-1]):
        assert idx[i] == -1
        assert status[i] == (N.VGB_HCA_KEY_NOT_FOUND if K.split(img)[1] == 56 else N.VGB_HCA_KEY_SKIPPED)
    assert idx[-1] == -1 and status[-1] == N.VGB_E_DATA
    assert ct.hca_key_outcomes(imgs, []).shape == (len(imgs), 0)


def test_zero_frames_and_all_empty_pass_the_first_key():
    names = dict(K.key_files(O))
    keys = [123, K.KEY, 456]
    for name in ("no_frames", "all_empty"):
        info, _, frames = K.split(names[name])
        assert K.find_key(info, frames, keys) == (0, 0)
        assert list(K.outcomes(info, frames, keys)[0]) == [0, 0, 0]


CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vgaudio_b200", "cli", "vgaudio_batch")


@pytest.mark.parametrize("text,line", [("# keys\n\n123\n0x1F\nzz\n", 5), ("  42  \n-3\n", 2), ("0x\n", 1),
                                       ("18446744073709551616\n", 1), ("0xFFFFFFFFFFFFFFFF\n12 34\n", 2)])
def test_cli_key_list_errors_name_the_line(tmp_path, text, line):
    """--hca-keys: a line that is not a decimal or 0x-hex code is an error naming its line, before any device is used."""
    import subprocess

    keys = tmp_path / "keys.txt"
    keys.write_text(text)
    (tmp_path / "in").mkdir()
    r = subprocess.run([CLI, "-i", str(tmp_path / "in"), "-o", str(tmp_path / "out"), "--out-format", "wav", "--hca-keys", str(keys)],
                       capture_output=True, text=True, timeout=60)
    assert r.returncode == 1
    assert f"keys.txt:{line}: not a key code" in r.stderr, r.stderr
