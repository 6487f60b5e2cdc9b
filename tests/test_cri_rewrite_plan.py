"""vgb_rewrite_batch's sizing pass, on the host without a device: for every .adx and .hca stimulus the size equals the
oracle chain's output file, and every file the rewrite refuses fails alone with its status and message."""
import ctypes as C

import numpy as np
import pytest

import cri_rewrite_oracle as R
from vgaudio_b200 import containers as ct

ADX_FEATURES = {"rev0", "rev8", "rev9", "out0", "out8", "out9", "9->9", "v3", "v4", "ch1", "ch2", "ch6", "ch255", "fs18", "fs34",
                "fixed", "linear", "exponential", "non-looping", "loop trimmed", "loop past source", "no_trim", "inserted v3",
                "no loop block", "empty", "empty after", "enc byte without key"}
HCA_FEATURES = {f"ciph{c}" for c in (0, 1, 56, 2)} | {f"out{o}" for o in (-1, 0, 1, 56)} | {
    "comm ascii", "comm utf8", "comm blank", "comm 0x01", "comm into frames", "rva 1", "rva 0.5", "rva nan", "ath", "vbr", "dec",
    "track 0", "loop", "overflow", "bad crc copied", "bad crc rekeyed"}


def _sizing(vg, out_type, img, opts, adx_key=None, hca_key=None):
    """(size, status, message) of one file's sizing pass."""
    f = np.ascontiguousarray(img, np.uint8)
    ftab, lens = (C.c_void_p * 1)(f.ctypes.data), (C.c_int64 * 1)(f.size)
    sz, st = (C.c_int64 * 1)(), (C.c_int32 * 1)()
    o = ct.convert_options(out_type, **opts)
    k = vg._native.VgbAdxKey(*adx_key) if adx_key is not None else None
    code = C.c_uint64(hca_key) if hca_key is not None else None
    assert vg.lib.vgb_rewrite_batch(ftab, lens, 1, C.byref(o), C.byref(k) if k is not None else None,
                                    C.byref(code) if code is not None else None, sz, None, st, None, None) == 0
    return int(sz[0]), int(st[0]), (vg.lib.vgb_last_error() or b"").decode() if st[0] else ""


def test_stimuli_reach_every_case():
    adx = set().union(*(c[4] for c in R.adx_cases()))
    hca = set().union(*(c[3] for c in R.hca_cases()))
    assert ADX_FEATURES <= adx, ADX_FEATURES - adx
    assert HCA_FEATURES <= hca, HCA_FEATURES - hca
    # the features are what the files hold: check the ones the headers show
    for name, img, opts, key, tags in R.adx_cases():
        st, h = R.RA.adx_parse(img)
        assert st == 0, name
        assert ("ch255" not in tags or h.channel_count == 255) and ("v3" not in tags or h.version == 3), name
        assert "inserted v3" not in tags or h.inserted_samples > 0, name
        assert "no loop block" not in tags or (h.looping == 0 and h.version == 4), name
        spf = 2 * h.frame_size - 4
        if "loop past source" in tags:  # TrimFile's LoopEnd + 3 frames reach past the frames the source holds
            assert -(-(h.loop_end_sample + 3 * spf) // spf) > h.audio_size // h.channel_count // h.frame_size, name
    for name, img, opts, tags in R.hca_cases():
        st, info, ciph, comment, rva = R.hca_parse(img)
        assert st == 0, name
        if "comm 0x01" in tags:
            assert comment == b"stop", name
        if "comm into frames" in tags:
            assert comment is not None and len(comment) + 5 > info.header_size - img.tobytes().index(b"comm"), name
        if "overflow" in tags:
            assert len(R.hca_chunks(info, opts["hca_key_type"] >= 0, 0, comment, rva)) > info.header_size - 2, name
        if "track 0" in tags:
            assert info.track_count == 1 and img[0x20] == 0, name


@pytest.mark.parametrize("case", R.adx_cases(), ids=lambda c: c[0])
def test_adx_sizes(vg, oracle, case):
    name, img, opts, key, _ = case
    want = R.expected_adx(img, opts.get("adx_encryption_type", 0),
                          (opts["adx_key_seed"], opts["adx_key_mult"], opts["adx_key_inc"]) if opts.get("adx_has_key") else None,
                          bool(opts.get("no_trim")), key)
    size, status, msg = _sizing(vg, R.ADX, img, opts, adx_key=key)
    assert status == 0, msg
    assert want is not None and size == want.size


@pytest.mark.parametrize("case", R.hca_cases(), ids=lambda c: c[0])
def test_hca_sizes(vg, oracle, case):
    name, img, opts, _ = case
    want = R.expected_hca(img, opts["hca_key_type"], opts["hca_key_code"], R.HCA_KEY)
    size, status, msg = _sizing(vg, R.HCA, img, opts, hca_key=R.HCA_KEY)
    assert status == 0, msg
    assert want is not None and size == want.size


@pytest.mark.parametrize("case", R.refused_cases(), ids=lambda c: c[0])
def test_refusals(vg, oracle, case):
    name, fmt, img, opts, adx_key, hca_key, want_status, part = case
    if fmt == R.ADX:
        assert R.expected_adx(img, in_key=adx_key) is None
    elif "overflow" not in name:
        assert R.expected_hca(img, in_key_code=hca_key) is None
    size, status, msg = _sizing(vg, fmt, img, opts, adx_key, hca_key)
    assert (size, status) == (0, want_status), msg
    assert part in msg and msg.startswith("file 0")


def test_mixed_batch_and_arguments(vg, oracle):
    """Statuses land on their own files in one call; an out_type that is not ADX or HCA, and a bad HCA key type, fail the call."""
    good = R.adx_cases()[0][1]
    bad = R.refused_cases()[0][2]
    files = [good, bad, good]
    arrs = [np.ascontiguousarray(f, np.uint8) for f in files]
    ftab = (C.c_void_p * 3)(*[a.ctypes.data for a in arrs])
    lens = (C.c_int64 * 3)(*[a.size for a in arrs])
    sz, st = (C.c_int64 * 3)(), (C.c_int32 * 3)()
    o = ct.convert_options(R.ADX)
    assert vg.lib.vgb_rewrite_batch(ftab, lens, 3, C.byref(o), None, None, sz, None, st, None, None) == 0
    assert list(st) == [0, -2, 0] and sz[1] == 0 and sz[0] == sz[2] == R.expected_adx(good).size
    for o in (ct.convert_options(1), ct.convert_options(R.HCA, hca_key_type=7)):
        assert vg.lib.vgb_rewrite_batch(ftab, lens, 3, C.byref(o), None, None, sz, None, st, None, None) == -1
