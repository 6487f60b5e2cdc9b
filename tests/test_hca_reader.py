"""HcaReader on the host (vgb_hca_parse) against the restatement of ReadHcaHeader in hca_reader_oracle.py and against the
HcaInfo each file was written from, a differential fuzz of the two parsers, and the sizing pass of the .hca -> WAVE converter, which
runs on the host only."""
import ctypes as C
import struct

import numpy as np
import pytest

import hca_reader_oracle as R
import hca_stimuli as H

KEY = 0x0123456789ABCDEF
INFO_FIELDS = ("channel_count", "sample_rate", "sample_count", "frame_count", "inserted_samples", "appended_samples", "header_size",
               "frame_size", "min_resolution", "max_resolution", "track_count", "channel_config", "total_band_count", "base_band_count",
               "stereo_band_count", "hfr_band_count", "bands_per_hfr_group", "hfr_group_count", "looping", "loop_start_frame",
               "loop_end_frame", "pre_loop_samples", "post_loop_samples", "use_ath_curve")


def _parse(vg, img):
    from vgaudio_b200 import _native as N

    img = np.ascontiguousarray(img, dtype=np.uint8)
    info, ciph = N.VgbHcaInfo(), C.c_int32(-1)
    st = vg.lib.vgb_hca_parse(img.ctypes.data if img.size else None, img.size, C.byref(info), C.byref(ciph))
    return st, info, int(ciph.value)


def _agree(vg, oracle, img):
    """Both parsers on one image: same decision, same fields, same ciph; returns (accepted, info, ciph)."""
    st, info, ciph = _parse(vg, img)
    ost, oinfo, ociph = R.hca_parse(img)
    assert (st == 0) == (ost == 0), (st, ost, vg.lib.vgb_last_error())
    if st == 0:
        for f in INFO_FIELDS:
            assert getattr(info, f) == getattr(oinfo, f), f
        assert ciph == ociph
    return st == 0, info, ciph


def _written(oracle, info, key_type=-1, comment=None, volume=1.0, seed=0):
    """An .hca image of `info` with random frame bytes (the parser does not look at them)."""
    frames = np.random.default_rng(seed).integers(0, 256, (info.frame_count, info.frame_size), dtype=np.uint8)
    enc = oracle.hca_key_tables(key_type, KEY)[1] if key_type >= 0 else None
    return oracle.hca_write(info, frames, enc, max(key_type, 0), comment=comment, volume=volume)


def _info(oracle, channels=2, rate=48000, n=20000, quality=2, loop=None):
    looping, ls, le = (1, loop[0], loop[1]) if loop else (0, 0, 0)
    return oracle.hca_init(oracle.HcaParams(quality, 0, 0, channels, rate, n, looping, ls, le))


def _check_written(vg, oracle, img, info, ciph):
    ok, got, got_ciph = _agree(vg, oracle, img)
    assert ok and got_ciph == ciph
    for f in INFO_FIELDS:
        assert getattr(got, f) == getattr(info, f), f


@pytest.mark.parametrize("key_type", [-1, 0, 1, 56])
@pytest.mark.parametrize("loop", [None, (3000, 15000)])
def test_written_files_parse_to_their_info(vg, oracle, key_type, loop):
    info = _info(oracle, loop=loop)
    _check_written(vg, oracle, _written(oracle, info, key_type), info, max(key_type, 0))


def test_comment_and_volume_chunks(vg, oracle):
    info = _info(oracle, 1, 32000, 9000)
    info.header_size += 32  # room for "comm" and "rva"
    _check_written(vg, oracle, _written(oracle, info, 1, comment="a comment", volume=0.5), info, 1)


@pytest.mark.parametrize("name,info", H.decoder_layouts(), ids=[n for n, _ in H.decoder_layouts()])
def test_decoder_layouts(vg, oracle, name, info):
    _check_written(vg, oracle, _written(oracle, info, 56), info, 56)


# ---- hand-assembled headers --------------------------------------------------------------------------------------------
def _chunk(cid, body):
    return cid + body


def _image(chunks, version=0x0200, frame_count=3, frame_size=64, pad_to=None):
    body = b"".join(chunks)
    header_size = pad_to or 8 + len(body) + 4
    head = b"HCA\0" + struct.pack(">hh", version, header_size) + body
    head = head + b"pad\0" + b"\0" * max(0, header_size - len(head) - 4)
    return np.frombuffer(head[:header_size] + bytes(frame_count * frame_size), dtype=np.uint8).copy()


def _fmt(channels=2, rate=44100, frames=3, inserted=128, appended=100):
    return _chunk(b"fmt\0", struct.pack(">BBHihh", channels, rate >> 16, rate & 0xffff, frames, inserted, appended))


def _comp(frame_size=64, total=100, base=60, stereo=20, per_hfr=5):
    return _chunk(b"comp", struct.pack(">hBBBBBBBBBB", frame_size, 1, 15, 1, 0, total, base, stereo, per_hfr, 0, 0))


def _dec(frame_size=64, total=100, base=60, tracks=1, config=0, stereo_type=1):
    return _chunk(b"dec\0", struct.pack(">hBBBBBB", frame_size, 1, 15, total - 1, base - 1, tracks << 4 | config, stereo_type))


@pytest.mark.parametrize("case", ["dec_stereo", "dec_mono_type0", "dec_then_comp", "v0100_no_ath", "v0100_ath0", "v0200_ath1",
                                  "vbr", "loop_trims", "masked_ids", "zero_tracks"])
def test_hand_assembled_headers(vg, oracle, case):
    chunks = {
        "dec_stereo": [_fmt(), _dec()],
        "dec_mono_type0": [_fmt(1), _dec(stereo_type=0)],
        "dec_then_comp": [_fmt(), _dec(), _comp(total=90)],
        "v0100_no_ath": [_fmt(), _comp()],
        "v0100_ath0": [_fmt(), _comp(), _chunk(b"ath\0", struct.pack(">h", 0))],
        "v0200_ath1": [_fmt(), _comp(), _chunk(b"ath\0", struct.pack(">h", 1))],
        "vbr": [_fmt(), _comp(), _chunk(b"vbr\0", struct.pack(">hh", 500, 3))],
        "loop_trims": [_fmt(frames=3), _comp(), _chunk(b"loop", struct.pack(">iihh", 0, 1, 200, 300))],
        "masked_ids": [_fmt(), _comp(), _chunk(b"ciph", struct.pack(">h", 56))],
        "zero_tracks": [_fmt(), _comp()],
    }[case]
    version = 0x0100 if case.startswith("v0100") else 0x0200
    img = _image(chunks, version)
    if case == "masked_ids":  # every id byte with 0x80 set, as keyed files carry them
        for at in (0, 8, 8 + 16, 8 + 16 + 16):
            for k in range(4):
                if img[at + k]:
                    img[at + k] |= 0x80
    ok, info, ciph = _agree(vg, oracle, img)
    assert ok
    want = {
        "dec_stereo": dict(total_band_count=100, base_band_count=60, stereo_band_count=40, use_ath_curve=0),
        "dec_mono_type0": dict(base_band_count=100, stereo_band_count=0),
        "dec_then_comp": dict(total_band_count=90, stereo_band_count=20, hfr_band_count=10, hfr_group_count=2),
        "v0100_no_ath": dict(use_ath_curve=1),
        "v0100_ath0": dict(use_ath_curve=0),
        "v0200_ath1": dict(use_ath_curve=1),
        "vbr": dict(sample_count=3 * 1024 - 228),
        "loop_trims": dict(looping=1, sample_count=2 * 1024 - 300 - 128),
        "masked_ids": dict(frame_size=64),
        "zero_tracks": dict(track_count=1),
    }[case]
    for f, v in want.items():
        assert getattr(info, f) == v, f
    assert ciph == (56 if case == "masked_ids" else 0)


@pytest.mark.parametrize("case", ["unknown_chunk", "bad_signature", "truncated_header", "truncated_frames", "comm_at_end", "negative_frames"])
def test_rejected_images(vg, oracle, case):
    from vgaudio_b200 import _native as N

    if case == "unknown_chunk":
        img = _image([_fmt(), _chunk(b"xyz\0", b"\0\0"), _comp()])
    elif case == "bad_signature":
        img = _image([_fmt(), _comp()])
        img[0] = ord("X")
    elif case == "truncated_header":
        img = _image([_fmt(), _comp()])[:20]
    elif case == "truncated_frames":
        img = _image([_fmt(), _comp()])[:-1]
    elif case == "comm_at_end":
        body = b"HCA\0" + struct.pack(">hh", 0x0200, 200) + _fmt(frames=0) + b"comm"
        img = np.frombuffer(body, dtype=np.uint8).copy()
    else:
        img = _image([_fmt(frames=-1), _comp()], frame_count=0)
    ok, _, _ = _agree(vg, oracle, img)
    assert not ok
    assert _parse(vg, img)[0] == N.VGB_E_DATA
    if case == "unknown_chunk":
        assert b"Chunk xyz" in vg.lib.vgb_last_error() and b"is not supported." in vg.lib.vgb_last_error()


def test_parsers_agree_on_mutated_and_truncated_hca_files(vg, oracle):
    """5000 images with random header bytes and random truncation through both parsers: same decision and fields."""
    rng = np.random.default_rng(20261016)
    base = [_written(oracle, _info(oracle, 2, 48000, 6000), -1), _written(oracle, _info(oracle, 1, 22050, 3000, loop=(100, 2500)), 56),
            _image([_fmt(), _dec(), _chunk(b"ath\0", struct.pack(">h", 1)), _chunk(b"vbr\0", b"\0\1\0\2")], 0x0100)]
    info = _info(oracle, 3, 32000, 4000)
    info.header_size += 32
    base.append(_written(oracle, info, 1, comment="x", volume=0.25))
    n_ok = 0
    for case in range(5000):
        img = base[case % len(base)].copy()
        head = min(img.size, 130)
        for _ in range(int(rng.integers(1, 4))):
            img[int(rng.integers(0, head))] = int(rng.integers(0, 256))
        if rng.random() < 0.3:
            img = img[: int(rng.integers(0, img.size + 1))].copy()
        n_ok += _agree(vg, oracle, img)[0]
    assert 300 < n_ok < 4700  # the mutations produce both outcomes


# ---- sizing pass of vgb_convert_hca_to_wave_batch (host only) ------------------------------------------------------------
def _expected_size(oracle, img, key_code):
    """(status is 0, WAVE file size) by the oracle's parse and the reader chain's checks."""
    st, info, ciph = R.hca_parse(img)
    if st != 0 or (ciph == 56 and key_code is None) or info.sample_count < 0 or not 1 <= info.channel_count <= 8:
        return False, 0
    if info.looping:
        ls = info.loop_start_frame * 1024 + info.pre_loop_samples - info.inserted_samples
        le = (info.loop_end_frame + 1) * 1024 - info.post_loop_samples - info.inserted_samples
        if not (0 <= ls <= info.sample_count and 0 <= le <= info.sample_count and ls <= le):
            return False, 0
    rows = [np.zeros(info.sample_count, np.int16)] * info.channel_count
    return True, oracle.wave_write16(rows, info.sample_rate, (0, 0) if info.looping else None).size


@pytest.mark.parametrize("key_code", [None, KEY])
def test_sizing_pass_matches_the_oracle(vg, oracle, key_code):
    from vgaudio_b200 import _native as N

    nine = _written(oracle, _info(oracle, 2, 48000, 5000), -1)
    nine[12] = 9  # fmt's channel count: more than the decoder takes
    imgs = [_written(oracle, _info(oracle, 2, 48000, 5000), -1), _written(oracle, _info(oracle, 1, 44100, 9000, loop=(10, 7000)), 1),
            _written(oracle, _info(oracle, 2, 48000, 5000), 56), nine, _written(oracle, _info(oracle, 1), -1)[:-7],
            _image([_fmt(2, 48000, frames=2, appended=2048 - 128), _comp()], frame_count=2)]  # sample_count == 0
    n = len(imgs)
    ftab = (C.c_void_p * n)(*[i.ctypes.data for i in imgs])
    lens = (C.c_int64 * n)(*[i.size for i in imgs])
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    code = C.c_uint64(key_code) if key_code is not None else None
    assert vg.lib.vgb_convert_hca_to_wave_batch(ftab, lens, n, C.byref(code) if code is not None else None, sizes, None, status) == 0
    for i, img in enumerate(imgs):
        ok, size = _expected_size(oracle, img, key_code)
        assert (status[i] == 0) == ok, (i, status[i])
        assert sizes[i] == size, i
    assert status[2] == (0 if key_code is not None else N.VGB_E_DATA)
    assert status[3] != 0 and status[4] == N.VGB_E_DATA and status[5] == 0
