"""AdxReader on the host (vgb_adx_parse) against the restatement in adx_reader_oracle.py and against the description each
file was written from, every rejection with its message, a differential fuzz of the two parsers, and the sizing pass of
the .adx -> WAVE converter, which runs on the host only."""
import ctypes as C

import numpy as np
import pytest

import adx_files as F
import adx_reader_oracle as R

FIELDS = ("header_size", "type", "frame_size", "bit_depth", "channel_count", "sample_rate", "sample_count", "highpass_frequency",
          "version", "revision", "inserted_samples", "loop_count", "looping", "loop_type", "loop_start_sample", "loop_start_byte",
          "loop_end_sample", "loop_end_byte", "samples_per_frame", "audio_offset", "audio_size")


def _parse(vg, img):
    from vgaudio_b200 import _native as N

    img = np.ascontiguousarray(img, dtype=np.uint8)
    info = N.VgbAdxFileInfo()
    st = vg.lib.vgb_adx_parse(img.ctypes.data if img.size else None, img.size, C.byref(info))
    return st, info


def _agree(vg, img):
    """Both parsers on one image: same decision, same fields and history; returns (accepted, info)."""
    st, info = _parse(vg, img)
    ost, oinfo = R.adx_parse(img)
    assert (st == 0) == (ost == 0), (st, ost, vg.lib.vgb_last_error())
    if st == 0:
        for f in FIELDS:
            assert getattr(info, f) == getattr(oinfo, f), f
        if info.version >= 4:
            assert [tuple(info.history[c]) for c in range(info.channel_count)] == oinfo.history
    return st == 0, info


@pytest.mark.parametrize("channels", [1, 2, 8])
@pytest.mark.parametrize("version", [3, 4])
@pytest.mark.parametrize("loop", [None, (1000, 7000)])
def test_written_files_parse_to_their_description(vg, oracle, channels, version, loop):
    img = F.encoded(oracle, channels, 9000, 44100, 18, version, 3, loop, seed=channels)
    ok, info = _agree(vg, img)
    assert ok
    align = F.alignment(loop[0], channels, 18) if loop else 0
    assert (info.channel_count, info.sample_rate, info.version, info.frame_size, info.type) == (channels, 44100, version, 18, 3)
    assert info.inserted_samples == align and info.looping == (loop is not None)
    if loop:
        assert (info.loop_start_sample, info.loop_end_sample) == (loop[0] + align, loop[1] + align)
        assert info.loop_start_byte % 0x800 == 0  # AdxWriter pads the header so the loop start sits on a sector
    else:
        assert info.sample_count == 9000


@pytest.mark.parametrize("frame_size,type", [(18, 2), (18, 4), (9, 3), (33, 3), (130, 4), (3, 3)])  # the oracle encodes frames of up to 256 samples
def test_other_types_and_frame_sizes(vg, oracle, frame_size, type):
    img = F.encoded(oracle, 2, 3000, 32000, frame_size, 4, type, None, seed=7)
    ok, info = _agree(vg, img)
    assert ok and info.samples_per_frame == (frame_size - 2) * 2 and info.type == type


@pytest.mark.parametrize("case", ["short_header_v4", "short_header_v3", "loop_count_zero", "loop_count_negative", "mono_v4_skip",
                                  "v5_header", "negative_header_size", "negative_inserted", "eight_channels_v4"])
def test_hand_assembled_headers(vg, oracle, case):
    img = {
        "short_header_v4": lambda: F.header(header_size=40, inserted=16, loop_count=1),  # 20 + 4 + 8 + 24 > 40: no loop fields
        "short_header_v3": lambda: F.header(version=3, header_size=43),
        "loop_count_zero": lambda: F.header(inserted=5, loop_count=0, header_size=80),
        "loop_count_negative": lambda: F.header(inserted=5, loop_count=-3, loop=(1, 2, 3, 4, 5), header_size=80),
        "mono_v4_skip": lambda: F.header(channels=1, inserted=7, loop_count=1, loop=(1, 10, 99, 90, 77), header_size=80, samples=200),
        "v5_header": lambda: F.header(version=5, inserted=3, loop_count=1, loop=(1, 4, 5, 50, 9), header_size=100),
        "negative_header_size": lambda: F.header(version=3, header_size=-4, samples=0),
        "negative_inserted": lambda: F.header(inserted=-20, loop_count=0, header_size=60),
        "eight_channels_v4": lambda: F.header(channels=8, inserted=0, loop_count=0, header_size=80,
                                              history=[(c * 100, -c * 7) for c in range(8)]),
    }[case]()
    ok, info = _agree(vg, img)
    assert ok
    want = {
        "short_header_v4": dict(inserted_samples=0, looping=0),
        "short_header_v3": dict(inserted_samples=0, looping=0),
        "loop_count_zero": dict(inserted_samples=5, loop_count=0, looping=0),
        "loop_count_negative": dict(loop_count=-3, looping=0, loop_start_sample=0),
        "mono_v4_skip": dict(inserted_samples=7, looping=1, loop_type=1, loop_start_sample=10, loop_start_byte=99, loop_end_sample=90),
        "v5_header": dict(looping=1, loop_end_sample=50),
        "negative_header_size": dict(header_size=-4, audio_offset=0),
        "negative_inserted": dict(inserted_samples=-20),
        "eight_channels_v4": dict(channel_count=8),
    }[case]
    for f, v in want.items():
        assert getattr(info, f) == v, f
    if case == "eight_channels_v4":
        assert tuple(info.history[7]) == (700, -49)


@pytest.mark.parametrize("case,message", [
    ("empty", b"not enough data"),
    ("bad_signature", b"File doesn't have ADX signature (0x80 0x00)"),
    ("truncated_header", b"past the end"),
    ("truncated_loop", b"past the end"),
    ("frame_size_0", b"divide by zero"),
    ("channels_0", b"divide by zero"),
    ("negative_offset", b"Non-negative number required"),
    ("short_audio", b"Specified length is greater than the number of bytes remaining in the Stream"),
    ("negative_length", b"negative audio length"),
    ("wrapped_length", b"divisible by the number of outputs"),
    ("frame_size_1", b"holds no whole sample"),
    ("frame_size_2", b"holds no whole sample"),
    ("inserted_before_audio", b"would index before the audio"),
])
def test_rejected_images(vg, oracle, case, message):
    from vgaudio_b200 import _native as N

    img = {
        "empty": lambda: np.zeros(0, np.uint8),
        "bad_signature": lambda: F.header()[:],
        "truncated_header": lambda: F.header()[:15],
        "truncated_loop": lambda: F.header(inserted=2, loop_count=1, loop=(1, 2, 3, 4, 5), header_size=100)[:50],
        "frame_size_0": lambda: F.header(frame_size=0, audio=b""),
        "channels_0": lambda: F.header(channels=0, audio=b""),
        "negative_offset": lambda: F.header(version=3, header_size=-5, samples=0),
        "short_audio": lambda: F.header()[:-1],
        "negative_length": lambda: F.header(samples=-100, audio=b""),
        "wrapped_length": lambda: F.header(channels=3, frame_size=255, samples=0x7FFFFF00, audio=b""),
        "frame_size_1": lambda: F.header(frame_size=1, samples=0, audio=b""),
        "frame_size_2": lambda: F.header(frame_size=2, samples=10, audio=b""),
        "inserted_before_audio": lambda: F.header(inserted=-32, loop_count=0, header_size=60),
    }[case]()
    if case == "bad_signature":
        img[1] = 1
    ok, _ = _agree(vg, img)
    assert not ok
    assert _parse(vg, img)[0] == N.VGB_E_DATA
    assert message in vg.lib.vgb_last_error(), vg.lib.vgb_last_error()


def test_parsers_agree_on_mutated_and_truncated_adx_files(vg, oracle):
    """5000 images with random header bytes and random truncation through both parsers: same decision and fields."""
    rng = np.random.default_rng(20261016)
    base = [F.encoded(oracle, 2, 3000, 48000, 18, 4, 3, None, seed=1), F.encoded(oracle, 1, 4000, 22050, 18, 4, 3, (100, 3000), seed=2),
            F.encoded(oracle, 3, 2000, 32000, 9, 3, 4, (10, 1500), seed=3), F.header(channels=1, version=3, inserted=4, loop_count=1,
                                                                                     loop=(1, 8, 9, 80, 10), header_size=64, samples=90)]
    n_ok = 0
    for case in range(5000):
        img = base[case % len(base)].copy()
        head = min(img.size, 64)
        for _ in range(int(rng.integers(1, 4))):
            img[int(rng.integers(0, head))] = int(rng.integers(0, 256))
        if rng.random() < 0.3:
            img = img[: int(rng.integers(0, img.size + 1))].copy()
        n_ok += _agree(vg, img)[0]
    assert 300 < n_ok < 4700  # the mutations produce both outcomes


# ---- sizing pass of vgb_convert_adx_to_wave_batch (host only) ------------------------------------------------------------
def _expected_size(oracle, img, key):
    """(status is 0, WAVE file size) by the oracle's parse and the reader chain's sizing checks (not the filter scan)."""
    st, h = R.adx_parse(img)
    if st != 0 or (h.revision in (8, 9) and key is None):
        return False, 0
    n = R._i32(h.sample_count - h.inserted_samples)
    loop = None
    if h.looping:
        loop = (R._i32(h.loop_start_sample - h.inserted_samples), R._i32(h.loop_end_sample - h.inserted_samples))
        if not (0 <= loop[0] <= n and 0 <= loop[1] <= n and loop[0] <= loop[1]):
            return False, 0
    if n < 0:
        return False, 0
    spf, pad = h.samples_per_frame, max(h.inserted_samples, 0)
    if n > 0 and (pad // spf + -(-n // spf)) * h.frame_size > h.audio_size // h.channel_count:
        return False, 0
    return True, oracle.wave_write16([np.zeros(n, np.int16)] * h.channel_count, h.sample_rate, (0, 0) if loop else None).size


def _short(img):
    _, h = R.adx_parse(img)
    return img[: h.audio_offset + h.audio_size - 1].copy()


@pytest.mark.parametrize("with_key", [False, True])
def test_sizing_pass_matches_the_oracle(vg, oracle, with_key):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    key = ct.adx_key(key_code=F.KEY_CODE) if with_key else None
    okey = oracle.adx_key(key_code=F.KEY_CODE)
    imgs = [F.encoded(oracle, 2, 5000, 48000, seed=1),
            F.encoded(oracle, 1, 6000, 44100, 18, 4, 3, (10, 5000), seed=2),
            F.encoded(oracle, 2, 5000, 48000, 18, 4, 3, None, okey, 9, seed=3),       # keyed: needs the key
            _short(F.encoded(oracle, 2, 5000, 48000, seed=4)),                           # short audio region
            F.header(samples=100, inserted=200, loop_count=0, header_size=60),         # negative unaligned count
            F.header(samples=64, inserted=8, loop_count=1, loop=(1, 4, 0, 100, 0), header_size=80),  # loop end past the count
            F.header(samples=0, inserted=0, loop_count=0, header_size=60),              # empty
            F.header(samples=32, inserted=-20, loop_count=0, header_size=60),           # the frames run past the audio
            F.header(samples=40, rate=0, inserted=0, loop_count=0, header_size=60),     # rate 0, Linear: decodes as in the reference
            F.header(samples=40, rate=0, type=2, inserted=0, loop_count=0, header_size=60)]  # rate 0, Fixed: converts
    n = len(imgs)
    ftab = (C.c_void_p * n)(*[i.ctypes.data for i in imgs])
    lens = (C.c_int64 * n)(*[i.size for i in imgs])
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    assert vg.lib.vgb_convert_adx_to_wave_batch(ftab, lens, n, C.byref(key) if key is not None else None, sizes, None, status) == 0
    for i, img in enumerate(imgs):
        ok, size = _expected_size(oracle, img, key)
        assert (status[i] == 0) == ok, (i, status[i])
        assert sizes[i] == size, i
    assert status[2] == (0 if with_key else N.VGB_E_DATA)
    assert [status[i] for i in (3, 4, 7)] == [N.VGB_E_DATA] * 3 and status[5] == N.VGB_E_ARG
    assert status[6] == 0 and status[8] == 0 and status[9] == 0
