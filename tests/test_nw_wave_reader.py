"""The NintendoWare wave and prefetch readers on the host (vgb_nw_file_parse with BRWAV, BCWAV, BFWAV, BCSTP, BFSTP)
against the restatement in nw_wave_reader_oracle.py, field by field and channel offset by channel offset; every
refusal with the reference's message; every prefix of a small file; a differential fuzz; the sizing pass of
vgb_convert_nw_to_wave_batch for the new types, which runs on the host only; and the converters without a writer for
them, which refuse them."""
import ctypes as C
import struct

import numpy as np
import pytest

import nw_files as NF
import nw_wave_files as F
import nw_wave_reader_oracle as R

FIELDS = ("codec", "looping", "channel_count", "sample_rate", "loop_start", "sample_count", "interleave_size", "big_endian",
          "version", "seek_table", "region_count", "track_count", "adpcm_channel_count", "samples_per_seek_entry",
          "loop_start_unaligned", "loop_end_unaligned", "output_size", "audio_offset", "audio_length")
WAVE_KINDS = [(F.BRWAV, None), (F.BCWAV, False), (F.BCWAV, True), (F.BFWAV, True), (F.BFWAV, False)]
PREFETCH_KINDS = [(F.BCSTP, False), (F.BFSTP, True), (F.BFSTP, False)]


def _parse(vg, img, kind):
    from vgaudio_b200 import _native as N

    img = np.ascontiguousarray(img, dtype=np.uint8)
    info = N.VgbNwInfo()
    offs = (C.c_int64 * N.VGB_NW_MAX_CHANNELS)()
    st = vg.lib.vgb_nw_file_parse(img.ctypes.data if img.size else None, img.size, kind, C.byref(info), offs)
    return st, info, list(offs), (vg.lib.vgb_last_error() or b"").decode() if st else ""


def _agree(vg, img, kind):
    """Both parsers on one image: same decision, fields, channel infos and channel offsets; (accepted, info, message)."""
    st, info, offs, msg = _parse(vg, img, kind)
    ost, o = R.parse(img, kind)
    assert (st == 0) == (ost == 0), (st, msg, ost, o)
    if st == 0:
        for f in FIELDS:
            assert getattr(info, f) == getattr(o, f), f
        for c, ch in enumerate(o.channels[: min(len(o.channels), 255)]):
            assert list(info.coefs[c]) == ch["coefs"] and info.gain[c] == ch["gain"]
            assert tuple(info.start_context[c]) == ch["start"] and tuple(info.loop_context[c]) == ch["loop"]
        want = [a for a, _ in o.rows] if o.rows is not None else []
        assert offs[: len(want)] == want and all(v == -1 for v in offs[len(want):])
    else:
        assert st == -2 and o in msg, (msg, o)
    return st == 0, info, msg


def _sizing(vg, imgs, kinds):
    n = len(imgs)
    imgs = [np.ascontiguousarray(i, dtype=np.uint8) for i in imgs]
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in imgs])
    lens = (C.c_int64 * n)(*[a.size for a in imgs])
    types = (C.c_int32 * n)(*kinds)
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    assert vg.lib.vgb_convert_nw_to_wave_batch(ftab, lens, types, n, sizes, None, status) == 0
    return list(sizes), list(status)


def _matrix(oracle):
    files = []
    i = 0
    for kind, be in WAVE_KINDS:
        for codec in (F.PCM8, F.PCM16, F.GCADPCM):
            for ch in (1, 2, 3, 8):
                for loop in (None, 321):
                    lay = ("ordered", "reversed", "overlap", "gaps")[i % 4]
                    files.append((kind, F.encoded(oracle, kind, codec, ch, 700 + 97 * (i % 5), loop=loop, seed=i, big_endian=be,
                                                  layout_kind=lay)))
                    i += 1
    for kind, be in PREFETCH_KINDS:
        for codec in (F.PCM8, F.PCM16, F.GCADPCM):
            for ch in (1, 2, 3):
                n = 5000
                per = F.samples_to_bytes(n, codec)
                files.append((kind, F.encoded(oracle, kind, codec, ch, n, loop=100 if ch == 2 else None, seed=i, big_endian=be,
                                              prefetch=[per // 2 // 8 * 8, per - per // 2 // 8 * 8] if ch != 1 else [per])))
                i += 1
    return files


def test_builder_matrix_parses_alike(vg, oracle):
    for kind, img in _matrix(oracle):
        ok, info, msg = _agree(vg, img, kind)
        assert ok, (kind, msg)
        assert info.interleave_size == (0 if kind <= F.BFWAV else 0x400)
        if kind >= F.BCSTP:
            assert info.looping == 0 and info.output_size == info.audio_length


@pytest.mark.parametrize("kind,versions", [(F.BCWAV, F.BCWAV_VERSIONS), (F.BFWAV, F.BFWAV_VERSIONS)])
def test_unaligned_loop_start_by_version(vg, oracle, kind, versions):
    for v, has in zip(versions, (False, True)):
        img = F.encoded(oracle, kind, F.GCADPCM, 2, 3000, loop=777, seed=4, version=v)
        ok, info, _ = _agree(vg, img, kind)
        assert ok and info.version == v and info.loop_start_unaligned == (777 if has else 0)


def test_stream_types_behave_as_the_stream_parsers(vg, oracle):
    from vgaudio_b200 import _native as N

    for kind, be in ((NF.BRSTM, None), (NF.BCSTM, False), (NF.BFSTM, True)):
        img = NF.encoded(oracle, kind, F.GCADPCM, 2, 3000, seed=2, big_endian=be)
        st, info, offs, _ = _parse(vg, img, kind)
        old = N.VgbNwInfo()
        fn = vg.lib.vgb_brstm_parse if kind == NF.BRSTM else vg.lib.vgb_bcfstm_parse
        assert st == 0 and fn(img.ctypes.data, img.size, C.byref(old)) == 0
        assert bytes(info) == bytes(old) and all(v == -1 for v in offs)
        # the stream types keep refusing wave and prefetch files on purpose
        for k2, wimg in ((F.BCWAV, F.encoded(oracle, F.BCWAV, F.PCM16, 1, 100)), (F.BFSTP, F.encoded(oracle, F.BFSTP, F.PCM16, 1, 100))):
            if kind != NF.BRSTM:
                st, _, _, msg = _parse(vg, wimg, kind)
                assert st == -2 and "are not read" in msg


def test_a_cstm_read_as_bcwav_is_accepted(vg, oracle):
    img = NF.encoded(oracle, NF.BCSTM, F.GCADPCM, 2, 2000, seed=5)
    for kind in (F.BCWAV, F.BFWAV, F.BCSTP, F.BFSTP):
        ok, info, _ = _agree(vg, img, kind)
        assert ok and info.audio_length == 2 * info.output_size
    wav = F.encoded(oracle, F.BFWAV, F.PCM8, 2, 500, seed=6)
    ok, _, _ = _agree(vg, wav, F.BCSTP)  # and a FWAV under a prefetch type
    assert ok


def _patch(img, at, fmt, *vals):
    b = bytearray(img.tobytes())
    struct.pack_into(fmt, b, at, *vals)
    return np.frombuffer(bytes(b), np.uint8).copy()


def test_refusals_with_the_reference_messages(vg, oracle):
    chans = F.channels(oracle, F.GCADPCM, 2, 1400, 7, False)
    n = 1400
    cases = [
        # a channel offset that puts the position before the image
        (F.BCWAV, F.cwav(F.BCWAV, F.GCADPCM, chans, n, offsets=[0, -0x10000]), "Non-negative number required"),
        (F.BRWAV, F.rwav(F.GCADPCM, chans, n, offsets=[-0x10000, 0]), "Non-negative number required"),
        # a channel reference that is not a wave channel: WaveAudioOffsets is short
        (F.BCWAV, F.cwav(F.BCWAV, F.GCADPCM, chans, n, wave_refs=[True, False]), "Index was out of range"),
        # a PDAT count of 0: PrefetchData[0]
        (F.BCSTP, F.cstp(F.BCSTP, F.GCADPCM, chans, n, [1000], count=0), "Index was out of range"),
        # a prefetch file of 0 channels: Size / ChannelCount
        (F.BFSTP, F.cstp(F.BFSTP, F.PCM8, [], 0, [0]), "Attempted to divide by zero"),
        # IMA ADPCM: ToAudioStream returns null
        (F.BFWAV, F.cwav(F.BFWAV, 3, chans, n), "IMA ADPCM is not decoded"),
        (F.BRWAV, F.rwav(3, chans, n), "IMA ADPCM is not decoded"),
        # more than 255 channels, on purpose
        (F.BCWAV, F.cwav(F.BCWAV, F.PCM8, [], 10, channel_count=256, wave_refs=[True] * 256, adpcm_info=False),
         "this reader takes 0..255"),
        # the signatures
        (F.BRWAV, F.rwav(F.GCADPCM, chans, n, magic=b"RWAX"), "File has no RWAV header"),
        (F.BCWAV, F.cwav(F.BCWAV, F.GCADPCM, chans, n, magic=b"CWAX"), "File has no CSTM or FSTM header"),
        (F.BRWAV, F.rwav(F.GCADPCM, chans, n, file_size_delta=1), "Actual file length is less than stated length"),
        # GC-ADPCM without channel info for every channel, on purpose
        (F.BCWAV, F.cwav(F.BCWAV, F.GCADPCM, chans, n, adpcm_info=False), "GC-ADPCM stream of"),
    ]
    for kind, img, msg in cases:
        ok, _, got = _agree(vg, img, kind)
        assert not ok and msg in got, (kind, msg, got)
    # the BOM of an RWAV and a stream data block under a wave info block (no audio reference)
    rw = F.rwav(F.GCADPCM, chans, n)
    ok, _, got = _agree(vg, _patch(rw, 4, ">H", 0xFFFE), F.BRWAV)
    assert not ok and "Expected 65279, but got 65534" in got
    cw = F.cwav(F.BCWAV, F.GCADPCM, chans, n)
    ok, _, got = _agree(vg, _patch(cw, 0x14 + 12, "<h", 0x4002), F.BCWAV)
    assert not ok and "Object reference not set" in got


def test_channels_running_past_the_image(vg, oracle):
    """ReadBytes returns what is left: the last channel's run is shorter, or empty past the end."""
    n = 1400
    for codec in (F.PCM8, F.PCM16, F.GCADPCM):
        for kind in (F.BRWAV, F.BCWAV):
            for ch, cut in ((1, 11), (2, 100), (2, F.samples_to_bytes(n, codec) + 64)):
                chans = F.channels(oracle, codec, ch, n, 3, kind == F.BRWAV)
                img = F.rwav(codec, chans, n, cut=cut) if kind == F.BRWAV else F.cwav(kind, codec, chans, n, cut=cut)
                ok, info, _ = _agree(vg, img, kind)
                assert ok
                rows = R.parse(img, kind)[1].rows
                assert rows[-1][1] == max(0, img.size - rows[-1][0]) < info.output_size
                assert info.audio_offset + info.audio_length <= img.size


@pytest.mark.parametrize("kind", [F.BRWAV, F.BCWAV, F.BFWAV, F.BCSTP, F.BFSTP])
def test_every_prefix_fails_at_the_same_read(vg, oracle, kind):
    codec = F.GCADPCM if kind != F.BFWAV else F.PCM16
    img = F.encoded(oracle, kind, codec, 2, 60, loop=14, seed=8)
    for k in range(img.size + 1):
        _agree(vg, img[:k], kind)


def test_mutated_and_truncated_images(vg, oracle):
    rng = np.random.default_rng(1234)
    seeds = [(kind, F.encoded(oracle, kind, codec, ch, 300, loop=loop, seed=s))
             for s, (kind, codec, ch, loop) in enumerate([(F.BRWAV, F.GCADPCM, 2, 28), (F.BRWAV, F.PCM16, 1, None),
                                                          (F.BCWAV, F.PCM8, 3, None), (F.BCWAV, F.GCADPCM, 1, 100),
                                                          (F.BFWAV, F.PCM16, 2, 10), (F.BCSTP, F.GCADPCM, 2, None),
                                                          (F.BFSTP, F.PCM16, 1, None)])]
    accepted = 0
    for t in range(5000):
        kind, base = seeds[t % len(seeds)]
        img = base.copy()
        for _ in range(int(rng.integers(1, 4))):
            at = int(rng.integers(0, img.size))
            img[at] = rng.integers(0, 256) if rng.random() < 0.7 else img[at] ^ (1 << int(rng.integers(0, 8)))
        if rng.random() < 0.1:
            img = img[: int(rng.integers(0, img.size))]
        kind2 = kind if rng.random() < 0.9 else int(rng.choice([F.BCWAV, F.BFWAV, F.BCSTP, F.BFSTP]))
        ok, info, _ = _agree(vg, img, kind2)
        accepted += ok
        if ok:
            assert 0 <= info.audio_offset and info.audio_offset + info.audio_length <= img.size
    assert 500 < accepted < 4900


def test_sizing_pass_matches_the_oracle(vg, oracle):
    """Status and WAVE size of every new type, good files and the builders' checks: short PCM rows (all alike or not),
    odd big-endian PCM16 rows, loops past a short row, prefetch rows, no channels, raw RWAV fields, other in_types."""
    files = list(_matrix(oracle))
    n = 1000
    for codec in (F.PCM8, F.PCM16):
        for loop in (None, 10, 990):
            for kind in (F.BRWAV, F.BCWAV, F.BFWAV):
                for ch, cut in ((1, 0), (1, 301), (2, 301), (3, 5)):
                    be = kind != F.BCWAV
                    chans = F.channels(oracle, codec, ch, n, ch + cut, be, loop)
                    same = F.layout("overlap", [F.samples_to_bytes(n, codec)] * ch) if cut == 5 else None
                    img = (F.rwav(codec, chans, n, loop=loop, offsets=same, cut=cut) if kind == F.BRWAV else
                           F.cwav(kind, codec, chans, n, loop=loop, offsets=same, cut=cut))
                    files.append((kind, img))
    chans = F.channels(oracle, F.GCADPCM, 2, n, 9, False)
    files.append((F.BCWAV, F.cwav(F.BCWAV, F.GCADPCM, chans, n, cut=40)))  # a short GC-ADPCM run
    files.append((F.BCWAV, F.cwav(F.BCWAV, F.PCM16, [], 100)))  # 0 channels: the builders refuse
    files.append((F.BRWAV, F.rwav(F.PCM16, F.channels(oracle, F.PCM16, 1, 200, 1, True), 200, nibble_fields=False)))  # raw fields
    files.append((7, files[0][1]))  # not a NintendoWare reader
    files.append((8, files[0][1]))
    sizes, status = _sizing(vg, [f for _, f in files], [k for k, _ in files])
    seen = set()
    for i, (kind, img) in enumerate(files):
        ost, msg, _, _, _ = R.plan(img, kind)
        assert status[i] == ost, (i, kind, status[i], ost, msg)
        assert sizes[i] == R.wave_size(img, kind), i
        seen.add(ost)
    assert seen == {0, -1, -2}


def test_converters_without_a_writer_refuse_the_new_types(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    img = F.encoded(oracle, F.BCWAV, F.PCM16, 1, 100)
    for t in range(F.BRWAV, F.BFSTP + 1):
        wave = oracle.wave_write16([np.zeros(100, np.int16)], 32000, None)
        with pytest.raises(N.VgbError) as e:
            ct.convert_wave_batch([wave], ct.convert_options(t))
        assert e.value.code == N.VGB_E_ARG
        _, status = ct.transcode_batch([img], [t], ct.convert_options(ct.CONTAINER_DSP))
        assert status == [N.VGB_E_ARG]
        assert f"in_type {t}" in vg.lib.vgb_last_error().decode()


def test_python_surface(vg, oracle):
    from vgaudio_b200 import containers as ct

    img = F.encoded(oracle, F.BFWAV, F.GCADPCM, 3, 900, seed=2, layout_kind="reversed")
    info, offs = ct.nw_file_parse(img, ct.CONTAINER_BFWAV)
    assert info.channel_count == 3 and offs == [a for a, _ in R.parse(img, F.BFWAV)[1].rows]
    assert offs[0] > offs[1] > offs[2]
    info, offs = ct.nw_file_parse(F.encoded(oracle, F.BCSTP, F.PCM8, 2, 900), ct.CONTAINER_BCSTP)
    assert offs == [] and info.output_size == 2 * 900
