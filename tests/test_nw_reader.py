"""BrstmReader / BCFstmReader on the host (vgb_brstm_parse, vgb_bcfstm_parse) against the restatement in
nw_reader_oracle.py, field by field; every rejection with its message in the reference's order; a differential fuzz of
the two parsers; the sizing pass of vgb_convert_nw_to_wave_batch, which runs on the host only; and the re-lock census
the time-parallel GC-ADPCM decoder's shortest segment rests on."""
import ctypes as C
import struct

import numpy as np
import pytest

import gc_relock as G
import nw_files as F
import nw_reader_oracle as R

FIELDS = ("codec", "looping", "channel_count", "sample_rate", "loop_start", "sample_count", "interleave_size", "big_endian",
          "version", "seek_table", "region_count", "track_count", "adpcm_channel_count", "samples_per_seek_entry",
          "loop_start_unaligned", "loop_end_unaligned", "output_size", "audio_offset", "audio_length")


def _parse(vg, img, kind):
    from vgaudio_b200 import _native as N

    img = np.ascontiguousarray(img, dtype=np.uint8)
    info = N.VgbNwInfo()
    fn = vg.lib.vgb_brstm_parse if kind == F.BRSTM else vg.lib.vgb_bcfstm_parse
    st = fn(img.ctypes.data if img.size else None, img.size, C.byref(info))
    return st, info, (vg.lib.vgb_last_error() or b"").decode() if st else ""


def _agree(vg, img, kind):
    """Both parsers on one image: same decision, same fields and channel infos; returns (accepted, info, message)."""
    st, info, msg = _parse(vg, img, kind)
    ost, o = R.parse(img, kind)
    assert (st == 0) == (ost == 0), (st, msg, ost, o)
    if st == 0:
        for f in FIELDS:
            assert getattr(info, f) == getattr(o, f), f
        for c, ch in enumerate(o.channels[: min(len(o.channels), 255)]):
            assert list(info.coefs[c]) == ch["coefs"] and info.gain[c] == ch["gain"]
            assert tuple(info.start_context[c]) == ch["start"] and tuple(info.loop_context[c]) == ch["loop"]
    else:
        assert st == -2 and o in msg, (msg, o)
    return st == 0, info, msg


KINDS = [(F.BRSTM, None), (F.BCSTM, False), (F.BFSTM, False), (F.BFSTM, True)]


@pytest.mark.parametrize("kind,be", KINDS)
@pytest.mark.parametrize("codec", [F.PCM8, F.PCM16, F.GCADPCM])
@pytest.mark.parametrize("channels", [1, 2, 8])
@pytest.mark.parametrize("loop", [None, 1234])
def test_written_files_parse_to_their_description(vg, oracle, kind, be, codec, channels, loop):
    n = 6000 + 13 * channels
    img = F.encoded(oracle, kind, codec, channels, n, loop=loop, seed=channels, big_endian=be, interleave=0x400)
    ok, info, _ = _agree(vg, img, kind)
    assert ok
    assert (info.codec, info.channel_count, info.sample_count, info.looping, info.sample_rate) == (codec, channels, n, loop is not None, 32000)
    assert info.loop_start == (loop or 0) and info.interleave_size == 0x400
    assert info.big_endian == (1 if kind == F.BRSTM else int(be))
    assert info.output_size == F.samples_to_bytes(n, codec) and info.audio_length == channels * info.output_size
    assert info.adpcm_channel_count == (channels if codec == F.GCADPCM or kind == F.BRSTM else channels)


@pytest.mark.parametrize("kind,version,regions", [(F.BCSTM, v, r) for v in F.BCSTM_VERSIONS for r in (0, 3)] +
                         [(F.BFSTM, v, r) for v in F.BFSTM_VERSIONS for r in (0, 2)])
def test_versions_regions_and_unaligned_loops(vg, oracle, kind, version, regions):
    img = F.encoded(oracle, kind, F.GCADPCM, 2, 3000, loop=500, seed=3, version=version, regions=regions)
    has_region = version >> 24 == 0 or version >= 0x02010000
    ok, info, msg = _agree(vg, img, kind)
    if regions and not has_region:  # REGN with no region reference: the reference dereferences null
        assert not ok and "Object reference not set" in msg
        return
    assert ok and info.version == version and info.region_count == regions
    unaligned = version in (0x02030000, 0x00040000, 0x00050000)
    assert (info.loop_start_unaligned, info.loop_end_unaligned) == ((500, 3000) if unaligned else (0, 0))


@pytest.mark.parametrize("kind", [F.BRSTM, F.BCSTM])
@pytest.mark.parametrize("seek", ["standard", "short", "unknown", "none"])
def test_seek_tables(vg, oracle, kind, seek):
    if kind == F.BCSTM and seek == "short":
        pytest.skip("the shortened size is a BRSTM reading")
    img = F.encoded(oracle, kind, F.GCADPCM, 2, 40000, seed=5, seek=seek, spe=0x800)
    ok, info, _ = _agree(vg, img, kind)
    assert ok
    want = {"standard": 1, "short": 2, "unknown": 0, "none": 0} if kind == F.BRSTM else {"standard": 1, "unknown": 1, "none": 0}
    assert info.seek_table == want[seek]


@pytest.mark.parametrize("kind,be", KINDS)
@pytest.mark.parametrize("delta", [-300, -1, 0, 1, 777])
def test_region_shorter_or_longer_than_the_samples(vg, oracle, kind, be, delta):
    """in_size != SamplesToBytes(sample_count): the rows are zero-filled or truncated; a last block shorter than the
    interleave either way."""
    n = 5000
    in_size = F.samples_to_bytes(n, F.GCADPCM) + delta
    img = F.encoded(oracle, kind, F.GCADPCM, 2, n, seed=9, big_endian=be, interleave=0x300, in_size=in_size)
    ok, info, _ = _agree(vg, img, kind)
    assert ok and info.audio_length == 2 * in_size and info.output_size == F.samples_to_bytes(n, F.GCADPCM)
    assert in_size % 0x300 != 0


@pytest.mark.parametrize("track_type,tracks", [(0, 1), (1, 3), (1, 0)])
def test_brstm_track_kinds(vg, oracle, track_type, tracks):
    img = F.encoded(oracle, F.BRSTM, F.PCM16, 2, 700, seed=2, track_type=track_type, tracks=tracks)
    ok, info, _ = _agree(vg, img, F.BRSTM)
    assert ok and info.track_count == tracks


def _patch(img, at, fmt, *vals):
    img = img.copy()
    b = bytearray(img.tobytes())
    struct.pack_into(fmt, b, at, *vals)
    return np.frombuffer(bytes(b), np.uint8).copy()


def _find(img, tag):
    return bytes(img).index(tag)


def _rej(oracle, case):
    """(kind, image) of one rejection case."""
    br = lambda **kw: F.encoded(oracle, F.BRSTM, F.GCADPCM, 2, 3000, seed=4, **kw)  # noqa: E731
    cs = lambda **kw: F.encoded(oracle, F.BCSTM, F.GCADPCM, 2, 3000, seed=4, **kw)  # noqa: E731
    b, c = br(), cs()
    return {
        "empty": (F.BRSTM, np.zeros(0, np.uint8)),
        "rstm_magic": (F.BRSTM, _patch(b, 0, "4s", b"RSTX")),
        "cstm_as_brstm": (F.BRSTM, c),
        "rstm_bom": (F.BRSTM, _patch(b, 4, ">H", 0xFFFE)),
        "rstm_length": (F.BRSTM, br(file_size_delta=1)),
        "head_id": (F.BRSTM, _patch(b, _find(b, b"HEAD"), "4s", b"HEAX")),
        "head_size": (F.BRSTM, _patch(b, 0x14, ">i", 1)),
        "stream_ref": (F.BRSTM, _patch(b, 0x48, ">h", 0x0101)),
        "track_ref": (F.BRSTM, _patch(b, 0x50, ">h", 0x0101)),
        "channel_ref": (F.BRSTM, _patch(b, 0x58, ">h", 0x0101)),
        "adpc_id": (F.BRSTM, _patch(b, _find(b, b"ADPC"), "4s", b"ADPX")),
        "adpc_size": (F.BRSTM, _patch(b, 0x1C, ">i", 0x60)),
        "adpc_spe_zero": (F.BRSTM, br(spe=0)),
        "data_id": (F.BRSTM, _patch(b, _find(b, b"DATA"), "4s", b"DATX")),
        "data_size": (F.BRSTM, _patch(b, 0x24, ">i", 7)),
        "truncated_audio": (F.BRSTM, b[:-3].copy()),
        "odd_split": (F.BRSTM, F.encoded(oracle, F.BRSTM, F.PCM8, 3, 100, seed=1, in_size=100, channel_count=7)),
        "truncated_head": (F.BRSTM, b[:0x50].copy()),
        "codec_ima": (F.BRSTM, _patch(b, 0x48 + 24, "B", 3)),
        "gc_no_channel_info": (F.BRSTM, br(adpcm_info=1)),
        "cstm_magic": (F.BCSTM, _patch(c, 0, "4s", b"XSTM")),
        "cstm_bom": (F.BCSTM, _patch(c, 4, "<H", 0x1234)),
        "cwav": (F.BCSTM, _patch(c, 0, "4s", b"CWAV")),
        "fstp": (F.BFSTM, _patch(c, 0, "4s", b"FSTP")),
        "cstm_length": (F.BCSTM, cs(file_size_delta=5)),
        "no_info": (F.BCSTM, _patch(c, 0x14, "<h", 0x4005)),
        "info_id": (F.BCSTM, _patch(c, _find(c, b"INFO"), "4s", b"INFX")),
        "info_size": (F.BCSTM, _patch(c, 0x14 + 8, "<i", 3)),
        "seek_id": (F.BCSTM, _patch(c, _find(c, b"SEEK"), "4s", b"SEEX")),
        "regn_id": (F.BCSTM, _patch(cs(regions=1), _find(cs(regions=1), b"REGN"), "4s", b"REGX")),
        "regn_old_version": (F.BCSTM, cs(regions=1, version=0x02000000)),
        "no_data": (F.BCSTM, _patch(c, 0x14 + 24, "<h", 0x4009)),
        "pdat_block": (F.BCSTM, _patch(_patch(c, 0x14 + 24, "<h", 0x4004), _find(c, b"DATA"), "4s", b"PDAT")),
        "data_size_cstm": (F.BCSTM, _patch(c, 0x14 + 24 + 8, "<i", 9)),
        "stream_ref_cstm": (F.BCSTM, _patch(c, _find(c, b"INFO") + 8, "<h", 0x4101)),
        "two_faults_head_first": (F.BRSTM, _patch(_patch(b, _find(b, b"HEAD"), "4s", b"HEAX"), _find(b, b"DATA"), "4s", b"DATX")),
    }[case]


REJECTIONS = [
    ("empty", "Index and count must refer to a location within the buffer"),
    ("rstm_magic", "File has no RSTM header"),
    ("cstm_as_brstm", "File has no RSTM header"),
    ("rstm_bom", "Expected 65279, but got 65534"),
    ("rstm_length", "Actual file length is less than stated length"),
    ("head_id", "Unknown or invalid HEAD block"),
    ("head_size", "HEAD block size in RSTM header doesn't match size in HEAD header"),
    ("stream_ref", "Could not read stream info."),
    ("track_ref", "Could not read track info."),
    ("channel_ref", "Could not read channel info."),
    ("adpc_id", "Unknown or invalid ADPC block"),
    ("adpc_size", "ADPC block size in RSTM header doesn't match size in ADPC header"),
    ("adpc_spe_zero", "Attempted to divide by zero."),
    ("data_id", "Unknown or invalid DATA block"),
    ("data_size", "DATA block size in main header doesn't match size in DATA header"),
    ("truncated_audio", "Actual file length is less than stated length"),
    ("odd_split", "must be divisible by the number of outputs."),
    ("truncated_head", "Actual file length is less than stated length"),
    ("codec_ima", "IMA ADPCM is not decoded"),
    ("gc_no_channel_info", "GC-ADPCM stream of 2 channels with GC-ADPCM info for 1"),
    ("cstm_magic", "File has no CSTM or FSTM header"),
    ("cstm_bom", "File has no byte order mark"),
    ("cwav", "CWAV files are not read"),
    ("fstp", "FSTP files are not read"),
    ("cstm_length", "Actual file length is less than stated length"),
    ("no_info", "File has no INFO block"),
    ("info_id", "Unknown or invalid INFO block"),
    ("info_size", "INFO block size in main header doesn't match size in INFO header"),
    ("seek_id", "Unknown or invalid SEEK block"),
    ("regn_id", "Unknown or invalid REGN block"),
    ("regn_old_version", "Object reference not set to an instance of an object."),
    ("no_data", "File has no DATA block"),
    ("pdat_block", "prefetch and wave data blocks are not read"),
    ("data_size_cstm", "DATA block size in main header doesn't match size in DATA header"),
    ("stream_ref_cstm", "Could not read stream info."),
    ("two_faults_head_first", "Unknown or invalid HEAD block"),
]


@pytest.mark.parametrize("case,message", REJECTIONS)
def test_rejected_images(vg, oracle, case, message):
    kind, img = _rej(oracle, case)
    ok, _, msg = _agree(vg, img, kind)
    assert not ok
    assert message in msg, msg


def test_truncated_images_fail_at_the_reads(vg, oracle):
    """Every prefix of a small file: the stated-length check, then the reads past the image, exactly as the oracle."""
    for kind, be in KINDS:
        img = F.encoded(oracle, kind, F.PCM16, 2, 40, seed=1, big_endian=be)
        for cut in range(img.size + 1):
            t = img[:cut].copy()
            if cut >= 16:  # keep the stated length honest so the reads themselves are reached
                t = _patch(t, 8, (">" if kind == F.BRSTM or be else "<") + "i", cut) if kind == F.BRSTM else \
                    _patch(t, 12, (">" if be else "<") + "i", cut)
            _agree(vg, t, kind)


def test_parsers_agree_on_mutated_and_truncated_images(vg, oracle):
    """5000 images with random header and table bytes and random truncation through both parsers: same decision, same
    fields; every outcome is VGB_OK or VGB_E_DATA."""
    rng = np.random.default_rng(20261016)
    base = [(F.BRSTM, F.encoded(oracle, F.BRSTM, F.GCADPCM, 2, 2000, loop=100, seed=1, spe=0x400)),
            (F.BRSTM, F.encoded(oracle, F.BRSTM, F.PCM8, 1, 900, seed=2, seek="short", spe=0x100)),
            (F.BCSTM, F.encoded(oracle, F.BCSTM, F.GCADPCM, 2, 1500, seed=3, regions=2, spe=0x400)),
            (F.BFSTM, F.encoded(oracle, F.BFSTM, F.PCM16, 2, 700, seed=4, big_endian=True, version=0x00050000, regions=1)),
            (F.BFSTM, F.encoded(oracle, F.BFSTM, F.GCADPCM, 1, 800, seed=5, version=0x00030000))]
    n_ok = 0
    for case in range(5000):
        kind, img = base[case % len(base)]
        img = img.copy()
        head = min(img.size, int(R.parse(img, kind)[1].audio_offset))
        for _ in range(int(rng.integers(1, 4))):
            at = int(rng.integers(0, head))
            img[at] = int(rng.integers(0, 256)) if rng.random() < 0.7 else img[at] ^ (1 << int(rng.integers(0, 8)))
        if rng.random() < 0.3:
            img = img[: int(rng.integers(0, img.size + 1))].copy()
        ok, _, _ = _agree(vg, img, kind)
        n_ok += ok
    assert 300 < n_ok < 4700  # the mutations produce both outcomes


# ---- sizing pass of vgb_convert_nw_to_wave_batch (host only) ------------------------------------------------------------
def test_sizing_pass_matches_the_oracle(vg, oracle):
    from vgaudio_b200 import _native as N

    jobs = [(F.BRSTM, F.encoded(oracle, F.BRSTM, F.GCADPCM, 2, 5000, loop=10, seed=1)),
            (F.BCSTM, F.encoded(oracle, F.BCSTM, F.PCM16, 1, 6000, seed=2)),
            (F.BFSTM, F.encoded(oracle, F.BFSTM, F.PCM8, 8, 300, seed=3, big_endian=True)),
            (F.BFSTM, F.encoded(oracle, F.BCSTM, F.PCM16, 3, 200, seed=4)),                 # BCFstmReader takes either magic
            (F.BRSTM, F.encoded(oracle, F.BCSTM, F.PCM16, 1, 200, seed=5)),                 # a .bcstm image read as BRSTM
            (F.BCSTM, F.encoded(oracle, F.BCSTM, F.PCM16, 1, 200, loop=201, seed=6)),       # loop start past the end
            (F.BCSTM, F.build(F.BCSTM, F.PCM16, [F.Channel(b"")], -4, in_size=0)),          # negative sample count
            (7, F.encoded(oracle, F.BCSTM, F.PCM16, 1, 200, seed=7)),                       # not a stream reader
            (F.BRSTM, F.encoded(oracle, F.BRSTM, F.GCADPCM, 1, 0, seed=8)),                 # empty
            (F.BCSTM, F.encoded(oracle, F.BCSTM, F.GCADPCM, 2, 100, seed=9, interleave=0)),  # interleave 0: zero rows
            (F.BRSTM, F.encoded(oracle, F.BRSTM, F.PCM16, 2, 100, loop=100, seed=10))]      # loop start == sample count
    n = len(jobs)
    imgs = [j[1] for j in jobs]
    ftab = (C.c_void_p * n)(*[i.ctypes.data for i in imgs])
    lens = (C.c_int64 * n)(*[i.size for i in imgs])
    types = (C.c_int32 * n)(*[j[0] for j in jobs])
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    assert vg.lib.vgb_convert_nw_to_wave_batch(ftab, lens, types, n, sizes, None, status) == 0
    for i, (kind, img) in enumerate(jobs):
        st = R.plan(img, kind)[0]
        assert status[i] == st, (i, status[i], st, vg.lib.vgb_last_error())
        assert sizes[i] == R.wave_size(img, kind), i
    assert [status[i] for i in (0, 1, 2, 3, 8, 9, 10)] == [0] * 7
    assert status[4] == N.VGB_E_DATA and status[5] == N.VGB_E_ARG and status[6] == N.VGB_E_DATA and status[7] == N.VGB_E_ARG


# ---- the re-lock census and the forced-silence stimulus (oracle only) ------------------------------------------------------
def test_relock_census_supports_the_shortest_segment(oracle):
    """From a wrong pair, the decoder re-locks within a few frames as a rule; the shortest segment (1024 frames,
    common.cuh) is longer than the 99th percentile on this material, so a boundary's run-on is a fraction of a segment."""
    from vgaudio_b200 import synth

    chans = [synth.channel(300 + i, 48000 * 3, 48000, degenerate=False) for i in range(6)]
    r = G.census(oracle, chans, every=37, cap=8192)
    assert r["never"] == 0 and r["trials"] > 1000
    assert r["median"] < 64 and r["p99"] < 1024, r


def test_wrong_pair_never_relocks_inside_digital_silence(oracle):
    """The stimulus the GPU tests use to force the cascade: inside the held silence a wrong pair stays wrong to the end
    of the stretch, and re-locks on the loud material after it."""
    from vgaudio_b200 import synth

    pcm = synth.channel(77, 14 * 3000, 48000, degenerate=False)
    co = oracle.calculate_coefficients(pcm)
    ad, co2 = G.silence_stimulus(oracle.encode(pcm, co), co, 200, 2200)
    truth = oracle.decode(ad, co2, len(pcm), 1000, -1000)
    assert truth[14 * 200 - 1] != 0 and np.all(truth[14 * 200: 14 * 2200] == truth[14 * 200 - 1])
    starts = list(range(200, 2200, 50))
    r = G.relock_frames(ad, co2, truth, starts, [(0, 0)] * len(starts), 8192)
    assert np.all(r > 2200 - np.array(starts)), r   # not before the stretch ends
    assert np.all(r > 0)                            # but after it
