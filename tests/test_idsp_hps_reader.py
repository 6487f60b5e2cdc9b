"""IdspReader / HpsReader on the host (vgb_idsp_parse, vgb_hps_parse) against the restatement in
idsp_hps_reader_oracle.py, field by field; files of the writer oracle parse to what was written; every rejection with
its message in the reference's order; hand-built HPS block chains; a differential fuzz of the two parsers; and the sizing
pass of vgb_convert_idsp_hps_to_wave_batch, which runs on the host only."""
import ctypes as C
import struct

import numpy as np
import pytest

import gc_container_writer_oracle as W
import idsp_hps_reader_oracle as R
from vgaudio_b200 import synth

IDSP_FIELDS = ("channel_count", "sample_rate", "sample_count", "loop_start", "loop_end", "interleave_size", "header_size",
               "channel_info_size", "audio_data_offset", "audio_data_length", "looping", "interleave", "output_size",
               "audio_offset", "audio_length")
HPS_FIELDS = ("sample_rate", "channel_count", "sample_count", "looping", "loop_start", "block_count", "first_block", "loop_block")


def _parse(vg, img, kind):
    from vgaudio_b200 import _native as N

    img = np.ascontiguousarray(img, dtype=np.uint8)
    ptr = img.ctypes.data if img.size else None
    if kind == R.IDSP:
        info = N.VgbIdspInfo()
        st = vg.lib.vgb_idsp_parse(ptr, img.size, C.byref(info))
        blocks = []
    else:
        info = N.VgbHpsInfo()
        st = vg.lib.vgb_hps_parse(ptr, img.size, C.byref(info), None, 0)
        blocks = []
        if st == 0 and info.block_count:
            tab = (N.VgbHpsBlock * info.block_count)()
            assert vg.lib.vgb_hps_parse(ptr, img.size, C.byref(info), tab, info.block_count) == 0
            blocks = list(tab)
    return st, info, blocks, (vg.lib.vgb_last_error() or b"").decode() if st else ""


def _agree(vg, img, kind):
    """Both parsers on one image: same decision, same fields; returns (accepted, info, blocks, message)."""
    st, info, blocks, msg = _parse(vg, img, kind)
    ost, o = R.parse(img, kind)
    assert (st == 0) == (ost == 0), (st, msg, ost, o)
    if st:
        assert st == -2 and o in msg, (msg, o)
        return False, info, blocks, msg
    for f in IDSP_FIELDS if kind == R.IDSP else HPS_FIELDS:
        assert getattr(info, f) == getattr(o, f), (f, getattr(info, f), getattr(o, f))
    for c, ch in enumerate(o.channels):
        assert list(info.coefs[c]) == ch["coefs"] and info.gain[c] == ch["gain"] and tuple(info.start_context[c]) == ch["start"]
        assert tuple(info.loop_context[c]) == ch.get("loop", (0, 0, 0))
        if kind == R.IDSP:
            for f in ("start_address", "end_address", "current_address"):
                assert getattr(info, f)[c] == ch[f]
            assert (info.ch_sample_count[c], info.ch_nibble_count[c], info.ch_sample_rate[c], info.ch_looping[c]) == \
                (ch["sample_count"], ch["nibble_count"], ch["sample_rate"], ch["looping"])
        else:
            assert (info.max_block_size[c], info.end_address[c]) == (ch["max_block_size"], ch["end_address"])
            assert info.channel_audio_bytes[c] == sum(g for _, g in o.pieces[c])
    if kind == R.HPS:
        assert [(b.offset, b.size, b.final_nibble, b.next_offset) for b in blocks] == \
            [(b["offset"], b["size"], b["final_nibble"], b["next_offset"]) for b in o.blocks]
    return True, info, blocks, ""


def _pcm(ch, n, seed):
    return list(synth.batch(ch, n, 32000, first_index=seed * 8, degenerate=False))


LOOPS = {"none": None, "zero": lambda n: (0, n), "aligned": lambda n: (28 * 300, n - 5), "unaligned": lambda n: (4321, n - 17)}


@pytest.mark.parametrize("channels", [1, 2, 3, 5, 6, 7])
@pytest.mark.parametrize("loop", list(LOOPS))
@pytest.mark.parametrize("trim", [True, False])
def test_written_idsp_files_parse_to_their_description(vg, oracle, channels, loop, trim):
    n = 20000 + 37 * channels
    lp = LOOPS[loop](n) if LOOPS[loop] else None
    st, img = W.write_idsp(_pcm(channels, n, channels), 32000, lp, trim)
    assert st == 0
    ok, info, _, _ = _agree(vg, img, R.IDSP)
    d = W.parse_idsp(img)
    assert ok and (info.channel_count, info.sample_rate, info.sample_count) == (channels, 32000, d["sample_count"])
    assert (info.looping, info.loop_start, info.loop_end) == (int(lp is not None), d["loop_start"], d["loop_end"])
    assert info.interleave == 16 and info.audio_length == channels * d["audio_data_size"]
    for c in range(channels):
        assert list(info.coefs[c]) == d["chans"][c]["coefs"] and tuple(info.loop_context[c]) == d["chans"][c]["loop"]


@pytest.mark.parametrize("channels", [1, 2, 5, 6])
@pytest.mark.parametrize("loop", list(LOOPS))
def test_written_hps_files_parse_to_their_description(vg, oracle, channels, loop):
    n = 70000 + 37 * channels
    lp = LOOPS[loop](n) if LOOPS[loop] else None
    st, img = W.write_hps(_pcm(channels, n, channels), 32000, lp)
    if st:  # the writer's own refusals (a block whose history lies past the first decode)
        return
    ok, info, blocks, _ = _agree(vg, img, R.HPS)
    d = W.parse_hps(img)
    assert ok and (info.channel_count, info.sample_count, info.looping, info.loop_start) == (channels, d["sample_count"], d["looping"], d["loop_start"])
    assert [(b.offset, b.next_offset) for b in blocks] == [(b["offset"], b["next"]) for b in d["blocks"]]
    assert all(info.channel_audio_bytes[c] == d["arrays"][c].size for c in range(channels))
    if lp:
        assert tuple(info.loop_context[0]) == d["blocks"][info.loop_block]["ctx"][0]


# ---- rejections ---------------------------------------------------------------------------------------------------------
def _patch(img, at, fmt, *vals):
    b = bytearray(np.asarray(img, np.uint8).tobytes())
    struct.pack_into(fmt, b, at, *vals)
    return np.frombuffer(bytes(b), np.uint8).copy()


def _enc(n, seed=1, ch=1):
    return [R.encoded(p, (seed * 31 % 500, -seed * 7 % 300)) for p in _pcm(ch, n, seed)]


def _idsp(n=3000, ch=2, **kw):
    return R.idsp_image(32000, _enc(n, 1, ch), n, **kw)


def _hps(pieces=(0x200, 0x200, 0x100), ch=2, **kw):
    n = sum(pieces) * 2 // 16 * 14
    return R.hps_chain(32000, _enc(n, 2, ch), list(pieces), **kw)


def _rej(case):
    i, h = _idsp(), _hps()
    return {
        "idsp_signature": (R.IDSP, _patch(i, 0, ">4s", b"IDSQ"), "File has no IDSP header"),
        "idsp_short_signature": (R.IDSP, i[:3], "Index and count must refer"),
        "idsp_main_header": (R.IDSP, i[:30], "Unable to read beyond the end of the stream"),
        "idsp_channel_info": (R.IDSP, _patch(i, 0x24, ">i", 0x7000), "Unable to read beyond the end of the stream"),
        "idsp_negative_info": (R.IDSP, _patch(i, 0x20, ">i", -0x100), "Non-negative number required"),
        "idsp_negative_audio_offset": (R.IDSP, _patch(i, 0x28, ">i", -1), "Non-negative number required"),
        "idsp_region": (R.IDSP, _patch(i, 0x2c, ">i", 100000), "Specified length is greater than the number of bytes remaining"),
        "idsp_divisibility": (R.IDSP, _patch(_idsp(ch=3), 0x2c, ">i", 0x55555556), "must be divisible by the number of outputs"),  # 3 * that wraps to 2
        "idsp_zero_channels": (R.IDSP, _patch(i, 0x08, ">i", 0), "Attempted to divide by zero"),
        "idsp_256_channels": (R.IDSP, _patch(i, 0x08, ">i", 256), "this reader takes 0..255"),
        "idsp_negative_output": (R.IDSP, _patch(i, 0x10, ">i", -100), "Arithmetic operation resulted in an overflow"),
        "hps_signature": (R.HPS, _patch(h, 0, ">8s", b" HALPSU\0"), "File has no HALPST header"),
        "hps_short_signature": (R.HPS, h[:7], "Index and count must refer"),
        "hps_header": (R.HPS, h[:0x30], "Unable to read beyond the end of the stream"),
        "hps_block_header": (R.HPS, h[:0x88], "Unable to read beyond the end of the stream"),
        "hps_zero_channels": (R.HPS, _patch(h, 0x0c, ">i", 0), "Sequence contains no elements"),
        "hps_256_channels": (R.HPS, _patch(h, 0x0c, ">i", 256), "this reader takes at most 255"),
        "hps_negative_audio_size": (R.HPS, _patch(h, 0x84, ">i", -3), "Non-negative number required"),
        "hps_negative_piece": (R.HPS, _patch(h, 0x80, ">i", -0x10000), "Non-negative number required"),
        "hps_differing_counts": (R.HPS, _patch(h, 0x10 + 0x38 + 8, ">i", 100), "Channels have differing sample counts"),
    }[case]


REJECTIONS = ["idsp_signature", "idsp_short_signature", "idsp_main_header", "idsp_channel_info", "idsp_negative_info",
              "idsp_negative_audio_offset", "idsp_region", "idsp_divisibility", "idsp_zero_channels", "idsp_256_channels",
              "idsp_negative_output", "hps_signature", "hps_short_signature", "hps_header", "hps_block_header",
              "hps_zero_channels", "hps_256_channels", "hps_negative_audio_size", "hps_negative_piece", "hps_differing_counts"]


@pytest.mark.parametrize("case", REJECTIONS)
def test_rejected_images(vg, oracle, case):
    kind, img, message = _rej(case)
    ok, _, _, msg = _agree(vg, img, kind)
    assert not ok and message in msg, msg


def test_truncated_images_fail_at_the_reads(vg, oracle):
    """Every prefix of a small file of each kind: the reads past the image and the region check, exactly as the oracle."""
    for kind, img in ((R.IDSP, _idsp(200, 2)), (R.HPS, _hps((0x40, 0x20)))):
        for cut in range(img.size + 1):
            _agree(vg, img[:cut].copy(), kind)


# ---- HPS block chains -----------------------------------------------------------------------------------------------------
def _chain_ok(vg, img):
    ok, info, blocks, msg = _agree(vg, img, R.HPS)
    assert ok, msg
    return info, blocks


@pytest.mark.parametrize("loop_block,want", [(0, 0), (1, 0x200 * 2 // 16 * 14), (2, 0x400 * 2 // 16 * 14)])
def test_chain_loops_to_the_first_and_a_middle_block(vg, oracle, loop_block, want):
    info, blocks = _chain_ok(vg, _hps(loop_block=loop_block))
    assert info.looping and info.loop_block == loop_block and info.loop_start == want and len(blocks) == 3


def test_chain_loop_to_an_offset_that_is_no_block(vg, oracle):
    img = _hps()
    info, blocks = _chain_ok(vg, img)
    last = blocks[-1].offset
    img = _patch(img, last + 8, ">i", blocks[1].offset + 4)  # before the last block, but no block starts there
    info, blocks = _chain_ok(vg, img)
    assert not info.looping and info.loop_block == -1 and len(blocks) == 3


def test_chain_ends_where_next_offset_is_not_past_the_block(vg, oracle):
    img = _hps((0x100,) * 5)
    _, blocks = _chain_ok(vg, img)
    for nxt in (blocks[2].offset, blocks[2].offset - 1, 0, -5):
        info, b = _chain_ok(vg, _patch(img, blocks[2].offset + 8, ">i", nxt))
        assert len(b) == 3 and info.looping == (nxt == blocks[2].offset)


def test_overlapping_blocks_and_odd_final_nibbles(vg, oracle):
    img = _hps((0x100, 0x80, 0x60), odd_final=True)
    _, blocks = _chain_ok(vg, img)
    # the third block moved 0x20 back, into the second block's audio: its header overlaps that audio, its audio its old header
    at = blocks[2].offset - 0x20
    img2 = _patch(img, blocks[1].offset + 8, ">i", at)
    img2[at: at + 28] = img[blocks[2].offset: blocks[2].offset + 28]
    info, b2 = _chain_ok(vg, img2)
    assert b2[2].offset == at and all(b.final_nibble % 2 == 0 for b in b2)
    # odd byte counts: FinalNibble 2k leaves k + 1 bytes
    img3 = _patch(img, blocks[0].offset + 4, ">i", 0x100 * 2 - 3)
    _chain_ok(vg, img3)


def test_piece_cut_short_by_the_end_of_the_image(vg, oracle):
    img = _hps((0x100, 0x100))
    _, blocks = _chain_ok(vg, img)
    cut = img[: img.size - 0x90].copy()  # the last block's second piece is short, and further cuts empty it
    info, _ = _chain_ok(vg, cut)
    assert info.channel_audio_bytes[1] < info.channel_audio_bytes[0]
    info, _ = _chain_ok(vg, img[: img.size - 0x180].copy())
    assert info.channel_audio_bytes[1] == 0x100


def hps_writer_3ch(pcm, rate):
    """HpsWriter on three channels: the block map leaves GetNextMultiple(4 + 8 * 3, 0x20) = 0x20 header bytes per block,
    WriteBlock writes 12 + 8 * 3 and pads to 0x40, so every later block lands 0x20 bytes further past its recorded
    offset."""
    ch, n = len(pcm), len(pcm[0])
    _, g = W.hps_geometry(ch, n, None)
    enc = [R.encoded(p) for p in pcm]
    out = R.hps_header(rate, [dict(coefs=co, end_address=W.sample_to_nibble(n - 1), start=st) for _, co, st in enc])
    pos = g["head"]
    for b in g["blocks"]:
        R.put(out, pos, struct.pack(">iii", b["written"], b["end_nibble"], b["next"]))
        pos = R._next_multiple(pos + 12 + 8 * ch, 0x20)
        for ad, _, _ in enc:
            R.put(out, pos, bytes(np.asarray(ad, np.uint8)[b["byte_in"]: b["byte_in"] + b["chan_size"]]))
            pos = R._next_multiple(pos + b["chan_size"], 0x20)
    return np.frombuffer(bytes(out), np.uint8).copy()


def test_three_channel_file_as_hps_writer_lays_it_out(vg, oracle):
    img = hps_writer_3ch(_pcm(3, 50000, 4), 32000)
    _agree(vg, img, R.HPS)
    assert R.plan(img, R.HPS)[0] == _sizing(vg, [(R.HPS, img)])[0][0]


# ---- differential fuzz --------------------------------------------------------------------------------------------------
def test_parsers_agree_on_mutated_and_truncated_images(vg, oracle):
    """3000 images with random header and block-header bytes and random truncation through both parsers: same decision,
    same fields; every outcome is VGB_OK or VGB_E_DATA."""
    rng = np.random.default_rng(20261017)
    base = [(R.IDSP, _idsp(900, 2)), (R.IDSP, _idsp(500, 3, interleave=0)), (R.HPS, _hps()),
            (R.HPS, _hps((0x60, 0x41, 0x20), ch=3, loop_block=1, stride=lambda n: n))]
    n_ok = 0
    for case in range(3000):
        kind, img = base[case % len(base)]
        img = img.copy()
        if kind == R.IDSP:
            spots = list(range(0, 0x40 + 0x60 * R.parse(img, kind)[1].channel_count))
        else:
            spots = list(range(0, 0x80)) + [b["offset"] + k for b in R.parse(img, kind)[1].blocks for k in range(12)]
        for _ in range(int(rng.integers(1, 4))):
            at = spots[int(rng.integers(0, len(spots)))]
            img[at] = int(rng.integers(0, 256)) if rng.random() < 0.7 else img[at] ^ (1 << int(rng.integers(0, 8)))
        if rng.random() < 0.3:
            img = img[: int(rng.integers(0, img.size + 1))].copy()
        ok, _, _, _ = _agree(vg, img, kind)
        n_ok += ok
    assert 300 < n_ok < 2700  # the mutations produce both outcomes


# ---- sizing pass of vgb_convert_idsp_hps_to_wave_batch (host only) -------------------------------------------------------
def _sizing(vg, jobs):
    n = len(jobs)
    imgs = [np.ascontiguousarray(j[1], np.uint8) for j in jobs]
    ftab = (C.c_void_p * n)(*[i.ctypes.data for i in imgs])
    lens = (C.c_int64 * n)(*[i.size for i in imgs])
    types = (C.c_int32 * n)(*[j[0] for j in jobs])
    sizes, status = (C.c_int64 * n)(), (C.c_int32 * n)()
    assert vg.lib.vgb_convert_idsp_hps_to_wave_batch(ftab, lens, types, n, sizes, None, status) == 0
    return [status[i] for i in range(n)], [sizes[i] for i in range(n)]


def _msg_of(vg, kind, img):
    imgs = np.ascontiguousarray(img, np.uint8)
    ftab, lens = (C.c_void_p * 1)(imgs.ctypes.data), (C.c_int64 * 1)(imgs.size)
    types, sizes = (C.c_int32 * 1)(kind), (C.c_int64 * 1)()
    st = vg.lib.vgb_convert_idsp_hps_to_wave_batch(ftab, lens, types, 1, sizes, None, None)
    assert st == 0
    status = (C.c_int32 * 1)()
    vg.lib.vgb_convert_idsp_hps_to_wave_batch(ftab, lens, types, 1, sizes, None, status)
    return status[0], (vg.lib.vgb_last_error() or b"").decode()


def sizing_jobs():
    i = _idsp(3000, 2, loop=(100, 2000))
    h = _hps()
    _, hb = R.parse(h, R.HPS)
    return [
        (R.IDSP, i),
        (R.HPS, h),
        (R.HPS, _hps(loop_block=1)),
        (R.IDSP, _idsp(3000, 1, loop=(0, 3000))),
        (R.IDSP, _patch(i, 0x10, ">i", -1)),                           # negative sample count
        (R.IDSP, _patch(i, 0x14, ">i", 3001)),                         # loop start past the end
        (R.IDSP, _patch(i, 0x18, ">i", -2)),                           # loop end negative
        (R.IDSP, _patch(i, 0x18, ">i", 50)),                           # loop end before the start
        (R.IDSP, _idsp(3000, 2, loop=(100, 2000), loop_flags=[0, 0])),  # loop points ignored without a looping channel
        (R.HPS, _patch(h, hb.blocks[0]["offset"] + 4, ">i", 0x80)),    # audio too short
        (R.HPS, _patch(_patch(h, 0x10 + 8, ">i", 0x7ff0), 0x10 + 0x38 + 8, ">i", 0x7ff0)),  # too short, long sample count
        (R.HPS, _patch(_patch(h, 0x10 + 8, ">i", -100), 0x10 + 0x38 + 8, ">i", -100)),      # negative sample count
        (R.HPS, _patch(_hps(loop_block=2), hb.blocks[0]["offset"] + 4, ">i", 0x7fff0000)),  # loop start past the end
        (3, i),                                                         # not IDSP or HPS
        (R.IDSP, _idsp(0, 1)),                                          # empty
        (R.IDSP, _idsp(3000, 2, interleave=0)),                         # one block per channel
        (R.IDSP, _idsp(3000, 2, interleave=-16)),                       # nothing copied: zero rows
    ]


def test_sizing_pass_matches_the_oracle(vg, oracle):
    from vgaudio_b200 import _native as N

    jobs = sizing_jobs()
    status, sizes = _sizing(vg, jobs)
    for k, (kind, img) in enumerate(jobs):
        assert status[k] == R.plan(img, kind)[0], (k, status[k], R.plan(img, kind)[0])
        assert sizes[k] == R.wave_size(img, kind), k
    assert status[:4] == [0] * 4 and status[8] == 0 and status[14:] == [0] * 3
    assert [status[k] for k in (4, 5, 6, 7, 9, 10, 11, 12, 13)] == [N.VGB_E_DATA] + [N.VGB_E_ARG] * 5 + [N.VGB_E_DATA] + [N.VGB_E_ARG] * 2


@pytest.mark.parametrize("k,message", [(4, "negative sample count"), (5, "Loop points must be less than the number of samples"),
                                       (6, "Loop points must be less than the number of samples"),
                                       (7, "The loop end must be greater than the loop start"),
                                       (9, "Audio array length is too short for the specified number of samples."),
                                       (11, "negative sample count"), (12, "Loop points must be less than the number of samples"),
                                       (13, "is not IDSP or HPS")])
def test_sizing_pass_messages(vg, oracle, k, message):
    kind, img = sizing_jobs()[k]
    st, msg = _msg_of(vg, kind, img)
    assert st != 0 and message in msg, msg
