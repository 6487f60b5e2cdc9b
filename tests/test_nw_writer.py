"""NintendoWare writers on the host: the oracle's files read back through both readers, the sizing pass of
vgb_convert_wave_batch against the oracle's file sizes, and every per-file refusal with its message."""
import ctypes as C
import itertools

import numpy as np
import pytest

import vgaudio_b200 as vg
from oracle import pyoracle as O
from vgaudio_b200 import _native as N
from vgaudio_b200 import containers as ct

import nw_reader_oracle as R
import nw_writer_oracle as W

KINDS = (W.BRSTM, W.BCSTM, W.BFSTM)
CODECS = (W.PCM8, W.PCM16, W.GCADPCM)


def _pcm(ch, n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return [(np.sin(t * (0.01 + 0.003 * c)) * 9000 + rng.normal(0, 300, n)).clip(-32768, 32767).astype(np.int16) for c in range(ch)]


def _loops(n):
    """no loop, aligned (loop start 0 and at the alignment), unaligned, loop end inside the last frame"""
    out = [None, (0, n)]
    if n > 200:
        out.append((100, n - 7))
        out.append((n // 3, n))
    if n > 14336 + 100:
        out.append((14336, n - 3))
    if n > 30:
        out.append((0, n - (n % 14 or 1)))
    return out


def size_pass(files, opts):
    n = len(files)
    arrs = [np.ascontiguousarray(f, dtype=np.uint8) for f in files]
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
    lens = (C.c_int64 * n)(*[a.size for a in arrs])
    sizes = (C.c_int64 * n)()
    status = (C.c_int32 * n)()
    N.check(N.lib.vgb_convert_wave_batch(ftab, lens, n, C.byref(opts), sizes, None, status, None, None))
    return list(sizes), list(status)


def _empty_wave():
    """a WAVE image whose data chunk holds no samples (a chunk behind it, so the chunk walk reaches the empty one)"""
    b = bytearray(O.wave_write16([np.zeros(0, np.int16)], 32000).tobytes()) + b"junk" + bytes(8)
    b[4:8] = (len(b) - 8).to_bytes(4, "little")
    return np.frombuffer(bytes(b), dtype=np.uint8)


def _opts(kind, codec, **kw):
    return ct.convert_options(kind, nw_codec_plus1=codec + 1, **kw)


@pytest.mark.parametrize("kind,codec", list(itertools.product(KINDS, CODECS)))
def test_oracle_files_parse_in_both_readers(kind, codec):
    for ch, n in ((1, 14336 * 3 + 5), (2, 100), (3, 14336)):
        for loop in _loops(n):
            st, f = W.write(kind, codec, _pcm(ch, n, ch), 32000, loop)
            assert st == 0
            assert f.size == W.file_size(kind, codec, ch, n, loop)
            info = ct.brstm_parse(f) if kind == W.BRSTM else ct.bcfstm_parse(f)
            rs, rinfo = R.parse(f, kind)
            assert rs == 0, rinfo
            floop = W.aligned_loop(codec, loop)[1]  # GC-ADPCM loops move to a multiple of 14336
            want_n = floop[1] if loop else n
            for got in (info, rinfo):
                assert (got.codec, got.channel_count, got.sample_rate, got.sample_count) == (codec, ch, 32000, want_n)
                assert (got.looping, got.loop_start) == ((1, floop[0]) if loop else (0, 0))
            if kind != W.BRSTM:
                assert info.big_endian == (kind == W.BFSTM)
            if codec == W.GCADPCM:
                for c in range(ch):
                    assert list(info.coefs[c]) == list(O.calculate_coefficients(_pcm(ch, n, ch)[c]))


def test_pcm_round_trips_through_the_reader_chain():
    pcm = _pcm(2, 5000, 7)
    for kind, codec in itertools.product(KINDS, (W.PCM8, W.PCM16)):
        st, f = W.write(kind, codec, pcm, 44100, (10, 4000))
        st2, got, loop = R.decoded_pcm(f, kind)
        assert st == 0 and st2 == 0 and loop == (10, 4000)
        want = [p[:4000] for p in pcm] if codec == W.PCM16 else [((p[:4000] >> 8) << 8).astype(np.int16) for p in pcm]
        for a, b in zip(got, want):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("kind", KINDS)
def test_sizing_pass_matches_the_oracle(kind):
    files, want = [], []
    for codec, ch, endian in itertools.product(CODECS, (1, 2, 3, 8), (0, 1, 2)):
        for n in (1, 13, 14336, 14336 * 2 + 77):
            for loop in _loops(n):
                pcm = _pcm(ch, n, n)
                files.append((codec, endian, O.wave_write16(pcm, 48000, loop)))
                want.append(W.file_size(kind, codec, ch, n, loop))
    for codec, endian in itertools.product(CODECS, (0, 1, 2)):
        idx = [i for i, (c, e, _) in enumerate(files) if c == codec and e == endian]
        sizes, status = size_pass([files[i][2] for i in idx], _opts(kind, codec, nw_endianness=endian))
        assert status == [0] * len(idx)
        assert sizes == [want[i] for i in idx]


def _refusal(kind, codec, wave, **kw):
    sizes, status = size_pass([wave], _opts(kind, codec, **kw))
    return sizes[0], status[0], vg.lib.vgb_last_error().decode()


def test_per_file_refusals_name_their_cause():
    pcm = _pcm(2, 20000, 3)
    cases = [(W.GCADPCM, _empty_wave(), {}, "no samples")]
    for kind in KINDS:
        for codec, wave, kw, msg in cases:
            size, status, err = _refusal(kind, codec, wave, **kw)
            assert (size, status) == (0, vg._native.VGB_E_ARG if "samples" not in msg else vg._native.VGB_E_DATA)
            assert msg in err
        # unaligned loops are aligned, not refused, and size as the oracle's WithAlignment says
        for m in (0, 1, 7, 50):
            size, status, _ = _refusal(kind, W.GCADPCM, O.wave_write16(pcm, 32000, (100, 19000)), nw_loop_point_alignment=m)
            assert status == 0 and size == W.file_size(kind, W.GCADPCM, 2, 20000, (100, 19000), m)
        # PCM codecs never align, and write empty streams
        assert _refusal(kind, W.PCM16, O.wave_write16(pcm, 32000, (100, 19000)))[1] == 0
        assert _refusal(kind, W.PCM16, _empty_wave())[1] == 0
    wide = O.wave_write16([np.zeros(4, np.int16)] * 256, 32000)
    assert "at most 255" in _refusal(W.BFSTM, W.PCM16, wide)[2]
    for bad, msg in (({"nw_codec_plus1": 4}, "nw_codec_plus1 4"), ({"nw_endianness": 3}, "nw_endianness 3")):
        o = ct.convert_options(W.BCSTM, **bad)
        assert size_pass([O.wave_write16(pcm, 32000)], o)[1] == [vg._native.VGB_E_ARG]
        assert msg in vg.lib.vgb_last_error().decode()


def test_oracle_refusals_match_the_sizing_pass():
    assert W.check(W.BRSTM, W.GCADPCM, 2, 20000, (100, 19000)) == 0
    assert W.check(W.BRSTM, W.GCADPCM, 2, 20000, (100, 19000), alignment=1) == 0
    assert W.check(W.BRSTM, W.GCADPCM, 1, 0, None) == W.E_DATA
    assert W.check(W.BRSTM, W.PCM16, 256, 4, None) == W.E_ARG


def test_transcode_still_refuses_nintendoware_targets():
    dsp = O.dsp_write([O.encode(_pcm(1, 100, 1)[0], O.calculate_coefficients(_pcm(1, 100, 1)[0]))],
                      np.stack([O.calculate_coefficients(_pcm(1, 100, 1)[0])]), 32000, 100)
    for kind in KINDS:
        with pytest.raises(Exception):
            ct.transcode_batch([dsp], [ct.CONTAINER_DSP], ct.convert_options(kind))
        assert "out_type" in vg.lib.vgb_last_error().decode()
