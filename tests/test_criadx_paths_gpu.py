"""GPU tests of the CRI ADX encoder on the stimuli of tests/adx_stimuli.py, whose reach into every rare path of
EncodeFrame on the 18-byte and the general path tests/test_oracle_adx_trace.py proves with the oracle's frame trace.

Encoder: vgb_adx_encode_batch and vgb_adx_encode_dev against the oracle, bytes and history bit for bit, serial, by the
library's own segment choice and at forced 3, 8 and 64 segments; the encode stats tap shows that run-ons lock on
fast-locking material and that the cascade carries never-locking material across segment ends.
Decoder: every stimulus's oracle bytes through vgb_adx_decode_batch and the segmented vgb_adx_decode_dev."""
import ctypes as C
import os

import numpy as np
import pytest

import adx_stimuli as A

pytestmark = pytest.mark.gpu

STIMS = A.build()


@pytest.fixture(scope="module")
def wanted(oracle):
    return [oracle.adx_encode_trace(s.pcm, *s.args) for s in STIMS]


@pytest.fixture
def env():
    """set(name, value) for VGB_* knobs; None removes one.  Restored after the test."""
    names = ("VGB_ADX_SEGMENTS", "VGB_ADX_MIN_SEG_FRAMES", "VGB_ADX_DEC_SEGMENTS", "VGB_ADX_DEC_MIN_SEG_FRAMES")
    saved = {k: os.environ.get(k) for k in names}

    def set_(name, value):
        if value is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = str(value)

    yield set_
    for k, v in saved.items():
        set_(k, v)


def _params(vg, s, history=0):
    return vg.criadx.CriAdxParameters(sample_rate=s.rate, frame_size=s.frame_size, version=s.version, padding=s.padding,
                                      type=s.type, filter=s.filter, history=history)


def encode_stats(vg):
    out = (C.c_uint64 * 5)()
    vg._native.check(vg.lib.vgb_adx_debug_encode_stats(out, 5))
    return dict(zip(("segments", "min_seg", "runon_frames", "cascade_frames", "repaired"), (int(v) for v in out)))


def encode_batch(vg, stims):
    adpcm, hist = vg.criadx.encode_batch([s.pcm for s in stims], [_params(vg, s) for s in stims])
    return [np.asarray(a, np.uint8) for a in adpcm], [int(h) for h in hist], encode_stats(vg)


def encode_dev(vg, stims):
    """vgb_adx_encode_dev on one slab; the stats are read while the workspace is still allocated."""
    import torch

    from vgaudio_b200 import _native as N

    n = len(stims)
    lens = np.array([len(s.pcm) for s in stims], np.int32)
    sizes = [vg.criadx.encoded_byte_count(len(s.pcm), s.padding, s.frame_size) for s in stims]
    p_off = np.cumsum([0] + [(int(v) + 15) // 8 * 8 for v in lens])[:-1].astype(np.int64)
    a_off = np.cumsum([0] + [(v + 31) // 16 * 16 for v in sizes])[:-1].astype(np.int64) + 2
    pcm = np.zeros(int(p_off[-1] + lens[-1] + 8), np.int16)
    for o, s in zip(p_off, stims):
        pcm[o: o + len(s.pcm)] = s.pcm
    d_pcm = torch.from_numpy(pcm).cuda()
    d_adpcm = torch.full((int(a_off[-1] + sizes[-1] + 16),), 0xA5, dtype=torch.uint8, device="cuda")
    d_hist = torch.full((n,), 0x5A5A, dtype=torch.int16, device="cuda")
    params = (N.VgbAdxParams * n)(*[N.VgbAdxParams(s.rate, 500, s.frame_size, s.version, 0, s.padding, s.type, s.filter)
                                    for s in stims])
    ws_bytes = int(vg.lib.vgb_adx_workspace_bytes(int(lens.astype(np.int64).sum()), n))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    N.check(vg.lib.vgb_adx_encode_dev(d_pcm.data_ptr(), p_off.ctypes.data, lens.ctypes.data, params, n, d_hist.data_ptr(),
                                      d_adpcm.data_ptr(), a_off.ctypes.data, ws.data_ptr(), ws_bytes, None))
    stats = encode_stats(vg)
    out = d_adpcm.cpu().numpy()
    return [out[o: o + z] for o, z in zip(a_off, sizes)], [int(h) for h in d_hist.cpu().numpy()], stats


ENCODERS = {"batch": encode_batch, "dev": encode_dev}


def check_encoded(stims, wanted, adpcm, hist, what):
    bad = []
    for s, (want, want_hist, trace), got in zip(stims, wanted, adpcm):
        if got.tobytes() != want.tobytes():
            f = int(np.flatnonzero(got != want)[0]) // s.frame_size
            path = "18-byte" if f < s.whole else "general"
            bad.append(f"{s.name}: first differing frame {f} ({path} path), categories {A.categories_at(s, trace, f) or 'none'}")
    for s, (_, want_hist, _), h in zip(stims, wanted, hist):
        if h != want_hist:
            bad.append(f"{s.name}: history {h}, want {want_hist}")
    assert not bad, f"{what}: " + "; ".join(bad)


@pytest.mark.parametrize("mode", list(ENCODERS))
@pytest.mark.parametrize("seg", [1, None, 3, 8, 64])
def test_every_stimulus_bit_exact(vg, wanted, env, mode, seg):
    """The whole set in one launch (18-byte and general-path channels side by side), serial, by the library's choice
    and at forced segment counts with segments as short as MIN_SEG_FRAMES (more segments than whole frames for the
    short channels, whole == 0 beside more than one segment)."""
    env("VGB_ADX_MIN_SEG_FRAMES", A.MIN_SEG_FRAMES)
    env("VGB_ADX_SEGMENTS", seg)
    adpcm, hist, stats = ENCODERS[mode](vg, STIMS)
    check_encoded(STIMS, wanted, adpcm, hist, f"{mode}, segments {seg}")
    if seg is not None:
        assert stats["segments"] == seg and stats["min_seg"] == A.MIN_SEG_FRAMES, stats
    if seg == 1:
        assert stats["runon_frames"] == stats["cascade_frames"] == stats["repaired"] == 0, stats


def _seg_len(whole, seg, min_seg):  # adx_seg_len (adx.cu)
    return max(-(-whole // seg), min_seg)


@pytest.mark.parametrize("mode", list(ENCODERS))
def test_run_ons_lock_on_fast_material(vg, wanted, env, mode):
    """8000 Hz material re-locks within a few frames: the run-ons run, and together encode far fewer frames than the
    segments they start hold (a run-on that ignored its lock would run to its segment's end).  No boundary is left to
    the cascade."""
    idx = [i for i, s in enumerate(STIMS) if s.role == "fast"]
    stims, want = [STIMS[i] for i in idx], [wanted[i] for i in idx]
    env("VGB_ADX_MIN_SEG_FRAMES", 16)
    env("VGB_ADX_SEGMENTS", 8)
    adpcm, hist, st = ENCODERS[mode](vg, stims)
    check_encoded(stims, want, adpcm, hist, f"{mode}, fast material")
    held = sum(s.whole - _seg_len(s.whole, 8, 16) for s in stims)   # frames of segments 1..7
    assert st["segments"] == 8 and st["runon_frames"] >= 7 * len(stims), st
    assert st["runon_frames"] * 20 < held, (st, held)
    assert st["cascade_frames"] == st["repaired"] == 0, st


@pytest.mark.parametrize("mode", list(ENCODERS))
def test_cascade_carries_never_locking_material(vg, oracle, wanted, env, mode):
    """500 Hz material never re-locks (test_oracle_adx_trace proves it), so each channel's cascade repairs a boundary
    and runs on to the channel's end: at least one repair, more cascade frames than one segment holds, and at most one
    repair per channel (a cascade that ignored how far it already carried the truth would repair every later
    boundary again)."""
    idx = [i for i, s in enumerate(STIMS) if s.role == "never"]
    stims, want = [STIMS[i] for i in idx], [wanted[i] for i in idx]
    env("VGB_ADX_MIN_SEG_FRAMES", 16)
    env("VGB_ADX_SEGMENTS", 8)
    adpcm, hist, st = ENCODERS[mode](vg, stims)
    check_encoded(stims, want, adpcm, hist, f"{mode}, never-locking material")
    seg_len = max(_seg_len(s.whole, 8, 16) for s in stims)
    assert 1 <= st["repaired"] <= len(stims), st
    assert st["cascade_frames"] > seg_len, (st, seg_len)
    assert st["runon_frames"] > 0, st


def test_serial_encode_leaves_the_counters_zero(vg, wanted, env):
    env("VGB_ADX_SEGMENTS", 1)
    idx = [i for i, s in enumerate(STIMS) if s.role in ("fast", "never")]
    adpcm, hist, st = encode_batch(vg, [STIMS[i] for i in idx])
    check_encoded([STIMS[i] for i in idx], [wanted[i] for i in idx], adpcm, hist, "serial")
    assert st["segments"] == 1 and st["runon_frames"] == st["cascade_frames"] == st["repaired"] == 0, st


@pytest.mark.parametrize("dec_segments", [None, 8])
def test_decode_of_every_stimulus(vg, oracle, wanted, env, dec_segments):
    """The oracle's bytes of every stimulus decode like oracle.adx_decode through vgb_adx_decode_batch and through the
    time-parallel vgb_adx_decode_dev."""
    import torch

    env("VGB_ADX_DEC_SEGMENTS", dec_segments)
    env("VGB_ADX_DEC_MIN_SEG_FRAMES", 8 if dec_segments else None)
    cfgs = [_params(vg, s, history=h) for s, (_, h, _) in zip(STIMS, wanted)]
    rows = [w for w, _, _ in wanted]
    counts = [len(s.pcm) for s in STIMS]
    want = [oracle.adx_decode(w, len(s.pcm), s.rate, 500, s.frame_size, s.version, h, s.padding, s.type)
            for s, (w, h, _) in zip(STIMS, wanted)]
    if dec_segments is None:
        got = vg.criadx.decode_batch(rows, counts, cfgs)
        for s, g, w in zip(STIMS, got, want):
            assert np.array_equal(g, w), f"decode_batch {s.name}: {int((g != w).sum())} samples differ"
    a_off = np.cumsum([0] + [(r.size + 31) // 16 * 16 for r in rows])[:-1].astype(np.int64)
    p_off = np.cumsum([0] + [c + 8 for c in counts])[:-1].astype(np.int64)
    d_adpcm = torch.zeros(int(a_off[-1] + rows[-1].size + 16), dtype=torch.uint8, device="cuda")
    for o, r in zip(a_off, rows):
        if r.size:
            d_adpcm[int(o): int(o) + r.size] = torch.from_numpy(r).cuda()
    d_pcm = torch.full((int(p_off[-1] + counts[-1] + 8),), 0x5555, dtype=torch.int16, device="cuda")
    vg.criadx.decode_dev(d_adpcm, a_off, [r.size for r in rows], counts, cfgs, d_pcm, p_off)
    pcm = d_pcm.cpu().numpy()
    for s, o, c, w in zip(STIMS, p_off, counts, want):
        g = pcm[o: o + c]
        assert np.array_equal(g, w), f"decode_dev {s.name}: {int((g != w).sum())} samples differ"
