"""The device-resident ("_dev") entry points on layouts a caller builds, against the oracle, bit for bit.

The host batch calls reach the same kernels through layouts the library packs itself: monotone, tight, 16-byte aligned
offsets, library-owned buffers, the library's own stream, one interleave item.  A caller of the _dev calls chooses all of
that.  Here every layout is scrambled (non-monotone offsets, gaps of assorted sizes), every gap and pad of an input slab
holds random poison (the oracle runs on the clean channel, so a read past a channel's end shows up as a wrong byte), and
every output slab starts as a sentinel that must survive outside each channel's documented region.  The calls run with
ragged lengths, per-channel params, given and aliased coefficients, forced segment counts, caller workspaces that are
exactly as large as the sizing functions say and full of stale bytes, caller streams behind a sleeping kernel, and
offsets past 2^32 bytes.

The base-pointer checks (a misaligned d_pcm, d_adpcm, d_coefs or d_workspace is VGB_E_ARG before any device work) are
CPU tests on fake addresses that are never dereferenced."""
import ctypes as C
import re

import numpy as np
import pytest

import gc_stimuli as G
import hca_stimuli as H
from vgaudio_b200 import synth

E_ARG, E_DATA, E_CUDA = -1, -2, -4
SENT8, SENT16 = 0xA5, 0x5A5A


def _has_gpu() -> bool:
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


# ---- base-pointer alignment: fake addresses, no device needed ---------------------------------------------------------
FAKE = 0x7F3000000000  # a 1 MiB-aligned address range nothing is ever read from or written to
BIG_WS = 1 << 40       # large enough for every workspace-size check


def _fake(k: int) -> int:
    return FAKE + k * (1 << 20)


def _dev_calls(vg):
    """name -> (alignment of each base pointer, call(pointers) -> status).  Every other argument is valid, so a call
    with aligned pointers gets past all argument checks."""
    from vgaudio_b200 import _native as N

    L = vg.lib
    n = np.array([1000, 29], np.int32)
    p_off = np.array([1008, 0], np.int64)
    a_off = np.array([0, 576], np.int64)
    gc_par = (N.VgbGcParams * 2)(N.VgbGcParams(1000, 0, 0), N.VgbGcParams(29, 0, 0))
    adx_par = (N.VgbAdxParams * 2)(*[N.VgbAdxParams(48000, 500, 18, 4, 0, 0, 3, 0)] * 2)
    hca_par = (N.VgbHcaParams * 1)(N.VgbHcaParams(2, 0, 0, 1, 48000, 3000, 0, 0, 0))
    info = (N.VgbHcaInfo * 1)()
    assert L.vgb_hca_query(hca_par, info) == 0
    one = np.zeros(1, np.int64)
    stride = np.array([3000], np.int64)
    nbytes = np.array([100000], np.int32)
    return {
        "gc_encode": ({"d_pcm": 16, "d_coefs_in": 2, "d_coefs_out": 2, "d_adpcm": 16, "d_workspace": 16},
                      lambda p: L.vgb_gcadpcm_encode_dev(p["d_pcm"], p_off.ctypes.data, n.ctypes.data, None, 2, p["d_coefs_in"],
                                                         p["d_coefs_out"], p["d_adpcm"], a_off.ctypes.data, p["d_workspace"], BIG_WS, None)),
        "gc_coefs": ({"d_pcm": 16, "d_coefs_out": 2, "d_workspace": 16},
                     lambda p: L.vgb_gcadpcm_coefs_dev(p["d_pcm"], p_off.ctypes.data, n.ctypes.data, 2, p["d_coefs_out"],
                                                       p["d_workspace"], BIG_WS, None)),
        "gc_decode": ({"d_adpcm": 16, "d_coefs": 2, "d_pcm": 16, "d_workspace": 16},
                      lambda p: L.vgb_gcadpcm_decode_dev(p["d_adpcm"], a_off.ctypes.data, p["d_coefs"], gc_par, 2, p["d_pcm"],
                                                         p_off.ctypes.data, p["d_workspace"], BIG_WS, None)),
        "adx_encode": ({"d_pcm": 16, "d_history_out": 2, "d_adpcm": 2, "d_workspace": 8},
                       lambda p: L.vgb_adx_encode_dev(p["d_pcm"], p_off.ctypes.data, n.ctypes.data, adx_par, 2, p["d_history_out"],
                                                      p["d_adpcm"], a_off.ctypes.data, p["d_workspace"], BIG_WS, None)),
        "adx_decode": ({"d_pcm": 2, "d_workspace": 8},
                       lambda p: L.vgb_adx_decode_dev(_fake(9), one.ctypes.data, nbytes.ctypes.data, n.ctypes.data, adx_par, 1,
                                                      p["d_pcm"], one.ctypes.data, p["d_workspace"], BIG_WS, None)),
        "hca_encode": ({"d_pcm": 2, "d_workspace": 8},
                       lambda p: L.vgb_hca_encode_dev(p["d_pcm"], one.ctypes.data, stride.ctypes.data, hca_par, 1, None, _fake(9),
                                                      one.ctypes.data, p["d_workspace"], BIG_WS, None)),
        "hca_decode": ({"d_pcm": 2, "d_workspace": 8},
                       lambda p: L.vgb_hca_decode_dev(_fake(9), one.ctypes.data, info, 1, p["d_pcm"], one.ctypes.data,
                                                      stride.ctypes.data, p["d_workspace"], BIG_WS, None)),
    }


ALIGN = {"gc_encode": {"d_pcm": 16, "d_coefs_in": 2, "d_coefs_out": 2, "d_adpcm": 16, "d_workspace": 16},
         "gc_coefs": {"d_pcm": 16, "d_coefs_out": 2, "d_workspace": 16},
         "gc_decode": {"d_adpcm": 16, "d_coefs": 2, "d_pcm": 16, "d_workspace": 16},
         "adx_encode": {"d_pcm": 16, "d_history_out": 2, "d_adpcm": 2, "d_workspace": 8},
         "adx_decode": {"d_pcm": 2, "d_workspace": 8},
         "hca_encode": {"d_pcm": 2, "d_workspace": 8},
         "hca_decode": {"d_pcm": 2, "d_workspace": 8}}
MISALIGNED = [(call, ptr, by) for call, ptrs in ALIGN.items() for ptr, a in ptrs.items() for by in sorted({1, 2, a // 2} - {0, a})]


def _aligned(ptrs):
    return {name: _fake(k) for k, name in enumerate(ptrs)}


def test_alignment_table_matches_the_calls(vg):
    assert {k: v[0] for k, v in _dev_calls(vg).items()} == ALIGN


@pytest.mark.parametrize("call,ptr,by", MISALIGNED)
def test_misaligned_base_pointer_is_refused(vg, call, ptr, by):
    """A base pointer the kernels cannot use is VGB_E_ARG, with a message naming it, before the call touches a device
    (the addresses are fake: any device work would fault or fail with VGB_E_CUDA)."""
    aligns, fn = _dev_calls(vg)[call]
    p = _aligned(aligns)
    p[ptr] += by
    before = vg.lib.vgb_kernel_launch_count()
    assert fn(p) == E_ARG
    msg = vg.lib.vgb_last_error().decode()
    assert ptr in msg and "aligned" in msg, msg
    assert vg.lib.vgb_kernel_launch_count() == before


@pytest.mark.skipif(_has_gpu(), reason="fake device addresses: only run where no device can be reached")
@pytest.mark.parametrize("call", list(ALIGN))
def test_aligned_base_pointers_pass_the_argument_checks(vg, call):
    """The same calls with aligned pointers get past every argument check and fail only at device init."""
    aligns, fn = _dev_calls(vg)[call]
    assert fn(_aligned(aligns)) == E_CUDA, vg.lib.vgb_last_error()


# ---- layouts ----------------------------------------------------------------------------------------------------------
def _up(x: int, a: int) -> int:
    return -(-x // a) * a


GAPS = (0, 1, 3, 2, 17, 5, 1, 40)


def _scatter(rng, sizes, unit: int, shift=None):
    """Offsets (elements) for regions of `sizes` elements: a shuffled, non-monotone order, each offset a multiple of
    `unit` plus shift[i], each region followed by its pad to `unit` and a gap of 0..40 units.  -> (offsets, slab length)"""
    n = len(sizes)
    order = list(rng.permutation(n))
    if n > 2 and order == sorted(order):
        order.reverse()
    shift = [0] * n if shift is None else shift
    off = np.zeros(n, np.int64)
    at = unit * int(rng.integers(1, 5))
    for k, i in enumerate(order):
        off[i] = at + shift[i]
        at = _up(at + shift[i] + int(sizes[i]), unit) + unit * GAPS[(k + int(rng.integers(0, 8))) % len(GAPS)]
    return off, at + unit


def _poisoned(rng, length: int, dtype, rows, offsets) -> np.ndarray:
    """A host slab of random poison with rows[i] at offsets[i]."""
    info = np.iinfo(dtype)
    slab = rng.integers(info.min, info.max + 1, length, dtype=dtype)
    for r, o in zip(rows, offsets):
        slab[int(o): int(o) + len(r)] = r
    return slab


def _check_regions(got: np.ndarray, offsets, wants, sentinel, what: str):
    """Each region equals its want; every element outside all regions still holds the sentinel."""
    outside = np.ones(got.size, bool)
    for i, (o, w) in enumerate(zip(offsets, wants)):
        o = int(o)
        seg = got[o: o + len(w)]
        if not np.array_equal(seg, w):
            bad = np.flatnonzero(seg != w)
            raise AssertionError(f"{what}: row {i}: {bad.size} of {len(w)} elements differ, first at {int(bad[0])}")
        outside[o: o + len(w)] = False
    stray = np.flatnonzero(outside & (got != sentinel))
    assert stray.size == 0, f"{what}: {stray.size} elements outside the rows were written, first at {int(stray[0])}"


def _torch():
    import torch

    return torch


def _cuda(a: np.ndarray):
    return _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def _arr(t) -> np.ndarray:
    return t.cpu().numpy()


def _need(vg, fn) -> int:
    """The workspace size a call asks for, from its 'workspace too small: need N bytes' refusal."""
    assert fn(0) == E_ARG
    m = re.search(r"need (\d+) bytes", vg.lib.vgb_last_error().decode())
    assert m, vg.lib.vgb_last_error()
    return int(m.group(1))


# ---- the calls, each with its inputs, its oracle outputs and its checks -------------------------------------------------
class Case:
    """One _dev call on a scrambled layout.  inputs: {name: (host slab, device slab)}; outputs: {name: device slab}
    reset to their sentinels by reset(); run(ws, ws_bytes, stream) -> status; check(outs) against the oracle."""

    sentinels: dict

    def reset(self):
        for k, t in self.outputs.items():
            t.fill_(self.sentinels[k])

    def poison_inputs(self):
        for _, d in self.inputs.values():
            d.fill_(0x11)

    def snapshot(self):
        return {k: _arr(t) for k, t in self.outputs.items()}

    def workspace(self, fill=0):
        return _torch().full((self.ws_bytes,), fill, dtype=_torch().uint8, device="cuda")


def _gc_params(N, rows):
    return (N.VgbGcParams * len(rows))(*[N.VgbGcParams(sc, h1, h2) for sc, h1, h2 in rows])


RAGGED = [0, 1, 13, 14, 15, 16, 28, 29] + [14 * 7 + r for r in range(14)] + [14 * 700 + 3, 14 * 2100 - 5]
EXTREMES = [(0, 0), (1234, -4321), (32767, -32768), (-32768, 32767), (-1, 1)]


def _gc_channels(rng, stims):
    """(pcm, coefs, (sample_count, h1, h2)) for the ragged lengths (every residue mod 14, with -1, shorter and 0 sample
    counts and extreme histories) and the rare-path stimulus channels of gc_stimuli with their own coefficients."""
    from oracle import pyoracle as O

    out = []
    for i, n in enumerate(RAGGED):
        pcm = synth.channel(100 + i, n, degenerate=False) if n else np.zeros(0, np.int16)
        h1, h2 = EXTREMES[i % len(EXTREMES)]
        sc = (-1, max(n - 1 - i % 13, 0), 0, -1, n)[i % 5]
        out.append((pcm, O.calculate_coefficients(pcm), (sc, h1, h2)))
    for s in stims:
        out.append((s.pcm, s.coefs, (s.sample_count, s.h1, s.h2)))
    order = rng.permutation(len(out))
    return [out[i] for i in order]


class GcEncode(Case):
    """vgb_gcadpcm_encode_dev (coefs: 'null' = analysis, 'given', 'alias' = d_coefs_in is d_coefs_out) or, with
    coefs='only', vgb_gcadpcm_coefs_dev."""

    def __init__(self, vg, oracle, chans, coefs: str, seed: int):
        from vgaudio_b200 import _native as N

        torch = _torch()
        self.vg, self.mode = vg, coefs
        rng = np.random.default_rng(seed)
        self.n = len(chans)
        self.lens = np.array([len(p) for p, _, _ in chans], np.int32)
        self.params = [p for _, _, p in chans]
        self.c_params = _gc_params(N, self.params)
        self.p_off, p_len = _scatter(rng, self.lens, 8)
        host = _poisoned(rng, p_len, np.int16, [p for p, _, _ in chans], self.p_off)
        self.inputs = {"pcm": (host, _cuda(host))}
        given = np.stack([c for _, c, _ in chans]).astype(np.int16)
        self.coefs_want = np.stack([oracle.calculate_coefficients(p) for p, _, _ in chans]) if coefs in ("null", "only") else given
        self.outputs = {"coefs": torch.empty((self.n + 1) * 16, dtype=torch.int16, device="cuda")}
        self.sentinels = {"coefs": SENT16, "adpcm": SENT8}
        self.coefs_in = None
        if coefs == "given":
            self.coefs_in = _cuda(given.ravel())
        self.given = given
        frames = int(sum(-(-int(n) // 14) for n in self.lens))
        self.ws_bytes = int(vg.lib.vgb_gcadpcm_workspace_bytes(frames, self.n))
        if coefs != "only":
            self.adpcm_want = [oracle.encode(p, self.coefs_want[i], *self.params[i]) for i, (p, _, _) in enumerate(chans)]
            self.a_off, a_len = _scatter(rng, [w.size for w in self.adpcm_want], 16)
            self.outputs["adpcm"] = torch.empty(a_len, dtype=torch.uint8, device="cuda")
        self.reset()

    def reset(self):
        super().reset()
        if self.mode == "alias":
            self.outputs["coefs"][: self.n * 16] = _cuda(self.given.ravel())

    def run(self, ws, ws_bytes=None, stream=0):
        L, o = self.vg.lib, self.outputs
        ws_bytes = ws.numel() if ws_bytes is None else ws_bytes
        d_pcm = self.inputs["pcm"][1].data_ptr()
        if self.mode == "only":
            return L.vgb_gcadpcm_coefs_dev(d_pcm, self.p_off.ctypes.data, self.lens.ctypes.data, self.n, o["coefs"].data_ptr(),
                                           ws.data_ptr(), ws_bytes, stream)
        c_in = {"null": None, "given": self.coefs_in.data_ptr() if self.coefs_in is not None else None,
                "alias": o["coefs"].data_ptr()}[self.mode]
        return L.vgb_gcadpcm_encode_dev(d_pcm, self.p_off.ctypes.data, self.lens.ctypes.data, self.c_params, self.n, c_in,
                                        o["coefs"].data_ptr(), o["adpcm"].data_ptr(), self.a_off.ctypes.data, ws.data_ptr(),
                                        ws_bytes, stream)

    def check(self, got=None):
        got = got or self.snapshot()
        _check_regions(got["coefs"], [0], [self.coefs_want.ravel()], SENT16, f"gc {self.mode}: coefficients")
        if "adpcm" in got:
            _check_regions(got["adpcm"], self.a_off, self.adpcm_want, SENT8, f"gc {self.mode}: adpcm")
        if self.coefs_in is not None:
            assert np.array_equal(_arr(self.coefs_in), self.given.ravel())


class GcDecode(Case):
    """vgb_gcadpcm_decode_dev of oracle-encoded channels, with `bad` channels whose frame headers select predictors
    8..15 (the device wraps the lookup, predictor & 7, and names the lowest such channel in the status word)."""

    def __init__(self, vg, oracle, chans, seed: int, bad=()):
        from vgaudio_b200 import _native as N

        torch = _torch()
        self.vg = vg
        rng = np.random.default_rng(seed)
        self.n = len(chans)
        coefs = np.stack([c for _, c, _ in chans]).astype(np.int16)
        rows, self.params, self.want = [], [], []
        for i, (pcm, co, (sc, h1, h2)) in enumerate(chans):
            adpcm = oracle.encode(pcm, co)
            count = len(pcm) if i % 3 else max(len(pcm) - (i % 29), 0)  # whole channels and shorter counts
            h1, h2 = EXTREMES[(i + 2) % len(EXTREMES)]
            wrapped = adpcm.copy()
            if i in bad and adpcm.size:
                f = int(rng.integers(0, adpcm.size // 8)) if adpcm.size >= 8 else 0
                f = min(f, max((count - 1) // 14, 0))  # a frame the decode reaches
                adpcm[8 * f] = (adpcm[8 * f] & 0x0F) | (int(rng.integers(8, 16)) << 4)
                wrapped[8 * f] = adpcm[8 * f] & 0x7F
            rows.append(adpcm)
            self.params.append((count, h1, h2))
            self.want.append(oracle.decode(wrapped, co, count, h1, h2))
        self.c_params = _gc_params(N, self.params)
        self.a_off, a_len = _scatter(rng, [r.size for r in rows], 16)
        host = _poisoned(rng, a_len, np.uint8, rows, self.a_off)
        self.inputs = {"adpcm": (host, _cuda(host))}
        self.coefs = _cuda(coefs.ravel())
        self.p_off, p_len = _scatter(rng, [w.size for w in self.want], 8)
        self.outputs = {"pcm": torch.empty(p_len, dtype=torch.int16, device="cuda")}
        self.sentinels = {"pcm": SENT16}
        self.ws_bytes = int(vg.lib.vgb_gcadpcm_workspace_bytes(32, self.n))
        self.reset()

    def run(self, ws, ws_bytes=None, stream=0):
        return self.vg.lib.vgb_gcadpcm_decode_dev(self.inputs["adpcm"][1].data_ptr(), self.a_off.ctypes.data, self.coefs.data_ptr(),
                                                  self.c_params, self.n, self.outputs["pcm"].data_ptr(), self.p_off.ctypes.data,
                                                  ws.data_ptr(), ws.numel() if ws_bytes is None else ws_bytes, stream)

    def status(self, ws, stream=0):
        return self.vg.lib.vgb_gcadpcm_decode_dev_status(ws.data_ptr(), self.n, stream)

    def check(self, got=None):
        got = got or self.snapshot()
        _check_regions(got["pcm"], self.p_off, self.want, SENT16, "gc decode")


# (frame size, version, type, filter, padding, sample rate): every type, both versions, frame sizes other than 18, padding
ADX_CONFIGS = [(18, 4, 3, 0, 0, 48000), (18, 3, 4, 0, 0, 44100), (18, 4, 2, 0, 0, 48000), (18, 4, 2, 3, 37, 32000),
               (9, 4, 3, 0, 3, 48000), (33, 3, 4, 0, 0, 22050), (3, 4, 2, 2, 1, 48000), (130, 4, 3, 0, 600, 48000),
               (18, 3, 3, 0, 1000, 48000), (18, 4, 4, 0, 0, 48000), (18, 4, 2, 1, 0, 44100), (11, 3, 2, 0, 0, 48000)]


class AdxEncode(Case):
    """vgb_adx_encode_dev; adpcm offsets cycle through 2, 6, 10 (mod 16) and 16-aligned values; history optional."""

    def __init__(self, vg, oracle, seed: int, history=True, long=False):
        from vgaudio_b200 import _native as N

        torch = _torch()
        self.vg = vg
        rng = np.random.default_rng(seed)
        rows, cfgs = [], []
        for i, (fs, version, type, filt, padding, rate) in enumerate(ADX_CONFIGS * 2):
            n = int(rng.integers(0, 300)) * 32 + int(rng.integers(0, 32))  # ragged, partial last frames
            if long and fs == 18 and padding == 0:
                n = 32 * 6000 + i  # long enough for forced segments
            if version == 4 and padding == 0:
                n = max(n, 1)
            rows.append(synth.channel(200 + i, n, rate, degenerate=False))
            cfgs.append((fs, version, type, filt, padding, rate))
        self.n = len(rows)
        self.lens = np.array([len(r) for r in rows], np.int32)
        self.c_params = (N.VgbAdxParams * self.n)(*[N.VgbAdxParams(rate, 500, fs, v, 0, pad, t, f) for fs, v, t, f, pad, rate in cfgs])
        enc = [oracle.adx_encode(r, rate, fs, v, pad, t, f) for r, (fs, v, t, f, pad, rate) in zip(rows, cfgs)]
        self.want = [e[0] for e in enc]
        self.hist_want = np.array([e[1] for e in enc], np.int64).astype(np.int16)
        self.p_off, p_len = _scatter(rng, self.lens, 8)
        host = _poisoned(rng, p_len, np.int16, rows, self.p_off)
        self.inputs = {"pcm": (host, _cuda(host))}
        self.a_off, a_len = _scatter(rng, [w.size for w in self.want], 16, shift=[(0, 2, 6, 10)[i % 4] for i in range(self.n)])
        self.outputs = {"adpcm": torch.empty(a_len, dtype=torch.uint8, device="cuda")}
        self.sentinels = {"adpcm": SENT8, "hist": SENT16}
        if history:
            self.outputs["hist"] = torch.empty(self.n + 8, dtype=torch.int16, device="cuda")
        self.ws_bytes = int(vg.lib.vgb_adx_workspace_bytes(int(self.lens.astype(np.int64).sum()), self.n))
        self.reset()

    def run(self, ws, ws_bytes=None, stream=0):
        o = self.outputs
        return self.vg.lib.vgb_adx_encode_dev(self.inputs["pcm"][1].data_ptr(), self.p_off.ctypes.data, self.lens.ctypes.data, self.c_params,
                                              self.n, o["hist"].data_ptr() if "hist" in o else None, o["adpcm"].data_ptr(),
                                              self.a_off.ctypes.data, ws.data_ptr(), ws.numel() if ws_bytes is None else ws_bytes, stream)

    def check(self, got=None):
        got = got or self.snapshot()
        _check_regions(got["adpcm"], self.a_off, self.want, SENT8, "adx encode")
        if "hist" in got:
            _check_regions(got["hist"], [0], [self.hist_want], SENT16, "adx history")


class HcaEncode(Case):
    """vgb_hca_encode_dev: streams of `nch` channels, channel_stride above sample_count with poisoned gaps, odd pcm and
    frame offsets, looping streams with different loop points; `streams` overrides the material (mono, with `bitrate`)."""

    def __init__(self, vg, oracle, seed: int, nch=2, quality=2, bitrate=0, streams=None, info=True):
        from vgaudio_b200 import _native as N

        torch = _torch()
        self.vg = vg
        rng = np.random.default_rng(seed)
        if streams is None:
            spec = [(3000, None), (12000, (1000, 9000)), (7777, (500, 7777)), (1, None), (5000, (4095, 4097))]
            streams = [([synth.channel(300 + 10 * s + c, n, degenerate=False) for c in range(nch)], loop) for s, (n, loop) in enumerate(spec)]
        self.n = len(streams)
        self.nch = len(streams[0][0])
        self.c_params = (N.VgbHcaParams * self.n)()
        self.want, self.info_want, pcm_rows, self.stride = [], [], [], []
        self.fails = []
        for s, (chans, loop) in enumerate(streams):
            n = len(chans[0])
            lp = (1, loop[0], loop[1]) if loop else (0, 0, 0)
            self.c_params[s] = N.VgbHcaParams(quality, bitrate, 0, self.nch, 48000, n, *lp)
            try:
                info, frames = oracle.hca_encode(chans, 48000, quality, bitrate, loop=loop)
                self.want.append(frames.ravel())
                self.info_want.append(info.as_dict())
                self.fails.append(False)
            except ValueError:  # "Bitrate is set too low."
                self.want.append(None)
                self.info_want.append(None)
                self.fails.append(True)
            stride = n + int(rng.integers(1, 40))
            self.stride.append(stride)
            row = rng.integers(-32768, 32768, stride * self.nch, dtype=np.int16)
            for c, x in enumerate(chans):
                row[c * stride: c * stride + n] = x
            pcm_rows.append(row[: (self.nch - 1) * stride + n])
        self.stride = np.array(self.stride, np.int64)
        self.p_off, p_len = _scatter(rng, [r.size for r in pcm_rows], 8, shift=[(1, 0, 3, 5, 2)[s % 5] for s in range(self.n)])
        host = _poisoned(rng, p_len, np.int16, pcm_rows, self.p_off)
        self.inputs = {"pcm": (host, _cuda(host))}
        sizes = []
        for s in range(self.n):
            q = (N.VgbHcaInfo * 1)()
            assert vg.lib.vgb_hca_query(C.byref(self.c_params[s]), q) == 0
            sizes.append(q[0].frame_count * q[0].frame_size)
            if self.want[s] is not None:
                assert sizes[-1] == self.want[s].size
        self.sizes = sizes
        self.f_off, f_len = _scatter(rng, sizes, 16, shift=[(3, 0, 1, 7, 0)[s % 5] for s in range(self.n)])
        self.outputs = {"frames": torch.empty(f_len, dtype=torch.uint8, device="cuda")}
        self.sentinels = {"frames": SENT8}
        self.info = (N.VgbHcaInfo * self.n)() if info else None
        self.ws_bytes = int(vg.lib.vgb_hca_workspace_bytes(self.n))
        self.reset()

    def run(self, ws, ws_bytes=None, stream=0):
        return self.vg.lib.vgb_hca_encode_dev(self.inputs["pcm"][1].data_ptr(), self.p_off.ctypes.data, self.stride.ctypes.data,
                                              self.c_params, self.n, self.info, self.outputs["frames"].data_ptr(), self.f_off.ctypes.data,
                                              ws.data_ptr(), ws.numel() if ws_bytes is None else ws_bytes, stream)

    def status(self, ws, stream=0):
        return self.vg.lib.vgb_hca_encode_dev_status(ws.data_ptr(), self.n, stream)

    def check(self, got=None):
        """Streams that encode equal the oracle; a failing stream's frames are unspecified, but stay inside its region."""
        frames = (got or self.snapshot())["frames"]
        wants = []
        for s in range(self.n):
            o = int(self.f_off[s])
            wants.append(frames[o: o + self.sizes[s]] if self.fails[s] else self.want[s])
        _check_regions(frames, self.f_off, wants, SENT8, "hca encode")
        if self.info is not None:
            for s in range(self.n):
                if not self.fails[s]:
                    assert self.info[s].as_dict() == self.info_want[s], s


# ---- GC-ADPCM ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def stims(oracle):
    return G.build()


@pytest.fixture(scope="module")
def gc_chans(oracle, stims):
    return _gc_channels(np.random.default_rng(7), stims)


@pytest.fixture
def env(monkeypatch):
    return monkeypatch.setenv


def _splice_stats(vg):
    from vgaudio_b200 import _native as N

    out = (C.c_uint64 * 4)()
    N.check(vg.lib.vgb_gcadpcm_debug_splice_stats(out, 4))
    return [int(v) for v in out]


@pytest.mark.gpu
@pytest.mark.parametrize("seg", [1, 3, 8])
def test_gc_encode_dev_scrambled_layout(vg, oracle, gc_chans, env, seg):
    """Every coefficient mode on the ragged and rare-path channels, cut into 1, 3 and 8 segments: coefficients and
    bytes equal the oracle's and nothing outside a channel's bytes is written."""
    env("VGB_GC_MIN_SEG_FRAMES", str(G.MIN_SEG_FRAMES))
    env("VGB_GC_SEGMENTS", str(seg))
    for k, mode in enumerate(("given", "null", "alias")):
        case = GcEncode(vg, oracle, gc_chans, mode, seed=10 * seg + k)
        ws = case.workspace()
        assert case.run(ws) == 0, vg.lib.vgb_last_error()
        case.check()
        assert _splice_stats(vg)[0] == seg  # the workspace is still allocated


@pytest.mark.gpu
def test_gc_encode_dev_runs_run_ons_and_the_cascade(vg, oracle, gc_chans, env):
    """The splice stats of _dev encodes (read while each call's workspace is alive): run-on and cascade frames occur."""
    env("VGB_GC_MIN_SEG_FRAMES", str(G.MIN_SEG_FRAMES))
    seen = []
    for seg in (3, 8):
        env("VGB_GC_SEGMENTS", str(seg))
        case = GcEncode(vg, oracle, gc_chans, "given", seed=90 + seg)
        ws = case.workspace(0xFF)
        assert case.run(ws) == 0, vg.lib.vgb_last_error()
        case.check()
        seen.append(_splice_stats(vg))
        del ws
    assert all(s[1] > 0 for s in seen), seen          # run-on frames
    assert max(s[2] for s in seen) > 0, seen          # cascade frames


@pytest.mark.gpu
def test_gc_coefs_dev_scrambled_layout(vg, oracle, gc_chans):
    case = GcEncode(vg, oracle, gc_chans, "only", seed=3)
    assert case.run(case.workspace()) == 0, vg.lib.vgb_last_error()
    case.check()


@pytest.mark.gpu
def test_gc_decode_dev_scrambled_layout_and_status(vg, oracle, gc_chans):
    """Clean channels decode exactly; predictors 8..15 in some channels make the status call name the lowest of them
    while every channel stays exact (the lookup wraps); the next clean call on the same workspace is VGB_OK."""
    clean = GcDecode(vg, oracle, gc_chans, seed=5)
    ws = clean.workspace(0xFF)
    assert clean.run(ws) == 0, vg.lib.vgb_last_error()
    assert clean.status(ws) == 0, vg.lib.vgb_last_error()
    clean.check()
    bad = [i for i, (p, _, _) in enumerate(gc_chans) if len(p) > 300][2:5]
    broken = GcDecode(vg, oracle, gc_chans, seed=5, bad=bad)
    assert broken.run(ws) == 0
    assert broken.status(ws) == E_DATA
    assert f"channel {bad[0]}:" in vg.lib.vgb_last_error().decode()
    broken.check()
    clean.reset()
    assert clean.run(ws) == 0
    assert clean.status(ws) == 0, vg.lib.vgb_last_error()
    clean.check()


# ---- ADX --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("history", [True, False])
def test_adx_encode_dev_scrambled_layout(vg, oracle, history):
    case = AdxEncode(vg, oracle, seed=21 + history, history=history)
    assert case.run(case.workspace()) == 0, vg.lib.vgb_last_error()
    case.check()


@pytest.mark.gpu
@pytest.mark.parametrize("segments,min_seg", [("1", "16"), ("5", "16"), ("64", "64")])
def test_adx_encode_dev_forced_segments(vg, oracle, env, segments, min_seg):
    env("VGB_ADX_SEGMENTS", segments)
    env("VGB_ADX_MIN_SEG_FRAMES", min_seg)
    case = AdxEncode(vg, oracle, seed=30, long=True)
    assert case.run(case.workspace(0xFF)) == 0, vg.lib.vgb_last_error()
    case.check()


# ---- HCA --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nch,quality,info", [(1, 2, True), (2, 1, False), (5, 3, True), (8, 4, True)])
def test_hca_encode_dev_scrambled_layout(vg, oracle, nch, quality, info):
    case = HcaEncode(vg, oracle, seed=40 + nch, nch=nch, quality=quality, info=info)
    ws = case.workspace(0xFF)
    assert case.run(ws) == 0, vg.lib.vgb_last_error()
    assert case.status(ws) == 0, vg.lib.vgb_last_error()
    case.check()


@pytest.mark.gpu
def test_hca_encode_dev_bitrate_too_low_fails_its_stream_alone(vg, oracle):
    """A stream the shared bitrate cannot carry, between streams that encode: the status call names it, the others equal
    the oracle, and a later clean call on the same workspace is VGB_OK."""
    s = H.bitrate_too_low()
    assert s.fails
    quiet = [([np.zeros(3000, np.int16)], None), ([np.zeros(5000, np.int16)], (100, 4000)), ([np.zeros(1, np.int16)], None)]
    case = HcaEncode(vg, oracle, seed=50, bitrate=s.bitrate, quality=s.quality, streams=quiet[:2] + [(s.streams[0], None)] + quiet[2:])
    assert case.fails == [False, False, True, False]
    ws = case.workspace()
    assert case.run(ws) == 0, vg.lib.vgb_last_error()
    assert case.status(ws) == E_DATA
    assert "stream 2: Bitrate is set too low." in vg.lib.vgb_last_error().decode()
    case.check()
    clean = HcaEncode(vg, oracle, seed=51, bitrate=s.bitrate, quality=s.quality, streams=quiet)
    assert clean.run(ws) == 0
    assert clean.status(ws) == 0, vg.lib.vgb_last_error()
    clean.check()


# ---- workspaces -------------------------------------------------------------------------------------------------------
def _cases(vg, oracle, gc_chans):
    few = gc_chans[:12] + [c for c in gc_chans if len(c[0]) > 20000][:2]
    return {"gc_encode": GcEncode(vg, oracle, few, "null", seed=61), "gc_coefs": GcEncode(vg, oracle, few, "only", seed=62),
            "gc_decode": GcDecode(vg, oracle, few, seed=63), "adx_encode": AdxEncode(vg, oracle, seed=64),
            "hca_encode": HcaEncode(vg, oracle, seed=65)}


@pytest.fixture(scope="module")
def cases(vg, oracle, gc_chans):
    return _cases(vg, oracle, gc_chans)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["gc_encode", "gc_coefs", "gc_decode", "adx_encode", "hca_encode"])
def test_workspace_exact_size_short_by_one_and_stale_bytes(vg, cases, name):
    """The least workspace the call takes works, one byte less is VGB_E_ARG with nothing launched or written, and a
    workspace full of 0xFF or random bytes gives the same output as a zeroed one."""
    torch = _torch()
    case = cases[name]
    case.reset()
    need = _need(vg, lambda b: case.run(case.workspace(), b))
    assert need <= case.ws_bytes
    if not name.startswith("gc"):
        assert need == case.ws_bytes  # the sizing function is the exact requirement
    ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    before = vg.lib.vgb_kernel_launch_count()
    assert case.run(ws, need - 1) == E_ARG
    assert "workspace too small" in vg.lib.vgb_last_error().decode()
    assert vg.lib.vgb_kernel_launch_count() == before
    for k, t in case.outputs.items():
        assert (t == case.sentinels[k]).all(), k  # untouched
    assert case.run(ws, need) == 0, vg.lib.vgb_last_error()
    first = case.snapshot()
    case.check(first)
    gen = torch.Generator(device="cuda").manual_seed(9)
    for fill in ("ff", "random"):
        case.reset()
        big = case.workspace(0xFF)
        if fill == "random":
            big = torch.randint(0, 256, (case.ws_bytes,), dtype=torch.uint8, device="cuda", generator=gen)
        assert case.run(big) == 0, vg.lib.vgb_last_error()
        again = case.snapshot()
        for k in first:
            assert np.array_equal(first[k], again[k]), (fill, k)


@pytest.mark.gpu
def test_one_workspace_across_calls_of_every_kind(vg, cases):
    """One workspace, reused by calls of different kinds and shapes in turn (each sees what the last one left), twice
    round: every output equals the oracle."""
    torch = _torch()
    ws = torch.randint(0, 256, (max(c.ws_bytes for c in cases.values()),), dtype=torch.uint8, device="cuda")
    for _ in range(2):
        for name in ("gc_encode", "adx_encode", "gc_decode", "hca_encode", "gc_coefs"):
            case = cases[name]
            case.reset()
            assert case.run(ws) == 0, (name, vg.lib.vgb_last_error())
            if hasattr(case, "status"):
                assert case.status(ws) == 0, (name, vg.lib.vgb_last_error())
            case.check()


# ---- streams ----------------------------------------------------------------------------------------------------------
SLEEP_CYCLES = 200_000_000  # ~0.1 s on an H100


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["gc_encode", "gc_coefs", "gc_decode", "adx_encode", "hca_encode"])
def test_call_is_ordered_on_the_callers_stream(vg, cases, name):
    """On a side stream: a long sleep, a non-blocking H2D copy of the real input over a poisoned device slab, the call,
    and a clone of its output, with no host synchronisation in between.  Work the library put on any other stream would
    see the poisoned input or race the clone."""
    torch = _torch()
    case = cases[name]
    case.reset()
    case.poison_inputs()
    pinned = {k: torch.from_numpy(h).pin_memory() for k, (h, _) in case.inputs.items()}
    ws = case.workspace()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for k, (_, d) in case.inputs.items():
            d.copy_(pinned[k], non_blocking=True)
        assert case.run(ws, stream=s.cuda_stream) == 0, vg.lib.vgb_last_error()
        clones = {k: t.clone() for k, t in case.outputs.items()}
    s.synchronize()
    if hasattr(case, "status"):
        assert case.status(ws, s.cuda_stream) == 0
    case.check({k: _arr(t) for k, t in clones.items()})


@pytest.mark.gpu
def test_two_streams_overlap_with_separate_workspaces(vg, oracle, gc_chans):
    """Two encode calls on two streams with their own workspaces and outputs, enqueued behind sleeps so they overlap."""
    torch = _torch()
    a = GcEncode(vg, oracle, gc_chans, "null", seed=71)
    b = AdxEncode(vg, oracle, seed=72)
    c = GcEncode(vg, oracle, gc_chans[::-1], "given", seed=73)
    wa, wb, wc = a.workspace(), b.workspace(), c.workspace()
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for s, case, w in ((s1, a, wa), (s2, b, wb), (s2, c, wc)):
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES // 4)
            assert case.run(w, stream=s.cuda_stream) == 0, vg.lib.vgb_last_error()
    torch.cuda.synchronize()
    for case in (a, b, c):
        case.check()


# ---- 64-bit offsets ---------------------------------------------------------------------------------------------------
FAR = 1 << 32  # bytes


@pytest.mark.gpu
def test_offsets_past_4_gib(vg, oracle):
    """One channel of each encode call at a sample and byte offset past 2^32 bytes (next to one near the start), and the
    GC-ADPCM decode back from there."""
    torch = _torch()
    from vgaudio_b200 import _native as N

    free, _ = torch.cuda.mem_get_info()
    if free < 12 * (1 << 30):
        pytest.skip(f"needs about 12 GB of free HBM for two 4 GiB slabs, {free / (1 << 30):.1f} GB free")
    L = vg.lib
    n = 14 * 300 + 5
    x = [synth.channel(500, n, degenerate=False), synth.channel(501, 999, degenerate=False)]
    p_far = FAR // 2 + 64  # samples: byte offset 2^32 + 128
    pcm = torch.empty(p_far + 4 * n + 4096, dtype=torch.int16, device="cuda")
    out = torch.empty(FAR + (1 << 20), dtype=torch.uint8, device="cuda")
    try:
        rng = np.random.default_rng(80)
        for o, ch in ((p_far, x[0]), (0, x[1])):
            pcm[o - 64 if o else 0: o + len(ch) + 64] = _cuda(rng.integers(-32768, 32768, len(ch) + (128 if o else 64), dtype=np.int16))
            pcm[o: o + len(ch)] = _cuda(ch)
        lens = np.array([n, 999], np.int32)
        p_off = np.array([p_far, 0], np.int64)

        def window(o, size):
            lo = max(o - 4096, 0)
            return lo, _arr(out[lo: o + size + 4096])

        # GC-ADPCM encode, then decode from there into a far PCM region
        a_far = FAR + 4096
        a_off = np.array([a_far, 0], np.int64)
        co = np.stack([oracle.calculate_coefficients(c) for c in x])
        want = [oracle.encode(c, co[i]) for i, c in enumerate(x)]
        out[a_far - 4096: a_far + want[0].size + 4096].fill_(SENT8)
        out[: 8192].fill_(SENT8)
        coefs = torch.full((48,), SENT16, dtype=torch.int16, device="cuda")
        ws = torch.zeros(L.vgb_gcadpcm_workspace_bytes(sum(-(-int(k) // 14) for k in lens), 2), dtype=torch.uint8, device="cuda")
        assert L.vgb_gcadpcm_encode_dev(pcm.data_ptr(), p_off.ctypes.data, lens.ctypes.data, None, 2, None, coefs.data_ptr(),
                                        out.data_ptr(), a_off.ctypes.data, ws.data_ptr(), ws.numel(), 0) == 0, L.vgb_last_error()
        _check_regions(_arr(coefs), [0], [co.ravel()], SENT16, "far gc coefficients")
        lo, got = window(a_far, want[0].size)
        _check_regions(got, [a_far - lo], [want[0]], SENT8, "far gc adpcm")
        _check_regions(_arr(out[:8192]), [0], [want[1]], SENT8, "near gc adpcm")
        d_far = p_far + 2 * n + 1024
        pcm[d_far - 256: d_far + n + 256].fill_(SENT16)
        dp = (N.VgbGcParams * 2)(N.VgbGcParams(n, 0, 0), N.VgbGcParams(999, 0, 0))
        d_off = np.array([d_far, p_far + n + 64 + 7], np.int64) // 8 * 8
        pcm[int(d_off[1]) - 64: int(d_off[1]) + 999 + 64].fill_(SENT16)
        assert L.vgb_gcadpcm_decode_dev(out.data_ptr(), a_off.ctypes.data, coefs.data_ptr(), dp, 2, pcm.data_ptr(), d_off.ctypes.data,
                                        ws.data_ptr(), ws.numel(), 0) == 0, L.vgb_last_error()
        assert L.vgb_gcadpcm_decode_dev_status(ws.data_ptr(), 2, 0) == 0
        for i, (o, k) in enumerate(zip(d_off, (n, 999))):
            o = int(o)
            got = _arr(pcm[o - 64: o + k + 64])
            _check_regions(got, [64], [oracle.decode(want[i], co[i], k)], SENT16, f"far gc decode {i}")
        # ADX encode from the far PCM into a far, odd-by-2 byte offset
        ap = (N.VgbAdxParams * 2)(*[N.VgbAdxParams(48000, 500, 18, 4, 0, 0, 3, 0)] * 2)
        x_far = FAR + (1 << 16) + 6
        ax_off = np.array([x_far, 4096], np.int64)
        wants = [oracle.adx_encode(c, 48000, 18, 4, 0, 3, 0)[0] for c in x]
        out[x_far - 4096: x_far + wants[0].size + 4096].fill_(SENT8)
        out[: 8192].fill_(SENT8)
        aws = torch.zeros(L.vgb_adx_workspace_bytes(int(lens.sum()), 2), dtype=torch.uint8, device="cuda")
        assert L.vgb_adx_encode_dev(pcm.data_ptr(), p_off.ctypes.data, lens.ctypes.data, ap, 2, None, out.data_ptr(), ax_off.ctypes.data,
                                    aws.data_ptr(), aws.numel(), 0) == 0, L.vgb_last_error()
        lo, got = window(x_far, wants[0].size)
        _check_regions(got, [x_far - lo], [wants[0]], SENT8, "far adx")
        _check_regions(_arr(out[:8192]), [4096], [wants[1]], SENT8, "near adx")
        # HCA encode (mono streams) from the far PCM into a far, odd byte offset
        hp = (N.VgbHcaParams * 2)(N.VgbHcaParams(2, 0, 0, 1, 48000, n, 0, 0, 0), N.VgbHcaParams(2, 0, 0, 1, 48000, 999, 0, 0, 0))
        h_far = FAR + (1 << 17) + 3
        h_off = np.array([h_far, 1], np.int64)
        stride = np.array([n, 999], np.int64)
        hw = [oracle.hca_encode([c], 48000, 2)[1].ravel() for c in x]
        out[h_far - 4096: h_far + hw[0].size + 4096].fill_(SENT8)
        out[: 8192].fill_(SENT8)
        hws = torch.zeros(L.vgb_hca_workspace_bytes(2), dtype=torch.uint8, device="cuda")
        assert L.vgb_hca_encode_dev(pcm.data_ptr(), p_off.ctypes.data, stride.ctypes.data, hp, 2, None, out.data_ptr(), h_off.ctypes.data,
                                    hws.data_ptr(), hws.numel(), 0) == 0, L.vgb_last_error()
        assert L.vgb_hca_encode_dev_status(hws.data_ptr(), 2, 0) == 0, L.vgb_last_error()
        lo, got = window(h_far, hw[0].size)
        _check_regions(got, [h_far - lo], [hw[0]], SENT8, "far hca")
        _check_regions(_arr(out[:8192]), [1], [hw[1]], SENT8, "near hca")
    finally:
        del pcm, out
        torch.cuda.empty_cache()


# ---- (de)interleave ---------------------------------------------------------------------------------------------------
def vector_width(values) -> int:
    """interleave.cu's vector_width: the widest of 16, 8, 4, 2, 1 bytes that divides every value."""
    w = 16
    for v in values:
        while w > 1 and v % w:
            w >>= 1
    return w


def _shape(count, in_size, ilv, out_size):
    in_blocks, out_blocks = -(-in_size // ilv), -(-out_size // ilv)
    return in_size - (in_blocks - 1) * ilv, out_size - (out_blocks - 1) * ilv


# (n_items, count, in_size, interleave, out_size, channel stride pad, item stride pad, in base, out base, width)
ILV_CASES = [
    (3, 2, 4096, 512, -1, 16, 48, 0, 0, 16),
    (5, 3, 1000, 200, 1000, 8, 24, 8, 0, 8),
    (2, 4, 900, 100, 1100, 4, 4, 0, 4, 4),
    (4, 2, 318, 18, 250, 2, 6, 2, 0, 2),
    (1, 5, 777, 64, 777, 3, 1, 1, 0, 1),
    (3, 3, 333, 1000, 400, 5, 9, 0, 0, 1),    # interleave larger than the size
    (2, 2, 512, 64, 0, 16, 16, 0, 0, 16),     # nothing to write
    (4, 6, 4800, 2048, 4096, 32, 16, 16, 32, 16),
    (2, 8, 64, 16, 128, 0, 16, 0, 0, 16),
    (4, 3, 8192, 4096, 8192, 48, 32, 16, 64, 16),   # equal sizes at width 16: the bulk-copy kernel under VGB_INTERLEAVE_TMA=1
    (2, 4, 4000, 1024, 4000, 16, 16, 0, 0, 16),     # ... with a short last block
]


def _ilv_layout(case, de: bool):
    n_items, count, in_size, ilv, out_size, cpad, ipad, b_in, b_out, _ = case
    out_eff = in_size if out_size == -1 else out_size
    if not de:
        ch_stride = in_size + cpad
        in_item = count * ch_stride + ipad
        out_item = out_eff * count + ipad
        return ch_stride, in_item, out_item, out_eff
    in_item = in_size * count + ipad
    ch_stride = out_eff + cpad
    out_item = count * ch_stride + ipad
    return ch_stride, in_item, out_item, out_eff


@pytest.mark.gpu
@pytest.mark.parametrize("tma", [False, True])
@pytest.mark.parametrize("de", [False, True])
@pytest.mark.parametrize("case", ILV_CASES, ids=[f"w{c[-1]}_{i}" for i, c in enumerate(ILV_CASES)])
def test_interleave_dev_items_and_strides(vg, oracle, monkeypatch, case, de, tma):
    """n_items payloads at item strides above the payload and channel strides above the size, against the oracle item by
    item, with the vector width each shape selects asserted and the sentinel between items intact."""
    torch = _torch()
    if tma:
        monkeypatch.setenv("VGB_INTERLEAVE_TMA", "1")
    n_items, count, in_size, ilv, out_size, cpad, ipad, b_in, b_out, want_w = case
    ch_stride, in_item, out_item, out_eff = _ilv_layout(case, de)
    rng = np.random.default_rng(hash(case) & 0xFFFF)
    in_len = b_in + n_items * in_item + 64
    out_len = b_out + n_items * out_item + 64
    host = rng.integers(0, 256, in_len, dtype=np.uint8)
    d_in = _cuda(host)
    d_out = torch.full((out_len,), SENT8, dtype=torch.uint8, device="cuda")
    last_in, last_out = _shape(count, in_size, ilv, out_eff) if out_eff else (0, 0)
    w = vector_width([ilv, in_size, out_eff, last_in, last_out, ch_stride, in_item, out_item, d_in.data_ptr() + b_in, d_out.data_ptr() + b_out])
    assert w == want_w
    L = vg.lib
    if not de:
        rc = L.vgb_interleave_dev(d_in.data_ptr() + b_in, ch_stride, in_item, d_out.data_ptr() + b_out, out_item, n_items, count, in_size, ilv,
                                  out_size, 0)
    else:
        rc = L.vgb_deinterleave_dev(d_in.data_ptr() + b_in, in_item, d_out.data_ptr() + b_out, ch_stride, out_item, n_items, count, in_size,
                                    ilv, out_size, 0)
    assert rc == 0, L.vgb_last_error()
    got = _arr(d_out)
    offs, wants = [], []
    for i in range(n_items):
        if not de:
            chans = [host[b_in + i * in_item + c * ch_stride: b_in + i * in_item + c * ch_stride + in_size] for c in range(count)]
            offs.append(b_out + i * out_item)
            wants.append(oracle.interleave(chans, ilv, out_size) if out_eff else np.zeros(0, np.uint8))
        else:
            data = host[b_in + i * in_item: b_in + i * in_item + in_size * count]
            outs = oracle.deinterleave(data, ilv, count, out_size) if out_eff else [np.zeros(0, np.uint8)] * count
            for c in range(count):
                offs.append(b_out + i * out_item + c * ch_stride)
                wants.append(outs[c])
    _check_regions(got, offs, wants, SENT8, f"{'de' if de else ''}interleave")
