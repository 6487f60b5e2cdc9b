"""Deterministic stimuli for the rare paths of the CRI HCA encoder and decoder.

Encoder: each builder is named after the EncodeFrame path it reaches; tests/test_oracle_hca_trace.py proves with the
oracle's frame trace (vgo_hca_encode_trace) that the set reaches every one of them, tests/test_crihca_paths_gpu.py
encodes the same set on the GPU.  All streams of one EncStim share the configuration, so they go through one batch call
with ragged lengths.

Decoder: frames the encoder never writes, built field by field with an MSB-first bit writer.  They are valid in the
sense of the reference's happy path (sync word, every scale-factor delta in range, intensity indices 0..14) unless a
fault is injected on purpose."""
from __future__ import annotations

import copy
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np

from oracle import pyoracle as O
from vgaudio_b200 import synth


@dataclass
class EncStim:
    name: str
    rate: int
    quality: int
    bitrate: int
    streams: List[List[np.ndarray]]   # [stream][channel] int16
    fails: bool = False               # the oracle stops with "Bitrate is set too low."


def _pair(first: int, n: int, rate: int = 48000):
    return [synth.channel(first, n, rate, degenerate=False), synth.channel(first + 1, n, rate, degenerate=False)]


def _square(n: int, k: int, phase: float = 0.0) -> np.ndarray:
    """Full-scale square wave at the centre frequency of MDCT bin k: coefficients above sqrt(128), so scale factor 63
    and coefficients clamped to +-0.999999999999."""
    t = np.arange(n)
    return np.where(np.cos(2 * np.pi * ((k + 0.5) / 256 * t + phase)) >= 0, 32767, -32768).astype(np.int16)


def _neg(x: np.ndarray) -> np.ndarray:
    return np.clip(-x.astype(np.int32), -32768, 32767).astype(np.int16)


def band_dropping() -> List[EncStim]:
    """No noise level fits the frame: `highest -= 2` rounds zero the top scale factors (CriHcaEncoder.cs:457-485)."""
    return [EncStim(f"band_dropping_{br}", 48000, 2, br, [_pair(10, 30000), _pair(12, 9000)]) for br in (20000, 30000)]


def hfr_groups_without_source_bands() -> List[EncStim]:
    """hfr_band_count > total_band_count - hfr_band_count: the last HFR groups average no band (0 / 0).  Frames of 22,
    28 and 33 bytes also fold the CRC over messages shorter than 32 bytes and not a multiple of 4."""
    return [EncStim(f"hfr_empty_groups_{br}", 48000, 2, br, [[synth.channel(20, 20000, degenerate=False)],
                                                              [synth.channel(21, 3000, degenerate=False)]])
            for br in (8500, 10500, 12500)]


def bitrate_too_low() -> EncStim:
    """Band dropping runs out of bands: "Bitrate is set too low." from inside the frame loop."""
    return EncStim("bitrate_too_low_6500", 48000, 2, 6500, [[synth.channel(22, 6000, degenerate=False)]], fails=True)


def intensity_pairs() -> List[EncStim]:
    n = 12000
    x = synth.channel(30, n, degenerate=False)
    low = (synth.reference_sine(n, 180, 48000) // 2).astype(np.int16)
    low2 = (synth.reference_sine(n, 310, 48000) // 3).astype(np.int16)
    return [
        EncStim("anti_phase_et_zero", 48000, 5, 0, [[x, _neg(x)], [low, _neg(low)]]),  # et == 0: ratio +inf, clamped
        EncStim("pair_equal", 48000, 5, 0, [[x, x.copy()]]),
        EncStim("pair_one_silent", 48000, 5, 0, [[x, np.zeros(n, np.int16)], [np.zeros(n, np.int16), x]]),
        EncStim("pair_high_bands_silent", 48000, 5, 0, [[low, low2]]),                # el == er == 0: index 0
    ]


def raw_scale_factors() -> List[EncStim]:
    """delta_bits == 6 (raw scale factors): found by a search of low custom bitrates with the frame trace; stereo at
    48 kHz and 16 000 bit/s after band dropping."""
    n = 16000
    return [EncStim("raw_scale_factors", 48000, 0, 16000,
                    [[synth.channel(seed * 8 + c, n, 48000, degenerate=False) for c in range(2)] for seed in (1, 3)])]


def delta_bits_5() -> List[EncStim]:
    n = 16000
    return [EncStim("delta_bits_5", 16000, 0, 10000,
                    [[synth.channel(32 + c, n, 16000, degenerate=False) for c in range(2)]])]


def clamped_coefficients() -> List[EncStim]:
    return [EncStim("clamped_full_scale_square", 48000, 1, 0, [[_square(8192, 40)], [_square(5000, 40, 0.25)]])]


def sample_rate_sweep() -> List[EncStim]:
    """Every quality at the rates the other tests never use, mono and stereo, plus 8 channels at 32 kHz / Highest: the
    4096-byte frame (frame size is 2048 * channels / ratio at every rate; at 96 kHz that configuration's bitrate * 1024
    leaves int32 and the reference fails, which vgb_hca_query reports)."""
    out = []
    for rate in (8000, 11025, 16000, 22050, 32000, 96000):
        for nch in (1, 2):
            for q in range(1, 6):
                n = 2500 + 700 * q
                out.append(EncStim(f"sweep_{rate}_{nch}ch_q{q}", rate, q, 0,
                                   [[synth.channel(40 + 3 * q + c, n, rate, degenerate=False) for c in range(nch)],
                                    [synth.channel(50 + c, 1100, rate, degenerate=False) for c in range(nch)]]))
    out.append(EncStim("sweep_32000_8ch_q1", 32000, 1, 0, [[synth.channel(60 + c, 3000, 32000, degenerate=False) for c in range(8)]]))
    return out


def encoder_stimuli() -> List[EncStim]:
    return (band_dropping() + hfr_groups_without_source_bands() + [bitrate_too_low()] + intensity_pairs()
            + raw_scale_factors() + delta_bits_5() + clamped_coefficients() + sample_rate_sweep())


# ---- decoder: structured frames ---------------------------------------------------------------------------------------

class BitWriter:
    """MSB-first, like the reference's BitWriter (Utilities/BitWriter.cs:26-98); bits past the end are dropped."""

    def __init__(self, size: int):
        self.buf = np.zeros(size, dtype=np.uint8)
        self.pos = 0

    def write(self, value: int, count: int):
        for i in range(count - 1, -1, -1):
            if (value >> i) & 1 and self.pos < self.buf.size * 8:
                self.buf[self.pos >> 3] |= 0x80 >> (self.pos & 7)
            self.pos += 1


def channel_types(info) -> List[int]:
    """CriHcaFrame.GetChannelTypes (CriHcaFrame.cs:34-52): 0 discrete, 1 stereo primary, 2 stereo secondary."""
    table = {2: [1, 2], 3: [1, 2, 0], 5: [1, 2, 0, 0, 0] if info.channel_config > 2 else [1, 2, 0, 1, 2],
             6: [1, 2, 0, 0, 1, 2], 7: [1, 2, 0, 0, 1, 2, 0], 8: [1, 2, 0, 0, 1, 2, 1, 2],
             4: [1, 2, 0, 0] if info.channel_config != 0 else [1, 2, 1, 2]}
    nch = info.channel_count
    if info.stereo_band_count == 0 or nch == 1:
        return [0] * nch
    return table[nch]


def coded_count(info, t: int) -> int:
    return info.base_band_count if t == 2 else info.base_band_count + info.stereo_band_count


def scale_chain(rng, n: int, delta_bits: int, style: int) -> List[int]:
    """n scale factors 0..63 whose chain holds in-range deltas, escapes and the values 0 and 63."""
    if n == 0:
        return []
    if style == 0:      # random walk: small deltas, clipped at both ends
        v = [int(rng.integers(0, 64))]
        for _ in range(n - 1):
            v.append(int(np.clip(v[-1] + rng.integers(-3, 4), 0, 63)))
    elif style == 1:    # jumps between the extremes: escapes in every delta width
        v = [int(rng.choice([0, 63, int(rng.integers(0, 64))])) for _ in range(n)]
    elif style == 2:    # the HFR conversion index's top end: low bands at 0 and 1 (index 127, 126 with HFR scale 63)
        v = [int(rng.choice([0, 1])) for _ in range(n)]
    else:               # its bottom end: low bands at 63 (index 1 with HFR scale 0)
        v = [63 if rng.random() < 0.8 else 62 for _ in range(n)]
    return v


def write_scale_factors(w: BitWriter, delta_bits: int, sfs: List[int], count: int):
    """WriteScaleFactors (CriHcaPacking.cs:262-295), with what DeltaDecode reads for a channel without coded bands."""
    w.write(delta_bits, 3)
    if delta_bits == 0:
        return
    if delta_bits >= 6:
        for v in sfs:
            w.write(v, 6)
        return
    w.write(sfs[0] if count else 0, 6)   # DeltaDecode reads output[0] even when count == 0 (:183-186)
    max_delta = (1 << (delta_bits - 1)) - 1
    for i in range(1, count):
        d = sfs[i] - sfs[i - 1]
        if abs(d) > max_delta:
            w.write((1 << delta_bits) - 1, delta_bits)
            w.write(sfs[i], 6)
        else:
            w.write(max_delta + d, delta_bits)


@dataclass
class Fault:
    frame: int
    channel: int
    kind: str          # "intensity15" or "bad_delta"
    subframe: int = 0


def build_frames(info, rng, n_frames: Optional[int] = None, fault: Optional[Fault] = None) -> np.ndarray:
    """Frames [frame_count, frame_size] for `info`, every field drawn over its full range."""
    types = channel_types(info)
    n_frames = info.frame_count if n_frames is None else n_frames
    frames = np.zeros((n_frames, info.frame_size), dtype=np.uint8)
    for k in range(n_frames):
        w = BitWriter(info.frame_size)
        w.write(0xFFFF, 16)
        style = int(rng.integers(0, 4))
        noise = int(rng.choice([0, 1, int(rng.integers(0, 512)), 511])) if k % 3 else int(rng.integers(0, 40))
        w.write(noise, 9)
        w.write(int(rng.integers(0, 128)), 7)
        for c, t in enumerate(types):
            n = coded_count(info, t)
            db = int(rng.integers(0, 8)) if k % 4 else (k // 4 + c) % 8
            if db == 0 and n and style == 2 and info.hfr_group_count:
                db = 6   # HFR index tests need the low bands' scale factors
            sfs = scale_chain(rng, n, db, style)
            if fault and fault.kind == "bad_delta" and fault.frame == k and fault.channel == c:
                db = max(2, min(db, 5)) if n >= 2 else 2
                sfs = [63] * n
                w.write(db, 3)
                w.write(63, 6)
                w.write((1 << (db - 1)), db)   # delta +1 above 63: DeltaDecode returns false
                for _ in range(2, n):
                    w.write((1 << (db - 1)) - 1, db)
            else:
                write_scale_factors(w, db, sfs, n)
            if t == 2:
                for sf in range(8):
                    v = int(rng.integers(0, 15))
                    if fault and fault.kind == "intensity15" and fault.frame == k and fault.channel == c and fault.subframe == sf:
                        v = 15
                    w.write(v, 4)
            elif info.hfr_group_count > 0:
                for _ in range(info.hfr_group_count):
                    w.write(63 if style == 2 else 0 if style == 3 else int(rng.integers(0, 64)), 6)
        # spectral codes: random bits up to the frame end; codes that run past it read zeros
        tail = info.frame_size * 8 - w.pos - (16 if k % 2 else 0)
        for _ in range(max(tail, 0) // 16):
            w.write(int(rng.integers(0, 1 << 16)), 16)
        frames[k] = w.buf
    return frames


def decoder_layouts() -> List[Tuple[str, object]]:
    """Infos the encoder's Initialize gives (vgb_hca_query computes the same) for 1..8 channels with intensity stereo
    and HFR on and off, plus hand-edited ones."""
    out = []
    for nch in range(1, 9):
        for q, rate in ((5, 48000), (1, 48000), (3, 22050)):
            info = O.hca_init(O.HcaParams(q, 0, 0, nch, rate, 4000, 0, 0, 0))
            out.append((f"{nch}ch_q{q}_{rate}", info))
    # a secondary channel without coded bands: base_band_count == 0, stereo_band_count > 0
    info = O.hca_init(O.HcaParams(5, 0, 0, 2, 48000, 4000, 0, 0, 0))
    edited = copy.copy(info)
    edited.base_band_count, edited.stereo_band_count = 0, 64
    out.append(("2ch_base0", edited))
    info6 = O.hca_init(O.HcaParams(5, 0, 0, 6, 48000, 4000, 0, 0, 0))
    edited6 = copy.copy(info6)
    edited6.base_band_count, edited6.stereo_band_count = 0, 64
    out.append(("6ch_base0", edited6))
    return out


@dataclass
class DecStim:
    name: str
    info: object
    streams: List[np.ndarray] = field(default_factory=list)   # frames [frame_count, frame_size] per stream


def decoder_stimuli(n_streams: int = 3) -> List[DecStim]:
    out = []
    for i, (name, info) in enumerate(decoder_layouts()):
        rng = np.random.default_rng(1000 + i)
        out.append(DecStim(name, info, [build_frames(info, rng) for _ in range(n_streams)]))
    return out


def fault_cases() -> List[Tuple[str, object, int, Fault]]:
    """(name, info, stream index, fault): intensity 15 in every secondary channel of 2-, 4-, 6- and 8-channel layouts, and
    a scale-factor delta out of range."""
    out = []
    for nch in (2, 4, 6, 8):
        info = O.hca_init(O.HcaParams(5, 0, 0, nch, 48000, 4000, 0, 0, 0))
        for c, t in enumerate(channel_types(info)):
            if t == 2:
                out.append((f"intensity15_{nch}ch_c{c}", info, c % 3, Fault(frame=(c + 1) % info.frame_count, channel=c,
                                                                             kind="intensity15", subframe=c % 8)))
    info = O.hca_init(O.HcaParams(2, 0, 0, 1, 48000, 4000, 0, 0, 0))
    out.append(("bad_delta_1ch", info, 1, Fault(frame=2, channel=0, kind="bad_delta")))
    info = O.hca_init(O.HcaParams(5, 0, 0, 4, 48000, 4000, 0, 0, 0))
    out.append(("bad_delta_4ch", info, 2, Fault(frame=1, channel=3, kind="bad_delta")))
    return out


def fault_streams(info, bad_stream: int, fault: Fault, seed: int, n_streams: int = 3) -> List[np.ndarray]:
    rng = np.random.default_rng(seed)
    return [build_frames(info, rng, fault=fault if s == bad_stream else None) for s in range(n_streams)]
