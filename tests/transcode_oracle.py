"""The oracle chain of a transcode (Convert.ConvertFile with a coded source): the source's reader restatement and the
oracle's decoder give what ToPcm16 yields (channels, sample count, loop points, rate), then the oracle's encoder and
writer of the target, configured from the options alone, give the file.  Also builders of .dsp / .hca source images on
the oracle (.adx images come from adx_files)."""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np

import adx_files as F
import adx_reader_oracle as RA
import hca_reader_oracle as RH
from oracle import pyoracle as O
from vgaudio_b200 import synth

DSP, ADX, HCA = 1, 2, 3
HCA_KEY = 0x00D7E1B6C2A94F03


# ---- sources ------------------------------------------------------------------------------------------------------------
def dsp_file(ch, n, rate, loop=None, seed=0, pcm=None):
    """A .dsp image the way the reference's encoder and DspWriter make it, with a start history in the header."""
    if pcm is None:
        pcm = [synth.channel(seed + c, max(n, 1), rate, degenerate=False)[:n] for c in range(ch)]
    coefs = np.stack([O.calculate_coefficients(p) for p in pcm])
    adpcm = [O.encode(p, c) for p, c in zip(pcm, coefs)]
    ctx = None
    if loop:
        ctx = np.stack([np.array(O.gc_loop_context(a, O.decode(a, c, n), loop[0]), dtype=np.int16) for a, c in zip(adpcm, coefs)])
    hist = np.array([[3 * c + seed % 7, -c] for c in range(ch)], dtype=np.int16)
    return O.dsp_write(adpcm, coefs, rate, n, loop, ctx, None, hist)


def hca_file(ch, rate, n, seed, quality=2, loop=None, key_type=-1, ath=False):
    pcm = [synth.channel(seed + c, n, rate, degenerate=False) for c in range(ch)]
    info, frames = O.hca_encode(pcm, rate, quality, loop=loop, ath=ath)
    enc = O.hca_key_tables(key_type, HCA_KEY)[1] if key_type >= 0 else None
    img = O.hca_write(info, frames, enc, max(key_type, 0))
    if ath:
        img[4:6] = (0x01, 0x00)  # version 1.0 without an "ath" chunk: HcaReader turns UseAthCurve on
    return img


def adx_file(oracle, ch, n, rate=48000, frame_size=18, version=4, type=3, loop=None, key=None, enc_type=0, seed=0):
    return F.encoded(oracle, ch, n, rate, frame_size, version, type, loop, key, enc_type, seed)


# ---- what ToPcm16 yields ------------------------------------------------------------------------------------------------
def source_pcm(img, in_type, adx_key=None, hca_key=None) -> Optional[Tuple[List[np.ndarray], int, Optional[tuple], int]]:
    """(channels, sample_count, loop or None, rate) of one source image, or None where the reader chain fails."""
    if in_type == DSP:
        st, info = O.dsp_parse(img)
        if st != 0:
            return None
        n = info.sample_count
        rows = O.dsp_read_data(img, info)
        pcm = [O.decode(rows[c], np.array(info.coefs[c][:], np.int16), n, info.start_ctx[c][1], info.start_ctx[c][2])
               for c in range(info.channel_count)]
        loop = (info.loop_start, info.loop_end) if info.looping else None
        return pcm, n, loop, info.sample_rate
    if in_type == HCA:
        st, info, ciph = RH.hca_parse(img)
        if st != 0 or (ciph == 56 and hca_key is None):
            return None
        frames = np.ascontiguousarray(img[info.header_size: info.header_size + info.frame_count * info.frame_size])
        if ciph in (1, 56):
            frames = O.hca_crypt_frames(frames, info.frame_size, O.hca_key_tables(ciph, hca_key or 0)[0])
        pcm = O.hca_decode(info, frames.reshape(info.frame_count, info.frame_size))
        loop = None
        if info.looping:
            loop = (info.loop_start_frame * 1024 + info.pre_loop_samples - info.inserted_samples,
                    (info.loop_end_frame + 1) * 1024 - info.post_loop_samples - info.inserted_samples)
        return [np.asarray(p, np.int16) for p in pcm], info.sample_count, loop, info.sample_rate
    # ADX: the reader chain of adx_reader_oracle (its WAVE image decides whether the chain succeeds)
    if RA.expected_wave(img, adx_key) is None:
        return None
    st, h = RA.adx_parse(img)
    rows = RA.audio_rows(img, h)
    if h.revision in (8, 9):
        rows = O.adx_crypt(rows, adx_key, h.revision, h.frame_size)
    n = RA._i32(h.sample_count - h.inserted_samples)
    pcm = [O.adx_decode(r, n, h.sample_rate, h.highpass_frequency, h.frame_size, h.version, 0, h.inserted_samples, h.type) for r in rows]
    loop = (RA._i32(h.loop_start_sample - h.inserted_samples), RA._i32(h.loop_end_sample - h.inserted_samples)) if h.looping else None
    return pcm, n, loop, h.sample_rate


# ---- the target, from a fresh configuration ---------------------------------------------------------------------------
def target_file(pcm, n, loop, rate, out_type, frame_size=18, version=4, type=3, filter=2, enc_type=0, adx_key=None, quality=2,
                hca_key_type=-1, hca_key_code=0) -> np.ndarray:
    ch = len(pcm)
    if out_type == DSP:
        coefs = np.stack([O.calculate_coefficients(p) for p in pcm])
        adpcm = [O.encode(p, c) for p, c in zip(pcm, coefs)]
        ctx = None
        if loop:
            ctx = np.stack([np.array(O.gc_loop_context(a, O.decode(a, c, n), loop[0]), dtype=np.int16) for a, c in zip(adpcm, coefs)])
        return O.dsp_write(adpcm, coefs, rate, n, loop, ctx)
    if out_type == ADX:
        align = F.alignment(loop[0], ch, frame_size) if loop else 0
        enc = [O.adx_encode(p, rate, frame_size, version, align, type, filter) for p in pcm]
        return O.adx_write([e[0] for e in enc], [e[1] for e in enc], rate, n, loop, align, frame_size, version, type, 500, enc_type, adx_key)
    info, frames = O.hca_encode(pcm, rate, quality, loop=loop)
    enc = O.hca_key_tables(hca_key_type, hca_key_code)[1] if hca_key_type >= 0 else None
    return O.hca_write(info, frames, enc, max(hca_key_type, 0))


def target_size(ch, n, loop, rate, out_type) -> int:
    """The size of the target file with the default configuration, from the geometry alone."""
    if out_type == DSP:
        zeros = [np.zeros(O.sample_count_to_byte_count(n), np.uint8) for _ in range(ch)]
        return O.dsp_write(zeros, np.zeros((ch, 16), np.int16), rate, n, loop, np.zeros((ch, 3), np.int16) if loop else None).size
    if out_type == ADX:
        align = F.alignment(loop[0], ch, 18) if loop else 0
        audio = [np.zeros(O.lib().vgo_adx_encoded_byte_count(n, align, 18), np.uint8) for _ in range(ch)]
        return O.adx_write(audio, [0] * ch, rate, n, loop, align).size
    info = O.hca_init(O.hca_params([np.zeros(n, np.int16)] * ch, rate, 2, 0, False, loop))
    return info.header_size + info.frame_size * info.frame_count


def expected(img, in_type, out_type, adx_key=None, hca_key=None, **target) -> Optional[np.ndarray]:
    """The whole chain for one file: the target image, or None where the source's reader fails."""
    src = source_pcm(img, in_type, adx_key, hca_key)
    return None if src is None else target_file(*src, out_type, **target)
