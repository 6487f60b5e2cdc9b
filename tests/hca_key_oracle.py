"""ctypes bindings of oracle/hcakeys.c, the C restatement of HcaReader.FindKey for type-56 .hca files - TEST
INFRASTRUCTURE: FindFirstNonEmptyFrame's window, TestKey's outcome per key (with each unpacked frame's Remaining) and
FindKey's first index, in oracle/libvgoracle.so.  Also the keyed images the key-search tests share."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import pyoracle

import hca_reader_oracle as R

FRAMES_TO_TEST = 10
NO_REMAINING = -(1 << 31)  # a window frame that did not reach UnpackingWasSuccessful


def lib() -> C.CDLL:
    return pyoracle.lib()


def split(image):
    """(HcaInfo, ciph, frames [frame_count, frame_size]) of an .hca image as HcaReader reads it."""
    st, info, ciph = R.hca_parse(np.asarray(image, dtype=np.uint8))
    assert st == 0, st
    img = np.asarray(image, dtype=np.uint8)
    frames = np.ascontiguousarray(img[info.header_size: info.header_size + info.frame_count * info.frame_size])
    return info, ciph, frames.reshape(info.frame_count, info.frame_size)


def window(frames: np.ndarray):
    """FindFirstNonEmptyFrame over the encrypted frames and TestKey's end: (start, end)."""
    L = lib()
    f = np.ascontiguousarray(frames, dtype=np.uint8)
    s, e = C.c_int(0), C.c_int(0)
    L.vgo_hca_key_window.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.vgo_hca_key_window.restype = None
    L.vgo_hca_key_window(f.ctypes.data, f.shape[0], f.shape[1] if f.ndim == 2 else 0, C.byref(s), C.byref(e))
    return s.value, e.value


def outcomes(info, frames: np.ndarray, keys, no_crc: bool = False):
    """TestKey per key: (outcome [n_keys], remaining [n_keys, 10]); outcome 0 pass, else 1 + 3 * j + r (r 0 bad sync, 1
    delta out of range, 2 UnpackingWasSuccessful false); remaining NO_REMAINING where a frame did not get that far.
    no_crc leaves the frame's last two bytes raw instead of CryptFrame's CRC."""
    L = lib()
    f = np.ascontiguousarray(frames, dtype=np.uint8)
    codes = np.ascontiguousarray([int(k) & 0xFFFFFFFFFFFFFFFF for k in keys], dtype=np.uint64)
    out = np.zeros(len(codes), dtype=np.int32)
    rem = np.full((len(codes), FRAMES_TO_TEST), NO_REMAINING, dtype=np.int32)
    L.vgo_hca_key_outcomes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.vgo_hca_key_outcomes.restype = None
    L.vgo_hca_key_outcomes(C.byref(info), f.ctypes.data, codes.ctypes.data, len(codes), int(no_crc), out.ctypes.data, rem.ctypes.data)
    return out, rem


def find_key(info, frames: np.ndarray, keys):
    """FindKey: (index or -1, status 0 found / 1 bad sync thrown / 2 no key)."""
    L = lib()
    f = np.ascontiguousarray(frames, dtype=np.uint8)
    codes = np.ascontiguousarray([int(k) & 0xFFFFFFFFFFFFFFFF for k in keys], dtype=np.uint64)
    st = C.c_int(0)
    L.vgo_hca_find_key.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    L.vgo_hca_find_key.restype = C.c_int
    idx = L.vgo_hca_find_key(C.byref(info), f.ctypes.data, codes.ctypes.data, len(codes), C.byref(st))
    return idx, st.value


def image_outcomes(image, keys):
    """outcomes() of an .hca image, or all -1 when it is not type 56."""
    info, ciph, frames = split(image)
    if ciph != 56:
        return np.full(len(keys), -1, dtype=np.int32)
    return outcomes(info, frames, keys)[0]


def image_find_key(image, keys):
    """find_key() of an .hca image as vgb_hca_find_keys reports it: (index, status) with status VGB_OK 0, VGB_E_DATA -2,
    VGB_HCA_KEY_SKIPPED 1, VGB_HCA_KEY_NOT_FOUND 2."""
    info, ciph, frames = split(image)
    if ciph != 56:
        return -1, 1
    idx, st = find_key(info, frames, keys)
    return idx, {0: 0, 1: -2, 2: 2}[st]


def keyed(oracle, info, frames, key_code):
    """The .hca image HcaWriter writes with a type-56 key."""
    return oracle.hca_write(info, frames, oracle.hca_key_tables(56, key_code)[1], 56)


def equivalent(code: int) -> int:
    """Another code with the same key: CriHcaKey(ulong) reads bytes 0..6 of code - 1, and this changes only byte 7 of
    code - 1."""
    k = (code - 1) & 0xFFFFFFFFFFFFFFFF
    return ((k ^ (0x5A << 56)) + 1) & 0xFFFFFFFFFFFFFFFF


KEY = 0x00D7E1B6C2A94F03
KEY2 = 0x0000000000001234


def _pcm(channels, n, rate, seed, lead=0):
    from vgaudio_b200 import synth

    out = []
    for c in range(channels):
        x = synth.channel(seed + c, n, rate, degenerate=False).copy()
        x[:lead] = 0
        out.append(x)
    return out


def _empty_frames(info, n):
    """n frames of the sync word followed by zero bytes: empty in FindFirstNonEmptyFrame's sense, and still so after
    HcaWriter's encryption (type-56 tables keep 0x00), apart from the CRC in the last two bytes."""
    f = np.zeros((n, info.frame_size), dtype=np.uint8)
    f[:, :2] = 0xFF
    return f


def key_files(oracle):
    """[(name, image)]: type-56 images under KEY of 1..8 channels (intensity stereo and HFR layouts, structured random
    frames), several qualities and frame sizes, silent lead-ins, files shorter than the window, a window that ends at
    the end of the file, a bad sync word inside the window, an all-empty file, a file with zero frames, frames whose
    outcome the CRC splice decides, a second key and a plain file."""
    import copy

    import hca_stimuli as H

    out = []
    for ch, q, rate, n in ((1, 1, 48000, 30000), (2, 3, 44100, 25000), (4, 5, 32000, 15000), (6, 2, 48000, 12000),
                           (8, 4, 22050, 9000), (2, 5, 48000, 3000)):
        info, frames = oracle.hca_encode(_pcm(ch, n, rate, 10 * ch + q), rate, q)
        out.append((f"enc_{ch}ch_q{q}_{rate}", keyed(oracle, info, frames, KEY)))
    for i, (name, info) in enumerate(H.decoder_layouts()):
        frames = H.build_frames(info, np.random.default_rng(700 + i))
        out.append((f"layout_{name}", keyed(oracle, info, frames, KEY)))
    # silent lead-in: three empty frames, then the encoder's frames; the window starts at frame 3
    info, frames = oracle.hca_encode(_pcm(2, 20000, 48000, 5), 48000, 2)
    frames = frames.copy()
    frames[:3] = _empty_frames(info, 3)
    out.append(("lead_in_3", keyed(oracle, info, frames, KEY)))
    # a window that ends at the end of the file: 12 frames, 5 of them empty lead-in
    info, frames = oracle.hca_encode(_pcm(1, 12 * 1024 - 2000, 48000, 6), 48000, 3)
    frames = frames.copy()
    frames[:5] = _empty_frames(info, 5)
    out.append(("window_to_end", keyed(oracle, info, frames, KEY)))
    # a bad sync word at window frame 4 (raw, after encryption)
    info, frames = oracle.hca_encode(_pcm(2, 30000, 48000, 7), 48000, 2)
    img = keyed(oracle, info, frames, KEY)
    img[info.header_size + 4 * info.frame_size] = 0x7F
    out.append(("bad_sync_4", img))
    # every frame empty: startFrame 0, every key passes through FrameEmpty
    info, frames = oracle.hca_encode(_pcm(2, 8000, 48000, 8), 48000, 2)
    out.append(("all_empty", keyed(oracle, info, _empty_frames(info, info.frame_count), KEY)))
    # zero frames: an empty window
    info0 = copy.copy(info)
    info0.frame_count = 0
    out.append(("no_frames", keyed(oracle, info0, np.zeros((0, info.frame_size), np.uint8), KEY)))
    # CryptFrame's CRC decides the outcome: a 37-byte mono frame whose scale-factor delta chain (2-bit deltas of 0 from
    # scale factor 0) runs on into the last two bytes, where a delta of -1 ends it out of range; with noise levels 4 and 5
    # the outcome differs between the CRC and the raw bytes
    info = oracle.hca_init(oracle.HcaParams(1, 0, 0, 1, 48000, 4000, 0, 0, 0))
    coded = info.base_band_count + info.stereo_band_count
    for noise in (4, 5):
        ic = copy.copy(info)
        ic.frame_size, ic.frame_count = (41 + 2 * (coded - 1)) // 8 + 1, 1
        w = H.BitWriter(ic.frame_size)
        for value, count in ((0xFFFF, 16), (noise, 9), (0, 7), (2, 3), (0, 6)):
            w.write(value, count)
        while w.pos < ic.frame_size * 8 - 16:
            w.write(1, 2)
        out.append((f"crc_tail_noise{noise}", keyed(oracle, ic, w.buf.reshape(1, -1), KEY)))
    # noise level 0 with coded scale factors that are all 0: no spectral bits, far more than 128 bits left, a pass
    info = oracle.hca_init(oracle.HcaParams(5, 0, 0, 1, 48000, 4000, 0, 0, 0))
    coded = info.base_band_count + info.stereo_band_count
    frames = np.zeros((12, info.frame_size), dtype=np.uint8)
    for k in range(12):
        w = H.BitWriter(info.frame_size)
        for value, count in [(0xFFFF, 16), (0, 9), (k, 7), (6, 3)] + [(0, 6)] * coded:
            w.write(value, count)
        frames[k] = w.buf
    out.append(("noise0_long", keyed(oracle, info, frames, KEY)))
    # a second key, and a plain file
    info, frames = oracle.hca_encode(_pcm(1, 15000, 44100, 9), 44100, 2)
    out.append(("key2", keyed(oracle, info, frames, KEY2)))
    out.append(("plain", oracle.hca_write(info, frames)))
    return out


def key_list(n: int, seed: int, planted=(KEY,), at: str = "end"):
    """n codes: random decoys with codes equivalent to the first planted key (and its neighbours, which are different
    keys) before the planted keys, which sit at the start, the middle or the end."""
    rng = np.random.default_rng(seed)
    decoys = [int(v) for v in rng.integers(1, 1 << 63, size=n, dtype=np.int64)]
    decoys[1] = planted[0] + 1
    decoys[2] = planted[0] - 1
    lead = [equivalent(planted[0])]
    body = decoys[:n - len(planted) - len(lead)]
    if at == "start":
        return list(planted) + lead + body
    if at == "middle":
        h = len(body) // 2
        return body[:h] + lead + list(planted) + body[h:]
    return body + lead + list(planted)
