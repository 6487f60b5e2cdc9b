"""The oracle chain of a same-codec rewrite (Convert.ConvertFile with .adx -> .adx or .hca -> .hca): the reader's
restatement decrypts the frames, the writer's restatement writes the source's own format with the output key.

ADX: adx_reader_oracle's parse and de-interleave, oracle.adx_crypt (decrypt) and oracle.adx_write (header, interleave,
encrypt, footer).  HCA: a copy of hca_reader_oracle.hca_parse that also returns the comment bytes (ReadUTF8Z) and the rva
bits, two oracle.hca_crypt_frames passes (decrypt, then encrypt) and a restatement of HcaWriter.WriteHeader with an explicit
"ciph" value, comment bytes, .NET's white-space test and the reference's writing past header_size - 2.  Also builders of
source images with every header feature the rewrite reads."""
from __future__ import annotations

import struct
from typing import List, Optional

import numpy as np

import adx_reader_oracle as RA
from oracle import pyoracle as O

ADX, HCA = 2, 3
HCA_KEY = 0x00D7E1B6C2A94F03
HCA_KEY_OUT = 0x0000A1B2C3D4E5F6
E_TRUNCATED, E_NOT_HCA, E_CHUNK, E_HEADER = -2, -13, -14, -15

# char.IsWhiteSpace (what string.IsNullOrWhiteSpace tests)
NET_SPACE = {*range(0x09, 0x0E), 0x20, 0x85, 0xA0, 0x1680, *range(0x2000, 0x200B), 0x2028, 0x2029, 0x202F, 0x205F, 0x3000}


def _i32(v: int) -> int:
    return (v + (1 << 31)) % (1 << 32) - (1 << 31)


def adx_stream(key, steps: int) -> List[int]:
    """CriAdxEncryption's xor value at steps 0 .. steps - 1 (CriAdxEncryption.cs:18-40)."""
    seed, mult, inc = key
    out, x = [], seed
    for _ in range(steps):
        out.append(x)
        x = (x * mult + inc) & 0x7FFF
    return out


# ---- ADX ----------------------------------------------------------------------------------------------------------------
def adx_source(channels, frames, frame_size=18, version=4, type=3, revision=0, key=None, loop=None, inserted=0, seed=0,
               rate=44100, empty=(), empty_after=(), trim=False, history=None) -> np.ndarray:
    """An .adx image whose frames are random bytes: `frames` frames per channel, written by AdxWriter's restatement
    (sample count frames * spf - inserted unaligned samples, AlignmentSamples = inserted).  Revision 8 / 9 files are
    encrypted with `key`; flat frames (j * channels + c) in `empty` are all zero, those in `empty_after` hold exactly
    the key stream's bytes, so they are empty only once decrypted."""
    rng = np.random.default_rng(seed)
    spf = (frame_size - 2) * 2
    rows = [rng.integers(0, 256, frames * frame_size, dtype=np.uint8) for _ in range(channels)]
    for r in rows:
        r[::frame_size] &= 0x1F if type != 2 else 0x7F  # scale high bits / filter as a real encoder leaves them
    for p in empty:
        j, c = divmod(p, channels)
        rows[c][j * frame_size:(j + 1) * frame_size] = 0
    if revision in (8, 9):
        rows = O.adx_crypt(rows, key, revision, frame_size)
        xs = adx_stream(key, frames * channels)
        for p in empty_after:
            j, c = divmod(p, channels)
            rows[c][j * frame_size:(j + 1) * frame_size] = 0
            rows[c][j * frame_size] = (xs[p] >> 8) & (0x1F if revision == 9 else 0xFF)
            rows[c][j * frame_size + 1] = xs[p] & 0xFF
    samples = frames * spf - inserted
    hist = history if history is not None else [(17 * c - 5) & 0x7FFF for c in range(channels)]
    return O.adx_write(rows, hist, rate, samples, loop, inserted, frame_size, version, type, 500, revision, None, trim)


def expected_adx(image, enc_type=0, out_key=None, no_trim=False, in_key=None) -> Optional[np.ndarray]:
    """The .adx file the reference writes for one source image (None where the rewrite refuses it)."""
    st, h = RA.adx_parse(image)
    if st != 0:
        return None
    rows = RA.audio_rows(image, h)
    if h.revision in (8, 9):
        if in_key is None:
            return None
        rows = O.adx_crypt(rows, in_key, h.revision, h.frame_size)
    samples = _i32(h.sample_count - h.inserted_samples)
    loop = None
    if h.looping:
        loop = (_i32(h.loop_start_sample - h.inserted_samples), _i32(h.loop_end_sample - h.inserted_samples))
        if not (0 <= loop[0] <= samples and 0 <= loop[1] <= samples and loop[0] <= loop[1]):
            return None
    if samples < 0 or h.inserted_samples < 0:
        return None
    history = [hh[0] for hh in h.history] if h.history else [0] * h.channel_count
    return O.adx_write(rows, history, h.sample_rate, samples, loop, h.inserted_samples, h.frame_size, h.version, h.type,
                       h.highpass_frequency, enc_type, out_key, not no_trim)


# ---- HCA ----------------------------------------------------------------------------------------------------------------
class _Past(Exception):
    pass


def hca_parse(image):
    """hca_reader_oracle.hca_parse, extended: (status, O.HcaInfo, ciph, comment bytes or None, rva float bits)."""
    data = np.ascontiguousarray(image, dtype=np.uint8).tobytes()
    info, ciph, comment, rva = O.HcaInfo(), 0, None, 0x3F800000
    pos = 0

    def take(n: int) -> bytes:
        nonlocal pos
        if pos + n > len(data):
            raise _Past
        pos += n
        return data[pos - n: pos]

    def u(n: int) -> int:
        return int.from_bytes(take(n), "big")

    def s(n: int) -> int:
        return int.from_bytes(take(n), "big", signed=True)

    def chunk_id() -> bytes:
        return bytes(b & 0x7F for b in take(4))

    try:
        sig = chunk_id()
        version = s(2)
        info.header_size = s(2)
        if sig != b"HCA\0":
            return E_NOT_HCA, info, ciph, comment, rva
        has_ath = False
        while pos < info.header_size:
            cid = chunk_id()
            if cid == b"fmt\0":
                info.channel_count = u(1)
                info.sample_rate = u(1) << 16 | u(2)
                info.frame_count = s(4)
                info.inserted_samples = s(2)
                info.appended_samples = s(2)
                info.sample_count = _i32(info.frame_count * 1024 - info.inserted_samples - info.appended_samples)
            elif cid == b"comp":
                info.frame_size = s(2)
                (info.min_resolution, info.max_resolution, info.track_count, info.channel_config, info.total_band_count,
                 info.base_band_count, info.stereo_band_count, info.bands_per_hfr_group) = take(8)
                take(2)
            elif cid == b"dec\0":
                info.frame_size = s(2)
                info.min_resolution, info.max_resolution = take(2)
                info.total_band_count = u(1) + 1
                info.base_band_count = u(1) + 1
                packed = u(1)
                info.track_count, info.channel_config = packed >> 4, packed & 0xF
                if u(1) == 0:
                    info.base_band_count = info.total_band_count
                else:
                    info.stereo_band_count = info.total_band_count - info.base_band_count
            elif cid == b"loop":
                info.looping = 1
                info.loop_start_frame, info.loop_end_frame = s(4), s(4)
                info.pre_loop_samples, info.post_loop_samples = s(2), s(2)
                loop_end = _i32((info.loop_end_frame + 1) * 1024 - info.post_loop_samples - info.inserted_samples)
                info.sample_count = min(info.sample_count, loop_end)
            elif cid == b"ath\0":
                info.use_ath_curve = int(s(2) == 1)
                has_ath = True
            elif cid == b"ciph":
                ciph = s(2)
            elif cid == b"rva\0":
                rva = u(4)
            elif cid == b"vbr\0":
                take(4)
            elif cid == b"comm":
                pos += 1
                if pos >= len(data):
                    raise _Past
                # ReadUTF8Z: bytes while ReadByte() - 1 > 0; Position - start - 1 of them, so at the end of the stream
                # (ReadByte -1, Position unchanged) the last byte read is not part of the text
                q = pos
                while q < len(data) and data[q] > 1:
                    q += 1
                comment = data[pos:q] if q < len(data) else data[pos:len(data) - 1]
                pos = info.header_size
            elif cid == b"pad\0":
                pos = info.header_size
            else:
                return E_CHUNK, info, ciph, comment, rva
    except _Past:
        return E_TRUNCATED, info, ciph, comment, rva
    if version < 0x0200 and not has_ath:
        info.use_ath_curve = 1
    if info.track_count < 1:
        info.track_count = 1
    if info.bands_per_hfr_group > 0:
        info.hfr_band_count = info.total_band_count - info.base_band_count - info.stereo_band_count
        info.hfr_group_count = -(-info.hfr_band_count // info.bands_per_hfr_group)
    if info.header_size < 0 or info.frame_count < 0 or (info.frame_count > 0 and info.frame_size < 2):
        return E_HEADER, info, ciph, comment, rva
    if info.frame_count * max(info.frame_size, 0) > len(data) - info.header_size:
        return E_TRUNCATED, info, ciph, comment, rva
    return 0, info, ciph, comment, rva


def comment_blank(text: str) -> bool:
    return all(ord(ch) in NET_SPACE for ch in text)


def hca_chunks(info, masked: bool, ciph: int, comment: Optional[bytes], rva_bits: int) -> bytes:
    """HcaWriter.WriteHeader's chunk stream (HcaWriter.cs:56-170), up to the CRC."""
    def cid(s: bytes) -> bytes:
        return bytes(b | 0x80 if masked and b else b for b in s)

    h = cid(b"HCA\0") + struct.pack(">Hh", 0x0200, info.header_size)
    h += cid(b"fmt\0") + struct.pack(">BBHiHH", info.channel_count & 0xFF, (info.sample_rate >> 16) & 0xFF, info.sample_rate & 0xFFFF,
                                     info.frame_count, info.inserted_samples & 0xFFFF, info.appended_samples & 0xFFFF)
    h += cid(b"comp") + struct.pack(">h8BH", info.frame_size, *(v & 0xFF for v in (
        info.min_resolution, info.max_resolution, info.track_count, info.channel_config, info.total_band_count,
        info.base_band_count, info.stereo_band_count, info.bands_per_hfr_group)), 0)
    if info.looping:
        h += cid(b"loop") + struct.pack(">iihh", info.loop_start_frame, info.loop_end_frame, info.pre_loop_samples, info.post_loop_samples)
    h += cid(b"ciph") + struct.pack(">h", ciph)
    if rva_bits != 0x3F800000:  # volume != 1, NaN included
        h += cid(b"rva\0") + struct.pack(">I", rva_bits)
    if comment is None or comment_blank(comment.decode("utf-8")):
        h += cid(b"pad")
    else:
        h += cid(b"comm\0") + comment + b"\0"
    return h


def expected_hca(image, out_key_type=-1, out_key_code=0, in_key_code=None) -> Optional[np.ndarray]:
    """The .hca file the reference writes for one source image (None where the rewrite refuses it)."""
    st, info, ciph, comment, rva = hca_parse(image)
    if st != 0:
        return None
    if comment is not None:
        try:
            comment.decode("utf-8")
        except UnicodeDecodeError:
            return None
    img = np.ascontiguousarray(image, np.uint8)
    fs, fc = info.frame_size, info.frame_count
    frames = img[info.header_size: info.header_size + fs * fc].copy()
    dec = None
    if ciph == 1:
        dec = O.hca_key_tables(1)[0]
    elif ciph == 56:
        if in_key_code is None:
            return None
        dec = O.hca_key_tables(56, in_key_code)[0]
    if dec is not None:
        frames = O.hca_crypt_frames(frames, fs, dec)
    keyed = out_key_type >= 0
    if keyed:
        frames = O.hca_crypt_frames(frames, fs, O.hca_key_tables(out_key_type, out_key_code)[1])
    out_ciph = out_key_type if keyed else 0 if dec is not None else ciph
    if info.header_size < 8:
        return None
    chunks = hca_chunks(info, keyed, out_ciph, comment, rva)
    total = info.header_size + fs * fc
    if len(chunks) > total:
        return None  # the reference would grow the file
    out = np.zeros(max(total, len(chunks)), np.uint8)
    out[:len(chunks)] = np.frombuffer(chunks, np.uint8)
    crc = O.crc16(out[:info.header_size - 2].tobytes())
    out[info.header_size - 2: info.header_size] = (crc >> 8, crc & 0xFF)
    out[info.header_size: total] = frames
    return out[:total]


def hca_info(channels=2, frame_count=6, frame_size=0x100, looping=False, track_count=1, rate=44100):
    info = O.HcaInfo()
    info.channel_count, info.sample_rate, info.frame_count, info.frame_size = channels, rate, frame_count, frame_size
    info.inserted_samples, info.appended_samples = 128, 200
    info.min_resolution, info.max_resolution, info.track_count, info.channel_config = 1, 15, track_count, 0
    info.total_band_count, info.base_band_count, info.stereo_band_count, info.bands_per_hfr_group = 128, 96, 16, 4
    if looping:
        info.looping, info.loop_start_frame, info.loop_end_frame, info.pre_loop_samples, info.post_loop_samples = 1, 1, frame_count - 2, 64, 32
    return info


def hca_frames(info, seed: int, bad_crc=(), text: bytes = b"") -> np.ndarray:
    """Random frames with their CRC-16 (frame k in bad_crc gets a wrong one); `text` starts frame 0's bytes."""
    rng = np.random.default_rng(seed)
    fs = info.frame_size
    fr = rng.integers(0, 256, (info.frame_count, fs), dtype=np.uint8)
    fr[:, :2] = 0xFF
    if text:
        fr[0, :len(text)] = np.frombuffer(text, np.uint8)
    for k in range(info.frame_count):
        crc = O.crc16(fr[k, :fs - 2].tobytes()) ^ (0x1234 if k in bad_crc else 0)
        fr[k, fs - 2:] = (crc >> 8, crc & 0xFF)
    return fr.ravel()


def hca_source(info, frames, ciph=0, key_code=HCA_KEY, header_size=None, comment: Optional[bytes] = None, terminator=b"\0",
               rva: Optional[int] = None, ath: Optional[int] = None, vbr: bool = False, dec: bool = False, version=0x0200,
               track_byte: Optional[int] = None) -> np.ndarray:
    """An .hca image: chunks in the order HcaReader reads them (ids masked when "ciph" is not 0), then the frames,
    encrypted with the "ciph" value's table (56: key_code; 2: left as they are).  comment: the bytes behind "comm\\0",
    then `terminator` (empty: the text runs on into whatever follows the header)."""
    masked = ciph != 0

    def cid(s: bytes) -> bytes:
        return bytes(b | 0x80 if masked and b else b for b in s)

    h = cid(b"fmt\0") + struct.pack(">BBHiHH", info.channel_count, info.sample_rate >> 16, info.sample_rate & 0xFFFF, info.frame_count,
                                     info.inserted_samples, info.appended_samples)
    tb = info.track_count if track_byte is None else track_byte
    if dec:
        h += cid(b"dec\0") + struct.pack(">hBBBBBB", info.frame_size, info.min_resolution, info.max_resolution, info.total_band_count - 1,
                                         info.base_band_count - 1, (tb << 4) | info.channel_config, 1)
    else:
        h += cid(b"comp") + struct.pack(">h8BH", info.frame_size, info.min_resolution, info.max_resolution, tb, info.channel_config,
                                        info.total_band_count, info.base_band_count, info.stereo_band_count, info.bands_per_hfr_group, 0)
    if info.looping:
        h += cid(b"loop") + struct.pack(">iihh", info.loop_start_frame, info.loop_end_frame, info.pre_loop_samples, info.post_loop_samples)
    if ath is not None:
        h += cid(b"ath\0") + struct.pack(">h", ath)
    if vbr:
        h += cid(b"vbr\0") + struct.pack(">hh", info.frame_size, 7)
    h += cid(b"ciph") + struct.pack(">h", ciph)
    if rva is not None:
        h += cid(b"rva\0") + struct.pack(">I", rva)
    if comment is not None:
        h += cid(b"comm\0") + comment + terminator
    else:
        h += cid(b"pad\0")
    size = 8 + len(h) + 2 if header_size is None else header_size
    head = bytearray((cid(b"HCA\0") + struct.pack(">Hh", version, size) + h).ljust(size, b"\0"))
    head = head[:size]
    if 8 + len(h) <= size - 2:  # else the comment runs on through where the CRC would go (the reader checks no CRC)
        head[size - 2:size] = struct.pack(">H", O.crc16(bytes(head[:size - 2])))
    fr = np.ascontiguousarray(frames, np.uint8).ravel()
    if ciph == 1:
        fr = O.hca_crypt_frames(fr, info.frame_size, O.hca_key_tables(1)[1])
    elif ciph == 56:
        fr = O.hca_crypt_frames(fr, info.frame_size, O.hca_key_tables(56, key_code)[1])
    return np.frombuffer(bytes(head) + fr.tobytes(), np.uint8).copy()


# ---- the stimuli: (name, image, options, input key, the features the file exercises) -----------------------------------
ADX_KEY_STRING, ADX_KEY_CODE, ADX_KEY_CODE_B = "vgaudio-b200", 0x0123456789ABCDEF, 0x00FEDCBA98765432


def adx_keys():
    """The input and output keys of the ADX cases: a type-8 key from a string, two type-9 keys from codes."""
    return O.adx_key(key_string=ADX_KEY_STRING), O.adx_key(key_code=ADX_KEY_CODE), O.adx_key(key_code=ADX_KEY_CODE_B)


def adx_out(enc_type=0, key=None, no_trim=False) -> dict:
    o = {"adx_encryption_type": enc_type, "no_trim": int(no_trim)}
    if key is not None:
        o.update(adx_has_key=1, adx_key_seed=key[0], adx_key_mult=key[1], adx_key_inc=key[2])
    return o


def adx_cases():
    k8, k9, k9b = adx_keys()
    key_of = {0: None, 8: k8, 9: k9}
    cases = []
    spf = 32
    for rev in (0, 8, 9):
        for out_type, out_key in ((0, None), (8, k8), (9, k9b)):
            img = adx_source(2, 24, revision=rev, key=key_of[rev], loop=(40, 9 * spf), seed=rev * 10 + out_type,
                             empty=(4, 9), empty_after=(6, 11) if rev else ())
            cases.append((f"rev{rev}->{out_type}", img, adx_out(out_type, out_key), key_of[rev],
                          {f"rev{rev}", f"out{out_type}", "empty", "loop trimmed", "v4", "fs18", "linear", "ch2"} | ({"empty after"} if rev else set())))
    img = adx_source(2, 16, revision=9, key=k9, seed=3, empty_after=(1, 2))
    cases.append(("9->9 other key", img, adx_out(9, k9b), k9, {"rev9", "out9", "9->9", "empty after", "no loop block", "non-looping"}))
    cases.append(("9->9 same key", img, adx_out(9, k9), k9, {"rev9", "out9"}))
    cases.append(("no key, type byte 8", adx_source(2, 10, seed=4), adx_out(8), None, {"rev0", "enc byte without key"}))
    cases.append(("v3 inserted", adx_source(2, 30, version=3, loop=(70, 20 * spf), inserted=45, seed=5), adx_out(), None,
                  {"v3", "inserted v3", "loop trimmed"}))
    cases.append(("v3 inserted keyed", adx_source(1, 30, version=3, revision=9, key=k9, loop=(64 * 3, 20 * spf), inserted=2 * spf + 7, seed=6),
                  adx_out(8, k8), k9, {"v3", "inserted v3", "ch1"}))
    cases.append(("mono v4", adx_source(1, 12, seed=7, loop=(0, 12 * spf)), adx_out(), None, {"ch1", "loop past source"}))
    cases.append(("6ch", adx_source(6, 9, revision=8, key=k8, seed=8, loop=(32, 5 * spf)), adx_out(9, k9), k8, {"ch6"}))
    cases.append(("255ch", adx_source(255, 3, version=3, revision=9, key=k9, seed=9), adx_out(8, k8), k9, {"ch255", "non-looping"}))
    cases.append(("fs34", adx_source(2, 10, frame_size=34, revision=8, key=k8, seed=10, loop=(60, 8 * 64)), adx_out(9, k9b), k8, {"fs34"}))
    cases.append(("fs34 odd offsets", adx_source(3, 7, frame_size=33, seed=11, loop=(10, 6 * 62)), adx_out(), None, {"odd frame size"}))
    cases.append(("fixed", adx_source(2, 10, type=2, revision=9, key=k9, seed=12, loop=(32, 6 * spf)), adx_out(9, k9b), k9, {"fixed"}))
    cases.append(("exponential", adx_source(2, 10, type=4, seed=13, loop=(32, 6 * spf)), adx_out(8, k8), None, {"exponential"}))
    cases.append(("loop end at source end", adx_source(2, 12, revision=9, key=k9, seed=14, loop=(64, 12 * spf - 10)), adx_out(9, k9b), k9,
                  {"loop past source"}))
    cases.append(("no trim", adx_source(2, 12, seed=15, loop=(64, 6 * spf)), adx_out(no_trim=True), None, {"no_trim"}))
    cases.append(("no trim keyed", adx_source(2, 12, revision=8, key=k8, seed=16, loop=(64, 6 * spf)), adx_out(9, k9, no_trim=True), k8, {"no_trim"}))
    return cases


def hca_out(key_type=-1) -> dict:
    return {"hca_key_type": key_type, "hca_key_code": HCA_KEY_OUT}


def hca_cases():
    cases = []
    for ciph in (0, 1, 56, 2):
        for out in (-1, 0, 1, 56):
            info = hca_info(looping=ciph == 1)
            img = hca_source(info, hca_frames(info, ciph * 7 + out + 1), ciph=ciph, comment=b"rewrite test")
            cases.append((f"ciph{ciph}->{out}", img, hca_out(out), {f"ciph{ciph}", f"out{out}", "comm ascii"}))
    info = hca_info(frame_count=4)
    add = lambda name, img, out, tags: cases.append((name, img, hca_out(out), tags))  # noqa: E731
    add("utf8", hca_source(info, hca_frames(info, 20), comment="café 日本 \U0001F600".encode()), 56, {"comm utf8"})
    add("white space", hca_source(info, hca_frames(info, 21), comment="   　\t\u0085".encode()), -1, {"comm blank"})
    add("0x01", hca_source(info, hca_frames(info, 22), ciph=56, comment=b"stop\x01here"), -1, {"comm 0x01", "ciph56"})
    text_info = hca_info(frame_count=5, frame_size=0x80)
    add("into frames", hca_source(text_info, hca_frames(text_info, 23, text=b" and on into the frames\0"), comment=b"comment text",
                                  terminator=b"", header_size=8 + 16 + 16 + 6 + 5 + 4), 1, {"comm into frames", "overflow"})
    for bits, tag in ((0x3F800000, "rva 1"), (0x3F000000, "rva 0.5"), (0x7FC00000, "rva nan")):
        add(tag, hca_source(info, hca_frames(info, 24), ciph=1, rva=bits), -1, {tag})
    add("ath v1", hca_source(info, hca_frames(info, 25), ath=1, version=0x0100), -1, {"ath"})
    add("vbr", hca_source(info, hca_frames(info, 26), vbr=True, ciph=56), 0, {"vbr"})
    dec_info = hca_info(frame_count=3)
    dec_info.stereo_band_count = dec_info.total_band_count - dec_info.base_band_count
    dec_info.bands_per_hfr_group = 0
    add("dec", hca_source(dec_info, hca_frames(dec_info, 27), dec=True), 56, {"dec"})
    # the dec chunk is 4 bytes shorter than comp: at its exact header size the rewritten chunks overflow into the frames
    exact = 8 + 16 + 12 + 6 + 4 + 2
    add("dec overflow", hca_source(dec_info, hca_frames(dec_info, 28), dec=True, header_size=exact), -1, {"dec", "overflow"})
    add("track 0", hca_source(info, hca_frames(info, 29), track_byte=0), 1, {"track 0"})
    loop_info = hca_info(frame_count=8, looping=True)
    add("loop", hca_source(loop_info, hca_frames(loop_info, 30), ciph=56, comment=b"loop"), 56, {"loop"})
    bad = hca_frames(info, 31, bad_crc=(1, 3))
    add("bad crc copied", hca_source(info, bad), -1, {"bad crc copied"})
    add("bad crc rekeyed", hca_source(info, bad), 56, {"bad crc rekeyed"})
    add("bad crc ciph2", hca_source(info, bad, ciph=2), -1, {"bad crc copied", "ciph2"})
    big = hca_info(frame_count=2, frame_size=0x300, channels=1)
    add("padded header", hca_source(big, hca_frames(big, 32), header_size=0x60, comment=b"x"), 0, {"comm ascii"})
    return cases


def refused_cases():
    """(name, format, image, options, adx key, hca key code, status, message part): files the rewrite refuses."""
    k8, k9, _ = adx_keys()
    import adx_files as F
    info = hca_info(frame_count=2)
    fr = hca_frames(info, 40)
    tiny = hca_info(frame_count=0)
    out = [
        ("adx keyed without key", ADX, adx_source(2, 4, revision=9, key=k9), adx_out(), None, None, -2, "no key"),
        ("adx bad loop", ADX, F.header(samples=320, inserted=0, loop_count=1, loop=(1, 10, 0, 400, 0), header_size=0x3C), adx_out(), None,
         None, -1, "Loop points"),
        ("adx loop end before start", ADX, F.header(samples=320, inserted=0, loop_count=1, loop=(1, 100, 0, 50, 0), header_size=0x3C),
         adx_out(), None, None, -1, "loop end must be greater"),
        ("adx signature", ADX, np.zeros(64, np.uint8), adx_out(), None, None, -2, "signature"),
        ("adx truncated", ADX, adx_source(2, 8)[:100], adx_out(), None, None, -2, "Specified length"),
        ("hca keyed without key", HCA, hca_source(info, fr, ciph=56), hca_out(), None, None, -2, "Cannot find key"),
        ("hca not hca", HCA, np.zeros(64, np.uint8), hca_out(), None, None, -2, "Not a valid HCA"),
        ("hca truncated", HCA, hca_source(info, fr)[:200], hca_out(), None, None, -2, "enough data"),
        ("hca overflow past the end", HCA, hca_source(tiny, np.zeros(0, np.uint8), comment=b"a long comment" * 4, header_size=0x30),
         hca_out(), None, None, -2, "past the end"),
    ]
    for bad in (b"\xc0\x80", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"ok\x80", b"\xe2\x82"):
        out.append((f"hca utf8 {bad!r}", HCA, hca_source(info, fr, comment=bad), hca_out(), None, None, -2, "UTF-8"))
    return out
