"""CriAdxCodec.Decode (Codecs/CriAdx/CriAdxCodec.cs:9-54) restated in plain Python from the C#, apart from the oracle's C,
so that the tests can hold every ADX decode path to the reference's verdict as well as to its PCM.

The restatement keeps what the C# does: int arithmetic wrapping at 32 bits, the (short) casts of the scale, the shift
count of `1 << (12 - scale)` masked to 5 bits as C# masks it, the version-3 and version-4 rounding orders, Clamp16, the
padding logic (startSample, the inIndex skip, zeros where no frame reaches) and the IndexOutOfRangeException at
`coefs[filterNum]`: four rows for the Fixed type, one (the computed pair) for every other type, indexed inside the
sample loop only, so a frame that yields no sample is never checked.

Also the stream geometry the product's decoders are built around (serial fast-path groups, the time-parallel decoder's
head / body / tail frames and segment boundaries), used to aim test streams at each path."""
from __future__ import annotations

import math

import numpy as np

FIXED, LINEAR, EXPONENTIAL = 2, 3, 4  # CriAdxType.cs:3-8
COEFS = ((0, 0), (0x0F00, 0), (0x1CC0, -0x0D00), (0x1880, -0x0DC0))  # CriAdxCodec.Coefs (:186-191) as shorts


class CoefsIndexError(IndexError):
    """coefs[filterNum] out of range (CriAdxCodec.cs:38 / :42): frame `frame` (0 = the first frame Decode reads) selects
    filter `filter_num` of a table with `rows` rows."""

    def __init__(self, frame: int, filter_num: int, rows: int):
        super().__init__(f"frame {frame}: filter {filter_num} indexes a {rows}-row coefficient table")
        self.frame, self.filter_num, self.rows = frame, filter_num, rows


def _s16(v: int) -> int:
    """C#'s (short) cast: keep the low 16 bits."""
    return ((v + 0x8000) & 0xFFFF) - 0x8000


def _trunc_div(a: int, b: int) -> int:
    """C#'s int division (rounds toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def calculate_coefficients(highpass_frequency: int, sample_rate: int):
    """CriAdxCodec.CalculateCoefficients (:173-184) for the finite results of positive rates."""
    sqrt2 = math.sqrt(2)
    a = sqrt2 - math.cos(2.0 * math.pi * highpass_frequency / sample_rate)
    b = sqrt2 - 1
    c = (a - math.sqrt((a + b) * (a - b))) / b
    return _s16(int(c * 8192)), _s16(int(c * c * -4096))  # (short) of a double truncates toward zero


def decode(adpcm, sample_count: int, sample_rate: int = 48000, highpass_frequency: int = 500, frame_size: int = 18,
           version: int = 4, history: int = 0, padding: int = 0, type: int = LINEAR):
    """CriAdxCodec.Decode: the PCM as a list of ints, or CoefsIndexError where the reference throws.  A read past
    `adpcm` raises IndexError as the reference does."""
    data = bytes(adpcm)
    spf = (frame_size - 2) * 2
    coefs = COEFS if type == FIXED else (calculate_coefficients(highpass_frequency, sample_rate),)
    pcm = [0] * sample_count
    hist1 = hist2 = history
    frame_count = -(-sample_count // spf)  # DivideByRoundUp
    current = 0
    start = padding % spf if padding > 0 else 0
    at = _trunc_div(padding, spf) * frame_size
    for i in range(frame_count):
        b0, b1 = data[at], data[at + 1]
        filter_num = (b0 >> 4) >> 1
        scale = _s16(((b0 << 8) | b1) & 0x1FFF)
        scale = _s16(1 << ((12 - scale) & 31)) if type == EXPONENTIAL else _s16(scale + 1)
        at += 2 + start // 2
        to_read = min(spf, sample_count - current)
        if start < to_read:  # the sample loop runs, and its first statement indexes coefs[filterNum]
            if filter_num >= len(coefs):
                raise CoefsIndexError(i, filter_num, len(coefs))
            c0, c1 = coefs[filter_num]
        for s in range(start, to_read):
            if s & 1:
                q = data[at] & 0xF
                at += 1
            else:
                q = data[at] >> 4
            q = q - 16 if q >= 8 else q
            if version == 4:
                p = ((hist1 * c0 + hist2 * c1 + 0x80000000) & 0xFFFFFFFF) - 0x80000000
                v = scale * q + (p >> 12)
            else:
                v = scale * q + (hist1 * c0 >> 12) + (hist2 * c1 >> 12)
            v = ((v + 0x80000000) & 0xFFFFFFFF) - 0x80000000
            v = -32768 if v < -32768 else (32767 if v > 32767 else v)  # Clamp16
            hist2, hist1 = hist1, v
            pcm[current] = v
            current += 1
        start = 0
    return pcm


def verdict(adpcm, sample_count: int, **params):
    """(pcm, None) where Decode returns, (None, CoefsIndexError) where it throws."""
    try:
        return decode(adpcm, sample_count, **params), None
    except CoefsIndexError as e:
        return None, e


# ---- geometry ------------------------------------------------------------------------------------------------------------
def frame_count(n: int, frame_size: int) -> int:
    return -(-n // ((frame_size - 2) * 2))


def head_row_frame(frame_size: int, padding: int) -> int:
    """The frame of the row that Decode reads first (inIndex = Padding / samplesPerFrame * FrameSize)."""
    return _trunc_div(padding, (frame_size - 2) * 2)


def head_yields(n: int, frame_size: int, padding: int) -> bool:
    spf = (frame_size - 2) * 2
    return n > 0 and min(spf, n) > (padding % spf if padding > 0 else 0)


def serial_fast_frames(n: int, frame_size: int, padding: int) -> int:
    """Frames the serial decoder (adx_decode_kernel) takes through its 8-frame groups: 18-byte frames without padding,
    every whole group of 256 samples."""
    return n // 256 * 8 if frame_size == 18 and padding == 0 else 0


def seg_boundaries(n: int, frame_size: int, padding: int, seg_count: int, min_seg: int):
    """Decode-order frame indices where the time-parallel decoder starts segments 1.. (its body frames are the frames
    after the head that yield all their samples; interior boundaries sit on 8-frame groups of the row)."""
    spf = (frame_size - 2) * 2
    start = padding % spf if padding > 0 else 0
    frames = frame_count(n, frame_size) if n > 0 else 0
    k0 = max(min(n, spf) - start, 0) if frames > 0 else 0
    body = min(1 + (n - k0) // spf, frames) - 1 if frames > 0 else 0
    per = -(-body // seg_count)
    seg_len = (max(per, min_seg) + 7) & ~7
    a1 = head_row_frame(frame_size, padding) + 1
    out = []
    for s in range(1, seg_count):
        lo = min(body, s * seg_len - (a1 & 7))
        if lo >= body:
            break
        out.append(1 + lo)
    return out


# ---- the stream matrix ---------------------------------------------------------------------------------------------------
class Stream:
    """One ADX channel row and the parameters Decode reads it with.  `fault` is the decode-order frame whose filter
    number was set to `filter` (None for a stream built clean), `placement` names the path that frame is aimed at."""

    def __init__(self, data, n, frame_size, version, padding, type, history=0, fault=None, filter=0, placement="clean"):
        self.data, self.n = data, n
        self.frame_size, self.version, self.padding, self.type, self.history = frame_size, version, padding, type, history
        self.fault, self.filter, self.placement = fault, filter, placement

    def params(self, history=None) -> dict:
        return dict(frame_size=self.frame_size, version=self.version, history=self.history if history is None else history,
                    padding=self.padding, type=self.type)

    def __repr__(self):
        return (f"Stream(type={self.type} v{self.version} fs={self.frame_size} pad={self.padding} n={self.n} "
                f"{self.placement} frame={self.fault} filter={self.filter})")


TYPES_VERSIONS = [(t, v) for t in (FIXED, LINEAR, EXPONENTIAL) for v in (3, 4)]
# (frame size, padding, n): padding 0, an odd padding % spf, padding >= spf; counts on the serial decoder's 256-sample
# groups (3072) and off them; every layout is also run at n + 1
LAYOUTS = [(18, 0, 3072), (18, 0, 3108), (18, 45, 2000), (18, 13, 1500), (3, 0, 301), (3, 7, 400), (9, 5, 1000), (9, 31, 777),
           (255, 0, 506 * 20 + 77), (255, 601, 506 * 12 + 1)]
# n <= padding % spf: the head frame yields no sample (n + 1 makes it yield)
SILENT_HEADS = [(18, 20, 20), (18, 45, 13), (3, 1, 1), (9, 5, 5), (255, 601, 95)]
# Exponential scale fields whose masked shift count (12 - scale) & 31 is 31, 16 and 15
EXP_SPECIAL_SCALES = (13, 28, 29)


def clean_row(rng, type, frame_size, padding, n, extra=2):
    """Random frames Decode accepts: Fixed frames cycle through the four table rows, other types select filter 0;
    Linear / Fixed scales are mostly moderate, Exponential ones mostly 0..12 with the special shift counts mixed in.  The
    frames in front of the head (skipped by inIndex) and `extra` frames past frameCount carry filter numbers the table
    cannot index: Decode never reads them."""
    head = head_row_frame(frame_size, padding)
    fc = frame_count(n, frame_size)
    frames = head + fc + extra
    a = rng.integers(0, 256, (frames, frame_size), dtype=np.uint8)
    k = np.arange(frames)
    if type == EXPONENTIAL:
        scale = rng.integers(0, 13, frames)
        scale[k % 5 == 4] = np.array(EXP_SPECIAL_SCALES)[(k[k % 5 == 4] // 5) % 3]
    else:
        scale = np.where(k % 9 == 8, rng.integers(0, 0x2000, frames), rng.integers(0, 0x180, frames))
    filt = (k + rng.integers(0, 4)) % 4 if type == FIXED else np.zeros(frames, np.int64)
    filt[:head] = 7
    filt[head + fc:] = (k[head + fc:] + n) % 8
    a[:, 0] = ((filt << 5) | (scale >> 8)).astype(np.uint8)
    a[:, 1] = (scale & 0xFF).astype(np.uint8)
    return a.ravel()


def burst_then_silence(rng, frames=600, loud=60):
    """Linear 18-byte frames: `loud` frames of random nibbles, then digital silence, where a wrong history pair stays
    fixed under the >> 12 and a segment boundary never re-locks."""
    a = rng.integers(0, 256, (frames, 18), dtype=np.uint8)
    a[:, 0] &= 0x0F
    a[loud:] = 0
    return a.ravel()


def clean_streams(seed=1):
    """Every type and version over every layout and silent head, at n and n + 1, and the silence stream."""
    rng = np.random.default_rng(seed)
    out = []
    for type, version in TYPES_VERSIONS:
        for fs, pad, n in LAYOUTS + SILENT_HEADS:
            for m in (n, n + 1):
                hist = int(rng.integers(-32768, 32768)) if len(out) % 3 else 0
                out.append(Stream(clean_row(rng, type, fs, pad, m), m, fs, version, pad, type, hist))
    out.append(Stream(burst_then_silence(rng), 600 * 32, 18, 4, 0, LINEAR, placement="silence"))
    return out


def placements(n, frame_size, padding, seg_count=8, min_seg=8):
    """{name: decode-order frame} of the points a fault frame is aimed at in one layout."""
    fc = frame_count(n, frame_size)
    p = {"head": 0, "past": fc}
    if fc > 1:
        p["tail"] = fc - 1
    fast = serial_fast_frames(n, frame_size, padding)
    if fast >= 32:
        p["group_first"], p["group_last"] = 24, 31
    if 0 < fast < fc - 1:
        p["remainder"] = fast
    b = seg_boundaries(n, frame_size, padding, seg_count, min_seg)
    if b:
        p["boundary"] = b[0]
        p["boundary_last"] = b[-1]
    if len(b) >= 3 and b[1] + 2 < b[2]:
        p["run_on"] = b[1] + 2
    return p


FAULT_LAYOUTS = [(18, 0, 3108), (18, 0, 3072), (18, 45, 2000), (9, 5, 1000), (3, 0, 301), (255, 0, 506 * 20 + 77)]


def fault_streams(seed=2, silent=False):
    """Every filter number 0..7 at every placement of FAULT_LAYOUTS (or, silent=True, in the head frame of every
    SILENT_HEADS stream and of the same stream with one more sample), for the three types; versions alternate."""
    rng = np.random.default_rng(seed)
    out = []
    for type in (FIXED, LINEAR, EXPONENTIAL):
        for fs, pad, n in (SILENT_HEADS if silent else FAULT_LAYOUTS):
            for m in ((n, n + 1) if silent else (n,)):
                base = clean_row(rng, type, fs, pad, m)
                for name, frame in ({"head": 0} if silent else placements(m, fs, pad)).items():
                    for f in range(8):
                        row = base.copy()
                        at = (head_row_frame(fs, pad) + frame) * fs
                        row[at] = (f << 5) | (row[at] & 0x1F)
                        out.append(Stream(row, m, fs, 3 + (f & 1), pad, type, int(rng.integers(-4000, 4000)), frame, f,
                                          ("silent_head" if not head_yields(m, fs, pad) else "yielding_head") if silent else name))
    return out



def adx_image(streams):
    """An .adx image (adx_files.header, Linear highpass 500 Hz at 48 kHz, history 0) whose channels are the rows of
    `streams`, which share type, version, frame size, padding (InsertedSamples) and n; each row cut to the frames of
    SampleCount = n + padding."""
    import adx_files

    s = streams[0]
    frames = frame_count(s.n + s.padding, s.frame_size)
    rows = [np.resize(np.asarray(x.data, np.uint8), frames * s.frame_size).reshape(frames, s.frame_size) for x in streams]
    audio = np.stack(rows, axis=1).tobytes()  # frame-interleaved (Interleave.cs)
    return adx_files.header(channels=len(streams), samples=s.n + s.padding, frame_size=s.frame_size, version=s.version,
                            type=s.type, inserted=s.padding, loop_count=0, header_size=60, audio=audio)
