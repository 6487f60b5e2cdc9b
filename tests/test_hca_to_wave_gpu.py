""".hca -> WAVE on the GPU: vgb_convert_hca_to_wave_batch against the oracle chain (hca_reader_oracle.hca_parse -> hca_crypt_frames with the
decryption table -> hca_decode -> wave_write16), per-file failures, the device-resident decode vgb_hca_decode_dev on torch
buffers, sharding over two bound devices, the .wav -> .hca -> .wav round trip and the CLI."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import hca_reader_oracle as R
import hca_stimuli as H
from vgaudio_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")
KEY = 0x00D7E1B6C2A94F03


def _expected(oracle, img, key_code=None):
    """The reader chain on the CPU: the WAVE image the reference would write for one .hca image."""
    st, info, ciph = R.hca_parse(img)
    assert st == 0
    frames = np.ascontiguousarray(img[info.header_size: info.header_size + info.frame_count * info.frame_size])
    if ciph in (1, 56):
        frames = oracle.hca_crypt_frames(frames, info.frame_size, oracle.hca_key_tables(ciph, key_code or 0)[0])
    pcm = oracle.hca_decode(info, frames.reshape(info.frame_count, info.frame_size))
    loop = None
    if info.looping:
        loop = (info.loop_start_frame * 1024 + info.pre_loop_samples - info.inserted_samples,
                (info.loop_end_frame + 1) * 1024 - info.post_loop_samples - info.inserted_samples)
    return oracle.wave_write16(list(pcm), info.sample_rate, loop)


def _encoded(oracle, channels, rate, n, seed, quality=2, loop=None, key_type=-1, ath=False):
    pcm = [synth.channel(seed + c, n, rate, degenerate=False) for c in range(channels)]
    info, frames = oracle.hca_encode(pcm, rate, quality, loop=loop, ath=ath)
    enc = oracle.hca_key_tables(key_type, KEY)[1] if key_type >= 0 else None
    img = oracle.hca_write(info, frames, enc, max(key_type, 0))
    if ath:
        img[4:6] = (0x01, 0x00)  # version 1.0 without an "ath" chunk: HcaReader turns UseAthCurve on
    return img


def _zero_samples(oracle):
    img = _encoded(oracle, 1, 48000, 900, 70)
    _, info, _ = R.hca_parse(img)
    img[8 + 4 + 10: 8 + 4 + 12] = np.frombuffer(struct.pack(">h", info.frame_count * 1024 - info.inserted_samples), np.uint8)
    return img


def _job(oracle):
    files = [_encoded(oracle, c, 48000, 7000 + 900 * c, 10 * c, quality=1 + c % 5) for c in range(1, 9)]
    files += [_encoded(oracle, 2, 44100, 30000, 90, loop=(4000, 21000)),              # looping, trimmed at loop_end
              _encoded(oracle, 1, 32000, 12000, 91, loop=(0, 12000), key_type=1),
              _encoded(oracle, 2, 48000, 15000, 92, quality=5, key_type=56),
              _encoded(oracle, 2, 22050, 9000, 93, ath=True),
              _zero_samples(oracle)]
    for i, (name, info) in enumerate(H.decoder_layouts()):  # intensity stereo and HFR layouts of 1..8 channels
        frames = H.build_frames(info, np.random.default_rng(500 + i))
        files.append(oracle.hca_write(info, frames))
    return files


def test_converter_matches_the_oracle_chain(vg, oracle):
    from vgaudio_b200 import containers as ct

    files = _job(oracle)
    outs, status = ct.convert_hca_to_wave_batch(files, key_code=KEY)
    assert status == [0] * len(files)
    for i, f in enumerate(files):
        assert outs[i].tobytes() == _expected(oracle, f, KEY).tobytes(), i


def test_bad_files_fail_alone(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    good = [_encoded(oracle, 2, 48000, 8000, 30), _encoded(oracle, 1, 48000, 6000, 31, key_type=1)]
    bad_sync = _encoded(oracle, 2, 48000, 8000, 32)
    _, info, _ = R.hca_parse(bad_sync)
    bad_sync[info.header_size + info.frame_size] ^= 0xff  # frame 1's sync word
    keyed = _encoded(oracle, 2, 48000, 8000, 33, key_type=56)
    short = _encoded(oracle, 1, 48000, 6000, 34)[:-5]
    files = [good[0], bad_sync, good[1], keyed, short]
    outs, status = ct.convert_hca_to_wave_batch(files)  # no key: the type-56 file cannot be decrypted
    assert status[0] == 0 and status[2] == 0
    assert status[1] == N.VGB_E_DATA and status[3] == N.VGB_E_DATA and status[4] == N.VGB_E_DATA
    assert outs[1] is None and outs[3] is None and outs[4] is None
    assert outs[0].tobytes() == _expected(oracle, good[0]).tobytes()
    assert outs[2].tobytes() == _expected(oracle, good[1]).tobytes()


def _decode_dev(vg, infos, frames):
    import torch

    from vgaudio_b200 import _native as N

    n = len(infos)
    arr = (N.VgbHcaInfo * n)(*infos)
    blobs = [np.ascontiguousarray(f, np.uint8).ravel() for f in frames]
    f_off = np.cumsum([0] + [b.size + 16 for b in blobs])[:-1].astype(np.int64)
    d_frames = torch.zeros(int(f_off[-1] + blobs[-1].size + 16), dtype=torch.uint8, device="cuda")
    for o, b in zip(f_off, blobs):
        d_frames[int(o): int(o) + b.size] = torch.from_numpy(b).cuda()
    nch = infos[0].channel_count
    stride = np.array([i.sample_count + 3 for i in infos], np.int64)
    p_off = np.cumsum([0] + [s * nch + 5 for s in stride])[:-1].astype(np.int64)
    d_pcm = torch.zeros(int(p_off[-1] + stride[-1] * nch + 5), dtype=torch.int16, device="cuda")
    ws_bytes = vg.lib.vgb_hca_decode_workspace_bytes(arr, n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    N.check(vg.lib.vgb_hca_decode_dev(d_frames.data_ptr(), f_off.ctypes.data, arr, n, d_pcm.data_ptr(), p_off.ctypes.data,
                                      stride.ctypes.data, ws.data_ptr(), ws_bytes, stream))
    st = vg.lib.vgb_hca_decode_dev_status(ws.data_ptr(), n, stream)
    pcm = d_pcm.cpu().numpy()
    return st, [[pcm[p_off[s] + c * stride[s]: p_off[s] + c * stride[s] + infos[s].sample_count] for c in range(nch)] for s in range(n)]


@pytest.mark.parametrize("stim", H.decoder_stimuli(), ids=lambda s: s.name)
def test_decode_dev_matches_batch_and_oracle(vg, oracle, stim):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import crihca

    infos = [N.VgbHcaInfo(*[getattr(stim.info, f) for f, _ in N.VgbHcaInfo._fields_]) for _ in stim.streams]
    st, dev = _decode_dev(vg, infos, stim.streams)
    assert st == 0
    host = crihca.decode_batch(infos, stim.streams)
    for s, frames in enumerate(stim.streams):
        want = oracle.hca_decode(stim.info, frames)
        for c in range(stim.info.channel_count):
            assert np.array_equal(dev[s][c], host[s][c]) and np.array_equal(dev[s][c], want[c]), (s, c)


@pytest.mark.parametrize("case", H.fault_cases(), ids=lambda c: c[0])
def test_decode_dev_status_maps_faults(vg, case):
    from vgaudio_b200 import _native as N

    name, info, bad, fault = case
    infos = [N.VgbHcaInfo(*[getattr(info, f) for f, _ in N.VgbHcaInfo._fields_]) for _ in range(3)]
    st, _ = _decode_dev(vg, infos, H.fault_streams(info, bad, fault, 7))
    assert st == N.VGB_E_DATA


def test_two_devices_give_the_same_bytes(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    files = _job(oracle)
    one, s1 = ct.convert_hca_to_wave_batch(files, key_code=KEY)
    N.check(vg.lib.vgb_shutdown())
    try:
        N.check(vg.lib.vgb_init_devices((C.c_int32 * 2)(0, 0), 2, 0))
        two, s2 = ct.convert_hca_to_wave_batch(files, key_code=KEY)
    finally:
        N.check(vg.lib.vgb_shutdown())
        N.check(vg.lib.vgb_init(0, 0))
    assert s1 == s2 == [0] * len(files)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(one, two))


def test_round_trip_wav_hca_wav(vg, oracle):
    from vgaudio_b200 import containers as ct

    waves = [oracle.wave_write16([synth.channel(40 + c, 20000, 48000, degenerate=False) for c in range(ch)], 48000, loop)
             for ch, loop in ((1, None), (2, (1000, 18000)), (6, None))]
    hcas, st = ct.convert_wave_batch(waves, ct.convert_options(ct.CONTAINER_HCA, hca_key_type=56, hca_key_code=KEY))
    assert st == [0, 0, 0]
    back, st = ct.convert_hca_to_wave_batch(hcas, key_code=KEY)
    assert st == [0, 0, 0]
    for h, w in zip(hcas, back):
        assert w.tobytes() == _expected(oracle, h, KEY).tobytes()


def test_cli_decodes_dsp_and_hca(tmp_path, vg, oracle):
    src, out = tmp_path / "in", tmp_path / "out"
    src.mkdir()
    pcm = [synth.channel(60, 5000, 32000, degenerate=False)]
    coefs = np.stack([oracle.calculate_coefficients(p) for p in pcm])
    dsp = oracle.dsp_write([oracle.encode(p, c) for p, c in zip(pcm, coefs)], coefs, 32000, 5000)
    plain, keyed = _encoded(oracle, 2, 48000, 9000, 61), _encoded(oracle, 1, 44100, 7000, 62, key_type=56)
    for name, data in (("a.dsp", dsp), ("b.hca", plain), ("c.HCA", keyed)):
        (src / name).write_bytes(data.tobytes())
    r = subprocess.run([CLI, "-i", str(src), "-o", str(out), "--out-format", "wav", "--keycode", str(KEY)], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.startswith("3 files converted, 0 failed"), r.stdout
    ok, info = oracle.dsp_parse(dsp)
    assert ok == 0
    assert (out / "b.wav").read_bytes() == _expected(oracle, plain).tobytes()
    assert (out / "c.wav").read_bytes() == _expected(oracle, keyed, KEY).tobytes()
    assert (out / "a.wav").stat().st_size == 44 + 5000 * 2
