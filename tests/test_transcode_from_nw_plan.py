"""vgb_transcode_from_nw_batch's sizing pass, on the host without a device: every NintendoWare stream, wave and prefetch
reader, IDSP and HPS into all eight targets, with every codec, byte order, loop point alignment, IDSP trimming and loop
setting, sized as the oracle chain sizes them (the reader restatement, SetLoop, then the target writer's geometry); every
per-file refusal fails its own file with its message and in its place in the order; the call's own refusals fail the
call and write nothing."""
import ctypes as C
import inspect
import os
import subprocess

import numpy as np
import pytest

import loop_override_oracle as LO
import transcode_from_nw_oracle as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "vgaudio_b200", "cli", "vgaudio_batch")


def _sizing(vg, files, in_types, opt):
    """(sizes, statuses, messages): the sizing pass file by file, so that each message belongs to its file."""
    sizes, status, msgs = [], [], []
    for f, t in zip(files, in_types):
        f = np.ascontiguousarray(f, np.uint8)
        ftab = (C.c_void_p * 1)(f.ctypes.data)
        lens = (C.c_int64 * 1)(f.size)
        types = (C.c_int32 * 1)(t)
        sz, st = (C.c_int64 * 1)(), (C.c_int32 * 1)()
        assert vg.lib.vgb_transcode_from_nw_batch(ftab, lens, types, 1, C.byref(opt), sz, None, st, None, None) == 0
        sizes.append(int(sz[0]))
        status.append(int(st[0]))
        msgs.append((vg.lib.vgb_last_error() or b"").decode() if st[0] else "")
    return sizes, status, msgs


# (codec, endianness, loop point alignment, trim) per target
CONFIGS = {X.DSP: [(X.GCADPCM, 0, 0, True)],
           X.ADX: [(X.GCADPCM, 0, 0, True)],
           X.HCA: [(X.GCADPCM, 0, 0, True)],
           X.BRSTM: [(X.GCADPCM, 0, 0, True), (X.GCADPCM, 0, 28, True), (X.PCM16, 0, 0, True), (X.PCM8, 0, 0, True)],
           X.BCSTM: [(X.GCADPCM, 0, 0, True), (X.GCADPCM, 2, 1000, True), (X.PCM16, 1, 0, True), (X.PCM8, 2, 0, True)],
           X.BFSTM: [(X.GCADPCM, 0, 0, True), (X.GCADPCM, 1, 14, True), (X.PCM16, 0, 0, True), (X.PCM8, 1, 0, True)],
           X.IDSP: [(X.GCADPCM, 0, 0, True), (X.GCADPCM, 0, 0, False)],
           X.HPS: [(X.GCADPCM, 0, 0, True)]}
LOOPS = [(LO.KEEP, 0, 0), (LO.SET, 700, 1500), (LO.SET, 1001, 1001), (LO.CLEAR, 0, 0)]


def _compare(got, want, ctx):
    size, status, msg = got
    want_size, why = want
    if want_size is not None:
        assert status == 0 and size == want_size, (ctx, status, msg)
        return 1
    assert status != 0 and size == 0, (ctx, why)
    if isinstance(why, str):
        assert msg.endswith(why), (ctx, msg, why)
    elif why is not None and why != -1:
        assert status == why, (ctx, status, why)
    return 0


@pytest.mark.parametrize("dst", X.TARGETS)
def test_sizing_pass_matches_the_oracle_chain(vg, oracle, dst):
    from vgaudio_b200 import containers as ct

    srcs = X.sources(oracle)
    files, types = [f for _, f, _ in srcs], [t for t, _, _ in srcs]
    sized = refused = 0
    for codec, endianness, alignment, trim in CONFIGS[dst]:
        for mode, s, e in LOOPS:
            loop = dict(loop=(s, e)) if mode == LO.SET else dict(no_loop=True) if mode == LO.CLEAR else {}
            opt = X.options(ct, dst, codec, endianness, alignment, trim, **loop)
            sizes, status, msgs = _sizing(vg, files, types, opt)
            for k, (t, f, note) in enumerate(srcs):
                want = X.expected_size(f, t, dst, codec, alignment, trim, mode, s, e)
                ok = _compare((sizes[k], status[k], msgs[k]), want, (note, codec, endianness, alignment, trim, mode, s, e))
                sized += ok
                refused += want[1] == X.MSG_REWRITE
    assert sized > 0 and (refused > 0) == (dst not in (X.ADX, X.HCA))  # no source holds ADX or HCA


def test_every_rewrite_cell_is_refused(vg, oracle):
    """GetFormat<T> hands back the source's own format: GC-ADPCM into .dsp, IDSP, HPS or GC-ADPCM NintendoWare, PCM16 into
    -f pcm16 and PCM8 into -f pcm8 (IDSP and HPS targets are GC-ADPCM whatever nw_codec_plus1 says)."""
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    srcs = X.sources(oracle)
    cells = [(X.DSP, 0), (X.IDSP, 0), (X.IDSP, 2), (X.HPS, 0), (X.HPS, 1)] + [(t, p) for t in X.NW_TARGETS for p in (0, 1, 2, 3)]
    seen = set()
    for dst, plus1 in cells:
        codec = plus1 - 1 if plus1 else X.GCADPCM
        opt = ct.convert_options(dst, nw_codec_plus1=plus1)
        sizes, status, msgs = _sizing(vg, [f for _, f, _ in srcs], [t for t, _, _ in srcs], opt)
        for k, (t, f, note) in enumerate(srcs):
            rewrite = X.source_codec(f, t) == X.target_codec(dst, codec)
            if rewrite:
                assert status[k] == N.VGB_E_ARG and sizes[k] == 0, (note, dst, plus1, status[k])
                assert msgs[k] == f"file 0: {X.MSG_REWRITE}", (note, msgs[k])
                seen.add((X.source_codec(f, t), X.target_codec(dst, codec)))
            else:
                assert X.MSG_REWRITE not in msgs[k], (note, dst, plus1)
    assert seen == {(X.GCADPCM, X.GCADPCM), (X.PCM16, X.PCM16), (X.PCM8, X.PCM8)}


def test_per_file_refusals_in_their_order(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    srcs = X.sources(oracle)
    gc_brstm, pcm16_bcstm = srcs[0][1], srcs[4][1]
    broken = np.frombuffer(b"IDSP" + bytes(60), np.uint8).copy()
    import nw_files as NF

    pcm16_3ch = NF.encoded(oracle, NF.BCSTM, X.PCM16, 3, 3001, seed=40)
    cases = [  # (image, in_type, options, status, message fragment)
        # 1. in_type
        (gc_brstm, 0, ct.convert_options(X.HCA), N.VGB_E_ARG, f"file 0: in_type 0 {X.MSG_IN_TYPE}"),
        (gc_brstm, X.DSP, ct.convert_options(X.HCA), N.VGB_E_ARG, f"file 0: in_type 1 {X.MSG_IN_TYPE}"),
        (gc_brstm, X.HCA, ct.convert_options(X.BRSTM), N.VGB_E_ARG, f"file 0: in_type 3 {X.MSG_IN_TYPE}"),
        (gc_brstm, 14, ct.convert_options(X.ADX), N.VGB_E_ARG, f"file 0: in_type 14 {X.MSG_IN_TYPE}"),
        # 2. IDSP / HPS into GC-ADPCM: the rewrite before the read, even for a file the reader refuses
        (broken, X.IDSP, ct.convert_options(X.HPS), N.VGB_E_ARG, X.MSG_REWRITE),
        (broken, X.HPS, ct.convert_options(X.DSP), N.VGB_E_ARG, X.MSG_REWRITE),
        (broken, X.IDSP, ct.convert_options(X.BFSTM), N.VGB_E_ARG, X.MSG_REWRITE),
        # 3. the reader and the loop setting first (the NintendoWare codec is only known after the parse)
        (broken, X.IDSP, ct.convert_options(X.HCA), N.VGB_E_DATA, None),
        (broken, X.BRSTM, ct.convert_options(X.DSP), N.VGB_E_DATA, None),
        (gc_brstm, X.BRSTM, ct.convert_options(X.DSP, loop=(0, 10 ** 6)), N.VGB_E_ARG, LO.MSG_RANGE),
        (gc_brstm, X.BRSTM, ct.convert_options(X.IDSP, loop=(9, 8)), N.VGB_E_ARG, LO.MSG_ORDER),
        # 4. then a NintendoWare file in the target's codec
        (gc_brstm, X.BRSTM, ct.convert_options(X.DSP, loop=(0, 100)), N.VGB_E_ARG, X.MSG_REWRITE),
        (pcm16_bcstm, X.BCSTM, ct.convert_options(X.BCSTM, nw_codec_plus1=2), N.VGB_E_ARG, X.MSG_REWRITE),
        # 5. the target's refusals
        (pcm16_3ch, X.BCSTM, ct.convert_options(X.HPS), N.VGB_E_ARG, "HpsWriter writes the block headers of 4k + 3 channels"),
        (pcm16_bcstm, X.BCSTM, ct.convert_options(X.BRSTM, loop=(1001, 1001)), N.VGB_E_ARG, None),
        (pcm16_bcstm, X.BCSTM, ct.convert_options(X.HCA, loop=(1001, 1001)), None, None),
    ]
    for k, (img, t, opt, st, frag) in enumerate(cases):
        sizes, status, msgs = _sizing(vg, [img], [t], opt)
        assert status[0] != 0 and sizes == [0], (k, status, msgs)
        if st is not None:
            assert status[0] == st, (k, status, msgs)
        if frag is not None:
            assert frag in msgs[0] and msgs[0].startswith("file 0: "), (k, msgs)
        else:
            assert X.MSG_REWRITE not in msgs[0], (k, msgs)


def test_failed_files_leave_the_others_sized(vg, oracle):
    """One call over every source with rewrites and refusals among them: each file's size and status is its own."""
    from vgaudio_b200 import containers as ct

    srcs = X.sources(oracle)
    files = [f for _, f, _ in srcs] + [np.zeros(16, np.uint8)]
    types = [t for t, _, _ in srcs] + [X.BFWAV]
    opt = X.options(ct, X.BCSTM, X.PCM16, loop=(700, 1500))
    n = len(files)
    arrs = [np.ascontiguousarray(f, np.uint8) for f in files]
    ftab = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
    lens = (C.c_int64 * n)(*[a.size for a in arrs])
    sizes, st = (C.c_int64 * n)(), (C.c_int32 * n)()
    assert vg.lib.vgb_transcode_from_nw_batch(ftab, lens, (C.c_int32 * n)(*types), n, C.byref(opt), sizes, None, st, None, None) == 0
    one, one_st, _ = _sizing(vg, files, types, opt)
    assert list(sizes) == one and list(st) == one_st
    assert one_st[-1] != 0 and sum(s == 0 for s in one_st) >= n // 2


def test_call_level_refusals_write_nothing(vg, oracle):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    f = np.ascontiguousarray(X.sources(oracle)[0][1], np.uint8)
    ftab, lens, types = (C.c_void_p * 1)(f.ctypes.data), (C.c_int64 * 1)(f.size), (C.c_int32 * 1)(X.BRSTM)

    def call(options, n=1, **null):
        sizes, st = (C.c_int64 * 1)(-7), (C.c_int32 * 1)(-7)
        args = dict(files=ftab, lens=lens, types=types, opt=C.byref(options), sizes=sizes)
        args.update(null)
        rc = vg.lib.vgb_transcode_from_nw_batch(args["files"], args["lens"], args["types"], n, args["opt"], args["sizes"], None, st, None, None)
        return rc, sizes[0], st[0]

    for out_type in (0, 9, 13, -1):
        assert call(ct.convert_options(out_type)) == (N.VGB_E_ARG, -7, -7), out_type
        assert b"out_type" in vg.lib.vgb_last_error()
    bad_loop = ct.convert_options(X.HCA)
    bad_loop.loop_mode = 3
    assert call(bad_loop) == (N.VGB_E_ARG, -7, -7)
    assert b"loop_mode 3" in vg.lib.vgb_last_error()
    assert call(ct.convert_options(X.HCA), n=-1) == (N.VGB_E_ARG, -7, -7)
    for name in ("files", "lens", "types", "opt", "sizes"):
        assert call(ct.convert_options(X.HCA), **{name: None}) == (N.VGB_E_ARG, -7, -7), name
    assert call(ct.convert_options(X.HCA), n=0) == (0, -7, -7)
    # the sizing pass itself
    assert call(ct.convert_options(X.HCA))[0] == 0


def test_python_keywords(vg):
    from vgaudio_b200 import _native as N
    from vgaudio_b200 import containers as ct

    params = list(inspect.signature(ct.transcode_from_nw_batch).parameters)
    assert params == ["files", "in_types", "options", "progress"]
    assert inspect.signature(ct.transcode_from_nw_batch).parameters["progress"].default is None
    assert len(N.SIGNATURES["vgb_transcode_from_nw_batch"][1]) == 10


def test_cli_nw_inputs_with_wav_is_a_usage_error(vg, tmp_path):
    r = subprocess.run([CLI, "-i", str(tmp_path), "-o", str(tmp_path / "out"), "--out-format", "wav", "--nw-inputs"], capture_output=True, text=True)
    assert r.returncode == 2, r.stdout + r.stderr
    assert "--nw-inputs takes --out-format dsp, adx, hca, brstm, bcstm, bfstm, idsp or hps" in r.stderr
    assert not (tmp_path / "out").exists()
