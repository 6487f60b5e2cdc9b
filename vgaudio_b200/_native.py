"""ctypes binding of libvgaudio_b200.so (C ABI in include/vgaudio_b200.h).

The library is the product; this module only loads it and declares the signatures.  There is no Python or CPU
fallback: if the shared object is missing the import fails loudly, and if no CUDA device is usable every codec call
raises VgbError(VGB_E_CUDA).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvgaudio_b200.so")

VGB_OK, VGB_E_ARG, VGB_E_DATA, VGB_E_STATE, VGB_E_CUDA, VGB_E_NCCL, VGB_E_NOMEM = 0, -1, -2, -3, -4, -5, -6


class VgbGcParams(C.Structure):
    """Mirror of GcAdpcmParameters (Codecs/GcAdpcm/GcAdpcmParameters.cs:3-7)."""

    _fields_ = [("sample_count", C.c_int32), ("history1", C.c_int16), ("history2", C.c_int16)]


class VgbAdxParams(C.Structure):
    """Mirror of CriAdxParameters (Codecs/CriAdx/CriAdxParameters.cs:3-13)."""

    _fields_ = [("sample_rate", C.c_int32), ("highpass_frequency", C.c_int32), ("frame_size", C.c_int32),
                ("version", C.c_int32), ("history", C.c_int32), ("padding", C.c_int32), ("type", C.c_int32),
                ("filter", C.c_int32)]


class VgbHcaParams(C.Structure):
    """Mirror of CriHcaParameters (Codecs/CriHca/CriHcaParameters.cs:3-15)."""

    _fields_ = [(n, C.c_int32) for n in ("quality", "bitrate", "limit_bitrate", "channel_count", "sample_rate",
                                         "sample_count", "looping", "loop_start", "loop_end")]


class VgbGcTapParams(C.Structure):
    _fields_ = [("sample_count", C.c_int32), ("samples_per_seek_table_entry", C.c_int32), ("loop_start", C.c_int32)]


class VgbGcAlignParams(C.Structure):
    """GcAdpcmAlignment's constructor arguments (Formats/GcAdpcm/GcAdpcmAlignment.cs:20)."""

    _fields_ = [("multiple", C.c_int32), ("loop_start", C.c_int32), ("loop_end", C.c_int32)]


class VgbGcAlignment(C.Structure):
    _fields_ = [("alignment_needed", C.c_int32), ("loop_start_aligned", C.c_int32), ("sample_count_aligned", C.c_int32)]


class VgbHcaInfo(C.Structure):
    """The HcaInfo fields the codec uses (Codecs/CriHca/HcaInfo.cs:5-48)."""

    _fields_ = [(n, C.c_int32) for n in (
        "channel_count", "sample_rate", "sample_count", "frame_count", "inserted_samples", "appended_samples",
        "header_size", "frame_size", "min_resolution", "max_resolution", "track_count", "channel_config",
        "total_band_count", "base_band_count", "stereo_band_count", "hfr_band_count", "bands_per_hfr_group",
        "hfr_group_count", "bitrate", "looping", "loop_start_frame", "loop_end_frame", "pre_loop_samples",
        "post_loop_samples", "use_ath_curve")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}



class VgbWaveInfo(C.Structure):
    """WaveStructure (Containers/Wave/WaveStructure.cs) + the data chunk's place in the file."""

    _fields_ = [(n, C.c_int32) for n in ("channel_count", "sample_rate", "bits_per_sample", "sample_count", "looping",
                                         "loop_start", "loop_end", "reserved")] + [("data_offset", C.c_int64), ("data_size", C.c_int64)]


class VgbDspDesc(C.Structure):
    """What DspWriter reads from GcAdpcmFormat + DspConfiguration (Containers/Dsp/DspWriter.cs:17-36)."""

    _fields_ = [(n, C.c_int32) for n in ("channel_count", "sample_rate", "sample_count", "looping", "loop_start", "loop_end",
                                         "samples_per_interleave", "loop_point_alignment", "no_trim")]


DSP_MAX_CHANNELS = 64


class VgbDspInfo(C.Structure):
    """DspStructure (Containers/Dsp/DspStructure.cs)."""

    _fields_ = [(n, C.c_int32) for n in ("sample_count", "nibble_count", "sample_rate", "looping", "format", "start_address",
                                         "end_address", "current_address", "channel_count", "frames_per_interleave",
                                         "loop_start", "loop_end")] + [
        ("coefs", (C.c_int16 * 16) * DSP_MAX_CHANNELS), ("gain", C.c_int16 * DSP_MAX_CHANNELS),
        ("start_context", (C.c_int16 * 3) * DSP_MAX_CHANNELS), ("loop_context", (C.c_int16 * 3) * DSP_MAX_CHANNELS)]


class VgbAdxDesc(C.Structure):
    """What AdxWriter reads from CriAdxFormat + AdxConfiguration (Containers/Adx/AdxWriter.cs:18-55)."""

    _fields_ = [(n, C.c_int32) for n in ("channel_count", "sample_rate", "sample_count", "looping", "loop_start", "loop_end",
                                         "alignment_samples", "frame_size", "version", "type", "highpass_frequency",
                                         "encryption_type", "no_trim")]


class VgbAdxKey(C.Structure):
    _fields_ = [("seed", C.c_int32), ("mult", C.c_int32), ("inc", C.c_int32)]


class VgbAdxFoundKey(C.Structure):
    """One key of vgb_adx_find_keys: the key, its confidence pass's status, CriAdxKey.KeyCode, the summed byte counts
    (differing and compared, short and full) and the two confidences."""
    _fields_ = [("key", VgbAdxKey), ("status", C.c_int32), ("key_code", C.c_uint64), ("diff_short", C.c_int64),
                ("total_short", C.c_int64), ("diff_full", C.c_int64), ("total_full", C.c_int64),
                ("confidence_short", C.c_double), ("confidence_full", C.c_double)]


VGB_ADX_KEY_SKIPPED = 1
VGB_ADX_KEYS_ONE_FILE = 1
VGB_ADX_MAX_CHANNELS = 255
VGB_HCA_KEY_SKIPPED = 1     # vgb_hca_find_keys: "ciph" is not 56, not searched
VGB_HCA_KEY_NOT_FOUND = 2   # no listed key passes


class VgbAdxFileInfo(C.Structure):
    """AdxStructure as AdxReader leaves it (Containers/Adx/AdxStructure.cs), plus where the audio sits."""

    _fields_ = [(n, C.c_int32) for n in ("header_size", "type", "frame_size", "bit_depth", "channel_count", "sample_rate",
                                         "sample_count", "highpass_frequency", "version", "revision", "inserted_samples",
                                         "loop_count", "looping", "loop_type", "loop_start_sample", "loop_start_byte",
                                         "loop_end_sample", "loop_end_byte", "samples_per_frame", "reserved")] + [
        ("audio_offset", C.c_int64), ("audio_size", C.c_int64), ("history", (C.c_int16 * 2) * VGB_ADX_MAX_CHANNELS)]


VGB_NW_MAX_CHANNELS = 255


class VgbNwInfo(C.Structure):
    """BxstmStructure as BrstmReader / BCFstmReader leave it, reduced to what decoding needs (see the header)."""

    _fields_ = [(n, C.c_int32) for n in ("codec", "looping", "channel_count", "sample_rate", "loop_start", "sample_count",
                                         "interleave_size", "big_endian")] + [("version", C.c_uint32)] + [
        (n, C.c_int32) for n in ("seek_table", "region_count", "track_count", "adpcm_channel_count", "samples_per_seek_entry",
                                 "loop_start_unaligned", "loop_end_unaligned", "output_size", "reserved")] + [
        ("audio_offset", C.c_int64), ("audio_length", C.c_int64),
        ("coefs", (C.c_int16 * 16) * VGB_NW_MAX_CHANNELS), ("gain", C.c_int16 * VGB_NW_MAX_CHANNELS),
        ("start_context", (C.c_int16 * 3) * VGB_NW_MAX_CHANNELS), ("loop_context", (C.c_int16 * 3) * VGB_NW_MAX_CHANNELS)]


class VgbIdspInfo(C.Structure):
    """IdspStructure as IdspReader leaves it, with the region Stream.DeInterleave reads (see the header)."""

    _fields_ = [(n, C.c_int32) for n in ("channel_count", "sample_rate", "sample_count", "loop_start", "loop_end", "interleave_size",
                                         "header_size", "channel_info_size", "audio_data_offset", "audio_data_length",
                                         "looping", "interleave", "output_size", "reserved")] + [
        ("audio_offset", C.c_int64), ("audio_length", C.c_int64)] + [
        (n, C.c_int32 * VGB_NW_MAX_CHANNELS) for n in ("ch_sample_count", "ch_nibble_count", "ch_sample_rate", "ch_looping", "start_address",
                                      "end_address", "current_address")] + [
        ("coefs", (C.c_int16 * 16) * VGB_NW_MAX_CHANNELS), ("gain", C.c_int16 * VGB_NW_MAX_CHANNELS),
        ("start_context", (C.c_int16 * 3) * VGB_NW_MAX_CHANNELS), ("loop_context", (C.c_int16 * 3) * VGB_NW_MAX_CHANNELS)]


class VgbHpsInfo(C.Structure):
    """HpsStructure as HpsReader leaves it (see the header)."""

    _fields_ = [(n, C.c_int32) for n in ("sample_rate", "channel_count", "sample_count", "looping", "loop_start", "block_count",
                                         "first_block", "loop_block")] + [
        ("max_block_size", C.c_int32 * VGB_NW_MAX_CHANNELS), ("end_address", C.c_int32 * VGB_NW_MAX_CHANNELS), ("channel_audio_bytes", C.c_int64 * VGB_NW_MAX_CHANNELS),
        ("coefs", (C.c_int16 * 16) * VGB_NW_MAX_CHANNELS), ("gain", C.c_int16 * VGB_NW_MAX_CHANNELS),
        ("start_context", (C.c_int16 * 3) * VGB_NW_MAX_CHANNELS), ("loop_context", (C.c_int16 * 3) * VGB_NW_MAX_CHANNELS)]


class VgbHpsBlock(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("offset", "size", "final_nibble", "next_offset")]


class VgbConvertOptions(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("out_type", "no_trim", "dsp_samples_per_interleave", "dsp_loop_point_alignment",
                                         "adx_version", "adx_frame_size", "adx_type", "adx_filter_plus1",
                                         "adx_encryption_type", "adx_has_key", "adx_key_seed", "adx_key_mult", "adx_key_inc",
                                         "hca_quality", "hca_bitrate", "hca_limit_bitrate", "hca_key_type", "reserved")] + [
        ("hca_key_code", C.c_uint64), ("group_bytes", C.c_int64)] + [
        (n, C.c_int32) for n in ("nw_codec_plus1", "nw_endianness", "nw_loop_point_alignment", "nw_pad",
                                 "loop_mode", "loop_start", "loop_end", "loop_pad")]


VGB_LOOP_SET, VGB_LOOP_CLEAR = 1, 2  # vgb_convert_options.loop_mode (0 keeps every source's loop)


PROGRESS_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_int64)

# name -> (restype, argtypes); also the list tests/test_abi.py checks against include/vgaudio_b200.h
SIGNATURES = {
    "vgb_abi_version": (C.c_int32, []),
    "vgb_init": (C.c_int32, [C.c_int32, C.c_uint32]),
    "vgb_shutdown": (C.c_int32, []),
    "vgb_init_devices": (C.c_int32, [C.c_void_p, C.c_int32, C.c_uint32]),
    "vgb_device_count": (C.c_int32, []),
    "vgb_nccl_unique_id": (C.c_int32, [C.c_void_p]),
    "vgb_nccl_init": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32]),
    "vgb_nccl_shutdown": (C.c_int32, []),
    "vgb_nccl_version": (C.c_int32, []),
    "vgb_scatterv_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_gatherv_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_sendrecv_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_partition_lpt": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vgb_last_error": (C.c_char_p, []),
    "vgb_host_alloc": (C.c_int32, [C.POINTER(C.c_void_p), C.c_uint64]),
    "vgb_host_free": (C.c_int32, [C.c_void_p]),
    "vgb_kernel_launch_count": (C.c_int64, []),
    "vgb_gcadpcm_sample_count_to_byte_count": (C.c_int32, [C.c_int32]),
    "vgb_gcadpcm_byte_count_to_sample_count": (C.c_int32, [C.c_int32]),
    "vgb_gcadpcm_sample_count_to_nibble_count": (C.c_int32, [C.c_int32]),
    "vgb_gcadpcm_nibble_count_to_sample_count": (C.c_int32, [C.c_int32]),
    "vgb_gcadpcm_sample_to_nibble": (C.c_int32, [C.c_int32]),
    "vgb_gcadpcm_nibble_to_sample": (C.c_int32, [C.c_int32]),
    "vgb_gcadpcm_coefs_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_gcadpcm_encode_batch": (
        C.c_int32,
        [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
    ),
    "vgb_gcadpcm_decode_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_gcadpcm_encode_frames": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_gcadpcm_workspace_bytes": (C.c_uint64, [C.c_int64, C.c_int32]),
    "vgb_gcadpcm_encode_dev": (
        C.c_int32,
        [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
         C.c_void_p, C.c_uint64, C.c_void_p],
    ),
    "vgb_gcadpcm_coefs_dev": (
        C.c_int32,
        [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p],
    ),
    "vgb_gcadpcm_decode_dev": (
        C.c_int32,
        [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
         C.c_void_p],
    ),
    "vgb_gcadpcm_decode_dev_status": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_adx_encoded_byte_count": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32]),
    "vgb_adx_encode_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p]),
    "vgb_adx_calculate_coefficients": (C.c_int32, [C.c_int32, C.c_int32, C.c_void_p]),
    "vgb_adx_decode_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_adx_decode_workspace_bytes": (C.c_uint64, [C.c_void_p, C.c_void_p, C.c_int32]),
    "vgb_adx_decode_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_uint64, C.c_void_p]),
    "vgb_adx_decode_dev_status": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_adx_debug_decode_stats": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_adx_debug_encode_stats": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_adx_workspace_bytes": (C.c_uint64, [C.c_int64, C.c_int32]),
    "vgb_adx_encode_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_uint64, C.c_void_p]),
    "vgb_hca_workspace_bytes": (C.c_uint64, [C.c_int32]),
    "vgb_hca_encode_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_uint64, C.c_void_p]),
    "vgb_hca_encode_dev_status": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_mdct128_batch": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "vgb_imdct128_batch": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "vgb_hca_query": (C.c_int32, [C.c_void_p, C.c_void_p]),
    "vgb_hca_encode_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_hca_decode_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_hca_decode_workspace_bytes": (C.c_uint64, [C.c_void_p, C.c_int32]),
    "vgb_hca_decode_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_uint64, C.c_void_p]),
    "vgb_hca_decode_dev_status": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_gcadpcm_seek_entry_count": (C.c_int32, [C.c_int32, C.c_int32]),
    "vgb_gcadpcm_seek_context_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "vgb_gcadpcm_alignment": (C.c_int32, [C.c_void_p, C.c_void_p]),
    "vgb_gcadpcm_align_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "vgb_interleave_dev": (C.c_int32, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int64,
                                       C.c_int32, C.c_int64, C.c_void_p]),
    "vgb_deinterleave_dev": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int64,
                                         C.c_int32, C.c_int64, C.c_void_p]),
    "vgb_interleave": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "vgb_deinterleave": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "vgb_set_kernel_timing": (C.c_int32, [C.c_int32]),
    "vgb_last_kernel_ms": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_debug_last_timeline": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_debug_last_coefs_done": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_gcadpcm_debug_records": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "vgb_gcadpcm_debug_refine_trace": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                                   C.c_void_p]),
    "vgb_gcadpcm_debug_splice_stats": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_wave_parse": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p]),
    "vgb_wave_read_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_dsp_file_size": (C.c_int64, [C.c_void_p]),
    "vgb_dsp_write_batch": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_dsp_parse": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p]),
    "vgb_dsp_read_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_adx_key_from_code": (C.c_int32, [C.c_uint64, C.c_void_p]),
    "vgb_adx_key_from_string": (C.c_int32, [C.c_char_p, C.c_void_p]),
    "vgb_adx_file_size": (C.c_int64, [C.c_void_p]),
    "vgb_adx_write_batch": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_adx_crypt_batch": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32]),
    "vgb_adx_parse": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p]),
    "vgb_adx_find_keys": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_adx_debug_find_keys_box": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32] + [C.c_int32] * 7 +
                                    [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_adx_debug_key_search_stats": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_adx_key_load": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "vgb_hca_parse": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "vgb_hca_key_tables": (C.c_int32, [C.c_int32, C.c_uint64, C.c_void_p, C.c_void_p]),
    "vgb_hca_find_keys": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "vgb_hca_debug_key_outcomes": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vgb_hca_debug_key_search_stats": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_hca_crypt_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_uint64, C.c_int32]),
    "vgb_hca_write_batch": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_convert_debug_stage_ms": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_convert_dsp_to_wave_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_convert_hca_to_wave_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_convert_adx_to_wave_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_brstm_parse": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p]),
    "vgb_bcfstm_parse": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p]),
    "vgb_nw_file_parse": (C.c_int32, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    "vgb_convert_nw_to_wave_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_idsp_parse": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p]),
    "vgb_hps_parse": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32]),
    "vgb_convert_idsp_hps_to_wave_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                                       C.c_void_p]),
    "vgb_convert_to_wave_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_gcadpcm_debug_decode_stats": (C.c_int32, [C.c_void_p, C.c_int32]),
    "vgb_convert_wave_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p]),
    "vgb_transcode_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_transcode_nw_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_transcode_from_nw_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_rewrite_gc_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vgb_rewrite_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p]),
}


class VgbError(RuntimeError):
    """Raised for a non-zero status.  `.code` is the VGB_E_* value; the C# shim maps the same codes to
    ArgumentException / InvalidDataException / InvalidOperationException (INTEGRATION.md)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"vgaudio_b200 error {code}: {message}")
        self.code = code


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  vgaudio_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here means header and library disagree
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(status: int) -> None:
    if status != VGB_OK:
        raise VgbError(status, (lib.vgb_last_error() or b"").decode("utf-8", "replace"))
