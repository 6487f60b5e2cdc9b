/*
 * oracle/gcalign.c — CPU ORACLE (test infrastructure, not product): GcAdpcmAlignment
 * (Formats/GcAdpcm/GcAdpcmAlignment.cs:20-63, paths relative to VGAudio's src/VGAudio/), restated line by line on top of
 * the oracle's decoder and encoder (gcadpcm.c), with Helpers.GetNextMultiple / LoopPointsAreAligned (Helpers.cs:71-83).
 * Pinning: GcAdpcmAlignmentTests.cs:13-108, replayed in tests/test_oracle_gc_alignment.py.
 * Built into libvgoracle.so with the rest of oracle/ (Makefile: every *.c); wrapped by oracle/pygcalign.py.
 */
#include "vgoracle.h"

#include <stdlib.h>
#include <string.h>

enum { FRAME_BYTES = 8, FRAME_SAMPLES = 14, FRAME_NIBBLES = 16 };

/* new GcAdpcmAlignment(multiple, loopStart, loopEnd, adpcm, coefs).  geom_out = AlignmentNeeded, LoopStartAligned,
 * SampleCountAligned (all 0 when no alignment is needed).  When it is needed, adpcm_aligned_out receives
 * SampleCountToByteCount(SampleCountAligned) bytes (AdpcmAligned) and pcm_aligned_out SampleCountAligned samples
 * (PcmAligned); either may be NULL.  adpcm_length < 0 asks for the geometry only (adpcm / coefs may then be NULL).
 * Returns 0; -1 where the reference throws an argument / overflow exception or its tail loop never ends (loopStart ==
 * loopEnd with a moving start), or adpcm_length is shorter than loopEnd samples; -2 where its first Decode throws
 * IndexOutOfRangeException (a frame header below loopEnd selects a predictor 8..15). */
int vgo_gc_align(int multiple, int loop_start, int loop_end, const uint8_t *adpcm, int adpcm_length, const int16_t coefs[16],
                 int32_t geom_out[3], uint8_t *adpcm_aligned_out, int16_t *pcm_aligned_out);

static int get_next_multiple(int value, int multiple) /* Helpers.cs:71-80 */
{
    if (multiple <= 0) return value;
    if (value % multiple == 0) return value;
    return value + multiple - value % multiple;
}

int vgo_gc_align(int multiple, int loop_start, int loop_end, const uint8_t *adpcm, int adpcm_length, const int16_t coefs[16],
                 int32_t geom_out[3], uint8_t *adpcm_aligned_out, int16_t *pcm_aligned_out)
{
    geom_out[0] = geom_out[1] = geom_out[2] = 0;
    if (multiple == -1 && loop_start == INT32_MIN) return -1; /* int.MinValue % -1: OverflowException */
    /* AlignmentNeeded = !Helpers.LoopPointsAreAligned (Helpers.cs:82-83) */
    int loop_points_are_aligned = !(multiple != 0 && (multiple == -1 ? 0 : loop_start % multiple) != 0);
    if (loop_points_are_aligned) return 0;                                 /* :27 */
    if (loop_start < 0 || loop_end < loop_start) return -1;                /* Array.Copy throws (:43, :50) */

    int loop_length = loop_end - loop_start;                               /* :29 */
    /* the same arithmetic without wrap-around: a wrapped SampleCountAligned or nibble count makes new byte[...] throw */
    int64_t aligned64 = multiple <= 0 || loop_start % multiple == 0 ? loop_start
                                                                      : (int64_t)loop_start + multiple - loop_start % multiple;
    int64_t count64 = (int64_t)loop_end + (aligned64 - loop_start);
    int64_t rest64 = count64 % FRAME_SAMPLES;
    if (count64 > INT32_MAX || FRAME_NIBBLES * (count64 / FRAME_SAMPLES) + (rest64 ? rest64 + 2 : 0) > INT32_MAX) return -1;
    int loop_start_aligned = get_next_multiple(loop_start, multiple);     /* :30 */
    int sample_count_aligned = loop_end + (loop_start_aligned - loop_start); /* :31 */

    int frames_to_keep = loop_end / FRAME_SAMPLES;                         /* :36-39 */
    int bytes_to_keep = frames_to_keep * FRAME_BYTES;
    int samples_to_keep = frames_to_keep * FRAME_SAMPLES;
    int samples_to_encode = sample_count_aligned - samples_to_keep;
    if (loop_length == 0 && loop_end - samples_to_keep < samples_to_encode) return -1; /* :48 steps by 0 forever */
    geom_out[0] = 1;
    geom_out[1] = loop_start_aligned;
    geom_out[2] = sample_count_aligned;
    if (adpcm_length < 0) return 0;                                        /* geometry only */
    if (adpcm_length < vgo_gc_sample_count_to_byte_count(loop_end)) return -1;
    for (int f = 0; f < vgo_divide_by_round_up(loop_end, FRAME_SAMPLES); f++)
        if ((adpcm[f * FRAME_BYTES] >> 4) >= 8) return -2;                 /* coefs[predictor * 2] out of range */

    int16_t *pcm_aligned = calloc((size_t)sample_count_aligned + 1, sizeof(int16_t)); /* :34 */
    int16_t *old_pcm = calloc((size_t)loop_end + 1, sizeof(int16_t));
    vgo_gc_decode(adpcm, coefs, loop_end, 0, 0, old_pcm);                  /* :41-42 */
    memcpy(pcm_aligned, old_pcm, (size_t)loop_end * sizeof(int16_t));      /* :43 */
    int16_t *new_pcm = calloc((size_t)samples_to_encode + 1, sizeof(int16_t));

    memcpy(new_pcm, old_pcm + samples_to_keep, (size_t)(loop_end - samples_to_keep) * sizeof(int16_t)); /* :46 */

    for (int current_sample = loop_end - samples_to_keep; current_sample < samples_to_encode; current_sample += loop_length) {
        int n = samples_to_encode - current_sample < loop_length ? samples_to_encode - current_sample : loop_length;
        memcpy(new_pcm + current_sample, pcm_aligned + loop_start, (size_t)n * sizeof(int16_t)); /* :50 */
    }

    int16_t history1 = samples_to_keep < 1 ? 0 : old_pcm[samples_to_keep - 1]; /* :54-55 */
    int16_t history2 = samples_to_keep < 2 ? 0 : old_pcm[samples_to_keep - 2];

    int new_bytes = vgo_gc_sample_count_to_byte_count(samples_to_encode);
    uint8_t *new_adpcm = calloc((size_t)new_bytes + 1, 1);
    vgo_gc_encode(new_pcm, samples_to_encode, coefs, samples_to_encode, history1, history2, new_adpcm); /* :57 */
    if (adpcm_aligned_out) {
        memcpy(adpcm_aligned_out, adpcm, (size_t)bytes_to_keep);           /* :58 */
        memcpy(adpcm_aligned_out + bytes_to_keep, new_adpcm, (size_t)new_bytes); /* :59 */
    }

    int16_t *decoded_pcm = calloc((size_t)samples_to_encode + 1, sizeof(int16_t));
    vgo_gc_decode(new_adpcm, coefs, samples_to_encode, history1, history2, decoded_pcm); /* :61 */
    memcpy(pcm_aligned + samples_to_keep, decoded_pcm, (size_t)samples_to_encode * sizeof(int16_t)); /* :62 */
    if (pcm_aligned_out) memcpy(pcm_aligned_out, pcm_aligned, (size_t)sample_count_aligned * sizeof(int16_t));

    free(decoded_pcm);
    free(new_adpcm);
    free(new_pcm);
    free(old_pcm);
    free(pcm_aligned);
    return 0;
}
