// tools/gc_err_check.c — checks the squared-error sums of gc_encode.cu's hot loop on the CPU: for a pass of 14 samples
// with |miss| <= 65535, the float32 sum F of fmaf(m, m, F) stays within 2^16 of the exact sum E (the kernel relies on
// 14 * 2^11), and from F and lo = E mod 2^32 the kernel's two uses are exact:
//   the saturated 32-bit key   F < 2^31 ? min(lo, 2^27 - 1) : 2^27 - 1   ==  min(E, 2^27 - 1)
//   the 64-bit error           (uint64)F + (int32)(lo - (uint32)F)      ==  E
// Sequences: every constant sequence, a beam search for the largest drift in each direction (each step tries every
// |m| in 0..65535 and keeps the widest drifts), sequences that cross 2^31 and every 2^32 * k, and 2e7 random ones.
// Build/run: gcc -O2 -ffp-contract=off -o /tmp/ec tools/gc_err_check.c -lm && /tmp/ec   (exit code 0 = all hold)
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define N 14
#define SAT ((1u << 27) - 1)
#define BOUND (14.0 * 2048.0)  // 14 roundings of at most half an ulp below 2^36
#define BEAM 48

static long bad = 0;
static double worst = 0;

static void check(float f, uint64_t e)
{
    const uint32_t lo = (uint32_t)e;
    const double d = (double)f - (double)e;
    if (fabs(d) > worst) worst = fabs(d);
    const uint64_t fi = (uint64_t)f;
    const uint32_t key = f < 2147483648.0f ? (lo < SAT ? lo : SAT) : SAT;
    const uint32_t want = e < SAT ? (uint32_t)e : SAT;
    const uint64_t rebuilt = fi + (uint64_t)(int64_t)(int32_t)(lo - (uint32_t)fi);
    if (fabs(d) > BOUND || (double)fi != (double)f || key != want || rebuilt != e) {
        if (bad++ < 10) printf("mismatch: F=%.1f E=%llu key=%u want=%u rebuilt=%llu\n", (double)f, (unsigned long long)e, key,
                               want, (unsigned long long)rebuilt);
    }
}

static void run(const uint32_t *m)
{
    float f = 0.0f;
    uint64_t e = 0;
    for (int s = 0; s < N; s++) {
        const float mf = (float)m[s];
        f = fmaf(mf, mf, f);
        e += (uint64_t)m[s] * m[s];
        check(f, e);  // every prefix is a shorter pass (the last frame of a channel)
    }
}

typedef struct { float f; uint64_t e; double d; } State;

static int by_d_desc(const void *a, const void *b)
{
    const double x = ((const State *)a)->d, y = ((const State *)b)->d;
    return x < y ? 1 : (x > y ? -1 : 0);
}

// keep the BEAM states of largest sign * drift after every step
static void beam(int sign)
{
    static State cur[BEAM], next[BEAM * 65536];
    int n = 1;
    cur[0].f = 0.0f; cur[0].e = 0; cur[0].d = 0;
    for (int s = 0; s < N; s++) {
        int k = 0;
        for (int i = 0; i < n; i++)
            for (uint32_t m = 0; m < 65536; m++) {
                const float mf = (float)m;
                State t;
                t.f = fmaf(mf, mf, cur[i].f);
                t.e = cur[i].e + (uint64_t)m * m;
                t.d = sign * ((double)t.f - (double)t.e);
                check(t.f, t.e);
                next[k++] = t;
            }
        qsort(next, k, sizeof(State), by_d_desc);
        n = k < BEAM ? k : BEAM;
        memcpy(cur, next, n * sizeof(State));
        printf("beam %+d step %2d: drift %.0f\n", sign, s + 1, cur[0].d);
    }
}

int main(void)
{
    uint32_t m[N];
    for (uint32_t v = 0; v < 65536; v++) {
        for (int s = 0; s < N; s++) m[s] = v;
        run(m);
    }
    beam(+1);
    beam(-1);
    // sums that end at or next to 2^31 and 2^32 * k (greedy: the largest square that fits, sample by sample)
    for (int k = 0; k <= 13; k++)
        for (int delta = -3; delta <= 3; delta++) {
            const int64_t target = (k == 0 ? (1ll << 31) : (int64_t)k << 32) + delta;
            uint64_t e = 0;
            for (int s = 0; s < N; s++) {
                const int64_t rest = target - (int64_t)e;
                uint32_t v = rest > 0 ? (uint32_t)sqrt((double)rest) : 0;
                if (v > 65535) v = 65535;
                while ((uint64_t)v * v > (uint64_t)(rest > 0 ? rest : 0)) v--;
                m[s] = v;
                e += (uint64_t)v * v;
            }
            run(m);
        }
    uint64_t x = 88172645463325252ull;
    for (long i = 0; i < 20000000; i++) {
        for (int s = 0; s < N; s++) {
            x ^= x << 13; x ^= x >> 7; x ^= x << 17;
            m[s] = (uint32_t)(x >> 48);
        }
        run(m);
    }
    printf("largest |F - E| %.0f (bound %.0f), mismatches %ld\n", worst, BOUND, bad);
    return bad != 0;
}
