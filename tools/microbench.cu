// tools/microbench.cu — dependent-chain latencies on sm_90a (H100) for the ops the codec kernels' critical paths use.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -o tools/microbench tools/microbench.cu
// One warp, one CTA; cycles per op = (clock after - clock before) / chain length.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define N_ITER 4096

template <int OP>
__global__ void chain(long long *out, int seed, double dseed, float fseed)
{
    int a = seed + threadIdx.x;
    int b = seed * 3 + 1;
    double d = dseed + threadIdx.x;
    float f = fseed + threadIdx.x;
    unsigned u = (unsigned)a;
    long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N_ITER; i++) {
        if (OP == 0) a = a * b + 7;                       // IMAD
        if (OP == 1) a = a + (a >> 3);                    // SHF + IADD
        if (OP == 2) a = min(max(a, -8), 7) + i;          // clamp (VIMNMX) + IADD
        if (OP == 3) d = __dadd_rn(d, 1.5);               // DADD
        if (OP == 4) d = __dmul_rn(d, 1.0000001);         // DMUL
        if (OP == 5) a = __float2int_rz(__int2float_rn(a) * 0.5f) + 1;   // I2F + FMUL + F2I
        if (OP == 6) a = __double2int_rz(__dadd_rn((double)__int2float_rn(a), 0.4999999)) ^ 1;  // literal quantiser chain
        if (OP == 7) a = __shfl_sync(0xFFFFFFFFu, a, (threadIdx.x + 1) & 31) + 1;   // SHFL
        if (OP == 8) a = (int)__reduce_min_sync(0xFFFFFFFFu, (unsigned)a) + threadIdx.x;  // REDUX
        if (OP == 9) a = (int)__ballot_sync(0xFFFFFFFFu, a & 1) + threadIdx.x;      // VOTE
        if (OP == 10) f = __fmaf_rn(f, 1.0001f, 0.5f);    // FFMA
        if (OP == 11) a = __float2int_ru(__int2float_rn(a)) + 1;  // I2F + F2I.CEIL
        if (OP == 12) u = __reduce_or_sync(0xFFFFFFFFu, u) + threadIdx.x;  // REDUX.OR
        if (OP == 13) a = abs(a) - 3;                     // IABS + IADD
        if (OP == 14) d = d / 1.0000001;                  // DDIV
        if (OP == 15) a = (a + ((a > 0) ? 5 : 6)) >> 1;   // compare-select add shift
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) { out[0] = t1 - t0; out[1] = a + (long long)d + (long long)f + u; }
}

template <int OP>
void run(const char *name, int ops_per_iter)
{
    long long *d_out, h[2];
    cudaMalloc(&d_out, 16);
    chain<OP><<<1, 32>>>(d_out, 3, 1.25, 0.75f);
    chain<OP><<<1, 32>>>(d_out, 3, 1.25, 0.75f);
    cudaMemcpy(h, d_out, 16, cudaMemcpyDeviceToHost);
    printf("%-44s %8.2f cycles/iter (%d dependent ops/iter)\n", name, (double)h[0] / N_ITER, ops_per_iter);
    cudaFree(d_out);
}

int main()
{
    run<0>("IMAD a=a*b+7", 1);
    run<1>("SHF+IADD a=a+(a>>3)", 2);
    run<2>("clamp4+IADD", 3);
    run<3>("DADD", 1);
    run<4>("DMUL", 1);
    run<5>("I2F+FMUL+F2I+IADD", 4);
    run<6>("I2F+F2D+DADD+D2I+LOP (literal quantiser)", 5);
    run<7>("SHFL+IADD", 2);
    run<8>("REDUX.MIN+IADD", 2);
    run<9>("VOTE.BALLOT+IADD", 2);
    run<10>("FFMA", 1);
    run<11>("I2F+F2I.CEIL+IADD", 3);
    run<12>("REDUX.OR+IADD", 2);
    run<13>("IABS+IADD", 2);
    run<14>("DDIV", 1);
    run<15>("ISETP+SEL+IADD+SHF", 4);
    return 0;
}
