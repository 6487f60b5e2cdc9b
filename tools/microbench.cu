// tools/microbench.cu — dependent-chain latencies on sm_90a (H100) for the ops the codec kernels' critical paths use.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -o tools/microbench tools/microbench.cu
// Default: one warp, one CTA; cycles per op = (clock after - clock before) / chain length.
// `microbench t`: issue throughput of the integer pipes with many warps and independent chains (run_tp below).
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

// ---- throughput mode: one 1024-thread CTA per SM (8 warps per sub-partition), 8 independent chains per thread, so
// neither latency nor a lone warp limits the rate; warp instructions per clock per sub-partition = 32 warps x iterations
// x instructions per iteration / (SM cycles x 4).  Each variant's loop body is checked in the SASS (cuobjdump -sass).
#define T_ITER 2048
#define T_CHAINS 8

__device__ __forceinline__ int t_imad(int a, int b, int c)
{
    int d;
    asm volatile("mad.lo.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

template <int OP>
__global__ void __launch_bounds__(1024, 1) throughput(long long *out, int seed)
{
    int a[T_CHAINS];
    long long w[T_CHAINS];
    const int b = seed * 3 + 1, c = seed ^ 0x55;
#pragma unroll
    for (int k = 0; k < T_CHAINS; k++) { a[k] = seed + threadIdx.x * 7 + k; w[k] = a[k]; }
    __syncthreads();
    const long long t0 = clock64();
#pragma unroll 4
    for (int i = 0; i < T_ITER; i++) {
#pragma unroll
        for (int k = 0; k < T_CHAINS; k++) {
            if (OP == 0) {  // 4 x IMAD
                a[k] = t_imad(a[k], b, c); a[k] = t_imad(a[k], b, k); a[k] = t_imad(a[k], c, b); a[k] = t_imad(a[k], b, i);
            }
            if (OP == 1)  // IMAD.WIDE x*x + 64-bit sum (as the encoder's squared error); x from the next chain's high word
            {
                const int x = (int)(w[(k + 1) % T_CHAINS] >> 32) ^ b;
                w[k] += (long long)x * x;
            }
            if (OP == 2) {  // LOP3, LEA.HI, SHF, VIMNMX, VIADDMNMX: 5 ALU ops (ptxas moves a lone add to IMAD.IADD)
                int x = a[k] ^ i;                                      // LOP3
                x = x + (int)((unsigned)x >> 31);                      // LEA.HI
                asm volatile("shr.s32 %0, %0, 3;" : "+r"(x));          // SHF
                x = min(x, c);                                         // VIMNMX
                a[k] = __viaddmin_s32_relu(x, 8, 15 + k);              // VIADDMNMX
            }
            if (OP == 3) {  // 2 x IMAD + 2 ALU (IADD3, VIADDMNMX)
                int x = t_imad(a[k], b, c);
                x = x + b + i;
                x = t_imad(x, c, k);
                a[k] = __viaddmin_s32_relu(x, 8, 15 + k);
            }
        }
    }
    const long long t1 = clock64();
    long long s = 0;
#pragma unroll
    for (int k = 0; k < T_CHAINS; k++) s += a[k] + w[k];
    if (threadIdx.x == 0) out[2 * blockIdx.x] = t1 - t0;
    if (s == 0x123456789LL) out[2 * blockIdx.x + 1] = s;  // keeps the chains alive
}

template <int OP>
void run_tp(const char *name, int ops_per_chain_iter)
{
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    long long *d_out;
    cudaMalloc(&d_out, 16ll * sms);
    throughput<OP><<<sms, 1024>>>(d_out, 3);
    throughput<OP><<<sms, 1024>>>(d_out, 3);
    long long *h = new long long[2 * sms];
    cudaMemcpy(h, d_out, 16ll * sms, cudaMemcpyDeviceToHost);
    double cyc = 0;
    for (int i = 0; i < sms; i++) cyc += (double)h[2 * i];
    cyc /= sms;
    const double warp_instr = 32.0 * T_ITER * T_CHAINS * ops_per_chain_iter;  // per CTA = per SM
    printf("%-44s %6.3f warp instr / clk / sub-partition (%d ops x %d chains per iter, %.0f cycles)\n", name,
           warp_instr / (cyc * 4.0), ops_per_chain_iter, T_CHAINS, cyc);
    delete[] h;
    cudaFree(d_out);
}

int main(int argc, char **argv)
{
    if (argc > 1 && argv[1][0] == 't') {
        run_tp<0>("IMAD only", 4);
        run_tp<1>("IMAD.WIDE + 64-bit sum (IMAD.WIDE only; +LOP3)", 1);
        run_tp<2>("ALU only (LOP3 LEA.HI SHF VIMNMX VIADDMNMX)", 5);
        run_tp<3>("IMAD / ALU 50/50 (IMAD IADD3 IMAD VIADDMNMX)", 4);
        return 0;
    }
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
