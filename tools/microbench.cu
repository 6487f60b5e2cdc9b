// tools/microbench.cu — dependent-chain latencies on sm_90a (H100) for the ops the codec kernels' critical paths use.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -o tools/microbench tools/microbench.cu
// Default: one warp, one CTA; cycles per op = (clock after - clock before) / chain length.
// `microbench t`: issue throughput of the integer and FP32 pipes with many warps and independent chains (run_tp below).
// `microbench d`: a dependent DADD chain's cycles per add with 1, 2 or 4 chain warps per sub-partition beside 0, 2 or 6
// warps that issue independent DMUL / DADD pairs (run_dc below), and the fp64 rate those warps reach.
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
    unsigned lo[T_CHAINS];
    float f[T_CHAINS];
    const int b = seed * 3 + 1, c = seed ^ 0x55;
    const int xs = seed * 5 + 1000, xb = xs | 0x4B000000;
    const float fb = 1.0f + seed * 1e-6f, fc = 0.25f * seed;
#pragma unroll
    for (int k = 0; k < T_CHAINS; k++) { a[k] = seed + threadIdx.x * 7 + k; w[k] = a[k]; lo[k] = a[k]; f[k] = (float)a[k]; }
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
            // The encoder's per-sample squared error, around a stand-in for its recurrence (IMAD, then the clamp of the
            // reconstructed sample as VIADDMNMX.RELU) so that every iteration squares a new value.
            if (OP == 4 || OP == 5) {
                const int ob = __viaddmin_s32_relu(t_imad(a[k], b, c), 32768, 65535);
                a[k] = ob;
                if (OP == 4) {  // miss, then IMAD.WIDE with a 64-bit accumulate: 4 instructions
                    const int miss = t_imad(ob, -1, xs);
                    w[k] += (long long)miss * miss;
                } else {  // float image (LOP3), miss, 32-bit IMAD sum, FADD, FFMA: 7 instructions
                    const int obb = ob | 0x4B000000;
                    const int miss = t_imad(obb, -1, xb);
                    lo[k] = (unsigned)t_imad(miss, miss, (int)lo[k]);
                    const float mf = __fsub_rn(__int_as_float(xb), __int_as_float(obb));
                    f[k] = __fmaf_rn(mf, mf, f[k]);
                }
            }
            if (OP == 6) {  // 4 x IMAD + 4 x FFMA: do FP32 instructions take IMAD slots?
                a[k] = t_imad(a[k], b, c); f[k] = __fmaf_rn(f[k], fb, fc);
                a[k] = t_imad(a[k], b, k); f[k] = __fmaf_rn(f[k], fc, fb);
                a[k] = t_imad(a[k], c, b); f[k] = __fmaf_rn(f[k], fb, fb);
                a[k] = t_imad(a[k], b, i); f[k] = __fmaf_rn(f[k], fc, fc);
            }
            if (OP == 7) {  // 2 x IMAD + 2 ALU (LOP3, VIADDMNMX) + FADD + FFMA
                int x = t_imad(a[k], b, c) ^ i;
                x = t_imad(x, c, k);
                a[k] = __viaddmin_s32_relu(x, 8, 15 + k);
                const float g = __fadd_rn(f[k], fb);
                f[k] = __fmaf_rn(g, fc, fb);
            }
            if (OP == 8) {  // 4 x FFMA
                f[k] = __fmaf_rn(f[k], fb, fc); f[k] = __fmaf_rn(f[k], fc, fb);
                f[k] = __fmaf_rn(f[k], fb, fb); f[k] = __fmaf_rn(f[k], fc, fc);
            }
        }
    }
    const long long t1 = clock64();
    long long s = 0;
#pragma unroll
    for (int k = 0; k < T_CHAINS; k++) s += a[k] + w[k] + lo[k] + (long long)f[k];
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
    // cycles per body: sub-partition cycles per loop body of one chain of one warp (8 warps per sub-partition)
    printf("%-52s %6.3f warp instr / clk / sub-partition, %5.2f cycles per body (%d ops x %d chains per iter, %.0f cycles)\n",
           name, warp_instr / (cyc * 4.0), cyc * 4.0 / (32.0 * T_ITER * T_CHAINS), ops_per_chain_iter, T_CHAINS, cyc);
    delete[] h;
    cudaFree(d_out);
}


// ---- fp64 contention mode: CTA warp w sits on sub-partition w % 4 (its warp slot modulo 4); warps w / 4 < chains run
// one dependent DADD chain each, the other warps run 8 independent DMUL -> DADD chains (--fmad=false keeps them two
// instructions) until every chain warp is done.  Configurations above 8 warps per sub-partition use two CTAs per SM.
#define D_ITER 8192

__global__ void __launch_bounds__(1024) dadd_contention(long long *out, int chains, double seed)
{
    __shared__ int done;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) done = 0;
    __syncthreads();
    long long *o = out + ((long long)blockIdx.x * 32 + w) * 2;
    if ((w >> 2) < chains) {
        double d = seed + threadIdx.x;
        const long long t0 = clock64();
#pragma unroll 16
        for (int i = 0; i < D_ITER; i++) d = __dadd_rn(d, 1.5);
        const long long t1 = clock64();
        if (lane == 0) { o[0] = t1 - t0; o[1] = -1; atomicAdd(&done, 1); }
        if (d == 0.125) o[1] = (long long)d;
    } else {
        double x[8];
#pragma unroll
        for (int k = 0; k < 8; k++) x[k] = seed + k + threadIdx.x;
        const double m = 1.0000001, a = 0.5;
        long long n = 0;
        const long long t0 = clock64();
        while (*(volatile int *)&done < chains * 4) {
#pragma unroll 4
            for (int i = 0; i < 16; i++) {
#pragma unroll
                for (int k = 0; k < 8; k++) x[k] = __dadd_rn(__dmul_rn(x[k], m), a);
            }
            n += 16 * 8 * 2;
        }
        const long long t1 = clock64();
        double s = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) s += x[k];
        if (lane == 0) { o[0] = t1 - t0; o[1] = n; }
        if (s == 0.125) o[1] = 0;
    }
}

void run_dc(int chains, int noise)
{
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int ctas = chains + noise > 8 ? 2 : 1;       // warps per sub-partition per CTA: (chains + noise) / ctas
    const int c_per = chains / ctas, warps = (chains + noise) / ctas * 4;
    long long *d_out;
    const size_t bytes = 16ull * 32 * sms * ctas;
    cudaMalloc(&d_out, bytes);
    dadd_contention<<<sms * ctas, warps * 32>>>(d_out, c_per, 1.25);
    dadd_contention<<<sms * ctas, warps * 32>>>(d_out, c_per, 1.25);
    long long *h = new long long[bytes / 8];
    cudaMemcpy(h, d_out, bytes, cudaMemcpyDeviceToHost);
    double chain_cyc = 0, noise_ops = 0, noise_cyc = 0;
    int nc = 0, nn = 0;
    for (int b = 0; b < sms * ctas; b++)
        for (int w = 0; w < warps; w++) {
            const long long *o = h + ((long long)b * 32 + w) * 2;
            if (o[1] < 0) { chain_cyc += (double)o[0]; nc++; }
            else { noise_ops += (double)o[1]; noise_cyc += (double)o[0]; nn++; }
        }
    chain_cyc /= nc;
    // fp64 warp instructions per cycle per sub-partition issued by the other warps while the chains ran
    const double rate = nn ? noise_ops / (noise_cyc / nn) / (sms * 4.0) : 0.0;
    printf("chains/sub %d  other fp64 warps/sub %d  %6.2f cycles per dependent DADD  %5.3f other fp64 warp instr / clk / sub\n",
           chains, noise, chain_cyc / D_ITER, rate);
    delete[] h;
    cudaFree(d_out);
}

int main(int argc, char **argv)
{
    if (argc > 1 && argv[1][0] == 'd') {
        const int chains[3] = {1, 2, 4}, noise[3] = {0, 2, 6};
        for (int c : chains)
            for (int k : noise) run_dc(c, k);
        return 0;
    }
    if (argc > 1 && argv[1][0] == 't') {
        run_tp<0>("IMAD only", 4);
        run_tp<1>("IMAD.WIDE + 64-bit sum (IMAD.WIDE only; +LOP3)", 1);
        run_tp<2>("ALU only (LOP3 LEA.HI SHF VIMNMX VIADDMNMX)", 5);
        run_tp<3>("IMAD / ALU 50/50 (IMAD IADD3 IMAD VIADDMNMX)", 4);
        run_tp<4>("error, 64-bit (IMAD VIADDMNMX IMAD IMAD.WIDE)", 4);
        run_tp<5>("error, IMAD + FP32 (IMAD VIADDMNMX LOP3 2xIMAD FADD FFMA)", 7);
        run_tp<6>("IMAD / FFMA 50/50", 8);
        run_tp<7>("IMAD / ALU / FP32 (2 IMAD, LOP3 VIADDMNMX, FADD FFMA)", 6);
        run_tp<8>("FFMA only", 4);
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
