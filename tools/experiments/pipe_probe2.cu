// pipe_probe2.cu — what does a carry cost on the integer-multiply pipe of sm_90a?  (standalone: nvcc -o pipe_probe2 pipe_probe2.cu)
// Every variant keeps 8 independent 64-bit accumulators per thread in aligned register pairs (declared as 64-bit operands and split
// inside the asm block, so ptxas needs no repacking moves) and issues 8 multiply-accumulates per loop iteration:
//   A  mad.wide.u32                                   -> IMAD.WIDE.U32             (no carry at all)
//   B  mad.lo.cc / madc.hi.cc / addc cc               -> IMAD.WIDE.U32 (P out) + IADD3.X on the ALU pipe (carry-save accumulation)
//   C  two chains of four: carry out feeds carry in   -> IMAD.WIDE.U32.X           (what the CIOS rows of fp_ptx.cuh are made of)
//   D  add.cc / addc.cc chains only                   -> IADD3 / IADD3.X           (ALU pipe alone)
//   E  C and D interleaved                            -> do the two pipes overlap?
//   F  mad.lo.cc / madc.hi (carry out dropped)        -> control for B: is the P output itself what costs?
//   G / H  mad.lo.u32 / mad.hi.u32                    -> IMAD / IMAD.HI: one 32-bit result word per lane
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define ACC8 "+l"(c0), "+l"(c1), "+l"(c2), "+l"(c3), "+l"(c4), "+l"(c5), "+l"(c6), "+l"(c7)

template <int V>
__global__ void __launch_bounds__(256) k_probe(uint64_t* out, int iters) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t a = t * 2654435761u + 12345u, b = t ^ 0x9e3779b9u;
    uint64_t c0 = t, c1 = t + 1, c2 = t + 2, c3 = t + 3, c4 = t + 4, c5 = t + 5, c6 = t + 6, c7 = t + 7;
    uint32_t k0 = 0, k1 = 0, k2 = 0, k3 = 0, k4 = 0, k5 = 0, k6 = 0, k7 = 0;
#pragma unroll 1
    for (int i = 0; i < iters; ++i) {
        const uint32_t x0 = (uint32_t)c1, x1 = (uint32_t)c2, x2 = (uint32_t)c3, x3 = (uint32_t)c4, x4 = (uint32_t)c5, x5 = (uint32_t)c6, x6 = (uint32_t)c7, x7 = (uint32_t)c0 ^ k0;
        if (V == 0) {
            asm volatile("mad.wide.u32 %0, %8, %16, %0;\n\tmad.wide.u32 %1, %9, %16, %1;\n\tmad.wide.u32 %2, %10, %16, %2;\n\tmad.wide.u32 %3, %11, %16, %3;\n\t"
                         "mad.wide.u32 %4, %12, %16, %4;\n\tmad.wide.u32 %5, %13, %16, %5;\n\tmad.wide.u32 %6, %14, %16, %6;\n\tmad.wide.u32 %7, %15, %16, %7;"
                         : ACC8 : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(x4), "r"(x5), "r"(x6), "r"(x7), "r"(b));
        } else if (V == 1 || V == 5) {
#define ONE_B(ACC, K, X) \
            if (V == 1) asm volatile("{\n\t.reg .u32 lo, hi;\n\tmov.b64 {lo, hi}, %0;\n\tmad.lo.cc.u32 lo, %2, %3, lo;\n\tmadc.hi.cc.u32 hi, %2, %3, hi;\n\taddc.u32 %1, %1, 0;\n\tmov.b64 %0, {lo, hi};\n\t}" \
                                     : "+l"(ACC), "+r"(K) : "r"(X), "r"(b)); \
            else asm volatile("{\n\t.reg .u32 lo, hi;\n\tmov.b64 {lo, hi}, %0;\n\tmad.lo.cc.u32 lo, %2, %3, lo;\n\tmadc.hi.u32 hi, %2, %3, hi;\n\tmov.b64 %0, {lo, hi};\n\t}" \
                              : "+l"(ACC), "+r"(K) : "r"(X), "r"(b));
            ONE_B(c0, k0, x0) ONE_B(c1, k1, x1) ONE_B(c2, k2, x2) ONE_B(c3, k3, x3) ONE_B(c4, k4, x4) ONE_B(c5, k5, x5) ONE_B(c6, k6, x6) ONE_B(c7, k7, x7)
        } else if (V == 2 || V == 4) {
#define CHAIN4(A0, A1, A2, A3, X0, X1, X2, X3) \
            asm volatile("{\n\t.reg .u32 l0, h0, l1, h1, l2, h2, l3, h3;\n\t" \
                         "mov.b64 {l0, h0}, %0;\n\tmov.b64 {l1, h1}, %1;\n\tmov.b64 {l2, h2}, %2;\n\tmov.b64 {l3, h3}, %3;\n\t" \
                         "mad.lo.cc.u32 l0, %4, %8, l0;\n\tmadc.hi.cc.u32 h0, %4, %8, h0;\n\t" \
                         "madc.lo.cc.u32 l1, %5, %8, l1;\n\tmadc.hi.cc.u32 h1, %5, %8, h1;\n\t" \
                         "madc.lo.cc.u32 l2, %6, %8, l2;\n\tmadc.hi.cc.u32 h2, %6, %8, h2;\n\t" \
                         "madc.lo.cc.u32 l3, %7, %8, l3;\n\tmadc.hi.u32 h3, %7, %8, h3;\n\t" \
                         "mov.b64 %0, {l0, h0};\n\tmov.b64 %1, {l1, h1};\n\tmov.b64 %2, {l2, h2};\n\tmov.b64 %3, {l3, h3};\n\t}" \
                         : "+l"(A0), "+l"(A1), "+l"(A2), "+l"(A3) : "r"(X0), "r"(X1), "r"(X2), "r"(X3), "r"(b));
            CHAIN4(c0, c1, c2, c3, x0, x1, x2, x3) CHAIN4(c4, c5, c6, c7, x4, x5, x6, x7)
            if (V == 4) {
                asm volatile("add.cc.u32 %0, %0, %8;\n\taddc.cc.u32 %1, %1, %9;\n\taddc.cc.u32 %2, %2, %8;\n\taddc.cc.u32 %3, %3, %9;\n\t"
                             "addc.cc.u32 %4, %4, %8;\n\taddc.cc.u32 %5, %5, %9;\n\taddc.cc.u32 %6, %6, %8;\n\taddc.u32 %7, %7, %9;"
                             : "+r"(k0), "+r"(k1), "+r"(k2), "+r"(k3), "+r"(k4), "+r"(k5), "+r"(k6), "+r"(k7) : "r"(a), "r"(b));
            }
        } else if (V == 6 || V == 7) {
#define ONE_G(K, X) \
            if (V == 6) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(K) : "r"(X), "r"(b)); \
            else asm volatile("mad.hi.u32 %0, %1, %2, %0;" : "+r"(K) : "r"(X), "r"(b));
            const uint32_t y0 = k1, y1 = k2, y2 = k3, y3 = k4, y4 = k5, y5 = k6, y6 = k7, y7 = k0 ^ a;
            ONE_G(k0, y0) ONE_G(k1, y1) ONE_G(k2, y2) ONE_G(k3, y3) ONE_G(k4, y4) ONE_G(k5, y5) ONE_G(k6, y6) ONE_G(k7, y7)
        } else if (V == 3) {
            asm volatile("add.cc.u32 %0, %0, %8;\n\taddc.cc.u32 %1, %1, %9;\n\taddc.cc.u32 %2, %2, %8;\n\taddc.cc.u32 %3, %3, %9;\n\t"
                         "addc.cc.u32 %4, %4, %8;\n\taddc.cc.u32 %5, %5, %9;\n\taddc.cc.u32 %6, %6, %8;\n\taddc.u32 %7, %7, %9;"
                         : "+r"(k0), "+r"(k1), "+r"(k2), "+r"(k3), "+r"(k4), "+r"(k5), "+r"(k6), "+r"(k7) : "r"(a), "r"(b));
        }
    }
    out[t] = c0 ^ c1 ^ c2 ^ c3 ^ c4 ^ c5 ^ c6 ^ c7 ^ (uint64_t)(k0 ^ k1 ^ k2 ^ k3 ^ k4 ^ k5 ^ k6 ^ k7);
}

template <int V>
static void run(const char* name, int per_iter_mul, int per_iter_add) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int clock_khz = 1980000;
    cudaDeviceGetAttribute(&clock_khz, cudaDevAttrClockRate, 0);
    for (int bps = 2; bps <= 8; bps *= 2) {
        const int blocks = sms * bps, threads = 256, iters = 4000;
        uint64_t* d; cudaMalloc(&d, 8ull * blocks * threads);
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        float ms = 0;
        for (int rep = 0; rep < 2; ++rep) {
            cudaEventRecord(e0);
            k_probe<V><<<blocks, threads>>>(d, iters);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
        }
        cudaEventElapsedTime(&ms, e0, e1);
        const double clk = ms * 1e-3 * clock_khz * 1e3;
        const double warp_iters_per_smsp = (double)blocks * threads / 32 * iters / (sms * 4.0);
        printf("%-64s threads/SM=%5d  %8.3f ms  %6.2f SMSP-cycles per warp-iteration (%d mul + %d add instr)\n", name, threads * bps, ms, clk / warp_iters_per_smsp,
               per_iter_mul, per_iter_add);
        cudaFree(d); cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
}

int main() {
    run<0>("A mad.wide.u32 (IMAD.WIDE)", 8, 0);
    run<5>("F mad.lo.cc + madc.hi (carry inside the pair only)", 8, 0);
    run<1>("B mad.lo.cc + madc.hi.cc + addc (IMAD.WIDE P-out, IADD3.X count)", 8, 8);
    run<2>("C carry chains of four (IMAD.WIDE.X)", 8, 0);
    run<6>("G mad.lo.u32 (IMAD, 32-bit result)", 8, 0);
    run<7>("H mad.hi.u32 (IMAD.HI, 32-bit result)", 8, 0);
    run<3>("D add.cc / addc.cc chain of eight (IADD3.X)", 0, 8);
    run<4>("E C + D interleaved", 8, 8);
    return 0;
}
