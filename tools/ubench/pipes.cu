// tools/ubench/pipes.cu — issue-rate probes for the integer instructions fe_mul is made of (sm_90a).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipes pipes.cu ;  run: ./pipes
// Prints warp-instructions per clock per SM for: IMAD.WIDE.U32 (independent), IMAD.WIDE.U32.X carry chains,
// IADD3 (independent), IADD3.X carry chains, and a 1:1 mix.  Diagnostic only (DESIGN.md compute model).
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#define REP 64
template <int KIND> __global__ void k(uint32_t* out, uint32_t a0, uint32_t b0, int iters) {
    uint32_t a = a0 + threadIdx.x, b = b0 ^ blockIdx.x;
    uint32_t r[16];
#pragma unroll
    for (int i = 0; i < 16; i++) r[i] = a * (i + 3) + b;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < REP / 8; u++) {
            if (KIND == 0) {  // 8 independent IMAD.WIDE.U32 (64-bit accumulate, no carry)
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    uint64_t acc = ((uint64_t)r[2 * i + 1] << 32) | r[2 * i];
                    asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc) : "r"(a), "r"(b));
                    r[2 * i] = (uint32_t)acc; r[2 * i + 1] = (uint32_t)(acc >> 32);
                }
            } else if (KIND == 1) {  // two carry chains of 4 fused IMAD.WIDE.U32.X each (like one fe_mul row)
                asm volatile(
                    "mad.lo.cc.u32 %0, %16, %17, %0;\n\tmadc.hi.cc.u32 %1, %16, %17, %1;\n\t"
                    "madc.lo.cc.u32 %2, %16, %17, %2;\n\tmadc.hi.cc.u32 %3, %16, %17, %3;\n\t"
                    "madc.lo.cc.u32 %4, %16, %17, %4;\n\tmadc.hi.cc.u32 %5, %16, %17, %5;\n\t"
                    "madc.lo.cc.u32 %6, %16, %17, %6;\n\tmadc.hi.u32 %7, %16, %17, %7;\n\t"
                    "mad.lo.cc.u32 %8, %17, %16, %8;\n\tmadc.hi.cc.u32 %9, %17, %16, %9;\n\t"
                    "madc.lo.cc.u32 %10, %17, %16, %10;\n\tmadc.hi.cc.u32 %11, %17, %16, %11;\n\t"
                    "madc.lo.cc.u32 %12, %17, %16, %12;\n\tmadc.hi.cc.u32 %13, %17, %16, %13;\n\t"
                    "madc.lo.cc.u32 %14, %17, %16, %14;\n\tmadc.hi.u32 %15, %17, %16, %15;\n\t"
                    : "+r"(r[0]), "+r"(r[1]), "+r"(r[2]), "+r"(r[3]), "+r"(r[4]), "+r"(r[5]), "+r"(r[6]), "+r"(r[7]),
                      "+r"(r[8]), "+r"(r[9]), "+r"(r[10]), "+r"(r[11]), "+r"(r[12]), "+r"(r[13]), "+r"(r[14]), "+r"(r[15])
                    : "r"(a), "r"(b));
            } else if (KIND == 2) {  // 8 independent IADD3
#pragma unroll
                for (int i = 0; i < 8; i++) asm volatile("add.u32 %0, %0, %1;" : "+r"(r[i]) : "r"(a));
            } else if (KIND == 3) {  // one carry chain of 8 IADD3.X
                asm volatile(
                    "add.cc.u32 %0, %0, %8;\n\taddc.cc.u32 %1, %1, %8;\n\taddc.cc.u32 %2, %2, %8;\n\taddc.cc.u32 %3, %3, %8;\n\t"
                    "addc.cc.u32 %4, %4, %8;\n\taddc.cc.u32 %5, %5, %8;\n\taddc.cc.u32 %6, %6, %8;\n\taddc.u32 %7, %7, %8;\n\t"
                    : "+r"(r[0]), "+r"(r[1]), "+r"(r[2]), "+r"(r[3]), "+r"(r[4]), "+r"(r[5]), "+r"(r[6]), "+r"(r[7]) : "r"(b));
            } else if (KIND == 4) {  // 4 IMAD.WIDE + 4 IADD3, independent
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    uint64_t acc = ((uint64_t)r[2 * i + 1] << 32) | r[2 * i];
                    asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc) : "r"(a), "r"(b));
                    r[2 * i] = (uint32_t)acc; r[2 * i + 1] = (uint32_t)(acc >> 32);
                    asm volatile("add.u32 %0, %0, %1;" : "+r"(r[8 + i]) : "r"(a));
                }
            } else if (KIND == 5) {  // 8 independent 32-bit IMAD (lo)
#pragma unroll
                for (int i = 0; i < 8; i++) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(r[i]) : "r"(a), "r"(b));
            }
        }
    }
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) x ^= r[i];
    if (x == 0x12345) out[0] = x;
}

template <int KIND> double run(const char* name, int per_rep_instr, int warps_per_sm) {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    uint32_t* out; cudaMalloc(&out, 4);
    int iters = 2000, threads = 128, blocks = sms * warps_per_sm * 32 / threads;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float ms = 0;
    for (int rep = 0; rep < 2; rep++) {
        cudaEventRecord(e0); k<KIND><<<blocks, threads>>>(out, 12345, 67891, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
    }
    double winstr = (double)iters * (REP / 8) * per_rep_instr * (blocks * threads / 32);
    double per_clk_sm = winstr / (ms * 1e-3) / sms / (clk * 1e3);
    printf("%-34s warps/SM %2d  %.3f warp-instr/clk/SM (%.2f cycles per warp-instr per SMSP) [clk %d kHz]\n", name, warps_per_sm, per_clk_sm, 4.0 / per_clk_sm, clk);
    cudaFree(out);
    return per_clk_sm;
}

int main() {
    for (int w : {8, 32}) {
        run<0>("IMAD.WIDE.U32 independent", 8, w);
        run<1>("IMAD.WIDE.U32.X carry chains", 8, w);   // 16 PTX mads = 8 fused SASS
        run<5>("IMAD (32-bit) independent", 8, w);
        run<2>("IADD3 independent", 8, w);
        run<3>("IADD3.X carry chain", 8, w);
        run<4>("4 IMAD.WIDE + 4 IADD3 mix", 8, w);
    }
    return 0;
}
