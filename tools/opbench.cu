// opbench.cu -- per-opcode issue rates of the integer pipes on this GPU (one SMSP's warp-instructions per clock), and which
// opcodes share a pipe with IMAD. Each kernel runs 8 independent register chains of one SASS opcode (checked with
// cuobjdump -sass) per thread, unrolled; MIX kernels interleave two opcodes 1:1.  Build: nvcc -arch=sm_90a -O3 -o opbench opbench.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <vector>
#include <string>

#define OP_LIST(X) \
    X(IMAD_REG) X(IMAD_IMM) X(IADD3) X(VIADD) X(LOP3) X(SHF) X(LEA) X(LEA_HI) X(I2IP) X(VIMNMX3) X(PRMT) X(IMAD_WIDE) X(IMAD_HI) \
    X(DP2A) X(DP4A) X(ISETP_SEL) X(IMAD_MOVISH) X(FFMA) \
    X(MIX_IMAD_IADD3) X(MIX_IMAD_SHF) X(MIX_IMAD_LEA) X(MIX_IMAD_I2IP) X(MIX_IMAD_VIMNMX3) X(MIX_IMAD_LOP3) X(MIX_IMAD_PRMT) \
    X(MIX_IADD3_SHF) X(MIX_IADD3_LEA) X(MIX_IMAD_FFMA) X(MIX_IADD3_FFMA) X(MIX_IMAD_DP2A) X(MIX_IADD3_DP2A) X(MIX3)

enum Op {
#define X(n) n,
    OP_LIST(X)
#undef X
    N_OPS
};
static const char *kNames[] = {
#define X(n) #n,
    OP_LIST(X)
#undef X
};

template <int OP>
__device__ __forceinline__ void step(int &x, int a, int b, int c) {
    if (OP == IMAD_REG) asm volatile("mad.lo.s32 %0, %0, %1, %2;" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == IMAD_IMM) asm volatile("mad.lo.s32 %0, %0, 277, %1;" : "+r"(x) : "r"(b));
    else if (OP == IADD3) asm volatile("{ .reg .s32 t; add.s32 t, %0, %1; add.s32 %0, t, %2; }" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == VIADD) asm volatile("add.s32 %0, %0, 12345;" : "+r"(x));
    else if (OP == LOP3) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == SHF) asm volatile("shf.r.wrap.b32 %0, %0, %1, 7;" : "+r"(x) : "r"(a));
    else if (OP == LEA) asm volatile("{ .reg .s32 t; shl.b32 t, %0, 3; add.s32 %0, t, %1; }" : "+r"(x) : "r"(a));
    else if (OP == LEA_HI) asm volatile("{ .reg .s32 t; shr.s32 t, %0, 2; add.s32 %0, t, %1; }" : "+r"(x) : "r"(a));
    else if (OP == I2IP) asm volatile("cvt.pack.sat.u8.s32.b32 %0, %0, %1, %2;" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == VIMNMX3) asm volatile("{ .reg .s32 t; max.s32 t, %0, %1; max.s32 %0, t, %2; }" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == PRMT) asm volatile("prmt.b32 %0, %0, %1, 0x3175;" : "+r"(x) : "r"(a));
    else if (OP == IMAD_WIDE) {
        long long t;
        asm volatile("mul.wide.s32 %0, %1, %2;" : "=l"(t) : "r"(x), "r"(a));
        asm volatile("{ .reg .b32 lo, hi; mov.b64 {lo, hi}, %1; xor.b32 %0, lo, hi; }" : "=r"(x) : "l"(t));
    } else if (OP == IMAD_HI) asm volatile("mul.hi.s32 %0, %0, %1;" : "+r"(x) : "r"(a));
    else if (OP == DP2A) asm volatile("dp2a.lo.s32.s32 %0, %0, %1, %2;" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == DP4A) asm volatile("dp4a.s32.s32 %0, %0, %1, %2;" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == ISETP_SEL) asm volatile("{ .reg .pred p; setp.lt.s32 p, %0, %1; selp.s32 %0, %2, %0, p; }" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == IMAD_MOVISH) asm volatile("mad.lo.s32 %0, %0, 1, %1;" : "+r"(x) : "r"(b));
    else if (OP == FFMA) asm volatile("{ .reg .f32 f; mov.b32 f, %0; fma.rn.f32 f, f, 0f3F800001, 0f3A000000; mov.b32 %0, f; }" : "+r"(x));
}

template <int OP>
__global__ void __launch_bounds__(256) bench(int *out, int iters, int a, int b) {
    int x[8];
#pragma unroll
    for (int i = 0; i < 8; i++) x[i] = threadIdx.x + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 8; u++) {
#pragma unroll
            for (int i = 0; i < 8; i++) {
                if (OP < MIX_IMAD_IADD3) step<OP>(x[i], a, b, 0);
                else if (OP == MIX_IMAD_IADD3) { if (i & 1) step<IMAD_IMM>(x[i], a, b, 0); else step<IADD3>(x[i], a, b, 0); }
                else if (OP == MIX_IMAD_SHF) { if (i & 1) step<IMAD_IMM>(x[i], a, b, 0); else step<SHF>(x[i], a, b, 0); }
                else if (OP == MIX_IMAD_LEA) { if (i & 1) step<IMAD_IMM>(x[i], a, b, 0); else step<LEA>(x[i], a, b, 0); }
                else if (OP == MIX_IMAD_I2IP) { if (i & 1) step<IMAD_IMM>(x[i], a, b, 0); else step<I2IP>(x[i], a, b, 0); }
                else if (OP == MIX_IMAD_VIMNMX3) { if (i & 1) step<IMAD_IMM>(x[i], a, b, 0); else step<VIMNMX3>(x[i], a, b, 0); }
                else if (OP == MIX_IMAD_LOP3) { if (i & 1) step<IMAD_IMM>(x[i], a, b, 0); else step<LOP3>(x[i], a, b, 0); }
                else if (OP == MIX_IMAD_PRMT) { if (i & 1) step<IMAD_IMM>(x[i], a, b, 0); else step<PRMT>(x[i], a, b, 0); }
                else if (OP == MIX_IADD3_SHF) { if (i & 1) step<IADD3>(x[i], a, b, 0); else step<SHF>(x[i], a, b, 0); }
                else if (OP == MIX_IADD3_LEA) { if (i & 1) step<IADD3>(x[i], a, b, 0); else step<LEA>(x[i], a, b, 0); }
                else if (OP == MIX_IMAD_FFMA) { if (i & 1) step<IMAD_IMM>(x[i], a, b, 0); else step<FFMA>(x[i], a, b, 0); }
                else if (OP == MIX_IADD3_FFMA) { if (i & 1) step<IADD3>(x[i], a, b, 0); else step<FFMA>(x[i], a, b, 0); }
                else if (OP == MIX_IMAD_DP2A) { if (i & 1) step<IMAD_IMM>(x[i], a, b, 0); else step<DP2A>(x[i], a, b, 0); }
                else if (OP == MIX_IADD3_DP2A) { if (i & 1) step<IADD3>(x[i], a, b, 0); else step<DP2A>(x[i], a, b, 0); }
                else if (OP == MIX3) { if (i % 3 == 0) step<IMAD_IMM>(x[i], a, b, 0); else if (i % 3 == 1) step<IADD3>(x[i], a, b, 0); else step<FFMA>(x[i], a, b, 0); }
            }
        }
    }
    int s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) s ^= x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int OP>
void run_one(int *buf, int grid, double clk_hz, int sms) {
    const int iters = 2048;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    bench<OP><<<grid, 256>>>(buf, iters / 8, 3, 7);
    cudaEventRecord(e0);
    bench<OP><<<grid, 256>>>(buf, iters, 3, 7);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    const double stmts = (double)grid * 256 / 32 * iters * 64.0;  // warp-level statements
    const double per_smsp_clk = stmts / (ms * 1e-3) / (sms * 4.0) / clk_hz;
    printf("%-18s %8.3f ms   %.3f statements/clk/SMSP\n", kNames[OP], ms, per_smsp_clk);
}

template <int OP>
struct Runner {
    static void go(int *buf, int grid, double clk, int sms) {
        run_one<OP>(buf, grid, clk, sms);
        Runner<OP + 1>::go(buf, grid, clk, sms);
    }
};
template <>
struct Runner<N_OPS> {
    static void go(int *, int, double, int) {}
};

int main() {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    int clk_khz = 0;
    cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    const int grid = prop.multiProcessorCount * 8;
    int *buf;
    cudaMalloc(&buf, sizeof(int) * (size_t)grid * 256);
    printf("%s, %d SMs, %d kHz (rates assume this clock)\n", prop.name, prop.multiProcessorCount, clk_khz);
    Runner<0>::go(buf, grid, clk_khz * 1e3, prop.multiProcessorCount);
    cudaFree(buf);
    return cudaGetLastError() != cudaSuccess;
}
