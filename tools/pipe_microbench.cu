// pipe_microbench.cu — issue-rate probes for the integer instructions Keccak-f is made of, on sm_90a.
// Answers: (1) LOP3 / SHF lanes per clock per SM (the ALU-pipe ceiling the keccak kernels are measured against),
// (2) whether 64-bit rotations expressed as IMAD.WIDE / IMAD.HI (FMA pipe) can be co-issued with LOP3 so that
// the rotation work leaves the ALU pipe.   Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 pipe_microbench.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__constant__ uint32_t MUL[8];

#define ACC 8

template <int MODE>
__global__ void probe(uint32_t *out, unsigned long long *cycles, int ITER) {
    uint32_t a[ACC], b[ACC];
    uint64_t w[ACC];
    uint32_t c[ACC];
    float fa[ACC], fb[ACC], fc = 1.0001f;
    for (int i = 0; i < ACC; i++) {
        a[i] = threadIdx.x * 2654435761u + i;
        b[i] = a[i] ^ 0x9e3779b9u;
        w[i] = ((uint64_t)a[i] << 32) | b[i];
        c[i] = a[i] + 7;
        fa[i] = (float)a[i];
        fb[i] = 1.0f + 1e-7f * i;
    }
    uint32_t m0 = MUL[0], m1 = MUL[1];
    __syncthreads();
    unsigned long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < ITER; it++) {
        // independent ops are grouped (8 accumulators) so that no instruction waits on its predecessor
#define L1(i) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b[i]), "r"(m0))
#define L2(i) asm volatile("lop3.b32 %0, %0, %1, %2, 0xd2;" : "+r"(b[i]) : "r"(a[i]), "r"(m1))
#define S1(i) asm volatile("shf.l.wrap.b32 %0, %0, %1, 7;" : "+r"(a[i]) : "r"(b[i]))
#define S2(i) asm volatile("shf.l.wrap.b32 %0, %0, %1, 13;" : "+r"(b[i]) : "r"(a[i]))
#define W1(i) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i]) : "r"(a[i]), "r"(m0))
#define W2(i) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(w[i]) : "r"(b[i]), "r"(m1))
#define H1(i) asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(m0))
#define H2(i) asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(b[i]) : "r"(m1))
#define M1(i) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(m0), "r"(b[i]))
#define M2(i) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(b[i]) : "r"(m1), "r"(a[i]))
#define M3(i) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(c[i]) : "r"(a[i]), "r"(m0))
#define P1(i) asm volatile("prmt.b32 %0, %0, %1, 0x2103;" : "+r"(a[i]) : "r"(b[i]))
#define P2(i) asm volatile("prmt.b32 %0, %0, %1, 0x1032;" : "+r"(b[i]) : "r"(a[i]))
#define A1(i) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(b[i]))
#define A2(i) asm volatile("add.u32 %0, %0, %1;" : "+r"(b[i]) : "r"(a[i]))
#define F1(i) asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(fa[i]) : "f"(fb[i]), "f"(fc))
#define R3a(i) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i]))
#define R3b(i) asm volatile("lop3.b32 %0, %0, %1, %2, 0xd2;" : "+r"(b[i]) : "r"(c[i]), "r"(a[i]))
#define R2a(i) asm volatile("lop3.b32 %0, %0, %1, %1, 0x96;" : "+r"(a[i]) : "r"(b[i]))
#define R2b(i) asm volatile("lop3.b32 %0, %0, %1, %1, 0xd2;" : "+r"(b[i]) : "r"(a[i]))
#define RIa(i) asm volatile("lop3.b32 %0, %0, %1, 0x5a5a1234, 0x96;" : "+r"(a[i]) : "r"(b[i]))
#define RIb(i) asm volatile("lop3.b32 %0, %0, %1, 0x0f0f4321, 0xd2;" : "+r"(b[i]) : "r"(a[i]))
#define X2a(i) asm volatile("xor.b32 %0, %0, %1;" : "+r"(a[i]) : "r"(b[i]))
#define X2b(i) asm volatile("xor.b32 %0, %0, %1;" : "+r"(b[i]) : "r"(a[i]))
#define H3(i) asm volatile("mul.hi.u32 %0, %1, %2;" : "=r"(c[i]) : "r"(a[i]), "r"(m0))
#define M4(i) asm volatile("mad.lo.u32 %0, %1, %2, %3;" : "=r"(c[i]) : "r"(b[i]), "r"(m1), "r"(c[i]))
#define ALL(X) X(0); X(1); X(2); X(3); X(4); X(5); X(6); X(7)
        if (MODE == 0) { ALL(L1); ALL(L2); }
        else if (MODE == 1) { ALL(S1); ALL(S2); }
        else if (MODE == 2) { ALL(W1); ALL(W2); }
        else if (MODE == 3) { ALL(L1); ALL(W1); ALL(L2); }
        else if (MODE == 4) { ALL(L1); ALL(S1); ALL(L2); }
        else if (MODE == 5) { ALL(H1); ALL(H2); }
        else if (MODE == 6) { ALL(M1); ALL(M2); }
        else if (MODE == 7) { ALL(L1); ALL(M3); ALL(L2); }
        else if (MODE == 8) { ALL(L1); ALL(W1); ALL(L2); ALL(W2); }
        else if (MODE == 9) { ALL(P1); ALL(P2); }
        else if (MODE == 10) { ALL(A1); ALL(A2); }
        else if (MODE == 11) { ALL(L1); ALL(M3); ALL(L2); ALL(M3); }
        else if (MODE == 12) { ALL(L1); ALL(F1); ALL(L2); ALL(F1); }
        else if (MODE == 13) { ALL(F1); ALL(F1); }
        else if (MODE == 14) { ALL(L1); ALL(S1); ALL(L2); ALL(M3); }
        else if (MODE == 15) { ALL(L1); ALL(H3); ALL(L2); }
        else if (MODE == 16) { ALL(L1); ALL(L2); ALL(H3); ALL(L1); ALL(L2); ALL(M4); }
        else if (MODE == 17) { ALL(L1); ALL(L2); ALL(H3); ALL(L1); ALL(M4); }
        else if (MODE == 20) { ALL(R3a); ALL(R3b); }
        else if (MODE == 21) { ALL(R2a); ALL(R2b); }
        else if (MODE == 22) { ALL(RIa); ALL(RIb); }
        else if (MODE == 23) { ALL(X2a); ALL(X2b); }
        else if (MODE == 24) { ALL(R3a); ALL(S1); ALL(R3b); }
    }
    unsigned long long t1 = clock64();
    uint32_t acc = 0;
    for (int i = 0; i < ACC; i++) acc ^= a[i] ^ b[i] ^ c[i] ^ __float_as_uint(fa[i]) ^ (uint32_t)w[i] ^ (uint32_t)(w[i] >> 32);
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int MODE>
void run(const char *name, int ops_per_acc, int sms, int warps_per_sm) {
    const int ITER = 1 << 18;  // tens of ms per launch: clocks are ramped, loop/launch overheads vanish
    int block = 256, blocks = sms * warps_per_sm * 32 / block;
    int resident = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, probe<MODE>, block, 0);
    if (resident * block < warps_per_sm * 32) {
        printf("%-28s warps/SM=%2d  skipped (only %d blocks resident)\n", name, warps_per_sm, resident);
        return;
    }
    uint32_t *out;
    unsigned long long *cyc;
    cudaMalloc(&out, (size_t)blocks * block * 4);
    cudaMalloc(&cyc, blocks * 8);
    probe<MODE><<<blocks, block>>>(out, cyc, ITER);
    probe<MODE><<<blocks, block>>>(out, cyc, ITER);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0);
    probe<MODE><<<blocks, block>>>(out, cyc, ITER);
    cudaEventRecord(e1);
    cudaDeviceSynchronize();
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    unsigned long long *h = new unsigned long long[blocks];
    cudaMemcpy(h, cyc, blocks * 8, cudaMemcpyDeviceToHost);
    double avg = 0;
    for (int i = 0; i < blocks; i++) avg += h[i];
    avg /= blocks;
    double ops_per_sm = (double)warps_per_sm * 32 * ITER * ACC * ops_per_acc;
    printf("%-28s warps/SM=%2d  %7.1f lane-ops/clk/SM by clock64 | %7.1f by events at 1.98 GHz  (%.3f ms, clock64 rate %.3f GHz)  err=%s\n",
           name, warps_per_sm, ops_per_sm / avg, ops_per_sm / (ms * 1e-3 * 1.98e9), ms, avg / (ms * 1e6),
           cudaGetErrorString(cudaGetLastError()));
    delete[] h;
    cudaFree(out);
    cudaFree(cyc);
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    uint32_t mul[8] = {8, 1u << 13, 3, 5, 7, 9, 11, 13};
    cudaMemcpyToSymbol(MUL, mul, sizeof mul);
    printf("SMs=%d\n", sms);
    for (int w : {8, 16, 24}) {
        run<0>("LOP3 (2 reg + uniform)", 2, sms, w);
        run<20>("LOP3 (3 distinct regs)", 2, sms, w);
        run<21>("LOP3 (2 distinct regs)", 2, sms, w);
        run<22>("LOP3 (2 regs + imm)", 2, sms, w);
        run<23>("XOR (2 regs)", 2, sms, w);
        run<24>("2 LOP3(3reg) + 1 SHF", 3, sms, w);
        run<1>("SHF", 2, sms, w);
        run<9>("PRMT", 2, sms, w);
        run<10>("IADD", 2, sms, w);
        run<6>("IMAD (mad.lo)", 2, sms, w);
        run<13>("FFMA", 2, sms, w);
        run<2>("IMAD.WIDE", 2, sms, w);
        run<5>("IMAD.HI (mul.hi)", 2, sms, w);
        run<4>("2 LOP3 + 1 SHF", 3, sms, w);
        run<7>("2 LOP3 + 1 IMAD", 3, sms, w);
        run<11>("2 LOP3 + 2 IMAD", 4, sms, w);
        run<12>("2 LOP3 + 2 FFMA", 4, sms, w);
        run<14>("2 LOP3 + 1 SHF + 1 IMAD", 4, sms, w);
        run<3>("2 LOP3 + 1 IMAD.WIDE", 3, sms, w);
        run<15>("2 LOP3 + 1 IMAD.HI", 3, sms, w);
        run<16>("4 LOP3 + 1 IMAD.HI + 1 IMAD", 6, sms, w);
        run<17>("3 LOP3 + 1 IMAD.HI + 1 IMAD", 5, sms, w);
    }
    return 0;
}
