// rot_pipes.cu — which pipe should a 64-bit rotate of the Keccak round run on?
//
// The round is 122 LOP3 + 58 SHF per thread, all on the ALU pipe (16 lanes/clk/SMSP) while the FMA pipe idles.
// A rotate by r of the pair (lo, hi) is also  lo' = lo*2^r + hi32(hi*2^r),  hi' = hi*2^r + hi32(lo*2^r)  (the
// two summands never share a bit), i.e. IMAD.HI + IMAD + IMAD.WIDE (with a 64-bit addend) on the FMA pipe.  The multipliers come from
// constant memory so that ptxas cannot turn them back into shifts.  This bench times N permutations per thread
// with K of the 29 rotates of every round moved over (K = 0: the shipping code).
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o rot_pipes rot_pipes.cu && ./rot_pipes 64
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

__constant__ uint32_t POW2[32] = {
    1u << 0,  1u << 1,  1u << 2,  1u << 3,  1u << 4,  1u << 5,  1u << 6,  1u << 7,  1u << 8,  1u << 9,  1u << 10,
    1u << 11, 1u << 12, 1u << 13, 1u << 14, 1u << 15, 1u << 16, 1u << 17, 1u << 18, 1u << 19, 1u << 20, 1u << 21,
    1u << 22, 1u << 23, 1u << 24, 1u << 25, 1u << 26, 1u << 27, 1u << 28, 1u << 29, 1u << 30, 1u << 31};

__constant__ uint64_t RC[24] = {
    0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL,
    0x000000000000808bULL, 0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL,
    0x000000000000008aULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000aULL,
    0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL, 0x8000000000008003ULL,
    0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
    0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};

template <int N>
__device__ __forceinline__ uint64_t rot_alu(uint64_t x) {
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32), nlo, nhi;
    if constexpr (N == 32) { nlo = hi; nhi = lo; }
    else if constexpr (N < 32) { nhi = __funnelshift_l(lo, hi, N); nlo = __funnelshift_l(hi, lo, N); }
    else { nhi = __funnelshift_l(hi, lo, N - 32); nlo = __funnelshift_l(lo, hi, N - 32); }
    return ((uint64_t)nhi << 32) | nlo;
}

__constant__ uint32_t ONE = 1;

// MODE 1: c = (lo*m)>>32 : (lo*m)<<0 swapped into a 64-bit addend of hi*m  (ptxas: 2 IMAD.WIDE + IADD3 + IMAD.X)
// MODE 2: X = lo*m, Y = hi*m (both wide); lo' = X.lo*1 + Y.hi, hi' = Y.lo*1 + X.hi      (2 IMAD.WIDE + 2 IMAD)
// MODE 3: lo' = lo*m + hi32(hi*m), hi' = hi*m + hi32(lo*m)                            (2 IMAD.HI + 2 IMAD)
template <int N, int MODE>
__device__ __forceinline__ uint64_t rot_fma(uint64_t x) {
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    if constexpr (N >= 32) { uint32_t t = lo; lo = hi; hi = t; }
    constexpr int S = N & 31;
    if constexpr (S == 0) return ((uint64_t)hi << 32) | lo;
    uint32_t m = POW2[S];
    uint32_t nlo, nhi;
    if constexpr (MODE == 1) {
        uint32_t clo, chi;
        uint64_t c, w;
        asm("mul.hi.u32 %0, %1, %2;" : "=r"(clo) : "r"(lo), "r"(m));
        asm("mul.lo.u32 %0, %1, %2;" : "=r"(chi) : "r"(lo), "r"(m));
        asm("mov.b64 %0, {%1, %2};" : "=l"(c) : "r"(clo), "r"(chi));
        asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(w) : "r"(hi), "r"(m), "l"(c));
        nhi = (uint32_t)w;
        nlo = (uint32_t)(w >> 32);
    } else if constexpr (MODE == 2) {
        uint64_t X, Y;
        uint32_t one = ONE;
        asm("mul.wide.u32 %0, %1, %2;" : "=l"(X) : "r"(lo), "r"(m));
        asm("mul.wide.u32 %0, %1, %2;" : "=l"(Y) : "r"(hi), "r"(m));
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(nlo) : "r"((uint32_t)X), "r"(one), "r"((uint32_t)(Y >> 32)));
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(nhi) : "r"((uint32_t)Y), "r"(one), "r"((uint32_t)(X >> 32)));
    } else {
        uint32_t t, u;
        asm("mul.hi.u32 %0, %1, %2;" : "=r"(t) : "r"(lo), "r"(m));
        asm("mul.hi.u32 %0, %1, %2;" : "=r"(u) : "r"(hi), "r"(m));
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(nhi) : "r"(hi), "r"(m), "r"(t));
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(nlo) : "r"(lo), "r"(m), "r"(u));
    }
    return ((uint64_t)nhi << 32) | nlo;
}

// rotate number `I` (0..28) of the round goes to the FMA pipe when I < K
template <int N, int I, int K, int MODE>
__device__ __forceinline__ uint64_t rot_sel(uint64_t x) {
    if constexpr (I < K) return rot_fma<N, MODE>(x); else return rot_alu<N>(x);
}
#define rot(N, I) rot_sel<N, I, K, MODE>

template <int K, int MODE>
__device__ __forceinline__ void round_k(uint64_t (&a)[25], uint64_t rc) {
    uint64_t c0 = a[0] ^ a[5] ^ a[10] ^ a[15] ^ a[20];
    uint64_t c1 = a[1] ^ a[6] ^ a[11] ^ a[16] ^ a[21];
    uint64_t c2 = a[2] ^ a[7] ^ a[12] ^ a[17] ^ a[22];
    uint64_t c3 = a[3] ^ a[8] ^ a[13] ^ a[18] ^ a[23];
    uint64_t c4 = a[4] ^ a[9] ^ a[14] ^ a[19] ^ a[24];
    uint64_t r0 = rot(1, 24)(c1), r1 = rot(1, 25)(c2), r2 = rot(1, 26)(c3), r3 = rot(1, 27)(c4),
             r4 = rot(1, 28)(c0);
#define TH(i, cm, rp) (a[i] ^ cm ^ rp)
    uint64_t b00 = TH(0, c4, r0);
    uint64_t b10 = rot(1, 0)(TH(1, c0, r1));
    uint64_t b20 = rot(62, 1)(TH(2, c1, r2));
    uint64_t b05 = rot(28, 2)(TH(3, c2, r3));
    uint64_t b15 = rot(27, 3)(TH(4, c3, r4));
    uint64_t b16 = rot(36, 4)(TH(5, c4, r0));
    uint64_t b01 = rot(44, 5)(TH(6, c0, r1));
    uint64_t b11 = rot(6, 6)(TH(7, c1, r2));
    uint64_t b21 = rot(55, 7)(TH(8, c2, r3));
    uint64_t b06 = rot(20, 8)(TH(9, c3, r4));
    uint64_t b07 = rot(3, 9)(TH(10, c4, r0));
    uint64_t b17 = rot(10, 10)(TH(11, c0, r1));
    uint64_t b02 = rot(43, 11)(TH(12, c1, r2));
    uint64_t b12 = rot(25, 12)(TH(13, c2, r3));
    uint64_t b22 = rot(39, 13)(TH(14, c3, r4));
    uint64_t b23 = rot(41, 14)(TH(15, c4, r0));
    uint64_t b08 = rot(45, 15)(TH(16, c0, r1));
    uint64_t b18 = rot(15, 16)(TH(17, c1, r2));
    uint64_t b03 = rot(21, 17)(TH(18, c2, r3));
    uint64_t b13 = rot(8, 18)(TH(19, c3, r4));
    uint64_t b14 = rot(18, 19)(TH(20, c4, r0));
    uint64_t b24 = rot(2, 20)(TH(21, c0, r1));
    uint64_t b09 = rot(61, 21)(TH(22, c1, r2));
    uint64_t b19 = rot(56, 22)(TH(23, c2, r3));
    uint64_t b04 = rot(14, 23)(TH(24, c3, r4));
#undef TH
    a[0] = b00 ^ (~b01 & b02) ^ rc;  a[1] = b01 ^ (~b02 & b03);  a[2] = b02 ^ (~b03 & b04);
    a[3] = b03 ^ (~b04 & b00);       a[4] = b04 ^ (~b00 & b01);
    a[5] = b05 ^ (~b06 & b07);  a[6] = b06 ^ (~b07 & b08);  a[7] = b07 ^ (~b08 & b09);
    a[8] = b08 ^ (~b09 & b05);  a[9] = b09 ^ (~b05 & b06);
    a[10] = b10 ^ (~b11 & b12); a[11] = b11 ^ (~b12 & b13); a[12] = b12 ^ (~b13 & b14);
    a[13] = b13 ^ (~b14 & b10); a[14] = b14 ^ (~b10 & b11);
    a[15] = b15 ^ (~b16 & b17); a[16] = b16 ^ (~b17 & b18); a[17] = b17 ^ (~b18 & b19);
    a[18] = b18 ^ (~b19 & b15); a[19] = b19 ^ (~b15 & b16);
    a[20] = b20 ^ (~b21 & b22); a[21] = b21 ^ (~b22 & b23); a[22] = b22 ^ (~b23 & b24);
    a[23] = b23 ^ (~b24 & b20); a[24] = b24 ^ (~b20 & b21);
}

template <int K, int MODE>
__global__ void __launch_bounds__(128) perm_kernel(uint64_t *out, int iters) {
    uint64_t a[25];
    uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
#pragma unroll
    for (int i = 0; i < 25; i++) a[i] = t * 0x9E3779B97F4A7C15ULL + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll 1
        for (int r = 0; r < 24; r++) round_k<K, MODE>(a, RC[r]);
    }
    uint64_t x = 0;
#pragma unroll
    for (int i = 0; i < 25; i++) x ^= a[i] * (2 * i + 1);
    out[t] = x;
}

template <int K, int MODE>
static void run(uint64_t *d_out, uint64_t *h_out, int blocks, int iters, uint64_t &sig, float &ms) {
    perm_kernel<K, MODE><<<blocks, 128>>>(d_out, iters);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0);
    for (int i = 0; i < 5; i++) perm_kernel<K, MODE><<<blocks, 128>>>(d_out, iters);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
    ms /= 5;
    cudaMemcpy(h_out, d_out, 1024 * 8, cudaMemcpyDeviceToHost);
    sig = 0;
    for (int i = 0; i < 1024; i++) sig = sig * 31 + h_out[i];
}

int main(int argc, char **argv) {
    int blocks = 132 * 16 * 4, iters = 64;  // 132 SMs (H100 SXM)
    if (argc > 1) iters = atoi(argv[1]);
    uint64_t *d_out, *h_out = (uint64_t *)malloc(1024 * 8);
    cudaMalloc(&d_out, (size_t)blocks * 128 * 8);
    double perms = (double)blocks * 128 * iters;
    uint64_t sig0 = 0, sig;
    float ms;
#define RUN(K, MODE)                                                                                             \
    run<K, MODE>(d_out, h_out, blocks, iters, sig, ms);                                                          \
    if (K == 0) sig0 = sig;                                                                                      \
    printf("{\"mode\": %d, \"K\": %d, \"ms\": %.3f, \"Gperm_s\": %.3f, \"same_result\": %s}\n", MODE, K, ms,      \
           perms / ms / 1e6, sig == sig0 ? "true" : "false");
    RUN(0, 1)
    RUN(8, 1) RUN(16, 1) RUN(24, 1) RUN(29, 1)
    RUN(8, 2) RUN(12, 2) RUN(16, 2) RUN(20, 2) RUN(24, 2) RUN(29, 2)
    RUN(8, 3) RUN(12, 3) RUN(16, 3) RUN(20, 3) RUN(24, 3) RUN(29, 3)
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("cuda error %s\n", cudaGetErrorString(e)); return 1; }
    return 0;
}
