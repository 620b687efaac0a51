// keccak_f1600.cuh — Keccak-f[1600] for sm_90a, one sponge per thread, state in registers.
//
// Why thread-per-message and not a warp-cooperative layout: the permutation is 122 LOP3 + 58 SHF per round
// on 32-bit halves (sm_90a SASS, tools/sass_count.py) (all on the ALU pipe: 64 lanes/clk/SM).  Spreading one state over 25 lanes of a warp turns
// every theta/pi/chi dependency into SHFL traffic (32 lanes/clk/SM, two SHFL per 64-bit lane) and idles 7/32
// lanes; it is ~5x slower than keeping the 25 lanes in registers.  The warp-shuffle formulation survives where latency, not
// throughput, is the bound: WarpKeccak in tk_warp.cuh (one warp per node for the sparse top levels of a trie and the dirty
// paths of an incremental update), measured against this one in DESIGN.md §5.
//
// What it computes: alloy-primitives `keccak256` (Keccak-256, rate 136, pad 0x01..0x80) as called from
// reth's KeccakKeyHasher (crates/trie/common/src/key.rs:4-18) and alloy-trie's RlpNode::from_rlp.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace b200 {

__constant__ uint64_t KECCAK_RC[24] = {
    0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL,
    0x000000000000808bULL, 0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL,
    0x000000000000008aULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000aULL,
    0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL, 0x8000000000008003ULL,
    0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
    0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};

template <int N>
__device__ __forceinline__ uint64_t rotl64(uint64_t x) {
    static_assert(N > 0 && N < 64, "rotation");
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    uint32_t nlo, nhi;
    if constexpr (N == 32) {
        nlo = hi;
        nhi = lo;
    } else if constexpr (N < 32) {
        nhi = __funnelshift_l(lo, hi, N);
        nlo = __funnelshift_l(hi, lo, N);
    } else {
        nhi = __funnelshift_l(hi, lo, N - 32);
        nlo = __funnelshift_l(lo, hi, N - 32);
    }
    return ((uint64_t)nhi << 32) | nlo;
}

// a ^ b ^ c as one three-input LOP3 (LUT 0x96) per 32-bit half.  Written out because ptxas for sm_90a re-factors
// theta: from `a[i] ^ c[x-1] ^ rotl1(c[x+1])` it hoists the common D[x] = c[x-1] ^ rotl1(c[x+1]) and then spends one
// two-input XOR per lane half on a[i] ^ D[x] (10 + 50 LOP3 per round instead of 50), and it splits the five-way
// column parities the same way.  Inline PTX is kept as written.  The asm is not volatile, so lanes whose result is
// dead (the last round of a squeeze) are still removed.  The plain C++ form serves host compilers (tools/emu) and
// rounds whose state holds compile-time zeros (PLAIN = true), which the compiler can only fold through plain XORs.
// One asm statement on 64-bit operands rather than one per half: with the latter, ptxas changed how it compiled
// unrelated code of the strip-based kernels (branch_kernel<128,16> and wavefront_thread_kernel<64> grew 4-5x).
template <bool PLAIN = false>
__device__ __forceinline__ uint64_t xor3(uint64_t a, uint64_t b, uint64_t c) {
#ifdef __CUDA_ARCH__
    if constexpr (!PLAIN) {
        uint64_t r;
        asm("{\n\t.reg .b32 al, ah, bl, bh, cl, ch, rl, rh;\n\t"
            "mov.b64 {al, ah}, %1;\n\tmov.b64 {bl, bh}, %2;\n\tmov.b64 {cl, ch}, %3;\n\t"
            "lop3.b32 rl, al, bl, cl, 0x96;\n\tlop3.b32 rh, ah, bh, ch, 0x96;\n\t"
            "mov.b64 %0, {rl, rh};\n\t}"
            : "=l"(r) : "l"(a), "l"(b), "l"(c));
        return r;
    }
#endif
    return a ^ b ^ c;
}

// One round: theta, rho, pi, chi, iota.  Written so that nothing moves: pi is pure renaming.  Per round on 32-bit
// halves: 20 LOP3 for the column parities, 50 for theta, 50 for chi, 1-2 for iota, 58 SHF for the rotations.
// PLAIN: see xor3 (the peeled first round of a single-block short message, where 20 lanes are zero).
template <bool PLAIN = false>
__device__ __forceinline__ void keccak_round(uint64_t (&a)[25], uint64_t rc) {
    uint64_t c0 = xor3<PLAIN>(xor3<PLAIN>(a[0], a[5], a[10]), a[15], a[20]);
    uint64_t c1 = xor3<PLAIN>(xor3<PLAIN>(a[1], a[6], a[11]), a[16], a[21]);
    uint64_t c2 = xor3<PLAIN>(xor3<PLAIN>(a[2], a[7], a[12]), a[17], a[22]);
    uint64_t c3 = xor3<PLAIN>(xor3<PLAIN>(a[3], a[8], a[13]), a[18], a[23]);
    uint64_t c4 = xor3<PLAIN>(xor3<PLAIN>(a[4], a[9], a[14]), a[19], a[24]);
    // d[x] = c[x-1] ^ rotl(c[x+1],1); folded into the 3-input xor below so that theta costs one LOP3 per half
    uint64_t r0 = rotl64<1>(c1), r1 = rotl64<1>(c2), r2 = rotl64<1>(c3), r3 = rotl64<1>(c4), r4 = rotl64<1>(c0);
#define TH(i, cm, rp) xor3<PLAIN>(a[i], cm, rp)
    uint64_t b00 = TH(0, c4, r0);
    uint64_t b10 = rotl64<1>(TH(1, c0, r1));
    uint64_t b20 = rotl64<62>(TH(2, c1, r2));
    uint64_t b05 = rotl64<28>(TH(3, c2, r3));
    uint64_t b15 = rotl64<27>(TH(4, c3, r4));
    uint64_t b16 = rotl64<36>(TH(5, c4, r0));
    uint64_t b01 = rotl64<44>(TH(6, c0, r1));
    uint64_t b11 = rotl64<6>(TH(7, c1, r2));
    uint64_t b21 = rotl64<55>(TH(8, c2, r3));
    uint64_t b06 = rotl64<20>(TH(9, c3, r4));
    uint64_t b07 = rotl64<3>(TH(10, c4, r0));
    uint64_t b17 = rotl64<10>(TH(11, c0, r1));
    uint64_t b02 = rotl64<43>(TH(12, c1, r2));
    uint64_t b12 = rotl64<25>(TH(13, c2, r3));
    uint64_t b22 = rotl64<39>(TH(14, c3, r4));
    uint64_t b23 = rotl64<41>(TH(15, c4, r0));
    uint64_t b08 = rotl64<45>(TH(16, c0, r1));
    uint64_t b18 = rotl64<15>(TH(17, c1, r2));
    uint64_t b03 = rotl64<21>(TH(18, c2, r3));
    uint64_t b13 = rotl64<8>(TH(19, c3, r4));
    uint64_t b14 = rotl64<18>(TH(20, c4, r0));
    uint64_t b24 = rotl64<2>(TH(21, c0, r1));
    uint64_t b09 = rotl64<61>(TH(22, c1, r2));
    uint64_t b19 = rotl64<56>(TH(23, c2, r3));
    uint64_t b04 = rotl64<14>(TH(24, c3, r4));
#undef TH
    a[0] = b00 ^ (~b01 & b02) ^ rc;
    a[1] = b01 ^ (~b02 & b03);
    a[2] = b02 ^ (~b03 & b04);
    a[3] = b03 ^ (~b04 & b00);
    a[4] = b04 ^ (~b00 & b01);
    a[5] = b05 ^ (~b06 & b07);
    a[6] = b06 ^ (~b07 & b08);
    a[7] = b07 ^ (~b08 & b09);
    a[8] = b08 ^ (~b09 & b05);
    a[9] = b09 ^ (~b05 & b06);
    a[10] = b10 ^ (~b11 & b12);
    a[11] = b11 ^ (~b12 & b13);
    a[12] = b12 ^ (~b13 & b14);
    a[13] = b13 ^ (~b14 & b10);
    a[14] = b14 ^ (~b10 & b11);
    a[15] = b15 ^ (~b16 & b17);
    a[16] = b16 ^ (~b17 & b18);
    a[17] = b17 ^ (~b18 & b19);
    a[18] = b18 ^ (~b19 & b15);
    a[19] = b19 ^ (~b15 & b16);
    a[20] = b20 ^ (~b21 & b22);
    a[21] = b21 ^ (~b22 & b23);
    a[22] = b22 ^ (~b23 & b24);
    a[23] = b23 ^ (~b24 & b20);
    a[24] = b24 ^ (~b20 & b21);
}

// Full permutation (state fully live afterwards: multi-block absorb).
__device__ __forceinline__ void keccak_f1600(uint64_t (&a)[25]) {
#pragma unroll 1
    for (int r = 0; r < 24; r++) keccak_round(a, KECCAK_RC[r]);
}

// Final permutation of a Keccak-256 squeeze: only lanes 0..3 are consumed, so the last round is peeled and
// the compiler drops the ~2/3 of it that feeds lanes 4..24.
__device__ __forceinline__ void keccak_f1600_final(uint64_t (&a)[25]) {
#pragma unroll 1
    for (int r = 0; r < 23; r++) keccak_round(a, KECCAK_RC[r]);
    keccak_round(a, 0x8000000080008008ULL);
}

// Rounds [R0, R1) of the permutation: lets a kernel interleave other work (the loads of its next item) between segments.
template <int R0, int R1>
__device__ __forceinline__ void keccak_rounds(uint64_t (&a)[25]) {
#pragma unroll 1
    for (int r = R0; r < R1; r++) keccak_round(a, KECCAK_RC[r]);
}

// Single-block message whose state is mostly compile-time zeros (a 20/32-byte key): round 0 is peeled too, and
// written with plain XORs, so that the compiler folds the XORs with the 20 zero lanes and the constant pad lanes.
// Rounds 1..22 stay a loop: unrolled in line with immediate round constants they are 2 % fewer ALU instructions
// (4141 against 4217 per digest) but ~67 KB of code, and keccak256_fixed32_kernel ran 14 % slower that way
// (3.41 against 3.91-3.98 G digests/s on one H100 SXM, 400 W), presumably limited by instruction fetch (not profiled).
__device__ __forceinline__ void keccak_f1600_sparse_final(uint64_t (&a)[25]) {
    keccak_round<true>(a, 0x0000000000000001ULL);
#pragma unroll 1
    for (int r = 1; r < 23; r++) keccak_round(a, KECCAK_RC[r]);
    keccak_round(a, 0x8000000080008008ULL);
}

}  // namespace b200
