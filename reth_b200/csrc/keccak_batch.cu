// keccak_batch.cu — batched Keccak-256 of many short messages (the AccountHashing / StorageHashing inner
// loop: crates/stages/stages/src/stages/hashing_account.rs:192-211, hashing_storage.rs:121-148; also
// HashedPostState::from_bundle_state, crates/trie/common/src/hashed_state.rs:49-69).
//
// Layout: message i at in + i*stride, digest i at out + 32*i.  One message per thread, sponge state in
// registers, grid-stride loop over a persistent grid (SM count x resident CTAs).  Algorithmic traffic is
// msg_len + 32 bytes per digest; the kernel is ALU-bound (one Keccak-f = ~4.2k LOP3/SHF), not HBM-bound.
#include "keccak_f1600.cuh"
#include "kernels.h"

namespace b200 {

static __device__ __forceinline__ uint64_t pack64(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// 32-byte messages, 16-byte aligned rows (stride % 16 == 0): two LDG.128 per key, two STG.128 per digest.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) keccak256_fixed32_kernel(const uint8_t *__restrict__ in, uint32_t stride,
                                                                  uint64_t n, uint4 *__restrict__ out) {
    const uint64_t step = (uint64_t)gridDim.x * BLOCK;
    for (uint64_t i = (uint64_t)blockIdx.x * BLOCK + threadIdx.x; i < n; i += step) {
        const uint4 *p = reinterpret_cast<const uint4 *>(in + i * stride);
        uint4 k0 = __ldg(p), k1 = __ldg(p + 1);
        uint64_t a[25];
        a[0] = pack64(k0.x, k0.y);
        a[1] = pack64(k0.z, k0.w);
        a[2] = pack64(k1.x, k1.y);
        a[3] = pack64(k1.z, k1.w);
        a[4] = 0x01;  // pad10*1 start, message ends at byte 32
#pragma unroll
        for (int l = 5; l < 25; l++) a[l] = 0;
        a[16] = 0x8000000000000000ULL;  // last byte of the 136-byte rate block
        keccak_f1600_sparse_final(a);
        uint4 d0 = make_uint4((uint32_t)a[0], (uint32_t)(a[0] >> 32), (uint32_t)a[1], (uint32_t)(a[1] >> 32));
        uint4 d1 = make_uint4((uint32_t)a[2], (uint32_t)(a[2] >> 32), (uint32_t)a[3], (uint32_t)(a[3] >> 32));
        out[2 * i] = d0;
        out[2 * i + 1] = d1;
    }
}

// 20-byte messages (addresses), rows 4-byte aligned (stride % 4 == 0): five LDG.32.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) keccak256_fixed20_kernel(const uint8_t *__restrict__ in, uint32_t stride,
                                                                  uint64_t n, uint4 *__restrict__ out) {
    const uint64_t step = (uint64_t)gridDim.x * BLOCK;
    for (uint64_t i = (uint64_t)blockIdx.x * BLOCK + threadIdx.x; i < n; i += step) {
        const uint32_t *p = reinterpret_cast<const uint32_t *>(in + i * stride);
        uint32_t w0 = __ldg(p), w1 = __ldg(p + 1), w2 = __ldg(p + 2), w3 = __ldg(p + 3), w4 = __ldg(p + 4);
        uint64_t a[25];
        a[0] = pack64(w0, w1);
        a[1] = pack64(w2, w3);
        a[2] = pack64(w4, 0x01);  // pad byte right after the 20 message bytes
#pragma unroll
        for (int l = 3; l < 25; l++) a[l] = 0;
        a[16] = 0x8000000000000000ULL;
        keccak_f1600_sparse_final(a);
        uint4 d0 = make_uint4((uint32_t)a[0], (uint32_t)(a[0] >> 32), (uint32_t)a[1], (uint32_t)(a[1] >> 32));
        uint4 d1 = make_uint4((uint32_t)a[2], (uint32_t)(a[2] >> 32), (uint32_t)a[3], (uint32_t)(a[3] >> 32));
        out[2 * i] = d0;
        out[2 * i + 1] = d1;
    }
}

// Any length / alignment: message i = data[begin_i, end_i).  Byte loads; the slow general path
// (contract code hashing, odd strides).  FIXED: begin = i*stride, len = msg_len; else offsets[i..i+1].
template <int BLOCK, bool FIXED>
__global__ void __launch_bounds__(BLOCK) keccak256_bytes_kernel(const uint8_t *__restrict__ data,
                                                                const uint64_t *__restrict__ offsets,
                                                                uint32_t msg_len, uint32_t stride, uint64_t n,
                                                                uint8_t *__restrict__ out) {
    const uint64_t step = (uint64_t)gridDim.x * BLOCK;
    for (uint64_t i = (uint64_t)blockIdx.x * BLOCK + threadIdx.x; i < n; i += step) {
        uint64_t beg, len;
        if (FIXED) {
            beg = i * stride;
            len = msg_len;
        } else {
            beg = offsets[i];
            len = offsets[i + 1] - beg;
        }
        const uint8_t *m = data + beg;
        uint64_t a[25];
#pragma unroll
        for (int l = 0; l < 25; l++) a[l] = 0;
        uint64_t done = 0;
        for (;;) {
            uint64_t rem = len - done;
            bool last = rem < 136;
#pragma unroll
            for (int l = 0; l < 17; l++) {
                uint64_t w = 0;
#pragma unroll
                for (int b = 0; b < 8; b++) {
                    uint64_t idx = (uint64_t)(8 * l + b);
                    uint64_t byte = 0;
                    if (idx < rem) byte = m[done + idx];
                    else if (idx == rem) byte = 0x01;
                    w |= byte << (8 * b);
                }
                a[l] ^= w;
            }
            if (last) {
                a[16] ^= 0x8000000000000000ULL;
                break;
            }
            keccak_f1600(a);
            done += 136;
        }
        keccak_f1600_final(a);
        uint8_t *o = out + 32 * i;
        if ((reinterpret_cast<uintptr_t>(o) & 15) == 0) {
            uint4 *o4 = reinterpret_cast<uint4 *>(o);
            o4[0] = make_uint4((uint32_t)a[0], (uint32_t)(a[0] >> 32), (uint32_t)a[1], (uint32_t)(a[1] >> 32));
            o4[1] = make_uint4((uint32_t)a[2], (uint32_t)(a[2] >> 32), (uint32_t)a[3], (uint32_t)(a[3] >> 32));
        } else {
#pragma unroll
            for (int l = 0; l < 4; l++)
#pragma unroll
                for (int b = 0; b < 8; b++) o[8 * l + b] = (uint8_t)(a[l] >> (8 * b));
        }
    }
}

// ---------------------------------------------------------------------------------------------- launchers
static int g_sm_count = 0;
static int sm_count() {
    if (!g_sm_count) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
        if (g_sm_count <= 0) g_sm_count = 132;
    }
    return g_sm_count;
}

template <typename K>
static int persistent_grid(K kernel, int block, uint64_t n) {
    int per_sm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, 0);
    if (per_sm < 1) per_sm = 1;
    uint64_t want = (n + block - 1) / block;
    uint64_t cap = (uint64_t)sm_count() * per_sm;  // multiple of the SM count: one full wave, grid-stride inside
    return (int)(want < cap ? (want ? want : 1) : cap);
}

cudaError_t launch_keccak256_fixed(const void *d_in, uint32_t msg_len, uint32_t stride, uint64_t n, void *d_out,
                                   cudaStream_t s, unsigned *launches) {
    if (n == 0) return cudaSuccess;
    constexpr int BLOCK = 256;
    const uint8_t *in = static_cast<const uint8_t *>(d_in);
    uintptr_t addr = reinterpret_cast<uintptr_t>(d_in);
    bool out_aligned = (reinterpret_cast<uintptr_t>(d_out) & 15) == 0;
    if (msg_len == 32 && (stride & 15) == 0 && (addr & 15) == 0 && out_aligned) {
        auto k = keccak256_fixed32_kernel<BLOCK>;
        k<<<persistent_grid(k, BLOCK, n), BLOCK, 0, s>>>(in, stride, n, static_cast<uint4 *>(d_out));
    } else if (msg_len == 20 && (stride & 3) == 0 && (addr & 3) == 0 && out_aligned) {
        auto k = keccak256_fixed20_kernel<BLOCK>;
        k<<<persistent_grid(k, BLOCK, n), BLOCK, 0, s>>>(in, stride, n, static_cast<uint4 *>(d_out));
    } else {
        auto k = keccak256_bytes_kernel<BLOCK, true>;
        k<<<persistent_grid(k, BLOCK, n), BLOCK, 0, s>>>(in, nullptr, msg_len, stride, n,
                                                          static_cast<uint8_t *>(d_out));
    }
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_keccak256_var(const void *d_data, const void *d_offsets, uint64_t n, void *d_out, cudaStream_t s,
                                 unsigned *launches) {
    if (n == 0) return cudaSuccess;
    constexpr int BLOCK = 128;
    auto k = keccak256_bytes_kernel<BLOCK, false>;
    k<<<persistent_grid(k, BLOCK, n), BLOCK, 0, s>>>(static_cast<const uint8_t *>(d_data),
                                                      static_cast<const uint64_t *>(d_offsets), 0, 0, n,
                                                      static_cast<uint8_t *>(d_out));
    if (launches) ++*launches;
    return cudaGetLastError();
}

}  // namespace b200
