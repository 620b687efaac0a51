// hash_sort.cu — "hash, then sort by digest": what AccountHashingStage / StorageHashingStage hand to the ETL
// collector (crates/stages/stages/src/stages/hashing_account.rs:192-230, crates/etl/src/lib.rs:31-60), done on
// the device: keccak of every key, then a radix sort of the 32-byte digests.
//
// Digests are keccak outputs: uniform.  (top 32 bits, index) pairs go through a four-pass radix sort; the few rows that
// agree in those bits (n^2 / 2^33 pairs) sit next to each other afterwards and the head of each such run orders it by the
// full 32 bytes, in place (fix_runs_kernel).  A last pass verifies the order of the full keys; only if it finds an unordered
// neighbour pair (runs longer than SORT_RUN_MAX: adversarial / equal-prefix input, not digests) the keys are re-sorted by a
// stable LSD over all four 64-bit words.  The composite 64-byte keys of the storage stage: the (few) address digests are sorted
// on their own, every entry takes the dense rank of its address, and the entries go through four passes over the top 32 bits
// of the slot digest plus ceil(log2(ranks)) bits of the rank (below).
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <cstring>
#include <mutex>

#include "engine.h"
#include "kernels.h"

using namespace b200;

namespace {

__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
}

// keys64[i] = big-endian word `w` (0 = most significant) of the digest at perm[i] (or i when perm is null)
__global__ void extract_word_kernel(const uint64_t *__restrict__ digests, const uint32_t *__restrict__ perm, int w,
                                    uint64_t n, uint64_t *__restrict__ keys64, uint32_t *__restrict__ idx_out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t src = perm ? perm[i] : i;
    keys64[i] = bswap64(digests[4 * src + w]);
    if (idx_out) idx_out[i] = (uint32_t)src;
}

__global__ void gather32_kernel(const uint4 *__restrict__ digests, const uint32_t *__restrict__ perm, uint64_t n,
                                uint4 *__restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t s = perm[i];
    out[2 * i] = digests[2 * s];
    out[2 * i + 1] = digests[2 * s + 1];
}

// flag = 1 if any neighbour pair is not strictly ascending (allow_equal: equal neighbours are fine — the caller dedups)
__global__ void check_sorted_kernel(const uint64_t *__restrict__ sorted, uint64_t n, int *__restrict__ flag, int allow_equal = 0) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 || i >= n) return;
    bool less = false, decided = false;
#pragma unroll
    for (int w = 0; w < 4; w++) {
        uint64_t a = bswap64(sorted[4 * (i - 1) + w]), b = bswap64(sorted[4 * i + w]);
        if (!decided && a != b) {
            decided = true;
            less = a < b;
        }
    }
    if (!less && !(allow_equal && !decided)) *flag = 1;  // equal keys also land here; harmless (the fallback is stable)
}

// keys32[i] = the four most significant bytes of digest i, idx[i] = i
__global__ void extract_top32_kernel(const uint32_t *__restrict__ digests, uint64_t n, uint32_t *__restrict__ keys32,
                                     uint32_t *__restrict__ idx_out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys32[i] = __byte_perm(digests[8 * i], 0, 0x0123);
    idx_out[i] = (uint32_t)i;
}

// After a stable sort on the top 32 bits: rows that agree in those bits form short runs (n^2 / 2^33 pairs among n uniform
// digests: 12 thousand at 10M, one row in a hundred at 100M).  The thread at the head of a run orders it by the full 32
// bytes, stably, rows and permutation entries alike.  Runs longer than SORT_RUN_MAX are left alone — check_sorted_kernel
// then sends the whole batch to the four-word LSD sort (keys with long common prefixes: not digests).
constexpr int SORT_RUN_MAX = 16;
__device__ __forceinline__ bool row_less(const uint32_t (&a)[8], const uint32_t (&b)[8]) {  // big-endian byte strings
#pragma unroll
    for (int w = 0; w < 8; w++) {
        uint32_t x = __byte_perm(a[w], 0, 0x0123), y = __byte_perm(b[w], 0, 0x0123);
        if (x != y) return x < y;
    }
    return false;
}
__global__ void fix_runs_kernel(uint32_t *__restrict__ sorted /* [n][8] */, uint32_t *__restrict__ perm, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i + 1 >= n) return;
    const uint32_t top = sorted[8 * i];
    if (sorted[8 * (i + 1)] != top || (i > 0 && sorted[8 * (i - 1)] == top)) return;  // not the head of a run of >= 2
    int len = 2;
    while (len <= SORT_RUN_MAX && i + len < n && sorted[8 * (i + len)] == top) len++;
    if (len > SORT_RUN_MAX) return;
    uint32_t row[SORT_RUN_MAX][8], src[SORT_RUN_MAX];
    for (int k = 0; k < len; k++) {
#pragma unroll
        for (int w = 0; w < 8; w++) row[k][w] = sorted[8 * (i + k) + w];
        src[k] = perm[i + k];
    }
    for (int k = 1; k < len; k++) {  // insertion sort: stable
        uint32_t r[8], sidx = src[k];
#pragma unroll
        for (int w = 0; w < 8; w++) r[w] = row[k][w];
        int j = k;
        while (j > 0 && row_less(r, row[j - 1])) {
#pragma unroll
            for (int w = 0; w < 8; w++) row[j][w] = row[j - 1][w];
            src[j] = src[j - 1];
            j--;
        }
#pragma unroll
        for (int w = 0; w < 8; w++) row[j][w] = r[w];
        src[j] = sidx;
    }
    for (int k = 0; k < len; k++) {
#pragma unroll
        for (int w = 0; w < 8; w++) sorted[8 * (i + k) + w] = row[k][w];
        perm[i + k] = src[k];
    }
}

inline unsigned nblk(uint64_t n) { return (unsigned)((n + 255) / 256); }

}  // namespace

// d_digests: [n][32] (input, unsorted) -> d_sorted [n][32], d_perm [n]
int32_t sort_digests_on_device(b200_ctx *c, const void *d_digests, uint64_t n, void *d_sorted, uint32_t *d_perm,
                               DevBuf &keys_a, DevBuf &keys_b, DevBuf &idx_a, DevBuf &flag, bool allow_equal) {
    if (n == 0) return B200_OK;
    if (n >= (1ull << 32)) return fail(c, B200_ERR_INVALID_ARG, "at most 2^32-1 keys per sort");
    cudaStream_t st = c->stream;
    TRY(ensure(c, keys_a, n * 8));
    TRY(ensure(c, keys_b, n * 8));
    TRY(ensure(c, idx_a, n * 4));
    TRY(ensure(c, flag, 16));
    uint64_t *ka = static_cast<uint64_t *>(keys_a.p), *kb = static_cast<uint64_t *>(keys_b.p);
    uint32_t *ia = static_cast<uint32_t *>(idx_a.p);
    const uint64_t *dig = static_cast<const uint64_t *>(d_digests);
    // fast path: four radix passes over the top 32 bits of every digest, then the short runs of equal tops ordered in place
    size_t temp = 0, temp32 = 0;
    uint32_t *ka32 = reinterpret_cast<uint32_t *>(ka), *kb32 = reinterpret_cast<uint32_t *>(kb);
    CU(cub::DeviceRadixSort::SortPairs(nullptr, temp, ka, kb, ia, d_perm, (int64_t)n, 0, 64, st));  // (the fallback's need)
    CU(cub::DeviceRadixSort::SortPairs(nullptr, temp32, ka32, kb32, ia, d_perm, (int64_t)n, 0, 32, st));
    TRY(ensure(c, c->cub_temp, std::max(temp, temp32)));
    extract_top32_kernel<<<nblk(n), 256, 0, st>>>(static_cast<const uint32_t *>(d_digests), n, ka32, ia);
    CU(cub::DeviceRadixSort::SortPairs(c->cub_temp.p, temp32, ka32, kb32, ia, d_perm, (int64_t)n, 0, 32, st));
    gather32_kernel<<<nblk(n), 256, 0, st>>>(static_cast<const uint4 *>(d_digests), d_perm, n,
                                             static_cast<uint4 *>(d_sorted));
    fix_runs_kernel<<<nblk(n), 256, 0, st>>>(static_cast<uint32_t *>(d_sorted), d_perm, n);
    CU(cudaMemsetAsync(flag.p, 0, 4, st));
    check_sorted_kernel<<<nblk(n), 256, 0, st>>>(static_cast<const uint64_t *>(d_sorted), n, static_cast<int *>(flag.p),
                                                 allow_equal ? 1 : 0);
    c->launches += 5;
    int *h_flag = reinterpret_cast<int *>(static_cast<uint8_t *>(c->pinned_small) + 3072);
    CU(cudaMemcpyAsync(h_flag, flag.p, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (*h_flag == 0) return B200_OK;
    // fallback: stable LSD over the four words, least significant first
    uint32_t *cur = nullptr;  // identity
    uint32_t *bufs[2] = {ia, d_perm};
    int which = 0;
    for (int w = 3; w >= 0; w--) {
        // keys of word w in the current order, then a stable sort carrying the source index
        uint32_t *idx_in = bufs[which], *idx_out = bufs[which ^ 1];
        extract_word_kernel<<<nblk(n), 256, 0, st>>>(dig, cur, w, n, ka, idx_in);
        CU(cub::DeviceRadixSort::SortPairs(c->cub_temp.p, temp, ka, kb, idx_in, idx_out, (int64_t)n, 0, 64, st));
        cur = idx_out;
        which ^= 1;
        c->launches += 2;
    }
    if (cur != d_perm) CU(cudaMemcpyAsync(d_perm, cur, n * 4, cudaMemcpyDeviceToDevice, st));
    gather32_kernel<<<nblk(n), 256, 0, st>>>(static_cast<const uint4 *>(d_digests), d_perm, n,
                                             static_cast<uint4 *>(d_sorted));
    c->launches++;
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------- composite keys (a3)
// StorageHashingStage (crates/stages/stages/src/stages/hashing_storage.rs:106-178) sorts by the 64-byte key
// keccak(address) || keccak(slot).  Element i belongs to address addr_index[i]; the address digest is computed
// once per address (the reference caches it across consecutive entries, :129-134).
namespace {

// big-endian word w (0..7) of the composite key of element src
__device__ __forceinline__ uint64_t composite_word(const uint64_t *__restrict__ ha, const uint32_t *__restrict__ addr_index,
                                                   const uint64_t *__restrict__ hs, uint64_t src, int w) {
    return bswap64(w < 4 ? ha[4 * (uint64_t)addr_index[src] + w] : hs[4 * src + (w - 4)]);
}

__global__ void extract_composite_kernel(const uint64_t *__restrict__ ha, const uint32_t *__restrict__ addr_index,
                                         const uint64_t *__restrict__ hs, const uint32_t *__restrict__ perm, int w, uint64_t n,
                                         uint64_t *__restrict__ keys64, uint32_t *__restrict__ idx_out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t src = perm ? perm[i] : i;
    keys64[i] = composite_word(ha, addr_index, hs, src, w);
    idx_out[i] = (uint32_t)src;
}

__global__ void gather_composite_kernel(const uint4 *__restrict__ ha, const uint32_t *__restrict__ addr_index,
                                        const uint4 *__restrict__ hs, const uint32_t *__restrict__ perm, uint64_t n,
                                        uint4 *__restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t s = perm[i], a = addr_index[s];
    out[4 * i] = ha[2 * a];
    out[4 * i + 1] = ha[2 * a + 1];
    out[4 * i + 2] = hs[2 * s];
    out[4 * i + 3] = hs[2 * s + 1];
}

// neighbours must be strictly ascending (a duplicate (address, slot) pair is reported separately)
__global__ void check_sorted_composite_kernel(const uint64_t *__restrict__ sorted, uint64_t n, int *__restrict__ flag,
                                              int allow_equal = 0) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 || i >= n) return;
    bool less = false, decided = false;
#pragma unroll
    for (int w = 0; w < 8; w++) {
        uint64_t a = bswap64(sorted[8 * (i - 1) + w]), b = bswap64(sorted[8 * i + w]);
        if (!decided && a != b) {
            decided = true;
            less = a < b;
        }
    }
    if (!decided) {
        if (!allow_equal) atomicMax(flag, 2);  // equal composite keys
    }
    else if (!less) atomicMax(flag, 1);     // out of order: the prefix passes were not enough
}

// ---- fast path of the composite sort: (dense rank of the address digest, top 32 bits of the slot digest)
// head[j] = 1 iff sorted address digest j differs from its predecessor (j = 0: 0), so that the inclusive sum is the dense rank
__global__ void addr_heads_kernel(const uint64_t *__restrict__ sorted_ha, uint32_t n_addr, uint32_t *__restrict__ head) {
    uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_addr) return;
    bool h = false;
    if (j > 0)
        for (int w = 0; w < 4; w++) h = h || sorted_ha[4 * (uint64_t)j + w] != sorted_ha[4 * (uint64_t)(j - 1) + w];
    head[j] = h ? 1u : 0u;
}
__global__ void addr_rank_scatter_kernel(const uint32_t *__restrict__ perm, const uint32_t *__restrict__ dense, uint32_t n_addr,
                                         uint32_t *__restrict__ rank) {
    uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n_addr) rank[perm[j]] = dense[j];
}
__global__ void extract_slot_top32_kernel(const uint32_t *__restrict__ hs, uint64_t n, uint32_t *__restrict__ keys32,
                                          uint32_t *__restrict__ idx_out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys32[i] = __byte_perm(hs[8 * i], 0, 0x0123);
    idx_out[i] = (uint32_t)i;
}
__global__ void extract_addr_rank_kernel(const uint32_t *__restrict__ addr_index, const uint32_t *__restrict__ rank,
                                         const uint32_t *__restrict__ order, uint64_t n, uint32_t *__restrict__ keys32) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keys32[i] = rank[addr_index[order[i]]];
}
// rows of 64 bytes that agree in the address digest and in the top 32 bits of the slot digest: ordered by the slot digest,
// in place, by the head of the run (fix_runs_kernel's job for the composite keys; longer runs are left to the fallback)
__global__ void fix_runs_composite_kernel(uint32_t *__restrict__ sorted /* [n][16] */, uint32_t *__restrict__ perm, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i + 1 >= n) return;
    auto same = [&](uint64_t x, uint64_t y) {  // address digest and slot top equal
        bool e = true;
#pragma unroll
        for (int w = 0; w < 9; w++) e = e && sorted[16 * x + w] == sorted[16 * y + w];
        return e;
    };
    if (!same(i, i + 1) || (i > 0 && same(i - 1, i))) return;
    int len = 2;
    while (len <= SORT_RUN_MAX && i + len < n && same(i, i + len)) len++;
    if (len > SORT_RUN_MAX) return;
    uint32_t row[SORT_RUN_MAX][8], src[SORT_RUN_MAX];  // the slot digests (the address part of the run is one value)
    for (int k = 0; k < len; k++) {
#pragma unroll
        for (int w = 0; w < 8; w++) row[k][w] = sorted[16 * (i + k) + 8 + w];
        src[k] = perm[i + k];
    }
    for (int k = 1; k < len; k++) {
        uint32_t r[8], sidx = src[k];
#pragma unroll
        for (int w = 0; w < 8; w++) r[w] = row[k][w];
        int j = k;
        while (j > 0 && row_less(r, row[j - 1])) {
#pragma unroll
            for (int w = 0; w < 8; w++) row[j][w] = row[j - 1][w];
            src[j] = src[j - 1];
            j--;
        }
#pragma unroll
        for (int w = 0; w < 8; w++) row[j][w] = r[w];
        src[j] = sidx;
    }
    for (int k = 0; k < len; k++) {
#pragma unroll
        for (int w = 0; w < 8; w++) sorted[16 * (i + k) + 8 + w] = row[k][w];
        perm[i + k] = src[k];
    }
}

__global__ void check_index_kernel(const uint32_t *__restrict__ addr_index, uint64_t n, uint32_t n_addr, int *__restrict__ flag) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && addr_index[i] >= n_addr) *flag = 3;
}

}  // namespace

// d_ha [n_addr][32], d_hs [n][32] digests; -> d_sorted [n][64], d_perm [n]
// keys_a / keys_b / idx_a serve both the entries and the nested sort of the address digests, so they are sized for
// max(n, n_addr) rows before their pointers are taken: the address table may be longer than the batch, and a block the
// nested sort had to grow would leave ka / kb / ia pointing at freed memory.
int32_t sort_composite_on_device(b200_ctx *c, const void *d_ha, uint32_t n_addr, const uint32_t *d_addr_index,
                                 const void *d_hs, uint64_t n, void *d_sorted, uint32_t *d_perm, DevBuf &keys_a,
                                 DevBuf &keys_b, DevBuf &idx_a, DevBuf &flag, bool allow_equal) {
    if (n == 0) return B200_OK;
    if (n >= (1ull << 32)) return fail(c, B200_ERR_INVALID_ARG, "at most 2^32-1 entries per sort");
    cudaStream_t st = c->stream;
    const uint64_t rows = std::max<uint64_t>(n, n_addr);
    TRY(ensure(c, keys_a, rows * 8));
    TRY(ensure(c, keys_b, rows * 8));
    TRY(ensure(c, idx_a, rows * 4));
    TRY(ensure(c, flag, 16));
    uint64_t *ka = static_cast<uint64_t *>(keys_a.p), *kb = static_cast<uint64_t *>(keys_b.p);
    uint32_t *ia = static_cast<uint32_t *>(idx_a.p);
    const uint64_t *ha = static_cast<const uint64_t *>(d_ha), *hs = static_cast<const uint64_t *>(d_hs);
    size_t temp = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, temp, ka, kb, ia, d_perm, (int64_t)n, 0, 64, st));
    TRY(ensure(c, c->cub_temp, temp));
    CU(cudaMemsetAsync(flag.p, 0, 4, st));
    check_index_kernel<<<nblk(n), 256, 0, st>>>(d_addr_index, n, n_addr, static_cast<int *>(flag.p));
    int *h_flag = reinterpret_cast<int *>(static_cast<uint8_t *>(c->pinned_small) + 3072);
    CU(cudaMemcpyAsync(h_flag, flag.p, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (*h_flag == 3) return fail(c, B200_ERR_INVALID_ARG, "addr_index entry out of range");
    auto lsd = [&](const int *words, int n_words) -> int32_t {
        uint32_t *cur = nullptr;
        uint32_t *bufs[2] = {ia, d_perm};
        int which = 0;
        for (int k = 0; k < n_words; k++) {
            uint32_t *idx_in = bufs[which], *idx_out = bufs[which ^ 1];
            extract_composite_kernel<<<nblk(n), 256, 0, st>>>(ha, d_addr_index, hs, cur, words[k], n, ka, idx_in);
            CU(cub::DeviceRadixSort::SortPairs(c->cub_temp.p, temp, ka, kb, idx_in, idx_out, (int64_t)n, 0, 64, st));
            cur = idx_out;
            which ^= 1;
            c->launches += 2;
        }
        if (cur != d_perm) CU(cudaMemcpyAsync(d_perm, cur, n * 4, cudaMemcpyDeviceToDevice, st));
        gather_composite_kernel<<<nblk(n), 256, 0, st>>>(static_cast<const uint4 *>(d_ha), d_addr_index,
                                                        static_cast<const uint4 *>(d_hs), d_perm, n,
                                                        static_cast<uint4 *>(d_sorted));
        CU(cudaMemsetAsync(flag.p, 0, 4, st));
        check_sorted_composite_kernel<<<nblk(n), 256, 0, st>>>(static_cast<const uint64_t *>(d_sorted), n,
                                                              static_cast<int *>(flag.p), allow_equal ? 1 : 0);
        c->launches += 2;
        CU(cudaMemcpyAsync(h_flag, flag.p, 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        return B200_OK;
    };
    // fast path: the addresses are few — sort their digests on their own and give every entry the dense rank of its
    // address; then four radix passes over the top 32 bits of the slot digests and ceil(log2(ranks)) bits of the rank
    // (stable: slot order survives inside an address), the rare rows that agree in both ordered in place, verification.
    {
        for (int k = 0; k < 4; k++) TRY(ensure(c, c->sort_aux[k], (size_t)n_addr * (k == 0 ? 32 : 4) + 16));
        uint8_t *sorted_ha = static_cast<uint8_t *>(c->sort_aux[0].p);
        uint32_t *perm_ha = static_cast<uint32_t *>(c->sort_aux[1].p), *dense = static_cast<uint32_t *>(c->sort_aux[2].p),
                 *rank = static_cast<uint32_t *>(c->sort_aux[3].p);
        TRY(sort_digests_on_device(c, d_ha, n_addr, sorted_ha, perm_ha, keys_a, keys_b, idx_a, flag, true));
        addr_heads_kernel<<<nblk(n_addr), 256, 0, st>>>(reinterpret_cast<const uint64_t *>(sorted_ha), n_addr, dense);
        size_t t_scan = 0, t32 = 0;
        CU(cub::DeviceScan::InclusiveSum(nullptr, t_scan, dense, dense, (int64_t)n_addr, st));
        uint32_t *ka32 = reinterpret_cast<uint32_t *>(ka), *kb32 = reinterpret_cast<uint32_t *>(kb);
        CU(cub::DeviceRadixSort::SortPairs(nullptr, t32, ka32, kb32, ia, d_perm, (int64_t)n, 0, 32, st));
        TRY(ensure(c, c->cub_temp, std::max(temp, std::max(t_scan, t32))));
        CU(cub::DeviceScan::InclusiveSum(c->cub_temp.p, t_scan, dense, dense, (int64_t)n_addr, st));
        addr_rank_scatter_kernel<<<nblk(n_addr), 256, 0, st>>>(perm_ha, dense, n_addr, rank);
        extract_slot_top32_kernel<<<nblk(n), 256, 0, st>>>(static_cast<const uint32_t *>(d_hs), n, ka32, ia);
        CU(cub::DeviceRadixSort::SortPairs(c->cub_temp.p, t32, ka32, kb32, ia, d_perm, (int64_t)n, 0, 32, st));
        extract_addr_rank_kernel<<<nblk(n), 256, 0, st>>>(d_addr_index, rank, d_perm, n, ka32);
        int rank_bits = 1;
        while (rank_bits < 32 && (1ull << rank_bits) < (uint64_t)n_addr) rank_bits++;
        CU(cub::DeviceRadixSort::SortPairs(c->cub_temp.p, t32, ka32, kb32, d_perm, ia, (int64_t)n, 0, rank_bits, st));
        CU(cudaMemcpyAsync(d_perm, ia, n * 4, cudaMemcpyDeviceToDevice, st));
        gather_composite_kernel<<<nblk(n), 256, 0, st>>>(static_cast<const uint4 *>(d_ha), d_addr_index,
                                                        static_cast<const uint4 *>(d_hs), d_perm, n,
                                                        static_cast<uint4 *>(d_sorted));
        fix_runs_composite_kernel<<<nblk(n), 256, 0, st>>>(static_cast<uint32_t *>(d_sorted), d_perm, n);
        CU(cudaMemsetAsync(flag.p, 0, 4, st));
        check_sorted_composite_kernel<<<nblk(n), 256, 0, st>>>(static_cast<const uint64_t *>(d_sorted), n,
                                                              static_cast<int *>(flag.p), allow_equal ? 1 : 0);
        c->launches += 11;
        CU(cudaMemcpyAsync(h_flag, flag.p, 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
    }
    if (*h_flag == 1) {
        const int full[8] = {7, 6, 5, 4, 3, 2, 1, 0};
        TRY(lsd(full, 8));
    }
    if (*h_flag == 2) return fail(c, B200_ERR_UNSORTED, "duplicate (address, slot) pair");
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------- changesets -> dirty set (a4)
// Incremental hashing of a block range: HashedPostStateSorted::from_reverts (crates/trie/db/src/state.rs:289-347),
// load_prefix_sets_with_provider (crates/trie/db/src/prefix_set.rs:22-60) and the key hashing of
// insert_account_for_hashing / insert_storage_for_hashing (crates/storage/provider/src/providers/database/provider.rs:
// 3206-3280) read the account / storage changesets of the range, keccak every address and slot, keep the FIRST (oldest)
// occurrence of every address and of every (address, slot) pair, and sort — HashSets and sort_unstable on one core.
// Here: one call.  Addresses of consecutive storage entries are hashed once per run (the changesets are ordered by
// (block, address), so a run is an account's slots in one block); stable radix sorts keep the oldest entry of equal keys
// in front, head flags + stream compaction drop the rest.
namespace {

__global__ void cs_run_heads_kernel(const uint8_t *__restrict__ addr20, uint64_t n, uint8_t *__restrict__ head) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool h = i == 0;
    if (!h) {
        const uint32_t *a = reinterpret_cast<const uint32_t *>(addr20 + 20 * (i - 1));
        const uint32_t *b = reinterpret_cast<const uint32_t *>(addr20 + 20 * i);
        h = a[0] != b[0] || a[1] != b[1] || a[2] != b[2] || a[3] != b[3] || a[4] != b[4];
    }
    head[i] = h ? 1 : 0;
}
// run index of every entry (inclusive scan of the heads, minus one) and the compacted run addresses
__global__ void cs_run_index_kernel(const uint8_t *__restrict__ addr20, const uint8_t *__restrict__ head,
                                    const uint32_t *__restrict__ incl, uint64_t n, uint32_t *__restrict__ run_of,
                                    uint8_t *__restrict__ run_addr20) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t r = incl[i] - 1;
    run_of[i] = r;
    if (head[i]) {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(addr20 + 20 * i);
        uint32_t *dst = reinterpret_cast<uint32_t *>(run_addr20 + 20 * (uint64_t)r);
#pragma unroll
        for (int w = 0; w < 5; w++) dst[w] = src[w];
    }
}
// head[i] = row i differs from row i-1 in its first `words` 64-bit words (rows of `stride` words)
__global__ void cs_row_heads_kernel(const uint64_t *__restrict__ rows, int stride, int words, uint64_t n, uint8_t *__restrict__ head) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool h = i == 0;
    if (!h)
        for (int w = 0; w < words; w++) h = h || rows[stride * (i - 1) + w] != rows[stride * i + w];
    head[i] = h ? 1 : 0;
}
// out32[j] = 32 bytes at word offset `off` of row sel[j]; first[j] = perm[sel[j]]
__global__ void cs_pick_rows_kernel(const uint64_t *__restrict__ rows, int stride, int off, const uint32_t *__restrict__ sel,
                                    const uint32_t *__restrict__ n_sel_p, const uint32_t *__restrict__ perm,
                                    uint64_t *__restrict__ out32, uint32_t *__restrict__ first) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= *n_sel_p) return;
    uint64_t i = sel[j];
#pragma unroll
    for (int w = 0; w < 4; w++) out32[4 * j + w] = rows[stride * i + off + w];
    if (first) first[j] = perm[i];
}
// heads of the address runs among the unique (address, slot) pairs sel[0 .. n_sel)
__global__ void cs_addr_heads_kernel(const uint64_t *__restrict__ rows64, const uint32_t *__restrict__ sel,
                                     const uint32_t *__restrict__ n_sel_p, uint8_t *__restrict__ head) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= *n_sel_p) return;
    bool h = j == 0;
    if (!h) {
        uint64_t a = sel[j - 1], b = sel[j];
        for (int w = 0; w < 4; w++) h = h || rows64[8 * a + w] != rows64[8 * b + w];
    }
    head[j] = h ? 1 : 0;
}
__global__ void cs_seg_offsets_kernel(const uint32_t *__restrict__ seg_start, const uint32_t *__restrict__ n_seg_p,
                                      const uint32_t *__restrict__ n_pairs_p, uint64_t *__restrict__ offs) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n_seg = *n_seg_p;
    if (j < n_seg) offs[j] = seg_start[j];
    if (j == n_seg) offs[j] = *n_pairs_p;
}
// sorted address key of segment j = the address half of the composite row of its first unique pair
__global__ void cs_seg_keys_kernel(const uint64_t *__restrict__ rows64, const uint32_t *__restrict__ sel,
                                   const uint32_t *__restrict__ seg_start, const uint32_t *__restrict__ n_seg_p,
                                   uint64_t *__restrict__ out32) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= *n_seg_p) return;
    uint64_t i = sel[seg_start[j]];
#pragma unroll
    for (int w = 0; w < 4; w++) out32[4 * j + w] = rows64[8 * i + w];
}

struct ChangesetOwner {
    void *host = nullptr;
};

}  // namespace

extern "C" B200_API void b200_changeset_hashes_release(b200_changeset_hashes *o) {
    if (!o) return;
    if (o->_owner) {
        ChangesetOwner *w = static_cast<ChangesetOwner *>(o->_owner);
        pinned_block_free(w->host);
        delete w;
    }
    memset(o, 0, sizeof *o);
}

extern "C" B200_API int32_t b200_hash_changesets(b200_ctx *c, const uint8_t *acct_addresses20, uint64_t n_acct,
                                                 const uint8_t *storage_addresses20, const uint8_t *storage_slots32,
                                                 uint64_t n_stor, b200_changeset_hashes *out) {
    if (!c || !out || (n_acct && !acct_addresses20) || (n_stor && (!storage_addresses20 || !storage_slots32)))
        return fail(c, B200_ERR_INVALID_ARG, "bad argument");
    if (n_acct >= (1ull << 31) || n_stor >= (1ull << 31)) return fail(c, B200_ERR_INVALID_ARG, "at most 2^31-1 changeset entries");
    memset(out, 0, sizeof *out);
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    uint32_t *ps = static_cast<uint32_t *>(c->pinned_small);
    thrust::counting_iterator<uint32_t> counting(0);
    auto up = [](size_t x) { return (x + 255) / 256 * 256; };

    // ---------------- device workspace (one block; sized from the entry counts)
    const uint64_t na = n_acct, ns = n_stor, nu = na + ns;  // nu bounds the union
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o += up(bytes ? bytes : 16); return at; };
    const size_t o_in_a = take(na * 20), o_in_sa = take(ns * 20), o_in_ss = take(ns * 32);
    const size_t o_dig_a = take(na * 32), o_sorted_a = take(na * 32), o_perm_a = take(na * 4), o_sel_a = take(na * 4);
    const size_t o_head = take(std::max(nu, (uint64_t)1)), o_incl = take(ns * 4), o_run_of = take(ns * 4), o_run_addr = take(ns * 20);
    const size_t o_ha = take(ns * 32), o_hs = take(ns * 32), o_sorted_s = take(ns * 64), o_perm_s = take(ns * 4), o_sel_s = take(ns * 4);
    const size_t o_seg = take(ns * 4), o_head2 = take(std::max(ns, (uint64_t)1));
    const size_t o_ukeys_a = take(na * 32), o_ufirst_a = take(na * 4);
    const size_t o_uslots = take(ns * 32), o_ufirst_s = take(ns * 4), o_segkeys = take(ns * 32), o_segoffs = take((ns + 1) * 8);
    const size_t o_cat = take(nu * 32), o_sorted_u = take(nu * 32), o_perm_u = take(nu * 4), o_sel_u = take(nu * 4), o_ukeys_u = take(nu * 32);
    const size_t o_cnt = take(64);
    TRY(ensure(c, c->in_a, o));
    uint8_t *W = static_cast<uint8_t *>(c->in_a.p);
    auto P = [&](size_t off) { return W + off; };
    uint32_t *cnt = reinterpret_cast<uint32_t *>(P(o_cnt));  // [0] unique accounts [1] runs(unused) [2] unique pairs [3] segments [4] union
    CU(cudaMemsetAsync(cnt, 0, 64, st));
    if (na) CU(cudaMemcpyAsync(P(o_in_a), acct_addresses20, na * 20, cudaMemcpyHostToDevice, st));
    if (ns) {
        CU(cudaMemcpyAsync(P(o_in_sa), storage_addresses20, ns * 20, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(P(o_in_ss), storage_slots32, ns * 32, cudaMemcpyHostToDevice, st));
    }
    size_t t1 = 0, t2 = 0;
    const uint64_t nmax = std::max<uint64_t>(nu, 1);
    CU(cub::DeviceSelect::Flagged(nullptr, t1, counting, P(o_head), reinterpret_cast<uint32_t *>(P(o_sel_u)), cnt, (int64_t)nmax, st));
    CU(cub::DeviceScan::InclusiveSum(nullptr, t2, P(o_head), reinterpret_cast<uint32_t *>(P(o_incl)), (int64_t)nmax, st));
    TRY(ensure(c, c->cub_temp, std::max(t1, t2)));

    // ---------------- accounts: hash, sort (oldest entry of equal keys first), keep the heads
    if (na) {
        CU(launch_keccak256_fixed(P(o_in_a), 20, 20, na, P(o_dig_a), st, &c->launches));
        TRY(sort_digests_on_device(c, P(o_dig_a), na, P(o_sorted_a), reinterpret_cast<uint32_t *>(P(o_perm_a)), c->sort_ka,
                                   c->sort_kb, c->sort_ia, c->sort_flag, true));
        cs_row_heads_kernel<<<nblk(na), 256, 0, st>>>(reinterpret_cast<const uint64_t *>(P(o_sorted_a)), 4, 4, na, P(o_head));
        CU(cub::DeviceSelect::Flagged(c->cub_temp.p, t1, counting, P(o_head), reinterpret_cast<uint32_t *>(P(o_sel_a)), cnt + 0,
                                      (int64_t)na, st));
        cs_pick_rows_kernel<<<nblk(na), 256, 0, st>>>(reinterpret_cast<const uint64_t *>(P(o_sorted_a)), 4, 0,
                                                      reinterpret_cast<const uint32_t *>(P(o_sel_a)), cnt + 0,
                                                      reinterpret_cast<const uint32_t *>(P(o_perm_a)),
                                                      reinterpret_cast<uint64_t *>(P(o_ukeys_a)), reinterpret_cast<uint32_t *>(P(o_ufirst_a)));
        c->launches += 3;
    }
    // ---------------- storage: address runs hashed once, slots hashed, composite sort, unique pairs, segments
    if (ns) {
        cs_run_heads_kernel<<<nblk(ns), 256, 0, st>>>(P(o_in_sa), ns, P(o_head));
        CU(cub::DeviceScan::InclusiveSum(c->cub_temp.p, t2, P(o_head), reinterpret_cast<uint32_t *>(P(o_incl)), (int64_t)ns, st));
        cs_run_index_kernel<<<nblk(ns), 256, 0, st>>>(P(o_in_sa), P(o_head), reinterpret_cast<const uint32_t *>(P(o_incl)), ns,
                                                      reinterpret_cast<uint32_t *>(P(o_run_of)), P(o_run_addr));
        CU(cudaMemcpyAsync(ps + 210, reinterpret_cast<uint32_t *>(P(o_incl)) + (ns - 1), 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        const uint32_t n_runs = ps[210];
        CU(launch_keccak256_fixed(P(o_run_addr), 20, 20, n_runs, P(o_ha), st, &c->launches));
        CU(launch_keccak256_fixed(P(o_in_ss), 32, 32, ns, P(o_hs), st, &c->launches));
        TRY(sort_composite_on_device(c, P(o_ha), n_runs, reinterpret_cast<const uint32_t *>(P(o_run_of)), P(o_hs), ns, P(o_sorted_s),
                                     reinterpret_cast<uint32_t *>(P(o_perm_s)), c->sort_ka, c->sort_kb, c->sort_ia, c->sort_flag, true));
        const uint64_t *rows = reinterpret_cast<const uint64_t *>(P(o_sorted_s));
        cs_row_heads_kernel<<<nblk(ns), 256, 0, st>>>(rows, 8, 8, ns, P(o_head));
        CU(cub::DeviceSelect::Flagged(c->cub_temp.p, t1, counting, P(o_head), reinterpret_cast<uint32_t *>(P(o_sel_s)), cnt + 2,
                                      (int64_t)ns, st));
        cs_pick_rows_kernel<<<nblk(ns), 256, 0, st>>>(rows, 8, 4, reinterpret_cast<const uint32_t *>(P(o_sel_s)), cnt + 2,
                                                      reinterpret_cast<const uint32_t *>(P(o_perm_s)),
                                                      reinterpret_cast<uint64_t *>(P(o_uslots)), reinterpret_cast<uint32_t *>(P(o_ufirst_s)));
        CU(cudaMemsetAsync(P(o_head2), 0, ns, st));
        cs_addr_heads_kernel<<<nblk(ns), 256, 0, st>>>(rows, reinterpret_cast<const uint32_t *>(P(o_sel_s)), cnt + 2, P(o_head2));
        CU(cub::DeviceSelect::Flagged(c->cub_temp.p, t1, counting, P(o_head2), reinterpret_cast<uint32_t *>(P(o_seg)), cnt + 3,
                                      (int64_t)ns, st));
        cs_seg_offsets_kernel<<<nblk(ns + 1), 256, 0, st>>>(reinterpret_cast<const uint32_t *>(P(o_seg)), cnt + 3, cnt + 2,
                                                            reinterpret_cast<uint64_t *>(P(o_segoffs)));
        cs_seg_keys_kernel<<<nblk(ns), 256, 0, st>>>(rows, reinterpret_cast<const uint32_t *>(P(o_sel_s)),
                                                     reinterpret_cast<const uint32_t *>(P(o_seg)), cnt + 3,
                                                     reinterpret_cast<uint64_t *>(P(o_segkeys)));
        c->launches += 10;
    }
    CU(cudaMemcpyAsync(ps + 212, cnt, 16, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint32_t ua = ps[212], up_ = ps[214], usa = ps[215];
    // ---------------- account prefix set: union of the two unique key lists
    const uint64_t ncat = (uint64_t)ua + usa;
    uint32_t uu = 0;
    if (ncat) {
        if (ua) CU(cudaMemcpyAsync(P(o_cat), P(o_ukeys_a), (size_t)ua * 32, cudaMemcpyDeviceToDevice, st));
        if (usa) CU(cudaMemcpyAsync(P(o_cat) + (size_t)ua * 32, P(o_segkeys), (size_t)usa * 32, cudaMemcpyDeviceToDevice, st));
        TRY(sort_digests_on_device(c, P(o_cat), ncat, P(o_sorted_u), reinterpret_cast<uint32_t *>(P(o_perm_u)), c->sort_ka,
                                   c->sort_kb, c->sort_ia, c->sort_flag, true));
        cs_row_heads_kernel<<<nblk(ncat), 256, 0, st>>>(reinterpret_cast<const uint64_t *>(P(o_sorted_u)), 4, 4, ncat, P(o_head));
        CU(cub::DeviceSelect::Flagged(c->cub_temp.p, t1, counting, P(o_head), reinterpret_cast<uint32_t *>(P(o_sel_u)), cnt + 4,
                                      (int64_t)ncat, st));
        cs_pick_rows_kernel<<<nblk(ncat), 256, 0, st>>>(reinterpret_cast<const uint64_t *>(P(o_sorted_u)), 4, 0,
                                                        reinterpret_cast<const uint32_t *>(P(o_sel_u)), cnt + 4, nullptr,
                                                        reinterpret_cast<uint64_t *>(P(o_ukeys_u)), nullptr);
        c->launches += 3;
        CU(cudaMemcpyAsync(ps + 216, cnt + 4, 4, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        uu = ps[216];
    }
    // ---------------- results: one page-locked block
    size_t h = 0;
    auto htake = [&](size_t bytes) { size_t at = h; h += (bytes + 15) / 16 * 16; return at; };
    const size_t h_ak = htake((size_t)ua * 32), h_af = htake((size_t)ua * 4), h_sk = htake((size_t)usa * 32),
                 h_so = htake(((size_t)usa + 1) * 8), h_lk = htake((size_t)up_ * 32), h_lf = htake((size_t)up_ * 4),
                 h_pk = htake((size_t)uu * 32);
    ChangesetOwner *owner = new ChangesetOwner();
    out->_owner = owner;
    if (!(owner->host = pinned_block_alloc(h ? h : 16))) return fail(c, B200_ERR_OOM, "page-locked result block");
    uint8_t *H = static_cast<uint8_t *>(owner->host);
    out->n_accounts = ua;
    out->account_keys32 = H + h_ak;
    out->account_first = reinterpret_cast<uint32_t *>(H + h_af);
    out->n_storage_accounts = usa;
    out->storage_account_keys32 = H + h_sk;
    out->storage_seg_offsets = reinterpret_cast<uint64_t *>(H + h_so);
    out->n_slots = up_;
    out->slot_keys32 = H + h_lk;
    out->slot_first = reinterpret_cast<uint32_t *>(H + h_lf);
    out->n_prefix = uu;
    out->account_prefix_keys32 = H + h_pk;
    out->storage_seg_offsets[0] = 0;
    if (ua) {
        CU(cudaMemcpyAsync(out->account_keys32, P(o_ukeys_a), (size_t)ua * 32, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(out->account_first, P(o_ufirst_a), (size_t)ua * 4, cudaMemcpyDeviceToHost, st));
    }
    if (up_) {
        CU(cudaMemcpyAsync(out->storage_account_keys32, P(o_segkeys), (size_t)usa * 32, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(out->storage_seg_offsets, P(o_segoffs), ((size_t)usa + 1) * 8, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(out->slot_keys32, P(o_uslots), (size_t)up_ * 32, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(out->slot_first, P(o_ufirst_s), (size_t)up_ * 4, cudaMemcpyDeviceToHost, st));
    }
    if (uu) CU(cudaMemcpyAsync(out->account_prefix_keys32, P(o_ukeys_u), (size_t)uu * 32, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return B200_OK;
}
