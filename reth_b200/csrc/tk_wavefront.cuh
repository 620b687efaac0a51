// tk_wavefront.cuh — incremental update: pending counters, climbing wavefront (warp and thread variants).
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ incremental wavefront
// pending[p] = number of dirty children of node p (dirty leaves and dirty branches), counted by walking up from
// every dirty leaf and stopping at the first ancestor somebody else already reached.
__global__ void mark_pending_kernel(ForestDev f, const uint32_t *__restrict__ idx, uint64_t m,
                                    const uint32_t *__restrict__ leaf_parent, const uint32_t *__restrict__ node_parent,
                                    uint32_t *__restrict__ pending) {
    if (*(volatile int *)f.err != B200_DEVERR_NONE) return;
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m) return;
    uint32_t p = leaf_parent[idx[t]];
    while (p != 0xFFFFFFFFu) {
        if (atomicAdd(&pending[p], 1u) != 0u) break;
        p = node_parent[p];
    }
}

// A warp that just finished a dirty item climbs from its parent p: whoever is the LAST dirty child to arrive at a
// node re-hashes it and goes on; everybody else retires.  Returns true iff this warp finished the root.
__device__ __forceinline__ bool warp_climb(const ForestDev &f, uint32_t p, const uint32_t *__restrict__ node_parent,
                                           uint32_t *__restrict__ pending, uint32_t *__restrict__ dirty_list,
                                           uint32_t *__restrict__ dirty_count, uint8_t *buf, const WarpKeccak &kw, int lane,
                                           uint32_t &hashed, uint32_t &exts, uint32_t (&out)[8]) {
    while (p != 0xFFFFFFFFu) {
        uint32_t last = 0;
        if (lane == 0) {
            __threadfence();  // publish what this warp wrote before announcing arrival
            last = atomicSub(&pending[p], 1u) == 1u;
            __threadfence();
        }
        last = __shfl_sync(0xffffffffu, last, 0);
        if (!last) return false;
        int d = f.node_masks[p].w;
        warp_build_node<true>(f, p, d, buf, kw, lane, hashed, exts, out);
        if (lane == 0) dirty_list[atomicAdd(dirty_count, 1u)] = p;
        p = node_parent[p];
    }
    return true;
}

// One warp per dirty leaf: overwrite + re-hash the leaf, then climb: whoever is the LAST dirty child to arrive at a
// node re-hashes it and continues to its parent; everybody else retires.  The whole dirty-path re-hash of an update
// is this single launch: its latency is (levels) x (one warp-built node), with no host round trip in between.
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) wavefront_kernel(ForestDev f, uint8_t *__restrict__ accts,
                                                              uint8_t *__restrict__ sroots,
                                                              const uint8_t *__restrict__ new_accts,
                                                              const uint8_t *__restrict__ new_sroots,
                                                              const uint32_t *__restrict__ idx, uint64_t m,
                                                              const uint32_t *__restrict__ leaf_parent,
                                                              const uint32_t *__restrict__ node_parent,
                                                              uint32_t *__restrict__ pending, uint32_t *__restrict__ dirty_list,
                                                              uint32_t *__restrict__ dirty_count, uint8_t *__restrict__ root_out) {
    __shared__ __align__(16) uint8_t sbuf[WARPS][WARP_BUF];
    if (*(volatile int *)f.err != B200_DEVERR_NONE) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t *buf = sbuf[warp];
    WarpKeccak kw;
    kw.init(lane);
    uint32_t hashed = 0, exts = 0;
    const uint64_t t = (uint64_t)blockIdx.x * WARPS + warp;
    if (t >= m) return;
    const uint32_t i = idx[t];
    // ---- the leaf
    if (lane == 0) {
        const uint64_t *src = reinterpret_cast<const uint64_t *>(new_accts + 72 * t);
        uint64_t *dst = reinterpret_cast<uint64_t *>(accts + 72 * (uint64_t)i);
#pragma unroll
        for (int w = 0; w < 9; w++) dst[w] = src[w];
        if (new_sroots && sroots) {
            uint32_t r[8];
            load32(new_sroots + 32 * t, r);
            store32(sroots + 32 * (uint64_t)i, r);
        }
    }
    uint32_t out[8];
    warp_leaf_ref(true, buf, f.keys + 32 * (uint64_t)i, parent_depth(f, i, i), new_accts + 72 * t,
                  sroots ? (new_sroots ? new_sroots + 32 * t : sroots + 32 * (uint64_t)i) : nullptr, f.err, kw, lane, hashed, out);
    if (lane == 0) {
        store32(f.leaf_ref + 32 * (uint64_t)i, out);
        f.leaf_meta[i] = 0;
    }
    __syncwarp();
    // ---- climb
    bool top = warp_climb(f, leaf_parent[i], node_parent, pending, dirty_list, dirty_count, buf, kw, lane, hashed, exts, out);
    if (top && lane == 0) store32(root_out, out);  // this warp re-hashed the root (or the only leaf)
    flush_warp_counters(f.counters, hashed, exts);
}

// ---- two-stage variant for large dirty sets -----------------------------------------------------------------------
// Stage A: one THREAD per dirty leaf (register-resident sponge: the ALU-efficient formulation) hashes the leaf and
// climbs through the populous deep levels (depth >= split_depth); when the next ancestor is shallower it hands the
// parent over.  Stage B (climb_kernel): one WARP per hand-over finishes the sparse upper levels with the
// latency-optimised warp-cooperative node builder.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) wavefront_thread_kernel(
    ForestDev f, uint8_t *__restrict__ accts, uint8_t *__restrict__ sroots, const uint8_t *__restrict__ new_accts,
    const uint8_t *__restrict__ new_sroots, const uint32_t *__restrict__ idx, uint64_t m,
    const uint32_t *__restrict__ leaf_parent, const uint32_t *__restrict__ node_parent, uint32_t *__restrict__ pending,
    uint32_t *__restrict__ dirty_list, uint32_t *__restrict__ dirty_count, uint32_t *__restrict__ handoff_list,
    uint32_t *__restrict__ handoff_count, uint8_t *__restrict__ root_out, int split_depth) {
    extern __shared__ uint32_t smem[];
    if (*(volatile int *)f.err != B200_DEVERR_NONE) return;
    Strip<BLOCK> s;
    uint32_t hashed = 0, exts = 0;
    uint64_t t = (uint64_t)blockIdx.x * BLOCK + threadIdx.x;
    if (t < m) {
        const uint32_t i = idx[t];
        s.init(smem);
        {
            const uint64_t *src = reinterpret_cast<const uint64_t *>(new_accts + 72 * t);
            uint64_t *dst = reinterpret_cast<uint64_t *>(accts + 72 * (uint64_t)i);
#pragma unroll
            for (int w = 0; w < 9; w++) dst[w] = src[w];
            if (new_sroots && sroots) {
                uint32_t r[8];
                load32(new_sroots + 32 * t, r);
                store32(sroots + 32 * (uint64_t)i, r);
            }
        }
        uint32_t k[8];
        load32(f.keys + 32 * (uint64_t)i, k);
        const int pd = parent_depth(f, i, i);
        uint32_t len = encode_leaf<Strip<BLOCK>, true>(
            s, k, pd, new_accts + 72 * t, sroots ? (new_sroots ? new_sroots + 32 * t : sroots + 32 * (uint64_t)i) : nullptr,
            f.err);
        uint32_t ref[8];
        uint32_t meta = strip_to_ref(s, len, pd < 0, ref, hashed);
        store32(f.leaf_ref + 32 * (uint64_t)i, ref);
        f.leaf_meta[i] = (uint8_t)meta;
        uint32_t p = leaf_parent[i];
        bool top = true;
        while (p != 0xFFFFFFFFu) {
            int d = f.node_masks[p].w;
            if (d < split_depth) {
                __threadfence();
                handoff_list[atomicAdd(handoff_count, 1u)] = p;
                top = false;
                break;
            }
            __threadfence();
            bool last = atomicSub(&pending[p], 1u) == 1u;
            __threadfence();
            if (!last) {
                top = false;
                break;
            }
            thread_build_node<BLOCK, 16, true>(s, smem, f, p, d, hashed, exts, ref);
            dirty_list[atomicAdd(dirty_count, 1u)] = p;
            p = node_parent[p];
        }
        if (top) store32(root_out, ref);
    }
    flush_counters(f.counters, hashed, exts);
}

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) climb_kernel(ForestDev f, const uint32_t *__restrict__ start_list,
                                                          const uint32_t *__restrict__ start_count_p,
                                                          const uint32_t *__restrict__ node_parent,
                                                          uint32_t *__restrict__ pending, uint32_t *__restrict__ dirty_list,
                                                          uint32_t *__restrict__ dirty_count, uint8_t *__restrict__ root_out) {
    __shared__ __align__(16) uint8_t sbuf[WARPS][WARP_BUF];
    if (*(volatile int *)f.err != B200_DEVERR_NONE) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpKeccak kw;
    kw.init(lane);
    uint32_t hashed = 0, exts = 0;
    const uint32_t count = *start_count_p;
    for (uint32_t e = blockIdx.x * WARPS + warp; e < count; e += gridDim.x * WARPS) {
        uint32_t out[8];
        bool top = warp_climb(f, start_list[e], node_parent, pending, dirty_list, dirty_count, sbuf[warp], kw, lane, hashed,
                              exts, out);
        if (top && lane == 0) store32(root_out, out);
    }
    flush_warp_counters(f.counters, hashed, exts);
}
