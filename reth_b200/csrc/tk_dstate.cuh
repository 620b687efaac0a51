// tk_dstate.cuh — dynamic state glue on top of tk_dtrie.cuh: sharded account buckets (frontier), storage wipes, routing of
// a block's slot entries to their storage tries.
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ sharded accounts
// Multi-GPU layout of §6 for the dynamic state: the account arena holds one trie per top-nibble bucket (trie id = nibble,
// every bucket a trie of its own, so its root hash is the frontier's as_root); as_child re-encodes the bucket's top item
// as a child of the depth-0 root branch.  One warp per bucket.
__global__ void dt_nibble_tries_kernel(const uint8_t *__restrict__ keys, uint64_t m, uint32_t *__restrict__ trie_of_key) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) trie_of_key[i] = keys[32 * i] >> 4;
}
__global__ void __launch_bounds__(512) dt_frontier_kernel(DTrieDev t, const uint8_t *__restrict__ bucket_roots,
                                                          FrontierEntryDev *__restrict__ out) {
    __shared__ __align__(16) uint8_t sbuf[16][WARP_BUF];
    const int lane = threadIdx.x & 31, b = threadIdx.x >> 5;
    uint8_t *buf = sbuf[b];
    WarpKeccak kw;
    kw.init(lane);
    FrontierEntryDev &e = out[b];
    for (int i = lane; i < (int)sizeof(FrontierEntryDev); i += 32) reinterpret_cast<uint8_t *>(&e)[i] = 0;
    __syncwarp();
    const uint32_t w = t.troot[b];
    if (w == DT_NONE || *(volatile int *)t.err != B200_DEVERR_NONE) return;
    uint32_t out8[8], hashed = 0, exts = 0, meta;
    if (w & DT_LEAF) {
        const uint32_t x = w & ~DT_LEAF;
        meta = warp_leaf_ref(true, buf, t.lkey + 32 * (uint64_t)x, 0, t.lval + 72 * (uint64_t)x,
                             t.lsroot ? t.lsroot + 32 * (uint64_t)x : nullptr, t.err, kw, lane, hashed, out8);
    } else {
        meta = dt_warp_build_node<0>(t, w, buf, kw, lane, hashed, exts, out8);
    }
    if (lane == 0) {
        e.as_root_len = 32;
        for (int i = 0; i < 32; i++) e.as_root[i] = bucket_roots[32 * b + i];
        LinBuf lb{e.as_child, 0};
        put_child(lb, out8, meta & META_LEN);
        e.as_child_len = (uint8_t)lb.n;
    }
}

// The bits this shard's buckets set in the masks of the depth-0 root branch: out[0] the hash mask, out[1] the tree mask
// (16 threads, thread k = bucket k).  The rule of dt_branch_payload at depth 0: the top node is a hashed child when it is a
// branch at depth 1, and a stored one when either of its own masks is set.  The top node's META_EXT is no help here: its
// reference was built with parent depth -1, as the root of its own trie.
__global__ void dt_frontier_masks_kernel(DTrieDev t, uint16_t *__restrict__ out) {
    const uint32_t k = threadIdx.x;
    const uint32_t w = t.troot[k];
    const bool node = w != DT_NONE && !(w & DT_LEAF);
    const bool hash = node && t.ndepth[w] == 1;
    bool tree = false;
    if (node) {
        const ushort4 mk = t.nmasks[w];
        tree = (mk.y | mk.z) != 0;
    }
    const uint32_t hm = __ballot_sync(0xFFFFu, hash), tm = __ballot_sync(0xFFFFu, tree);
    if (k == 0) {
        out[0] = (uint16_t)hm;
        out[1] = (uint16_t)tm;
    }
}

// ------------------------------------------------------------------------------------------------ dynamic state glue
// Which storage tries a block wipes: the tries of destroyed accounts and of accounts flagged "storage wiped"
// (HashedStorage::wiped, crates/trie/common/src/hashed_state.rs:423-428).  Trie id = id of the account's leaf.
__global__ void dt_wipe_list_kernel(const uint8_t *__restrict__ kind, const uint8_t *__restrict__ flags,
                                    const uint32_t *__restrict__ leaf_of, uint64_t m, uint32_t *__restrict__ tries,
                                    uint32_t *__restrict__ count) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    uint8_t k = kind[i];
    bool wiped = flags != nullptr && (flags[i] & 4);
    if (k == DK_DELETE || (wiped && (k == DK_UPDATE || k == DK_TOUCH))) tries[atomicAdd(count, 1u)] = leaf_of[i];
}
static __device__ __forceinline__ void dt_wipe_leaf(const DTrieDev &t, uint32_t x) {
    t.lmeta[x] = DT_DEAD;
    t.leaf_free[atomicAdd(&t.g[DG_LEAF_FREE], 1u)] = x;
    atomicSub(&t.g[DG_NLEAVES], 1u);
}
// Breadth-first release of whole tries; no removed-node records (reth reports a wiped storage trie as is_deleted).  The
// free stack doubles as the BFS queue: a released node is pushed onto node_free at once (nothing pops during a wipe), and
// the next round visits exactly the stack region the previous round pushed — its child words are still intact.
__global__ void dt_wipe_begin_kernel(DTrieDev t, const uint32_t *__restrict__ tries, const uint32_t *__restrict__ count_p) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *count_p) return;
    uint32_t r = tries[i], w = t.troot[r];
    if (w == DT_NONE) return;
    dt_set_child(t, r, DT_NONE, 0, DT_NONE);
    if (w & DT_LEAF) dt_wipe_leaf(t, w & ~DT_LEAF);
    else t.node_free[atomicAdd(&t.g[DG_NODE_FREE], 1u)] = w;
}
__global__ void dt_wipe_round_kernel(DTrieDev t, uint32_t lo, uint32_t hi) {  // node_free[lo, hi): pushed by the round before
    uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hi) return;
    uint32_t v = t.node_free[i];
    const uint32_t *ch = t.nchild + 16 * (uint64_t)v;
    for (int s = 0; s < 16; s++) {
        uint32_t w = ch[s];
        if (w == DT_NONE) continue;
        if (w & DT_LEAF) dt_wipe_leaf(t, w & ~DT_LEAF);
        else t.node_free[atomicAdd(&t.g[DG_NODE_FREE], 1u)] = w;
    }
    t.ndepth[v] = DT_DEAD;
    t.nmeta[v] = 0;
    t.npending[v] = 0;
}
// trie_of_key[j] for storage entry j of account entry i (seg_offsets[i] <= j < seg_offsets[i+1]): the account's leaf if
// the account exists after the block, DT_NONE (entry ignored) otherwise
__global__ void dt_expand_tries_kernel(const uint64_t *__restrict__ seg_offsets, uint64_t m, const uint8_t *__restrict__ kind,
                                       const uint32_t *__restrict__ leaf_of, uint64_t n_entries, uint32_t *__restrict__ trie_of_key) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_entries) return;
    uint64_t lo = 0, hi = m;  // last account with offset <= j
    while (hi - lo > 1) {
        uint64_t mid = (lo + hi) >> 1;
        if (seg_offsets[mid] <= j) lo = mid;
        else hi = mid;
    }
    uint8_t k = kind[lo];
    trie_of_key[j] = (k == DK_UPDATE || k == DK_TOUCH || k == DK_INSERT) ? leaf_of[lo] : DT_NONE;
}

