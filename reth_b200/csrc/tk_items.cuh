// tk_items.cuh — leaf pass of an "items" build: the input stream of an incremental HashBuilder run.
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, after tk_ordered.cuh).
//
// reth's incremental root (StateRoot / StorageRoot over TrieWalker + TrieNodeIter, crates/trie/trie/src/walker.rs:161-388,
// node_iter.rs:200-304) feeds HashBuilder two kinds of elements in key order: `add_leaf(key, value)` for the changed leaves
// and the leaves no stored hash covers, and `add_branch(path, hash, children_are_in_trie)` for every unchanged subtree whose
// hash the trie tables still hold.  Here such a stream is one sorted item array: a hash item sits at one position like a
// leaf (key = its path, zero-padded; paths and keys are prefix-free, so the structure pass runs unchanged) but stands for
// a branch node of depth L = its path length: it is wrapped in an extension when its parent is more than one nibble away,
// and its parent sets the hash-mask bit (cleared by the extension) and, with children_are_in_trie, the tree-mask bit —
// alloy-trie HashBuilder::update for a `HashBuilderValue::Hash` (SURVEY.md Appendix A).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) item_leaf_kernel(ForestDev f, ItemLeavesDev it, const uint8_t *__restrict__ values,
                                                          const uint8_t *__restrict__ storage_roots) {
    extern __shared__ uint32_t smem[];
    if (*(volatile int *)f.err == B200_DEVERR_UNSORTED || *(volatile int *)f.err == B200_DEVERR_BAD_OFFSETS) return;
    Strip<BLOCK> s;
    uint32_t hashed = 0, exts = 0;
    const uint32_t stride = it.account ? (uint32_t)sizeof(b200_account_dev) : 32u;
    const uint64_t step = (uint64_t)gridDim.x * BLOCK;
    for (uint64_t i = (uint64_t)blockIdx.x * BLOCK + threadIdx.x; i < f.n; i += step) {
        s.init(smem);
        const int pd = parent_depth(f, i, i);
        const uint32_t L = it.key_nibs[i];
        uint32_t ref[8], meta;
        if (L >= 64) {
            uint32_t k[8];
            load32(f.keys + 32 * i, k);
            const uint8_t *vp = values + (uint64_t)stride * i;
            uint32_t len = it.account ? encode_leaf<Strip<BLOCK>, true>(s, k, pd, vp, storage_roots ? storage_roots + 32 * i : nullptr, f.err)
                                      : encode_leaf<Strip<BLOCK>, false>(s, k, pd, vp, nullptr, f.err);
            meta = strip_to_ref(s, len, pd < 0, ref, hashed);
        } else {
            if (pd >= (int)L) atomicExch(f.err, B200_DEVERR_UNSORTED);  // another item lies below this path: not prefix-free
            {  // rows of 72 bytes are only 8-byte aligned
                const uint2 *q = reinterpret_cast<const uint2 *>(values + (uint64_t)stride * i);
#pragma unroll
                for (int w = 0; w < 4; w++) {
                    uint2 t = __ldg(q + w);
                    ref[2 * w] = t.x;
                    ref[2 * w + 1] = t.y;
                }
            }
            // an extension node when more than one nibble below its parent (or alone in its trie): >= 35 bytes, hashed
            meta = META_ISNODE | ((it.flags[i] & 1) ? META_STORED : 0u) |
                   thread_finish_node(s, ref, 0u, pd, (int)L, f.keys + 32 * i, hashed, exts);
        }
        store32(f.leaf_ref + 32 * i, ref);
        f.leaf_meta[i] = (uint8_t)meta;
        f.S[i] = (uint32_t)i;
        f.E[i] = (uint32_t)i;
    }
    flush_counters(f.counters, hashed, exts);
}

cudaError_t launch_item_leaves(const ForestDev &f, const ItemLeavesDev &it, const uint8_t *values, const uint8_t *storage_roots,
                               cudaStream_t st) {
    if (f.n == 0) return cudaSuccess;
    auto k = item_leaf_kernel<LEAF_BLOCK>;
    size_t smem = (size_t)LEAF_WORDS_ACCOUNT * LEAF_BLOCK * 4;
    k<<<persistent_grid(k, LEAF_BLOCK, smem, f.n), LEAF_BLOCK, smem, st>>>(f, it, values, storage_roots);
    return cudaGetLastError();
}
