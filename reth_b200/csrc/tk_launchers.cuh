// tk_launchers.cuh — host-side launchers (grid sizing, dynamic shared memory opt-in).
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ launchers
static inline unsigned blocks_for(uint64_t n, unsigned block) { return (unsigned)((n + block - 1) / block); }

static int g_sms = 0;
static int sms() {
    if (!g_sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_sms <= 0) g_sms = 132;
    }
    return g_sms;
}

// grid = min(work, SM count x resident CTAs): a single full wave, grid-stride inside the kernel
template <typename K>
static unsigned persistent_grid(K kernel, int block, size_t smem, uint64_t work_items) {
    static std::mutex mu;
    static std::unordered_map<const void *, int> cache;
    int per_sm;
    {
        std::lock_guard<std::mutex> g(mu);
        auto it = cache.find((const void *)kernel);
        if (it == cache.end()) {
            cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            per_sm = 1;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, smem);
            if (per_sm < 1) per_sm = 1;
            cache.emplace((const void *)kernel, per_sm);
        } else {
            per_sm = it->second;
        }
    }
    uint64_t want = (work_items + block - 1) / block;
    uint64_t cap = (uint64_t)sms() * per_sm;
    return (unsigned)(want < cap ? (want ? want : 1) : cap);
}

cudaError_t launch_latch_error(int *err, int *sticky, unsigned long long *counters, cudaStream_t st) {
    latch_error_kernel<<<1, 1, 0, st>>>(err, sticky, counters);
    return cudaGetLastError();
}
cudaError_t launch_mark_boundaries(const uint64_t *d_seg_offsets, uint64_t n_segs, uint64_t n, uint8_t *Lp, int *err,
                                   cudaStream_t st) {
    mark_boundaries_kernel<<<blocks_for(n_segs + 1, 256), 256, 0, st>>>(d_seg_offsets, n_segs, n, Lp, err);
    return cudaGetLastError();
}
cudaError_t launch_lcp(const uint8_t *keys, uint64_t n, uint8_t *Lp, uint8_t *nibs, int *err, cudaStream_t st) {
    lcp_kernel<<<blocks_for(n + 1, 256), 256, 0, st>>>(keys, n, Lp, nibs, err);
    return cudaGetLastError();
}
cudaError_t launch_iota(uint32_t *out, uint64_t n, uint32_t first, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    iota_kernel<<<blocks_for(n, 256), 256, 0, st>>>(out, n, first);
    return cudaGetLastError();
}
cudaError_t launch_fill_u32(uint32_t *out, uint64_t n, uint32_t value, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    fill_u32_kernel<<<blocks_for(n, 256), 256, 0, st>>>(out, n, value);
    return cudaGetLastError();
}
cudaError_t launch_gap_keys(const uint8_t *Lp, uint64_t G, uint16_t *key, uint32_t *val, uint32_t *unresolved, cudaStream_t st) {
    if (G == 0) return cudaSuccess;
    gap_keys_kernel<<<blocks_for(G, 256), 256, 0, st>>>(Lp, G, key, val, unresolved);
    return cudaGetLastError();
}
cudaError_t launch_bucket_offsets(const uint16_t *key_sorted, uint64_t G, uint32_t *bucket_off, cudaStream_t st) {
    bucket_offsets_kernel<<<1, 96, 0, st>>>(key_sorted, G, bucket_off);
    return cudaGetLastError();
}
cudaError_t launch_head_fix(const uint8_t *keys, uint16_t *key_sorted, const uint32_t *gap_sorted, const uint64_t *seg_offsets,
                            uint64_t n_segs, const uint32_t *unresolved, uint64_t G, cudaStream_t st) {
    if (G == 0) return cudaSuccess;
    head_fix_kernel<<<blocks_for(G, 256), 256, 0, st>>>(keys, key_sorted, gap_sorted, seg_offsets, n_segs, unresolved, G);
    return cudaGetLastError();
}
cudaError_t launch_level_ranges(uint32_t *node_start, const uint32_t *n_nodes_p, const uint32_t *bucket_off,
                                uint32_t *level_lo, cudaStream_t st) {
    level_ranges_kernel<<<1, 96, 0, st>>>(node_start, n_nodes_p, bucket_off, level_lo, node_start);
    return cudaGetLastError();
}

constexpr int LEAF_BLOCK = 128;
constexpr int LEAF_WORDS_STORAGE = 34;   // <= 70 bytes -> one rate block
constexpr int LEAF_WORDS_ACCOUNT = 68;   // <= 148 bytes -> two rate blocks
constexpr int BRANCH_BLOCK = 128;
constexpr int BRANCH_WORDS = 136;        // <= 532 bytes -> four rate blocks

cudaError_t launch_leaves(const ForestDev &f, bool account, const uint8_t *values, const uint8_t *storage_roots,
                          cudaStream_t st) {
    if (f.n == 0) return cudaSuccess;
    if (account) {
        auto k = leaf_kernel<LEAF_BLOCK, true>;
        size_t smem = (size_t)LEAF_WORDS_ACCOUNT * LEAF_BLOCK * 4;
        k<<<persistent_grid(k, LEAF_BLOCK, smem, f.n), LEAF_BLOCK, smem, st>>>(f, values, storage_roots);
    } else {
        auto k = leaf_storage_kernel<LEAF_BLOCK>;
        size_t smem = (size_t)LEAF_WORDS_STORAGE * LEAF_BLOCK * 4;  // the strip of the rare leaves outside the register path
        k<<<blocks_for(f.n, LEAF_BLOCK), LEAF_BLOCK, smem, st>>>(f, values);
    }
    return cudaGetLastError();
}

template <int MAXC, int WORDS>
static cudaError_t launch_branch_class(const ForestDev &f, const uint32_t *node_order, uint32_t pos_lo, uint32_t pos_hi,
                                       int d, cudaStream_t st) {
    auto k = branch_kernel<BRANCH_BLOCK, MAXC>;
    size_t smem = (size_t)WORDS * BRANCH_BLOCK * 4;
    k<<<persistent_grid(k, BRANCH_BLOCK, smem, pos_hi - pos_lo), BRANCH_BLOCK, smem, st>>>(f, node_order, pos_lo,
                                                                                          pos_hi, d);
    return cudaGetLastError();
}

// cls: child-count class of every node in the range (0: <=3, 1: <=7, 2: <=12, 3: <=16 children), or 3 for a
// mixed range.  The extension wrapper (<= 70 bytes) fits the smallest strip.
cudaError_t launch_branch_level(const ForestDev &f, const uint32_t *node_order, uint32_t pos_lo, uint32_t pos_hi,
                                int d, int cls, cudaStream_t st) {
    if (pos_hi <= pos_lo) return cudaSuccess;
    if (cls < 0) {  // latency path: one warp per node
        constexpr int WARPS = 4;
        uint32_t cnt = pos_hi - pos_lo;
        unsigned blocks = (cnt + WARPS - 1) / WARPS;
        unsigned cap = (unsigned)sms() * 16;
        branch_warp_kernel<WARPS><<<blocks < cap ? blocks : cap, WARPS * 32, 0, st>>>(f, node_order, pos_lo, pos_hi, d);
        return cudaGetLastError();
    }
    switch (cls) {
        case 0: {  // 2 / 3 children: register path, gather of the next node pipelined under the permutation of this one
            auto k = branch3_pipelined_kernel<BRANCH_BLOCK>;
            size_t smem = (size_t)34 * BRANCH_BLOCK * 4;  // the strip of the rare extension / inline-child nodes
            k<<<persistent_grid(k, BRANCH_BLOCK, smem, pos_hi - pos_lo), BRANCH_BLOCK, smem, st>>>(f, node_order, pos_lo, pos_hi, d);
            return cudaGetLastError();
        }
        case 1: return launch_branch_class<7, 68>(f, node_order, pos_lo, pos_hi, d, st);
        case 2: return launch_branch_class<12, 102>(f, node_order, pos_lo, pos_hi, d, st);
        default: return launch_branch_class<16, BRANCH_WORDS>(f, node_order, pos_lo, pos_hi, d, st);
    }
}

// sort key of node v: deepest level first, then by the number of rate blocks its RLP needs when every child
// is a 33-byte hash reference (children <= 3 -> 1 block, <= 7 -> 2, <= 12 -> 3, else 4)
// hist[key] counts the nodes of every (depth, class); runs before the host knows the node count, hence the
// device-side bound.
__global__ void node_class_keys_kernel(const uint32_t *__restrict__ node_start, const uint16_t *__restrict__ key_sorted,
                                       const uint32_t *__restrict__ n_nodes_p, uint8_t *__restrict__ keys,
                                       uint32_t *__restrict__ ids, uint32_t *__restrict__ hist) {
    __shared__ uint32_t sh[256];
    sh[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t n_nodes = *n_nodes_p;
    for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n_nodes; v += gridDim.x * blockDim.x) {
        uint32_t j0 = node_start[v], children = node_start[v + 1] - j0 + 1;
        uint32_t cls = children <= 3 ? 0 : (children <= 7 ? 1 : (children <= 12 ? 2 : 3));
        uint32_t key = ((63u - (key_sorted[j0] & 0xFFu)) << 2) | cls;
        keys[v] = (uint8_t)key;
        ids[v] = v;
        atomicAdd(&sh[key], 1u);
    }
    __syncthreads();
    if (sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}
cudaError_t launch_node_class_keys(const uint32_t *node_start, const uint16_t *key_sorted, const uint32_t *n_nodes_p,
                                   uint64_t max_nodes, uint8_t *keys, uint32_t *ids, uint32_t *hist, cudaStream_t st) {
    if (max_nodes == 0) return cudaSuccess;
    unsigned blocks = blocks_for(max_nodes, 256);
    if (blocks > (unsigned)sms() * 8) blocks = (unsigned)sms() * 8;
    node_class_keys_kernel<<<blocks, 256, 0, st>>>(node_start, key_sorted, n_nodes_p, keys, ids, hist);
    return cudaGetLastError();
}

cudaError_t launch_segment_roots(const ForestDev &f, const uint64_t *d_seg_offsets, uint64_t n_segs, uint8_t *roots,
                                 cudaStream_t st) {
    if (n_segs == 0) return cudaSuccess;
    segment_roots_kernel<<<blocks_for(n_segs, 256), 256, 0, st>>>(f, d_seg_offsets, n_segs, roots);
    return cudaGetLastError();
}

cudaError_t launch_stored_flags(const ForestDev &f, uint32_t n_nodes, uint8_t *flags, uint32_t *n_hashes,
                                cudaStream_t st) {
    if (n_nodes == 0) return cudaSuccess;
    stored_flags_kernel<<<blocks_for(n_nodes, 256), 256, 0, st>>>(f, n_nodes, flags, n_hashes);
    return cudaGetLastError();
}
cudaError_t launch_table_order_keys(const ForestDev &f, const uint32_t *ids, uint32_t count, uint64_t *keys, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    table_order_keys_kernel<<<blocks_for(count, 256), 256, 0, st>>>(f, ids, count, keys);
    return cudaGetLastError();
}
cudaError_t launch_row_sizes(const ForestDev &f, const uint32_t *ids, uint32_t count, int packed, int storage, uint64_t *size,
                             uint32_t *key_len, cudaStream_t st) {
    row_sizes_kernel<<<blocks_for((uint64_t)count + 1, 256), 256, 0, st>>>(f, ids, count, packed, storage, size, key_len);
    return cudaGetLastError();
}
cudaError_t launch_encode_rows(const ForestDev &f, const uint32_t *ids, uint32_t count, int packed, int storage,
                               const uint64_t *d_seg_offsets, uint64_t n_segs, const uint8_t *acct_keys,
                               const uint64_t *row_off, uint8_t *out, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    constexpr int WARPS = 8;
    encode_rows_kernel<WARPS><<<blocks_for(count, WARPS), WARPS * 32, 0, st>>>(f, ids, count, packed, storage, d_seg_offsets,
                                                                              n_segs, acct_keys, row_off, out);
    return cudaGetLastError();
}
cudaError_t launch_gather_updates(const ForestDev &f, const uint32_t *stored_ids, uint32_t n_stored,
                                  const uint32_t *hash_prefix, const uint32_t *prefix_by_record,
                                  const uint64_t *d_seg_offsets, uint64_t n_segs, const UpdatesDev &out,
                                  cudaStream_t st) {
    if (n_stored == 0) return cudaSuccess;
    gather_updates_kernel<<<blocks_for(n_stored, 128), 128, 0, st>>>(f, stored_ids, n_stored, hash_prefix,
                                                                     prefix_by_record, d_seg_offsets, n_segs, out);
    return cudaGetLastError();
}

cudaError_t launch_nibble_buckets(const uint8_t *keys, uint64_t n, uint64_t *offs, cudaStream_t st) {
    nibble_buckets_kernel<<<1, 32, 0, st>>>(keys, n, offs);
    return cudaGetLastError();
}
cudaError_t launch_frontier(const ForestDev &f, const uint64_t *bucket_offsets, const uint8_t *values,
                            const uint8_t *storage_roots, FrontierEntryDev *out, cudaStream_t st) {
    constexpr int B = 32;
    auto k = frontier_kernel<B, true>;
    size_t smem = (size_t)BRANCH_WORDS * B * 4;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k<<<1, B, smem, st>>>(f, bucket_offsets, values, storage_roots, out);
    return cudaGetLastError();
}
cudaError_t launch_merge_frontiers(const FrontierEntryDev *all, int world, FrontierEntryDev *out, int *err, cudaStream_t st) {
    merge_frontiers_kernel<<<1, 32, 0, st>>>(all, world, out, err);
    return cudaGetLastError();
}
cudaError_t launch_partition_owner(const uint8_t *digests, uint64_t n, int world, uint8_t *owner, unsigned long long *counts,
                                   cudaStream_t st) {
    if (n) partition_owner_kernel<<<blocks_for(n, 256), 256, 0, st>>>(digests, n, world, owner, counts);
    return cudaGetLastError();
}
cudaError_t launch_gather_values(const uint8_t *values, uint32_t vb, const uint32_t *perm, uint64_t n, uint8_t *out_v, cudaStream_t st) {
    if (!n || !vb) return cudaSuccess;
    const uintptr_t al = reinterpret_cast<uintptr_t>(values) | reinterpret_cast<uintptr_t>(out_v) | vb;
    if (!(al & 7)) {
        gather_rows_kernel<uint64_t><<<blocks_for(n * (vb / 8), 256), 256, 0, st>>>(reinterpret_cast<const uint64_t *>(values), vb / 8, perm, n,
                                                                                 reinterpret_cast<uint64_t *>(out_v));
    } else if (!(al & 3)) {
        gather_rows_kernel<uint32_t><<<blocks_for(n * (vb / 4), 256), 256, 0, st>>>(reinterpret_cast<const uint32_t *>(values), vb / 4, perm, n,
                                                                                 reinterpret_cast<uint32_t *>(out_v));
    } else {
        gather_rows_kernel<uint8_t><<<blocks_for(n * vb, 256), 256, 0, st>>>(values, vb, perm, n, out_v);
    }
    return cudaGetLastError();
}
cudaError_t launch_partition_gather(const uint8_t *digests, const uint8_t *values, uint32_t vb, const uint32_t *perm, uint64_t n,
                                    uint8_t *out_d, uint8_t *out_v, cudaStream_t st) {
    if (!n) return cudaSuccess;
    partition_gather_kernel<<<blocks_for(n, 256), 256, 0, st>>>(digests, perm, n, out_d);
    cudaError_t e = cudaGetLastError();
    return e != cudaSuccess ? e : launch_gather_values(values, vb, perm, n, out_v, st);
}
cudaError_t launch_root_from_frontier(const FrontierEntryDev *fr, uint8_t *root, cudaStream_t st) {
    constexpr int B = 32;
    auto k = root_from_frontier_kernel<B>;
    size_t smem = (size_t)BRANCH_WORDS * B * 4;
    k<<<1, B, smem, st>>>(fr, root);
    return cudaGetLastError();
}

// ---- resident trie launchers
cudaError_t launch_locate_classify(const uint8_t *keys, uint64_t n, const uint8_t *dirty_keys, const uint8_t *present,
                                   uint64_t m, uint32_t *lb, uint8_t *kind, uint32_t *counts, int *err, cudaStream_t st) {
    if (m == 0) return cudaSuccess;
    locate_classify_kernel<<<blocks_for(m, 128), 128, 0, st>>>(keys, n, dirty_keys, present, m, lb, kind, counts, err);
    return cudaGetLastError();
}
cudaError_t launch_merge_marks(const uint32_t *lb, const uint8_t *kind, uint64_t m, uint32_t *ins_at, uint32_t *del,
                               uint32_t *ins_flag, cudaStream_t st) {
    if (m == 0) return cudaSuccess;
    merge_marks_kernel<<<blocks_for(m, 256), 256, 0, st>>>(lb, kind, m, ins_at, del, ins_flag);
    return cudaGetLastError();
}
cudaError_t launch_merge_scatter(const uint8_t *keys, const uint8_t *accts, const uint8_t *sroots, uint64_t n,
                                 const uint32_t *ins_incl, const uint32_t *del_excl, const uint32_t *del,
                                 const uint8_t *dirty_keys, const uint8_t *new_accts, const uint8_t *new_sroots,
                                 const uint32_t *lb, const uint8_t *kind, const uint32_t *ins_rank, uint64_t m, uint8_t *nkeys,
                                 uint8_t *naccts, uint8_t *nsroots, cudaStream_t st) {
    if (n) merge_scatter_base_kernel<<<blocks_for(n, 256), 256, 0, st>>>(keys, accts, sroots, n, ins_incl, del_excl, del, nkeys,
                                                                        naccts, nsroots);
    if (m) merge_scatter_dirty_kernel<<<blocks_for(m, 256), 256, 0, st>>>(dirty_keys, new_accts, new_sroots, lb, kind, ins_rank, m,
                                                                         n, ins_incl, del_excl, nkeys, naccts, nsroots);
    return cudaGetLastError();
}
cudaError_t launch_wavefront_two_stage(const ForestDev &f, uint8_t *accts, uint8_t *sroots, const uint8_t *new_accts,
                                       const uint8_t *new_sroots, const uint32_t *idx, uint64_t m,
                                       const uint32_t *leaf_parent, const uint32_t *node_parent, uint32_t *pending,
                                       uint32_t *dirty_list, uint32_t *dirty_count, uint32_t *handoff_list,
                                       uint32_t *handoff_count, uint64_t max_handoff, uint8_t *root_out, int split_depth,
                                       cudaStream_t st) {
    if (m == 0) return cudaSuccess;
    constexpr int TB = 64;
    auto ka = wavefront_thread_kernel<TB>;
    size_t smem = (size_t)BRANCH_WORDS * TB * 4;
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(ka, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        attr_set = true;
    }
    ka<<<blocks_for(m, TB), TB, smem, st>>>(f, accts, sroots, new_accts, new_sroots, idx, m, leaf_parent, node_parent, pending,
                                            dirty_list, dirty_count, handoff_list, handoff_count, root_out, split_depth);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    constexpr int WARPS = 4;
    unsigned blocks = blocks_for(max_handoff ? max_handoff : 1, WARPS);
    unsigned cap = (unsigned)sms() * 16;
    climb_kernel<WARPS><<<blocks < cap ? blocks : cap, WARPS * 32, 0, st>>>(f, handoff_list, handoff_count, node_parent, pending,
                                                                         dirty_list, dirty_count, root_out);
    return cudaGetLastError();
}
cudaError_t launch_mark_pending(const ForestDev &f, const uint32_t *idx, uint64_t m, const uint32_t *leaf_parent,
                                const uint32_t *node_parent, uint32_t *pending, cudaStream_t st) {
    if (m == 0) return cudaSuccess;
    mark_pending_kernel<<<blocks_for(m, 128), 128, 0, st>>>(f, idx, m, leaf_parent, node_parent, pending);
    return cudaGetLastError();
}
cudaError_t launch_wavefront(const ForestDev &f, uint8_t *accts, uint8_t *sroots, const uint8_t *new_accts,
                             const uint8_t *new_sroots, const uint32_t *idx, uint64_t m, const uint32_t *leaf_parent,
                             const uint32_t *node_parent, uint32_t *pending, uint32_t *dirty_list, uint32_t *dirty_count,
                             uint8_t *root_out, cudaStream_t st) {
    if (m == 0) return cudaSuccess;
    constexpr int WARPS = 4;
    wavefront_kernel<WARPS><<<blocks_for(m, WARPS), WARPS * 32, 0, st>>>(f, accts, sroots, new_accts, new_sroots, idx, m,
                                                                        leaf_parent, node_parent, pending, dirty_list,
                                                                        dirty_count, root_out);
    return cudaGetLastError();
}
cudaError_t launch_stored_flags_subset(const ForestDev &f, const uint32_t *ids, uint32_t count, uint8_t *flags,
                                       uint32_t *n_hashes, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    stored_flags_subset_kernel<<<blocks_for(count, 256), 256, 0, st>>>(f, ids, count, flags, n_hashes);
    return cudaGetLastError();
}
cudaError_t launch_pick_subset(const uint32_t *ids, const uint32_t *prefix, const uint32_t *sel_pos, uint32_t n_sel,
                               uint32_t *out_ids, uint32_t *out_prefix, cudaStream_t st) {
    if (n_sel == 0) return cudaSuccess;
    pick_subset_kernel<<<blocks_for(n_sel, 256), 256, 0, st>>>(ids, prefix, sel_pos, n_sel, out_ids, out_prefix);
    return cudaGetLastError();
}
cudaError_t launch_parent_links(const ForestDev &f, uint32_t n_nodes, uint32_t *leaf_parent, uint32_t *node_parent,
                                cudaStream_t st) {
    if (n_nodes == 0) return cudaSuccess;
    parent_links_kernel<<<blocks_for(n_nodes, 256), 256, 0, st>>>(f, n_nodes, leaf_parent, node_parent);
    return cudaGetLastError();
}
cudaError_t launch_locate(const uint8_t *keys, uint64_t n, const uint8_t *dirty_keys, uint64_t m, uint32_t *idx_out,
                          int *err, cudaStream_t st) {
    if (m == 0) return cudaSuccess;
    locate_kernel<<<blocks_for(m, 128), 128, 0, st>>>(keys, n, dirty_keys, m, idx_out, err);
    return cudaGetLastError();
}
