// tk_dtrie_launchers.cuh — host-side launchers of the dynamic trie / state / proof kernels.
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ launchers
// leaf_trie: trie (segment) of every leaf of a forest build, nullptr for a single trie
cudaError_t launch_dt_convert(const ForestDev &f, uint32_t n_nodes, const uint32_t *leaf_parent, const uint32_t *node_parent,
                              const uint32_t *leaf_trie, const DTrieDev &t, cudaStream_t st) {
    if (f.n) dt_convert_leaves_kernel<<<blocks_for(f.n, 256), 256, 0, st>>>(f.n, leaf_parent, leaf_trie, t);
    if (n_nodes) dt_convert_nodes_kernel<<<blocks_for(n_nodes, 128), 128, 0, st>>>(f, n_nodes, node_parent, leaf_trie, t);
    return cudaGetLastError();
}
cudaError_t launch_dt_leaf_segments(const uint64_t *seg_offsets, uint64_t n_segs, uint64_t n, uint32_t *leaf_trie, cudaStream_t st) {
    if (n) dt_leaf_segments_kernel<<<blocks_for(n, 256), 256, 0, st>>>(seg_offsets, n_segs, n, leaf_trie);
    return cudaGetLastError();
}
cudaError_t launch_dt_locate(const DTrieDev &t, const uint32_t *trie_of_key, const uint8_t *keys, const uint8_t *vals,
                             const uint8_t *flags, uint64_t m, uint8_t *kind, uint32_t *leaf_of, cudaStream_t st) {
    dt_locate_kernel<<<blocks_for(m, 128), 128, 0, st>>>(t, trie_of_key, keys, vals, flags, m, kind, leaf_of);
    return cudaGetLastError();
}
cudaError_t launch_dt_update_detach(const DTrieDev &t, const uint8_t *accts, const uint8_t *sroots, uint64_t m,
                                    const uint8_t *kind, const uint32_t *leaf_of, uint32_t *touched, cudaStream_t st) {
    dt_update_detach_kernel<<<blocks_for(m, 128), 128, 0, st>>>(t, accts, sroots, m, kind, leaf_of, touched);
    return cudaGetLastError();
}
// one collapse round over `list` (count on the device, at most max_count): begin / act / end
cudaError_t launch_dt_collapse_round(const DTrieDev &t, const uint32_t *list, const uint32_t *count_p, uint32_t max_count,
                                     uint8_t *defer, uint32_t *next, uint32_t *next_count, cudaStream_t st) {
    unsigned blocks = blocks_for(max_count, 128);
    dt_round_begin_kernel<<<blocks, 128, 0, st>>>(t, list, count_p);
    dt_round_defer_kernel<<<blocks, 128, 0, st>>>(t, list, count_p, defer);
    dt_collapse_round_kernel<<<blocks, 128, 0, st>>>(t, list, count_p, defer, next, next_count);
    dt_round_end_kernel<<<blocks, 128, 0, st>>>(t, list, count_p);
    return cudaGetLastError();
}
// the whole restructure of a small block in one CTA (dt_restructure_fused_kernel)
cudaError_t launch_dt_restructure_fused(const DTrieDev &t, const uint32_t *trie_of_key, const uint8_t *keys, const uint8_t *vals,
                                        const uint8_t *flags, const uint8_t *sroots, uint32_t m, uint8_t *kind, uint32_t *leaf_of,
                                        uint32_t *list_a, uint32_t *list_b, uint8_t *defer, uint32_t *idx_a, uint32_t *idx_b,
                                        uint64_t *attach, uint8_t *pending, uint32_t max_per_run, cudaStream_t st) {
    dt_restructure_fused_kernel<1024><<<1, 1024, 0, st>>>(t, trie_of_key, keys, vals, flags, sroots, m, kind, leaf_of, list_a, list_b,
                                                         defer, idx_a, idx_b, attach, pending, max_per_run);
    return cudaGetLastError();
}
// one insertion round: attach points of the (remaining) insert entries, then at most max_per_run keys per run
cudaError_t launch_dt_insert(const DTrieDev &t, const uint32_t *trie_of_key, const uint8_t *keys, const uint8_t *vals,
                             const uint8_t *sroots, const uint32_t *ins_idx, const uint32_t *n_ins_p, uint64_t max_ins,
                             uint64_t *attach, uint32_t *leaf_of, uint32_t max_per_run, uint8_t *pending, uint32_t *leftover,
                             cudaStream_t st) {
    unsigned blocks = blocks_for(max_ins, 128);
    dt_insert_locate_kernel<<<blocks, 128, 0, st>>>(t, trie_of_key, keys, ins_idx, n_ins_p, attach);
    dt_insert_runs_kernel<<<blocks, 128, 0, st>>>(t, trie_of_key, keys, vals, sroots, ins_idx, n_ins_p, attach, leaf_of, max_per_run,
                                                  pending, leftover);
    dt_insert_unlock_kernel<<<blocks, 128, 0, st>>>(t, n_ins_p, attach);
    return cudaGetLastError();
}
// mark -> starts -> wavefront -> finish (empty-trie root, recycling of this apply's freed nodes)
__global__ void dt_finish_kernel(DTrieDev t) {
    t.g[DG_NODE_FREE] += t.g[DG_FREED_NOW];
    t.g[DG_FREED_NOW] = 0;
}
// handoff != nullptr selects the two-stage form (thread per seed below split_depth's levels, warps above)
cudaError_t launch_dt_rehash(const DTrieDev &t, uint32_t max_seeds, uint32_t *handoff, uint32_t *handoff_count, int split_depth,
                             bool already_marked, cudaStream_t st) {
    constexpr int WARPS = 4;
    const uint32_t *count_p = t.g + DG_SEEDS;
    unsigned blocks = blocks_for(max_seeds, 128);
    if (!already_marked) {  // (the fused restructure of a small block has done both)
        dt_mark_kernel<<<blocks, 128, 0, st>>>(t, count_p);
        dt_starts_kernel<<<blocks, 128, 0, st>>>(t, count_p);
    }
    unsigned cap = (unsigned)sms() * 16;
    if (handoff == nullptr) {
        unsigned wblocks = blocks_for(max_seeds, WARPS);
        dt_wavefront_kernel<WARPS><<<wblocks < cap ? wblocks : cap, WARPS * 32, 0, st>>>(t, count_p);
        return cudaGetLastError();
    }
    constexpr int TB = 64;
    auto ka = dt_wavefront_thread_kernel<TB>;
    size_t smem = (size_t)BRANCH_WORDS * TB * 4;
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(ka, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        attr_set = true;
    }
    ka<<<blocks_for(max_seeds, TB), TB, smem, st>>>(t, count_p, handoff, handoff_count, split_depth);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    unsigned wblocks = blocks_for(max_seeds, WARPS);
    dt_climb_kernel<WARPS><<<wblocks < cap ? wblocks : cap, WARPS * 32, 0, st>>>(t, handoff, handoff_count);
    return cudaGetLastError();
}
cudaError_t launch_dt_finish(const DTrieDev &t, uint32_t max_freed, cudaStream_t st) {
    if (max_freed) dt_recycle_kernel<<<blocks_for(max_freed, 128), 128, 0, st>>>(t);
    dt_finish_kernel<<<1, 1, 0, st>>>(t);
    return cudaGetLastError();
}
cudaError_t launch_dt_stored_flags(const DTrieDev &t, uint32_t max_built, uint8_t *flags, uint32_t *n_hashes, cudaStream_t st) {
    if (max_built) dt_stored_flags_kernel<<<blocks_for(max_built, 256), 256, 0, st>>>(t, t.g + DG_BUILT, flags, n_hashes);
    return cudaGetLastError();
}
cudaError_t launch_dt_gather_updates(const DTrieDev &t, const uint32_t *stored_ids, uint32_t n_stored,
                                     const uint32_t *hash_prefix_by_record, const UpdatesDev &out, cudaStream_t st) {
    if (n_stored) dt_gather_updates_kernel<<<blocks_for(n_stored, 128), 128, 0, st>>>(t, stored_ids, n_stored, hash_prefix_by_record, out);
    return cudaGetLastError();
}
cudaError_t launch_dt_removed_paths(const DTrieDev &t, uint32_t n_removed, uint8_t *path_len, uint8_t *path_packed,
                                    uint32_t *trie_id, cudaStream_t st) {
    if (n_removed) dt_removed_paths_kernel<<<blocks_for(n_removed, 128), 128, 0, st>>>(t, n_removed, path_len, path_packed, trie_id);
    return cudaGetLastError();
}
cudaError_t launch_dt_wipe_list(const uint8_t *kind, const uint8_t *flags, const uint32_t *leaf_of, uint64_t m, uint32_t *tries,
                                uint32_t *count, cudaStream_t st) {
    if (m) dt_wipe_list_kernel<<<blocks_for(m, 256), 256, 0, st>>>(kind, flags, leaf_of, m, tries, count);
    return cudaGetLastError();
}
cudaError_t launch_dt_wipe_begin(const DTrieDev &t, const uint32_t *tries, const uint32_t *count_p, uint32_t max_count,
                                 cudaStream_t st) {
    if (max_count) dt_wipe_begin_kernel<<<blocks_for(max_count, 128), 128, 0, st>>>(t, tries, count_p);
    return cudaGetLastError();
}
cudaError_t launch_dt_wipe_round(const DTrieDev &t, uint32_t lo, uint32_t hi, cudaStream_t st) {
    if (hi > lo) dt_wipe_round_kernel<<<blocks_for(hi - lo, 128), 128, 0, st>>>(t, lo, hi);
    return cudaGetLastError();
}
cudaError_t launch_dt_expand_tries(const uint64_t *seg_offsets, uint64_t m, const uint8_t *kind, const uint32_t *leaf_of,
                                   uint64_t n_entries, uint32_t *trie_of_key, cudaStream_t st) {
    if (n_entries) dt_expand_tries_kernel<<<blocks_for(n_entries, 256), 256, 0, st>>>(seg_offsets, m, kind, leaf_of, n_entries, trie_of_key);
    return cudaGetLastError();
}
cudaError_t launch_dt_nibble_tries(const uint8_t *keys, uint64_t m, uint32_t *trie_of_key, cudaStream_t st) {
    if (m) dt_nibble_tries_kernel<<<blocks_for(m, 256), 256, 0, st>>>(keys, m, trie_of_key);
    return cudaGetLastError();
}
cudaError_t launch_dt_frontier(const DTrieDev &t, const uint8_t *bucket_roots, FrontierEntryDev *out, cudaStream_t st) {
    dt_frontier_kernel<<<1, 512, 0, st>>>(t, bucket_roots, out);
    return cudaGetLastError();
}
cudaError_t launch_dt_proof_sizes(const DTrieDev &t, const DTrieDev &alt, const uint32_t *trie_of_target, const uint8_t *keys, uint64_t n,
                                  uint32_t *node_count, uint64_t *byte_count, cudaStream_t st) {
    if (n) dt_proof_size_kernel<<<blocks_for(n, 64), 64, 0, st>>>(t, alt, trie_of_target, keys, n, node_count, byte_count);
    return cudaGetLastError();
}
cudaError_t launch_dt_proof_write(const DTrieDev &t, const DTrieDev &alt, const uint32_t *trie_of_target, const uint8_t *keys, uint64_t n,
                                  const uint64_t *node_base, const uint64_t *byte_base, uint8_t *rlp, uint64_t *rlp_offset,
                                  uint8_t *node_depth, uint32_t *node_masks, cudaStream_t st) {
    if (n) dt_proof_write_kernel<<<blocks_for(n, 64), 64, 0, st>>>(t, alt, trie_of_target, keys, n, node_base, byte_base, rlp, rlp_offset, node_depth,
                                                                  node_masks);
    return cudaGetLastError();
}
cudaError_t launch_dt_sharded_proof_sizes(const DTrieDev &t, const ShardRootDev &r, const uint8_t *keys, uint64_t n, uint32_t *node_count,
                                          uint64_t *byte_count, cudaStream_t st) {
    if (n) dt_sharded_proof_size_kernel<<<blocks_for(n, 64), 64, 0, st>>>(t, r, keys, n, node_count, byte_count);
    return cudaGetLastError();
}
cudaError_t launch_dt_sharded_proof_write(const DTrieDev &t, const ShardRootDev &r, const uint8_t *keys, uint64_t n, const uint64_t *node_base,
                                          const uint64_t *byte_base, uint8_t *rlp, uint64_t *rlp_offset, uint8_t *node_depth,
                                          uint32_t *node_masks, cudaStream_t st) {
    if (n) dt_sharded_proof_write_kernel<<<blocks_for(n, 64), 64, 0, st>>>(t, r, keys, n, node_base, byte_base, rlp, rlp_offset, node_depth,
                                                                          node_masks);
    return cudaGetLastError();
}
cudaError_t launch_dt_frontier_masks(const DTrieDev &t, uint16_t *out, cudaStream_t st) {
    dt_frontier_masks_kernel<<<1, 16, 0, st>>>(t, out);
    return cudaGetLastError();
}
cudaError_t launch_root_branch(const FrontierEntryDev *fr, uint8_t *out, cudaStream_t st) {
    root_branch_kernel<<<1, 1, 0, st>>>(fr, out);
    return cudaGetLastError();
}
cudaError_t launch_dt_find_leaves(const DTrieDev &t, const uint8_t *keys, uint64_t n, uint32_t *leaf_out, uint8_t *sroot_out, cudaStream_t st) {
    if (n) dt_find_leaves_kernel<<<blocks_for(n, 128), 128, 0, st>>>(t, keys, n, leaf_out, sroot_out);
    return cudaGetLastError();
}
cudaError_t launch_dt_target_tries(const uint64_t *seg_offsets, uint64_t n_accounts, const uint32_t *leaf_of, uint64_t n_targets,
                                   uint32_t *trie_of_target, cudaStream_t st) {
    if (n_targets) dt_target_tries_kernel<<<blocks_for(n_targets, 256), 256, 0, st>>>(seg_offsets, n_accounts, leaf_of, n_targets, trie_of_target);
    return cudaGetLastError();
}
cudaError_t launch_dt_find_leaf(const DTrieDev &t, const uint8_t *key, uint32_t *out, uint64_t n_copies, cudaStream_t st) {
    if (n_copies) dt_find_leaf_kernel<<<blocks_for(n_copies, 128), 128, 0, st>>>(t, key, out, n_copies);
    return cudaGetLastError();
}

