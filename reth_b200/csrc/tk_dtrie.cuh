// tk_dtrie.cuh — dynamic resident trie: an arena of branch nodes with 16 child slots each, kept in HBM, that takes
// inserts and deletes in place (SURVEY.md §8 f1 "sparse-trie update path" / row a10).
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).
//
// What reth does with ParallelSparseTrie (crates/trie/sparse/src/parallel.rs: update_leaf / remove_leaf, then
// update_subtrie_hashes / root) and, on the database path, with TrieWalker + prefix sets (crates/trie/trie/src/walker.rs
// :161-202): touch only the paths of the changed keys.  Here:
//   * a child word is NONE, a leaf id (DT_LEAF set) or a node id; extension nodes stay implicit (a node whose parent
//     is more than one nibble shallower), exactly as in the level-synchronous builder;
//   * every phase is its own launch and is written so that concurrent threads never touch the same word:
//       locate        read-only descent per dirty key
//       update/detach value writes to found leaves; deleted leaves leave their parent's slot (distinct slots)
//       collapse      rounds over the nodes that lost children: a node acts only if its parent is not in the same
//                     round (so the acting nodes are never adjacent); 0 children -> the node leaves its parent,
//                     1 child -> the child moves up (path compression), >= 2 -> the node is just dirty
//       insert        keys that attach at the same (parent, slot) form a run of the sorted dirty list; one thread
//                     inserts a run serially, so different threads work in disjoint subtrees
//       mark / wavefront   dirty leaves and nodes are seeds; pending[] counts dirty children; the last dirty child
//                     to arrive re-hashes the parent (same scheme as tk_wavefront.cuh)
//   * stored-node changes are reported as reth's TrieUpdates: re-hashed nodes with tree|hash mask != 0 are "updated",
//     freed nodes and nodes whose masks became empty are "removed" (crates/trie/common/src/updates.rs:17-26).

// ------------------------------------------------------------------------------------------------ helpers
static __device__ __forceinline__ uint32_t dt_nib(const uint8_t *key, uint32_t i) { return key_nibble_mem(key, i); }

// common prefix of two keys in nibbles, at most `limit`, knowing the first `from` nibbles agree
static __device__ __forceinline__ uint32_t dt_lcp(const uint8_t *a, const uint8_t *b, uint32_t from, uint32_t limit) {
    uint32_t i = from & ~1u;
    for (; i < limit; i += 2) {
        uint32_t x = a[i >> 1] ^ b[i >> 1];
        if (x) {
            uint32_t l = (x & 0xF0) ? i : i + 1;
            return l < limit ? l : limit;
        }
    }
    return limit;
}

static __device__ __forceinline__ void dt_copy32(uint8_t *dst, const uint8_t *src) {
    const uint4 *s = reinterpret_cast<const uint4 *>(src);
    uint4 *d = reinterpret_cast<uint4 *>(dst);
    d[0] = s[0];
    d[1] = s[1];
}
static __device__ __forceinline__ void dt_copy72(uint8_t *dst, const uint8_t *src) {
    const uint64_t *s = reinterpret_cast<const uint64_t *>(src);
    uint64_t *d = reinterpret_cast<uint64_t *>(dst);
#pragma unroll
    for (int w = 0; w < 9; w++) d[w] = s[w];
}

static __device__ __forceinline__ uint32_t dt_trie_of(const DTrieDev &t, uint32_t word) {
    if (!t.ltrie) return 0;
    return (word & DT_LEAF) ? t.ltrie[word & ~DT_LEAF] : t.ntrie[word];
}
static __device__ __forceinline__ void dt_put_empty_root(uint8_t *dst) {  // EMPTY_ROOT_HASH
    uint32_t *w = reinterpret_cast<uint32_t *>(dst);
    w[0] = 0x171fe856u; w[1] = 0xa655cc1bu; w[2] = 0xe64583ffu; w[3] = 0x6ef8c092u;
    w[4] = 0x1be0485bu; w[5] = 0xc0ad6c99u; w[6] = 0xb52f6201u; w[7] = 0x21b463e3u;
}
// parent == NONE addresses the root word of `trie`; a trie that becomes empty gets EMPTY_ROOT_HASH as its root right
// away (no wavefront will visit it)
static __device__ __forceinline__ void dt_set_child(const DTrieDev &t, uint32_t trie, uint32_t parent, uint32_t slot, uint32_t word) {
    if (parent == DT_NONE) {
        t.troot[trie] = word;
        if (word == DT_NONE) dt_put_empty_root(t.top_out + (uint64_t)t.top_stride * trie);
    } else {
        t.nchild[16 * (uint64_t)parent + slot] = word;
    }
}
static __device__ __forceinline__ void dt_copy_val(const DTrieDev &t, uint32_t x, const uint8_t *src) {
    if (t.account) dt_copy72(t.lval + 72 * (uint64_t)x, src);
    else dt_copy32(t.lval + 32 * (uint64_t)x, src);
}
static __device__ __forceinline__ void dt_set_parent(const DTrieDev &t, uint32_t word, uint32_t parent) {
    if (word & DT_LEAF) t.lparent[word & ~DT_LEAF] = parent;
    else t.nparent[word] = parent;
}
// exact test-and-set on a byte-flag array (the flag arrays are 4-byte aligned)
static __device__ __forceinline__ bool dt_test_and_set(uint8_t *base, uint32_t idx) {
    unsigned int *w = reinterpret_cast<unsigned int *>(base + (idx & ~3u));
    unsigned int bit = 1u << (8 * (idx & 3u));
    return (atomicOr(w, bit) & bit) != 0;
}
// a dirty item: must be re-hashed even if nothing below it changed
static __device__ __forceinline__ void dt_seed(const DTrieDev &t, uint32_t word) {
    bool was = (word & DT_LEAF) ? dt_test_and_set(t.lseed, word & ~DT_LEAF) : dt_test_and_set(t.nseed, word);
    if (!was) t.seeds[atomicAdd(&t.g[DG_SEEDS], 1u)] = word;
}

// Pop of a free stack, or a fresh slot from the bump region when it is empty.  Only pops run side by side (the kernels that
// push — detach, collapse, wipe, recycle — are other launches / other phases of the fused kernel), so one atomic does: a
// count driven below zero means "empty" and is put back to zero by dt_pop_settle once the phase is over.  (A CAS loop here
// serialised the ~30 000 allocations of a block on one L2 round trip each.)
static __device__ __forceinline__ uint32_t dt_pop(uint32_t *count, const uint32_t *stack, uint32_t *bump) {
    int c = (int)atomicSub(count, 1u);
    if (c > 0) return stack[c - 1];
    return atomicAdd(bump, 1u);
}
static __device__ __forceinline__ void dt_pop_settle(const DTrieDev &t) {  // one thread, after every pop of the phase
    if ((int)t.g[DG_LEAF_FREE] < 0) t.g[DG_LEAF_FREE] = 0;
    if ((int)t.g[DG_NODE_FREE] < 0) t.g[DG_NODE_FREE] = 0;
}
static __device__ __forceinline__ uint32_t dt_alloc_leaf(const DTrieDev &t) {
    // (the seed flag of a free slot is already clear: dt_starts_kernel clears every flag it listed, fresh capacity is
    // zero-filled; no plain store here, other threads of this kernel update neighbouring flags with atomics)
    return dt_pop(&t.g[DG_LEAF_FREE], t.leaf_free, &t.g[DG_LEAF_ALLOC]);
}
static __device__ __forceinline__ uint32_t dt_alloc_node(const DTrieDev &t, uint32_t trie, uint32_t depth, const uint8_t *key,
                                                        uint32_t parent) {
    uint32_t v = dt_pop(&t.g[DG_NODE_FREE], t.node_free, &t.g[DG_NODE_ALLOC]);
    if (t.ntrie) t.ntrie[v] = trie;
    uint4 none = make_uint4(DT_NONE, DT_NONE, DT_NONE, DT_NONE);
    uint4 *ch = reinterpret_cast<uint4 *>(t.nchild + 16 * (uint64_t)v);
    ch[0] = none; ch[1] = none; ch[2] = none; ch[3] = none;
    t.ndepth[v] = (uint8_t)depth;
    t.nparent[v] = parent;
    t.nmeta[v] = 0;
    t.nmasks[v] = make_ushort4(0, 0, 0, (unsigned short)depth);
    dt_copy32(t.nkey + 32 * (uint64_t)v, key);
    t.npending[v] = 0;  // (nseed / ncur / nnext of a free slot are clear already, see dt_alloc_leaf)
    return v;
}
// A stored node that ceases to exist (or to be stored) is one of reth's removed_nodes; its path is read from nkey /
// nmasks.w when the apply gathers its output, so a freed slot is only recycled after that (freed_now list).
static __device__ __forceinline__ void dt_record_removed(const DTrieDev &t, uint32_t v) {
    if (t.nmasks[v].w == 0) return;  // the empty path is never stored (updates.rs:140-158)
    t.removed[atomicAdd(&t.g[DG_REMOVED], 1u)] = v;
}
static __device__ __forceinline__ void dt_free_node(const DTrieDev &t, uint32_t v) {
    if (t.nmeta[v] & META_STORED) dt_record_removed(t, v);
    t.ndepth[v] = DT_DEAD;
    t.nmeta[v] = 0;
    t.freed_now[atomicAdd(&t.g[DG_FREED_NOW], 1u)] = v;
}
__global__ void dt_recycle_kernel(DTrieDev t) {  // end of an apply: this apply's freed nodes become allocatable
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.g[DG_FREED_NOW]) return;
    t.node_free[t.g[DG_NODE_FREE] + i] = t.freed_now[i];
}
// byte b of the first d nibbles of key, packed high-first and zero padded (the path layout of b200_updates)
static __device__ __forceinline__ uint8_t dt_path_byte(const uint8_t *key, uint32_t d, uint32_t b) {
    return (uint8_t)(2 * b + 1 < d ? key[b] : (2 * b < d ? (key[b] & 0xF0) : 0));
}
static __device__ __forceinline__ void dt_pack_path(const uint8_t *key, uint32_t d, uint8_t *pp) {
    for (uint32_t b = 0; b < 32; b++) pp[b] = dt_path_byte(key, d, b);
}
__global__ void dt_removed_paths_kernel(DTrieDev t, uint32_t n_removed, uint8_t *__restrict__ path_len, uint8_t *__restrict__ path_packed,
                                        uint32_t *__restrict__ trie_id) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_removed) return;
    uint32_t v = t.removed[i];
    uint32_t d = t.nmasks[v].w;
    dt_pack_path(t.nkey + 32 * (uint64_t)v, d, path_packed + 32 * (uint64_t)i);
    path_len[i] = (uint8_t)d;
    trie_id[i] = t.ntrie ? t.ntrie[v] : 0;
}

// ------------------------------------------------------------------------------------------------ create
// Conversion of a finished level-synchronous build (ForestDev, one trie) into the arena: node ids and leaf ids carry
// over unchanged.
__global__ void dt_convert_nodes_kernel(ForestDev f, uint32_t n_nodes, const uint32_t *__restrict__ node_parent,
                                        const uint32_t *__restrict__ leaf_trie, DTrieDev t) {
    uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_nodes) return;
    uint32_t j0 = f.node_start[v], k = f.node_start[v + 1] - j0;
    uint32_t *ch = t.nchild + 16 * (uint64_t)v;
    for (int s = 0; s < 16; s++) ch[s] = DT_NONE;
    for (uint32_t c = 0; c <= k; c++) {
        ChildInfo ci = fetch_child(f, j0, c);
        ch[ci.nib] = ci.id < f.n ? (ci.id | DT_LEAF) : ci.id - (uint32_t)f.n;
    }
    ushort4 m = f.node_masks[v];
    t.ndepth[v] = (uint8_t)m.w;
    t.nmasks[v] = m;
    t.nparent[v] = node_parent[v];
    t.nmeta[v] = f.node_meta[v];
    dt_copy32(t.nref + 32 * (uint64_t)v, f.node_ref + 32 * (uint64_t)v);
    dt_copy32(t.nkey + 32 * (uint64_t)v, f.keys + 32 * (uint64_t)f.node_l[v]);
    t.npending[v] = 0;
    t.nseed[v] = 0;
    t.ncur[v] = 0;
    t.nnext[v] = 0;
    uint32_t trie = leaf_trie ? leaf_trie[f.node_l[v]] : 0;
    if (t.ntrie) t.ntrie[v] = trie;
    if (node_parent[v] == DT_NONE) t.troot[trie] = v;
}
// single-leaf tries: the root word is the leaf itself (leaf_parent == NONE)
__global__ void dt_convert_leaves_kernel(uint64_t n, const uint32_t *__restrict__ leaf_parent, const uint32_t *__restrict__ leaf_trie,
                                         DTrieDev t) {
    uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= n) return;
    uint32_t trie = leaf_trie ? leaf_trie[x] : 0;
    if (t.ltrie) t.ltrie[x] = trie;
    t.lparent[x] = leaf_parent[x];
    if (leaf_parent[x] == DT_NONE) t.troot[trie] = (uint32_t)x | DT_LEAF;
}
// leaf_trie[x] = segment (trie) of leaf x of a forest build
__global__ void dt_leaf_segments_kernel(const uint64_t *__restrict__ seg_offsets, uint64_t n_segs, uint64_t n, uint32_t *__restrict__ leaf_trie) {
    uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= n) return;
    uint64_t lo = 0, hi = n_segs;  // last segment with offset <= x
    while (hi - lo > 1) {
        uint64_t mid = (lo + hi) >> 1;
        if (seg_offsets[mid] <= x) lo = mid;
        else hi = mid;
    }
    leaf_trie[x] = (uint32_t)lo;
}

// ------------------------------------------------------------------------------------------------ locate

struct DtLoc {
    uint32_t parent, slot, child;  // attach point and what hangs there now
    bool found;                    // child is the leaf holding exactly this key
};
static __device__ __forceinline__ DtLoc dt_descend(const DTrieDev &t, uint32_t trie, const uint8_t *key) {
    DtLoc r;
    r.parent = DT_NONE;
    r.slot = 0;
    r.found = false;
    uint32_t cur = t.troot[trie];
    uint32_t matched = 0;  // nibbles known to agree with everything below `cur`
    for (int hops = 0;; hops++) {
        if (hops > DT_MAX_HOPS) {  // depth grows with every hop: more than 64 means a damaged structure, never a long path
            atomicExch(t.err, B200_DEVERR_CORRUPT);
            r.child = DT_NONE;
            return r;
        }
        r.child = cur;
        if (cur == DT_NONE) return r;
        if (cur & DT_LEAF) {
            r.found = dt_lcp(key, t.lkey + 32 * (uint64_t)(cur & ~DT_LEAF), matched, 64) == 64;
            return r;
        }
        uint32_t d = t.ndepth[cur];
        if (dt_lcp(key, t.nkey + 32 * (uint64_t)cur, matched, d) < d) return r;  // diverges inside the edge above `cur`
        r.parent = cur;
        r.slot = dt_nib(key, d);
        matched = d + 1;
        cur = t.nchild[16 * (uint64_t)cur + r.slot];
    }
}

// flags[i] (accounts): bit 0 = present (0 deletes), bit 1 = touch only (the leaf's data is unchanged but it must be
// re-hashed: its storage root changes); nullptr = all present.  Storage slots: a zero value deletes.
// trie_of_key (forest arenas): the trie each key belongs to, DT_NONE = skip the entry.
static __device__ __forceinline__ void dt_locate_entry(const DTrieDev &t, const uint32_t *__restrict__ trie_of_key,
                                                       const uint8_t *__restrict__ keys, const uint8_t *__restrict__ vals,
                                                       const uint8_t *__restrict__ flags, uint64_t i, uint8_t *__restrict__ kind,
                                                       uint32_t *__restrict__ leaf_of) {
    const uint32_t trie = trie_of_key ? trie_of_key[i] : 0;
    if (trie == DT_NONE) {
        kind[i] = DK_NOOP;
        leaf_of[i] = DT_NONE;
        return;
    }
    if (i && (!trie_of_key || trie_of_key[i - 1] == trie)) {  // strictly ascending inside a trie: the insert runs rely on it
        const uint8_t *a = keys + 32 * (i - 1), *b = keys + 32 * i;
        uint32_t l = dt_lcp(a, b, 0, 64);
        if (l == 64 || dt_nib(a, l) > dt_nib(b, l)) atomicExch(t.err, B200_DEVERR_UNSORTED);
    }
    DtLoc loc = dt_descend(t, trie, keys + 32 * i);
    bool want, touch = false;
    if (t.account) {
        want = flags == nullptr || (flags[i] & 1);
        touch = flags != nullptr && (flags[i] & 2);
    } else {
        const uint64_t *v = reinterpret_cast<const uint64_t *>(vals + 32 * i);
        want = (v[0] | v[1] | v[2] | v[3]) != 0;
    }
    uint8_t k;
    if (touch) k = (want && loc.found) ? DK_TOUCH : DK_NOOP;
    else k = loc.found ? (want ? DK_UPDATE : DK_DELETE) : (want ? DK_INSERT : DK_NOOP);
    kind[i] = k;
    leaf_of[i] = loc.found ? (loc.child & ~DT_LEAF) : DT_NONE;
}
__global__ void dt_locate_kernel(DTrieDev t, const uint32_t *__restrict__ trie_of_key, const uint8_t *__restrict__ keys,
                                 const uint8_t *__restrict__ vals, const uint8_t *__restrict__ flags, uint64_t m,
                                 uint8_t *__restrict__ kind, uint32_t *__restrict__ leaf_of) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) dt_locate_entry(t, trie_of_key, keys, vals, flags, i, kind, leaf_of);
}

// value changes of existing leaves; deleted leaves leave their parent's slot
static __device__ __forceinline__ void dt_update_detach_entry(const DTrieDev &t, const uint8_t *__restrict__ vals,
                                                              const uint8_t *__restrict__ sroots, uint64_t i,
                                                              const uint8_t *__restrict__ kind, const uint32_t *__restrict__ leaf_of,
                                                              uint32_t *__restrict__ touched) {
    uint32_t x = leaf_of[i];
    if (kind[i] == DK_UPDATE) {
        dt_copy_val(t, x, vals + (uint64_t)t.val_stride * i);
        if (sroots && t.lsroot) dt_copy32(t.lsroot + 32 * (uint64_t)x, sroots + 32 * i);
        dt_seed(t, x | DT_LEAF);
    } else if (kind[i] == DK_TOUCH) {
        dt_seed(t, x | DT_LEAF);
    } else if (kind[i] == DK_DELETE) {
        uint32_t p = t.lparent[x];
        if (p == DT_NONE) {
            dt_set_child(t, dt_trie_of(t, x | DT_LEAF), DT_NONE, 0, DT_NONE);
        } else {
            t.nchild[16 * (uint64_t)p + dt_nib(t.lkey + 32 * (uint64_t)x, t.ndepth[p])] = DT_NONE;
            if (!dt_test_and_set(t.nnext, p)) touched[atomicAdd(&t.g[DG_LIST_A], 1u)] = p;
        }
        t.lmeta[x] = DT_DEAD;
        t.leaf_free[atomicAdd(&t.g[DG_LEAF_FREE], 1u)] = x;
        atomicSub(&t.g[DG_NLEAVES], 1u);
    }
}
__global__ void dt_update_detach_kernel(DTrieDev t, const uint8_t *__restrict__ vals, const uint8_t *__restrict__ sroots,
                                        uint64_t m, const uint8_t *__restrict__ kind, const uint32_t *__restrict__ leaf_of,
                                        uint32_t *__restrict__ touched) {
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) dt_update_detach_entry(t, vals, sroots, i, kind, leaf_of, touched);
}

// ------------------------------------------------------------------------------------------------ collapse rounds
// ncur = member of the round being processed, nnext = already listed for the following round
__global__ void dt_round_begin_kernel(DTrieDev t, const uint32_t *__restrict__ list, const uint32_t *__restrict__ count_p) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *count_p) return;
    uint32_t v = list[i];
    t.ncur[v] = 1;
    t.nnext[v] = 0;
}
// snapshot of "my parent is a member of this round", taken before anybody acts: the decision must not depend on
// parent links that an acting node re-writes during the round
__global__ void dt_round_defer_kernel(DTrieDev t, const uint32_t *__restrict__ list, const uint32_t *__restrict__ count_p,
                                      uint8_t *__restrict__ defer) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *count_p) return;
    uint32_t v = list[i];
    uint32_t gp = t.ndepth[v] == DT_DEAD ? DT_NONE : t.nparent[v];
    defer[i] = (gp != DT_NONE && t.ncur[gp]) ? 1 : 0;
}
__global__ void dt_round_end_kernel(DTrieDev t, const uint32_t *__restrict__ list, const uint32_t *__restrict__ count_p) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *count_p) return;
    t.ncur[list[i]] = 0;
}

// One round over the nodes that lost children.  ncur marks the members of this round; a node whose parent was a
// member when the round began waits for the next round, so two acting nodes are never parent and child and every
// word has one writer.
static __device__ __forceinline__ void dt_collapse_entry(const DTrieDev &t, const uint32_t *__restrict__ list, uint32_t i,
                                                         const uint8_t *__restrict__ defer, uint32_t *__restrict__ next,
                                                         uint32_t *next_count) {
    uint32_t v = list[i];
    if (t.ndepth[v] == DT_DEAD) return;
    uint32_t gp = t.nparent[v];
    auto push_next = [&](uint32_t node) {
        if (!dt_test_and_set(t.nnext, node)) next[atomicAdd(next_count, 1u)] = node;
    };
    if (defer[i]) {
        push_next(v);
        return;
    }
    const uint32_t *ch = t.nchild + 16 * (uint64_t)v;
    uint32_t cnt = 0, only = DT_NONE;
    for (int s = 0; s < 16; s++)
        if (ch[s] != DT_NONE) {
            cnt++;
            only = ch[s];
        }
    if (cnt >= 2) {
        dt_seed(t, v);
        return;
    }
    uint32_t slot = gp == DT_NONE ? 0 : dt_nib(t.nkey + 32 * (uint64_t)v, t.ndepth[gp]);
    const uint32_t trie = dt_trie_of(t, v);
    if (cnt == 1) {  // path compression: the only child takes this node's place
        dt_set_child(t, trie, gp, slot, only);
        dt_set_parent(t, only, gp);
        dt_seed(t, only);  // its parent depth changed: the leaf path / extension above it is different now
    } else {
        dt_set_child(t, trie, gp, slot, DT_NONE);
        if (gp != DT_NONE) push_next(gp);
    }
    dt_free_node(t, v);
}
__global__ void dt_collapse_round_kernel(DTrieDev t, const uint32_t *__restrict__ list, const uint32_t *__restrict__ count_p,
                                         const uint8_t *__restrict__ defer, uint32_t *__restrict__ next, uint32_t *next_count) {
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < *count_p) dt_collapse_entry(t, list, i, defer, next, next_count);
}

// ------------------------------------------------------------------------------------------------ insert
// attach[j] identifies where insert key j hangs in the structure left by the deletes: (parent << 4 | slot), or, at a
// trie's root word, (1 << 63 | trie).  Keys with equal attach words are consecutive (same trie, same leading prefix).
static __device__ __forceinline__ void dt_insert_locate_entry(const DTrieDev &t, const uint32_t *__restrict__ trie_of_key,
                                                              const uint8_t *__restrict__ keys, const uint32_t *__restrict__ ins_idx,
                                                              uint32_t j, uint64_t *__restrict__ attach) {
    const uint32_t i = ins_idx[j];
    const uint32_t trie = trie_of_key ? trie_of_key[i] : 0;
    DtLoc loc = dt_descend(t, trie, keys + 32 * (uint64_t)i);
    attach[j] = loc.parent == DT_NONE ? ((1ull << 63) | trie) : (((uint64_t)loc.parent << 4) | loc.slot);
}
__global__ void dt_insert_locate_kernel(DTrieDev t, const uint32_t *__restrict__ trie_of_key, const uint8_t *__restrict__ keys,
                                        const uint32_t *__restrict__ ins_idx, const uint32_t *__restrict__ n_ins_p,
                                        uint64_t *__restrict__ attach) {
    uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < *n_ins_p) dt_insert_locate_entry(t, trie_of_key, keys, ins_idx, j, attach);
}

// returns the id of the new leaf.  `top` is the value of the attach word (the child word at (parent, slot), or the trie's
// root word): the run that owns the attach point keeps it in a register — the word in memory holds DT_LOCKED for the
// whole round — and stores the final value afterwards (dt_insert_unlock_entry).
static __device__ __forceinline__ uint32_t dt_insert_one(const DTrieDev &t, uint32_t trie, const uint8_t *key, const uint8_t *val,
                                                         const uint8_t *sroot, uint32_t parent, uint32_t slot, uint32_t &top) {
    uint32_t matched = parent == DT_NONE ? 0 : (uint32_t)t.ndepth[parent] + 1;
    uint32_t cur = top;
    bool at_top = true;  // `cur` is the attach word itself: updates go to `top`, not to memory
    // the new leaf
    uint32_t x = dt_alloc_leaf(t);
    dt_copy32(t.lkey + 32 * (uint64_t)x, key);
    dt_copy_val(t, x, val);
    if (t.ltrie) t.ltrie[x] = trie;
    if (t.lsroot) {
        if (sroot) dt_copy32(t.lsroot + 32 * (uint64_t)x, sroot);
        else dt_put_empty_root(t.lsroot + 32 * (uint64_t)x);
    }
    t.lmeta[x] = 0;
    atomicAdd(&t.g[DG_NLEAVES], 1u);
    for (int hops = 0;; hops++) {
        if (hops > DT_MAX_HOPS) {
            atomicExch(t.err, B200_DEVERR_CORRUPT);
            break;
        }
        if (cur == DT_NONE) {
            if (at_top) top = x | DT_LEAF;
            else dt_set_child(t, trie, parent, slot, x | DT_LEAF);
            t.lparent[x] = parent;
            break;
        }
        const uint8_t *other = (cur & DT_LEAF) ? t.lkey + 32 * (uint64_t)(cur & ~DT_LEAF) : t.nkey + 32 * (uint64_t)cur;
        uint32_t limit = (cur & DT_LEAF) ? 64u : (uint32_t)t.ndepth[cur];
        uint32_t l = dt_lcp(key, other, matched, limit);
        if (l < limit) {  // diverges above `cur`: a new branch at depth l holds both
            uint32_t b = dt_alloc_node(t, trie, l, key, parent);
            t.nchild[16 * (uint64_t)b + dt_nib(key, l)] = x | DT_LEAF;
            t.nchild[16 * (uint64_t)b + dt_nib(other, l)] = cur;
            t.lparent[x] = b;
            dt_set_parent(t, cur, b);
            if (at_top) top = b;
            else dt_set_child(t, trie, parent, slot, b);
            dt_seed(t, b);
            dt_seed(t, cur);  // parent depth changed
            break;
        }
        // (a leaf can never match all 64 nibbles here: the key is new)
        parent = cur;
        slot = dt_nib(key, limit);
        matched = limit + 1;
        cur = t.nchild[16 * (uint64_t)cur + slot];
        at_top = false;
    }
    dt_seed(t, x | DT_LEAF);
    return x;
}

// One thread per run inserts its first `max_per_run` keys; the rest of a long run is left for the next round, by which
// time the keys just inserted have fanned the attach point out into up to 16 deeper ones per level — a run of r keys
// needs ~log(r) rounds instead of r serial inserts (a new contract with 100k slots, a bulk load into an empty trie).
// pending[j] = 1 for every entry that is still to be inserted; *leftover counts them.
//
// The keys of one attach point are NOT always neighbours in the sorted list: with K1 < K2 < K3, K1 and K3 can both diverge
// inside the edge above a node N (same attach word) while K2 matches that edge and attaches below N — long edges (clustered
// keys, small storage tries) make that common.  Two heads with the same attach word must not work concurrently, so a head
// takes the attach word itself as the lock: atomicExch(word, DT_LOCKED).  The winner keeps the word's value in a register
// and leaves DT_LOCKED in memory until the round is over (t.unlock[j] = the final value, stored by dt_insert_unlock_entry
// after the barrier / kernel boundary); a head that finds DT_LOCKED leaves its keys for the next round.  Nothing else reads
// an attach word during this phase: descents happen in the locate phase, and runs below N start from their own attach word.
static __device__ __forceinline__ uint32_t *dt_attach_word(const DTrieDev &t, uint64_t a) {
    return (a >> 63) ? t.troot + (uint32_t)a : t.nchild + a;  // (parent << 4 | slot) == 16 * parent + slot
}
static __device__ __forceinline__ void dt_insert_run_entry(const DTrieDev &t, const uint32_t *__restrict__ trie_of_key,
                                                           const uint8_t *__restrict__ keys, const uint8_t *__restrict__ vals,
                                                           const uint8_t *__restrict__ sroots, const uint32_t *__restrict__ ins_idx,
                                                           uint32_t n_ins, uint32_t j, const uint64_t *__restrict__ attach,
                                                           uint32_t *__restrict__ leaf_of, uint32_t max_per_run,
                                                           uint8_t *__restrict__ pending, uint32_t *__restrict__ leftover) {
    t.unlock[j] = DT_LOCKED;  // nothing to store back for this entry (unless it turns out to own an attach word)
    uint64_t a = attach[j];
    if (j && attach[j - 1] == a) return;  // not the head of its run
    const bool at_root = (a >> 63) != 0;
    uint32_t parent = at_root ? DT_NONE : (uint32_t)(a >> 4), slot = at_root ? 0u : (uint32_t)(a & 15);
    uint32_t top = atomicExch(dt_attach_word(t, a), DT_LOCKED);
    const bool owner = top != DT_LOCKED;
    uint32_t done = 0, left = 0;
    for (uint32_t q = j; q < n_ins && attach[q] == a; q++) {
        if (!owner || done == max_per_run) {
            pending[q] = 1;
            left++;
            continue;
        }
        uint64_t i = ins_idx[q];
        uint32_t trie = trie_of_key ? trie_of_key[i] : 0;
        leaf_of[i] = dt_insert_one(t, trie, keys + 32 * i, vals + (uint64_t)t.val_stride * i, sroots ? sroots + 32 * i : nullptr,
                                   parent, slot, top);
        pending[q] = 0;
        done++;
    }
    if (owner) t.unlock[j] = top;
    if (left) atomicAdd(leftover, left);
}
// after every head of the round has run: the owners store the final value of their attach word (never DT_LOCKED)
static __device__ __forceinline__ void dt_insert_unlock_entry(const DTrieDev &t, uint32_t j, const uint64_t *__restrict__ attach) {
    uint32_t v = t.unlock[j];
    if (v != DT_LOCKED) *dt_attach_word(t, attach[j]) = v;
}
__global__ void dt_insert_runs_kernel(DTrieDev t, const uint32_t *__restrict__ trie_of_key, const uint8_t *__restrict__ keys,
                                      const uint8_t *__restrict__ vals, const uint8_t *__restrict__ sroots,
                                      const uint32_t *__restrict__ ins_idx, const uint32_t *__restrict__ n_ins_p,
                                      const uint64_t *__restrict__ attach, uint32_t *__restrict__ leaf_of, uint32_t max_per_run,
                                      uint8_t *__restrict__ pending, uint32_t *__restrict__ leftover) {
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;
    const uint32_t n_ins = *n_ins_p;
    uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n_ins) dt_insert_run_entry(t, trie_of_key, keys, vals, sroots, ins_idx, n_ins, j, attach, leaf_of, max_per_run, pending, leftover);
}
__global__ void dt_insert_unlock_kernel(DTrieDev t, const uint32_t *__restrict__ n_ins_p, const uint64_t *__restrict__ attach) {
    uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j == 0) dt_pop_settle(t);
    if (j < *n_ins_p) dt_insert_unlock_entry(t, j, attach);
}

// ------------------------------------------------------------------------------------------------ mark + wavefront
static __device__ __forceinline__ bool dt_alive(const DTrieDev &t, uint32_t word) {
    return (word & DT_LEAF) ? t.lmeta[word & ~DT_LEAF] != DT_DEAD : t.ndepth[word] != DT_DEAD;
}
static __device__ __forceinline__ uint32_t dt_parent_of(const DTrieDev &t, uint32_t word) {
    return (word & DT_LEAF) ? t.lparent[word & ~DT_LEAF] : t.nparent[word];
}

// pending[p] = number of dirty children of p.  A walk stops at the first ancestor somebody already reached, and at a
// seed (which walks on its own behalf).
static __device__ __forceinline__ void dt_mark_entry(const DTrieDev &t, uint32_t i) {
    uint32_t s = t.seeds[i];
    if (!dt_alive(t, s)) return;
    uint32_t p = dt_parent_of(t, s);
    for (int hops = 0; p != DT_NONE; hops++) {
        if (hops > DT_MAX_HOPS) {
            atomicExch(t.err, B200_DEVERR_CORRUPT);
            break;
        }
        if (atomicAdd(&t.npending[p], 1u) != 0u) break;
        if (t.nseed[p]) break;
        p = t.nparent[p];
    }
}
__global__ void dt_mark_kernel(DTrieDev t, const uint32_t *__restrict__ count_p) {
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < *count_p) dt_mark_entry(t, i);
}

// After marking: clears the seed flags and keeps only the wavefront's starting points in the list — live leaves, and
// live nodes without a dirty child (a seed node that has dirty children is re-hashed by the last of them to arrive).
static __device__ __forceinline__ void dt_starts_entry(const DTrieDev &t, uint32_t i) {
    uint32_t s = t.seeds[i];
    if (s & DT_LEAF) {
        t.lseed[s & ~DT_LEAF] = 0;
        if (t.lmeta[s & ~DT_LEAF] == DT_DEAD) t.seeds[i] = DT_NONE;
    } else {
        t.nseed[s] = 0;
        if (t.ndepth[s] == DT_DEAD || t.npending[s] != 0u) t.seeds[i] = DT_NONE;
    }
}
__global__ void dt_starts_kernel(DTrieDev t, const uint32_t *__restrict__ count_p) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < *count_p) dt_starts_entry(t, i);
}

// ------------------------------------------------------------------------------------------------ fused restructure
// Small blocks (the live path: a few hundred accounts, a few thousand slots) are latency-bound by launches and host round
// trips, not by work.  One CTA runs the whole restructure — locate, update / detach, every collapse round, every insert
// round, then mark / starts — with __syncthreads where the multi-launch form has kernel boundaries and host-driven
// loops; the phase bodies are the same device functions.  Ordered compaction (the insert lists must stay sorted) is a block-wide scan.
template <int BLOCK>
static __device__ __forceinline__ uint32_t dt_block_exclusive_scan(uint32_t v, uint32_t *sh /* BLOCK/32 + 1 */, uint32_t &total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += up;
    }
    if (lane == 31) sh[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < BLOCK / 32 ? sh[lane] : 0, wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t up = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += up;
        }
        if (lane < BLOCK / 32) sh[lane] = wi - w;  // exclusive offset of every warp
        if (lane == 31) sh[BLOCK / 32] = wi;      // grand total
    }
    __syncthreads();
    uint32_t res = sh[warp] + incl - v;
    total = sh[BLOCK / 32];
    __syncthreads();  // sh is reused by the next call
    return res;
}
// dst[0 .. count) = the src entries (positions 0 .. n) whose flag is set, order kept; returns count
template <int BLOCK, class FlagOf>
static __device__ __forceinline__ uint32_t dt_block_compact(const uint32_t *src, bool identity, uint32_t n, FlagOf flag_of,
                                                            uint32_t *dst, uint32_t *sh) {
    uint32_t base = 0;
    for (uint32_t lo = 0; lo < n; lo += BLOCK) {
        uint32_t j = lo + threadIdx.x;
        uint32_t f = j < n && flag_of(j) ? 1u : 0u, total;
        uint32_t pos = dt_block_exclusive_scan<BLOCK>(f, sh, total);
        if (f) dst[base + pos] = identity ? j : src[j];
        base += total;
    }
    __syncthreads();
    return base;
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) dt_restructure_fused_kernel(DTrieDev t, const uint32_t *__restrict__ trie_of_key,
                                                                    const uint8_t *__restrict__ keys, const uint8_t *__restrict__ vals,
                                                                    const uint8_t *__restrict__ flags, const uint8_t *__restrict__ sroots,
                                                                    uint32_t m, uint8_t *__restrict__ kind, uint32_t *__restrict__ leaf_of,
                                                                    uint32_t *list_a, uint32_t *list_b, uint8_t *__restrict__ defer,
                                                                    uint32_t *idx_a, uint32_t *idx_b, uint64_t *__restrict__ attach,
                                                                    uint8_t *__restrict__ pending, uint32_t max_per_run) {
    __shared__ uint32_t sh[BLOCK / 32 + 1];
    __shared__ uint32_t s_count;
    const uint32_t tid = threadIdx.x;
    // ---- locate
    for (uint32_t i = tid; i < m; i += BLOCK) dt_locate_entry(t, trie_of_key, keys, vals, flags, i, kind, leaf_of);
    __syncthreads();
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;  // uniform: every thread reads the same word after the barrier
    // ---- value updates, detach deleted leaves
    for (uint32_t i = tid; i < m; i += BLOCK) dt_update_detach_entry(t, vals, sroots, i, kind, leaf_of, list_a);
    __syncthreads();
    // ---- collapse rounds
    uint32_t *cur = list_a, *next = list_b;
    uint32_t *cnt_cur = t.g + DG_LIST_A, *cnt_next = t.g + DG_LIST_B;
    for (int round = 0; round < 256; round++) {
        const uint32_t n = *(volatile uint32_t *)cnt_cur;
        if (n == 0) break;
        if (tid == 0) *cnt_next = 0;
        for (uint32_t e = tid; e < n; e += BLOCK) {
            uint32_t v = cur[e];
            t.ncur[v] = 1;
            t.nnext[v] = 0;
        }
        __syncthreads();
        for (uint32_t e = tid; e < n; e += BLOCK) {
            uint32_t v = cur[e];
            uint32_t gp = t.ndepth[v] == DT_DEAD ? DT_NONE : t.nparent[v];
            defer[e] = (gp != DT_NONE && t.ncur[gp]) ? 1 : 0;
        }
        __syncthreads();
        for (uint32_t e = tid; e < n; e += BLOCK) dt_collapse_entry(t, cur, e, defer, next, cnt_next);
        __syncthreads();
        for (uint32_t e = tid; e < n; e += BLOCK) t.ncur[cur[e]] = 0;
        __syncthreads();
        uint32_t *tp = cur; cur = next; next = tp;
        uint32_t *tc = cnt_cur; cnt_cur = cnt_next; cnt_next = tc;
    }
    __syncthreads();
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;
    // ---- inserts, in rounds
    uint32_t n_ins = dt_block_compact<BLOCK>(nullptr, true, m, [&](uint32_t j) { return kind[j] == DK_INSERT; }, idx_a, sh);
    uint32_t *icur = idx_a, *inext = idx_b;
    for (int round = 0; round < 128 && n_ins; round++) {
        if (tid == 0) s_count = 0;
        for (uint32_t j = tid; j < n_ins; j += BLOCK) dt_insert_locate_entry(t, trie_of_key, keys, icur, j, attach);
        __syncthreads();
        for (uint32_t j = tid; j < n_ins; j += BLOCK)
            dt_insert_run_entry(t, trie_of_key, keys, vals, sroots, icur, n_ins, j, attach, leaf_of, max_per_run, pending, &s_count);
        __syncthreads();
        for (uint32_t j = tid; j < n_ins; j += BLOCK) dt_insert_unlock_entry(t, j, attach);
        if (tid == 0) dt_pop_settle(t);
        __syncthreads();
        if (s_count == 0) break;
        n_ins = dt_block_compact<BLOCK>(icur, false, n_ins, [&](uint32_t j) { return pending[j] != 0; }, inext, sh);
        uint32_t *tp = icur; icur = inext; inext = tp;
    }
    __syncthreads();
    // ---- mark the dirty paths and pick the wavefront's starting points (dt_mark_kernel / dt_starts_kernel)
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;
    const uint32_t n_seeds = *(volatile uint32_t *)(t.g + DG_SEEDS);
    for (uint32_t e = tid; e < n_seeds; e += BLOCK) dt_mark_entry(t, e);
    __syncthreads();
    for (uint32_t e = tid; e < n_seeds; e += BLOCK) dt_starts_entry(t, e);
}

// ------------------------------------------------------------------------------------------------ node encoding
// Payload length of the RLP of node v (16 child slots + the empty value slot) and its masks.  COHERENT: loads that
// bypass L1 (the wavefronts read what other SMs wrote earlier in the same kernel).
template <bool COHERENT>
static __device__ __forceinline__ uint32_t dt_branch_payload(const DTrieDev &t, uint32_t v, uint32_t &state_mask,
                                                            uint32_t &tree_mask, uint32_t &hash_mask) {
    const uint32_t *ch = t.nchild + 16 * (uint64_t)v;
    uint32_t payload = 1;
    state_mask = tree_mask = hash_mask = 0;
    for (int k = 0; k < 16; k++) {
        uint32_t cw = ch[k];
        if (cw == DT_NONE) {
            payload += 1;
            continue;
        }
        bool leaf = (cw & DT_LEAF) != 0;
        const uint8_t *mp = leaf ? t.lmeta + (cw & ~DT_LEAF) : t.nmeta + cw;
        uint32_t m = COHERENT ? __ldcg(mp) : *mp;
        payload += (m & META_LEN) ? (m & META_LEN) : 33u;
        state_mask |= 1u << k;
        if (!leaf) {
            if (!(m & META_EXT)) {
                hash_mask |= 1u << k;
                if (COHERENT && (m & META_LEN)) atomicExch(t.err, B200_DEVERR_INLINE_HASH_CHILD);  // builders only
            }
            if (m & META_STORED) tree_mask |= 1u << k;
        }
    }
    return payload;
}
// The RLP of node v, given its payload length
template <bool COHERENT, class W>
static __device__ __forceinline__ void dt_put_branch(W &s, const DTrieDev &t, uint32_t v, uint32_t payload) {
    const uint32_t *ch = t.nchild + 16 * (uint64_t)v;
    put_list_header(s, payload);
    for (int k = 0; k < 16; k++) {
        uint32_t cw = ch[k];
        if (cw == DT_NONE) {
            s.byte(0x80);
            continue;
        }
        bool leaf = (cw & DT_LEAF) != 0;
        uint32_t id = cw & ~DT_LEAF;
        const uint8_t *mp = leaf ? t.lmeta + id : t.nmeta + id;
        const uint8_t *rp = (leaf ? t.lref : t.nref) + 32 * (uint64_t)id;
        uint32_t ref[8];
        if (COHERENT) load32_cg(rp, ref);
        else load32_nc(rp, ref);
        const uint32_t il = (COHERENT ? __ldcg(mp) : *mp) & META_LEN;
        if (il == 0) {
            s.byte(0xa0);
            s.words8(ref);
        } else {  // (not put_child: with it, ptxas keeps the leaf arrays of dt_wavefront_thread_kernel in local memory)
            for (uint32_t b = 0; b < il; b++) s.byte(byte_at(ref, b));
        }
    }
    s.byte(0x80);
}

// One warp builds node v from its 16 child slots (lane = nibble).  All 32 lanes must call.
// PD_OVERRIDE >= -1: encode as if the parent were at that depth and leave the arena untouched (multi-GPU frontier:
// a bucket's top node as child of the depth-0 root branch); returns the RlpNode meta (inline length | META_EXT ...).
template <int PD_OVERRIDE = -2>
__device__ __forceinline__ uint32_t dt_warp_build_node(const DTrieDev &t, uint32_t v, uint8_t *buf, const WarpKeccak &kw, int lane,
                                                       uint32_t &hashed, uint32_t &exts, uint32_t (&out)[8]) {
    uint32_t *bufw = reinterpret_cast<uint32_t *>(buf);
    const int d = t.ndepth[v];
    const uint32_t cw = lane < 16 ? t.nchild[16 * (uint64_t)v + lane] : DT_NONE;
    const bool has = cw != DT_NONE;
    const bool is_leaf = has && (cw & DT_LEAF);
    const uint32_t id = cw & ~DT_LEAF;
    uint32_t ref[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint32_t cmeta = 0;
    if (has) {
        cmeta = __ldcg(is_leaf ? t.lmeta + id : t.nmeta + id);
        load32_cg((is_leaf ? t.lref : t.nref) + 32 * (uint64_t)id, ref);
    }
    const uint32_t clen = lane < 16 ? (has ? ((cmeta & META_LEN) ? (cmeta & META_LEN) : 33u) : 1u) : 0u;
    const uint32_t bit = has ? (1u << lane) : 0u;
    const bool is_branch = has && !is_leaf;
    const uint32_t hbit = (is_branch && !(cmeta & META_EXT)) ? bit : 0u;
    const uint32_t tbit = (is_branch && (cmeta & META_STORED)) ? bit : 0u;
    if (hbit && (cmeta & META_LEN)) atomicExch(t.err, B200_DEVERR_INLINE_HASH_CHILD);
    const uint32_t state_mask = __reduce_or_sync(0xffffffffu, bit);
    const uint32_t hash_mask = __reduce_or_sync(0xffffffffu, hbit);
    const uint32_t tree_mask = __reduce_or_sync(0xffffffffu, tbit);
    uint32_t incl = clen;
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {
        uint32_t up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += up;
    }
    const uint32_t payload = __shfl_sync(0xffffffffu, incl, 15) + 1;  // + the empty value slot
    const uint32_t hdr = list_header_len(payload), total = hdr + payload;
    const uint32_t blocks = total / 136 + 1;
    for (uint32_t w = lane; w < blocks * 34; w += 32) bufw[w] = 0;
    __syncwarp();
    if (lane == 0) {
        LinBuf lb{buf, 0};
        put_list_header(lb, payload);
    }
    if (lane < 16) {
        LinBuf lb{buf + hdr + incl - clen, 0};
        if (has) put_child(lb, ref, cmeta & META_LEN);
        else lb.byte(0x80);
    }
    if (lane == 16) {
        buf[total - 1] = 0x80;
        buf[total] |= 0x01;
        buf[blocks * 136 - 1] |= 0x80;
    }
    __syncwarp();
    const uint32_t par = t.nparent[v];
    const int pd = PD_OVERRIDE >= -1 ? PD_OVERRIDE : (par == DT_NONE ? -1 : (int)t.ndepth[par]);
    uint32_t meta = warp_finish_node(buf, total, blocks, d, pd, t.nkey + 32 * (uint64_t)v, kw, lane, hashed, exts, out);
    if (PD_OVERRIDE >= -1) {
        __syncwarp();
        return meta;
    }
    if (lane == 0) {
        if ((tree_mask | hash_mask) != 0) meta |= META_STORED;
        if ((t.nmeta[v] & META_STORED) && !(meta & META_STORED)) dt_record_removed(t, v);
        store32(t.nref + 32 * (uint64_t)v, out);
        t.nmeta[v] = (uint8_t)meta;
        t.nmasks[v] = make_ushort4((unsigned short)state_mask, (unsigned short)tree_mask, (unsigned short)hash_mask,
                                   (unsigned short)d);
        t.built[atomicAdd(&t.g[DG_BUILT], 1u)] = v;
    }
    __syncwarp();
    return meta;
}

// The last-arriver climb of a warp from node p (see warp_climb); true iff this warp re-hashed the root of its trie.
static __device__ __forceinline__ bool dt_warp_climb(const DTrieDev &t, uint32_t p, uint8_t *buf, const WarpKeccak &kw, int lane,
                                                     uint32_t &hashed, uint32_t &exts, uint32_t (&out)[8]) {
    for (int hops = 0; p != DT_NONE; hops++) {
        if (hops > DT_MAX_HOPS) {  // uniform across the warp
            if (lane == 0) atomicExch(t.err, B200_DEVERR_CORRUPT);
            return false;
        }
        uint32_t last = 0;
        if (lane == 0) {
            __threadfence();
            last = atomicSub(&t.npending[p], 1u) == 1u;
            __threadfence();
        }
        last = __shfl_sync(0xffffffffu, last, 0);
        if (!last) return false;
        dt_warp_build_node(t, p, buf, kw, lane, hashed, exts, out);
        p = t.nparent[p];
    }
    return true;
}

// One warp per seed: re-hash the item if nothing below it is dirty, then climb; the last dirty child to arrive at a
// node re-hashes it.  The warp that runs out of parents holds the new root reference.
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) dt_wavefront_kernel(DTrieDev t, const uint32_t *__restrict__ count_p) {
    __shared__ __align__(16) uint8_t sbuf[WARPS][WARP_BUF];
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t *buf = sbuf[warp];
    WarpKeccak kw;
    kw.init(lane);
    uint32_t hashed = 0, exts = 0;
    const uint32_t count = *count_p;
    for (uint32_t e = blockIdx.x * WARPS + warp; e < count; e += gridDim.x * WARPS) {
        const uint32_t s = t.seeds[e];
        if (s == DT_NONE) continue;  // not a starting point (dt_starts_kernel)
        uint32_t out[8];
        uint32_t p;
        if (s & DT_LEAF) {
            const uint32_t x = s & ~DT_LEAF;
            const uint32_t lp = t.lparent[x];
            const uint32_t lmeta = warp_leaf_ref(t.account, buf, t.lkey + 32 * (uint64_t)x, lp == DT_NONE ? -1 : (int)t.ndepth[lp],
                                                 t.lval + (uint64_t)t.val_stride * x, t.lsroot ? t.lsroot + 32 * (uint64_t)x : nullptr,
                                                 t.err, kw, lane, hashed, out);
            if (lane == 0) {
                store32(t.lref + 32 * (uint64_t)x, out);
                t.lmeta[x] = (uint8_t)lmeta;
            }
            __syncwarp();
            p = t.lparent[x];  // (read again, not kept live across the leaf encode: that cost the kernel a spill)
        } else {
            dt_warp_build_node(t, s, buf, kw, lane, hashed, exts, out);
            p = t.nparent[s];
        }
        if (dt_warp_climb(t, p, buf, kw, lane, hashed, exts, out) && lane == 0)
            store32(t.top_out + (uint64_t)t.top_stride * dt_trie_of(t, s), out);  // the trie's new root
    }
    flush_warp_counters(t.counters, hashed, exts);
}

// ------------------------------------------------------------------------------------------------ two-stage re-hash
// Large dirty sets (sync catch-up, thousands of blocks per commit): the warp-per-seed wavefront spends ~14x the
// instructions of the register-resident sponge.  Stage A: one THREAD per seed hashes its item and climbs while the
// ancestors are deep (depth >= split_depth: the populous levels); where the trie thins out it hands the arrival over.
// Stage B (dt_climb_kernel): one WARP per hand-over finishes the sparse top with the latency-optimised builder.
// Same last-arriver protocol as dt_wavefront_kernel; the two stages are separate launches.
template <int BLOCK>
__device__ __forceinline__ void dt_thread_build_node(Strip<BLOCK> &s, uint32_t *smem, const DTrieDev &t, uint32_t v,
                                                     uint32_t &hashed, uint32_t &exts, uint32_t (&ref)[8]) {
    s.init(smem);
    const int d = t.ndepth[v];
    uint32_t state_mask, tree_mask, hash_mask;
    const uint32_t payload = dt_branch_payload<true>(t, v, state_mask, tree_mask, hash_mask);
    dt_put_branch<true>(s, t, v, payload);
    const uint32_t par = t.nparent[v];
    const int pd = par == DT_NONE ? -1 : (int)t.ndepth[par];
    uint32_t meta = strip_to_ref(s, list_header_len(payload) + payload, pd < 0 && pd + 1 >= d, ref, hashed);
    meta = thread_finish_node(s, ref, meta, pd, d, t.nkey + 32 * (uint64_t)v, hashed, exts);
    if ((tree_mask | hash_mask) != 0) meta |= META_STORED;
    if ((t.nmeta[v] & META_STORED) && !(meta & META_STORED)) dt_record_removed(t, v);
    store32(t.nref + 32 * (uint64_t)v, ref);
    t.nmeta[v] = (uint8_t)meta;
    t.nmasks[v] = make_ushort4((unsigned short)state_mask, (unsigned short)tree_mask, (unsigned short)hash_mask, (unsigned short)d);
    t.built[atomicAdd(&t.g[DG_BUILT], 1u)] = v;
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) dt_wavefront_thread_kernel(DTrieDev t, const uint32_t *__restrict__ count_p,
                                                                   uint32_t *__restrict__ handoff_list,
                                                                   uint32_t *__restrict__ handoff_count, int split_depth) {
    extern __shared__ uint32_t smem[];
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;
    Strip<BLOCK> s;
    uint32_t hashed = 0, exts = 0;
    const uint32_t e = blockIdx.x * BLOCK + threadIdx.x;
    const uint32_t sd = e < *count_p ? t.seeds[e] : DT_NONE;
    if (sd != DT_NONE) {
        uint32_t ref[8];
        uint32_t p;
        if (sd & DT_LEAF) {
            const uint32_t x = sd & ~DT_LEAF;
            s.init(smem);
            p = t.lparent[x];
            const int pd = p == DT_NONE ? -1 : (int)t.ndepth[p];
            uint32_t k[8];
            load32_nc(t.lkey + 32 * (uint64_t)x, k);
            uint32_t len = t.account ? encode_leaf<Strip<BLOCK>, true>(s, k, pd, t.lval + 72 * (uint64_t)x,
                                                                        t.lsroot ? t.lsroot + 32 * (uint64_t)x : nullptr, t.err)
                                     : encode_leaf<Strip<BLOCK>, false>(s, k, pd, t.lval + 32 * (uint64_t)x, nullptr, t.err);
            uint32_t meta = strip_to_ref(s, len, pd < 0, ref, hashed);
            store32(t.lref + 32 * (uint64_t)x, ref);
            t.lmeta[x] = (uint8_t)meta;
        } else {
            dt_thread_build_node<BLOCK>(s, smem, t, sd, hashed, exts, ref);
            p = t.nparent[sd];
        }
        bool top = true;
        for (int hops = 0; p != DT_NONE; hops++) {
            if (hops > DT_MAX_HOPS) {
                atomicExch(t.err, B200_DEVERR_CORRUPT);
                top = false;
                break;
            }
            if ((int)t.ndepth[p] < split_depth) {  // the sparse top belongs to the warps: hand the arrival over
                __threadfence();
                handoff_list[atomicAdd(handoff_count, 1u)] = p;
                top = false;
                break;
            }
            __threadfence();
            bool last = atomicSub(&t.npending[p], 1u) == 1u;
            __threadfence();
            if (!last) {
                top = false;
                break;
            }
            dt_thread_build_node<BLOCK>(s, smem, t, p, hashed, exts, ref);
            p = t.nparent[p];
        }
        if (top) store32(t.top_out + (uint64_t)t.top_stride * dt_trie_of(t, sd), ref);
    }
    flush_counters(t.counters, hashed, exts);
}

// Stage B: every list entry is one arrival at node p (a dirty child that stage A finished).
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) dt_climb_kernel(DTrieDev t, const uint32_t *__restrict__ arrivals,
                                                             const uint32_t *__restrict__ count_p) {
    __shared__ __align__(16) uint8_t sbuf[WARPS][WARP_BUF];
    if (*(volatile int *)t.err != B200_DEVERR_NONE) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t *buf = sbuf[warp];
    WarpKeccak kw;
    kw.init(lane);
    uint32_t hashed = 0, exts = 0;
    const uint32_t count = *count_p;
    for (uint32_t e = blockIdx.x * WARPS + warp; e < count; e += gridDim.x * WARPS) {
        const uint32_t p = arrivals[e];
        uint32_t out[8];
        if (dt_warp_climb(t, p, buf, kw, lane, hashed, exts, out) && lane == 0)
            store32(t.top_out + (uint64_t)t.top_stride * dt_trie_of(t, p), out);
    }
    flush_warp_counters(t.counters, hashed, exts);
}

// ------------------------------------------------------------------------------------------------ TrieUpdates
// flags[i] = 1 iff re-hashed node built[i] is stored (tree|hash mask != 0, path not empty); n_hashes[i] its hash count
__global__ void dt_stored_flags_kernel(DTrieDev t, const uint32_t *__restrict__ count_p, uint8_t *__restrict__ flags,
                                       uint32_t *__restrict__ n_hashes) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *count_p) return;
    uint32_t v = t.built[i];
    bool stored = t.ndepth[v] != DT_DEAD && t.ndepth[v] != 0 && (t.nmeta[v] & META_STORED);
    flags[i] = stored ? 1 : 0;
    n_hashes[i] = stored ? (uint32_t)__popc(t.nmasks[v].z) : 0u;
}
// record i of `out`: stored node v as a BranchNodeCompact of trie trie_id, its child hashes from hash slot h on
static __device__ __forceinline__ void dt_put_record(const DTrieDev &t, uint32_t v, uint32_t trie_id, uint32_t h, const UpdatesDev &out,
                                                     uint32_t i) {
    const ushort4 m = t.nmasks[v];
    out.trie_id[i] = trie_id;
    out.path_len[i] = (uint8_t)m.w;
    dt_pack_path(t.nkey + 32 * (uint64_t)v, m.w, out.path_packed + 32 * (uint64_t)i);
    out.state_mask[i] = m.x;
    out.tree_mask[i] = m.y;
    out.hash_mask[i] = m.z;
    out.hash_offset[i] = h;
    const uint32_t *ch = t.nchild + 16 * (uint64_t)v;
    for (int s = 0; s < 16; s++)
        if ((m.z >> s) & 1) {
            dt_copy32(out.hashes + 32 * (uint64_t)h, t.nref + 32 * (uint64_t)ch[s]);
            h++;
        }
}
__global__ void dt_gather_updates_kernel(DTrieDev t, const uint32_t *__restrict__ stored_ids, uint32_t n_stored,
                                         const uint32_t *__restrict__ hash_prefix_by_record, UpdatesDev out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_stored) return;
    const uint32_t v = stored_ids[i];
    dt_put_record(t, v, t.ntrie ? t.ntrie[v] : 0, hash_prefix_by_record[i], out, i);
}

