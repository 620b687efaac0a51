// tk_overlay.cuh — post-block state roots of candidate blocks on top of the resident state, read-only
// (b200_dstate_overlay_roots, eng_overlay.inl).  Part of the single translation unit trie_kernels.cu (included inside
// namespace b200, after tk_stateless.cuh: it produces the items that the stateless tail sorts, merges and folds).
//
// reth's StateRootProvider::state_root(hashed_state) on the latest state.  Every block of the batch is its own
// computation against the arenas as they are: the tries are revealed from the arenas, level by level, along the paths of
// the block's keys, into the items of tk_stateless.cuh — leaves (full key, value in the encoding a witness carries) and
// the hashes of the branches no key reaches (kind SL_BLIND_BRANCH at the branch's own path, so the fold re-creates the
// extension above it).  Trie ids as in the stateless path: storage trie of account entry a = a, account trie of block
// b = m + b.  A queued branch carries the contiguous range of its trie's targets that pass through it: the block's
// sorted account keys, or the entry's sorted slot keys.  Nothing is written into the arenas.
//
// With TrieUpdates (b200_dstate_overlay_roots_with_updates) a hash item also carries its parent's tree-mask bit as the arena
// holds it (reth's CursorSubNode::tree_flag: the branch is stored), so that the fold rebuilds the stored records of the
// branches on the keys' paths; and every stored branch the reveal queues (not at the empty path) is a removed-node
// candidate, dropped later when the fold stores a record at the same path.
//
// With proof targets (b200_dstate_overlay_multiproof, one block) a queued branch also carries the range of its trie's sorted
// targets that pass through it: the account targets, or the slot targets of the account target whose key is the entry's.
// A branch is queued when either range is non-empty.  Targets are not entries: the merge, the rows and the folds do not
// change.  Afterwards the fold builds every node of the post-block trie on a target's path; the only hash item a target
// can reach is a branch below an extension that the target leaves.

// nibbles [from, to) of `key` against those of `path`: -1 / 0 / 1
__device__ __forceinline__ int ov_cmp_nibbles(const uint8_t *key, const uint8_t *path, uint32_t from, uint32_t to) {
    for (uint32_t i = from; i < to; i++) {
        const uint32_t a = sl_nib(key, i), b = sl_nib(path, i);
        if (a != b) return a < b ? -1 : 1;
    }
    return 0;
}
// first target in [lo, hi) whose nibbles [from, to) compare above `bound` against `path` (ascending keys that share the
// first `from` nibbles)
__device__ __forceinline__ uint32_t ov_first_above(const uint8_t *keys, uint32_t lo, uint32_t hi, const uint8_t *path, uint32_t from,
                                                   uint32_t to, int bound) {
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (ov_cmp_nibbles(keys + 32 * (uint64_t)mid, path, from, to) <= bound) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// The value of leaf x as its trie's leaf carries it: rlp(TrieAccount) with the leaf's storage root, or rlp(U256).
__device__ uint32_t ov_leaf_value(const DTrieDev &t, uint32_t x, uint8_t *out) {
    const uint8_t *v = t.lval + (uint64_t)t.val_stride * x;
    uint32_t n = 0;
    auto u256 = [&](const uint8_t *be, uint32_t width) {  // big-endian integer of `width` bytes, leading zeros stripped
        uint32_t z = 0;
        while (z < width && be[z] == 0) z++;
        if (z == width) out[n++] = 0x80;
        else if (z == width - 1 && be[z] < 0x80) out[n++] = be[z];
        else {
            out[n++] = (uint8_t)(0x80 + width - z);
            for (uint32_t k = z; k < width; k++) out[n++] = be[k];
        }
    };
    if (!t.account) {
        u256(v, 32);
        return n;
    }
    const b200_account_dev &a = *reinterpret_cast<const b200_account_dev *>(v);
    uint8_t nonce[8];
    for (int k = 0; k < 8; k++) nonce[k] = (uint8_t)(a.nonce >> (8 * (7 - k)));
    n = 2;  // [0xf8, payload]: the payload holds two 33-byte hashes
    u256(nonce, 8);
    u256(a.balance_be, 32);
    out[n++] = 0xa0;
    for (int k = 0; k < 32; k++) out[n++] = t.lsroot[32 * (uint64_t)x + k];
    out[n++] = 0xa0;
    for (int k = 0; k < 32; k++) out[n++] = a.code_hash[k];
    out[0] = 0xf8;
    out[1] = (uint8_t)(n - 2);
    return n;
}

__device__ __forceinline__ SlItem &ov_item(SlItem *items, uint32_t *n_items, uint32_t trie, uint32_t block, uint32_t &idx) {
    idx = atomicAdd(n_items, 1u);
    SlItem &it = items[idx];
    it.off = (uint64_t)OV_STRIDE * idx;
    it.trie = trie;
    it.block = block;
    it.entry = SL_NONE;
    it.tree = 0;
    return it;
}

// Child word w of a branch at depth pd (-1: w is the root word of its trie) with the entries [lo, hi) and the proof targets
// [tlo, thi) that pass through the child's slot, and the parent's tree-mask bit for that slot (`tree`; for a root word ov_root_tree): a leaf is an
// item; a branch is queued with the keys that share its whole path, or, when none do and its RLP is at least 32 bytes,
// is an item holding the hash of the branch itself (under an implicit extension the reference its parent holds is the
// extension's, so the branch is re-hashed).  A branch shorter than 32 bytes has no hash form: it is queued with its
// (possibly empty) range and its children become items.
__device__ void ov_word(const DTrieDev &t, const StatelessDev &s, uint32_t w, int pd, uint32_t tree, uint32_t trie, uint32_t block,
                        uint32_t lo, uint32_t hi, uint32_t tlo, uint32_t thi, OvNode *next, uint32_t *n_next, SlItem *items,
                        uint32_t *n_items, uint8_t *vals) {
    uint32_t idx;
    if (w & DT_LEAF) {
        const uint32_t x = w & ~DT_LEAF;
        SlItem &it = ov_item(items, n_items, trie, block, idx);
        for (int k = 0; k < 32; k++) it.key[k] = t.lkey[32 * (uint64_t)x + k];
        it.len = ov_leaf_value(t, x, vals + it.off);
        it.nib = 64;
        it.kind = SL_LEAF;
        return;
    }
    const uint32_t d = t.ndepth[w];
    const uint8_t *nk = t.nkey + 32 * (uint64_t)w;
    const bool ext = (int)d > pd + 1;
    if (ext && lo < hi) {  // the keys that diverge inside the extension do not reach the branch
        const uint8_t *keys = trie >= s.m ? s.akeys : s.skeys;
        lo = ov_first_above(keys, lo, hi, nk, (uint32_t)(pd + 1), d, -1);
        hi = ov_first_above(keys, lo, hi, nk, (uint32_t)(pd + 1), d, 0);
    }
    if (ext && tlo < thi) {
        const uint8_t *keys = trie >= s.m ? s.tkeys : s.tskeys;
        tlo = ov_first_above(keys, tlo, thi, nk, (uint32_t)(pd + 1), d, -1);
        thi = ov_first_above(keys, tlo, thi, nk, (uint32_t)(pd + 1), d, 0);
    }
    uint32_t sm, tm, hm;
    const uint32_t payload = dt_branch_payload<false>(t, w, sm, tm, hm), blen = list_header_len(payload) + payload;
    if (lo < hi || tlo < thi || blen < 32) {
        OvNode &e = next[atomicAdd(n_next, 1u)];
        e.node = w;
        e.trie = trie;
        e.block = block;
        e.lo = lo;
        e.hi = hi;
        e.tlo = tlo;
        e.thi = thi;
        return;
    }
    SlItem &it = ov_item(items, n_items, trie, block, idx);
    uint8_t *h = vals + it.off;
    if (ext) {
        uint8_t br[544];
        LinBuf lb{br, 0};
        dt_put_branch<false>(lb, t, w, payload);
        uint32_t dig[8];
        dt_keccak_global(br, blen, dig);
        for (int k = 0; k < 32; k++) h[k] = (uint8_t)(dig[k >> 2] >> (8 * (k & 3)));
    } else {
        for (int k = 0; k < 32; k++) h[k] = t.nref[32 * (uint64_t)w + k];
    }
    for (int k = 0; k < 32; k++) it.key[k] = 0;
    for (uint32_t k = 0; k < d; k++) sl_set_nib(it.key, k, sl_nib(nk, k));
    it.len = 32;
    it.nib = (uint8_t)d;
    it.kind = SL_BLIND_BRANCH;
    it.tree = (uint8_t)tree;
}

// A root word has no parent branch, but when every key leaves the extension above it, the fold builds a new branch above
// it whose tree-mask bit for it is what the arena's parent would hold: whether the branch itself is stored.
__device__ __forceinline__ uint32_t ov_root_tree(const DTrieDev &t, uint32_t w) {
    return !(w & DT_LEAF) && (t.nmeta[w] & META_STORED) ? 1u : 0u;
}

// Threads [0, n_blocks): the account root of every block with entries (and the block's parent root for the finish: the
// current root).  Threads [n_blocks, n_blocks + m): the storage root of every entry that is live, not wiped, has slots (or,
// with reveal_targets, is an account target) and whose account exists with a non-empty storage trie — so the storage tries
// are revealed at the same levels as the account tries.  found (nullable): found[a] = entry a's account is in the account
// arena.  With bucket_tries the account arena is a shard's 16 bucket tries and every block lies in one bucket: a block
// starts from its bucket's trie, and an entry's account is looked up in the trie of its top key nibble.
__global__ void ov_seed_kernel(DTrieDev ta, DTrieDev ts, StatelessDev s, const uint8_t *root, uint8_t *parent, OvNode *q,
                               uint32_t *n_q, SlItem *items, uint32_t *n_items, uint8_t *vals, uint8_t *found) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < s.n_blocks) {
        for (int k = 0; k < 32; k++) parent[32 * i + k] = root[k];
        const uint32_t lo = (uint32_t)s.block_acct[i], hi = (uint32_t)s.block_acct[i + 1];
        const uint32_t w = !s.bucket_tries ? ta.troot[0] : lo < hi ? ta.troot[s.akeys[32 * (uint64_t)lo] >> 4] : DT_NONE;
        if (lo < hi && w != DT_NONE)
            ov_word(ta, s, w, -1, ov_root_tree(ta, w), (uint32_t)(s.m + i), (uint32_t)i, lo, hi, 0, (uint32_t)s.n_t, q, n_q, items, n_items,
                    vals);
        return;
    }
    const uint64_t a = i - s.n_blocks;
    if (a >= s.m) return;
    const uint32_t fl = sl_flags(s, a);
    const bool has_slots = s.seg[a + 1] != s.seg[a];
    const bool reveal = (fl & 1) && !(fl & 4) && (has_slots || s.reveal_targets);
    if (!reveal && !found) return;
    const DtLoc loc = dt_descend(ta, s.bucket_tries ? (uint32_t)(s.akeys[32 * a] >> 4) : 0u, s.akeys + 32 * a);
    if (found) found[a] = loc.found ? 1 : 0;
    if (!reveal || !loc.found) return;
    const uint32_t w = ts.troot[loc.child & ~DT_LEAF];
    if (w == DT_NONE) return;
    uint32_t tlo = 0, thi = 0;  // the slot targets of the account target with this entry's key
    bool target = false;
    if (s.n_t) {
        const uint8_t *key = s.akeys + 32 * a;
        uint64_t lo = 0, hi = s.n_t;  // first account target >= key
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if (ov_cmp_nibbles(s.tkeys + 32 * mid, key, 0, 64) < 0) lo = mid + 1;
            else hi = mid;
        }
        if (lo < s.n_t && ov_cmp_nibbles(s.tkeys + 32 * lo, key, 0, 64) == 0) {
            tlo = (uint32_t)s.tseg[lo];
            thi = (uint32_t)s.tseg[lo + 1];
            target = true;
        }
    }
    if (!has_slots && !target) return;
    ov_word(ts, s, w, -1, ov_root_tree(ts, w), (uint32_t)a, sl_block_of_entry(s, a), (uint32_t)s.seg[a], (uint32_t)s.seg[a + 1], tlo, thi, q,
            n_q, items, n_items, vals);
}

// One level: every queued branch splits its entries and its targets by the nibble at its depth and hands each child its
// parts; a stored one
// (not at the empty path) is a removed-node candidate when rm keeps them.
__global__ void ov_reveal_kernel(DTrieDev ta, DTrieDev ts, StatelessDev s, const OvNode *q, uint32_t nq, OvNode *next, uint32_t *n_next,
                                 SlItem *items, uint32_t *n_items, uint8_t *vals, OvRemoved rm) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const OvNode e = q[i];
    const bool account = e.trie >= s.m;
    const DTrieDev &t = account ? ta : ts;
    const uint8_t *keys = account ? s.akeys : s.skeys;
    const uint32_t d = t.ndepth[e.node];
    const uint32_t *ch = t.nchild + 16 * (uint64_t)e.node;
    const uint32_t tree_mask = t.nmasks[e.node].y;
    if (rm.acc && (t.nmeta[e.node] & META_STORED) && d != 0) {
        uint32_t *cand = account ? rm.acc : rm.sto;
        const uint32_t k = atomicAdd(account ? rm.n_acc : rm.n_sto, 1u);
        cand[2 * k] = e.trie;
        cand[2 * k + 1] = e.node;
    }
    const uint8_t *tkeys = account ? s.tkeys : s.tskeys;
    // first key in [lo, top) whose nibble d is above c
    auto split = [d](const uint8_t *ks, uint32_t lo, uint32_t top, uint32_t c) {
        while (lo < top) {
            const uint32_t mid = (lo + top) >> 1;
            if (sl_nib(ks + 32 * (uint64_t)mid, d) <= c) lo = mid + 1;
            else top = mid;
        }
        return lo;
    };
    uint32_t lo = e.lo, tlo = e.tlo;
    for (uint32_t c = 0; c < 16; c++) {
        const uint32_t hi = split(keys, lo, e.hi, c), thi = tlo < e.thi ? split(tkeys, tlo, e.thi, c) : tlo;
        if (ch[c] != DT_NONE)
            ov_word(t, s, ch[c], (int)d, (tree_mask >> c) & 1u, e.trie, e.block, lo, hi, tlo, thi, next, n_next, items, n_items, vals);
        lo = hi;
        tlo = thi;
    }
}

// Candidate k -> (trie id - trie_base, path length, packed path): the rows of the removed records (as dt_removed_paths_kernel)
__global__ void ov_removed_paths_kernel(DTrieDev t, const uint32_t *__restrict__ cand, uint32_t n, uint32_t trie_base,
                                        uint8_t *__restrict__ path_len, uint8_t *__restrict__ path_packed, uint32_t *__restrict__ trie_id) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t v = cand[2 * i + 1], d = t.nmasks[v].w;
    const uint8_t *key = t.nkey + 32 * (uint64_t)v;
    uint8_t *pp = path_packed + 32 * (uint64_t)i;
    for (uint32_t b = 0; b < 32; b++) pp[b] = (uint8_t)(2 * b + 1 < d ? key[b] : (2 * b < d ? (key[b] & 0xF0) : 0));
    path_len[i] = (uint8_t)d;
    trie_id[i] = cand[2 * i] - trie_base;
}

// b200_dstate_overlay_frontiers: thread 16 b + k writes the entry of bucket k after block b.  seg[v] (the fold's account
// segments) of virtual block v = vblock[16 b + k], block b's entries in bucket k, is the bucket's trie after the block;
// vblock < 0: the block does not touch the bucket, which keeps its entry of `cur`.  An empty segment is a bucket the block
// empties: an all-zero entry.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) ov_frontier_kernel(ForestDev f, const uint64_t *__restrict__ seg, const int32_t *__restrict__ vblock,
                                                           uint64_t n, const uint8_t *__restrict__ values, const uint8_t *__restrict__ sroots,
                                                           const uint8_t *__restrict__ nibs, const FrontierEntryDev *__restrict__ cur,
                                                           FrontierEntryDev *__restrict__ out) {
    extern __shared__ uint32_t smem[];
    const uint64_t i = (uint64_t)blockIdx.x * BLOCK + threadIdx.x;
    Strip<BLOCK> s;
    s.init(smem);
    if (i >= n || *(volatile int *)f.err != B200_DEVERR_NONE) return;
    const int32_t v = vblock[i];
    FrontierEntryDev &e = out[i];
    if (v < 0) {
        e = cur[i & 15];
        return;
    }
    for (int k = 0; k < 33; k++) e.as_child[k] = e.as_root[k] = 0;
    e.as_child_len = e.as_root_len = 0;
    const uint64_t lo = seg[v], hi = seg[v + 1];
    if (lo < hi) frontier_entry<BLOCK, true, true>(s, f, f.S[lo], values, sroots, nibs, e);
}

cudaError_t launch_ov_frontier(const ForestDev &f, const uint64_t *seg, const int32_t *vblock, uint64_t n, const uint8_t *values,
                               const uint8_t *sroots, const uint8_t *nibs, const FrontierEntryDev *cur, FrontierEntryDev *out,
                               cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    constexpr int B = 32;
    auto k = ov_frontier_kernel<B>;
    const size_t smem = (size_t)BRANCH_WORDS * B * 4;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k<<<blocks_for(n, B), B, smem, st>>>(f, seg, vblock, n, values, sroots, nibs, cur, out);
    return cudaGetLastError();
}

cudaError_t launch_ov_seed(const DTrieDev &ta, const DTrieDev &ts, const StatelessDev &s, const uint8_t *root, uint8_t *parent, OvNode *q,
                           uint32_t *n_q, SlItem *items, uint32_t *n_items, uint8_t *vals, uint8_t *found, cudaStream_t st) {
    ov_seed_kernel<<<blocks_for(s.n_blocks + s.m, 128), 128, 0, st>>>(ta, ts, s, root, parent, q, n_q, items, n_items, vals, found);
    return cudaGetLastError();
}
cudaError_t launch_ov_reveal(const DTrieDev &ta, const DTrieDev &ts, const StatelessDev &s, const OvNode *q, uint32_t nq, OvNode *next,
                             uint32_t *n_next, SlItem *items, uint32_t *n_items, uint8_t *vals, OvRemoved rm, cudaStream_t st) {
    ov_reveal_kernel<<<blocks_for(nq, 128), 128, 0, st>>>(ta, ts, s, q, nq, next, n_next, items, n_items, vals, rm);
    return cudaGetLastError();
}
cudaError_t launch_ov_removed_paths(const DTrieDev &t, const uint32_t *cand, uint32_t n, uint32_t trie_base, uint8_t *path_len,
                                    uint8_t *path_packed, uint32_t *trie_id, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    ov_removed_paths_kernel<<<blocks_for(n, 128), 128, 0, st>>>(t, cand, n, trie_base, path_len, path_packed, trie_id);
    return cudaGetLastError();
}
