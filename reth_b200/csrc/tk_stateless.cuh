// tk_stateless.cuh — post-block state roots from execution witnesses (b200_witness_roots, eng_stateless.inl).
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, after tk_witness.cuh).
//
// Stateless validation of a batch of blocks (reth: DecodedMultiProofV2::from_witness, crates/trie/common/src/proofs.rs:469-544,
// revealed into a SparseStateTrie, crates/trie/sparse/src/state.rs).  Every block is its own computation: its witness nodes
// (hashed once for the whole batch and sorted by digest) are decoded breadth-first from its parent root into "items" — the
// leaves of the revealed tries and the hashes of the hashed children the witness does not hold ("blind" items).  The block's
// entries are merged into those items by rank, and the final items of every trie go through the items fold
// (tk_items.cuh): storage tries first, then one account trie per block.  Trie ids: storage trie of account entry a = a,
// account trie of block b = m + b; items sort by (trie, zero-padded path).

__device__ __forceinline__ uint32_t sl_flags(const StatelessDev &s, uint64_t a) { return s.aflags ? s.aflags[a] : 1u; }
__device__ __forceinline__ uint32_t sl_nib(const uint8_t *k, uint32_t d) { return (d & 1) ? (k[d >> 1] & 15u) : (k[d >> 1] >> 4); }
__device__ __forceinline__ void sl_set_nib(uint8_t *k, uint32_t d, uint32_t v) { k[d >> 1] |= (uint8_t)((d & 1) ? v : v << 4); }
__device__ __forceinline__ int sl_cmp32(const uint8_t *a, const uint8_t *b) {
    for (int i = 0; i < 32; i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return 0;
}
__device__ __forceinline__ bool sl_is_empty_root(const uint8_t *h) {
    const uint8_t e[32] = {0x56, 0xe8, 0x1f, 0x17, 0x1b, 0xcc, 0x55, 0xa6, 0xff, 0x83, 0x45, 0xe6, 0x92, 0xc0, 0xf8, 0x6e,
                           0x5b, 0x48, 0xe0, 0x1b, 0x99, 0x6c, 0xad, 0xc0, 0x01, 0x62, 0x2f, 0xb5, 0xe3, 0x63, 0xb4, 0x21};
    return sl_cmp32(h, e) == 0;
}
// first index in [lo, hi) whose offs value is > v (offs non-decreasing)
__device__ __forceinline__ uint64_t sl_upper(const uint64_t *offs, uint64_t lo, uint64_t hi, uint64_t v) {
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (offs[mid] <= v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ uint32_t sl_block_of_entry(const StatelessDev &s, uint64_t a) {
    return (uint32_t)(sl_upper(s.block_acct, 0, s.n_blocks + 1, a) - 1);
}
// (trie, key) order of items against a probe
__device__ __forceinline__ int sl_cmp_item(const SlItem &it, uint32_t trie, const uint8_t *key) {
    if (it.trie != trie) return it.trie < trie ? -1 : 1;
    return sl_cmp32(it.key, key);
}
__device__ __forceinline__ uint64_t sl_lower_item(const SlItem *items, uint64_t n, uint32_t trie, const uint8_t *key) {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (sl_cmp_item(items[mid], trie, key) < 0) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
// the first L nibbles of `path` equal those of `key`
__device__ __forceinline__ bool sl_prefix(const uint8_t *path, uint32_t L, const uint8_t *key) {
    for (uint32_t i = 0; i < (L >> 1); i++)
        if (path[i] != key[i]) return false;
    return !(L & 1) || (path[L >> 1] >> 4) == (key[L >> 1] >> 4);
}

// One RLP item at p[i, end): payload p[pay, pay + len), list or string.  false when malformed or running past `end`.
__device__ bool sl_rlp(const uint8_t *p, uint64_t i, uint64_t end, uint64_t &pay, uint64_t &len, bool &list) {
    if (i >= end) return false;
    const uint32_t x = p[i];
    list = x >= 0xc0;
    if (x < 0x80) {
        pay = i;
        len = 1;
    } else if (x < 0xb8 || (x >= 0xc0 && x < 0xf8)) {
        pay = i + 1;
        len = x - (list ? 0xc0 : 0x80);
    } else {
        const uint32_t ll = x - (list ? 0xf7 : 0xb7);
        if (ll > 4 || i + 1 + ll > end || p[i + 1] == 0) return false;
        len = 0;
        for (uint32_t k = 0; k < ll; k++) len = len << 8 | p[i + 1 + k];
        if (len < 56) return false;
        pay = i + 1 + ll;
    }
    return pay + len <= end;
}

// A TrieAccount [nonce, balance, storage_root, code_hash] filling exactly p[i, i + n).  out / sroot may be null.
__device__ bool sl_account(const uint8_t *p, uint64_t i, uint64_t n, b200_account_dev *out, const uint8_t **sroot) {
    uint64_t pay, len, q;
    bool list;
    if (!sl_rlp(p, i, i + n, pay, len, list) || !list || pay + len != i + n) return false;
    const uint64_t end = pay + len;
    uint64_t f[4], fl[4];
    q = pay;
    for (int k = 0; k < 4; k++) {
        if (!sl_rlp(p, q, end, f[k], fl[k], list) || list) return false;
        q = f[k] + fl[k];
    }
    if (q != end || fl[0] > 8 || fl[1] > 32 || fl[2] != 32 || fl[3] != 32) return false;
    if (out) {
        uint64_t nonce = 0;
        for (uint64_t k = 0; k < fl[0]; k++) nonce = nonce << 8 | p[f[0] + k];
        out->nonce = nonce;
        for (int k = 0; k < 32; k++) out->balance_be[k] = k < 32 - (int)fl[1] ? 0 : p[f[1] + k - (32 - fl[1])];
        for (int k = 0; k < 32; k++) out->code_hash[k] = p[f[3] + k];
    }
    if (sroot) *sroot = p + f[2];
    return true;
}
// A storage leaf value: the RLP of a non-zero U256 of at most 32 bytes, filling exactly p[i, i + n).  out32: big-endian.
__device__ bool sl_slot_value(const uint8_t *p, uint64_t i, uint64_t n, uint8_t *out32) {
    uint64_t pay, len;
    bool list;
    if (!sl_rlp(p, i, i + n, pay, len, list) || list || pay + len != i + n || len == 0 || len > 32 || p[pay] == 0) return false;
    if (out32)
        for (int k = 0; k < 32; k++) out32[k] = k < 32 - (int)len ? 0 : p[pay + k - (32 - len)];
    return true;
}

// node of block b whose digest is h, or -1: binary search, then the run of equal digests
__device__ int64_t sl_find(const StatelessDev &s, uint32_t b, const uint8_t *h) {
    uint64_t lo = 0, hi = s.n_nodes;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (sl_cmp32(s.dig_sorted + 32 * mid, h) < 0) lo = mid + 1;
        else hi = mid;
    }
    for (; lo < s.n_nodes && sl_cmp32(s.dig_sorted + 32 * lo, h) == 0; lo++) {
        const uint32_t n = s.dig_perm[lo];
        if (n >= s.block_node[b] && n < s.block_node[b + 1]) return n;
    }
    return -1;
}

__device__ __forceinline__ void sl_push(SlNode *q, uint32_t *n_q, const uint8_t *path, uint32_t depth, uint64_t off, uint32_t len,
                                        uint32_t trie, uint32_t block) {
    SlNode &e = q[atomicAdd(n_q, 1u)];
    for (int k = 0; k < 32; k++) e.path[k] = path[k];
    e.off = off;
    e.len = len;
    e.trie = trie;
    e.block = block;
    e.depth = depth;
}
__device__ __forceinline__ void sl_emit(SlItem *items, uint32_t *n_items, const uint8_t *key, uint32_t nib, uint32_t kind, uint64_t off,
                                        uint32_t len, uint32_t trie, uint32_t block) {
    SlItem &it = items[atomicAdd(n_items, 1u)];
    for (int k = 0; k < 32; k++) it.key[k] = key[k];
    it.off = off;
    it.len = len;
    it.trie = trie;
    it.block = block;
    it.entry = SL_NONE;
    it.nib = (uint8_t)nib;
    it.kind = (uint8_t)kind;
    it.tree = 0;  // (a witness node does not say whether a hashed child is stored)
}

// The root node of every block with entries and a non-empty parent state starts the walk; a missing one: incomplete.
__global__ void sl_seed_kernel(StatelessDev s, SlNode *q, uint32_t *n_q) {
    const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.n_blocks || s.block_acct[b] == s.block_acct[b + 1] || sl_is_empty_root(s.parent + 32 * b)) return;
    const int64_t n = sl_find(s, (uint32_t)b, s.parent + 32 * b);
    if (n < 0) {
        atomicOr(s.status + b, SL_INCOMPLETE);
        return;
    }
    const uint8_t zero[32] = {};
    sl_push(q, n_q, zero, 0, s.rlp_off[n], (uint32_t)(s.rlp_off[n + 1] - s.rlp_off[n]), (uint32_t)(s.m + b), (uint32_t)b);
}

// A child reference at p[i, end of item): inline node (a list shorter than 32 bytes) -> next level; 32-byte hash -> its
// node in the block's witness, or a blind item.  A blind child at depth 64 (a hashed leaf with an empty path, keys that
// share 63 nibbles) has no item form in the fold: incomplete.
__device__ bool sl_child(const StatelessDev &s, const SlNode &e, const uint8_t *path, uint32_t depth, uint64_t i, uint64_t end,
                         bool known_branch, SlNode *next, uint32_t *n_next, SlItem *items, uint32_t *n_items) {
    uint64_t pay, len;
    bool list;
    if (!sl_rlp(s.rlp, i, end, pay, len, list)) return false;
    if (list) {
        if (pay + len - i >= 32) return false;
        sl_push(next, n_next, path, depth, i, (uint32_t)(pay + len - i), e.trie, e.block);
        return true;
    }
    if (len != 32) return false;
    const int64_t n = sl_find(s, e.block, s.rlp + pay);
    if (n >= 0) sl_push(next, n_next, path, depth, s.rlp_off[n], (uint32_t)(s.rlp_off[n + 1] - s.rlp_off[n]), e.trie, e.block);
    else if (depth >= 64) atomicOr(s.status + e.block, SL_INCOMPLETE);
    else sl_emit(items, n_items, path, depth, known_branch ? SL_BLIND_BRANCH : SL_BLIND, pay, 32, e.trie, e.block);
    return true;
}

// One level of the walk: every queued node is decoded; leaves become items, children go to the next level.  An account
// leaf whose entry changes its storage (live, not wiped, with slots) queues the storage root node under trie id = entry.
__global__ void sl_reveal_kernel(StatelessDev s, const SlNode *q, uint32_t nq, SlNode *next, uint32_t *n_next, SlItem *items,
                                 uint32_t *n_items) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nq) return;
    const SlNode e = q[t];
    const uint8_t *p = s.rlp;
    const uint64_t end = e.off + e.len;
    uint64_t pay, len, it[17];
    bool list;
    bool ok = sl_rlp(p, e.off, end, pay, len, list) && list && pay + len == end;
    int cnt = 0;
    for (uint64_t i = pay; ok && i < end; cnt++) {
        uint64_t ip, il;
        if (cnt == 17 || !sl_rlp(p, i, end, ip, il, list)) ok = false;
        else {
            it[cnt] = i;
            i = ip + il;
        }
    }
    ok = ok && (cnt == 2 || cnt == 17);
    if (ok && cnt == 17) {  // branch
        uint64_t ip, il;
        ok = e.depth < 64 && sl_rlp(p, it[16], end, ip, il, list) && !list && il == 0;
        for (int c = 0; ok && c < 16; c++) {
            ok = sl_rlp(p, it[c], end, ip, il, list);
            if (!ok || (!list && il == 0)) continue;
            uint8_t path[32];
            for (int k = 0; k < 32; k++) path[k] = e.path[k];
            sl_set_nib(path, e.depth, (uint32_t)c);
            ok = sl_child(s, e, path, e.depth + 1, it[c], it[c + 1], false, next, n_next, items, n_items);
        }
    } else if (ok) {  // leaf or extension: [hex-prefix path, value | child]
        uint64_t pp, pl, vp, vl;
        ok = sl_rlp(p, it[0], end, pp, pl, list) && !list && pl > 0;
        const uint32_t flag = ok ? p[pp] >> 4 : 0, odd = flag & 1;
        ok = ok && flag <= 3 && (odd || (p[pp] & 15) == 0);
        const uint32_t nn = ok ? 2 * (uint32_t)(pl - 1) + odd : 0, d2 = e.depth + nn;
        const bool leaf = flag >= 2;
        ok = ok && (leaf ? d2 == 64 : (nn > 0 && d2 < 64));
        uint8_t path[32];
        for (int k = 0; k < 32; k++) path[k] = e.path[k];
        for (uint32_t k = 0; ok && k < nn; k++) {
            const uint32_t pos = k + 2 - odd;  // nibble index inside the hex-prefix bytes (flag nibble, [pad nibble])
            sl_set_nib(path, e.depth + k, (pos & 1) ? (p[pp + (pos >> 1)] & 15u) : (p[pp + (pos >> 1)] >> 4));
        }
        if (ok && !leaf) ok = sl_child(s, e, path, d2, it[1], end, true, next, n_next, items, n_items);
        else if (ok) {
            ok = sl_rlp(p, it[1], end, vp, vl, list) && !list;
            const bool account = e.trie >= s.m;
            const uint8_t *sroot = nullptr;
            ok = ok && (account ? sl_account(p, vp, vl, nullptr, &sroot) : sl_slot_value(p, vp, vl, nullptr));
            if (ok) {
                sl_emit(items, n_items, path, 64, SL_LEAF, vp, (uint32_t)vl, e.trie, e.block);
                if (account) {  // the entry of this account, if the block has one
                    uint64_t lo = s.block_acct[e.block], hi = s.block_acct[e.block + 1];
                    while (lo < hi) {
                        uint64_t mid = (lo + hi) >> 1;
                        if (sl_cmp32(s.akeys + 32 * mid, path) < 0) lo = mid + 1;
                        else hi = mid;
                    }
                    const uint64_t a = lo;
                    if (a < s.block_acct[e.block + 1] && sl_cmp32(s.akeys + 32 * a, path) == 0) {
                        const uint32_t fl = sl_flags(s, a);
                        if ((fl & 1) && !(fl & 4) && s.seg[a + 1] > s.seg[a] && !sl_is_empty_root(sroot)) {
                            const int64_t n = sl_find(s, e.block, sroot);
                            const uint8_t zero[32] = {};
                            if (n < 0) atomicOr(s.status + e.block, SL_INCOMPLETE);
                            else sl_push(next, n_next, zero, 0, s.rlp_off[n], (uint32_t)(s.rlp_off[n + 1] - s.rlp_off[n]), (uint32_t)a, e.block);
                        }
                    }
                }
            }
        }
    }
    if (!ok) atomicOr(s.status + e.block, SL_INVALID);
}

// LSD sort key of pass w: big-endian path word w (0 = most significant) or, w = 4, the trie id; of item perm[i] (or i)
__global__ void sl_sort_key_kernel(const SlItem *items, const uint32_t *perm, uint64_t n, int w, uint64_t *keys, uint32_t *idx) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t j = perm ? perm[i] : (uint32_t)i;
    uint64_t k = 0;
    if (w == 4) k = items[j].trie;
    else
        for (int b = 0; b < 8; b++) k = k << 8 | items[j].key[8 * w + b];
    keys[i] = k;
    idx[i] = j;
}
__global__ void sl_gather_kernel(const SlItem *items, const uint32_t *perm, uint64_t n, SlItem *out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = items[perm[i]];
}

// Entry j (slot entries [0, n_e), then account entries) against the sorted items of its trie: a leaf is updated (entry
// recorded) or deleted, a blind item on the key's path makes the block incomplete, otherwise the key is inserted (live,
// non-zero) or nothing happens.  lb[j]: the rank of the key among the items (non-decreasing in j).
__global__ void sl_merge_kernel(StatelessDev s, SlItem *items, uint64_t n_it, uint32_t *dead, uint32_t *ins, uint32_t *lb,
                                uint32_t *eblock) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= s.n_e + s.m) return;
    const bool slot = j < s.n_e;
    const uint64_t a = slot ? sl_upper(s.seg, 0, s.m + 1, j) - 1 : j - s.n_e;
    const uint32_t b = sl_block_of_entry(s, a), fl = sl_flags(s, a);
    const uint32_t trie = slot ? (uint32_t)a : (uint32_t)(s.m + b);
    const uint8_t *key = slot ? s.skeys + 32 * j : s.akeys + 32 * a;
    const uint64_t r = sl_lower_item(items, n_it, trie, key);
    bool blind = false, found = false;
    if (r < n_it && items[r].trie == trie) {
        if (items[r].nib == 64) found = sl_cmp32(items[r].key, key) == 0;
        else blind = sl_prefix(items[r].key, items[r].nib, key);
    }
    if (r > 0 && items[r - 1].trie == trie && items[r - 1].nib < 64) blind |= sl_prefix(items[r - 1].key, items[r - 1].nib, key);
    bool zero = true;
    if (slot)
        for (int k = 0; k < 32; k++) zero &= s.svals[32 * j + k] == 0;
    uint32_t insert = 0;
    if (blind) atomicOr(s.status + b, SL_INCOMPLETE);
    else if (found) {
        if (!(fl & 1) || (slot && zero)) {
            if (fl & 1 || !slot) dead[r] = 1;
        } else items[r].entry = slot ? (uint32_t)j : (uint32_t)a;
    } else insert = slot ? ((fl & 1) && !zero) : ((fl & 1) && !(fl & 2));
    ins[j] = insert;
    lb[j] = (uint32_t)r;
    eblock[j] = b;
}
// survivors: items not deleted and entries inserted, of blocks that have not failed
__global__ void sl_keep_kernel(const uint32_t *status, const SlItem *items, uint64_t n_it, uint32_t *keep, const uint32_t *eblock,
                               uint64_t n_ent, uint32_t *ins) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_it) keep[i] = !keep[i] && !status[items[i].block];
    else if (i - n_it < n_ent) ins[i - n_it] = ins[i - n_it] && !status[eblock[i - n_it]];
}
// totals[0] = final items, totals[1] = final items of the storage tries (trie < m)
__global__ void sl_totals_kernel(StatelessDev s, const SlItem *items, uint64_t n_it, const uint32_t *kscan, const uint32_t *iscan,
                                 uint64_t *totals) {
    uint64_t lo = 0, hi = n_it;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (items[mid].trie < s.m) lo = mid + 1;
        else hi = mid;
    }
    totals[0] = (uint64_t)kscan[n_it] + iscan[s.n_e + s.m];
    totals[1] = (uint64_t)kscan[lo] + iscan[s.n_e];
}
// Final positions by rank: an inserted entry goes before the item at its rank, after the entries inserted before it.
__global__ void sl_place_kernel(StatelessDev s, const SlItem *items, uint64_t n_it, const uint32_t *keep, const uint32_t *kscan,
                                const uint32_t *ins, const uint32_t *iscan, const uint32_t *lb, const uint32_t *eblock, SlItem *fin) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t n_ent = s.n_e + s.m;
    if (i < n_it) {
        if (!keep[i]) return;
        uint64_t lo = 0, hi = n_ent;  // entries ranked at or before item i
        while (lo < hi) {
            uint64_t mid = (lo + hi) >> 1;
            if (lb[mid] <= i) lo = mid + 1;
            else hi = mid;
        }
        fin[kscan[i] + iscan[lo]] = items[i];
    } else if (i - n_it < n_ent) {
        const uint64_t j = i - n_it;
        if (!ins[j]) return;
        SlItem &f = fin[kscan[lb[j]] + iscan[j]];
        const bool slot = j < s.n_e;
        const uint64_t a = slot ? sl_upper(s.seg, 0, s.m + 1, j) - 1 : j - s.n_e;
        const uint8_t *key = slot ? s.skeys + 32 * j : s.akeys + 32 * a;
        for (int k = 0; k < 32; k++) f.key[k] = key[k];
        f.off = 0;
        f.len = 0;  // no decoded value: the entry's
        f.trie = slot ? (uint32_t)a : (uint32_t)(s.m + eblock[j]);
        f.block = eblock[j];
        f.entry = slot ? (uint32_t)j : (uint32_t)a;
        f.nib = 64;
        f.kind = SL_LEAF;
        f.tree = 0;
    }
}
// Segment offsets of the two forests: storage segment a (m of them), account segment b (n_blocks), from the final items.
__global__ void sl_segments_kernel(StatelessDev s, const SlItem *fin, uint64_t n_fin, uint64_t n_sto, uint64_t *sto_offs,
                                   uint64_t *acc_offs) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t > s.m + s.n_blocks) return;
    uint64_t lo = 0, hi = n_fin;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (fin[mid].trie < t) lo = mid + 1;
        else hi = mid;
    }
    if (t <= s.m) sto_offs[t] = lo;
    if (t >= s.m) acc_offs[t - s.m] = lo - n_sto;
}
// Rule (b): a blind item of unknown kind that ends up more than one nibble below its nearest branch would be wrapped in an
// extension by the fold, which is only right for a branch node.  Its parent depth is the longer common prefix with its
// neighbours in the same trie (none: the item is the root of its trie).
__global__ void sl_sufficiency_kernel(StatelessDev s, const SlItem *fin, uint64_t n_fin) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_fin || fin[i].kind != SL_BLIND) return;
    int pd = -1;
    for (int side = 0; side < 2; side++) {
        const uint64_t o = side ? i + 1 : i - 1;
        if ((side ? i + 1 >= n_fin : i == 0) || fin[o].trie != fin[i].trie) continue;
        int l = 0;
        while (l < 64 && sl_nib(fin[o].key, l) == sl_nib(fin[i].key, l)) l++;
        pd = l > pd ? l : pd;
    }
    if ((int)fin[i].nib > pd + 1) atomicOr(s.status + fin[i].block, SL_INCOMPLETE);
}
// Fold inputs of final items [lo, hi): keys, nibbles, flags (the item's tree bit: children_are_in_trie), and the value rows — storage: U256 (entry or decoded leaf);
// accounts: b200_account (entry unless "unchanged", else the decoded leaf) and the storage root (the new root when the entry
// changes the storage or the account is new, else the leaf's).  A blind item's row starts with its hash.
__global__ void sl_rows_kernel(StatelessDev s, const SlItem *fin, uint64_t lo, uint64_t hi, uint8_t *keys, uint8_t *nibs, uint8_t *flags,
                               uint8_t *values, uint8_t *sroots, const uint8_t *sto_roots) {
    const uint64_t i = lo + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hi) return;
    const SlItem &f = fin[i];
    const uint64_t r = i - lo;
    for (int k = 0; k < 32; k++) keys[32 * r + k] = f.key[k];
    nibs[r] = f.nib;
    flags[r] = f.tree;
    const bool account = sroots != nullptr;
    uint8_t *row = values + (account ? 72 : 32) * r;
    if (f.kind != SL_LEAF) {
        for (int k = 0; k < 32; k++) row[k] = s.rlp[f.off + k];
        return;
    }
    if (!account) {
        if (f.entry != SL_NONE)
            for (int k = 0; k < 32; k++) row[k] = s.svals[32 * (uint64_t)f.entry + k];
        else sl_slot_value(s.rlp, f.off, f.len, row);
        return;
    }
    b200_account_dev acc;
    const uint8_t *old = nullptr;
    if (f.len) sl_account(s.rlp, f.off, f.len, &acc, &old);
    const uint64_t a = f.entry;
    const uint32_t fl = f.entry != SL_NONE ? sl_flags(s, a) : 0;
    if (f.entry != SL_NONE && !(fl & 2)) acc = reinterpret_cast<const b200_account_dev *>(s.accts)[a];
    const uint8_t *b = reinterpret_cast<const uint8_t *>(&acc);
    for (int k = 0; k < 72; k++) row[k] = b[k];
    const bool fresh = f.entry != SL_NONE && (!f.len || (fl & 4) || s.seg[a + 1] > s.seg[a]);
    const uint8_t *sr = fresh ? sto_roots + 32 * a : old;
    for (int k = 0; k < 32; k++) sroots[32 * r + k] = sr[k];
}
// roots32 [n_blocks][32] then the statuses int32 [n_blocks]: a block without entries keeps its parent root
__global__ void sl_finish_kernel(StatelessDev s, const uint8_t *acc_roots, uint8_t *out) {
    const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= s.n_blocks) return;
    const bool empty = s.block_acct[b] == s.block_acct[b + 1];
    const uint32_t st = empty ? 0 : s.status[b];
    const uint8_t *src = empty ? s.parent + 32 * b : acc_roots + 32 * b;
    for (int k = 0; k < 32; k++) out[32 * b + k] = st ? 0 : src[k];
    reinterpret_cast<int32_t *>(out + 32 * s.n_blocks)[b] =
        (st & SL_INVALID) ? SL_STATUS_INVALID : (st & SL_INCOMPLETE) ? SL_STATUS_INCOMPLETE : 0;
}

cudaError_t launch_sl_seed(const StatelessDev &s, SlNode *q, uint32_t *n_q, cudaStream_t st) {
    sl_seed_kernel<<<blocks_for(s.n_blocks, 256), 256, 0, st>>>(s, q, n_q);
    return cudaGetLastError();
}
cudaError_t launch_sl_reveal(const StatelessDev &s, const SlNode *q, uint32_t nq, SlNode *next, uint32_t *n_next, SlItem *items,
                             uint32_t *n_items, cudaStream_t st) {
    sl_reveal_kernel<<<blocks_for(nq, 128), 128, 0, st>>>(s, q, nq, next, n_next, items, n_items);
    return cudaGetLastError();
}
cudaError_t launch_sl_sort_key(const SlItem *items, const uint32_t *perm, uint64_t n, int w, uint64_t *keys, uint32_t *idx,
                               cudaStream_t st) {
    sl_sort_key_kernel<<<blocks_for(n, 256), 256, 0, st>>>(items, perm, n, w, keys, idx);
    return cudaGetLastError();
}
cudaError_t launch_sl_gather(const SlItem *items, const uint32_t *perm, uint64_t n, SlItem *out, cudaStream_t st) {
    sl_gather_kernel<<<blocks_for(n, 256), 256, 0, st>>>(items, perm, n, out);
    return cudaGetLastError();
}
cudaError_t launch_sl_merge(const StatelessDev &s, SlItem *items, uint64_t n_it, uint32_t *dead, uint32_t *ins, uint32_t *lb,
                            uint32_t *eblock, cudaStream_t st) {
    sl_merge_kernel<<<blocks_for(s.n_e + s.m, 256), 256, 0, st>>>(s, items, n_it, dead, ins, lb, eblock);
    return cudaGetLastError();
}
cudaError_t launch_sl_keep(const StatelessDev &s, const SlItem *items, uint64_t n_it, uint32_t *keep, const uint32_t *eblock,
                           uint32_t *ins, cudaStream_t st) {
    sl_keep_kernel<<<blocks_for(n_it + s.n_e + s.m, 256), 256, 0, st>>>(s.status, items, n_it, keep, eblock, s.n_e + s.m, ins);
    return cudaGetLastError();
}
cudaError_t launch_sl_totals(const StatelessDev &s, const SlItem *items, uint64_t n_it, const uint32_t *kscan, const uint32_t *iscan,
                             uint64_t *totals, cudaStream_t st) {
    sl_totals_kernel<<<1, 1, 0, st>>>(s, items, n_it, kscan, iscan, totals);
    return cudaGetLastError();
}
cudaError_t launch_sl_place(const StatelessDev &s, const SlItem *items, uint64_t n_it, const uint32_t *keep, const uint32_t *kscan,
                            const uint32_t *ins, const uint32_t *iscan, const uint32_t *lb, const uint32_t *eblock, SlItem *fin,
                            cudaStream_t st) {
    sl_place_kernel<<<blocks_for(n_it + s.n_e + s.m, 256), 256, 0, st>>>(s, items, n_it, keep, kscan, ins, iscan, lb, eblock, fin);
    return cudaGetLastError();
}
cudaError_t launch_sl_segments(const StatelessDev &s, const SlItem *fin, uint64_t n_fin, uint64_t n_sto, uint64_t *sto_offs,
                               uint64_t *acc_offs, cudaStream_t st) {
    sl_segments_kernel<<<blocks_for(s.m + s.n_blocks + 1, 256), 256, 0, st>>>(s, fin, n_fin, n_sto, sto_offs, acc_offs);
    return cudaGetLastError();
}
cudaError_t launch_sl_sufficiency(const StatelessDev &s, const SlItem *fin, uint64_t n_fin, cudaStream_t st) {
    if (n_fin == 0) return cudaSuccess;
    sl_sufficiency_kernel<<<blocks_for(n_fin, 256), 256, 0, st>>>(s, fin, n_fin);
    return cudaGetLastError();
}
cudaError_t launch_sl_rows(const StatelessDev &s, const SlItem *fin, uint64_t lo, uint64_t hi, uint8_t *keys, uint8_t *nibs,
                           uint8_t *flags, uint8_t *values, uint8_t *sroots, const uint8_t *sto_roots, cudaStream_t st) {
    if (hi <= lo) return cudaSuccess;
    sl_rows_kernel<<<blocks_for(hi - lo, 128), 128, 0, st>>>(s, fin, lo, hi, keys, nibs, flags, values, sroots, sto_roots);
    return cudaGetLastError();
}
cudaError_t launch_sl_finish(const StatelessDev &s, const uint8_t *acc_roots, uint8_t *out, cudaStream_t st) {
    sl_finish_kernel<<<blocks_for(s.n_blocks, 256), 256, 0, st>>>(s, acc_roots, out);
    return cudaGetLastError();
}
