// tk_witness.cuh — execution witness of a block (TrieWitness::compute, crates/trie/trie/src/witness.rs) out of the
// dynamic arenas, read-only.  Part of the single translation unit trie_kernels.cu (included inside namespace b200, after
// tk_proofs.cuh).
//
// The witness is every node of the proofs of the block's targets, plus the nodes a sparse trie has to reveal to collapse a
// branch that keeps a single child (the sibling of removed leaves), plus in Legacy mode the storage-root node of every
// account without storage targets.  The sparse trie asks for a sibling exactly when, after the removal phase, a branch on a
// removal path keeps one child and that child is hashed (RLP >= 32 bytes) and lies on no target's path.  Here:
//   * every target key walks down once: each branch slot it passes is "seen" (a target path goes through that child);
//     in Canonical mode an inserted key also marks the slots it passes as surviving (upserts are applied first);
//   * a removed leaf climbs: it sets its bit in the parent's "gone" mask; the thread whose bit completes the mask of the
//     parent's children (the last arriver) carries on with the parent, so a subtree all of whose leaves go is gone for
//     its own parent, in one launch and without ordering between the threads;
//   * every branch that lost a child (listed by its first arriver) with exactly one surviving, unseen, hashed child c
//     emits the proof target (key = path ‖ c ‖ 0…0, min_len = |path ‖ c|): what the sparse trie's blinded-node callback
//     asks for (crates/trie/sparse/src/parallel.rs:1004-1013).
// Per-node scratch: two words per node slot of the arena, cleared for every call.
//
// b200_dstate_overlay_witness runs the same kernels on the folds of an overlay (da_from_fold): every target path is opened
// there, and a hash leaf (lmeta META_ISNODE: an unchanged resident subtree) counts as a surviving, hashed, unseen child.
// The walks that go below a hash leaf (the branch under a diverging extension, a collapse sibling, the leaves of a wiped
// storage) carry on, read-only, in the resident arena of the same trie (wt_fall).  Storage trie ids are then the overlay's
// entries (entry_trie), and res_trie[trie] names the resident storage trie behind one.

static __device__ __forceinline__ uint32_t wt_child_mask(const DTrieDev &t, uint32_t v) {
    uint32_t m = 0;
    const uint32_t *ch = t.nchild + 16 * (uint64_t)v;
#pragma unroll
    for (int s = 0; s < 16; s++) m |= (ch[s] != DT_NONE ? 1u : 0u) << s;
    return m;
}

// One key of one trie: marks the slots it passes; remove = a removal (an existing leaf is removed), insert = an upsert
// whose slots count as survivors.  Returns whether the key is in the trie.
static __device__ bool wt_walk(const DTrieDev &t, const WitnessMarks &w, uint32_t trie, const uint8_t *key, bool remove, bool insert) {
    uint32_t cur = t.troot[trie], matched = 0, parent = DT_NONE, slot = 0;
    bool found = false;
    for (int hops = 0;; hops++) {
        if (hops > DT_MAX_HOPS) {
            atomicExch(t.err, B200_DEVERR_CORRUPT);
            return false;
        }
        if (cur == DT_NONE) break;
        if (cur & DT_LEAF) {
            found = dt_lcp(key, t.lkey + 32 * (uint64_t)(cur & ~DT_LEAF), matched, 64) == 64;
            break;
        }
        const uint32_t d = t.ndepth[cur];
        if (dt_lcp(key, t.nkey + 32 * (uint64_t)cur, matched, d) < d) break;  // diverges inside the extension above cur
        slot = dt_nib(key, d);
        atomicOr(&w.seen[cur], (1u << slot) | (insert ? 1u << (16 + slot) : 0u));
        parent = cur;
        matched = d + 1;
        cur = t.nchild[16 * (uint64_t)cur + slot];
    }
    if (!(remove && found)) return found;
    // the climb: (v, s) = a branch and the slot of the child that is gone
    uint32_t v = parent, s = slot;
    for (int hops = 0;; hops++) {
        if (v == DT_NONE) {  // the trie's root is gone: the trie becomes empty
            if (w.trie_flags) w.trie_flags[trie] |= WF_EMPTIED;
            return true;
        }
        if (hops > DT_MAX_HOPS) {
            atomicExch(t.err, B200_DEVERR_CORRUPT);
            return true;
        }
        const uint32_t bit = 1u << s, old = atomicOr(&w.gone[v], bit);
        if (old == 0) w.list[atomicAdd(w.n_list, 1u)] = v;
        if ((old | bit) != wt_child_mask(t, v)) return true;  // a sibling survives, or arrives later
        const uint32_t p = t.nparent[v];
        if (p != DT_NONE) s = dt_nib(t.nkey + 32 * (uint64_t)v, t.ndepth[p]);
        v = p;
    }
}

// reth's Account::is_empty on a b200_account row: nonce 0, balance 0, code hash KECCAK_EMPTY (the row of a None hash)
static __device__ __forceinline__ bool wt_account_empty(const uint8_t *a) {
    static constexpr uint8_t KE[32] = {0xc5, 0xd2, 0x46, 0x01, 0x86, 0xf7, 0x23, 0x3c, 0x92, 0x7e, 0x7d, 0xb2, 0xdc, 0xc7, 0x03, 0xc0,
                                       0xe5, 0x00, 0xb6, 0x53, 0xca, 0x82, 0x27, 0x3b, 0x7b, 0xfa, 0xd8, 0x04, 0x5d, 0x85, 0xa4, 0x70};
    for (int b = 0; b < 40; b++)
        if (a[b]) return false;
    for (int b = 0; b < 32; b++)
        if (a[40 + b] != KE[b]) return false;
    return true;
}

// The resident branch behind hash leaf x of fold arena f: the node of resident trie rt at depth lnib[x] on the path lkey[x],
// whose own hash must be the one the leaf holds (nref is the reference its resident parent holds: below an implicit
// extension that is the extension's, so the branch is re-hashed).  Anything else latches B200_DEVERR_CORRUPT: DT_NONE.
static __device__ uint32_t wt_fall(const DTrieDev &f, uint32_t x, const DTrieDev &r, uint32_t rt) {
    const uint8_t *hk = f.lkey + 32 * (uint64_t)x, *want = f.lval + (uint64_t)f.val_stride * x;
    const uint32_t L = f.lnib[x];
    uint32_t cur = rt == DT_NONE ? DT_NONE : r.troot[rt];
    int pd = -1;
    for (int hops = 0; hops <= DT_MAX_HOPS && cur != DT_NONE && !(cur & DT_LEAF); hops++) {
        const uint32_t d = r.ndepth[cur];
        if (d > L || dt_lcp(hk, r.nkey + 32 * (uint64_t)cur, (uint32_t)(pd + 1), d) < d) break;
        if (d < L) {
            pd = (int)d;
            cur = r.nchild[16 * (uint64_t)cur + dt_nib(hk, d)];
            continue;
        }
        bool same = true;
        if (pd + 1 == (int)L) {
            for (int k = 0; k < 32; k++) same &= r.nref[32 * (uint64_t)cur + k] == want[k];
        } else {
            uint32_t sm, tm, hm, dig[8];
            const uint32_t payload = dt_branch_payload<false>(r, cur, sm, tm, hm), blen = list_header_len(payload) + payload;
            uint8_t br[544];
            LinBuf lb{br, 0};
            dt_put_branch<false>(lb, r, cur, payload);
            dt_keccak_global(br, blen, dig);
            for (int k = 0; k < 32; k++) same &= (uint8_t)(dig[k >> 2] >> (8 * (k & 3))) == want[k];
        }
        if (same) return cur;
        break;
    }
    atomicExch(f.err, B200_DEVERR_CORRUPT);
    return DT_NONE;
}
static __device__ __forceinline__ bool wt_hash_leaf(const DTrieDev &t, uint32_t w) {
    return (w & DT_LEAF) && t.lnib && (t.lmeta[w & ~DT_LEAF] & META_ISNODE);
}

static __device__ __forceinline__ uint32_t wt_account_of(const uint64_t *__restrict__ seg_offsets, uint64_t m, uint64_t j) {
    uint64_t lo = 0, hi = m;  // last account with offset <= j
    while (hi - lo > 1) {
        uint64_t mid = (lo + hi) >> 1;
        if (seg_offsets[mid] <= j) lo = mid;
        else hi = mid;
    }
    return (uint32_t)lo;
}
static __device__ __forceinline__ bool wt_wiped(const uint8_t *flags, uint64_t i) {  // destroyed, or storage wiped
    return flags != nullptr && (!(flags[i] & 1) || (flags[i] & 4));
}

// Accounts, first pass: the account leaf and the storage trie (entry_trie, nullable: the leaf) of every account entry, the
// key order, the wiped storage tries.  acct_trie (nullable: trie 0): the account trie of every entry, a bucket trie of a
// sharded state.
__global__ void wt_accounts_kernel(DTrieDev ta, DTrieDev ts, const uint8_t *__restrict__ keys, const uint8_t *__restrict__ flags,
                                   uint64_t m, const uint32_t *__restrict__ entry_trie, const uint32_t *__restrict__ acct_trie,
                                   uint32_t *__restrict__ leaf_of, uint32_t *__restrict__ trie_of, uint8_t *__restrict__ trie_flags) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint8_t *key = keys + 32 * i;
    if (i) {
        uint32_t l = dt_lcp(key - 32, key, 0, 64);
        if (l == 64 || dt_nib(key - 32, l) > dt_nib(key, l)) atomicExch(ta.err, B200_DEVERR_UNSORTED);
    }
    DtLoc loc = dt_descend(ta, acct_trie ? acct_trie[i] : 0u, key);
    const uint32_t leaf = loc.found ? (loc.child & ~DT_LEAF) : DT_NONE;
    const uint32_t trie = leaf == DT_NONE ? DT_NONE : entry_trie ? entry_trie[i] : leaf;
    leaf_of[i] = leaf;
    trie_of[i] = trie;
    if (trie != DT_NONE && wt_wiped(flags, i) && ts.troot[trie] != DT_NONE) trie_flags[trie] = WF_WIPED;
}

// Slot entries: the storage target j (trie, key), the key order, and the walk of every entry of a storage trie that is not
// wiped (a wiped trie loses every leaf: no branch of it keeps a pre-state child, so it reveals nothing).
__global__ void wt_slots_kernel(DTrieDev ts, WitnessMarks w, const uint64_t *__restrict__ seg_offsets, uint64_t m,
                                const uint32_t *__restrict__ trie_of, const uint8_t *__restrict__ flags,
                                const uint8_t *__restrict__ keys, const uint8_t *__restrict__ vals, uint64_t n, int canonical,
                                uint32_t *__restrict__ trie_of_target, uint8_t *__restrict__ nonzero) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t i = wt_account_of(seg_offsets, m, j);
    const uint8_t *key = keys + 32 * j;
    if (j > seg_offsets[i]) {
        uint32_t l = dt_lcp(key - 32, key, 0, 64);
        if (l == 64 || dt_nib(key - 32, l) > dt_nib(key, l)) atomicExch(ts.err, B200_DEVERR_UNSORTED);
    }
    const uint64_t *v = reinterpret_cast<const uint64_t *>(vals + 32 * j);
    const bool upsert = (v[0] | v[1] | v[2] | v[3]) != 0;
    if (upsert) nonzero[i] = 1;
    const uint32_t trie = trie_of[i];
    trie_of_target[j] = trie;
    if (trie == DT_NONE || wt_wiped(flags, i)) return;
    const bool found = wt_walk(ts, w, trie, key, !upsert, false);
    if (canonical && upsert && !found) wt_walk(ts, w, trie, key, false, true);
}

// Accounts, second pass (after the storage walks): removal or upsert (TrieWitness: removal iff the account is empty and
// its storage root after the block is EMPTY_ROOT_HASH), the walk in the account trie (acct_trie as wt_accounts_kernel), and
// the Legacy storage-root target.
__global__ void wt_account_walk_kernel(DTrieDev ta, DTrieDev ts, WitnessMarks w, const uint8_t *__restrict__ keys,
                                       const uint8_t *__restrict__ accts, const uint8_t *__restrict__ flags,
                                       const uint64_t *__restrict__ seg_offsets, uint64_t m, const uint32_t *__restrict__ acct_trie,
                                       const uint32_t *__restrict__ leaf_of,
                                       const uint32_t *__restrict__ trie_of, const uint8_t *__restrict__ trie_flags, const uint8_t *__restrict__ nonzero, int canonical,
                                       uint32_t *__restrict__ root_trie, uint16_t *__restrict__ root_meta) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint32_t leaf = leaf_of[i], trie = trie_of[i];
    const uint8_t f = flags ? flags[i] : 1;
    const bool wiped = wt_wiped(flags, i);
    const bool pre_empty = trie == DT_NONE || ts.troot[trie] == DT_NONE;
    const bool has_targets = seg_offsets[i + 1] > seg_offsets[i] || (wiped && !pre_empty);
    bool post_empty;
    if (has_targets) post_empty = (pre_empty || wiped || (trie_flags[trie] & WF_EMPTIED)) && !nonzero[i];
    else post_empty = pre_empty;
    // as b200_dstate_apply does: a destroyed account goes whatever its slot entries say, and an "unchanged" entry of an
    // absent account is ignored with its slots (its key is still a target: its proof shows the absence)
    const bool ignored = (f & 1) && (f & 2) && leaf == DT_NONE;
    bool removal;
    if (!(f & 1)) removal = true;
    else if (ignored) removal = false;
    else if (f & 2) removal = wt_account_empty(ta.lval + 72 * (uint64_t)leaf) && post_empty;  // unchanged: the resident one
    else removal = wt_account_empty(accts + 72 * i) && post_empty;
    root_trie[i] = trie;
    root_meta[i] = (!canonical && !has_targets) ? WM_ROOT_ONLY : WM_SKIP;
    const uint32_t at = acct_trie ? acct_trie[i] : 0u;
    const bool found = wt_walk(ta, w, at, keys + 32 * i, removal, false);
    if (canonical && !removal && !ignored && !found) wt_walk(ta, w, at, keys + 32 * i, false, true);
}

// Reveal targets: every listed branch with exactly one surviving child that no target walks through and whose node is
// hashed.  Written at [*n_out) of (trie, key, meta).
__global__ void wt_reveal_kernel(DTrieDev t, WitnessMarks w, uint32_t max_list, int canonical, uint32_t *__restrict__ out_trie,
                                 uint8_t *__restrict__ out_keys, uint16_t *__restrict__ out_meta, uint32_t *__restrict__ n_out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= max_list || i >= *w.n_list) return;
    const uint32_t v = w.list[i], seen = w.seen[v];
    const uint32_t surv = (wt_child_mask(t, v) & ~w.gone[v]) | (canonical ? seen >> 16 : 0u);
    if (__popc(surv) != 1 || (seen & surv)) return;
    const uint32_t c = __ffs(surv) - 1, d = t.ndepth[v], child = t.nchild[16 * (uint64_t)v + c];
    uint32_t len;
    if (wt_hash_leaf(t, child)) {
        len = 32;  // an unopened branch of at least 32 bytes, or the extension above one
    } else if (child & DT_LEAF) {
        const uint32_t x = child & ~DT_LEAF;
        uint32_t k[8];
        load32_nc(t.lkey + 32 * (uint64_t)x, k);
        const uint8_t *val = t.lval + (uint64_t)t.val_stride * x;
        CountBuf cb{0};
        len = t.account ? encode_leaf<CountBuf, true>(cb, k, (int)d, val, t.lsroot + 32 * (uint64_t)x, t.err)
                        : encode_leaf<CountBuf, false>(cb, k, (int)d, val, nullptr, t.err);
    } else {
        uint32_t sm, tm, hm;
        const uint32_t payload = dt_branch_payload<false>(t, child, sm, tm, hm);
        const uint32_t blen = list_header_len(payload) + payload, dc = t.ndepth[child];
        len = blen;
        if (dc > d + 1) {  // the node at path ‖ c is the extension above the child branch
            uint32_t e = dc - (d + 1), hp_len = 1 + (e >> 1), path_str = hp_len == 1 ? 1 : 1 + hp_len;
            uint32_t epayload = path_str + (blen >= 32 ? 33 : blen);
            len = list_header_len(epayload) + epayload;
        }
    }
    if (len < 32) return;  // embedded in the branch: revealed with it
    const uint32_t o = atomicAdd(n_out, 1u);
    out_trie[o] = t.ntrie ? t.ntrie[v] : 0;
    out_meta[o] = (uint16_t)(d + 1);
    const uint8_t *nk = t.nkey + 32 * (uint64_t)v;
    uint8_t *k = out_keys + 32 * (uint64_t)o;
    for (uint32_t b = 0; b < 32; b++) {
        const uint32_t hi = 2 * b, lo = 2 * b + 1;
        uint32_t nh = hi < d ? (nk[b] >> 4) : (hi == d ? c : 0), nl = lo < d ? (nk[b] & 15) : (lo == d ? c : 0);
        k[b] = (uint8_t)(nh << 4 | nl);
    }
}

// Wipe expansion: a read-only breadth-first walk of the wiped storage tries (the traversal of the apply's release path,
// dt_wipe_*_kernel, on a queue of its own), so its cost follows the size of those tries, not of the arena.  Every live leaf
// of a wiped trie becomes a storage target.  A queue entry is a pair (node, trie): the node is one of ts, or with DT_ALT one
// of res, the resident arena below a hash leaf of a fold; the trie is ts's, the one its leaves prove in.
static __device__ __forceinline__ void wt_wipe_push(uint32_t *queue, uint32_t *n_queue, uint32_t node, uint32_t trie) {
    const uint32_t k = atomicAdd(n_queue, 1u);
    queue[2 * (uint64_t)k] = node;
    queue[2 * (uint64_t)k + 1] = trie;
}
// child word w of a wiped trie (alt: a word of res): a node is queued, a leaf counted, a hash leaf queues the branch behind it
static __device__ void wt_wipe_child(const DTrieDev &ts, const DTrieDev &res, const uint32_t *res_trie, uint32_t w, uint32_t trie,
                                     uint32_t alt, uint32_t *queue, uint32_t *n_queue, uint32_t *n_leaves) {
    if (w == DT_NONE) return;
    if (!alt && wt_hash_leaf(ts, w)) {
        const uint32_t r = wt_fall(ts, w & ~DT_LEAF, res, res_trie ? res_trie[trie] : 0u);
        if (r != DT_NONE) wt_wipe_push(queue, n_queue, r | DT_ALT, trie);
    } else if (w & DT_LEAF) {
        atomicAdd(n_leaves, 1u);
    } else {
        wt_wipe_push(queue, n_queue, w | alt, trie);
    }
}
// roots: a leaf root is counted (WRITE: written as a target); a node root is queued (count pass only).  trie_flags nullable:
// every trie of trie_of is expanded (DT_NONE: none).
template <bool WRITE>
__global__ void wt_wipe_roots_kernel(DTrieDev ts, DTrieDev res, const uint32_t *__restrict__ res_trie, const uint32_t *__restrict__ trie_of,
                                     const uint8_t *__restrict__ trie_flags, uint64_t m, uint32_t *__restrict__ queue,
                                     uint32_t *__restrict__ n_queue, uint32_t *__restrict__ n_out, uint32_t *__restrict__ out_trie,
                                     uint8_t *__restrict__ out_keys) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint32_t trie = trie_of[i];
    if (trie == DT_NONE || (trie_flags && !(trie_flags[trie] & WF_WIPED))) return;
    const uint32_t w = ts.troot[trie];
    if (!WRITE) {
        wt_wipe_child(ts, res, res_trie, w, trie, 0u, queue, n_queue, n_out);
    } else if ((w & DT_LEAF) && !wt_hash_leaf(ts, w)) {
        const uint32_t o = atomicAdd(n_out, 1u);
        out_trie[o] = trie;
        dt_copy32(out_keys + 32 * (uint64_t)o, ts.lkey + 32 * (uint64_t)(w & ~DT_LEAF));
    }
}
// one level: queue[lo, hi) was pushed by the level before; child nodes are queued, child leaves counted
__global__ void wt_wipe_round_kernel(DTrieDev ts, DTrieDev res, const uint32_t *__restrict__ res_trie, uint32_t *__restrict__ queue,
                                     uint32_t lo, uint32_t hi, uint32_t *__restrict__ n_queue, uint32_t *__restrict__ n_leaves) {
    uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hi) return;
    const uint32_t v = queue[2 * (uint64_t)i], trie = queue[2 * (uint64_t)i + 1], alt = v & DT_ALT;
    const uint32_t *ch = (alt ? res.nchild : ts.nchild) + 16 * (uint64_t)(v & ~DT_ALT);
    for (int s = 0; s < 16; s++) wt_wipe_child(ts, res, res_trie, ch[s], trie, alt, queue, n_queue, n_leaves);
}
// every node the walk queued writes its leaf children as targets
__global__ void wt_wipe_leaves_kernel(DTrieDev ts, DTrieDev res, const uint32_t *__restrict__ queue, uint32_t n, uint32_t *__restrict__ n_out,
                                      uint32_t *__restrict__ out_trie, uint8_t *__restrict__ out_keys) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t v = queue[2 * (uint64_t)i], trie = queue[2 * (uint64_t)i + 1], alt = v & DT_ALT;
    const uint32_t *ch = (alt ? res.nchild : ts.nchild) + 16 * (uint64_t)(v & ~DT_ALT);
    const uint8_t *lkey = alt ? res.lkey : ts.lkey;
    for (int s = 0; s < 16; s++) {
        const uint32_t w = ch[s];
        if (w == DT_NONE || !(w & DT_LEAF) || (!alt && wt_hash_leaf(ts, w))) continue;
        const uint32_t o = atomicAdd(n_out, 1u);
        out_trie[o] = trie;
        dt_copy32(out_keys + 32 * (uint64_t)o, lkey + 32 * (uint64_t)(w & ~DT_LEAF));
    }
}

// After the call: the marks go back to zero along the same walks that set them (every marked branch lies on the path of
// an entry: the climbs only visit ancestors of the leaves they start from), and so do the storage trie flags, so that
// no call pays for clearing the whole arena.  trie_of: nullptr = trie 0; leaf_of (nullable): trie_flags entries to clear.
__global__ void wt_clear_kernel(DTrieDev t, WitnessMarks w, const uint32_t *__restrict__ trie_of, const uint8_t *__restrict__ keys,
                                uint64_t n, const uint32_t *__restrict__ leaf_of, uint8_t *__restrict__ trie_flags) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (leaf_of && leaf_of[i] != DT_NONE) trie_flags[leaf_of[i]] = 0;
    const uint32_t trie = trie_of ? trie_of[i] : 0;
    if (trie == DT_NONE) return;
    const uint8_t *key = keys + 32 * i;
    uint32_t cur = t.troot[trie], matched = 0;
    for (int hops = 0; hops <= DT_MAX_HOPS && cur != DT_NONE && !(cur & DT_LEAF); hops++) {
        const uint32_t d = t.ndepth[cur];
        if (dt_lcp(key, t.nkey + 32 * (uint64_t)cur, matched, d) < d) return;
        w.seen[cur] = 0;
        w.gone[cur] = 0;
        matched = d + 1;
        cur = t.nchild[16 * (uint64_t)cur + dt_nib(key, d)];
    }
}

// Proof walks of the targets [0, n_fixed + *n_extra) (meta: min_len | stop bits; trie DT_NONE = the empty trie).  A walk
// that reaches a hash leaf of a fold goes on in res, in trie res_trie[trie] (nullptr: trie 0).
template <bool WRITE>
static __device__ __forceinline__ void wt_target(const DTrieDev &t, const DTrieDev &res, const uint32_t *__restrict__ res_trie,
                                                 const uint32_t *__restrict__ trie_of, const uint8_t *__restrict__ keys,
                                                 const uint16_t *__restrict__ meta, uint64_t i, uint32_t &nn, uint64_t &nb,
                                                 uint8_t *rlp, uint64_t byte_base, uint64_t *rlp_offset, uint64_t node_base) {
    const uint32_t trie = trie_of ? trie_of[i] : 0;
    const uint16_t mt = meta ? meta[i] : 0;
    nn = 0;
    nb = 0;
    if (mt & WM_SKIP) return;
    if (trie == DT_NONE) {
        if ((mt & 0xFF) == 0) {
            if (WRITE) {
                rlp[byte_base] = 0x80;
                rlp_offset[node_base] = byte_base;
            }
            nn = 1;
            nb = 1;
        }
        return;
    }
    const uint32_t x = dt_proof_walk<WRITE, true>(t, trie, keys + 32 * i, nn, nb, rlp, byte_base, rlp_offset, nullptr, nullptr, node_base,
                                                  mt & 0xFF, mt >> 8);
    if (x == DT_NONE) return;
    const uint32_t r = wt_fall(t, x, res, res_trie ? res_trie[trie] : 0u), p = t.lparent[x];
    if (r != DT_NONE)
        dt_proof_steps<WRITE, true>(res, r, p == DT_NONE ? -1 : (int)t.ndepth[p], keys + 32 * i, nn, nb, rlp, byte_base, rlp_offset, nullptr,
                                    nullptr, node_base, mt & 0xFF, mt >> 8);
}
__global__ void wt_proof_size_kernel(DTrieDev t, DTrieDev res, const uint32_t *__restrict__ res_trie, const uint32_t *__restrict__ trie_of, const uint8_t *__restrict__ keys,
                                     const uint16_t *__restrict__ meta, uint64_t n_fixed, const uint32_t *__restrict__ n_extra, uint64_t n_max,
                                     uint32_t *__restrict__ node_count, uint64_t *__restrict__ byte_count) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    uint32_t nn = 0;
    uint64_t nb = 0;
    if (i < n_fixed + (n_extra ? *n_extra : 0u)) wt_target<false>(t, res, res_trie, trie_of, keys, meta, i, nn, nb, nullptr, 0, nullptr, 0);
    node_count[i] = nn;
    byte_count[i] = nb;
}
__global__ void wt_proof_write_kernel(DTrieDev t, DTrieDev res, const uint32_t *__restrict__ res_trie, const uint32_t *__restrict__ trie_of, const uint8_t *__restrict__ keys,
                                      const uint16_t *__restrict__ meta, uint64_t n_fixed, const uint32_t *__restrict__ n_extra,
                                      uint64_t n_max, const uint64_t *__restrict__ node_base, const uint64_t *__restrict__ byte_base,
                                      uint64_t node_shift, uint64_t byte_shift, uint8_t *__restrict__ rlp, uint64_t *__restrict__ rlp_offset) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max || i >= n_fixed + (n_extra ? *n_extra : 0u)) return;
    uint32_t nn;
    uint64_t nb;
    wt_target<true>(t, res, res_trie, trie_of, keys, meta, i, nn, nb, rlp, byte_shift + byte_base[i], rlp_offset, node_shift + node_base[i]);
}

// The account targets of a sharded state (b200_dstate_sharded_witness): t holds the 16 bucket tries and the walks start at
// the gathered root (ShardRootDev), as dt_sharded_proof_walk does.  With the root branch (two or more non-empty buckets) it
// is kept when min_len is 0, then the walk goes on from the top of the key's bucket at parent depth 0 (nothing more when the
// bucket is empty); with `only` bucket only's trie is the whole trie, walked from parent depth -1 (trie 0 of an empty state
// gives 0x80).  The bucket follows from the key; trie ids are not read.
template <bool WRITE>
static __device__ __forceinline__ void wt_sharded_target(const DTrieDev &t, const ShardRootDev &r, const uint8_t *__restrict__ keys,
                                                         const uint16_t *__restrict__ meta, uint64_t i, uint32_t &nn, uint64_t &nb,
                                                         uint8_t *rlp, uint64_t byte_base, uint64_t *rlp_offset, uint64_t node_base) {
    const uint16_t mt = meta[i];
    const uint8_t *key = keys + 32 * i;
    const uint32_t min_len = mt & 0xFF, stop = mt >> 8;
    nn = 0;
    nb = 0;
    if (mt & WM_SKIP) return;
    if (r.only >= 0) {
        dt_proof_walk<WRITE, true>(t, (uint32_t)r.only, key, nn, nb, rlp, byte_base, rlp_offset, nullptr, nullptr, node_base, min_len, stop);
        return;
    }
    if (min_len == 0) {
        const uint32_t len = *reinterpret_cast<const uint32_t *>(r.branch);
        if (WRITE) {
            for (uint32_t b = 0; b < len; b++) rlp[byte_base + b] = r.branch[4 + b];
            rlp_offset[node_base] = byte_base;
        }
        nn = 1;
        nb = len;
        if (stop & (WT_ROOT_ONLY | WT_FIRST_ONLY)) return;
    }
    const uint32_t cur = t.troot[key[0] >> 4];
    if (cur != DT_NONE)
        dt_proof_steps<WRITE, true>(t, cur, 0, key, nn, nb, rlp, byte_base, rlp_offset, nullptr, nullptr, node_base, min_len, stop);
}
__global__ void wt_sharded_proof_size_kernel(DTrieDev t, ShardRootDev r, const uint8_t *__restrict__ keys, const uint16_t *__restrict__ meta,
                                             uint64_t n_fixed, const uint32_t *__restrict__ n_extra, uint64_t n_max,
                                             uint32_t *__restrict__ node_count, uint64_t *__restrict__ byte_count) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max) return;
    uint32_t nn = 0;
    uint64_t nb = 0;
    if (i < n_fixed + *n_extra) wt_sharded_target<false>(t, r, keys, meta, i, nn, nb, nullptr, 0, nullptr, 0);
    node_count[i] = nn;
    byte_count[i] = nb;
}
__global__ void wt_sharded_proof_write_kernel(DTrieDev t, ShardRootDev r, const uint8_t *__restrict__ keys, const uint16_t *__restrict__ meta,
                                              uint64_t n_fixed, const uint32_t *__restrict__ n_extra, uint64_t n_max,
                                              const uint64_t *__restrict__ node_base, const uint64_t *__restrict__ byte_base,
                                              uint8_t *__restrict__ rlp, uint64_t *__restrict__ rlp_offset) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_max || i >= n_fixed + *n_extra) return;
    uint32_t nn;
    uint64_t nb;
    wt_sharded_target<true>(t, r, keys, meta, i, nn, nb, rlp, byte_base[i], rlp_offset, node_base[i]);
}

// After the sort by hash: keep[i] = 1 for the first of every run of equal hashes (Canonical: not the empty node 0x80),
// kept_bytes[i] its length.
__global__ void wt_unique_kernel(const uint8_t *__restrict__ sorted32, const uint32_t *__restrict__ perm, const uint64_t *__restrict__ rlp_offset,
                                 const uint8_t *__restrict__ rlp, uint64_t n, int drop_empty, uint32_t *__restrict__ keep,
                                 uint64_t *__restrict__ kept_bytes) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool head = true;
    if (i) {
        const uint4 *a = reinterpret_cast<const uint4 *>(sorted32 + 32 * (i - 1)), *b = reinterpret_cast<const uint4 *>(sorted32 + 32 * i);
        uint4 a0 = a[0], a1 = a[1], b0 = b[0], b1 = b[1];
        head = a0.x != b0.x || a0.y != b0.y || a0.z != b0.z || a0.w != b0.w || a1.x != b1.x || a1.y != b1.y || a1.z != b1.z || a1.w != b1.w;
    }
    const uint32_t k = perm[i];
    const uint64_t beg = rlp_offset[k], len = rlp_offset[k + 1] - beg;
    if (head && drop_empty && len == 1 && rlp[beg] == 0x80) head = false;
    keep[i] = head ? 1u : 0u;
    kept_bytes[i] = head ? len : 0;
}
__global__ void wt_gather_kernel(const uint8_t *__restrict__ sorted32, const uint32_t *__restrict__ perm, const uint64_t *__restrict__ rlp_offset,
                                 const uint8_t *__restrict__ rlp, uint64_t n, const uint32_t *__restrict__ keep,
                                 const uint32_t *__restrict__ pos, const uint64_t *__restrict__ byte_pos, uint8_t *__restrict__ out_hash,
                                 uint64_t *__restrict__ out_offset, uint8_t *__restrict__ out_rlp) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !keep[i]) return;
    const uint32_t o = pos[i], k = perm[i];
    dt_copy32(out_hash + 32 * (uint64_t)o, sorted32 + 32 * i);
    const uint64_t beg = rlp_offset[k], len = rlp_offset[k + 1] - beg, at = byte_pos[i];
    out_offset[o] = at;
    for (uint64_t b = 0; b < len; b++) out_rlp[at + b] = rlp[beg + b];
}

// ------------------------------------------------------------------------------------------------ launchers
cudaError_t launch_wt_accounts(const DTrieDev &ta, const DTrieDev &ts, const uint8_t *keys, const uint8_t *flags, uint64_t m,
                               const uint32_t *entry_trie, const uint32_t *acct_trie, uint32_t *leaf_of, uint32_t *trie_of,
                               uint8_t *trie_flags, cudaStream_t st) {
    if (m) wt_accounts_kernel<<<blocks_for(m, 128), 128, 0, st>>>(ta, ts, keys, flags, m, entry_trie, acct_trie, leaf_of, trie_of, trie_flags);
    return cudaGetLastError();
}
cudaError_t launch_wt_slots(const DTrieDev &ts, const WitnessMarks &w, const uint64_t *seg_offsets, uint64_t m, const uint32_t *trie_of,
                            const uint8_t *flags, const uint8_t *keys, const uint8_t *vals, uint64_t n, int canonical,
                            uint32_t *trie_of_target, uint8_t *nonzero, cudaStream_t st) {
    if (n) wt_slots_kernel<<<blocks_for(n, 128), 128, 0, st>>>(ts, w, seg_offsets, m, trie_of, flags, keys, vals, n, canonical, trie_of_target, nonzero);
    return cudaGetLastError();
}
cudaError_t launch_wt_account_walk(const DTrieDev &ta, const DTrieDev &ts, const WitnessMarks &w, const uint8_t *keys, const uint8_t *accts,
                                   const uint8_t *flags, const uint64_t *seg_offsets, uint64_t m, const uint32_t *acct_trie,
                                   const uint32_t *leaf_of, const uint32_t *trie_of, const uint8_t *trie_flags, const uint8_t *nonzero,
                                   int canonical, uint32_t *root_trie, uint16_t *root_meta, cudaStream_t st) {
    if (m)
        wt_account_walk_kernel<<<blocks_for(m, 128), 128, 0, st>>>(ta, ts, w, keys, accts, flags, seg_offsets, m, acct_trie, leaf_of, trie_of,
                                                                   trie_flags, nonzero, canonical, root_trie, root_meta);
    return cudaGetLastError();
}
cudaError_t launch_wt_reveal(const DTrieDev &t, const WitnessMarks &w, uint32_t max_list, int canonical, uint32_t *out_trie,
                             uint8_t *out_keys, uint16_t *out_meta, uint32_t *n_out, cudaStream_t st) {
    if (max_list) wt_reveal_kernel<<<blocks_for(max_list, 128), 128, 0, st>>>(t, w, max_list, canonical, out_trie, out_keys, out_meta, n_out);
    return cudaGetLastError();
}
cudaError_t launch_wt_wipe_roots(const DTrieDev &ts, const DTrieDev &res, const uint32_t *res_trie, const uint32_t *trie_of,
                                 const uint8_t *trie_flags, uint64_t m, bool write, uint32_t *queue, uint32_t *n_queue, uint32_t *n_out,
                                 uint32_t *out_trie, uint8_t *out_keys, cudaStream_t st) {
    if (!m) return cudaSuccess;
    if (write)
        wt_wipe_roots_kernel<true><<<blocks_for(m, 128), 128, 0, st>>>(ts, res, res_trie, trie_of, trie_flags, m, queue, n_queue, n_out, out_trie,
                                                                        out_keys);
    else
        wt_wipe_roots_kernel<false><<<blocks_for(m, 128), 128, 0, st>>>(ts, res, res_trie, trie_of, trie_flags, m, queue, n_queue, n_out, out_trie,
                                                                         out_keys);
    return cudaGetLastError();
}
cudaError_t launch_wt_wipe_round(const DTrieDev &ts, const DTrieDev &res, const uint32_t *res_trie, uint32_t *queue, uint32_t lo, uint32_t hi,
                                 uint32_t *n_queue, uint32_t *n_leaves, cudaStream_t st) {
    if (hi > lo) wt_wipe_round_kernel<<<blocks_for(hi - lo, 128), 128, 0, st>>>(ts, res, res_trie, queue, lo, hi, n_queue, n_leaves);
    return cudaGetLastError();
}
cudaError_t launch_wt_wipe_leaves(const DTrieDev &ts, const DTrieDev &res, const uint32_t *queue, uint32_t n, uint32_t *n_out,
                                  uint32_t *out_trie, uint8_t *out_keys, cudaStream_t st) {
    if (n) wt_wipe_leaves_kernel<<<blocks_for(n, 128), 128, 0, st>>>(ts, res, queue, n, n_out, out_trie, out_keys);
    return cudaGetLastError();
}
cudaError_t launch_wt_clear(const DTrieDev &t, const WitnessMarks &w, const uint32_t *trie_of, const uint8_t *keys, uint64_t n,
                            const uint32_t *leaf_of, uint8_t *trie_flags, cudaStream_t st) {
    if (n) wt_clear_kernel<<<blocks_for(n, 128), 128, 0, st>>>(t, w, trie_of, keys, n, leaf_of, trie_flags);
    return cudaGetLastError();
}
cudaError_t launch_wt_proof_sizes(const DTrieDev &t, const DTrieDev &res, const uint32_t *res_trie, const uint32_t *trie_of, const uint8_t *keys, const uint16_t *meta, uint64_t n_fixed,
                                  const uint32_t *n_extra, uint64_t n_max, uint32_t *node_count, uint64_t *byte_count, cudaStream_t st) {
    if (n_max) wt_proof_size_kernel<<<blocks_for(n_max, 64), 64, 0, st>>>(t, res, res_trie, trie_of, keys, meta, n_fixed, n_extra, n_max, node_count,
                                                                   byte_count);
    return cudaGetLastError();
}
cudaError_t launch_wt_proof_write(const DTrieDev &t, const DTrieDev &res, const uint32_t *res_trie, const uint32_t *trie_of, const uint8_t *keys, const uint16_t *meta, uint64_t n_fixed,
                                  const uint32_t *n_extra, uint64_t n_max, const uint64_t *node_base, const uint64_t *byte_base,
                                  uint64_t node_shift, uint64_t byte_shift, uint8_t *rlp, uint64_t *rlp_offset, cudaStream_t st) {
    if (n_max)
        wt_proof_write_kernel<<<blocks_for(n_max, 64), 64, 0, st>>>(t, res, res_trie, trie_of, keys, meta, n_fixed, n_extra, n_max, node_base, byte_base,
                                                                    node_shift, byte_shift, rlp, rlp_offset);
    return cudaGetLastError();
}
cudaError_t launch_wt_sharded_proof_sizes(const DTrieDev &t, const ShardRootDev &r, const uint8_t *keys, const uint16_t *meta, uint64_t n_fixed,
                                          const uint32_t *n_extra, uint64_t n_max, uint32_t *node_count, uint64_t *byte_count, cudaStream_t st) {
    if (n_max) wt_sharded_proof_size_kernel<<<blocks_for(n_max, 64), 64, 0, st>>>(t, r, keys, meta, n_fixed, n_extra, n_max, node_count, byte_count);
    return cudaGetLastError();
}
cudaError_t launch_wt_sharded_proof_write(const DTrieDev &t, const ShardRootDev &r, const uint8_t *keys, const uint16_t *meta, uint64_t n_fixed,
                                          const uint32_t *n_extra, uint64_t n_max, const uint64_t *node_base, const uint64_t *byte_base,
                                          uint8_t *rlp, uint64_t *rlp_offset, cudaStream_t st) {
    if (n_max)
        wt_sharded_proof_write_kernel<<<blocks_for(n_max, 64), 64, 0, st>>>(t, r, keys, meta, n_fixed, n_extra, n_max, node_base, byte_base, rlp,
                                                                            rlp_offset);
    return cudaGetLastError();
}
cudaError_t launch_wt_unique(const uint8_t *sorted32, const uint32_t *perm, const uint64_t *rlp_offset, const uint8_t *rlp, uint64_t n,
                             int drop_empty, uint32_t *keep, uint64_t *kept_bytes, cudaStream_t st) {
    if (n) wt_unique_kernel<<<blocks_for(n, 256), 256, 0, st>>>(sorted32, perm, rlp_offset, rlp, n, drop_empty, keep, kept_bytes);
    return cudaGetLastError();
}
cudaError_t launch_wt_gather(const uint8_t *sorted32, const uint32_t *perm, const uint64_t *rlp_offset, const uint8_t *rlp, uint64_t n,
                             const uint32_t *keep, const uint32_t *pos, const uint64_t *byte_pos, uint8_t *out_hash, uint64_t *out_offset,
                             uint8_t *out_rlp, cudaStream_t st) {
    if (n) wt_gather_kernel<<<blocks_for(n, 128), 128, 0, st>>>(sorted32, perm, rlp_offset, rlp, n, keep, pos, byte_pos, out_hash, out_offset, out_rlp);
    return cudaGetLastError();
}
