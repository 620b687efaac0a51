// tk_proofs.cuh — Merkle proofs from the dynamic arenas (tk_dtrie.cuh).
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ proofs
// Merkle proofs from the resident arenas (SURVEY §8 f4): for a target key, the RLP of every node whose position is a prefix
// of the key, root first — what alloy-trie's ProofRetainer keeps while reth's Proof::account_proof / storage_proof walk
// the trie (crates/trie/trie/src/proof/mod.rs).  An extension node and the branch below it are two proof nodes; the walk
// stops at a leaf (inclusion, or exclusion by a different key), at an empty slot, or inside an extension whose nibbles
// differ from the key.  One thread per target; two passes (sizes, then bytes) around an exclusive scan.

// keccak256 of `len` bytes at an arbitrarily aligned global address (thread-serial; proofs are not a throughput path)
static __device__ void dt_keccak_global(const uint8_t *p, uint32_t len, uint32_t (&dig)[8]) {
    uint64_t a[25];
#pragma unroll
    for (int i = 0; i < 25; i++) a[i] = 0;
    uint32_t off = 0;
    for (;;) {
        uint32_t take = len - off < 136 ? len - off : 136;
        for (uint32_t lane = 0; lane < 17; lane++) {
            uint64_t w = 0;
            for (uint32_t b = 0; b < 8; b++) {
                uint32_t i = 8 * lane + b;
                uint32_t x = i < take ? p[off + i] : 0;
                if (take < 136 && i == take) x ^= 0x01;
                if (take < 136 && i == 135) x ^= 0x80;
                w |= (uint64_t)x << (8 * b);
            }
#pragma unroll
            for (int q = 0; q < 17; q++)
                if ((uint32_t)q == lane) a[q] ^= w;
        }
        keccak_f1600(a);
        off += take;
        if (take < 136) break;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        dig[2 * i] = (uint32_t)a[i];
        dig[2 * i + 1] = (uint32_t)(a[i] >> 32);
    }
}

// Walks target `key` in trie `trie`.  WRITE = false: returns node / byte counts.  WRITE = true: writes the nodes at
// rlp + byte_base and their start offsets at rlp_offset[node_base ..].
// WITNESS (tk_witness.cuh; node_depth / node_masks unused): an extension and the branch below it are one node of reth's V2
// proofs (BranchNodeV2 with a key) and TrieWitness records both RLPs (crates/trie/trie/src/witness.rs:328-343), so the
// branch below a diverging extension is kept too; only nodes whose path is at least `min_len` nibbles long are kept (an
// extension and its branch by the extension's path: ProofV2Target::with_min_len); WT_ROOT_ONLY stops after the root
// node (with its branch when it is an extension), WT_FIRST_ONLY after the first node.
// An arena made from an items fold (b200_dstate_overlay_multiproof) also holds hash leaves (lmeta META_ISNODE): the hash of a
// branch at path lkey[..lnib) that the fold did not open.  A target reaches one only where it leaves the extension above
// that branch: the proof ends with the extension node, whose child is the hash.  A target that shares the whole path
// would need the branch itself, which the fold does not have: a sticky B200_DEVERR_CORRUPT, never a wrong proof.
// dt_proof_steps: the walk goes on from child word `cur` below a node at depth pd, adding to n_nodes / n_bytes.  WITNESS, in an arena made
// from a fold: a hash leaf ends the walk with nothing kept and is returned (the caller continues in the resident arena,
// tk_witness.cuh); DT_NONE otherwise.
template <bool WRITE, bool WITNESS = false>
static __device__ uint32_t dt_proof_steps(const DTrieDev &t, uint32_t cur, int pd, const uint8_t *key, uint32_t &n_nodes, uint64_t &n_bytes,
                                          uint8_t *rlp, uint64_t byte_base, uint64_t *rlp_offset, uint8_t *node_depth,
                                          uint32_t *node_masks, uint64_t node_base, uint32_t min_len, uint32_t stop) {
    // depth = number of key nibbles that lead to the node: its path in a ProofNodes / MultiProof map is key[..depth]
    // masks: hash_mask << 16 | tree_mask of a branch node reth would store (BranchNodeMasks), 0 for everything else
    auto begin_node = [&](uint32_t len, int depth, uint32_t masks = 0) {
        if (WRITE) {
            rlp_offset[node_base + n_nodes] = byte_base + n_bytes;
            if (!WITNESS) {
                node_depth[node_base + n_nodes] = (uint8_t)depth;
                node_masks[node_base + n_nodes] = masks;
            }
        }
        n_nodes++;
        n_bytes += len;
    };
    for (int hops = 0; hops <= DT_MAX_HOPS; hops++) {
        if (cur & DT_LEAF) {
            const uint32_t x = cur & ~DT_LEAF;
            if (WITNESS && t.lnib && (t.lmeta[x] & META_ISNODE)) return x;
            const uint8_t *val = t.lval + (uint64_t)t.val_stride * x;
            if (!WITNESS && (t.lmeta[x] & META_ISNODE)) {
                const uint8_t *hk = t.lkey + 32 * (uint64_t)x;
                const uint32_t L = t.lnib[x];
                if ((int)L <= pd + 1 || dt_lcp(key, hk, (uint32_t)(pd + 1), L) == L) {
                    atomicExch(t.err, B200_DEVERR_CORRUPT);
                    return DT_NONE;
                }
                uint32_t child[8];
                for (int w = 0; w < 8; w++)
                    child[w] = (uint32_t)val[4 * w] | ((uint32_t)val[4 * w + 1] << 8) | ((uint32_t)val[4 * w + 2] << 16) |
                               ((uint32_t)val[4 * w + 3] << 24);
                const uint32_t m = L - (uint32_t)(pd + 1), hp_len = 1 + (m >> 1), path_str = hp_len == 1 ? 1 : 1 + hp_len;
                const uint32_t epayload = path_str + 33, elen = list_header_len(epayload) + epayload;
                if (WRITE) {
                    LinBuf lb{rlp + byte_base + n_bytes, 0};
                    encode_extension(lb, hk, (uint32_t)(pd + 1), L, child, 0u);
                }
                begin_node(elen, pd + 1);
                return DT_NONE;
            }
            uint32_t k[8];
            load32_nc(t.lkey + 32 * (uint64_t)x, k);
            const uint8_t *sr = t.lsroot ? t.lsroot + 32 * (uint64_t)x : nullptr;
            if (WITNESS && (uint32_t)(pd + 1) < min_len) return DT_NONE;
            CountBuf cb{0};
            uint32_t len = t.account ? encode_leaf<CountBuf, true>(cb, k, pd, val, sr, t.err) : encode_leaf<CountBuf, false>(cb, k, pd, val, nullptr, t.err);
            if (WRITE) {
                LinBuf lb{rlp + byte_base + n_bytes, 0};
                if (t.account) encode_leaf<LinBuf, true>(lb, k, pd, val, sr, t.err);
                else encode_leaf<LinBuf, false>(lb, k, pd, val, nullptr, t.err);
            }
            begin_node(len, pd + 1);
            return DT_NONE;
        }
        const uint32_t v = cur;
        const int d = t.ndepth[v];
        const uint8_t *nk = t.nkey + 32 * (uint64_t)v;
        uint32_t sm, tm, hm;
        const uint32_t payload = dt_branch_payload<false>(t, v, sm, tm, hm);
        const uint32_t blen = list_header_len(payload) + payload;
        const ushort4 mk = t.nmasks[v];
        const uint32_t masks = ((uint32_t)mk.z << 16) | mk.y;
        const bool ext = pd + 1 < d;
        const bool matches = dt_lcp(key, nk, (uint32_t)(pd + 1), (uint32_t)d) == (uint32_t)d;
        if (WITNESS && !(ext ? (uint32_t)(pd + 1) >= min_len : (uint32_t)d >= min_len)) {
            // above the wanted depth: walk on without keeping the node
            if (!matches) return DT_NONE;
        } else if (ext) {  // the extension node sits at a prefix of the key (we got here); the branch only if its nibbles match
            uint32_t m = (uint32_t)(d - (pd + 1)), hp_len = 1 + (m >> 1), path_str = hp_len == 1 ? 1 : 1 + hp_len;
            uint32_t clen = blen >= 32 ? 33 : blen;
            uint32_t epayload = path_str + clen, elen = list_header_len(epayload) + epayload;
            if (WRITE) {
                // the branch's RLP is needed first (its hash, or itself when shorter than 32 bytes, is the extension's
                // child): written to its final place right after the extension when it belongs to the proof, to a
                // thread-local buffer otherwise
                uint8_t *ext_at = rlp + byte_base + n_bytes;
                uint8_t tmp[544];
                // (WT_FIRST_ONLY keeps the extension alone: its branch was not counted, whatever the key's nibbles)
                const bool keep_br = WITNESS ? !(stop & WT_FIRST_ONLY) : matches;
                uint8_t *br_at = keep_br ? ext_at + elen : tmp;
                LinBuf br{br_at, 0};
                dt_put_branch<false>(br, t, v, payload);
                uint32_t child[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                if (blen >= 32) dt_keccak_global(br_at, blen, child);
                else
                    for (uint32_t b = 0; b < blen; b++) child[b >> 2] |= (uint32_t)br_at[b] << (8 * (b & 3));
                LinBuf lb{ext_at, 0};
                encode_extension(lb, nk, (uint32_t)(pd + 1), (uint32_t)d, child, blen >= 32 ? 0u : blen);
            }
            begin_node(elen, pd + 1);
            if (WITNESS) {
                if (stop & WT_FIRST_ONLY) return DT_NONE;
                begin_node(blen, d);
                if (!matches || (stop & (WT_ROOT_ONLY | WT_FIRST_ONLY))) return DT_NONE;
            } else {
                if (!matches) return DT_NONE;
                begin_node(blen, d, masks);
            }
        } else {
            if (WRITE) {
                LinBuf br{rlp + byte_base + n_bytes, 0};
                dt_put_branch<false>(br, t, v, payload);
            }
            begin_node(blen, d, masks);
            if (WITNESS && (stop & (WT_ROOT_ONLY | WT_FIRST_ONLY))) return DT_NONE;
        }
        pd = d;
        cur = t.nchild[16 * (uint64_t)v + dt_nib(key, (uint32_t)d)];
        if (cur == DT_NONE) return DT_NONE;  // exclusion: the branch has no child for the key's next nibble
    }
    atomicExch(t.err, B200_DEVERR_CORRUPT);
    return DT_NONE;
}
template <bool WRITE, bool WITNESS = false>
static __device__ uint32_t dt_proof_walk(const DTrieDev &t, uint32_t trie, const uint8_t *key, uint32_t &n_nodes, uint64_t &n_bytes,
                                         uint8_t *rlp, uint64_t byte_base, uint64_t *rlp_offset, uint8_t *node_depth, uint32_t *node_masks,
                                         uint64_t node_base, uint32_t min_len = 0, uint32_t stop = 0) {
    n_nodes = 0;
    n_bytes = 0;
    const uint32_t cur = t.troot[trie];
    if (cur == DT_NONE) {  // empty trie: the proof is the empty string (EMPTY_STRING_CODE), proof.rs:121-126
        if (WITNESS && min_len) return DT_NONE;
        if (WRITE) rlp[byte_base] = 0x80;
        n_nodes = 1;
        n_bytes = 1;
        if (WRITE) rlp_offset[node_base] = byte_base;
        if (WRITE && !WITNESS) {
            node_depth[node_base] = 0;
            node_masks[node_base] = 0;
        }
        return DT_NONE;
    }
    return dt_proof_steps<WRITE, WITNESS>(t, cur, -1, key, n_nodes, n_bytes, rlp, byte_base, rlp_offset, node_depth, node_masks, node_base,
                                          min_len, stop);
}

// trie_of_target: nullptr = trie 0 of t; DT_NONE entries (storage of an absent account) prove against the empty trie;
// DT_ALT | r: trie r of alt
__global__ void dt_proof_size_kernel(DTrieDev t, DTrieDev alt, const uint32_t *__restrict__ trie_of_target, const uint8_t *__restrict__ keys,
                                     uint64_t n, uint32_t *__restrict__ node_count, uint64_t *__restrict__ byte_count) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t trie = trie_of_target ? trie_of_target[i] : 0;
    uint32_t nn;
    uint64_t nb;
    if (trie == DT_NONE) {
        nn = 1;
        nb = 1;
    } else {
        dt_proof_walk<false>(trie & DT_ALT ? alt : t, trie & ~DT_ALT, keys + 32 * i, nn, nb, nullptr, 0, nullptr, nullptr, nullptr, 0);
    }
    node_count[i] = nn;
    byte_count[i] = nb;
}
__global__ void dt_proof_write_kernel(DTrieDev t, DTrieDev alt, const uint32_t *__restrict__ trie_of_target, const uint8_t *__restrict__ keys,
                                      uint64_t n, const uint64_t *__restrict__ node_base, const uint64_t *__restrict__ byte_base,
                                      uint8_t *__restrict__ rlp, uint64_t *__restrict__ rlp_offset, uint8_t *__restrict__ node_depth,
                                      uint32_t *__restrict__ node_masks) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t trie = trie_of_target ? trie_of_target[i] : 0;
    uint32_t nn;
    uint64_t nb;
    if (trie == DT_NONE) {
        rlp[byte_base[i]] = 0x80;
        rlp_offset[node_base[i]] = byte_base[i];
        node_depth[node_base[i]] = 0;
        node_masks[node_base[i]] = 0;
    } else {
        dt_proof_walk<true>(trie & DT_ALT ? alt : t, trie & ~DT_ALT, keys + 32 * i, nn, nb, rlp, byte_base[i], rlp_offset, node_depth,
                            node_masks, node_base[i]);
    }
}

// ---- proofs of a sharded state: the account arena holds the 16 bucket tries, the depth-0 root branch above them is in no
// arena (ShardRootDev, trie_kernels.h).  With the root branch, the proof is that node, then the walk from the top of the
// key's bucket at parent depth 0 (nothing more when the bucket is empty); with `only` the bucket's trie is the whole trie.
template <bool WRITE>
static __device__ void dt_sharded_proof_walk(const DTrieDev &t, const ShardRootDev &r, const uint8_t *key, uint32_t &n_nodes,
                                             uint64_t &n_bytes, uint8_t *rlp, uint64_t byte_base, uint64_t *rlp_offset,
                                             uint8_t *node_depth, uint32_t *node_masks, uint64_t node_base) {
    if (r.only >= 0) {
        dt_proof_walk<WRITE>(t, (uint32_t)r.only, key, n_nodes, n_bytes, rlp, byte_base, rlp_offset, node_depth, node_masks, node_base);
        return;
    }
    const uint32_t len = *reinterpret_cast<const uint32_t *>(r.branch);
    if (WRITE) {
        for (uint32_t b = 0; b < len; b++) rlp[byte_base + b] = r.branch[4 + b];
        rlp_offset[node_base] = byte_base;
        node_depth[node_base] = 0;
        node_masks[node_base] = r.masks;
    }
    n_nodes = 1;
    n_bytes = len;
    const uint32_t cur = t.troot[key[0] >> 4];
    if (cur != DT_NONE)
        dt_proof_steps<WRITE>(t, cur, 0, key, n_nodes, n_bytes, rlp, byte_base, rlp_offset, node_depth, node_masks, node_base, 0, 0);
}
__global__ void dt_sharded_proof_size_kernel(DTrieDev t, ShardRootDev r, const uint8_t *__restrict__ keys, uint64_t n,
                                             uint32_t *__restrict__ node_count, uint64_t *__restrict__ byte_count) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t nn;
    uint64_t nb;
    dt_sharded_proof_walk<false>(t, r, keys + 32 * i, nn, nb, nullptr, 0, nullptr, nullptr, nullptr, 0);
    node_count[i] = nn;
    byte_count[i] = nb;
}
__global__ void dt_sharded_proof_write_kernel(DTrieDev t, ShardRootDev r, const uint8_t *__restrict__ keys, uint64_t n,
                                              const uint64_t *__restrict__ node_base, const uint64_t *__restrict__ byte_base,
                                              uint8_t *__restrict__ rlp, uint64_t *__restrict__ rlp_offset,
                                              uint8_t *__restrict__ node_depth, uint32_t *__restrict__ node_masks) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t nn;
    uint64_t nb;
    dt_sharded_proof_walk<true>(t, r, keys + 32 * i, nn, nb, rlp, byte_base[i], rlp_offset, node_depth, node_masks, node_base[i]);
}

// the account leaf (= storage trie id) of one account key, DT_NONE when the account does not exist
__global__ void dt_find_leaf_kernel(DTrieDev t, const uint8_t *__restrict__ key, uint32_t *__restrict__ out, uint64_t n_copies) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_copies) return;
    DtLoc loc = dt_descend(t, t.ltrie ? (uint32_t)(key[0] >> 4) : 0u, key);
    out[i] = loc.found ? (loc.child & ~DT_LEAF) : DT_NONE;
}


// ---- multiproof batch (MultiProofTargets: accounts with their slot targets)
// leaf_out[i] = the account leaf (= storage trie id) of account key i, DT_NONE when the account does not exist; its storage
// root goes to sroot_out (nullable; EMPTY_ROOT_HASH for a missing account)
__global__ void dt_find_leaves_kernel(DTrieDev t, const uint8_t *__restrict__ keys, uint64_t n, uint32_t *__restrict__ leaf_out,
                                      uint8_t *__restrict__ sroot_out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t *key = keys + 32 * i;
    DtLoc loc = dt_descend(t, t.ltrie ? (uint32_t)(key[0] >> 4) : 0u, key);
    uint32_t leaf = loc.found ? (loc.child & ~DT_LEAF) : DT_NONE;
    leaf_out[i] = leaf;
    if (!sroot_out) return;
    if (leaf != DT_NONE && t.lsroot) dt_copy32(sroot_out + 32 * i, t.lsroot + 32 * (uint64_t)leaf);
    else dt_put_empty_root(sroot_out + 32 * i);
}
// trie_of_target[j] = leaf of the account whose slot-target segment holds j
__global__ void dt_target_tries_kernel(const uint64_t *__restrict__ seg_offsets, uint64_t n_accounts, const uint32_t *__restrict__ leaf_of,
                                       uint64_t n_targets, uint32_t *__restrict__ trie_of_target) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_targets) return;
    uint64_t lo = 0, hi = n_accounts;  // last account with offset <= j
    while (hi - lo > 1) {
        uint64_t mid = (lo + hi) >> 1;
        if (seg_offsets[mid] <= j) lo = mid;
        else hi = mid;
    }
    trie_of_target[j] = leaf_of[lo];
}
