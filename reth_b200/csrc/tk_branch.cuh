// tk_branch.cuh — branch / extension encoding, the thread-per-node builder and the class-specialised branch kernel.
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ branches
struct ChildInfo {
    uint32_t id;    // < n: leaf, else n + node
    uint32_t nib;
    uint32_t meta;  // low 5 bits inline length (0 = hashed), META_EXT, META_STORED
};

// COHERENT: loads that bypass L1 (data produced by other SMs earlier in the SAME kernel: the wavefront)
template <bool COHERENT = false>
__device__ __forceinline__ ChildInfo fetch_child(const ForestDev &f, uint32_t j0, uint32_t c) {
    ChildInfo ci;
    if (c == 0) {
        uint32_t g = f.gap_sorted[j0];
        ci.id = f.E[g - 1];
        ci.nib = f.nibs[g] >> 4;
    } else {
        uint32_t g = f.gap_sorted[j0 + c - 1];
        ci.id = f.S[g];
        ci.nib = f.nibs[g] & 15;
    }
    if (COHERENT) ci.meta = ci.id < f.n ? __ldcg(f.leaf_meta + ci.id) : __ldcg(f.node_meta + (ci.id - (uint32_t)f.n));
    else ci.meta = ci.id < f.n ? f.leaf_meta[ci.id] : f.node_meta[ci.id - (uint32_t)f.n];
    return ci;
}

// hex-prefix string of key nibbles [from, to) (extension flag), as an RLP string
template <class W>
__device__ __forceinline__ uint32_t put_ext_path(W &s, const uint8_t *key, uint32_t from, uint32_t to) {
    uint32_t m = to - from;
    uint32_t hp_len = 1 + (m >> 1);
    uint32_t i = from;
    uint32_t first = 0;
    if (m & 1) {
        first = 0x10u | key_nibble_mem(key, i);
        i++;
    }
    if (hp_len > 1) s.byte(0x80 + hp_len);
    s.byte(first);  // 0x00 or 0x1n: a lone byte < 0x80 is its own RLP
    for (; i < to; i += 2) s.byte((key_nibble_mem(key, i) << 4) | key_nibble_mem(key, i + 1));
    return hp_len == 1 ? 1 : 1 + hp_len;
}

// Wraps `child` (ref words + inline length, 0 = hashed) into an extension over key nibbles [from,to).
template <class W>
__device__ __forceinline__ uint32_t encode_extension(W &s, const uint8_t *key, uint32_t from, uint32_t to,
                                                     const uint32_t (&child)[8], uint32_t child_inline_len) {
    uint32_t m = to - from;
    uint32_t hp_len = 1 + (m >> 1);
    uint32_t path_str = hp_len == 1 ? 1 : 1 + hp_len;
    uint32_t clen = child_inline_len ? child_inline_len : 33;
    uint32_t payload = path_str + clen;
    put_list_header(s, payload);
    put_ext_path(s, key, from, to);
    put_child(s, child, child_inline_len);
    return list_header_len(payload) + payload;
}

// Builds the branch node over gaps [j0, j0 + k) into the strip; returns its RLP length and the node's masks / extent.
// At most MAXC children: every per-child quantity lives in registers and all the dependent global loads of a phase
// (gap -> S/E -> meta -> ref) are issued back to back for the whole node before any of them is consumed, so one
// thread keeps up to MAXC requests in flight.
template <int BLOCK, int MAXC, bool COHERENT = false>
__device__ __forceinline__ uint32_t encode_branch_u(Strip<BLOCK> &s, const ForestDev &f, uint32_t j0, uint32_t k,
                                                    uint32_t &state_mask, uint32_t &tree_mask, uint32_t &hash_mask,
                                                    uint32_t &l, uint32_t &r) {
    const uint32_t n = (uint32_t)f.n;
    uint32_t g[MAXC - 1];
#pragma unroll
    for (int c = 0; c < MAXC - 1; c++) g[c] = (uint32_t)c < k ? f.gap_sorted[j0 + c] : 0u;
    uint32_t id[MAXC], nm[MAXC];  // nm = nibble | meta << 8
    id[0] = f.E[g[0] - 1];
    nm[0] = f.nibs[g[0]] >> 4;
#pragma unroll
    for (int c = 1; c < MAXC; c++) {
        id[c] = 0;
        nm[c] = 0;
        if ((uint32_t)c <= k) {
            id[c] = f.S[g[c - 1]];
            nm[c] = f.nibs[g[c - 1]] & 15;
        }
    }
#pragma unroll
    for (int c = 0; c < MAXC; c++)
        if ((uint32_t)c <= k) {
            const uint8_t *mp = id[c] < n ? f.leaf_meta + id[c] : f.node_meta + (id[c] - n);
            nm[c] |= (uint32_t)(COHERENT ? __ldcg(mp) : *mp) << 8;
        }
    uint32_t payload = 17;
    state_mask = tree_mask = hash_mask = 0;
    uint32_t last = id[0];
#pragma unroll
    for (int c = 0; c < MAXC; c++) {
        if ((uint32_t)c <= k) {
            uint32_t meta = nm[c] >> 8;
            payload += ((meta & META_LEN) ? (meta & META_LEN) : 33u) - 1;
            uint32_t bit = 1u << (nm[c] & 15);
            state_mask |= bit;
            if (id[c] >= n || (meta & META_ISNODE)) {
                if (!(meta & META_EXT)) {
                    hash_mask |= bit;
                    if ((meta & META_LEN) && f.retain_updates) atomicExch(f.err, B200_DEVERR_INLINE_HASH_CHILD);
                }
                if (meta & META_STORED) tree_mask |= bit;
            }
            last = id[c];
        }
    }
    l = id[0] < n ? id[0] : f.node_l[id[0] - n];
    r = last < n ? last : f.node_r[last - n];
    put_list_header(s, payload);
    uint32_t cur = 0;
#pragma unroll
    for (int c = 0; c < MAXC; c++) {
        if ((uint32_t)c <= k) {
            const uint8_t *rp = id[c] < n ? f.leaf_ref + 32 * (uint64_t)id[c] : f.node_ref + 32 * (uint64_t)(id[c] - n);
            uint32_t ref[8];
            if (COHERENT) load32_cg(rp, ref);
            else load32_nc(rp, ref);
            uint32_t nibble = nm[c] & 15;
            s.fill80(nibble - cur);
            cur = nibble;
            put_child(s, ref, (nm[c] >> 8) & META_LEN);
            cur++;
        }
    }
    s.fill80(16 - cur + 1);  // trailing empty slots + the value slot
    return list_header_len(payload) + payload;
}

// ------------------------------------------------------------------------------------------------ 2 / 3 children, register path
// The most frequent branch nodes by far (the sparse bottom of every trie: 4.8M of the 5.8M nodes of the C3 build) have two or
// three children, and all of them hashed.  Their RLP is one rate block with a fixed skeleton:
//     f8 LL | 0x80 per empty slot | a0 + 32 bytes per child | 0x80 (value)          LL = 17 + 32 c,  83 or 115 bytes
// child j (nibble n_j) starts at byte 2 + n_j + 32 j.  Start from the skeleton with 0x80 in EVERY payload byte and XOR each
// child in as (a0 | ref) ^ (80 | 80..80) moved to its offset: wherever a child lands the 0x80 cancels.  The move is a barrel
// shifter over registers (byte funnel + conditional word moves by 4 / 2 / 1, as in storage_leaf_words); no shared memory, no
// byte loop, uniform control flow.  ~320 ALU instructions against ~930 through the strip.
__device__ __forceinline__ void xor_child33(uint32_t (&m)[34], const int base_word, const uint32_t (&ref)[8], uint32_t nib, bool present) {
    // D = 0x20 | (ref ^ 0x80..80) << 8: the child's 33 bytes XOR the 0x80 they replace
    uint32_t D[11];
    uint32_t r[8];
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = present ? (ref[i] ^ 0x80808080u) : 0u;
    D[0] = 0;
    D[1] = (present ? 0x20u : 0u) | (r[0] << 8);
#pragma unroll
    for (int i = 1; i < 8; i++) D[i + 1] = __funnelshift_l(r[i - 1], r[i], 8);
    D[9] = r[7] >> 24;
    D[10] = 0;
    const uint32_t s = nib + 2, sw = s >> 2, sb8 = 8 * (s & 3);  // byte offset inside the window: 2 .. 17
    uint32_t T0[14], T1[14], T2[14];
#pragma unroll
    for (int i = 0; i < 14; i++) T0[i] = i < 10 ? __funnelshift_l(D[i], D[i + 1], sb8) : 0u;
#pragma unroll
    for (int i = 0; i < 14; i++) T1[i] = (sw & 4) ? (i >= 4 ? T0[i - 4] : 0u) : T0[i];
#pragma unroll
    for (int i = 0; i < 14; i++) T2[i] = (sw & 2) ? (i >= 2 ? T1[i - 2] : 0u) : T1[i];
#pragma unroll
    for (int i = 0; i < 14; i++) {
        const uint32_t t3 = (sw & 1) ? (i >= 1 ? T2[i - 1] : 0u) : T2[i];
        if (base_word + i < 34) m[base_word + i] ^= t3;
    }
}

// children = 2 | 3, all hashed: the padded single block of the node's RLP as 34 words
__device__ __forceinline__ void branch23_words(const uint32_t (&r0)[8], const uint32_t (&r1)[8], const uint32_t (&r2)[8], uint32_t n0,
                                               uint32_t n1, uint32_t n2, bool three, uint32_t (&m)[34]) {
    // skeleton: f8 LL, 0x80 up to the end of the payload (83 / 115 bytes), pad 0x01 behind it, 0x80 in the last rate byte
#pragma unroll
    for (int w = 0; w < 34; w++) {
        uint32_t two_v = w == 0 ? 0x808051f8u : (w < 20 ? 0x80808080u : (w == 20 ? 0x01808080u : 0u));
        uint32_t three_v = w == 0 ? 0x808071f8u : (w < 28 ? 0x80808080u : (w == 28 ? 0x01808080u : 0u));
        if (w == 33) {
            two_v = 0x80000000u;
            three_v = 0x80000000u;
        }
        m[w] = two_v == three_v ? two_v : (three ? three_v : two_v);
    }
    xor_child33(m, 0, r0, n0, true);
    xor_child33(m, 8, r1, n1, true);
    xor_child33(m, 16, r2, n2, three);
}

// The reference (ref, meta) of a node of depth d as seen from its parent at depth pd: wrapped into an extension node over
// key nibbles [pd + 1, d) when more than one nibble separates the two (through the strip, which the node's own RLP no
// longer needs).  Returns the new meta.
template <int BLOCK>
__device__ __forceinline__ uint32_t thread_finish_node(Strip<BLOCK> &s, uint32_t (&ref)[8], uint32_t meta, int pd, int d,
                                                       const uint8_t *key, uint32_t &hashed, uint32_t &exts) {
    if (pd + 1 >= d) return meta;
    s.reset();
    uint32_t elen = encode_extension(s, key, (uint32_t)(pd + 1), (uint32_t)d, ref, meta);
    exts++;
    return strip_to_ref(s, elen, pd < 0, ref, hashed) | META_EXT;
}

// One thread builds branch node v of depth d into its strip, hashes it and publishes it (node arrays, S/E).
template <int BLOCK, int MAXC, bool COHERENT>
__device__ __forceinline__ void thread_build_node(Strip<BLOCK> &s, uint32_t *smem, const ForestDev &f, uint32_t v, int d,
                                                  uint32_t &hashed, uint32_t &exts, uint32_t (&ref)[8]) {
    s.init(smem);
    uint32_t j0 = f.node_start[v], k = f.node_start[v + 1] - j0;
    if (k + 1 > (uint32_t)MAXC) k = MAXC - 1;  // cannot happen for well-formed input; keeps the strip in bounds
    uint32_t state_mask, tree_mask, hash_mask, l, r;
    uint32_t meta;
    bool done = false;
    if constexpr (MAXC == 3 && !COHERENT) {
        // ---- register path: gather as encode_branch_u does, then assemble the block in registers
        const uint32_t n = (uint32_t)f.n;
        const uint32_t g0 = f.gap_sorted[j0], g1 = k >= 2 ? f.gap_sorted[j0 + 1] : g0;
        uint32_t id[3], nb[3], mt[3];
        id[0] = f.E[g0 - 1];
        nb[0] = f.nibs[g0] >> 4;
        id[1] = f.S[g0];
        nb[1] = f.nibs[g0] & 15;
        id[2] = k >= 2 ? f.S[g1] : id[1];
        nb[2] = k >= 2 ? (uint32_t)(f.nibs[g1] & 15) : 15u;
#pragma unroll
        for (int c = 0; c < 3; c++) mt[c] = id[c] < n ? f.leaf_meta[id[c]] : f.node_meta[id[c] - n];
        const bool three = k >= 2;
        if (k >= 1 && ((mt[0] | mt[1] | (three ? mt[2] : 0u)) & META_LEN) == 0) {
            uint32_t rr[3][8];
#pragma unroll
            for (int c = 0; c < 3; c++)
                load32_nc(id[c] < n ? f.leaf_ref + 32 * (uint64_t)id[c] : f.node_ref + 32 * (uint64_t)(id[c] - n), rr[c]);
            state_mask = tree_mask = hash_mask = 0;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                if (c < 2 || three) {
                    const uint32_t bit = 1u << nb[c];
                    state_mask |= bit;
                    if (id[c] >= n || (mt[c] & META_ISNODE)) {
                        if (!(mt[c] & META_EXT)) hash_mask |= bit;
                        if (mt[c] & META_STORED) tree_mask |= bit;
                    }
                }
            }
            const uint32_t last = three ? id[2] : id[1];
            l = id[0] < n ? id[0] : f.node_l[id[0] - n];
            r = last < n ? last : f.node_r[last - n];
            uint32_t m[34];
            branch23_words(rr[0], rr[1], rr[2], nb[0], nb[1], nb[2], three, m);
            uint64_t a[25];
#pragma unroll
            for (int q = 0; q < 17; q++) a[q] = ((uint64_t)m[2 * q + 1] << 32) | m[2 * q];
#pragma unroll
            for (int q = 17; q < 25; q++) a[q] = 0;
            keccak_f1600_final(a);
#pragma unroll
            for (int q = 0; q < 4; q++) {
                ref[2 * q] = (uint32_t)a[q];
                ref[2 * q + 1] = (uint32_t)(a[q] >> 32);
            }
            hashed++;
            meta = 0;
            done = true;
        }
    }
    uint32_t len = 0;
    if (!done) len = encode_branch_u<BLOCK, MAXC, COHERENT>(s, f, j0, k, state_mask, tree_mask, hash_mask, l, r);
    const int pd = parent_depth(f, l, r);
    if (!done) meta = strip_to_ref(s, len, pd < 0 && pd + 1 >= d, ref, hashed);
    meta = thread_finish_node(s, ref, meta, pd, d, f.keys + 32 * (uint64_t)l, hashed, exts);
    bool stored = (tree_mask | hash_mask) != 0;
    if (stored) meta |= META_STORED;
    store32(f.node_ref + 32 * (uint64_t)v, ref);
    f.node_meta[v] = (uint8_t)meta;
    f.node_l[v] = l;
    f.node_r[v] = r;
    f.node_masks[v] = make_ushort4((unsigned short)state_mask, (unsigned short)tree_mask, (unsigned short)hash_mask,
                                   (unsigned short)d);
    f.S[l] = (uint32_t)f.n + v;
    f.E[r] = (uint32_t)f.n + v;
}

// ------------------------------------------------------------------------------------------------ class 0, software-pipelined
// The thread-per-node kernels gather through four dependent loads (node -> gap -> S/E -> meta/ref); ncu shows them stalled
// on exactly that (long-scoreboard stalls).  For the
// class that holds most nodes (2 / 3 children, register path) the gather of node i+1 is therefore spread over the
// permutation of node i: one level of the chain is issued after every six rounds, so every load has six rounds of ALU work of
// the same thread (and of its neighbours) in front of its first use.
struct PrefetchedNode3 {
    uint32_t v, j0, k;      // node, first gap (sorted order), number of gaps (children - 1)
    uint32_t g0, g1;        // gap positions
    uint32_t id[3], nb[3], mt[3];
    uint32_t rr[3][8];
    uint32_t nl, nr;        // node_l / node_r of the first / last child when those are nodes
    bool valid;
};

template <int BLOCK>
__device__ __forceinline__ void pf3_stage_a(const ForestDev &f, const uint32_t *__restrict__ node_order, uint64_t p, uint32_t pos_hi,
                                            PrefetchedNode3 &x) {
    x.valid = p < pos_hi;
    if (x.valid) {
        x.v = __ldg(node_order + p);
        x.j0 = f.node_start[x.v];
        x.k = f.node_start[x.v + 1] - x.j0;
    }
}
__device__ __forceinline__ void pf3_stage_b(const ForestDev &f, PrefetchedNode3 &x) {
    if (x.valid) {
        x.g0 = f.gap_sorted[x.j0];
        x.g1 = x.k >= 2 ? f.gap_sorted[x.j0 + 1] : x.g0;
    }
}
__device__ __forceinline__ void pf3_stage_c(const ForestDev &f, PrefetchedNode3 &x) {
    if (x.valid) {
        const uint32_t nib0 = f.nibs[x.g0], nib1 = f.nibs[x.g1];
        x.id[0] = f.E[x.g0 - 1];
        x.id[1] = f.S[x.g0];
        x.id[2] = x.k >= 2 ? f.S[x.g1] : x.id[1];
        x.nb[0] = nib0 >> 4;
        x.nb[1] = nib0 & 15;
        x.nb[2] = x.k >= 2 ? (nib1 & 15) : 15u;
    }
}
__device__ __forceinline__ void pf3_stage_d(const ForestDev &f, PrefetchedNode3 &x) {
    if (x.valid) {
        const uint32_t n = (uint32_t)f.n;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            x.mt[c] = x.id[c] < n ? f.leaf_meta[x.id[c]] : f.node_meta[x.id[c] - n];
            load32_nc(x.id[c] < n ? f.leaf_ref + 32 * (uint64_t)x.id[c] : f.node_ref + 32 * (uint64_t)(x.id[c] - n), x.rr[c]);
        }
        const uint32_t last = x.k >= 2 ? x.id[2] : x.id[1];
        x.nl = x.id[0] < n ? x.id[0] : f.node_l[x.id[0] - n];
        x.nr = last < n ? last : f.node_r[last - n];
    }
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 4) branch3_pipelined_kernel(ForestDev f, const uint32_t *__restrict__ node_order,
                                                                  uint32_t pos_lo, uint32_t pos_hi, int d) {
    extern __shared__ uint32_t smem[];
    if (*(volatile int *)f.err != B200_DEVERR_NONE) return;
    Strip<BLOCK> s;
    s.init(smem);
    uint32_t hashed = 0, exts = 0;
    const uint32_t step = gridDim.x * BLOCK;
    const uint32_t n = (uint32_t)f.n;
    uint64_t p = (uint64_t)pos_lo + blockIdx.x * BLOCK + threadIdx.x;
    PrefetchedNode3 cur;
    pf3_stage_a<BLOCK>(f, node_order, p, pos_hi, cur);
    pf3_stage_b(f, cur);
    pf3_stage_c(f, cur);
    pf3_stage_d(f, cur);
    while (cur.valid) {
        PrefetchedNode3 nx;
        pf3_stage_a<BLOCK>(f, node_order, p + step, pos_hi, nx);
        const uint32_t v = cur.v, l = cur.nl, r = cur.nr;
        const bool three = cur.k >= 2;
        const bool fast = cur.k >= 1 && cur.k <= 2 && ((cur.mt[0] | cur.mt[1] | (three ? cur.mt[2] : 0u)) & META_LEN) == 0;
        const uint8_t lpl = f.Lp[l], lpr = f.Lp[(uint64_t)r + 1];  // consumed after the permutation
        uint32_t ref[8], meta = 0, state_mask = 0, tree_mask = 0, hash_mask = 0;
        if (fast) {
#pragma unroll
            for (int c = 0; c < 3; c++) {
                if (c < 2 || three) {
                    const uint32_t bit = 1u << cur.nb[c];
                    state_mask |= bit;
                    if (cur.id[c] >= n || (cur.mt[c] & META_ISNODE)) {
                        if (!(cur.mt[c] & META_EXT)) hash_mask |= bit;
                        if (cur.mt[c] & META_STORED) tree_mask |= bit;
                    }
                }
            }
            uint64_t a[25];
            {
                uint32_t m[34];
                branch23_words(cur.rr[0], cur.rr[1], cur.rr[2], cur.nb[0], cur.nb[1], cur.nb[2], three, m);
#pragma unroll
                for (int q = 0; q < 17; q++) a[q] = ((uint64_t)m[2 * q + 1] << 32) | m[2 * q];
#pragma unroll
                for (int q = 17; q < 25; q++) a[q] = 0;
            }
            keccak_rounds<0, 6>(a);
            pf3_stage_b(f, nx);
            keccak_rounds<6, 12>(a);
            pf3_stage_c(f, nx);
            keccak_rounds<12, 17>(a);
            pf3_stage_d(f, nx);
            keccak_rounds<17, 23>(a);
            keccak_round(a, 0x8000000080008008ULL);  // last round: only lanes 0..3 are consumed
#pragma unroll
            for (int q = 0; q < 4; q++) {
                ref[2 * q] = (uint32_t)a[q];
                ref[2 * q + 1] = (uint32_t)(a[q] >> 32);
            }
            hashed++;
            int pdl = depth_of(lpl), pdr = depth_of(lpr);
            int pd = pdl > pdr ? pdl : pdr;
            meta = thread_finish_node(s, ref, 0u, pd, d, f.keys + 32 * (uint64_t)l, hashed, exts);  // rare for hashed keys
            if ((tree_mask | hash_mask) != 0) meta |= META_STORED;
            store32(f.node_ref + 32 * (uint64_t)v, ref);
            f.node_meta[v] = (uint8_t)meta;
            f.node_l[v] = l;
            f.node_r[v] = r;
            f.node_masks[v] = make_ushort4((unsigned short)state_mask, (unsigned short)tree_mask, (unsigned short)hash_mask,
                                           (unsigned short)d);
            f.S[l] = n + v;
            f.E[r] = n + v;
        } else {  // an inline (< 32 byte) child, or a node outside the class: the general builder (loads everything again)
            pf3_stage_b(f, nx);
            pf3_stage_c(f, nx);
            pf3_stage_d(f, nx);
            thread_build_node<BLOCK, 3, false>(s, smem, f, v, d, hashed, exts, ref);
        }
        cur = nx;
        p += step;
    }
    flush_counters(f.counters, hashed, exts);
}

// One thread per branch node of depth d.  MAXC bounds the children of every node in [pos_lo, pos_hi) (the level's
// nodes are grouped by child-count class); the strip is sized for that class, which is what sets the occupancy.
template <int BLOCK, int MAXC>
__global__ void __launch_bounds__(BLOCK) branch_kernel(ForestDev f, const uint32_t *__restrict__ node_order,
                                                       uint32_t pos_lo, uint32_t pos_hi, int d) {
    extern __shared__ uint32_t smem[];
    if (*(volatile int *)f.err != B200_DEVERR_NONE) return;  // malformed input: the structure arrays are not trustworthy
    Strip<BLOCK> s;
    uint32_t hashed = 0, exts = 0;
    const uint32_t step = gridDim.x * BLOCK;
    for (uint64_t p64 = (uint64_t)pos_lo + blockIdx.x * BLOCK + threadIdx.x; p64 < pos_hi; p64 += step) {
        uint32_t ref[8];
        thread_build_node<BLOCK, MAXC, false>(s, smem, f, __ldg(node_order + p64), d, hashed, exts, ref);
    }
    flush_counters(f.counters, hashed, exts);
}
