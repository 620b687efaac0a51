// tk_frontier.cuh — multi-GPU: top-nibble bucket frontier and the root from a gathered frontier.
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ multi-GPU frontier
// The frontier entry of a trie of forest f whose keys share their first nibble, from its top item (f.S of its first leaf):
// as_root is the trie's root (the item's reference as the top of its trie, which is always hashed), as_child re-encodes
// only the top node with parent depth 0.  The item is a leaf, a branch node (f.n + node id), or, when `nibs` is given (an
// items fold), possibly a hash item of depth L = nibs[item] < 64: the hash of an unrevealed branch at depth L, whose
// reference from depth 0 is that hash, wrapped in an extension over nibbles 1 .. L-1 when L > 1.
template <int BLOCK, bool ACCOUNT, bool ITEMS>
__device__ __forceinline__ void frontier_entry(Strip<BLOCK> &s, const ForestDev &f, uint32_t item, const uint8_t *__restrict__ values,
                                               const uint8_t *__restrict__ storage_roots, const uint8_t *__restrict__ nibs,
                                               FrontierEntryDev &e) {
    uint32_t ref[8], hashed = 0, exts = 0, meta;
    const uint8_t *rootp =
        item < f.n ? f.leaf_ref + 32 * (uint64_t)item : f.node_ref + 32 * (uint64_t)(item - (uint32_t)f.n);
    load32_nc(rootp, ref);
    e.as_root_len = 32;
    for (int i = 0; i < 32; i++) e.as_root[i] = (uint8_t)(ref[i >> 2] >> (8 * (i & 3)));
    const uint32_t stride = ACCOUNT ? (uint32_t)sizeof(b200_account_dev) : 32u;
    if (ITEMS && item < f.n && nibs[item] < 64) {
        const uint2 *q = reinterpret_cast<const uint2 *>(values + (uint64_t)stride * item);  // rows are 8-byte aligned
        for (int w = 0; w < 4; w++) {
            const uint2 t = __ldg(q + w);
            ref[2 * w] = t.x;
            ref[2 * w + 1] = t.y;
        }
        meta = thread_finish_node(s, ref, 0u, 0, (int)nibs[item], f.keys + 32 * (uint64_t)item, hashed, exts);
    } else if (item < f.n) {
        uint32_t k[8];
        load32(f.keys + 32 * (uint64_t)item, k);
        const uint8_t *vp = values + (uint64_t)stride * item;
        const uint8_t *sp = (ACCOUNT && storage_roots) ? storage_roots + 32 * (uint64_t)item : nullptr;
        uint32_t len = encode_leaf<Strip<BLOCK>, ACCOUNT>(s, k, 0, vp, sp, f.err);
        meta = strip_to_ref(s, len, false, ref, hashed);
    } else {
        uint32_t v = item - (uint32_t)f.n;
        uint32_t d = f.node_masks[v].w;
        uint32_t j0 = f.node_start[v], k = f.node_start[v + 1] - j0;
        uint32_t sm, tm, hm, l, r;
        uint32_t len = encode_branch_u<BLOCK, 16>(s, f, j0, k, sm, tm, hm, l, r);
        meta = strip_to_ref(s, len, false, ref, hashed);
        meta = thread_finish_node(s, ref, meta, 0, (int)d, f.keys + 32 * (uint64_t)l, hashed, exts);
    }
    LinBuf lb{e.as_child, 0};
    put_child(lb, ref, meta & META_LEN);
    e.as_child_len = (uint8_t)lb.n;
}

// For each of the 16 top-nibble buckets of this rank's account shard: the bucket's node as child of a depth-0
// root branch (as_child) and as a trie of its own (as_root).  The build treated every bucket as a separate
// trie (boundary gaps), so as_root is simply the segment root.
template <int BLOCK, bool ACCOUNT>
__global__ void frontier_kernel(ForestDev f, const uint64_t *__restrict__ bucket_offsets /*17*/,
                                const uint8_t *__restrict__ values, const uint8_t *__restrict__ storage_roots,
                                FrontierEntryDev *__restrict__ out) {
    extern __shared__ uint32_t smem[];
    uint32_t b = threadIdx.x;
    Strip<BLOCK> s;
    s.init(smem);
    if (b >= 16 || *(volatile int *)f.err != B200_DEVERR_NONE) return;
    FrontierEntryDev &e = out[b];
    for (int i = 0; i < 33; i++) e.as_child[i] = e.as_root[i] = 0;
    e.as_child_len = e.as_root_len = 0;
    uint64_t lo = bucket_offsets[b], hi = bucket_offsets[b + 1];
    if (lo < hi) frontier_entry<BLOCK, ACCOUNT, false>(s, f, f.S[lo], values, storage_roots, nullptr, e);
}

// The depth-0 root branch over a gathered frontier with two or more non-empty entries: every bucket's as_child (0x80 for an
// empty one) and an empty value; at most 3 + 16 x 33 + 1 = 532 bytes.
template <class W>
__device__ __forceinline__ void put_root_branch(W &s, const FrontierEntryDev *__restrict__ fr) {
    uint32_t payload = 1;
    for (uint32_t b = 0; b < 16; b++) payload += fr[b].as_child_len ? fr[b].as_child_len : 1;
    put_list_header(s, payload);
    for (uint32_t b = 0; b < 16; b++) {
        if (fr[b].as_child_len == 0) s.byte(0x80);
        else
            for (uint32_t i = 0; i < fr[b].as_child_len; i++) s.byte(fr[b].as_child[i]);
    }
    s.byte(0x80);
}

// Proofs of a sharded state (b200_dstate_sharded_multiproof): the root branch of the merged frontier as a proof node,
// its length (u32) at out and its RLP at out + 4 (single thread).
__global__ void root_branch_kernel(const FrontierEntryDev *__restrict__ fr, uint8_t *__restrict__ out) {
    if (threadIdx.x != 0) return;
    LinBuf lb{out + 4, 0};
    put_root_branch(lb, fr);
    *reinterpret_cast<uint32_t *>(out) = lb.n;
}

// Root from the gathered 16-entry frontier (single thread).
template <int BLOCK>
__global__ void root_from_frontier_kernel(const FrontierEntryDev *__restrict__ fr, uint8_t *__restrict__ root) {
    extern __shared__ uint32_t smem[];
    if (threadIdx.x != 0) return;
    Strip<BLOCK> s;
    s.init(smem);
    uint32_t nonempty = 0, only = 0;
    for (uint32_t b = 0; b < 16; b++)
        if (fr[b].as_root_len) {
            nonempty++;
            only = b;
        }
    uint32_t ref[8];
    if (nonempty == 0) {
        ref[0] = 0x171fe856u; ref[1] = 0xa655cc1bu; ref[2] = 0xe64583ffu; ref[3] = 0x6ef8c092u;
        ref[4] = 0x1be0485bu; ref[5] = 0xc0ad6c99u; ref[6] = 0xb52f6201u; ref[7] = 0x21b463e3u;
    } else if (nonempty == 1) {
        for (int i = 0; i < 8; i++) {
            const uint8_t *p = fr[only].as_root + 4 * i;
            ref[i] = p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24);
        }
    } else {
        put_root_branch(s, fr);
        uint32_t blocks = s.finish();
        strip_keccak(s, blocks, ref);
    }
    store32(root, ref);
}

// bucket_offsets[b] = first account whose top nibble >= b (b = 0..16)
__global__ void nibble_buckets_kernel(const uint8_t *__restrict__ keys, uint64_t n, uint64_t *__restrict__ offs) {
    uint32_t b = threadIdx.x;
    if (b > 16) return;
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if ((uint32_t)(keys[32 * mid] >> 4) < b) lo = mid + 1;
        else hi = mid;
    }
    offs[b] = lo;
}

// Multi-GPU: out[i] = the one non-empty entry of nibble i among the gathered frontiers of all ranks (rank r's 16 entries at
// all[16 * r ..]); two ranks claiming the same nibble is an input error (a rank owns whole top-nibble buckets).
__global__ void merge_frontiers_kernel(const FrontierEntryDev *__restrict__ all, int world, FrontierEntryDev *__restrict__ out,
                                       int *__restrict__ err) {
    int i = threadIdx.x;
    if (i >= 16) return;
    FrontierEntryDev e;
    e.as_child_len = 0;
    e.as_root_len = 0;
    int owners = 0;
    for (int r = 0; r < world; r++) {
        const FrontierEntryDev &c = all[16 * r + i];
        if (c.as_child_len || c.as_root_len) {
            if (!owners) e = c;
            owners++;
        }
    }
    if (owners > 1) atomicExch(err, B200_DEVERR_BAD_OFFSETS);
    if (!owners)
        for (int b = 0; b < 33; b++) e.as_child[b] = e.as_root[b] = 0;
    out[i] = e;
}

// Hash-partition (AccountHashing / StorageHashing at N > 1): owner rank of every digest by top nibble, histogram per rank
__global__ void partition_owner_kernel(const uint8_t *__restrict__ digests, uint64_t n, int world, uint8_t *__restrict__ owner,
                                       unsigned long long *__restrict__ counts) {
    __shared__ unsigned int sh[16];
    if (threadIdx.x < 16) sh[threadIdx.x] = 0;
    __syncthreads();
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t r = 0xFFu;
    if (i < n) {
        r = (uint32_t)(digests[32 * i] >> 4) * (uint32_t)world / 16u;
        owner[i] = (uint8_t)r;
    }
    // one shared-memory atomic per (warp, owner) instead of one per row
    for (int o = 0; o < world; o++) {
        const unsigned peers = __ballot_sync(0xFFFFFFFFu, r == (uint32_t)o);
        if ((threadIdx.x & 31) == 0 && peers) atomicAdd(&sh[o], (unsigned)__popc(peers));
    }
    __syncthreads();
    if (threadIdx.x < 16 && sh[threadIdx.x]) atomicAdd(&counts[threadIdx.x], (unsigned long long)sh[threadIdx.x]);
}
// digests gathered in destination order
__global__ void partition_gather_kernel(const uint8_t *__restrict__ digests, const uint32_t *__restrict__ perm, uint64_t n,
                                        uint8_t *__restrict__ out_d) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t s = perm[i];
    const uint4 *q = reinterpret_cast<const uint4 *>(digests + 32 * s);
    uint4 *o = reinterpret_cast<uint4 *>(out_d + 32 * i);
    o[0] = q[0];
    o[1] = q[1];
}
// out row i = in row perm[i], rows of `words` elements of T: one thread per element, so that a warp writes 32 consecutive
// elements and reads runs of up to `words` consecutive ones (a row of 72 bytes = 9 x 8 bytes; a thread-per-row byte loop
// is many times slower than the traffic it moves)
template <typename T>
__global__ void gather_rows_kernel(const T *__restrict__ in, uint32_t words, const uint32_t *__restrict__ perm, uint64_t n,
                                   T *__restrict__ out) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n * words) return;
    uint64_t i = g / words;
    uint32_t w = (uint32_t)(g - i * words);
    out[g] = in[(uint64_t)perm[i] * words + w];
}
