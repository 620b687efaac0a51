// tk_warp.cuh — warp-per-node builder: 16 lanes assemble the child slots, shuffle-based Keccak-f over 25 lanes.
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ warp-per-node
// Small levels (the top of every trie, the dirty paths of an incremental update) hold too few nodes to fill the
// machine; there the cost is the LATENCY of one node: 1-4 dependent Keccak-f on one thread.  Here one
// warp builds one node: the 16 child slots are assembled by 16 lanes in parallel, and the permutation runs with
// the 25 lanes of the sponge state spread over 25 threads (theta/pi/chi as warp shuffles) — the layout the task
// statement sketches.  It is ~5x less ALU-efficient than the register-resident sponge but ~5x shorter in latency,
// so it is used only where a level fits in about one wave of warps.
__constant__ uint8_t KW_ROT[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};
__constant__ uint8_t KW_SRC[25] = {0, 6, 12, 18, 24, 3, 9, 10, 16, 22, 1, 7, 13, 19, 20, 4, 5, 11, 17, 23, 2, 8, 14, 15, 21};

static __device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) {
    uint32_t lo = __shfl_sync(0xffffffffu, (uint32_t)v, src);
    uint32_t hi = __shfl_sync(0xffffffffu, (uint32_t)(v >> 32), src);
    return ((uint64_t)hi << 32) | lo;
}
static __device__ __forceinline__ uint64_t rotl64_var(uint64_t x, uint32_t n) {
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    if (n & 32) {
        uint32_t t = lo;
        lo = hi;
        hi = t;
    }
    n &= 31;
    return ((uint64_t)__funnelshift_l(lo, hi, n) << 32) | __funnelshift_l(hi, lo, n);
}

struct WarpKeccak {
    int l5, l10, l15, l20, xm1, xp1, src, n1, n2;
    uint32_t rot;
    bool lane0;
    __device__ __forceinline__ void init(int lane) {
        int i = lane % 25, x = i % 5, y = i / 5;
        l5 = (i + 5) % 25; l10 = (i + 10) % 25; l15 = (i + 15) % 25; l20 = (i + 20) % 25;
        xm1 = (x + 4) % 5; xp1 = (x + 1) % 5;
        src = KW_SRC[i]; rot = KW_ROT[i];
        n1 = 5 * y + (x + 1) % 5; n2 = 5 * y + (x + 2) % 5;
        lane0 = lane == 0;
    }
    __device__ __forceinline__ void permute(uint64_t &a) const {
#pragma unroll 1
        for (int r = 0; r < 24; r++) {
            uint64_t c = a ^ shfl64(a, l5) ^ shfl64(a, l10) ^ shfl64(a, l15) ^ shfl64(a, l20);
            uint64_t d = shfl64(c, xm1) ^ rotl64<1>(shfl64(c, xp1));
            uint64_t b = shfl64(rotl64_var(a ^ d, rot), src);
            a = b ^ (~shfl64(b, n1) & shfl64(b, n2));
            if (lane0) a ^= KECCAK_RC[r];
        }
    }
    // keccak256 of buf[0 .. blocks*136) (already padded) -> 8 little-endian digest words in every lane
    __device__ __forceinline__ void digest(const uint8_t *buf, uint32_t blocks, int lane, uint32_t (&out)[8]) const {
        uint64_t a = 0;
        const uint64_t *w = reinterpret_cast<const uint64_t *>(buf);
        for (uint32_t b = 0; b < blocks; b++) {
            if (lane < 17) a ^= w[17 * b + lane];
            permute(a);
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {  // digest word i is in lane i
            uint64_t x = shfl64(a, i);
            out[2 * i] = (uint32_t)x;
            out[2 * i + 1] = (uint32_t)(x >> 32);
        }
    }
};

constexpr int WARP_BUF = 560;  // 4 rate blocks + slack, 16-byte multiple

// The assembled branch RLP (`total` bytes, padded into `blocks` rate blocks of `buf`) -> RlpNode of the node as seen from a
// parent at depth pd: hashed if >= 32 bytes (or a trie root), wrapped in an extension node when more than one nibble
// separates it from the parent.  Uniform control flow: all 32 lanes call.  Returns the meta byte (inline length | META_EXT).
__device__ __forceinline__ uint32_t warp_finish_node(uint8_t *buf, uint32_t total, uint32_t blocks, int d, int pd,
                                                     const uint8_t *key, const WarpKeccak &kw, int lane, uint32_t &hashed,
                                                     uint32_t &exts, uint32_t (&out)[8]) {
    uint32_t *bufw = reinterpret_cast<uint32_t *>(buf);
    bool is_root = pd < 0, need_ext = pd + 1 < d;
    uint32_t meta;
    if (total >= 32 || (is_root && !need_ext)) {
        kw.digest(buf, blocks, lane, out);
        meta = 0;
        hashed += lane == 0;
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) out[i] = bufw[i];
        meta = total;
    }
    if (need_ext) {
        __syncwarp();
        for (uint32_t w = lane; w < 34; w += 32) bufw[w] = 0;
        __syncwarp();
        uint32_t elen = 0;
        if (lane == 0) {
            LinBuf lb{buf, 0};
            elen = encode_extension(lb, key, (uint32_t)(pd + 1), (uint32_t)d, out, meta);
            buf[elen] |= 0x01;
            buf[135] |= 0x80;
        }
        elen = __shfl_sync(0xffffffffu, elen, 0);
        __syncwarp();
        if (elen >= 32 || is_root) {
            kw.digest(buf, 1, lane, out);
            meta = META_EXT;
            hashed += lane == 0;
        } else {
#pragma unroll
            for (int i = 0; i < 8; i++) out[i] = bufw[i];
            meta = elen | META_EXT;
        }
        exts += lane == 0;
    }
    return meta;
}

// One warp re-encodes a leaf with parent depth pd (lane 0 writes the RLP) -> its RlpNode in `out`: hashed when >= 32 bytes
// or a whole trie, else the RLP itself.  Account leaves are >= 70 bytes: always hashed.  All 32 lanes call; returns the
// meta byte (inline length, 0 = hashed).
__device__ __forceinline__ uint32_t warp_leaf_ref(bool account, uint8_t *buf, const uint8_t *key, int pd, const uint8_t *val,
                                                  const uint8_t *sroot, int *err, const WarpKeccak &kw, int lane, uint32_t &hashed,
                                                  uint32_t (&out)[8]) {
    uint32_t *bufw = reinterpret_cast<uint32_t *>(buf);
    for (uint32_t w = lane; w < 68; w += 32) bufw[w] = 0;
    __syncwarp();
    uint32_t len = 0;
    if (lane == 0) {
        uint32_t k[8];
        load32_nc(key, k);
        LinBuf lb{buf, 0};
        len = account ? encode_leaf<LinBuf, true>(lb, k, pd, val, sroot, err) : encode_leaf<LinBuf, false>(lb, k, pd, val, nullptr, err);
    }
    len = __shfl_sync(0xffffffffu, len, 0);
    if (len >= 32 || pd < 0) {
        if (lane == 0) {
            buf[len] |= 0x01;
            buf[(len / 136 + 1) * 136 - 1] |= 0x80;
        }
        __syncwarp();
        kw.digest(buf, len / 136 + 1, lane, out);
        hashed += lane == 0;
        return 0;
    }
    __syncwarp();
#pragma unroll
    for (int q = 0; q < 8; q++) out[q] = bufw[q];
    return len;
}

// One warp builds branch node v of depth d (all 32 lanes must call).  Returns through lane 0's stores.
template <bool COHERENT>
__device__ __forceinline__ void warp_build_node(const ForestDev &f, uint32_t v, int d, uint8_t *buf, const WarpKeccak &kw,
                                                int lane, uint32_t &hashed, uint32_t &exts, uint32_t (&out)[8]) {
    uint32_t *bufw = reinterpret_cast<uint32_t *>(buf);
    const uint32_t n = (uint32_t)f.n;
    uint32_t j0 = f.node_start[v], k = f.node_start[v + 1] - j0;
    if (k > 15) k = 15;
    // ---- lane c <= k owns child c
    const bool has = (uint32_t)lane <= k;
    ChildInfo ci{0, 0, 0};
    uint32_t ref[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint32_t lext = 0, rext = 0;
    if (has) {
        ci = fetch_child<COHERENT>(f, j0, (uint32_t)lane);
        const uint8_t *rp = ci.id < n ? f.leaf_ref + 32 * (uint64_t)ci.id : f.node_ref + 32 * (uint64_t)(ci.id - n);
        if (COHERENT) load32_cg(rp, ref);
        else load32_nc(rp, ref);
        if (lane == 0) lext = ci.id < n ? ci.id : f.node_l[ci.id - n];
        if ((uint32_t)lane == k) rext = ci.id < n ? ci.id : f.node_r[ci.id - n];
    }
    uint32_t clen = has ? ((ci.meta & META_LEN) ? (ci.meta & META_LEN) : 33u) : 0u;
    uint32_t bit = has ? (1u << ci.nib) : 0u;
    bool is_branch = has && (ci.id >= n || (ci.meta & META_ISNODE));
    uint32_t hbit = (is_branch && !(ci.meta & META_EXT)) ? bit : 0u;
    uint32_t tbit = (is_branch && (ci.meta & META_STORED)) ? bit : 0u;
    if (hbit && (ci.meta & META_LEN) && f.retain_updates) atomicExch(f.err, B200_DEVERR_INLINE_HASH_CHILD);
    uint32_t state_mask = __reduce_or_sync(0xffffffffu, bit);
    uint32_t hash_mask = __reduce_or_sync(0xffffffffu, hbit);
    uint32_t tree_mask = __reduce_or_sync(0xffffffffu, tbit);
    uint32_t incl = clen;  // inclusive prefix sum of child lengths
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    uint32_t children_len = __shfl_sync(0xffffffffu, incl, (int)k);
    uint32_t l = __shfl_sync(0xffffffffu, lext, 0), r = __shfl_sync(0xffffffffu, rext, (int)k);
    uint32_t payload = children_len + (15 - k) + 1;
    uint32_t hdr = list_header_len(payload), total = hdr + payload;
    uint32_t blocks = total / 136 + 1;
    for (uint32_t w = lane; w < blocks * 34; w += 32) bufw[w] = 0;
    __syncwarp();
    if (lane == 0) {
        LinBuf lb{buf, 0};
        put_list_header(lb, payload);
    }
    if (has) {  // child bytes at hdr + (lengths of earlier children) + (empty slots before this nibble)
        LinBuf lb{buf + hdr + (incl - clen) + (ci.nib - (uint32_t)lane), 0};
        put_child(lb, ref, ci.meta & META_LEN);
    }
    {  // empty slots: lane e < 16 owns nibble e
        uint32_t cb = __popc(state_mask & ((1u << (lane & 15)) - 1));
        uint32_t before = __shfl_sync(0xffffffffu, incl, cb ? (int)cb - 1 : 0);
        if (lane < 16 && !((state_mask >> lane) & 1)) buf[hdr + (cb ? before : 0u) + ((uint32_t)lane - cb)] = 0x80;
    }
    if (lane == 16) {
        buf[total - 1] = 0x80;  // value slot
        buf[total] |= 0x01;     // pad10*1
        buf[blocks * 136 - 1] |= 0x80;
    }
    __syncwarp();
    uint32_t meta = warp_finish_node(buf, total, blocks, d, parent_depth(f, l, r), f.keys + 32 * (uint64_t)l, kw, lane, hashed,
                                     exts, out);
    if (lane == 0) {
        if ((tree_mask | hash_mask) != 0) meta |= META_STORED;
        store32(f.node_ref + 32 * (uint64_t)v, out);
        f.node_meta[v] = (uint8_t)meta;
        f.node_l[v] = l;
        f.node_r[v] = r;
        f.node_masks[v] = make_ushort4((unsigned short)state_mask, (unsigned short)tree_mask,
                                       (unsigned short)hash_mask, (unsigned short)d);
        f.S[l] = n + v;
        f.E[r] = n + v;
    }
    __syncwarp();
}

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) branch_warp_kernel(ForestDev f, const uint32_t *__restrict__ node_order,
                                                                uint32_t pos_lo, uint32_t pos_hi, int d) {
    __shared__ __align__(16) uint8_t sbuf[WARPS][WARP_BUF];
    if (*(volatile int *)f.err != B200_DEVERR_NONE) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpKeccak kw;
    kw.init(lane);
    uint32_t hashed = 0, exts = 0;
    const uint32_t stride = gridDim.x * WARPS;
    for (uint64_t p64 = (uint64_t)pos_lo + blockIdx.x * WARPS + warp; p64 < pos_hi; p64 += stride) {
        uint32_t out[8];
        warp_build_node<false>(f, __ldg(node_order + p64), d, sbuf[warp], kw, lane, hashed, exts, out);
    }
    flush_warp_counters(f.counters, hashed, exts);
}
