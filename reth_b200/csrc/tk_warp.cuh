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
    // keccak256 of buf[0 .. blocks*136) (already padded); digest word i ends up in lane i (i < 4)
    __device__ __forceinline__ uint64_t hash(const uint8_t *buf, uint32_t blocks, int lane) const {
        uint64_t a = 0;
        const uint64_t *w = reinterpret_cast<const uint64_t *>(buf);
        for (uint32_t b = 0; b < blocks; b++) {
            if (lane < 17) a ^= w[17 * b + lane];
            permute(a);
        }
        return a;
    }
};

// byte writer over a warp's linear shared buffer (single-lane use)
struct LinBuf {
    uint8_t *p;
    uint32_t n;
    __device__ __forceinline__ void byte(uint32_t b) { p[n++] = (uint8_t)b; }
    __device__ __forceinline__ void tail32(const uint32_t (&x)[8], uint32_t b0) {
        for (uint32_t b = b0; b < 32; b++) byte(byte_at(x, b));
    }
    __device__ __forceinline__ void words8(const uint32_t (&x)[8]) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            p[n++] = (uint8_t)x[i];
            p[n++] = (uint8_t)(x[i] >> 8);
            p[n++] = (uint8_t)(x[i] >> 16);
            p[n++] = (uint8_t)(x[i] >> 24);
        }
    }
};

constexpr int WARP_BUF = 560;  // 4 rate blocks + slack, 16-byte multiple

// fetch_child with loads that bypass L1 (data produced by other SMs earlier in the SAME kernel: the wavefront)
template <bool COHERENT>
__device__ __forceinline__ ChildInfo fetch_child_c(const ForestDev &f, uint32_t j0, uint32_t c) {
    if (!COHERENT) return fetch_child(f, j0, c);
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
    ci.meta = ci.id < f.n ? __ldcg(f.leaf_meta + ci.id) : __ldcg(f.node_meta + (ci.id - (uint32_t)f.n));
    return ci;
}

// (Same steps as the tail of warp_build_node below, which keeps its own copy so that its SASS stays as measured.)
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
        uint64_t a = kw.hash(buf, blocks, lane);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            uint64_t w = shfl64(a, i);
            out[2 * i] = (uint32_t)w;
            out[2 * i + 1] = (uint32_t)(w >> 32);
        }
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
            uint64_t a = kw.hash(buf, 1, lane);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                uint64_t w = shfl64(a, i);
                out[2 * i] = (uint32_t)w;
                out[2 * i + 1] = (uint32_t)(w >> 32);
            }
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
        ci = fetch_child_c<COHERENT>(f, j0, (uint32_t)lane);
        const uint8_t *rp = ci.id < n ? f.leaf_ref + 32 * (uint64_t)ci.id : f.node_ref + 32 * (uint64_t)(ci.id - n);
        if (COHERENT) {
            const uint4 *q = reinterpret_cast<const uint4 *>(rp);
            uint4 x = __ldcg(q), y = __ldcg(q + 1);
            ref[0] = x.x; ref[1] = x.y; ref[2] = x.z; ref[3] = x.w;
            ref[4] = y.x; ref[5] = y.y; ref[6] = y.z; ref[7] = y.w;
        } else {
            load32_nc(rp, ref);
        }
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
        uint32_t off = hdr + (incl - clen) + (ci.nib - (uint32_t)lane);
        if ((ci.meta & META_LEN) == 0) {
            buf[off++] = 0xa0;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                buf[off++] = (uint8_t)ref[i];
                buf[off++] = (uint8_t)(ref[i] >> 8);
                buf[off++] = (uint8_t)(ref[i] >> 16);
                buf[off++] = (uint8_t)(ref[i] >> 24);
            }
        } else {
            for (uint32_t b = 0; b < clen; b++) buf[off++] = (uint8_t)byte_at(ref, b);
        }
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
    // ---- parent depth, extension, hash (uniform control flow)
    int pdl = depth_of(f.Lp[l]), pdr = depth_of(f.Lp[(uint64_t)r + 1]);
    int pd = pdl > pdr ? pdl : pdr;
    bool is_root = pd < 0, need_ext = pd + 1 < d;
    uint32_t meta;
    if (total >= 32 || (is_root && !need_ext)) {
        uint64_t a = kw.hash(buf, blocks, lane);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            uint64_t w = shfl64(a, i);
            out[2 * i] = (uint32_t)w;
            out[2 * i + 1] = (uint32_t)(w >> 32);
        }
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
            elen = encode_extension(lb, f.keys + 32 * (uint64_t)l, (uint32_t)(pd + 1), (uint32_t)d, out, meta);
            buf[elen] |= 0x01;
            buf[135] |= 0x80;
        }
        elen = __shfl_sync(0xffffffffu, elen, 0);
        __syncwarp();
        if (elen >= 32 || is_root) {
            uint64_t a = kw.hash(buf, 1, lane);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                uint64_t w = shfl64(a, i);
                out[2 * i] = (uint32_t)w;
                out[2 * i + 1] = (uint32_t)(w >> 32);
            }
            meta = META_EXT;
            hashed += lane == 0;
        } else {
#pragma unroll
            for (int i = 0; i < 8; i++) out[i] = bufw[i];
            meta = elen | META_EXT;
        }
        exts += lane == 0;
    }
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
    if (lane == 0) {
        if (hashed) atomicAdd(&f.counters[CNT_HASHED], (unsigned long long)hashed);
        if (exts) atomicAdd(&f.counters[CNT_EXT], (unsigned long long)exts);
    }
}
