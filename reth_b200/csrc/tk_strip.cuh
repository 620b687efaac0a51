// tk_strip.cuh — thread-private shared-memory byte stream (Strip), its Keccak absorb, load/store and RLP helpers.
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ sponge strip
// Thread-private byte stream in shared memory.  Word w of thread t lives at base[w*BLOCK + t].
template <int BLOCK>
struct Strip {
    uint32_t *w;
    uint32_t prev;  // pending bytes are the top `nb` bytes of prev, stream order low->high
    uint32_t nb;
    uint32_t nw;
    __device__ __forceinline__ void init(uint32_t *smem) {
        w = smem + threadIdx.x;
        prev = 0;
        nb = 0;
        nw = 0;
    }
    __device__ __forceinline__ void byte(uint32_t b) {
        prev = (prev >> 8) | (b << 24);
        if (++nb == 4) {
            w[nw * BLOCK] = prev;
            nw++;
            nb = 0;
        }
    }
    // 4 stream bytes given as a little-endian word
    __device__ __forceinline__ void word(uint32_t x) {
        w[nw * BLOCK] = __funnelshift_rc(prev, x, 32 - 8 * nb);
        nw++;
        prev = x;
    }
    __device__ __forceinline__ void words8(const uint32_t (&x)[8]) {
#pragma unroll
        for (int i = 0; i < 8; i++) word(x[i]);
    }
    // `cnt` empty-slot markers (0x80), four at a time whatever the current byte alignment
    __device__ __forceinline__ void fill80(uint32_t cnt) {
        while (cnt >= 4) {
            word(0x80808080u);
            cnt -= 4;
        }
        while (cnt--) byte(0x80);
    }
    // bytes [b0, 32) of a 32-byte string held as 8 little-endian words
    __device__ __forceinline__ void tail32(const uint32_t (&x)[8], uint32_t b0) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            if (4u * i >= b0) {
                word(x[i]);
            } else if (4u * i + 3 >= b0) {
                for (uint32_t b = b0 - 4u * i; b < 4; b++) byte((x[i] >> (8 * b)) & 0xff);
            }
        }
    }
    __device__ __forceinline__ uint32_t length() const { return nw * 4 + nb; }
    __device__ __forceinline__ uint32_t read_word(uint32_t i) const { return w[i * BLOCK]; }
    // Keccak pad10*1 to a multiple of the 136-byte rate; returns the number of rate blocks.
    __device__ __forceinline__ uint32_t finish() {
        uint32_t blocks = length() / 136 + 1;
        uint32_t total_words = blocks * 34;
        byte(0x01);
        while (nb != 0) byte(0);
        while (nw < total_words) {
            w[nw * BLOCK] = 0;
            nw++;
        }
        w[(total_words - 1) * BLOCK] |= 0x80000000u;
        return blocks;
    }
    __device__ __forceinline__ void reset() {
        prev = 0;
        nb = 0;
        nw = 0;
    }
};

// keccak256 of the finished strip -> 8 little-endian digest words
template <int BLOCK>
__device__ __forceinline__ void strip_keccak(const Strip<BLOCK> &s, uint32_t blocks, uint32_t (&dig)[8]) {
    uint64_t a[25];
#pragma unroll
    for (int l = 0; l < 25; l++) a[l] = 0;
    uint32_t base = 0;
    for (uint32_t b = 0; b + 1 < blocks; b++) {
#pragma unroll
        for (int l = 0; l < 17; l++)
            a[l] ^= ((uint64_t)s.read_word(base + 2 * l + 1) << 32) | s.read_word(base + 2 * l);
        keccak_f1600(a);
        base += 34;
    }
#pragma unroll
    for (int l = 0; l < 17; l++) a[l] ^= ((uint64_t)s.read_word(base + 2 * l + 1) << 32) | s.read_word(base + 2 * l);
    keccak_f1600_final(a);
#pragma unroll
    for (int l = 0; l < 4; l++) {
        dig[2 * l] = (uint32_t)a[l];
        dig[2 * l + 1] = (uint32_t)(a[l] >> 32);
    }
}

// ------------------------------------------------------------------------------------------------ helpers
static __device__ __forceinline__ void load32(const uint8_t *p, uint32_t (&x)[8]) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    uint4 a = __ldg(q), b = __ldg(q + 1);
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w;
    x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
}
static __device__ __forceinline__ void load32_nc(const uint8_t *p, uint32_t (&x)[8]) {
    // plain (coherent) loads: data written by earlier kernels of the same build
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    uint4 a = q[0], b = q[1];
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w;
    x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
}
static __device__ __forceinline__ void load32_cg(const uint8_t *p, uint32_t (&x)[8]) {
    // L1-bypassing loads: data written by other SMs earlier in the same kernel (the wavefronts)
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    uint4 a = __ldcg(q), b = __ldcg(q + 1);
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w;
    x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
}
static __device__ __forceinline__ void store32(uint8_t *p, const uint32_t (&x)[8]) {
    uint4 *q = reinterpret_cast<uint4 *>(p);
    q[0] = make_uint4(x[0], x[1], x[2], x[3]);
    q[1] = make_uint4(x[4], x[5], x[6], x[7]);
}
// nibble i (0 = most significant) of a 32-byte big-endian key held as LE words
static __device__ __forceinline__ uint32_t key_nibble_mem(const uint8_t *key, uint32_t i) {
    uint32_t b = key[i >> 1];
    return (i & 1) ? (b & 15) : (b >> 4);
}
static __device__ __forceinline__ int depth_of(uint8_t lp) { return lp == 0xFF ? -1 : (int)lp; }
// depth of the parent of the item spanning leaves [l, r]: the deeper of its two boundary gaps (-1: the item is a whole trie)
static __device__ __forceinline__ int parent_depth(const ForestDev &f, uint64_t l, uint64_t r) {
    const int pdl = depth_of(f.Lp[l]), pdr = depth_of(f.Lp[r + 1]);
    return pdl > pdr ? pdl : pdr;
}

// Node / extension counts of a build (CNT_HASHED, CNT_EXT).  Warp-per-item kernels: lane 0 holds the warp's counts.
static __device__ __forceinline__ void flush_warp_counters(unsigned long long *counters, uint32_t hashed, uint32_t exts) {
    if ((threadIdx.x & 31) == 0) {
        if (hashed) atomicAdd(&counters[CNT_HASHED], (unsigned long long)hashed);
        if (exts) atomicAdd(&counters[CNT_EXT], (unsigned long long)exts);
    }
}
// thread-per-item kernels: one atomic per warp and counter
static __device__ __forceinline__ void flush_counters(unsigned long long *counters, uint32_t hashed, uint32_t exts) {
    for (int o = 16; o; o >>= 1) {
        hashed += __shfl_xor_sync(0xffffffffu, hashed, o);
        exts += __shfl_xor_sync(0xffffffffu, exts, o);
    }
    flush_warp_counters(counters, hashed, exts);
}

// number of leading zero BYTES of a 32-byte big-endian integer held as LE words (32 if zero)
static __device__ __forceinline__ uint32_t leading_zero_bytes(const uint32_t (&x)[8]) {
    uint32_t z = 32;
#pragma unroll
    for (int i = 7; i >= 0; i--)
        if (x[i] != 0) z = 4u * i + ((__ffs(x[i]) - 1) >> 3);
    return z;
}
static __device__ __forceinline__ uint32_t byte_at(const uint32_t (&x)[8], uint32_t j) {
    uint32_t w = 0;
#pragma unroll
    for (int i = 0; i < 8; i++)
        if ((j >> 2) == (uint32_t)i) w = x[i];
    return (w >> (8 * (j & 3))) & 0xff;
}

// byte writer over a linear buffer (a warp's shared buffer written by one lane, a proof node in global memory)
struct LinBuf {
    uint8_t *p;
    uint32_t n;
    __device__ __forceinline__ void byte(uint32_t b) { p[n++] = (uint8_t)b; }
    __device__ __forceinline__ void word(uint32_t x) {
        p[n++] = (uint8_t)x;
        p[n++] = (uint8_t)(x >> 8);
        p[n++] = (uint8_t)(x >> 16);
        p[n++] = (uint8_t)(x >> 24);
    }
    __device__ __forceinline__ void words8(const uint32_t (&x)[8]) {
#pragma unroll
        for (int i = 0; i < 8; i++) word(x[i]);
    }
    __device__ __forceinline__ void tail32(const uint32_t (&x)[8], uint32_t b0) {
        for (uint32_t b = b0; b < 32; b++) byte(byte_at(x, b));
    }
};
struct CountBuf {  // sizing pass: same interface as LinBuf, nothing is written
    uint32_t n;
    __device__ __forceinline__ void byte(uint32_t) { n++; }
    __device__ __forceinline__ void word(uint32_t) { n += 4; }
    __device__ __forceinline__ void words8(const uint32_t (&)[8]) { n += 32; }
    __device__ __forceinline__ void tail32(const uint32_t (&)[8], uint32_t b0) { n += 32 - b0; }
};

// RLP list header for a payload < 65536 bytes
template <class W>
static __device__ __forceinline__ void put_list_header(W &s, uint32_t payload) {
    if (payload < 56) {
        s.byte(0xc0 + payload);
    } else if (payload < 256) {
        s.byte(0xf8);
        s.byte(payload);
    } else {
        s.byte(0xf9);
        s.byte(payload >> 8);
        s.byte(payload & 0xff);
    }
}
static __device__ __forceinline__ uint32_t list_header_len(uint32_t payload) {
    return payload < 56 ? 1 : (payload < 256 ? 2 : 3);
}

// A child's RlpNode inside its parent: 0xa0 + the 32-byte hash (inline_len == 0), or the child's own RLP of inline_len
// < 32 bytes, written as whole words and then the 0..3 bytes of the partial one.  Every word index is a constant, so
// the reference stays in registers (a run-time byte index would put it in local memory).
template <class W>
static __device__ __forceinline__ void put_child(W &s, const uint32_t (&ref)[8], uint32_t inline_len) {
    if (inline_len == 0) {
        s.byte(0xa0);
        s.words8(ref);
        return;
    }
    uint32_t part = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        if (4u * i + 4 <= inline_len) s.word(ref[i]);
        part |= (4u * i < inline_len && inline_len < 4u * i + 4) ? ref[i] : 0u;
    }
#pragma unroll
    for (uint32_t b = 0; b < 3; b++)
        if (b < (inline_len & 3)) s.byte((part >> (8 * b)) & 0xff);
}
