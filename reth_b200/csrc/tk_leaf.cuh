// tk_leaf.cuh — leaf encoding (storage slot / account) and the leaf kernel.
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ leaves
// One leaf -> RlpNode.  ACCOUNT: value = rlp(TrieAccount) built on the fly (crates/trie/trie/src/trie.rs:429-432,
// crates/trie/common/src/account.rs:16-31); else value = rlp(U256) (trie.rs:668-671).
// Encodes with parent depth `pd` (suffix starts at nibble pd+1); `force_hash` for a leaf that is a whole trie.
template <class W, bool ACCOUNT>
__device__ __forceinline__ uint32_t encode_leaf(W &s, const uint32_t (&k)[8], int pd, const uint8_t *val_ptr,
                                                const uint8_t *sroot_ptr, int *err) {
    uint32_t p = (uint32_t)(pd + 1);  // first suffix nibble
    uint32_t m = 64 - p;              // suffix nibbles (1..64)
    uint32_t hp_len = 1 + (m >> 1);
    uint32_t hp_str = hp_len == 1 ? 1 : 1 + hp_len;
    uint32_t first = (p & 1) ? (0x30u | (byte_at(k, p >> 1) & 15)) : 0x20u;
    uint32_t b0 = (p + 1) >> 1;  // key bytes [b0,32) follow the flag byte

    if (!ACCOUNT) {
        uint32_t v[8];
        load32(val_ptr, v);
        uint32_t z = leading_zero_bytes(v);
        if (z == 32) {
            atomicExch(err, B200_DEVERR_ZERO_VALUE);
            z = 31;
        }
        uint32_t vb = 32 - z;
        uint32_t fb = byte_at(v, z);
        bool single = vb == 1 && fb < 0x80;
        uint32_t rlp_v = single ? 1 : 1 + vb;     // alloy_rlp::encode_fixed_size(U256)
        uint32_t val_str = single ? 1 : 1 + rlp_v;  // ... wrapped as an RLP string inside the leaf
        uint32_t payload = hp_str + val_str;
        put_list_header(s, payload);
        if (hp_len > 1) s.byte(0x80 + hp_len);
        s.byte(first);
        s.tail32(k, b0);
        if (single) {
            s.byte(fb);
        } else {
            s.byte(0x80 + rlp_v);
            s.byte(0x80 + vb);
            s.tail32(v, z);
        }
        return list_header_len(payload) + payload;
    } else {
        const uint64_t *ap = reinterpret_cast<const uint64_t *>(val_ptr);
        uint64_t nonce = __ldg(ap);
        uint32_t bal[8], code[8], sroot[8];
        {
            const uint2 *q = reinterpret_cast<const uint2 *>(val_ptr + 8);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                uint2 t = __ldg(q + i);
                bal[2 * i] = t.x;
                bal[2 * i + 1] = t.y;
            }
#pragma unroll
            for (int i = 0; i < 4; i++) {
                uint2 t = __ldg(q + 4 + i);
                code[2 * i] = t.x;
                code[2 * i + 1] = t.y;
            }
        }
        if (sroot_ptr) {
            load32_nc(sroot_ptr, sroot);
        } else {  // EMPTY_ROOT_HASH
            sroot[0] = 0x171fe856u; sroot[1] = 0xa655cc1bu; sroot[2] = 0xe64583ffu; sroot[3] = 0x6ef8c092u;
            sroot[4] = 0x1be0485bu; sroot[5] = 0xc0ad6c99u; sroot[6] = 0xb52f6201u; sroot[7] = 0x21b463e3u;
        }
        uint32_t nn = nonce == 0 ? 0 : (8 - (__clzll((long long)nonce) >> 3));
        uint32_t nonce_rlp = (nn == 0 || (nn == 1 && nonce < 0x80)) ? 1 : 1 + nn;
        uint32_t bz = leading_zero_bytes(bal);
        uint32_t bb = 32 - bz;
        uint32_t bfb = bb ? byte_at(bal, bz) : 0;
        uint32_t bal_rlp = (bb == 0 || (bb == 1 && bfb < 0x80)) ? 1 : 1 + bb;
        uint32_t inner_payload = nonce_rlp + bal_rlp + 66;  // >= 68: two-byte list header
        uint32_t inner_total = 2 + inner_payload;           // 70..110: two-byte string header
        uint32_t payload = hp_str + 2 + inner_total;        // 73..146: two-byte list header
        s.byte(0xf8);
        s.byte(payload);
        if (hp_len > 1) s.byte(0x80 + hp_len);
        s.byte(first);
        s.tail32(k, b0);
        s.byte(0xb8);
        s.byte(inner_total);
        s.byte(0xf8);
        s.byte(inner_payload);
        if (nn == 0) {
            s.byte(0x80);
        } else {
            if (nonce_rlp > 1) s.byte(0x80 + nn);
            for (int i = (int)nn - 1; i >= 0; i--) s.byte((uint32_t)(nonce >> (8 * i)) & 0xff);
        }
        if (bb == 0) {
            s.byte(0x80);
        } else if (bal_rlp == 1) {
            s.byte(bfb);
        } else {
            s.byte(0x80 + bb);
            s.tail32(bal, bz);
        }
        s.byte(0xa0);
        s.words8(sroot);
        s.byte(0xa0);
        s.words8(code);
        return 2 + payload;
    }
}

// ------------------------------------------------------------------------------------------------ storage leaf, register path
// The RLP of a storage leaf is at most 70 bytes — one rate block — and has only three variable-position pieces:
//     A (3 or 4 bytes: list header, hex-prefix string header, first path byte) | key bytes [b0, 32) | value part
// with the value part = [0x80 + 1 + vb][0x80 + vb] v[z .. 32)  (or the lone byte v[31] < 0x80).  Instead of streaming
// bytes through the shared-memory strip (~840 of the old leaf kernel's ~4950 instructions per leaf, branchy), the two
// 32-byte inputs are moved into place with barrel shifters over registers: a constant word move (free), then conditional
// word moves by 4 / 2 / 1 words (SEL) and one byte-granular funnel shift (SHF) per word — uniform control flow, no
// shared memory, ~220 ALU instructions.  The pad byte 0x01 rides along as "value byte 32".
// Valid for parent depth pd in [0, 26] (p = pd + 1 in [1, 27]): every trie that fits a GPU; other leaves take the strip.
// RLP length 22 .. 69 bytes; below 32 the leaf stays inline (meta = length) like in the strip path.
// Returns the RLP length (22 .. 69).
__device__ __forceinline__ uint32_t storage_leaf_words(const uint32_t (&k)[8], const uint32_t (&v)[8], uint32_t p, uint32_t z,
                                                       uint32_t (&mw)[18]) {
    const uint32_t hp_len = 1 + ((64 - p) >> 1);  // 19..32: the hex-prefix string always has a header byte
    const uint32_t b0 = (p + 1) >> 1;             // 1..14: key bytes [b0, 32) follow the first path byte
    const uint32_t kb = p >> 1;                   // byte holding nibble p (0..13)
    const uint32_t kw = kb < 4 ? k[0] : (kb < 8 ? k[1] : (kb < 12 ? k[2] : k[3]));
    const uint32_t first = (p & 1) ? (0x30u | ((kw >> (8 * (kb & 3))) & 15u)) : 0x20u;
    const uint32_t vb = 32 - z;                   // 1..32 value bytes
    const uint32_t fb = v[7] >> 24;               // v[31]
    const bool single = z == 31 && fb < 0x80;
    const uint32_t val_str = single ? 1u : 2u + vb;
    const uint32_t payload = 1 + hp_len + val_str;  // 21..67
    const bool two = payload >= 56;                 // two-byte list header
    const uint32_t a = two ? 4u : 3u;               // bytes in front of the key tail
    const uint32_t A = two ? (0xf8u | (payload << 8) | ((0x80u + hp_len) << 16) | (first << 24))
                           : ((0xc0u + payload) | ((0x80u + hp_len) << 8) | (first << 16));

    // ---- value: [v0 .. v31, 0x01] moved up by 2 bytes (room for its two header bytes), then down by z bytes
    uint32_t U[14];
    U[0] = v[0] << 16;
#pragma unroll
    for (int j = 1; j < 8; j++) U[j] = __funnelshift_l(v[j - 1], v[j], 16);
    U[8] = (1u << 16) | (v[7] >> 16);
#pragma unroll
    for (int j = 9; j < 14; j++) U[j] = 0;
    const uint32_t zw = z >> 2, zb8 = 8 * (z & 3);
    uint32_t W1[12], W2[11], W3[11];
#pragma unroll
    for (int j = 0; j < 12; j++) W1[j] = (zw & 4) ? (j + 4 < 14 ? U[j + 4] : 0u) : U[j];
#pragma unroll
    for (int j = 0; j < 11; j++) W2[j] = (zw & 2) ? (j + 2 < 12 ? W1[j + 2] : 0u) : W1[j];
#pragma unroll
    for (int j = 0; j < 11; j++) W3[j] = (zw & 1) ? (j + 1 < 11 ? W2[j + 1] : 0u) : W2[j];
    uint32_t Y[11];  // Y[1 .. 9] = value part at offset 0; Y[0] = Y[10] = 0 (neighbours for the shift below)
    Y[0] = 0;
    Y[10] = 0;
#pragma unroll
    for (int j = 0; j < 9; j++) Y[j + 1] = __funnelshift_r(W3[j], W3[j + 1], zb8);
    Y[1] = single ? (Y[1] >> 16) : (Y[1] | (0x81u + vb) | ((0x80u + vb) << 8));

    // ---- key: moved up by one word (free), then down by b0 + 4 - a bytes, so that key byte b0 lands at offset a
    const uint32_t dsh = b0 + 4 - a, dw = dsh >> 2, db8 = 8 * (dsh & 3);  // 1..15
    uint32_t K1[11], K2[10], X[9];
#pragma unroll
    for (int j = 0; j < 11; j++) {
        const uint32_t lo = (j >= 1 && j <= 8) ? k[j - 1] : 0u;           // KU[j]
        const uint32_t hi = (j + 2 >= 1 && j + 2 <= 8) ? k[j + 1] : 0u;   // KU[j + 2]
        K1[j] = (dw & 2) ? hi : lo;
    }
#pragma unroll
    for (int j = 0; j < 10; j++) K2[j] = (dw & 1) ? K1[j + 1] : K1[j];
#pragma unroll
    for (int j = 0; j < 9; j++) X[j] = __funnelshift_r(K2[j], K2[j + 1], db8);
    X[0] = (two ? 0u : (X[0] & 0xFF000000u)) | A;

    // ---- value part to offset a + 32 - b0 (21..35): byte shift, then up by 0..3 words from word 5
    const uint32_t ov = a + 32 - b0, bv8 = 8 * (ov & 3), rel = (ov >> 2) - 5;
    uint32_t T0[13], T1[13];
#pragma unroll
    for (int i = 0; i < 13; i++) T0[i] = i < 10 ? __funnelshift_l(Y[i], Y[i + 1], bv8) : 0u;
#pragma unroll
    for (int i = 0; i < 13; i++) T1[i] = (rel & 2) ? (i >= 2 ? T0[i - 2] : 0u) : T0[i];
#pragma unroll
    for (int i = 0; i < 5; i++) mw[i] = X[i];
#pragma unroll
    for (int i = 0; i < 13; i++) {
        const uint32_t t2 = (rel & 1) ? (i >= 1 ? T1[i - 1] : 0u) : T1[i];
        mw[5 + i] = (5 + i < 9 ? X[5 + i] : 0u) | t2;
    }
    return (two ? 2u : 1u) + payload;
}

// keccak256 of a single-block message held as 18 words (bytes 0 .. 71 of the rate block, pad 0x01 included)
__device__ __forceinline__ void keccak_single_block18(const uint32_t (&mw)[18], uint32_t (&dig)[8]) {
    uint64_t a[25];
#pragma unroll
    for (int l = 0; l < 9; l++) a[l] = ((uint64_t)mw[2 * l + 1] << 32) | mw[2 * l];
#pragma unroll
    for (int l = 9; l < 25; l++) a[l] = 0;
    a[16] = 0x8000000000000000ULL;  // last byte of the rate block
    keccak_f1600_sparse_final(a);
#pragma unroll
    for (int l = 0; l < 4; l++) {
        dig[2 * l] = (uint32_t)a[l];
        dig[2 * l + 1] = (uint32_t)(a[l] >> 32);
    }
}

// strip -> (ref words, meta): hashed when >= 32 bytes or forced
template <int BLOCK>
__device__ __forceinline__ uint32_t strip_to_ref(Strip<BLOCK> &s, uint32_t len, bool force_hash, uint32_t (&ref)[8],
                                                 uint32_t &hashed) {
    if (len >= 32 || force_hash) {
        uint32_t blocks = s.finish();
        strip_keccak(s, blocks, ref);
        hashed++;
        return 0;  // meta: hashed
    }
    while (s.nb != 0) s.byte(0);
#pragma unroll
    for (int i = 0; i < 8; i++) ref[i] = (uint32_t)i < s.nw ? s.read_word(i) : 0;
    return len;  // meta: inline length 1..31
}

template <int BLOCK, bool ACCOUNT>
__global__ void __launch_bounds__(BLOCK) leaf_kernel(ForestDev f, const uint8_t *__restrict__ values,
                                                     const uint8_t *__restrict__ storage_roots) {
    extern __shared__ uint32_t smem[];
    if (*(volatile int *)f.err == B200_DEVERR_UNSORTED || *(volatile int *)f.err == B200_DEVERR_BAD_OFFSETS) return;
    Strip<BLOCK> s;
    uint32_t hashed = 0;
    const uint64_t step = (uint64_t)gridDim.x * BLOCK;
    for (uint64_t i = (uint64_t)blockIdx.x * BLOCK + threadIdx.x; i < f.n; i += step) {
        s.init(smem);
        uint32_t k[8];
        load32(f.keys + 32 * i, k);
        const int pd = parent_depth(f, i, i);
        const uint8_t *vp = ACCOUNT ? values + (uint64_t)sizeof(b200_account_dev) * i : values + 32 * i;
        const uint8_t *sp = (ACCOUNT && storage_roots) ? storage_roots + 32 * i : nullptr;
        uint32_t len = encode_leaf<Strip<BLOCK>, ACCOUNT>(s, k, pd, vp, sp, f.err);
        uint32_t ref[8];
        uint32_t meta = strip_to_ref(s, len, pd < 0, ref, hashed);
        store32(f.leaf_ref + 32 * i, ref);
        f.leaf_meta[i] = (uint8_t)meta;
        f.S[i] = (uint32_t)i;
        f.E[i] = (uint32_t)i;
    }
    // one atomic per warp
    for (int o = 16; o; o >>= 1) hashed += __shfl_xor_sync(0xffffffffu, hashed, o);
    if ((threadIdx.x & 31) == 0 && hashed) atomicAdd(&f.counters[CNT_HASHED], (unsigned long long)hashed);
}

// Storage leaves, one per thread, plain grid (short-lived CTAs: the structure pass running next to this kernel on the
// high-priority stream gets SM slots as they free up).  Leaves outside the register path's range (a single-leaf trie,
// parent depth > 26) go through the strip like every other node.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) leaf_storage_kernel(ForestDev f, const uint8_t *__restrict__ values) {
    extern __shared__ uint32_t smem[];
    __shared__ uint32_t s_hashed;
    if (*(volatile int *)f.err == B200_DEVERR_UNSORTED || *(volatile int *)f.err == B200_DEVERR_BAD_OFFSETS) return;
    if (threadIdx.x == 0) s_hashed = 0;
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * BLOCK + threadIdx.x;
    uint32_t hashed = 0;
    if (i < f.n) {
        uint32_t k[8], v[8], ref[8];
        load32(f.keys + 32 * i, k);
        load32(values + 32 * i, v);
        const int pd = parent_depth(f, i, i);
        uint32_t meta;
        if (pd >= 0 && pd <= 26) {
            uint32_t zi = 8, zword = 0;
#pragma unroll
            for (int w = 7; w >= 0; w--)
                if (v[w] != 0) {
                    zi = (uint32_t)w;
                    zword = v[w];
                }
            uint32_t z = 4 * zi + ((uint32_t)(__ffs((int)zword) - 1) >> 3);
            if (zi == 8) {
                atomicExch(f.err, B200_DEVERR_ZERO_VALUE);
                z = 31;
            }
            uint32_t mw[18];
            const uint32_t len = storage_leaf_words(k, v, (uint32_t)(pd + 1), z, mw);
            if (len >= 32) {
                keccak_single_block18(mw, ref);
                hashed = 1;
                meta = 0;
            } else {  // inline leaf (a tiny value deep in a dense trie): the RLP itself, without the pad byte behind it
#pragma unroll
                for (int w = 0; w < 8; w++) ref[w] = (uint32_t)w == (len >> 2) ? (mw[w] & ~(0xFFu << (8 * (len & 3)))) : mw[w];
                meta = len;
            }
        } else {
            Strip<BLOCK> s;
            s.init(smem);
            uint32_t len = encode_leaf<Strip<BLOCK>, false>(s, k, pd, values + 32 * i, nullptr, f.err);
            meta = strip_to_ref(s, len, pd < 0, ref, hashed);
        }
        store32(f.leaf_ref + 32 * i, ref);
        f.leaf_meta[i] = (uint8_t)meta;
        f.S[i] = (uint32_t)i;
        f.E[i] = (uint32_t)i;
    }
    for (int o = 16; o; o >>= 1) hashed += __shfl_xor_sync(0xffffffffu, hashed, o);
    if ((threadIdx.x & 31) == 0 && hashed) atomicAdd(&s_hashed, hashed);
    __syncthreads();
    if (threadIdx.x == 0 && s_hashed) atomicAdd(&f.counters[CNT_HASHED], (unsigned long long)s_hashed);
}
