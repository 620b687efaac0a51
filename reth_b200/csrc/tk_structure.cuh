// tk_structure.cuh — structure pass: gap depths, boundaries, bucket offsets, node heads, level ranges.
// Part of the single translation unit trie_kernels.cu (included inside namespace b200, in this order: the later
// files use the device functions of the earlier ones).

// ------------------------------------------------------------------------------------------------ structure pass
// Lp[g] for every gap; nibs[g] = (nibble of left key at Lp) << 4 | nibble of right key.  Boundaries were
// pre-marked with 0xFF by mark_boundaries_kernel and are left alone.
__global__ void lcp_kernel(const uint8_t *__restrict__ keys, uint64_t n, uint8_t *__restrict__ Lp,
                           uint8_t *__restrict__ nibs, int *__restrict__ err) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g == 0) {
        Lp[0] = 0xFF;
        Lp[n] = 0xFF;
    }
    if (g == 0 || g >= n) return;
    if (Lp[g] == 0xFF) return;
    uint32_t a[8], b[8];
    load32(keys + 32 * (g - 1), a);
    load32(keys + 32 * g, b);
    uint32_t lcp = 64, na = 0, nbb = 0;
    bool ascending = false;
#pragma unroll
    for (int i = 7; i >= 0; i--) {
        uint32_t x = __byte_perm(a[i], 0, 0x0123), y = __byte_perm(b[i], 0, 0x0123);  // big-endian numeric
        uint32_t d = x ^ y;
        if (d != 0) {
            uint32_t nz = __clz(d) >> 2;
            lcp = 8u * i + nz;
            na = (x >> (28 - 4 * nz)) & 15;
            nbb = (y >> (28 - 4 * nz)) & 15;
            ascending = x < y;
        }
    }
    if (!ascending) {  // equal or descending keys inside one trie: flag it; later kernels of the build bail out
        atomicExch(err, B200_DEVERR_UNSORTED);
        Lp[g] = 0xFF;
        return;
    }
    Lp[g] = (uint8_t)lcp;
    nibs[g] = (uint8_t)((na << 4) | nbb);
}

__global__ void mark_boundaries_kernel(const uint64_t *__restrict__ seg_offsets, uint64_t n_segs, uint64_t n,
                                       uint8_t *__restrict__ Lp, int *__restrict__ err) {
    uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s > n_segs) return;
    uint64_t o = seg_offsets[s];
    if (s == 0 && o != 0) atomicExch(err, B200_DEVERR_BAD_OFFSETS);
    if (s == n_segs && o != n) atomicExch(err, B200_DEVERR_BAD_OFFSETS);
    if (s < n_segs && seg_offsets[s + 1] < o) atomicExch(err, B200_DEVERR_BAD_OFFSETS);
    if (o > 0 && o < n) Lp[o] = 0xFF;
}

// Start of a build: the error word of the previous (possibly still unreported) build is latched into the sticky word —
// first error wins — and cleared, together with the build counters, so that this build starts clean without erasing
// what b200_sync / b200_dev_status still has to report (include/b200trie.h: violations of async calls are sticky).
__global__ void latch_error_kernel(int *__restrict__ err, int *__restrict__ sticky, unsigned long long *__restrict__ counters) {
    int e = *err;
    if (e != B200_DEVERR_NONE && *sticky == B200_DEVERR_NONE) *sticky = e;
    *err = B200_DEVERR_NONE;
    for (int i = 0; i < CNT_COUNT; i++) counters[i] = 0;
}

__global__ void iota_kernel(uint32_t *__restrict__ out, uint64_t n, uint32_t first) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = first + (uint32_t)i;
}
__global__ void fill_u32_kernel(uint32_t *__restrict__ out, uint64_t n, uint32_t value) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = value;
}

// Sort input of the gaps, in position order: val[g-1] = g, key[g-1] = depth | head << 8 | unresolved << 9 (a boundary
// gap: 0xFF, it sorts behind the real ones).  The sort looks at bits 0..7 only and is stable, so the flags travel with
// their gap.  Gap g of depth d starts a new branch node iff the nearest gap to its left that is not deeper than d is
// shallower (or a trie boundary): the run of depth-d gaps it would continue is cut there.  Forests of small tries and the
// populous deep levels of a big trie find that gap within a few bytes of Lp; a thread that has not found it after
// GAP_SCAN steps leaves the answer to head_fix_kernel (unresolved, counted).
constexpr int GAP_SCAN = 32;
constexpr uint16_t GK_HEAD = 0x100, GK_UNRESOLVED = 0x200;
__global__ void __launch_bounds__(256) gap_keys_kernel(const uint8_t *__restrict__ Lp, uint64_t G, uint16_t *__restrict__ key,
                                                       uint32_t *__restrict__ val, uint32_t *__restrict__ unresolved) {
    __shared__ uint8_t win[GAP_SCAN + 256];  // Lp[g0 - GAP_SCAN .. g0 + 255], g0 = first gap of the block
    const uint64_t g0 = (uint64_t)blockIdx.x * 256 + 1;
    for (int i = threadIdx.x; i < GAP_SCAN + 256; i += 256) {
        int64_t q = (int64_t)g0 - GAP_SCAN + i;
        win[i] = (q < 0 || (uint64_t)q > G) ? 0xFF : Lp[q];  // Lp[0] = 0xFF: the left end is a boundary
    }
    __syncthreads();
    const uint64_t g = g0 + threadIdx.x;
    if (g > G) return;
    const uint32_t d = win[GAP_SCAN + threadIdx.x];
    val[g - 1] = (uint32_t)g;
    if (d == 0xFF) {
        key[g - 1] = 0xFF;
        return;
    }
    uint32_t x = 0xFF;
    int steps = 0;
    for (; steps < GAP_SCAN; steps++) {
        x = win[GAP_SCAN + threadIdx.x - 1 - steps];
        if (x <= d || x == 0xFF) break;
    }
    uint16_t k = (uint16_t)d;
    if (steps == GAP_SCAN) {
        k |= GK_UNRESOLVED;
        atomicAdd(unresolved, 1u);
    } else if (x != d) {
        k |= GK_HEAD;
    }
    key[g - 1] = k;
}

// bucket_off[d] = first sorted position whose depth >= d, d = 0..64 (64 => number of real gaps)
__global__ void bucket_offsets_kernel(const uint16_t *__restrict__ key_sorted, uint64_t G,
                                      uint32_t *__restrict__ bucket_off) {
    uint32_t d = threadIdx.x;
    if (d > 64) return;
    uint64_t lo = 0, hi = G;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if ((key_sorted[mid] & 0xFFu) < d) lo = mid + 1;
        else hi = mid;
    }
    bucket_off[d] = (uint32_t)lo;
}

// The gaps gap_keys_kernel left open, now that the sort has put every gap next to the previous gap of its depth: sorted
// gap j (position g) continues the node of sorted gap j-1 (position gp, same depth d, more than GAP_SCAN to the left, every
// gap in the last GAP_SCAN deeper) iff both lie in one trie and the leaves gp .. g-1 share more than d nibbles.
// seg_offsets == nullptr: one trie.  Exits at once when nothing was left open (the rule for forests of small tries).
__global__ void head_fix_kernel(const uint8_t *__restrict__ keys, uint16_t *__restrict__ key_sorted,
                                const uint32_t *__restrict__ gap_sorted, const uint64_t *__restrict__ seg_offsets,
                                uint64_t n_segs, const uint32_t *__restrict__ unresolved, uint64_t G) {
    if (*unresolved == 0) return;
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= G) return;
    const uint32_t k = key_sorted[j];
    if (!(k & GK_UNRESOLVED)) return;
    const uint32_t d = k & 0xFFu;
    bool h = true;
    if (j > 0 && (key_sorted[j - 1] & 0xFFu) == d) {
        const uint32_t gp = gap_sorted[j - 1], g = gap_sorted[j];
        bool same_seg = true;
        if (seg_offsets) {  // does a trie start in (gp, g)?  first offset > gp
            uint64_t lo = 0, hi = n_segs + 1;
            while (lo < hi) {
                uint64_t mid = (lo + hi) >> 1;
                if (seg_offsets[mid] <= gp) lo = mid + 1;
                else hi = mid;
            }
            same_seg = lo > n_segs || seg_offsets[lo] >= g;
        }
        if (same_seg) {
            uint32_t a[8], b[8];
            load32(keys + 32 * (uint64_t)gp, a);
            load32(keys + 32 * (uint64_t)(g - 1), b);
            uint32_t lcp = 64;
#pragma unroll
            for (int i = 7; i >= 0; i--) {
                uint32_t x = __byte_perm(a[i] ^ b[i], 0, 0x0123);
                if (x != 0) lcp = 8u * i + (__clz(x) >> 2);
            }
            h = !(lcp > d);
        }
    }
    key_sorted[j] = (uint16_t)(d | (h ? GK_HEAD : 0));
}

// level_lo[d] = first node id whose depth >= d  (node_start is ascending in sorted-gap position)
__global__ void level_ranges_kernel(const uint32_t *__restrict__ node_start, const uint32_t *__restrict__ n_nodes_p,
                                    const uint32_t *__restrict__ bucket_off, uint32_t *__restrict__ level_lo,
                                    uint32_t *__restrict__ node_start_sentinel_target) {
    uint32_t d = threadIdx.x;
    uint32_t B = *n_nodes_p;
    if (d == 0) node_start_sentinel_target[B] = bucket_off[64];
    if (d > 64) return;
    uint32_t target = bucket_off[d];
    uint32_t lo = 0, hi = B;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (node_start[mid] < target) lo = mid + 1;
        else hi = mid;
    }
    level_lo[d] = lo;
    if (d == 0) level_lo[65] = B;
}
