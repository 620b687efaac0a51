// tk_changesets.cuh — trie changesets of a block out of the dynamic arenas, read-only: reth's compute_trie_changesets
// (crates/trie/trie/src/changesets.rs:50-239) with the resident state as the trie cursor factory.  Part of the single
// translation unit trie_kernels.cu (included inside namespace b200, after tk_witness.cuh).
//
// A changeset record is a path of a trie and the stored node the tables hold at exactly that path before the block, or
// None.  The records come from the block's changed paths (one thread each walks down: cs_find) and, for a deleted storage
// trie, from every stored node of it (the wipe walk of tk_witness.cuh queues every node of those tries).  A row names one
// record: output trie id << 32 | source, the source being a changed-path index or CS_NODE | a node id.  A changed path of a
// deleted trie that finds a stored node is left out: the wipe walk lists that node, so the merge keeps the stored node.

constexpr uint32_t CS_NODE = 0x80000000u;

// a node reth stores: a branch with tree_mask | hash_mask != 0, at a non-empty path (dt_stored_flags_kernel's rule)
static __device__ __forceinline__ bool cs_stored(const DTrieDev &t, uint32_t v) {
    return t.ndepth[v] != DT_DEAD && t.ndepth[v] != 0 && (t.nmeta[v] & META_STORED);
}

// The stored node of `trie` at exactly the first `len` nibbles of `path`, or DT_NONE: the walk ends at an empty slot, at a
// leaf, at a node deeper than the path (the path ends inside the extension above it) or where the keys disagree.
static __device__ uint32_t cs_find(const DTrieDev &t, uint32_t trie, const uint8_t *path, uint32_t len) {
    uint32_t cur = trie == DT_NONE ? DT_NONE : t.troot[trie], matched = 0;
    for (int hops = 0; cur != DT_NONE && !(cur & DT_LEAF); hops++) {
        if (hops > DT_MAX_HOPS) {
            atomicExch(t.err, B200_DEVERR_CORRUPT);
            return DT_NONE;
        }
        const uint32_t d = t.ndepth[cur];
        if (d > len || dt_lcp(path, t.nkey + 32 * (uint64_t)cur, matched, d) < d) return DT_NONE;
        if (d == len) return cs_stored(t, cur) ? cur : DT_NONE;
        matched = d + 1;
        cur = t.nchild[16 * (uint64_t)cur + dt_nib(path, d)];
    }
    return DT_NONE;
}

// Changed paths: node_of[j] = the stored node at path j, and the row of j.  Storage paths (offs non-null): path j belongs to
// key i (offs[i] <= j < offs[i+1]) whose trie is leaf_of[i] (DT_NONE: no account); a key with kflags bit 0 is deleted.
// n_rows null: row j at position j; otherwise rows are appended, and a path of a deleted trie that finds a node is left out.
__global__ void cs_lookup_kernel(DTrieDev t, const uint64_t *__restrict__ offs, uint64_t n_keys, const uint32_t *__restrict__ leaf_of,
                                 const uint8_t *__restrict__ kflags, const uint8_t *__restrict__ len, const uint8_t *__restrict__ paths,
                                 uint64_t n, uint32_t *__restrict__ node_of, uint64_t *__restrict__ rows, uint32_t *__restrict__ n_rows) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t i = offs ? wt_account_of(offs, n_keys, j) : 0u;
    const uint32_t v = cs_find(t, offs ? leaf_of[i] : 0u, paths + 32 * j, len[j]);
    node_of[j] = v;
    const uint64_t row = (uint64_t)i << 32 | j;
    if (!n_rows) rows[j] = row;
    else if (v == DT_NONE || !(kflags && (kflags[i] & 1))) rows[atomicAdd(n_rows, 1u)] = row;
}

// The stored nodes the wipe walk queued ((node, trie) pairs of ts): a row each, under the index of the trie's account key
// (ta's leaf `trie`) among the n_keys ascending keys32.
__global__ void cs_wiped_rows_kernel(DTrieDev ts, DTrieDev ta, const uint32_t *__restrict__ queue, uint32_t n_queue,
                                     const uint8_t *__restrict__ keys32, uint64_t n_keys, uint64_t *__restrict__ rows,
                                     uint32_t *__restrict__ n_rows) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_queue) return;
    const uint32_t v = queue[2 * (uint64_t)k], trie = queue[2 * (uint64_t)k + 1];
    if (!cs_stored(ts, v)) return;
    const uint8_t *key = ta.lkey + 32 * (uint64_t)trie;
    uint64_t lo = 0, hi = n_keys;  // the key equal to `key` (the trie was queued from it)
    while (hi - lo > 1) {
        const uint64_t mid = (lo + hi) >> 1;
        const uint8_t *b = keys32 + 32 * mid;
        const uint32_t l = dt_lcp(b, key, 0, 64);
        if (l == 64 || dt_nib(b, l) < dt_nib(key, l)) lo = mid;
        else hi = mid;
    }
    rows[atomicAdd(n_rows, 1u)] = lo << 32 | CS_NODE | v;
}

// The sort key of a row is 40 bytes: trie id (big-endian) | packed path | length | 0 0 0.  keys64[r] = its big-endian word w
// (0 = most significant), for the stable LSD passes that order the rows by (trie, path, length).
__global__ void cs_sort_word_kernel(DTrieDev t, const uint8_t *__restrict__ len, const uint8_t *__restrict__ paths,
                                    const uint64_t *__restrict__ rows, uint32_t n, int w, uint64_t *__restrict__ keys64) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint64_t row = rows[r];
    const uint32_t src = (uint32_t)row, tid = (uint32_t)(row >> 32);
    const bool node = (src & CS_NODE) != 0;
    const uint32_t id = src & ~CS_NODE;
    const uint8_t *key = node ? t.nkey + 32 * (uint64_t)id : paths + 32 * (uint64_t)id;
    const uint32_t d = node ? t.ndepth[id] : len[id];
    uint64_t word = 0;
    for (int q = 8 * w; q < 8 * w + 8; q++) {
        uint32_t b = 0;
        if (q < 4) b = (tid >> (8 * (3 - q))) & 0xFF;
        else if (q < 36) b = dt_path_byte(key, d, (uint32_t)(q - 4));
        else if (q == 36) b = d;
        word = word << 8 | b;
    }
    keys64[r] = word;
}

// the stored node of row r (DT_NONE: a None record)
static __device__ __forceinline__ uint32_t cs_node_of_row(uint64_t row, const uint32_t *node_of) {
    const uint32_t src = (uint32_t)row;
    return (src & CS_NODE) ? (src & ~CS_NODE) : node_of[src];
}
// hash counts of the records, in row order
__global__ void cs_hash_counts_kernel(DTrieDev t, const uint64_t *__restrict__ rows, uint32_t n, const uint32_t *__restrict__ node_of,
                                      uint32_t *__restrict__ n_hashes) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint32_t v = cs_node_of_row(rows[r], node_of);
    n_hashes[r] = v == DT_NONE ? 0u : (uint32_t)__popc(t.nmasks[v].z);
}
// record r: the stored node (dt_put_record), or None (the changed path with all three masks 0 and no hashes)
__global__ void cs_write_kernel(DTrieDev t, const uint64_t *__restrict__ rows, uint32_t n, const uint32_t *__restrict__ node_of,
                                const uint8_t *__restrict__ len, const uint8_t *__restrict__ paths, const uint32_t *__restrict__ hash_prefix,
                                UpdatesDev out) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint64_t row = rows[r];
    const uint32_t tid = (uint32_t)(row >> 32), v = cs_node_of_row(row, node_of);
    if (v != DT_NONE) {
        dt_put_record(t, v, tid, hash_prefix[r], out, r);
        return;
    }
    const uint32_t j = (uint32_t)row;
    out.trie_id[r] = tid;
    out.path_len[r] = len[j];
    dt_copy32(out.path_packed + 32 * (uint64_t)r, paths + 32 * (uint64_t)j);
    out.state_mask[r] = out.tree_mask[r] = out.hash_mask[r] = 0;
    out.hash_offset[r] = hash_prefix[r];
}

// ------------------------------------------------------------------------------------------------ launchers
cudaError_t launch_cs_lookup(const DTrieDev &t, const uint64_t *offs, uint64_t n_keys, const uint32_t *leaf_of, const uint8_t *kflags,
                             const uint8_t *len, const uint8_t *paths, uint64_t n, uint32_t *node_of, uint64_t *rows, uint32_t *n_rows,
                             cudaStream_t st) {
    if (n) cs_lookup_kernel<<<blocks_for(n, 128), 128, 0, st>>>(t, offs, n_keys, leaf_of, kflags, len, paths, n, node_of, rows, n_rows);
    return cudaGetLastError();
}
cudaError_t launch_cs_wiped_rows(const DTrieDev &ts, const DTrieDev &ta, const uint32_t *queue, uint32_t n_queue, const uint8_t *keys32,
                                 uint64_t n_keys, uint64_t *rows, uint32_t *n_rows, cudaStream_t st) {
    if (n_queue) cs_wiped_rows_kernel<<<blocks_for(n_queue, 128), 128, 0, st>>>(ts, ta, queue, n_queue, keys32, n_keys, rows, n_rows);
    return cudaGetLastError();
}
cudaError_t launch_cs_sort_word(const DTrieDev &t, const uint8_t *len, const uint8_t *paths, const uint64_t *rows, uint32_t n, int w,
                                uint64_t *keys64, cudaStream_t st) {
    if (n) cs_sort_word_kernel<<<blocks_for(n, 256), 256, 0, st>>>(t, len, paths, rows, n, w, keys64);
    return cudaGetLastError();
}
cudaError_t launch_cs_hash_counts(const DTrieDev &t, const uint64_t *rows, uint32_t n, const uint32_t *node_of, uint32_t *n_hashes,
                                  cudaStream_t st) {
    if (n) cs_hash_counts_kernel<<<blocks_for(n, 256), 256, 0, st>>>(t, rows, n, node_of, n_hashes);
    return cudaGetLastError();
}
cudaError_t launch_cs_write(const DTrieDev &t, const uint64_t *rows, uint32_t n, const uint32_t *node_of, const uint8_t *len,
                            const uint8_t *paths, const uint32_t *hash_prefix, const UpdatesDev &out, cudaStream_t st) {
    if (n) cs_write_kernel<<<blocks_for(n, 128), 128, 0, st>>>(t, rows, n, node_of, len, paths, hash_prefix, out);
    return cudaGetLastError();
}
