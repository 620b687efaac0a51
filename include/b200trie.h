/*
 * b200trie.h — C ABI of the GPU state-root engine (libb200trie.so, built for the H100, sm_90a).
 *
 * This is the drop-in boundary for reth's Merkle-Patricia-Trie commitment path.  reth has no FFI for this
 * path (it is all Rust traits/closures); each entry point below names the reference interface a thin Rust
 * shim would route to it (paths relative to the reth workspace; the shim itself is shown in INTEGRATION.md).
 *
 * Conventions
 *   - plain pointers and sizes only; all multi-byte integers little-endian host order unless a field says BE
 *   - every function returns B200_OK (0) or a negative b200_status; b200_last_error(ctx) gives the text
 *   - the library never aborts/throws across the boundary and never falls back to a CPU path: without a
 *     usable CUDA device b200_create fails with B200_ERR_NO_DEVICE
 *   - a b200_ctx is internally locked: calls on one ctx are serialised, different ctxs run concurrently
 *     (ParallelStateRoot calls StorageRoot from many threads: crates/trie/parallel/src/root.rs:111-125)
 *   - host-pointer entry points copy inputs to the device and results back (these are what the e2e
 *     benchmark times); *_dev entry points take device pointers (inputs and outputs) and leave their results in
 *     device memory without a final synchronisation (b200_sync to wait, or order later work on the ctx stream).
 *     They are not fire-and-forget: a trie build reads its level histogram back once (322 integers, on an internal
 *     stream while the leaf pass keeps running on the ctx stream), and a scratch buffer that has to grow
 *     synchronises before it is replaced
 *   - hashed keys are 32-byte big-endian strings exactly as reth's B256; sorted means ascending bytewise
 */
#ifndef B200TRIE_H
#define B200TRIE_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200_ctx b200_ctx;

typedef enum {
    B200_OK = 0,
    B200_ERR_NO_DEVICE = -1,   /* no CUDA device / driver */
    B200_ERR_CUDA = -2,        /* CUDA runtime error (text in b200_last_error) */
    B200_ERR_INVALID_ARG = -3, /* null pointer, bad length, offsets not monotone ... */
    B200_ERR_UNSORTED = -4,    /* keys not strictly ascending inside a trie (HashBuilder::add_leaf asserts this) */
    B200_ERR_ZERO_VALUE = -5,  /* a storage slot with value 0: reth treats zero as deletion
                                  (crates/trie/common/src/hashed_state.rs:423-455), it is never a leaf */
    B200_ERR_OOM = -6,
    B200_ERR_INLINE_HASH_CHILD = -7, /* a <32-byte branch child under a hash_mask bit while retaining updates:
                                        alloy-trie's child_hashes would panic here; unreachable for keccak keys */
    B200_ERR_NOT_FOUND = -8, /* b200_trie_update: a dirty key is not in the resident trie */
    B200_ERR_WITNESS_INCOMPLETE = -9 /* b200_witness_roots (per block): a node the post-block root needs is not in the witness */
} b200_status;

/* ------------------------------------------------------------------------------------------------ lifecycle */
/* Number of usable CUDA devices (0 when there is no driver). */
B200_API int32_t b200_device_count(void);
/* One context per device ordinal (one process per GPU in the multi-GPU layout). NULL on failure;
 * b200_create_status() then tells why. */
B200_API b200_ctx *b200_create(int32_t device_ordinal);
B200_API int32_t b200_create_status(void);
B200_API void b200_destroy(b200_ctx *);
B200_API const char *b200_last_error(const b200_ctx *);
B200_API const char *b200_version(void);
/* Use an existing CUDA stream (cudaStream_t passed as void*) instead of the context's own stream, so that a
 * host runtime (torch, the Rust shim's stream) can order and time the work.  NULL is the CUDA legacy default
 * stream (what a cudaStream_t of 0 means everywhere); (void*)-1 restores the context's own stream. */
B200_API int32_t b200_set_stream(b200_ctx *, void *cuda_stream);
B200_API int32_t b200_sync(b200_ctx *);
/* Page-locked host buffers for the host-pointer entry points (pageable memory works too, but is slower). */
/* Binds the CALLING thread to the host NUMA node the GPU hangs off (its CPUs and, as preferred memory policy, its DRAM),
 * so that page-locked staging buffers allocated afterwards (b200_host_alloc, or the caller's own) and the copies out of them
 * stay on the GPU's socket — the placement a one-process-per-GPU host wants before it allocates (reth's stage pipeline
 * drains cursors into such buffers, hashing_account.rs:176-238).  Returns the node (>= 0), -1 when the platform exposes no
 * NUMA topology for the device (nothing is changed then).  Never fails hard; needs no context. */
B200_API int32_t b200_numa_bind_thread(int32_t device_ordinal);
B200_API void *b200_host_alloc(size_t bytes);
B200_API void b200_host_free(void *);
/* Scratch the context currently holds on the device, bytes. */
B200_API uint64_t b200_device_bytes(const b200_ctx *);
/* Kernel launches issued through this context so far (what bench.py reports as gpu_launches). */
B200_API uint64_t b200_launch_count(const b200_ctx *);

/* ------------------------------------------------------------------------------------------------ key hashing
 * Replaces the per-key `keccak256` of KeccakKeyHasher::hash_key (crates/trie/common/src/key.rs:4-18) as
 * batched by AccountHashingStage (crates/stages/stages/src/stages/hashing_account.rs:192-211, 20-byte
 * addresses), StorageHashingStage (hashing_storage.rs:121-148, 20-byte address + 32-byte slot),
 * HashedPostState::from_bundle_state (crates/trie/common/src/hashed_state.rs:49-69) and
 * load_prefix_sets_with_provider (crates/trie/db/src/prefix_set.rs:42-60).
 *
 * in: n messages of msg_len bytes, message i at in + i*stride (stride >= msg_len). out32: n*32 bytes. */
B200_API int32_t b200_keccak256_fixed(b200_ctx *, const uint8_t *in, uint32_t msg_len, uint32_t stride, uint64_t n,
                             uint8_t *out32);
B200_API int32_t b200_keccak256_fixed_dev(b200_ctx *, const void *d_in, uint32_t msg_len, uint32_t stride, uint64_t n,
                                 void *d_out32);
/* Variable-length messages (contract code -> code hash, arbitrary RLP): message i is
 * data[offsets[i] .. offsets[i+1]). */
B200_API int32_t b200_keccak256_var(b200_ctx *, const uint8_t *data, const uint64_t *offsets, uint64_t n, uint8_t *out32);
B200_API int32_t b200_keccak256_var_dev(b200_ctx *, const void *d_data, const void *d_offsets, uint64_t n, void *d_out32);

/* Hash then sort: what the hashing stages feed to the ETL collector (crates/etl/src/lib.rs:31-60,
 * hashing_account.rs:207-230).  out_sorted32 receives the digests in ascending order, out_perm[i] is the
 * input index whose digest landed at position i (the shim permutes the values with it). */
B200_API int32_t b200_hash_sort_keys(b200_ctx *, const uint8_t *in, uint32_t msg_len, uint32_t stride, uint64_t n,
                            uint8_t *out_sorted32, uint32_t *out_perm);
B200_API int32_t b200_hash_sort_keys_dev(b200_ctx *, const void *d_in, uint32_t msg_len, uint32_t stride, uint64_t n,
                                void *d_sorted32, void *d_perm_u32);
/* StorageHashingStage full pass (hashing_storage.rs:106-178): entry i is (addresses20[addr_index[i]], slots32[i]).
 * Every address is hashed once, every slot key once, and the entries are sorted by the 64-byte composite key
 * keccak(address) || keccak(slot): out_sorted64[i] is the i-th smallest composite key, out_perm[i] the entry it
 * came from.  A duplicate (address, slot) pair yields B200_ERR_UNSORTED. */
B200_API int32_t b200_hash_sort_storage(b200_ctx *, const uint8_t *addresses20, uint32_t n_addr, const uint32_t *addr_index,
                                        const uint8_t *slots32, uint64_t n, uint8_t *out_sorted64, uint32_t *out_perm);
/* The same with every array in device memory (d_sorted64: n x 64 bytes, d_perm_u32: n x u32); synchronises once for the
 * verification of the order, like b200_hash_sort_keys_dev. */
B200_API int32_t b200_hash_sort_storage_dev(b200_ctx *, const void *d_addresses20, uint32_t n_addr, const void *d_addr_index_u32,
                                            const void *d_slots32, uint64_t n, void *d_sorted64, void *d_perm_u32);
/* The sort half alone: n 32-byte keys (already digests) -> ascending order + permutation. */
B200_API int32_t b200_sort_keys32_dev(b200_ctx *, const void *d_keys32, uint64_t n, void *d_sorted32, void *d_perm_u32);

/* ------------------------------------------------------------------------------------------------ trie inputs
 * reth's Account (reth-primitives-traits: nonce u64, balance U256, bytecode_hash Option<B256>) flattened;
 * the shim writes KECCAK_EMPTY when bytecode_hash is None (crates/trie/common/src/account.rs:16-31). */
typedef struct {
    uint64_t nonce;
    uint8_t balance_be[32];
    uint8_t code_hash[32];
} b200_account; /* 72 bytes */

/* TrieUpdates / StorageTrieUpdates after finalize (crates/trie/common/src/updates.rs:17-26,140-158,235-245):
 * one record per stored BranchNodeCompact, empty path excluded.  Record order is deterministic (by path
 * length, then key order) but carries no meaning: reth keeps these in hash maps.  All arrays are owned by the library (pinned host memory); release with b200_updates_release. */
typedef struct {
    uint64_t n_nodes;
    uint32_t *trie_id;     /* storage tries: index of the account (segment); account trie: 0 */
    uint8_t *path_len;     /* nibbles, 1..63 */
    uint8_t *path_packed;  /* [n_nodes][32] nibbles packed high-first, zero padded */
    uint16_t *state_mask, *tree_mask, *hash_mask;
    uint64_t *hash_offset; /* [n_nodes+1] into hashes */
    uint8_t *hashes;       /* [hash_offset[n_nodes]][32] child hashes, ascending nibble */
    void *_owner;
} b200_updates;
B200_API void b200_updates_release(b200_updates *);

/* ------------------------------------------------------------------------------------------------ table rows
 * Byte-exact rows of reth's trie tables from a b200_updates, in MDBX key order, ready for a cursor append /
 * upsert loop (write_trie_updates_sorted, crates/storage/provider/src/providers/database/provider.rs:3125-3160;
 * DatabaseStorageTrieCursor::write_storage_trie_updates_sorted, crates/trie/db/src/trie_cursor.rs:280-312).
 * Host-only (no device work).  Row r occupies bytes[row_offset[r] .. row_offset[r+1]): the first key_len[r]
 * bytes are the table key, the rest is the value.
 *   AccountsTrie (crates/storage/db-api/src/tables/mod.rs:484-487): key = StoredNibbles (LEGACY: one nibble per
 *     byte, crates/trie/common/src/nibbles.rs:27-66) or PackedStoredNibbles (PACKED: 32 packed bytes + nibble
 *     count, nibbles.rs:143-213); value = BranchNodeCompact Compact (three big-endian u16 masks, then hashes).
 *   StoragesTrie (tables/mod.rs:490-494, dup-sorted): key = hashed address = acct_keys32[trie_id]; value =
 *     StorageTrieEntry = StoredNibblesSubKey (65 B) or PackedStoredNibblesSubKey (33 B) followed by the node
 *     (crates/trie/common/src/storage.rs:24-44,70-86).
 * Deleted storage tries (StorageTrieUpdates::deleted) have no rows; the caller clears those duplicates. */
typedef enum {
    B200_KEYS_LEGACY = 0, /* StoredNibbles / StoredNibblesSubKey */
    B200_KEYS_PACKED = 1  /* storage v2: PackedStoredNibbles / PackedStoredNibblesSubKey */
} b200_key_format;

typedef struct {
    uint64_t n_rows;
    uint64_t *row_offset; /* [n_rows+1] into bytes */
    uint32_t *key_len;    /* [n_rows] */
    uint8_t *bytes;
    void *_owner;
} b200_rows;

B200_API int32_t b200_account_trie_rows(const b200_updates *account_updates, int32_t key_format, b200_rows *out);
B200_API int32_t b200_storage_trie_rows(const b200_updates *storage_updates, const uint8_t *acct_keys32,
                                        uint64_t n_accounts, int32_t key_format, b200_rows *out);
B200_API void b200_rows_release(b200_rows *);
/* (b200_state_root_full_rows, below, delivers the same rows straight from a build: encoded on the device.) */

/* TrieStats / TrieRootMetrics (crates/trie/trie/src/stats.rs, metrics.rs:22-40) plus device timing. */
typedef struct {
    uint64_t leaves_added;
    uint64_t branches_added;   /* branch nodes built (reth counts add_branch calls; a from-scratch build has none) */
    uint64_t extension_nodes;
    uint64_t hashed_nodes;     /* keccak digests produced (node RLP >= 32 bytes, plus roots) */
    uint64_t levels;           /* populated trie levels processed */
    double device_ms;          /* stream time of the build, measured with CUDA events */
    uint64_t keccak_f;         /* Keccak-f[1600] permutations of a from-scratch build: hashed_nodes + the second .. fourth rate
                                  block of every branch node by its child-count class (4-7 children: 2 blocks, 8-12: 3, 13-16: 4;
                                  exact when no child of such a node is inlined, i.e. for hashed keys).  0 where it is not
                                  counted (ordered roots, resident / dynamic updates). */
} b200_stats;

/* ------------------------------------------------------------------------------------------------ roots
 * StorageRoot::calculate for n_accounts tries in one call (crates/trie/trie/src/trie.rs:615-721; the
 * fan-out of ParallelStateRoot, crates/trie/parallel/src/root.rs:101-127).  Segment a holds slots
 * seg_offsets[a] .. seg_offsets[a+1]: slot_keys32 = keccak(slot) sorted ascending inside the segment,
 * values32_be = U256 big-endian, non-zero.  Empty segment -> EMPTY_ROOT_HASH (trie.rs:622-629).
 * roots32: n_accounts*32. opt_updates may be NULL (root(): no updates retained). */
B200_API int32_t b200_storage_roots(b200_ctx *, const uint8_t *slot_keys32, const uint8_t *values32_be,
                           const uint64_t *seg_offsets, uint64_t n_accounts, uint8_t *roots32,
                           b200_updates *opt_updates, b200_stats *opt_stats);

/* The account-trie fold of StateRoot::calculate (trie.rs:247-309): leaf i = rlp(TrieAccount{nonce, balance,
 * storage_roots32[i], code_hash}) under key acct_keys32[i] (trie.rs:429-432).  storage_roots32 may be NULL
 * (all EMPTY_ROOT_HASH).  n == 0 -> EMPTY_ROOT_HASH. */
B200_API int32_t b200_state_root(b200_ctx *, const uint8_t *acct_keys32, const b200_account *accts,
                        const uint8_t *storage_roots32, uint64_t n, uint8_t root32[32],
                        b200_updates *opt_updates, b200_stats *opt_stats);

/* StateRoot::root_with_updates / ParallelStateRoot::incremental_root_with_updates over a complete
 * HashedPostStateSorted-shaped input (crates/trie/common/src/hashed_state.rs:519-524,710-715): all storage
 * tries, then all account leaves, then the account trie, without leaving the device.
 * seg_offsets has n_accounts+1 entries (segment a = storage of account a). */
B200_API int32_t b200_state_root_full(b200_ctx *, const uint8_t *acct_keys32, const b200_account *accts,
                             uint64_t n_accounts, const uint8_t *slot_keys32, const uint8_t *values32_be,
                             const uint64_t *seg_offsets, uint8_t root32[32],
                             b200_updates *opt_account_updates, b200_updates *opt_storage_updates,
                             b200_stats *opt_stats);

/* b200_state_root_full whose stored nodes arrive as finished table rows — MerkleStage's rebuild leg writing
 * AccountsTrie / StoragesTrie (crates/stages/stages/src/stages/merkle.rs:216-253 → write_trie_updates,
 * crates/storage/provider/src/providers/database/provider.rs:2545-2627): rows are sized, ordered and laid out on the
 * device and cross in one copy; byte-identical to b200_account_trie_rows / b200_storage_trie_rows over the records.
 * Release both with b200_rows_release. */
B200_API int32_t b200_state_root_full_rows(b200_ctx *, const uint8_t *acct_keys32, const b200_account *accts,
                                           uint64_t n_accounts, const uint8_t *slot_keys32, const uint8_t *values32_be,
                                           const uint64_t *seg_offsets, int32_t key_format, uint8_t root32[32],
                                           b200_rows *account_rows, b200_rows *storage_rows, b200_stats *opt_stats);

/* Device-resident variants: every pointer is a device pointer (seg_offsets included), results are written
 * to device memory and no host buffer is touched (one internal read-back of the level histogram per build, see the
 * conventions above).  d_root32 / d_roots32 are device buffers.
 * Input violations (unsorted keys, zero values) are reported by the next b200_sync / b200_dev_status. */
B200_API int32_t b200_storage_roots_dev(b200_ctx *, const void *d_slot_keys32, const void *d_values32_be,
                               const void *d_seg_offsets, uint64_t n_accounts, uint64_t n_slots,
                               void *d_roots32);
B200_API int32_t b200_state_root_dev(b200_ctx *, const void *d_acct_keys32, const void *d_accts,
                            const void *d_storage_roots32, uint64_t n, void *d_root32);
B200_API int32_t b200_state_root_full_dev(b200_ctx *, const void *d_acct_keys32, const void *d_accts, uint64_t n_accounts,
                                 const void *d_slot_keys32, const void *d_values32_be, const void *d_seg_offsets,
                                 uint64_t n_slots, void *d_root32);
/* Sticky status of the asynchronous entry points (B200_OK / B200_ERR_UNSORTED / ...); synchronises. */
B200_API int32_t b200_dev_status(b200_ctx *);
/* Stats of the last build on this ctx (synchronises). */
B200_API int32_t b200_last_stats(b200_ctx *, b200_stats *out);

/* ------------------------------------------------------------------------------------------------ multi-GPU
 * Key-range sharding of the account trie (SURVEY.md §8e): a rank owns whole top-nibble buckets of the hashed
 * address space together with the storage tries of its accounts.  It builds its buckets with
 * b200_subtrie_frontier, the 16 frontier entries of all ranks are all-gathered (NCCL, 16 x 2 x 34 bytes), and
 * every rank finishes the root with b200_root_from_frontier.
 *
 * Each bucket yields two RlpNode candidates (len byte + up to 33 bytes):
 *   as_child: the node as child `nibble` of a depth-0 root branch (used when >= 2 buckets are non-empty)
 *   as_root : the bucket alone as the whole trie (used when it is the only non-empty bucket)
 * len == 0 means the bucket is empty. */
typedef struct {
    uint8_t as_child_len;
    uint8_t as_child[33];
    uint8_t as_root_len; /* 0 or 32: root hash */
    uint8_t as_root[33];
} b200_frontier_entry; /* 68 bytes */

/* acct_keys32/accts/storage as in b200_state_root_full but holding only this rank's accounts (any subset of
 * top nibbles). frontier: 16 entries, entries of nibbles this rank does not own are zeroed. */
B200_API int32_t b200_subtrie_frontier(b200_ctx *, const uint8_t *acct_keys32, const b200_account *accts,
                              uint64_t n_accounts, const uint8_t *slot_keys32, const uint8_t *values32_be,
                              const uint64_t *seg_offsets, b200_frontier_entry frontier[16],
                              b200_stats *opt_stats);
B200_API int32_t b200_subtrie_frontier_dev(b200_ctx *, const void *d_acct_keys32, const void *d_accts, uint64_t n_accounts,
                                  const void *d_slot_keys32, const void *d_values32_be, const void *d_seg_offsets,
                                  uint64_t n_slots, void *d_frontier /* 16 x b200_frontier_entry */);
/* Combine the gathered frontier (entry i = bucket of top nibble i, from whichever rank owns it). Host-side,
 * 17 node hashes at most; runs on the device like everything else. */
B200_API int32_t b200_root_from_frontier(b200_ctx *, const b200_frontier_entry frontier[16], uint8_t root32[32]);
B200_API int32_t b200_root_from_frontier_dev(b200_ctx *, const void *d_frontier, void *d_root32);

/* ------------------------------------------------------------------------------------------------ incremental root, trie not resident
 * The fold of an incremental HashBuilder run over the element stream reth's TrieWalker + TrieNodeIter produce from the
 * stored trie nodes and the prefix sets (crates/trie/trie/src/walker.rs:161-388, node_iter.rs:200-304; PrefixSet::contains,
 * crates/trie/common/src/prefix_set.rs:205-231; StateRoot::calculate, trie.rs:247-309; StorageRoot::calculate, :659-698):
 * item i is either a leaf (key_nibbles[i] == 64: HashBuilder::add_leaf) or the stored hash of an unchanged subtree
 * (key_nibbles[i] = length of its path in nibbles, 0..63: HashBuilder::add_branch(path, hash, children_are_in_trie)).
 *   keys32      : leaf key, or the path left-aligned (two nibbles per byte) and zero-padded; strictly ascending inside a
 *                 trie and prefix-free (the walker never yields anything below a hash it yields)
 *   item_flags  : bit 0 = children_are_in_trie of a hash item (sets the parent's tree-mask bit)
 *   values      : rows of 72 bytes (account != 0: b200_account; storage_roots32 gives their storage roots, NULL = empty)
 *                 or 32 bytes (U256 big-endian slot values, non-zero); a hash item's row starts with its 32-byte hash
 *   seg_offsets : a forest of storage tries in one call (n_segs + 1 entries), or NULL for one trie (n_segs ignored)
 * roots32: one root per trie (an empty segment gives EMPTY_ROOT_HASH; a lone hash at the empty path is returned as is).
 * opt_updates: the branch nodes built by THIS fold that the tables must store (TrieUpdates::account_nodes /
 * storage_nodes; trie_id = segment) — the removed_nodes of the walk are the walker's (every stored node it descended into
 * and that is not among the updated ones, walker.rs:336-344). */
B200_API int32_t b200_root_from_items(b200_ctx *, const uint8_t *keys32, const uint8_t *key_nibbles, const uint8_t *item_flags,
                                      const uint8_t *values, const uint8_t *storage_roots32, const uint64_t *seg_offsets,
                                      uint64_t n_segs, uint64_t n_items, int32_t account, uint8_t *roots32,
                                      b200_updates *opt_updates, b200_stats *opt_stats);

/* ------------------------------------------------------------------------------------------------ changesets -> dirty set
 * Incremental hashing of a block range in one call: what HashedPostStateSorted::from_reverts (crates/trie/db/src/state.rs:
 * 289-347), load_prefix_sets_with_provider (crates/trie/db/src/prefix_set.rs:22-60) and insert_account_for_hashing /
 * insert_storage_for_hashing (crates/storage/provider/src/providers/database/provider.rs:3206-3280) do with HashSets and
 * sort_unstable: keccak every changed address and slot, keep the FIRST (oldest) changeset entry of every address and of every
 * (address, slot) pair, sort.  Input: the account changeset addresses and the storage changeset (address, slot) rows of the
 * range, in changeset order (block, address).  Output (page-locked, released with b200_changeset_hashes_release):
 *   accounts  : unique keccak(address) ascending + index of the first entry of each (the caller picks AccountBeforeTx there)
 *   storages  : unique (keccak(address), keccak(slot)) pairs as a CSR — addresses ascending, slot keys ascending inside a
 *               segment, index of the first entry of each pair — i.e. HashedStorageSorted per address, and at the same
 *               time the storage prefix sets (sorted, deduplicated changed keys; prefix_set.rs:165-177)
 *   prefix set: the account prefix set — union of both address key sets, ascending, deduplicated.
 * destroyed_accounts needs the HashedAccounts table (prefix_set.rs:40-42) and stays with the caller. */
typedef struct {
    uint64_t n_accounts;
    uint8_t *account_keys32;
    uint32_t *account_first;
    uint64_t n_storage_accounts;
    uint8_t *storage_account_keys32;
    uint64_t *storage_seg_offsets; /* [n_storage_accounts + 1] */
    uint64_t n_slots;
    uint8_t *slot_keys32;
    uint32_t *slot_first;
    uint64_t n_prefix;
    uint8_t *account_prefix_keys32;
    void *_owner;
} b200_changeset_hashes;
B200_API int32_t b200_hash_changesets(b200_ctx *, const uint8_t *acct_addresses20, uint64_t n_acct_entries,
                                      const uint8_t *storage_addresses20, const uint8_t *storage_slots32,
                                      uint64_t n_storage_entries, b200_changeset_hashes *out);
B200_API void b200_changeset_hashes_release(b200_changeset_hashes *);

/* ------------------------------------------------------------------------------------------------ streamed / resumable root
 * StateRoot::with_threshold / root_with_progress / with_intermediate_state (crates/trie/trie/src/trie.rs:73-85,156-330;
 * progress.rs) and MerkleStage's chunked rebuild with its MerkleCheckpoint (crates/stages/stages/src/stages/merkle.rs:
 * 118-148,184-366): the state is committed in ascending account-key ranges, e.g. when it does not fit HBM or host memory
 * at once.  Each push carries a range of accounts (strictly after every key pushed before) with their complete storage, in
 * the layout of b200_state_root_full.  A push builds the storage tries of its accounts and every top-nibble bucket of the
 * account trie that the range closes; closed buckets survive as 68-byte frontier entries (the entries of the multi-GPU
 * path), the accounts of the still open bucket (at most 1/16 of the state, 136 bytes each) stay on the device.  Stored
 * nodes leave with the push that closes them (account nodes: trie_id = top nibble; storage nodes: trie_id = index of the
 * account inside that push), like the per-chunk TrieUpdates of StateRootProgress::Progress.  finish closes the last bucket
 * and folds the frontier.  k pushes give exactly the root and the union of updates of one b200_state_root_full call. */
typedef struct b200_root_stream b200_root_stream;
typedef struct {
    uint64_t accounts;         /* pushed so far */
    uint64_t slots;
    uint64_t open_accounts;    /* carried in HBM: the accounts of the open bucket */
    uint32_t closed_buckets;   /* bit i: top nibble i is finished */
} b200_stream_progress;
/* What survives a restart (the role of MerkleCheckpoint): frontier of the closed buckets + where to resume.  After
 * b200_root_stream_resume the caller pushes again from the first key whose top nibble is resume_nibble (16: nothing left). */
typedef struct {
    b200_frontier_entry frontier[16];
    uint32_t closed_mask;
    uint32_t resume_nibble;
    uint32_t retain_updates;
    uint32_t _reserved;
} b200_stream_checkpoint;
B200_API int32_t b200_root_stream_begin(b200_ctx *, int32_t retain_updates, b200_root_stream **out);
B200_API int32_t b200_root_stream_push(b200_root_stream *, const uint8_t *acct_keys32, const b200_account *accts,
                                       uint64_t n_accounts, const uint8_t *slot_keys32, const uint8_t *values32_be,
                                       const uint64_t *seg_offsets, b200_updates *opt_account_updates,
                                       b200_updates *opt_storage_updates, b200_stream_progress *opt_progress);
B200_API int32_t b200_root_stream_finish(b200_root_stream *, uint8_t root32[32], b200_updates *opt_account_updates);
B200_API int32_t b200_root_stream_checkpoint(const b200_root_stream *, b200_stream_checkpoint *out);
B200_API int32_t b200_root_stream_resume(b200_ctx *, const b200_stream_checkpoint *, b200_root_stream **out);
B200_API void b200_root_stream_free(b200_root_stream *);

/* Communicator: the two exchange steps of the path behind the C ABI (SURVEY.md §8b `b200_create(device, n_devices)`, §8e).
 * One process (or thread) per GPU, each with its own b200_ctx; rank 0 makes the id (b200_comm_unique_id = ncclGetUniqueId),
 * the host ships its 128 bytes to the other ranks over whatever channel it has, every rank calls b200_comm_create
 * (ncclCommInitRank: collective, blocks until all ranks joined).  NCCL is loaded at run time (libnccl.so.2; B200_NCCL_LIB
 * overrides), so a host that never creates a communicator needs no NCCL.  At most 16 ranks (one top-nibble bucket each). */
#define B200_COMM_ID_BYTES 128
typedef struct b200_comm b200_comm;
B200_API int32_t b200_comm_unique_id(uint8_t id[B200_COMM_ID_BYTES]);
B200_API int32_t b200_comm_create(b200_ctx *, const uint8_t id[B200_COMM_ID_BYTES], int32_t n_ranks, int32_t rank, b200_comm **out);
B200_API void b200_comm_destroy(b200_comm *);
B200_API int32_t b200_comm_rank(const b200_comm *);
B200_API int32_t b200_comm_size(const b200_comm *);
/* b200_subtrie_frontier -> ncclAllGather of the 16 x 68-byte frontier -> b200_root_from_frontier in ONE call on the ctx
 * stream: every rank passes its own shard (whole top-nibble buckets, any subset) and receives the state root.  The _dev form
 * takes device pointers and leaves the root in device memory without a final synchronisation (d_root32: device). */
B200_API int32_t b200_state_root_sharded(b200_comm *, const uint8_t *acct_keys32, const b200_account *accts, uint64_t n_accounts,
                                         const uint8_t *slot_keys32, const uint8_t *values32_be, const uint64_t *seg_offsets,
                                         uint8_t root32[32], b200_stats *opt_stats);
B200_API int32_t b200_state_root_sharded_dev(b200_comm *, const void *d_acct_keys32, const void *d_accts, uint64_t n_accounts,
                                             const void *d_slot_keys32, const void *d_values32_be, const void *d_seg_offsets,
                                             uint64_t n_slots, void *d_root32);
/* The live path at N > 1: every rank has applied its part of the block to its shard (b200_dstate_create_sharded +
 * b200_dstate_apply); this gathers the resident 16-entry frontiers of all ranks (one ncclAllGather) and returns the state root
 * on every rank.  (b200_dstate is declared further down.) */
struct b200_dstate;
B200_API int32_t b200_dstate_root_sharded(b200_comm *, struct b200_dstate *, uint8_t root32[32]);
/* AccountHashingStage / StorageHashingStage at N > 1 (hashing_account.rs:176-238, hashing_storage.rs:106-178; SURVEY.md §8e
 * last sentence): every rank holds an arbitrary slice of the plain table — n messages (msg_len 20 | 32) with one
 * value_bytes-wide row each (the account, the slot value; may be 0).  One call hashes them, sends every (digest, row) to the
 * rank that owns the digest's top nibble (rank = nibble * n_ranks / 16; one grouped all-to-all over NVLink) and sorts what
 * arrives by digest: the rank's shard of HashedAccounts in table order, ready for b200_state_root_sharded.  Device pointers;
 * the outputs hold `capacity` rows, *n_out receives the rows this rank owns (error if it exceeds capacity). Synchronises. */
B200_API int32_t b200_hash_partition_dev(b200_comm *, const void *d_in, uint32_t msg_len, uint32_t stride, uint64_t n,
                                         const void *d_values, uint32_t value_bytes, uint64_t capacity, void *d_sorted_keys32,
                                         void *d_sorted_values, uint64_t *n_out);

/* ------------------------------------------------------------------------------------------------ ordered roots
 * Transactions / receipts / withdrawals roots of a batch of lists in one call (SURVEY.md §8f-4): what
 * OrderedTrieRootEncodedBuilder::finalize (crates/trie/common/src/ordered_root.rs:240-257) and alloy's
 * ordered_trie_root_with_encoder behind proofs::calculate_{transaction,receipt,withdrawals}_root
 * (crates/ethereum/evm/src/build.rs:56-68, crates/ethereum/consensus/src/validation.rs:108,
 * crates/consensus/common/src/validation.rs:59) return, for pre-encoded items.
 * List l holds items seg_offsets[l] .. seg_offsets[l+1] in list (execution) order; item i is the byte string
 * values[value_offsets[i] .. value_offsets[i+1]) — the EIP-2718 encoding the reference's encoder closure writes.
 * Keys (rlp(index)) and their insertion order are derived on the device.  Empty list -> EMPTY_ROOT_HASH.
 * roots32: n_lists*32.  At most 2^31-1 items per call, each below 2 GiB. */
B200_API int32_t b200_ordered_roots(b200_ctx *, const uint8_t *values, const uint64_t *value_offsets,
                                    const uint64_t *seg_offsets, uint64_t n_lists, uint8_t *roots32,
                                    b200_stats *opt_stats);
/* Device-resident variant (all pointers device pointers; d_values 8-byte aligned for the fast path, any alignment
 * accepted; values_len = bytes readable at d_values).  Violations are reported by the next b200_sync. */
B200_API int32_t b200_ordered_roots_dev(b200_ctx *, const void *d_values, uint64_t values_len,
                                        const void *d_value_offsets, const void *d_seg_offsets, uint64_t n_lists,
                                        uint64_t n_items, void *d_roots32);

/* ------------------------------------------------------------------------------------------------ resident trie
 * Incremental state root (BASELINE config 5; reth: StateRoot::with_prefix_sets over stored branch nodes,
 * crates/trie/trie/src/walker.rs:172-202, node_iter.rs:205-300, DatabaseStateRoot::incremental_root_with_updates
 * crates/trie/db/src/state.rs:184-193).  The whole account trie — keys, accounts, storage roots and the node-hash
 * frontier of every level — stays in HBM; an update re-hashes only the root paths of the dirty accounts.
 *
 * Scope: value changes of EXISTING accounts (nonce / balance / code hash / storage root).  A key that is not in the
 * trie yields B200_ERR_NOT_FOUND and leaves the trie untouched (inserts and deletes change the trie shape: rebuild).
 * Dirty keys of one call must be distinct.  Storage roots of dirty accounts are computed by the caller with
 * b200_storage_roots over their complete post-state storage. */
typedef struct b200_trie b200_trie;
B200_API int32_t b200_trie_create(b200_ctx *, const uint8_t *acct_keys32, const b200_account *accts,
                                  const uint8_t *storage_roots32 /* nullable: all EMPTY_ROOT_HASH, not updatable */,
                                  uint64_t n, b200_trie **out, uint8_t root32[32]);
B200_API int32_t b200_trie_create_dev(b200_ctx *, const void *d_acct_keys32, const void *d_accts,
                                      const void *d_storage_roots32, uint64_t n, b200_trie **out, void *d_root32);
/* opt_updates: the stored BranchNodeCompact records on the dirty paths (what HashBuilder re-emits when reth
 * re-walks them), same format as above. */
B200_API int32_t b200_trie_update(b200_trie *, const uint8_t *dirty_keys32, const b200_account *new_accts,
                                  const uint8_t *new_storage_roots32 /* nullable: unchanged */, uint64_t m,
                                  uint8_t root32[32], b200_updates *opt_updates, b200_stats *opt_stats);
B200_API int32_t b200_trie_update_dev(b200_trie *, const void *d_dirty_keys32, const void *d_new_accts,
                                      const void *d_new_storage_roots32, uint64_t m, void *d_root32);
/* General commit of a dirty set with HashedPostStateSorted semantics (crates/trie/common/src/hashed_state.rs:519-524):
 * keys32 strictly ascending; present[i] != 0 (or present == NULL) = upsert accts[i], present[i] == 0 = delete (a delete
 * of an absent key is a no-op).  Value changes of existing accounts take the in-place path of b200_trie_update; any
 * insert or delete merges the keys on the device and rebuilds the trie there (*out_rebuilt = 1; opt_updates then holds
 * the complete node set of the new trie, to be written after clearing AccountsTrie as MerkleStage's rebuild path does,
 * crates/stages/stages/src/stages/merkle.rs:237-238). */
B200_API int32_t b200_trie_apply(b200_trie *, const uint8_t *keys32, const b200_account *accts, const uint8_t *present,
                                 const uint8_t *storage_roots32, uint64_t m, uint8_t root32[32], int32_t *out_rebuilt,
                                 b200_updates *opt_updates, b200_stats *opt_stats);
B200_API int32_t b200_trie_root(b200_trie *, uint8_t root32[32]);
B200_API uint64_t b200_trie_device_bytes(const b200_trie *);
B200_API uint64_t b200_trie_leaves(const b200_trie *);
B200_API void b200_trie_destroy(b200_trie *);

/* ------------------------------------------------------------------------------------------------ dynamic resident trie
 * The account trie as an arena of 16-slot branch nodes in HBM that takes a block's upserts AND deletes in place: only
 * the paths of the changed keys are restructured and re-hashed, whatever the size of the trie.  This is the role of
 * reth's sparse trie on the live path (ParallelSparseTrie::update_leaf / remove_leaf / root,
 * crates/trie/sparse/src/parallel.rs) and of TrieWalker + prefix sets on the database path
 * (crates/trie/trie/src/walker.rs:161-202, crates/trie/common/src/prefix_set.rs).
 * STATUS: validated bit-exact against the oracle on the GPU (tests/test_gpu_dtrie.py) and under tools/emu.
 *
 * b200_dtrie_apply: keys32 strictly ascending; present[i] == 0 deletes key i (NULL: all upserts); deleting an absent
 * key is a no-op.  storage_roots32 may be NULL (new accounts get EMPTY_ROOT_HASH, existing ones keep theirs).
 * opt_updated = the block's TrieUpdates::account_nodes (re-hashed nodes with tree_mask|hash_mask != 0);
 * opt_removed = TrieUpdates::removed_nodes as records whose masks are 0 (paths of stored nodes that ceased to exist or to
 * be stored; updated paths take precedence, crates/trie/common/src/updates.rs:160-167).  Release both with
 * b200_updates_release. */
typedef struct b200_dtrie b200_dtrie;
B200_API int32_t b200_dtrie_create(b200_ctx *, const uint8_t *acct_keys32 /* sorted */, const b200_account *accts,
                                   const uint8_t *storage_roots32 /* nullable */, uint64_t n, b200_dtrie **out,
                                   uint8_t root32[32] /* nullable */);
B200_API int32_t b200_dtrie_create_dev(b200_ctx *, const void *d_acct_keys32, const void *d_accts,
                                       const void *d_storage_roots32, uint64_t n, b200_dtrie **out, void *d_root32);
B200_API int32_t b200_dtrie_apply(b200_dtrie *, const uint8_t *keys32, const b200_account *accts, const uint8_t *present,
                                  const uint8_t *storage_roots32, uint64_t m, uint8_t root32[32],
                                  b200_updates *opt_updated, b200_updates *opt_removed, b200_stats *opt_stats);
B200_API int32_t b200_dtrie_root(b200_dtrie *, uint8_t root32[32]);
B200_API uint64_t b200_dtrie_leaves(const b200_dtrie *);
B200_API uint64_t b200_dtrie_nodes(const b200_dtrie *);   /* node slots allocated so far */
B200_API uint64_t b200_dtrie_device_bytes(const b200_dtrie *);
B200_API void b200_dtrie_destroy(b200_dtrie *);

/* ------------------------------------------------------------------------------------------------ dynamic resident state
 * b200_dtrie plus every storage trie: the whole hashed state (HashedAccounts + HashedStorages) lives in HBM as two arenas
 * and a block's HashedPostStateSorted (crates/trie/common/src/hashed_state.rs:519-524,710-715) is applied in place —
 * account upserts / destructions, per-account slot upserts / deletions (zero value) / wipes.  Storage roots flow into the
 * account leaves on the device; only the touched paths of the touched tries are re-hashed.  This is the complete role
 * of reth's SparseStateTrie on the live path (crates/trie/sparse/src/state.rs) and of StateRoot::overlay_root_with_updates
 * (crates/trie/db/src/state.rs:184-230).  STATUS as b200_dtrie (tests/test_gpu_dstate.py).
 *
 * create: like b200_state_root_full (segment a = storage of account a).
 * apply:  m account entries, keys strictly ascending; acct_flags[i]: bit 0 = exists after the block (0 = destroyed: its
 *         storage trie is released), bit 1 = account data unchanged (accts[i] ignored; its leaf is re-hashed because its
 *         storage root changes), bit 2 = storage wiped before this block's slots apply (HashedStorage::wiped); NULL =
 *         all plain upserts.  Slots of entry i: seg_offsets[i] .. seg_offsets[i+1], keys ascending, zero value deletes.
 *         Every account whose storage changes needs an entry.  Entries for absent accounts with bit 0 clear / bit 1 set
 *         are ignored together with their slots.
 * outputs (all optional): account TrieUpdates as in b200_dtrie_apply; storage records with trie_id = account entry
 *         index; opt_storage_deleted[i] = 1 when entry i's storage trie was released (StorageTrieUpdates::is_deleted). */
typedef struct b200_dstate b200_dstate;
B200_API int32_t b200_dstate_create(b200_ctx *, const uint8_t *acct_keys32, const b200_account *accts, uint64_t n_accounts,
                                    const uint8_t *slot_keys32, const uint8_t *values32_be, const uint64_t *seg_offsets,
                                    b200_dstate **out, uint8_t root32[32] /* nullable */);
B200_API int32_t b200_dstate_apply(b200_dstate *, const uint8_t *acct_keys32, const b200_account *accts,
                                   const uint8_t *acct_flags, uint64_t m, const uint8_t *slot_keys32,
                                   const uint8_t *values32_be, const uint64_t *seg_offsets, uint8_t root32[32],
                                   b200_updates *opt_acct_updated, b200_updates *opt_acct_removed,
                                   b200_updates *opt_storage_updated, b200_updates *opt_storage_removed,
                                   uint8_t *opt_storage_deleted, b200_stats *opt_stats);
/* Multi-GPU: one rank's shard of a state split by top key nibble (SURVEY.md §8e; the layout of b200_subtrie_frontier).
 * The shard keeps its accounts as 16 bucket tries; after every apply b200_dstate_frontier returns its 16 entries (empty
 * for buckets it does not hold), the ranks all-gather them (NCCL, 16 x 68 bytes) and b200_root_from_frontier gives the
 * state root.  root32 of create / apply is the root of the shard on its own (equal to the state root when one rank
 * holds every bucket).  TrieUpdates are unaffected by the sharding (the depth-0 root branch is never stored). */
B200_API int32_t b200_dstate_create_sharded(b200_ctx *, const uint8_t *acct_keys32, const b200_account *accts,
                                            uint64_t n_accounts, const uint8_t *slot_keys32, const uint8_t *values32_be,
                                            const uint64_t *seg_offsets, b200_dstate **out, uint8_t root32[32]);
/* Device-resident seed: every pointer is a device pointer (a state too large to stage through one host call is uploaded
 * in pieces by the caller); n_slots = d_seg_offsets[n_accounts]; sharded != 0 selects the sharded layout. */
B200_API int32_t b200_dstate_create_dev(b200_ctx *, const void *d_acct_keys32, const void *d_accts, uint64_t n_accounts,
                                        const void *d_slot_keys32, const void *d_values32_be, const void *d_seg_offsets,
                                        uint64_t n_slots, int32_t sharded, b200_dstate **out, void *d_root32 /* nullable */);
B200_API int32_t b200_dstate_frontier(b200_dstate *, b200_frontier_entry out16[16]);
/* The frontier entries of a sharded state after each of a batch of candidate blocks, each applied on its own to the state
 * as it is (siblings, not a chain); the state does not change.  The ranks all-gather out (n_blocks x 16 x 68 bytes) and
 * b200_root_from_frontier of block b's merged entries is the root b200_dstate_overlay_roots gives on an unsharded state:
 * payload validation and payload building over a sharded state, before b200_dstate_apply keeps one block.  Inputs in the
 * layout and with the rules of b200_dstate_overlay_roots (each rank passes its part of every block).  out[16b .. 16b + 15]
 * = what b200_dstate_frontier returns after b200_dstate_apply of block b alone: a bucket the block does not touch keeps its
 * entry, a bucket it empties gives an all-zero entry.  A block without entries gives the current frontier.  Errors:
 * B200_ERR_INVALID_ARG for an unsharded state and as b200_dstate_overlay_roots (null pointers, bad offsets, the limits),
 * B200_ERR_UNSORTED; out is zeroed on any error. */
B200_API int32_t b200_dstate_overlay_frontiers(b200_dstate *, uint64_t n_blocks, const uint8_t *acct_keys32, const b200_account *accts,
                                               const uint8_t *acct_flags /* nullable */, const uint64_t *block_acct_offset /* [n_blocks+1] */,
                                               const uint8_t *slot_keys32, const uint8_t *values32_be, const uint64_t *seg_offsets /* [M+1] */,
                                               b200_frontier_entry *out /* [n_blocks][16] */, b200_stats *opt_stats);
/* Merkle proofs from the resident state (SURVEY.md §8 f4; eth_getProof / reth's Proof::account_proof and storage_proof,
 * crates/trie/trie/src/proof/mod.rs): target t's proof is nodes node_offset[t] .. node_offset[t+1], node k's RLP is
 * rlp[rlp_offset[k] .. rlp_offset[k+1]), root first — every node whose position is a prefix of the target key (what
 * alloy-trie's ProofRetainer keeps): extension and branch are separate nodes, the walk ends at a leaf (inclusion, or
 * exclusion by another key), at an empty branch slot or inside a diverging extension.  An empty trie gives the single
 * node 0x80.  Pinned by reth's own vectors (crates/trie/db/tests/proof.rs:44-165).  Not for sharded states: see
 * b200_dstate_sharded_multiproof. */
typedef struct {
    uint64_t n_targets;
    uint64_t *node_offset; /* [n_targets+1] */
    uint64_t n_nodes;
    uint64_t *rlp_offset;  /* [n_nodes+1] */
    uint8_t *rlp;
    uint8_t *node_depth;   /* [n_nodes] nibbles of the target key that lead to the node: its path in a ProofNodes /
                              MultiProof map (crates/trie/common/src/proofs.rs) is target[..node_depth] */
    uint32_t *node_masks;  /* [n_nodes] hash_mask << 16 | tree_mask of a branch node that reth stores in its trie tables (either
                              mask non-empty), 0 otherwise (leaves, extensions, unstored branches): the entries of
                              MultiProof::branch_node_masks / StorageMultiProof::branch_node_masks (proofs.rs:185,601;
                              BranchNodeMasks, crates/trie/common/src/trie.rs:13-18) that Proof::with_branch_node_masks(true)
                              collects from the hash builder's updated_branch_nodes (proof/mod.rs) */
    void *_owner;
} b200_proofs;
B200_API int32_t b200_dstate_account_proofs(b200_dstate *, const uint8_t *acct_keys32, uint64_t n, b200_proofs *out);
B200_API int32_t b200_dstate_storage_proofs(b200_dstate *, const uint8_t *acct_key32, const uint8_t *slot_keys32, uint64_t n,
                                            uint8_t storage_root32[32] /* nullable */, b200_proofs *out);
/* Multiproof batch (Proof::multiproof over MultiProofTargets, crates/trie/trie/src/proof/mod.rs:143-193; the unit of work of
 * the proof workers in crates/trie/parallel/src/proof_task.rs): n target accounts, account i with the hashed slot targets
 * slot_seg_offsets[i] .. slot_seg_offsets[i+1] of slot_keys32.  One call returns the account proofs (target i = account i),
 * storage_roots32[i] (EMPTY_ROOT_HASH for an absent account) and the proofs of all slot targets (target j = slot j; an
 * absent account's slots prove with the single node 0x80).  MultiProof::account_subtree = { key[..node_depth] -> rlp } over
 * account_proofs; StorageMultiProof{root, subtree} per account the same over its slot targets. */
B200_API int32_t b200_dstate_multiproof(b200_dstate *, const uint8_t *acct_keys32, uint64_t n_accounts,
                                        const uint64_t *slot_seg_offsets, const uint8_t *slot_keys32, b200_proofs *account_proofs,
                                        uint8_t *storage_roots32, b200_proofs *storage_proofs);
B200_API void b200_proofs_release(b200_proofs *);
/* Proofs over a sharded state (b200_dstate_create_sharded): eth_getProof and the proof workers' Proof::multiproof when the
 * state is spread over several GPUs.  The depth-0 root branch of the whole state is in no shard; each rank gives its part of
 * that node (b200_dstate_frontier and b200_dstate_frontier_masks), the ranks all-gather them, and each rank proves the
 * targets of its own buckets with b200_dstate_sharded_multiproof.
 *
 * The bits this shard's buckets set in the masks of the depth-0 root branch of the whole state.
 * hash bit k: bucket k's top node is a branch at depth 1.
 * tree bit k: bucket k's top node is a branch that reth stores (tree_mask | hash_mask != 0), at any depth.
 * Buckets the shard does not hold, leaf tops and empty buckets give 0.  The ranks OR their masks.
 * An unsharded state gives B200_ERR_INVALID_ARG. */
B200_API int32_t b200_dstate_frontier_masks(b200_dstate *, uint16_t *hash_mask, uint16_t *tree_mask);
/* b200_dstate_multiproof on one rank's shard.  merged[16]: the entry of every bucket from its owner, as passed to
 * b200_root_from_frontier.  root_hash_mask / root_tree_mask: the OR of every rank's b200_dstate_frontier_masks.
 *
 * Equality: every output is byte for byte what b200_dstate_multiproof gives for the same targets on an unsharded state of
 * all accounts: node RLPs, node order, node_depth, node_masks, storage_roots32, and the 0x80 proofs of an absent account's
 * slots.
 *
 * The root, decided by the number of non-empty buckets in merged:
 *   none: every account proof is the single node 0x80;
 *   exactly one, bucket j: its trie is the whole trie and every proof walks it from parent depth -1 (its top node is the
 *     root: an extension over nibble j when the top is a branch), also for targets whose own bucket is empty;
 *   two or more: node 0 is the root branch, at depth 0, with node_masks hash << 16 | tree (0 when both are 0).  A target
 *     whose bucket is non-empty continues from that bucket's top node at parent depth 0; for a target whose bucket is
 *     empty the proof ends with the root branch.
 *
 * The answering bucket of a target is its own top nibble when that bucket is non-empty, otherwise in the one-bucket case
 * that one bucket, otherwise none (any shard can answer).  A shard answers a target only when it holds the answering bucket
 * or there is none; a target of another shard, storage targets of its account included, is B200_ERR_INVALID_ARG.  The
 * call never returns a partial proof.
 *
 * Checks against the shard's own data, all B200_ERR_INVALID_ARG, so that a stale or foreign frontier cannot give a wrong
 * proof: for every bucket the shard holds, merged[k] equals its current frontier entry byte for byte (so it is not empty)
 * and the two mask bits of bit k equal its own; every entry is well formed (as_root_len 0 or 32, as_child_len at most 33,
 * both zero together) and no mask bit is set for an empty entry.
 *
 * Everything else is as for b200_dstate_multiproof: null pointers, offsets and the 2^24 target limit; B200_ERR_INVALID_ARG
 * for an unsharded state.  On error both b200_proofs are released and zeroed.  The state does not change. */
B200_API int32_t b200_dstate_sharded_multiproof(b200_dstate *, const b200_frontier_entry merged[16],
                                                uint16_t root_hash_mask, uint16_t root_tree_mask,
                                                const uint8_t *acct_keys32, uint64_t n_accounts,
                                                const uint64_t *slot_seg_offsets, const uint8_t *slot_keys32,
                                                b200_proofs *account_proofs, uint8_t *storage_roots32,
                                                b200_proofs *storage_proofs);
/* Execution witness of one block (reth's TrieWitness::compute, crates/trie/trie/src/witness.rs; what debug_executionWitness
 * and stateless re-execution consume): { keccak(node) -> node RLP } of every trie node needed to apply the block to this
 * state, computed on the device from the resident state, which stays unchanged.  The block comes in exactly the layout of
 * b200_dstate_apply and with its rules: a destroyed entry is removed and its storage counts as wiped, an entry with bit 1 set
 * for an absent account is ignored (its key and slots are still proved); the slot entries of every entry are targets.
 * The map holds, keyed by the keccak of its RLP (nodes shorter than 32 bytes included):
 *   - every node of the proof of every target — the account entries, their slot entries, and every slot a wiped storage
 *     holds — with both nodes of every extension on a proof path, the branch below a diverging extension included;
 *   - the nodes a sparse trie has to reveal when a branch on a removal path keeps a single child: after the removal phase
 *     (Legacy: removals before upserts; Canonical: upserts first, so inserted keys keep a branch alive) a branch with exactly
 *     one surviving child c whose node is hashed and on no target's path adds the proof of path ‖ c ‖ 0…0 from depth
 *     |path ‖ c| on.  Storage tries first; a live account entry is a removal iff its account (the resident one with flag
 *     bit 1) is empty and its storage root after the block is EMPTY_ROOT_HASH;
 *   - Legacy only: the storage-root node (both nodes of an extension root, 0x80 for an empty storage) of every account entry
 *     without storage targets.
 * Canonical drops every 0x80 node.  An empty block (m = 0) gives the empty map, or with always_include_root the single
 * entry { state root: root node } ({ EMPTY_ROOT_HASH: 0x80 } for an empty state).  Entries are sorted by hash, without
 * duplicates: entry i is hashes32[32i ..], rlp[rlp_offset[i] .. rlp_offset[i+1]).  Keys must be strictly ascending
 * (B200_ERR_UNSORTED).  Not for sharded states (B200_ERR_INVALID_ARG): see b200_dstate_sharded_witness. */
enum { B200_WITNESS_LEGACY = 0, B200_WITNESS_CANONICAL = 1 };
typedef struct {
    uint64_t n;
    uint8_t *hashes32;     /* [n][32] ascending */
    uint64_t *rlp_offset;  /* [n+1] */
    uint8_t *rlp;
    void *_owner;
} b200_witness;
B200_API int32_t b200_dstate_witness(b200_dstate *, const uint8_t *acct_keys32, const b200_account *accts, const uint8_t *acct_flags,
                                     uint64_t m, const uint8_t *slot_keys32, const uint8_t *values32_be, const uint64_t *seg_offsets,
                                     int32_t mode, int32_t always_include_root, b200_witness *out);
B200_API void b200_witness_release(b200_witness *);
/* The execution witness of a block over a sharded state (b200_dstate_create_sharded): debug_executionWitness, the
 * invalid-block witness hook and stateless clients when the state is spread over several GPUs.  Each rank passes its part
 * of the block; the union of the ranks' maps, duplicates removed, is byte for byte the map b200_dstate_witness gives for the
 * whole block on an unsharded state of all accounts, in both modes, and every rank's map is a subset of it.  The depth-0
 * root branch is in no shard, and whether it keeps a single child after the removal phase is the one decision no shard
 * makes alone: each rank gives its kept mask (b200_dstate_witness_root_kept), and the ranks OR the masks and all-gather
 * them with the frontier (b200_dstate_frontier) and the root masks (b200_dstate_frontier_masks).
 *
 * This shard's kept mask for its part of the block (a block in the b200_dstate_apply layout, as b200_dstate_witness takes
 * it).  The entries are routed by their own top nibble; an entry of a bucket this shard does not hold counts as an absent
 * account.  Bit k: after the mode's removal phase (Legacy: the removals; Canonical: the upserts, then the removals) bucket
 * k still holds a leaf: the shard holds bucket k and not every leaf of it is removed, or in Canonical mode the part inserts
 * a live account into bucket k.  The OR of every rank's mask, each over the entries of its own buckets, is the set of
 * surviving children of the unsharded root branch.  Errors as b200_dstate_witness (*kept is then 0); an unsharded state is
 * B200_ERR_INVALID_ARG.  The state does not change. */
B200_API int32_t b200_dstate_witness_root_kept(b200_dstate *, const uint8_t *acct_keys32, const b200_account *accts,
                                               const uint8_t *acct_flags, uint64_t m, const uint8_t *slot_keys32,
                                               const uint8_t *values32_be, const uint64_t *seg_offsets, int32_t mode, uint16_t *kept);
/* b200_dstate_witness on one rank's shard.  merged, root_hash_mask, root_tree_mask: as for b200_dstate_sharded_multiproof;
 * root_kept: the OR of every rank's b200_dstate_witness_root_kept (for the same block and mode).
 *
 * The rule of b200_dstate_witness, split by the number of non-empty buckets in merged:
 *   none: the state is empty, every proof is the single node 0x80 (dropped in Canonical mode);
 *   exactly one, bucket j: its trie is the whole trie, walked from parent depth -1 (the root is an extension over nibble j
 *     when its top is a branch; both nodes belong to the witness), removal reveals included, also at the top branch;
 *   two or more: every account proof starts with the depth-0 root branch and goes on from the top of the key's own bucket
 *     at parent depth 0 (nothing more when that bucket is empty).  The reveal at depth 0 applies when root_kept has the
 *     single bit c, merged[c] is hashed (as_child_len 33) and no entry of the block has top nibble c: the owner of bucket c
 *     then adds the proof of c ‖ 0…0 from depth 1 on.
 * Storage targets, the Legacy storage-root nodes and the wipe expansion stay in the shard that owns the account.
 *
 * An entry belongs to the owner of its own bucket when that bucket is non-empty in merged, in the one-bucket case to the
 * owner of that bucket, and with no bucket to any shard; an entry of another shard, its slots included, is
 * B200_ERR_INVALID_ARG.  With two or more buckets, an entry whose bucket is empty in merged belongs to every shard: every
 * part holds it (its nodes are the same from any shard, and the union removes the duplicates).  A part without entries gives the empty map, or with always_include_root the single entry { state
 * root: root node } (in the one-bucket case only from the owner of that bucket; the others give the empty map), unless the
 * shard owes the depth-0 reveal.  The caller sets always_include_root only when the whole block is empty: on an empty state
 * in Canonical mode a part's root entry would otherwise be a 0x80 the unsharded map drops.
 *
 * Checks, all B200_ERR_INVALID_ARG: those of b200_dstate_sharded_multiproof on merged and the masks, and these on root_kept:
 *   - for every bucket k this shard holds, bit k equals the kept bit this call computes for its part;
 *   - for every bucket k empty in merged: in Legacy mode bit k is 0; in Canonical mode with two or more buckets, bit k is
 *     set exactly when this part inserts a live account into bucket k.
 * So every bit of root_kept is checked by some rank (a non-empty bucket's by its owner, an empty bucket's by every rank):
 * a stale or foreign kept mask makes at least one rank's call fail, and never makes all of them succeed with a wrong
 * union.  (With fewer than two buckets the mask does not enter the witness.)  Everything else is as for b200_dstate_witness (B200_ERR_UNSORTED, the 2^24 limit, the modes).  On
 * any error out is released and zeroed.  The state does not change.  opt_stats (nullable): the call's counters. */
B200_API int32_t b200_dstate_sharded_witness(b200_dstate *, const b200_frontier_entry merged[16], uint16_t root_hash_mask,
                                             uint16_t root_tree_mask, uint16_t root_kept, const uint8_t *acct_keys32,
                                             const b200_account *accts, const uint8_t *acct_flags, uint64_t m,
                                             const uint8_t *slot_keys32, const uint8_t *values32_be, const uint64_t *seg_offsets,
                                             int32_t mode, int32_t always_include_root, b200_witness *out, b200_stats *opt_stats);
/* Post-block state roots from execution witnesses: stateless validation (reth: DecodedMultiProofV2::from_witness,
 * crates/trie/common/src/proofs.rs:469-544, revealed into a SparseStateTrie and updated, crates/trie/sparse/src/state.rs).
 * A batch of n_blocks independent blocks, each with its own parent state root and witness; no b200_dstate is involved.
 *   witness of block b : nodes block_node_offset[b] .. block_node_offset[b+1]; node i is
 *                        node_rlp[node_rlp_offset[i] .. node_rlp_offset[i+1]) (ExecutionWitness.state: RLPs only — every
 *                        node is hashed on the device).  Duplicates and unrelated nodes are allowed; a block only uses its
 *                        own nodes.
 *   block b            : account entries block_acct_offset[b] .. block_acct_offset[b+1] in the layout of b200_dstate_apply and
 *                        with its rules (keys strictly ascending inside a block; seg_offsets [M+1] over all M entries of the
 *                        call; flag bit 0 clear = destroyed, its slots ignored; bit 1 = account data unchanged; bit 2 = storage
 *                        wiped first; zero value deletes a slot; an unchanged entry of an absent account is ignored with its
 *                        slots; a live entry is an upsert, also of an empty account with an empty storage).
 * Per block (block_status[b], roots32[32b..]; a failed block's root is zeroed, other blocks are unaffected):
 *   B200_OK                     : the post-block state root.  A block without entries keeps its parent root and needs no node;
 *                                 a parent root of EMPTY_ROOT_HASH is the empty state and needs no node.
 *   B200_ERR_WITNESS_INCOMPLETE : a node the computation needs is missing (also: a parent root whose node is missing).
 *   B200_ERR_INVALID_ARG        : a node reached from the parent root fails one of these checks, and only these are made
 *                                 (non-minimal RLP, a branch with fewer than two children or an extension above a leaf or an
 *                                 extension are accepted as they are): bad RLP, trailing
 *                                 bytes, a branch with a non-empty 17th item, a leaf path that does not end at nibble 64, an
 *                                 inline child of 32 bytes or more, a hashed child that is not 32 bytes, an account value
 *                                 that is not a TrieAccount, a storage value that is zero or longer than 32 bytes).  Wins over
 *                                 INCOMPLETE.
 * The nodes needed: (a) every node on the path to each account key of the block, and to each slot key of every live storage
 * trie the block changes and does not wipe (the path ends at the leaf, an empty slot, or a diverging leaf or extension);
 * (b) every hashed child on no such path that in the post-block trie hangs more than one nibble below its nearest branch
 * (its encoding changes), except the child of an extension, which is a branch and keeps its hash.  Nothing of a wiped storage
 * trie is needed.  A missing node of kind (a) or (b) gives B200_ERR_WITNESS_INCOMPLETE, never a wrong root; so does a
 * missing hashed leaf at depth 64 (two keys sharing 63 nibbles), which the fold cannot represent.  The witness
 * b200_dstate_witness returns, in either mode, holds every node of kind (a) and (b).
 * Call-level errors: null pointers, offsets that do not start at 0 or are not monotone (B200_ERR_INVALID_ARG); keys not
 * strictly ascending inside a block or an entry (B200_ERR_UNSORTED).  Limit: nodes, entries, and revealed items plus entries
 * each below 2^31-1 per call (B200_ERR_INVALID_ARG). */
B200_API int32_t b200_witness_roots(b200_ctx *, uint64_t n_blocks, const uint8_t *parent_roots32, const uint8_t *node_rlp,
                                    const uint64_t *node_rlp_offset /* [N+1] */, const uint64_t *block_node_offset /* [n_blocks+1] */,
                                    const uint8_t *acct_keys32, const b200_account *accts, const uint8_t *acct_flags /* nullable */,
                                    const uint64_t *block_acct_offset /* [n_blocks+1] */, const uint8_t *slot_keys32,
                                    const uint8_t *values32_be, const uint64_t *seg_offsets /* [M+1] */, uint8_t *roots32,
                                    int32_t *block_status, b200_stats *opt_stats);
/* Post-block state roots of a batch of candidate blocks, each applied on its own to the state as it is (siblings, not a
 * chain); the state does not change (reth: StateRootProvider::state_root(hashed_state) on the latest state — payload
 * validation, payload building, sibling payloads; a chain of uncommitted blocks is one block with their merged entries).
 * Block b: account entries block_acct_offset[b] .. block_acct_offset[b+1], in the layout of b200_dstate_apply and with its
 * rules (flags bit 0/1/2, zero value deletes, seg_offsets [M+1] over all M entries of the call).  roots32[32b..] = the root
 * b200_dstate_apply of that block alone would return.  A block without entries gives the current root.  There is no per-block
 * status: the resident state holds every node a block needs.  Call-level errors as b200_witness_roots (B200_ERR_INVALID_ARG
 * for null pointers, offsets that do not start at 0 or are not monotone, and the limits; B200_ERR_UNSORTED); a sharded state
 * gives B200_ERR_INVALID_ARG.  The same as b200_dstate_overlay_roots_with_updates without outputs. */
B200_API int32_t b200_dstate_overlay_roots(b200_dstate *, uint64_t n_blocks, const uint8_t *acct_keys32, const b200_account *accts,
                                           const uint8_t *acct_flags /* nullable */, const uint64_t *block_acct_offset /* [n_blocks+1] */,
                                           const uint8_t *slot_keys32, const uint8_t *values32_be, const uint64_t *seg_offsets /* [M+1] */,
                                           uint8_t *roots32, b200_stats *opt_stats);
/* b200_dstate_overlay_roots plus the TrieUpdates of every block (reth: StateRoot::overlay_root_with_updates, what
 * state_root_with_updates(hashed_state) returns); the state still does not change.  Inputs, roots and call-level errors as
 * b200_dstate_overlay_roots.  Outputs, all nullable, as b200_dstate_apply's: account records with trie_id = block index;
 * storage records with trie_id = account entry index over the whole call (block b owns entries block_acct_offset[b] ..
 * [b+1]); opt_storage_deleted[M].  On error every list is released and zeroed, and opt_storage_deleted is zeroed (all M
 * bytes, once block_acct_offset has passed its checks; before that M is not known and the array is left as it is); with no
 * entries every requested list is valid and empty.  opt_stats covers the whole call, both folds included.  The records follow reth's walker (TrieWalker + HashBuilder):
 *   updated : every stored branch the block's keys pass through, rebuilt — also on the path of a key that changes nothing
 *             (the delete of an absent slot, an ignored unchanged entry); unchanged siblings stay hashes and get no record;
 *   removed : every stored branch on such a path that is no longer a stored branch at the same path afterwards; masks 0, no
 *             hashes, the empty path never; a path that is also updated (same trie) is not removed (updates.rs:160-167);
 *   storage_deleted[i] : exactly b200_dstate_apply's flag — entry i's account exists and is destroyed, or exists and its
 *             storage is wiped.
 * Where a block changes the structure, the records can differ from b200_dstate_apply's of the same block in records that
 * restate a stored node as it is (both describe the same tables after the block). */
B200_API int32_t b200_dstate_overlay_roots_with_updates(b200_dstate *, uint64_t n_blocks, const uint8_t *acct_keys32,
                                                        const b200_account *accts, const uint8_t *acct_flags /* nullable */,
                                                        const uint64_t *block_acct_offset /* [n_blocks+1] */, const uint8_t *slot_keys32,
                                                        const uint8_t *values32_be, const uint64_t *seg_offsets /* [M+1] */,
                                                        uint8_t *roots32, b200_updates *opt_acct_updated, b200_updates *opt_acct_removed,
                                                        b200_updates *opt_storage_updated, b200_updates *opt_storage_removed,
                                                        uint8_t *opt_storage_deleted /* [M] */, b200_stats *opt_stats);
/* Merkle proofs of the state after one candidate block, against the state as it is, which does not change (reth:
 * Proof::overlay_multiproof, crates/trie/db/src/proof.rs, which StateProofProvider::multiproof / proof of a
 * MemoryOverlayStateProvider reach with the in-memory blocks prepended to the input — eth_getProof at a block that is not
 * persisted, and the proof workers of the state-root task over an OverlayStateProviderFactory).  A chain of in-memory blocks
 * is one block whose entries are merged, as for b200_dstate_overlay_roots.
 *   the block   : m account entries in the layout of b200_dstate_apply and with its rules (flags bit 0/1/2, zero value
 *                 deletes, seg_offsets [m+1]; keys strictly ascending).
 *   the targets : the layout of b200_dstate_multiproof: n_targets account keys, target i with the slot keys
 *                 target_slot_offsets[i] .. [i+1] of target_slot_keys32; account keys strictly ascending, and the slot keys
 *                 of each target (B200_ERR_UNSORTED).
 * Every output is byte for byte what b200_dstate_apply(block) followed by b200_dstate_multiproof(targets) gives on a twin
 * state: root32 (nullable) the apply's root; every target's nodes in account_proofs / storage_proofs with the same RLPs, in
 * the same order, with the same node_depth and node_masks; storage_roots32[i] the storage root of target i after the block
 * (EMPTY_ROOT_HASH when the account does not exist after it, and each of its slot targets then proves with the single node
 * 0x80).  m = 0 gives b200_dstate_multiproof of the targets.  Call-level errors are those of b200_dstate_overlay_roots plus
 * those of b200_dstate_multiproof: B200_ERR_INVALID_ARG for null pointers, offsets that do not start at 0 or are not monotone,
 * 2^24 or more account targets or slot targets, 2^31-1 or more entries plus revealed items, and a sharded state.  On error
 * both b200_proofs are released and zeroed.  opt_stats covers the whole call. */
B200_API int32_t b200_dstate_overlay_multiproof(b200_dstate *, const uint8_t *acct_keys32, const b200_account *accts,
                                                const uint8_t *acct_flags /* nullable */, uint64_t m, const uint8_t *slot_keys32,
                                                const uint8_t *values32_be, const uint64_t *seg_offsets /* [m+1] */,
                                                const uint8_t *target_keys32, uint64_t n_targets,
                                                const uint64_t *target_slot_offsets /* [n_targets+1] */, const uint8_t *target_slot_keys32,
                                                uint8_t root32[32] /* nullable */, b200_proofs *account_proofs,
                                                uint8_t *storage_roots32 /* [n_targets][32] */, b200_proofs *storage_proofs,
                                                b200_stats *opt_stats);
/* Execution witness of a block whose parent is a candidate block on top of the state as it is, which does not change
 * (reth: StateProofProvider::witness(input, target, mode) of a MemoryOverlayStateProvider — debug_executionWitness and the
 * invalid-block witness hook when the parent block is not persisted).  A chain of in-memory blocks is one overlay block whose
 * entries are merged, as for b200_dstate_overlay_roots.  Both blocks come in the layout of b200_dstate_apply and with its
 * rules; the target block exactly as b200_dstate_witness takes it.
 * out is byte for byte the map that b200_dstate_apply(overlay) followed by b200_dstate_witness(target, mode,
 * always_include_root) gives on a twin state, and overlay_root32 (nullable) that apply's root: the parent root a stateless
 * client checks the witness against.  Hence:
 *   - ov_m = 0 gives b200_dstate_witness of the target (overlay_root32: the current root);
 *   - m = 0 gives the empty map, or with always_include_root { overlay root: its root node } ({ EMPTY_ROOT_HASH: 0x80 } when
 *     the overlay empties the state);
 *   - both modes as b200_dstate_witness, the removal rule of a live account entry judged on the account after the overlay.
 * Call-level errors are those of b200_dstate_witness and b200_dstate_overlay_roots: B200_ERR_INVALID_ARG for null pointers,
 * offsets that do not start at 0 or are not monotone, a bad mode, 2^24 or more target entries or slots, 2^31-1 or more
 * entries plus revealed items, and a sharded state; B200_ERR_UNSORTED for keys not strictly ascending in either block.  On
 * error out is released and zeroed.  opt_stats covers the whole call. */
B200_API int32_t b200_dstate_overlay_witness(
    b200_dstate *,
    /* the overlay: in-memory blocks merged, b200_dstate_apply layout and rules */
    const uint8_t *ov_acct_keys32, const b200_account *ov_accts, const uint8_t *ov_acct_flags /* nullable */, uint64_t ov_m,
    const uint8_t *ov_slot_keys32, const uint8_t *ov_values32_be, const uint64_t *ov_seg_offsets /* [ov_m+1] */,
    /* the target block: the same layout, exactly what b200_dstate_witness takes */
    const uint8_t *acct_keys32, const b200_account *accts, const uint8_t *acct_flags /* nullable */, uint64_t m,
    const uint8_t *slot_keys32, const uint8_t *values32_be, const uint64_t *seg_offsets /* [m+1] */,
    int32_t mode, int32_t always_include_root,
    uint8_t overlay_root32[32] /* nullable */, b200_witness *out, b200_stats *opt_stats);
/* Trie changesets of a block: the values its changed trie nodes had before it, against the state as it is, which does not
 * change (reth: compute_trie_changesets(factory, &trie_updates), crates/trie/trie/src/changesets.rs:50-239, which the payload
 * validator calls for every block, crates/engine/tree/src/tree/payload_validator.rs:1795, and the changeset cache,
 * crates/trie/db/src/changesets.rs:69-170; written next to the block, they are applied backwards on unwind).  The input is
 * the block's TrieUpdatesSorted (crates/trie/common/src/updates.rs:550-556,759-765) reduced to what reth reads of it: paths
 * and is_deleted.  Paths use the packing of b200_updates (nibbles high-first, zero padded, lengths 1..63) and must be
 * strictly ascending in reth's Nibbles order, which is the order of (the 32 packed bytes, then the length): a prefix before
 * its extensions.
 *   account paths : n_acct_paths of them.
 *   storage tries : n_storage_tries hashed addresses, strictly ascending; storage_flags[i] bit 0 = is_deleted (nullable: none);
 *                   trie i's paths are storage_path_offsets[i] .. [i+1] (offsets start at 0, monotone), strictly ascending.
 * A stored node is a branch whose tree_mask | hash_mask != 0 at a non-empty path: what AccountsTrie / StoragesTrie hold.
 *   account_out : one record per account path, in input order, trie_id 0: the stored node at exactly that path (seek_exact),
 *                 or None — all three masks 0 and no hashes, as removed records are.
 *   storage_out : ordered by trie, then path, trie_id = index into storage_keys32.  A trie that is not deleted: one record per
 *                 path, as above.  A deleted trie (storage_trie_wiped_changeset_iter, changesets.rs:198-239): the merge by path
 *                 of its paths with every stored node of the trie — a path the trie holds gives its node, a path it does not
 *                 gives None, a stored node on no path gives itself.  A key without a resident account, or with an empty
 *                 storage, has an empty trie: its paths are all None and a deleted one adds nothing.  A trie without records
 *                 has none in the list (reth leaves an empty storage changeset out); is_deleted is the caller's to copy.
 * The state is left as it is, so this call comes before the b200_dstate_apply of the block, which overwrites the old nodes.
 * No paths at all give two valid, empty lists.  Errors: B200_ERR_INVALID_ARG for null pointers with non-zero counts, offsets
 * that do not start at 0 or are not monotone, a path length of 0 or over 63, non-zero padding, a sharded state, and 2^31-1 or
 * more records in or out of a list; B200_ERR_UNSORTED for any order violation, duplicates included.  On error both outputs
 * are released and zeroed.  Release them with b200_updates_release. */
B200_API int32_t b200_dstate_trie_changesets(
    b200_dstate *,
    const uint8_t *acct_path_len, const uint8_t *acct_path_packed /* [n][32] */, uint64_t n_acct_paths,
    const uint8_t *storage_keys32, const uint8_t *storage_flags /* nullable; bit 0 = is_deleted */, uint64_t n_storage_tries,
    const uint64_t *storage_path_offsets /* [n_storage_tries+1] */, const uint8_t *storage_path_len,
    const uint8_t *storage_path_packed /* [N][32] */,
    b200_updates *account_out, b200_updates *storage_out, b200_stats *opt_stats);
/* b200_dstate_apply with the block already in device memory (every input pointer and d_root32 are device pointers;
 * n_entries = d_seg_offsets[m]); the update records, if wanted, still arrive in host memory. */
B200_API int32_t b200_dstate_apply_dev(b200_dstate *, const void *d_acct_keys32, const void *d_accts, const void *d_acct_flags,
                                       uint64_t m, const void *d_slot_keys32, const void *d_values32_be,
                                       const void *d_seg_offsets, uint64_t n_entries, void *d_root32,
                                       b200_updates *opt_acct_updated, b200_updates *opt_acct_removed,
                                       b200_updates *opt_storage_updated, b200_updates *opt_storage_removed,
                                       uint8_t *opt_storage_deleted, b200_stats *opt_stats);
B200_API int32_t b200_dstate_root(b200_dstate *, uint8_t root32[32]);
B200_API uint64_t b200_dstate_accounts(const b200_dstate *);
B200_API uint64_t b200_dstate_slots(const b200_dstate *);
B200_API uint64_t b200_dstate_device_bytes(const b200_dstate *);
B200_API void b200_dstate_destroy(b200_dstate *);

#ifdef __cplusplus
}
#endif
#endif /* B200TRIE_H */
