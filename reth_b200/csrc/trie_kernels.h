// trie_kernels.h — device-side data layout of one forest build and the kernel launch interface
// (internal to libb200trie.so).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace b200 {

// sticky device error codes (mapped to b200_status by the engine)
enum : int {
    B200_DEVERR_NONE = 0,
    B200_DEVERR_UNSORTED = 1,
    B200_DEVERR_ZERO_VALUE = 2,
    B200_DEVERR_INLINE_HASH_CHILD = 3,
    B200_DEVERR_BAD_OFFSETS = 4,
    B200_DEVERR_NOT_FOUND = 5,
    B200_DEVERR_CORRUPT = 6,  // dynamic trie: a walk did not terminate within 64 hops
};

// node / leaf meta byte
// META_ISNODE (leaf_meta only): the position holds the hash of a whole unchanged subtree (HashBuilder::add_branch,
// tk_items.cuh), which its parent treats like a branch child (hash / tree mask bits)
enum : uint32_t { META_LEN = 31u, META_EXT = 32u, META_STORED = 64u, META_ISNODE = 128u };

enum : int { CNT_HASHED = 0, CNT_EXT = 1, CNT_COUNT = 4 };

struct b200_account_dev {  // == b200_account (include/b200trie.h), 72 bytes
    uint64_t nonce;
    uint8_t balance_be[32];
    uint8_t code_hash[32];
};
static_assert(sizeof(b200_account_dev) == 72, "account layout");

struct FrontierEntryDev {  // == b200_frontier_entry
    uint8_t as_child_len;
    uint8_t as_child[33];
    uint8_t as_root_len;
    uint8_t as_root[33];
};
static_assert(sizeof(FrontierEntryDev) == 68, "frontier layout");

// All arrays live in HBM for the duration of one build (and stay resident afterwards: the node-hash
// frontier of every level is exactly node_ref/leaf_ref).
//
//   per leaf  (n)    : keys 32 B (input) | Lp 1 | nibs 1 | leaf_ref 32 | leaf_meta 1 | S 4 | E 4
//   per gap   (n-1)  : key_sorted 2 (depth | head flag << 8) | gap_sorted 4   (gaps ordered by (depth, position))
//   per branch (B)   : node_start 4 (CSR into gap_sorted) | node_ref 32 | node_meta 1 | node_l 4 | node_r 4 |
//                      node_masks 8 (state, tree, hash, depth)
struct ForestDev {
    uint64_t n;             // leaves
    const uint8_t *keys;    // [n][32] sorted inside each trie
    uint8_t *Lp;            // [n+1] gap depth; Lp[0] = Lp[n] = 0xFF; 0xFF = trie boundary
    uint8_t *nibs;          // [n+1] (left nibble << 4) | right nibble at depth Lp
    uint8_t *leaf_ref;      // [n][32] digest, or inline RLP (< 32 bytes)
    uint8_t *leaf_meta;     // [n] 0 = hashed, else inline length
    uint32_t *S, *E;        // [n] frontier item starting / ending at this leaf (< n leaf, else n + node id)
    const uint32_t *gap_sorted;   // [n-1]
    const uint32_t *node_start;   // [B+1]
    uint8_t *node_ref;      // [B][32]
    uint8_t *node_meta;     // [B] inline length | META_EXT | META_STORED
    uint32_t *node_l, *node_r;    // [B] leaf extent
    ushort4 *node_masks;    // [B]
    int *err;               // sticky error code
    unsigned long long *counters;  // [CNT_COUNT]
    int retain_updates;
};

struct UpdatesDev {
    uint32_t *trie_id;
    uint8_t *path_len;
    uint8_t *path_packed;
    uint16_t *state_mask, *tree_mask, *hash_mask;
    uint32_t *hash_offset;  // [n_stored] (exclusive); the engine appends the total
    uint8_t *hashes;
};

cudaError_t launch_latch_error(int *err, int *sticky, unsigned long long *counters, cudaStream_t st);
cudaError_t launch_mark_boundaries(const uint64_t *d_seg_offsets, uint64_t n_segs, uint64_t n, uint8_t *Lp, int *err,
                                   cudaStream_t st);
cudaError_t launch_lcp(const uint8_t *keys, uint64_t n, uint8_t *Lp, uint8_t *nibs, int *err, cudaStream_t st);
cudaError_t launch_iota(uint32_t *out, uint64_t n, uint32_t first, cudaStream_t st);
cudaError_t launch_fill_u32(uint32_t *out, uint64_t n, uint32_t value, cudaStream_t st);
cudaError_t launch_gap_keys(const uint8_t *Lp, uint64_t G, uint16_t *key, uint32_t *val, uint32_t *unresolved, cudaStream_t st);
cudaError_t launch_bucket_offsets(const uint16_t *key_sorted, uint64_t G, uint32_t *bucket_off, cudaStream_t st);
cudaError_t launch_head_fix(const uint8_t *keys, uint16_t *key_sorted, const uint32_t *gap_sorted, const uint64_t *seg_offsets,
                            uint64_t n_segs, const uint32_t *unresolved, uint64_t G, cudaStream_t st);
cudaError_t launch_level_ranges(uint32_t *node_start, const uint32_t *n_nodes_p, const uint32_t *bucket_off,
                                uint32_t *level_lo, cudaStream_t st);
cudaError_t launch_leaves(const ForestDev &f, bool account, const uint8_t *values, const uint8_t *storage_roots,
                          cudaStream_t st);
cudaError_t launch_branch_level(const ForestDev &f, const uint32_t *node_order, uint32_t pos_lo, uint32_t pos_hi,
                                int d, int cls, cudaStream_t st);
cudaError_t launch_node_class_keys(const uint32_t *node_start, const uint16_t *key_sorted, const uint32_t *n_nodes_p,
                                   uint64_t max_nodes, uint8_t *keys, uint32_t *ids, uint32_t *hist, cudaStream_t st);
cudaError_t launch_segment_roots(const ForestDev &f, const uint64_t *d_seg_offsets, uint64_t n_segs, uint8_t *roots,
                                 cudaStream_t st);
cudaError_t launch_stored_flags(const ForestDev &f, uint32_t n_nodes, uint8_t *flags, uint32_t *n_hashes,
                                cudaStream_t st);
cudaError_t launch_table_order_keys(const ForestDev &f, const uint32_t *ids, uint32_t count, uint64_t *keys, cudaStream_t st);
cudaError_t launch_row_sizes(const ForestDev &f, const uint32_t *ids, uint32_t count, int packed, int storage, uint64_t *size,
                             uint32_t *key_len, cudaStream_t st);
cudaError_t launch_encode_rows(const ForestDev &f, const uint32_t *ids, uint32_t count, int packed, int storage,
                               const uint64_t *d_seg_offsets, uint64_t n_segs, const uint8_t *acct_keys,
                               const uint64_t *row_off, uint8_t *out, cudaStream_t st);
cudaError_t launch_gather_updates(const ForestDev &f, const uint32_t *stored_ids, uint32_t n_stored,
                                  const uint32_t *hash_prefix, const uint32_t *prefix_by_record,
                                  const uint64_t *d_seg_offsets, uint64_t n_segs, const UpdatesDev &out,
                                  cudaStream_t st);
cudaError_t launch_nibble_buckets(const uint8_t *keys, uint64_t n, uint64_t *offs, cudaStream_t st);
cudaError_t launch_frontier(const ForestDev &f, const uint64_t *bucket_offsets, const uint8_t *values,
                            const uint8_t *storage_roots, FrontierEntryDev *out, cudaStream_t st);
cudaError_t launch_root_from_frontier(const FrontierEntryDev *fr, uint8_t *root, cudaStream_t st);
cudaError_t launch_merge_frontiers(const FrontierEntryDev *all, int world, FrontierEntryDev *out, int *err, cudaStream_t st);
cudaError_t launch_partition_owner(const uint8_t *digests, uint64_t n, int world, uint8_t *owner, unsigned long long *counts,
                                   cudaStream_t st);
cudaError_t launch_partition_gather(const uint8_t *digests, const uint8_t *values, uint32_t vb, const uint32_t *perm, uint64_t n,
                                    uint8_t *out_d, uint8_t *out_v, cudaStream_t st);
cudaError_t launch_gather_values(const uint8_t *values, uint32_t vb, const uint32_t *perm, uint64_t n, uint8_t *out_v, cudaStream_t st);

cudaError_t launch_parent_links(const ForestDev &f, uint32_t n_nodes, uint32_t *leaf_parent, uint32_t *node_parent,
                                cudaStream_t st);
cudaError_t launch_locate(const uint8_t *keys, uint64_t n, const uint8_t *dirty_keys, uint64_t m, uint32_t *idx_out,
                          int *err, cudaStream_t st);
cudaError_t launch_mark_pending(const ForestDev &f, const uint32_t *idx, uint64_t m, const uint32_t *leaf_parent,
                                const uint32_t *node_parent, uint32_t *pending, cudaStream_t st);
cudaError_t launch_wavefront(const ForestDev &f, uint8_t *accts, uint8_t *sroots, const uint8_t *new_accts,
                             const uint8_t *new_sroots, const uint32_t *idx, uint64_t m, const uint32_t *leaf_parent,
                             const uint32_t *node_parent, uint32_t *pending, uint32_t *dirty_list, uint32_t *dirty_count,
                             uint8_t *root_out, cudaStream_t st);
cudaError_t launch_wavefront_two_stage(const ForestDev &f, uint8_t *accts, uint8_t *sroots, const uint8_t *new_accts,
                                       const uint8_t *new_sroots, const uint32_t *idx, uint64_t m,
                                       const uint32_t *leaf_parent, const uint32_t *node_parent, uint32_t *pending,
                                       uint32_t *dirty_list, uint32_t *dirty_count, uint32_t *handoff_list,
                                       uint32_t *handoff_count, uint64_t max_handoff, uint8_t *root_out, int split_depth,
                                       cudaStream_t st);
cudaError_t launch_locate_classify(const uint8_t *keys, uint64_t n, const uint8_t *dirty_keys, const uint8_t *present,
                                   uint64_t m, uint32_t *lb, uint8_t *kind, uint32_t *counts, int *err, cudaStream_t st);
cudaError_t launch_merge_marks(const uint32_t *lb, const uint8_t *kind, uint64_t m, uint32_t *ins_at, uint32_t *del,
                               uint32_t *ins_flag, cudaStream_t st);
cudaError_t launch_merge_scatter(const uint8_t *keys, const uint8_t *accts, const uint8_t *sroots, uint64_t n,
                                 const uint32_t *ins_incl, const uint32_t *del_excl, const uint32_t *del,
                                 const uint8_t *dirty_keys, const uint8_t *new_accts, const uint8_t *new_sroots,
                                 const uint32_t *lb, const uint8_t *kind, const uint32_t *ins_rank, uint64_t m, uint8_t *nkeys,
                                 uint8_t *naccts, uint8_t *nsroots, cudaStream_t st);
cudaError_t launch_stored_flags_subset(const ForestDev &f, const uint32_t *ids, uint32_t count, uint8_t *flags,
                                       uint32_t *n_hashes, cudaStream_t st);
cudaError_t launch_pick_subset(const uint32_t *ids, const uint32_t *prefix, const uint32_t *sel_pos, uint32_t n_sel,
                               uint32_t *out_ids, uint32_t *out_prefix, cudaStream_t st);

// ------------------------------------------------------------------------------------------------ ordered tries (tk_ordered.cuh)
struct OrderedLeavesDev {
    const uint8_t *key_nibs;  // [n] true key length in nibbles (the padded keys are ForestDev::keys)
    const uint32_t *item;     // [n] item (in list order) carried by the leaf at this sorted position
    const uint32_t *order;    // [n] leaf positions in the order the leaf pass visits them (longest item first)
    const uint16_t *sched_sorted;  // [n] the sorted scheduling keys (65535 - Keccak blocks of the item)
    uint32_t *n_long;         // device word: leading entries of `order` that get a warp each
    const uint8_t *values;    // concatenated pre-encoded items
    const uint64_t *val_off;  // [n+1] byte offsets of the items in `values`
    uint64_t blob_len;
};
cudaError_t launch_ordered_keys(const uint64_t *d_seg_offsets, uint64_t n_segs, uint64_t n, const uint64_t *val_off,
                                uint8_t *keys, uint8_t *key_nibs, uint32_t *item, uint16_t *sched_key, uint32_t *pos, int *err,
                                cudaStream_t st);
cudaError_t launch_ordered_leaves(const ForestDev &f, const OrderedLeavesDev &o, cudaStream_t st);

// ------------------------------------------------------------------------------------------------ mixed items (tk_items.cuh)
// The input stream of an incremental HashBuilder run (TrieNodeIter, crates/trie/trie/src/node_iter.rs:200-304): changed /
// uncovered leaves and the stored hashes of unchanged subtrees, in key order.
struct ItemLeavesDev {
    const uint8_t *key_nibs;  // [n] 64 = a leaf; 0..63 = hash of the subtree rooted at the path of that many nibbles
    const uint8_t *flags;     // [n] bit 0: the subtree's nodes are in the trie tables (children_are_in_trie -> tree mask)
    int account;              // leaf values: b200_account (72-byte rows) | U256 BE (32-byte rows); hashes: first 32 bytes of the row
};
cudaError_t launch_item_leaves(const ForestDev &f, const ItemLeavesDev &it, const uint8_t *values, const uint8_t *storage_roots,
                               cudaStream_t st);

// ------------------------------------------------------------------------------------------------ dynamic trie (tk_dtrie.cuh)
constexpr uint32_t DT_NONE = 0xFFFFFFFFu;
constexpr uint32_t DT_LEAF = 0x80000000u;
constexpr uint32_t DT_LOCKED = 0xFFFFFFFEu;  // an attach word owned by an insert run for the duration of a round (never a valid id: ids < 2^31 - 2)
constexpr uint8_t DT_DEAD = 0xFF;  // ndepth / lmeta of a freed slot
constexpr int DT_MAX_HOPS = 66;

enum : int {
    DG_UNUSED0 = 0,
    DG_NLEAVES,       // live leaves
    DG_LEAF_ALLOC,    // bump pointers
    DG_NODE_ALLOC,
    DG_LEAF_FREE,     // free-stack heights
    DG_NODE_FREE,
    DG_SEEDS,         // list lengths of the current apply
    DG_BUILT,
    DG_REMOVED,
    DG_LIST_A,
    DG_LIST_B,
    DG_NINSERT,
    DG_FREED_NOW,
    DG_WORDS = 16
};

struct DTrieDev {
    // leaves [lcap]
    uint8_t *lkey, *lval, *lsroot, *lref, *lmeta;  // lval: 72-byte account or 32-byte slot value; lsroot: accounts only
    const uint8_t *lnib;  // arenas made from an items fold only (else null): path length of a hash leaf (lmeta META_ISNODE)
    uint32_t *lparent, *ltrie;                     // ltrie / ntrie: owning trie (nullptr = a single trie, id 0)
    uint8_t *lseed;
    // nodes [ncap]
    uint32_t *nchild;  // [ncap][16]
    uint8_t *ndepth;
    uint32_t *nparent;
    uint8_t *nref, *nmeta;
    ushort4 *nmasks;
    uint8_t *nkey;  // [ncap][32] a key of the subtree: its first ndepth nibbles are the node's path
    uint32_t *npending, *ntrie;
    uint8_t *nseed, *ncur, *nnext;
    // tries
    uint32_t *troot;     // [n_tries] child word of every trie's root
    uint8_t *top_out;    // the warp that finishes trie r stores its new root hash at top_out + top_stride * r
    uint32_t top_stride;
    uint32_t val_stride;  // 72 | 32
    int account;          // leaf encoding: rlp(TrieAccount) | rlp(U256)
    // free stacks, lists, globals
    uint32_t *leaf_free, *node_free;
    uint32_t *seeds, *built, *removed, *freed_now;
    uint32_t *unlock;  // [insert entries of the round] final value of the attach word a run owned, DT_LOCKED = none
    uint32_t *g;
    int *err;
    unsigned long long *counters;
    uint32_t lcap, ncap;
};

enum : uint8_t { DK_NOOP = 0, DK_UPDATE = 1, DK_DELETE = 2, DK_INSERT = 3, DK_TOUCH = 4 };

cudaError_t launch_dt_convert(const ForestDev &f, uint32_t n_nodes, const uint32_t *leaf_parent, const uint32_t *node_parent,
                              const uint32_t *leaf_trie, const DTrieDev &t, cudaStream_t st);
cudaError_t launch_dt_leaf_segments(const uint64_t *seg_offsets, uint64_t n_segs, uint64_t n, uint32_t *leaf_trie, cudaStream_t st);
cudaError_t launch_dt_locate(const DTrieDev &t, const uint32_t *trie_of_key, const uint8_t *keys, const uint8_t *vals,
                             const uint8_t *flags, uint64_t m, uint8_t *kind, uint32_t *leaf_of, cudaStream_t st);
cudaError_t launch_dt_update_detach(const DTrieDev &t, const uint8_t *accts, const uint8_t *sroots, uint64_t m,
                                    const uint8_t *kind, const uint32_t *leaf_of, uint32_t *touched, cudaStream_t st);
cudaError_t launch_dt_collapse_round(const DTrieDev &t, const uint32_t *list, const uint32_t *count_p, uint32_t max_count,
                                     uint8_t *defer, uint32_t *next, uint32_t *next_count, cudaStream_t st);
cudaError_t launch_dt_insert(const DTrieDev &t, const uint32_t *trie_of_key, const uint8_t *keys, const uint8_t *vals,
                             const uint8_t *sroots, const uint32_t *ins_idx, const uint32_t *n_ins_p, uint64_t max_ins,
                             uint64_t *attach, uint32_t *leaf_of, uint32_t max_per_run, uint8_t *pending, uint32_t *leftover,
                             cudaStream_t st);
cudaError_t launch_dt_rehash(const DTrieDev &t, uint32_t max_seeds, uint32_t *handoff, uint32_t *handoff_count, int split_depth,
                             bool already_marked, cudaStream_t st);
cudaError_t launch_dt_finish(const DTrieDev &t, uint32_t max_freed, cudaStream_t st);
cudaError_t launch_dt_stored_flags(const DTrieDev &t, uint32_t max_built, uint8_t *flags, uint32_t *n_hashes, cudaStream_t st);
cudaError_t launch_dt_gather_updates(const DTrieDev &t, const uint32_t *stored_ids, uint32_t n_stored,
                                     const uint32_t *hash_prefix_by_record, const UpdatesDev &out, cudaStream_t st);
cudaError_t launch_dt_removed_paths(const DTrieDev &t, uint32_t n_removed, uint8_t *path_len, uint8_t *path_packed,
                                    uint32_t *trie_id, cudaStream_t st);

cudaError_t launch_dt_wipe_list(const uint8_t *kind, const uint8_t *flags, const uint32_t *leaf_of, uint64_t m, uint32_t *tries,
                                uint32_t *count, cudaStream_t st);
cudaError_t launch_dt_wipe_begin(const DTrieDev &t, const uint32_t *tries, const uint32_t *count_p, uint32_t max_count,
                                 cudaStream_t st);
cudaError_t launch_dt_wipe_round(const DTrieDev &t, uint32_t lo, uint32_t hi, cudaStream_t st);
cudaError_t launch_dt_expand_tries(const uint64_t *seg_offsets, uint64_t m, const uint8_t *kind, const uint32_t *leaf_of,
                                   uint64_t n_entries, uint32_t *trie_of_key, cudaStream_t st);

cudaError_t launch_dt_nibble_tries(const uint8_t *keys, uint64_t m, uint32_t *trie_of_key, cudaStream_t st);
cudaError_t launch_dt_frontier(const DTrieDev &t, const uint8_t *bucket_roots, FrontierEntryDev *out, cudaStream_t st);

// Proof targets: trie_of_target[i] = a trie of t, DT_NONE (the empty trie), or DT_ALT | a trie of `alt` (the second arena
// of a call whose targets prove against two: the resident state and an overlay's fold); nullptr = trie 0 of t.
constexpr uint32_t DT_ALT = 0x80000000u;
cudaError_t launch_dt_proof_sizes(const DTrieDev &t, const DTrieDev &alt, const uint32_t *trie_of_target, const uint8_t *keys, uint64_t n,
                                  uint32_t *node_count, uint64_t *byte_count, cudaStream_t st);
cudaError_t launch_dt_proof_write(const DTrieDev &t, const DTrieDev &alt, const uint32_t *trie_of_target, const uint8_t *keys, uint64_t n,
                                  const uint64_t *node_base, const uint64_t *byte_base, uint8_t *rlp, uint64_t *rlp_offset,
                                  uint8_t *node_depth, uint32_t *node_masks, cudaStream_t st);
// Account proofs of a sharded state (b200_dstate_sharded_multiproof): `only` >= 0 when at most one bucket of the whole
// state is non-empty (its trie, or the empty trie 0x80 when none is, is then the whole trie); -1: every proof starts with
// the depth-0 root branch, its length (u32) at `branch` and its RLP at branch + 4 (device memory), masks hash << 16 | tree.
struct ShardRootDev {
    const uint8_t *branch;
    uint32_t masks;
    int32_t only;
};
cudaError_t launch_dt_sharded_proof_sizes(const DTrieDev &t, const ShardRootDev &r, const uint8_t *keys, uint64_t n, uint32_t *node_count,
                                          uint64_t *byte_count, cudaStream_t st);
cudaError_t launch_dt_sharded_proof_write(const DTrieDev &t, const ShardRootDev &r, const uint8_t *keys, uint64_t n, const uint64_t *node_base,
                                          const uint64_t *byte_base, uint8_t *rlp, uint64_t *rlp_offset, uint8_t *node_depth,
                                          uint32_t *node_masks, cudaStream_t st);
cudaError_t launch_dt_frontier_masks(const DTrieDev &t, uint16_t *out, cudaStream_t st);
cudaError_t launch_root_branch(const FrontierEntryDev *fr, uint8_t *out, cudaStream_t st);
cudaError_t launch_dt_find_leaves(const DTrieDev &t, const uint8_t *keys, uint64_t n, uint32_t *leaf_out, uint8_t *sroot_out, cudaStream_t st);
cudaError_t launch_dt_target_tries(const uint64_t *seg_offsets, uint64_t n_accounts, const uint32_t *leaf_of, uint64_t n_targets,
                                   uint32_t *trie_of_target, cudaStream_t st);
cudaError_t launch_dt_find_leaf(const DTrieDev &t, const uint8_t *key, uint32_t *out, uint64_t n_copies, cudaStream_t st);

// ------------------------------------------------------------------------------------------------ witness (tk_witness.cuh)
constexpr uint32_t WT_ROOT_ONLY = 1, WT_FIRST_ONLY = 2;  // dt_proof_walk stops: after the root node / after the first node kept
constexpr uint8_t WF_WIPED = 1, WF_EMPTIED = 2;          // storage trie flags: wiped by the block / every leaf removed
// target meta (u16): low byte min_len (nodes on shorter paths are skipped), then the stop bits; WM_SKIP = no node
constexpr uint16_t WM_ROOT_ONLY = WT_ROOT_ONLY << 8, WM_FIRST_ONLY = WT_FIRST_ONLY << 8, WM_SKIP = 0x8000;
struct WitnessMarks {       // per-call scratch of one arena
    uint32_t *gone;         // [ncap] bit c: every leaf below child c is removed
    uint32_t *seen;         // [ncap] bit c: a target walks through child c; bit 16 + c: an inserted key does (Canonical)
    uint32_t *list;         // branches that lost a child, [0, *n_list)
    uint32_t *n_list;
    uint8_t *trie_flags;    // WF_* per trie: storage forest [account leaf capacity]; account arena of a shard
                            // (b200_dstate_sharded_witness) [16], WF_EMPTIED per bucket; null otherwise
};
// b200_dstate_overlay_witness runs these on an overlay's folds: entry_trie (nullable: the account leaf) is the storage trie of
// every entry; res / res_trie: the resident arena, and its trie behind each trie of the fold, below the fold's hash leaves
// (res_trie nullptr: trie 0).  On the resident arenas res is the arena itself and holds no hash leaf.
// acct_trie (nullable: trie 0): the account trie of every entry (b200_dstate_sharded_witness: a bucket trie of the shard).
cudaError_t launch_wt_accounts(const DTrieDev &ta, const DTrieDev &ts, const uint8_t *keys, const uint8_t *flags, uint64_t m,
                               const uint32_t *entry_trie, const uint32_t *acct_trie, uint32_t *leaf_of, uint32_t *trie_of,
                               uint8_t *trie_flags, cudaStream_t st);
cudaError_t launch_wt_slots(const DTrieDev &ts, const WitnessMarks &w, const uint64_t *seg_offsets, uint64_t m, const uint32_t *trie_of,
                            const uint8_t *flags, const uint8_t *keys, const uint8_t *vals, uint64_t n, int canonical,
                            uint32_t *trie_of_target, uint8_t *nonzero, cudaStream_t st);
cudaError_t launch_wt_account_walk(const DTrieDev &ta, const DTrieDev &ts, const WitnessMarks &w, const uint8_t *keys, const uint8_t *accts,
                                   const uint8_t *flags, const uint64_t *seg_offsets, uint64_t m, const uint32_t *acct_trie,
                                   const uint32_t *leaf_of, const uint32_t *trie_of, const uint8_t *trie_flags, const uint8_t *nonzero,
                                   int canonical, uint32_t *root_trie, uint16_t *root_meta, cudaStream_t st);
cudaError_t launch_wt_reveal(const DTrieDev &t, const WitnessMarks &w, uint32_t max_list, int canonical, uint32_t *out_trie,
                             uint8_t *out_keys, uint16_t *out_meta, uint32_t *n_out, cudaStream_t st);
// the wipe queue holds (node, trie) pairs: node | DT_ALT = a node of res; trie_flags nullable: every trie of trie_of is wiped
cudaError_t launch_wt_wipe_roots(const DTrieDev &ts, const DTrieDev &res, const uint32_t *res_trie, const uint32_t *trie_of,
                                 const uint8_t *trie_flags, uint64_t m, bool write, uint32_t *queue, uint32_t *n_queue, uint32_t *n_out,
                                 uint32_t *out_trie, uint8_t *out_keys, cudaStream_t st);
cudaError_t launch_wt_wipe_round(const DTrieDev &ts, const DTrieDev &res, const uint32_t *res_trie, uint32_t *queue, uint32_t lo, uint32_t hi,
                                 uint32_t *n_queue, uint32_t *n_leaves, cudaStream_t st);
cudaError_t launch_wt_wipe_leaves(const DTrieDev &ts, const DTrieDev &res, const uint32_t *queue, uint32_t n, uint32_t *n_out,
                                  uint32_t *out_trie, uint8_t *out_keys, cudaStream_t st);
cudaError_t launch_wt_clear(const DTrieDev &t, const WitnessMarks &w, const uint32_t *trie_of, const uint8_t *keys, uint64_t n,
                            const uint32_t *leaf_of, uint8_t *trie_flags, cudaStream_t st);
cudaError_t launch_wt_proof_sizes(const DTrieDev &t, const DTrieDev &res, const uint32_t *res_trie, const uint32_t *trie_of,
                                  const uint8_t *keys, const uint16_t *meta, uint64_t n_fixed, const uint32_t *n_extra, uint64_t n_max,
                                  uint32_t *node_count, uint64_t *byte_count, cudaStream_t st);
cudaError_t launch_wt_proof_write(const DTrieDev &t, const DTrieDev &res, const uint32_t *res_trie, const uint32_t *trie_of,
                                  const uint8_t *keys, const uint16_t *meta, uint64_t n_fixed, const uint32_t *n_extra, uint64_t n_max,
                                  const uint64_t *node_base, const uint64_t *byte_base, uint64_t node_shift, uint64_t byte_shift,
                                  uint8_t *rlp, uint64_t *rlp_offset, cudaStream_t st);
// Account targets of a sharded state: the proofs start at the gathered root (trie ids unused, the bucket is the key's)
cudaError_t launch_wt_sharded_proof_sizes(const DTrieDev &t, const ShardRootDev &r, const uint8_t *keys, const uint16_t *meta, uint64_t n_fixed,
                                          const uint32_t *n_extra, uint64_t n_max, uint32_t *node_count, uint64_t *byte_count, cudaStream_t st);
cudaError_t launch_wt_sharded_proof_write(const DTrieDev &t, const ShardRootDev &r, const uint8_t *keys, const uint16_t *meta, uint64_t n_fixed,
                                          const uint32_t *n_extra, uint64_t n_max, const uint64_t *node_base, const uint64_t *byte_base,
                                          uint8_t *rlp, uint64_t *rlp_offset, cudaStream_t st);
cudaError_t launch_wt_unique(const uint8_t *sorted32, const uint32_t *perm, const uint64_t *rlp_offset, const uint8_t *rlp, uint64_t n,
                             int drop_empty, uint32_t *keep, uint64_t *kept_bytes, cudaStream_t st);
cudaError_t launch_wt_gather(const uint8_t *sorted32, const uint32_t *perm, const uint64_t *rlp_offset, const uint8_t *rlp, uint64_t n,
                             const uint32_t *keep, const uint32_t *pos, const uint64_t *byte_pos, uint8_t *out_hash, uint64_t *out_offset,
                             uint8_t *out_rlp, cudaStream_t st);

// ------------------------------------------------------------------------------------------------ trie changesets (tk_changesets.cuh)
// a row is (output trie id << 32 | source): a changed-path index, or CS_NODE | a node id of a deleted trie
cudaError_t launch_cs_lookup(const DTrieDev &t, const uint64_t *offs, uint64_t n_keys, const uint32_t *leaf_of, const uint8_t *kflags,
                             const uint8_t *len, const uint8_t *paths, uint64_t n, uint32_t *node_of, uint64_t *rows, uint32_t *n_rows,
                             cudaStream_t st);
cudaError_t launch_cs_wiped_rows(const DTrieDev &ts, const DTrieDev &ta, const uint32_t *queue, uint32_t n_queue, const uint8_t *keys32,
                                 uint64_t n_keys, uint64_t *rows, uint32_t *n_rows, cudaStream_t st);
cudaError_t launch_cs_sort_word(const DTrieDev &t, const uint8_t *len, const uint8_t *paths, const uint64_t *rows, uint32_t n, int w,
                                uint64_t *keys64, cudaStream_t st);
cudaError_t launch_cs_hash_counts(const DTrieDev &t, const uint64_t *rows, uint32_t n, const uint32_t *node_of, uint32_t *n_hashes,
                                  cudaStream_t st);
cudaError_t launch_cs_write(const DTrieDev &t, const uint64_t *rows, uint32_t n, const uint32_t *node_of, const uint8_t *len,
                            const uint8_t *paths, const uint32_t *hash_prefix, const UpdatesDev &out, cudaStream_t st);

// ------------------------------------------------------------------------------------------------ stateless roots (tk_stateless.cuh)
enum : uint32_t { SL_INCOMPLETE = 1u, SL_INVALID = 2u, SL_NONE = 0xFFFFFFFFu };
enum : int32_t { SL_STATUS_INVALID = -3, SL_STATUS_INCOMPLETE = -9 };  // == B200_ERR_INVALID_ARG, B200_ERR_WITNESS_INCOMPLETE
enum : uint8_t { SL_LEAF = 0, SL_BLIND = 1, SL_BLIND_BRANCH = 2 };  // item kinds: leaf, hashed child not in the witness (of
                                                                    // unknown kind / the child of an extension: a branch)
struct StatelessDev {
    const uint8_t *rlp;          // witness nodes of all blocks, node i = rlp[rlp_off[i], rlp_off[i+1])
    const uint64_t *rlp_off;     // [n_nodes + 1]
    const uint64_t *block_node;  // [n_blocks + 1] nodes of block b
    const uint8_t *dig_sorted;   // [n_nodes][32] node digests, ascending
    const uint32_t *dig_perm;    // [n_nodes] node of each sorted digest
    uint64_t n_nodes;
    const uint8_t *parent;       // [n_blocks][32]
    const uint64_t *block_acct;  // [n_blocks + 1] account entries of block b
    const uint8_t *akeys;        // [m][32]
    const uint8_t *accts;        // [m] b200_account rows
    const uint8_t *aflags;       // [m] or null (all plain upserts)
    const uint64_t *seg;         // [m + 1] slot entries of account entry a
    const uint8_t *skeys, *svals;  // [n_e][32]
    uint64_t n_blocks, m, n_e;
    uint32_t *status;            // [n_blocks] SL_INCOMPLETE | SL_INVALID
    // overlay multiproof (one block): the proof targets, which the reveal follows as well as the entries
    const uint8_t *tkeys;        // [n_t][32] account targets, ascending
    const uint64_t *tseg;        // [n_t + 1] slot targets of account target i
    const uint8_t *tskeys;       // [tseg[n_t]][32]
    uint64_t n_t;
    int reveal_targets;          // overlay witness: an entry whose key is an account target also reveals its storage without slots
    int bucket_tries;            // overlay frontiers: the account arena holds 16 top-nibble bucket tries, each block lies in one
};
struct SlNode {  // a queued node: trie, path (packed nibbles, zero-padded) and depth, RLP at rlp[off, off + len)
    uint8_t path[32];
    uint64_t off;
    uint32_t len, trie, block, depth;
};
struct SlItem {  // leaf (nib 64, value RLP at rlp[off, off + len); len 0: an inserted entry) or blind child (hash at rlp[off])
    uint8_t key[32];
    uint64_t off;
    uint32_t len, trie, block, entry;  // entry: the slot / account entry that updates or inserts it, or SL_NONE
    uint8_t nib, kind;
    uint8_t tree;  // a hash item whose branch is stored (children_are_in_trie: its parent's tree-mask bit); 0 otherwise
    uint8_t pad[5];
};
cudaError_t launch_sl_seed(const StatelessDev &s, SlNode *q, uint32_t *n_q, cudaStream_t st);
cudaError_t launch_sl_reveal(const StatelessDev &s, const SlNode *q, uint32_t nq, SlNode *next, uint32_t *n_next, SlItem *items,
                             uint32_t *n_items, cudaStream_t st);
cudaError_t launch_sl_sort_key(const SlItem *items, const uint32_t *perm, uint64_t n, int w, uint64_t *keys, uint32_t *idx,
                               cudaStream_t st);
cudaError_t launch_sl_gather(const SlItem *items, const uint32_t *perm, uint64_t n, SlItem *out, cudaStream_t st);
cudaError_t launch_sl_merge(const StatelessDev &s, SlItem *items, uint64_t n_it, uint32_t *dead, uint32_t *ins, uint32_t *lb,
                            uint32_t *eblock, cudaStream_t st);
cudaError_t launch_sl_keep(const StatelessDev &s, const SlItem *items, uint64_t n_it, uint32_t *keep, const uint32_t *eblock,
                           uint32_t *ins, cudaStream_t st);
cudaError_t launch_sl_totals(const StatelessDev &s, const SlItem *items, uint64_t n_it, const uint32_t *kscan, const uint32_t *iscan,
                             uint64_t *totals, cudaStream_t st);
cudaError_t launch_sl_place(const StatelessDev &s, const SlItem *items, uint64_t n_it, const uint32_t *keep, const uint32_t *kscan,
                            const uint32_t *ins, const uint32_t *iscan, const uint32_t *lb, const uint32_t *eblock, SlItem *fin,
                            cudaStream_t st);
cudaError_t launch_sl_segments(const StatelessDev &s, const SlItem *fin, uint64_t n_fin, uint64_t n_sto, uint64_t *sto_offs,
                               uint64_t *acc_offs, cudaStream_t st);
cudaError_t launch_sl_sufficiency(const StatelessDev &s, const SlItem *fin, uint64_t n_fin, cudaStream_t st);
cudaError_t launch_sl_rows(const StatelessDev &s, const SlItem *fin, uint64_t lo, uint64_t hi, uint8_t *keys, uint8_t *nibs,
                           uint8_t *flags, uint8_t *values, uint8_t *sroots, const uint8_t *sto_roots, cudaStream_t st);
cudaError_t launch_sl_finish(const StatelessDev &s, const uint8_t *acc_roots, uint8_t *out, cudaStream_t st);

// ------------------------------------------------------------------------------------------------ overlay roots (tk_overlay.cuh)
struct OvNode {  // a queued branch of an arena: trie id of the call, block, the entries [lo, hi) and the proof targets [tlo, thi)
                 // that pass through it
    uint32_t node, trie, block, lo, hi, tlo, thi;
};
constexpr uint32_t OV_STRIDE = 112;  // value bytes of item i at OV_STRIDE * i: rlp(TrieAccount) (<= 110), rlp(U256) (<= 33), a hash
// Removed-node candidates of an overlay with TrieUpdates: (trie id of the call, arena node) of every stored branch that the
// reveal queues, account tries and storage tries apart; null lists: none are kept (the root-only call).
struct OvRemoved {
    uint32_t *acc, *sto;      // [2][..] pairs
    uint32_t *n_acc, *n_sto;  // counts
};
cudaError_t launch_ov_seed(const DTrieDev &ta, const DTrieDev &ts, const StatelessDev &s, const uint8_t *root, uint8_t *parent, OvNode *q,
                           uint32_t *n_q, SlItem *items, uint32_t *n_items, uint8_t *vals, uint8_t *found, cudaStream_t st);
cudaError_t launch_ov_reveal(const DTrieDev &ta, const DTrieDev &ts, const StatelessDev &s, const OvNode *q, uint32_t nq, OvNode *next,
                             uint32_t *n_next, SlItem *items, uint32_t *n_items, uint8_t *vals, OvRemoved rm, cudaStream_t st);
cudaError_t launch_ov_removed_paths(const DTrieDev &t, const uint32_t *cand, uint32_t n, uint32_t trie_base, uint8_t *path_len,
                                    uint8_t *path_packed, uint32_t *trie_id, cudaStream_t st);
// b200_dstate_overlay_frontiers: the n = 16 x blocks entries from the account fold f (segments seg, rows values / sroots /
// nibs) and the current frontier cur; vblock[i]: the segment of entry i, or -1 (cur[i % 16])
cudaError_t launch_ov_frontier(const ForestDev &f, const uint64_t *seg, const int32_t *vblock, uint64_t n, const uint8_t *values,
                               const uint8_t *sroots, const uint8_t *nibs, const FrontierEntryDev *cur, FrontierEntryDev *out,
                               cudaStream_t st);

cudaError_t launch_dt_restructure_fused(const DTrieDev &t, const uint32_t *trie_of_key, const uint8_t *keys, const uint8_t *vals,
                                        const uint8_t *flags, const uint8_t *sroots, uint32_t m, uint8_t *kind, uint32_t *leaf_of,
                                        uint32_t *list_a, uint32_t *list_b, uint8_t *defer, uint32_t *idx_a, uint32_t *idx_b,
                                        uint64_t *attach, uint8_t *pending, uint32_t max_per_run, cudaStream_t st);

}  // namespace b200
