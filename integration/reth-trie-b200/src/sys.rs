//! Raw bindings of include/b200trie.h (hand-written; `bindgen` over the header gives the same).
//! UNCOMPILED SKETCH — see Cargo.toml.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_void};

#[repr(C)]
pub struct b200_ctx {
    _p: [u8; 0],
}
#[repr(C)]
pub struct b200_trie {
    _p: [u8; 0],
}
#[repr(C)]
pub struct b200_dtrie {
    _p: [u8; 0],
}
#[repr(C)]
pub struct b200_dstate {
    _p: [u8; 0],
}
#[repr(C)]
#[derive(Clone, Copy)]
pub struct b200_frontier_entry {
    pub as_child_len: u8,
    pub as_child: [u8; 33],
    pub as_root_len: u8,
    pub as_root: [u8; 33],
}

#[repr(C)]
#[derive(Clone, Copy)]
pub struct b200_account {
    pub nonce: u64,
    pub balance_be: [u8; 32],
    pub code_hash: [u8; 32],
}

#[repr(C)]
pub struct b200_updates {
    pub n_nodes: u64,
    pub trie_id: *mut u32,
    pub path_len: *mut u8,
    pub path_packed: *mut u8,
    pub state_mask: *mut u16,
    pub tree_mask: *mut u16,
    pub hash_mask: *mut u16,
    pub hash_offset: *mut u64,
    pub hashes: *mut u8,
    pub _owner: *mut c_void,
}

#[repr(C)]
#[derive(Default, Clone, Copy)]
pub struct b200_stats {
    pub leaves_added: u64,
    pub branches_added: u64,
    pub extension_nodes: u64,
    pub hashed_nodes: u64,
    pub levels: u64,
    pub device_ms: f64,
    pub keccak_f: u64,
}

#[repr(C)]
pub struct b200_rows {
    pub n_rows: u64,
    pub row_offset: *mut u64,
    pub key_len: *mut u32,
    pub bytes: *mut u8,
    pub _owner: *mut c_void,
}
pub const B200_KEYS_LEGACY: i32 = 0;
pub const B200_KEYS_PACKED: i32 = 1;

// ---- round-2 entry points (include/b200trie.h): stream, items, changesets, communicator, multiproof
#[repr(C)] pub struct b200_root_stream { _p: [u8; 0] }
#[repr(C)] pub struct b200_comm { _p: [u8; 0] }
#[repr(C)] #[derive(Default, Clone, Copy)]
pub struct b200_stream_progress { pub accounts: u64, pub slots: u64, pub open_accounts: u64, pub closed_buckets: u32 }
#[repr(C)] #[derive(Clone, Copy)]
pub struct b200_stream_checkpoint {
    pub frontier: [b200_frontier_entry; 16], pub closed_mask: u32, pub resume_nibble: u32, pub retain_updates: u32, pub _reserved: u32,
}
#[repr(C)]
pub struct b200_changeset_hashes {
    pub n_accounts: u64, pub account_keys32: *mut u8, pub account_first: *mut u32,
    pub n_storage_accounts: u64, pub storage_account_keys32: *mut u8, pub storage_seg_offsets: *mut u64,
    pub n_slots: u64, pub slot_keys32: *mut u8, pub slot_first: *mut u32,
    pub n_prefix: u64, pub account_prefix_keys32: *mut u8, pub _owner: *mut c_void,
}
#[repr(C)]
pub struct b200_proofs {
    pub n_targets: u64, pub node_offset: *mut u64, pub n_nodes: u64, pub rlp_offset: *mut u64, pub rlp: *mut u8,
    pub node_depth: *mut u8, pub node_masks: *mut u32, pub _owner: *mut c_void,
}
#[repr(C)]
pub struct b200_witness {
    pub n: u64, pub hashes32: *mut u8, pub rlp_offset: *mut u64, pub rlp: *mut u8, pub _owner: *mut c_void,
}
pub const B200_WITNESS_LEGACY: i32 = 0;
pub const B200_WITNESS_CANONICAL: i32 = 1;
pub const B200_COMM_ID_BYTES: usize = 128;

pub const B200_OK: i32 = 0;
pub const B200_ERR_NOT_FOUND: i32 = -8;

#[link(name = "b200trie")]
unsafe extern "C" {
    pub fn b200_create(device_ordinal: i32) -> *mut b200_ctx;
    pub fn b200_create_status() -> i32;
    pub fn b200_destroy(ctx: *mut b200_ctx);
    pub fn b200_last_error(ctx: *const b200_ctx) -> *const c_char;

    pub fn b200_keccak256_fixed(ctx: *mut b200_ctx, input: *const u8, msg_len: u32, stride: u32, n: u64, out32: *mut u8) -> i32;
    pub fn b200_hash_sort_keys(ctx: *mut b200_ctx, input: *const u8, msg_len: u32, stride: u32, n: u64,
                               out_sorted32: *mut u8, out_perm: *mut u32) -> i32;
    pub fn b200_hash_sort_storage_dev(ctx: *mut b200_ctx, d_addresses20: *const c_void, n_addr: u32, d_addr_index: *const c_void,
                                      d_slots32: *const c_void, n: u64, d_sorted64: *mut c_void, d_perm: *mut c_void) -> i32;
    pub fn b200_hash_sort_storage(ctx: *mut b200_ctx, addresses20: *const u8, n_addr: u32, addr_index: *const u32,
                                  slots32: *const u8, n: u64, out_sorted64: *mut u8, out_perm: *mut u32) -> i32;

    pub fn b200_storage_roots(ctx: *mut b200_ctx, slot_keys32: *const u8, values32_be: *const u8, seg_offsets: *const u64,
                              n_accounts: u64, roots32: *mut u8, updates: *mut b200_updates, stats: *mut b200_stats) -> i32;
    pub fn b200_state_root_full(ctx: *mut b200_ctx, acct_keys32: *const u8, accts: *const b200_account, n_accounts: u64,
                                slot_keys32: *const u8, values32_be: *const u8, seg_offsets: *const u64, root32: *mut u8,
                                account_updates: *mut b200_updates, storage_updates: *mut b200_updates,
                                stats: *mut b200_stats) -> i32;
    pub fn b200_updates_release(u: *mut b200_updates);
    pub fn b200_account_trie_rows(account_updates: *const b200_updates, key_format: i32, out: *mut b200_rows) -> i32;
    pub fn b200_storage_trie_rows(storage_updates: *const b200_updates, acct_keys32: *const u8, n_accounts: u64,
                                  key_format: i32, out: *mut b200_rows) -> i32;
    pub fn b200_rows_release(rows: *mut b200_rows);

    pub fn b200_trie_create(ctx: *mut b200_ctx, acct_keys32: *const u8, accts: *const b200_account,
                            storage_roots32: *const u8, n: u64, out: *mut *mut b200_trie, root32: *mut u8) -> i32;
    pub fn b200_trie_apply(trie: *mut b200_trie, keys32: *const u8, accts: *const b200_account, present: *const u8,
                           storage_roots32: *const u8, m: u64, root32: *mut u8, out_rebuilt: *mut i32,
                           updates: *mut b200_updates, stats: *mut b200_stats) -> i32;
    pub fn b200_trie_destroy(trie: *mut b200_trie);

    // dynamic resident trie / state (emulation-validated; include/b200trie.h)
    pub fn b200_dtrie_create(ctx: *mut b200_ctx, acct_keys32: *const u8, accts: *const b200_account, storage_roots32: *const u8,
                             n: u64, out: *mut *mut b200_dtrie, root32: *mut u8) -> i32;
    pub fn b200_dtrie_apply(trie: *mut b200_dtrie, keys32: *const u8, accts: *const b200_account, present: *const u8,
                            storage_roots32: *const u8, m: u64, root32: *mut u8, updated: *mut b200_updates,
                            removed: *mut b200_updates, stats: *mut b200_stats) -> i32;
    pub fn b200_dtrie_destroy(trie: *mut b200_dtrie);
    pub fn b200_dstate_create(ctx: *mut b200_ctx, acct_keys32: *const u8, accts: *const b200_account, n_accounts: u64,
                              slot_keys32: *const u8, values32_be: *const u8, seg_offsets: *const u64,
                              out: *mut *mut b200_dstate, root32: *mut u8) -> i32;
    pub fn b200_dstate_create_sharded(ctx: *mut b200_ctx, acct_keys32: *const u8, accts: *const b200_account, n_accounts: u64,
                                      slot_keys32: *const u8, values32_be: *const u8, seg_offsets: *const u64,
                                      out: *mut *mut b200_dstate, root32: *mut u8) -> i32;
    pub fn b200_dstate_apply(state: *mut b200_dstate, acct_keys32: *const u8, accts: *const b200_account, acct_flags: *const u8,
                             m: u64, slot_keys32: *const u8, values32_be: *const u8, seg_offsets: *const u64, root32: *mut u8,
                             acct_updated: *mut b200_updates, acct_removed: *mut b200_updates,
                             storage_updated: *mut b200_updates, storage_removed: *mut b200_updates,
                             storage_deleted: *mut u8, stats: *mut b200_stats) -> i32;
    pub fn b200_dstate_frontier(state: *mut b200_dstate, out16: *mut b200_frontier_entry) -> i32;
    /// the frontier entries of a sharded state after each sibling block (out: [n_blocks][16]), the state unchanged; the ranks
    /// all-gather them and b200_root_from_frontier gives each block's root (payload validation over a sharded state)
    pub fn b200_dstate_overlay_frontiers(state: *mut b200_dstate, n_blocks: u64, acct_keys32: *const u8, accts: *const b200_account,
                                         acct_flags: *const u8, block_acct_offset: *const u64, slot_keys32: *const u8,
                                         values32_be: *const u8, seg_offsets: *const u64, out: *mut b200_frontier_entry,
                                         stats: *mut b200_stats) -> i32;
    pub fn b200_root_from_frontier(ctx: *mut b200_ctx, frontier16: *const b200_frontier_entry, root32: *mut u8) -> i32;
    pub fn b200_dstate_destroy(state: *mut b200_dstate);
    /// transactions / receipts / withdrawals roots of a batch of lists (ordered_root.rs:240-257 per list)
    pub fn b200_ordered_roots(ctx: *mut b200_ctx, values: *const u8, value_offsets: *const u64, seg_offsets: *const u64,
                              n_lists: u64, roots32: *mut u8, opt_stats: *mut b200_stats) -> i32;

    /// StateRoot::with_threshold / root_with_progress / with_intermediate_state; MerkleStage's chunked rebuild + MerkleCheckpoint
    pub fn b200_root_stream_begin(ctx: *mut b200_ctx, retain_updates: i32, out: *mut *mut b200_root_stream) -> i32;
    pub fn b200_root_stream_push(s: *mut b200_root_stream, acct_keys32: *const u8, accts: *const b200_account, n_accounts: u64,
                                 slot_keys32: *const u8, values32_be: *const u8, seg_offsets: *const u64,
                                 account_updates: *mut b200_updates, storage_updates: *mut b200_updates,
                                 progress: *mut b200_stream_progress) -> i32;
    pub fn b200_root_stream_finish(s: *mut b200_root_stream, root32: *mut u8, account_updates: *mut b200_updates) -> i32;
    pub fn b200_root_stream_checkpoint(s: *const b200_root_stream, out: *mut b200_stream_checkpoint) -> i32;
    pub fn b200_root_stream_resume(ctx: *mut b200_ctx, cp: *const b200_stream_checkpoint, out: *mut *mut b200_root_stream) -> i32;
    pub fn b200_root_stream_free(s: *mut b200_root_stream);
    /// the fold of TrieNodeIter's element stream: HashBuilder::add_leaf / add_branch (trie.rs:247-309,659-698)
    pub fn b200_root_from_items(ctx: *mut b200_ctx, keys32: *const u8, key_nibbles: *const u8, item_flags: *const u8,
                                values: *const u8, storage_roots32: *const u8, seg_offsets: *const u64, n_segs: u64,
                                n_items: u64, account: i32, roots32: *mut u8, updates: *mut b200_updates, stats: *mut b200_stats) -> i32;
    /// HashedPostStateSorted::from_reverts + load_prefix_sets_with_provider over the changesets of a block range
    pub fn b200_hash_changesets(ctx: *mut b200_ctx, acct_addresses20: *const u8, n_acct: u64, storage_addresses20: *const u8,
                                storage_slots32: *const u8, n_storage: u64, out: *mut b200_changeset_hashes) -> i32;
    pub fn b200_changeset_hashes_release(o: *mut b200_changeset_hashes);
    /// the two exchange steps of the path (NCCL behind the C ABI)
    pub fn b200_comm_unique_id(id: *mut u8) -> i32;
    pub fn b200_comm_create(ctx: *mut b200_ctx, id: *const u8, n_ranks: i32, rank: i32, out: *mut *mut b200_comm) -> i32;
    pub fn b200_comm_destroy(comm: *mut b200_comm);
    pub fn b200_state_root_sharded(comm: *mut b200_comm, acct_keys32: *const u8, accts: *const b200_account, n_accounts: u64,
                                   slot_keys32: *const u8, values32_be: *const u8, seg_offsets: *const u64, root32: *mut u8,
                                   stats: *mut b200_stats) -> i32;
    pub fn b200_dstate_root_sharded(comm: *mut b200_comm, state: *mut b200_dstate, root32: *mut u8) -> i32;
    pub fn b200_hash_partition_dev(comm: *mut b200_comm, d_in: *const c_void, msg_len: u32, stride: u32, n: u64,
                                   d_values: *const c_void, value_bytes: u32, capacity: u64, d_sorted_keys32: *mut c_void,
                                   d_sorted_values: *mut c_void, n_out: *mut u64) -> i32;
    /// Proof::multiproof(MultiProofTargets) from the resident state
    pub fn b200_dstate_multiproof(state: *mut b200_dstate, acct_keys32: *const u8, n_accounts: u64, slot_seg_offsets: *const u64,
                                  slot_keys32: *const u8, account_proofs: *mut b200_proofs, storage_roots32: *mut u8,
                                  storage_proofs: *mut b200_proofs) -> i32;
    pub fn b200_proofs_release(p: *mut b200_proofs);
    /// the bits this shard's buckets set in the hash / tree masks of the depth-0 root branch; the ranks OR them
    pub fn b200_dstate_frontier_masks(state: *mut b200_dstate, hash_mask: *mut u16, tree_mask: *mut u16) -> i32;
    /// b200_dstate_multiproof on one shard, from the gathered frontier (merged16) and the ORed root masks
    pub fn b200_dstate_sharded_multiproof(state: *mut b200_dstate, merged16: *const b200_frontier_entry, root_hash_mask: u16,
                                          root_tree_mask: u16, acct_keys32: *const u8, n_accounts: u64, slot_seg_offsets: *const u64,
                                          slot_keys32: *const u8, account_proofs: *mut b200_proofs, storage_roots32: *mut u8,
                                          storage_proofs: *mut b200_proofs) -> i32;
    /// multiproof of the state after one candidate block (layout of b200_dstate_apply), the state unchanged
    pub fn b200_dstate_overlay_multiproof(state: *mut b200_dstate, acct_keys32: *const u8, accts: *const b200_account,
                                          acct_flags: *const u8, m: u64, slot_keys32: *const u8, values32_be: *const u8,
                                          seg_offsets: *const u64, target_keys32: *const u8, n_targets: u64,
                                          target_slot_offsets: *const u64, target_slot_keys32: *const u8, root32: *mut u8,
                                          account_proofs: *mut b200_proofs, storage_roots32: *mut u8,
                                          storage_proofs: *mut b200_proofs, opt_stats: *mut b200_stats) -> i32;
    /// execution witness of a target block on the state after an overlay block (both in the layout of b200_dstate_apply),
    /// the state unchanged
    pub fn b200_dstate_overlay_witness(state: *mut b200_dstate, ov_acct_keys32: *const u8, ov_accts: *const b200_account,
                                       ov_acct_flags: *const u8, ov_m: u64, ov_slot_keys32: *const u8, ov_values32_be: *const u8,
                                       ov_seg_offsets: *const u64, acct_keys32: *const u8, accts: *const b200_account,
                                       acct_flags: *const u8, m: u64, slot_keys32: *const u8, values32_be: *const u8,
                                       seg_offsets: *const u64, mode: i32, always_include_root: i32, overlay_root32: *mut u8,
                                       out: *mut b200_witness, opt_stats: *mut b200_stats) -> i32;
    /// trie changesets (compute_trie_changesets) of a block's TrieUpdatesSorted paths against the state, which is unchanged
    pub fn b200_dstate_trie_changesets(state: *mut b200_dstate, acct_path_len: *const u8, acct_path_packed: *const u8,
                                       n_acct_paths: u64, storage_keys32: *const u8, storage_flags: *const u8,
                                       n_storage_tries: u64, storage_path_offsets: *const u64, storage_path_len: *const u8,
                                       storage_path_packed: *const u8, account_out: *mut b200_updates,
                                       storage_out: *mut b200_updates, opt_stats: *mut b200_stats) -> i32;
    pub fn b200_witness_release(w: *mut b200_witness);
    /// this shard's kept mask for its part of a block (the entries of its own buckets): bit k = bucket k still holds a
    /// leaf after the mode's removal phase; the ranks OR the masks for b200_dstate_sharded_witness
    pub fn b200_dstate_witness_root_kept(state: *mut b200_dstate, acct_keys32: *const u8, accts: *const b200_account,
                                         acct_flags: *const u8, m: u64, slot_keys32: *const u8, values32_be: *const u8,
                                         seg_offsets: *const u64, mode: i32, kept: *mut u16) -> i32;
    /// b200_dstate_witness of one shard's part of a block, from the gathered frontier (merged16), the ORed root masks and
    /// the ORed kept masks; the union of the ranks' maps is the unsharded witness
    pub fn b200_dstate_sharded_witness(state: *mut b200_dstate, merged16: *const b200_frontier_entry, root_hash_mask: u16,
                                       root_tree_mask: u16, root_kept: u16, acct_keys32: *const u8, accts: *const b200_account,
                                       acct_flags: *const u8, m: u64, slot_keys32: *const u8, values32_be: *const u8,
                                       seg_offsets: *const u64, mode: i32, always_include_root: i32, out: *mut b200_witness,
                                       opt_stats: *mut b200_stats) -> i32;
    /// CPUs + preferred memory of the calling thread on the GPU's NUMA node (before allocating staging buffers)
    pub fn b200_numa_bind_thread(device_ordinal: i32) -> i32;
}
