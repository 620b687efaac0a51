//! reth-trie-b200 — routes reth's state-commitment seams to the GPU engine (libb200trie.so).
//!
//! UNCOMPILED SKETCH (no Rust toolchain in the build image).  Seams (SURVEY.md §8b):
//!   * `CustomStateRoot` closure   crates/engine/tree/src/tree/payload_validator.rs:2291-2310
//!   * `StateRoot`-shaped wrapper  crates/trie/trie/src/trie.rs:54-158
//!   * replacement stages          crates/stages/api/src/stage.rs:241-300 (see INTEGRATION.md §3)
pub mod sys;

use alloy_primitives::{keccak256, map::B256Map, B256, U256};
use alloy_trie::{BranchNodeCompact, Nibbles, TrieMask, EMPTY_ROOT_HASH, KECCAK_EMPTY};
use reth_storage_errors::{db::DatabaseError, provider::{ProviderError, ProviderResult}};
use reth_trie_common::{updates::{StorageTrieUpdates, TrieUpdates}, HashedPostStateSorted};
use std::{ffi::CStr, sync::Arc};

/// Owning handle on a `b200_ctx` (one per GPU; internally locked, so it is `Send + Sync`).
pub struct B200Handle(*mut sys::b200_ctx);
unsafe impl Send for B200Handle {}
unsafe impl Sync for B200Handle {}

impl B200Handle {
    pub fn new(device: i32) -> ProviderResult<Self> {
        let p = unsafe { sys::b200_create(device) };
        if p.is_null() {
            // no CPU fallback exists on purpose: the caller decides (e.g. fall back to reth's own StateRoot)
            return Err(other(format!("b200_create({device}) failed, status {}", unsafe { sys::b200_create_status() })));
        }
        Ok(Self(p))
    }
    pub fn raw(&self) -> *mut sys::b200_ctx { self.0 }
    pub fn last_error(&self) -> String {
        unsafe { CStr::from_ptr(sys::b200_last_error(self.0)) }.to_string_lossy().into_owned()
    }
    fn check(&self, rc: i32) -> ProviderResult<()> {
        if rc == sys::B200_OK { Ok(()) } else { Err(other(format!("b200 status {rc}: {}", self.last_error()))) }
    }
}
impl Drop for B200Handle {
    fn drop(&mut self) { unsafe { sys::b200_destroy(self.0) } }
}

/// Same convention the reference uses for internal failures (crates/trie/parallel/src/root.rs:153-158).
fn other(msg: String) -> ProviderError { ProviderError::Database(DatabaseError::Other(msg)) }

/// `HashedPostStateSorted` flattened into the layout of include/b200trie.h.
#[derive(Default)]
pub struct FlatState {
    pub acct_keys: Vec<u8>,                 // n x 32
    pub accts: Vec<sys::b200_account>,      // n
    pub slot_keys: Vec<u8>,                 // m x 32
    pub slot_values: Vec<u8>,               // m x 32, big-endian
    pub seg_offsets: Vec<u64>,              // n + 1
}

impl FlatState {
    /// Destroyed accounts (`None`) and zero-valued slots are dropped exactly where the reference's cursors skip them
    /// (crates/trie/trie/src/hashed_cursor/post_state.rs:260-297).
    pub fn from_sorted(state: &HashedPostStateSorted) -> Self {
        let mut f = Self { seg_offsets: vec![0], ..Default::default() };
        for (hashed_address, account) in state.accounts() {
            let Some(account) = account else { continue };
            f.acct_keys.extend_from_slice(hashed_address.as_slice());
            f.accts.push(sys::b200_account {
                nonce: account.nonce,
                balance_be: account.balance.to_be_bytes(),
                code_hash: account.bytecode_hash.unwrap_or(KECCAK_EMPTY).0, // account.rs:16-31
            });
            let mut count = 0u64;
            if let Some(storage) = state.account_storages().get(hashed_address) {
                for (slot, value) in storage.storage_slots_ref() {
                    if value.is_zero() { continue }
                    f.slot_keys.extend_from_slice(slot.as_slice());
                    f.slot_values.extend_from_slice(&value.to_be_bytes::<32>());
                    count += 1;
                }
            }
            f.seg_offsets.push(f.seg_offsets.last().unwrap() + count);
        }
        f
    }
    pub fn n_accounts(&self) -> u64 { self.accts.len() as u64 }
    pub fn account_key(&self, i: u32) -> B256 { B256::from_slice(&self.acct_keys[32 * i as usize..32 * i as usize + 32]) }
}

fn branch_node(u: &sys::b200_updates, i: usize) -> (Nibbles, BranchNodeCompact) {
    unsafe {
        let len = *u.path_len.add(i) as usize;
        let packed = std::slice::from_raw_parts(u.path_packed.add(32 * i), 32);
        let path = Nibbles::unpack(packed).slice(..len);
        let (lo, hi) = (*u.hash_offset.add(i) as usize, *u.hash_offset.add(i + 1) as usize);
        let hashes = (lo..hi).map(|h| B256::from_slice(std::slice::from_raw_parts(u.hashes.add(32 * h), 32))).collect();
        (path, BranchNodeCompact::new(TrieMask::new(*u.state_mask.add(i)), TrieMask::new(*u.tree_mask.add(i)),
                                      TrieMask::new(*u.hash_mask.add(i)), hashes, None))
    }
}

/// `TrieUpdates` as `StateRoot::root_with_updates` returns them (crates/trie/common/src/updates.rs:17-26,140-158).
fn trie_updates_from(flat: &FlatState, mut au: sys::b200_updates, mut su: sys::b200_updates) -> TrieUpdates {
    let mut out = TrieUpdates::default();
    for i in 0..au.n_nodes as usize {
        let (path, node) = branch_node(&au, i);
        out.account_nodes.insert(path, node);
    }
    let mut per_trie: B256Map<StorageTrieUpdates> = Default::default();
    for i in 0..su.n_nodes as usize {
        let (path, node) = branch_node(&su, i);
        let addr = flat.account_key(unsafe { *su.trie_id.add(i) });
        per_trie.entry(addr).or_default().storage_nodes.insert(path, node);
    }
    for a in 0..flat.n_accounts() as usize {
        let addr = flat.account_key(a as u32);
        if flat.seg_offsets[a + 1] == flat.seg_offsets[a] {
            out.insert_storage_updates(addr, StorageTrieUpdates::deleted()); // trie.rs:622-629
        } else if let Some(u) = per_trie.remove(&addr) {
            out.insert_storage_updates(addr, u);
        }
    }
    unsafe {
        sys::b200_updates_release(&mut au);
        sys::b200_updates_release(&mut su);
    }
    out
}

/// `StateRoot::root_with_updates` over a complete hashed state (MerkleStage rebuild, `StateRootProvider::state_root`).
pub fn state_root_with_updates(ctx: &B200Handle, state: &HashedPostStateSorted) -> ProviderResult<(B256, TrieUpdates)> {
    let flat = FlatState::from_sorted(state);
    let mut root = B256::ZERO;
    let (mut au, mut su): (sys::b200_updates, sys::b200_updates) = unsafe { (std::mem::zeroed(), std::mem::zeroed()) };
    ctx.check(unsafe {
        sys::b200_state_root_full(ctx.raw(), flat.acct_keys.as_ptr(), flat.accts.as_ptr(), flat.n_accounts(),
                                  flat.slot_keys.as_ptr(), flat.slot_values.as_ptr(), flat.seg_offsets.as_ptr(),
                                  root.as_mut_ptr(), &mut au, &mut su, std::ptr::null_mut())
    })?;
    Ok((root, trie_updates_from(&flat, au, su)))
}

/// The `CustomStateRoot` closure (payload_validator.rs:2291-2310; template: examples/custom-state-root/src/main.rs:45-112).
/// `merged_state(input)` must yield the parent state overlaid with the block's `HashedPostStateSorted`, exactly what
/// `compute_state_root_parallel` builds its cursors over (payload_validator.rs:1264-1280); with a resident trie
/// (`b200_trie_apply`, INTEGRATION.md §5b) only the block's dirty set is needed instead.
pub fn custom_state_root<N, F>(ctx: Arc<B200Handle>, merged_state: F)
    -> Arc<dyn Fn(reth_engine_tree::tree::CustomStateRootInput<'_, N>) -> ProviderResult<(B256, TrieUpdates)> + Send + Sync>
where
    F: Fn(&reth_engine_tree::tree::CustomStateRootInput<'_, N>) -> ProviderResult<HashedPostStateSorted> + Send + Sync + 'static,
    N: 'static,
{
    Arc::new(move |input| {
        let state = merged_state(&input)?;
        state_root_with_updates(&ctx, &state)
    })
}

/// Batched `KeccakKeyHasher` (crates/trie/common/src/key.rs:4-18): n keys of `LEN` bytes in, n digests out.
pub fn hash_keys<const LEN: usize>(ctx: &B200Handle, keys: &[[u8; LEN]]) -> ProviderResult<Vec<B256>> {
    let mut out = vec![B256::ZERO; keys.len()];
    ctx.check(unsafe {
        sys::b200_keccak256_fixed(ctx.raw(), keys.as_ptr().cast(), LEN as u32, LEN as u32, keys.len() as u64,
                                  out.as_mut_ptr().cast())
    })?;
    debug_assert!(keys.is_empty() || out[0] == keccak256(keys[0]));
    let _ = (EMPTY_ROOT_HASH, U256::ZERO);
    Ok(out)
}

/// `proofs::calculate_transaction_root` for every block of a batch in one device call (INTEGRATION.md §5d): the encoder
/// is the one `ordered_trie_root_with_encoder` is given — `encode_2718` — so the trie sees the same bytes.
pub fn transaction_roots<T: alloy_eips::eip2718::Encodable2718>(ctx: &B200Handle, blocks: &[&[T]]) -> ProviderResult<Vec<B256>> {
    let (mut blob, mut offs, mut segs) = (Vec::<u8>::new(), vec![0u64], vec![0u64]);
    for txs in blocks {
        for tx in txs.iter() {
            tx.encode_2718(&mut blob);
            offs.push(blob.len() as u64);
        }
        segs.push(offs.len() as u64 - 1);
    }
    let mut roots = vec![B256::ZERO; blocks.len()];
    ctx.check(unsafe {
        sys::b200_ordered_roots(ctx.raw(), blob.as_ptr(), offs.as_ptr(), segs.as_ptr(), blocks.len() as u64,
                                roots.as_mut_ptr().cast(), std::ptr::null_mut())
    })?;
    Ok(roots)
}
