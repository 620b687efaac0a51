"""Host-side mirror of reth's root calculators (crates/trie/trie/src/trie.rs, crates/trie/parallel/src/root.rs,
crates/trie/common/src/updates.rs) over the C ABI.

The calculators take the hashed state itself where reth takes cursor factories over it: with no stored trie nodes
underneath (from-scratch build: MerkleStage's rebuild path `merkle.rs:210-254`, `StateRootProvider::state_root`
on a full state, every test that uses `MockHashedCursorFactory` + `NoopTrieCursor`) the walk degenerates to
"stream all leaves in key order" (SURVEY.md §3.2), which is what the device consumes.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from ._lib import ERR_WITNESS_INCOMPLETE
from .engine import EMPTY_ROOT_HASH, Engine
from .hashed_state import HashedPostStateSorted, HashedStorageSorted, TriePrefixSets

B256 = bytes
Nibbles = bytes


@dataclass(frozen=True)
class BranchNodeCompact:
    """alloy_trie::BranchNodeCompact as reth stores it (crates/storage/db-api/src/tables/mod.rs:484-494)."""
    state_mask: int
    tree_mask: int
    hash_mask: int
    hashes: Tuple[bytes, ...]
    root_hash: Optional[bytes] = None


@dataclass
class StorageTrieUpdates:
    """crates/trie/common/src/updates.rs:235-245."""
    is_deleted: bool = False
    storage_nodes: Dict[Nibbles, BranchNodeCompact] = field(default_factory=dict)
    removed_nodes: set = field(default_factory=set)

    @classmethod
    def deleted(cls):
        return cls(is_deleted=True)

    def is_empty(self) -> bool:
        return not self.is_deleted and not self.storage_nodes and not self.removed_nodes

    def __len__(self):
        return int(self.is_deleted) + len(self.storage_nodes) + len(self.removed_nodes)

    def into_sorted(self) -> "StorageTrieUpdatesSorted":
        """updates.rs:364-379: updated nodes, then the removed paths that are not updated as None, sorted by path."""
        nodes = [(p, n) for p, n in self.storage_nodes.items()]
        nodes += [(p, None) for p in self.removed_nodes if p not in self.storage_nodes]
        nodes.sort(key=lambda e: e[0])
        return StorageTrieUpdatesSorted(self.is_deleted, nodes)


@dataclass
class StorageTrieUpdatesSorted:
    """crates/trie/common/src/updates.rs:759-765: (path, Some(node) | None) sorted by path."""
    is_deleted: bool = False
    storage_nodes: List[Tuple[Nibbles, Optional[BranchNodeCompact]]] = field(default_factory=list)

    def is_empty(self) -> bool:
        return not self.is_deleted and not self.storage_nodes


@dataclass
class TrieUpdatesSorted:
    """crates/trie/common/src/updates.rs:550-556: account (path, Some(node) | None) sorted by path, and the sorted updates
    of every storage trie by hashed address."""
    account_nodes: List[Tuple[Nibbles, Optional[BranchNodeCompact]]] = field(default_factory=list)
    storage_tries: Dict[B256, StorageTrieUpdatesSorted] = field(default_factory=dict)


@dataclass
class TrieUpdates:
    """crates/trie/common/src/updates.rs:17-26."""
    account_nodes: Dict[Nibbles, BranchNodeCompact] = field(default_factory=dict)
    removed_nodes: set = field(default_factory=set)
    storage_tries: Dict[B256, StorageTrieUpdates] = field(default_factory=dict)

    def insert_storage_updates(self, hashed_address: B256, updates: StorageTrieUpdates):
        if updates.is_empty():  # updates.rs:132-134
            return
        assert hashed_address not in self.storage_tries
        self.storage_tries[hashed_address] = updates

    def is_empty(self) -> bool:
        return not self.account_nodes and not self.removed_nodes and not self.storage_tries

    def into_sorted(self) -> TrieUpdatesSorted:
        """updates.rs:160-180: updated takes precedence over removed, then every list is sorted by path."""
        nodes = [(p, n) for p, n in self.account_nodes.items()]
        nodes += [(p, None) for p in self.removed_nodes if p not in self.account_nodes]
        nodes.sort(key=lambda e: e[0])
        return TrieUpdatesSorted(nodes, {k: v.into_sorted() for k, v in self.storage_tries.items()})


@dataclass
class IntermediateStateRootState:
    """crates/trie/trie/src/progress.rs:24-30.  reth keeps the HashBuilder stack and the walker position; here the open
    right edge of the build is a b200_root_stream (frontier of the closed top-nibble buckets + the accounts of the open
    bucket in HBM) and the position is the index of the next account of the sorted state."""
    stream: object            # engine.RootStream
    next_account: int
    last_hashed_key: bytes

    def checkpoint(self) -> bytes:
        """What MerkleStage persists between runs (MerkleCheckpoint, merkle.rs:118-148): 1104 bytes."""
        return self.stream.checkpoint()


@dataclass
class StateRootProgress:
    """crates/trie/trie/src/progress.rs:12-21: `Complete(root, walked, updates)` (complete = True, state = None) or
    `Progress(state, walked, updates)` (complete = False, root = None; `updates` are the nodes finished so far by this call)."""
    root: Optional[bytes]
    hashed_entries_walked: int
    updates: TrieUpdates
    complete: bool = True
    state: Optional[IntermediateStateRootState] = None


class StateRootError(RuntimeError):
    """StateRootError::Database(DatabaseError::Other(msg)) in the Rust shim."""


def _records_to_nodes(records) -> Dict[int, Dict[Nibbles, BranchNodeCompact]]:
    out: Dict[int, Dict[Nibbles, BranchNodeCompact]] = {}
    for tid, path, sm, tm, hm, hashes in records:
        out.setdefault(tid, {})[bytes(path)] = BranchNodeCompact(sm, tm, hm, tuple(hashes))
    return out


class StorageRoot:
    """StorageRoot::new_hashed(..).root() / root_with_updates() — crates/trie/trie/src/trie.rs:479-615."""

    def __init__(self, engine: Engine, hashed_address: B256, storage: HashedStorageSorted):
        self.engine, self.hashed_address, self.storage = engine, hashed_address, storage
        self.prefix_set = None
        self.threshold = 100_000

    def with_prefix_set(self, prefix_set):
        """Kept for interface parity (trie.rs:512-516).  This calculator is given every slot of the trie and hashes all of
        them, so a changed-key set cannot alter its result; the skipping that prefix sets drive in reth happens in
        IncrementalStateRoot (stored nodes + prefix sets) and in the resident paths."""
        self.prefix_set = prefix_set
        return self

    def with_threshold(self, threshold: int):
        """trie.rs:523-527.  One storage trie is one device build (a 10M-slot trie takes milliseconds): `calculate`
        always returns the Complete variant, whatever the threshold — the thresholded, resumable build is StateRoot's
        (account ranges; every storage trie of a range is finished inside its push)."""
        self.threshold = threshold
        return self

    def with_no_threshold(self):
        self.threshold = 2**64 - 1
        return self

    def _flat(self):
        slots = [(k, v) for k, v in self.storage.storage_slots if v != 0]
        m = len(slots)
        keys = np.frombuffer(b"".join(k for k, _ in slots), np.uint8).reshape(m, 32) if m else np.zeros((0, 32), np.uint8)
        vals = np.frombuffer(b"".join(int(v).to_bytes(32, "big") for _, v in slots), np.uint8).reshape(m, 32) \
            if m else np.zeros((0, 32), np.uint8)
        return keys, vals, np.array([0, m], np.uint64)

    def root(self) -> bytes:
        return self.calculate(False)[0]

    def root_with_updates(self) -> Tuple[bytes, int, StorageTrieUpdates]:
        return self.calculate(True)

    def calculate(self, retain_updates: bool) -> Tuple[bytes, int, StorageTrieUpdates]:
        """-> (root, storage_slots_walked, updates) like StorageRootProgress::Complete (trie.rs:615-721)."""
        keys, vals, offs = self._flat()
        if len(keys) == 0:  # trie.rs:622-629
            return EMPTY_ROOT_HASH, 0, StorageTrieUpdates.deleted()
        try:
            if retain_updates:
                roots, recs = self.engine.storage_roots(keys, vals, offs, want_updates=True)
                upd = StorageTrieUpdates(storage_nodes=_records_to_nodes(recs).get(0, {}))
            else:
                roots, upd = self.engine.storage_roots(keys, vals, offs), StorageTrieUpdates()
        except Exception as e:  # noqa: BLE001 - mapped like the shim maps native errors
            raise StateRootError(str(e)) from e
        return roots[0].tobytes(), len(keys), upd


class StateRoot:
    """StateRoot::{root, root_with_updates, root_with_progress} — crates/trie/trie/src/trie.rs:54-158.

    with_threshold(t) + root_with_progress(): the build stops after a range of accounts holding at least `t` hashed
    entries (accounts + slots; reth counts retained trie updates, trie.rs:296-306 — a device build knows the entries of a
    range before it runs, the updates only afterwards) and returns StateRootProgress(complete=False, state=...); feeding the
    state back through with_intermediate_state() continues where it stopped.  root() / root_with_updates() ignore the
    threshold like the reference (trie.rs:126-140)."""

    def __init__(self, engine: Engine, hashed_state: HashedPostStateSorted):
        self.engine, self.state = engine, hashed_state
        self.prefix_sets = TriePrefixSets()
        self.threshold = 100_000  # DEFAULT_INTERMEDIATE_THRESHOLD, trie.rs:25
        self.previous_state: Optional[IntermediateStateRootState] = None

    def with_prefix_sets(self, prefix_sets: TriePrefixSets):
        """A from-scratch build hashes every leaf it is given, so the changed-key sets have nothing to skip; only
        `destroyed_accounts` is consumed (TrieUpdates::finalize).  The skip logic lives in IncrementalStateRoot (stored
        nodes + prefix sets) and in the resident paths."""
        self.prefix_sets = prefix_sets
        return self

    def with_threshold(self, threshold: int):
        self.threshold = threshold
        return self

    def with_no_threshold(self):
        self.threshold = 2**64 - 1
        return self

    def with_intermediate_state(self, state: Optional[IntermediateStateRootState]):
        self.previous_state = state
        return self

    def root(self) -> bytes:
        return self._calculate(False).root

    def root_with_updates(self) -> Tuple[bytes, TrieUpdates]:
        p = self._calculate(True)
        return p.root, p.updates

    def root_with_progress(self) -> StateRootProgress:
        if self.threshold >= 2**64 - 1 and self.previous_state is None:
            return self._calculate(True)
        return self._calculate_range()

    def _finalize(self, updates: TrieUpdates):
        # TrieUpdates::finalize (updates.rs:140-158): destroyed accounts -> is_deleted
        for destroyed in self.prefix_sets.destroyed_accounts:
            updates.storage_tries.setdefault(destroyed, StorageTrieUpdates()).is_deleted = True

    def _calculate(self, retain_updates: bool) -> StateRootProgress:
        keys, accts, skeys, svals, offs = self.state.to_flat()
        try:
            if retain_updates:
                root, acct_recs, stor_recs = self.engine.state_root_full(keys, accts, skeys, svals, offs,
                                                                         want_updates=True)
            else:
                root = self.engine.state_root_full(keys, accts, skeys, svals, offs)
                acct_recs = stor_recs = []
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e
        updates = TrieUpdates()
        if retain_updates:
            updates.account_nodes = _records_to_nodes(acct_recs).get(0, {})
            per_trie = _records_to_nodes(stor_recs)
            for i in range(len(keys)):
                addr = keys[i].tobytes()
                if offs[i + 1] == offs[i]:
                    # StorageRoot::calculate returns StorageTrieUpdates::deleted() for empty storage (trie.rs:622-629)
                    updates.insert_storage_updates(addr, StorageTrieUpdates.deleted())
                else:
                    updates.insert_storage_updates(addr, StorageTrieUpdates(storage_nodes=per_trie.get(i, {})))
            self._finalize(updates)
        walked = int(len(keys) + len(skeys))
        return StateRootProgress(root, walked, updates)

    def _calculate_range(self) -> StateRootProgress:
        """One step of the thresholded build: push the next range of accounts into the stream; Complete when none is left."""
        from .engine import RootStream
        keys, accts, skeys, svals, offs = self.state.to_flat()
        n = len(keys)
        st = self.previous_state
        try:
            if st is None:
                st = IntermediateStateRootState(RootStream(self.engine, retain_updates=True), 0, b"")
            a0 = st.next_account
            # the range: accounts a0 .. a1 holding >= threshold hashed entries (at least one account)
            target = int(offs[a0]) + a0 + min(self.threshold, 2**62) if a0 < n else 0
            entries = offs[a0:n + 1].astype(np.int64) + np.arange(a0, n + 1)      # entries before account i
            a1 = min(n, max(a0 + 1, int(np.searchsorted(entries, target, side="left")))) if a0 < n else n
            updates = TrieUpdates()
            walked = 0
            if a1 > a0:
                s0, s1 = int(offs[a0]), int(offs[a1])
                _, acct_recs, stor_recs = st.stream.push(keys[a0:a1], accts[a0:a1], skeys[s0:s1], svals[s0:s1],
                                                         (offs[a0:a1 + 1] - offs[a0]).astype(np.uint64))
                for _, path, sm, tm, hm, hashes in acct_recs:
                    updates.account_nodes[bytes(path)] = BranchNodeCompact(sm, tm, hm, tuple(hashes))
                per_trie = _records_to_nodes(stor_recs)
                for i in range(a0, a1):
                    addr = keys[i].tobytes()
                    if offs[i + 1] == offs[i]:
                        updates.insert_storage_updates(addr, StorageTrieUpdates.deleted())
                    else:
                        updates.insert_storage_updates(addr, StorageTrieUpdates(storage_nodes=per_trie.get(i - a0, {})))
                walked = (a1 - a0) + (s1 - s0)
                st.next_account = a1
                st.last_hashed_key = keys[a1 - 1].tobytes()
            if a1 < n:
                return StateRootProgress(None, walked, updates, complete=False, state=st)
            root, acct_recs = st.stream.finish()
            st.stream.close()
            for _, path, sm, tm, hm, hashes in acct_recs:
                updates.account_nodes[bytes(path)] = BranchNodeCompact(sm, tm, hm, tuple(hashes))
            self._finalize(updates)
            return StateRootProgress(root, walked, updates)
        except StateRootError:
            raise
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e


class ParallelStateRoot(StateRoot):
    """ParallelStateRoot::{incremental_root, incremental_root_with_updates} — crates/trie/parallel/src/root.rs:35-77.
    On the device the storage-root fan-out and the account fold are the same launches."""

    def incremental_root(self) -> bytes:
        return self.root()

    def incremental_root_with_updates(self) -> Tuple[bytes, TrieUpdates]:
        return self.root_with_updates()


class ResidentStateRoot:
    """Live-path commitment with the account trie resident in HBM (BASELINE config 5).

    Plays the part of `StateRoot::overlay_root_with_updates` / `ParallelStateRoot::incremental_root_with_updates`
    (crates/trie/db/src/state.rs:184-230, crates/trie/parallel/src/root.rs:35-77): `commit(HashedPostState)` folds one
    block's hashed post state into the committed state and returns the new root.  The hashed tables the reference
    reads through cursors (`HashedAccounts`, `HashedStorages`) are kept here as host dictionaries; the trie itself —
    every node hash of every level — lives on the device and only the dirty paths are re-hashed
    (`b200_trie_apply`).  Storage roots of the touched accounts are recomputed from their complete post-block storage
    in one `b200_storage_roots` call."""

    def __init__(self, engine: Engine, state: HashedPostStateSorted, dynamic: bool = False):
        """dynamic=True keeps the account trie in a `DynamicTrie` (b200_dtrie_*): new and destroyed accounts are applied in
        place instead of through merge + rebuild (`commit` then always reports rebuilt=False)."""
        from .engine import ACCOUNT_DTYPE, DynamicTrie, ResidentTrie
        self.engine = engine
        self.accounts = {k: a for k, a in state.accounts if a is not None}
        self.storages = {k: {s: v for s, v in st.storage_slots if v != 0} for k, st in state.storages.items()
                         if k in self.accounts}
        keys, accts, skeys, svals, offs = state.to_flat()
        sroots = engine.storage_roots(skeys, svals, offs) if len(keys) else np.zeros((0, 32), np.uint8)
        self.dynamic = dynamic
        self.trie = (DynamicTrie if dynamic else ResidentTrie).create(engine, keys, accts, sroots)
        self._dtype = ACCOUNT_DTYPE

    def root(self) -> bytes:
        return self.trie.root()

    def commit(self, post) -> Tuple[bytes, bool]:
        """post: HashedPostState.  -> (new root, rebuilt) where rebuilt tells whether the trie shape changed."""
        from .hashed_state import Account
        touched = set(post.accounts) | set(post.storages)
        # 1. storage overlay: wiped hides everything older, zero deletes (hashed_cursor/post_state.rs:185-195,260-297)
        for addr, hs in post.storages.items():
            cur = {} if hs.wiped else dict(self.storages.get(addr, {}))
            for slot, val in hs.storage.items():
                if val == 0:
                    cur.pop(slot, None)
                else:
                    cur[slot] = val
            self.storages[addr] = cur
        # 2. account overlay
        for addr, acc in post.accounts.items():
            if acc is None:
                self.accounts.pop(addr, None)
                self.storages.pop(addr, None)
            else:
                self.accounts[addr] = acc
        dirty = sorted(touched)
        if not dirty:
            return self.trie.root(), False
        live = [k for k in dirty if k in self.accounts]
        # 3. storage roots of the live touched accounts, all tries in one device call
        slot_keys, slot_vals, offs = [], [], [0]
        for k in live:
            st = sorted(self.storages.get(k, {}).items())
            slot_keys += [s for s, _ in st]
            slot_vals += [int(v).to_bytes(32, "big") for _, v in st]
            offs.append(offs[-1] + len(st))
        m = len(slot_keys)
        sk = np.frombuffer(b"".join(slot_keys), np.uint8).reshape(m, 32) if m else np.zeros((0, 32), np.uint8)
        sv = np.frombuffer(b"".join(slot_vals), np.uint8).reshape(m, 32) if m else np.zeros((0, 32), np.uint8)
        roots = self.engine.storage_roots(sk, sv, np.array(offs, np.uint64)) if live else np.zeros((0, 32), np.uint8)
        root_of = {k: roots[i] for i, k in enumerate(live)}
        # 4. one sorted dirty set for the device: upserts and deletes
        keys = np.frombuffer(b"".join(dirty), np.uint8).reshape(len(dirty), 32)
        accts = np.zeros(len(dirty), self._dtype)
        present = np.zeros(len(dirty), np.uint8)
        sroots = np.zeros((len(dirty), 32), np.uint8)
        for i, k in enumerate(dirty):
            a = self.accounts.get(k)
            if a is None:
                continue  # destroyed (or storage of an account that does not exist): delete / no-op
            present[i] = 1
            accts[i]["nonce"] = a.nonce
            accts[i]["balance"] = np.frombuffer(int(a.balance).to_bytes(32, "big"), np.uint8)
            accts[i]["code_hash"] = np.frombuffer(a.code_hash(), np.uint8)
            sroots[i] = root_of[k]
        try:
            if self.dynamic:
                return self.trie.apply(keys, accts, present, sroots), False
            return self.trie.apply(keys, accts, present, sroots)
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e

    def close(self):
        self.trie.close()


def apply_layout(post, destroyed_slots: bool):
    """post: HashedPostState -> (touched keys, the b200_dstate_apply arrays).  destroyed_slots: keep the slot entries
    of a destroyed account (the witness proves them; an apply ignores them)."""
    from .engine import ACCOUNT_DTYPE, DynamicState as DS
    touched = sorted(set(post.accounts) | set(post.storages))
    m = len(touched)
    keys = np.frombuffer(b"".join(touched), np.uint8).reshape(m, 32) if m else np.zeros((0, 32), np.uint8)
    accts = np.zeros(m, ACCOUNT_DTYPE)
    flags = np.zeros(m, np.uint8)
    sk, sv, offs = [], [], [0]
    for i, k in enumerate(touched):
        hs = post.storages.get(k)
        if k in post.accounts:
            a = post.accounts[k]
            if a is None:
                if destroyed_slots and hs is not None:
                    for s, v in sorted(hs.storage.items()):
                        sk.append(s)
                        sv.append(int(v).to_bytes(32, "big"))
                offs.append(len(sk))  # destroyed: flags 0, its storage is wiped
                continue
            flags[i] = DS.EXISTS
            accts[i]["nonce"] = a.nonce
            accts[i]["balance"] = np.frombuffer(int(a.balance).to_bytes(32, "big"), np.uint8)
            accts[i]["code_hash"] = np.frombuffer(a.code_hash(), np.uint8)
        else:
            flags[i] = DS.EXISTS | DS.UNCHANGED  # storage-only change
        if hs is not None:
            if hs.wiped:
                flags[i] |= DS.WIPED
            for s, v in sorted(hs.storage.items()):
                sk.append(s)
                sv.append(int(v).to_bytes(32, "big"))
        offs.append(len(sk))
    skeys = np.frombuffer(b"".join(sk), np.uint8).reshape(-1, 32) if sk else np.zeros((0, 32), np.uint8)
    svals = np.frombuffer(b"".join(sv), np.uint8).reshape(-1, 32) if sv else np.zeros((0, 32), np.uint8)
    return touched, (keys, accts, flags, skeys, svals, np.array(offs, np.uint64))


def _trie_updates(touched, au, ar, su, sr, deleted) -> TrieUpdates:
    """TrieUpdates of one block from the records of `DynamicState.apply(..., want_updates=True)` (or of an overlay), entry i
    being the account touched[i]."""
    upd = TrieUpdates()
    upd.account_nodes = _records_to_nodes(au).get(0, {})
    upd.removed_nodes = {bytes(p) for p in ar}
    per_entry = _records_to_nodes(su)
    removed_per_entry: Dict[int, set] = {}
    for entry, p in sr:
        removed_per_entry.setdefault(entry, set()).add(bytes(p))
    for i, k in enumerate(touched):
        st = StorageTrieUpdates(bool(deleted[i]), per_entry.get(i, {}), removed_per_entry.get(i, set()))
        upd.insert_storage_updates(k, st)
    return upd


class DynamicStateRoot:
    """Live-path commitment with the WHOLE hashed state resident in HBM (b200_dstate_*): accounts and every storage trie.

    The role of reth's `SparseStateTrie` fed by the state-root task (crates/trie/sparse/src/state.rs,
    crates/engine/tree/src/tree/payload_processor/sparse_trie.rs) and of `StateRoot::overlay_root_with_updates`
    (crates/trie/db/src/state.rs:184-230): `commit(HashedPostState)` applies one block in place — new / changed /
    destroyed accounts, slot writes, zeroed slots, wiped storages — and returns the new root with the block's
    `TrieUpdates` (account_nodes, removed_nodes, storage_tries with is_deleted).  Nothing of the state is kept on the host.
    Validated against the oracle on the GPU (tests/test_gpu_dstate.py)."""

    def __init__(self, engine: Engine, state: HashedPostStateSorted, sharded: bool = False):
        """sharded=True: this object is one rank's shard (see reth_b200.sharded.ShardedDynamicStateRoot); `commit`'s root is
        then the shard's own root and the state root comes from the gathered frontiers."""
        from .engine import ACCOUNT_DTYPE, DynamicState
        keys, accts, skeys, svals, offs = state.to_flat()
        self.ds = DynamicState.create(engine, keys, accts, skeys, svals, offs, sharded=sharded)
        self._dtype = ACCOUNT_DTYPE

    def root(self) -> bytes:
        return self.ds.root()

    def _block(self, post, destroyed_slots: bool):
        return apply_layout(post, destroyed_slots)

    def commit(self, post) -> Tuple[bytes, TrieUpdates]:
        """post: HashedPostState -> (root, TrieUpdates of the block)."""
        touched, block = self._block(post, destroyed_slots=False)
        try:
            res = self.ds.apply(*block, want_updates=True)
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e
        return res[0], _trie_updates(touched, *res[1:])

    def witness(self, post, mode: str = "legacy", always_include_root_node: bool = False) -> Dict[bytes, bytes]:
        """TrieWitness::compute(post) against the state as it is (crates/trie/trie/src/witness.rs): {keccak(node): node RLP}
        of every trie node a stateless client needs to apply `post` to this state.  mode: "legacy" (reth's default) or
        "canonical" (ExecutionWitnessMode).  The state is not changed; commit the block afterwards.  Raises StateRootError
        for a storage entry without an account entry (TrieWitnessError::MissingAccount).

        One difference from reth: the block goes through the layout `commit` uses, in which a destroyed account (None)
        always loses its storage.  reth's HashedPostState can also say "destroyed, storage not wiped" (no `storages` entry
        marked wiped); TrieWitness then keeps the account's storage root and upserts the default account, which needs
        other nodes.  Blocks from execution always wipe the storage of a destroyed account, so both give the same map."""
        for k in post.storages:
            if k not in post.accounts:
                raise StateRootError(f"missing account {k.hex()}")
        _, block = self._block(post, destroyed_slots=True)
        try:
            return self.ds.witness(*block, mode=mode, always_include_root_node=always_include_root_node)
        except ValueError:
            raise
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e

    def overlay_witness(self, input_post, post, mode: str = "legacy", always_include_root_node: bool = False) -> Dict[bytes, bytes]:
        """StateProofProvider::witness(input, target, mode) of a MemoryOverlayStateProvider (crates/chain-state/src/
        memory_overlay.rs) in one device call (b200_dstate_overlay_witness): witness(post) on the state after `input_post`,
        with the state left as it is — debug_executionWitness and the invalid-block witness hook when the parent block is
        not persisted.  A chain of in-memory blocks is one input_post merged with HashedPostState.extend.  The map is exactly
        what commit(input_post) and then witness(post, ...) give; `overlay_root(input_post)` is the parent root a stateless
        client checks it against.  Raises StateRootError for a storage entry of `post` without an account entry
        (TrieWitnessError::MissingAccount); the layout note of `witness` holds for `post` as well."""
        for k in post.storages:
            if k not in post.accounts:
                raise StateRootError(f"missing account {k.hex()}")
        _, overlay = self._block(input_post, destroyed_slots=False)
        _, block = self._block(post, destroyed_slots=True)
        try:
            return self.ds.overlay_witness(overlay, block, mode=mode, always_include_root_node=always_include_root_node)[1]
        except ValueError:
            raise
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e

    def overlay_roots(self, posts) -> List[bytes]:
        """StateRootProvider::state_root(hashed_state) on the latest state (crates/storage/storage-api/src/trie.rs) for a batch
        of candidate blocks, in one device call (b200_dstate_overlay_roots): the root `commit` of each post alone would
        return, with the state left as it is — to validate a payload, or to finish every payload built on this parent, before
        `commit` keeps one of them.  The posts are siblings on the current state, not a chain.  A chain of uncommitted blocks
        is one post merged with HashedPostState.extend, as MemoryOverlayStateProvider merges its in-memory blocks
        (crates/chain-state/src/memory_overlay.rs).  `overlay_roots_with_updates` also returns each block's TrieUpdates."""
        return self._overlay(posts, False)

    def overlay_root(self, post) -> bytes:
        """overlay_roots for one post: the root `commit(post)` would return, without changing the state."""
        return self.overlay_roots([post])[0]

    def overlay_roots_with_updates(self, posts) -> List[Tuple[bytes, TrieUpdates]]:
        """StateRoot::overlay_root_with_updates (crates/trie/db/src/state.rs:219-230) for a batch of candidate blocks, in one
        device call (b200_dstate_overlay_roots_with_updates): for each post, (root, TrieUpdates) that describe the same trie
        tables after the block as `commit(post)`'s, with the state left as it is — what payload validation, BlockBuilder::finish
        and debug_stateRootWithUpdates keep with a block until it is persisted."""
        return self._overlay(posts, True)

    def overlay_root_with_updates(self, post) -> Tuple[bytes, TrieUpdates]:
        """overlay_roots_with_updates for one post."""
        return self.overlay_roots_with_updates([post])[0]

    def overlay_multiproof(self, post, targets) -> dict:
        """StateProofProvider::multiproof(input, targets) of a MemoryOverlayStateProvider (crates/chain-state/src/
        memory_overlay.rs; Proof::overlay_multiproof, crates/trie/db/src/proof.rs) in one device call
        (b200_dstate_overlay_multiproof): the proofs of `targets` ({hashed address: hashed slots}) in the state after `post`,
        with the state left as it is — eth_getProof at a block that is not persisted, and the proof workers of the state-root
        task.  A chain of in-memory blocks is one post merged with HashedPostState.extend.  -> the dict of
        DynamicState.multiproof plus "root", the root `commit(post)` would return."""
        _, block = self._block(post, destroyed_slots=False)
        try:
            return self.ds.overlay_multiproof(block, targets)
        except ValueError:
            raise
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e

    def trie_changesets(self, updates) -> TrieUpdatesSorted:
        """compute_trie_changesets(factory, &trie_updates) (crates/trie/trie/src/changesets.rs:50-239) with this state as the
        trie cursor factory, in one device call (b200_dstate_trie_changesets): the values the nodes a block changes had before
        it, which reth writes next to the block and applies backwards on unwind.  updates: the block's TrieUpdatesSorted (a
        TrieUpdates is sorted first); only its paths and is_deleted are read.  -> TrieUpdatesSorted of the old values: each
        account path, and each path of a storage trie that is not deleted, with the node stored at exactly that path or None;
        a deleted storage trie gets every node it stored merged in by path (storage_trie_wiped_changeset_iter); storage tries
        with an empty changeset are left out.  The state does not change.

        On the live path the order is overlay_root_with_updates(post) -> trie_changesets(updates) -> commit(post): the call
        reads the nodes as they are before the block, and the commit overwrites them.  The parent is the resident state itself;
        changesets against a parent that is an unpersisted overlay (reth's InMemoryTrieCursorFactory over cumulative updates)
        are not covered."""
        if isinstance(updates, TrieUpdates):
            updates = updates.into_sorted()
        addrs = sorted(updates.storage_tries)
        storage = {a: (updates.storage_tries[a].is_deleted, [p for p, _ in updates.storage_tries[a].storage_nodes]) for a in addrs}
        try:
            acct, stor = self.ds.trie_changesets([p for p, _ in updates.account_nodes], storage)
        except ValueError:
            raise
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e
        node = lambda r: BranchNodeCompact(r[2], r[3], r[4], tuple(r[5])) if r[2] else None  # state_mask 0: None
        out = TrieUpdatesSorted([(r[1], node(r)) for r in acct])
        per_trie: Dict[int, list] = {}
        for r in stor:
            per_trie.setdefault(r[0], []).append((r[1], node(r)))
        for i, a in enumerate(addrs):
            if per_trie.get(i):
                out.storage_tries[a] = StorageTrieUpdatesSorted(updates.storage_tries[a].is_deleted, per_trie[i])
        return out

    def _overlay(self, posts, want_updates: bool):
        layouts = [self._block(post, destroyed_slots=False) for post in posts]
        try:
            res = self.ds.overlay_roots([block for _, block in layouts], want_updates=want_updates)
        except ValueError:
            raise
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e
        if not want_updates:
            return res
        return [(r[0], _trie_updates(touched, *r[1:])) for (touched, _), r in zip(layouts, res)]

    def close(self):
        self.ds.close()


def stateless_state_roots(engine: Engine, parent_roots, witnesses, posts) -> List[bytes]:
    """Stateless validation of a batch of blocks (b200_witness_roots): the post-block state root of every block from its
    parent root, its execution witness (ExecutionWitness.state: a list of node RLPs, or a {hash: rlp} map) and its
    HashedPostState alone.  Raises StateRootError for a storage entry without an account entry, and for the first block
    whose witness is incomplete or holds a malformed node (naming the block and the status)."""
    blocks = []
    for post in posts:
        for k in post.storages:
            if k not in post.accounts:
                raise StateRootError(f"missing account {k.hex()}")
        blocks.append(apply_layout(post, destroyed_slots=False)[1])
    try:
        roots, statuses = engine.witness_roots(list(parent_roots), list(witnesses), blocks)
    except ValueError:
        raise
    except Exception as e:  # noqa: BLE001
        raise StateRootError(str(e)) from e
    for b, st in enumerate(statuses):
        if st:
            what = "witness incomplete" if st == ERR_WITNESS_INCOMPLETE else "malformed witness node"
            raise StateRootError(f"block {b}: {what} (status {int(st)})")
    return [r.tobytes() for r in roots]


def stateless_state_root(engine: Engine, parent_root: bytes, witness, post) -> bytes:
    """stateless_state_roots for one block."""
    return stateless_state_roots(engine, [parent_root], [witness], [post])[0]
