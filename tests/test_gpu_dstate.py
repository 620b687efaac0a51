"""Dynamic resident state (b200_dstate_*, SURVEY §8 f1): accounts and every storage trie resident; blocks of account
upserts / destructions and slot upserts / deletions / wipes applied in place.  After every block the root equals the
oracle's from-scratch StateRoot over the merged state, and the account / storage TrieUpdates applied to a model of
AccountsTrie / StoragesTrie reproduce the oracle's full node sets (reth's incremental == full criterion,
crates/trie/db/tests/trie.rs:680-717, crates/trie/parallel/src/root.rs:287-400)."""
import os

import numpy as np
import pytest

import oracle
from tests.util import to_device_ptrs

pytestmark = [pytest.mark.gpu]

EXISTS, UNCHANGED, WIPED = 1, 2, 4


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def acct(nonce, balance=0):
    a = np.zeros((), oracle.ACCOUNT_DTYPE)
    a["nonce"] = nonce
    a["balance"] = np.frombuffer(int(balance).to_bytes(32, "big"), np.uint8)
    a["code_hash"] = np.frombuffer(oracle.KECCAK_EMPTY, np.uint8)
    return a


def flatten(state):
    """state: {addr: (account, {slot: int})} -> flat sorted arrays"""
    ks = sorted(state)
    n = len(ks)
    keys = np.frombuffer(b"".join(ks), np.uint8).reshape(n, 32) if n else np.zeros((0, 32), np.uint8)
    accs = np.zeros(n, oracle.ACCOUNT_DTYPE)
    sk, sv, offs = [], [], [0]
    for i, k in enumerate(ks):
        accs[i] = state[k][0]
        for s in sorted(state[k][1]):
            sk.append(s)
            sv.append(int(state[k][1][s]).to_bytes(32, "big"))
        offs.append(len(sk))
    skeys = np.frombuffer(b"".join(sk), np.uint8).reshape(-1, 32) if sk else np.zeros((0, 32), np.uint8)
    svals = np.frombuffer(b"".join(sv), np.uint8).reshape(-1, 32) if sv else np.zeros((0, 32), np.uint8)
    return ks, keys, accs, skeys, svals, np.array(offs, np.uint64)


def model(state):
    ks, keys, accs, skeys, svals, offs = flatten(state)
    root, au, su = oracle.state_root_full(keys, accs, skeys, svals, offs, want_updates=True)
    acct_nodes = {r[1]: r[2:] for r in au}
    storage_nodes = {}
    for r in su:
        storage_nodes.setdefault(ks[r[0]], {})[r[1]] = r[2:]
    return root, acct_nodes, storage_nodes


class Harness:
    def __init__(self, eng, state):
        from reth_b200 import DynamicState
        self.state = {k: (a.copy(), dict(s)) for k, (a, s) in state.items()}
        _, keys, accs, skeys, svals, offs = flatten(self.state)
        self.ds = DynamicState.create(eng, keys, accs, skeys, svals, offs)
        root, self.adb, self.sdb = model(self.state)
        assert self.ds._root == root

    def commit(self, block):
        """block: {addr: (flags, account, {slot: value})}"""
        ks = sorted(block)
        m = len(ks)
        keys = np.frombuffer(b"".join(ks), np.uint8).reshape(m, 32) if m else np.zeros((0, 32), np.uint8)
        accs = np.zeros(m, oracle.ACCOUNT_DTYPE)
        flags = np.zeros(m, np.uint8)
        sk, sv, offs = [], [], [0]
        for i, k in enumerate(ks):
            fl, a, slots = block[k]
            flags[i], accs[i] = fl, a
            for s in sorted(slots):
                sk.append(s)
                sv.append(int(slots[s]).to_bytes(32, "big"))
            offs.append(len(sk))
            # the model: HashedPostState overlay rules (hashed_cursor/post_state.rs:185-195,260-297)
            if not (fl & EXISTS):
                self.state.pop(k, None)
                continue
            if fl & UNCHANGED:
                if k not in self.state:
                    continue
                cur_a, cur_s = self.state[k]
            else:
                cur_a, cur_s = a.copy(), (self.state[k][1] if k in self.state else {})
            cur_s = {} if (fl & WIPED) else dict(cur_s)
            for s, v in slots.items():
                if v == 0:
                    cur_s.pop(s, None)
                else:
                    cur_s[s] = v
            self.state[k] = (cur_a, cur_s)
        skeys = np.frombuffer(b"".join(sk), np.uint8).reshape(-1, 32) if sk else np.zeros((0, 32), np.uint8)
        svals = np.frombuffer(b"".join(sv), np.uint8).reshape(-1, 32) if sv else np.zeros((0, 32), np.uint8)
        root, au, ar, su, sr, deleted = self.ds.apply(keys, accs, flags, skeys, svals, np.array(offs, np.uint64),
                                                      want_updates=True)
        o_root, o_adb, o_sdb = model(self.state)
        assert root == o_root == self.ds.root()
        assert self.ds.accounts() == len(self.state)
        assert self.ds.slots() == sum(len(s) for _, s in self.state.values())
        for p in ar:
            self.adb.pop(p, None)
        for r in au:
            self.adb[r[1]] = r[2:]
        assert self.adb == o_adb
        for i, k in enumerate(ks):
            if deleted[i]:
                self.sdb.pop(k, None)          # StorageTrieUpdates::is_deleted: clear the account's duplicates
        for entry, p in sr:
            self.sdb.get(ks[entry], {}).pop(p, None)
        for r in su:
            self.sdb.setdefault(ks[r[0]], {})[r[1]] = r[2:]
        assert {k: v for k, v in self.sdb.items() if v} == o_sdb
        return root


def rkey(rng):
    return rng.integers(0, 256, 32, dtype=np.uint8).tobytes()


def random_state(rng, n, with_storage=0.4, max_slots=40):
    st = {}
    for _ in range(n):
        slots = {}
        if rng.random() < with_storage:
            slots = {rkey(rng): int(rng.integers(1, 2**62)) for _ in range(int(rng.integers(1, max_slots)))}
        st[rkey(rng)] = (acct(int(rng.integers(0, 50)), int(rng.integers(1, 2**60))), slots)
    return st


def random_block(rng, state, n_touch, step):
    block = {}
    live = sorted(state)
    for _ in range(n_touch):
        r = rng.integers(0, 7)
        if r == 0 or not live:                                   # new account, maybe with storage
            slots = {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(int(rng.integers(0, 12)))}
            block[rkey(rng)] = (EXISTS, acct(step, 5), slots)
        elif r == 1:                                             # destroyed
            block[live[rng.integers(0, len(live))]] = (0, acct(0), {})
        elif r == 2:                                             # balance change only
            k = live[rng.integers(0, len(live))]
            a = state[k][0].copy()
            a["nonce"] += 1
            block[k] = (EXISTS, a, {})
        elif r in (3, 4):                                        # storage-only change: new slots, changed slots, zeroed slots
            k = live[rng.integers(0, len(live))]
            cur = sorted(state[k][1])
            slots = {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(int(rng.integers(1, 6)))}
            for s in cur[:int(rng.integers(0, 4))]:
                slots[s] = 0 if rng.random() < 0.5 else int(rng.integers(1, 2**50))
            block[k] = (EXISTS | UNCHANGED, acct(0), slots)
        elif r == 5:                                             # wipe + refill (selfdestruct & recreate)
            k = live[rng.integers(0, len(live))]
            slots = {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(int(rng.integers(0, 5)))}
            block[k] = (EXISTS | WIPED, state[k][0].copy(), slots)
        else:                                                    # storage for an account that does not exist: ignored
            block[rkey(rng)] = (EXISTS | UNCHANGED, acct(0), {rkey(rng): 7})
    return block


@pytest.mark.parametrize("n0,blocks,touch", [(0, 5, 6), (3, 6, 5), (200, 8, 40), (1500, 5, 150)])
def test_random_blocks_match_full_state_root(eng, n0, blocks, touch):
    rng = np.random.default_rng(400 + n0)
    h = Harness(eng, random_state(rng, n0))
    for step in range(blocks):
        h.commit(random_block(rng, h.state, touch, step + 1))
    h.ds.close()


def test_storage_lifecycle_of_one_account(eng):
    rng = np.random.default_rng(9)
    st = random_state(rng, 50, with_storage=0.0)
    h = Harness(eng, st)
    k = sorted(h.state)[7]
    slots = [rkey(rng) for _ in range(300)]
    h.commit({k: (EXISTS | UNCHANGED, acct(0), {s: i + 1 for i, s in enumerate(slots[:1])})})      # first slot: root = leaf
    h.commit({k: (EXISTS | UNCHANGED, acct(0), {s: i + 1 for i, s in enumerate(slots)})})          # grows
    h.commit({k: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in slots[::2]})})                        # half deleted
    h.commit({k: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in slots[1::2]})})                       # empty again
    assert h.ds.slots() == 0
    h.commit({k: (EXISTS | UNCHANGED, acct(0), {s: 9 for s in slots[:40]})})
    h.commit({k: (EXISTS | WIPED, h.state[k][0].copy(), {slots[0]: 1})})                            # wiped, one slot back
    h.commit({k: (0, acct(0), {})})                                                                 # destroyed
    assert h.ds.slots() == 0
    h.commit({k: (EXISTS, acct(1, 1), {slots[5]: 5})})                                              # re-created
    h.ds.close()


def test_destroyed_and_recreated_in_neighbouring_blocks_reuses_slots(eng):
    rng = np.random.default_rng(10)
    h = Harness(eng, random_state(rng, 120, with_storage=0.8, max_slots=25))
    for step in range(4):
        live = sorted(h.state)
        kill = {live[i]: (0, acct(0), {}) for i in rng.choice(len(live), 30, replace=False)}
        h.commit(kill)
        born = {rkey(rng): (EXISTS, acct(step), {rkey(rng): int(rng.integers(1, 2**40)) for _ in range(int(rng.integers(0, 20)))})
                for _ in range(30)}
        h.commit(born)
    h.ds.close()


def test_dynamic_state_root_commits_hashed_post_states(eng):
    """The host mirror: blocks arrive as reth's HashedPostState (accounts: Some / None = destroyed; storages with wiped
    flag and zero = delete); after every block root and TrieUpdates agree with a from-scratch StateRoot over the merged
    state (crates/trie/db/tests/trie.rs:680-717)."""
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage, StateRoot
    rng = np.random.default_rng(78)
    rk = lambda: bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    base = HashedPostState()
    for _ in range(500):
        k = rk()
        base.accounts[k] = Account(int(rng.integers(0, 50)), int(rng.integers(1, 2**62)))
        if rng.random() < 0.3:
            base.storages[k] = HashedStorage(False, {rk(): int(rng.integers(1, 2**62)) for _ in range(int(rng.integers(1, 30)))})
    merged = HashedPostState(dict(base.accounts), {k: HashedStorage(False, dict(v.storage)) for k, v in base.storages.items()})
    ds = DynamicStateRoot(eng, base.into_sorted())
    root0, full0 = StateRoot(eng, base.into_sorted()).root_with_updates()
    assert ds.root() == root0
    acct_db = dict(full0.account_nodes)
    stor_db = {k: dict(v.storage_nodes) for k, v in full0.storage_tries.items() if v.storage_nodes}
    for block in range(5):
        post = HashedPostState()
        live = [k for k, a in merged.accounts.items() if a is not None]
        for i in rng.choice(len(live), 30, replace=False):
            a = merged.accounts[live[i]]
            post.accounts[live[i]] = Account(a.nonce + 1, a.balance + 7, a.bytecode_hash)
        for _ in range(8):
            k = rk()
            post.accounts[k] = Account(0, int(rng.integers(1, 10**18)))
            if rng.random() < 0.5:
                post.storages[k] = HashedStorage(False, {rk(): int(rng.integers(1, 2**60)) for _ in range(5)})
        for i in rng.choice(len(live), 4, replace=False):
            post.accounts[live[i]] = None
            post.storages[live[i]] = HashedStorage(True, {})
        with_storage = [k for k in merged.storages if merged.accounts.get(k) is not None and k not in post.accounts]
        for k in with_storage[:6]:
            slots = list(merged.storages[k].storage)
            changes = {slots[0]: 0} if slots else {}
            changes[rk()] = int(rng.integers(1, 2**60))
            post.storages[k] = HashedStorage(block == 3, changes)
        root, upd = ds.commit(post)
        for k, hs in post.storages.items():
            cur = {} if hs.wiped else dict(merged.storages.get(k, HashedStorage()).storage)
            for s, v in hs.storage.items():
                if v == 0:
                    cur.pop(s, None)
                else:
                    cur[s] = v
            merged.storages[k] = HashedStorage(False, cur)
        for k, a in post.accounts.items():
            if a is None:
                merged.accounts.pop(k, None)
                merged.storages.pop(k, None)
            else:
                merged.accounts[k] = a
        o_root, o_full = StateRoot(eng, merged.into_sorted()).root_with_updates()
        assert root == o_root, block
        for p in upd.removed_nodes:
            acct_db.pop(p, None)
        acct_db.update(upd.account_nodes)
        assert acct_db == o_full.account_nodes
        for k, st in upd.storage_tries.items():
            if st.is_deleted:
                stor_db.pop(k, None)
            cur = stor_db.setdefault(k, {})
            for p in st.removed_nodes:
                cur.pop(p, None)
            cur.update(st.storage_nodes)
        assert {k: v for k, v in stor_db.items() if v} == {k: v.storage_nodes for k, v in o_full.storage_tries.items() if v.storage_nodes}
    ds.close()


class ShardedHarness:
    """`world` shards of one state (rank r owns top nibbles [16r/world, 16(r+1)/world)), as separate b200_dstate objects in
    one process; a block is routed by top nibble, the frontiers are merged the way the NCCL all-gather would."""

    def __init__(self, eng, state, world):
        from reth_b200 import DynamicState
        self.eng, self.world = eng, world
        self.state = {k: (a.copy(), dict(s)) for k, (a, s) in state.items()}
        self.shards = []
        for r in range(world):
            part = {k: v for k, v in self.state.items() if self.rank_of(k) == r}
            _, keys, accs, skeys, svals, offs = flatten(part)
            self.shards.append(DynamicState.create(eng, keys, accs, skeys, svals, offs, sharded=True))
        root, self.adb, self.sdb = model(self.state)
        assert self.global_root() == root

    def rank_of(self, k):
        return (k[0] >> 4) * self.world // 16

    def global_root(self):
        merged = np.zeros((16, 68), np.uint8)
        for r, ds in enumerate(self.shards):
            fr = ds.frontier()
            lo, hi = -(-16 * r // self.world), -(-16 * (r + 1) // self.world)
            mine = [b for b in range(16) if b * self.world // 16 == r]
            assert not fr[[b for b in range(16) if b not in mine]].any()
            merged[mine] = fr[mine]
        return self.eng.root_from_frontier(merged)

    def commit(self, block):
        for k, (fl, a, slots) in block.items():           # the model (same overlay rules as Harness.commit)
            if not (fl & EXISTS):
                self.state.pop(k, None)
                continue
            if fl & UNCHANGED:
                if k not in self.state:
                    continue
                cur_a, cur_s = self.state[k]
            else:
                cur_a, cur_s = a.copy(), (self.state[k][1] if k in self.state else {})
            cur_s = {} if (fl & WIPED) else dict(cur_s)
            for s, v in slots.items():
                if v == 0:
                    cur_s.pop(s, None)
                else:
                    cur_s[s] = v
            self.state[k] = (cur_a, cur_s)
        for r, ds in enumerate(self.shards):
            ks = sorted(k for k in block if self.rank_of(k) == r)
            m = len(ks)
            keys = np.frombuffer(b"".join(ks), np.uint8).reshape(m, 32) if m else np.zeros((0, 32), np.uint8)
            accs = np.zeros(m, oracle.ACCOUNT_DTYPE)
            flags = np.zeros(m, np.uint8)
            sk, sv, offs = [], [], [0]
            for i, k in enumerate(ks):
                flags[i], accs[i] = block[k][0], block[k][1]
                for s in sorted(block[k][2]):
                    sk.append(s)
                    sv.append(int(block[k][2][s]).to_bytes(32, "big"))
                offs.append(len(sk))
            skeys = np.frombuffer(b"".join(sk), np.uint8).reshape(-1, 32) if sk else np.zeros((0, 32), np.uint8)
            svals = np.frombuffer(b"".join(sv), np.uint8).reshape(-1, 32) if sv else np.zeros((0, 32), np.uint8)
            _, au, ar, su, sr, deleted = ds.apply(keys, accs, flags, skeys, svals, np.array(offs, np.uint64), want_updates=True)
            for p in ar:
                self.adb.pop(p, None)
            for rec in au:
                self.adb[rec[1]] = rec[2:]
            for i, k in enumerate(ks):
                if deleted[i]:
                    self.sdb.pop(k, None)
            for entry, p in sr:
                self.sdb.get(ks[entry], {}).pop(p, None)
            for rec in su:
                self.sdb.setdefault(ks[rec[0]], {})[rec[1]] = rec[2:]
        o_root, o_adb, o_sdb = model(self.state)
        assert self.global_root() == o_root
        assert self.adb == o_adb                      # the union of the shards' TrieUpdates == the unsharded node set
        assert {k: v for k, v in self.sdb.items() if v} == o_sdb
        assert sum(ds.accounts() for ds in self.shards) == len(self.state)


@pytest.mark.parametrize("world", [1, 2, 8, 16])
def test_sharded_state_matches_full_root(eng, world):
    rng = np.random.default_rng(900 + world)
    h = ShardedHarness(eng, random_state(rng, 400), world)
    for step in range(4):
        h.commit(random_block(rng, h.state, 60, step + 1))
    for ds in h.shards:
        ds.close()


def test_sharded_state_degenerate_buckets(eng):
    """All accounts in one bucket (the global root is not a depth-0 branch), then a second bucket appears and vanishes."""
    rng = np.random.default_rng(31)
    st = {}
    for _ in range(40):
        k = bytearray(rkey(rng))
        k[0] = 0x30 | (k[0] & 15)
        st[bytes(k)] = (acct(1, 5), {})
    h = ShardedHarness(eng, st, 4)
    other = bytearray(rkey(rng))
    other[0] = 0xC1
    h.commit({bytes(other): (EXISTS, acct(2, 2), {rkey(rng): 9})})
    h.commit({bytes(other): (0, acct(0), {})})
    h.commit({k: (0, acct(0), {}) for k in sorted(h.state)[1:]})      # a single account left
    h.commit({k: (0, acct(0), {}) for k in sorted(h.state)})           # empty state
    for ds in h.shards:
        ds.close()


@pytest.mark.parametrize("sharded", [False, True])
def test_device_resident_seed(eng, sharded):
    """b200_dstate_create_dev: the seed arrays already live in device memory (tests/util.py:to_device_ptrs)."""
    from reth_b200 import DynamicState
    rng = np.random.default_rng(55)
    state = random_state(rng, 600)
    _, keys, accs, skeys, svals, offs = flatten(state)
    ptrs, hold = to_device_ptrs((keys, accs, skeys, svals, offs))
    ds = DynamicState.create_dev(eng, ptrs[0], ptrs[1], len(keys), ptrs[2], ptrs[3], ptrs[4], len(skeys), sharded=sharded)
    root, _, _ = model(state)
    if sharded:
        assert eng.root_from_frontier(ds.frontier()) == root
    assert ds.root() == root and ds.accounts() == len(state)
    ds.close()


def test_new_contract_with_many_slots_in_one_block(eng):
    """A whole storage trie appears in one block: every slot attaches at the new trie's root word, i.e. one long insert
    run — handled in rounds (8 keys per run and round), not serially."""
    rng = np.random.default_rng(77)
    h = Harness(eng, random_state(rng, 100, with_storage=0.2))
    big = {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(5000)}
    h.commit({rkey(rng): (EXISTS, acct(1, 1), big)})
    k = next(a for a, (_, s) in h.state.items() if len(s) == 5000)
    h.commit({k: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in sorted(big)[::2]})})          # half of it deleted again
    h.commit({k: (EXISTS | UNCHANGED, acct(0), {rkey(rng): 5 for _ in range(2000)})})       # and 2000 more
    h.ds.close()


def clustered_slots(rng, n_clusters):
    """Slots in clusters of 2..16 keys that differ only in their last nibble.  A cluster is one depth-63 branch whose
    leaves are inline: 3, 5 or 6 bytes of RLP for a value < 0x80, < 0x100 or < 0x10000.  The branch is 18 - n + (the
    leaves' lengths) bytes; below 32 it is itself inline, under the extension that leads to it from the shallow branch
    where the clusters part."""
    slots = {}
    for _ in range(n_clusters):
        key = bytearray(rkey(rng))
        for nib in rng.choice(16, int(rng.integers(2, 17)), replace=False):
            key[31] = (key[31] & 0xF0) | int(nib)
            slots[bytes(key)] = int(rng.integers(1, (0x80, 0x100, 0x10000)[rng.integers(0, 3)]))
    return slots


def test_inline_children_of_clustered_slots(eng):
    """Storage tries whose branches have inline (< 32 byte) children: the inline-child paths of the warp and thread node
    builders and of the proof encoder.  Small blocks first, then one block of more than 8192 slot entries (the multi-launch
    restructure and the two-stage re-hash at the default thresholds); the slot proofs of clustered keys chain to the roots."""
    from tests.test_gpu_proofs import verify
    rng = np.random.default_rng(515)
    st = random_state(rng, 200, with_storage=0.0)
    owners = sorted(st)[:24]
    for k in owners:
        st[k] = (st[k][0], clustered_slots(rng, int(rng.integers(1, 5))))
    h = Harness(eng, st)
    for step in range(3):
        block = {}
        for i in rng.choice(len(owners), 6, replace=False):
            k = owners[i]
            slots = clustered_slots(rng, 2)
            for s in sorted(h.state[k][1])[:4]:               # changed and deleted members of existing clusters
                slots[s] = 0 if rng.random() < 0.5 else int(rng.integers(1, 0x10000))
            block[k] = (EXISTS | UNCHANGED, acct(0), slots)
        h.commit(block)
    block, n = {}, 0
    for k in owners:
        slots = clustered_slots(rng, 40)
        n += len(slots)
        block[k] = (EXISTS | UNCHANGED, acct(0), slots)
    assert n > 8192
    h.commit(block)
    _, keys, _, skeys, svals, offs = flatten(h.state)
    sroots = oracle.storage_roots(skeys, svals, offs)
    index = {k: i for i, k in enumerate(sorted(h.state))}
    inline_lengths = set()
    for k in owners:
        have = sorted(h.state[k][1])
        near = [s[:31] + bytes([s[31] ^ 0x0F]) for s in have[:4]]   # same cluster prefix, maybe absent
        tgt = have[:12] + near
        sroot, proofs = h.ds.storage_proofs(k, np.frombuffer(b"".join(tgt), np.uint8).reshape(-1, 32))
        assert sroot == sroots[index[k]].tobytes()
        for s, proof in zip(tgt, proofs):
            v = h.state[k][1].get(s)
            verify(sroot, s, proof, None if v is None else oracle.encode_u256(v))
            inline_lengths |= {len(node) for node in proof[1:] if len(node) < 32}
    assert {n % 4 for n in inline_lengths} == {0, 1, 2, 3}      # every tail length of an inline child reference
    h.ds.close()


def test_merkle_stage_incremental_equals_rebuild(eng):
    """The three stages end to end: a full pass (AccountHashing, StorageHashing, MerkleStage rebuild), then ranges of
    changes through MerkleStage.execute_incremental (incremental hashing + the resident state).  After every range the
    root and the trie tables equal what a rebuild over the updated plain state produces
    (crates/stages/stages/src/stages/merkle.rs:520-618 execute_small_merkle / execute_chunked_merkle)."""
    from reth_b200 import Account, AccountHashingStage, MerkleStage, StorageHashingStage
    from reth_b200.stages import Tables
    rng = np.random.default_rng(88)
    ra = lambda: bytes(rng.integers(0, 256, 20, dtype=np.uint8))
    t = Tables()
    for _ in range(400):
        a = ra()
        t.plain_accounts[a] = Account(int(rng.integers(0, 9)), int(rng.integers(1, 2**60)))
        if rng.random() < 0.3:
            t.plain_storage[a] = {int(rng.integers(0, 2**63)): int(rng.integers(1, 2**60)) for _ in range(int(rng.integers(1, 25)))}
    AccountHashingStage(eng).execute(t)
    StorageHashingStage(eng).execute(t)
    stage = MerkleStage(eng)
    stage.execute(t)

    def rebuild(plain_accounts, plain_storage):
        r = Tables(plain_accounts=dict(plain_accounts), plain_storage={a: dict(s) for a, s in plain_storage.items()})
        AccountHashingStage(eng).execute(r)
        StorageHashingStage(eng).execute(r)
        root = MerkleStage(eng).execute(r)
        return root, r

    for rng_no in range(4):
        live = sorted(t.plain_accounts)
        changed_accounts, changed_storage, wiped = {}, {}, set()
        for i in rng.choice(len(live), 25, replace=False):
            acc = t.plain_accounts[live[i]]
            changed_accounts[live[i]] = Account(acc.nonce + 1, acc.balance + 3, acc.bytecode_hash)
        for _ in range(6):
            a = ra()
            changed_accounts[a] = Account(0, 5)
            changed_storage[a] = {int(rng.integers(0, 2**63)): 9 for _ in range(4)}
        for i in rng.choice(len(live), 3, replace=False):
            changed_accounts[live[i]] = None
            changed_storage.pop(live[i], None)
        with_storage = [a for a in t.plain_storage if t.plain_storage[a] and changed_accounts.get(a, 0) is not None]
        for a in with_storage[:5]:
            slots = sorted(t.plain_storage[a])
            changed_storage[a] = {slots[0]: 0, int(rng.integers(0, 2**63)): int(rng.integers(1, 2**40))}
        if rng_no == 2 and with_storage:
            wiped.add(with_storage[-1])
            changed_storage[with_storage[-1]] = {7: 7}
        root = stage.execute_incremental(t, changed_accounts, changed_storage, wiped)
        o_root, r = rebuild(t.plain_accounts, t.plain_storage)
        assert root == o_root
        assert t.hashed_accounts == r.hashed_accounts and t.hashed_storages == r.hashed_storages
        assert t.trie_updates.account_nodes == r.trie_updates.account_nodes
        mine = {k: v.storage_nodes for k, v in t.trie_updates.storage_tries.items() if v.storage_nodes}
        theirs = {k: v.storage_nodes for k, v in r.trie_updates.storage_tries.items() if v.storage_nodes}
        assert mine == theirs
    with pytest.raises(Exception):
        stage.execute_incremental(t, {ra(): Account(1, 1)}, {}, expected_state_root=b"\\x00" * 32)
    stage.close()


def test_block_updates_as_table_rows(eng):
    """The block's storage records (trie_id = account entry index) feed b200_storage_trie_rows with the block's own account
    keys: rows come out in StoragesTrie key order (address, then sub-key), ready for the cursor upsert loop."""
    from reth_b200 import tables
    rng = np.random.default_rng(91)
    h = Harness(eng, random_state(rng, 300, with_storage=0.6, max_slots=80))
    block = random_block(rng, h.state, 80, 1)
    ks = sorted(block)
    keys = np.frombuffer(b"".join(ks), np.uint8).reshape(-1, 32)
    accs = np.zeros(len(ks), oracle.ACCOUNT_DTYPE)
    flags = np.zeros(len(ks), np.uint8)
    sk, sv, offs = [], [], [0]
    for i, k in enumerate(ks):
        flags[i], accs[i] = block[k][0], block[k][1]
        for s in sorted(block[k][2]):
            sk.append(s)
            sv.append(int(block[k][2][s]).to_bytes(32, "big"))
        offs.append(len(sk))
    skeys = np.frombuffer(b"".join(sk), np.uint8).reshape(-1, 32) if sk else np.zeros((0, 32), np.uint8)
    svals = np.frombuffer(b"".join(sv), np.uint8).reshape(-1, 32) if sv else np.zeros((0, 32), np.uint8)
    _, au, _, su, _, _ = h.ds.apply(keys, accs, flags, skeys, svals, np.array(offs, np.uint64), want_updates=True)
    arows = tables.account_trie_rows(au, tables.KEYS_PACKED)
    assert [k for k, _ in arows] == sorted(k for k, _ in arows) and len(arows) == len(au)
    srows = tables.storage_trie_rows(su, keys, tables.KEYS_PACKED)
    assert len(srows) == len(su)
    order = [(k, v[:33]) for k, v in srows]
    assert order == sorted(order)
    assert {k for k, _ in srows} <= set(ks)
    h.ds.close()


def test_bad_arguments_are_rejected_not_crashed(eng):
    """The C ABI never aborts: null pointers, malformed segment tables, unsorted keys and misuse of a plain state as a
    sharded one come back as error codes, and the state stays usable."""
    import ctypes as C
    from reth_b200 import DynamicState
    from reth_b200._lib import B200Error
    lib, ctx = eng.lib, eng.ctx
    h = C.c_void_p()
    assert lib.b200_dstate_create(ctx, None, None, 5, None, None, None, C.byref(h), None) < 0          # null inputs, n > 0
    assert lib.b200_dstate_create(None, None, None, 0, None, None, None, C.byref(h), None) < 0         # null context
    rng = np.random.default_rng(1)
    state = random_state(rng, 50)
    _, keys, accs, skeys, svals, offs = flatten(state)
    bad_offs = offs.copy()
    bad_offs[3] = bad_offs[-1] + 5                                                                      # not monotone
    assert lib.b200_dstate_create(ctx, keys.ctypes.data, accs.ctypes.data, len(keys), skeys.ctypes.data, svals.ctypes.data,
                                  bad_offs.ctypes.data, C.byref(h), None) < 0
    ds = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    root = ds.root()
    with pytest.raises(B200Error):                                                                      # unsorted account keys
        ds.apply(keys[[5, 2]], accs[[5, 2]], None, np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8), np.zeros(3, np.uint64))
    with pytest.raises(ValueError):                                                                     # segment table vs slot rows
        ds.apply(keys[:2], accs[:2], None, np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8), np.array([0, 0, 9], np.uint64))
    with pytest.raises(B200Error):                                                                      # segment table not monotone
        ds.apply(keys[:2], accs[:2], None, skeys[:4], svals[:4], np.array([0, 5, 4], np.uint64))
    with pytest.raises(B200Error):                                                                      # not a sharded state
        ds.frontier()
    assert lib.b200_dstate_apply(ds.handle, None, None, None, 3, None, None, None, None, None, None, None, None, None, None) < 0
    assert lib.b200_dstate_account_proofs(ds.handle, None, 4, None) < 0
    assert lib.b200_dstate_root(None, None) < 0
    lib.b200_dstate_destroy(None)                                                                       # no-op
    lib.b200_proofs_release(None)
    assert ds.root() == root                                                                            # untouched by all of the above
    assert ds.apply(keys[:1], accs[:1], None, np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8), np.zeros(2, np.uint64)) == root
    ds.close()


def test_device_resident_block(eng):
    """b200_dstate_apply_dev: the block's arrays and the root buffer live in device memory; same result as the host-pointer
    call on a twin state."""
    from reth_b200 import DynamicState
    rng = np.random.default_rng(66)
    state = random_state(rng, 400)
    _, keys, accs, skeys, svals, offs = flatten(state)
    a = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    b = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    for step in range(3):
        block = random_block(rng, state, 60, step + 1)
        ks = sorted(block)
        m = len(ks)
        bk = np.frombuffer(b"".join(ks), np.uint8).reshape(m, 32)
        ba = np.zeros(m, oracle.ACCOUNT_DTYPE)
        bf = np.zeros(m, np.uint8)
        sk, sv, so = [], [], [0]
        for i, k in enumerate(ks):
            bf[i], ba[i] = block[k][0], block[k][1]
            for s in sorted(block[k][2]):
                sk.append(s)
                sv.append(int(block[k][2][s]).to_bytes(32, "big"))
            so.append(len(sk))
        bsk = np.frombuffer(b"".join(sk), np.uint8).reshape(-1, 32) if sk else np.zeros((1, 32), np.uint8)[:0]
        bsv = np.frombuffer(b"".join(sv), np.uint8).reshape(-1, 32) if sv else np.zeros((1, 32), np.uint8)[:0]
        so = np.array(so, np.uint64)
        root_host = a.apply(bk, ba, bf, bsk, bsv, so)
        pad = lambda x: x if len(x) else np.zeros((1, 32), np.uint8)            # a valid address even when empty
        ptrs, hold = to_device_ptrs((bk, ba, bf, pad(bsk), pad(bsv), so, np.zeros(32, np.uint8)))
        b.apply_dev(ptrs[0], ptrs[1], ptrs[2], m, ptrs[3], ptrs[4], ptrs[5], len(sk), ptrs[6])
        assert b.root() == root_host
        assert b.accounts() == a.accounts() and b.slots() == a.slots()
        # (the host model only steers the block generator)
        for k in ks:
            fl, acc, slots = block[k]
            if not (fl & EXISTS):
                state.pop(k, None)
            elif not (fl & UNCHANGED) or k in state:
                cur_a, cur_s = (state[k] if (fl & UNCHANGED) else (acc, state[k][1] if k in state else {}))
                cur_s = {} if (fl & WIPED) else dict(cur_s)
                for s_, v in slots.items():
                    if v == 0:
                        cur_s.pop(s_, None)
                    else:
                        cur_s[s_] = v
                state[k] = (cur_a, cur_s)
    a.close()
    b.close()
