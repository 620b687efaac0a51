"""Merkle proofs and multiproofs of a sharded state (b200_dstate_sharded_multiproof, b200_dstate_frontier_masks).

Every case runs 1 to 16 shards in one process (tests/test_gpu_dstate.py's ShardedHarness layout) next to an unsharded
twin of the same accounts, and checks:
(a) each shard answers the targets routed to it, and every target's node list (RLP, order, depth, masks) and storage root
    equal b200_dstate_multiproof of the same targets on the twin;
(b) the merged dicts of all shards equal the twin's multiproof dict;
(c) keccak of every account proof's first node is root_from_frontier(merged), which is the oracle's root."""
import ctypes as C

import numpy as np
import pytest

import oracle
from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, ShardedHarness, acct, random_block, random_state, rkey
from tests.test_gpu_proofs import MAINNET_PROOF_HEADS, MAINNET_TARGET, TESTSPEC
from tests.test_gpu_witness import block_arrays, make_state
from tests.util import alloc_to_flat

pytestmark = [pytest.mark.gpu]
H = bytes.fromhex


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def gather(shards, world):
    """-> (merged (16, 68), hash mask, tree mask): what the all-gather of ShardedDynamicStateRoot.multiproof gives."""
    merged = np.zeros((16, 68), np.uint8)
    hm = tm = 0
    for r, ds in enumerate(shards):
        fr = ds.frontier()
        mine = [b for b in range(16) if b * world // 16 == r]
        merged[mine] = fr[mine]
        h, t = ds.frontier_masks()
        assert not (h | t) & ~sum(1 << b for b in mine)
        hm, tm = hm | h, tm | t
    return merged, hm, tm


def route(key, merged, world):
    """the rank that answers a target: the owner of its bucket, or of the only non-empty bucket"""
    nonempty = [k for k in range(16) if merged[k, 34]]
    k = key[0] >> 4
    if k not in nonempty and len(nonempty) == 1:
        k = nonempty[0]
    return k * world // 16


def check_proofs(eng, shards, world, u, targets, root):
    merged, hm, tm = gather(shards, world)
    assert eng.root_from_frontier(merged) == root
    want = u.multiproof(targets)
    got = {"account_subtree": {}, "branch_node_masks": {}, "storages": {}}
    for r, ds in enumerate(shards):
        share = {a: s for a, s in targets.items() if route(a, merged, world) == r}
        part = ds.sharded_multiproof(merged, hm, tm, share, with_nodes=True)
        assert part == u.multiproof(share, with_nodes=True), r             # (a)
        for nodes in part["account_nodes"]:                                  # (c)
            assert oracle.keccak256(nodes[0][1]) == root
        for name in got:
            got[name].update(part[name])
    assert got == want                                                       # (b)


class Rig:
    def __init__(self, eng, state, world):
        self.eng, self.world = eng, world
        self.h = ShardedHarness(eng, state, world)                           # checks the initial root against the oracle
        self.u = make_state(eng, self.h.state)

    def root(self):
        return self.h.global_root()

    def commit(self, block):
        self.h.commit(block)
        assert self.u.apply(*block_arrays(block)) == self.root()

    def check(self, targets):
        check_proofs(self.eng, self.h.shards, self.world, self.u, targets, self.root())

    def targets(self, rng, n_present=12):
        return make_targets(rng, self.h.state, n_present)

    def close(self):
        for ds in self.h.shards:
            ds.close()
        self.u.close()


def with_prefix(rng, prefix_nibbles):
    k = bytearray(rkey(rng))
    for i, x in enumerate(prefix_nibbles):
        k[i // 2] = (k[i // 2] & 0x0F) | (x << 4) if i % 2 == 0 else (k[i // 2] & 0xF0) | x
    return bytes(k)


def nibble_at(key, i):
    return (key[i // 2] >> 4) if i % 2 == 0 else key[i // 2] & 15


def make_targets(rng, state, n_present=12):
    """present accounts (with and without storage, present and absent slots), absent keys in held and empty buckets, near
    misses sharing 1 to 6 nibbles with a present key, and absent accounts with slot targets"""
    keys = sorted(state)
    t = {}
    for i in rng.permutation(len(keys))[:n_present]:
        k = keys[i]
        slots = sorted(state[k][1])
        t[k] = slots[:3] + [rkey(rng)]                                      # present and absent slots (or absent only)
    if keys:
        t[keys[0]] = []                                                      # an account target without slot targets
        base = keys[int(rng.integers(0, len(keys)))]
        for n in range(1, 7):                                                # near misses
            nibs = [nibble_at(base, i) for i in range(n)] + [nibble_at(base, n) ^ int(rng.integers(1, 16))]
            t[with_prefix(rng, nibs)] = [rkey(rng)]
    buckets = {k[0] >> 4 for k in keys}
    for b in range(16):
        if b in buckets and rng.random() < 0.3:
            t[with_prefix(rng, [b])] = []                                    # absent, held bucket
        elif b not in buckets and rng.random() < 0.5:
            t[with_prefix(rng, [b])] = [rkey(rng), rkey(rng)]                # absent, empty bucket, with slots
    return t


def bucket_state(rng, prefixes, n_each, slots=True):
    st = {}
    for p in prefixes:
        for _ in range(n_each):
            sl = {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(int(rng.integers(0, 6)))} if slots and rng.random() < 0.5 else {}
            st[with_prefix(rng, p)] = (acct(int(rng.integers(0, 9)), int(rng.integers(1, 2**50))), sl)
    return st


WORLDS = [1, 2, 4, 8, 16]


@pytest.mark.parametrize("world", WORLDS)
def test_random_state_through_blocks(eng, world):
    """all 16 buckets, then commit chains"""
    rng = np.random.default_rng(7100 + world)
    rig = Rig(eng, random_state(rng, 300), world)
    rig.check(rig.targets(rng, 30))
    for step in range(3):
        rig.commit(random_block(rng, rig.h.state, 40, step + 1))
        rig.check(rig.targets(rng, 20))
    rig.close()


@pytest.mark.parametrize("world", WORLDS)
def test_bucket_shapes(eng, world):
    """the empty state; one bucket topped by a leaf, a depth-1 branch or a branch four nibbles deep; two buckets"""
    rng = np.random.default_rng(7200 + world)
    shapes = [
        {},
        bucket_state(rng, [[0xA]], 1),
        bucket_state(rng, [[0x3]], 25),
        bucket_state(rng, [[0x5, 0x1, 0xC, 0x7]], 20),
        bucket_state(rng, [[0x0], [0xF, 0x2, 0x2]], 10),
        bucket_state(rng, [[0x6], [0x9]], 1),
    ]
    for st in shapes:
        rig = Rig(eng, st, world)
        rig.check(rig.targets(rng))
        rig.close()


@pytest.mark.parametrize("world", [2, 4, 16])
def test_commits_that_create_empty_and_destroy_buckets(eng, world):
    rng = np.random.default_rng(7300 + world)
    rig = Rig(eng, bucket_state(rng, [[0x3, 0x3]], 15), world)
    rig.check(rig.targets(rng))
    other = with_prefix(rng, [0xC, 0x1])
    steps = [
        {other: (EXISTS, acct(2, 2), {rkey(rng): 9})},                                    # a second bucket appears
        {with_prefix(rng, [0xC, 0x1]): (EXISTS, acct(3, 3), {})},                          # ... and grows a branch
        {k: (0, acct(0), {}) for k in sorted(rig.h.state)},                                 # bucket 3 destroyed
        {with_prefix(rng, [0x8]): (EXISTS, acct(4, 4), {}), with_prefix(rng, [0xE]): (EXISTS, acct(5, 5), {})},
    ]
    for block in steps:
        rig.commit(block)
        rig.check(rig.targets(rng))
    keys = sorted(rig.h.state)
    rig.commit({k: (0, acct(0), {}) for k in keys[1:]})                                     # one account left
    rig.check(rig.targets(rng))
    rig.commit({k: (EXISTS | UNCHANGED, acct(0), {rkey(rng): 5}) for k in keys[:1]})
    rig.commit({k: (EXISTS | WIPED, rig.h.state[k][0].copy(), {}) for k in keys[:1]})
    rig.check(rig.targets(rng))
    rig.commit({k: (0, acct(0), {}) for k in sorted(rig.h.state)})                          # empty state
    rig.check(rig.targets(rng))
    rig.close()


def flat_shards(eng, flat, world):
    from reth_b200 import DynamicState
    keys, accs, skeys, svals, offs = flat
    shards = []
    for r in range(world):
        idx = [i for i in range(len(keys)) if (keys[i][0] >> 4) * world // 16 == r]
        offs_r, sk, sv = [0], [], []
        for i in idx:
            a, b = int(offs[i]), int(offs[i + 1])
            sk.append(skeys[a:b])
            sv.append(svals[a:b])
            offs_r.append(offs_r[-1] + b - a)
        cat = lambda xs: np.concatenate(xs).reshape(-1, 32) if xs else np.zeros((0, 32), np.uint8)
        shards.append(DynamicState.create(eng, keys[idx].reshape(-1, 32), accs[idx], cat(sk), cat(sv), np.array(offs_r, np.uint64),
                                          sharded=True))
    return shards


def sharded_account_proof(eng, shards, world, key):
    merged, hm, tm = gather(shards, world)
    r = route(key, merged, world)
    return shards[r].sharded_multiproof(merged, hm, tm, {key: []}, with_nodes=True)["account_nodes"][0]


@pytest.mark.parametrize("world", [1, 4, 16])
def test_reth_proof_vectors(eng, golden_allocs, world):
    """crates/trie/db/tests/proof.rs: testspec_proofs and mainnet_genesis_account_proof, from the shards"""
    shards = flat_shards(eng, alloc_to_flat(golden_allocs["testspec"]["alloc"]), world)
    for addr, proof in TESTSPEC.items():
        nodes = sharded_account_proof(eng, shards, world, oracle.keccak256(H(addr)))
        assert [n[1].hex() for n in nodes] == proof, addr
    for ds in shards:
        ds.close()
    shards = flat_shards(eng, alloc_to_flat(golden_allocs["mainnet"]["alloc"]), world)
    merged, _, _ = gather(shards, world)
    assert eng.root_from_frontier(merged) == H(golden_allocs["mainnet"]["state_root"])
    nodes = sharded_account_proof(eng, shards, world, oracle.keccak256(H(MAINNET_TARGET)))
    assert len(nodes) == len(MAINNET_PROOF_HEADS)
    for (_, node, _), (head, tail, length) in zip(nodes, MAINNET_PROOF_HEADS):
        assert node.hex().startswith(head) and node.hex().endswith(tail) and len(node) == length
    for ds in shards:
        ds.close()


@pytest.mark.parametrize("world", [2, 16])
def test_storage_proofs_on_a_shard(eng, world):
    rng = np.random.default_rng(7400 + world)
    rig = Rig(eng, random_state(rng, 120, with_storage=0.8), world)
    for k in sorted(rig.h.state)[::7] + [rkey(rng)]:
        slots = np.frombuffer(b"".join(sorted(rig.h.state[k][1])[:4] + [rkey(rng)]) if k in rig.h.state else rkey(rng),
                              np.uint8).reshape(-1, 32)
        ds = rig.h.shards[rig.h.rank_of(k)]
        assert ds.storage_proofs(k, slots) == rig.u.storage_proofs(k, slots)
    rig.close()


def test_errors_leave_the_shard_unchanged(eng):
    from reth_b200._lib import ERR_INVALID_ARG, FrontierEntry, Proofs
    world = 4
    rng = np.random.default_rng(7500)
    state = random_state(rng, 200)
    rig = Rig(eng, state, world)
    ctl = ShardedHarness(eng, state, world)
    lib = eng.lib
    merged, hm, tm = gather(rig.h.shards, world)
    stale = merged.copy()
    ds = rig.h.shards[1]                                                     # buckets 4..7
    own = [4, 5, 6, 7]

    def call(target, fr=None, masks=None, n=None, offs=None, slot_targets=0, null=()):
        """-> the status of b200_dstate_sharded_multiproof; on error both outputs must be zeroed.  null: arguments passed
        as NULL ("merged", "keys", "offsets")."""
        fr = merged if fr is None else fr
        h, t = (hm, tm) if masks is None else masks
        keys = np.frombuffer(target, np.uint8).reshape(-1, 32)
        n = len(keys) if n is None else n
        offs = np.array([0] * n + [slot_targets], np.uint64) if offs is None else offs
        skeys = np.zeros((1, 32), np.uint8)
        pa, ps = Proofs(), Proofs()
        pa.n_targets = ps.n_targets = 99
        sroots = np.zeros((max(len(keys), 1), 32), np.uint8)
        arr = None if "merged" in null else (FrontierEntry * 16).from_buffer_copy(np.ascontiguousarray(fr).tobytes())
        rc = lib.b200_dstate_sharded_multiproof(target_ds[0].handle, arr, h, t, None if "keys" in null else keys.ctypes.data, n,
                                                None if "offsets" in null else offs.ctypes.data, skeys.ctypes.data,
                                                C.byref(pa), sroots.ctypes.data, C.byref(ps))
        if rc:
            assert (pa.n_targets, pa.n_nodes, ps.n_targets, ps.n_nodes) == (0, 0, 0, 0)
            assert not (pa._owner or ps._owner)
        lib.b200_proofs_release(C.byref(pa))
        lib.b200_proofs_release(C.byref(ps))
        return rc

    target_ds = [ds]
    mine = with_prefix(rng, [5])
    assert call(mine) == 0
    target_ds[0] = rig.u                                                     # an unsharded state
    assert call(mine) == ERR_INVALID_ARG
    h, t = C.c_uint16(), C.c_uint16()
    assert lib.b200_dstate_frontier_masks(rig.u.handle, C.byref(h), C.byref(t)) == ERR_INVALID_ARG
    target_ds[0] = ds
    assert lib.b200_dstate_frontier_masks(ds.handle, None, C.byref(t)) == ERR_INVALID_ARG
    for arg in ("merged", "keys", "offsets"):                                # null pointers
        assert call(mine, null=(arg,)) == ERR_INVALID_ARG
    for b in own:                                                            # one flipped byte in an own entry
        if merged[b, 34]:
            for pos in (1, 5, 33, 40, 67):                                   # as_child, its padding, as_root
                bad = merged.copy()
                bad[b, pos] ^= 0x01
                assert call(mine, fr=bad) == ERR_INVALID_ARG
            bad = merged.copy()
            bad[b] = 0                                                       # own bucket given as empty
            assert call(mine, fr=bad) == ERR_INVALID_ARG
            bit = 1 << b
            assert call(mine, masks=(hm ^ bit, tm)) == ERR_INVALID_ARG     # wrong own mask bits
            assert call(mine, masks=(hm, tm ^ bit)) == ERR_INVALID_ARG
    bad = merged.copy()
    bad[0, 34] = 31                                                          # malformed entries
    assert call(mine, fr=bad) == ERR_INVALID_ARG
    bad = merged.copy()
    bad[0, 0] = 34
    assert call(mine, fr=bad) == ERR_INVALID_ARG
    foreign = with_prefix(rng, [0xB])
    assert call(foreign) == ERR_INVALID_ARG                                  # a foreign target
    assert call(b"".join([mine, foreign])) == ERR_INVALID_ARG
    assert call(mine, n=1 << 24, offs=np.zeros((1 << 24) + 1, np.uint64)) == ERR_INVALID_ARG
    assert call(mine, slot_targets=1 << 24) == ERR_INVALID_ARG              # the target limits
    # an empty-bucket target when the only non-empty bucket is foreign: a state of one bucket (0xB, rank 2)
    single = ShardedHarness(eng, {with_prefix(rng, [0xB, 1]): (acct(1, 1), {}), with_prefix(rng, [0xB, 2]): (acct(1, 2), {})}, world)
    m1, h1, t1 = gather(single.shards, world)
    target_ds[0] = single.shards[1]
    assert call(with_prefix(rng, [5]), fr=m1, masks=(h1, t1)) == ERR_INVALID_ARG
    target_ds[0] = single.shards[2]
    assert call(with_prefix(rng, [5]), fr=m1, masks=(h1, t1)) == 0
    for s in single.shards:
        s.close()
    # a stale frontier, from before a commit that changes this shard's buckets
    block = {with_prefix(rng, [6, 1]): (EXISTS, acct(9, 9), {rkey(rng): 3})}
    rig.h.commit(block)
    ctl.commit(block)
    target_ds[0] = ds
    assert call(mine, fr=stale) == ERR_INVALID_ARG
    # every shard unchanged: same root and frontier as the control, same next apply and TrieUpdates
    for a, b in zip(rig.h.shards, ctl.shards):
        assert a.root() == b.root() and np.array_equal(a.frontier(), b.frontier())
    block = random_block(rng, rig.h.state, 30, 5)
    for r, (a, b) in enumerate(zip(rig.h.shards, ctl.shards)):
        part = {k: v for k, v in block.items() if rig.h.rank_of(k) == r}
        arrays = block_arrays(part)
        ra, rb = a.apply(*arrays, want_updates=True), b.apply(*arrays, want_updates=True)
        assert ra[:5] == rb[:5] and np.array_equal(ra[5], rb[5])
    for s in ctl.shards:
        s.close()
    rig.close()
