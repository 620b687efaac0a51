"""Frontier entries of a sharded state after candidate blocks, the shards unchanged (b200_dstate_overlay_frontiers).

Every case checks, for every shard of 1 to 16 in one process (tests/test_gpu_dstate.py's ShardedHarness layout):
(a) the 16 entries after every block equal, byte for byte, the frontier of a twin shard after `apply` of that block;
(b) the root merged over all shards equals `overlay_roots` of the whole block on an unsharded state and the oracle's root;
(c) every shard afterwards has the root and frontier it had before, and its next `apply` returns the same root and
    TrieUpdates as on a control shard that never saw the call."""
import ctypes as C

import numpy as np
import pytest

import oracle
from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, ShardedHarness, acct, flatten, random_block, random_state, rkey
from tests.test_gpu_witness import apply_to_model, block_arrays, make_state

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def oracle_root(state):
    _, keys, accs, skeys, svals, offs = flatten(state)
    return oracle.state_root_full(keys, accs, skeys, svals, offs)


def sharded_state(eng, state):
    from reth_b200 import DynamicState
    _, keys, accs, skeys, svals, offs = flatten(state)
    return DynamicState.create(eng, keys, accs, skeys, svals, offs, sharded=True)


class Rig:
    """The shards under test, control shards that never see an overlay call (a ShardedHarness, which also checks the
    initial global root against the oracle), and an unsharded state of the same accounts."""

    def __init__(self, eng, state, world):
        self.eng, self.world = eng, world
        self.ctl = ShardedHarness(eng, state, world)
        self.state = self.ctl.state
        self.shards = [sharded_state(eng, self.part_state(r)) for r in range(world)]
        self.u = make_state(eng, self.state)

    def part_state(self, r):
        return {k: v for k, v in self.state.items() if self.ctl.rank_of(k) == r}

    def part(self, block, r):
        return {k: v for k, v in block.items() if self.ctl.rank_of(k) == r}

    def owned(self, r):
        return [b for b in range(16) if b * self.world // 16 == r]

    def check(self, blocks):
        """(a), (b) and the first half of (c) for a batch of sibling blocks on the current state."""
        before = [(ds.root(), ds.frontier()) for ds in self.shards]
        frs = [ds.overlay_frontiers([block_arrays(self.part(b, r)) for b in blocks]) for r, ds in enumerate(self.shards)]
        u_roots = self.u.overlay_roots([block_arrays(b) for b in blocks])
        for (root, fr), ds in zip(before, self.shards):
            assert ds.root() == root
            assert np.array_equal(ds.frontier(), fr)
        for r, fr in enumerate(frs):
            assert fr.shape == (len(blocks), 16, 68) and fr.dtype == np.uint8
        for i, block in enumerate(blocks):
            merged = np.zeros((16, 68), np.uint8)
            for r in range(self.world):
                mine = self.part(block, r)
                if mine:
                    twin = sharded_state(self.eng, self.part_state(r))
                    twin.apply(*block_arrays(mine))
                    want = twin.frontier()
                    twin.close()
                else:
                    want = before[r][1]
                assert np.array_equal(frs[r][i], want), (i, r)
                others = [b for b in range(16) if b not in self.owned(r)]
                assert not frs[r][i][others].any()
                merged[self.owned(r)] = frs[r][i][self.owned(r)]
            root = self.eng.root_from_frontier(merged)
            assert root == u_roots[i] == oracle_root(apply_to_model(self.state, block)), i
        return frs

    def commit(self, block):
        """(c): the shards under test and the control shards apply the block alike; the unsharded state follows."""
        for r, (ds, cs) in enumerate(zip(self.shards, self.ctl.shards)):
            arrays = block_arrays(self.part(block, r))
            got, want = ds.apply(*arrays, want_updates=True), cs.apply(*arrays, want_updates=True)
            assert got[:5] == want[:5]
            assert np.array_equal(got[5], want[5])
            assert np.array_equal(ds.frontier(), cs.frontier())
        self.ctl.state = self.state = apply_to_model(self.state, block)
        assert self.u.apply(*block_arrays(block)) == self.ctl.global_root() == oracle_root(self.state)

    def close(self):
        for ds in self.shards + self.ctl.shards + [self.u]:
            ds.close()


def in_bucket(rng, nib, prefix=()):
    """a random key in top-nibble bucket `nib`, its next nibbles fixed to `prefix`"""
    k = bytearray(rkey(rng))
    nibs = (nib,) + tuple(prefix)
    for i, n in enumerate(nibs):
        k[i // 2] = (k[i // 2] & 0x0F) | (n << 4) if i % 2 == 0 else (k[i // 2] & 0xF0) | n
    return bytes(k)


@pytest.mark.parametrize("world", [1, 2, 8, 16])
def test_random_chains(eng, world):
    """Each step: the overlay of a block and of a sibling, then the commit of the block, so that later overlays run on
    arenas with freed and reused slots."""
    rng = np.random.default_rng(1200 + world)
    rig = Rig(eng, random_state(rng, 300), world)
    for step in range(4):
        block = random_block(rng, rig.state, 40, step + 1)
        rig.check([block, random_block(rng, rig.state, 25, step + 1)])
        rig.commit(block)
    rig.close()


def test_sibling_batches_with_empty_blocks(eng):
    rng = np.random.default_rng(1301)
    rig = Rig(eng, random_state(rng, 200), 4)
    blocks = [random_block(rng, rig.state, 20, 1), {}, random_block(rng, rig.state, 5, 2), {}, {}]
    frs = rig.check(blocks)
    for r, ds in enumerate(rig.shards):
        assert np.array_equal(frs[r][1], ds.frontier()) and np.array_equal(frs[r][4], ds.frontier())
    rig.check([{}])
    for ds in rig.shards:                                     # no blocks: nothing to do
        assert ds.overlay_frontiers([]).shape == (0, 16, 68)
    rig.commit(blocks[0])
    rig.check(blocks[2:])
    rig.close()


def test_bucket_shapes(eng):
    """A block that empties a bucket, one that creates a bucket in a shard that held none, a bucket left as one account
    leaf, and buckets whose top after the block is a branch the block never reaches (a hash item of the fold): two
    nibbles deep (below an extension over nibble 1) and five nibbles deep.  A hash item one nibble deep cannot occur:
    every key of a block passes through its bucket's depth-1 branch."""
    rng = np.random.default_rng(77)
    st = {}
    for _ in range(6):                                        # bucket 3: emptied
        st[in_bucket(rng, 3)] = (acct(1, 1), {rkey(rng): 5} if rng.random() < 0.5 else {})
    for _ in range(5):                                        # bucket 5: reduced to one account leaf
        st[in_bucket(rng, 5)] = (acct(2, 2), {})
    for _ in range(8):                                        # bucket 9: an untouched branch at depth 2 below nibble 9.7
        st[in_bucket(rng, 9, (7,))] = (acct(3, 3), {rkey(rng): 1})
    lone9 = in_bucket(rng, 9, (2,))
    st[lone9] = (acct(4, 4), {})
    for _ in range(6):                                        # bucket 10: an untouched branch at depth 5 below 10.1.2.3.4
        st[in_bucket(rng, 10, (1, 2, 3, 4))] = (acct(5, 5), {})
    lone10 = in_bucket(rng, 10, (6,))
    st[lone10] = (acct(6, 6), {rkey(rng): 9})
    for _ in range(20):                                       # other buckets, 0xC excluded
        k = rkey(rng)
        if k[0] >> 4 not in (3, 5, 9, 10, 12):
            st[k] = (acct(7, 7), {})
    rig = Rig(eng, st, 4)                                     # rank 3 holds buckets 12..15: 0xC is empty
    b3 = sorted(k for k in rig.state if k[0] >> 4 == 3)
    b5 = sorted(k for k in rig.state if k[0] >> 4 == 5)
    empties = {k: (0, acct(0), {}) for k in b3}
    creates = {in_bucket(rng, 12): (EXISTS, acct(8, 8), {rkey(rng): 3}), in_bucket(rng, 12): (EXISTS, acct(9, 9), {})}
    one_leaf = {k: (0, acct(0), {}) for k in b5[1:]}
    blind2 = {lone9: (0, acct(0), {})}
    blind5 = {lone10: (0, acct(0), {})}
    alone = {in_bucket(rng, 13): (EXISTS, acct(1, 1), {})}    # a single leaf in a new bucket
    mixed = dict(empties)
    mixed.update(creates)
    mixed.update(blind5)
    rig.check([empties, creates, one_leaf, blind2, blind5, alone, mixed])
    for block in (empties, creates, blind2, one_leaf, blind5):
        rig.commit(block)
        rig.check([{k: (EXISTS, acct(11, 11), {}) for k in list(rig.state)[:3]}, blind5, empties])
    rig.close()


def test_degenerate_states(eng):
    """test_sharded_state_degenerate_buckets' shapes: every account in one bucket, a second bucket that appears and
    vanishes, a single account, the empty state."""
    rng = np.random.default_rng(31)
    st = {}
    for _ in range(40):
        k = bytearray(rkey(rng))
        k[0] = 0x30 | (k[0] & 15)
        st[bytes(k)] = (acct(1, 5), {})
    rig = Rig(eng, st, 4)
    other = bytearray(rkey(rng))
    other[0] = 0xC1
    steps = [{bytes(other): (EXISTS, acct(2, 2), {rkey(rng): 9})}, {bytes(other): (0, acct(0), {})}]
    for block in steps:
        rig.check([block])
        rig.commit(block)
    block = {k: (0, acct(0), {}) for k in sorted(rig.state)[1:]}
    rig.check([block])
    rig.commit(block)                                         # a single account left
    block = {k: (0, acct(0), {}) for k in sorted(rig.state)}
    back = {rkey(rng): (EXISTS, acct(3, 3), {}) for _ in range(3)}
    rig.check([block, back])
    rig.commit(block)                                         # the empty state
    rig.check([back, {}, {rkey(rng): (EXISTS | UNCHANGED, acct(0), {rkey(rng): 1})}])
    rig.commit(back)
    rig.close()
    empty = Rig(eng, {}, 2)                                   # created empty
    empty.check([back, {}])
    empty.close()


def test_entry_kinds(eng):
    """Storage-only entries, destroyed accounts with storage, wipes with and without refill, and entries of absent
    accounts that change nothing (storage of an account that does not exist, destruction of one)."""
    rng = np.random.default_rng(5)
    rig = Rig(eng, random_state(rng, 160, with_storage=0.8, max_slots=30), 4)
    with_storage = sorted(k for k, (_, s) in rig.state.items() if s)
    sto_only, destroyed, wiped, refill = with_storage[:6], with_storage[6:10], with_storage[10:13], with_storage[13:16]
    blocks = [
        {k: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in list(rig.state[k][1])[:2]} | {rkey(rng): 4}) for k in sto_only},
        {k: (0, acct(0), {}) for k in destroyed},
        {k: (EXISTS | WIPED, rig.state[k][0].copy(), {}) for k in wiped},
        {k: (EXISTS | WIPED, rig.state[k][0].copy(), {rkey(rng): 6}) for k in refill},
        {rkey(rng): (EXISTS | UNCHANGED, acct(0), {rkey(rng): 7}) for _ in range(5)},
        {rkey(rng): (0, acct(0), {}) for _ in range(5)},
        {k: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in rig.state[k][1]}) for k in with_storage[16:20]},  # storage emptied
    ]
    rig.check(blocks)
    for block in blocks:
        rig.commit(block)
    rig.close()


def test_large_block_and_wide_batch(eng):
    """A block of more than 8192 entries on each of two shards, and 32 siblings in one call."""
    rng = np.random.default_rng(8192)
    rig = Rig(eng, random_state(rng, 9000, with_storage=0.2, max_slots=8), 2)
    big = random_block(rng, rig.state, 3000, 1)
    for i in range(18000):                                    # new accounts, some with storage
        big[rkey(rng)] = (EXISTS, acct(1, i + 1), {rkey(rng): i + 1} if i % 4 == 0 else {})
    assert all(len(rig.part(big, r)) > 8192 for r in range(2))
    rig.check([big])
    rig.commit(big)
    rig.check([random_block(rng, rig.state, 30, b + 2) for b in range(32)])
    rig.close()


def test_errors_zero_the_output(eng):
    from reth_b200._lib import ERR_INVALID_ARG, ERR_UNSORTED, FrontierEntry
    from reth_b200.engine import _ptr, block_batch_arrays
    rng = np.random.default_rng(3)
    state = random_state(rng, 60)
    ds, flat = sharded_state(eng, state), make_state(eng, state)
    blocks = [block_arrays(random_block(rng, state, 8, 1)), block_arrays(random_block(rng, state, 8, 2))]
    lib = eng.lib

    def call(target, args, n=2, out=True):
        buf = (FrontierEntry * 32)()
        C.memset(buf, 0xAB, C.sizeof(buf))
        r = lib.b200_dstate_overlay_frontiers(target.handle, n, *(_ptr(a) for a in args), buf if out else None, None)
        return r, np.frombuffer(bytes(buf), np.uint8)

    good = block_batch_arrays(blocks)
    r, out = call(ds, good)
    assert r == 0 and not (out[:2 * 16 * 68] == 0xAB).all()
    assert call(flat, good)[0] == ERR_INVALID_ARG                       # an unsharded state
    assert call(ds, good, out=False)[0] == ERR_INVALID_ARG              # no output
    assert call(ds, good, n=0, out=False)[0] == 0                       # nothing to do
    cases = []
    bad = list(good)
    bad[3] = good[3].copy()
    bad[3][0] = 1                                                       # block offsets not from 0
    cases.append((bad, ERR_INVALID_ARG))
    bad = list(good)
    bad[3] = good[3].copy()
    bad[3][1], bad[3][2] = bad[3][2] + 1, bad[3][2]                     # not monotone
    cases.append((bad, ERR_INVALID_ARG))
    bad = list(good)
    bad[6] = good[6].copy()
    bad[6][0] = 1                                                       # slot offsets not from 0
    cases.append((bad, ERR_INVALID_ARG))
    bad = list(good)
    bad[0] = good[0].copy()
    lo = int(good[3][1])
    bad[0][[lo, lo + 1]] = bad[0][[lo + 1, lo]]                         # account keys out of order in block 1
    cases.append((bad, ERR_UNSORTED))
    bad = list(good)
    bad[4] = good[4].copy()
    a = int(np.argmax(np.diff(good[6].astype(np.int64)) >= 2))          # an entry with two slots or more
    assert good[6][a + 1] - good[6][a] >= 2
    s0 = int(good[6][a])
    bad[4][[s0, s0 + 1]] = bad[4][[s0 + 1, s0]]                         # slot keys out of order
    cases.append((bad, ERR_UNSORTED))
    bad = list(good)
    bad[1] = None                                                       # accounts missing
    cases.append((bad, ERR_INVALID_ARG))
    for args, code in cases:
        r, out = call(ds, args)
        assert r == code
        assert not out[:2 * 16 * 68].any()                              # zeroed on any error
    r, out = call(flat, good)
    assert not out[:2 * 16 * 68].any()
    root, fr = ds.root(), ds.frontier()
    assert np.array_equal(ds.overlay_frontiers(blocks)[0], ds.overlay_frontiers(blocks[:1])[0])
    assert ds.root() == root and np.array_equal(ds.frontier(), fr)
    ds.close()
    flat.close()
