"""Execution witness of a block over a sharded state (b200_dstate_witness_root_kept, b200_dstate_sharded_witness).

Every case runs 1 to 16 shards in one process (tests/test_gpu_dstate.py's ShardedHarness layout) next to an unsharded
twin of the same accounts, in both modes, with and without always_include_root, and checks:
(a) every shard's map is a subset of b200_dstate_witness of the whole block on the twin;
(b) the union of the shards' maps equals the twin's map;
(c) the union, the parent root and the block give, statelessly (b200_witness_roots), the root of the twin's apply;
(d) no call changes a shard: root, frontier and root masks stay, and the next commit is checked against the oracle
    (ShardedHarness.commit: root and the union of the shards' TrieUpdates)."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, ShardedHarness, acct, random_block, random_state, rkey
from tests.test_gpu_sharded_proofs import bucket_state, gather, route, with_prefix
from tests.test_gpu_witness import block_arrays, make_state

pytestmark = [pytest.mark.gpu]
MODES = ("legacy", "canonical")
WORLDS = [1, 2, 4, 8, 16]


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def root_kept(shards, world, block, mode):
    """the OR of every rank's kept mask, each over the entries of its own buckets"""
    kept = 0
    for r, ds in enumerate(shards):
        kept |= ds.witness_root_kept(block_arrays({k: v for k, v in block.items() if (k[0] >> 4) * world // 16 == r}), mode)
    return kept


def part_of(block, merged, world, r):
    """rank r's part, routed as ShardedDynamicStateRoot.witness routes it: the answering rank, and with two or more
    non-empty buckets every rank for an entry of an empty bucket"""
    every = sum(1 for b in range(16) if merged[b, 34]) >= 2
    return {k: v for k, v in block.items() if route(k, merged, world) == r or (every and not merged[k[0] >> 4, 34])}


def shard_maps(shards, world, block, mode, always):
    """every shard's part of the witness"""
    merged, hm, tm = gather(shards, world)
    kept = root_kept(shards, world, block, mode)
    return [ds.sharded_witness(merged, hm, tm, kept, block_arrays(part_of(block, merged, world, r)), mode,
                               always_include_root_node=always and not block)
            for r, ds in enumerate(shards)]


def snapshot(shards):
    return [(ds.root(), ds.frontier().tobytes(), ds.frontier_masks()) for ds in shards]


class Rig:
    def __init__(self, eng, state, world):
        self.eng, self.world = eng, world
        self.h = ShardedHarness(eng, state, world)                           # checks the initial root against the oracle
        self.u = make_state(eng, self.h.state)

    def root(self):
        return self.h.global_root()

    def check(self, block):
        """(a), (b) and the unchanged shards for both modes and both root flags -> {mode: union without the root flag}"""
        arrays = block_arrays(block)
        before = snapshot(self.h.shards)
        unions = {}
        for mode in MODES:
            for always in (False, True):
                want = self.u.witness(*arrays, mode=mode, always_include_root_node=always)
                union = {}
                for r, part in enumerate(shard_maps(self.h.shards, self.world, block, mode, always)):
                    assert all(want.get(h) == rlp for h, rlp in part.items()), (mode, always, r)     # (a)
                    union.update(part)
                assert union == want, (mode, always, len(set(want) - set(union)), len(set(union) - set(want)))  # (b)
                if not always:
                    unions[mode] = union
        assert snapshot(self.h.shards) == before                             # (d)
        return unions

    def step(self, block):
        """check the block, commit it (twin and oracle agree), then (c)"""
        parent = self.root()
        unions = self.check(block)
        self.h.commit(block)
        new = self.u.apply(*block_arrays(block))
        assert new == self.root()
        for mode, union in unions.items():
            roots, status = self.eng.witness_roots([parent], [union], [block_arrays(block)])
            assert status[0] == 0 and roots[0].tobytes() == new, mode           # (c)

    def close(self):
        for ds in self.h.shards:
            ds.close()
        self.u.close()


def keys_in(state, nibble):
    return sorted(k for k in state if k[0] >> 4 == nibble)


@pytest.mark.parametrize("world", WORLDS)
def test_random_blocks_and_commit_chains(eng, world):
    """all sixteen buckets: random blocks (destroyed accounts, wiped storages, storage-only changes, ignored entries)"""
    rng = np.random.default_rng(8100 + world)
    rig = Rig(eng, random_state(rng, 300, with_storage=0.5), world)
    for step in range(3):
        rig.step(random_block(rng, rig.h.state, 40, step + 1))
    rig.close()


@pytest.mark.parametrize("world", WORLDS)
def test_bucket_shapes(eng, world):
    """the empty state; one bucket topped by a leaf, a depth-1 branch or a branch four nibbles deep under a root
    extension; two buckets: random blocks, a block that touches one bucket only (empty parts), the empty block"""
    rng = np.random.default_rng(8200 + world)
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
        rig.check({})
        live = sorted(rig.h.state)
        if live:
            k = live[0]
            rig.check({k: (EXISTS, acct(77, 7), {rkey(rng): 3})})              # one bucket touched, the other parts empty
        rig.step(random_block(rng, rig.h.state, 12, 1))
        rig.step(random_block(rng, rig.h.state, 12, 2))
        rig.close()


@pytest.mark.parametrize("world", [1, 2, 4, 16])
def test_removals_at_the_root_branch(eng, world):
    """removals that empty a bucket, and that leave the root branch with one bucket, unseen and seen; a bucket emptied and
    refilled in one block (Legacy reveals the other bucket at depth 0, Canonical does not); a single-leaf bucket left"""
    rng = np.random.default_rng(8300 + world)
    st = bucket_state(rng, [[0x2], [0x7, 0x7], [0xD]], 6)
    destroy = lambda ks: {k: (0, acct(0), {}) for k in ks}
    cases = [
        destroy(keys_in(st, 0x2)),                                              # one bucket emptied, two left
        destroy(keys_in(st, 0x2) + keys_in(st, 0xD)),                           # one left, unseen
        {**destroy(keys_in(st, 0x2) + keys_in(st, 0xD)), keys_in(st, 0x7)[0]: (EXISTS, acct(5, 5), {})},   # ... seen
        {**destroy(keys_in(st, 0x2) + keys_in(st, 0xD)), with_prefix(rng, [0x7, 0x1]): (0, acct(0), {})},  # ... seen by an absent key
        {**destroy(keys_in(st, 0x2) + keys_in(st, 0xD)), with_prefix(rng, [0x2, 0x9]): (EXISTS, acct(1, 1), {})},  # refilled
        # an empty bucket filled: Legacy reveals bucket 7, Canonical keeps two children
        {**destroy(keys_in(st, 0x2) + keys_in(st, 0xD)), with_prefix(rng, [0xE, 0x4]): (EXISTS, acct(1, 1), {})},
        # an empty account and an ignored entry in empty buckets insert nothing: both modes reveal bucket 7
        {**destroy(keys_in(st, 0x2) + keys_in(st, 0xD)), with_prefix(rng, [0xE, 0x4]): (EXISTS, acct(0), {}),
         with_prefix(rng, [0x0, 0x4]): (EXISTS | UNCHANGED, acct(0), {rkey(rng): 2})},
        {**destroy(keys_in(st, 0x2)[1:] + keys_in(st, 0xD)), keys_in(st, 0x2)[0]: (EXISTS, acct(0), {})},  # empty account: removal
        destroy(keys_in(st, 0x2) + keys_in(st, 0x7) + keys_in(st, 0xD)),        # every bucket emptied
    ]
    for block in cases:
        rig = Rig(eng, st, world)
        rig.step(block)
        rig.close()
    # storage-only removals: an empty account loses its last slot and with it its leaf
    st2 = {with_prefix(rng, [0x4]): (acct(0), {rkey(rng): 9}), with_prefix(rng, [0xB, 1]): (acct(3, 3), {}),
           with_prefix(rng, [0xB, 2]): (acct(4, 4), {})}
    k4 = keys_in(st2, 0x4)[0]
    for fl, a in ((EXISTS | UNCHANGED, acct(0)), (EXISTS, acct(0)), (EXISTS | WIPED, acct(0))):
        rig = Rig(eng, st2, world)
        rig.step({k4: (fl, a, {s: 0 for s in st2[k4][1]})})
        rig.close()
    # the last bucket shrinks to a single leaf, then goes
    rig = Rig(eng, bucket_state(rng, [[0x9]], 4), world)
    ks = sorted(rig.h.state)
    rig.step(destroy(ks[1:]))
    rig.step({**destroy(ks[:1]), with_prefix(rng, [0x1]): (EXISTS, acct(2, 2), {})})
    rig.step(destroy(sorted(rig.h.state)))
    rig.step({})
    rig.close()


@pytest.mark.parametrize("world", [2, 8])
def test_absent_ignored_and_destroyed_entries(eng, world):
    rng = np.random.default_rng(8400 + world)
    rig = Rig(eng, random_state(rng, 80, with_storage=0.7), world)
    live = sorted(rig.h.state)
    block = {
        rkey(rng): (0, acct(0), {rkey(rng): 5}),                                 # destroyed, absent, with slots
        rkey(rng): (EXISTS | UNCHANGED, acct(0), {rkey(rng): 7}),               # ignored
        rkey(rng): (EXISTS, acct(0), {}),                                        # an empty account, absent: removal of nothing
        live[0]: (0, acct(0), {s: 1 for s in list(rig.h.state[live[0]][1])[:2]}),  # destroyed with slot entries
        live[1]: (EXISTS | WIPED, rig.h.state[live[1]][0].copy(), {}),           # wiped
        live[2]: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in rig.h.state[live[2]][1]}),   # every slot zeroed
    }
    rig.step(block)
    rig.close()


def test_kept_mask_paths_agree(eng):
    """the kept mask of a part that cannot remove anything is read from the frontier; with a possible removal the walks
    run: both give the mask of the unsharded root branch's surviving children"""
    rng = np.random.default_rng(8500)
    world = 4
    rig = Rig(eng, bucket_state(rng, [[0x1], [0x5], [0x9], [0xC]], 3), world)
    upserts = {k: (EXISTS, acct(9, 9), {}) for k in sorted(rig.h.state)[::2]}
    upserts[with_prefix(rng, [0xE])] = (EXISTS, acct(1, 1), {})                # a new bucket (Canonical only)
    held = sum(1 << b for b in (0x1, 0x5, 0x9, 0xC))
    assert root_kept(rig.h.shards, world, upserts, "legacy") == held
    assert root_kept(rig.h.shards, world, upserts, "canonical") == held | 1 << 0xE
    with_removal = dict(upserts)
    with_removal.update({k: (0, acct(0), {}) for k in keys_in(rig.h.state, 0x5)})
    assert root_kept(rig.h.shards, world, with_removal, "legacy") == held & ~(1 << 0x5)
    assert root_kept(rig.h.shards, world, with_removal, "canonical") == (held & ~(1 << 0x5)) | 1 << 0xE
    rig.step(with_removal)
    rig.close()


@pytest.mark.parametrize("world", [2, 4])
def test_kept_bits_of_empty_buckets(eng, world):
    """Every bit of root_kept is checked by some rank: a bucket empty in merged by every rank (Legacy: the bit is 0;
    Canonical: it is set exactly when the part inserts there, every part holding every entry of an empty bucket).  A
    mask of the other mode, a spurious bit or an entry of an empty bucket missing from a part makes a call fail, with the
    output zeroed; a correct one gives the unsharded witness."""
    from reth_b200._lib import ERR_INVALID_ARG, B200Error
    rng = np.random.default_rng(8700 + world)
    rig = Rig(eng, bucket_state(rng, [[0x2], [0x7, 0x7], [0xD]], 6), world)
    shards = rig.h.shards
    merged, hm, tm = gather(shards, world)
    new = with_prefix(rng, [0xE, 0x4])
    block = {**{k: (0, acct(0), {}) for k in keys_in(rig.h.state, 0x2) + keys_in(rig.h.state, 0xD)}, new: (EXISTS, acct(1, 1), {})}
    kept = {mode: root_kept(shards, world, block, mode) for mode in MODES}
    assert kept["legacy"] == 1 << 0x7 and kept["canonical"] == 1 << 0x7 | 1 << 0xE

    def statuses(mode, k, parts=None):
        out = []
        for r, ds in enumerate(shards):
            part = part_of(block, merged, world, r) if parts is None else parts[r]
            try:
                ds.sharded_witness(merged, hm, tm, k, block_arrays(part), mode)
                out.append(0)
            except B200Error as e:
                out.append(e.status)
        return out

    assert statuses("legacy", kept["legacy"]) == [0] * world and statuses("canonical", kept["canonical"]) == [0] * world
    bad = [ERR_INVALID_ARG] * world
    assert statuses("legacy", kept["canonical"]) == bad                 # the Canonical mask in a Legacy call
    assert statuses("canonical", kept["legacy"]) == bad                 # the Legacy mask in a Canonical call
    for mode in MODES:
        assert statuses(mode, kept[mode] | 1 << 0xF) == bad             # a spurious bit of an empty bucket
    owner_only = [{k: v for k, v in block.items() if route(k, merged, world) == r} for r in range(world)]
    st = statuses("canonical", kept["canonical"], owner_only)           # the insert given to one rank only
    assert st.count(0) == 1 and st.count(ERR_INVALID_ARG) == world - 1
    rig.step(block)
    rig.close()


def test_errors_leave_the_shards_unchanged(eng):
    from reth_b200._lib import ERR_INVALID_ARG, ERR_UNSORTED, FrontierEntry, Stats, Witness
    world = 4
    rng = np.random.default_rng(8600)
    state = random_state(rng, 200)
    rig = Rig(eng, state, world)
    ctl = ShardedHarness(eng, state, world)
    lib = eng.lib
    shards = rig.h.shards
    ds = shards[1]                                                           # buckets 4..7
    merged, hm, tm = gather(shards, world)
    stale = merged.copy()
    mine = {with_prefix(rng, [5]): (EXISTS, acct(3, 3), {rkey(rng): 1}),
            keys_in(rig.h.state, 6)[0]: (0, acct(0), {})}
    kept = root_kept(shards, world, mine, "legacy")

    def call(block, target=None, fr=None, masks=None, k=None, mode=0, null=(), swap=False):
        """-> the status of b200_dstate_sharded_witness; on error the output must be zeroed"""
        target = ds if target is None else target
        fr = merged if fr is None else fr
        h, t = (hm, tm) if masks is None else masks
        keys, accs, flags, sk, sv, offs = block_arrays(block)
        if swap:
            keys = keys[::-1].copy()
        w = Witness()
        w.n = 99
        arr = None if "merged" in null else (FrontierEntry * 16).from_buffer_copy(np.ascontiguousarray(fr).tobytes())
        rc = lib.b200_dstate_sharded_witness(target.handle, arr, h, t, kept if k is None else k,
                                             None if "keys" in null else keys.ctypes.data, accs.ctypes.data, flags.ctypes.data,
                                             len(keys), sk.ctypes.data, sv.ctypes.data, offs.ctypes.data, mode, 0, C.byref(w),
                                             C.byref(Stats()))
        if rc:
            assert (w.n, bool(w.hashes32), bool(w.rlp_offset), bool(w.rlp), w._owner) == (0, False, False, False, None)
        lib.b200_witness_release(C.byref(w))
        return rc

    def kept_call(block, target=None, mode=0, swap=False):
        keys, accs, flags, sk, sv, offs = block_arrays(block)
        if swap:
            keys = keys[::-1].copy()
        out = C.c_uint16(0xFFFF)
        rc = lib.b200_dstate_witness_root_kept((target or ds).handle, keys.ctypes.data, accs.ctypes.data, flags.ctypes.data, len(keys),
                                               sk.ctypes.data, sv.ctypes.data, offs.ctypes.data, mode, C.byref(out))
        if rc:
            assert out.value == 0
        return rc

    assert call(mine) == 0 and call(mine, mode=1, k=root_kept(shards, world, mine, "canonical")) == 0
    assert call(mine, target=rig.u) == ERR_INVALID_ARG                         # an unsharded state
    assert kept_call(mine, target=rig.u) == ERR_INVALID_ARG
    with pytest.raises(Exception):
        ds.witness(*block_arrays(mine))                                        # b200_dstate_witness on a shard
    for mode in (2, -1):                                                       # a bad mode
        assert call(mine, mode=mode) == ERR_INVALID_ARG and kept_call(mine, mode=mode) == ERR_INVALID_ARG
    for arg in ("merged", "keys"):                                             # null pointers
        assert call(mine, null=(arg,)) == ERR_INVALID_ARG
    for b in (4, 5, 6, 7):
        if not merged[b, 34]:
            continue
        bad = merged.copy()
        bad[b, 3] ^= 0x01                                                      # a foreign or corrupted entry
        assert call(mine, fr=bad) == ERR_INVALID_ARG
        bad = merged.copy()
        bad[b] = 0                                                             # own bucket given as empty
        assert call(mine, fr=bad) == ERR_INVALID_ARG
        assert call(mine, masks=(hm ^ 1 << b, tm)) == ERR_INVALID_ARG          # wrong masks
        assert call(mine, masks=(hm, tm ^ 1 << b)) == ERR_INVALID_ARG
        assert call(mine, k=kept ^ 1 << b) == ERR_INVALID_ARG                  # a stale kept mask
        assert call({}, k=kept ^ 1 << b) == ERR_INVALID_ARG                    # ... also for an empty part
    assert call(mine, k=kept ^ 1 << 0xB) == 0                                   # (a foreign bucket's bit is not this shard's)
    foreign = with_prefix(rng, [0xB])
    assert call({foreign: (EXISTS, acct(1), {})}) == ERR_INVALID_ARG            # an entry of another shard
    assert call({**mine, foreign: (EXISTS, acct(1), {})}) == ERR_INVALID_ARG
    two = {with_prefix(rng, [5, 1]): (EXISTS, acct(1, 1), {}), with_prefix(rng, [5, 2]): (EXISTS, acct(2, 2), {})}
    assert call(two, swap=True) == ERR_UNSORTED                                 # unsorted keys
    assert kept_call(two, swap=True) == ERR_UNSORTED                            # (no removal: the host path)
    two_rm = {**two, keys_in(rig.h.state, 6)[0]: (0, acct(0), {})}
    assert kept_call(two_rm, swap=True) == ERR_UNSORTED                         # (a removal: the device path)
    assert call(two_rm, swap=True) == ERR_UNSORTED
    # a stale frontier, from before a commit that changes this shard's buckets
    block = {with_prefix(rng, [6, 1]): (EXISTS, acct(9, 9), {rkey(rng): 3})}
    rig.h.commit(block)
    ctl.commit(block)
    rig.u.apply(*block_arrays(block))
    assert call(mine, fr=stale) == ERR_INVALID_ARG
    # every shard unchanged: same root and frontier as the control, same next apply and TrieUpdates
    for a, b in zip(shards, ctl.shards):
        assert a.root() == b.root() and np.array_equal(a.frontier(), b.frontier()) and a.frontier_masks() == b.frontier_masks()
    block = random_block(rng, rig.h.state, 30, 5)
    for r, (a, b) in enumerate(zip(shards, ctl.shards)):
        arrays = block_arrays({k: v for k, v in block.items() if rig.h.rank_of(k) == r})
        ra, rb = a.apply(*arrays, want_updates=True), b.apply(*arrays, want_updates=True)
        assert ra[:5] == rb[:5] and np.array_equal(ra[5], rb[5])
    for s in ctl.shards:
        s.close()
    rig.close()
