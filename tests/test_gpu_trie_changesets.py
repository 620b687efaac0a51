"""Trie changesets of a block from the resident state (b200_dstate_trie_changesets; reth's compute_trie_changesets,
crates/trie/trie/src/changesets.rs:50-239).  The reference restates compute_trie_changesets and
storage_trie_wiped_changeset_iter over the oracle's tables of the parent state (tests/test_gpu_dstate.py's `model`): every
changed path looked up exactly, and a deleted storage trie merged by path with every node it stored."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, acct, clustered_slots, model, random_block, random_state, rkey
from tests.test_gpu_overlay_updates import tables_after
from tests.test_gpu_witness import apply_to_model, block_arrays, make_state

pytestmark = [pytest.mark.gpu]

NONE = (0, 0, 0, ())


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def norm(records):
    return [(r[0], bytes(r[1]), r[2], r[3], r[4], tuple(r[5])) for r in records]


def lookup(db, p):
    return (db[p][0], db[p][1], db[p][2], tuple(db[p][3])) if p in db else NONE


def reference(tables, acct_paths, storage):
    """compute_trie_changesets over the parent's tables: seek_exact per path; a deleted trie is the merge-join of its changed
    paths with every node it stores (storage_trie_wiped_changeset_iter)"""
    _, adb, sdb = tables
    acct_out = [(0, p) + lookup(adb, p) for p in acct_paths]
    stor_out = []
    for i, a in enumerate(sorted(storage)):
        deleted, paths = storage[a]
        db = sdb.get(a, {})
        ps = sorted(set(paths) | set(db)) if deleted else paths
        stor_out += [(i, p) + lookup(db, p) for p in ps]
    return acct_out, stor_out


def changeset_input(block, res):
    """the paths and is_deleted flags of one block's updates (the result tuple of apply / overlay_roots with updates)"""
    ks = sorted(block)
    _, au, ar, su, sr, deleted = res
    acct_paths = sorted({r[1] for r in au} | set(ar))
    per = {}
    for r in su:
        per.setdefault(r[0], set()).add(r[1])
    for e, p in sr:
        per.setdefault(e, set()).add(p)
    storage = {ks[i]: (bool(deleted[i]), sorted(per.get(i, ()))) for i in range(len(ks)) if deleted[i] or per.get(i)}
    return acct_paths, storage


def reverted(tables_post, storage, got):
    """the changesets written back over the tables after the block: Some upserts, None deletes, a deleted trie cleared first"""
    adb, sdb = tables_post
    adb, sdb = dict(adb), {k: dict(v) for k, v in sdb.items()}
    acct_recs, stor_recs = got
    for r in acct_recs:
        if r[2]:
            adb[r[1]] = (r[2], r[3], r[4], list(r[5]))
        else:
            adb.pop(r[1], None)
    addrs = sorted(storage)
    for i, a in enumerate(addrs):
        if storage[a][0] and any(r[0] == i for r in stor_recs):
            sdb.pop(a, None)
    for r in stor_recs:
        db = sdb.setdefault(addrs[r[0]], {})
        if r[2]:
            db[r[1]] = (r[2], r[3], r[4], list(r[5]))
        else:
            db.pop(r[1], None)
    return adb, {k: v for k, v in sdb.items() if v}


def tables_eq(a, b):
    canon = lambda db: {p: (v[0], v[1], v[2], tuple(v[3])) for p, v in db.items()}
    return canon(a[0]) == canon(b[0]) and {k: canon(v) for k, v in a[1].items()} == {k: canon(v) for k, v in b[1].items()}


def check(ds, pre, block, res):
    acct_paths, storage = changeset_input(block, res)
    got = tuple(norm(x) for x in ds.trie_changesets(acct_paths, storage))
    want = reference(pre, acct_paths, storage)
    assert got[0] == want[0]
    assert got[1] == want[1]
    post = tables_after(pre, block, res)
    assert tables_eq(reverted(post, storage, got), (pre[1], {k: v for k, v in pre[2].items() if v}))
    return got


@pytest.mark.parametrize("n0,touch", [(5, 6), (300, 40), (3000, 250)])
def test_random_blocks_match_the_reference_and_revert(eng, n0, touch):
    rng = np.random.default_rng(1300 + n0)
    state = random_state(rng, n0, with_storage=0.5, max_slots=40)
    ds, twin = make_state(eng, state), make_state(eng, state)
    try:
        for step in range(4):
            block = random_block(rng, state, touch, step + 1)
            arrays = block_arrays(block)
            pre = model(state)
            root = ds.root()
            ov = ds.overlay_roots([arrays], want_updates=True)[0]
            check(ds, pre, block, ov)
            ap = twin.apply(*arrays, want_updates=True)
            check(ds, pre, block, ap)
            assert ds.root() == root == pre[0]
            after = ds.apply(*arrays, want_updates=True)  # the queries left nothing behind: same root, same updates
            assert after[:5] == ap[:5] and (after[5] == ap[5]).all()
            state = apply_to_model(state, block)
    finally:
        ds.close()
        twin.close()


def branch_paths(keys):
    """every branch of the trie over `keys` (sorted): the common prefix of neighbours, as nibble paths"""
    nib = lambda k: bytes(x for b in k for x in (b >> 4, b & 15))
    ks = [nib(k) for k in sorted(keys)]
    out = set()
    for a, b in zip(ks, ks[1:]):
        l = next(i for i in range(64) if a[i] != b[i])
        out.add(a[:l])
    return out, ks


def test_lookup_shapes(eng):
    """every kind of path against its own tries: stored branches, unstored branches, paths ending inside an extension, paths
    below a leaf, length 1 and the deepest stored branch; absent accounts, deleted or not; an empty storage"""
    rng = np.random.default_rng(1401)
    state = {k: v for k, v in random_state(rng, 400, with_storage=0.3, max_slots=30).items() if k[0] != 0xAB}
    for c in range(40):  # clustered accounts: long extensions and deep branches
        k = bytes([0xAB, 0xCD, 0xE0 | (c >> 4)]) + bytes([c & 15 | 0x50]) + rkey(rng)[4:]
        state[k] = (acct(c, 3), {})
    rich = sorted(state)[7]
    state[rich] = (state[rich][0], {s: 5 for s in clustered_slots(rng, 12)})
    empty, empty2 = sorted(state)[9], sorted(state)[11]
    state[empty] = (state[empty][0], {})
    state[empty2] = (state[empty2][0], {})
    tables = model(state)
    ds = make_state(eng, state)
    try:
        branches, nibs = branch_paths(list(state))
        stored = set(tables[1])
        paths = set(stored) | branches | {bytes([n]) for n in range(16)}
        paths |= {k[:l] for k in nibs[::5] for l in (2, 5, 33, 63)}
        paths |= {bytes([0xA, 0xB]), bytes([0xA, 0xB, 0xC])}  # inside the extension above the clustered branch
        paths.discard(b"")
        assert branches - stored - {b""}, "the state has unstored branches"
        assert bytes([0xA, 0xB, 0xC, 0xD, 0xE]) in branches
        deepest = max(stored, key=len)
        sbranches, snibs = branch_paths(list(state[rich][1]))
        spaths = sorted((set(tables[2].get(rich, {})) | sbranches | {k[:l] for k in snibs for l in (1, 3, 40)}) - {b""})
        absent = [rkey(rng) for _ in range(2)]
        storage = {rich: (False, spaths), empty: (False, [bytes([1]), bytes([2, 3])]), absent[0]: (False, [bytes([4])]),
                   absent[1]: (True, [bytes([5])]), empty2: (True, [])}
        acct_paths = sorted(paths)
        got = tuple(norm(x) for x in ds.trie_changesets(acct_paths, storage))
        want = reference(tables, acct_paths, storage)
        assert got == want
        by_path = {r[1]: r for r in got[0]}
        assert by_path[deepest][2] and by_path[bytes([0xA, 0xB])][2:] == NONE
        assert all(by_path[p][2:] == NONE for p in branches - stored - {b""})
        assert all(by_path[k[:63]][2:] == NONE for k in nibs[::5])
    finally:
        ds.close()


def test_destroyed_contract_spanning_several_levels_and_ctas(eng):
    """a deleted storage trie of 60 000 slots: the breadth-first walk runs over several levels, each wider than one CTA"""
    rng = np.random.default_rng(1402)
    state = random_state(rng, 50, with_storage=0.5, max_slots=20)
    big = sorted(state)[3]
    state[big] = (state[big][0], {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(60_000)})
    tables = model(state)
    assert len(tables[2][big]) > 2000
    ds = make_state(eng, state)
    try:
        block = {big: (0, acct(0), {}), sorted(state)[5]: (EXISTS | WIPED, state[sorted(state)[5]][0], {rkey(rng): 9})}
        res = ds.overlay_roots([block_arrays(block)], want_updates=True)[0]
        check(ds, tables, block, res)
        # a new path in the wiped trie, merged in at its place (None)
        new = sorted(tables[2][big])[100] + bytes([3] * 10)
        got = norm(ds.trie_changesets([], {big: (True, [new])})[1])
        want = reference(tables, [], {big: (True, [new])})[1]
        assert got == want and len(got) == len(tables[2][big]) + 1
    finally:
        ds.close()


def test_empty_state_and_empty_updates(eng):
    ds = make_state(eng, {})
    try:
        assert ds.trie_changesets([], {}) == ([], [])
        got = ds.trie_changesets([bytes([1]), bytes([1, 2])], {b"\x11" * 32: (True, [bytes([3])]), b"\x22" * 32: (False, [])})
        assert norm(got[0]) == [(0, bytes([1])) + NONE, (0, bytes([1, 2])) + NONE]
        assert norm(got[1]) == [(0, bytes([3])) + NONE]
    finally:
        ds.close()


def test_reth_cases_through_the_host_mirror(eng):
    """changesets.rs:246-476 restated on real tries, through DynamicStateRoot: empty updates, account changesets, storage
    changesets, a wiped storage, a wiped storage with a new path; then the live-path order overlay_root_with_updates ->
    trie_changesets -> commit, and the changesets revert the commit's tables"""
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage, StateRoot
    from reth_b200.trie import StorageTrieUpdatesSorted, TrieUpdates, TrieUpdatesSorted
    rng = np.random.default_rng(1403)
    rk = lambda: bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    base = HashedPostState()
    for _ in range(400):
        k = rk()
        base.accounts[k] = Account(int(rng.integers(0, 50)), int(rng.integers(1, 2**62)))
        if rng.random() < 0.3:
            base.storages[k] = HashedStorage(False, {rk(): int(rng.integers(1, 2**62)) for _ in range(int(rng.integers(1, 300)))})
    dsr = DynamicStateRoot(eng, base.into_sorted())
    _, full = StateRoot(eng, base.into_sorted()).root_with_updates()
    adb = dict(full.account_nodes)
    sdb = {k: dict(v.storage_nodes) for k, v in full.storage_tries.items() if v.storage_nodes}
    try:
        assert dsr.trie_changesets(TrieUpdatesSorted()) == TrieUpdatesSorted()
        ap = sorted(sorted(adb)[:2] + [bytes([15] * 9)])  # two stored paths and one where nothing is stored
        got = dsr.trie_changesets(TrieUpdatesSorted([(p, None) for p in ap]))
        assert got.account_nodes == [(p, adb.get(p)) for p in ap] and not got.storage_tries
        addr = max(sdb, key=lambda a: len(sdb[a]))
        sp = sorted(sdb[addr])[:2] + [bytes([15] * 9)]
        su = StorageTrieUpdatesSorted(False, [(p, None) for p in sorted(sp)])
        got = dsr.trie_changesets(TrieUpdatesSorted([], {addr: su}))
        assert got.storage_tries == {addr: StorageTrieUpdatesSorted(False, [(p, sdb[addr].get(p)) for p in sorted(sp)])}
        got = dsr.trie_changesets(TrieUpdatesSorted([], {addr: StorageTrieUpdatesSorted(True, [])}))
        assert got.storage_tries == {addr: StorageTrieUpdatesSorted(True, sorted(sdb[addr].items()))}
        new = bytes([15] * 9)
        got = dsr.trie_changesets(TrieUpdatesSorted([], {addr: StorageTrieUpdatesSorted(True, [(new, None)])}))
        assert got.storage_tries == {addr: StorageTrieUpdatesSorted(True, sorted(list(sdb[addr].items()) + [(new, None)]))}
        # the live path: updates of the candidate block, its changesets, then the commit
        post = HashedPostState()
        live = sorted(base.accounts)
        for i in rng.choice(len(live), 40, replace=False):
            post.accounts[live[i]] = Account(1, 2)
        for k in [k for k in base.storages if k not in post.accounts][:5]:
            post.storages[k] = HashedStorage(False, {rk(): 3, next(iter(base.storages[k].storage)): 0})
        post.accounts[addr] = None
        post.storages[addr] = HashedStorage(True, {})
        root, upd = dsr.overlay_root_with_updates(post)
        cs = dsr.trie_changesets(upd)
        assert dsr.trie_changesets(upd.into_sorted()) == cs
        assert isinstance(upd, TrieUpdates) and cs.storage_tries[addr].is_deleted
        assert dsr.commit(post)[0] == root
        # the tables after the commit, with the changesets written back, are the tables before it
        for p in upd.removed_nodes:
            adb.pop(p, None)
        adb.update(upd.account_nodes)
        for k, st in upd.storage_tries.items():
            if st.is_deleted:
                sdb.pop(k, None)
            cur = sdb.setdefault(k, {})
            for p in st.removed_nodes:
                cur.pop(p, None)
            cur.update(st.storage_nodes)
        for p, n in cs.account_nodes:
            adb.pop(p, None) if n is None else adb.__setitem__(p, n)
        for k, st in cs.storage_tries.items():
            if st.is_deleted:
                sdb.pop(k, None)
            cur = sdb.setdefault(k, {})
            for p, n in st.storage_nodes:
                cur.pop(p, None) if n is None else cur.__setitem__(p, n)
        assert adb == dict(full.account_nodes)
        assert {k: v for k, v in sdb.items() if v} == {k: dict(v.storage_nodes) for k, v in full.storage_tries.items() if v.storage_nodes}
    finally:
        dsr.close()


def test_large_block_on_a_large_state(eng):
    """a 20 000-entry block on a 100 000-account state"""
    rng = np.random.default_rng(1404)
    state = random_state(rng, 100_000, with_storage=0.2, max_slots=12)
    tables = model(state)
    ds = make_state(eng, state)
    try:
        block = random_block(rng, state, 20_000, 1)
        assert len(block) > 15_000
        res = ds.overlay_roots([block_arrays(block)], want_updates=True)[0]
        got = check(ds, tables, block, res)
        assert len(got[0]) > 4000
    finally:
        ds.close()


def test_errors_release_and_zero_the_outputs(eng):
    from reth_b200._lib import B200Error, Stats, Updates
    state = random_state(np.random.default_rng(1405), 50)
    ds = make_state(eng, state)
    lib = eng.lib
    k1, k2 = b"\x10" * 32, b"\x20" * 32

    def call(alen, apk, n_a, keys, flags, n_s, offs, slen, spk, handle=None):
        au, su = Updates(), Updates()
        au.n_nodes = su.n_nodes = 77
        p = lambda a: None if a is None else a.ctypes.data
        rc = lib.b200_dstate_trie_changesets(handle or ds.handle, p(alen), p(apk), n_a, p(keys), p(flags), n_s, p(offs), p(slen), p(spk),
                                             C.byref(au), C.byref(su), C.byref(Stats()))
        if rc:
            assert au.n_nodes == su.n_nodes == 0 and not au._owner and not su._owner and not au.trie_id
        else:
            lib.b200_updates_release(C.byref(au))
            lib.b200_updates_release(C.byref(su))
        return rc

    def paths(*ps):
        from reth_b200.engine import _pack_paths
        return _pack_paths(list(ps))

    z0 = np.zeros(1, np.uint64)
    keys2 = np.frombuffer(k1 + k2, np.uint8).reshape(2, 32).copy()
    l, pk = paths(bytes([1]), bytes([1, 2]))
    try:
        assert call(l, pk, 2, None, None, 0, z0, None, None) == 0
        assert call(None, None, 0, None, None, 0, z0, None, None) == 0
        ERR_INVALID, ERR_UNSORTED = -3, -4
        assert call(None, pk, 2, None, None, 0, z0, None, None) == ERR_INVALID            # null with a count
        assert call(l, pk, 2, None, None, 0, None, None, None) == ERR_INVALID             # no offsets
        assert call(l, pk, 2, None, None, 2, np.array([0, 0, 0], np.uint64), None, None) == ERR_INVALID  # null keys
        assert call(None, None, 0, keys2, None, 2, np.array([1, 1, 1], np.uint64), l, pk) == ERR_INVALID  # not from 0
        assert call(None, None, 0, keys2, None, 2, np.array([0, 2, 1], np.uint64), l, pk) == ERR_INVALID  # not monotone
        bad = l.copy(); bad[0] = 0
        assert call(bad, pk, 2, None, None, 0, z0, None, None) == ERR_INVALID             # length 0
        bad = l.copy(); bad[1] = 64
        assert call(bad, pk, 2, None, None, 0, z0, None, None) == ERR_INVALID             # length over 63
        bad = pk.copy(); bad[0, 0] |= 0x0F
        assert call(l, bad, 2, None, None, 0, z0, None, None) == ERR_INVALID              # padding after an odd length
        bad = pk.copy(); bad[1, 31] = 1
        assert call(l, bad, 2, None, None, 0, z0, None, None) == ERR_INVALID              # padding in the last byte
        rl, rp = paths(bytes([1, 2]), bytes([1]))
        assert call(rl, rp, 2, None, None, 0, z0, None, None) == ERR_UNSORTED            # extension before its prefix
        dl, dp = paths(bytes([1]), bytes([1]))
        assert call(dl, dp, 2, None, None, 0, z0, None, None) == ERR_UNSORTED            # duplicate
        assert call(None, None, 0, keys2, None, 2, np.array([0, 1, 2], np.uint64), rl, rp) == 0  # one path per trie: fine
        assert call(None, None, 0, keys2, None, 2, np.array([0, 2, 2], np.uint64), rl, rp) == ERR_UNSORTED  # inside a trie
        keys_rev = keys2[::-1].copy()
        assert call(None, None, 0, keys_rev, None, 2, np.array([0, 0, 0], np.uint64), None, None) == ERR_UNSORTED
        keys_dup = np.stack([keys2[0], keys2[0]])
        assert call(None, None, 0, keys_dup, None, 2, np.array([0, 0, 0], np.uint64), None, None) == ERR_UNSORTED
        assert call(l, pk, 1 << 31, None, None, 0, z0, None, None) == ERR_INVALID         # 2^31-1 or more records
        with pytest.raises(B200Error):
            ds.trie_changesets([bytes([2]), bytes([1])], {})
    finally:
        ds.close()
    # a sharded state
    from reth_b200 import DynamicState
    from tests.test_gpu_dstate import flatten
    _, keys, accs, skeys, svals, offs = flatten(state)
    sh = DynamicState.create(eng, keys, accs, skeys, svals, offs, sharded=True)
    try:
        assert call(l, pk, 2, None, None, 0, z0, None, None, handle=sh.handle) == -3
    finally:
        sh.close()
