"""TrieUpdates of candidate blocks on top of the resident state, without changing it (b200_dstate_overlay_roots_with_updates;
reth's StateRoot::overlay_root_with_updates).  The reference is always a twin state built from the same state, on which the
same block is committed with DynamicState.apply(..., want_updates=True); the tables are the oracle's full node sets
(tests/test_gpu_dstate.py's `model`)."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, acct, clustered_slots, flatten, model, random_block, random_state, rkey
from tests.test_gpu_witness import EMPTY_ROOT, KECCAK, apply_to_model, block_arrays, make_state

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def twin_apply(eng, state, block):
    twin = make_state(eng, state)
    try:
        return twin.apply(*block_arrays(block), want_updates=True)
    finally:
        twin.close()


def tables_after(pre, block, res):
    """the pre-state's tables with one block's records applied: removed paths, then is_deleted, then updated records (as
    Harness.commit does)"""
    _, adb, sdb = pre
    adb, sdb = dict(adb), {k: dict(v) for k, v in sdb.items()}
    ks = sorted(block)
    _, au, ar, su, sr, deleted = res
    for p in ar:
        adb.pop(p, None)
    for r in au:
        adb[r[1]] = r[2:]
    for entry, p in sr:
        sdb.get(ks[entry], {}).pop(p, None)
    for i, k in enumerate(ks):
        if deleted[i]:
            sdb.pop(k, None)
    for r in su:
        sdb.setdefault(ks[r[0]], {})[r[1]] = r[2:]
    return adb, {k: v for k, v in sdb.items() if v}


def check_block(state, block, got, want, pre=None):
    """one block's overlay result against the twin apply's, and the tables it gives against the oracle's"""
    pre = pre or model(state)
    root, au, ar, su, sr, deleted = got
    assert root == want[0]
    assert set(ar) == set(want[2])
    assert len(set(ar)) == len(ar)
    assert set(sr) == set(want[4])
    assert np.array_equal(deleted, want[5])
    ks = sorted(block)
    for mine, theirs, old in (({r[1]: r[2:] for r in au}, {r[1]: r[2:] for r in want[1]}, lambda p: pre[1].get(p)),
                              ({(ks[r[0]], r[1]): r[2:] for r in su}, {(ks[r[0]], r[1]): r[2:] for r in want[3]},
                               lambda p: pre[2].get(p[0], {}).get(p[1]))):
        for p in mine.keys() | theirs.keys():
            if p in mine and p in theirs:
                assert mine[p] == theirs[p], p
            else:   # reported by one side only: a record that restates the pre-state's stored node
                assert old(p) == mine.get(p, theirs.get(p)), p
    _, o_adb, o_sdb = model(apply_to_model(state, block))
    assert tables_after(pre, block, got) == (o_adb, o_sdb)


def check_siblings(eng, state, blocks):
    """every block on its own against `state`, in one overlay call, then one call per block; the state does not change"""
    ds = make_state(eng, state)
    try:
        parent = ds.root()
        pre = model(state)
        wants = [twin_apply(eng, state, b) for b in blocks]
        got = ds.overlay_roots([block_arrays(b) for b in blocks], want_updates=True)
        assert len(got) == len(blocks)
        for b, g, w in zip(blocks, got, wants):
            check_block(state, b, g, w, pre)
        assert ds.overlay_roots([block_arrays(b) for b in blocks]) == [w[0] for w in wants]
        for b, w in zip(blocks, wants):
            check_block(state, b, ds.overlay_roots([block_arrays(b)], want_updates=True)[0], w, pre)
        assert ds.root() == parent
    finally:
        ds.close()
    return got


@pytest.mark.parametrize("n0,touch", [(5, 6), (300, 40), (3000, 250)])
def test_random_blocks(eng, n0, touch):
    """overlay updates == twin apply's; then both commit the block, so later steps run on arenas with freed and reused slots"""
    rng = np.random.default_rng(1900 + n0)
    state = random_state(rng, n0, with_storage=0.5, max_slots=30)
    ds, twin = make_state(eng, state), make_state(eng, state)
    for step in range(4):
        block = random_block(rng, state, touch, step + 1)
        arrays = block_arrays(block)
        parent = ds.root()
        got = ds.overlay_roots([arrays], want_updates=True)[0]
        assert ds.root() == parent
        check_block(state, block, got, twin.apply(*arrays, want_updates=True))
        assert ds.apply(*arrays) == got[0]
        state = apply_to_model(state, block)
    ds.close()
    twin.close()


def test_sibling_batch_with_empty_and_repeated_blocks(eng):
    rng = np.random.default_rng(1901)
    state = random_state(rng, 400, with_storage=0.5, max_slots=20)
    blocks = [random_block(rng, state, 30, b + 1) for b in range(6)]
    blocks.insert(2, {})
    blocks.append(blocks[1])
    blocks.append({})
    got = check_siblings(eng, state, blocks)
    for a, b in zip(got[1], got[-2]):
        assert np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b
    for g in (got[2], got[-1]):
        assert g[1:5] == ([], [], [], []) and len(g[5]) == 0
    ds = make_state(eng, state)
    assert ds.overlay_roots([], want_updates=True) == []
    ds.close()


def test_stored_siblings_keep_their_tree_bits(eng):
    """a storage trie of thousands of slots touched in one slot: the rebuilt branches keep the tree-mask bits of stored
    children that no key reaches (they come from the hash items, not from the fold)"""
    rng = np.random.default_rng(1902)
    state = random_state(rng, 200, with_storage=0.3, max_slots=10)
    big = sorted(state)[7]
    state[big] = (state[big][0], {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(6000)})
    slots = sorted(state[big][1])
    blocks = [{big: (EXISTS | UNCHANGED, acct(0), {slots[1234]: 99})},
              {big: (EXISTS | UNCHANGED, acct(0), {slots[77]: 0})},
              {big: (EXISTS | UNCHANGED, acct(0), {rkey(rng): 5})}]
    got = check_siblings(eng, state, blocks)
    nib = lambda k: bytes(x for b in k for x in (b >> 4, b & 15))
    for block, g in zip(blocks, got):
        keys = [nib(s) for s in block[big][2]]
        unreached = [(r[1], c) for r in g[3] for c in range(16)
                     if r[3] >> c & 1 and not any(k.startswith(r[1] + bytes([c])) for k in keys)]
        assert unreached, "no record keeps a tree-mask bit of a child outside the block's paths"


def test_collapse_inline_and_extension_shapes(eng):
    rng = np.random.default_rng(1903)
    state = random_state(rng, 300, with_storage=0.3, max_slots=20)
    owners = sorted(state)[:30]
    for k in owners:
        state[k] = (state[k][0], {s: int(rng.integers(1, 4)) for s in clustered_slots(rng, 5)})
    for step in range(3):
        block = {}
        for k in owners[step * 10:(step + 1) * 10]:
            slots = sorted(state[k][1])
            ch = {s: 0 for s in slots[int(rng.integers(0, 3)):]}
            near = bytearray(slots[0])
            near[20] ^= 0x10
            ch[bytes(near)] = int(rng.integers(1, 3)) if step else 0
            split = bytearray(slots[-1])
            split[1] ^= 0x01
            ch[bytes(split)] = 7
            block[k] = (EXISTS | UNCHANGED, acct(0), ch)
        live = sorted(set(state) - set(owners))
        for i in rng.choice(len(live), 25, replace=False):
            block[live[i]] = (0, acct(0), {})
        check_siblings(eng, state, [block])
        state = apply_to_model(state, block)
    # accounts under one long extension: keys that diverge inside it, inserts that split it, a collapse onto one account
    state = {}
    for i in range(12):
        k = bytearray(KECCAK(b"ext")[:20] + bytes(12))
        k[20:] = KECCAK(bytes([i]))[:12]
        state[bytes(k)] = (acct(i + 1, 10**18 + i), {KECCAK(bytes([i, j])): j + 1 for j in range(i % 4)})
    for i in range(40):
        state[KECCAK(bytes([100, i]))] = (acct(1, i + 1), {})
    ext = [k for k in sorted(state) if k[:20] == KECCAK(b"ext")[:20]]
    diverge = bytearray(ext[0])
    diverge[10] ^= 0x01
    blocks = [{bytes(diverge): (EXISTS, acct(7), {})}, {bytes(diverge): (0, acct(0), {})},
              dict(sorted({ext[0]: (0, acct(0), {}), bytes(diverge): (EXISTS, acct(9), {})}.items())),
              {k: (0, acct(0), {}) for k in ext[1:]}]
    check_siblings(eng, state, blocks)


def prefixed(rng, prefix: bytes, nibbles: int):
    """a random key whose first `nibbles` nibbles are those of `prefix`"""
    k = bytearray(rkey(rng))
    for i in range(nibbles):
        v = (prefix[i >> 1] >> (4 * (1 - (i & 1)))) & 15
        k[i >> 1] = (k[i >> 1] & (0x0F if i & 1 == 0 else 0xF0)) | (v << (4 * (1 - (i & 1))))
    return bytes(k)


def diverging(rng, prefix: bytes, at: int):
    """a random key that shares the first `at` nibbles of `prefix` and differs at nibble `at`"""
    while True:
        k = prefixed(rng, prefix, at)
        if (k[at >> 1] >> (4 * (1 - (at & 1)))) & 15 != (prefix[at >> 1] >> (4 * (1 - (at & 1)))) & 15:
            return k


@pytest.mark.parametrize("depth", [2, 4, 5])
def test_root_extension_divergence(eng, depth):
    """a trie whose root is an extension over a stored branch, and blocks whose keys all leave that extension below its first
    nibble: the new branch above the stored one needs its tree-mask bit (account trie, then one storage trie)"""
    rng = np.random.default_rng(1910 + depth)
    prefix = bytes([0x7a, 0xbc, 0xd1])
    state = {prefixed(rng, prefix, depth): (acct(int(rng.integers(1, 9)), int(rng.integers(1, 2**40))), {}) for _ in range(400)}
    blocks = [{diverging(rng, prefix, at): (EXISTS, acct(1, 1), {})} for at in range(1, depth)]
    blocks.append({diverging(rng, prefix, depth - 1): (0, acct(0), {})})              # a delete of an absent key: changes nothing
    blocks.append({diverging(rng, prefix, 1): (EXISTS, acct(2), {}), sorted(state)[5]: (0, acct(0), {})})   # control: reaches B
    check_siblings(eng, state, [dict(sorted(b.items())) for b in blocks])
    sprefix = bytes([0x5e, 0x3f, 0x90])
    state = random_state(rng, 50, with_storage=0.3, max_slots=10)
    owner = sorted(state)[3]
    state[owner] = (state[owner][0], {prefixed(rng, sprefix, depth): int(rng.integers(1, 2**60)) for _ in range(400)})
    blocks = [{owner: (EXISTS | UNCHANGED, acct(0), {diverging(rng, sprefix, at): 5})} for at in range(1, depth)]
    blocks.append({owner: (EXISTS | UNCHANGED, acct(0), {diverging(rng, sprefix, depth - 1): 0})})
    blocks.append({owner: (EXISTS | UNCHANGED, acct(0), {diverging(rng, sprefix, 1): 6, sorted(state[owner][1])[9]: 0})})
    check_siblings(eng, state, blocks)


def test_account_and_storage_lifecycle(eng):
    """destroyed accounts, wipes with and without new slots, storages emptied by zero values, destroyed and re-created,
    no-op keys (deletes of absent slots, unchanged entries of absent accounts, also with many slots)"""
    rng = np.random.default_rng(1904)
    state = random_state(rng, 200, with_storage=0.6, max_slots=40)
    live = sorted(state)
    with_sto = sorted((k for k in live if state[k][1]), key=lambda k: -len(state[k][1]))
    blocks = [
        {with_sto[0]: (EXISTS | WIPED, state[with_sto[0]][0].copy(), {rkey(rng): 5, rkey(rng): 6})},
        {with_sto[1]: (EXISTS | WIPED, acct(9), {})},
        {with_sto[2]: (EXISTS | UNCHANGED | WIPED, acct(0), {rkey(rng): 1})},
        {with_sto[3]: (0, acct(0), {})},
        {with_sto[4]: (0, acct(0), {rkey(rng): 1})},
        {with_sto[5]: (EXISTS | WIPED, acct(3, 3), {rkey(rng): v + 1 for v in range(40)})},      # destroyed and re-created
        {k: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in state[k][1]}) for k in with_sto[6:9]},  # emptied, no wipe
        {with_sto[9]: (EXISTS | UNCHANGED, acct(0), {rkey(rng): 0 for _ in range(5)})},          # deletes of absent slots
        {rkey(rng): (EXISTS | UNCHANGED, acct(0), {rkey(rng): v + 1 for v in range(300)})},      # absent account: ignored
        {rkey(rng): (0, acct(0), {})},                                                            # delete of an absent account
        {live[0]: (EXISTS, state[live[0]][0].copy(), {})},                                         # an unchanged account
    ]
    check_siblings(eng, state, [dict(sorted(b.items())) for b in blocks])
    mixed = {}
    for b in blocks:
        mixed.update(b)
    check_siblings(eng, state, [dict(sorted(mixed.items()))])


def test_empty_state_emptying_blocks_and_one_top_nibble(eng):
    rng = np.random.default_rng(1905)
    new = {rkey(rng): (EXISTS, acct(3), {rkey(rng): 4 for _ in range(30)}) for _ in range(40)}
    assert check_siblings(eng, {}, [dict(sorted(new.items())), {}])[1][0] == EMPTY_ROOT
    state = random_state(rng, 300, with_storage=0.5, max_slots=30)
    gone = check_siblings(eng, state, [{k: (0, acct(0), {}) for k in state}])[0]
    assert gone[0] == EMPTY_ROOT and gone[1] == [] and gone[3] == []
    state = {}
    for _ in range(300):
        k = bytearray(rkey(rng))
        k[0] = 0x70 | (k[0] & 0x0F)
        state[bytes(k)] = (acct(int(rng.integers(1, 9)), int(rng.integers(1, 2**40))),
                           {rkey(rng): int(rng.integers(1, 2**40)) for _ in range(int(rng.integers(0, 20)))})
    outside = bytearray(rkey(rng))
    outside[0] = 0x30
    check_siblings(eng, state, [random_block(rng, state, 20, b + 1) for b in range(3)] + [{bytes(outside): (EXISTS, acct(1), {})}])


def test_state_is_unchanged(eng):
    """overlay calls with updates leave no trace: root, the next apply's TrieUpdates, a multiproof and a witness equal those of
    a twin that never saw the call; the root-only and with-updates calls give the same roots"""
    rng = np.random.default_rng(1906)
    state = random_state(rng, 500, with_storage=0.5, max_slots=30)
    ds, twin = make_state(eng, state), make_state(eng, state)
    for step in range(3):
        block = random_block(rng, state, 40, step + 1)
        siblings = [block_arrays(b) for b in [random_block(rng, state, 25, 10 + step) for _ in range(3)] + [block]]
        with_upd = ds.overlay_roots(siblings, want_updates=True)
        assert [g[0] for g in with_upd] == ds.overlay_roots(siblings)
        arrays = block_arrays(block)
        got, want = ds.apply(*arrays, want_updates=True), twin.apply(*arrays, want_updates=True)
        for a, b in zip(got, want):
            assert np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b
        state = apply_to_model(state, block)
        targets = {k: list(state[k][1])[:5] for k in sorted(state)[:40]}
        nxt = block_arrays(random_block(rng, state, 30, 20 + step))
        ds.overlay_roots([nxt], want_updates=True)
        assert ds.root() == twin.root()
        assert ds.multiproof(targets) == twin.multiproof(targets)
        assert ds.witness(*nxt) == twin.witness(*nxt)
    ds.close()
    twin.close()


def test_host_mirror_and_chains(eng):
    """DynamicStateRoot.overlay_root_with_updates(post) gives the tables commit(post) gives on a twin; a chain merged with
    HashedPostState.extend gives the tables of committing its blocks one by one"""
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage
    from reth_b200.trie import BranchNodeCompact
    rng = np.random.default_rng(1907)
    state = random_state(rng, 300, with_storage=0.5, max_slots=40)
    base = HashedPostState()
    for k, (a, slots) in state.items():
        base.accounts[k] = Account(int(a["nonce"]), int.from_bytes(a["balance"].tobytes(), "big"))
        if slots:
            base.storages[k] = HashedStorage(False, dict(slots))
    live = sorted(state)

    def post_of(seed):
        r = np.random.default_rng(seed)
        p = HashedPostState()
        for i in r.choice(len(live), 25, replace=False):
            k = live[i]
            x = int(r.integers(0, 4))
            if x == 0:
                p.accounts[k] = None
                p.storages[k] = HashedStorage(True, {})
            elif x == 1:
                p.accounts[k] = Account(int(r.integers(50, 99)), int(r.integers(1, 2**62)))
            else:
                p.accounts[k] = base.accounts[k]
                old = sorted(state[k][1])
                ch = {rkey(r): int(r.integers(1, 2**60)) for _ in range(3)}
                for s in old[:2]:
                    ch[s] = 0
                p.storages[k] = HashedStorage(x == 3, ch)
        p.accounts[rkey(r)] = Account(1, 1)
        return p

    _, adb, sdb = model(state)
    node = lambda rec: BranchNodeCompact(rec[0], rec[1], rec[2], tuple(rec[3]))
    s_tables = ({p: node(v) for p, v in adb.items()}, {k: {p: node(v) for p, v in t.items()} for k, t in sdb.items()})

    def apply_updates(tables, upd):
        a, s = dict(tables[0]), {k: dict(v) for k, v in tables[1].items()}
        for p in upd.removed_nodes:
            a.pop(p, None)
        a.update(upd.account_nodes)
        for k, st in upd.storage_tries.items():
            t = {} if st.is_deleted else s.get(k, {})
            for p in st.removed_nodes:
                t.pop(p, None)
            t.update(st.storage_nodes)
            s[k] = t
        return a, {k: v for k, v in s.items() if v}

    ds, twin = DynamicStateRoot(eng, base.into_sorted()), DynamicStateRoot(eng, base.into_sorted())
    parent = ds.root()
    p1, p2 = post_of(1), post_of(2)
    chain = HashedPostState(dict(p1.accounts), {k: HashedStorage(v.wiped, dict(v.storage)) for k, v in p1.storages.items()})
    chain.extend(p2)
    (r1, u1), (rc, uc) = ds.overlay_roots_with_updates([p1, chain])
    assert ds.overlay_root_with_updates(p1)[0] == r1 and ds.root() == parent
    t1, tw1 = twin.commit(p1)
    assert r1 == t1
    assert apply_updates(s_tables, u1) == apply_updates(s_tables, tw1)
    t2, tw2 = twin.commit(p2)
    assert rc == t2
    assert apply_updates(s_tables, uc) == apply_updates(apply_updates(s_tables, tw1), tw2)
    ds.close()
    twin.close()


def test_call_level_errors_and_null_outputs(eng):
    from reth_b200 import B200Error, DynamicState
    from reth_b200._lib import Stats, Updates
    from reth_b200.engine import _ptr, block_batch_arrays, updates_to_records
    rng = np.random.default_rng(1909)
    state = random_state(rng, 200, with_storage=0.5, max_slots=40)
    ds = make_state(eng, state)
    parent = ds.root()
    block = random_block(rng, state, 40, 1)
    want = ds.overlay_roots([block_arrays(block)], want_updates=True)[0]
    packed = list(block_batch_arrays([block_arrays(block)]))
    m = len(packed[0])
    roots = np.zeros((1, 32), np.uint8)

    def call(args, outs, n=1):
        return eng.lib.b200_dstate_overlay_roots_with_updates(ds.handle, n, *(_ptr(x) for x in args), _ptr(roots), *outs,
                                                              C.byref(Stats()))
    # each output on its own
    lib = eng.lib
    for i in range(5):
        us = [Updates() for _ in range(4)]
        deleted = np.zeros(max(m, 1), np.uint8)
        outs = [None] * 5
        outs[i] = _ptr(deleted) if i == 4 else C.byref(us[i])
        assert call(packed, outs) == 0
        assert roots[0].tobytes() == want[0]
        if i == 4:
            assert np.array_equal(deleted[:m], want[5])
            continue
        recs = updates_to_records(us[i], lib)
        expect = {0: [(0,) + r[1:] for r in want[1]], 1: want[2], 2: want[3], 3: want[4]}[i]
        if i == 1:
            recs = [r[1] for r in recs]
        elif i == 3:
            recs = [(r[0], r[1]) for r in recs]
        assert sorted(recs) == sorted(expect)
    # the stats cover the whole call: the same counts as the root-only call
    st_root, st_upd = Stats(), Stats()
    us = [Updates() for _ in range(4)]
    assert eng.lib.b200_dstate_overlay_roots(ds.handle, 1, *(_ptr(x) for x in packed), _ptr(roots), C.byref(st_root)) == 0
    assert eng.lib.b200_dstate_overlay_roots_with_updates(ds.handle, 1, *(_ptr(x) for x in packed), _ptr(roots),
                                                          *(C.byref(u) for u in us), None, C.byref(st_upd)) == 0
    for u in us:
        lib.b200_updates_release(C.byref(u))
    for f in ("leaves_added", "branches_added", "extension_nodes", "hashed_nodes", "levels"):
        assert getattr(st_upd, f) == getattr(st_root, f), f
    # call-level errors: outputs released and zeroed (storage_deleted too, once the block offsets give M)
    us = [Updates() for _ in range(4)]
    deleted = np.full(m, 0xAA, np.uint8)
    outs = [C.byref(u) for u in us] + [_ptr(deleted)]
    for idx, bad, m_known in ((3, np.array([1, 2], np.uint64), False), (6, None, True)):
        args = list(packed)
        args[idx] = bad
        deleted[:] = 0xAA
        assert call(args, outs) == -3
        assert all(int(u.n_nodes) == 0 and not u._owner for u in us)
        assert (deleted == (0 if m_known else 0xAA)).all()
    k0, k1 = sorted([rkey(rng), rkey(rng)])
    unsorted = (np.stack([np.frombuffer(k1, np.uint8), np.frombuffer(k0, np.uint8)]), np.stack([acct(1), acct(2)]), None,
                np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8), np.zeros(3, np.uint64))
    with pytest.raises(B200Error) as e:
        ds.overlay_roots([unsorted], want_updates=True)
    assert e.value.status == -4
    # no entries: valid empty lists
    empty = list(block_batch_arrays([block_arrays({})] * 2))
    roots2 = np.zeros((2, 32), np.uint8)
    assert eng.lib.b200_dstate_overlay_roots_with_updates(ds.handle, 2, *(_ptr(x) for x in empty), _ptr(roots2), *outs,
                                                          C.byref(Stats())) == 0
    assert all(int(u.n_nodes) == 0 and u._owner for u in us)
    for u in us:
        assert updates_to_records(u, lib) == []
    assert [roots2[0].tobytes(), roots2[1].tobytes()] == [parent, parent]
    assert ds.root() == parent
    _, keys, accs, skeys, svals, offs = flatten(state)
    sh = DynamicState.create(eng, keys, accs, skeys, svals, offs, sharded=True)
    with pytest.raises(B200Error) as e:
        sh.overlay_roots([block_arrays(block)], want_updates=True)
    assert e.value.status == -3
    sh.close()
    ds.close()
