"""Post-block state roots from execution witnesses (b200_witness_roots; reth's stateless validation: from_witness, a revealed
SparseStateTrie, root()).  The reference in every test is the root DynamicState.apply gives on a twin state; witnesses come
from b200_dstate_witness (both modes) or are built by hand."""
import ctypes as C

import numpy as np
import pytest

import oracle
from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, acct, clustered_slots, random_block, random_state, rkey
from tests.test_gpu_witness import (EMPTY_ROOT, KECCAK, apply_to_model, block_arrays, decode, hex_prefix, is_empty, make_state,
                                    nib, rlp_list, rlp_str, rlp_uint, stateless_root)

pytestmark = [pytest.mark.gpu]

OK, INVALID, INCOMPLETE = 0, -3, -9


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def roots_of(eng, parents, witnesses, blocks):
    roots, st = eng.witness_roots(parents, witnesses, [block_arrays(b) for b in blocks])
    return [r.tobytes() for r in roots], [int(x) for x in st]


def one(eng, parent, witness, block):
    r, s = roots_of(eng, [parent], [witness], [block])
    return r[0], s[0]


def setup(eng, state, block):
    """-> (parent root, {mode: witness}, the root an apply of the block gives)"""
    ds, twin = make_state(eng, state), make_state(eng, state)
    arrays = block_arrays(block)
    w = {mode: ds.witness(*arrays, mode=mode) for mode in ("legacy", "canonical")}
    parent, want = ds.root(), twin.apply(*arrays)
    ds.close()
    twin.close()
    return parent, w, want


def has_live_empty(block):
    return any((fl & EXISTS) and not (fl & UNCHANGED) and is_empty(a) for fl, a, _ in block.values())


@pytest.mark.parametrize("n0,touch", [(5, 6), (300, 40), (3000, 250)])
def test_random_blocks(eng, n0, touch):
    rng = np.random.default_rng(700 + n0)
    state = random_state(rng, n0, with_storage=0.5, max_slots=30)
    for step in range(3):
        block = random_block(rng, state, touch, step + 1)
        parent, w, want = setup(eng, state, block)
        for mode in ("legacy", "canonical"):
            assert one(eng, parent, w[mode], block) == (want, OK), mode
            if n0 <= 300 and not has_live_empty(block):
                assert stateless_root(w[mode], parent, block, mode == "canonical") == want
        state = apply_to_model(state, block)


def test_chain_in_one_call(eng):
    rng = np.random.default_rng(71)
    state = random_state(rng, 400, with_storage=0.5, max_slots=20)
    ds = make_state(eng, state)
    parents, witnesses, blocks, wants = [], [], [], []
    for step in range(6):
        block = random_block(rng, state, 30, step + 1)
        arrays = block_arrays(block)
        parents.append(ds.root())
        witnesses.append(ds.witness(*arrays, mode="legacy" if step % 2 else "canonical"))
        wants.append(ds.apply(*arrays))
        blocks.append(block)
        state = apply_to_model(state, block)
    ds.close()
    assert roots_of(eng, parents, witnesses, blocks) == (wants, [OK] * 6)
    for b in range(6):
        assert one(eng, parents[b], list(witnesses[b].values()), blocks[b]) == (wants[b], OK)


def test_collapse_shapes(eng):
    """clustered slots with small values (inline leaves and branches), removals that collapse onto hashed, inline and revealed
    siblings, keys that diverge inside extensions, inserts that split an extension, destroyed accounts"""
    rng = np.random.default_rng(72)
    state = random_state(rng, 300, with_storage=0.3, max_slots=20)
    owners = sorted(state)[:30]
    for k in owners:
        # small values: slots that share 63 nibbles have inline leaves (a hashed leaf at depth 64 is not representable)
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
            split[1] ^= 0x01   # splits the extension below the first nibbles
            ch[bytes(split)] = 7
            block[k] = (EXISTS | UNCHANGED, acct(0), ch)
        live = sorted(set(state) - set(owners))
        for i in rng.choice(len(live), 25, replace=False):
            block[live[i]] = (0, acct(0), {})
        parent, w, want = setup(eng, state, block)
        for mode in ("legacy", "canonical"):
            assert one(eng, parent, w[mode], block) == (want, OK), mode
        state = apply_to_model(state, block)


# ---- rule (b), hand-built ---------------------------------------------------------------------------------------------------
BIG = 2**250  # leaves of more than 32 bytes: hashed in their branch


def slot_key(*nibs):
    k = bytearray(32)
    for i, x in enumerate(nibs):
        k[i // 2] |= x << (4 if i % 2 == 0 else 0)
    return bytes(k)


def storage_case(eng, slots, change):
    a = KECCAK(b"rule-b")
    state = {a: (acct(1), slots)}
    block = {a: (EXISTS | UNCHANGED, acct(0), change)}
    parent, w, want = setup(eng, state, block)
    return parent, w["legacy"], want, block


def drop(w, pred):
    kept = {h: r for h, r in w.items() if not pred(decode(r))}
    assert len(kept) == len(w) - 1
    return kept


def test_rule_b_hashed_leaf_sibling_is_needed(eng):
    s1, s2 = slot_key(1), slot_key(2)
    parent, w, want, block = storage_case(eng, {s1: BIG, s2: BIG + 1}, {s1: 0})
    assert one(eng, parent, w, block) == (want, OK)
    w2 = drop(w, lambda d: len(d) == 2 and d[1] == rlp_uint(BIG + 1))
    assert one(eng, parent, w2, block) == (bytes(32), INCOMPLETE)


def test_rule_b_branch_behind_an_extension_is_not_needed(eng):
    s1, s2, s3 = slot_key(1), slot_key(2, 10, 5), slot_key(2, 10, 6)
    below = lambda d: len(d) == 17 and d[5] != b"" and d[6] != b""
    parent, w, want, block = storage_case(eng, {s1: BIG, s2: BIG, s3: BIG + 1}, {s1: 0})
    assert one(eng, parent, drop(w, below), block) == (want, OK)
    parent, w, want, block = storage_case(eng, {s1: BIG, s2: BIG, s3: BIG + 1}, {slot_key(2, 11): 9})  # splits the extension
    assert one(eng, parent, drop(w, below), block) == (want, OK)


def path_nodes(w, root, key):
    """-> (hashes of the nodes on the path from `root` to `key` in the node map w, the leaf's value or None): the walk ends
    at the leaf, at an empty branch slot, or at a diverging leaf or extension (the branch below it is not on the path)"""
    if root == EMPTY_ROOT:
        return set(), None
    nk, d, out, node = nib(key), 0, {root}, decode(w[root])
    while True:
        if len(node) == 17:
            child = node[nk[d]]
            d += 1
        else:
            b = node[0]
            part = ((b[0] & 15,) if b[0] & 0x10 else ()) + tuple(x for y in b[1:] for x in (y >> 4, y & 15))
            if b[0] >> 4 >= 2:
                return out, (node[1] if nk[d:] == part else None)
            if nk[d:d + len(part)] != part:
                return out, None
            d += len(part)
            child = node[1]
        if child == b"":
            return out, None
        if not isinstance(child, list):
            out.add(child)
            child = decode(w[child])
        node = child


def test_never_a_wrong_root(eng):
    """Dropping any one witness node gives the right root or INCOMPLETE; dropping a node on the path to a key of the block
    (account keys, and the slot keys of live, unwiped, existing storage tries) always gives INCOMPLETE."""
    rng = np.random.default_rng(73)
    state = random_state(rng, 40, with_storage=0.6, max_slots=12)
    for step in range(2):
        block = random_block(rng, state, 5, step + 1)
        parent, w, want = setup(eng, state, block)
        for mode in ("legacy", "canonical"):
            path = set()
            for k, (fl, _, slots) in block.items():
                nodes, leaf = path_nodes(w[mode], parent, k)
                path |= nodes
                if (fl & EXISTS) and not (fl & WIPED) and slots and leaf is not None:
                    for sk in slots:
                        path |= path_nodes(w[mode], decode(leaf)[2], sk)[0]
            assert path and path <= set(w[mode])
            items = list(w[mode].items())
            for h, _ in items:
                r, s = one(eng, parent, {k: v for k, v in items if k != h}, block)
                assert (r, s) in ((want, OK), (bytes(32), INCOMPLETE)), (mode, h.hex())
                if h in path:
                    assert s == INCOMPLETE, (mode, h.hex())
        state = apply_to_model(state, block)


def test_tampering_and_extra_nodes(eng):
    rng = np.random.default_rng(74)
    state = random_state(rng, 200, with_storage=0.5, max_slots=10)
    blocks, parents, ws, wants = [], [], [], []
    ds = make_state(eng, state)
    for step in range(3):
        block = random_block(rng, state, 10, step + 1)
        arrays = block_arrays(block)
        parents.append(ds.root())
        ws.append(ds.witness(*arrays, mode="legacy"))
        wants.append(ds.apply(*arrays))
        blocks.append(block)
        state = apply_to_model(state, block)
    ds.close()
    root_node = bytearray(ws[0][parents[0]])
    root_node[-1] ^= 1
    tampered = dict(ws[0])
    tampered[parents[0]] = bytes(root_node)
    assert one(eng, parents[0], tampered, blocks[0]) == (bytes(32), INCOMPLETE)
    assert one(eng, bytes(31) + b"\1", ws[0], blocks[0]) == (bytes(32), INCOMPLETE)
    junk = [rng.bytes(int(rng.integers(1, 600))) for _ in range(50)]
    noisy = [list(ws[0].values()) * 2 + list(ws[1].values()) + junk, list(ws[1].values()) + junk, list(ws[2].values()) + junk[:3]]
    assert roots_of(eng, parents, noisy, blocks) == (wants, [OK] * 3)
    # a node block 0 needs, carried only by block 1
    moved = [{k: v for k, v in ws[0].items() if k != parents[0]}, {**ws[1], parents[0]: ws[0][parents[0]]}, ws[2]]
    r, s = roots_of(eng, parents, moved, blocks)
    assert s == [INCOMPLETE, OK, OK] and r[1:] == wants[1:]


def account_rlp(nonce, bal, sroot):
    return rlp_list([rlp_uint(nonce), rlp_uint(bal), rlp_str(sroot), rlp_str(oracle.KECCAK_EMPTY)])


def test_malformed_nodes(eng):
    a = KECCAK(b"malformed")
    leaf = lambda nibs, value: rlp_list([rlp_str(hex_prefix(list(nibs), True)), rlp_str(value)])
    good = leaf(nib(a), account_rlp(1, 1, EMPTY_ROOT))
    slot = slot_key(3)
    sleaf = lambda v: leaf(nib(slot), v)
    bad_storage_root = lambda v: leaf(nib(a), account_rlp(1, 1, KECCAK(sleaf(v))))
    cases = {
        "bad rlp": [b"\xf8\x02\x01"],
        "trailing bytes": [good + b"\x00"],
        "17th item": [rlp_list([rlp_str(b"")] * 3 + [rlp_str(KECCAK(good))] + [rlp_str(b"")] * 12 + [rlp_str(b"x")])],
        "short leaf path": [leaf(nib(a)[:63], account_rlp(1, 1, EMPTY_ROOT))],
        "long leaf path": [leaf(nib(a) + (1,), account_rlp(1, 1, EMPTY_ROOT))],
        "inline child of 33 bytes": [rlp_list([rlp_str(b"")] * 3 + [rlp_list([rlp_str(b"\x20"), rlp_str(bytes(30))])] + [rlp_str(b"")] * 13)],
        "hashed child of 31 bytes": [rlp_list([rlp_str(b"")] * 3 + [rlp_str(bytes(31))] + [rlp_str(b"")] * 13)],
        "account value": [leaf(nib(a), rlp_list([rlp_str(bytes(9)), rlp_uint(1), rlp_str(EMPTY_ROOT), rlp_str(oracle.KECCAK_EMPTY)]))],
        "zero storage value": [bad_storage_root(b"\x80"), sleaf(b"\x80")],
        "long storage value": [bad_storage_root(rlp_str(b"\x01" * 33)), sleaf(rlp_str(b"\x01" * 33))],
    }
    good_block = {a: (EXISTS, acct(5), {})}
    store_block = {a: (EXISTS | UNCHANGED, acct(0), {slot: 2})}
    parents, ws, blocks = [KECCAK(good)], [[good]], [good_block]
    for name, nodes in cases.items():
        parents.append(KECCAK(nodes[0]))
        ws.append(nodes)
        blocks.append(store_block if "storage" in name else good_block)
    r, s = roots_of(eng, parents, ws, blocks)
    assert s == [OK] + [INVALID] * len(cases), dict(zip(["good"] + list(cases), s))
    assert r[0] == make_state(eng, {a: (acct(5), {})}).root() and all(x == bytes(32) for x in r[1:])


def test_wipe_needs_nothing_of_the_wiped_trie(eng):
    rng = np.random.default_rng(75)
    state = random_state(rng, 100, with_storage=0.2)
    big = sorted(state)[50]
    state[big] = (state[big][0], {rkey(rng): int(rng.integers(1, 2**40)) for _ in range(9000)})
    block = {big: (EXISTS | WIPED, state[big][0].copy(), {rkey(rng): 5})}
    parent, w, want = setup(eng, state, block)
    ds = make_state(eng, state)
    sroot = ds.multiproof({big: []})["storages"][big]["root"]
    sub = ds.multiproof({big: list(state[big][1])[:50]})["storages"][big]["subtree"]
    ds.close()
    wiped = set(sub.values())
    lean = {h: r for h, r in w["legacy"].items() if r not in wiped and h != sroot}
    assert len(lean) < len(w["legacy"])
    assert one(eng, parent, lean, block) == (want, OK)


def test_edge_semantics(eng):
    rng = np.random.default_rng(76)
    state = random_state(rng, 50, with_storage=0.5, max_slots=5)
    ds = make_state(eng, state)
    parent = ds.root()
    ds.close()
    assert one(eng, parent, [], {}) == (parent, OK)
    r, s = eng.witness_roots([], [], [])
    assert r.shape == (0, 32) and s.shape == (0,)
    new = {rkey(rng): (EXISTS, acct(3), {rkey(rng): 4}) for _ in range(5)}
    assert one(eng, EMPTY_ROOT, [], new) == (make_state(eng, {k: (a, s) for k, (_, a, s) in new.items()}).root(), OK)
    k0, k1 = sorted(state)[:2]
    absent = rkey(rng)
    block = {k0: (EXISTS, acct(0), {}),                                # live empty account: stays a leaf
             k1: (0, acct(0), {rkey(rng): 9}),                          # destroyed: its slots are ignored
             absent: (EXISTS | UNCHANGED, acct(0), {rkey(rng): 1})}    # unchanged entry of an absent account: ignored
    block = dict(sorted(block.items()))
    parent, w, want = setup(eng, state, block)
    for mode in ("legacy", "canonical"):
        assert one(eng, parent, w[mode], block) == (want, OK)


def test_reth_witness_cases(eng):
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage, stateless_state_root
    a, slot = KECCAK(b"addr"), KECCAK(b"slot")
    s1, s2 = bytes([1]) * 32, bytes([2]) * 32
    a2 = KECCAK(bytes(20))
    cases = [
        (HashedPostState({a: Account()}, {}), HashedPostState({a: Account()}, {a: HashedStorage(False, {slot: 1})})),
        (HashedPostState({a: Account()}, {a: HashedStorage(False, {slot: 1})}), HashedPostState({a: None}, {a: HashedStorage(True, {})})),
        (HashedPostState({a2: Account()}, {a2: HashedStorage(False, {s1: 1, s2: 1})}),
         HashedPostState({a2: Account()}, {a2: HashedStorage(False, {s1: 2, s2: 2})})),
        (HashedPostState({a: Account(1, 1)}, {a: HashedStorage(False, {KECCAK(bytes([i])): i + 1 for i in range(4)})}),
         HashedPostState({a: Account(2, 1)}, {})),
        (HashedPostState({a: Account(1)}, {a: HashedStorage(False, {bytes([0x10]) + bytes(31): BIG, bytes([0x20]) + bytes(31): BIG + 1})}),
         HashedPostState({a: Account(1)}, {a: HashedStorage(False, {bytes([0x10]) + bytes(31): 0, bytes([0x30]) + bytes(31): 1})})),
    ]
    for pre, post in cases:
        for mode in ("legacy", "canonical"):
            ds, twin = DynamicStateRoot(eng, pre.into_sorted()), DynamicStateRoot(eng, pre.into_sorted())
            parent, w = ds.root(), ds.witness(post, mode)
            want, _ = twin.commit(post)
            assert stateless_state_root(eng, parent, w, post) == want
            ds.close()
            twin.close()


def test_argument_errors(eng):
    from reth_b200 import Account, B200Error, HashedPostState, HashedStorage, StateRootError, stateless_state_root
    rng = np.random.default_rng(77)
    k0, k1 = sorted([rkey(rng), rkey(rng)])
    unsorted = (np.stack([np.frombuffer(k1, np.uint8), np.frombuffer(k0, np.uint8)]), np.stack([acct(1), acct(2)]),
                np.array([EXISTS, EXISTS], np.uint8), np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8), np.zeros(3, np.uint64))
    with pytest.raises(B200Error) as e:
        eng.witness_roots([EMPTY_ROOT], [[]], [unsorted])
    assert e.value.status == -4
    # the C entry point's own checks: offsets that do not start at 0, non-monotone offsets, a null pointer
    from reth_b200._lib import Stats
    from reth_b200.engine import _ptr, witness_batch_arrays
    two = (np.stack([np.frombuffer(k0, np.uint8), np.frombuffer(k1, np.uint8)]), np.stack([acct(1), acct(2)]), None,
           np.zeros((1, 32), np.uint8), np.ones((1, 32), np.uint8), np.array([0, 1, 1], np.uint64))
    good = list(witness_batch_arrays([EMPTY_ROOT], [[]], [two]))
    roots, status = np.zeros((1, 32), np.uint8), np.zeros(1, np.int32)

    def call(args):
        return eng.lib.b200_witness_roots(eng.ctx, args[0], *(_ptr(x) for x in args[1:]), _ptr(roots), _ptr(status), C.byref(Stats()))
    assert call(good) == 0 and status[0] == OK
    for i, bad in ((8, np.array([1, 2], np.uint64)), (11, np.array([0, 1, 0], np.uint64)), (4, np.array([1, 1], np.uint64)),
                   (1, None)):
        args = list(good)
        args[i] = bad
        assert call(args) == -3, i
    with pytest.raises(StateRootError, match=r"block 0: witness incomplete \(status -9\)"):
        stateless_state_root(eng, KECCAK(b"x"), [], HashedPostState({k0: Account(1)}, {}))
    with pytest.raises(StateRootError):
        stateless_state_root(eng, EMPTY_ROOT, [], HashedPostState({}, {k0: HashedStorage(False, {k1: 1})}))
