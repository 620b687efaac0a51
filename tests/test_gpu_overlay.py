"""Post-block state roots of candidate blocks on top of the resident state, without changing it (b200_dstate_overlay_roots;
reth's StateRootProvider::state_root on the latest state).  The reference in every test is the root DynamicState.apply of the
same block gives on a twin state."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, acct, clustered_slots, flatten, random_block, random_state, rkey
from tests.test_gpu_witness import EMPTY_ROOT, KECCAK, apply_to_model, block_arrays, make_state

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def twin_root(eng, state, block):
    """the root an apply of `block` gives on a fresh state built from `state`"""
    twin = make_state(eng, state)
    try:
        return twin.apply(*block_arrays(block))
    finally:
        twin.close()


def check_siblings(eng, state, blocks):
    """every block on its own against `state`, in one overlay call, then one call per block"""
    ds = make_state(eng, state)
    try:
        parent = ds.root()
        wants = [twin_root(eng, state, b) for b in blocks]
        assert ds.overlay_roots([block_arrays(b) for b in blocks]) == wants
        for b, want in zip(blocks, wants):
            assert ds.overlay_roots([block_arrays(b)]) == [want]
        assert ds.root() == parent
    finally:
        ds.close()
    return wants


@pytest.mark.parametrize("n0,touch", [(5, 6), (300, 40), (3000, 250)])
def test_random_blocks(eng, n0, touch):
    """overlay == twin apply; then both commit the block, so later steps overlay on an arena with freed and reused slots"""
    rng = np.random.default_rng(900 + n0)
    state = random_state(rng, n0, with_storage=0.5, max_slots=30)
    ds, twin = make_state(eng, state), make_state(eng, state)
    for step in range(4):
        block = random_block(rng, state, touch, step + 1)
        arrays = block_arrays(block)
        parent = ds.root()
        got = ds.overlay_roots([arrays])
        assert ds.root() == parent
        want = twin.apply(*arrays)
        assert got == [want], step
        assert ds.apply(*arrays) == want
        state = apply_to_model(state, block)
    ds.close()
    twin.close()


def test_sibling_batch(eng):
    rng = np.random.default_rng(901)
    state = random_state(rng, 400, with_storage=0.5, max_slots=20)
    blocks = [random_block(rng, state, 30, b + 1) for b in range(8)]
    blocks.insert(3, {})
    blocks.append({})
    wants = check_siblings(eng, state, blocks)
    ds = make_state(eng, state)
    assert wants[3] == wants[-1] == ds.root()
    assert ds.overlay_roots([]) == []
    assert ds.overlay_roots([block_arrays({})] * 3) == [ds.root()] * 3
    ds.close()


def test_collapse_shapes(eng):
    """clustered slots with small values (inline leaves and inline branches), removals that collapse onto hashed, inline and
    revealed siblings, keys that diverge inside extensions, inserts that split an extension, destroyed accounts"""
    rng = np.random.default_rng(902)
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
            split[1] ^= 0x01   # splits the extension below the first nibbles
            ch[bytes(split)] = 7
            block[k] = (EXISTS | UNCHANGED, acct(0), ch)
        live = sorted(set(state) - set(owners))
        for i in rng.choice(len(live), 25, replace=False):
            block[live[i]] = (0, acct(0), {})
        check_siblings(eng, state, [block])
        state = apply_to_model(state, block)


def test_inline_subtrees_without_targets(eng):
    """inline branches that no key reaches: they have no hash form, so their leaves become items of the fold"""
    rng = np.random.default_rng(903)
    state = random_state(rng, 40, with_storage=0.0)
    owners = sorted(state)[:6]
    for k in owners:
        state[k] = (state[k][0], clustered_slots(rng, 4))
    blocks = []
    for k in owners:
        slots = sorted(state[k][1])
        blocks.append({k: (EXISTS | UNCHANGED, acct(0), {slots[0]: 0})})                        # a cluster loses a leaf
        blocks.append({k: (EXISTS | UNCHANGED, acct(0), {rkey(rng): 3})})                       # a new slot elsewhere
        near = bytearray(slots[-1])
        near[31] ^= 0x01 if near[31] & 0x0F != 0x0F else 0x02
        blocks.append({k: (EXISTS | UNCHANGED, acct(0), {bytes(near): 0x7f})})                 # into a cluster (or beside it)
    check_siblings(eng, state, blocks)


def test_diverging_keys_and_extension_splits(eng):
    """keys that diverge inside the extension above a branch (all of them, or some), and inserts that split the extension"""
    state = {}
    for i in range(12):   # accounts under one long extension: they share their first 40 nibbles
        k = bytearray(KECCAK(b"ext")[:20] + bytes(12))
        k[20:] = KECCAK(bytes([i]))[:12]
        state[bytes(k)] = (acct(i + 1, 10**18 + i), {KECCAK(bytes([i, j])): j + 1 for j in range(i % 4)})
    for i in range(40):
        state[KECCAK(bytes([100, i]))] = (acct(1, i + 1), {})
    keys = sorted(state)
    ext = [k for k in keys if k[:20] == KECCAK(b"ext")[:20]]
    diverge = bytearray(ext[0])
    diverge[10] ^= 0x01            # leaves the extension at nibble 21
    diverge2 = bytearray(ext[0])
    diverge2[19] ^= 0x10           # at nibble 38
    blocks = [
        {bytes(diverge): (EXISTS, acct(7), {})},                                     # insert splitting the extension
        {bytes(diverge): (0, acct(0), {})},                                          # delete of an absent key inside it
        {bytes(diverge): (EXISTS, acct(7), {}), bytes(diverge2): (EXISTS, acct(8), {KECCAK(b"s"): 1})},
        {bytes(diverge2): (EXISTS | UNCHANGED, acct(0), {KECCAK(b"s"): 1})},          # unchanged entry of an absent account
        {ext[0]: (0, acct(0), {}), bytes(diverge): (EXISTS, acct(9), {})},           # a removal and an insert
        {k: (0, acct(0), {}) for k in ext[1:]},                                      # collapse onto the last one
        {ext[3]: (EXISTS, acct(3, 1), {}), bytes(diverge2): (0, acct(0), {})},
    ]
    check_siblings(eng, state, [dict(sorted(b.items())) for b in blocks])


def test_accounts_and_storage_lifecycle(eng):
    """destroyed accounts, wipes with re-created storage, new accounts with storage, unchanged entries of absent accounts"""
    rng = np.random.default_rng(904)
    state = random_state(rng, 200, with_storage=0.6, max_slots=25)
    live = sorted(state)
    with_sto = [k for k in live if state[k][1]]
    blocks = [
        {with_sto[0]: (EXISTS | WIPED, state[with_sto[0]][0].copy(), {rkey(rng): 5, rkey(rng): 6})},
        {with_sto[1]: (EXISTS | WIPED, acct(9), {})},
        {with_sto[2]: (EXISTS | UNCHANGED | WIPED, acct(0), {rkey(rng): 1})},
        {with_sto[3]: (0, acct(0), {})},
        {with_sto[4]: (0, acct(0), {rkey(rng): 1})},                                # destroyed: its slots are ignored
        {rkey(rng): (EXISTS | UNCHANGED, acct(0), {rkey(rng): 1})},                 # unchanged entry of an absent account
        {rkey(rng): (EXISTS, acct(0), {})},                                          # a live empty account
        {rkey(rng): (EXISTS, acct(2), {rkey(rng): 3 for _ in range(4)})},
        {k: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in state[k][1]}) for k in with_sto[5:9]},   # storages emptied
    ]
    check_siblings(eng, state, [dict(sorted(b.items())) for b in blocks])


def test_empty_state_and_emptying_blocks(eng):
    rng = np.random.default_rng(905)
    new = {rkey(rng): (EXISTS, acct(3), {rkey(rng): 4}) for _ in range(5)}
    one = {rkey(rng): (EXISTS, acct(1), {})}
    assert check_siblings(eng, {}, [dict(sorted(new.items())), one, {}])[2] == EMPTY_ROOT
    state = random_state(rng, 30, with_storage=0.5, max_slots=6)
    gone = {k: (0, acct(0), {}) for k in state}
    assert check_siblings(eng, state, [gone])[0] == EMPTY_ROOT
    single = {sorted(state)[0]: state[sorted(state)[0]]}
    assert check_siblings(eng, single, [{k: (0, acct(0), {}) for k in single}, {rkey(rng): (EXISTS, acct(1), {})}])[0] == EMPTY_ROOT


def test_accounts_in_one_top_nibble(eng):
    rng = np.random.default_rng(906)
    state = {}
    for _ in range(300):
        k = bytearray(rkey(rng))
        k[0] = 0x70 | (k[0] & 0x0F)
        state[bytes(k)] = (acct(int(rng.integers(1, 9)), int(rng.integers(1, 2**40))),
                           {rkey(rng): int(rng.integers(1, 2**40)) for _ in range(int(rng.integers(0, 4)))})
    blocks = [random_block(rng, state, 20, b + 1) for b in range(4)]
    outside = bytearray(rkey(rng))
    outside[0] = 0x30
    blocks.append({bytes(outside): (EXISTS, acct(1), {})})
    check_siblings(eng, state, blocks)


def test_state_is_unchanged(eng):
    """overlay calls between applies leave no trace: after every apply, root, TrieUpdates, multiproof and witness are those of
    a twin that never saw an overlay call"""
    rng = np.random.default_rng(907)
    state = random_state(rng, 500, with_storage=0.5, max_slots=30)
    ds, twin = make_state(eng, state), make_state(eng, state)
    for step in range(4):
        block = random_block(rng, state, 40, step + 1)
        siblings = [random_block(rng, state, 25, 10 + step) for _ in range(3)] + [block]
        ds.overlay_roots([block_arrays(b) for b in siblings])
        arrays = block_arrays(block)
        got, want = ds.apply(*arrays, want_updates=True), twin.apply(*arrays, want_updates=True)
        assert got[0] == want[0]
        for a, b in zip(got[1:], want[1:]):
            if isinstance(a, np.ndarray):
                assert np.array_equal(a, b)
            else:
                assert a == b
        state = apply_to_model(state, block)
        targets = {k: list(state[k][1])[:5] for k in sorted(state)[:40]}
        assert ds.multiproof(targets) == twin.multiproof(targets)
        nxt = block_arrays(random_block(rng, state, 30, 20 + step))
        ds.overlay_roots([nxt])
        for mode in ("legacy", "canonical"):
            assert ds.witness(*nxt, mode=mode) == twin.witness(*nxt, mode=mode)
    ds.close()
    twin.close()


def test_host_mirror_against_stateless_and_chains(eng):
    """overlay_root(post) == the stateless root from the state's own witness; two uncommitted blocks merged with extend ==
    the root after committing both"""
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage, stateless_state_root
    rng = np.random.default_rng(908)
    rk = lambda: bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    base = HashedPostState()
    for _ in range(300):
        k = rk()
        base.accounts[k] = Account(int(rng.integers(0, 50)), int(rng.integers(1, 2**62)))
        if rng.random() < 0.5:
            base.storages[k] = HashedStorage(False, {rk(): int(rng.integers(1, 2**60)) for _ in range(int(rng.integers(1, 10)))})
    live = sorted(base.accounts)

    def post_of(seed):
        r = np.random.default_rng(seed)
        p = HashedPostState()
        for i in r.choice(len(live), 20, replace=False):
            k = live[i]
            x = int(r.integers(0, 4))
            if x == 0:
                p.accounts[k] = None
                p.storages[k] = HashedStorage(True, {})
            elif x == 1:
                p.accounts[k] = Account(int(r.integers(50, 99)), int(r.integers(1, 2**62)))
            else:
                p.accounts[k] = base.accounts[k]
                old = sorted(base.storages[k].storage) if k in base.storages else []
                ch = {rk(): int(r.integers(1, 2**60))}
                if old:
                    ch[old[0]] = 0
                p.storages[k] = HashedStorage(x == 3, ch)
        p.accounts[rk()] = Account(1, 1)
        return p

    ds, twin = DynamicStateRoot(eng, base.into_sorted()), DynamicStateRoot(eng, base.into_sorted())
    p1, p2 = post_of(1), post_of(2)
    parent = ds.root()
    for p in (p1, p2):
        assert ds.overlay_root(p) == stateless_state_root(eng, parent, ds.witness(p), p)
    chain = HashedPostState(dict(p1.accounts), {k: HashedStorage(v.wiped, dict(v.storage)) for k, v in p1.storages.items()})
    chain.extend(p2)
    r1, _ = twin.commit(p1)
    r2, _ = twin.commit(p2)
    assert ds.overlay_roots([p1, chain]) == [r1, r2]
    assert ds.root() == parent
    ds.close()
    twin.close()


def test_call_level_errors(eng):
    from reth_b200 import B200Error, DynamicState
    from reth_b200._lib import Stats
    from reth_b200.engine import _ptr, block_batch_arrays
    rng = np.random.default_rng(909)
    state = random_state(rng, 60, with_storage=0.5, max_slots=6)
    ds = make_state(eng, state)
    parent = ds.root()
    k0, k1 = sorted([rkey(rng), rkey(rng)])
    s0, s1 = sorted([rkey(rng), rkey(rng)])
    a2 = np.stack([acct(1), acct(2)])
    one = lambda k: np.frombuffer(k, np.uint8)
    unsorted_accts = (np.stack([one(k1), one(k0)]), a2, None, np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8),
                      np.zeros(3, np.uint64))
    unsorted_slots = (np.stack([one(k0)]), a2[:1], None, np.stack([one(s1), one(s0)]), np.ones((2, 32), np.uint8),
                      np.array([0, 2], np.uint64))
    for bad in (unsorted_accts, unsorted_slots):
        with pytest.raises(B200Error) as e:
            ds.overlay_roots([bad])
        assert e.value.status == -4
    good_block = (np.stack([one(k0), one(k1)]), a2, None, np.stack([one(s0)]), np.ones((1, 32), np.uint8),
                  np.array([0, 1, 1], np.uint64))
    good = list(block_batch_arrays([good_block]))
    roots = np.zeros((2, 32), np.uint8)

    def call(args, n=1):
        return eng.lib.b200_dstate_overlay_roots(ds.handle, n, *(_ptr(x) for x in args), _ptr(roots), C.byref(Stats()))
    assert call(good) == 0
    want = twin_root(eng, state, {k0: (EXISTS, acct(1), {s0: int.from_bytes(bytes([1]) * 32, "big")}), k1: (EXISTS, acct(2), {})})
    assert roots[0].tobytes() == want
    for i, bad, n in ((3, np.array([1, 2], np.uint64), 1), (3, np.array([0, 2, 1], np.uint64), 2), (6, np.array([0, 1, 0], np.uint64), 1),
                      (6, np.array([1, 1, 1], np.uint64), 1), (0, None, 1)):
        args = list(good)
        args[i] = bad
        assert call(args, n) == -3, (i, bad)
    assert call(good, n=0) == 0   # no blocks: nothing to do
    assert ds.root() == parent
    assert ds.overlay_roots([block_arrays({})]) == [parent]
    _, keys, accs, skeys, svals, offs = flatten(state)
    sh = DynamicState.create(eng, keys, accs, skeys, svals, offs, sharded=True)
    with pytest.raises(B200Error) as e:
        sh.overlay_roots([good_block])
    assert e.value.status == -3
    sh.close()
    block = random_block(rng, state, 10, 1)
    assert ds.overlay_roots([block_arrays(block)]) == [twin_root(eng, state, block)]
    assert ds.root() == parent
    ds.close()
