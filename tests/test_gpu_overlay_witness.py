"""Execution witness of a block on top of a candidate block, without changing the resident state
(b200_dstate_overlay_witness; reth's StateProofProvider::witness of a MemoryOverlayStateProvider).  The reference in every
test is a twin state on which the overlay is applied, followed by witness of the target block: the whole map and the
overlay root must be equal.  Where the shape allows, the map is also checked against the model of tests/test_gpu_witness.py
on the post-overlay state, and a stateless run (b200_witness_roots) from the overlay root must give the twin's root after
the target block."""
import ctypes as C

import numpy as np
import oracle
import pytest

from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, acct, flatten, random_block, random_state, rkey
from tests.test_gpu_witness import apply_to_model, block_arrays, make_state, model_witness

pytestmark = [pytest.mark.gpu]

MODES = ("legacy", "canonical")
EMPTY_BLOCK = (np.zeros((0, 32), np.uint8), np.zeros(0, oracle.ACCOUNT_DTYPE), None, np.zeros((0, 32), np.uint8),
               np.zeros((0, 32), np.uint8), np.zeros(1, np.uint64))


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def check(eng, ds, state, overlay, target, model=True):
    """ds (the resident `state`) against a twin: apply(overlay), then witness(target), in both modes, with and without
    always_include_root"""
    ov, tg = block_arrays(overlay), block_arrays(target)
    twin = make_state(eng, state)
    try:
        ov_root = twin.apply(*ov)
        post = apply_to_model(state, overlay)
        for mode in MODES:
            for incl in (False, True):
                want = twin.witness(*tg, mode=mode, always_include_root_node=incl)
                root, got = ds.overlay_witness(ov, tg, mode=mode, always_include_root_node=incl)
                assert root == ov_root, (mode, incl)
                assert got == want, (mode, incl, len(set(got) - set(want)), len(set(want) - set(got)))
                if model and not incl:
                    assert got == model_witness(post, target, mode), mode
                if target:
                    roots, status = eng.witness_roots([ov_root], [got], [tg])
                    assert status[0] == 0
                    after = roots[0].tobytes()
        if target:
            assert after == twin.apply(*tg)
    finally:
        twin.close()


@pytest.mark.parametrize("n0,touch", [(5, 6), (300, 40), (3000, 250)])
def test_random_blocks(eng, n0, touch):
    rng = np.random.default_rng(1300 + n0)
    state = random_state(rng, n0, with_storage=0.5, max_slots=30)
    ds = make_state(eng, state)
    try:
        for step in range(3):
            overlay = random_block(rng, state, touch, 2 * step + 1)
            target = random_block(rng, apply_to_model(state, overlay), touch, 2 * step + 2)
            check(eng, ds, state, overlay, target)
            block = random_block(rng, state, touch, 2 * step + 1)   # committed: the folds and marks meet a changed state
            ds.apply(*block_arrays(block))
            state = apply_to_model(state, block)
    finally:
        ds.close()


def two_groups(rng, first, second, n_first=2, n_second=12):
    """keys under top nibble `first` (n_first of them) and `second` (n_second): the `second` subtree is hashed"""
    def under(nib):
        k = bytearray(rkey(rng))
        k[0] = (nib << 4) | (k[0] & 15)
        return bytes(k)
    return sorted(under(first) for _ in range(n_first)), sorted(under(second) for _ in range(n_second))


def under_extension(rng, n=12, shared=5):
    """n slots that share their first 2 * shared nibbles: the storage root is an extension above a hashed branch"""
    head = rkey(rng)[:shared]
    return {head + rkey(rng)[shared:]: int(rng.integers(1, 2**60)) for _ in range(n)}


def test_removal_onto_an_unopened_sibling(eng):
    """A target removal whose only surviving sibling is a hashed subtree the overlay never opened: the collapse sibling lies
    below a hash leaf of the fold, in the storage trie and in the account trie."""
    rng = np.random.default_rng(1310)
    a, b = two_groups(rng, 1, 2)
    owner = rkey(rng)
    s_few, s_many = two_groups(rng, 3, 9)
    state = {k: (acct(1, 1), {}) for k in a + b}
    state[owner] = (acct(1, 1), {s: int(rng.integers(1, 2**60)) for s in s_few + s_many})
    ds = make_state(eng, state)
    try:
        other = b[0]
        overlay = {other: (EXISTS, acct(7, 7), {}), owner: (EXISTS, acct(2, 2), {})}  # nothing under s_many / most of b
        target = {owner: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in s_few})}
        check(eng, ds, state, overlay, target)
        target = {k: (0, acct(0), {}) for k in a}   # both accounts under nibble 1 go: collapse onto nibble 2 ... and owner's
        check(eng, ds, state, overlay, target)
    finally:
        ds.close()


def test_divergence_inside_an_unopened_extension(eng):
    """A target key that diverges inside an extension above a branch the overlay did not open: the witness holds the branch."""
    rng = np.random.default_rng(1311)
    state = random_state(rng, 200, with_storage=0.3, max_slots=10)
    owner = sorted(state)[17]
    state[owner] = (state[owner][0], under_extension(rng))
    slots = sorted(state[owner][1])
    ds = make_state(eng, state)
    try:
        overlay = {owner: (EXISTS, acct(3, 3), {}), sorted(state)[90]: (0, acct(0), {})}
        for shared in (2, 5, 9):
            near = bytearray(slots[0])
            b, hi = divmod(shared, 2)
            near[b] ^= 0x80 if hi == 0 else 0x08
            for value in (0, 5):
                check(eng, ds, state, overlay, {owner: (EXISTS | UNCHANGED, acct(0), {bytes(near): value})})
    finally:
        ds.close()


def test_wipes_of_storages_the_overlay_changed_in_part_or_left_alone(eng):
    rng = np.random.default_rng(1312)
    state = random_state(rng, 300, with_storage=0.0)
    ks = sorted(state)
    for k in ks[:6]:
        state[k] = (state[k][0], {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(40)})
    ds = make_state(eng, state)
    try:
        some = sorted(state[ks[0]][1])
        new = rkey(rng)
        overlay = {
            ks[0]: (EXISTS | UNCHANGED, acct(0), {some[0]: 0, some[1]: 9, rkey(rng): 4}),   # changed in part
            ks[1]: (EXISTS, acct(5, 5), {}),                                              # account only
            ks[2]: (EXISTS | WIPED, state[ks[2]][0].copy(), {rkey(rng): 1, rkey(rng): 2}),  # wiped and refilled
            new: (EXISTS, acct(1, 1), {rkey(rng): 3 for _ in range(5)}),                   # created
        }
        for k in (ks[0], ks[1], ks[2], ks[3], new):          # ks[3]: left alone
            for fl in (EXISTS | WIPED, 0):                   # wiped / destroyed
                check(eng, ds, state, overlay, {k: (fl, acct(2, 2), {rkey(rng): 8} if fl else {})})
    finally:
        ds.close()


def test_account_lifecycles_across_the_two_blocks(eng):
    rng = np.random.default_rng(1313)
    state = random_state(rng, 200, with_storage=0.5, max_slots=8)
    ks = sorted(state)
    owner = next(k for k in ks if state[k][1])
    ds = make_state(eng, state)
    try:
        created = rkey(rng)
        check(eng, ds, state, {created: (EXISTS, acct(1, 1), {rkey(rng): 5})}, {created: (0, acct(0), {})})
        check(eng, ds, state, {ks[5]: (0, acct(0), {})}, {ks[5]: (EXISTS, acct(4, 4), {rkey(rng): 6})})
        emptied = {owner: (EXISTS, acct(0), {s: 0 for s in state[owner][1]})}     # empty account, empty storage
        for fl in (EXISTS | UNCHANGED, EXISTS):
            check(eng, ds, state, emptied, {owner: (fl, acct(0), {})})
    finally:
        ds.close()


def test_legacy_storage_root_nodes(eng):
    """Target entries without slots: the storage-root node, also an extension root whose branch the overlay did not open."""
    rng = np.random.default_rng(1314)
    state = random_state(rng, 150, with_storage=0.5, max_slots=12)
    ks = sorted(state)
    ext_owner = ks[3]
    state[ext_owner] = (state[ext_owner][0], under_extension(rng))
    ds = make_state(eng, state)
    try:
        overlay = {ks[40]: (EXISTS, acct(9, 9), {}), ks[41]: (EXISTS | UNCHANGED, acct(0), {rkey(rng): 1})}
        target = {k: (EXISTS, acct(2, 2), {}) for k in (ext_owner, ks[10], ks[11], ks[40], ks[41], rkey(rng))}
        check(eng, ds, state, overlay, target)
        check(eng, ds, state, {ext_owner: (EXISTS, acct(1, 2), {})}, {ext_owner: (EXISTS, acct(3, 3), {})})
    finally:
        ds.close()


def test_empty_states_one_top_nibble_and_empty_blocks(eng):
    rng = np.random.default_rng(1315)
    state = random_state(rng, 60, with_storage=0.5, max_slots=6)
    ds = make_state(eng, state)
    try:
        all_gone = {k: (0, acct(0), {}) for k in state}
        check(eng, ds, state, all_gone, {rkey(rng): (EXISTS, acct(1, 1), {rkey(rng): 2})})
        check(eng, ds, state, all_gone, {})
        check(eng, ds, state, random_block(rng, state, 8, 1), {})                     # m = 0
        # ov_m = 0: exactly b200_dstate_witness
        target = block_arrays(random_block(rng, state, 8, 2))
        for mode in MODES:
            for incl in (False, True):
                root, got = ds.overlay_witness(EMPTY_BLOCK, target, mode=mode, always_include_root_node=incl)
                assert root == ds.root()
                assert got == ds.witness(*target, mode=mode, always_include_root_node=incl)
    finally:
        ds.close()
    one = {}
    for _ in range(80):
        k = bytearray(rkey(rng))
        k[0] = 0x70 | (k[0] & 15)
        one[bytes(k)] = (acct(1, 1), {rkey(rng): 3} if rng.random() < 0.3 else {})
    ds = make_state(eng, one)
    try:
        ks = sorted(one)
        check(eng, ds, one, {ks[0]: (0, acct(0), {}), rkey(rng): (EXISTS, acct(1, 1), {})},
              {ks[1]: (0, acct(0), {}), ks[2]: (EXISTS, acct(5, 5), {})})
    finally:
        ds.close()


def test_the_state_is_unchanged(eng):
    rng = np.random.default_rng(1316)
    state = random_state(rng, 400, with_storage=0.5, max_slots=20)
    ds, twin = make_state(eng, state), make_state(eng, state)
    try:
        root = ds.root()
        for step in range(3):
            overlay = random_block(rng, state, 30, 1)
            ds.overlay_witness(block_arrays(overlay), block_arrays(random_block(rng, apply_to_model(state, overlay), 30, 2)))
        assert ds.root() == twin.root() == root
        block = block_arrays(random_block(rng, state, 30, 3))
        for mode in MODES:
            assert ds.witness(*block, mode=mode) == twin.witness(*block, mode=mode)
        targets = {k: tuple(sorted(s)[:3]) for k, (_, s) in list(state.items())[:50]}
        assert ds.multiproof(targets) == twin.multiproof(targets)
        assert ds.apply(*block) == twin.apply(*block)
    finally:
        ds.close()
        twin.close()


def raw_call(eng, ds, ov, tg, mode=0, null=None):
    from reth_b200.engine import Witness, _ptr
    ok, oa, of, osk, osv, oso = ov
    k, a, f, sk, sv, so = tg
    root = np.zeros(32, np.uint8)
    w = Witness()
    args = [ds.handle, _ptr(ok), _ptr(oa), _ptr(of), len(ok), _ptr(osk), _ptr(osv), _ptr(oso), _ptr(k), _ptr(a), _ptr(f), len(k),
            _ptr(sk), _ptr(sv), _ptr(so), mode, 0, _ptr(root), C.byref(w), None]
    if null is not None:
        args[null] = None
    r = eng.lib.b200_dstate_overlay_witness(*args)
    if r != 0:
        assert w.n == 0 and not w._owner and not w.hashes32 and not w.rlp and not w.rlp_offset
    else:
        eng.lib.b200_witness_release(C.byref(w))
    return r


def test_errors(eng):
    from reth_b200 import DynamicState
    rng = np.random.default_rng(1317)
    state = random_state(rng, 60, with_storage=0.5, max_slots=6)
    ds = make_state(eng, state)
    try:
        ov = block_arrays(random_block(rng, state, 6, 1))
        tg = block_arrays({rkey(rng): (EXISTS, acct(1, 1), {rkey(rng): 1, rkey(rng): 2}), rkey(rng): (EXISTS, acct(1, 1), {})})
        assert raw_call(eng, ds, ov, tg) == 0
        rev = lambda b: (b[0][::-1].copy(),) + tuple(b[1:])
        swap_slots = lambda b: b[:3] + (b[3][::-1].copy(), b[4], b[5])
        bad_offs = lambda b: b[:5] + (np.array([0, int(b[5][-1]), 0], np.uint64),)
        one_first = lambda b: b[:5] + (b[5] + np.uint64(1),)
        cases = [
            (-4, ov, rev(tg), 0, None),            # unsorted target accounts
            (-4, ov, swap_slots(tg), 0, None),     # unsorted target slots (the first entry holds both)
            (-4, rev(ov), tg, 0, None) if len(ov[0]) > 1 else None,
            (-3, ov, bad_offs(tg), 0, None),       # target offsets not monotone
            (-3, ov, one_first(tg), 0, None),      # target offsets not starting at 0
            (-3, one_first(ov), tg, 0, None),      # overlay offsets not starting at 0
            (-3, ov, tg, 2, None),                 # bad mode
            (-3, ov, tg, 0, 1),                    # null overlay keys
            (-3, ov, tg, 0, 7),                    # null overlay offsets
            (-3, ov, tg, 0, 8),                    # null target keys
            (-3, ov, tg, 0, 14),                   # null target offsets
            (-3, ov, tg, 0, 18),                   # null out
        ]
        for case in filter(None, cases):
            want, o, t, mode, null = case
            assert raw_call(eng, ds, o, t, mode, null) == want, (want, mode, null)
        check(eng, ds, state, {}, {})   # still usable
        _, keys, accs, skeys, svals, offs = flatten(state)
        sh = DynamicState.create(eng, keys, accs, skeys, svals, offs, sharded=True)
        try:
            assert raw_call(eng, sh, ov, tg) == -3
        finally:
            sh.close()
    finally:
        ds.close()


def test_chain_of_two_posts(eng):
    """DynamicStateRoot.overlay_witness(p1.extend(p2), p3) == a twin that committed p1 and p2 and then witness(p3)"""
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage, StateRootError
    rng = np.random.default_rng(1318)
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
    try:
        p1, p2, p3 = post_of(1), post_of(2), post_of(3)
        chain = HashedPostState(dict(p1.accounts), {k: HashedStorage(v.wiped, dict(v.storage)) for k, v in p1.storages.items()})
        chain.extend(p2)
        root = ds.overlay_root(chain)
        twin.commit(p1)
        assert twin.commit(p2)[0] == root
        for mode in MODES:
            for incl in (False, True):
                assert ds.overlay_witness(chain, p3, mode, incl) == twin.witness(p3, mode, incl)
        bad = HashedPostState({}, {rk(): HashedStorage(False, {rk(): 1})})
        with pytest.raises(StateRootError):
            ds.overlay_witness(chain, bad)
    finally:
        ds.close()
        twin.close()
