"""Merkle multiproofs of a candidate block on top of the resident state, without changing it (b200_dstate_overlay_multiproof;
reth's Proof::overlay_multiproof, what StateProofProvider::multiproof of a MemoryOverlayStateProvider returns).  The
reference in every test is a twin state on which the block is applied, followed by multiproof of the same targets: the full
dict (account subtree, branch masks, every storage's root, subtree and masks) and every target's node list in order must be
equal, and every proof must verify against the returned root."""
import ctypes as C

import numpy as np
import oracle
import pytest

from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, acct, clustered_slots, random_block, random_state, rkey
from tests.test_gpu_proofs import verify
from tests.test_gpu_witness import EMPTY_ROOT, KECCAK, account_enc, apply_to_model, block_arrays, make_state

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def near(rng, key, shared):
    """a key that shares exactly `shared` nibbles with `key` (1..63)"""
    k = bytearray(key)
    b, hi = divmod(shared, 2)
    nib = (k[b] >> 4, k[b] & 15)[hi]
    new = (nib + int(rng.integers(1, 16))) % 16
    k[b] = (new << 4 | (k[b] & 15)) if hi == 0 else ((k[b] & 0xF0) | new)
    for i in range(b + 1, 32):
        k[i] = int(rng.integers(0, 256))
    if hi == 0:
        k[b] = (k[b] & 0xF0) | int(rng.integers(0, 16))
    return bytes(k)


def targets_for(rng, state, block, n_untouched=20, n_absent=10):
    """every entry with its written, deleted, untouched and absent slots; untouched accounts with slots; absent and
    near-miss keys (sharing 1..63 nibbles with a block or resident key) with slots"""
    t = {}
    post = apply_to_model(state, block)
    for k, (_, _, slots) in block.items():
        cur = sorted(state[k][1]) if k in state else []
        after = sorted(post[k][1]) if k in post else []
        sel = set(slots) | set(cur[:3]) | set(after[:3]) | {rkey(rng)}
        if slots:
            sel.add(near(rng, sorted(slots)[0], int(rng.integers(1, 64))))
        t[k] = sel
    live = sorted(state)
    for i in rng.choice(len(live), min(n_untouched, len(live)), replace=False) if live else []:
        k = live[i]
        t.setdefault(k, set()).update(sorted(state[k][1])[:3] + [rkey(rng)])
    refs = sorted(set(block) | set(state))
    for _ in range(n_absent):
        t[rkey(rng)] = {rkey(rng)}
        if refs:
            k = refs[int(rng.integers(0, len(refs)))]
            t[near(rng, k, int(rng.integers(1, 64)))] = {rkey(rng)}
    return t


def check_account_proofs(got, post):
    """every account proof verifies against the returned root, with the post-state's leaf"""
    for i, a in enumerate(sorted(got["storages"])):
        proof = [rlp for _, rlp, _ in got["account_nodes"][i]]
        sroot = got["storages"][a]["root"]
        if got["root"] == EMPTY_ROOT:
            assert a not in post and sroot == EMPTY_ROOT and proof == [b"\x80"]
        elif a in post:
            verify(got["root"], a, proof, account_enc(post[a][0], sroot))
        else:
            assert sroot == EMPTY_ROOT
            verify(got["root"], a, proof, None)


def check(eng, state, block, targets, ds=None):
    """overlay multiproof on `ds` (or a fresh state) == apply + multiproof on a twin; returns the twin's root"""
    own = ds is None
    if own:
        ds = make_state(eng, state)
    twin = make_state(eng, state)
    try:
        parent = ds.root()
        arrays = block_arrays(block)
        got = ds.overlay_multiproof(arrays, targets, with_nodes=True)
        assert ds.root() == parent
        root = twin.apply(*arrays)
        want = twin.multiproof(targets, with_nodes=True)
        assert got["root"] == root
        for key in want:
            assert got[key] == want[key], key
        post = apply_to_model(state, block)
        check_account_proofs(got, post)
        addrs = sorted(targets)
        j = 0
        for a in addrs:
            sroot = got["storages"][a]["root"]
            slots = post[a][1] if a in post else {}
            for s in sorted(set(bytes(x) for x in targets[a])):
                proof = [rlp for _, rlp, _ in got["storage_nodes"][j]]
                j += 1
                if sroot == EMPTY_ROOT:
                    assert proof == [b"\x80"]
                    continue
                v = slots.get(s)
                verify(sroot, s, proof, None if v is None else oracle.encode_u256(int(v)))
        return root
    finally:
        twin.close()
        if own:
            ds.close()


@pytest.mark.parametrize("n0,touch", [(5, 6), (300, 40), (3000, 250)])
def test_random_blocks(eng, n0, touch):
    """four steps, the block committed between steps, so later overlays see freed and reused arena slots"""
    rng = np.random.default_rng(1200 + n0)
    state = random_state(rng, n0, with_storage=0.5, max_slots=30)
    ds = make_state(eng, state)
    try:
        for step in range(4):
            block = random_block(rng, state, touch, step + 1)
            root = check(eng, state, block, targets_for(rng, state, block), ds=ds)
            assert ds.apply(*block_arrays(block)) == root
            state = apply_to_model(state, block)
    finally:
        ds.close()


def test_collapse_and_inline_shapes(eng):
    """clustered slots with small values (inline leaves and branches); removals that collapse onto hashed, inline and revealed
    survivors; inserts that split an extension; destroyed accounts"""
    rng = np.random.default_rng(1210)
    state = random_state(rng, 300, with_storage=0.3, max_slots=20)
    owners = sorted(state)[:30]
    for k in owners:
        state[k] = (state[k][0], {s: int(rng.integers(1, 4)) for s in clustered_slots(rng, 5)})
    for step in range(3):
        block = {}
        for k in owners[step * 10:(step + 1) * 10]:
            slots = sorted(state[k][1])
            ch = {s: 0 for s in slots[int(rng.integers(0, 3)):]}
            nb = bytearray(slots[0])
            nb[20] ^= 0x10
            ch[bytes(nb)] = int(rng.integers(1, 3)) if step else 0
            split = bytearray(slots[-1])
            split[1] ^= 0x01
            ch[bytes(split)] = 7
            block[k] = (EXISTS | UNCHANGED, acct(0), ch)
        live = sorted(set(state) - set(owners))
        for i in rng.choice(len(live), 25, replace=False):
            block[live[i]] = (0, acct(0), {})
        targets = targets_for(rng, state, block)
        for k in owners:   # every slot of every clustered trie, touched or not
            targets.setdefault(k, set()).update(state[k][1])
        check(eng, state, block, targets)
        state = apply_to_model(state, block)


def test_extension_divergence(eng):
    """targets that leave an extension the block does not touch, and inserts that split it"""
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
    diverge2 = bytearray(ext[0])
    diverge2[19] ^= 0x10
    outside = KECCAK(bytes([100, 0]))
    targets = {bytes(diverge): {KECCAK(b"s")}, bytes(diverge2): {KECCAK(b"s")}, ext[0]: set(state[ext[0]][1]),
               ext[5]: set(state[ext[5]][1]) | {KECCAK(b"x")}}
    blocks = [
        {outside: (EXISTS, acct(5), {})},                                            # the extension is not touched
        {bytes(diverge): (EXISTS, acct(7), {})},                                     # insert splitting the extension
        {bytes(diverge2): (EXISTS | UNCHANGED, acct(0), {KECCAK(b"s"): 1})},          # ignored entry of an absent account
        {ext[0]: (0, acct(0), {}), bytes(diverge): (EXISTS, acct(9), {})},
        {k: (0, acct(0), {}) for k in ext[1:]},                                      # collapse onto the last one
    ]
    for b in blocks:
        check(eng, state, dict(sorted(b.items())), targets)


def test_storage_lifecycle(eng):
    """wiped, destroyed, created and emptied storages; unchanged entries of absent accounts; account-only changes"""
    rng = np.random.default_rng(1211)
    state = random_state(rng, 200, with_storage=0.6, max_slots=25)
    with_sto = [k for k in sorted(state) if state[k][1]]
    blocks = [
        {with_sto[0]: (EXISTS | WIPED, state[with_sto[0]][0].copy(), {rkey(rng): 5, rkey(rng): 6})},
        {with_sto[1]: (EXISTS | WIPED, acct(9), {})},
        {with_sto[2]: (EXISTS | UNCHANGED | WIPED, acct(0), {rkey(rng): 1})},
        {with_sto[3]: (0, acct(0), {})},
        {with_sto[4]: (0, acct(0), {rkey(rng): 1})},
        {rkey(rng): (EXISTS | UNCHANGED, acct(0), {rkey(rng): 1})},
        {rkey(rng): (EXISTS, acct(0), {})},
        {rkey(rng): (EXISTS, acct(2), {rkey(rng): 3 for _ in range(4)})},
        {k: (EXISTS | UNCHANGED, acct(0), {s: 0 for s in state[k][1]}) for k in with_sto[5:9]},
        {with_sto[9]: (EXISTS, acct(4, 4), {})},
    ]
    for b in blocks:
        b = dict(sorted(b.items()))
        targets = targets_for(rng, state, b, n_untouched=10, n_absent=4)
        for k in b:
            targets[k] = set(targets[k]) | set(state[k][1] if k in state else {})
        check(eng, state, b, targets)


def test_empty_state_and_emptying_blocks(eng):
    rng = np.random.default_rng(1212)
    new = dict(sorted({rkey(rng): (EXISTS, acct(3), {rkey(rng): 4}) for _ in range(5)}.items()))
    check(eng, {}, new, targets_for(rng, {}, new))
    check(eng, {}, {rkey(rng): (0, acct(0), {})}, {rkey(rng): {rkey(rng)}})
    state = random_state(rng, 30, with_storage=0.5, max_slots=6)
    gone = {k: (0, acct(0), {}) for k in state}
    assert check(eng, state, gone, targets_for(rng, state, gone)) == EMPTY_ROOT


def test_accounts_in_one_top_nibble(eng):
    rng = np.random.default_rng(1213)
    state = {}
    for _ in range(300):
        k = bytearray(rkey(rng))
        k[0] = 0x70 | (k[0] & 0x0F)
        state[bytes(k)] = (acct(int(rng.integers(1, 9)), int(rng.integers(1, 2**40))),
                           {rkey(rng): int(rng.integers(1, 2**40)) for _ in range(int(rng.integers(0, 4)))})
    block = random_block(rng, state, 20, 1)
    outside = bytearray(rkey(rng))
    outside[0] = 0x30
    block[bytes(outside)] = (EXISTS, acct(1), {})
    block = dict(sorted(block.items()))
    check(eng, state, block, targets_for(rng, state, block))


def test_empty_block_zero_targets_and_no_slot_targets(eng):
    rng = np.random.default_rng(1214)
    state = random_state(rng, 100, with_storage=0.5, max_slots=10)
    ds = make_state(eng, state)
    try:
        targets = targets_for(rng, state, {})
        got = ds.overlay_multiproof(block_arrays({}), targets, with_nodes=True)
        want = ds.multiproof(targets, with_nodes=True)
        assert got.pop("root") == ds.root()
        assert got == want
        block = random_block(rng, state, 10, 1)
        check(eng, state, block, {}, ds=ds)
        check(eng, state, block, {k: () for k in targets_for(rng, state, block)}, ds=ds)
    finally:
        ds.close()


def test_chain_of_two_posts(eng):
    """DynamicStateRoot.overlay_multiproof(p1.extend(p2)) == a twin that committed p1 and then p2"""
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage
    rng = np.random.default_rng(1215)
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
        p1, p2 = post_of(1), post_of(2)
        chain = HashedPostState(dict(p1.accounts), {k: HashedStorage(v.wiped, dict(v.storage)) for k, v in p1.storages.items()})
        chain.extend(p2)
        targets = {}
        for p in (p1, p2):
            for k in p.accounts:
                targets[k] = set(p.storages[k].storage if k in p.storages else ()) | {rk()}
        for k in live[:10]:
            targets.setdefault(k, set()).update(base.storages[k].storage if k in base.storages else ())
        targets[rk()] = {rk()}
        parent = ds.root()
        got = ds.overlay_multiproof(chain, targets)
        twin.commit(p1)
        root, _ = twin.commit(p2)
        want = twin.ds.multiproof(targets)
        assert got.pop("root") == root
        assert got == want
        assert ds.root() == parent
    finally:
        ds.close()
        twin.close()


def test_state_is_unchanged(eng):
    """overlay multiproofs interleaved with overlay roots leave root, multiproof, witness and the next apply as a twin's"""
    rng = np.random.default_rng(1216)
    state = random_state(rng, 300, with_storage=0.5, max_slots=20)
    ds, twin = make_state(eng, state), make_state(eng, state)
    try:
        for step in range(3):
            block = random_block(rng, state, 30, step + 1)
            ds.overlay_multiproof(block_arrays(block), targets_for(rng, state, block))
            ds.overlay_roots([block_arrays(block)])
        nxt = random_block(rng, state, 30, 9)
        targets = targets_for(rng, state, nxt)
        assert ds.root() == twin.root()
        assert ds.multiproof(targets, with_nodes=True) == twin.multiproof(targets, with_nodes=True)
        arrays = block_arrays(nxt)
        assert ds.witness(*arrays) == twin.witness(*arrays)
        assert ds.apply(*arrays) == twin.apply(*arrays)
        assert ds.multiproof(targets, with_nodes=True) == twin.multiproof(targets, with_nodes=True)
    finally:
        ds.close()
        twin.close()


def raw_call(eng, ds, block, keys, offs, skeys, null=None):
    from reth_b200.engine import Proofs, _ptr
    k, a, f, sk, sv, so = block
    n = len(keys)
    ak = np.frombuffer(b"".join(keys), np.uint8).reshape(n, 32) if n else np.zeros((0, 32), np.uint8)
    tk = np.frombuffer(b"".join(skeys), np.uint8).reshape(len(skeys), 32) if skeys else np.zeros((0, 32), np.uint8)
    to = np.array(offs, np.uint64)
    sroots = np.zeros((max(n, 1), 32), np.uint8)
    root = np.zeros(32, np.uint8)
    pa, ps = Proofs(), Proofs()
    args = [ds.handle, _ptr(k), _ptr(a), _ptr(f), len(k), _ptr(sk), _ptr(sv), _ptr(so), _ptr(ak), n, _ptr(to), _ptr(tk), _ptr(root),
            C.byref(pa), _ptr(sroots), C.byref(ps), None]
    if null is not None:
        args[null] = None
    r = eng.lib.b200_dstate_overlay_multiproof(*args)
    return r, pa, ps


def test_errors(eng):
    from reth_b200 import DynamicState
    from tests.test_gpu_dstate import flatten
    rng = np.random.default_rng(1217)
    state = random_state(rng, 50, with_storage=0.5, max_slots=6)
    ds = make_state(eng, state)
    try:
        block = random_block(rng, state, 5, 1)
        arrays = block_arrays(block)
        a, b = sorted([rkey(rng), rkey(rng)])
        s1, s2 = sorted([rkey(rng), rkey(rng)])
        ok = raw_call(eng, ds, arrays, [a, b], [0, 1, 2], [s1, s2])
        assert ok[0] == 0
        for p in ok[1:]:
            eng.lib.b200_proofs_release(C.byref(p))
        cases = [
            (-4, ([b, a], [0, 1, 2], [s1, s2], None)),          # unsorted account targets
            (-4, ([a, b], [0, 2, 2], [s2, s1], None)),          # unsorted slot targets
            (-4, ([a, a], [0, 0, 0], [], None)),                # duplicate account targets
            (-3, ([a, b], [1, 1, 2], [s1, s2], None)),          # offsets not starting at 0
            (-3, ([a, b], [0, 2, 1], [s1, s2], None)),          # offsets not monotone
            (-3, ([a, b], [0, 1, 2], [s1, s2], 13)),            # null account proofs
            (-3, ([a, b], [0, 1, 2], [s1, s2], 14)),            # null storage roots
            (-3, ([a, b], [0, 1, 2], [s1, s2], 15)),            # null storage proofs
            (-3, ([a, b], [0, 1, 2], [s1, s2], 10)),            # null target offsets
            (-3, ([a, b], [0, 1, 2], [s1, s2], 11)),            # null slot target keys
            (-3, ([a, b], [0, 1, 2], [s1, s2], 1)),             # null block keys
        ]
        for want, (keys, offs, skeys, null) in cases:
            r, pa, ps = raw_call(eng, ds, arrays, keys, offs, skeys, null)
            assert r == want, (want, keys == [b, a], offs, null)
            for p in (pa, ps):
                assert p.n_targets == 0 and p.n_nodes == 0 and not p._owner and not p.rlp
        if len(arrays[0]) >= 2:   # unsorted block keys
            k = arrays[0][::-1].copy()
            bad = (k,) + tuple(arrays[1:])
            assert raw_call(eng, ds, bad, [a, b], [0, 1, 2], [s1, s2])[0] == -4
        _, keys, accs, skeys, svals, offs = flatten(state)
        sh = DynamicState.create(eng, keys, accs, skeys, svals, offs, sharded=True)
        try:
            r, pa, ps = raw_call(eng, sh, arrays, [a, b], [0, 1, 2], [s1, s2])
            assert r == -3
        finally:
            sh.close()
    finally:
        ds.close()
