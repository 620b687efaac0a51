"""The overlay, witness and stateless paths at large blocks and wide batches (b200_dstate_overlay_roots(_with_updates),
b200_dstate_overlay_multiproof, b200_dstate_overlay_witness, b200_dstate_witness, b200_witness_roots).

They share one pipeline: a breadth-first reveal from the arenas (one launch and one read-back per level; the queue, item and
value buffers sized from the previous level and grown mid-call, keeping what was written), a key sort and merge, then two
folds through build_forest (the storage forest, then one account trie per block) that keep their stored nodes for
TrieUpdates or copy them into scratch arenas for proofs.  The other test files run it at a few hundred entries, where every
fold depth has at most WARP_LEVEL_MAX nodes (summed over the tries of the call) and takes the one-warp-per-node launch.
Every case here is sized from that threshold so that a fold depth goes past it and takes the class-split thread kernels
(`big<=3` ... `big<=16`), and asserts from the launch labels of its own call (B200_PHASE_TIMING) that they ran.  Under
the CPU emulation the threshold is lower and the same cases run at a few percent of the device sizes.

Every result is compared with a twin DynamicState on which the block is applied, followed by the same query, and at least
once per case the post-block root is also checked against the oracle's from-scratch state root over the merged state."""
import os
import re

import numpy as np
import pytest

import oracle
from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, acct, clustered_slots, flatten, model, random_block, random_state, rkey
from tests.test_gpu_level_classes import BIG, DISPATCH, launch_threshold
from tests.test_gpu_overlay_proofs import check_account_proofs, near, targets_for
from tests.test_gpu_overlay_updates import check_block as check_updates
from tests.test_gpu_proofs import verify
from tests.test_gpu_witness import EMPTY_ROOT, apply_to_model, block_arrays, model_witness

pytestmark = [pytest.mark.gpu]

MODES = ("legacy", "canonical")
# model_witness (a recursive trie in Python over the whole state) takes about 0.75 s per 10 000 accounts and slots on one
# x86 core, per mode; above this many it is left out and the witness rests on the twin and the stateless rebuild.
MODEL_WITNESS_MAX = 40_000


def scaled(n):
    """n at the device's WARP_LEVEL_MAX (4096), scaled to the threshold of the library under test"""
    return max(1, n * launch_threshold() // 4096)


def engine_with_timing():
    from reth_b200 import Engine
    old = os.environ.get("B200_PHASE_TIMING")
    os.environ["B200_PHASE_TIMING"] = "1"
    try:
        return Engine(0)
    finally:
        if old is None:
            del os.environ["B200_PHASE_TIMING"]
        else:
            os.environ["B200_PHASE_TIMING"] = old


@pytest.fixture(scope="module")
def timed():
    """the context of the states under test: every call prints its phase labels and buffer growth on stderr"""
    e = engine_with_timing()
    yield e
    e.close()


@pytest.fixture(scope="module")
def eng():
    """the context of the twins (no timing output)"""
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


class Flat:
    """a state flattened once, so that many twins can be built from it"""

    def __init__(self, state):
        self.state = state
        _, *self.arrays = flatten(state)

    def make(self, eng):
        from reth_b200 import DynamicState
        return DynamicState.create(eng, *self.arrays)


def traced(capfd, call):
    """-> (call(), {"storage": labels, "account": labels, "grows": [(from, to, keep)]}) of that call alone.  The labels are
    the launch labels of build_forest (small-level, small-class, big<=N), split at the `stateless-storage` mark that
    eng_stateless.inl sets between the storage fold and the account fold."""
    capfd.readouterr()
    out = call()
    names, grows = [], []
    for line in capfd.readouterr().err.splitlines():
        if line.startswith("[b200 phases]"):
            names += line.split(":", 1)[1].split()[0::2]
        elif line.startswith("[b200 grow]"):
            grows.append(tuple(int(x) for x in re.findall(r"\d+", line.split("]", 1)[1])))
    cut = names.index("stateless-storage") if "stateless-storage" in names else len(names)
    fold = lambda xs: [x for x in xs if x in DISPATCH]
    return out, {"storage": fold(names[:cut]), "account": fold(names[cut:]), "grows": grows}


def has_big(labels, want=None):
    """a class-split thread kernel ran (want: that one in particular)"""
    return (want in labels) if want else any(x in BIG for x in labels)


def oracle_root(state):
    return oracle.state_root_full(*flatten(state)[1:])


def same_updates(block, got, want, pre):
    """an overlay's TrieUpdates against the twin apply's (the rules of test_gpu_overlay_updates.check_block, without the
    from-scratch tables, which that function adds for a sample)"""
    root, au, ar, su, sr, deleted = got
    assert root == want[0]
    assert set(ar) == set(want[2]) and len(set(ar)) == len(ar)
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


def check_proofs(got, targets, post):
    """every account and storage proof of an overlay multiproof verifies against the returned roots (as
    test_gpu_overlay_proofs.check)"""
    check_account_proofs(got, post)
    j = 0
    for a in sorted(targets):
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
    assert j == len(got["storage_nodes"])


def multiproof_vs_twin(ds, twin_post, arrays, targets, post, trace=None):
    """ds.overlay_multiproof == twin_post.multiproof (twin_post: the block already applied), every proof verifies"""
    got = ds.overlay_multiproof(arrays, targets, with_nodes=True) if trace is None else trace(
        lambda: ds.overlay_multiproof(arrays, targets, with_nodes=True))
    mp = got[0] if trace is not None else got
    want = twin_post.multiproof(targets, with_nodes=True)
    assert mp["root"] == twin_post.root()
    for key in want:
        assert mp[key] == want[key], key
    check_proofs(mp, targets, post)
    return got


def witness_vs_twin(eng, witness_of, twin_post, target, post=None):
    """witness_of(mode) -> (overlay root, map) against twin_post.witness (twin_post: the overlay applied), in both modes;
    the stateless rebuild from the overlay root gives the twin's root after the target block.  -> node counts per mode"""
    tg = block_arrays(target)
    sizes = {}
    for mode in MODES:
        root, got = witness_of(mode)
        assert root == twin_post.root(), mode
        want = twin_post.witness(*tg, mode=mode)
        assert got == want, (mode, len(set(got) - set(want)), len(set(want) - set(got)))
        if post is not None:
            assert got == model_witness(post, target, mode), mode
        roots, status = eng.witness_roots([root], [got], [tg])
        assert status[0] == 0, mode
        sizes[mode] = (len(got), sum(len(v) for v in got.values()))
        after = roots[0].tobytes()
    return after, sizes


def report(record_property, name, info):
    """recorded as a test property, and printed (pytest -s / -rP)"""
    record_property(name, info)
    print(name, info)


def model_size(state):
    return len(state) + sum(len(s) for _, s in state.values())


# ---- 1. a wide batch of sibling blocks ---------------------------------------------------------------------------------
def test_wide_sibling_batch(timed, eng, capfd, record_property):
    """About WARP_LEVEL_MAX / 12 sibling blocks of 100 touched accounts: every block's account fold has 16 depth-1 branches
    of 16 children, so depth 1 sums past the threshold and takes the 13-16 class kernel; with updates the folds retain
    their nodes.  Empty and repeated blocks are in the batch."""
    rng = np.random.default_rng(2100)
    state = random_state(rng, scaled(20_000), with_storage=0.5, max_slots=30)
    flat = Flat(state)
    blocks = [random_block(rng, state, 100, b + 1) for b in range(launch_threshold() // 12 - 2)]
    blocks.insert(3, {})
    blocks += [blocks[1], blocks[7], {}]
    arrays = [block_arrays(b) for b in blocks]
    ds = flat.make(timed)
    try:
        parent, n_acc, n_slots = ds.root(), ds.accounts(), ds.slots()
        wants = {}
        for b, a in zip(blocks, arrays):
            if id(b) not in wants:
                twin = flat.make(eng)
                wants[id(b)] = twin.apply(*a, want_updates=True)
                twin.close()
        roots, tr = traced(capfd, lambda: ds.overlay_roots(arrays))
        assert roots == [wants[id(b)][0] for b in blocks]
        assert roots[3] == roots[-1] == parent
        assert has_big(tr["account"], "big<=16"), tr
        for i in (0, len(blocks) // 2, len(blocks) - 3):   # the independent root, the repeated block among them
            assert roots[i] == oracle_root(apply_to_model(state, blocks[i])), i
        got, tr_u = traced(capfd, lambda: ds.overlay_roots(arrays, want_updates=True))
        assert has_big(tr_u["account"], "big<=16"), tr_u
        pre = model(state)
        for i, (b, g) in enumerate(zip(blocks, got)):
            same_updates(b, g, wants[id(b)], pre)
        for i in (0, len(blocks) - 4):
            check_updates(state, blocks[i], got[i], wants[id(blocks[i])], pre)
        assert ds.root() == parent and ds.accounts() == n_acc and ds.slots() == n_slots
        report(record_property, "wide_batch", {"blocks": len(blocks), "entries": int(sum(len(a[0]) for a in arrays)),
                                               "slot_entries": int(sum(len(a[3]) for a in arrays)), "account_fold": tr["account"],
                                               "storage_fold": tr["storage"], "account_fold_with_updates": tr_u["account"]})
    finally:
        ds.close()


# ---- 2. one big block on a big state -----------------------------------------------------------------------------------
def big_state(rng):
    """scaled(200 000) accounts; scaled(5 000) contracts with 6-30 slots, scaled(400) of them with clustered slots of small
    values (inline leaves and branches); one contract with scaled(80 000) slots.  -> (state, contracts, clustered, whale)"""
    state = random_state(rng, scaled(200_000), with_storage=0.0)
    ks = sorted(state)
    pick = rng.choice(len(ks), scaled(5_000) + 1, replace=False)
    contracts = [ks[i] for i in pick[1:]]
    whale = ks[pick[0]]
    clustered = contracts[:scaled(400)]
    for k in contracts:
        slots = {rkey(rng): int(rng.integers(1, 2**62)) for _ in range(int(rng.integers(6, 31)))}
        if k in clustered:
            slots.update({s: int(rng.integers(1, 4)) for s in clustered_slots(rng, 3)})
        state[k] = (state[k][0], slots)
    state[whale] = (state[whale][0], {rkey(rng): int(rng.integers(1, 2**62)) for _ in range(scaled(80_000))})
    return state, contracts, clustered, whale


def big_block(rng, state, contracts, clustered, whale, n_touch, step):
    """About n_touch entries: scaled(5 000) contracts with slot changes (inserts, deletes, value-only changes; most of each
    cluster removed), the whale with scaled(50 000) slot changes, creations, destructions (with and without storage),
    wipes, destroyed-and-re-created accounts, balance changes and "unchanged" entries of absent accounts."""
    block = {}
    live = [k for k in sorted(state) if k != whale]
    for j, k in enumerate(k for k in contracts if k in state):
        cur = sorted(state[k][1])
        new = {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(int(rng.integers(0, 4)))}
        if j % 20 == 19:
            block[k] = (0, acct(0), {})                                                           # destroyed with storage
        elif j % 20 == 18:
            block[k] = (EXISTS | WIPED, state[k][0].copy(), new)                                   # wiped, maybe refilled
        elif j % 20 == 17:
            block[k] = (EXISTS | WIPED, acct(step, 3), new)                                        # destroyed and re-created
        else:
            ch = dict(new)
            for s in cur[:int(rng.integers(0, len(cur))) + 1 if cur else 0]:
                ch[s] = 0 if rng.random() < 0.4 else int(rng.integers(1, 2**60))
            if k in clustered:
                ch.update({s: 0 for s in cur if state[k][1][s] < 4 and rng.random() < 0.8})
            block[k] = (EXISTS | UNCHANGED, acct(0), ch)
    cur = sorted(state[whale][1])
    n = scaled(50_000)
    sel = rng.choice(len(cur), min(len(cur), 2 * n // 3), replace=False)
    wch = {cur[i]: (0 if j % 2 else int(rng.integers(1, 2**60))) for j, i in enumerate(sel)}
    while len(wch) < n:
        wch[rkey(rng)] = int(rng.integers(1, 2**60))
    block[whale] = (EXISTS | UNCHANGED, acct(0), wch)
    rest = [k for k in live if k not in block]
    order = rng.permutation(len(rest))
    n_other = max(0, n_touch - len(block))
    for j, i in enumerate(order[:n_other * 3 // 4]):
        k = rest[i]
        r = j % 8
        if r == 0:
            block[k] = (0, acct(0), {})                                                           # destroyed
        elif r == 2:
            block[k] = (EXISTS | WIPED, acct(step, 9), {rkey(rng): v + 1 for v in range(int(rng.integers(0, 6)))})   # re-created
        else:
            a = state[k][0].copy()
            a["nonce"] += 1
            block[k] = (EXISTS, a, {})                                                            # balance / nonce change
    for j in range(n_other - n_other * 3 // 4):
        if j % 10 == 0:
            block[rkey(rng)] = (EXISTS | UNCHANGED, acct(0), {rkey(rng): 7})                     # absent: ignored
        else:
            block[rkey(rng)] = (EXISTS, acct(step, 5), {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(j % 4)})
    return dict(sorted(block.items()))


def proof_targets(rng, state, block, whale, n):
    """about n targets from targets_for over a sample of the block (the whale with a sample of its slots), untouched
    accounts, absent and near-miss keys"""
    keys = sorted(block)
    sub = {keys[i]: block[keys[i]] for i in rng.choice(len(keys), min(len(keys), n * 3 // 4), replace=False)}
    wch = sorted(block[whale][2])
    sub[whale] = (block[whale][0], block[whale][1], {s: block[whale][2][s] for s in wch[::max(1, 6 * len(wch) // n)]})
    t = targets_for(rng, state, dict(sorted(sub.items())), n_untouched=n // 8, n_absent=n // 16)
    t[whale] |= {near(rng, s, int(rng.integers(1, 64))) for s in wch[:40]}
    return t


def test_big_block_on_a_big_state(timed, eng, capfd, record_property):
    rng = np.random.default_rng(2200)
    state, contracts, clustered, whale = big_state(rng)
    block = big_block(rng, state, contracts, clustered, whale, scaled(20_000), 1)
    arrays = block_arrays(block)
    post = apply_to_model(state, block)
    flat = Flat(state)
    ds, twin = flat.make(timed), flat.make(eng)
    info = {"accounts": len(state), "slots": ds.slots(), "entries": len(arrays[0]), "slot_entries": len(arrays[3]),
            "whale_slot_entries": len(block[whale][2])}
    try:
        parent = ds.root()
        want = twin.apply(*arrays, want_updates=True)
        assert want[0] == oracle_root(post)
        # roots, with and without TrieUpdates (storage-deleted flags among them)
        roots, tr = traced(capfd, lambda: ds.overlay_roots([arrays]))
        assert roots == [want[0]]
        assert has_big(tr["storage"]) and has_big(tr["account"]), tr
        got, tr_u = traced(capfd, lambda: ds.overlay_roots([arrays], want_updates=True))
        assert has_big(tr_u["storage"]) and has_big(tr_u["account"]), tr_u
        assert got[0][5].any()
        check_updates(state, block, got[0], want, model(state))
        info.update(storage_fold=tr["storage"], account_fold=tr["account"])
        # multiproof of about 2 000 targets
        targets = proof_targets(rng, state, block, whale, scaled(2_000))
        (_, tr_p) = multiproof_vs_twin(ds, twin, arrays, targets, post, trace=lambda f: traced(capfd, f))
        assert has_big(tr_p["storage"]) and has_big(tr_p["account"]), tr_p
        info.update(proof_targets=len(targets), proof_slot_targets=sum(len(v) for v in targets.values()))
        # the witness of a second big block on top of this one
        target = big_block(rng, post, [k for k in contracts if k in post], [k for k in clustered if k in post], whale,
                           scaled(10_000), 2)
        ov_w = lambda mode: traced(capfd, lambda: ds.overlay_witness(arrays, block_arrays(target), mode=mode))
        labels = {}

        def witness_of(mode):
            out, t = ov_w(mode)
            labels[mode] = t
            return out
        after, sizes = witness_vs_twin(eng, witness_of, twin, target,
                                       post if model_size(post) <= MODEL_WITNESS_MAX else None)
        assert all(has_big(t["storage"]) and has_big(t["account"]) for t in labels.values()), labels
        assert after == twin.apply(*block_arrays(target))
        info.update(overlay_witness_nodes=sizes)
        # the witness of the big block itself, from the resident state
        pre = Flat(state).make(eng)
        try:
            after, sizes = witness_vs_twin(eng, lambda mode: (ds.root(), ds.witness(*arrays, mode=mode)), pre, block,
                                           state if model_size(state) <= MODEL_WITNESS_MAX else None)
        finally:
            pre.close()
        assert after == want[0]
        info.update(witness_nodes=sizes)
        assert ds.root() == parent
        report(record_property, "big_block", info)
    finally:
        ds.close()
        twin.close()


# ---- 3. scratch that grows in the middle of a call ---------------------------------------------------------------------
def test_growth_from_a_fresh_context(eng, capfd, record_property):
    """The first call on a new context is a big overlay with TrieUpdates: the reveal's queue, item, value and candidate
    buffers start at the size of the seeds and grow level by level, keeping what the earlier levels wrote (eng_overlay.inl
    grow(..., keep)).  A large multiproof follows, then a tiny call, then the big ones again: all outputs equal, and equal
    to the twin's.

    The block seeds the reveal with four roots (the account trie's and three storage tries'), each of which fans out to
    16 children on the first level: the next-level queue must take the full fan-out of a branch, not an average one."""
    rng = np.random.default_rng(2300)
    state = random_state(rng, scaled(20_000), with_storage=0.5, max_slots=30)
    live = sorted(state)
    big = live[:3]
    block = {}
    for k in big:   # three storage tries with many slot changes: inserts, deletes, value-only changes
        slots = {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(scaled(30_000))}
        state[k] = (state[k][0], slots)
        ch = {s: (0 if j % 2 else 9) for j, s in enumerate(sorted(slots)[::3])}
        ch.update({rkey(rng): 5 for _ in range(scaled(1_000))})
        block[k] = (EXISTS | UNCHANGED, acct(0), ch)
    for j, i in enumerate(rng.choice(np.arange(3, len(live)), scaled(8_000), replace=False)):   # account-only changes
        k = live[i]
        if j % 5 == 0:
            block[k] = (0, acct(0), {})
        else:
            a = state[k][0].copy()
            a["nonce"] += 1
            block[k] = (EXISTS, a, {})
    block.update({rkey(rng): (EXISTS, acct(3, 3), {}) for _ in range(scaled(1_000))})
    block = dict(sorted(block.items()))
    arrays = block_arrays(block)
    post = apply_to_model(state, block)
    flat = Flat(state)
    fresh = engine_with_timing()
    ds = twin = None
    try:
        ds, twin = flat.make(fresh), flat.make(eng)
        want = twin.apply(*arrays, want_updates=True)
        assert want[0] == oracle_root(post)
        first, tr = traced(capfd, lambda: ds.overlay_roots([arrays], want_updates=True))
        kept = [g for g in tr["grows"] if g[2] > 0]
        assert kept, tr["grows"]          # the reveal grew its buffers mid-call, keeping what it had written
        assert has_big(tr["storage"]), tr
        same_updates(block, first[0], want, model(state))
        targets = targets_for(rng, state, block, n_untouched=scaled(2_000), n_absent=scaled(500))
        mp_first = multiproof_vs_twin(ds, twin, arrays, targets, post)
        small = random_block(rng, state, 3, 2)
        tiny = flat.make(eng)
        try:
            assert ds.overlay_roots([block_arrays(small)]) == [tiny.apply(*block_arrays(small))]
        finally:
            tiny.close()
        again = ds.overlay_roots([arrays], want_updates=True)
        for a, b in zip(first[0], again[0]):
            assert np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b
        assert ds.overlay_multiproof(arrays, targets, with_nodes=True) == mp_first
        report(record_property, "growth", {"entries": len(arrays[0]), "slot_entries": len(arrays[3]), "grows": tr["grows"],
                                           "grows_keeping": len(kept), "account_fold": tr["account"], "storage_fold": tr["storage"]})
    finally:
        for x in (ds, twin):
            if x is not None:
                x.close()
        fresh.close()


# ---- 4. deep and one-sided shapes at scale ------------------------------------------------------------------------------
def under(rng, head, nibbles):
    """a random key whose first `nibbles` nibbles are those of `head`"""
    k = bytearray(rkey(rng))
    full, odd = divmod(nibbles, 2)
    k[:full] = head[:full]
    if odd:
        k[full] = (head[full] & 0xF0) | (k[full] & 0x0F)
    return bytes(k)


def test_deep_and_one_sided_shapes(timed, eng, capfd, record_property):
    """Thousands of accounts under one top nibble and one storage trie under a 10-nibble extension, with blocks that put one
    depth of each past the threshold; then removals of every key outside one subtree of each, so that a big subtree
    collapses onto a sibling no key reaches (a hash item of the fold), with proof targets in the collapsed region."""
    rng = np.random.default_rng(2400)
    top = bytes([0x70])
    state = {under(rng, top, 1): (acct(int(rng.integers(1, 9)), int(rng.integers(1, 2**40))), {})
             for _ in range(scaled(40_000))}
    state.update(random_state(rng, 300, with_storage=0.3, max_slots=10))
    owner = sorted(k for k in state if k[0] >> 4 != 7)[0]
    head = rkey(rng)
    state[owner] = (state[owner][0], {under(rng, head, 10): int(rng.integers(1, 2**60)) for _ in range(scaled(40_000))})
    flat = Flat(state)
    ds = flat.make(timed)
    info = {"accounts": len(state), "owner_slots": len(state[owner][1])}
    try:
        parent = ds.root()
        seven = sorted(k for k in state if k[0] >> 4 == 7)
        slots = sorted(state[owner][1])
        # three siblings that touch a third of the nibble-7 accounts each; the first also rewrites 40 % of the owner's slots
        blocks = []
        for b in range(3):
            blk = {seven[i]: (EXISTS, acct(b + 10, i), {}) for i in rng.choice(len(seven), len(seven) // 3, replace=False)}
            blk[under(rng, bytes([0x30]), 1)] = (EXISTS, acct(1), {})
            if b == 0:
                ch = {slots[i]: (0 if i % 3 == 0 else int(rng.integers(1, 2**60)))
                      for i in rng.choice(len(slots), len(slots) * 2 // 5, replace=False)}
                ch.update({under(rng, head, 10): 3 for _ in range(scaled(2_000))})
                blk[owner] = (EXISTS | UNCHANGED, acct(0), ch)
            blocks.append(dict(sorted(blk.items())))
        arrays = [block_arrays(b) for b in blocks]
        wants = []
        for a in arrays:
            twin = flat.make(eng)
            wants.append(twin.apply(*a, want_updates=True))
            twin.close()
        got, tr = traced(capfd, lambda: ds.overlay_roots(arrays, want_updates=True))
        assert has_big(tr["account"]) and has_big(tr["storage"]), tr
        pre = model(state)
        for b, g, w in zip(blocks, got, wants):
            same_updates(b, g, w, pre)
        assert got[0][0] == oracle_root(apply_to_model(state, blocks[0]))
        info.update(sibling_account_fold=tr["account"], sibling_storage_fold=tr["storage"])
        # collapse: every nibble-7 account outside 7a.., every owner slot outside head + one nibble
        keep_a = lambda k: k[0] == 0x7A
        keep_nib = (head[5] >> 4)
        keep_s = lambda s: s[5] >> 4 == keep_nib
        block = {k: (0, acct(0), {}) for k in seven if not keep_a(k)}
        block[owner] = (EXISTS | UNCHANGED, acct(0), {s: 0 for s in slots if not keep_s(s)})
        block = dict(sorted(block.items()))
        a = block_arrays(block)
        post = apply_to_model(state, block)
        twin = flat.make(eng)
        try:
            want = twin.apply(*a, want_updates=True)
            assert want[0] == oracle_root(post)
            g, tr_c = traced(capfd, lambda: ds.overlay_roots([a], want_updates=True))
            check_updates(state, block, g[0], want, pre)
            gone = [k for k in seven if not keep_a(k)]
            kept = [k for k in seven if keep_a(k)]
            targets = {k: set() for k in gone[::max(1, len(gone) // 300)] + kept[::max(1, len(kept) // 100)]}
            targets.update({near(rng, kept[0], d): set() for d in range(1, 20)})
            targets.update({under(rng, bytes([0x7A]), 2): set() for _ in range(20)})
            targets.update({under(rng, top, 1): set() for _ in range(20)})
            live = sorted(s for s in slots if keep_s(s))
            dead = [s for s in slots if not keep_s(s)]
            targets[owner] = set(live[::max(1, len(live) // 200)] + dead[::max(1, len(dead) // 200)] +
                                 [near(rng, live[0], d) for d in range(1, 40)] + [under(rng, head, 11) for _ in range(20)])
            targets = {k: targets[k] for k in sorted(targets)}
            _, tr_p = multiproof_vs_twin(ds, twin, a, targets, post, trace=lambda f: traced(capfd, f))
            info.update(collapse_entries=len(a[0]), collapse_slot_entries=len(a[3]), collapse_account_fold=tr_c["account"],
                        collapse_storage_fold=tr_c["storage"], proof_targets=len(targets))
        finally:
            twin.close()
        assert ds.root() == parent
        report(record_property, "deep_shapes", info)
    finally:
        ds.close()
