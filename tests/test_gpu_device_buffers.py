"""Device-memory accounting across owner lifecycles.  Every owner of device memory (resident trie, dynamic trie, dynamic
state, root stream, and the context's own scratch) is charged for what it allocates and gives back exactly that when it
releases it: identical rounds of create / use / close in one Engine leave identical byte counts, so a leak or a counting
drift shows up as a difference between rounds."""
import numpy as np
import pytest

from tests.test_gpu_dstate import flatten, random_block, random_state, rkey
from tests.test_gpu_witness import block_arrays

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def one_round(eng, seed):
    """-> {owner: its device_bytes() just before it is closed}; every owner is created, used and closed"""
    from reth_b200 import DynamicState, DynamicTrie, ResidentTrie, RootStream
    rng = np.random.default_rng(seed)
    state = random_state(rng, 300, with_storage=0.5, max_slots=20)
    _, keys, accs, skeys, svals, offs = flatten(state)
    n = len(keys)
    seen = {}

    # resident trie: an in-place update, then an apply with inserts and deletes (device merge + rebuild)
    t = ResidentTrie.create(eng, keys, accs)
    bumped = accs.copy()
    bumped["nonce"] += 1
    t.update(keys[::7], bumped[::7])
    inserted = sorted({rkey(rng) for _ in range(20)} - {k.tobytes() for k in keys})
    dirty = sorted([(k.tobytes(), 0) for k in keys[::5]] + [(k, 1) for k in inserted])
    dkeys = np.frombuffer(b"".join(k for k, _ in dirty), np.uint8).reshape(-1, 32)
    daccs = np.zeros(len(dirty), accs.dtype)
    daccs[:] = accs[0]
    present = np.array([p for _, p in dirty], np.uint8)
    _, rebuilt = t.apply(dkeys, daccs, present)
    assert rebuilt
    seen["trie"] = t.device_bytes()
    t.close()

    # dynamic trie: create and apply the same dirty set
    dt = DynamicTrie.create(eng, keys, accs)
    dt.apply(dkeys, daccs, present)
    seen["dtrie"] = dt.device_bytes()
    dt.close()

    # dynamic state: witness, apply, multiproof; the witness then gives the same root without the state
    ds = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    block = random_block(rng, state, 30, 1)
    arrays = block_arrays(block)
    parent, witness = ds.root(), ds.witness(*arrays)
    root = ds.apply(*arrays)
    targets = {keys[i].tobytes(): [skeys[j].tobytes() for j in range(int(offs[i]), int(offs[i + 1]))][:3] for i in range(0, n, 25)}
    targets[rkey(rng)] = [rkey(rng)]
    ds.multiproof(targets)
    seen["dstate"] = ds.device_bytes()
    ds.close()
    roots, status = eng.witness_roots([parent], [witness], [arrays])
    assert (roots[0].tobytes(), int(status[0])) == (root, 0)

    # root stream (charged to the context): three pushes of ascending key ranges, finish, close
    rs = RootStream(eng)
    for lo, hi in ((0, n // 3), (n // 3, 2 * n // 3), (2 * n // 3, n)):
        a, b = int(offs[lo]), int(offs[hi])
        rs.push(keys[lo:hi], accs[lo:hi], skeys[a:b], svals[a:b], offs[lo:hi + 1] - offs[lo])
    assert rs.finish() == eng.state_root_full(keys, accs, skeys, svals, offs)
    rs.close()
    return seen


def test_owners_release_what_they_were_charged(eng):
    rounds, after = [], []
    for _ in range(3):
        rounds.append(one_round(eng, 4242))
        after.append(eng.device_bytes())
    assert all(v > 0 for v in rounds[0].values())
    assert rounds[1] == rounds[0] and rounds[2] == rounds[0]
    assert after[2] == after[1]
