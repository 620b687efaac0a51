"""Dynamic resident trie (b200_dtrie_*, SURVEY §8 f1 / a10): inserts, deletes and value updates applied in place,
checked after every block against a from-scratch oracle build — the root, and the stored-node set a database would hold
after applying the block's TrieUpdates (updated nodes written, removed paths deleted).  Modelled on reth's
fuzz_in_memory_account_nodes / incremental-vs-full tests (crates/trie/db/tests/trie.rs, fuzz_in_memory_nodes.rs)."""
import os

import numpy as np
import pytest

import oracle
from tests.util import synth_accounts

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def acct(nonce):
    a = np.zeros((), oracle.ACCOUNT_DTYPE)
    a["nonce"] = nonce
    a["code_hash"] = np.frombuffer(oracle.KECCAK_EMPTY, np.uint8)
    return a


def model(state):
    ks = sorted(state)
    k = np.frombuffer(b"".join(ks), np.uint8).reshape(-1, 32) if ks else np.zeros((0, 32), np.uint8)
    acc = np.zeros(len(ks), oracle.ACCOUNT_DTYPE)
    for i, kk in enumerate(ks):
        acc[i] = state[kk]
    root, upd = oracle.state_root(k, acc, want_updates=True)
    return root, {r[1]: r[2:] for r in upd}


class Harness:
    def __init__(self, eng, n0, seed):
        from reth_b200 import DynamicTrie
        keys, accs = synth_accounts(seed, n0)
        self.state = {keys[i].tobytes(): accs[i].copy() for i in range(n0)}
        self.trie = DynamicTrie.create(eng, keys, accs)
        root, nodes = model(self.state)
        assert self.trie._root == root
        self.db = dict(nodes)

    def commit(self, dirty):
        """dirty: {key: (present, account)}"""
        ks = sorted(dirty)
        dk = np.frombuffer(b"".join(ks), np.uint8).reshape(-1, 32) if ks else np.zeros((0, 32), np.uint8)
        da = np.zeros(len(ks), oracle.ACCOUNT_DTYPE)
        pres = np.zeros(len(ks), np.uint8)
        for i, k in enumerate(ks):
            pres[i], da[i] = dirty[k]
            if dirty[k][0]:
                self.state[k] = dirty[k][1]
            else:
                self.state.pop(k, None)
        root, updated, removed = self.trie.apply(dk, da, pres, want_updates=True)
        o_root, o_nodes = model(self.state)
        assert root == o_root == self.trie.root()
        assert len(self.trie) == len(self.state)
        for p in removed:
            self.db.pop(p, None)
        for r in updated:
            assert r[1] not in removed            # updated nodes take precedence (updates.rs:160-167)
            self.db[r[1]] = r[2:]
        assert self.db == o_nodes                  # what AccountsTrie would hold == the full rebuild's node set
        return updated, removed


def random_block(rng, state, m, step):
    existing = sorted(state)
    dirty = {}
    for _ in range(m):
        r = rng.integers(0, 5)
        if r == 0 and existing:
            k = existing[rng.integers(0, len(existing))]
            a = state[k].copy()
            a["nonce"] += 1
            dirty[k] = (1, a)
        elif r == 1 and existing:
            dirty[existing[rng.integers(0, len(existing))]] = (0, acct(0))
        elif r == 2:
            dirty[rng.integers(0, 256, 32, dtype=np.uint8).tobytes()] = (1, acct(step + 1))
        elif r == 3 and existing:   # a new key sharing a long prefix with an existing one: deep splits
            b = bytearray(existing[rng.integers(0, len(existing))])
            b[int(rng.integers(1, 32))] ^= int(rng.integers(1, 256))
            dirty[bytes(b)] = (1, acct(5))
        else:                        # deleting an absent key is a no-op
            dirty[rng.integers(0, 256, 32, dtype=np.uint8).tobytes()] = (0, acct(0))
    return dirty


@pytest.mark.parametrize("n0,blocks,m", [(0, 6, 5), (1, 6, 4), (2, 8, 6), (50, 10, 20), (2000, 6, 200)])
def test_random_blocks_match_full_rebuild(eng, n0, blocks, m):
    rng = np.random.default_rng(1000 + n0)
    h = Harness(eng, n0, seed=n0 + 1)
    for step in range(blocks):
        h.commit(random_block(rng, h.state, m, step))
    h.trie.close()


def test_shrink_to_empty_and_regrow(eng):
    h = Harness(eng, 300, seed=11)
    h.commit({k: (0, acct(0)) for k in h.state})                      # everything
    assert h.trie.root() == oracle.EMPTY_ROOT_HASH and len(h.trie) == 0
    rng = np.random.default_rng(5)
    h.commit({rng.integers(0, 256, 32, dtype=np.uint8).tobytes(): (1, acct(3)) for _ in range(100)})
    h.commit({k: (0, acct(0)) for k in sorted(h.state)[1:]})          # down to a single leaf (root = that leaf)
    assert len(h.trie) == 1
    h.commit({rng.integers(0, 256, 32, dtype=np.uint8).tobytes(): (1, acct(4)) for _ in range(3)})
    h.commit({k: (0, acct(0)) for k in h.state})
    assert h.trie.root() == oracle.EMPTY_ROOT_HASH
    h.trie.close()


def test_repeated_halving_then_deep_siblings(eng):
    h = Harness(eng, 500, seed=12)
    for _ in range(3):                                                 # collapse cascades
        h.commit({k: (0, acct(0)) for k in sorted(h.state)[::2]})
    rng = np.random.default_rng(6)
    h.commit({rng.integers(0, 256, 32, dtype=np.uint8).tobytes(): (1, acct(3)) for _ in range(400)})
    deep = {}
    for k in sorted(h.state)[:40]:
        for flip in (0x01, 0x10):                                      # keys sharing 63 / 62 nibbles with an existing one
            b = bytearray(k)
            b[31] ^= flip
            deep[bytes(b)] = (1, acct(9))
    h.commit(deep)
    h.commit({k: (0, acct(0)) for k in h.state if k[31] & 1})
    h.commit(deep)
    h.trie.close()


def test_bulk_insert_into_empty_trie_runs(eng):
    # every key of the first block attaches at the root: one long run per root nibble afterwards
    h = Harness(eng, 0, seed=13)
    rng = np.random.default_rng(7)
    h.commit({rng.integers(0, 256, 32, dtype=np.uint8).tobytes(): (1, acct(1)) for _ in range(1500)})
    h.commit({k: (0, acct(0)) for k in sorted(h.state)[::2]})
    h.commit({rng.integers(0, 256, 32, dtype=np.uint8).tobytes(): (1, acct(2)) for _ in range(1500)})
    h.trie.close()


def test_value_only_blocks_report_no_removals(eng):
    h = Harness(eng, 3000, seed=14)
    rng = np.random.default_rng(8)
    ks = sorted(h.state)
    dirty = {}
    for i in rng.choice(len(ks), 300, replace=False):
        a = h.state[ks[i]].copy()
        a["balance"][31] ^= 1
        dirty[ks[i]] = (1, a)
    updated, removed = h.commit(dirty)
    assert removed == [] and len(updated) > 0
    h.trie.close()


def test_storage_roots_follow_accounts(eng):
    from reth_b200 import DynamicTrie
    n = 400
    keys, accs = synth_accounts(15, n)
    rng = np.random.default_rng(9)
    sroots = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    t = DynamicTrie.create(eng, keys, accs, sroots)
    assert t._root == oracle.state_root(keys, accs, sroots)
    # update 50 storage roots, insert 20 accounts (with roots), delete 30
    idx = rng.choice(n, 80, replace=False)
    new_keys = rng.integers(0, 256, (20, 32), dtype=np.uint8)
    dirty = {}
    for i in idx[:50]:
        dirty[keys[i].tobytes()] = (1, accs[i], rng.integers(0, 256, 32, dtype=np.uint8))
    for i in idx[50:]:
        dirty[keys[i].tobytes()] = (0, accs[i], np.zeros(32, np.uint8))
    for k in new_keys:
        dirty[k.tobytes()] = (1, acct(1), rng.integers(0, 256, 32, dtype=np.uint8))
    ks = sorted(dirty)
    dk = np.frombuffer(b"".join(ks), np.uint8).reshape(-1, 32)
    da = np.zeros(len(ks), oracle.ACCOUNT_DTYPE)
    pres = np.zeros(len(ks), np.uint8)
    dsr = np.zeros((len(ks), 32), np.uint8)
    state = {keys[i].tobytes(): (accs[i], sroots[i]) for i in range(n)}
    for i, k in enumerate(ks):
        pres[i], da[i], dsr[i] = dirty[k]
        if pres[i]:
            state[k] = (da[i], dsr[i])
        else:
            state.pop(k)
    root = t.apply(dk, da, pres, dsr)
    sk = sorted(state)
    fk = np.frombuffer(b"".join(sk), np.uint8).reshape(-1, 32)
    fa = np.zeros(len(sk), oracle.ACCOUNT_DTYPE)
    fs = np.zeros((len(sk), 32), np.uint8)
    for i, k in enumerate(sk):
        fa[i], fs[i] = state[k]
    assert root == oracle.state_root(fk, fa, fs)
    t.close()


def test_rejects_unsorted_or_duplicate_keys_and_stays_consistent(eng):
    from reth_b200._lib import B200Error
    h = Harness(eng, 100, seed=16)
    ks = sorted(h.state)
    before = h.trie.root()
    bad = np.frombuffer(ks[5] + ks[3], np.uint8).reshape(2, 32)
    with pytest.raises(B200Error):
        h.trie.apply(bad, np.zeros(2, oracle.ACCOUNT_DTYPE))
    dup = np.frombuffer(ks[5] + ks[5], np.uint8).reshape(2, 32)
    with pytest.raises(B200Error):
        h.trie.apply(dup, np.zeros(2, oracle.ACCOUNT_DTYPE))
    assert h.trie.root() == before
    h.commit({ks[0]: (0, acct(0))})      # still usable
    h.trie.close()


def test_split_runs_share_an_attach_point(eng):
    """K1 < K2 < K3 where K1 and K3 diverge inside the (long) edge above a node N and K2 passes through it: K1 and K3 have the
    same attach point without being neighbours in the sorted insert list.  The first GPU run caught this shape (two threads
    inserting at one attach word concurrently; sequential emulation could not see it): many such triples per block here."""
    rng = np.random.default_rng(31)
    state0 = {}
    stems = []
    for _ in range(64):                                   # 64 deep two-leaf subtries: root -> long edge -> N -> {a, b}
        stem = rng.integers(0, 256, 20, dtype=np.uint8).tobytes()
        stems.append(stem)
        for last in (0x10, 0xE0):
            state0[stem + bytes([last]) + rng.integers(0, 256, 11, dtype=np.uint8).tobytes()] = acct(1)
    h = Harness(eng, 0, seed=32)
    h.commit({k: (1, a) for k, a in state0.items()})
    for step in range(3):
        dirty = {}
        for stem in stems:
            cut = int(rng.integers(2 + step, 19))         # diverge inside the edge at byte `cut`, below and above
            lo, hi = bytearray(stem), bytearray(stem)
            if lo[cut] == 0 or hi[cut] == 255:
                continue
            lo[cut] -= 1
            hi[cut] += 1
            tail = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            dirty[bytes(lo[:cut + 1]) + tail(31 - cut)] = (1, acct(2))          # K1: below the edge
            dirty[stem + bytes([0x70 + step]) + tail(11)] = (1, acct(3))        # K2: through the edge, into N
            dirty[bytes(hi[:cut + 1]) + tail(31 - cut)] = (1, acct(4))          # K3: above the edge
        h.commit(dirty)
    h.trie.close()


def test_clustered_keys_long_extensions(eng):
    """Keys drawn from a few long shared prefixes: deep branches under long extension nodes, so inserts split extensions at
    every depth and deletes merge them back (the shapes uniform keccak keys almost never produce)."""
    rng = np.random.default_rng(21)
    prefixes = [rng.integers(0, 256, int(rng.integers(3, 31)), dtype=np.uint8).tobytes() for _ in range(6)]
    prefixes += [prefixes[0][:5] + bytes([prefixes[0][5] ^ 0x01]) + prefixes[0][6:], prefixes[1][:9]]

    def clustered():
        p = prefixes[int(rng.integers(0, len(prefixes)))]
        cut = int(rng.integers(1, len(p) + 1))
        return p[:cut] + rng.integers(0, 256, 32 - cut, dtype=np.uint8).tobytes()

    h = Harness(eng, 0, seed=30)
    h.commit({clustered(): (1, acct(1)) for _ in range(400)})
    for step in range(6):
        existing = sorted(h.state)
        dirty = {}
        for _ in range(120):
            r = rng.integers(0, 3)
            if r == 0:
                dirty[clustered()] = (1, acct(step + 2))
            elif r == 1:
                dirty[existing[int(rng.integers(0, len(existing)))]] = (0, acct(0))
            else:
                k = bytearray(existing[int(rng.integers(0, len(existing)))])
                k[int(rng.integers(0, 32))] ^= 1 << int(rng.integers(0, 8))     # one bit away: splits deep inside an edge
                dirty[bytes(k)] = (1, acct(7))
        h.commit(dirty)
    h.commit({k: (0, acct(0)) for k in sorted(h.state)[3:]})                    # collapse almost everything
    h.trie.close()
