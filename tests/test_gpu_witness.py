"""Execution witness of a block from the resident state (b200_dstate_witness; reth's TrieWitness::compute,
crates/trie/trie/src/witness.rs).  The device map is compared with a test-side model of the rule in include/b200trie.h
(a recursive trie built from the same flat state, "revealed" tracked as a set of node paths), with reth's own cases
(crates/trie/db/tests/witness.rs), and with a stateless client that rebuilds the post-block root from the witness alone."""
import numpy as np
import pytest

import oracle
from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, acct, clustered_slots, flatten, random_block, random_state, rkey

pytestmark = [pytest.mark.gpu]

EMPTY_ROOT = bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421")
KECCAK = oracle.keccak256


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


# ---- RLP and a recursive trie ------------------------------------------------------------------------------------------
def rlp_str(b):
    if len(b) == 1 and b[0] < 0x80:
        return b
    if len(b) < 56:
        return bytes([0x80 + len(b)]) + b
    ln = len(b).to_bytes((len(b).bit_length() + 7) // 8, "big")
    return bytes([0xb7 + len(ln)]) + ln + b


def rlp_list(items):
    p = b"".join(items)
    if len(p) < 56:
        return bytes([0xc0 + len(p)]) + p
    ln = len(p).to_bytes((len(p).bit_length() + 7) // 8, "big")
    return bytes([0xf7 + len(ln)]) + ln + p


def rlp_uint(v):
    return rlp_str(int(v).to_bytes((int(v).bit_length() + 7) // 8, "big"))


def hex_prefix(nibs, leaf):
    f = 2 if leaf else 0
    if len(nibs) % 2:
        out, rest = [(f + 1) << 4 | nibs[0]], nibs[1:]
    else:
        out, rest = [f << 4], nibs
    return bytes(out + [rest[i] << 4 | rest[i + 1] for i in range(0, len(rest), 2)])


def ref(rlp):
    return rlp if len(rlp) < 32 else rlp_str(KECCAK(rlp))


def nib(key):
    return tuple(x for b in key for x in (b >> 4, b & 15))


class Node:
    def __init__(self, kind, path, rlp, children=None, child=None):
        self.kind, self.path, self.rlp, self.children, self.child = kind, path, rlp, children, child


def build(items, depth=0):
    """items: sorted [(nibbles, value encoding)] -> the node at depth `depth` (None for an empty trie)"""
    if not items:
        return None
    if len(items) == 1:
        k, v = items[0]
        return Node("leaf", k[:depth], rlp_list([rlp_str(hex_prefix(k[depth:], True)), rlp_str(v)]))
    a, b = items[0][0], items[-1][0]
    cp = depth
    while a[cp] == b[cp]:
        cp += 1
    br = build_branch(items, cp)
    if cp == depth:
        return br
    return Node("ext", a[:depth], rlp_list([rlp_str(hex_prefix(a[depth:cp], False)), ref(br.rlp)]), child=br)


def build_branch(items, d):
    groups = {}
    for k, v in items:
        groups.setdefault(k[d], []).append((k, v))
    ch = {c: build(g, d + 1) for c, g in groups.items()}
    rlp = rlp_list([ref(ch[c].rlp) if c in ch else b"\x80" for c in range(16)] + [b"\x80"])
    return Node("branch", items[0][0][:d], rlp, children=ch)


def proof(node, key, min_len=0, root_only=False):
    """[(path, rlp)] of the witness walk of `key` (tk_proofs.cuh dt_proof_walk, witness form)"""
    if node is None:
        return [((), b"\x80")] if min_len == 0 else []
    out = []
    while True:
        keep = len(node.path) >= min_len
        if node.kind == "leaf":
            if keep:
                out.append((node.path, node.rlp))
            return out
        if node.kind == "ext":
            br = node.child
            if keep:
                out += [(node.path, node.rlp), (br.path, br.rlp)]
                if root_only:
                    return out
            if key[:len(br.path)] != br.path:
                return out
            node = br
        elif keep:
            out.append((node.path, node.rlp))
            if root_only:
                return out
        nxt = node.children.get(key[len(node.path)])
        if nxt is None:
            return out
        node = nxt


def branches(node):
    if node is None:
        return
    if node.kind == "ext":
        node = node.child
    if node.kind == "branch":
        yield node
        for c in node.children.values():
            yield from branches(c)


def storage_trie(slots):
    return build(sorted((nib(s), rlp_uint(v)) for s, v in slots.items()))


def trie_root(node):
    return EMPTY_ROOT if node is None else KECCAK(node.rlp)


def account_enc(a, sroot):
    return rlp_list([rlp_uint(int(a["nonce"])), rlp_uint(int.from_bytes(bytes(a["balance"]), "big")), rlp_str(sroot),
                     rlp_str(bytes(a["code_hash"]))])


def is_empty(a):
    return int(a["nonce"]) == 0 and not any(bytes(a["balance"])) and bytes(a["code_hash"]) == oracle.KECCAK_EMPTY


def model_witness(state, block, mode):
    """Steps 1-7 of the rule (include/b200trie.h) over the fully known pre-state.
    state: {addr: (account, {slot: int})}; block: {addr: (flags, account, {slot: int})}"""
    if not block:
        return {}
    canonical = mode == "canonical"
    w = {}

    def add(rlp):
        w[KECCAK(rlp)] = rlp

    def run(trie, targets, removed, survivors):
        """targets: keys whose proofs go in; removed: existing keys removed; survivors: keys alive after the removal phase"""
        revealed = set()
        for k in targets:
            for p, rlp in proof(trie, nib(k)):
                add(rlp)
                revealed.add(p)
        rem = [nib(k) for k in removed]
        surv = [nib(k) for k in survivors]
        for br in branches(trie):
            p = br.path
            if not any(r[:len(p)] == p for r in rem):
                continue
            alive = {s[len(p)] for s in surv if s[:len(p)] == p}
            if len(alive) != 1:
                continue
            c = next(iter(alive))
            child = br.children.get(c)
            if child is None or len(child.rlp) < 32 or child.path in revealed:
                continue
            for _, rlp in proof(trie, p + (c,) + (0,) * (63 - len(p)), min_len=len(p) + 1):
                add(rlp)

    tries = {k: storage_trie(s) for k, (_, s) in state.items()}
    removal = {}
    for k in sorted(block):
        fl, a, slots = block[k]
        pre = state[k][1] if k in state else {}
        wiped = not (fl & EXISTS) or bool(fl & WIPED)
        entries = dict(slots)
        if wiped:
            for s in pre:
                entries.setdefault(s, 0)
        if entries:
            removed = {s for s, v in entries.items() if v == 0 and s in pre}
            inserts = {s for s, v in entries.items() if v != 0 and s not in pre}
            survivors = (set(pre) - removed) | (inserts if canonical else set())
            run(tries.get(k), sorted(entries), removed, survivors)
            post = {} if wiped else dict(pre)
            for s, v in entries.items():
                if v:
                    post[s] = v
                else:
                    post.pop(s, None)
            post_empty = not post
        else:
            post_empty = not pre
            if not canonical:
                for _, rlp in proof(tries.get(k), (0,) * 64, root_only=True):
                    add(rlp)
        # as an apply: a destroyed account goes, an "unchanged" entry of an absent account is ignored
        if not (fl & EXISTS):
            removal[k] = True
        elif fl & UNCHANGED:
            removal[k] = False if k not in state else is_empty(state[k][0]) and post_empty
        else:
            removal[k] = is_empty(a) and post_empty
    acc_trie = build(sorted((nib(k), account_enc(a, trie_root(tries[k]))) for k, (a, _) in state.items()))
    removed = {k for k in block if removal[k] and k in state}
    inserts = {k for k in block if not removal[k] and k not in state and not (block[k][0] & UNCHANGED)}
    run(acc_trie, sorted(block), removed, (set(state) - removed) | (inserts if canonical else set()))
    if canonical:
        w = {h: r for h, r in w.items() if r != b"\x80"}
    return w


# ---- the device side -----------------------------------------------------------------------------------------------------
def block_arrays(block):
    ks = sorted(block)
    m = len(ks)
    keys = np.frombuffer(b"".join(ks), np.uint8).reshape(m, 32) if m else np.zeros((0, 32), np.uint8)
    accs = np.zeros(m, oracle.ACCOUNT_DTYPE)
    flags = np.zeros(m, np.uint8)
    sk, sv, offs = [], [], [0]
    for i, k in enumerate(ks):
        fl, a, slots = block[k]
        flags[i], accs[i] = fl, a
        for s in sorted(slots):
            sk.append(s)
            sv.append(int(slots[s]).to_bytes(32, "big"))
        offs.append(len(sk))
    skeys = np.frombuffer(b"".join(sk), np.uint8).reshape(-1, 32) if sk else np.zeros((0, 32), np.uint8)
    svals = np.frombuffer(b"".join(sv), np.uint8).reshape(-1, 32) if sv else np.zeros((0, 32), np.uint8)
    return keys, accs, flags, skeys, svals, np.array(offs, np.uint64)


def make_state(eng, state):
    from reth_b200 import DynamicState
    _, keys, accs, skeys, svals, offs = flatten(state)
    return DynamicState.create(eng, keys, accs, skeys, svals, offs)


def apply_to_model(state, block):
    """the post-block state (HashedPostState overlay rules, as tests/test_gpu_dstate.py's Harness)"""
    state = {k: (a.copy(), dict(s)) for k, (a, s) in state.items()}
    for k, (fl, a, slots) in block.items():
        if not (fl & EXISTS):
            state.pop(k, None)
            continue
        if fl & UNCHANGED:
            if k not in state:
                continue
            cur_a, cur_s = state[k]
        else:
            cur_a, cur_s = a.copy(), (state[k][1] if k in state else {})
        cur_s = {} if (fl & WIPED) else dict(cur_s)
        for s, v in slots.items():
            if v == 0:
                cur_s.pop(s, None)
            else:
                cur_s[s] = v
        state[k] = (cur_a, cur_s)
    return state


def check_block(eng, ds, state, block):
    arrays = block_arrays(block)
    for mode in ("legacy", "canonical"):
        got = ds.witness(*arrays, mode=mode)
        want = model_witness(state, block, mode)
        assert set(got) == set(want), (mode, len(set(got) - set(want)), len(set(want) - set(got)))
        assert got == want
        for h, rlp in got.items():
            assert KECCAK(rlp) == h
    return arrays


def blocks_of(rng, state, n_blocks, touch):
    for step in range(n_blocks):
        block = random_block(rng, state, touch, step + 1)
        yield block
        state = apply_to_model(state, block)


@pytest.mark.parametrize("n0,touch", [(3, 5), (300, 40), (3000, 250)])
def test_random_blocks_match_the_model(eng, n0, touch):
    rng = np.random.default_rng(900 + n0)
    state = random_state(rng, n0, with_storage=0.5, max_slots=40)
    ds = make_state(eng, state)
    for step in range(4):
        block = random_block(rng, state, touch, step + 1)
        arrays = check_block(eng, ds, state, block)
        ds.apply(*arrays)
        state = apply_to_model(state, block)
    ds.close()


def test_removals_collapse_onto_every_kind_of_sibling(eng):
    """Clustered slots with small values (inline leaves), removals that empty a branch, collapse it onto a hashed, an inline
    or a revealed sibling, and keys that diverge inside an extension."""
    rng = np.random.default_rng(31)
    state = random_state(rng, 400, with_storage=0.3, max_slots=20)
    owners = sorted(state)[:40]
    for k in owners:
        state[k] = (state[k][0], {s: int(rng.integers(1, 4)) for s in clustered_slots(rng, 6)})
    ds = make_state(eng, state)
    for step in range(4):
        block = {}
        for k in owners[step * 10:(step + 1) * 10]:
            slots = sorted(state[k][1])
            pick = rng.choice(len(slots), int(rng.integers(1, len(slots))), replace=False)
            ch = {slots[i]: 0 for i in pick}
            # a key that shares a long prefix with an existing slot: diverges inside its extension
            near = bytearray(slots[0])
            near[20] ^= 0x10
            ch[bytes(near)] = 0 if step % 2 else int(rng.integers(1, 3))
            block[k] = (EXISTS | UNCHANGED, acct(0), ch)
        live = sorted(set(state) - set(owners))
        for i in rng.choice(len(live), 20, replace=False):   # account removals: destroyed
            block[live[i]] = (0, acct(0), {})
        arrays = check_block(eng, ds, state, block)
        ds.apply(*arrays)
        state = apply_to_model(state, block)
    ds.close()


def test_wipe_of_a_large_storage_trie(eng):
    rng = np.random.default_rng(32)
    state = random_state(rng, 200, with_storage=0.2)
    big = sorted(state)[50]
    state[big] = (state[big][0], {rkey(rng): int(rng.integers(1, 2**40)) for _ in range(9000)})
    ds = make_state(eng, state)
    block = {big: (EXISTS | WIPED, state[big][0].copy(), {rkey(rng): 5})}
    check_block(eng, ds, state, block)
    check_block(eng, ds, state, {big: (0, acct(0), {})})
    ds.close()


# ---- sufficiency: a stateless client rebuilds the post-block root from the witness alone ----------------------------------
def decode(rlp):
    """RLP item -> bytes or list (recursively)"""
    def item(b, i):
        x = b[i]
        if x < 0x80:
            return b[i:i + 1], i + 1
        if x < 0xb8:
            return b[i + 1:i + 1 + x - 0x80], i + 1 + x - 0x80
        if x < 0xc0:
            ll = x - 0xb7
            n = int.from_bytes(b[i + 1:i + 1 + ll], "big")
            return b[i + 1 + ll:i + 1 + ll + n], i + 1 + ll + n
        if x < 0xf8:
            s, e = i + 1, i + 1 + x - 0xc0
        else:
            ll = x - 0xf7
            s = i + 1 + ll
            e = s + int.from_bytes(b[i + 1:i + 1 + ll], "big")
        out, j = [], s
        while j < e:
            v, j = item(b, j)
            out.append(v)
        return out, e
    return item(rlp, 0)[0]


class Stateless:
    """A stateless client: tries resolved lazily from the witness map (every hashed node fetched by its hash; a node it
    needs and cannot fetch fails the test), updated with MPT inserts and deletes (a branch left with one child merges
    with it, which needs that child's node)."""

    def __init__(self, w):
        self.w = w

    # nodes: None | ("hash", h) | ("leaf", path, value) | ("ext", path, child) | ("branch", [16 children])
    def node_of(self, item):
        if isinstance(item, bytes):
            if len(item) == 0:
                return None
            assert len(item) == 32
            return ("hash", item)
        if len(item) == 17:
            return ("branch", [self.node_of(c) for c in item[:16]])
        hp = item[0]
        f = hp[0] >> 4
        path = ((hp[0] & 15,) if f & 1 else ()) + tuple(x for b in hp[1:] for x in (b >> 4, b & 15))
        return ("leaf", path, item[1]) if f & 2 else ("ext", path, self.node_of(item[1]))

    def open(self, n):
        if n is not None and n[0] == "hash":
            assert n[1] in self.w, f"the witness lacks node {n[1].hex()}"
            return self.node_of(decode(self.w[n[1]]))
        return n

    def root_node(self, root):
        return None if root == EMPTY_ROOT else ("hash", root)

    def get(self, n, path):
        n = self.open(n)
        if n is None:
            return None
        if n[0] == "leaf":
            return n[2] if n[1] == path else None
        if n[0] == "ext":
            return self.get(n[2], path[len(n[1]):]) if path[:len(n[1])] == n[1] else None
        return self.get(n[1][path[0]], path[1:])

    def leaves(self, n, path=()):
        """every (path, value) below n, opening every node"""
        n = self.open(n)
        if n is None:
            return
        if n[0] == "leaf":
            yield path + n[1], n[2]
        elif n[0] == "ext":
            yield from self.leaves(n[2], path + n[1])
        else:
            for c in range(16):
                yield from self.leaves(n[1][c], path + (c,))

    def insert(self, n, path, value):
        n = self.open(n)
        if n is None:
            return ("leaf", path, value)
        if n[0] == "leaf":
            if n[1] == path:
                return ("leaf", path, value)
            return self.split(n, n[1], path, value)
        if n[0] == "ext":
            ep = n[1]
            if path[:len(ep)] == ep:
                return ("ext", ep, self.insert(n[2], path[len(ep):], value))
            return self.split(n, ep, path, value)
        ch = list(n[1])
        ch[path[0]] = self.insert(ch[path[0]], path[1:], value)
        return ("branch", ch)

    def split(self, n, npath, path, value):
        cp = 0
        while npath[cp] == path[cp]:
            cp += 1
        ch = [None] * 16
        if n[0] == "leaf":
            ch[npath[cp]] = ("leaf", npath[cp + 1:], n[2])
        else:
            rest = npath[cp + 1:]
            ch[npath[cp]] = ("ext", rest, n[2]) if rest else n[2]
        ch[path[cp]] = ("leaf", path[cp + 1:], value)
        br = ("branch", ch)
        return ("ext", path[:cp], br) if cp else br

    def delete(self, n, path):
        n = self.open(n)
        if n is None:
            return None
        if n[0] == "leaf":
            return None if n[1] == path else n
        if n[0] == "ext":
            ep = n[1]
            if path[:len(ep)] != ep:
                return n
            return self.prefix(ep, self.delete(n[2], path[len(ep):]))
        ch = list(n[1])
        ch[path[0]] = self.delete(ch[path[0]], path[1:])
        left = [c for c in range(16) if ch[c] is not None]
        if len(left) != 1:
            return ("branch", ch) if left else None
        return self.prefix((left[0],), ch[left[0]])

    def prefix(self, p, child):
        """the node that is `child` reached through the nibbles p (merging with a leaf or an extension: child opened)"""
        if child is None:
            return None
        if child[0] == "branch":
            return ("ext", p, child)
        child = self.open(child)
        if child[0] == "leaf":
            return ("leaf", p + child[1], child[2])
        if child[0] == "ext":
            return ("ext", p + child[1], child[2])
        return ("ext", p, child)

    def enc(self, n):
        if n[0] == "leaf":
            return rlp_list([rlp_str(hex_prefix(n[1], True)), rlp_str(n[2])])
        if n[0] == "ext":
            return rlp_list([rlp_str(hex_prefix(n[1], False)), self.ref(n[2])])
        return rlp_list([self.ref(c) if c is not None else b"\x80" for c in n[1]] + [b"\x80"])

    def ref(self, n):
        if n[0] == "hash":
            return rlp_str(n[1])
        e = self.enc(n)
        return e if len(e) < 32 else rlp_str(KECCAK(e))

    def root(self, n):
        if n is None:
            return EMPTY_ROOT
        return n[1] if n[0] == "hash" else KECCAK(self.enc(n))

    def apply(self, n, updates, canonical):
        """updates: {key: value bytes or None (removal)} in the phase order of the mode"""
        rem = [k for k, v in sorted(updates.items()) if v is None]
        ups = [(k, v) for k, v in sorted(updates.items()) if v is not None]
        phases = ("ups", "rem") if canonical else ("rem", "ups")
        for ph in phases:
            if ph == "rem":
                for k in rem:
                    n = self.delete(n, nib(k))
            else:
                for k, v in ups:
                    n = self.insert(n, nib(k), v)
        return n


def stateless_root(w, parent_root, block, canonical):
    """The post-block state root from the witness, the parent root and the block alone (block in the apply layout, with
    its rules: a destroyed account's storage is wiped, an "unchanged" entry of an absent account is ignored)."""
    sc = Stateless(w)
    acc = sc.root_node(parent_root)
    acc_updates = {}
    for k in sorted(block):
        fl, a, slots = block[k]
        leaf = sc.get(acc, nib(k))
        if (fl & EXISTS) and (fl & UNCHANGED) and leaf is None:
            continue
        if not (fl & EXISTS):
            acc_updates[k] = None
            continue
        fields = decode(leaf) if leaf is not None else None
        sroot = fields[2] if fields else EMPTY_ROOT
        st = sc.root_node(sroot)
        entries = {s: (rlp_uint(v) if v else None) for s, v in slots.items()}
        if fl & WIPED:   # the wiped storage's slots, read from the witness, become removals
            for path, _ in list(sc.leaves(st)):
                key = bytes(path[i] << 4 | path[i + 1] for i in range(0, 64, 2))
                entries.setdefault(key, None)
        if entries:
            sroot = sc.root(sc.apply(st, entries, canonical))
        if fl & UNCHANGED:
            nonce, bal, code = fields[0], fields[1], fields[3]
            empty = not nonce and not bal and code == oracle.KECCAK_EMPTY
            enc = rlp_list([rlp_str(nonce), rlp_str(bal), rlp_str(sroot), rlp_str(code)])
        else:
            empty = is_empty(a)
            enc = account_enc(a, sroot)
        acc_updates[k] = None if empty and sroot == EMPTY_ROOT else enc
    return sc.root(sc.apply(acc, acc_updates, canonical))


def check_stateless(eng, state, block):
    """witness in both modes -> the stateless root == the root an apply of the block gives on a twin state"""
    ds, twin = make_state(eng, state), make_state(eng, state)
    parent = ds.root()
    arrays = block_arrays(block)
    want = twin.apply(*arrays)
    for mode in ("legacy", "canonical"):
        w = ds.witness(*arrays, mode=mode)
        assert stateless_root(w, parent, block, mode == "canonical") == want, mode
    ds.close()
    twin.close()


@pytest.mark.parametrize("seed,n0,touch", [(41, 5, 6), (42, 300, 40), (43, 1500, 150)])
def test_stateless_rebuild_of_random_blocks(eng, seed, n0, touch):
    """Sufficiency, independent of the model: a stateless client rebuilds the post-block root from the witness, the parent
    root and the block alone, and gets the root the apply of the block gives."""
    rng = np.random.default_rng(seed)
    state = random_state(rng, n0, with_storage=0.6, max_slots=30)
    for step in range(3):
        block = random_block(rng, state, touch, step + 1)
        check_stateless(eng, state, block)
        state = apply_to_model(state, block)


def test_stateless_rebuild_of_collapses(eng):
    """The same on blocks that empty branches and collapse them onto hashed, inline and revealed siblings: clustered slots
    with small values, removals of most of a cluster, keys that diverge inside an extension, destroyed accounts."""
    rng = np.random.default_rng(44)
    state = random_state(rng, 300, with_storage=0.3, max_slots=20)
    owners = sorted(state)[:30]
    for k in owners:
        state[k] = (state[k][0], {s: int(rng.integers(1, 4)) if rng.random() < 0.5 else int.from_bytes(rng.bytes(31), "big") | 1
                                  for s in clustered_slots(rng, 5)})
    for step in range(3):
        block = {}
        for k in owners[step * 10:(step + 1) * 10]:
            slots = sorted(state[k][1])
            keep = int(rng.integers(0, 3))
            ch = {s: 0 for s in slots[keep:]} if step != 1 else {s: 0 for s in slots[:-1]}
            near = bytearray(slots[0])
            near[20] ^= 0x10
            ch[bytes(near)] = int(rng.integers(1, 3)) if step == 2 else 0
            block[k] = (EXISTS | UNCHANGED, acct(0), ch)
        live = sorted(set(state) - set(owners))
        for i in rng.choice(len(live), 25, replace=False):
            block[live[i]] = (0, acct(0), {})
        check_stateless(eng, state, block)
        state = apply_to_model(state, block)


# ---- reth's cases (crates/trie/db/tests/witness.rs) ------------------------------------------------------------------------
def test_includes_empty_node_preimage(eng):
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage
    a, slot = bytes(range(32)), bytes(range(1, 33))
    empty = DynamicStateRoot(eng, HashedPostState().into_sorted())
    post = HashedPostState({a: Account()}, {})
    assert empty.witness(post, "legacy") == {EMPTY_ROOT: b"\x80"}
    assert empty.witness(post, "canonical") == {}
    assert empty.witness(HashedPostState(), "legacy", always_include_root_node=True) == {EMPTY_ROOT: b"\x80"}
    assert empty.witness(HashedPostState(), "legacy") == {}
    empty.close()
    ds = DynamicStateRoot(eng, HashedPostState({a: Account()}, {}).into_sorted())
    root = ds.root()
    mp = ds.ds.multiproof({a: [slot]})
    post = HashedPostState({a: Account()}, {a: HashedStorage(False, {slot: 1})})
    legacy = ds.witness(post, "legacy")
    assert root in legacy
    for node in mp["account_subtree"].values():
        assert legacy[KECCAK(node)] == node
    assert legacy[EMPTY_ROOT] == b"\x80"
    canonical = ds.witness(post, "canonical")
    assert root in canonical and EMPTY_ROOT not in canonical
    for node in mp["account_subtree"].values():
        assert canonical[KECCAK(node)] == node
    assert ds.witness(HashedPostState(), "canonical", always_include_root_node=True) == {root: legacy[root]}
    ds.close()


def test_includes_nodes_for_destroyed_storage_nodes(eng):
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage
    a, slot = KECCAK(b"addr"), KECCAK(b"slot")
    ds = DynamicStateRoot(eng, HashedPostState({a: Account()}, {a: HashedStorage(False, {slot: 1})}).into_sorted())
    root = ds.root()
    mp = ds.ds.multiproof({a: [slot]})
    w = ds.witness(HashedPostState({a: None}, {a: HashedStorage(True, {})}))
    assert root in w
    for node in mp["account_subtree"].values():
        assert w[KECCAK(node)] == node
    for node in mp["storages"][a]["subtree"].values():
        assert w[KECCAK(node)] == node
    ds.close()


def test_correctly_decodes_branch_node_values(eng):
    """Two slots 0x0101… and 0x0202… under one account, both rewritten to 2: every node of the multiproof (account and
    storage) and the state root are in the witness."""
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage
    a = KECCAK(bytes(20))
    s1, s2 = bytes([1]) * 32, bytes([2]) * 32
    ds = DynamicStateRoot(eng, HashedPostState({a: Account()}, {a: HashedStorage(False, {s1: 1, s2: 1})}).into_sorted())
    root = ds.root()
    mp = ds.ds.multiproof({a: [s1, s2]})
    for mode in ("legacy", "canonical"):
        w = ds.witness(HashedPostState({a: Account()}, {a: HashedStorage(False, {s1: 2, s2: 2})}), mode)
        assert root in w
        for node in mp["account_subtree"].values():
            assert w[KECCAK(node)] == node
        for node in mp["storages"][a]["subtree"].values():
            assert w[KECCAK(node)] == node
    ds.close()


def test_root_node_of_a_state_whose_root_is_an_extension(eng):
    """always_include_root_node on an empty block returns the root node alone: here an extension whose nibbles are all
    zero (accounts 0x00… and 0x01…), the case in which the walk of key 0…0 also matches the branch below it."""
    from reth_b200 import Account, DynamicStateRoot, HashedPostState
    a0, a1 = bytes(32), bytes([0x01]) + bytes(31)
    ds = DynamicStateRoot(eng, HashedPostState({a0: Account(1, 1), a1: Account(2, 2)}).into_sorted())
    root = ds.root()
    for mode in ("legacy", "canonical"):
        w = ds.witness(HashedPostState(), mode, always_include_root_node=True)
        assert list(w) == [root]
        assert decode(w[root])[0] == bytes([0x10])   # an extension of the single nibble 0
    ds.close()


def test_storage_root_node_for_account_only_changes(eng):
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage
    a = KECCAK(b"acct")
    slots = {KECCAK(bytes([i])): i + 1 for i in range(4)}
    ds = DynamicStateRoot(eng, HashedPostState({a: Account(1, 1)}, {a: HashedStorage(False, slots)}).into_sorted())
    root = ds.root()
    sroot = ds.ds.multiproof({a: []})["storages"][a]["root"]
    post = HashedPostState({a: Account(2, 1)}, {})
    legacy = ds.witness(post, "legacy")
    assert root in legacy and sroot in legacy
    canonical = ds.witness(post, "canonical")
    assert root in canonical and sroot not in canonical
    ds.close()


def test_canonical_mode_handles_mixed_storage_inserts_and_removals(eng):
    """Two slots under one branch: the block removes one and inserts a new one next to them.  Legacy removes first, so the
    branch collapses onto the retained leaf, which has to be revealed; Canonical inserts first and never needs it."""
    from reth_b200 import Account, DynamicStateRoot, HashedPostState, HashedStorage
    a = KECCAK(b"mixed")
    s1, s2, s3 = (bytes([0x10]) + bytes(31)), (bytes([0x20]) + bytes(31)), (bytes([0x30]) + bytes(31))
    big = 2**250  # leaves of more than 32 bytes: hashed in their branch
    ds = DynamicStateRoot(eng, HashedPostState({a: Account(1)}, {a: HashedStorage(False, {s1: big, s2: big + 1})}).into_sorted())
    root = ds.root()
    retained = rlp_list([rlp_str(hex_prefix(nib(s2)[1:], True)), rlp_str(rlp_uint(big + 1))])
    assert len(retained) >= 32
    post = HashedPostState({a: Account(1)}, {a: HashedStorage(False, {s1: 0, s3: 1})})
    legacy = ds.witness(post, "legacy")
    assert root in legacy and legacy.get(KECCAK(retained)) == retained
    canonical = ds.witness(post, "canonical")
    assert root in canonical and KECCAK(retained) not in canonical
    assert all(v != b"\x80" for v in canonical.values())
    ds.close()


# ---- read-only, errors ---------------------------------------------------------------------------------------------------
def test_witness_leaves_the_state_unchanged(eng):
    rng = np.random.default_rng(34)
    state = random_state(rng, 300, with_storage=0.5)
    a, b = make_state(eng, state), make_state(eng, state)
    block = random_block(rng, state, 40, 1)
    arrays = block_arrays(block)
    targets = {k: list(state[k][1])[:3] if k in state else [] for k in sorted(block)}
    before = a.multiproof(targets)
    a.witness(*arrays, mode="legacy")
    a.witness(*arrays, mode="canonical")
    assert a.multiproof(targets) == before
    assert a.apply(*arrays, want_updates=True)[:5] == b.apply(*arrays, want_updates=True)[:5]
    a.close()
    b.close()


def test_errors(eng):
    from reth_b200 import B200Error, DynamicState, DynamicStateRoot, HashedPostState, HashedStorage, StateRootError
    rng = np.random.default_rng(35)
    state = random_state(rng, 50, with_storage=0.5)
    _, keys, accs, skeys, svals, offs = flatten(state)
    sharded = DynamicState.create(eng, keys, accs, skeys, svals, offs, sharded=True)
    block = block_arrays({sorted(state)[0]: (EXISTS, acct(1), {})})
    with pytest.raises(B200Error) as e:
        sharded.witness(*block)
    assert e.value.status == -3   # B200_ERR_INVALID_ARG
    sharded.close()
    ds = make_state(eng, state)
    k0, k1 = sorted(state)[:2]
    keys2 = np.stack([np.frombuffer(k1, np.uint8), np.frombuffer(k0, np.uint8)])
    with pytest.raises(B200Error) as e:
        ds.witness(keys2, np.stack([acct(1), acct(2)]), np.array([EXISTS, EXISTS], np.uint8), np.zeros((0, 32), np.uint8),
                   np.zeros((0, 32), np.uint8), np.zeros(3, np.uint64))
    assert e.value.status == -4   # B200_ERR_UNSORTED
    ds.close()
    from reth_b200 import Account
    dsr = DynamicStateRoot(eng, HashedPostState({k0: Account(1)}, {}).into_sorted())
    with pytest.raises(StateRootError):
        dsr.witness(HashedPostState({}, {k0: HashedStorage(False, {k1: 1})}))
    dsr.close()
