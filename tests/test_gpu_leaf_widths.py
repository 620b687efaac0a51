"""Leaf encoders at every field width.  Every root, proof and witness starts with a leaf RLP built on the device: storage
leaves (the register barrel shifter of `storage_leaf_words` for parent depths 0..26, the strip everywhere else) and account
leaves of 75..148 bytes (one or two Keccak rate blocks).  Here storage values of every width 1..32 hang at every parent
depth -1..62, and accounts carry nonces of 0..8 bytes and balances of 0..32 bytes at parent depths that produce every leaf
length; every build path, in-place path, proof, witness and the stateless decode are compared bit-exactly with the oracle
and with a plain RLP encoder written out below.  A census over that encoder asserts that each case reaches the widths,
depths, lengths and shifter cells it is meant to reach."""
import numpy as np
import pytest

import oracle

EMPTY = oracle.EMPTY_ROOT_HASH
KEMPTY = oracle.KECCAK_EMPTY
KECCAK = oracle.keccak256
EXISTS, UNCHANGED, WIPED = 1, 2, 4
OK, INVALID = 0, -3


# ---- a plain reference encoder -------------------------------------------------------------------------------------------
def be(v):
    return int(v).to_bytes((int(v).bit_length() + 7) // 8, "big")


def rlp_str(b):
    if len(b) == 1 and b[0] < 0x80:
        return bytes(b)
    if len(b) < 56:
        return bytes([0x80 + len(b)]) + bytes(b)
    return bytes([0xb7 + len(be(len(b)))]) + be(len(b)) + bytes(b)


def rlp_list(items):
    p = b"".join(items)
    if len(p) < 56:
        return bytes([0xc0 + len(p)]) + p
    return bytes([0xf7 + len(be(len(p)))]) + be(len(p)) + p


def rlp_uint(v):
    return rlp_str(be(v))


def nib(key):
    return tuple(x for b in key for x in (b >> 4, b & 15))


def hex_prefix(nibs, leaf):
    f = 2 if leaf else 0
    head, rest = ([(f + 1) << 4 | nibs[0]], nibs[1:]) if len(nibs) % 2 else ([f << 4], nibs)
    return bytes(head + [rest[i] << 4 | rest[i + 1] for i in range(0, len(rest), 2)])


def account_enc(nonce, balance, sroot=EMPTY, code=KEMPTY):
    return rlp_list([rlp_uint(nonce), rlp_uint(balance), rlp_str(sroot), rlp_str(code)])


def leaf_node(key, pd, value_enc):
    """The leaf of `key` hanging below a branch at depth pd (-1: the leaf is the whole trie)."""
    return rlp_list([rlp_str(hex_prefix(nib(key)[pd + 1:], True)), rlp_str(value_enc)])


def lcp(a, b):
    for i in range(32):
        if a[i] != b[i]:
            return 2 * i + (0 if (a[i] ^ b[i]) & 0xF0 else 1)
    return 64


def parent_depths(keys):
    """keys sorted: the depth of the branch every leaf hangs from (-1 for the only leaf of a trie)"""
    g = [lcp(keys[i], keys[i + 1]) for i in range(len(keys) - 1)]
    return [max(g[i - 1] if i else -1, g[i] if i < len(g) else -1) for i in range(len(keys))]


def payload_len(rlp):
    return len(rlp) - (1 if rlp[0] < 0xf8 else 1 + rlp[0] - 0xf7)


# ---- field values --------------------------------------------------------------------------------------------------------
NONCES = [0, 1, 0x7f, 0x80, 0xff, 0x100, 0xffff, 0x10000, 0xffffff, 2**24, 2**32 - 1, 2**32, 2**40 + 5, 2**48 + 7, 2**56 + 9,
          2**63, 2**64 - 1]


def wide(rng, w):
    """a value of exactly w bytes"""
    return int.from_bytes(bytes([int(rng.integers(1, 256))]) + rng.integers(0, 256, w - 1, dtype=np.uint8).tobytes(), "big")


def balances(rng):
    return [0, 1, 0x7f, 0x80, 0xff] + [wide(rng, w) for w in range(2, 33)] + [2**255, 2**256 - 1]


def slot_values(rng):
    """every width 1..32, and the single-byte edges"""
    return [0x01, 0x7f, 0x80] + [wide(rng, w) for w in range(1, 33)]


def rkey(rng):
    return rng.integers(0, 256, 32, dtype=np.uint8).tobytes()


def with_nibble(key, d, x):
    k = bytearray(key)
    k[d // 2] = (k[d // 2] & 0x0F) | (x << 4) if d % 2 == 0 else (k[d // 2] & 0xF0) | x
    return bytes(k)


def rows(ks):
    return np.frombuffer(b"".join(ks), np.uint8).reshape(-1, 32).copy() if ks else np.zeros((0, 32), np.uint8)


def u256_rows(vs):
    return rows([int(v).to_bytes(32, "big") for v in vs])


def acc(nonce, balance, code=None):
    a = np.zeros((), oracle.ACCOUNT_DTYPE)
    a[()] = oracle.make_accounts([(nonce, balance, code)])[0]
    return a


def fields(a):
    return int(a["nonce"]), int.from_bytes(bytes(a["balance"]), "big"), bytes(a["code_hash"])


def width(v):
    return len(be(v))


# ---- the storage grid ----------------------------------------------------------------------------------------------------
def storage_grid(seed=1):
    """A forest of two-leaf tries (key B = key A with nibble d changed: both leaves at parent depth d, d = 0..62) for every
    value, single-slot tries for every value, and one dense trie of all widths (stored branch nodes).
    -> (tries [[(key, value)]], keys, values, seg_offsets)"""
    rng = np.random.default_rng(seed)
    vals = slot_values(rng)
    tries = []
    for d in range(63):
        for i, v in enumerate(vals):
            a = rkey(rng)
            x = nib(a)[d]
            b = with_nibble(a, d, x ^ (1 + i % 15))
            tries.append(sorted([(a, v), (b, vals[(i + 11) % len(vals)])]))
    tries += [[(rkey(rng), v)] for v in vals]
    tries.append(sorted((rkey(rng), vals[j % len(vals)]) for j in range(600)))
    offs = np.cumsum([0] + [len(t) for t in tries]).astype(np.uint64)
    keys = rows([k for t in tries for k, _ in t])
    values = u256_rows([v for t in tries for _, v in t])
    return tries, keys, values, offs


def storage_census(tries):
    """[(parent depth, value width, leaf RLP length, list payload length)] of every leaf"""
    out = []
    for t in tries:
        for (k, v), pd in zip(t, parent_depths([k for k, _ in t])):
            leaf = leaf_node(k, pd, rlp_uint(v))
            out.append((pd, width(v), len(leaf), payload_len(leaf)))
    return out


def check_storage_census(cells):
    reg = [c for c in cells if 0 <= c[0] <= 26]                                  # the register path of the leaf kernel
    assert {(pd + 1, 32 - w) for pd, w, _, _ in reg} == {(p, z) for p in range(1, 28) for z in range(32)}
    assert {ln for _, _, ln, _ in reg if ln < 32} == set(range(22, 32))          # inline register-path leaves
    assert {55, 56} <= {pl for _, _, _, pl in reg}                              # one- / two-byte list header
    assert {pd for pd, _, _, _ in cells} >= set(range(-1, 63))
    assert {w for _, w, _, _ in cells} == set(range(1, 33))
    assert {(pd, w) for pd, w, _, _ in cells if pd > 26} >= {(pd, w) for pd in range(27, 63) for w in range(1, 33)}


# ---- the account grid ----------------------------------------------------------------------------------------------------
def account_len(pd, nonce, balance):
    return len(leaf_node(bytes(32), pd, account_enc(nonce, balance)))


def fields_of_length(rest):
    """(hex-prefix string length, nonce, balance) with 72 + their encoded lengths == 72 + rest, parent depth >= 3"""
    if rest <= 43:
        hp = 1
        br = min(33, rest - 2)
        nr = rest - 1 - br
    elif rest - 42 == 2:
        hp, nr, br = 3, 8, 33
    else:
        hp, nr, br = rest - 42, 9, 33
    num = lambda r: 0 if r == 1 else 1 << (8 * (r - 1) - 1)     # r-byte encoding: 0, or an (r-1)-byte value with the top bit
    pd = 62 if hp == 1 else 63 - 2 * (hp - 2)
    return pd, num(nr), num(br)


def account_states(seed=2):
    """-> {name: (sorted keys, [(nonce, balance, code_hash)])}:
    "grid": two-account groups under distinct 3-nibble prefixes, both at parent depth 3..62, every (nonce, balance) pair of
    the value lists and every leaf length 75..146;  "top": 8 top-nibble buckets with one account (parent depth 0) and 8
    with two accounts that part at nibble 1;  "single-*": one account, the leaf is the root (up to 148 bytes)."""
    rng = np.random.default_rng(seed)
    bals = balances(rng)
    code = lambda i: KEMPTY if i % 3 else rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    want = [(3 + i % 60, n, b) for i, (n, b) in enumerate((n, b) for n in NONCES for b in bals)]
    want += [fields_of_length(L - 72) for L in range(75, 147)]
    by_pd = {}
    for pd, n, b in want:
        by_pd.setdefault(pd, []).append((n, b))
    groups = iter(rng.permutation(4096))
    keys, accs = [], []
    for pd, fl in sorted(by_pd.items()):
        if len(fl) % 2:
            fl.append((1, 1))
        for j in range(0, len(fl), 2):
            g = int(next(groups))
            a = bytes([g >> 4, ((g & 15) << 4) | int(rng.integers(0, 16))]) + rng.integers(0, 256, 30, dtype=np.uint8).tobytes()
            b = with_nibble(a, pd, nib(a)[pd] ^ int(rng.integers(1, 16)))
            for k, (n, bal) in zip((a, b), fl[j:j + 2]):
                keys.append(k)
                accs.append((n, bal, code(len(keys))))
    states = {"grid": (keys, accs)}
    top, tacc = [], []
    wide_fields = [(2**64 - 1, 2**256 - 1), (2**64 - 1, 2**255), (2**56 + 9, 2**256 - 1), (0, 0), (0x80, 0x80), (0x7f, 0x7f)]
    for bucket in range(16):
        k = bytes([bucket << 4 | int(rng.integers(0, 16))]) + rng.integers(0, 256, 31, dtype=np.uint8).tobytes()
        ks = [k] if bucket < 8 else [k, with_nibble(k, 1, nib(k)[1] ^ 5)]
        for k2 in ks:
            top.append(k2)
            tacc.append(wide_fields[len(top) % len(wide_fields)] + (code(len(top)),))
    states["top"] = (top, tacc)
    for i, (n, b) in enumerate([(2**64 - 1, 2**256 - 1), (0, 0), (0x80, 2**248), (2**63, 0x7f)]):
        states[f"single-{i}"] = ([rkey(rng)], [(n, b, code(i + 1))])
    for name, (ks, ac) in states.items():
        order = sorted(range(len(ks)), key=lambda i: ks[i])
        states[name] = ([ks[i] for i in order], [ac[i] for i in order])
    return states


def account_census(states):
    """{(parent depth, nonce width, balance width, leaf length)} over all states"""
    out = set()
    for ks, ac in states.values():
        for k, (n, b, c), pd in zip(ks, ac, parent_depths(ks)):
            out.add((pd, width(n), width(b), len(leaf_node(k, pd, account_enc(n, b, EMPTY, c)))))
    return out


def check_account_census(cells):
    assert {c[3] for c in cells} == set(range(75, 149))
    assert {c[1] for c in cells} == set(range(9)) and {c[2] for c in cells} == set(range(33))
    assert {-1, 0, 1} | set(range(3, 63)) <= {c[0] for c in cells}


def arrays(state):
    ks, ac = state
    return rows(ks), oracle.make_accounts(ac)


def mixed_sroots(rng, n):
    sr = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    sr[::3] = np.frombuffer(EMPTY, np.uint8)
    return sr


# ---- 1. the reference encoder against the oracle (no GPU) ---------------------------------------------------------------
def test_reference_encoder_matches_oracle():
    rng = np.random.default_rng(0)
    vals = [0] + slot_values(rng) + [2**(8 * w) - 1 for w in range(1, 33)] + [2**(8 * w - 8) for w in range(1, 33)]
    for v in vals:
        assert rlp_uint(v) == oracle.encode_u256(v), v
    sr = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    code = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    bals = balances(rng)
    for n in NONCES:
        for b in bals:
            assert account_enc(n, b, sr, code) == oracle.encode_trie_account(n, b, sr, code), (n, b)
            assert account_enc(n, b) == oracle.encode_trie_account(n, b)
    assert len(account_enc(2**64 - 1, 2**256 - 1)) == 110
    # leaf nodes: the HashBuilder's own leaf RLPs of two-leaf tries at every parent depth and of single-leaf tries
    for d in range(-1, 64):
        a = rkey(rng)
        ks = [a] if d < 0 else sorted([a, with_nibble(a, d, nib(a)[d] ^ 9)])
        for enc in ([rlp_uint(v) for v in slot_values(rng)] + [account_enc(n, b) for n, b in
                                                              ((0, 0), (2**64 - 1, 2**256 - 1), (0x80, 0x7f))]):
            hb = oracle.HashBuilder(retain_nodes=True)
            for k in ks:
                hb.add_leaf(bytes(nib(k)), enc)
            root = hb.root()
            nodes = hb.nodes()
            for k, pd in zip(ks, parent_depths(ks)):
                assert pd == d
                assert leaf_node(k, pd, enc) in nodes, (d, enc.hex())
            if d < 0:
                assert root == KECCAK(leaf_node(ks[0], -1, enc))
    # the cases below reach what they claim
    check_storage_census(storage_census(storage_grid()[0]))
    check_account_census(account_census(account_states()))
    assert account_len(-1, 2**64 - 1, 2**256 - 1) == 148


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


def oracle_hashed_nodes(fn, *args):
    oracle.stats_reset()
    fn(*args)
    return oracle.stats()["hashed_nodes"]


# ---- 2. the storage grid (from-scratch forest) ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_storage_grid_every_width_at_every_parent_depth(eng):
    tries, keys, values, offs = storage_grid()
    check_storage_census(storage_census(tries))
    roots, upd, stats = eng.storage_roots(keys, values, offs, want_updates=True, want_stats=True)
    o_roots, o_upd = oracle.storage_roots(keys, values, offs, want_updates=True, threads=4)
    for i, t in enumerate(tries[:-1]):                         # the reference encoder agrees on every small trie
        if len(t) == 1:
            assert o_roots[i].tobytes() == KECCAK(leaf_node(t[0][0], -1, rlp_uint(t[0][1])))
    assert (roots == o_roots).all(), np.nonzero((roots != o_roots).any(1))[0][:20]
    assert upd == o_upd and upd
    assert stats["hashed_nodes"] == oracle_hashed_nodes(oracle.storage_roots, keys, values, offs)
    assert stats["leaves_added"] == len(keys)


@pytest.mark.gpu
def test_storage_grid_device_buffers(eng):
    import torch
    _, keys, values, offs = storage_grid()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
    m = len(offs) - 1
    d_roots = torch.zeros(m * 32, dtype=torch.uint8, device="cuda")
    eng.use_torch_stream()
    try:
        eng.storage_roots_dev(t(keys), t(values), t(offs), m, len(keys), d_roots)
        eng.dev_status()
    finally:
        eng.set_stream(None)
    assert (d_roots.cpu().numpy().reshape(m, 32) == oracle.storage_roots(keys, values, offs, threads=4)).all()


# ---- 3. the account grid -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["grid", "top", "single-0", "single-1", "single-2", "single-3"])
def test_account_grid_state_root_and_items(eng, name):
    state = account_states()[name]
    keys, accs = arrays(state)
    rng = np.random.default_rng(3)
    sroots = mixed_sroots(rng, len(keys))
    for sr in (None, sroots):
        want = oracle.state_root(keys, accs, sr, want_updates=True)
        assert eng.state_root(keys, accs, sr, want_updates=True) == want
        if len(keys) == 1:
            n, b, c = fields(accs[0])
            assert want[0] == KECCAK(leaf_node(state[0][0], -1, account_enc(n, b, EMPTY if sr is None else sr[0].tobytes(), c)))
        n = len(keys)
        roots, recs = eng.root_from_items(keys, np.full(n, 64, np.uint8), np.zeros(n, np.uint8),
                                          accs.view(np.uint8).reshape(n, 72), sr, None, account=True, want_updates=True)
        assert roots[0].tobytes() == want[0]
        assert {r[1]: r[2:] for r in recs} == {r[1]: r[2:] for r in want[1]}


def account_slots(keys, rng, every=4):
    """one or two slots of wide values on every `every`-th account (arbitrary storage roots in the full-state paths)"""
    n = len(keys)
    counts = np.where(np.arange(n) % every == 1, 1 + np.arange(n) % 2, 0)
    vals = slot_values(rng)
    sk = rows(sorted(rkey(rng) for _ in range(int(counts.sum()))))      # ascending, so inside every account's run too
    offs = np.cumsum([0] + list(counts)).astype(np.uint64)
    sv = u256_rows([vals[(3 * i + 5) % len(vals)] for i in range(len(sk))])
    return sk, sv, offs


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["grid", "top"])
def test_account_grid_frontier(eng, name):
    keys, accs = arrays(account_states()[name])
    if name == "top":                                            # buckets 0..7 hold one account each
        assert [int((keys[:, 0] >> 4 == b).sum()) for b in range(16)] == [1] * 8 + [2] * 8
    for sk, sv, offs in ((np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8), np.zeros(len(keys) + 1, np.uint64)),
                         account_slots(keys, np.random.default_rng(4))):
        fr = eng.subtrie_frontier(keys, accs, sk, sv, offs)
        assert eng.root_from_frontier(fr) == oracle.state_root_full(keys, accs, sk, sv, offs)


@pytest.mark.gpu
def test_account_grid_root_stream_cut_inside(eng):
    from reth_b200 import RootStream
    keys, accs = arrays(account_states()["grid"])
    sk, sv, offs = account_slots(keys, np.random.default_rng(5))
    o_root, o_au, _ = oracle.state_root_full(keys, accs, sk, sv, offs, want_updates=True)
    n = len(keys)
    bounds = [0, 1, n // 3, n // 3 + 1, 2 * n // 3, n]
    s = RootStream(eng, retain_updates=True)
    au = {}
    for a0, a1 in zip(bounds, bounds[1:]):
        s0, s1 = int(offs[a0]), int(offs[a1])
        prog, ua, _ = s.push(keys[a0:a1], accs[a0:a1], sk[s0:s1], sv[s0:s1], (offs[a0:a1 + 1] - offs[a0]).astype(np.uint64))
        assert prog["accounts"] == a1
        au.update({r[1]: r[2:] for r in ua})
    root, ua = s.finish()
    au.update({r[1]: r[2:] for r in ua})
    s.close()
    assert root == o_root
    assert au == {r[1]: r[2:] for r in o_au}


# ---- 4. in-place paths ---------------------------------------------------------------------------------------------------
def narrow_wide_blocks(accs, rng):
    """three blocks of new account fields: every account wide, then every account narrow, then wide on every other one"""
    n = len(accs)
    bals = balances(rng)
    wide_ = [(NONCES[(i * 5) % len(NONCES)], bals[(i * 7) % len(bals)]) for i in range(n)]
    narrow = [(i % 3, (i % 2) * 0x7f) for i in range(n)]
    mk = lambda fl, idx: (idx, oracle.make_accounts([(fl[i][0], fl[i][1], bytes(accs[i]["code_hash"])) for i in idx]))
    every = np.arange(n)
    return [mk(wide_, every), mk(narrow, every), mk(wide_[::-1], every[::2])]


@pytest.mark.gpu
def test_resident_trie_narrow_wide_narrow(eng):
    from reth_b200 import ResidentTrie
    keys, accs = arrays(account_states()["grid"])
    rng = np.random.default_rng(6)
    sroots = mixed_sroots(rng, len(keys))
    t = ResidentTrie.create(eng, keys, accs, sroots)
    assert t.root() == oracle.state_root(keys, accs, sroots)
    for idx, new in narrow_wide_blocks(accs, rng):
        new_sr = mixed_sroots(rng, len(idx))
        root, upd = t.update(keys[idx], new, new_sr, want_updates=True)
        accs[idx], sroots[idx] = new, new_sr
        o_root, o_upd = oracle.state_root(keys, accs, sroots, want_updates=True)
        assert root == o_root
        full = {r[1]: r for r in o_upd}
        assert upd and all(full[r[1]] == r for r in upd)
    t.close()


@pytest.mark.gpu
def test_resident_trie_update_dev_narrow_wide_narrow(eng):
    import torch
    from reth_b200 import ResidentTrie
    keys, accs = arrays(account_states()["grid"])
    rng = np.random.default_rng(7)
    t = ResidentTrie.create(eng, keys, accs)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
    d_root = torch.zeros(32, dtype=torch.uint8, device="cuda")
    eng.use_torch_stream()
    try:
        for idx, new in narrow_wide_blocks(accs, rng):
            t.update_dev(dev(keys[idx]), dev(new), None, len(idx), d_root)
            eng.dev_status()
            accs[idx] = new
            assert d_root.cpu().numpy().tobytes() == oracle.state_root(keys, accs)
    finally:
        eng.set_stream(None)
    t.close()


@pytest.mark.gpu
def test_resident_trie_large_block_above_the_warp_split(eng):
    """more than 4096 dirty leaves and a level with more than 4096 branch nodes: the thread-per-leaf stage of the wavefront"""
    from reth_b200 import ResidentTrie
    from tests.util import synth_accounts
    keys, accs = synth_accounts(81, 40_000)
    t = ResidentTrie.create(eng, keys, accs)
    rng = np.random.default_rng(8)
    bals = balances(rng)
    for step in range(2):
        idx = np.sort(rng.choice(len(keys), 6000, replace=False))
        new = oracle.make_accounts([(NONCES[(i + step) % len(NONCES)], bals[(i * 3 + step) % len(bals)] if step == 0 else i % 200,
                                     bytes(accs[i]["code_hash"])) for i in idx])
        accs[idx] = new
        assert t.update(keys[idx], new) == oracle.state_root(keys, accs)
    t.close()


@pytest.mark.gpu
def test_dynamic_trie_widths_inserts_deletes(eng):
    from tests.test_gpu_dtrie import Harness
    h = Harness(eng, 300, seed=90)
    rng = np.random.default_rng(9)
    bals = balances(rng)
    wide_acc = lambda i: acc(NONCES[i % len(NONCES)], bals[(i * 7) % len(bals)], rkey(rng) if i % 2 else None)
    for step in range(4):
        live = sorted(h.state)
        dirty = {}
        for j, i in enumerate(rng.choice(len(live), 80, replace=False)):
            dirty[live[i]] = (1, wide_acc(j + step) if step % 2 == 0 else acc(j % 2, 0x80 * (j % 2)))
        for i in rng.choice(len(live), 20, replace=False):
            dirty[live[i]] = (0, acc(0, 0))
        for j in range(30):
            dirty[rkey(rng)] = (1, wide_acc(j * 3 + step))
        for i in rng.choice(len(live), 10, replace=False):               # deep siblings of wide leaves
            b = bytearray(live[i])
            b[31 - step] ^= 0x01
            dirty[bytes(b)] = (1, wide_acc(int(i) + step))
        h.commit(dirty)
    h.trie.close()


def dstate_leaves(state):
    """{("a", key) | ("s", key, slot): leaf RLP} of a {key: (account, {slot: value})} state, by the reference encoder"""
    from tests.test_gpu_dstate import flatten
    ks, keys, accs, skeys, svals, offs = flatten(state)
    sroots = oracle.storage_roots(skeys, svals, offs) if len(ks) else []
    out = {}
    for i, (k, pd) in enumerate(zip(ks, parent_depths(ks))):
        n, b, c = fields(state[k][0])
        out[("a", k)] = leaf_node(k, pd, account_enc(n, b, sroots[i].tobytes(), c))
        sl = sorted(state[k][1])
        for s, spd in zip(sl, parent_depths(sl)):
            out[("s", k, s)] = leaf_node(s, spd, rlp_uint(state[k][1][s]))
    return out


def deep_pairs(rng, depths):
    out = []
    for d in depths:
        a = rkey(rng)
        out += [a, with_nibble(a, d, nib(a)[d] ^ 3)]
    return out


def slot_widths_state(rng, deep=True):
    """accounts with wide and narrow fields; their storage: a shallow trie of 200 slots, pairs at parent depths 20..62 and
    (deep=True) clusters of slots that share 63 nibbles"""
    from tests.test_gpu_dstate import clustered_slots
    bals = balances(rng)
    st = {}
    for i in range(60):
        st[rkey(rng)] = (acc(NONCES[i % len(NONCES)], bals[(i * 11) % len(bals)], rkey(rng) if i % 4 == 0 else None), {})
    owners = sorted(st)[:3]
    st[owners[0]] = (st[owners[0]][0], {rkey(rng): 1 + i % 100 for i in range(200)})
    st[owners[1]] = (st[owners[1]][0], {s: 1 + i % 100 for i, s in enumerate(deep_pairs(rng, range(20, 63)))})
    if deep:
        st[owners[2]] = (st[owners[2]][0], {s: 1 + i % 100 for i, s in enumerate(clustered_slots(rng, 8))})
    return st, owners


@pytest.mark.gpu
def test_dynamic_state_slot_widths_and_inline_flips(eng):
    """every slot width at shallow and deep parent depths, narrow -> wide -> narrow; deep clustered slots widening from 1 byte
    to 32 and back flip their branch's child references between inline and hashed; accounts wide and narrow; then proofs"""
    from tests.test_gpu_dstate import Harness
    from tests.test_gpu_proofs import verify
    rng = np.random.default_rng(10)
    st, owners = slot_widths_state(rng)
    vals = slot_values(rng)
    h = Harness(eng, st)
    inline_seen = []
    for step, widen in enumerate((True, False, True, False)):
        block = {}
        for o in owners:
            sl = sorted(h.state[o][1])
            wide_v = (lambda i: vals[-1 - i % 3]) if o == owners[2] else (lambda i: vals[(i + step) % len(vals)])
            ch = {s: (wide_v(i) if widen else 1 + i % 0x7f) for i, s in enumerate(sl)}
            for s in sl[:3]:
                ch[s] = 0
            ch[rkey(rng)] = vals[step * 5 % len(vals)]
            block[o] = (EXISTS | UNCHANGED, acc(0, 0), ch)
        bals = balances(rng)
        for i, k in enumerate(sorted(set(h.state) - set(owners))[step::3]):
            a = acc(NONCES[(i + step) % len(NONCES)], bals[(i * 5 + step) % len(bals)]) if widen else acc(i % 2, i % 3)
            block[k] = (EXISTS | UNCHANGED if i % 5 == 0 else EXISTS, a, {rkey(rng): vals[i % len(vals)]} if i % 4 == 0 else {})
        root = h.commit(block)
        leaves = dstate_leaves(h.state)
        sl = sorted(h.state[owners[2]][1])
        clus = [leaves[("s", owners[2], s)] for s, pd in zip(sl, parent_depths(sl)) if pd == 63]
        assert len(clus) >= 8
        inline_seen.append({len(x) < 32 for x in clus})
        # proofs of every account and of every slot of the owners: leaves == the reference encoder's, chains to the root
        ks = sorted(h.state)
        proofs = h.ds.account_proofs(rows(ks))
        for k, p in zip(ks, proofs):
            assert p[-1] == leaves[("a", k)]
            verify(root, k, p, rlp_items_value(p[-1]))
        mp = h.ds.multiproof({o: sorted(h.state[o][1])[:40] for o in owners})
        pds = dict(zip(ks, parent_depths(ks)))
        for o in owners:
            assert mp["account_subtree"][bytes(nib(o)[:pds[o] + 1])] == leaves[("a", o)]
            sl = sorted(h.state[o][1])
            sroot, sp = h.ds.storage_proofs(o, rows(sl))
            spds = dict(zip(sl, parent_depths(sl)))
            for s, p in zip(sl, sp):
                assert p[-1] == leaves[("s", o, s)]
                verify(sroot, s, p, rlp_uint(h.state[o][1][s]))
            for s in sl[:40]:
                assert mp["storages"][o]["subtree"][bytes(nib(s)[:spds[s] + 1])] == leaves[("s", o, s)]
    assert inline_seen == [{False}, {True}, {False}, {True}]
    h.ds.close()


def rlp_items_value(leaf):
    from tests.test_gpu_proofs import rlp_items
    return rlp_items(leaf)[1]


@pytest.mark.gpu
@pytest.mark.parametrize("n_block", [300, 9000], ids=["small_block", "large_block"])
def test_dynamic_state_wide_accounts(eng, n_block):
    """wide accounts through the dynamic state at the default thresholds, in a small block and in a block of more than 8192
    entries (the multi-launch restructure and the two-stage re-hash)"""
    from tests.test_gpu_dstate import Harness
    rng = np.random.default_rng(11 + n_block)
    bals = balances(rng)
    st = {rkey(rng): (acc(i % 3, i % 200), {}) for i in range(2000)}
    h = Harness(eng, st)
    for step in range(3):
        live = sorted(h.state)
        block = {}
        for j, i in enumerate(rng.choice(len(live), min(n_block // 2, len(live)), replace=False)):
            a = acc(NONCES[(j + step) % len(NONCES)], bals[(j * 3 + step) % len(bals)]) if step != 1 else acc(j % 2, j % 0x81)
            block[live[i]] = (EXISTS, a, {})
        while len(block) < n_block:
            block[rkey(rng)] = (EXISTS, acc(NONCES[len(block) % len(NONCES)], bals[len(block) % len(bals)]), {})
        h.commit(block)
    h.ds.close()


# ---- 5. witnesses, the stateless decode, malformed widths ----------------------------------------------------------------
def is_leaf(node):
    from tests.test_gpu_proofs import rlp_items
    if node == b"\x80":
        return False
    items = rlp_items(node)
    return len(items) == 2 and items[0][0] >> 4 in (2, 3)


@pytest.mark.gpu
def test_witness_leaves_and_stateless_roots(eng):
    from tests.test_gpu_witness import apply_to_model, block_arrays, make_state
    rng = np.random.default_rng(12)
    state, owners = slot_widths_state(rng, deep=False)
    vals = slot_values(rng)
    bals = balances(rng)
    for step in range(3):
        block = {}
        for j, o in enumerate(owners[:2]):
            sl = sorted(state[o][1])
            ch = {s: vals[(i * 7 + step + j) % len(vals)] if (i + step) % 2 else 1 + i % 0x7f for i, s in enumerate(sl[::3])}
            ch[sl[1]] = 0
            ch[rkey(rng)] = vals[-1 - step]
            block[o] = (EXISTS | UNCHANGED, acc(0, 0), ch)
        rest = sorted(set(state) - set(owners))
        for i, k in enumerate(rest[step::4]):
            block[k] = (EXISTS, acc(NONCES[-1 - (i + step) % len(NONCES)], bals[-1 - (i * 3) % len(bals)]) if i % 2 else acc(i, 1), {})
        for i, k in enumerate(rest[step + 1::9]):                         # storage-only change of a wide account
            block[k] = (EXISTS | UNCHANGED, acc(0, 0), {rkey(rng): vals[i % len(vals)]})
        for i in range(4):
            block[rkey(rng)] = (EXISTS, acc(2**64 - 1, 2**256 - 1 - i), {rkey(rng): vals[-1]})
        arrs = block_arrays(block)
        ds, twin = make_state(eng, state), make_state(eng, state)
        parent = ds.root()
        want = twin.apply(*arrs)
        leaves = dstate_leaves(state)
        ref = set(leaves.values())
        for mode in ("legacy", "canonical"):
            w = ds.witness(*arrs, mode=mode)
            got = [r for r in w.values() if is_leaf(r)]
            assert got and set(got) <= ref
            for k, (fl, _, slots) in block.items():                   # the leaves on the paths of the block's keys
                if k in state:
                    assert leaves[("a", k)] in w.values()
                    if fl & EXISTS and not fl & WIPED and len(state[k][1]) > 1:
                        for s in slots:
                            x = leaves.get(("s", k, s))
                            assert x is None or len(x) < 32 or x in w.values()
            roots, status = eng.witness_roots([parent], [w], [arrs])
            assert (roots[0].tobytes(), int(status[0])) == (want, OK), mode
        ds.close()
        twin.close()
        state = apply_to_model(state, block)


@pytest.mark.gpu
def test_stateless_field_widths_out_of_range(eng):
    """single-leaf tries written by the reference encoder with fields the decoder must refuse (9-byte nonce, 33-byte balance,
    33-byte or zero storage value) or accept (the widest legal fields; a nonce with a leading zero byte, which the header
    accepts as non-minimal RLP), all in one call: a refused block does not disturb the others"""
    from tests.test_gpu_dstate import flatten
    from tests.test_gpu_witness import block_arrays
    a, slot = KECCAK(b"widths"), KECCAK(b"slot")
    raw_acct = lambda nonce_b, bal_b, sroot: rlp_list([rlp_str(nonce_b), rlp_str(bal_b), rlp_str(sroot), rlp_str(KEMPTY)])
    acct_leaf = lambda enc: leaf_node(a, -1, enc)
    slot_leaf = lambda enc: leaf_node(slot, -1, enc)

    def with_slot(nonce_b, bal_b, slot_enc):
        s = slot_leaf(slot_enc)
        return [acct_leaf(raw_acct(nonce_b, bal_b, KECCAK(s))), s]
    block = {a: (EXISTS | UNCHANGED, acc(0, 0), {KECCAK(b"new"): 2**256 - 1})}
    cases = [
        ("widest", with_slot(be(2**64 - 1), be(2**256 - 1), rlp_uint(2**256 - 1)), OK, (2**64 - 1, 2**256 - 1, 2**256 - 1)),
        ("9-byte nonce", [acct_leaf(raw_acct(b"\x01" + bytes(8), be(5), EMPTY))], INVALID, None),
        ("33-byte balance", [acct_leaf(raw_acct(be(5), b"\x01" + bytes(32), EMPTY))], INVALID, None),
        ("33-byte slot value", with_slot(be(5), be(5), rlp_str(b"\x01" * 33)), INVALID, None),
        ("zero slot value", with_slot(be(5), be(5), b"\x80"), INVALID, None),
        ("nonce with a leading zero", with_slot(b"\x00\x05", be(7), rlp_uint(0x80)), OK, (5, 7, 0x80)),
        ("32-byte balance", with_slot(be(0x80), be(2**255), rlp_uint(1)), OK, (0x80, 2**255, 1)),
    ]
    parents = [KECCAK(nodes[0]) for _, nodes, _, _ in cases]
    roots, status = eng.witness_roots(parents, [nodes for _, nodes, _, _ in cases], [block_arrays(block)] * len(cases))
    assert [int(s) for s in status] == [c[2] for c in cases], [c[0] for c in cases]
    for (name, _, st, f), r in zip(cases, roots):
        if st != OK:
            assert r.tobytes() == bytes(32), name
            continue
        n, b, v = f
        post = {a: (acc(n, b), {slot: v, KECCAK(b"new"): 2**256 - 1})}
        _, keys, accs, skeys, svals, offs = flatten(post)
        assert r.tobytes() == oracle.state_root_full(keys, accs, skeys, svals, offs), name
