"""The hash-and-sort paths of hash_sort.cu at their edges, against the oracle's keccak and a plain host ordering.

The sorts order rows by the top 32 bits of their digests; the head of every run of equal tops orders its run by the full
key in place (fix_runs_kernel, fix_runs_composite_kernel: runs of up to SORT_RUN_MAX = 16 rows), a verification pass
catches longer runs and sends the batch to a stable LSD sort over every word (32-byte digests: four words, 64-byte
composite keys: eight).  Uniform digests almost never reach those mechanisms, so the inputs here are crafted: pairs of
addresses / slots whose digests agree in the top 32 bits (found by a birthday search with the oracle), placed in runs of
equal keys just below and above the run limit.  In the changeset sorts (b200_hash_changesets) equal neighbours are legal
and stability alone keeps the oldest entry of a key in front.  Which path ran is read off the launch counter, so that a
test cannot silently stop covering a fallback.  Also: address tables longer than the batch (the composite sort's scratch
is shared with its nested sort of the address digests), the storage stage over accounts whose slots are all zero, and
the device-resident entry points through raw device pointers."""
import functools

import numpy as np
import pytest

import oracle
from tests.test_gpu_changesets import check, restate
from tests.util import random_keys, read_device, to_device_ptrs

pytestmark = [pytest.mark.gpu]

RUN_MAX = 16                # hash_sort.cu SORT_RUN_MAX: the longest run of equal tops ordered in place
DIGEST_FALLBACK = 4 * 2 + 1  # extra launches of the four-word LSD sort: (extract + radix pass) per word, one gather
COMPOSITE_FALLBACK = 8 * 2 + 2  # ... of the eight-word one: (extract + radix pass) per word, gather and check


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


@functools.lru_cache(maxsize=None)
def top32_pairs(width: int, seed: int, n: int = 1 << 18):
    """Pairs (x, y) of distinct `width`-byte messages whose keccak digests agree in their top 32 bits, found by a birthday
    search over n seeded random messages (about n^2 / 2^33 pairs).  keccak(y) < keccak(x): a sort that meets x first has to
    move y in front of it."""
    msgs = random_keys(seed, n)[:, :width].copy()
    dig = oracle.keccak256_fixed(msgs, threads=4)
    top = dig[:, :4].copy().view(">u4").ravel()
    order = np.argsort(top, kind="stable")
    pairs = []
    for h in np.nonzero(top[order][1:] == top[order][:-1])[0]:
        i, j = int(order[h]), int(order[h + 1])
        if dig[i].tobytes() == dig[j].tobytes():
            continue
        x, y = (i, j) if dig[i].tobytes() > dig[j].tobytes() else (j, i)
        pairs.append((msgs[x].copy(), msgs[y].copy()))
    assert pairs, "the birthday search found no pair with equal top 32 bits"
    return pairs


def address_pairs():
    return top32_pairs(20, 1001)


def slot_pairs():
    return top32_pairs(32, 1002)


def _launches(eng, fn):
    l0 = eng.launch_count()
    fn()
    return eng.launch_count() - l0


def _replace_rows(rows, old, new):
    out = rows.copy()
    out[(rows == old).all(axis=1)] = new
    return out


def _composite_ref(addrs, owner, slots):
    """keccak(addresses[owner[i]]) || keccak(slots[i]) for every entry, and their ascending (stable) order."""
    comp = np.concatenate([oracle.keccak256_fixed(addrs, threads=4)[owner], oracle.keccak256_fixed(slots, threads=4)], axis=1)
    v = comp.view(">u8")
    order = np.lexsort(tuple(v[:, i] for i in range(7, -1, -1)))
    return comp[order], order


def _digest_ref(msgs, msg_len):
    dig = oracle.keccak256_fixed(np.ascontiguousarray(msgs[:, :msg_len]), threads=4) if len(msgs) else np.zeros((0, 32), np.uint8)
    v = dig.view(">u8")
    order = np.lexsort((v[:, 3], v[:, 2], v[:, 1], v[:, 0]))
    return dig[order], order


def _dev_hash_sort_keys(eng, msgs, msg_len):
    """b200_hash_sort_keys_dev with input and outputs in device memory."""
    n, stride = msgs.shape
    pad = lambda a: a if n else np.zeros((1,) + a.shape[1:], a.dtype)
    (p_in, p_out, p_perm), hold = to_device_ptrs([pad(msgs), np.zeros((max(n, 1), 32), np.uint8), np.zeros(max(n, 1), np.uint32)])
    eng._check(eng.lib.b200_hash_sort_keys_dev(eng.ctx, p_in, msg_len, stride, n, p_out, p_perm))
    eng.sync()
    return read_device(hold[1]).reshape(-1, 32)[:n], read_device(hold[2], np.uint32)[:n]


def _dev_hash_sort_storage(eng, addrs, owner, slots):
    """b200_hash_sort_storage_dev with inputs and outputs in device memory."""
    n = len(slots)
    (p_a, p_i, p_s, p_out, p_perm), hold = to_device_ptrs([addrs, np.asarray(owner, np.uint32), slots,
                                                           np.zeros((max(n, 1), 64), np.uint8), np.zeros(max(n, 1), np.uint32)])
    eng._check(eng.lib.b200_hash_sort_storage_dev(eng.ctx, p_a, len(addrs), p_i, p_s, n, p_out, p_perm))
    eng.sync()
    return read_device(hold[3]).reshape(-1, 64)[:n], read_device(hold[4], np.uint32)[:n]


def _hash_sort_storage(eng, entry, addrs, owner, slots):
    if entry == "host":
        return eng.hash_sort_storage(addrs, owner, slots)
    return _dev_hash_sort_storage(eng, addrs, owner, slots)


def _storage_block(rng, addrs, slots_per):
    """Storage changeset rows of one block: a run of slots per address, addresses in ascending order."""
    sa, ss = [], []
    for a in sorted(addrs, key=lambda x: x.tobytes()):
        for _ in range(slots_per):
            sa.append(a)
            ss.append(rng.integers(0, 256, 32, dtype=np.uint8))
    return sa, ss


# ---------------------------------------------------------------------------------------------- changesets at the run limit
@pytest.mark.parametrize("where", ["start", "middle", "end"])
@pytest.mark.parametrize("k", [1, 14, 15, 16, 17, 40])
def test_account_run_limit(eng, k, where):
    """Account changesets: address A changed k times and B (same top 32 bits, smaller digest) inside A's run and once more
    later on.  The sorted top-32 run holds k + 2 rows: up to 16 are ordered in place, longer ones by the four-word fallback;
    either way the first occurrence of A and of B must come out."""
    a, b = address_pairs()[0]
    rng = np.random.default_rng(100 + k)
    other = rng.integers(0, 256, (60, 20), dtype=np.uint8)
    run = [a] * k
    run.insert({"start": 0, "middle": k // 2, "end": k}[where], b)
    acct = np.stack(list(other[:20]) + run + list(other[20:35]) + [b] + list(other[35:]))
    sa, ss = _storage_block(rng, list(other[:6]), 3)
    sa, ss = np.stack(sa), np.stack(ss)
    got = _launches(eng, lambda: check(eng, acct, sa, ss))
    control = _replace_rows(acct, b, rng.integers(0, 256, 20, dtype=np.uint8))
    base = _launches(eng, lambda: check(eng, control, sa, ss))
    assert got - base == (DIGEST_FALLBACK if k + 2 > RUN_MAX else 0)


@pytest.mark.parametrize("where", ["start", "middle", "end"])
@pytest.mark.parametrize("k", [1, 14, 15, 16, 17, 40])
def test_storage_run_limit(eng, k, where):
    """Storage changesets: under one address X, slot S1 changed k times and S2 (same top 32 bits of the digest, smaller
    digest) inside that run, and X again in a later block with S2.  The composite rows of X agreeing in the slot top form a
    run of k + 2: up to 16 ordered in place, longer ones by the eight-word fallback."""
    s1, s2 = slot_pairs()[0]
    rng = np.random.default_rng(200 + k)
    x = rng.integers(0, 256, 20, dtype=np.uint8)
    other = rng.integers(0, 256, (24, 20), dtype=np.uint8)
    run = [s1] * k
    run.insert({"start": 0, "middle": k // 2, "end": k}[where], s2)
    sa0, ss0 = _storage_block(rng, list(other[:8]), 3)
    sa1, ss1 = _storage_block(rng, list(other[8:16]), 2)
    sa2, ss2 = _storage_block(rng, list(other[16:]), 4)
    sa = np.stack(sa0 + [x] * len(run) + sa1 + [x, x] + sa2)
    ss = np.stack(ss0 + run + ss1 + [rng.integers(0, 256, 32, dtype=np.uint8), s2] + ss2)
    acct = np.stack([x] + list(other[::3]))
    got = _launches(eng, lambda: check(eng, acct, sa, ss))
    control = _replace_rows(ss, s2, rng.integers(0, 256, 32, dtype=np.uint8))
    base = _launches(eng, lambda: check(eng, acct, sa, control))
    assert got - base == (COMPOSITE_FALLBACK if k + 2 > RUN_MAX else 0)


@pytest.mark.parametrize("layout", ["a_accounts_b_storage", "b_accounts_a_storage", "both_in_both"])
def test_prefix_union_collision(eng, layout):
    """A colliding pair that meets in the sort of the account prefix set, the union of the hashed account keys and the
    hashed addresses of the storage changesets."""
    a, b = address_pairs()[-1]
    rng = np.random.default_rng(301)
    other = rng.integers(0, 256, (30, 20), dtype=np.uint8)
    in_acct, in_stor = {"a_accounts_b_storage": ([a], [b]), "b_accounts_a_storage": ([b], [a]),
                        "both_in_both": ([a, b], [a, b])}[layout]
    acct = np.stack(list(other[:10]) + in_acct + list(other[10:15]))
    sa, ss = _storage_block(rng, list(other[15:]) + in_stor, 2)
    sa, ss = np.stack(sa), np.stack(ss)
    got = _launches(eng, lambda: check(eng, acct, sa, ss))
    c = rng.integers(0, 256, 20, dtype=np.uint8)
    base = _launches(eng, lambda: check(eng, _replace_rows(acct, b, c), _replace_rows(sa, b, c), ss))
    assert got == base, "a fallback ran: a run of 2 to 4 rows is ordered in place"
    prefix = restate(acct, sa, ss)[2]
    assert oracle.keccak256(b.tobytes()) in prefix and oracle.keccak256(a.tobytes()) in prefix


def test_hot_keys_keep_first_occurrence_without_fallback(eng):
    """One address changed in each of 40 blocks, one of its slots changed in each of them, between ordinary rows: runs of
    40 equal keys in every sort.  The oldest entry is kept, and no fallback runs: equal neighbours are left alone."""
    rng = np.random.default_rng(401)
    hot_a = rng.integers(0, 256, 20, dtype=np.uint8)
    hot_s = rng.integers(0, 256, 32, dtype=np.uint8)

    def blocks(hot_a, hot_s):
        """40 blocks; hot_a / hot_s: the hot address / slot, or None for a fresh one in every block"""
        acct, sa, ss = [], [], []
        for _ in range(40):
            h = hot_a if hot_a is not None else rng.integers(0, 256, 20, dtype=np.uint8)
            s = hot_s if hot_s is not None else rng.integers(0, 256, 32, dtype=np.uint8)
            addrs = sorted([rng.integers(0, 256, 20, dtype=np.uint8) for _ in range(4)] + [h], key=lambda x: x.tobytes())
            acct += addrs
            for a in addrs:
                row_slots = [rng.integers(0, 256, 32, dtype=np.uint8), s, rng.integers(0, 256, 32, dtype=np.uint8)] \
                    if a is h else [rng.integers(0, 256, 32, dtype=np.uint8) for _ in range(3)]
                sa += [a] * 3
                ss += row_slots
        return np.stack(acct), np.stack(sa), np.stack(ss)

    acct, sa, ss = blocks(hot_a, hot_s)
    assert ((sa == hot_a).all(axis=1) & (ss == hot_s).all(axis=1)).sum() == 40
    got = _launches(eng, lambda: check(eng, acct, sa, ss))
    c_acct, c_sa, c_ss = blocks(None, None)
    base = _launches(eng, lambda: check(eng, c_acct, c_sa, c_ss))
    assert got == base, "a fallback ran on runs of equal keys"


# ---------------------------------------------------------------------------------------------- the full-pass composite sort
@pytest.mark.parametrize("entry", ["host", "dev"])
def test_storage_repeated_address_and_collisions(eng, entry):
    """An address table listing A 20 times with B (same top 32 bits, smaller digest) between its copies: the nested sort of
    the address digests (equal neighbours allowed) needs its four-word fallback, and every copy of A takes one rank.  Slot
    pairs with equal tops under one address (one of them split over two copies of A) are ordered in place."""
    a, b = address_pairs()[0]
    rng = np.random.default_rng(501)
    other = rng.integers(0, 256, (40, 20), dtype=np.uint8)
    table = np.stack(list(other[:10]) + [a] * 9 + [b] + [a] * 11 + list(other[10:]))
    owner = np.repeat(np.arange(len(table)), 3)
    slots = rng.integers(0, 256, (len(owner), 32), dtype=np.uint8)
    copies_of_a = np.nonzero((table == a).all(axis=1))[0]
    extra_owner, extra_slots = [], []
    for j, (s1, s2) in enumerate(slot_pairs()):
        o1, o2 = (copies_of_a[3], copies_of_a[7]) if j == 0 else (j % 10, j % 10)
        extra_owner += [o1, o2]
        extra_slots += [s1, s2]
    owner = np.concatenate([owner, np.array(extra_owner)]).astype(np.uint32)
    slots = np.concatenate([slots, np.stack(extra_slots)])   # each pair larger digest first: the in-place fixer swaps it
    keys_ref, order_ref = _composite_ref(table, owner, slots)
    l0 = eng.launch_count()
    keys, perm = _hash_sort_storage(eng, entry, table, owner, slots)
    n_launch = eng.launch_count() - l0
    assert (keys == keys_ref).all()
    assert (perm.astype(np.int64) == order_ref).all()
    control = _replace_rows(table, b, rng.integers(0, 256, 20, dtype=np.uint8))
    base = _launches(eng, lambda: _hash_sort_storage(eng, entry, control, owner, slots))
    assert n_launch - base == DIGEST_FALLBACK


@pytest.mark.parametrize("entry", ["host", "dev"])
@pytest.mark.parametrize("n_addr,n", [(200_000, 20_000), (100_000, 1), (24_100, 20_000)], ids=["addr10x", "one_entry", "addr1.2x"])
def test_address_table_longer_than_batch(entry, n_addr, n):
    """More addresses than entries, on a fresh context: the scratch of the composite sort has to hold the nested sort of
    all address digests as well as the entries."""
    from reth_b200 import Engine
    rng = np.random.default_rng(n_addr + n)
    addrs = rng.integers(0, 256, (n_addr, 20), dtype=np.uint8)
    owner = rng.integers(0, n_addr, n).astype(np.uint32)
    slots = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    keys_ref, order_ref = _composite_ref(addrs, owner, slots)
    e = Engine(0)
    try:
        keys, perm = _hash_sort_storage(e, entry, addrs, owner, slots)
    finally:
        e.close()
    assert (keys == keys_ref).all()
    assert (perm.astype(np.int64) == order_ref).all()


def test_address_table_grows_between_calls():
    """One context, the address table growing from call to call while the batch stays small, through both entry points."""
    from reth_b200 import Engine
    rng = np.random.default_rng(601)
    e = Engine(0)
    try:
        for n_addr, n, entry in [(40, 3000, "host"), (50_000, 3000, "host"), (60, 2500, "dev"), (90_000, 2500, "dev"),
                                 (130_000, 10, "host"), (3, 40_000, "dev")]:
            addrs = rng.integers(0, 256, (n_addr, 20), dtype=np.uint8)
            owner = rng.integers(0, n_addr, n).astype(np.uint32)
            slots = rng.integers(0, 256, (n, 32), dtype=np.uint8)
            keys, perm = _hash_sort_storage(e, entry, addrs, owner, slots)
            keys_ref, order_ref = _composite_ref(addrs, owner, slots)
            assert (keys == keys_ref).all(), (n_addr, n, entry)
            assert (perm.astype(np.int64) == order_ref).all(), (n_addr, n, entry)
    finally:
        e.close()


def test_storage_stage_with_zero_only_accounts():
    """StorageHashingStage.execute hands every account with a non-empty storage dict to the sort and drops the zero-valued
    slots: a state in which most accounts hold only zeros has far more addresses than entries."""
    from reth_b200 import Engine, StorageHashingStage
    from reth_b200.stages import Tables
    rng = np.random.default_rng(701)
    t = Tables()
    for i in range(4000):
        t.plain_storage[bytes(rng.integers(0, 256, 20, dtype=np.uint8))] = {int(rng.integers(0, 2**40)): 0 for _ in range(2)}
        if i % 200 == 0:
            live = {int(rng.integers(0, 2**40)): int(rng.integers(1, 2**62)) for _ in range(int(rng.integers(1, 12)))}
            live[int(rng.integers(0, 2**40))] = 0
            t.plain_storage[bytes(rng.integers(0, 256, 20, dtype=np.uint8))] = live
    want = {}
    for a, st in t.plain_storage.items():
        rows = sorted((oracle.keccak256(s.to_bytes(32, "big")), v) for s, v in st.items() if v)
        if rows:
            want[oracle.keccak256(a)] = rows
    e = Engine(0)
    try:
        total = StorageHashingStage(e).execute(t)
    finally:
        e.close()
    assert total == sum(len(v) for v in want.values()) and total < len(t.plain_storage) // 10
    assert list(t.hashed_storages) == sorted(want)
    assert t.hashed_storages == want


# ---------------------------------------------------------------------------------------------- device entry points
@pytest.mark.parametrize("stride", [20, 32])
@pytest.mark.parametrize("n", [0, 1, 2, (1 << 17) + 4099])
def test_hash_sort_keys_dev(eng, stride, n):
    """b200_hash_sort_keys_dev: 20-byte messages at strides 20 and 32 equal b200_hash_sort_keys and the oracle; the larger
    batches hold colliding address pairs, listed larger digest first."""
    rng = np.random.default_rng(800 + n + stride)
    msgs = rng.integers(0, 256, (n, stride), dtype=np.uint8)
    pairs = address_pairs()
    if n >= 2:
        for j, (x, y) in enumerate(pairs[: n // 2]):
            msgs[j, :20], msgs[n - 1 - j, :20] = x, y
    dig_ref, order_ref = _digest_ref(msgs, 20)
    keys, perm = _dev_hash_sort_keys(eng, msgs, 20)
    assert (keys == dig_ref).all() and (perm.astype(np.int64) == order_ref).all()
    h_keys, h_perm = eng.hash_sort_keys(msgs, 20)
    assert (h_keys == keys).all() and (h_perm == perm).all()


def test_hash_sort_storage_dev_matches_host_and_rejects_bad_input(eng):
    """b200_hash_sort_storage_dev equals b200_hash_sort_storage and the oracle; an addr_index entry out of range is
    ERR_INVALID_ARG, a repeated (address, slot) pair ERR_UNSORTED, and the context goes on working after either."""
    from reth_b200 import B200Error, _lib
    rng = np.random.default_rng(901)
    n_addr, n = 300, 30_000
    addrs = rng.integers(0, 256, (n_addr, 20), dtype=np.uint8)
    addrs[11] = addrs[250]
    owner = rng.integers(0, n_addr, n).astype(np.uint32)
    owner[:12_000] = 42
    slots = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    keys_ref, order_ref = _composite_ref(addrs, owner, slots)

    def ok():
        keys, perm = _dev_hash_sort_storage(eng, addrs, owner, slots)
        assert (keys == keys_ref).all() and (perm.astype(np.int64) == order_ref).all()
        h_keys, h_perm = eng.hash_sort_storage(addrs, owner, slots)
        assert (h_keys == keys).all() and (h_perm == perm).all()

    ok()
    bad = owner.copy()
    bad[n // 2] = n_addr
    with pytest.raises(B200Error) as err:
        _dev_hash_sort_storage(eng, addrs, bad, slots)
    assert err.value.status == _lib.ERR_INVALID_ARG
    ok()
    dup_owner, dup_slots = owner.copy(), slots.copy()
    dup_owner[7], dup_slots[7] = dup_owner[20_000], dup_slots[20_000]
    with pytest.raises(B200Error) as err:
        _dev_hash_sort_storage(eng, addrs, dup_owner, dup_slots)
    assert err.value.status == _lib.ERR_UNSORTED
    dup_owner, dup_slots = owner.copy(), slots.copy()
    dup_owner[7], dup_owner[8], dup_slots[8] = 11, 250, dup_slots[7]   # one address under its two indices, one slot
    with pytest.raises(B200Error) as err:
        _dev_hash_sort_storage(eng, addrs, dup_owner, dup_slots)
    assert err.value.status == _lib.ERR_UNSORTED
    ok()
