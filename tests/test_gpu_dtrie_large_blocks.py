"""The large-block paths of the dynamic tries (b200_dtrie_apply, b200_dstate_apply; eng_darena.inl).

A block of at most 8192 entries per arena is restructured by one CTA (dt_restructure_fused_kernel); a bigger one takes the
multi-launch form: locate + detach, collapse rounds over many CTAs (dt_round_defer / dt_collapse_round, one host read-back
per round), then insert rounds (dt_insert_locate / dt_insert_runs / dt_insert_unlock, at most 8 keys per run per round,
the leftover compacted between rounds).  Its re-hash has more than WARP_LEVEL_MAX dirty entries, so it takes the two-stage
form (one thread per seed, then the hand-off climb).  These forms are correct only because of properties that concurrency
between CTAs can break (one writer per word in a collapse round, the locked attach words of an insert round, the free-stack
pops settled once per phase, the last-arriver climb), so every case here sends blocks of more than 8192 entries through
them at the default thresholds and compares, after every block, the root, the stored-node sets after the block's
TrieUpdates, the counters and the storage-deleted flags with a from-scratch oracle build (the harnesses of
test_gpu_dtrie.py / test_gpu_dstate.py).  The phase labels the library prints with B200_PHASE_TIMING set prove which form
ran and how many collapse and insert rounds it took.

The last tests run other parts of the suite in child processes with every size switch forced each way: the switches are
read once per process."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import oracle
from tests.test_gpu_dstate import EXISTS, UNCHANGED, WIPED, Harness as StateHarness, ShardedHarness
from tests.test_gpu_dstate import acct as sacct, random_block as state_block, random_state, rkey
from tests.test_gpu_dtrie import Harness as TrieHarness, acct, random_block as trie_block
from tests.test_gpu_level_classes import launch_threshold

pytestmark = [pytest.mark.gpu]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUSED_DEFAULT = 8192   # reth_b200/csrc/eng_darena.inl dt_fused_max: the one-CTA restructure up to this many entries per arena


def fused_max():
    """the fused-form limit of the library under test (B200_DT_FUSED_MAX; the CPU emulation keeps the default)"""
    return int(os.environ.get("B200_DT_FUSED_MAX", FUSED_DEFAULT))


def two_stage_min():
    """the re-hash switch-over (B200_DT_TWO_STAGE_MIN, default WARP_LEVEL_MAX, which the CPU emulation lowers)"""
    v = os.environ.get("B200_DT_TWO_STAGE_MIN")
    return int(v) if v is not None else launch_threshold()


@pytest.fixture(scope="module")
def timed():
    """A context with B200_PHASE_TIMING set: every apply prints its phase labels on stderr."""
    from reth_b200 import Engine
    old = os.environ.get("B200_PHASE_TIMING")
    os.environ["B200_PHASE_TIMING"] = "1"
    try:
        e = Engine(0)
    finally:
        if old is None:
            del os.environ["B200_PHASE_TIMING"]
        else:
            os.environ["B200_PHASE_TIMING"] = old
    yield e
    e.close()


def applies(capfd, call, marker=None):
    """-> the phase labels of every apply that call() made (one list per [b200 phases] line that contains `marker`)"""
    capfd.readouterr()
    call()
    out = []
    for line in capfd.readouterr().err.splitlines():
        if line.startswith("[b200 phases]"):
            names = line.split(":", 1)[1].split()[0::2]       # " name ms" pairs after "total X ms:"
            if marker is None or marker in names:
                out.append(names)
    return out


def rounds(names):
    """restructure labels of one arena -> (multi-launch form ran, collapse rounds, insert rounds)"""
    multi = "r:locate+detach" in names
    if not multi:
        assert not [x for x in names if x.startswith("r:")], names
        return False, 0, 0
    return True, names.count("r:collapse-sync") - 1, names.count("r:insert-round")


def arenas(names):
    """the labels of one b200_dstate_apply split by arena: (account restructure, storage restructure)"""
    a = names.index("acct-restructure")
    if "storage-restructure" not in names:
        return names[:a], []
    return names[:a], names[names.index("wipes") + 1:names.index("storage-restructure")]


def check_form(names, m, record, tag, min_collapse=0, min_insert=0):
    """The arena got m > 8192 entries: the multi-launch form ran unless B200_DT_FUSED_MAX says otherwise, with at least the
    expected rounds.  -> (collapse rounds, insert rounds)"""
    assert m > FUSED_DEFAULT, m
    multi, nc, ni = rounds(names)
    assert multi == (m > fused_max()), (m, fused_max(), names)
    if multi:
        assert nc >= min_collapse, (nc, names)
        assert ni >= min_insert, (ni, names)
    # (the re-hash form follows from m alone: two-stage above two_stage_min())
    record(tag, {"entries": m, "multi": multi, "collapse_rounds": nc, "insert_rounds": ni, "two_stage_rehash": m > two_stage_min()})
    return nc, ni


def absent_deletes(rng, state, n):
    """n deletions of keys that are not in the trie (no-ops that still count as block entries)"""
    out = {}
    while len(out) < n:
        k = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
        if k not in state:
            out[k] = (0, acct(0))
    return out


# ---- DynamicTrie: the account arena alone ------------------------------------------------------------------------------
def test_small_block_control(timed, capfd):
    """a block below the limit: no multi-launch labels unless B200_DT_FUSED_MAX forces that form"""
    h = TrieHarness(timed, 3000, seed=41)
    rng = np.random.default_rng(41)
    block = trie_block(rng, h.state, 600, 1)
    (names,) = applies(capfd, lambda: h.commit(block))
    assert rounds(names)[0] == (len(block) > fused_max()), names
    h.trie.close()


def test_small_block_control_state(timed, capfd):
    rng = np.random.default_rng(42)
    h = StateHarness(timed, random_state(rng, 600))
    block = state_block(rng, h.state, 150, 1)
    m, n = len(block), sum(len(s) for _, _, s in block.values())
    (names,) = applies(capfd, lambda: h.commit(block), "acct-restructure")
    a, s = arenas(names)
    assert rounds(a)[0] == (m > fused_max()) and rounds(s)[0] == (n > fused_max()), names
    h.ds.close()


def test_halving_cascades(timed, capfd, record_property):
    """every other key deleted three times from 84 000 leaves: 42 000, 21 000, 10 500 deletions, chained collapses"""
    h = TrieHarness(timed, 84_000, seed=43)
    for step in range(3):
        block = {k: (0, acct(0)) for k in sorted(h.state)[::2]}
        (names,) = applies(capfd, lambda: h.commit(block))
        check_form(names, len(block), record_property, f"halving_{step}", min_collapse=2)
    h.trie.close()


def unused_prefixes(rng, state, n, nibbles=5):
    """n distinct random prefixes of `nibbles` nibbles that no key of `state` starts with"""
    bits = 4 * nibbles
    taken = {int.from_bytes(k[:4], "big") >> (32 - bits) for k in state}
    out = set()
    while len(out) < n:
        p = int(rng.integers(0, 1 << bits))
        if p not in taken:
            out.add(p)
    return sorted(out)


def long_run_groups(rng, state, n_groups):
    """Insert keys in groups of 9..40 that share an 8-nibble prefix whose first 5 nibbles no existing key has: every key of
    a group attaches at the same word (an empty slot, or an existing leaf whose edge the group branches off inside).  Within
    a group the keys fall into sub-clusters A < B < C by their 9th nibble, A and B of 8 keys: round 1 inserts A (a branch
    at depth 9 below an extension), B and C then diverge inside that edge, so they attach at one word again; round 2
    inserts B and round 3 the keys of C, now at a slot of their own.  -> {key: (1, account)}"""
    dirty = {}
    for p in unused_prefixes(rng, state, n_groups):
        g = int(rng.integers(9, 41))
        head = ((p << 12) | int(rng.integers(0, 1 << 12))).to_bytes(4, "big")      # 8 nibbles
        subs = np.sort(rng.choice(16, 3, replace=False))
        for nib, size in zip(subs, (8, min(8, g - 8), max(g - 16, 0))):
            for _ in range(size):
                tail = rng.integers(0, 256, 28, dtype=np.uint8).tobytes()
                dirty[head + bytes([(int(nib) << 4) | (tail[0] & 0x0F)]) + tail[1:]] = (1, acct(g))
    return dirty


def test_long_insert_runs(timed, capfd, record_property):
    rng = np.random.default_rng(44)
    h = TrieHarness(timed, 20_000, seed=44)
    block = long_run_groups(rng, h.state, 400)
    (names,) = applies(capfd, lambda: h.commit(block))
    check_form(names, len(block), record_property, "long_runs", min_insert=2)
    # and the same shape once more on top, in the same block as the deletion of every seventh key
    block = long_run_groups(rng, h.state, 400)
    block.update({k: (0, acct(0)) for k in sorted(h.state)[::7]})
    (names,) = applies(capfd, lambda: h.commit(block))
    check_form(names, len(block), record_property, "long_runs_with_deletes", min_insert=2)
    h.trie.close()


def test_split_runs_at_scale(timed, capfd, record_property):
    """test_gpu_dtrie.py::test_split_runs_share_an_attach_point with 3 100 triples per block: K1 and K3 diverge inside the
    long edge above a node N (one attach word), K2 passes through it and attaches below N"""
    rng = np.random.default_rng(45)
    stems, state0 = [], {}
    for _ in range(3100):
        stem = rng.integers(0, 256, 20, dtype=np.uint8).tobytes()
        stems.append(stem)
        for last in (0x10, 0xE0):
            state0[stem + bytes([last]) + rng.integers(0, 256, 11, dtype=np.uint8).tobytes()] = acct(1)
    h = TrieHarness(timed, 0, seed=46)
    h.commit({k: (1, a) for k, a in state0.items()})
    for step in range(2):
        dirty = {}
        for stem in stems:
            cut = int(rng.integers(2 + step, 19))
            lo, hi = bytearray(stem), bytearray(stem)
            if lo[cut] == 0 or hi[cut] == 255:
                continue
            lo[cut] -= 1
            hi[cut] += 1
            tail = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            dirty[bytes(lo[:cut + 1]) + tail(31 - cut)] = (1, acct(2))
            dirty[stem + bytes([0x70 + step]) + tail(11)] = (1, acct(3))
            dirty[bytes(hi[:cut + 1]) + tail(31 - cut)] = (1, acct(4))
        (names,) = applies(capfd, lambda: h.commit(dirty))
        check_form(names, len(dirty), record_property, f"split_runs_{step}", min_insert=1)
    h.trie.close()


def test_mixed_blocks(timed, capfd, record_property):
    rng = np.random.default_rng(47)
    h = TrieHarness(timed, 20_000, seed=47)
    for step in range(2):
        block = trie_block(rng, h.state, 9600, step)
        (names,) = applies(capfd, lambda: h.commit(block))
        check_form(names, len(block), record_property, f"mixed_{step}", min_collapse=1, min_insert=1)
    h.trie.close()


def test_shrink_to_one_then_empty_then_regrow(timed, capfd, record_property):
    """each block has more than 8192 entries: deletions of absent keys pad the ones that delete only a few"""
    rng = np.random.default_rng(48)
    h = TrieHarness(timed, 9000, seed=48)
    keep = sorted(h.state)[4321]
    block = {k: (0, acct(0)) for k in h.state if k != keep}
    (names,) = applies(capfd, lambda: h.commit(block))
    check_form(names, len(block), record_property, "shrink_to_one", min_collapse=2)
    assert len(h.trie) == 1
    block = {keep: (0, acct(0)), **absent_deletes(rng, h.state, 8500)}
    (names,) = applies(capfd, lambda: h.commit(block))
    check_form(names, len(block), record_property, "shrink_to_empty")
    assert h.trie.root() == oracle.EMPTY_ROOT_HASH and len(h.trie) == 0
    block = {rng.integers(0, 256, 32, dtype=np.uint8).tobytes(): (1, acct(7)) for _ in range(9000)}   # one run at the root
    (names,) = applies(capfd, lambda: h.commit(block))
    check_form(names, len(block), record_property, "regrow", min_insert=2)
    block = {k: (0, acct(0)) for k in sorted(h.state)[1:]}
    block.update(absent_deletes(rng, h.state, 100))
    (names,) = applies(capfd, lambda: h.commit(block))
    check_form(names, len(block), record_property, "shrink_to_one_again", min_collapse=2)
    h.trie.close()


# ---- DynamicState: both arenas ------------------------------------------------------------------------------------------
def slot_entries(block):
    return sum(len(s) for _, _, s in block.values())


def commit_state(h, capfd, block):
    """-> (account restructure labels, storage restructure labels) of the block's apply"""
    (names,) = applies(capfd, lambda: h.commit(block), "acct-restructure")
    return arenas(names)


def test_mass_slot_deletion_across_storage_tries(timed, capfd, record_property):
    """about half the slots of 300 storage tries deleted in one block, 40 of the tries emptied"""
    rng = np.random.default_rng(50)
    st = random_state(rng, 800, with_storage=0.0)
    owners = sorted(st)[:300]
    for k in owners:
        st[k] = (st[k][0], {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(int(rng.integers(30, 80)))})
    h = StateHarness(timed, st)
    block = {}
    for i, k in enumerate(owners):
        slots = sorted(h.state[k][1])
        gone = slots if i % 7 == 0 else slots[::2]
        block[k] = (EXISTS | UNCHANGED, sacct(0), {s: 0 for s in gone})
    _, s = commit_state(h, capfd, block)
    check_form(s, slot_entries(block), record_property, "mass_slot_deletion", min_collapse=2)
    assert sum(1 for k in owners if not h.state[k][1]) >= 40
    h.ds.close()


def test_wipe_and_refill_then_destroy_and_recreate(timed, capfd, record_property):
    rng = np.random.default_rng(51)
    st = random_state(rng, 300, with_storage=0.2, max_slots=20)
    big = sorted(st)[:3]
    for j, k in enumerate(big):
        st[k] = (st[k][0], {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(20_500 if j == 0 else 6000)})
    h = StateHarness(timed, st)
    # the 20 500-slot trie wiped and refilled with 8 600 new slots (and a few of its old ones) in the same block
    old = sorted(h.state[big[0]][1])
    refill = {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(8600)}
    refill.update({s: 5 for s in old[:50]})
    block = {big[0]: (EXISTS | WIPED, h.state[big[0]][0].copy(), refill)}
    _, s = commit_state(h, capfd, block)
    check_form(s, slot_entries(block), record_property, "wipe_and_refill", min_insert=2)
    assert len(h.state[big[0]][1]) == 8650
    # the accounts with large storage destroyed ...
    block = {k: (0, sacct(0), {}) for k in big}
    commit_state(h, capfd, block)
    assert h.ds.slots() == sum(len(x) for _, x in h.state.values())
    # ... and re-created in the next block, two of them with more than 8192 new slots between them
    block = {k: (EXISTS, sacct(3, 9), {rkey(rng): int(rng.integers(1, 2**60)) for _ in range(4400 if j < 2 else 10)})
             for j, k in enumerate(big)}
    _, s = commit_state(h, capfd, block)
    check_form(s, slot_entries(block), record_property, "recreate", min_insert=2)
    h.ds.close()


def test_large_account_side_with_destructions_and_storage(timed, capfd, record_property):
    """9 000+ account entries (a fifth destroyed, storage tries among them) and storage changes in the same block"""
    rng = np.random.default_rng(52)
    h = StateHarness(timed, random_state(rng, 20_000, with_storage=0.15, max_slots=12))
    live = sorted(h.state)
    block = {}
    for n, i in enumerate(rng.choice(len(live), 8000, replace=False)):
        k = live[i]
        if n % 5 == 0:
            block[k] = (0, sacct(0), {})
        elif n % 5 == 1 and h.state[k][1]:
            block[k] = (EXISTS | UNCHANGED, sacct(0), {s: (0 if j % 2 else 11) for j, s in enumerate(sorted(h.state[k][1]))})
        else:
            a = h.state[k][0].copy()
            a["nonce"] += 1
            block[k] = (EXISTS, a, {})
    for _ in range(1200):
        block[rkey(rng)] = (EXISTS, sacct(1, 2), {rkey(rng): 3 for _ in range(int(rng.integers(0, 3)))})
    a, _ = commit_state(h, capfd, block)
    check_form(a, len(block), record_property, "account_side", min_collapse=1, min_insert=1)
    h.ds.close()


@pytest.mark.parametrize("seed", [0, 1])
def test_random_state_blocks_above_the_limit(timed, capfd, record_property, seed):
    rng = np.random.default_rng(53 + seed)
    h = StateHarness(timed, random_state(rng, 3000))
    for step in range(2):
        block = state_block(rng, h.state, 3600, step + 1)
        for k in list(block)[:400]:                      # more slots per touch for a few hundred of them
            fl, a, slots = block[k]
            if fl & EXISTS:
                slots.update({rkey(rng): int(rng.integers(1, 2**60)) for _ in range(8)})
        _, s = commit_state(h, capfd, block)
        check_form(s, slot_entries(block), record_property, f"random_state_{seed}_{step}", min_insert=1)
    h.ds.close()


def skewed_state(rng, n, world):
    """random accounts, three quarters of them moved into the top nibbles of rank 0 (world 2: 0-7, world 16: 0)"""
    mask = 0x7F if world == 2 else 0x0F
    st = {}
    for i, (k, v) in enumerate(random_state(rng, n, with_storage=0.1, max_slots=10).items()):
        st[bytes([k[0] & mask]) + k[1:] if i % 4 != 3 else k] = v
    return st


@pytest.mark.parametrize("world", [2, 16])
def test_sharded_big_block(timed, capfd, record_property, world):
    """one block with more than 8192 account entries in rank 0's shard (its account arena is a forest of bucket tries,
    re-hashed with split depth 3) and storage changes in every shard"""
    rng = np.random.default_rng(54 + world)
    h = ShardedHarness(timed, skewed_state(rng, 12_000, world), world)
    mine = [k for k in sorted(h.state) if h.rank_of(k) == 0]
    block = state_block(rng, h.state, 800, 1)
    for n, i in enumerate(rng.choice(len(mine), 8600, replace=False)):
        k = mine[i]
        if n % 6 == 0:
            block[k] = (0, sacct(0), {})
        else:
            a = h.state[k][0].copy()
            a["nonce"] += 1
            block[k] = (EXISTS, a, {rkey(rng): 4} if n % 6 == 1 else {})
    m0 = sum(1 for k in block if h.rank_of(k) == 0)
    labels = applies(capfd, lambda: h.commit(block), "acct-restructure")
    a, _ = arenas(labels[0])                             # the shards apply in rank order
    check_form(a, m0, record_property, f"sharded_{world}", min_collapse=1, min_insert=1)
    for ds in h.shards:
        ds.close()


# ---- every size switch forced both ways, in child processes --------------------------------------------------------------
LARGE_BLOCK_TESTS = ("tests/test_gpu_leaf_widths.py::test_dynamic_state_wide_accounts",
                     "tests/test_gpu_dstate.py::test_inline_children_of_clustered_slots")
FORCED = {   # name: (settings, test paths, -k selection, minimum passed)
    # every block takes the multi-launch restructure and the two-stage re-hash
    "large_forms": ({"B200_DT_FUSED_MAX": "0", "B200_DT_TWO_STAGE_MIN": "0"},
                    ["tests/test_gpu_dtrie.py", "tests/test_gpu_dstate.py", "tests/test_gpu_leaf_widths.py",
                     "tests/test_gpu_dtrie_large_blocks.py"],
                    "(not test_gpu_leaf_widths or dynamic_) and (not test_gpu_dtrie_large_blocks or small_block_control)", 36),
    # every block takes the one-CTA restructure and the one-warp-per-seed re-hash
    "small_forms": ({"B200_DT_FUSED_MAX": "4294967295", "B200_DT_TWO_STAGE_MIN": "4294967295"},
                    ["tests/test_gpu_dtrie_large_blocks.py", *LARGE_BLOCK_TESTS], None, 17),
    "wavefront_two_stage": ({"B200_WAVEFRONT_TWO_STAGE_MIN": "0"},
                            ["tests/test_gpu_trie.py", "tests/test_gpu_leaf_widths.py"], "resident_trie_", 8),
    "wavefront_one_stage": ({"B200_WAVEFRONT_TWO_STAGE_MIN": "4294967295"},
                            ["tests/test_gpu_trie.py", "tests/test_gpu_leaf_widths.py"], "resident_trie_", 8),
    "one_stream_build": ({"B200_OVERLAP_STRUCTURE": "0"}, ["tests/test_gpu_trie.py", "tests/test_gpu_level_classes.py"],
                         "genesis or testspec or account_and_storage or extension or empty_and_single or forest or node_heads "
                         "or account_trie_random or c1_config or full_state_random or inline_children or extensions "
                         "or threshold_edges or ordered_roots_of_tiny", 25),
}
# Under the CPU emulation every warp shuffle is 32 context switches: it leaves out the biggest sizes, and the one-warp-per-seed
# re-hash of blocks above 8192 entries, so that this file rehearses in minutes there.  The device runs every row in full.
EMU_SKIP = "not 200000 and not one_million"
EMU_ROWS = {"small_forms": ("small_block_control", 2)}


def child_selection(name):
    """-> (test paths, -k expression, minimum passed) of a row of FORCED in this process (emulated or not)"""
    _, paths, k, min_passed = FORCED[name]
    ks = ["not forced_"] + ([f"({k})"] if k else [])
    if os.environ.get("B200_EMU"):
        ks.append(EMU_SKIP)
        if name in EMU_ROWS:
            k, min_passed = EMU_ROWS[name]
            ks.append(f"({k})")
    return paths, " and ".join(ks), min_passed


@pytest.mark.parametrize("name", sorted(FORCED))
def test_forced_switch(name):
    paths, kexpr, min_passed = child_selection(name)
    cmd = [sys.executable, "-m", "pytest", *paths, "-m", "gpu", "-q", "-p", "no:cacheprovider", "-k", kexpr]
    if os.environ.get("B200_EMU"):
        cmd.append("--emu")
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=3000, env=dict(os.environ, **FORCED[name][0]))
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    passed = re.search(r"(\d+) passed", r.stdout)
    assert passed and int(passed.group(1)) >= min_passed, tail
