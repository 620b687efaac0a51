"""The class-split branch kernels of the forest build (eng_build.inl build_forest) on the shapes that take their strip path:
inline (< 32 byte) children, extension wrappers, stored-hash items and trie roots shorter than 32 bytes.

build_forest sends a depth with at most WARP_LEVEL_MAX branch nodes (summed over every trie of the call) to one warp per
node; a bigger depth gets one thread-per-node launch per child-count class (2-3: branch3_pipelined_kernel, 4-7 / 8-12 /
13-16: branch_kernel<128, 7|12|16>), except that a class of at most WARP_LEVEL_MAX / 4 nodes still goes to the warp kernel.
Random 32-byte keys reach the thread kernels only with hashed children and the occasional extension, so every case here
builds its keys so that the (depth, class) it is about is a thread-kernel launch, and proves it twice:
  * a census of the branch nodes computed on the host from the sorted keys (`Census`), checked at the product thresholds;
  * the launch labels the library prints per build with B200_PHASE_TIMING set (`big<=3` ... `big<=16`, `small-class`,
    `small-level`), which must be exactly the sequence the census predicts.
Every root, TrieUpdates record set and node counter is compared bit-exactly with the CPU oracle (pinned by reth's golden
vectors), or for the items fold with the oracle's HashBuilder fed the same stream."""
import os

import numpy as np
import pytest

import oracle
from tests.test_gpu_dstate import clustered_slots, flatten, random_block, random_state
from tests.test_gpu_witness import apply_to_model, block_arrays, make_state
from tests.util import synth_accounts

pytestmark = [pytest.mark.gpu]

WARP_LEVEL_MAX = 4096                  # reth_b200/csrc/engine.cu: a depth of at most this many nodes: one warp per node
CLASS_WARP_MAX = WARP_LEVEL_MAX // 4   # a class of at most this many nodes inside a bigger depth: one warp per node too
CLASS_LO = np.array([2, 4, 8, 13])     # child-count classes 2-3, 4-7, 8-12, 13-16
CLASS_HI = np.array([4, 8, 13, 17])
BIG = ("big<=3", "big<=7", "big<=12", "big<=16")
DISPATCH = {"small-level", "small-class", *BIG}


def launch_threshold():
    """WARP_LEVEL_MAX of the library under test: the CPU emulation lowers it (tools/emu/translate.py, EMU_WARP_LEVEL_MAX)."""
    if os.environ.get("B200_EMU"):
        return int(os.environ.get("EMU_WARP_LEVEL_MAX", "192"))
    return WARP_LEVEL_MAX


@pytest.fixture(scope="module")
def eng():
    from reth_b200 import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def timed():
    """A second context with B200_PHASE_TIMING set: every sync prints the launch labels of its builds on stderr."""
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


def with_phases(capfd, call):
    """-> (call(), the phase names the library printed while it ran, in order)"""
    capfd.readouterr()
    out = call()
    names = []
    for line in capfd.readouterr().err.splitlines():
        if line.startswith("[b200 phases]"):
            names += line.split(":", 1)[1].split()[0::2]       # " name ms" pairs after "total X ms:"
    return out, names


def launches(names):
    return [x for x in names if x in DISPATCH]


# ---- census of the branch nodes, from the keys alone --------------------------------------------------------------------
class Census:
    """Every branch node of a forest of sorted, prefix-free keys: its depth, child count, class, whether it is wrapped in an
    extension (its parent lies more than one nibble up, or it is a root below depth 0) and whether it is a trie root.

    Keys are rows of bytes (32 for hashed keys, fewer for zero-padded RLP(index) keys or item paths: prefix-free keys differ
    before the shorter one ends, so the padding never counts).  The gap between keys i-1 and i has the length of their
    common nibble prefix, -1 across a trie boundary.  A node of depth d is a run of depth-d gaps with no shallower gap
    between them; its parent's depth is the deeper of the two shallower gaps that enclose the run."""

    def __init__(self, keys, seg_offsets=None):
        keys = np.ascontiguousarray(keys, np.uint8).reshape(len(keys), -1)
        n = len(keys)
        lcp = np.full(n + 1, -1, np.int64)
        if n > 1:
            diff = keys[1:] ^ keys[:-1]
            j = (diff != 0).argmax(1)
            lcp[1:n] = 2 * j + (diff[np.arange(n - 1), j] < 16)
        if seg_offsets is not None:
            lcp[np.asarray(seg_offsets, np.int64)] = -1
        depth, kids, parent, first = [], [], [], []
        for d in np.unique(lcp[lcp >= 0]):
            pos = np.nonzero(lcp == d)[0]
            low = np.nonzero(lcp < d)[0]
            cut = np.searchsorted(low, pos)                  # the first shallower gap to the right of each depth-d gap
            head = np.ones(len(pos), bool)
            head[1:] = cut[1:] != cut[:-1]
            k = np.bincount(np.cumsum(head) - 1) + 1
            left, right = low[cut[head] - 1], low[cut[head]]
            depth.append(np.full(len(k), d))
            kids.append(k)
            parent.append(np.maximum(lcp[left], lcp[right]))
            first.append(left)                               # index of the node's first key
        cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.int64)
        self.depth, self.kids, self.parent, self.first = cat(depth), cat(kids), cat(parent), cat(first)
        self.cls = np.searchsorted(CLASS_LO[1:], self.kids, side="right")
        self.wrapped = self.parent + 1 < self.depth
        self.root = self.parent < 0

    def count(self, d, cls=None):
        sel = self.depth == d
        if cls is not None:
            sel &= self.cls == cls
        return int(sel.sum())

    def dispatch(self, threshold):
        """the launch labels build_forest prints for this forest, deepest level first"""
        out = []
        for d in range(63, -1, -1):
            hc = [self.count(d, c) for c in range(4)]
            if not sum(hc):
                continue
            if sum(hc) <= threshold:
                out.append("small-level")
            else:
                out += ["small-class" if h <= threshold // 4 else BIG[c] for c, h in enumerate(hc) if h]
        return out

    def assert_thread_launch(self, d, classes):
        """depth d is a class split at the product thresholds, and each of `classes` gets its own thread-per-node kernel"""
        assert self.count(d) > WARP_LEVEL_MAX, (d, self.count(d))
        for c in classes:
            assert self.count(d, c) > CLASS_WARP_MAX, (d, c, self.count(d, c))


def check_dispatch(census, names):
    got = launches(names)
    assert got == census.dispatch(launch_threshold())
    return got


# ---- key generators -----------------------------------------------------------------------------------------------------
def set_nibble(keys, pos, nib):
    rows = np.arange(len(keys))
    pos = np.broadcast_to(np.asarray(pos, np.int64), rows.shape)
    byte = pos // 2
    cur = keys[rows, byte]
    keys[rows, byte] = np.where(pos % 2 == 0, (cur & 0x0F) | (nib << 4), (cur & 0xF0) | nib).astype(np.uint8)


def fan_out(rng, keys, pos, counts):
    """Row i of keys becomes counts[i] rows that differ only in nibble pos[i] (distinct random nibbles): a branch node at
    depth pos[i] when counts[i] > 1.  -> (rows, index of the parent row of each)."""
    counts = np.broadcast_to(np.asarray(counts, np.int64), (len(keys),))
    pos = np.broadcast_to(np.asarray(pos, np.int64), (len(keys),))
    order = np.argsort(rng.random((len(keys), 16)), axis=1)
    parent = np.repeat(np.arange(len(keys)), counts)
    out = keys[parent]
    set_nibble(out, pos[parent], order[np.arange(16)[None, :] < counts[:, None]].astype(np.uint8))
    return out, parent


def random_rows(rng, n):
    return rng.integers(0, 256, (n, 32), dtype=np.uint8)


def class_sizes(rng, cls):
    return rng.integers(CLASS_LO[cls], CLASS_HI[cls])


def big_values(rng, n):
    """full 32-byte slot values: every leaf is hashed in its branch"""
    v = random_rows(rng, n)
    v[:, 0] |= 1
    return v


def small_values(rng, n):
    """values < 0x80, < 0x100 or < 0x10000: leaves of 3, 5 or 6 bytes when their path is at most one nibble"""
    x = rng.integers(1, np.array([0x80, 0x100, 0x10000])[rng.integers(0, 3, n)])
    v = np.zeros((n, 32), np.uint8)
    v[:, 30], v[:, 31] = x >> 8, x & 0xFF
    return v


def forest(keys, seg, *rows):
    """sort by (trie, key) -> (keys, seg_offsets, rows...)"""
    v = keys.view(">u8")
    o = np.lexsort((v[:, 3], v[:, 2], v[:, 1], v[:, 0], seg))
    offs = np.zeros(int(seg.max()) + 2, np.uint64)
    offs[1:] = np.cumsum(np.bincount(seg))
    return (keys[o], offs) + tuple(r[o] for r in rows)


def clustered_forest(rng, per_class):
    """4 * per_class storage tries.  Each is one depth-62 branch (behind its root extension of 62 nibbles) with a cluster
    of 2..16 slots that differ only in their last nibble and one or two lone slots; every value is small.  The clusters are
    depth-63 branches of inline leaves, per_class of them in each child-count class; the small ones are inline themselves,
    so their depth-62 parent has an inline branch child under a hash-mask bit."""
    t = 4 * per_class
    k = class_sizes(rng, np.repeat(np.arange(4), per_class))
    kids, tr = fan_out(rng, random_rows(rng, t), 62, rng.integers(2, 4, t))
    cluster = np.r_[True, tr[1:] != tr[:-1]]
    leaves, p = fan_out(rng, kids, 63, np.where(cluster, k[tr], 1))
    return forest(leaves, tr[p], small_values(rng, len(leaves)))


# ---- a. inline children in every class ----------------------------------------------------------------------------------
def test_inline_children_in_every_class(timed, capfd):
    rng = np.random.default_rng(801)
    keys, offs, vals = clustered_forest(rng, 1100)
    c = Census(keys, offs)
    c.assert_thread_launch(63, range(4))
    c.assert_thread_launch(62, [0])
    assert (c.root == (c.depth == 62)).all() and c.wrapped[c.root].all()     # every root: a 62-nibble extension
    (roots, stats), names = with_phases(capfd, lambda: timed.storage_roots(keys, vals, offs, want_stats=True))
    assert set(BIG) <= set(check_dispatch(c, names))
    oracle.stats_reset()
    assert (roots == oracle.storage_roots(keys, vals, offs)).all()
    want = oracle.stats()
    assert want["branch_nodes"] == len(c.depth) == stats["branches_added"]
    assert want["extension_nodes"] == int(c.wrapped.sum()) == stats["extension_nodes"]
    assert stats["hashed_nodes"] == want["hashed_nodes"]


# ---- b. the same keys with updates retained -----------------------------------------------------------------------------
def test_inline_branch_child_with_updates_is_an_error_and_the_context_recovers(eng):
    """alloy-trie's HashBuilder panics on an inline branch child under a hash-mask bit (B200_ERR_INLINE_HASH_CHILD).  Here
    the only such children hang under the depth-62 nodes, all of which the thread kernel of class 2-3 builds.  The call
    that hits it reports the error; include/b200trie.h: reporting clears it, so the next calls on the context succeed."""
    from reth_b200 import B200Error, _lib
    rng = np.random.default_rng(801)
    keys, offs, vals = clustered_forest(rng, 1100)
    Census(keys, offs).assert_thread_launch(62, [0])
    with pytest.raises(B200Error) as e:
        eng.storage_roots(keys, vals, offs, want_updates=True)
    assert e.value.status == _lib.ERR_INLINE_HASH_CHILD
    want = oracle.storage_roots(keys, vals, offs)
    assert (eng.storage_roots(keys, vals, offs) == want).all()
    assert (eng.storage_roots(keys, vals, offs) == want).all()
    # and a build that retains updates, on the same context
    k2, o2, v2 = extension_forest(np.random.default_rng(5), 60, (3, 20))
    roots, upd = eng.storage_roots(k2, v2, o2, want_updates=True)
    o_roots, o_upd = oracle.storage_roots(k2, v2, o2, want_updates=True)
    assert (roots == o_roots).all()
    assert upd == o_upd


# ---- c. extensions of every length at big levels ------------------------------------------------------------------------
DEPTHS = (3, 6, 20, 40, 62)


def extension_forest(rng, per_class, depths, spread=False):
    """4 * per_class storage tries; each has one group of keys per depth d of `depths` (plus one at a random depth with
    spread), hanging from a depth-0 root.  A group is 2..16 keys that share their first d nibbles: a depth-d branch behind an
    extension of d - 1 nibbles.  All groups of a trie are of one child-count class, per_class tries per class."""
    t = 4 * per_class
    g = len(depths) + spread
    tops, tr = fan_out(rng, random_rows(rng, t), 0, g)
    gd = np.tile(np.array(depths + ((0,) if spread else ()), np.int64), t)
    if spread:
        gd[g - 1::g] = rng.integers(2, 63, t)
    leaves, p = fan_out(rng, tops, gd, class_sizes(rng, np.repeat(np.arange(4), per_class))[tr])
    return forest(leaves, tr[p], big_values(rng, len(leaves)))


def test_extensions_of_every_length_storage_forest(timed, capfd):
    rng = np.random.default_rng(802)
    keys, offs, vals = extension_forest(rng, 1100, DEPTHS, spread=True)
    c = Census(keys, offs)
    for d in DEPTHS:
        c.assert_thread_launch(d, range(4))
        assert c.wrapped[c.depth == d].all()
    c.assert_thread_launch(0, [1])
    assert set((c.depth - c.parent - 1)[c.wrapped]) == set(range(1, 62))   # every extension length
    (res, names) = with_phases(capfd, lambda: timed.storage_roots(keys, vals, offs, want_updates=True, want_stats=True))
    roots, upd, stats = res
    check_dispatch(c, names)
    oracle.stats_reset()
    o_roots, o_upd = oracle.storage_roots(keys, vals, offs, want_updates=True)
    want = oracle.stats()
    assert (roots == o_roots).all()
    assert upd == o_upd
    assert want["branch_nodes"] == len(c.depth) == stats["branches_added"]
    assert want["extension_nodes"] == int(c.wrapped.sum()) == stats["extension_nodes"]
    assert stats["hashed_nodes"] == want["hashed_nodes"]


def test_extensions_at_big_levels_account_trie(timed, capfd):
    rng = np.random.default_rng(803)
    depths = DEPTHS[1:]
    per = 1100
    gd = np.repeat(np.array(depths), 4 * per)
    cls = np.tile(np.repeat(np.arange(4), per), len(depths))
    keys, _ = fan_out(rng, random_rows(rng, len(gd)), gd, class_sizes(rng, cls))
    keys, _ = forest(keys, np.zeros(len(keys), np.int64))
    _, accs = synth_accounts(804, len(keys))
    sroots = random_rows(rng, len(keys))
    c = Census(keys)
    for d in depths:
        c.assert_thread_launch(d, range(4))
    assert c.wrapped[c.depth >= 20].all()
    (res, names) = with_phases(capfd, lambda: timed.state_root(keys, accs, sroots, want_updates=True, want_stats=True))
    root, upd, stats = res
    check_dispatch(c, names)
    oracle.stats_reset()
    o_root, o_upd = oracle.state_root(keys, accs, sroots, want_updates=True)
    want = oracle.stats()
    assert root == o_root
    assert upd == o_upd
    assert want["branch_nodes"] == len(c.depth) == stats["branches_added"]
    assert want["extension_nodes"] == int(c.wrapped.sum()) == stats["extension_nodes"]
    assert stats["hashed_nodes"] == want["hashed_nodes"]


# ---- d. the thresholds themselves -----------------------------------------------------------------------------------------
EDGE_LEVELS = {30: (1024, 1025, 1024, 1025),   # a big level of warp and thread launches in turn
               20: (1025, 1024, 1024, 1024),   # 4097 nodes: class split; 1025 -> thread kernel, 1024 -> warp kernel
               10: (1024, 1024, 1024, 1024)}   # exactly 4096 nodes: one warp per node
EDGE_LAUNCHES = ["small-class", "big<=7", "small-class", "big<=16", "big<=3", "small-class", "small-class", "small-class",
                 "small-level"]


@pytest.mark.parametrize("shape", ["storage_forest", "account_trie"])
def test_threshold_edges(timed, capfd, shape):
    rng = np.random.default_rng(805)
    gd = np.concatenate([np.full(sum(h), d) for d, h in EDGE_LEVELS.items()])
    cls = np.concatenate([np.repeat(np.arange(4), h) for h in EDGE_LEVELS.values()])
    keys, grp = fan_out(rng, random_rows(rng, len(gd)), gd, class_sizes(rng, cls))
    if shape == "storage_forest":          # one group per trie: only the group nodes are branches
        keys, offs, vals = forest(keys, grp, big_values(rng, len(keys)))
        c = Census(keys, offs)
        (res, names) = with_phases(capfd, lambda: timed.storage_roots(keys, vals, offs, want_updates=True, want_stats=True))
        (roots, upd, stats), (o_roots, o_upd) = res, oracle.storage_roots(keys, vals, offs, want_updates=True)
        assert (roots == o_roots).all()
        assert check_dispatch(c, names) == (EDGE_LAUNCHES if launch_threshold() == WARP_LEVEL_MAX else launches(names))
        assert len(c.depth) == sum(map(sum, EDGE_LEVELS.values()))
    else:                                  # all groups in one trie: shallow levels join them
        keys, _ = forest(keys, np.zeros(len(keys), np.int64))
        _, accs = synth_accounts(806, len(keys))
        c = Census(keys)
        (res, names) = with_phases(capfd, lambda: timed.state_root(keys, accs, want_updates=True, want_stats=True))
        (root, upd, stats), (o_root, o_upd) = res, oracle.state_root(keys, accs, want_updates=True)
        assert root == o_root
        got = check_dispatch(c, names)
        if launch_threshold() == WARP_LEVEL_MAX:
            assert got[:len(EDGE_LAUNCHES)] == EDGE_LAUNCHES
    assert upd == o_upd
    for d, h in EDGE_LEVELS.items():
        assert [c.count(d, k) for k in range(4)] == list(h)
    assert stats["branches_added"] == len(c.depth) and stats["extension_nodes"] == int(c.wrapped.sum())


# ---- e. more than one persistent wave -------------------------------------------------------------------------------------
def two_level_forest(rng, n_tries, cls, p_single=0.35, p_inline=0.3):
    """Storage tries of depth-62 branches with `cls`-class child counts over depth-63 leaves.  Most tries join two or three
    of them under a depth-61 root: those need no extension and, when all their leaves are hashed, take the fast path.  The
    others (p_single) are a lone depth-62 branch behind a 62-nibble root extension, and p_inline of the depth-62 branches
    get one small (inline) leaf: both take the strip path.  -> (keys, offs, vals, strip flag per depth-62 node in key
    order)"""
    n61 = np.where(rng.random(n_tries) < p_single, 1, rng.integers(2, 4, n_tries))
    mids, tr = fan_out(rng, random_rows(rng, n_tries), 61, n61)
    leaves, m = fan_out(rng, mids, 62, class_sizes(rng, np.full(len(mids), cls)))
    first = np.r_[True, m[1:] != m[:-1]]
    vals = big_values(rng, len(leaves))
    small = first & (rng.random(len(mids)) < p_inline)[m]
    vals[small] = small_values(rng, int(small.sum()))
    keys, offs, vals, small = forest(leaves, tr[m], vals, small)
    return keys, offs, vals, small


@pytest.mark.parametrize("cls,n_tries,wave_nodes", [(0, 110_000, 200_000), (3, 36_000, 60_000)])
def test_strip_and_fast_nodes_interleaved_across_persistent_waves(timed, capfd, cls, n_tries, wave_nodes):
    """A class-2-3 depth of more than 200 k nodes (branch3_pipelined_kernel keeps 4 CTAs of 128 threads per SM: about three
    grid strides on an H100) and a class-13-16 depth of more than one wave of branch_kernel<128,16>.  Strip-path nodes (an
    inline leaf, or a root extension) lie between fast ones in key order, so a thread meets both kinds across its strides
    and the pipelined kernel prefetches the next node from both arms."""
    rng = np.random.default_rng(807 + cls)
    keys, offs, vals, small = two_level_forest(rng, n_tries, cls)
    c = Census(keys, offs)
    c.assert_thread_launch(62, [cls])
    assert c.count(62, cls) == c.count(62) > wave_nodes
    at = np.nonzero(c.depth == 62)[0]
    at = at[np.argsort(c.first[at])]
    cs = np.r_[0, np.cumsum(small)]
    f, k = c.first[at], c.kids[at]
    strip = c.wrapped[at] | (cs[f + k] - cs[f] > 0)
    assert 0.3 < strip.mean() < 0.7 and (strip[1:] != strip[:-1]).mean() > 0.3
    (res, names) = with_phases(capfd, lambda: timed.storage_roots(keys, vals, offs, want_stats=True))
    roots, stats = res
    check_dispatch(c, names)
    oracle.stats_reset()
    assert (roots == oracle.storage_roots(keys, vals, offs)).all()
    want = oracle.stats()
    assert want["extension_nodes"] == int(c.wrapped.sum()) == stats["extension_nodes"]
    assert stats["hashed_nodes"] == want["hashed_nodes"]


# ---- f. ordered roots -----------------------------------------------------------------------------------------------------
def rlp_index(i):
    if i == 0:
        return b"\x80"
    if i < 0x80:
        return bytes([i])
    b = i.to_bytes((i.bit_length() + 7) // 8, "big")
    return bytes([0x80 + len(b)]) + b


def ordered_census(lists):
    """the census of the index-keyed tries of `lists`: keys RLP(index), zero-padded to 4 bytes, sorted per list"""
    rows, seg = [], []
    for li, items in enumerate(lists):
        ks = sorted(rlp_index(i) for i in range(len(items)))
        rows += [k.ljust(4, b"\0") for k in ks]
        seg += [li] * len(ks)
    keys = np.frombuffer(b"".join(rows), np.uint8).reshape(-1, 4)
    offs = np.zeros(len(lists) + 1, np.uint64)
    offs[1:] = np.cumsum([len(x) for x in lists])
    return Census(keys, offs)


def test_ordered_roots_of_tiny_items(timed, capfd):
    """Three lists of 66 000 tiny items: about 12 000 class-13-16 nodes at depth 5 over inline leaves.  2 000 lists of 300:
    depth 1.  5 000 lists of 2 or 3 one-byte items: a depth-0 level of class-2-3 roots whose children are all inline and
    whose RLP is shorter than 32 bytes; a root is hashed all the same."""
    tiny = lambda i: (i * 2654435761 % 251).to_bytes(1, "big") * (1 + i % 3)
    cases = [([[tiny(i + j) for i in range(66_000)] for j in range(3)], [(5, [3])]),
             ([[tiny(i + j) for i in range(300)] for j in range(2000)], [(1, [0, 3])]),
             ([[bytes([(j + i) % 0x7f + 1]) for i in range(2 + j % 2)] for j in range(5000)], [(0, [0])])]
    for lists, targets in cases:
        c = ordered_census(lists)
        for d, classes in targets:
            c.assert_thread_launch(d, classes)
        packed = oracle.pack_lists(lists)
        roots, names = with_phases(capfd, lambda: timed.ordered_roots(*packed))
        check_dispatch(c, names)
        assert (roots == oracle.ordered_roots(*packed)).all()
    assert c.root.sum() == 5000 and (c.depth[c.root] == 0).all()


# ---- g. the items fold ----------------------------------------------------------------------------------------------------
def test_items_fold_with_stored_hashes_at_a_big_level(timed, capfd):
    """root_from_items over a storage forest: depth-8 branches (4400 of them, every class) whose children mix leaves,
    stored hashes at the next nibble (with and without children_are_in_trie) and stored hashes deeper down, which the fold
    wraps in an extension.  The streams are built directly, sorted and prefix-free.  Reference: the oracle's HashBuilder
    fed the same add_leaf / add_branch stream, trie by trie."""
    rng = np.random.default_rng(808)
    per_class, d = 1100, 8
    tops, tr = fan_out(rng, random_rows(rng, 2 * per_class), 0, 2)     # two depth-8 branches per trie
    keys, g = fan_out(rng, tops, d, class_sizes(rng, np.repeat(np.arange(4), per_class)))
    n = len(keys)
    kind = rng.integers(0, 3, n)                  # 0 leaf, 1 hash at depth d + 1, 2 hash deeper
    nibs = np.where(kind == 0, 64, np.where(kind == 1, d + 1, d + 1 + rng.integers(1, 20, n))).astype(np.uint8)
    flags = ((kind != 0) & (rng.random(n) < 0.5)).astype(np.uint8)
    for i in np.nonzero(kind != 0)[0]:           # a path of nibs[i] nibbles, zero-padded
        p = int(nibs[i])
        keys[i, (p + 1) // 2:] = 0
        if p % 2:
            keys[i, p // 2] &= 0xF0
    vals = big_values(rng, n)
    keys, offs, nibs, flags, vals = forest(keys, tr[g], nibs, flags, vals)
    c = Census(keys, offs)
    c.assert_thread_launch(d, range(4))
    (res, names) = with_phases(capfd, lambda: timed.root_from_items(keys, nibs, flags, vals, None, offs, account=False,
                                                                    want_updates=True))
    roots, recs = res
    check_dispatch(c, names)
    got = {}
    for r in recs:
        got.setdefault(r[0], {})[bytes(r[1])] = (r[2], r[3], r[4], list(r[5]))
    for s in range(len(offs) - 1):
        hb = oracle.HashBuilder(retain_updates=True)
        for i in range(int(offs[s]), int(offs[s + 1])):
            path = oracle.unpack_nibbles(keys[i].tobytes())[:int(nibs[i])]
            if nibs[i] == 64:
                hb.add_leaf(path, oracle.encode_u256(int.from_bytes(vals[i].tobytes(), "big")))
            else:
                hb.add_branch(path, vals[i].tobytes(), bool(flags[i]))
        assert roots[s].tobytes() == hb.root(), s
        want = {p: (u["state_mask"], u["tree_mask"], u["hash_mask"], u["hashes"]) for p, u in hb.updates().items() if p != b""}
        assert got.get(s, {}) == want, s


# ---- h. a stateless batch -------------------------------------------------------------------------------------------------
def test_witness_roots_batch_folds_a_big_account_level(eng, timed, capfd):
    """witness_roots over 24 consecutive blocks (400 entries each) of a 20 000-account state, some of whose storage tries are clustered slots
    (inline leaves and branches): the account fold of the batch holds more than 4096 nodes at one depth.  Every root equals
    the oracle's from-scratch root of the post-block state; the twin DynamicState's apply gives the same."""
    rng = np.random.default_rng(809)
    state = random_state(rng, 20_000, with_storage=0.1, max_slots=10)
    for k in sorted(state)[::40]:
        state[k] = (state[k][0], clustered_slots(rng, int(rng.integers(1, 6))))
    ds = make_state(eng, state)
    parents, witnesses, blocks, wants = [], [], [], []
    for step in range(24):
        block = random_block(rng, state, 400, step + 1)
        arrays = block_arrays(block)
        parents.append(ds.root())
        witnesses.append(ds.witness(*arrays, mode="legacy" if step % 2 else "canonical"))
        twin = ds.apply(*arrays)
        state = apply_to_model(state, block)
        _, keys, accs, skeys, svals, offs = flatten(state)
        wants.append(oracle.state_root_full(keys, accs, skeys, svals, offs, threads=4))
        assert twin == wants[-1], step
        blocks.append(arrays)
    ds.close()
    (res, names) = with_phases(capfd, lambda: timed.witness_roots(parents, witnesses, blocks))
    roots, status = res
    assert [int(x) for x in status] == [0] * 24
    assert [r.tobytes() for r in roots] == wants
    after = names[names.index("stateless-storage") + 1:]
    assert any(x in BIG for x in launches(after)), after
