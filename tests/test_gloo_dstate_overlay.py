"""world_size-2 CPU test (gloo) of the overlay roots of a sharded dynamic state (ShardedDynamicStateRoot.overlay_roots):
every rank computes its frontier entries after each sibling post with its shard unchanged, the n x 16 entries are
all-gathered once and both ranks must arrive at the oracle's root of base + post, with root() unchanged; then one post is
committed and the overlay roots of new siblings are checked again.  The shards run on tools/emu's CPU emulation of the
CUDA sources (test-side redirection of the loader, as `pytest --emu` does); on GPUs the same class runs over NCCL."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "emu")


def _posts(seed):
    """deterministic base state, two batches of sibling posts (the first on base, the second after committing posts[0][0])"""
    from reth_b200 import Account, HashedPostState, HashedStorage
    rng = np.random.default_rng(seed)
    rk = lambda: bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    base = HashedPostState()
    for _ in range(250):
        k = rk()
        base.accounts[k] = Account(int(rng.integers(0, 9)), int(rng.integers(1, 2**60)))
        if rng.random() < 0.3:
            base.storages[k] = HashedStorage(False, {rk(): int(rng.integers(1, 2**60)) for _ in range(int(rng.integers(1, 12)))})
    live = sorted(base.accounts)

    def post(n_upd, n_new, n_kill):
        p = HashedPostState()
        for i in rng.choice(len(live), n_upd, replace=False):
            p.accounts[live[i]] = Account(7, int(rng.integers(1, 2**50)))
        for _ in range(n_new):
            k = rk()
            p.accounts[k] = Account(0, 1)
            p.storages[k] = HashedStorage(False, {rk(): 9})
        for i in rng.choice(len(live), n_kill, replace=False):
            if live[i] not in p.accounts:
                p.accounts[live[i]] = None
                p.storages[live[i]] = HashedStorage(True, {})
        return p

    first = [post(20, 5, 2), post(3, 0, 0), post(0, 0, 0), post(0, 4, 6)]
    second = [post(10, 3, 1), post(1, 1, 1)]
    return base, first, second


def _merge(state, post):
    from reth_b200 import HashedPostState, HashedStorage
    out = HashedPostState(dict(state.accounts), {k: HashedStorage(False, dict(v.storage)) for k, v in state.storages.items()})
    for k, hs in post.storages.items():
        cur = {} if hs.wiped else dict(out.storages.get(k, HashedStorage()).storage)
        for sk, v in hs.storage.items():
            if v == 0:
                cur.pop(sk, None)
            else:
                cur[sk] = v
        out.storages[k] = HashedStorage(False, cur)
    for k, a in post.accounts.items():
        if a is None:
            out.accounts.pop(k, None)
            out.storages.pop(k, None)
        else:
            out.accounts[k] = a
    return out


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), B200_EMU="1")
    from reth_b200 import _lib
    _lib.LIB_PATH = os.path.join(EMU, "build", "libb200trie_emu.so")   # test-side redirection only
    from reth_b200 import Engine, ShardedDynamicStateRoot
    dist.init_process_group("gloo", rank=rank, world_size=world)
    base, first, second = _posts(11)
    eng = Engine(0)
    sh = ShardedDynamicStateRoot(eng, base, rank, world)
    res = {"root0": sh.root().hex()}
    res["first"] = [r.hex() for r in sh.overlay_roots(first)]
    res["one"] = sh.overlay_root(first[3]).hex()
    res["root_after_overlay"] = sh.root().hex()
    res["commit"] = sh.commit(first[0])[0].hex()
    res["second"] = [r.hex() for r in sh.overlay_roots(second)]
    res["root_end"] = sh.root().hex()
    sh.close()
    with open(os.path.join(out_dir, f"rank_{rank}.json"), "w") as f:
        json.dump(res, f)
    dist.destroy_process_group()


def test_two_rank_sharded_overlay_roots(tmp_path):
    subprocess.run(["make", "-j8", "-C", EMU], check=True, capture_output=True)
    world = 2
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    r0 = json.load(open(tmp_path / "rank_0.json"))
    r1 = json.load(open(tmp_path / "rank_1.json"))
    assert r0 == r1
    import oracle
    base, first, second = _posts(11)

    def oracle_root(st):
        keys, accts, skeys, svals, offs = st.into_sorted().to_flat()
        return oracle.state_root_full(keys, accts, skeys, svals, offs).hex()

    assert r0["root0"] == r0["root_after_overlay"] == oracle_root(base)
    assert r0["first"] == [oracle_root(_merge(base, p)) for p in first]
    assert r0["first"][2] == r0["root0"]                                # an empty post keeps the root
    assert r0["one"] == r0["first"][3]
    committed = _merge(base, first[0])
    assert r0["commit"] == r0["first"][0] == r0["root_end"] == oracle_root(committed)
    assert r0["second"] == [oracle_root(_merge(committed, p)) for p in second]
