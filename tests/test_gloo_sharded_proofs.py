"""world_size-2 CPU test (gloo) of the multiproof of a sharded dynamic state (ShardedDynamicStateRoot.multiproof): both
ranks call it with the same targets and must both get the dict DynamicState.multiproof gives on an unsharded state of all
accounts, before and after a commit.  The shards run on tools/emu's CPU emulation of the CUDA sources (test-side
redirection of the loader, as `pytest --emu` does); on GPUs the same class runs over NCCL."""
import os
import pickle
import socket
import subprocess
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_gloo_dstate_overlay import EMU, ROOT, _posts


def _targets(base, seed):
    """present accounts with present and absent slots, accounts without slot targets, absent accounts with slots"""
    rng = np.random.default_rng(seed)
    rk = lambda: bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    live = sorted(base.accounts)
    t = {}
    for i in rng.choice(len(live), 30, replace=False):
        k = live[i]
        t[k] = sorted(base.storages[k].storage)[:2] + [rk()] if k in base.storages else []
    for _ in range(8):
        t[rk()] = [rk()]
    return t


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), B200_EMU="1")
    from reth_b200 import _lib
    _lib.LIB_PATH = os.path.join(EMU, "build", "libb200trie_emu.so")   # test-side redirection only
    from reth_b200 import DynamicStateRoot, Engine, ShardedDynamicStateRoot
    dist.init_process_group("gloo", rank=rank, world_size=world)
    base, first, _ = _posts(11)
    targets = _targets(base, 12)
    eng = Engine(0)
    sh = ShardedDynamicStateRoot(eng, base, rank, world)
    full = DynamicStateRoot(eng, base.into_sorted())
    res = {"before": (sh.multiproof(targets), full.ds.multiproof(targets))}
    sh.commit(first[0])
    full.commit(first[0])
    res["after"] = (sh.multiproof(targets), full.ds.multiproof(targets))
    sh.close()
    full.close()
    with open(os.path.join(out_dir, f"rank_{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    dist.destroy_process_group()


def test_two_rank_sharded_multiproof(tmp_path):
    subprocess.run(["make", "-j8", "-C", EMU], check=True, capture_output=True)
    world = 2
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    r0 = pickle.load(open(tmp_path / "rank_0.pkl", "rb"))
    r1 = pickle.load(open(tmp_path / "rank_1.pkl", "rb"))
    for when in ("before", "after"):
        sharded0, full = r0[when]
        assert sharded0 == full and r1[when][0] == full, when
        assert full["account_subtree"] and any(s["subtree"] for s in full["storages"].values())
    assert r0["before"][1] != r0["after"][1]
