"""world_size-2 CPU test (gloo) of the execution witness of a sharded dynamic state (ShardedDynamicStateRoot.witness): both
ranks call it with the same post and must both get the map DynamicStateRoot.witness gives on an unsharded state of all
accounts, in both modes, before and after a commit.  The shards run on tools/emu's CPU emulation of the CUDA sources
(test-side redirection of the loader, as `pytest --emu` does); on GPUs the same class runs over NCCL."""
import os
import pickle
import socket
import subprocess
import sys

import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_gloo_dstate_overlay import EMU, ROOT, _posts


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), B200_EMU="1")
    from reth_b200 import _lib
    _lib.LIB_PATH = os.path.join(EMU, "build", "libb200trie_emu.so")   # test-side redirection only
    from reth_b200 import DynamicStateRoot, Engine, HashedPostState, HashedStorage, ShardedDynamicStateRoot
    from reth_b200.trie import StateRootError
    dist.init_process_group("gloo", rank=rank, world_size=world)
    base, first, second = _posts(17)
    # every account goes but those of bucket 0xF, which no entry touches: rank 1 owes the depth-0 reveal, decided by the
    # kept masks of both ranks
    keep_one = HashedPostState({k: None for k in base.accounts if k[0] >> 4 != 0xF},
                               {k: HashedStorage(True, {}) for k in base.storages if k[0] >> 4 != 0xF})
    eng = Engine(0)
    sh = ShardedDynamicStateRoot(eng, base, rank, world)
    full = DynamicStateRoot(eng, base.into_sorted())
    res = {}
    for name, post, always in (("before", first[0], False), ("empty", first[2], True), ("keep_one", keep_one, False)):
        for mode in ("legacy", "canonical"):
            res[name, mode] = (sh.witness(post, mode, always), full.witness(post, mode, always))
    missing = HashedPostState({}, {bytes(32): HashedStorage(False, {bytes(32): 1})})
    try:
        sh.witness(missing)
        res["missing"] = False
    except StateRootError:
        res["missing"] = True
    sh.commit(first[0])
    full.commit(first[0])
    for mode in ("legacy", "canonical"):
        res["after", mode] = (sh.witness(second[0], mode), full.witness(second[0], mode))
    sh.close()
    full.close()
    with open(os.path.join(out_dir, f"rank_{rank}.pkl"), "wb") as f:
        pickle.dump(res, f)
    dist.destroy_process_group()


def test_two_rank_sharded_witness(tmp_path):
    subprocess.run(["make", "-j8", "-C", EMU], check=True, capture_output=True)
    world = 2
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    r0 = pickle.load(open(tmp_path / "rank_0.pkl", "rb"))
    r1 = pickle.load(open(tmp_path / "rank_1.pkl", "rb"))
    assert r0["missing"] and r1["missing"]
    for key in [k for k in r0 if k != "missing"]:
        sharded0, full = r0[key]
        assert full and sharded0 == full and r1[key][0] == full, key
    assert r0["before", "legacy"][1] != r0["after", "legacy"][1]
    assert len(r0["empty", "legacy"][1]) == 1
    assert r0["keep_one", "legacy"][1] != r0["keep_one", "canonical"][1]
