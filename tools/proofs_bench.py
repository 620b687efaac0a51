#!/usr/bin/env python3
"""Cost of the multiproof of a sharded state (b200_dstate_sharded_multiproof: eth_getProof and the proof workers of the
state-root task over a state spread across GPUs), next to the multiproof of the same targets on one unsharded state.

    python -m pytest tests/test_gpu_sharded_proofs.py -m gpu -q     # correctness first
    python tools/proofs_bench.py --accounts 1000000 --slots 16 --targets 2000 --shards 4

Seeds the state of tools/witness_bench.py (--accounts accounts x --slots slots) once unsharded and once as --shards shards
on the same GPU, and takes --targets account targets (a twentieth of them absent) with every slot of the present ones.
Each target goes to the shard that owns its top nibble.  Alternating rep by rep, it times b200_dstate_multiproof of all
targets on the unsharded state and b200_dstate_sharded_multiproof of every shard's share, each call with its
b200_proofs_release.  CUDA-event time on the call's stream and host-call time, after warm-ups, median / min / max over
--reps; per shard, and the maximum and sum over the shards (the shards run one after another here; on one GPU per rank
they run side by side).  Kernel launches (b200_launch_count), device-to-host read-backs and host-to-device copies from a
separate torch.profiler run of one call.  Afterwards the merged dicts of the shards are checked against the unsharded
multiproof.  Reads the card's name, power limit and SM clock in the same run.  Prints one JSON line."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.stateless_bench import card, spread  # noqa: E402
from tools.witness_bench import make_state  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--targets", type=int, default=2000)
    ap.add_argument("--shards", type=int, default=4)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    S = args.shards
    if not 1 <= S <= 16:
        raise SystemExit("--shards: 1 to 16")
    import torch

    from reth_b200 import DynamicState, Engine
    from reth_b200._lib import FrontierEntry, Proofs
    from reth_b200.engine import _ptr
    out = {"card": card()}
    eng = Engine(0)
    keys, accs, skeys, svals, offs = make_state(np.random.default_rng(3), args.accounts, args.slots)
    ds = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    owner = lambda k: (k[:, 0].astype(np.int64) >> 4) * S // 16
    bounds = np.searchsorted(owner(keys), np.arange(S + 1))           # keys are sorted: every shard holds a run of them

    def state_part(r):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        so = offs[lo:hi + 1]
        return keys[lo:hi], accs[lo:hi], skeys[int(so[0]):int(so[-1])], svals[int(so[0]):int(so[-1])], so - so[0]
    shards = [DynamicState.create(eng, *state_part(r), sharded=True) for r in range(S)]
    merged = np.zeros((16, 68), np.uint8)
    hm = tm = 0
    for r, d in enumerate(shards):
        mine = [b for b in range(16) if b * S // 16 == r]
        merged[mine] = d.frontier()[mine]
        h, t = d.frontier_masks()
        hm, tm = hm | h, tm | t
    assert eng.root_from_frontier(merged) == ds.root()

    rng = np.random.default_rng(5)
    n_absent = args.targets // 20
    picks = rng.choice(len(keys), args.targets - n_absent, replace=False)
    targets = {keys[i].tobytes(): [skeys[j].tobytes() for j in range(int(offs[i]), int(offs[i + 1]))] for i in picks}
    for _ in range(n_absent):
        targets[rng.integers(0, 256, 32, dtype=np.uint8).tobytes()] = [rng.integers(0, 256, 32, dtype=np.uint8).tobytes()]
    shares = [{a: s for a, s in targets.items() if (a[0] >> 4) * S // 16 == r} for r in range(S)]
    out.update({"accounts": args.accounts, "slots": args.accounts * args.slots, "shards": S, "account_targets": len(targets),
                "slot_targets": sum(len(s) for s in targets.values()), "account_targets_per_shard": [len(s) for s in shares]})
    fr = (FrontierEntry * 16).from_buffer_copy(merged.tobytes())

    def call_of(target_set, sharded_on=None):
        _, ak, so, sk, _ = DynamicState._multiproof_targets(target_set)
        n = len(ak)
        sroots = np.zeros((max(n, 1), 32), np.uint8)

        def call():
            pa, ps = Proofs(), Proofs()
            if sharded_on is None:
                rc = eng.lib.b200_dstate_multiproof(ds.handle, _ptr(ak), n, _ptr(so), _ptr(sk), C.byref(pa), _ptr(sroots), C.byref(ps))
            else:
                rc = eng.lib.b200_dstate_sharded_multiproof(sharded_on.handle, fr, hm, tm, _ptr(ak), n, _ptr(so), _ptr(sk), C.byref(pa),
                                                            _ptr(sroots), C.byref(ps))
            eng._check(rc)
            eng.lib.b200_proofs_release(C.byref(pa))
            eng.lib.b200_proofs_release(C.byref(ps))
        return call
    calls = {"multiproof": call_of(targets)}
    for r in range(S):
        calls[f"shard_{r}"] = call_of(shares[r], shards[r])

    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for k, c in calls.items():
        l0 = eng.launch_count()
        c()
        launches = eng.launch_count() - l0
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            c()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        res[k] = {"launches": launches, "readbacks_dtoh": sum(1 for n in names if "DtoH" in n),
                  "copies_htod": sum(1 for n in names if "HtoD" in n)}
    for _ in range(args.warmup):
        for c in calls.values():
            c()
    dev, host = {k: [] for k in calls}, {k: [] for k in calls}
    for _ in range(args.reps):
        for k, c in calls.items():
            torch.cuda.synchronize()
            ev0.record(stream)
            t0 = time.perf_counter()
            c()
            host[k].append((time.perf_counter() - t0) * 1e3)
            ev1.record(stream)
            ev1.synchronize()
            dev[k].append(ev0.elapsed_time(ev1))
    out["multiproof"] = dict(res["multiproof"], device_ms=spread(dev["multiproof"]), host_call_ms=spread(host["multiproof"]))
    sd = np.array([dev[f"shard_{r}"] for r in range(S)])
    out["sharded_multiproof"] = {
        "per_shard": [dict(res[f"shard_{r}"], device_ms=spread(dev[f"shard_{r}"]), host_call_ms=spread(host[f"shard_{r}"]))
                      for r in range(S)],
        "max_over_shards_ms": spread(sd.max(axis=0)), "sum_over_shards_ms": spread(sd.sum(axis=0))}
    mo = out["multiproof"]["device_ms"]["median"]
    out["ratios"] = {"max_shard_over_unsharded": round(out["sharded_multiproof"]["max_over_shards_ms"]["median"] / mo, 2),
                     "sum_shards_over_unsharded": round(out["sharded_multiproof"]["sum_over_shards_ms"]["median"] / mo, 2)}
    got = {"account_subtree": {}, "branch_node_masks": {}, "storages": {}}
    for r in range(S):
        part = shards[r].sharded_multiproof(merged, hm, tm, shares[r])
        for name in got:
            got[name].update(part[name])
    out["matches_unsharded"] = got == ds.multiproof(targets)
    for d in shards + [ds]:
        d.close()
    eng.close()
    print(json.dumps(out))
    if not out["matches_unsharded"]:
        raise SystemExit("the merged sharded multiproof differs from the unsharded one")


if __name__ == "__main__":
    main()
