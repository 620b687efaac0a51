#!/usr/bin/env python3
"""Cost of the trie changesets of a block from the resident state (b200_dstate_trie_changesets; reth's
compute_trie_changesets, which the payload validator runs for every block), next to the calls around it on the live path.

    python -m pytest tests/test_gpu_trie_changesets.py -m gpu -q     # correctness first
    python tools/changesets_bench.py --accounts 1000000 --slots 16 --touch 2000

Seeds the state of tools/witness_bench.py (--accounts accounts x --slots slots) as a resident b200_dstate, and a twin of it,
and makes one block of the 2 000-account shape of tools/overlay_bench.py.  Alternating rep by rep, it times:
  - overlay_with_updates : b200_dstate_overlay_roots_with_updates of the block (its TrieUpdates);
  - trie_changesets      : b200_dstate_trie_changesets of those updates (their paths and is_deleted flags);
  - apply_twin           : b200_dstate_apply with updates on the twin, a fresh block of the same shape every rep (an apply
                           changes the state it runs on).
CUDA-event time on the call's stream and host-call time of the C ABI call alone (inputs packed beforehand), after warm-ups,
median / min / max over --reps; kernel launches (b200_launch_count), device-to-host read-backs and host-to-device copies
from a separate torch.profiler run of one call; record counts.  Afterwards the revert property is checked on the block: the
tables of the state (a full build with TrieUpdates) with the block's updates applied and the changesets written back are
the tables before the block, for the account trie and every storage trie the block touches.  Reads the card's name, power
limit and SM clock in the same run.  Prints one JSON line."""
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
from tools.witness_bench import block_arrays, make_block, make_state  # noqa: E402


def changeset_input(keys_sorted, res):
    """paths and is_deleted of one block's updates (the tuple of DynamicState.overlay_roots(..., want_updates=True))"""
    _, au, ar, su, sr, deleted = res
    per = {}
    for r in su:
        per.setdefault(r[0], set()).add(r[1])
    for e, p in sr:
        per.setdefault(e, set()).add(p)
    storage = {keys_sorted[i]: (bool(deleted[i]), sorted(per.get(i, ()))) for i in range(len(keys_sorted)) if deleted[i] or per.get(i)}
    return sorted({r[1] for r in au} | set(ar)), storage


def revert_holds(pre_adb, pre_sdb, keys_sorted, res, storage, changesets) -> bool:
    """tables after the block (removed, is_deleted, updated), then the changesets written back (a deleted trie cleared
    first, Some upserts, None deletes): equal to the tables before, on the account trie and the block's storage tries"""
    _, au, ar, su, sr, deleted = res
    adb, sdb = dict(pre_adb), {k: dict(pre_sdb.get(k, {})) for k in keys_sorted}
    for p in ar:
        adb.pop(p, None)
    for r in au:
        adb[r[1]] = tuple(r[2:5]) + (tuple(r[5]),)
    for e, p in sr:
        sdb[keys_sorted[e]].pop(p, None)
    for i, k in enumerate(keys_sorted):
        if deleted[i]:
            sdb[k] = {}
    for r in su:
        sdb[keys_sorted[r[0]]][r[1]] = tuple(r[2:5]) + (tuple(r[5]),)
    acct_cs, stor_cs = changesets
    for r in acct_cs:
        if r[2]:
            adb[r[1]] = tuple(r[2:5]) + (tuple(r[5]),)
        else:
            adb.pop(r[1], None)
    addrs = sorted(storage)
    for i in {r[0] for r in stor_cs}:
        if storage[addrs[i]][0]:
            sdb[addrs[i]] = {}
    for r in stor_cs:
        if r[2]:
            sdb[addrs[r[0]]][r[1]] = tuple(r[2:5]) + (tuple(r[5]),)
        else:
            sdb[addrs[r[0]]].pop(r[1], None)
    return adb == pre_adb and all(sdb[k] == pre_sdb.get(k, {}) for k in keys_sorted)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--touch", type=int, default=2000)
    ap.add_argument("--slot-writes", type=int, default=10)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    from reth_b200 import DynamicState, Engine
    from reth_b200._lib import Stats, Updates
    from reth_b200.engine import _pack_paths, _ptr, block_batch_arrays
    out = {"card": card()}
    eng = Engine(0)
    keys, accs, skeys, svals, offs = make_state(np.random.default_rng(3), args.accounts, args.slots)
    ds = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    twin = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    parent = ds.root()
    rng = np.random.default_rng(77)
    block = make_block(rng, keys, skeys, offs, args.touch, args.slot_writes)
    a0 = block_arrays(block)
    ks = sorted(block)
    out.update({"accounts": args.accounts, "slots": args.accounts * args.slots, "block_accounts": len(a0[0]),
                "block_slot_entries": len(a0[3])})
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    # the block's updates, and its changeset inputs packed once
    res = ds.overlay_roots([a0], want_updates=True)[0]
    acct_paths, storage = changeset_input(ks, res)
    alen, apk = _pack_paths(acct_paths)
    addrs = sorted(storage)
    skeys_cs = np.frombuffer(b"".join(addrs), np.uint8).reshape(len(addrs), 32) if addrs else np.zeros((0, 32), np.uint8)
    sflags = np.array([1 if storage[a][0] else 0 for a in addrs], np.uint8)
    spaths = [p for a in addrs for p in storage[a][1]]
    soffs = np.cumsum([0] + [len(storage[a][1]) for a in addrs]).astype(np.uint64)
    slen, spk = _pack_paths(spaths)
    packed = block_batch_arrays([a0])
    roots = np.zeros((1, 32), np.uint8)
    deleted = np.zeros(max(len(a0[0]), 1), np.uint8)
    recs = {}

    def overlay_with_updates():
        us = [Updates() for _ in range(4)]
        eng._check(eng.lib.b200_dstate_overlay_roots_with_updates(ds.handle, 1, *(_ptr(x) for x in packed), _ptr(roots),
                                                                  *(C.byref(u) for u in us), _ptr(deleted), C.byref(Stats())))
        recs["overlay_with_updates"] = sum(int(u.n_nodes) for u in us)
        for u in us:
            eng.lib.b200_updates_release(C.byref(u))

    def trie_changesets():
        au, su = Updates(), Updates()
        eng._check(eng.lib.b200_dstate_trie_changesets(ds.handle, _ptr(alen), _ptr(apk), len(alen), _ptr(skeys_cs), _ptr(sflags), len(addrs),
                                                       _ptr(soffs), _ptr(slen), _ptr(spk), C.byref(au), C.byref(su), C.byref(Stats())))
        recs["trie_changesets"] = {"account": int(au.n_nodes), "storage": int(su.n_nodes)}
        eng.lib.b200_updates_release(C.byref(au))
        eng.lib.b200_updates_release(C.byref(su))

    chain = iter(block_arrays(make_block(rng, keys, skeys, offs, args.touch, args.slot_writes)) for _ in range(args.warmup + args.reps + 4))
    cur = {}
    root = np.zeros(32, np.uint8)

    def apply_twin():
        a = cur["a"]
        us = [Updates() for _ in range(4)]
        dl = np.zeros(max(len(a[0]), 1), np.uint8)
        eng._check(eng.lib.b200_dstate_apply(twin.handle, _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), len(a[0]), _ptr(a[3]), _ptr(a[4]), _ptr(a[5]),
                                             _ptr(root), *(C.byref(u) for u in us), _ptr(dl), C.byref(Stats())))
        recs["apply_twin"] = sum(int(u.n_nodes) for u in us)
        for u in us:
            eng.lib.b200_updates_release(C.byref(u))
    calls = {"overlay_with_updates": (overlay_with_updates, None), "trie_changesets": (trie_changesets, None),
             "apply_twin": (apply_twin, lambda: cur.__setitem__("a", next(chain)))}

    from torch.profiler import ProfilerActivity, profile
    res_t = {}
    for k, (c, before) in calls.items():
        if before:
            before()
        l0 = eng.launch_count()
        c()
        launches = eng.launch_count() - l0
        if before:
            before()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            c()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        res_t[k] = {"launches": launches, "readbacks_dtoh": sum(1 for n in names if "DtoH" in n),
                    "copies_htod": sum(1 for n in names if "HtoD" in n)}
    for _ in range(args.warmup):
        for c, before in calls.values():
            if before:
                before()
            c()
    dev, host = {k: [] for k in calls}, {k: [] for k in calls}
    for _ in range(args.reps):
        for k, (c, before) in calls.items():
            if before:
                before()
            torch.cuda.synchronize()
            ev0.record(stream)
            t0 = time.perf_counter()
            c()
            host[k].append((time.perf_counter() - t0) * 1e3)
            ev1.record(stream)
            ev1.synchronize()
            dev[k].append(ev0.elapsed_time(ev1))
    for k in calls:
        res_t[k].update({"device_ms": spread(dev[k]), "host_call_ms": spread(host[k]), "records": recs[k]})
    res_t["apply_twin"]["note"] = "every rep applies a fresh block of the same shape on the twin, on top of the previous one"
    out.update(res_t)
    out["changeset_input"] = {"account_paths": len(acct_paths), "storage_tries": len(addrs), "deleted_tries": int(sflags.sum()),
                              "storage_paths": len(spaths)}
    assert ds.root() == parent and roots[0].tobytes() == res[0]
    # ---- the revert property on the block, against the tables of a full build of the state
    _, au, su = eng.state_root_full(keys, accs, skeys, svals, offs, want_updates=True)
    pre_adb = {r[1]: tuple(r[2:5]) + (tuple(r[5]),) for r in au}
    index = {keys[i].tobytes(): i for i in range(len(keys))}
    want = {index[k] for k in ks if k in index}
    pre_sdb = {}
    for r in su:
        if r[0] in want:
            pre_sdb.setdefault(keys[r[0]].tobytes(), {})[r[1]] = tuple(r[2:5]) + (tuple(r[5]),)
    cs = ds.trie_changesets(acct_paths, storage)
    out["revert_check"] = revert_holds(pre_adb, pre_sdb, ks, res, storage, cs)
    assert out["revert_check"], "the changesets do not revert the block's updates"
    mo = out["overlay_with_updates"]["device_ms"]["median"]
    out["ratios"] = {"changesets_over_overlay_with_updates": round(out["trie_changesets"]["device_ms"]["median"] / mo, 3),
                     "changesets_over_apply": round(out["trie_changesets"]["device_ms"]["median"] / out["apply_twin"]["device_ms"]["median"], 3)}
    out["card_after"] = card()
    print(json.dumps(out))
    ds.close()
    twin.close()
    eng.close()


if __name__ == "__main__":
    main()
