#!/usr/bin/env python3
"""Cost of post-block roots of candidate blocks on top of the resident state (b200_dstate_overlay_roots), against the routes
it replaces, on the C3-shaped state.

    python -m pytest tests/test_gpu_overlay.py -m gpu -q      # correctness first
    python tools/overlay_bench.py --accounts 1000000 --slots 16 --touch 2000 --siblings 16

Seeds the state of tools/witness_bench.py (--accounts accounts x --slots slots) as a resident b200_dstate and makes
--siblings blocks of its 2 000-account shape, all on that one parent.  Times, with the state unchanged: the overlay of the
first block; the overlay of all siblings in one call; b200_dstate_witness (Legacy) + b200_witness_roots of the first block.
Then times b200_dstate_apply over a chain of fresh blocks of the same shape (an apply changes the state, so every rep
applies a new block); the first apply is the first sibling, and its root must equal the overlay's.  Every sibling's overlay
root must equal its witness_roots root on the unchanged state.  CUDA-event time on the call's stream and host-call time
of the C ABI call alone (inputs packed beforehand), after warm-ups, median / min / max over --reps.  Counts per call:
kernel launches (b200_launch_count), device-to-host read-backs and host-to-device copies from a separate torch.profiler
run of one call.  Reads the card's name, power limit and SM clock in the same run.  Prints one JSON line.

    python tools/overlay_bench.py --updates

--updates measures the TrieUpdates instead (b200_dstate_overlay_roots_with_updates): the root-only overlay of the first block
and of all siblings, each alternating rep by rep with the with-updates call of the same blocks, then b200_dstate_apply with
updates over a chain of fresh blocks of the same shape.  Each with its time, launches, read-backs and record count
(updated + removed records of both tries).

    python tools/overlay_bench.py --proofs

--proofs measures the overlay multiproof (b200_dstate_overlay_multiproof) of the first block, alternating rep by rep: with
the block's accounts and their written slots as targets (what the proof workers ask for); with --touch untouched accounts
as targets; b200_dstate_multiproof of those untouched targets on the resident state; and b200_dstate_overlay_roots of the
block.  Each with its time, launches, read-backs and proof node count (account + storage proofs).

    python tools/overlay_bench.py --witness

--witness measures the overlay witness (b200_dstate_overlay_witness, Legacy): the first block is the overlay, and the target
is a second block of the same shape on top of it.  Alternating rep by rep: the overlay witness; b200_dstate_overlay_roots of
the overlay block; b200_dstate_witness of the target block on the resident state.  Each with its time, launches, read-backs
and node count.  Afterwards the overlay block is applied, and b200_dstate_witness of the target on the changed state must
give the same map and the overlay root."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--touch", type=int, default=2000)
    ap.add_argument("--slot-writes", type=int, default=10)
    ap.add_argument("--siblings", type=int, default=16)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--updates", action="store_true", help="measure the overlay with TrieUpdates (see above)")
    ap.add_argument("--proofs", action="store_true", help="measure the overlay multiproof (see above)")
    ap.add_argument("--witness", action="store_true", help="measure the overlay witness (see above)")
    args = ap.parse_args()
    import torch

    from reth_b200 import DynamicState, Engine
    from reth_b200._lib import Proofs, Stats, Updates, Witness
    from reth_b200.engine import _ptr, block_batch_arrays, witness_batch_arrays
    out = {"card": card()}
    eng = Engine(0)
    keys, accs, skeys, svals, offs = make_state(np.random.default_rng(3), args.accounts, args.slots)
    ds = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    parent = ds.root()
    rng = np.random.default_rng(77)
    arrays = [block_arrays(make_block(rng, keys, skeys, offs, args.touch, args.slot_writes)) for _ in range(args.siblings)]
    out.update({"accounts": args.accounts, "slots": args.accounts * args.slots, "block_accounts": len(arrays[0][0]),
                "block_slot_entries": len(arrays[0][3]), "siblings": args.siblings})
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def measure(call, reps=args.reps, before=None):
        l0 = eng.launch_count()
        if before:
            before()
        call()
        launches = eng.launch_count() - l0
        for _ in range(args.warmup):
            if before:
                before()
            call()
        dev, host = [], []
        for _ in range(reps):
            if before:
                before()
            torch.cuda.synchronize()
            ev0.record(stream)
            t0 = time.perf_counter()
            call()
            host.append((time.perf_counter() - t0) * 1e3)
            ev1.record(stream)
            ev1.synchronize()
            dev.append(ev0.elapsed_time(ev1))
        from torch.profiler import ProfilerActivity, profile
        if before:
            before()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        return {"device_ms": spread(dev), "host_call_ms": spread(host), "launches": launches,
                "readbacks_dtoh": sum(1 for n in names if "DtoH" in n), "copies_htod": sum(1 for n in names if "HtoD" in n)}

    def counts(call):
        """launches, then device-to-host read-backs and host-to-device copies from a torch.profiler run of one call"""
        l0 = eng.launch_count()
        call()
        launches = eng.launch_count() - l0
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        return {"launches": launches, "readbacks_dtoh": sum(1 for n in names if "DtoH" in n),
                "copies_htod": sum(1 for n in names if "HtoD" in n)}

    def alternating(calls):
        """{name: call}: warmed up, then timed rep by rep in turn, so that both see the same machine"""
        res = {k: counts(c) for k, c in calls.items()}
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
        for k in calls:
            res[k].update({"device_ms": spread(dev[k]), "host_call_ms": spread(host[k])})
        return res

    if args.proofs:
        a0 = arrays[0]
        m = len(a0[0])
        block_keys = {a0[0][i].tobytes() for i in range(m)}
        # the block's accounts with their written slots; untouched resident accounts (no slot targets)
        written = (a0[0], np.asarray(a0[5], np.uint64), a0[3])
        picks = np.sort(rng.choice(len(keys), 2 * args.touch, replace=False))
        untouched = np.ascontiguousarray(np.stack([keys[i] for i in picks if keys[i].tobytes() not in block_keys][:args.touch]))
        plain = (untouched, np.zeros(len(untouched) + 1, np.uint64), np.zeros((0, 32), np.uint8))
        root = np.zeros(32, np.uint8)
        roots = np.zeros((1, 32), np.uint8)
        nodes = {}

        def take(name, pa, ps):
            nodes[name] = int(pa.n_nodes) + int(ps.n_nodes)
            eng.lib.b200_proofs_release(C.byref(pa))
            eng.lib.b200_proofs_release(C.byref(ps))

        def overlay_proof(name, tg):
            tk, to, ts = tg
            sroots = np.zeros((max(len(tk), 1), 32), np.uint8)

            def call():
                pa, ps = Proofs(), Proofs()
                eng._check(eng.lib.b200_dstate_overlay_multiproof(
                    ds.handle, *(_ptr(x) for x in a0[:3]), m, *(_ptr(x) for x in a0[3:]), _ptr(tk), len(tk), _ptr(to), _ptr(ts),
                    _ptr(root), C.byref(pa), _ptr(sroots), C.byref(ps), C.byref(Stats())))
                take(name, pa, ps)
            return call

        def resident_proof():
            pa, ps = Proofs(), Proofs()
            sroots = np.zeros((len(untouched), 32), np.uint8)
            eng._check(eng.lib.b200_dstate_multiproof(ds.handle, _ptr(plain[0]), len(plain[0]), _ptr(plain[1]), _ptr(plain[2]),
                                                      C.byref(pa), _ptr(sroots), C.byref(ps)))
            take("resident_multiproof_untouched", pa, ps)

        packed = block_batch_arrays(arrays[:1])

        def overlay_root():
            eng._check(eng.lib.b200_dstate_overlay_roots(ds.handle, 1, *(_ptr(x) for x in packed), _ptr(roots), C.byref(Stats())))
        calls = {"overlay_multiproof_block_targets": overlay_proof("overlay_multiproof_block_targets", written),
                 "overlay_multiproof_untouched": overlay_proof("overlay_multiproof_untouched", plain),
                 "resident_multiproof_untouched": resident_proof, "overlay_roots": overlay_root}
        res = alternating(calls)
        for k in res:
            res[k]["proof_nodes"] = nodes.get(k)
        out.update(res)
        out["targets"] = {"block_accounts": m, "block_written_slots": int(len(a0[3])), "untouched_accounts": len(untouched)}
        assert root.tobytes() == roots[0].tobytes() and ds.root() == parent
        mo = out["overlay_roots"]["device_ms"]["median"]
        out["ratios"] = {k + "_over_overlay_roots": round(out[k]["device_ms"]["median"] / mo, 2)
                         for k in ("overlay_multiproof_block_targets", "overlay_multiproof_untouched", "resident_multiproof_untouched")}
        out["card_after"] = card()
        print(json.dumps(out))
        ds.close()
        eng.close()
        return

    if args.witness:
        a0 = arrays[0]
        tg = block_arrays(make_block(rng, keys, skeys, offs, args.touch, args.slot_writes))
        packed = block_batch_arrays(arrays[:1])
        root, roots = np.zeros(32, np.uint8), np.zeros((1, 32), np.uint8)
        nodes = {}

        def keep(name, w):
            nodes[name] = int(w.n)
            eng.lib.b200_witness_release(C.byref(w))

        def overlay_witness():
            w = Witness()
            eng._check(eng.lib.b200_dstate_overlay_witness(ds.handle, *(_ptr(x) for x in a0[:3]), len(a0[0]), *(_ptr(x) for x in a0[3:]),
                                                           *(_ptr(x) for x in tg[:3]), len(tg[0]), *(_ptr(x) for x in tg[3:]), 0, 0,
                                                           _ptr(root), C.byref(w), C.byref(Stats())))
            keep("overlay_witness", w)

        def overlay_root():
            eng._check(eng.lib.b200_dstate_overlay_roots(ds.handle, 1, *(_ptr(x) for x in packed), _ptr(roots), C.byref(Stats())))

        def resident_witness():
            w = Witness()
            eng._check(eng.lib.b200_dstate_witness(ds.handle, *(_ptr(x) for x in tg[:3]), len(tg[0]), *(_ptr(x) for x in tg[3:]), 0, 0,
                                                   C.byref(w)))
            keep("resident_witness", w)
        res = alternating({"overlay_witness": overlay_witness, "overlay_roots": overlay_root, "resident_witness": resident_witness})
        for k in res:
            res[k]["witness_nodes"] = nodes.get(k)
        out.update(res)
        out["target"] = {"block_accounts": int(len(tg[0])), "block_slot_entries": int(len(tg[3]))}
        assert root.tobytes() == roots[0].tobytes() and ds.root() == parent
        ov_root, got = ds.overlay_witness(a0, tg, mode="legacy")
        assert len(got) == nodes["overlay_witness"] and ov_root == root.tobytes()
        assert ds.apply(*a0) == ov_root
        assert got == ds.witness(*tg, mode="legacy"), "overlay witness differs from apply + witness"
        mo = out["overlay_roots"]["device_ms"]["median"]
        out["ratios"] = {k + "_over_overlay_roots": round(out[k]["device_ms"]["median"] / mo, 2) for k in ("overlay_witness", "resident_witness")}
        out["card_after"] = card()
        print(json.dumps(out))
        ds.close()
        eng.close()
        return

    if args.updates:
        def overlay_calls(nb):
            packed = block_batch_arrays(arrays[:nb])
            roots = np.zeros((nb, 32), np.uint8)
            deleted = np.zeros(max(len(packed[0]), 1), np.uint8)
            recs = {}

            def root_only():
                eng._check(eng.lib.b200_dstate_overlay_roots(ds.handle, nb, *(_ptr(x) for x in packed), _ptr(roots), C.byref(Stats())))

            def with_updates():
                us = [Updates() for _ in range(4)]
                eng._check(eng.lib.b200_dstate_overlay_roots_with_updates(ds.handle, nb, *(_ptr(x) for x in packed), _ptr(roots),
                                                                          *(C.byref(u) for u in us), _ptr(deleted), C.byref(Stats())))
                recs["records"] = [int(u.n_nodes) for u in us]
                for u in us:
                    eng.lib.b200_updates_release(C.byref(u))
            r = alternating({"root_only": root_only, "with_updates": with_updates})
            r["with_updates"]["records"] = dict(zip(["acct_updated", "acct_removed", "storage_updated", "storage_removed"],
                                                    recs["records"]))
            r["with_updates"]["records"]["total"] = sum(recs["records"])
            r["blocks"] = nb
            return r
        out["overlay_one"] = overlay_calls(1)
        out["overlay_batch"] = overlay_calls(args.siblings)
        assert ds.root() == parent
        chain = iter(block_arrays(make_block(rng, keys, skeys, offs, args.touch, args.slot_writes))
                     for _ in range(args.warmup + args.reps + 4))
        cur, recs = {}, {}
        root = np.zeros(32, np.uint8)

        def apply_updates():
            a = cur["a"]
            us = [Updates() for _ in range(4)]
            deleted = np.zeros(max(len(a[0]), 1), np.uint8)
            eng._check(eng.lib.b200_dstate_apply(ds.handle, _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), len(a[0]), _ptr(a[3]), _ptr(a[4]),
                                                 _ptr(a[5]), _ptr(root), *(C.byref(u) for u in us), _ptr(deleted), C.byref(Stats())))
            recs["records"] = sum(int(u.n_nodes) for u in us)
            for u in us:
                eng.lib.b200_updates_release(C.byref(u))
        out["apply_with_updates_chain"] = measure(apply_updates, before=lambda: cur.__setitem__("a", next(chain)))
        out["apply_with_updates_chain"]["records"] = recs["records"]
        out["apply_with_updates_chain"]["note"] = "every rep applies a fresh block of the same shape on top of the previous one"
        o1 = out["overlay_one"]["with_updates"]["device_ms"]["median"]
        out["ratios"] = {"updates_over_root_only_one": round(o1 / out["overlay_one"]["root_only"]["device_ms"]["median"], 2),
                         "updates_over_root_only_batch": round(out["overlay_batch"]["with_updates"]["device_ms"]["median"] /
                                                               out["overlay_batch"]["root_only"]["device_ms"]["median"], 2),
                         "overlay_updates_over_apply_updates": round(o1 / out["apply_with_updates_chain"]["device_ms"]["median"], 2)}
        out["card_after"] = card()
        print(json.dumps(out))
        ds.close()
        eng.close()
        return

    # ---- overlay: one block, then every sibling in one call
    def overlay_case(nb):
        packed = block_batch_arrays(arrays[:nb])
        roots = np.zeros((nb, 32), np.uint8)
        s = Stats()

        def call():
            eng._check(eng.lib.b200_dstate_overlay_roots(ds.handle, nb, *(_ptr(x) for x in packed), _ptr(roots), C.byref(s)))
        r = measure(call)
        r["blocks"] = nb
        r["host_call_ms_per_block"] = round(r["host_call_ms"]["median"] / nb, 3)
        return r, [x.tobytes() for x in roots]

    out["overlay_one"], one_root = overlay_case(1)
    out["overlay_batch"], batch_roots = overlay_case(args.siblings)
    assert batch_roots[0] == one_root[0] and ds.root() == parent

    # ---- the read-only route it replaces: witness, then witness_roots, of the first block
    a0 = arrays[0]
    wit_roots = []
    for a in arrays:
        w = ds.witness(*a, mode="legacy")
        r, st = eng.witness_roots([parent], [w], [a])
        assert int(st[0]) == 0
        wit_roots.append(r[0].tobytes())
    assert wit_roots == batch_roots, "overlay root differs from the witness_roots root"
    w0 = ds.witness(*a0, mode="legacy")
    packed_w = witness_batch_arrays([parent], [w0], [a0])
    roots_w, status_w = np.zeros((1, 32), np.uint8), np.zeros(1, np.int32)

    def witness_route():
        w = Witness()
        eng._check(eng.lib.b200_dstate_witness(ds.handle, _ptr(a0[0]), _ptr(a0[1]), _ptr(a0[2]), len(a0[0]), _ptr(a0[3]),
                                               _ptr(a0[4]), _ptr(a0[5]), 0, 0, C.byref(w)))
        eng.lib.b200_witness_release(C.byref(w))  # (the witness reaches the host: a caller would pass it on as it is)
        eng._check(eng.lib.b200_witness_roots(eng.ctx, 1, *(_ptr(x) for x in packed_w[1:]), _ptr(roots_w), _ptr(status_w),
                                              C.byref(Stats())))
    out["witness_plus_witness_roots"] = measure(witness_route)
    assert roots_w[0].tobytes() == one_root[0] and ds.root() == parent

    # ---- apply: the first sibling, then a chain of fresh blocks of the same shape
    root0 = ds.apply(*a0)
    assert root0 == one_root[0], "overlay root differs from the apply"
    chain = iter(block_arrays(make_block(rng, keys, skeys, offs, args.touch, args.slot_writes))
                 for _ in range(args.warmup + args.reps + 2))
    cur = {}
    root = np.zeros(32, np.uint8)

    def next_block():
        cur["a"] = next(chain)

    def apply_call():
        a = cur["a"]
        eng._check(eng.lib.b200_dstate_apply(ds.handle, _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), len(a[0]), _ptr(a[3]), _ptr(a[4]),
                                             _ptr(a[5]), _ptr(root), None, None, None, None, None, C.byref(Stats())))
    out["apply_chain"] = measure(apply_call, before=next_block)
    out["apply_chain"]["note"] = "every rep applies a fresh block of the same shape on top of the previous one"
    o1, ob = out["overlay_one"]["device_ms"]["median"], out["overlay_batch"]["device_ms"]["median"]
    out["ratios"] = {"witness_route_over_overlay": round(out["witness_plus_witness_roots"]["device_ms"]["median"] / o1, 2),
                     "batch_over_one": round(ob / o1, 2),
                     "overlay_over_apply": round(o1 / out["apply_chain"]["device_ms"]["median"], 2)}
    out["card_after"] = card()
    print(json.dumps(out))
    ds.close()
    eng.close()


if __name__ == "__main__":
    main()
