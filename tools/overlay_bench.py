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
give the same map and the overlay root.

    python tools/overlay_bench.py --shards 4

--shards S measures the overlay frontiers of a sharded state (b200_dstate_overlay_frontiers): the same state as S shards in
one process on one GPU (rank r owns top nibbles [16r/S, 16(r+1)/S), as reth_b200.sharded does), the first block split by
owner.  Alternating rep by rep: the overlay-frontiers call of every shard on its part of the block, each timed on its own;
the root from the merged frontier (b200_root_from_frontier); b200_dstate_overlay_roots of the whole block on the unsharded
state; and b200_dstate_apply on sharded twins, each shard timed on its own (the first rep applies the first block, every
later rep a fresh block of the same shape on top).  Reported per shard call: time, and their maximum (what S GPUs would
spend before the all-gather) and sum; launches and read-backs.  Checked in the run: the merged root equals the unsharded
overlay root and the twins' root after the block, and every shard keeps its root and frontier."""
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
    ap.add_argument("--shards", type=int, nargs="?", const=4, default=0,
                    help="measure the overlay frontiers of a state in this many shards (default 4; see above)")
    args = ap.parse_args()
    import torch

    from reth_b200 import DynamicState, Engine
    from reth_b200._lib import FrontierEntry, Proofs, Stats, Updates, Witness
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

    if args.shards:
        S = args.shards
        if not 1 <= S <= 16:
            raise SystemExit("--shards: 1 to 16")
        owner = lambda k: (k[:, 0].astype(np.int64) >> 4) * S // 16
        bounds = np.searchsorted(owner(keys), np.arange(S + 1))       # keys are sorted: every rank holds a run of them

        def state_part(r):
            lo, hi = int(bounds[r]), int(bounds[r + 1])
            so = offs[lo:hi + 1]
            return keys[lo:hi], accs[lo:hi], skeys[int(so[0]):int(so[-1])], svals[int(so[0]):int(so[-1])], so - so[0]

        def block_part(a, r):
            bb = np.searchsorted(owner(a[0]), np.arange(S + 1))
            lo, hi = int(bb[r]), int(bb[r + 1])
            so = np.asarray(a[5], np.uint64)[lo:hi + 1]
            return (a[0][lo:hi], a[1][lo:hi], a[2][lo:hi], a[3][int(so[0]):int(so[-1])], a[4][int(so[0]):int(so[-1])], so - so[0])
        shards = [DynamicState.create(eng, *state_part(r), sharded=True) for r in range(S)]
        twins = [DynamicState.create(eng, *state_part(r), sharded=True) for r in range(S)]
        pick = np.arange(16) * S // 16                                # owner of every bucket

        def merge(frs):
            return np.ascontiguousarray(np.stack(frs)[pick, np.arange(16)])
        shard_root0 = [(d.root(), d.frontier()) for d in shards]
        assert eng.root_from_frontier(merge([f for _, f in shard_root0])) == parent
        a0 = arrays[0]
        packed = [block_batch_arrays([block_part(a0, r)]) for r in range(S)]
        frs = [(FrontierEntry * 16)() for _ in range(S)]
        as_np = lambda fr: np.frombuffer(bytes(fr), np.uint8).reshape(16, 68)
        packed_u, roots = block_batch_arrays([a0]), np.zeros((1, 32), np.uint8)

        def frontiers(r):
            return lambda: eng._check(eng.lib.b200_dstate_overlay_frontiers(shards[r].handle, 1, *(_ptr(x) for x in packed[r]), frs[r],
                                                                            C.byref(Stats())))

        def merged_root():
            return eng.root_from_frontier(merge([as_np(f) for f in frs]))

        def overlay_root():
            eng._check(eng.lib.b200_dstate_overlay_roots(ds.handle, 1, *(_ptr(x) for x in packed_u), _ptr(roots), C.byref(Stats())))
        chain = iter([a0] + [block_arrays(make_block(rng, keys, skeys, offs, args.touch, args.slot_writes))
                             for _ in range(args.warmup + args.reps + 1)])
        root = np.zeros(32, np.uint8)

        def twin_apply(r):
            def call():
                a = cur[r]
                eng._check(eng.lib.b200_dstate_apply(twins[r].handle, _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), len(a[0]), _ptr(a[3]),
                                                     _ptr(a[4]), _ptr(a[5]), _ptr(root), None, None, None, None, None, C.byref(Stats())))
            return call
        # ---- the cross-checks: merged overlay root == unsharded overlay root == the twins' root after the block
        for r in range(S):
            frontiers(r)()
        overlay_root()
        a = next(chain)
        cur = [block_part(a, r) for r in range(S)]
        for r in range(S):
            twin_apply(r)()
        twin_root = eng.root_from_frontier(merge([t.frontier() for t in twins]))
        assert merged_root() == roots[0].tobytes() == twin_root, "merged overlay root differs"
        assert [as_np(f).tobytes() for f in frs] == [t.frontier().tobytes() for t in twins], "overlay frontier differs from the apply"
        # ---- counts of one call each
        res = {"overlay_frontiers": [counts(frontiers(r)) for r in range(S)], "root_from_frontier": counts(merged_root),
               "overlay_roots_unsharded": counts(overlay_root)}
        # ---- timed, alternating rep by rep (warm-ups included in the same loop)
        t = {"overlay_frontiers": [[] for _ in range(S)], "root_from_frontier": [], "overlay_roots_unsharded": [],
             "apply_twins": [[] for _ in range(S)]}
        host_t = {k: [] for k in ("overlay_frontiers", "root_from_frontier", "overlay_roots_unsharded", "apply_twins")}

        def timed(call):
            torch.cuda.synchronize()
            ev0.record(stream)
            t0 = time.perf_counter()
            call()
            h = (time.perf_counter() - t0) * 1e3
            ev1.record(stream)
            ev1.synchronize()
            return ev0.elapsed_time(ev1), h
        apply_launches = []
        for rep in range(args.warmup + args.reps):
            keep = rep >= args.warmup
            hs = 0.0
            for r in range(S):
                d, h = timed(frontiers(r))
                hs += h
                if keep:
                    t["overlay_frontiers"][r].append(d)
            if keep:
                host_t["overlay_frontiers"].append(hs)
            for k, call in (("root_from_frontier", merged_root), ("overlay_roots_unsharded", overlay_root)):
                d, h = timed(call)
                if keep:
                    t[k].append(d)
                    host_t[k].append(h)
            a = next(chain)
            cur = [block_part(a, r) for r in range(S)]
            hs, l0 = 0.0, eng.launch_count()
            for r in range(S):
                d, h = timed(twin_apply(r))
                hs += h
                if keep:
                    t["apply_twins"][r].append(d)
            apply_launches.append(eng.launch_count() - l0)
            if keep:
                host_t["apply_twins"].append(hs)
        for d, (r0, f0) in zip(shards, shard_root0):
            assert d.root() == r0 and np.array_equal(d.frontier(), f0), "a shard changed"
        assert merged_root() == roots[0].tobytes()

        def per_shard(xs):
            xs = np.array(xs)                                          # [shard][rep]
            return {"per_shard_ms": [spread(x) for x in xs], "max_over_shards_ms": spread(xs.max(axis=0)),
                    "sum_over_shards_ms": spread(xs.sum(axis=0))}
        res["overlay_frontiers"] = dict(per_shard(t["overlay_frontiers"]), host_call_ms_all_shards=spread(host_t["overlay_frontiers"]),
                                        launches=[c["launches"] for c in res["overlay_frontiers"]],
                                        readbacks_dtoh=[c["readbacks_dtoh"] for c in res["overlay_frontiers"]],
                                        copies_htod=[c["copies_htod"] for c in res["overlay_frontiers"]])
        for k in ("root_from_frontier", "overlay_roots_unsharded"):
            res[k].update({"device_ms": spread(t[k]), "host_call_ms": spread(host_t[k])})
        res["apply_twins"] = dict(per_shard(t["apply_twins"]), host_call_ms_all_shards=spread(host_t["apply_twins"]),
                                  launches_all_shards=int(np.median(apply_launches)),
                                  note="every rep applies a fresh block of the same shape on top of the previous one")
        out.update(res)
        out["shards"] = S
        out["block_accounts_per_shard"] = [int(len(p[0])) for p in packed]
        mo = out["overlay_roots_unsharded"]["device_ms"]["median"]
        out["ratios"] = {"max_shard_over_unsharded_overlay": round(out["overlay_frontiers"]["max_over_shards_ms"]["median"] / mo, 2),
                         "sum_shards_over_unsharded_overlay": round(out["overlay_frontiers"]["sum_over_shards_ms"]["median"] / mo, 2),
                         "max_shard_overlay_over_max_shard_apply": round(out["overlay_frontiers"]["max_over_shards_ms"]["median"] /
                                                                         out["apply_twins"]["max_over_shards_ms"]["median"], 2)}
        out["card_after"] = card()
        print(json.dumps(out))
        for d in shards + twins + [ds]:
            d.close()
        eng.close()
        return

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
