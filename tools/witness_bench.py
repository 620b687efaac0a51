#!/usr/bin/env python3
"""Cost of the execution witness of one block (b200_dstate_witness) on the C3-shaped resident state.

    python -m pytest tests/test_gpu_witness.py -m gpu -q        # correctness first
    python tools/witness_bench.py --accounts 1000000 --slots 16 --touch 2000 --slot-writes 10

Seeds --accounts accounts x --slots slots, builds one block of the shape tools/dstate_bench.py commits (60 % storage-only
with --slot-writes slot writes, 25 % balance changes, 10 % new accounts with storage, 5 % destroyed), and times the witness
of that block in both modes: the C ABI call alone (stream time between CUDA events, and host-call time) after warm-ups,
and the Python mirror that also builds the result dict.  For comparison it times b200_dstate_multiproof over the same
account and slot keys (without the wipe expansion and the reveals).  It reports the node count, the witness bytes and the kernel
launches of one call; --cpu-sample N also times the test-side model of tests/test_gpu_witness.py on an N-account state
with a block scaled down in proportion (the model holds the whole state as Python tries, so it cannot take the full size).
Prints one JSON line.

    python tools/witness_bench.py --accounts 1000000 --slots 16 --touch 2000 --shards 4

--shards N seeds the same state once unsharded and once as N shards on the same GPU (rank r owns the top nibbles
[16r/N, 16(r+1)/N)) and times, alternating rep by rep, b200_dstate_witness of the block on the unsharded state and every
shard's b200_dstate_witness_root_kept (its kept pre-pass) plus b200_dstate_sharded_witness of its part (Legacy mode): CUDA-
event time per shard, the slowest shard and the sum over the shards (they run one after another here; on one GPU per rank
side by side), and the launches of each call.  The merged map is checked against the unsharded one in both modes.  Reads the
card's name, power limit and SM clock in the same run.  Prints one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KECCAK_EMPTY = bytes.fromhex("c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470")


def make_state(g, n, slots):
    from reth_b200 import ACCOUNT_DTYPE

    def sorted_keys(count, groups=None):
        k = g.integers(0, 256, (count, 32), dtype=np.uint8)
        cols = tuple(k[:, i] for i in range(31, -1, -1))
        order = np.lexsort(cols if groups is None else cols + (groups,))
        return k[order]
    keys = sorted_keys(n)
    accs = np.zeros(n, ACCOUNT_DTYPE)
    accs["nonce"] = g.integers(0, 1 << 16, n)
    accs["balance"][:, 24:] = g.integers(0, 256, (n, 8), dtype=np.uint8)
    accs["code_hash"] = np.frombuffer(KECCAK_EMPTY, np.uint8)
    total = n * slots
    skeys = sorted_keys(total, np.repeat(np.arange(n), slots))
    svals = np.zeros((total, 32), np.uint8)
    svals[:, 24:] = g.integers(0, 256, (total, 8), dtype=np.uint8)
    svals[:, 31] |= 1
    offs = np.arange(n + 1, dtype=np.uint64) * np.uint64(slots)
    return keys, accs, skeys, svals, offs


def make_block(rng, keys, skeys, offs, touch, slot_writes):
    """{key: (flags, account row or None, {slot: value int})}: the dstate_bench block shape, zeroing / changing two existing
    slots of the storage-only accounts"""
    from reth_b200 import ACCOUNT_DTYPE, DynamicState
    EX, UN = DynamicState.EXISTS, DynamicState.UNCHANGED
    block = {}
    for q, pi in enumerate(rng.choice(len(keys), touch, replace=False)):
        k, r = keys[pi].tobytes(), q / touch
        if r < 0.60:
            slots = {rng.integers(0, 256, 32, dtype=np.uint8).tobytes(): int(rng.integers(1, 2**60)) for _ in range(slot_writes)}
            lo = int(offs[pi])
            for j in range(lo, min(lo + 2, int(offs[pi + 1]))):
                slots[skeys[j].tobytes()] = 0 if rng.random() < 0.5 else int(rng.integers(1, 2**60))
            block[k] = (EX | UN, None, slots)
        elif r < 0.85:
            a = np.zeros((), ACCOUNT_DTYPE)
            a["nonce"] = 1
            a["balance"][24:] = rng.integers(0, 256, 8, dtype=np.uint8)
            a["code_hash"] = np.frombuffer(KECCAK_EMPTY, np.uint8)
            block[k] = (EX, a, {})
        elif r < 0.95:
            a = np.zeros((), ACCOUNT_DTYPE)
            a["code_hash"] = np.frombuffer(KECCAK_EMPTY, np.uint8)
            block[rng.integers(0, 256, 32, dtype=np.uint8).tobytes()] = (
                EX, a, {rng.integers(0, 256, 32, dtype=np.uint8).tobytes(): int(rng.integers(1, 2**60)) for _ in range(slot_writes)})
        else:
            block[k] = (0, None, {})
    return block


def block_arrays(block):
    from reth_b200 import ACCOUNT_DTYPE
    ks = sorted(block)
    m = len(ks)
    bk = np.frombuffer(b"".join(ks), np.uint8).reshape(m, 32)
    ba, bf = np.zeros(m, ACCOUNT_DTYPE), np.zeros(m, np.uint8)
    sk, sv, so = [], [], [0]
    for i, k in enumerate(ks):
        fl, a, slots = block[k]
        bf[i] = fl
        if a is not None:
            ba[i] = a
        for s in sorted(slots):
            sk.append(s)
            sv.append(int(slots[s]).to_bytes(32, "big"))
        so.append(len(sk))
    bsk = np.frombuffer(b"".join(sk), np.uint8).reshape(-1, 32) if sk else np.zeros((0, 32), np.uint8)
    bsv = np.frombuffer(b"".join(sv), np.uint8).reshape(-1, 32) if sv else np.zeros((0, 32), np.uint8)
    return bk, ba, bf, bsk, bsv, np.array(so, np.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--touch", type=int, default=2000)
    ap.add_argument("--slot-writes", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-sample", type=int, default=0, help="accounts of the state the CPU model is timed on (0 = skip)")
    ap.add_argument("--shards", type=int, default=0, help="time the witness of a state sharded this many ways (0 = unsharded only)")
    args = ap.parse_args()
    if args.shards:
        return sharded_main(args)
    import torch

    from reth_b200 import DynamicState, Engine
    eng = Engine(0)
    g = np.random.default_rng(3)
    keys, accs, skeys, svals, offs = make_state(g, args.accounts, args.slots)
    ds = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    block = make_block(np.random.default_rng(77), keys, skeys, offs, args.touch, args.slot_writes)
    arrays = block_arrays(block)
    root0 = ds.root()
    out = {"accounts": args.accounts, "slots": args.accounts * args.slots, "block_accounts": len(arrays[0]),
           "block_slot_entries": len(arrays[3])}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        dev, host = [], []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            ev0.record(stream)
            t0 = time.perf_counter()
            r = fn()
            host.append((time.perf_counter() - t0) * 1e3)
            ev1.record(stream)
            ev1.synchronize()
            dev.append(ev0.elapsed_time(ev1))
        return r, float(np.median(dev)), float(np.median(host))

    import ctypes as C

    from reth_b200._lib import Witness
    from reth_b200.engine import _ptr
    bk, ba, bf, bsk, bsv, bso = arrays

    def c_call(mode):  # the C ABI call alone (the Python dict of the result is not built)
        w = Witness()
        eng._check(eng.lib.b200_dstate_witness(ds.handle, _ptr(bk), _ptr(ba), _ptr(bf), len(bk), _ptr(bsk), _ptr(bsv), _ptr(bso),
                                               mode, 0, C.byref(w)))
        n = int(w.n)
        eng.lib.b200_witness_release(C.byref(w))
        return n

    for code, mode in enumerate(("legacy", "canonical")):
        l0 = eng.launch_count()
        w = ds.witness(*arrays, mode=mode)
        launches = eng.launch_count() - l0
        n, dev_ms, host_ms = timed(lambda: c_call(code))
        assert n == len(w)
        _, _, py_ms = timed(lambda: ds.witness(*arrays, mode=mode))
        out[mode] = {"device_ms": round(dev_ms, 3), "host_call_ms": round(host_ms, 3), "python_mirror_ms": round(py_ms, 3),
                     "nodes": len(w), "bytes": sum(len(v) for v in w.values()), "launches": launches}
    from reth_b200._lib import Proofs
    sroots = np.zeros((len(bk), 32), np.uint8)

    def c_multiproof():  # b200_dstate_multiproof over the same accounts and slot keys, C ABI call alone
        pa, ps = Proofs(), Proofs()
        eng._check(eng.lib.b200_dstate_multiproof(ds.handle, _ptr(bk), len(bk), _ptr(bso), _ptr(bsk), C.byref(pa), _ptr(sroots),
                                                  C.byref(ps)))
        n = int(pa.n_nodes) + int(ps.n_nodes)
        eng.lib.b200_proofs_release(C.byref(pa))
        eng.lib.b200_proofs_release(C.byref(ps))
        return n

    n, dev_ms, host_ms = timed(c_multiproof)
    out["multiproof_same_targets"] = {"device_ms": round(dev_ms, 3), "host_call_ms": round(host_ms, 3), "proof_nodes": n}
    assert ds.root() == root0, "the witness changed the state"
    if args.cpu_sample:
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
        from tests.test_gpu_witness import model_witness
        n = args.cpu_sample
        gs = np.random.default_rng(5)
        k2, a2, sk2, sv2, of2 = make_state(gs, n, args.slots)
        state = {k2[i].tobytes(): (a2[i], {sk2[j].tobytes(): int.from_bytes(sv2[j].tobytes(), "big")
                                           for j in range(int(of2[i]), int(of2[i + 1]))}) for i in range(n)}
        touch = max(1, args.touch * n // args.accounts)
        b2 = make_block(np.random.default_rng(78), k2, sk2, of2, touch, args.slot_writes)
        b2 = {k: (fl, a if a is not None else np.zeros((), a2.dtype), s) for k, (fl, a, s) in b2.items()}
        t0 = time.perf_counter()
        model_witness(state, b2, "legacy")
        out["cpu_model"] = {"accounts": n, "block_accounts": len(b2), "legacy_s": round(time.perf_counter() - t0, 3),
                            "note": "Python model, includes building every trie of the sampled state"}
    out["gpu"] = torch.cuda.get_device_name(0)
    print(json.dumps(out))
    ds.close()
    eng.close()


def sharded_main(args):
    S = args.shards
    if not 1 <= S <= 16:
        raise SystemExit("--shards: 1 to 16")
    import ctypes as C

    import torch

    from reth_b200 import DynamicState, Engine
    from reth_b200._lib import FrontierEntry, Witness
    from reth_b200.engine import _ptr
    from tools.stateless_bench import card, spread
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
    block = make_block(np.random.default_rng(77), keys, skeys, offs, args.touch, args.slot_writes)
    arrays = block_arrays(block)
    parts = [block_arrays({k: v for k, v in block.items() if (k[0] >> 4) * S // 16 == r}) for r in range(S)]
    out.update({"accounts": args.accounts, "slots": args.accounts * args.slots, "shards": S, "block_accounts": len(arrays[0]),
                "block_slot_entries": len(arrays[3]), "block_accounts_per_shard": [len(p[0]) for p in parts]})
    fr = (FrontierEntry * 16).from_buffer_copy(merged.tobytes())
    kept_of = {}

    def kept_call(r, mode=0):
        bk, ba, bf, bsk, bsv, bso = parts[r]
        kept = C.c_uint16()
        eng._check(eng.lib.b200_dstate_witness_root_kept(shards[r].handle, _ptr(bk), _ptr(ba), _ptr(bf), len(bk), _ptr(bsk), _ptr(bsv),
                                                         _ptr(bso), mode, C.byref(kept)))
        return kept.value

    def witness_call(r=None, mode=0):  # the C ABI call alone (the Python dict of the result is not built)
        bk, ba, bf, bsk, bsv, bso = arrays if r is None else parts[r]
        w = Witness()
        if r is None:
            rc = eng.lib.b200_dstate_witness(ds.handle, _ptr(bk), _ptr(ba), _ptr(bf), len(bk), _ptr(bsk), _ptr(bsv), _ptr(bso), mode, 0,
                                             C.byref(w))
        else:
            rc = eng.lib.b200_dstate_sharded_witness(shards[r].handle, fr, hm, tm, kept_of[mode], _ptr(bk), _ptr(ba), _ptr(bf), len(bk),
                                                     _ptr(bsk), _ptr(bsv), _ptr(bso), mode, 0, C.byref(w), None)
        eng._check(rc)
        n = int(w.n)
        eng.lib.b200_witness_release(C.byref(w))
        return n

    for mode in (0, 1):
        kept_of[mode] = 0
        for r in range(S):
            kept_of[mode] |= kept_call(r, mode)
    calls = {"unsharded": lambda: witness_call()}
    for r in range(S):
        calls[f"kept_{r}"] = lambda r=r: kept_call(r)
        calls[f"witness_{r}"] = lambda r=r: witness_call(r)
    launches = {}
    for k, c in calls.items():
        l0 = eng.launch_count()
        c()
        launches[k] = eng.launch_count() - l0
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.warmup):
        for c in calls.values():
            c()
    dev = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, c in calls.items():
            torch.cuda.synchronize()
            ev0.record(stream)
            c()
            ev1.record(stream)
            ev1.synchronize()
            dev[k].append(ev0.elapsed_time(ev1))
    kd, wd = np.array([dev[f"kept_{r}"] for r in range(S)]), np.array([dev[f"witness_{r}"] for r in range(S)])
    out["unsharded_witness"] = {"device_ms": spread(dev["unsharded"]), "launches": launches["unsharded"]}
    out["sharded_witness"] = {
        "per_shard": [{"kept_ms": spread(dev[f"kept_{r}"]), "witness_ms": spread(dev[f"witness_{r}"]),
                       "kept_launches": launches[f"kept_{r}"], "witness_launches": launches[f"witness_{r}"]} for r in range(S)],
        "max_over_shards_ms": spread((kd + wd).max(axis=0)), "sum_over_shards_ms": spread((kd + wd).sum(axis=0)),
        "kept_share_of_sum": round(float(np.median(kd.sum(axis=0)) / np.median((kd + wd).sum(axis=0))), 3)}
    matches = {}
    for mode in ("legacy", "canonical"):
        kept = 0
        for r in range(S):
            kept |= shards[r].witness_root_kept(parts[r], mode)
        union = {}
        for r in range(S):
            union.update(shards[r].sharded_witness(merged, hm, tm, kept, parts[r], mode))
        matches[mode] = union == ds.witness(*arrays, mode=mode)
    out["matches_unsharded"] = matches
    for d in shards + [ds]:
        d.close()
    eng.close()
    print(json.dumps(out))
    if not all(matches.values()):
        raise SystemExit("the merged sharded witness differs from the unsharded one")


if __name__ == "__main__":
    main()
