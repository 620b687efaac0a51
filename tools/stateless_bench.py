#!/usr/bin/env python3
"""Cost of post-block roots from execution witnesses (b200_witness_roots) on the C3-shaped state.

    python -m pytest tests/test_gpu_stateless.py -m gpu -q      # correctness first
    python tools/stateless_bench.py --accounts 1000000 --slots 16 --touch 2000 --blocks 16

Seeds the state of tools/witness_bench.py (--accounts accounts x --slots slots) as a resident b200_dstate and builds a chain
of --blocks blocks of its 2 000-account shape; the Legacy witness of each block is taken before that block is applied, and
the apply gives the reference root.  Times the C ABI call alone (inputs packed beforehand) for the first block and for the
whole chain as one batch: CUDA-event time on the call's stream and host-call time, after warm-ups, median / min / max over
--reps.  Counts per call: kernel launches (b200_launch_count); device-to-host read-backs and host-to-device copies from a
separate torch.profiler run of one call; nodes, witness bytes and the host-to-device bytes of the inputs.  --python-model
also times the test-side Python model (tests/test_gpu_witness.py Stateless) on the first block: a Python model, not reth.
Reads the card's name, power limit and SM clock in the same run.  Prints one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.witness_bench import block_arrays, make_block, make_state  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().split("\n")[0]
    name, power, sm, sm_max = [x.strip() for x in q.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def spread(xs):
    return {"median": round(float(np.median(xs)), 3), "min": round(float(np.min(xs)), 3), "max": round(float(np.max(xs)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--touch", type=int, default=2000)
    ap.add_argument("--slot-writes", type=int, default=10)
    ap.add_argument("--blocks", type=int, default=16)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--python-model", action="store_true", help="also time the test-side Python model on the first block")
    args = ap.parse_args()
    import torch

    from reth_b200 import DynamicState, Engine
    from reth_b200._lib import Stats
    from reth_b200.engine import _ptr, witness_batch_arrays
    out = {"card": card()}
    eng = Engine(0)
    keys, accs, skeys, svals, offs = make_state(np.random.default_rng(3), args.accounts, args.slots)
    ds = DynamicState.create(eng, keys, accs, skeys, svals, offs)
    parents, witnesses, blocks, arrays, wants = [], [], [], [], []
    rng = np.random.default_rng(77)
    for _ in range(args.blocks):
        block = make_block(rng, keys, skeys, offs, args.touch, args.slot_writes)
        a = block_arrays(block)
        parents.append(ds.root())
        witnesses.append(ds.witness(*a, mode="legacy"))
        wants.append(ds.apply(*a))
        blocks.append(block)
        arrays.append(a)
    ds.close()
    out.update({"accounts": args.accounts, "slots": args.accounts * args.slots, "block_accounts": len(arrays[0][0]),
                "block_slot_entries": len(arrays[0][3]), "witness": "legacy"})
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def case(nb):
        packed = witness_batch_arrays(parents[:nb], witnesses[:nb], arrays[:nb])
        roots, status = np.zeros((nb, 32), np.uint8), np.zeros(nb, np.int32)
        s = Stats()

        def call():  # the C ABI call alone
            eng._check(eng.lib.b200_witness_roots(eng.ctx, nb, *(_ptr(x) for x in packed[1:]), _ptr(roots), _ptr(status), C.byref(s)))

        l0 = eng.launch_count()
        call()
        launches = eng.launch_count() - l0
        assert status.tolist() == [0] * nb and [r.tobytes() for r in roots] == wants[:nb], "root differs from the apply"
        for _ in range(args.warmup):
            call()
        dev, host = [], []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            ev0.record(stream)
            t0 = time.perf_counter()
            call()
            host.append((time.perf_counter() - t0) * 1e3)
            ev1.record(stream)
            ev1.synchronize()
            dev.append(ev0.elapsed_time(ev1))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        dtoh = sum(1 for n in names if "DtoH" in n)
        htod = sum(1 for n in names if "HtoD" in n)
        input_bytes = sum(x.nbytes for x in packed[1:]) - (packed[2].nbytes if packed[3][-1] == 0 else 0)
        n_nodes, wbytes = int(packed[4][-1]), int(packed[3][-1])
        host_med = float(np.median(host))
        return {"blocks": nb, "device_ms": spread(dev), "host_call_ms": spread(host), "host_call_ms_per_block": round(host_med / nb, 3),
                "launches": launches, "readbacks_dtoh": dtoh, "copies_htod": htod, "nodes": n_nodes, "witness_bytes": wbytes,
                "h2d_input_bytes": int(input_bytes)}

    out["one_block"] = case(1)
    if args.blocks > 1:
        out["batch"] = case(args.blocks)
    if args.python_model:
        from tests.test_gpu_witness import stateless_root
        from reth_b200 import ACCOUNT_DTYPE
        b0 = {k: (fl, a if a is not None else np.zeros((), ACCOUNT_DTYPE), s) for k, (fl, a, s) in blocks[0].items()}
        t0 = time.perf_counter()
        r = stateless_root(witnesses[0], parents[0], b0, False)
        out["python_model"] = {"blocks": 1, "s": round(time.perf_counter() - t0, 3), "root_matches": r == wants[0],
                               "note": "test-side Python model (tests/test_gpu_witness.py Stateless), not reth"}
    out["card_after"] = card()
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
