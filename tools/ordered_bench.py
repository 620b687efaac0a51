#!/usr/bin/env python3
"""Round-2 measurement aid for b200_ordered_roots (transactions / receipts roots of a batch of blocks, DESIGN.md §8c).

    python tools/ordered_bench.py --blocks 2000 --items 200 --shape receipts

Synthesizes --blocks lists of about --items items (receipt-shaped: 262..700 bytes; tx-shaped: mostly 110..200 bytes with a
tail of large calldata), runs them through the host-pointer C ABI (H2D of the items and D2H of the roots inside — the
call a reth shim makes) and prints one JSON line: median wall ms, device ms from the build stats, items/s and item GB/s,
next to the CPU oracle (1 thread) on a bounded sample of the same lists.  Roots are compared on the sample."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=2000)
    ap.add_argument("--items", type=int, default=200)
    ap.add_argument("--shape", choices=["receipts", "transactions"], default="receipts")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--cpu-sample", type=int, default=200, help="lists given to the CPU oracle")
    args = ap.parse_args()
    import oracle
    from reth_b200 import Engine
    rng = np.random.default_rng(99)
    counts = rng.integers(max(0, args.items // 2), args.items * 3 // 2 + 1, args.blocks)
    n = int(counts.sum())
    if args.shape == "receipts":
        lens = 262 + rng.integers(0, 440, n)
    else:
        lens = rng.choice([110, 115, 150, 200, 700, 3000, 20000], n, p=[.35, .2, .15, .15, .1, .04, .01])
    value_offsets = np.zeros(n + 1, np.uint64)
    value_offsets[1:] = np.cumsum(lens, dtype=np.uint64)
    seg_offsets = np.zeros(args.blocks + 1, np.uint64)
    seg_offsets[1:] = np.cumsum(counts, dtype=np.uint64)
    values = rng.integers(0, 256, int(value_offsets[-1]), dtype=np.uint8)
    eng = Engine(0)
    roots = eng.ordered_roots(values, value_offsets, seg_offsets)  # warm-up (allocations)
    pageable = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        eng.ordered_roots(values, value_offsets, seg_offsets)
        pageable.append((time.perf_counter() - t0) * 1e3)
    # the same call with the caller's buffers page-locked (b200_host_alloc): the H2D copy is a plain DMA
    pv, po, ps = (eng.pinned_empty(a.shape, a.dtype) for a in (values, value_offsets, seg_offsets))
    pv[:], po[:], ps[:] = values, value_offsets, seg_offsets
    wall, dev = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        roots, st = eng.ordered_roots(pv, po, ps, want_stats=True)
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(st["device_ms"])
    k = min(args.cpu_sample, args.blocks)
    so = seg_offsets[:k + 1]
    vo = value_offsets[:int(so[-1]) + 1]
    t0 = time.perf_counter()
    want = oracle.ordered_roots(values[:int(vo[-1])], vo, so)
    cpu_s = time.perf_counter() - t0
    ok = bool((roots[:k] == want).all())
    w, d = float(np.median(wall)), float(np.median(dev))
    print(json.dumps({
        "tool": "ordered_bench", "shape": args.shape, "lists": args.blocks, "items": n, "item_bytes": int(value_offsets[-1]),
        "wall_ms": round(w, 3), "wall_ms_pageable_buffers": round(float(np.median(pageable)), 3), "device_ms": round(d, 3), "items_per_s_e2e": round(n / (w / 1e3)),
        "items_per_s_device": round(n / (d / 1e3)) if d else None,
        "item_GBps_device": round(int(value_offsets[-1]) / (d / 1e3) / 1e9, 2) if d else None,
        "cpu_oracle_items_per_s": round(int(so[-1]) / cpu_s), "cpu_sample_lists": k, "roots_match_oracle": ok,
    }))
    eng.close()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
