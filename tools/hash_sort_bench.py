#!/usr/bin/env python3
"""AccountHashing full pass (hash + sort, SURVEY.md §8 a2 / f2): b200_hash_sort_keys over --keys 20-byte addresses.

    python tools/hash_sort_bench.py --keys 10000000

Prints one JSON line: device time of b200_hash_sort_keys_dev (inputs resident in HBM, CUDA events), wall time of the
host-pointer call on page-locked buffers (H2D of the addresses, D2H of the sorted digests + permutation inside; once more
with ordinary pageable arrays), keys/s of both, the algorithmic
GB/s (20 B read + 32 B digest written + 32 B sorted digest + 4 B permutation written per key), and the CPU restatement
(oracle keccak on all host threads + numpy lexsort) on a bounded sample.  The sorted digests of the sample are compared."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--cpu-sample", type=int, default=1_000_000)
    args = ap.parse_args()
    import torch

    import oracle
    from bench import random_keys_torch
    from reth_b200 import Engine
    from tests.util import sort_rows
    n = args.keys
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    eng.use_torch_stream()
    d_addr = random_keys_torch(7, n, dev).view(torch.uint8).view(n, 32)[:, :20].contiguous().view(-1)
    d_sorted = torch.empty(n * 32, dtype=torch.uint8, device=dev)
    d_perm = torch.empty(n, dtype=torch.int32, device=dev)
    eng.hash_sort_keys_dev(d_addr, 20, 20, n, d_sorted, d_perm)
    torch.cuda.synchronize()
    dev_ms = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.hash_sort_keys_dev(d_addr, 20, 20, n, d_sorted, d_perm)
        e1.record()
        torch.cuda.synchronize()
        dev_ms.append(e0.elapsed_time(e1))
    eng.dev_status()
    eng.set_stream(None)
    h_addr = eng.pinned_empty((n, 20))
    h_addr[:] = d_addr.view(n, 20).cpu().numpy()
    h_sorted, h_perm = eng.pinned_empty((n, 32)), eng.pinned_empty((n,), np.uint32)
    eng.hash_sort_keys(h_addr, 20, out=h_sorted, perm=h_perm)
    wall = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        eng.hash_sort_keys(h_addr, 20, out=h_sorted, perm=h_perm)
        wall.append((time.perf_counter() - t0) * 1e3)
    pageable_in = np.array(h_addr)
    t0 = time.perf_counter()
    eng.hash_sort_keys(pageable_in, 20)
    wall_pageable = (time.perf_counter() - t0) * 1e3
    same = bool((h_sorted == d_sorted.view(n, 32).cpu().numpy()).all())
    # CPU restatement on a bounded sample: keccak on all threads, then the sort the ETL collector would do
    cs = min(args.cpu_sample, n)
    threads = len(os.sched_getaffinity(0))
    t0 = time.perf_counter()
    dig = oracle.keccak256_fixed(h_addr[:cs], threads=threads)
    order = sort_rows(dig)
    cpu_s = time.perf_counter() - t0
    g_sorted, g_perm = eng.hash_sort_keys(h_addr[:cs], 20)
    ok = bool((g_sorted == dig[order]).all() and (dig[g_perm] == g_sorted).all())
    d = float(np.median(dev_ms))
    w = float(np.median(wall))
    print(json.dumps({
        "tool": "hash_sort_bench", "keys": n, "msg_len": 20, "device_ms": d, "keys_per_s_device": n / (d * 1e-3),
        "algorithmic_gb_per_s_device": n * (20 + 32 + 32 + 4) / (d * 1e-3) / 1e9,
        "wall_ms_e2e": w, "keys_per_s_e2e": n / (w * 1e-3), "wall_ms_e2e_pageable_buffers": wall_pageable,
        "e2e_api": "b200_hash_sort_keys, page-locked caller buffers: H2D of chunk k+1 under the hashing of chunk k, sort, D2H", "h2d_bytes": n * 20, "d2h_bytes": n * 36,
        "cpu_baseline": {"value": cs / cpu_s, "unit": "keys/s", "cores": threads, "kind": "port",
                         "sample": f"{cs} addresses: oracle keccak on {threads} threads + numpy lexsort of the digests"},
        "device_equals_host_path": same, "sorted_digests_match_oracle_on_sample": ok}))


if __name__ == "__main__":
    main()
