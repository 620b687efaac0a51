#!/usr/bin/env python3
"""StorageHashing full pass (hash + sort by keccak(address) || keccak(slot), SURVEY.md §8 a3 / f2): b200_hash_sort_storage over
--slots entries of --accounts contracts (Zipf-sized: a few large storages, a long tail of small ones).

    python tools/hash_sort_storage_bench.py --slots 10000000 --accounts 200000

Prints one JSON line: device time of b200_hash_sort_storage_dev (inputs resident in HBM, CUDA events), wall time of the
host-pointer call on page-locked buffers, entries/s of both, and the CPU restatement (oracle keccak on all host threads +
numpy lexsort of the composite keys) on a bounded sample; the sample's sorted keys and permutation are compared."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=10_000_000)
    ap.add_argument("--accounts", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--cpu-sample", type=int, default=1_000_000)
    args = ap.parse_args()
    import torch

    import oracle
    from bench import random_keys_torch
    from reth_b200 import Engine
    n, na = args.slots, args.accounts
    rng = np.random.default_rng(5)
    w = np.arange(1, na + 1, dtype=np.float64) ** -1.1
    counts = np.maximum(1, np.floor(w / w.sum() * n)).astype(np.int64)
    counts[0] += n - int(counts.sum())
    owner = np.repeat(rng.permutation(na).astype(np.uint32), counts)   # entries arrive grouped by address (the plain table)
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    eng.use_torch_stream()
    d_addr = random_keys_torch(17, na, dev).view(torch.uint8).view(na, 32)[:, :20].contiguous().view(-1)
    d_slots = random_keys_torch(19, n, dev).view(torch.uint8).view(-1)
    d_owner = torch.from_numpy(owner.view(np.int32)).to(dev)
    d_sorted = torch.empty(n * 64, dtype=torch.uint8, device=dev)
    d_perm = torch.empty(n, dtype=torch.int32, device=dev)
    eng.hash_sort_storage_dev(d_addr, na, d_owner, d_slots, n, d_sorted, d_perm)
    torch.cuda.synchronize()
    dev_ms = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.hash_sort_storage_dev(d_addr, na, d_owner, d_slots, n, d_sorted, d_perm)
        e1.record()
        torch.cuda.synchronize()
        dev_ms.append(e0.elapsed_time(e1))
    eng.dev_status()
    eng.set_stream(None)
    h_addr = eng.pinned_empty((na, 20))
    h_addr[:] = d_addr.view(na, 20).cpu().numpy()
    h_slots = eng.pinned_empty((n, 32))
    h_slots[:] = d_slots.view(n, 32).cpu().numpy()
    h_owner = eng.pinned_empty((n,), np.uint32)
    h_owner[:] = owner
    h_sorted, h_perm = eng.pinned_empty((n, 64)), eng.pinned_empty((n,), np.uint32)
    eng.hash_sort_storage(h_addr, h_owner, h_slots, out=h_sorted, perm=h_perm)
    wall = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        eng.hash_sort_storage(h_addr, h_owner, h_slots, out=h_sorted, perm=h_perm)
        wall.append((time.perf_counter() - t0) * 1e3)
    same = bool((h_sorted == d_sorted.view(n, 64).cpu().numpy()).all())
    # CPU restatement on a bounded sample (whole accounts): keccak on all threads, then the collector's sort
    cs = min(args.cpu_sample, n)
    threads = len(os.sched_getaffinity(0))
    sl, ow = np.array(h_slots[:cs]), np.array(h_owner[:cs])
    t0 = time.perf_counter()
    ha = oracle.keccak256_fixed(np.array(h_addr), threads=threads)
    hs = oracle.keccak256_fixed(sl, threads=threads)
    comp = np.concatenate([ha[ow], hs], axis=1)
    v = comp.view(">u8")
    order = np.lexsort(tuple(v[:, i] for i in range(7, -1, -1)))
    cpu_s = time.perf_counter() - t0
    g_sorted, g_perm = eng.hash_sort_storage(np.array(h_addr), ow, sl)
    ok = bool((g_sorted == comp[order]).all() and (g_perm.astype(np.int64) == order).all())
    d, wl = float(np.median(dev_ms)), float(np.median(wall))
    print(json.dumps({
        "tool": "hash_sort_storage_bench", "entries": n, "accounts": na, "largest_storage": int(counts.max()),
        "device_ms": d, "entries_per_s_device": n / (d * 1e-3),
        "algorithmic_gb_per_s_device": (n * (32 + 4 + 32 + 64 + 4) + na * 52) / (d * 1e-3) / 1e9,
        "wall_ms_e2e": wl, "entries_per_s_e2e": n / (wl * 1e-3), "h2d_bytes": n * 36 + na * 20, "d2h_bytes": n * 68,
        "e2e_api": "b200_hash_sort_storage, page-locked caller buffers",
        "cpu_baseline": {"value": cs / cpu_s, "unit": "entries/s", "cores": threads, "kind": "port",
                         "sample": f"{cs} entries: oracle keccak on {threads} threads + numpy lexsort of the 64-byte keys"},
        "device_equals_host_path": same, "sorted_keys_match_oracle_on_sample": ok}))
    eng.close()
    return 0 if (same and ok) else 1


if __name__ == "__main__":
    sys.exit(main())
