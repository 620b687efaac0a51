#!/usr/bin/env python3
"""Latency of the dynamic resident trie (b200_dtrie_*) on the GPU (a leg of bench.py).

    python -m pytest tests/test_gpu_dtrie.py -m gpu -q      # correctness first
    python tools/dtrie_bench.py --base 100000000 --dirty 10000 --mix 80,10,10   # then latency

Builds a base trie of --base accounts on the device, then applies blocks of --dirty keys with the given
update,insert,delete percentages through the host-pointer C ABI (the call a reth shim makes: H2D of the dirty set and D2H
of the root inside) and prints one JSON line: median wall µs, device ms of the build stats, re-hashed nodes, and the same
block through b200_trie_apply (merge + rebuild) for comparison.  Roots of the two paths are compared every block."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", type=int, default=10_000_000)
    ap.add_argument("--dirty", type=int, default=10_000)
    ap.add_argument("--mix", default="80,10,10", help="update,insert,delete percent")
    ap.add_argument("--blocks", type=int, default=12)
    ap.add_argument("--cpu-sample", type=int, default=0, help="accounts of the oracle's from-scratch fold timed as the CPU baseline (0 = skip)")
    ap.add_argument("--compare", action="store_true", help="also run every block through b200_trie_apply and compare roots")
    args = ap.parse_args()
    T0 = time.perf_counter()

    def note(msg):  # progress on stderr: where the wall time of a 100M-key run goes
        print(f"[dtrie_bench {time.perf_counter() - T0:7.1f}s] {msg}", file=sys.stderr, flush=True)
    import torch
    from bench import be_sort_key, random_keys_torch, splitmix64_torch
    from reth_b200 import ACCOUNT_DTYPE, DynamicTrie, Engine, ResidentTrie
    dev = torch.device("cuda", 0)
    eng = Engine(0)
    eng.use_torch_stream()
    n, m = args.base, args.dirty
    pu, pi, pd = (int(x) for x in args.mix.split(","))
    keys = random_keys_torch(5, n, dev)
    keys = keys[torch.sort(be_sort_key(keys), stable=True).indices].contiguous()
    accts = torch.zeros((n, 72), dtype=torch.uint8, device=dev)
    accts[:, 32:40] = splitmix64_torch(5 ^ 0xACC0, n, dev).view(torch.uint8).view(n, 8)
    accts[:, 40:72] = torch.frombuffer(bytearray(bytes.fromhex(
        "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470")), dtype=torch.uint8).to(dev)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()   # the generator's temporaries: the library allocates outside torch's cache
    t0 = time.perf_counter()
    trie = DynamicTrie.create_dev(eng, keys.view(torch.uint8).view(-1), accts.view(-1), None, n)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    note("dynamic trie created")
    ref = ResidentTrie.create_dev(eng, keys.view(torch.uint8).view(-1), accts.view(-1), None, n) if args.compare else None
    assert ref is None or trie.root() == ref.root()
    # both tries hold their own copies of the inputs: keep host copies and hand the device memory back (two resident tries of
    # 100M leaves and a merge + rebuild have to fit one 80 GB GPU)
    base_keys_np = keys.view(torch.uint8).view(n, 32).cpu().numpy()
    h_accts = accts.cpu().numpy().view(ACCOUNT_DTYPE).reshape(-1)
    del keys, accts
    torch.cuda.empty_cache()
    eng.set_stream(None)
    rng = np.random.default_rng(55)
    live = base_keys_np.copy()   # host copy of the key set, kept in step with the trie
    live_set = None
    lat, dev_ms, built, mismatches, lat_rebuild, launches = [], [], [], 0, [], []
    base_root = trie.root()
    base_index = {}          # key -> row in the base arrays, for every key a block touched (the final undo block needs the base value)
    inserted_total = set()
    note("host copies ready")
    for b in range(args.blocks):
        note(f"block {b}")
        n_upd, n_ins, n_del = m * pu // 100, m * pi // 100, m * pd // 100
        pick = rng.choice(len(live), n_upd + n_del, replace=False)
        upd_keys, del_keys = live[pick[:n_upd]], live[pick[n_upd:]]
        ins_keys = rng.integers(0, 256, (n_ins, 32), dtype=np.uint8)
        dk = np.concatenate([upd_keys, del_keys, ins_keys])
        present = np.concatenate([np.ones(n_upd, np.uint8), np.zeros(n_del, np.uint8), np.ones(n_ins, np.uint8)])
        order = np.lexsort(tuple(dk[:, i] for i in range(31, -1, -1)))
        dk, present = np.ascontiguousarray(dk[order]), np.ascontiguousarray(present[order])
        da = np.zeros(len(dk), ACCOUNT_DTYPE)
        da["nonce"] = b + 1
        da["balance"][:, 24:] = rng.integers(0, 256, (len(dk), 8), dtype=np.uint8)
        da["code_hash"] = np.frombuffer(bytes.fromhex("c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"), np.uint8)
        l0 = eng.launch_count()
        t0 = time.perf_counter()
        root, stats = trie.apply(dk, da, present, want_stats=True)
        wall = time.perf_counter() - t0
        if b >= 2:
            lat.append(wall * 1e6)
            dev_ms.append(stats["device_ms"])
            built.append(stats["branches_added"])
            launches.append(eng.launch_count() - l0)
        if ref is not None:  # the same block through merge + from-scratch rebuild (the static, oracle-pinned path)
            t0 = time.perf_counter()
            r2 = ref.apply(dk, da, present)[0]
            if b >= 2:
                lat_rebuild.append((time.perf_counter() - t0) * 1e6)
            mismatches += r2 != root
        for kk in ins_keys:
            inserted_total.add(kk.tobytes())
        for kk in list(upd_keys) + list(del_keys):
            base_index.setdefault(kk.tobytes(), None)
        mask = np.ones(len(live), bool)
        mask[pick[n_upd:]] = False
        live = np.concatenate([live[mask], ins_keys])
    note("blocks done")
    import faulthandler
    faulthandler.dump_traceback_later(240, exit=True)   # a hang below says where
    # ---- undo everything in one block: base values back, deleted base keys re-inserted, inserted keys deleted.  The root must
    # return to the root of the from-scratch build the trie was created from (independent of any model of the state).
    # sorted with the keys; NATIVE byte order (searchsorted on a non-native array converts the whole array on every call)
    prefix = np.ascontiguousarray(base_keys_np[:, :8]).view(">u8").reshape(-1).astype(np.uint64)

    def find_row(kb):
        want = int.from_bytes(kb[:8], "big")
        row = int(np.searchsorted(prefix, np.uint64(want)))   # (a Python int would promote the whole array on every call)
        while row < n and int(prefix[row]) == want:
            if base_keys_np[row].tobytes() == kb:
                return row
            row += 1
        return -1
    note("base key prefixes ready")
    undo = {}
    for kb in base_index:
        if kb in inserted_total:
            continue
        row = find_row(kb)
        if row >= 0:
            undo[kb] = (1, h_accts[row])
    for kb in inserted_total:
        if kb not in undo:
            undo[kb] = (0, h_accts[0])
    note("undo entries looked up")
    uk = sorted(undo)
    dk = np.frombuffer(b"".join(uk), np.uint8).reshape(-1, 32)
    da = np.zeros(len(uk), ACCOUNT_DTYPE)
    present = np.zeros(len(uk), np.uint8)
    for i, kb in enumerate(uk):
        present[i], da[i] = undo[kb]
    note(f"undo block of {len(uk)} entries")
    undo_root = trie.apply(dk, da, present)
    note("undo applied")
    undo_ok = bool(undo_root == base_root and len(trie) == n)
    faulthandler.cancel_dump_traceback_later()
    cpu = None
    if args.cpu_sample:
        import oracle
        from tests.util import synth_accounts
        ak, ac = synth_accounts(5, args.cpu_sample)
        t0 = time.perf_counter()
        oracle.state_root(ak, ac)
        dt = time.perf_counter() - t0
        cpu = {"value": args.cpu_sample / dt, "unit": "leaves/s", "cores": 1, "kind": "port",
               "sample": f"from-scratch account-trie fold over {args.cpu_sample} accounts (the CPU restatement has no in-place update path)",
               "equivalent_rebuild_s_at_base_size": n / (args.cpu_sample / dt)}
    print(json.dumps({"undo_block_restores_base_root": undo_ok, "launches_per_block": float(np.median(launches)) if launches else None,
                      "merge_rebuild_wall_us_median": float(np.median(lat_rebuild)) if lat_rebuild else None,
                      "cpu_baseline": cpu,
                      "base_leaves": n, "dirty": m, "mix_update_insert_delete": [pu, pi, pd], "blocks": args.blocks,
                      "apply_wall_us_median": float(np.median(lat)), "apply_device_ms_median": float(np.median(dev_ms)),
                      "rehashed_nodes_median": float(np.median(built)), "base_build_ms": build_s * 1e3,
                      "leaves_after": len(trie), "resident_bytes": trie.device_bytes(),
                      "root_mismatches_vs_trie_apply": mismatches if ref is not None else None}))


if __name__ == "__main__":
    main()
