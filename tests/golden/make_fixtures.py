#!/usr/bin/env python
"""Regenerates tests/golden/genesis_allocs.json from the reference's genesis files.

Run against a checkout of reth (the tests only read the generated file):
    python tests/golden/make_fixtures.py /path/to/reth

Sources (data, not code): <reth>/crates/chainspec/res/genesis/{mainnet,sepolia,holesky,goerli}.json
(alloc + the `stateRoot` each file states) and <reth>/crates/trie/trie/testdata/proof-genesis.json.
Only the fields that enter the state root are kept: address -> balance, nonce, code, storage.
"""
import json
import os
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "."
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "genesis_allocs.json")


def slim(alloc):
    out = {}
    for addr, a in alloc.items():
        addr = addr.lower().removeprefix("0x")
        e = {"balance": hex(int(a.get("balance", "0x0"), 16) if a.get("balance", "0x0").startswith("0x")
                            else int(a["balance"]))}
        if a.get("nonce"):
            e["nonce"] = hex(int(a["nonce"], 16) if str(a["nonce"]).startswith("0x") else int(a["nonce"]))
        if a.get("code") and a["code"] not in ("0x", ""):
            e["code"] = a["code"].lower()
        if a.get("storage"):
            e["storage"] = {k.lower(): v.lower() for k, v in a["storage"].items()}
        out[addr] = e
    return out


def main():
    res = {}
    for name in ("mainnet", "sepolia", "holesky", "goerli"):  # dev.json's stateRoot is a stale copy of sepolia's
   
        g = json.load(open(f"{REF}/crates/chainspec/res/genesis/{name}.json"))
        res[name] = {"source": f"crates/chainspec/res/genesis/{name}.json",
                     "state_root": g["stateRoot"].lower().removeprefix("0x"),
                     "alloc": slim(g["alloc"])}
    g = json.load(open(f"{REF}/crates/trie/trie/testdata/proof-genesis.json"))
    res["testspec"] = {"source": "crates/trie/trie/testdata/proof-genesis.json; root node RLP "
                                 "crates/trie/db/tests/proof.rs:55",
                       "state_root": None, "alloc": slim(g["alloc"])}
    with open(OUT, "w") as f:
        json.dump(res, f, separators=(",", ":"), sort_keys=True)
    print(OUT, os.path.getsize(OUT), "bytes", {k: len(v["alloc"]) for k, v in res.items()})


if __name__ == "__main__":
    main()
