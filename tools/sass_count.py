#!/usr/bin/env python3
"""ALU-pipe instructions per digest of the key-hash kernels, counted from their SASS (the constant behind `alu_frac` in
bench.py):

    python tools/sass_count.py                  # keccak256_fixed32_kernel<256> of the in-tree build
    python tools/sass_count.py --kernel fixed20 --obj path/to/keccak_batch.o

The kernel is a grid-stride loop whose body hashes one key: 24 Keccak rounds, of which the first (sparse state) and
the last (only lanes 0..3 live) are peeled.  The 22 rounds between them are either a loop (one round per trip) or
unrolled in line; both shapes are counted.  LOP3 / SHF / ISETP / VIADD / LEA / IADD3 / SEL / PRMT issue to the ALU
pipe (64 lanes/clk/SM on compute capability 9.0); IMAD / MOV go to the FMA pipe, LDG / STG to the LSU.

The LUT histogram of the LOP3s is the check on the code shape: a round should be ~70 x 0x96 (three-input XOR:
column parities and theta), 50 x 0xb4 (chi) and 1-2 for iota.  Two-input XORs (0x3c, 0x5a, 0x66) in bulk mean
ptxas has re-factored theta again (see keccak_f1600.cuh)."""
import argparse
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "reth_b200", "csrc", "build", "keccak_batch.o")
FUN = {"fixed32": "_ZN4b20024keccak256_fixed32_kernelILi256EEEvPKhjmP5uint4",
       "fixed20": "_ZN4b20024keccak256_fixed20_kernelILi256EEEvPKhjmP5uint4"}
ALU = ("LOP3", "SHF", "ISETP", "VIADD", "LEA", "IADD3", "SEL", "PRMT", "IADD")
ROUNDS = 24
LOOP_TRIPS = 22  # rounds 1..22 when they are a loop


def parse(txt):
    """[(address, opcode without modifiers, branch target or None, LOP3 LUT or None)] in address order"""
    ins = []
    for l in txt.splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", l)
        if not m:
            continue
        rest = m.group(2).split()
        if rest[0].startswith("@"):
            rest = rest[1:]
        op = rest[0].split(".")[0]
        target = int(rest[-1], 16) if op == "BRA" and rest[-1].startswith("0x") else None
        lut = None
        if op == "LOP3":
            luts = [t.rstrip(",") for t in rest[1:] if re.fullmatch(r"0x[0-9a-f]{1,2},?", t)]
            lut = luts[-1] if luts else "?"
        ins.append((int(m.group(1), 16), op, target, lut))
    return ins


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--obj", default=OBJ, help="object file (default: the in-tree build of keccak_batch.cu)")
    ap.add_argument("--kernel", choices=sorted(FUN), default="fixed32")
    args = ap.parse_args()
    txt = subprocess.run(["cuobjdump", "-sass", "-fun", FUN[args.kernel], args.obj], capture_output=True, text=True,
                         check=True).stdout
    ins = parse(txt)
    back = [(a, t) for a, _, t, _ in ins if t is not None and t < a]
    outer_end, outer_start = max(back, key=lambda x: x[0] - x[1])  # the grid-stride loop: one digest per trip
    inner = [(e, s) for e, s in back if outer_start <= s and e < outer_end]
    body = [x for x in ins if outer_start <= x[0] <= outer_end]
    if inner:  # the 22 middle rounds are a loop: its body is one round
        loop_end, loop_start = min(inner, key=lambda x: x[0] - x[1])
        loop = [x for x in body if loop_start <= x[0] <= loop_end]
        rest = [x for x in body if not loop_start <= x[0] <= loop_end]
        shape = f"round loop of {len(loop)} instructions x {LOOP_TRIPS} trips"
    else:
        loop, rest = [], body
        shape = "rounds unrolled in line"
    ops = lambda xs: collections.Counter(o for _, o, _, _ in xs)
    luts = lambda xs: collections.Counter(u for _, o, _, u in xs if o == "LOP3")
    n_alu = lambda c: sum(v for k, v in c.items() if k in ALU)
    per_digest = ops(rest) + collections.Counter({k: LOOP_TRIPS * v for k, v in ops(loop).items()})
    lut_digest = luts(rest) + collections.Counter({k: LOOP_TRIPS * v for k, v in luts(loop).items()})
    fmt = lambda c: ", ".join(f"{k} {v}" for k, v in sorted(c.items(), key=lambda kv: -kv[1]))

    print(f"keccak256_{args.kernel}_kernel<256>: {len(ins)} SASS instructions, {shape}")
    if loop:
        c = ops(loop)
        print(f"  per round (loop body): {n_alu(c)} ALU = {c['LOP3']} LOP3 + {c['SHF']} SHF + "
              f"{n_alu(c) - c['LOP3'] - c['SHF']} other;  LOP3 LUTs: {fmt(luts(loop))}")
        c = ops(rest)
        print(f"  outside the loop (loads, peeled rounds 0 and 23, stores, control): {sum(c.values())} instr, "
              f"{n_alu(c)} ALU;  LOP3 LUTs: {fmt(luts(rest))}")
    alu = n_alu(per_digest)
    print(f"  per round, mean of {ROUNDS}: {per_digest['LOP3'] / ROUNDS:.1f} LOP3 + {per_digest['SHF'] / ROUNDS:.1f} SHF")
    print(f"  LOP3 LUTs per digest: {fmt(lut_digest)}")
    print(f"per digest: {sum(per_digest.values())} instructions, {alu} on the ALU pipe")
    print(f"ALU ceiling per SM: {64 / alu * 1e3:.3f} digests per 1000 clocks (x 132 SMs x SM clock on an H100 SXM; "
          f"{132 * 64 * 1.98e9 / alu / 1e9:.2f} G/s at 1980 MHz)")


if __name__ == "__main__":
    main()
