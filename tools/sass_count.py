#!/usr/bin/env python3
"""ALU-pipe instructions per digest of keccak256_fixed32_kernel, counted from its SASS (the constant behind `alu_frac` in
bench.py):   python tools/sass_count.py
The kernel is a grid-stride loop whose body is: loads + the peeled first round (`pre`), a 22-trip loop of one round each
(`loop`), the peeled last round + stores (`post`).  LOP3 / SHF / ISETP / VIADD / LEA / IADD3 / SEL issue to the ALU pipe
(64 lanes/clk/SM on compute capability 9.0); IMAD / MOV go to the FMA pipe, LDG / STG to the LSU."""
import collections
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "reth_b200", "csrc", "build", "keccak_batch.o")
FUN = "_ZN4b20024keccak256_fixed32_kernelILi256EEEvPKhjmP5uint4"
ALU = ("LOP3", "SHF", "ISETP", "VIADD", "LEA", "IADD3", "SEL", "PRMT", "IADD")


def main():
    txt = subprocess.run(["cuobjdump", "-sass", "-fun", FUN, OBJ], capture_output=True, text=True, check=True).stdout
    ins = []
    for l in txt.splitlines():
        l = l.strip()
        if not l.startswith("/*") or "*/" not in l[2:]:
            continue
        try:
            a = int(l[2:l.index("*/")], 16)
        except ValueError:
            continue
        rest = l[l.index("*/") + 2:].split("/*")[0].strip().rstrip(";").split()
        if not rest:
            continue
        op = rest[1] if rest[0].startswith("@") else rest[0]
        target = None
        if op.startswith("BRA") and rest[-1].startswith("0x"):
            target = int(rest[-1], 16)
        ins.append((a, op.split(".")[0], target))
    back = [(a, t) for a, o, t in ins if o == "BRA" and t is not None and t < a]
    (loop_end, loop_start) = min(back, key=lambda x: x[0] - x[1])          # the innermost backward branch: the round loop
    pre = [o for a, o, _ in ins if a < loop_start]
    loop = [o for a, o, _ in ins if loop_start <= a <= loop_end]
    outer_end = max(a for a, o, t in ins if o == "BRA" and t is not None and t < a)
    post = [o for a, o, _ in ins if loop_end < a <= outer_end]
    n_alu = lambda ops: sum(o in ALU for o in ops)
    c = lambda ops: dict(collections.Counter(ops).most_common(6))
    print(f"keccak256_fixed32_kernel<256>: {len(ins)} SASS instructions")
    print(f"  before the round loop (loads, peeled round 0): {len(pre)} instr, {n_alu(pre)} ALU  {c(pre)}")
    print(f"  round loop body (x22):                          {len(loop)} instr, {n_alu(loop)} ALU  {c(loop)}")
    print(f"  after it (peeled round 23, stores, loop control): {len(post)} instr, {n_alu(post)} ALU  {c(post)}")
    total, alu = len(pre) + 22 * len(loop) + len(post), n_alu(pre) + 22 * n_alu(loop) + n_alu(post)
    print(f"per digest: {total} instructions, {alu} on the ALU pipe")
    print(f"ALU ceiling per SM: {64 / alu * 1e3:.3f} digests per 1000 clocks (x 132 SMs x SM clock on an H100 SXM)")


if __name__ == "__main__":
    main()
