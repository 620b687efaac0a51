#!/usr/bin/env python3
"""Are the device functions of two builds the same machine code?

    python tools/sass_diff.py <git-rev>          # build <git-rev>'s reth_b200/csrc in /tmp and compare with the working tree

Compiles both trees for sm_90a, dumps SASS with cuobjdump and compares every function of the OLD build instruction by
instruction (opcodes, operands and encodings; addresses, -lineinfo comments and column padding ignored; anonymous-
namespace name hashes normalised).  Used to show that kernels measured on the GPU are untouched by later work that
could only be checked under tools/emu."""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNITS = ["trie_kernels", "keccak_batch", "hash_sort", "engine"]
NVCC = ["nvcc", "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler",
        "-fPIC,-O3,-fvisibility=hidden"]


def build(src_root, out_dir):
    csrc = os.path.join(src_root, "reth_b200", "csrc")
    for u in UNITS:
        obj = os.path.join(out_dir, u + ".o")
        subprocess.run(NVCC + ["-I" + os.path.join(src_root, "include"), "-c", u + ".cu", "-o", obj], cwd=csrc, check=True,
                       capture_output=True)
        with open(os.path.join(out_dir, u + ".sass"), "w") as f:
            subprocess.run(["cuobjdump", "-sass", obj], stdout=f, check=True)


def functions(path):
    out, cur = {}, None
    for line in open(path):
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+", "ANON", m.group(1))
            out[cur] = []
            continue
        if cur is None:
            continue
        text = line.strip()
        if not text or text.startswith("//##"):
            continue
        text = re.sub(r"^/\*[0-9a-f]{4}\*/", "", text)
        out[cur].append(re.sub(r"\s+", " ", text).strip())
    return out


def main():
    rev = sys.argv[1]
    with tempfile.TemporaryDirectory() as tmp:
        old_src, old_out, new_out = (os.path.join(tmp, d) for d in ("src", "old", "new"))
        for d in (old_src, old_out, new_out):
            os.makedirs(d)
        tar = subprocess.run(["git", "archive", rev, "reth_b200/csrc", "include"], cwd=ROOT, check=True, capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", old_src], input=tar, check=True)
        build(old_src, old_out)
        build(ROOT, new_out)
        total = same = 0
        for u in UNITS:
            a, b = functions(os.path.join(old_out, u + ".sass")), functions(os.path.join(new_out, u + ".sass"))
            for name, body in a.items():
                total += 1
                if name not in b:
                    print(f"{u}: MISSING {name}")
                elif body != b[name]:
                    print(f"{u}: DIFFERENT {name} ({len(body)} vs {len(b[name])} lines)")
                else:
                    same += 1
            print(f"{u}: {len(a)} functions at {rev}, {len([k for k in b if k not in a])} new since")
        print(f"{same} of {total} device functions of {rev} are bit-identical in the working tree")
        return 0 if same == total else 1


if __name__ == "__main__":
    sys.exit(main())
