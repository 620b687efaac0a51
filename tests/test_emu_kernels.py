"""Kernel logic without a GPU: the CUDA sources of reth_b200/csrc, translated and run by tools/emu (fibers for the
threads of a block, yield-based barriers and warp collectives), pass the fast part of the `gpu` parity tests
bit-exact against the oracle and the golden vectors.

This is a check of the *sources* (indexing, masks, RLP assembly, barrier placement), not a product path: only this
test process points the loader at the emulated build (tests/conftest.py --emu); the GPU results come from the
`-m gpu` run of the very same tests on the real library."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAST = ("not one_million and not pipelined and not reentrancy and not frontier_sharding and not commits_blocks "
        "and not 200000 and not receipt_and_transaction_shaped and not persistent_waves and not large_block")


def test_cuda_sources_pass_parity_under_cpu_emulation():
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_trie.py", "tests/test_gpu_keccak.py",
                        "tests/test_gpu_host_mirror.py", "tests/test_gpu_dtrie.py", "tests/test_gpu_dstate.py", "tests/test_gpu_proofs.py",
                        "tests/test_gpu_zz_ordered_roots.py", "tests/test_gpu_zz_table_rows_device.py", "tests/test_gpu_level_classes.py",
                        "tests/test_gpu_leaf_widths.py", "tests/test_gpu_hash_sort_edges.py", "-m", "gpu", "--emu", "-q", "-x", "-k", FAST,
                        "-p", "no:cacheprovider"],
                       cwd=ROOT, capture_output=True, text=True, timeout=1500)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail


def test_dynamic_tries_two_stage_rehash_under_cpu_emulation():
    """The dynamic tries again on their large-block code paths, forced for every block size: the multi-launch restructure
    (B200_DT_FUSED_MAX=0; by default blocks up to 8192 entries are restructured by one CTA) and the thread-per-seed +
    warp-climb re-hash (B200_DT_TWO_STAGE_MIN=0; by default only dirty sets above 4096 entries take it)."""
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_dtrie.py", "tests/test_gpu_dstate.py", "-m", "gpu",
                        "--emu", "-q", "-x", "-p", "no:cacheprovider", "-k",
                        "random_blocks or shrink or clustered or sharded_state_matches or new_contract or lifecycle or inline_children"],
                       cwd=ROOT, capture_output=True, text=True, timeout=1500,
                       env=dict(os.environ, B200_DT_TWO_STAGE_MIN="0", B200_DT_FUSED_MAX="0"))
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail


def test_overlay_witness_and_stateless_paths_under_cpu_emulation():
    """tk_overlay.cuh, tk_witness.cuh and tk_stateless.cuh: the overlay roots, TrieUpdates, multiproofs and witnesses, the
    execution witness and the stateless roots, and tests/test_gpu_overlay_large.py, whose sizes follow the emulated
    threshold.  The six random-block cases of 3 000 accounts are left out (about 190 s of the run on an 8-core x86 host,
    where the rest takes about 8 minutes): test_gpu_overlay_large.py covers those paths at larger sizes."""
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_overlay.py", "tests/test_gpu_overlay_updates.py",
                        "tests/test_gpu_overlay_proofs.py", "tests/test_gpu_overlay_witness.py", "tests/test_gpu_witness.py",
                        "tests/test_gpu_stateless.py", "tests/test_gpu_overlay_large.py", "-m", "gpu", "--emu", "-q", "-x",
                        "-p", "no:cacheprovider", "-k", "not 3000"],
                       cwd=ROOT, capture_output=True, text=True, timeout=1500)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail


def test_cpp_host_mirror_under_cpu_emulation(tmp_path):
    """tests/cpp/host_test.cpp (reth's trie tests restated over the C++ host mirror) linked against the emulated build."""
    emu = os.path.join(ROOT, "tools", "emu")
    subprocess.run(["make", "-j8", "-C", emu], check=True, capture_output=True)
    import oracle
    oracle.build()
    exe = str(tmp_path / "host_test_emu")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "cpp", "host_test.cpp"), "-o", exe,
                        os.path.join(emu, "build", "libb200trie_emu.so"), os.path.join(ROOT, "oracle", "liboracle.so"),
                        "-Wl,-rpath," + os.path.join(emu, "build"), "-Wl,-rpath," + os.path.join(ROOT, "oracle")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=dict(os.environ, B200_EMU="1"))
    assert r.returncode == 0 and "all checks passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
