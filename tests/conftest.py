import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_addoption(parser):
    parser.addoption("--emu", action="store_true", default=False,
                     help="development aid: run the `gpu` tests against tools/emu's CPU emulation of the CUDA sources "
                          "(bit-exact logic check without a GPU; never used by the product or the driver)")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    if config.getoption("--emu"):
        import subprocess
        emu_dir = os.path.join(ROOT, "tools", "emu")
        build = os.environ.get("EMU_BUILD", "build")   # e.g. build_asan, made by hand (tools/emu/README.md)
        if build == "build":
            subprocess.run(["make", "-j8", "-C", emu_dir], check=True, capture_output=True)
        from reth_b200 import _lib
        _lib.LIB_PATH = os.path.join(emu_dir, build, "libb200trie_emu.so")   # test-side redirection only
        os.environ["B200_EMU"] = "1"


def pytest_collection_modifyitems(config, items):
    if not config.getoption("--emu"):
        return
    import inspect
    for item in items:
        reason = None
        src = inspect.getsource(item.function) if hasattr(item, "function") else ""
        if "torch" in src:
            reason = "needs torch CUDA tensors"
        elif item.fspath.basename in ("test_gpu_fullsize.py", "test_cpp_host.py"):
            reason = "full-size / native-binary test"
        if reason:
            item.add_marker(pytest.mark.skip(reason="--emu: " + reason))


@pytest.fixture(scope="session")
def golden_allocs():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "genesis_allocs.json")) as f:
        return json.load(f)
