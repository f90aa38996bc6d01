"""Every C entry point the Python side binds (every function of include/vilbert_b200.h: vilbert_b200._lib.FUNCTIONS) is called by
name from a test that runs on the GPU, or is listed below with the test that covers it. A new entry point without a kernel test
then fails here, on any machine."""
import glob
import os
import re

from vilbert_b200 import _lib as L

TESTS = os.path.dirname(os.path.abspath(__file__))

# entry points reached through a wrapper rather than by name: {name: "test that covers it and how"}
COVERED_ELSEWHERE = {
    "vb_gemm_plan": "tests/test_host_cpu.py: host-only tile-plan query, no GPU work",
    "vb_version": "tests/test_host_cpu.py: the ABI version the library reports, no GPU work",
}


def _gpu_run_sources():
    files = sorted(glob.glob(os.path.join(TESTS, "test_*_gpu.py")))
    files += [os.path.join(TESTS, f) for f in ("test_optim.py", "test_radam.py", "_gpu_util.py")]
    return {os.path.basename(f): open(f).read() for f in files if os.path.exists(f)}


def test_every_header_function_has_a_gpu_test():
    sources = _gpu_run_sources()
    missing = [n for n in L.FUNCTIONS
               if n not in COVERED_ELSEWHERE and not any(re.search(rf"\b{n}\b", t) for t in sources.values())]
    assert not missing, f"entry points no GPU test calls: {missing}"


def test_covered_elsewhere_names_header_functions():
    """Each listed entry point still exists, and the test file named for it exists and mentions it or the wrapper that calls it."""
    for name, where in COVERED_ELSEWHERE.items():
        assert name in L.FUNCTIONS, name
        path = os.path.join(os.path.dirname(TESTS), where.split(":")[0])
        assert os.path.exists(path), (name, where)
        text = open(path).read()
        assert re.search(rf"\b{name}\b|FusedAdamW|FusedRAdam", text), (name, where)
