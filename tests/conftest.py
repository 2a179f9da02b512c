import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


# BP_TEST_MOCK_ENGINE=1 (set only by tests/test_host_mirror_cpu.py for its child process): the C++ host mirror and the Python binding run
# against tests/mock_engine (the oracle's CPU arithmetic behind the same C ABI), so that the mirror's own logic is exercised without a GPU.
# The product never does this: bulletproofs_b200 loads libbpmsm.so only.
MOCK_ENGINE = os.environ.get("BP_TEST_MOCK_ENGINE") == "1"
if MOCK_ENGINE:
    import bulletproofs_b200 as _bp
    _bp.LIB_PATH = os.path.join(ROOT, "tests", "mock_engine", "libmockbpmsm.so")
    _bp.HOST_LIB_PATH = os.path.join(ROOT, "tests", "mock_engine", "libbulletproofs_host_mock.so")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def built():
    """Make sure the oracle, the host-emulation library and the CUDA library exist (build is incremental)."""
    from bulletproofs_b200 import build as b
    b.build_oracle()
    b.build_emul()
    b.build_cuda()
    b.build_host()
    if MOCK_ENGINE:
        sys.path.insert(0, os.path.join(ROOT, "tests", "mock_engine"))
        import build_mock
        build_mock.build_mock_engine()
    return True


@pytest.fixture(scope="session")
def orc(built):
    from oracle_binding import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def golden():
    import json
    return json.load(open(os.path.join(ROOT, "tests", "golden", "range_proof_v1.json")))


@pytest.fixture(scope="session")
def gpu_ctx(built):
    import bulletproofs_b200 as bp
    ctx = bp.Context(0)           # raises if there is no H100: GPU tests must not pass on a fallback
    yield ctx
    ctx.close()
