"""CPU tier: the C++ host mirror of the reference API (bulletproofs_b200/host: RangeProof single and batched, InnerProductProof, LinearProof,
r1cs::{Prover,Verifier}, mpc::{Party,Dealer}) against the oracle, WITHOUT a GPU.

The mirror reaches the engine only through the C ABI of include/bpmsm.h.  tests/mock_engine implements that ABI on the oracle's CPU arithmetic
(test infrastructure, see its header); a child pytest process with BP_TEST_MOCK_ENGINE=1 binds the Python package and a copy of the mirror to it
and runs the mirror's own parity tests -- the ones the GPU tier runs against libbpmsm.so -- so that the mirror's transcript order, scalar algebra,
wire formats and error mapping are checked byte for byte on every CPU run.  The engine itself is not under test here (the -m gpu tier does that).
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIRROR_TESTS = ["tests/test_gpu_prover.py", "tests/test_linear_proof.py", "tests/test_mpc.py", "tests/test_r1cs.py"]


def test_host_mirror_against_oracle_through_the_mock_engine(built):
    sys.path.insert(0, os.path.join(ROOT, "tests", "mock_engine"))
    import build_mock
    build_mock.build_mock_engine()
    env = dict(os.environ, BP_TEST_MOCK_ENGINE="1")
    # the two largest R1CS sizes are left to the GPU tier (the mock's MSMs are single-threaded CPU code)
    r = subprocess.run([sys.executable, "-m", "pytest"] + MIRROR_TESTS + ["-m", "gpu", "-x", "-q", "-k", "not config5", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    tail = "\n".join(r.stdout.splitlines()[-15:])
    assert r.returncode == 0, tail + r.stderr[-2000:]
    assert " passed" in tail and "failed" not in tail, tail
    n_passed = int(tail.split(" passed")[0].split()[-1])
    assert n_passed >= 48, tail          # 29 prover/IPP (up to m = 32), 5 linear-proof, 6 MPC, 8 R1CS cases (incl. 2049 inputs = 4096 multipliers)


def test_package_never_points_at_the_mock_engine_by_default():
    """the product binds libbpmsm.so / libbulletproofs_host.so; the mock is reachable only through the test-only environment switch"""
    r = subprocess.run([sys.executable, "-c", "import bulletproofs_b200 as bp; print(bp.LIB_PATH); print(bp.HOST_LIB_PATH)"],
                       cwd=ROOT, env={k: v for k, v in os.environ.items() if k != "BP_TEST_MOCK_ENGINE"}, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    lib, host = r.stdout.split()
    assert lib.endswith("bulletproofs_b200/libbpmsm.so") and host.endswith("bulletproofs_b200/libbulletproofs_host.so")
    src = open(os.path.join(ROOT, "bulletproofs_b200", "__init__.py")).read() + open(os.path.join(ROOT, "bulletproofs_b200", "build.py")).read()
    assert "mock" not in src.lower()
