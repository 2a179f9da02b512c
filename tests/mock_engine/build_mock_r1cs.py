"""Builds the TEST-ONLY mock engine with bp_r1cs_verify_batch (mock_r1cs.c: mock_bpmsm.c plus that entry point) and a copy of the C++
host mirror, r1cs::verify_batch included, linked against it.  Test infrastructure for tests/test_r1cs_batch.py, never used by the package."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
MOCK = os.path.join(HERE, "libmockbpmsm_r1cs.so")
HOST = os.path.join(HERE, "libbulletproofs_host_mock_r1cs.so")


def _stale(target, sources):
    return not os.path.exists(target) or any(os.path.getmtime(s) > os.path.getmtime(target) for s in sources)


def _run(cmd):
    print("+", " ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)


def build(force=False):
    odir, hdir, csrc = os.path.join(ROOT, "oracle"), os.path.join(ROOT, "bulletproofs_b200", "host"), os.path.join(ROOT, "bulletproofs_b200", "csrc")
    srcs = [os.path.join(HERE, f) for f in ("mock_r1cs.c", "mock_stubs.c")]
    deps = srcs + [os.path.join(HERE, "mock_bpmsm.c")] + [os.path.join(odir, f) for f in ("ge.h", "sc.h", "fe51.h", "hashes.h", "liboracle.so")] + [os.path.join(ROOT, "include", "bpmsm.h")]
    if force or _stale(MOCK, deps):
        _run(["gcc", "-O2", "-fPIC", "-shared", "-o", MOCK] + srcs + ["-L" + odir, "-loracle", "-Wl,-rpath,$ORIGIN/../../oracle"])
    hsrcs = [os.path.join(hdir, f) for f in ("bulletproofs.cpp", "r1cs.cpp", "r1cs_batch.cpp", "mpc.cpp")]
    hdeps = [os.path.join(hdir, f) for f in os.listdir(hdir)] + [os.path.join(csrc, f) for f in ("sc.cuh", "merlin.cuh", "fe.cuh")] + [MOCK]
    if force or _stale(HOST, hdeps):
        _run(["g++", "-O2", "-std=c++17", "-pthread", "-shared", "-fPIC", "-o", HOST] + hsrcs + ["-L" + HERE, "-lmockbpmsm_r1cs", "-Wl,-rpath,$ORIGIN"])
    return MOCK, HOST


if __name__ == "__main__":
    build(force=True)
