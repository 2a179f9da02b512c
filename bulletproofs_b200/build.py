"""In-tree builds: the sm_90a (H100) CUDA library (product), the C oracle and the host-emulation test library
(both test infrastructure).  nvcc cross-compiles without a GPU; the built .so files are git-ignored and
are rebuilt from source by build()."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bulletproofs_b200", "csrc")
LIB = os.path.join(ROOT, "bulletproofs_b200", "libbpmsm.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "--shared", "-Xcompiler", "-fPIC", "-diag-suppress", "177,550"]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _run(cmd, cwd=None):
    print("+", " ".join(cmd), flush=True)
    subprocess.run(cmd, cwd=cwd, check=True)


def build_cuda(force=False, verbose=False):
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "bpmsm.h")]
    if not force and _newer(LIB, srcs):
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = "nvcc"
    flags = NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else [])
    _run([nvcc] + flags + ["-o", LIB, os.path.join(CSRC, "bpmsm.cu")])
    return LIB


def build_host(force=False):
    """C++ mirror of the reference API (bulletproofs_b200/host), linked against libbpmsm.so"""
    hdir = os.path.join(ROOT, "bulletproofs_b200", "host")
    lib = os.path.join(ROOT, "bulletproofs_b200", "libbulletproofs_host.so")
    srcs = [os.path.join(hdir, f) for f in os.listdir(hdir)] + [os.path.join(CSRC, f) for f in ("sc.cuh", "merlin.cuh", "fe.cuh")] + [LIB]
    if force or not _newer(lib, srcs):
        _run(["g++", "-O2", "-std=c++17", "-pthread", "-shared", "-fPIC", "-o", lib, os.path.join(hdir, "bulletproofs.cpp"), os.path.join(hdir, "r1cs.cpp"),
              os.path.join(hdir, "r1cs_batch.cpp"), os.path.join(hdir, "mpc.cpp"),
              "-L" + os.path.join(ROOT, "bulletproofs_b200"), "-lbpmsm", "-Wl,-rpath,$ORIGIN"])
    return lib


def build_oracle(force=False):
    odir = os.path.join(ROOT, "oracle")
    lib = os.path.join(odir, "liboracle.so")
    srcs = [os.path.join(odir, f) for f in ("bp_oracle.c", "fe51.h", "sc.h", "ge.h", "hashes.h", "r1cs.h", "mpc.h")]
    if force or not _newer(lib, srcs):
        _run(["make", "-B", "-C", odir, "liboracle.so"])
    return lib


def build_emul(force=False):
    edir = os.path.join(ROOT, "tests", "host_emul")
    lib = os.path.join(edir, "libemul.so")
    cpps = [os.path.join(edir, f) for f in ("emul.cpp", "emul_r1cs.cpp", "emul_linear.cpp", "emul_transcript.cpp", "emul_head.cpp", "emul_mixed.cpp",
                                          "emul_decompress.cpp", "emul_debug.cpp", "emul_transcript_records.cpp",
                                          "emul_mixed_fit.cpp", "emul_tab_layout.cpp", "emul_mixed_place.cpp", "emul_exact.cpp",
                                          "emul_linear_device.cpp", "emul_linear_mixed.cpp", "emul_linear_mixed_place.cpp")]
    srcs = cpps + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    if force or not _newer(lib, srcs):
        _run(["g++", "-O2", "-std=c++17", "-pthread", "-shared", "-fPIC", "-o", lib] + cpps)
    return lib


if __name__ == "__main__":
    build_cuda(force="--force" in sys.argv, verbose="-v" in sys.argv)
    build_host()
    build_oracle()
    build_emul()
