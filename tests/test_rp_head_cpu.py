"""CPU tier: the device's range-proof head (rp_head_lean, specialised to k as k_rp_head_seq instantiates it, host build in
tests/host_emul/emul_head.cpp) against the sequential reference (rp_reduce_challenges + rp_scalars_head + rp_scalars_dynamic) on the
same challenge rows, and the built library's resource table: the head keeps every scalar in registers (no stack frame)."""
import ctypes
import os
import random
import re
import shutil
import subprocess

import pytest

from oracle_binding import L_ORDER as l

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RAW_U = 6                                   # rows y, z, x, w, c, rho, then u_0..u_{k-1}
ROW_Y, ROW_Z, ROW_RHO = 0, 1, 5


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    for f in (E.emul_rp_head_lean, E.emul_rp_head_ref):
        f.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_char_p]
    E.emul_rp_tab_size.argtypes = [ctypes.c_uint32, ctypes.c_uint32]; E.emul_rp_tab_size.restype = ctypes.c_uint32
    return E


def le(x, n=32):
    return x.to_bytes(n, "little")


def cells(k):
    """the (n, m) of the reference grid with n m = 2^k"""
    return [(n, (1 << k) // n) for n in (8, 16, 32, 64) if (1 << k) % n == 0 and 1 <= (1 << k) // n <= 32]


def fake_proof(rnd, k):
    """t_x, t_x_blinding, e_blinding, a, b canonical; the point encodings are not read by the head"""
    pb = bytearray(rnd.randbytes(32 * (9 + 2 * k)))
    for off in (128, 160, 192, 224 + 64 * k, 256 + 64 * k):
        pb[off:off + 32] = le(rnd.randrange(l))
    return bytes(pb)


def run(E, raw, proof, k, n, m):
    size = 32 * (3 + 4 + 2 * k + m + E.emul_rp_tab_size(k, m))
    a, b = ctypes.create_string_buffer(size), ctypes.create_string_buffer(size)
    sa = E.emul_rp_head_lean(raw, proof, k, n, m, a)
    sb = E.emul_rp_head_ref(raw, proof, k, n, m, b)
    return sa, sb, a.raw, b.raw


@pytest.mark.parametrize("k", range(3, 12))
def test_lean_head_matches_the_sequential_head(E, k):
    """zL, the base-point and blinding scalars, the D dynamic scalars and the nine tables, byte for byte, at every (n, m) with
    n m = 2^k; a zero y or u_j (a row of zeros, or l itself) rejects the proof in both; a zero rho weighs the proof with 1 in both."""
    rnd = random.Random(300 + k)
    zero_rows = [bytes(64), le(l) + bytes(32), le(l, 64)]
    for n, m in cells(k):
        for case in ("random", "random", "zero y", "zero u", "zero rho", "zero z", "top rows"):
            rows = [rnd.randbytes(64) for _ in range(RAW_U + k)]
            if case == "zero y": rows[ROW_Y] = rnd.choice(zero_rows)
            if case == "zero u": rows[RAW_U + rnd.randrange(k)] = rnd.choice(zero_rows)
            if case == "zero rho": rows[ROW_RHO] = rnd.choice(zero_rows)
            if case == "zero z": rows[ROW_Z] = bytes(64)
            if case == "top rows": rows = [b"\xff" * 64 for _ in rows]
            sa, sb, a, b = run(E, b"".join(rows), fake_proof(rnd, k), k, n, m)
            want_status = 1 if case in ("zero y", "zero u") else 0
            assert (sa, sb) == (want_status, want_status), (n, m, case)
            if want_status == 0:
                assert a == b, (n, m, case)


def test_lean_head_beyond_the_grid(E):
    """k up to 20 (n m = 2^20) has an instance too; two cells well past the grid"""
    rnd = random.Random(399)
    for k, n, m in ((14, 64, 256), (20, 16, 65536)):
        rows = b"".join(rnd.randbytes(64) for _ in range(RAW_U + k))
        sa, sb, a, b = run(E, rows, fake_proof(rnd, k), k, n, m)
        assert sa == sb == 0 and a == b, (k, n, m)


def test_head_kernel_has_no_stack_frame(built):
    """every k_rp_head_seq<K> instance of the built library keeps its scalars in registers: a stack frame here means an operand or a
    per-j array went through local memory again"""
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.exists(cuobjdump):
        cuobjdump = shutil.which("cuobjdump")
    assert cuobjdump, "cuobjdump (CUDA toolkit) is needed to read the resource table"
    out = subprocess.run([cuobjdump, "--dump-resource-usage", os.path.join(ROOT, "bulletproofs_b200", "libbpmsm.so")],
                         check=True, capture_output=True, text=True).stdout
    heads = {}
    for fn, body in re.findall(r"Function (\S+):\s*\n?\s*(REG:\d+ STACK:\d+[^\n]*)", out):
        mk = re.match(r"_Z\d+k_rp_head_seqILj(\d+)E", fn)
        if mk:
            heads[int(mk.group(1))] = int(re.search(r"STACK:(\d+)", body).group(1))
    assert sorted(heads) == list(range(3, 21)), sorted(heads)
    assert {k: s for k, s in heads.items() if s} == {}, "k_rp_head_seq instances with a stack frame"
