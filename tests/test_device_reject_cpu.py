"""CPU tier: the pass arithmetic of the exact entry points' device reject path (rp.cuh: rp_x_slice, rp_x_unit_live, rp_x_listed,
rp_x_clamp, rp_x_iters; host build in tests/host_emul/emul_exact.cpp) against a Python model: the failing-proof list over partial last
chunks and groups with fewer live proofs than slots, P at every admitted geometry up to n m = 2^20, and the bound on the level-2 loop."""
import ctypes
import os
import random

import pytest

from test_rp_large_cpu import admitted

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = 32                                  # RP_CHUNK
BUDGET = 1 << 18                            # RP_X_BUDGET


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    u32 = ctypes.c_uint32
    for name, args in (("emul_rp_x_slice", [u32, u32, u32]), ("emul_rp_x_clamp", [u32, u32]), ("emul_rp_x_iters", [u32, u32]),
                       ("emul_rp_x_list", [u32, u32, u32, ctypes.c_char_p, ctypes.POINTER(u32)])):
        getattr(E, name).argtypes = args
        getattr(E, name).restype = u32
    return E


def list_model(count, nbatch, live, fail):
    """the live proofs of the failing chunks, batch after batch: proof b count + q is live when b count + q < live"""
    nch = -(-count // CHUNK)
    return [b * count + q for b in range(nbatch) for q in range(count) if b * count + q < live and fail[b * nch + q // CHUNK]]


def run_list(E, count, nbatch, live, fail):
    out = (ctypes.c_uint32 * max(count * nbatch, 1))()
    n = E.emul_rp_x_list(count, nbatch, live, bytes(fail), out)
    return list(out[:n])


@pytest.mark.parametrize("count,nbatch", [(1, 1), (31, 1), (32, 1), (33, 1), (100, 3), (1024, 8), (70, 5)])
def test_failing_proof_list(E, count, nbatch):
    rnd = random.Random(count * 1000 + nbatch)
    nch = -(-count // CHUNK)
    total = count * nbatch
    patterns = [[0] * (nch * nbatch), [1] * (nch * nbatch), [1 if (i % nch) == nch - 1 else 0 for i in range(nch * nbatch)]]   # none, all, last chunks
    patterns += [[rnd.random() < 0.3 for _ in range(nch * nbatch)] for _ in range(5)]
    for fail in patterns:
        fail = [1 if f else 0 for f in fail]
        for live in sorted({total, max(total - 1, 0), total // 2, 1, 0, rnd.randrange(total + 1)}):
            got = run_list(E, count, nbatch, live, fail)
            assert got == list_model(count, nbatch, live, fail), (count, nbatch, live)
            assert len(got) <= live


def test_slice_every_admitted_geometry(E):
    """P = bp_recheck_slice(np, S + D, RP_X_BUDGET): at least one proof, at most np and 65535, and P (S + D) terms stay within the budget
    unless a single proof exceeds it"""
    for n, m in admitted():
        N = n * m
        k = N.bit_length() - 1
        S, D = 2 + 2 * N, 4 + 2 * k + m
        for np_ in (0, 1, 7, 32, 1000, 8192, 1 << 20):
            P = E.emul_rp_x_slice(np_, S, D)
            want = min(max(1, min(BUDGET // (S + D), 65535)), max(np_, 1))
            assert P == want, (n, m, np_, P, want)
            assert 1 <= P <= max(np_, 1)
            assert P * (S + D) <= BUDGET or P == 1


def test_iteration_bound(E):
    """the loop runs ceil(n / P) times over the clamped length, so a count the compaction could never leave (larger than the live proofs,
    or near 2^32) still gives at most ceil(live / P) iterations"""
    rnd = random.Random(7)
    for _ in range(2000):
        live = rnd.choice([0, 1, 31, 32, 33, 8192, rnd.randrange(1 << 24)])
        n = rnd.choice([0, live, live + 1, 2 * live + 5, 0xFFFFFFFF, rnd.randrange(1 << 32)])
        P = rnd.choice([1, 2, 7, 1783, 65535, rnd.randrange(1, 65536)])
        clamped = E.emul_rp_x_clamp(n, live)
        assert clamped == min(n, live)
        iters = E.emul_rp_x_iters(clamped, P)
        assert iters == -(-clamped // P)
        assert iters <= -(-live // P)
        assert (iters - 1) * P < clamped <= iters * P or clamped == iters == 0
    assert E.emul_rp_x_iters(0xFFFFFFFF, 1) == 0xFFFFFFFF and E.emul_rp_x_iters(0xFFFFFFFF, 2) == 1 << 31
