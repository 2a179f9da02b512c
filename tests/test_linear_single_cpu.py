"""CPU tier of the fused LinearProof path (k_lin_single, linear_single.cuh): its host part, compiled for the host by
tests/host_emul/emul_linear_single.cpp, against a Python restatement.

- The shared-memory layout of every k <= LIN_SINGLE_MAX_K, under its own plan and under the plan of any longer proof of the same launch,
  fits the per-block limit; LIN_SINGLE_MAX_K + 1 does not, so LIN_SINGLE_MAX_K is the largest k that fits.
- The regions, their sizes and order: window sums, the proof's points, the s tables, the recoded terms and the bucket lists.  The lists
  hold 15-bit term ids (the sign in bit 15), and a CTA's (window, bucket) threads fit its block.
- The routing rule at its edges."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32 = ctypes.c_uint32


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    E.emul_lin_single_consts.argtypes = [ctypes.POINTER(ctypes.c_uint64)]
    E.emul_lin_single_layout.argtypes = [U32, U32, ctypes.POINTER(U32), ctypes.POINTER(U32)]
    E.emul_lin_single_layout.restype = U32
    E.emul_lin_single_routed.argtypes = [ctypes.c_size_t, ctypes.c_size_t]
    return E


@pytest.fixture(scope="module")
def K(E):
    out = (ctypes.c_uint64 * 6)()
    E.emul_lin_single_consts(out)
    return dict(zip(("max_k", "max_count", "smem_limit", "route_count", "route_n", "threads"), out))


def layout(E, k, kmax):
    plan, lay = (U32 * 5)(), (U32 * 6)()
    T = E.emul_lin_single_layout(k, kmax, plan, lay)
    return T, dict(zip(("c", "W", "nb", "cl", "wpc"), plan)), dict(zip(("wsum", "niels", "tabs", "rec", "lists", "total"), lay))


def model(k, P):
    """the layout restated: (T, regions in order with their byte sizes)"""
    n, D = 1 << k, 2 + 2 * k
    T = n + 2 + D
    kl = (k + 1) // 2
    tab = (1 << kl) + (1 << (k - kl))
    return T, [("wsum", P["W"] * 128), ("niels", D * 96), ("tabs", tab * 32), ("rec", T * 36), ("lists", P["wpc"] * T * 2)]


def test_limits(K):
    assert K["smem_limit"] <= 227 * 1024
    assert 1 <= K["max_count"] <= 64 and K["max_k"] >= 10


@pytest.mark.parametrize("kmax", range(0, 14))
def test_every_layout_fits_up_to_max_k(E, K, kmax):
    T, P, L = layout(E, kmax, kmax)
    if kmax > K["max_k"]:
        assert L["total"] > K["smem_limit"], (kmax, L)          # the next k no longer fits
        return
    assert L["total"] <= K["smem_limit"], (kmax, L)
    # the plan: windows cover 255 bits, a window's buckets are whole lanes of one warp, a CTA's (window, bucket) threads fit its block,
    # and the cluster's CTAs own every window
    assert P["c"] * P["W"] >= 255 and P["nb"] == 1 << (P["c"] - 1) and 32 % P["nb"] == 0
    assert P["wpc"] * P["nb"] <= K["threads"] and P["wpc"] * P["cl"] >= P["W"]
    assert P["cl"] in (4, 8) and P["c"] == (5 if T <= 320 else 6)
    # term ids and their sign fit the 16-bit list entries
    assert T < 1 << 15
    for k in range(kmax + 1):
        Tk, Pk, Lk = layout(E, k, kmax)
        assert Pk == P
        Tm, regions = model(k, P)
        assert Tk == Tm
        o = 0
        for name, size in regions:
            assert Lk[name] == o, (k, kmax, name)
            o += size
        assert Lk["total"] == (o + 15) & ~15 and Lk["total"] <= L["total"]
        # the bucket lists of the CTA's windows hold every term once per window
        assert Lk["total"] - Lk["lists"] >= P["wpc"] * Tk * 2
        assert Lk["wsum"] % 16 == 0 and Lk["niels"] % 16 == 0 and Lk["tabs"] % 16 == 0 and Lk["rec"] % 4 == 0


def test_routing_edges(E, K):
    C, N = K["route_count"], K["route_n"]
    assert 1 <= C <= K["max_count"] and N <= 1 << K["max_k"]
    routed = lambda c, n: E.emul_lin_single_routed(c, n) == 1
    assert not routed(0, 1)
    assert routed(1, 1) and routed(1, N) and routed(C, 1) and routed(C, N)
    assert not routed(C + 1, 1) and not routed(1, 2 * N) and not routed(C + 1, N)
