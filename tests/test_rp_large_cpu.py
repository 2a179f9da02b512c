"""CPU tier: k_rp_decompress's shared-memory stage (rp_dec_block, rp_dec_offset, rp_dec_smem_bytes in rp.cuh, host build in
tests/host_emul/emul_decompress.cpp) at every geometry the verifier admits, n in {8, 16, 32, 64} and m = 2^j with n m <= 2^20.  A block
stages the proofs it touches and the commitments of its own points only, so the stage stays within what an H100 block can have whatever m
is; each point's encoding comes from the byte the naive proof + 32 idx / L_j / R_j / V_j address names."""
import ctypes
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_LG_N = 20                               # BP_MAX_LG_N
H100_SMEM_PER_BLOCK = 227 * 1024            # cudaDevAttrMaxSharedMemoryPerBlockOptin on an H100
COMMIT = 1 << 63                            # emul_rp_dec_sources: a source in the commitment array


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    E.emul_rp_dec_smem.argtypes = [ctypes.c_uint32, ctypes.c_uint32]; E.emul_rp_dec_smem.restype = ctypes.c_uint32
    E.emul_rp_dec_smem_max.restype = ctypes.c_uint32
    E.emul_rp_dec_sources.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p]
    E.emul_rp_dec_sources.restype = ctypes.c_uint32
    return E


def admitted():
    return [(n, 1 << j) for n in (8, 16, 32, 64) for j in range(0, MAX_LG_N + 1) if n << j <= 1 << MAX_LG_N]


def test_stage_fits_the_attribute_and_the_sm(E):
    """the size every launch asks for is at most the limit bp_ctx_create sets, and that limit is at most what an H100 block can have"""
    attr = E.emul_rp_dec_smem_max()
    assert attr <= H100_SMEM_PER_BLOCK, attr
    sizes = {(n, m): E.emul_rp_dec_smem(n, m) for n, m in admitted()}
    over = {nm: s for nm, s in sizes.items() if s > attr or s > H100_SMEM_PER_BLOCK}
    assert not over, (attr, over)
    assert attr == max(sizes.values())
    assert len(sizes) == 18 + 17 + 16 + 15         # m from 1 to 2^20 / n for each n


def naive_sources(n, m, count):
    """byte offset of point i's encoding in the proof array, or COMMIT | offset in the commitment array"""
    k = (n * m).bit_length() - 1
    D, plen = 4 + 2 * k + m, 32 * (9 + 2 * k)
    i = np.arange(count * D, dtype=np.uint64)
    p, idx = i // np.uint64(D), i % np.uint64(D)
    base = p * np.uint64(plen)
    out = np.where(idx < 4, base + 32 * idx, np.uint64(0))
    lr = idx - np.uint64(4)
    out = np.where((idx >= 4) & (idx < 4 + k), base + np.uint64(224) + 64 * lr, out)
    out = np.where((idx >= 4 + k) & (idx < 4 + 2 * k), base + np.uint64(224 + 32) + 64 * (lr - np.uint64(k)), out)
    v = p * np.uint64(m) + (idx - np.uint64(4 + 2 * k))
    return np.where(idx >= 4 + 2 * k, np.uint64(COMMIT) | (32 * v), out)


@pytest.mark.parametrize("n,m", [(64, 1), (8, 1), (8, 64), (8, 128), (8, 2048), (64, 16384), (8, 131072)])
@pytest.mark.parametrize("count", [1, 3, 40])
def test_every_point_reads_its_own_bytes(E, n, m, count):
    """every block of the launch: what it stages stays inside its bounds, and each point reads the bytes of its own field.  D = 4+2k+m
    points per proof: (8, 64) and (8, 128) put D just below and just above one block of 128 points"""
    D = 4 + 2 * ((n * m).bit_length() - 1) + m
    got = np.zeros(count * D, dtype=np.uint64)
    assert E.emul_rp_dec_sources(n, m, count, got.ctypes.data) == 0, "a block reads outside its stage"
    want = naive_sources(n, m, count)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(int(i), int(i) // D, int(i) % D, hex(int(got[i])), hex(int(want[i]))) for i in bad[:5]]
