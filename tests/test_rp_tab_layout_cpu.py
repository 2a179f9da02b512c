"""CPU tier: the chunk-major layout of the range-proof head's product tables (rp.cuh: rp_tab_index, rp_tab_slice, host build in
tests/host_emul/emul_tab_layout.cpp).  The head writes a proof of any slice position through the addressing function, touches no other
slot and reads back what the sequential reference computes; the fixed-geometry, mixed and reject-path slices give every (proof, entry)
a distinct slot inside their allocation, the last partial chunk included; and k_rp_scalars_sum, like k_rp_head_seq, has no stack frame."""
import ctypes
import os
import random
import re
import shutil
import subprocess

import pytest

from test_rp_head_cpu import RAW_U, cells, fake_proof

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = 32
U32P, U64P = ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint64)


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    E.emul_rp_head_ref.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_char_p]
    E.emul_rp_head_slice.argtypes = [ctypes.c_char_p, ctypes.c_char_p] + [ctypes.c_uint32] * 5 + [ctypes.c_char_p]
    E.emul_rp_tab_size.argtypes = [ctypes.c_uint32, ctypes.c_uint32]; E.emul_rp_tab_size.restype = ctypes.c_uint32
    E.emul_rp_tab_slice.argtypes = [ctypes.c_uint32] * 3; E.emul_rp_tab_slice.restype = ctypes.c_uint64
    E.emul_rp_tab_slot.argtypes = [ctypes.c_uint32] * 4; E.emul_rp_tab_slot.restype = ctypes.c_uint64
    E.emul_rp_sum_indices.argtypes = [ctypes.c_uint32] * 3 + [U32P]; E.emul_rp_sum_indices.restype = ctypes.c_uint32
    E.emul_rp_mix_tab_slices.argtypes = [ctypes.c_uint32, U32P, U32P, U32P, U64P, U64P, U32P, U32P]
    E.emul_rp_mix_tab_slices.restype = ctypes.c_uint64
    return E


def slots(E, count, k, m):
    """the slot of every (proof, entry) of a slice of count proofs, in (proof, entry) order"""
    tsz = E.emul_rp_tab_size(k, m)
    return [E.emul_rp_tab_slot(p, e, k, m) for p in range(count) for e in range(tsz)]


def assert_distinct_inside(E, count, k, m):
    size = E.emul_rp_tab_slice(count, k, m)
    assert size == -(-count // CHUNK) * CHUNK * E.emul_rp_tab_size(k, m)
    s = slots(E, count, k, m)
    assert len(set(s)) == len(s), (count, k, m)
    assert max(s) < size, (count, k, m)


@pytest.mark.parametrize("k", [3, 6, 9])
def test_head_writes_its_own_entries_at_any_slice_position(E, k):
    """the head through rp_tab_proof with entries RP_CHUNK apart: the first, a middle and the last proof of a slice ending in a partial
    chunk; the values equal the sequential head's, and every other slot of the slice keeps its marker"""
    rnd = random.Random(700 + k)
    for n, m in cells(k)[:2]:
        D = 4 + 2 * k + m
        size = 32 * (3 + D + E.emul_rp_tab_size(k, m))
        for count, p in ((1, 0), (45, 0), (45, 33), (45, 44), (64, 31)):
            raw = b"".join(rnd.randbytes(64) for _ in range(RAW_U + k))
            proof = fake_proof(rnd, k)
            a, b = ctypes.create_string_buffer(size), ctypes.create_string_buffer(size)
            assert E.emul_rp_head_slice(raw, proof, k, n, m, count, p, a) == 0, (n, m, count, p)
            assert E.emul_rp_head_ref(raw, proof, k, n, m, b) == 0
            assert a.raw == b.raw, (n, m, count, p)


@pytest.mark.parametrize("count", [1, 31, 32, 33, 64, 97])
def test_fixed_slices_give_distinct_slots(E, count):
    """every (proof, entry) of a fixed-geometry group of count proofs has its own slot inside rp_tab_slice, at k = 3, 6 and 8"""
    for k, m in ((3, 1), (6, 1), (8, 4)):
        assert_distinct_inside(E, count, k, m)


def test_large_k_slot_bounds(E):
    """k = 20 (9216 entries per proof): the first and last entries of the first and last proofs of a 33-proof slice"""
    k, m = 20, 16384
    tsz, size = E.emul_rp_tab_size(k, m), E.emul_rp_tab_slice(33, k, m)
    assert tsz == 9216 and size == 64 * tsz
    got = [E.emul_rp_tab_slot(p, e, k, m) for p in (0, 31, 32) for e in (0, tsz - 1)]
    assert got == [0, (tsz - 1) * CHUNK, 31, (tsz - 1) * CHUNK + 31, CHUNK * tsz, CHUNK * tsz + (tsz - 1) * CHUNK]
    assert max(got) < size


@pytest.mark.parametrize("count,nbatch", [(1024, 8), (45, 3), (32, 2), (1, 5), (97, 1)])
def test_sums_read_the_slots_the_head_wrote(E, count, nbatch):
    """k_rp_scalars_sum's blocks read each proof of the group once, at the slice index the head wrote it to (its group index); the
    reject path's one-proof geometry over the proofs [p0, p0 + n) (a failing chunk, the last partial one, or the whole batch) with
    tab_p0 = p0 reads the same indices"""
    total = count * nbatch
    nch = -(-count // CHUNK)
    idx = (ctypes.c_uint32 * (nbatch * nch * CHUNK))(*([0xffffffff] * (nbatch * nch * CHUNK)))
    assert E.emul_rp_sum_indices(count, nbatch, 0, idx) == nbatch * nch
    got = sorted(v for v in idx if v != 0xffffffff)
    assert got == list(range(total))
    for batch in {0, nbatch - 1}:
        ranges = [(batch * count + ch * CHUNK, min(CHUNK, count - ch * CHUNK)) for ch in {0, nch - 1}] + [(batch * count, count)]
        for p0, n in ranges:
            one = (ctypes.c_uint32 * (n * CHUNK))(*([0xffffffff] * (n * CHUNK)))
            assert E.emul_rp_sum_indices(1, n, p0, one) == n
            assert [one[b * CHUNK] for b in range(n)] == list(range(p0, p0 + n)), (p0, n)


@pytest.mark.parametrize("seed", range(4))
def test_mixed_class_slices_are_whole_chunks(E, seed):
    """a reserved mix of classes of any size: every class's slice starts where the one before ends, holds whole chunks, and the
    slots of its proofs lie inside it; the slices are disjoint and fill the arena"""
    rnd = random.Random(900 + seed)
    grid = [(n, m) for n in (8, 16, 32, 64) for m in (1, 2, 4, 8)]
    classes = rnd.sample(grid, rnd.randint(1, 6))
    C = len(classes)
    n = (ctypes.c_uint32 * C)(*[c[0] for c in classes]); m = (ctypes.c_uint32 * C)(*[c[1] for c in classes])
    cap = (ctypes.c_uint32 * C)(*[rnd.choice([1, 5, 31, 32, 33, 70]) for _ in classes])
    off, ln = (ctypes.c_uint64 * C)(), (ctypes.c_uint64 * C)()
    cnt, tsz = (ctypes.c_uint32 * C)(), (ctypes.c_uint32 * C)()
    total = E.emul_rp_mix_tab_slices(C, n, m, cap, off, ln, cnt, tsz)
    assert total > 0
    end = 0
    for c in range(C):
        assert off[c] == end, (c, classes)
        assert ln[c] == -(-cnt[c] // CHUNK) * CHUNK * tsz[c]
        k = (n[c] * m[c]).bit_length() - 1
        s = slots(E, cnt[c], k, m[c])
        assert len(set(s)) == len(s) and max(s) < ln[c], (c, classes)
        end += ln[c]
    assert end == total


def test_sums_kernel_has_no_stack_frame(built):
    """k_rp_scalars_sum keeps the entries of the proofs it has in flight in registers: a stack frame here means the prefetch spilled"""
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.exists(cuobjdump):
        cuobjdump = shutil.which("cuobjdump")
    assert cuobjdump, "cuobjdump (CUDA toolkit) is needed to read the resource table"
    out = subprocess.run([cuobjdump, "--dump-resource-usage", os.path.join(ROOT, "bulletproofs_b200", "libbpmsm.so")],
                         check=True, capture_output=True, text=True).stdout
    found = [(fn, body) for fn, body in re.findall(r"Function (\S+):\s*\n?\s*(REG:\d+ STACK:\d+[^\n]*)", out) if re.match(r"_Z\d+k_rp_scalars_sum", fn)]
    assert len(found) == 1, found
    assert int(re.search(r"STACK:(\d+)", found[0][1]).group(1)) == 0
    assert int(re.search(r"REG:(\d+)", found[0][1]).group(1)) <= 128
