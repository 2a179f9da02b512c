"""CPU tier: the device planner of a mixed call on device inputs (bulletproofs_b200/csrc/rp_mixed_device.cuh: the per-proof and per-block
steps of k_mix_admit, k_mix_scan and k_mix_place, compiled into tests/host_emul and run block by block) against the host planner
(rp_mixed_make_plan, rp_mixed_fit, rp_mixed_slots) on the same calls: parameter codes, live counts and (input, slot) pairs of calls that
fit; the unplaced proofs of calls that do not; the per-proof FormatError of bad offsets; and counts around the 256-proof block."""
import ctypes
import os
import random
import struct

import pytest

from test_mixed_plan_cpu import FORMAT_ERROR, OK, commitments, proof

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_SLOT = 0xFFFFFFFF
TX = {(64, 1): 8, (64, 2): 4, (64, 4): 2, (64, 8): 1}
CAP, PARTIES = 64, 32


@pytest.fixture(scope="module")
def E(built):
    e = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    u32p, u64p, sz = ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint64), ctypes.c_size_t
    e.emul_rp_mixed_place.argtypes = [sz, u32p, u32p, u32p, sz, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64,
                                      ctypes.c_void_p, sz, sz, u32p, u32p, u32p]
    e.emul_rp_mixed_host_place.argtypes = [sz, u32p, u32p, u32p, sz, ctypes.c_char_p, u64p, u32p, u64p, sz, sz, u32p, u32p, u32p, u32p, ctypes.POINTER(sz)]
    return e


def u32s(v):
    return (ctypes.c_uint32 * max(len(v), 1))(*v)


def mix_args(mix):
    keys = list(mix)
    return len(keys), u32s([n for n, _ in keys]), u32s([m for _, m in keys]), u32s([mix[k] for k in keys])


def offsets(items):
    poffs, coffs = [0], [0]
    for p, V, _ in items:
        poffs.append(poffs[-1] + len(p))
        coffs.append(coffs[-1] + len(V) // 32)
    return poffs, coffs


def device_place(E, mix, items, poffs=None, coffs=None, shift=0, prefix=0, proof_bytes=None, n_commit=None):
    """(codes, slots, live) of the device planner; the offset and n arrays start `shift` bytes into their buffers, the proofs after
    `prefix` bytes"""
    count = len(items)
    po, co = offsets(items)
    poffs, coffs = poffs or po, coffs or co
    proofs = bytes(prefix) + b"".join(p for p, _, _ in items) + bytes(64)
    bufs = [ctypes.create_string_buffer(bytes(shift) + b) for b in (struct.pack(f"<{count + 1}Q", *poffs), struct.pack(f"<{count}I", *[it[2] for it in items]),
                                                                     struct.pack(f"<{count + 1}Q", *coffs))]
    pa, na, ca = (ctypes.addressof(b) + shift for b in bufs)
    C, n, m, cap = mix_args(mix)
    codes, slots, live = (ctypes.c_uint32 * count)(), (ctypes.c_uint32 * count)(), (ctypes.c_uint32 * C)()
    rc = E.emul_rp_mixed_place(C, n, m, cap, count, proofs, po[-1] if proof_bytes is None else proof_bytes, pa, na, co[-1] if n_commit is None else n_commit,
                               ca, CAP, PARTIES, codes, slots, live)
    assert rc == 0
    return list(codes), list(slots), list(live)


def host_place(E, mix, items):
    """(rc, codes, live, pairs) of the host planner, rc as emul_rp_mixed_host_place"""
    count = len(items)
    poffs, coffs = offsets(items)
    C, n, m, cap = mix_args(mix)
    codes, live = (ctypes.c_uint32 * count)(), (ctypes.c_uint32 * C)()
    src, slot, na = (ctypes.c_uint32 * count)(), (ctypes.c_uint32 * count)(), ctypes.c_size_t()
    rc = E.emul_rp_mixed_host_place(C, n, m, cap, count, b"".join(p for p, _, _ in items) + bytes(64), (ctypes.c_uint64 * (count + 1))(*poffs),
                                    u32s([it[2] for it in items]), (ctypes.c_uint64 * (count + 1))(*coffs), CAP, PARTIES, codes, live, src, slot, ctypes.byref(na))
    return rc, list(codes), list(live), sorted(zip(src[:na.value], slot[:na.value]))


class Pool:
    """a few random proofs per (n, m), tiled: placement depends on the parameters only"""

    def __init__(self, seed):
        self.rnd, self.cache = random.Random(seed), {}

    def item(self, n, m, **kw):
        key = (n, m, tuple(sorted(kw.items())))
        if key not in self.cache:
            self.cache[key] = [(proof(n, m, self.rnd, **kw), commitments(m, self.rnd), n) for _ in range(3)]
        return self.rnd.choice(self.cache[key])


def check_fits(E, mix, items):
    codes, slots, live = device_place(E, mix, items)
    rc, hcodes, hlive, pairs = host_place(E, mix, items)
    assert rc == 1
    assert codes == hcodes and live == hlive
    assert sorted((i, s) for i, s in enumerate(slots) if s != NO_SLOT) == pairs
    return live


def test_fitting_calls_match_the_host_planner(E):
    pool = Pool(1)
    for fill in ({1: 8, 2: 4, 4: 2, 8: 1}, {1: 3, 2: 0, 4: 1, 8: 1}, {1: 0, 2: 0, 4: 0, 8: 1}):
        items = [pool.item(64, m) for m, c in fill.items() for _ in range(c)]
        random.Random(len(items)).shuffle(items)
        assert check_fits(E, TX, items) == [fill[m] for _, m in TX]


def test_fitting_calls_with_rejected_proofs(E):
    """rejected proofs take no slot and keep the host planner's codes, non-canonical scalars included"""
    pool, rnd = Pool(2), random.Random(2)
    mix = {(n, m): 6 for n in (8, 16, 32, 64) for m in (1, 2, 4, 8, 16, 32)}
    items = [pool.item(n, m) for (n, m) in mix for _ in range(rnd.randrange(0, 6))]
    items += [pool.item(64, 1, length=33), pool.item(12, 1), pool.item(64, 2, length=32 * 9), pool.item(64, 64), pool.item(8, 2, noncanonical=3),
              (proof(16, 4, rnd, noncanonical=0), commitments(0, rnd), 16)]
    rnd.shuffle(items)
    check_fits(E, mix, items)


def expected_unplaced(mix, items, codes):
    """admitted proofs of an unreserved class, and those past the capacity of theirs, in input order"""
    seen, out = {}, []
    for i, (p, V, n) in enumerate(items):
        if codes[i] != OK:
            continue
        key = (n, len(V) // 32)
        seen[key] = seen.get(key, 0) + 1
        if key not in mix or seen[key] > mix[key]:
            out.append(i)
    return out


@pytest.mark.parametrize("count", [1, 255, 256, 257, 3000])
def test_overfull_and_unreserved_classes(E, count):
    """calls that do not fit, classes interleaved across blocks: the unplaced proofs are exactly the later ones of over-full classes and
    every proof of an unreserved class; the others take the slots the host planner gives them once the excess is dropped"""
    pool, rnd = Pool(count), random.Random(count)
    mix = {(64, 1): max(1, count // 5), (64, 2): max(1, count // 9), (64, 4): 3, (32, 8): 2}
    keys = list(mix) + [(64, 8), (16, 2)]
    items = [pool.item(*rnd.choice(keys)) if rnd.random() > 0.05 else pool.item(12, 1) for _ in range(count)]
    codes, slots, live = device_place(E, mix, items)
    rc, hcodes, _, _ = host_place(E, mix, items)
    assert rc in (0, 1) and codes == hcodes
    unplaced = expected_unplaced(mix, items, codes)
    assert [i for i, s in enumerate(slots) if s == NO_SLOT and codes[i] == OK] == unplaced
    kept = [it for i, it in enumerate(items) if codes[i] == OK and i not in set(unplaced)]
    idx = [i for i in range(count) if codes[i] == OK and i not in set(unplaced)]
    if kept:
        rc, _, hlive, pairs = host_place(E, mix, kept)
        assert rc == 1 and live == hlive
        assert sorted((idx[j], s) for j, s in pairs) == sorted((i, slots[i]) for i in idx)


@pytest.mark.parametrize("count", [1, 255, 256, 257, 4100])
def test_block_boundaries(E, count):
    """fitting calls of every size around the block of 256 proofs, classes interleaved"""
    pool, rnd = Pool(count + 7), random.Random(count + 7)
    mix = {(64, 1): count, (64, 2): count, (16, 4): count}
    items = [pool.item(*rnd.choice(list(mix))) for _ in range(count)]
    check_fits(E, mix, items)


def test_bad_offsets_are_per_proof_format_errors(E):
    """decreasing offsets and bytes past proof_bytes / n_commitments give that proof FormatError and no slot; the offsets need not start
    at 0 and may sit at any alignment, and the other proofs are placed as usual"""
    pool, base = Pool(9), 5
    items = [pool.item(64, 1) for _ in range(7)]
    L = len(items[0][0])
    poffs, coffs = [base + i * L for i in range(8)], list(range(8))
    poffs[2] = base                 # proof 1 decreases; proof 2 spans three proofs' bytes (a wrong length)
    coffs[4] = 8                    # proof 3's commitments reach past n_commitments = 7; proof 4's decrease
    codes, slots, live = device_place(E, TX, items, poffs=poffs, coffs=coffs, shift=3, prefix=base, proof_bytes=base + 7 * L - 1, n_commit=7)
    assert codes[2] != OK           # a parameter code, whichever the three proofs' bytes give
    assert codes[:2] + codes[3:] == [OK, FORMAT_ERROR, FORMAT_ERROR, FORMAT_ERROR, OK, FORMAT_ERROR]      # proof 6 ends past proof_bytes
    assert slots == [0, NO_SLOT, NO_SLOT, NO_SLOT, NO_SLOT, 1, NO_SLOT] and live == [2, 0, 0, 0]
