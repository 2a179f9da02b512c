"""CPU tier: the device planner of a mixed-length LinearProof call on device inputs (bulletproofs_b200/csrc/linear_mixed_device.cuh: the
per-proof and per-block steps of k_linm_admit, k_linm_scan and k_linm_place, compiled into tests/host_emul and run block by block)
against the host plan (linm_make_plan) and a Python model on the same calls: parameter codes, the (input, slot) pairs, gather entries and
live counts of calls that fit; exactly the later proofs of over-full classes and every proof of an unreserved n unplaced; counts around
the 256-proof block; offsets at odd byte offsets, not starting at 0; and the per-proof FormatError of bad offsets, without a read.
Also the refusals of the reserved mix itself (linm_mix)."""
import ctypes
import os
import random
import struct

import pytest

from test_linear_mixed_cpu import model_code, proof_bytes, run
from test_linear_verify_batch import FORMAT_ERROR, INVALID_GENERATORS_LENGTH, OK, VERIFICATION_ERROR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_SLOT = 0xFFFFFFFF
U32, U64, SZ = ctypes.c_uint32, ctypes.c_uint64, ctypes.c_size_t
SET_N = (1 << 10) + 2


@pytest.fixture(scope="module")
def E(built):
    e = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    u32p, u64p = ctypes.POINTER(U32), ctypes.POINTER(U64)
    e.emul_linm_plan.argtypes = [SZ, ctypes.c_char_p, u64p, u64p, SZ, ctypes.c_char_p, u32p, u64p, u64p]
    e.emul_linm_mix.argtypes = [SZ, u32p, u32p, SZ, u32p, u64p]
    e.emul_linm_mixed_place.argtypes = [SZ, u32p, u32p, SZ, SZ, ctypes.c_char_p, U64, ctypes.c_void_p, ctypes.c_void_p, U64, u32p, u32p, u32p, u64p]
    return e


def u32s(v):
    return (U32 * max(len(v), 1))(*v)


def mix_first(mix):
    first, out = 0, {}
    for n, cap in mix.items():
        out[n] = first
        first += cap
    return out, first


def device_place(E, mix, proofs, ns, set_n=SET_N, po=None, bo=None, shift=0, prefix=0, proof_bytes_=None, n_b=None):
    """(codes, slots, live, gather) of the device planner; the offset arrays start `shift` bytes into their buffers, the proofs after
    `prefix` bytes"""
    count = len(proofs)
    if po is None:
        po, bo = [prefix], [0]
        for p, n in zip(proofs, ns):
            po.append(po[-1] + len(p)); bo.append(bo[-1] + n)
    blob = bytes(prefix) + b"".join(proofs) + bytes(64)
    bufs = [ctypes.create_string_buffer(bytes(shift) + struct.pack(f"<{count + 1}Q", *o)) for o in (po, bo)]
    pa, ba = (ctypes.addressof(b) + shift for b in bufs)
    _, slots_total = mix_first(mix)
    codes, slots, live = (U32 * count)(), (U32 * count)(), (U32 * len(mix))()
    gather = (U64 * (3 * slots_total))(*([0xFFFFFFFFFFFFFFFF] * (3 * slots_total)))
    rc = E.emul_linm_mixed_place(len(mix), u32s(list(mix)), u32s(list(mix.values())), set_n, count, blob, po[-1] if proof_bytes_ is None else proof_bytes_,
                                 pa, ba, bo[-1] if n_b is None else n_b, codes, slots, live, gather)
    assert rc == 0
    return list(codes), list(slots), list(live), [tuple(gather[3 * s:3 * s + 3]) for s in range(slots_total)]


def model_place(mix, codes, ns):
    """the expected slot of every proof (NO_SLOT when rejected or unplaced) and live count per class"""
    first, _ = mix_first(mix)
    seen, slots = {}, []
    for code, n in zip(codes, ns):
        if code != OK or n not in mix or seen.get(n, 0) >= mix[n]:
            slots.append(NO_SLOT)
        else:
            slots.append(first[n] + seen.get(n, 0))
        if code == OK:
            seen[n] = seen.get(n, 0) + 1
    return slots, [min(seen.get(n, 0), cap) for n, cap in mix.items()]


class Pool:
    """a few proofs per rounds k, tiled (placement depends on lengths and a, r only); bad ones on request"""

    def __init__(self, seed):
        self.rnd = random.Random(seed)

    def item(self, n, **kw):
        k = max(n.bit_length() - 1, 0) if n else 0
        return proof_bytes(k, a=self.rnd.randrange(1, 1 << 250), r=self.rnd.randrange(1, 1 << 250), **kw), n


def check(E, mix, proofs, ns, **kw):
    codes, slots, live, gather = device_place(E, mix, proofs, ns, **kw)
    assert codes == [model_code(p, n, kw.get("set_n", SET_N))[0] for p, n in zip(proofs, ns)]
    want, wlive = model_place(mix, codes, ns)
    assert slots == want and live == wlive
    po, bo = [kw.get("prefix", 0)], [0]
    for p, n in zip(proofs, ns):
        po.append(po[-1] + len(p)); bo.append(bo[-1] + n)
    for i, s in enumerate(slots):
        if s != NO_SLOT:
            assert gather[s] == (po[i], bo[i], i)
    return codes, slots, live


def test_fitting_calls_match_the_host_plan(E):
    """a call that fits: the same codes as linm_make_plan, and each class's proofs, in the host plan's class order, take the mix's slots
    of their n in turn"""
    pool = Pool(1)
    mix = {64: 8, 256: 4, 1024: 2, 1: 3}
    for fill in ({64: 8, 256: 4, 1024: 2, 1: 3}, {64: 3, 256: 0, 1024: 1, 1: 1}, {64: 0, 256: 0, 1024: 1, 1: 0}):
        items = [pool.item(n) for n, c in fill.items() for _ in range(c)]
        random.Random(len(items)).shuffle(items)
        proofs, ns = [p for p, _ in items], [n for _, n in items]
        codes, slots, live = check(E, mix, proofs, ns)
        assert live == [fill[n] for n in mix]
        hcodes, order, cls, _ = run(E, proofs, ns, SET_N)
        assert codes == hcodes
        first, _ = mix_first(mix)
        pairs = sorted((order[K["first"] + j], first[K["n"]] + j) for K in cls for j in range(K["count"]))
        assert sorted((i, s) for i, s in enumerate(slots) if s != NO_SLOT) == pairs


def test_parameter_codes_among_placed_proofs(E):
    """rejected proofs take no slot and keep linm_make_plan's codes: bad lengths, non-canonical a or r, a set too short, n != 2^k"""
    pool, rnd = Pool(2), random.Random(2)
    mix = {1: 4, 16: 4, 64: 4, 1024: 4}
    items = [pool.item(n) for n in mix for _ in range(rnd.randrange(1, 5))]
    items += [pool.item(64, length=32 * 15 - 1), pool.item(64, length=64), (proof_bytes(4, a=(1 << 256) - 1), 16), (proof_bytes(6), 48),
              (proof_bytes(0), 0), (proof_bytes(10), 1024)]
    rnd.shuffle(items)
    proofs, ns = [p for p, _ in items], [n for _, n in items]
    codes, _, _ = check(E, mix, proofs, ns)
    assert codes == run(E, proofs, ns, SET_N)[0]
    assert codes.count(FORMAT_ERROR) == 3 and codes.count(VERIFICATION_ERROR) == 2
    short = check(E, {1: 4, 16: 4, 64: 4}, proofs, ns, set_n=66)[0]        # InvalidGeneratorsLength for every n above 64
    assert short == run(E, proofs, ns, 66)[0] and short.count(INVALID_GENERATORS_LENGTH) > 0


@pytest.mark.parametrize("count", [1, 255, 256, 257, 3000])
def test_overfull_and_unreserved_classes(E, count):
    """calls that do not fit, lengths interleaved across blocks: the unplaced proofs are exactly the later ones of over-full classes and
    every proof of an unreserved n"""
    pool, rnd = Pool(count), random.Random(count)
    mix = {64: max(1, count // 5), 256: max(1, count // 9), 1024: 3, 4: 2}
    lengths = list(mix) + [8, 512]
    items = [pool.item(rnd.choice(lengths)) if rnd.random() > 0.05 else (proof_bytes(3), 12) for _ in range(count)]
    proofs, ns = [p for p, _ in items], [n for _, n in items]
    codes, slots, live = check(E, mix, proofs, ns)
    assert all(s == NO_SLOT for c, s, n in zip(codes, slots, ns) if c == OK and n not in mix)


@pytest.mark.parametrize("count", [1, 255, 256, 257, 4100])
def test_block_boundaries(E, count):
    """fitting calls of every size around the block of 256 proofs, lengths interleaved"""
    pool, rnd = Pool(count + 7), random.Random(count + 7)
    mix = {2: count, 32: count, 128: count}
    items = [pool.item(rnd.choice(list(mix))) for _ in range(count)]
    codes, slots, live = check(E, mix, [p for p, _ in items], [n for _, n in items])
    assert sum(live) == count and NO_SLOT not in slots


def test_odd_offsets_not_starting_at_zero(E):
    """offset arrays at odd byte offsets of their buffers, proof offsets starting past a prefix: the same placement and gather entries"""
    pool, rnd = Pool(5), random.Random(5)
    mix = {16: 6, 256: 6}
    items = [pool.item(rnd.choice([16, 256])) for _ in range(10)]
    for shift, prefix in ((1, 3), (3, 0), (7, 13)):
        check(E, mix, [p for p, _ in items], [n for _, n in items], shift=shift, prefix=prefix)


def test_bad_offsets_are_per_proof_format_errors(E):
    """decreasing offsets and bytes past proof_bytes / n_b give that proof FormatError and no slot, and none of its bytes is read: the
    proof bytes beyond proof_bytes are a valid proof that would otherwise be admitted"""
    pool, base = Pool(9), 5
    items = [pool.item(64) for _ in range(7)]
    L = len(items[0][0])
    proofs = [p for p, _ in items]
    po, bo = [base + i * L for i in range(8)], [64 * i for i in range(8)]
    po[2] = base                    # proof 1 decreases; proof 2 spans three proofs' bytes (a wrong length)
    bo[4] = 64 * 7 + 1              # proof 3's b reaches past n_b = 448; proof 4's decreases
    codes, slots, live, _ = device_place(E, {64: 8}, proofs, [64] * 7, po=po, bo=bo, shift=3, prefix=base, proof_bytes_=base + 7 * L - 1, n_b=64 * 7)
    assert codes[2] != OK           # a parameter code, whichever the three proofs' bytes give
    assert codes[:2] + codes[3:] == [OK, FORMAT_ERROR, FORMAT_ERROR, FORMAT_ERROR, OK, FORMAT_ERROR]      # proof 6 ends past proof_bytes
    assert slots == [0, NO_SLOT, NO_SLOT, NO_SLOT, NO_SLOT, 1, NO_SLOT] and live == [2]


def mix_rc(E, ns, caps, set_n=SET_N):
    first, sums = (U32 * 32)(), (U64 * 2)()
    return E.emul_linm_mix(len(ns), u32s(ns), u32s(caps), set_n, first, sums), list(first[:len(ns)]), list(sums)


def test_mix_layout_and_refusals(E):
    rc, first, sums = mix_rc(E, [64, 1, 1024], [8, 3, 2])
    assert rc == 3 and first == [0, 8, 11] and sums == [13, 1024 + 2 + 8 * 14 + 3 * 2 + 2 * 22]
    assert mix_rc(E, [1 << k for k in range(21)], [1] * 21, set_n=(1 << 20) + 2)[0] == 21
    for ns, caps, set_n in (([], [], SET_N), ([1 << k for k in range(21)] + [3], [1] * 22, (1 << 20) + 2),      # 0 and 22 classes
                            ([64, 64], [1, 1], SET_N), ([0], [1], SET_N), ([48], [1], SET_N), ([1 << 21], [1], 1 << 22),
                            ([2048], [1], SET_N),                                                            # set shorter than n + 2
                            ([64], [0], SET_N), ([64], [(1 << 20) + 1], SET_N)):
        assert mix_rc(E, ns, caps, set_n)[0] == -1, (ns, caps)
