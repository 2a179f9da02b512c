"""CPU tier: the fit of a mixed-geometry range-proof call to a reserved mix (bulletproofs_b200/csrc/rp_mixed.cuh: rp_mixed_mix,
rp_mixed_fit, rp_mixed_slots, compiled into tests/host_emul) against a Python model: which calls fit, each class's slot base and live
count, the slot order of the gather table on shuffled inputs, and the mixes the reservation refuses."""
import ctypes
import os
import random

import pytest

from test_mixed_plan_cpu import commitments, model, proof

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TX = {(64, 1): 8, (64, 2): 4, (64, 4): 2, (64, 8): 1}


@pytest.fixture(scope="module")
def E(built):
    e = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    u32p, u64p = ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint64)
    e.emul_rp_mixed_fit.argtypes = [ctypes.c_size_t, u32p, u32p, u32p, ctypes.c_size_t, ctypes.c_char_p, u64p, u32p, u64p, ctypes.c_size_t, ctypes.c_size_t,
                                    u32p, u32p, u32p, u32p, ctypes.POINTER(ctypes.c_size_t)]
    return e


def run_fit(E, mix, items, cap=64, parties=32):
    """(rc, base, live, gather) with gather = [(input index, slot)]; rc as emul_rp_mixed_fit"""
    u32, u64 = ctypes.c_uint32, ctypes.c_uint64
    pairs = list(mix.items()) if isinstance(mix, dict) else list(mix)       # a list of ((n, m), capacity) may repeat a class
    C, count = len(pairs), len(items)
    keys = [key for key, _ in pairs]
    poffs, coffs = [0], [0]
    for p, V, _ in items:
        poffs.append(poffs[-1] + len(p))
        coffs.append(coffs[-1] + len(V) // 32)
    base, live = (u32 * max(C, 1))(), (u32 * max(C, 1))()
    src, slot, na = (u32 * max(count, 1))(), (u32 * max(count, 1))(), ctypes.c_size_t()
    rc = E.emul_rp_mixed_fit(C, (u32 * max(C, 1))(*[n for n, _ in keys]), (u32 * max(C, 1))(*[m for _, m in keys]), (u32 * max(C, 1))(*[c for _, c in pairs]),
                             count, b"".join(p for p, _, _ in items) + bytes(64), (u64 * (count + 1))(*poffs), (u32 * max(count, 1))(*[it[2] for it in items]),
                             (u64 * (count + 1))(*coffs), cap, parties, base, live, src, slot, ctypes.byref(na))
    if rc != 1:
        return rc, None, None, None
    return rc, list(base[:C]), list(live[:C]), list(zip(src[:na.value], slot[:na.value]))


def fit_model(mix, items, cap=64, parties=32):
    """None when the call does not fit, else (base, live, gather): class c's slots start after the capacities of the classes before it,
    and its admitted proofs take its first slots in input order"""
    codes, _, cls, _, _ = model(items, cap, parties)
    members = {}
    for i, (p, V, n) in enumerate(items):
        if codes[i] == 0:
            members.setdefault((n, len(V) // 32), []).append(i)
    if any(key not in mix or len(ids) > mix[key] for key, ids in members.items()):
        return None
    base, live, gather, b = [], [], [], 0
    for key, capacity in mix.items():
        ids = members.get(key, [])
        base.append(b)
        live.append(len(ids))
        gather += [(i, b + q) for q, i in enumerate(ids)]
        b += capacity
    return base, live, gather


def tx_items(rnd, counts):
    return [(proof(64, m, rnd), commitments(m, rnd), 64) for m, c in counts.items() for _ in range(c)]


def check(E, mix, items, fits=True, **kw):
    rc, base, live, gather = run_fit(E, mix, items, **kw)
    want = fit_model(mix, items, **kw)
    assert (rc == 1) == fits == (want is not None)
    if fits:
        assert (base, live, gather) == want
    return live


def test_full_and_partial_fill(E):
    rnd = random.Random(1)
    assert check(E, TX, tx_items(rnd, {1: 8, 2: 4, 4: 2, 8: 1})) == [8, 4, 2, 1]
    assert check(E, TX, tx_items(rnd, {1: 3, 2: 4, 4: 1, 8: 1})) == [3, 4, 1, 1]
    assert check(E, TX, tx_items(rnd, {1: 1})) == [1, 0, 0, 0]


def test_empty_class_fits(E):
    rnd = random.Random(2)
    assert check(E, TX, tx_items(rnd, {1: 5, 4: 2, 8: 1})) == [5, 0, 2, 1]


def test_unreserved_class_does_not_fit(E):
    rnd = random.Random(3)
    items = tx_items(rnd, {1: 2}) + [(proof(32, 2, rnd), commitments(2, rnd), 32)]
    check(E, TX, items, fits=False)


def test_one_proof_over_capacity_does_not_fit(E):
    rnd = random.Random(4)
    check(E, TX, tx_items(rnd, {1: 8, 2: 5}), fits=False)
    check(E, TX, tx_items(rnd, {1: 8, 2: 4, 4: 2, 8: 2}), fits=False)


def test_rejected_proofs_take_no_slot(E):
    """rejected proofs of an unreserved (n, m) or over a class's capacity leave the fit alone; every proof rejected fits, with no live proof"""
    rnd = random.Random(5)
    rejected = [(proof(8, 1, rnd), commitments(1, rnd), 12), (proof(8, 4, rnd), commitments(3, rnd), 8), (proof(64, 8, rnd), commitments(8, rnd), 64)]
    rejected[2] = (rejected[2][0][:-32], rejected[2][1], 64)          # no proof length: FormatError
    items = tx_items(rnd, {1: 8, 8: 1}) + rejected
    rnd.shuffle(items)
    assert check(E, TX, items) == [8, 0, 0, 1]
    assert check(E, TX, rejected) == [0, 0, 0, 0]


def test_gather_slot_order_on_shuffled_inputs(E):
    """every class of the 64 x 32 grid reserved in a shuffled order; proofs shuffled; classes partly filled, some empty"""
    rnd = random.Random(6)
    keys = [(n, m) for n in (8, 16, 32, 64) for m in (1, 2, 4, 8, 16, 32)]
    rnd.shuffle(keys)
    mix = {key: rnd.randrange(1, 6) for key in keys}
    for trial in range(5):
        items = [(proof(n, m, rnd), commitments(m, rnd), n) for (n, m), capacity in mix.items() for _ in range(rnd.randrange(0, capacity + 1))]
        rnd.shuffle(items)
        live = check(E, mix, items)
        assert sum(live) == len(items)


def test_mixes_the_reservation_refuses(E):
    rnd = random.Random(7)
    items = tx_items(rnd, {1: 1})
    assert run_fit(E, {}, items)[0] == -2                                            # no class
    assert run_fit(E, {(64, 1): 0}, items)[0] == -2                                  # zero capacity
    assert run_fit(E, {(12, 1): 4}, items)[0] == -2                                  # bit size the generators reject
    assert run_fit(E, {(64, 64): 4}, items)[0] == -2                                 # more parties than the table has
    assert run_fit(E, {(64, 1): 1 << 24}, items)[0] == -2                            # 2^24 proof slots
    assert run_fit(E, [((64, 1), 4), ((64, 2), 4), ((64, 1), 4)], items)[0] == -2     # a duplicate class
    assert run_fit(E, [((n, m), 1) for n in (8, 16, 32, 64) for m in (1, 2, 4, 8, 16, 32)] + [((64, 1), 1)], items)[0] == -2   # 25 classes
    assert run_fit(E, {(8, m): 1 for m in (1, 2, 4, 8, 16, 32)} | {(16, m): 1 for m in (1, 2, 4, 8, 16, 32)}
                   | {(32, m): 1 for m in (1, 2, 4, 8, 16, 32)} | {(64, m): 1 for m in (1, 2, 4, 8, 16, 32)}, items)[0] == 1       # 24 classes
    assert run_fit(E, {(64, 1): (1 << 24) - 1}, items)[0] == 1
