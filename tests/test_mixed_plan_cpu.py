"""CPU tier: the plan of a mixed-geometry range-proof call (bulletproofs_b200/csrc/rp_mixed.cuh, compiled into tests/host_emul) against a
Python model: per-proof parameter codes, class membership and order, segment offsets, S and D per class, the total number of MSM terms
and the global dynamic point indices, and the calls the plan refuses."""
import ctypes
import os
import random

import pytest

from oracle_binding import L_ORDER as l

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, VERIFICATION_ERROR, FORMAT_ERROR, INVALID_BITSIZE, INVALID_GENERATORS_LENGTH = 0, 1, 2, 3, 4
RP_CHUNK = 32
FIELDS = ["n", "m", "k", "S", "D", "count", "first", "seg", "dyn", "proof_off", "commit_off", "part_off"]


@pytest.fixture(scope="module")
def E(built):
    e = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    u64p = ctypes.POINTER(ctypes.c_uint64)
    e.emul_rp_mixed_plan.argtypes = [ctypes.c_size_t, ctypes.c_char_p, u64p, ctypes.POINTER(ctypes.c_uint32), u64p, ctypes.c_size_t, ctypes.c_size_t,
                                     ctypes.c_char_p, ctypes.POINTER(ctypes.c_uint32), u64p, u64p]
    return e


def plen(n, m):
    return 32 * (9 + 2 * ((n * m).bit_length() - 1))


def param_code(proof, n, m, cap, parties):
    """rp_param_verdict, then rp_rejected_proof_verdict (mod.rs:358-366, 497-538)"""
    L = len(proof)
    if L % 32 or L < 7 * 32:
        return FORMAT_ERROR
    ne = (L - 7 * 32) // 32
    if ne < 2 or (ne - 2) % 2 or (ne - 2) // 2 >= 32:
        return FORMAT_ERROR
    k = (ne - 2) // 2
    if n not in (8, 16, 32, 64):
        code = INVALID_BITSIZE
    elif cap < n or parties < m:
        code = INVALID_GENERATORS_LENGTH
    elif m == 0 or n * m != 1 << k or k > 20:
        code = VERIFICATION_ERROR
    else:
        return OK
    ab = 224 + 64 * k
    if any(int.from_bytes(proof[o:o + 32], "little") >= l for o in (128, 160, 192, ab, ab + 32)):
        return FORMAT_ERROR
    return code


def model(items, cap, parties):
    codes = [param_code(p, n, len(V) // 32, cap, parties) for p, V, n in items]
    keys, members = [], {}
    for i, (p, V, n) in enumerate(items):
        if codes[i] == OK:
            key = (n, len(V) // 32)
            if key not in members:
                keys.append(key)
                members[key] = []
            members[key].append(i)
    cls, order, seg, dyn, poff, coff, part = [], [], 0, 0, 0, 0, 0
    for n, m in keys:
        k = (n * m).bit_length() - 1
        S, D, cnt = 2 + 2 * n * m, 4 + 2 * k + m, len(members[(n, m)])
        cls.append(dict(n=n, m=m, k=k, S=S, D=D, count=cnt, first=len(order), seg=seg, dyn=dyn, proof_off=poff, commit_off=coff, part_off=part))
        order += members[(n, m)]
        seg += S + cnt * D
        dyn += cnt * D
        poff += cnt * plen(n, m)
        coff += cnt * m * 32
        part += -(-cnt // RP_CHUNK) * S
    return codes, order, cls, seg, dyn


def run_plan(E, items, cap, parties, poffs=None, coffs=None):
    count = len(items)
    u64 = ctypes.c_uint64
    if poffs is None:
        poffs = [0]
        for p, _, _ in items:
            poffs.append(poffs[-1] + len(p))
    if coffs is None:
        coffs = [0]
        for _, V, _ in items:
            coffs.append(coffs[-1] + len(V) // 32)
    blob = b"".join(p for p, _, _ in items) + bytes(64)
    codes = ctypes.create_string_buffer(max(count, 1))
    order = (ctypes.c_uint32 * max(count, 1))()
    cls = (u64 * (12 * max(count, 1)))()
    sums = (u64 * 4)()
    C = E.emul_rp_mixed_plan(count, blob, (u64 * (count + 1))(*poffs), (ctypes.c_uint32 * max(count, 1))(*[it[2] for it in items]), (u64 * (count + 1))(*coffs),
                             cap, parties, codes, order, cls, sums)
    if C < 0:
        return None
    A = sums[2]
    return (list(codes.raw[:count]), list(order[:A]), [dict(zip(FIELDS, cls[12 * c:12 * c + 12])) for c in range(C)], sums[0], sums[1], sums[3])


def proof(n, m, rnd, length=None, noncanonical=None):
    L = plen(n, m) if length is None else length
    b = bytearray(rnd.getrandbits(8) for _ in range(L))
    k = max(0, (L // 32 - 9) // 2)
    for o in (128, 160, 192, 224 + 64 * k, 256 + 64 * k):          # canonical scalars where a proof of this length has them
        if o + 32 <= L:
            b[o:o + 32] = (rnd.randrange(l)).to_bytes(32, "little")
    if noncanonical is not None:
        o = (128, 160, 192, 224 + 64 * k, 256 + 64 * k)[noncanonical]
        b[o:o + 32] = b"\xff" * 32
    return bytes(b)


def commitments(m, rnd):
    return bytes(rnd.getrandbits(8) for _ in range(32 * m))


def test_plan_matches_model_on_shuffled_classes(E):
    """every (n, m) of a 64 x 32 table, several proofs each, shuffled"""
    rnd = random.Random(5)
    items = [(proof(n, m, rnd), commitments(m, rnd), n) for n in (8, 16, 32, 64) for m in (1, 2, 4, 8, 16, 32) for _ in range(rnd.randrange(1, 4))]
    rnd.shuffle(items)
    codes, order, cls, terms, dyn, T0 = run_plan(E, items, 64, 32)
    want_codes, want_order, want_cls, want_terms, want_dyn = model(items, 64, 32)
    assert codes == want_codes == [OK] * len(items)
    assert order == want_order and sorted(order) == list(range(len(items)))
    assert cls == want_cls and len(cls) == 24
    assert (terms, dyn) == (want_terms, want_dyn)
    assert T0 == cls[0]["S"] + cls[0]["count"] * cls[0]["D"]
    # a term's dynamic point index is global: class c's proof q, point d is dyn_c + q*D_c + d, and the classes' points tile [0, dyn)
    ends = sorted((c["dyn"], c["dyn"] + c["count"] * c["D"]) for c in cls)
    assert ends[0][0] == 0 and ends[-1][1] == dyn and all(a[1] == b[0] for a, b in zip(ends, ends[1:]))
    segs = sorted((c["seg"], c["seg"] + c["S"] + c["count"] * c["D"]) for c in cls)
    assert segs[0][0] == 0 and segs[-1][1] == terms and all(a[1] == b[0] for a, b in zip(segs, segs[1:]))


def test_plan_per_proof_parameter_codes(E):
    """the rejected-parameter cases of a single-geometry call, one proof each, between admitted proofs of two classes"""
    rnd = random.Random(7)
    good = [(proof(64, 1, rnd), commitments(1, rnd), 64), (proof(32, 4, rnd), commitments(4, rnd), 32)]
    bad = [
        ((proof(8, 1, rnd), commitments(1, rnd), 12), INVALID_BITSIZE),                       # n = 12
        ((proof(8, 1, rnd), commitments(1, rnd), 128), INVALID_BITSIZE),
        ((proof(8, 64, rnd), commitments(64, rnd), 8), INVALID_GENERATORS_LENGTH),             # m above the table's parties
        ((proof(64, 1, rnd), commitments(1, rnd), 64), OK),                                    # rejected with a table of 32 generators
        ((proof(8, 4, rnd), commitments(3, rnd), 8), VERIFICATION_ERROR),                      # m = 3
        ((proof(8, 1, rnd), b"", 8), VERIFICATION_ERROR),                                      # m = 0
        ((proof(8, 32, rnd), commitments(16, rnd), 8), VERIFICATION_ERROR),                    # length of n*m = 256, verified as 128
        ((proof(8, 1, rnd, length=100), commitments(1, rnd), 8), FORMAT_ERROR),                # not a multiple of 32
        ((proof(8, 1, rnd, length=32 * 10), commitments(1, rnd), 8), FORMAT_ERROR),            # odd number of inner-product elements
        ((proof(8, 1, rnd, length=32 * 6), commitments(1, rnd), 8), FORMAT_ERROR),             # too short
        ((proof(8, 4, rnd, noncanonical=0), commitments(3, rnd), 8), FORMAT_ERROR),            # m = 3 and a non-canonical t_x
        ((proof(8, 1, rnd, noncanonical=4), commitments(1, rnd), 12), FORMAT_ERROR),           # n = 12 and a non-canonical b
        ((proof(8, 1, rnd, noncanonical=3), commitments(1, rnd), 8), OK),                      # admitted: the device decides
    ]
    for cap, parties in ((64, 32), (32, 32)):
        items = []
        for i, (it, _) in enumerate(bad):
            items += [good[i % 2], it]
        items += good
        codes, order, cls, terms, dyn, _ = run_plan(E, items, cap, parties)
        want_codes, want_order, want_cls, want_terms, want_dyn = model(items, cap, parties)
        assert (codes, order, cls, terms, dyn) == (want_codes, want_order, want_cls, want_terms, want_dyn)
        expect = [c for _, c in bad]
        if cap == 32:           # every n = 64 proof lacks generators now, the good ones included
            expect[3] = INVALID_GENERATORS_LENGTH
            assert [codes[2 * i] for i in range(len(bad))] == [INVALID_GENERATORS_LENGTH if i % 2 == 0 else OK for i in range(len(bad))]
        assert [codes[2 * i + 1] for i in range(len(bad))] == expect


def test_plan_with_every_proof_rejected(E):
    rnd = random.Random(9)
    items = [(proof(8, 1, rnd), commitments(1, rnd), 12), (proof(8, 4, rnd), commitments(3, rnd), 8)]
    codes, order, cls, terms, dyn, T0 = run_plan(E, items, 64, 32)
    assert codes == [INVALID_BITSIZE, VERIFICATION_ERROR] and order == [] and cls == [] and terms == dyn == T0 == 0


def test_plan_refuses_bad_offsets(E):
    rnd = random.Random(11)
    items = [(proof(8, 1, rnd), commitments(1, rnd), 8), (proof(8, 1, rnd), commitments(1, rnd), 8)]
    L = plen(8, 1)
    assert run_plan(E, items, 64, 32) is not None
    assert run_plan(E, [], 64, 32) is None                                           # no proofs
    assert run_plan(E, items, 64, 32, poffs=[32, L + 32, 2 * L + 32]) is None        # proof offsets not starting at 0
    assert run_plan(E, items, 64, 32, coffs=[1, 2, 3]) is None                       # commitment offsets not starting at 0
    assert run_plan(E, items, 64, 32, poffs=[0, L, L - 32]) is None                  # decreasing
    assert run_plan(E, items, 64, 32, coffs=[0, 2, 1]) is None
