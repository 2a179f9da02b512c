"""CPU tier of the mixed-length LinearProof call (bp_linear_verify_mixed): its host plan (linear_mixed.cuh), compiled for the host by
tests/host_emul/emul_linear_mixed.cpp, against a Python restatement.

- Per-proof parameter codes in the reference's order: a length no proof can have, then a non-canonical a or r (FormatError, whatever the
  other parameters), a set of fewer than n + 2 points (InvalidGeneratorsLength), n != 2^rounds and n = 0 (VerificationError).
- Classes: one per n among the admitted proofs, in the order of their first proof, proofs in input order within a class.
- Every class's arena offsets, its first G-sum chunk and dynamic-point base, and the totals, with the combined row's Nmax + 2 + sum D terms.
- Refusals: no proof, more than 2^20, offsets that do not start at 0 or that decrease, an n above 2^20, and 2^31 MSM terms or more."""
import ctypes
import os
import random

import pytest

from oracle_binding import L_ORDER as l
from test_linear_verify_batch import FORMAT_ERROR, INVALID_GENERATORS_LENGTH, OK, VERIFICATION_ERROR, le

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("n", "k", "first", "count", "proof_len", "D", "chunk0", "tiles", "proof_off", "b_off", "raw_off", "tab_off", "part_off", "b0_off", "dyn")
SUMS = ("nmax", "chunks", "terms", "dyn_points", "proof_bytes", "b_scalars", "raw_rows", "tab_scalars", "part_scalars", "b0_scalars")
CHUNK, TILE = 32, 128
U64 = ctypes.c_uint64


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    E.emul_linm_plan.argtypes = [ctypes.c_size_t, ctypes.c_char_p, ctypes.POINTER(U64), ctypes.POINTER(U64), ctypes.c_size_t, ctypes.c_char_p,
                                 ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(U64), ctypes.POINTER(U64)]
    E.emul_linm_layout.argtypes = [ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(U64), ctypes.POINTER(U64)]
    return E


def proof_bytes(k, a=1, r=2, length=None):
    """a proof of k rounds (points are never decoded by the plan) with the given a and r; length: cut or padded to that many bytes"""
    p = bytes(range(64)) * k + bytes(32) + le(a) + le(r)
    return p if length is None else (p + bytes(length))[:length]


def run(E, proofs, ns, set_n, offsets=None):
    count = len(proofs)
    po, bo = [0], [0]
    for p, n in zip(proofs, ns):
        po.append(po[-1] + len(p)); bo.append(bo[-1] + n)
    if offsets:
        po, bo = offsets(po, bo)
    codes = ctypes.create_string_buffer(max(count, 1)); order = (ctypes.c_uint32 * max(count, 1))()
    cls = (U64 * (len(FIELDS) * 21))(); sums = (U64 * len(SUMS))()
    C = E.emul_linm_plan(count, b"".join(proofs) + bytes(1), (U64 * len(po))(*po), (U64 * len(bo))(*bo), set_n, codes, order, cls, sums)
    if C < 0:
        return None
    codes = list(codes.raw[:count])
    return codes, list(order[:codes.count(OK)]), [dict(zip(FIELDS, cls[len(FIELDS) * c:len(FIELDS) * (c + 1)])) for c in range(C)], dict(zip(SUMS, sums))


def model_code(p, n, set_n):
    ne = len(p) // 32
    if len(p) % 32 or ne < 3 or (ne - 3) % 2 or (ne - 3) // 2 >= 32:
        return FORMAT_ERROR, None
    k = (ne - 3) // 2
    a, r = int.from_bytes(p[64 * k + 32:64 * k + 64], "little"), int.from_bytes(p[64 * k + 64:64 * k + 96], "little")
    if a >= l or r >= l:
        return FORMAT_ERROR, k
    if set_n < n + 2:
        return INVALID_GENERATORS_LENGTH, k
    if n != 1 << k:
        return VERIFICATION_ERROR, k
    return OK, k


def tab_size(k):
    kl = (k + 1) // 2
    return (1 << kl) + (1 << (k - kl))


def model_layout(classes):
    """classes: [(n, k, count)] in order -> (per-class dicts, sums)"""
    out, s = [], dict.fromkeys(SUMS, 0)
    first = 0
    for n, k, count in classes:
        D, nch, tiles = 2 + 2 * k, -(-count // CHUNK), -(-n // TILE)
        out.append(dict(n=n, k=k, first=first, count=count, proof_len=32 * (2 * k + 3), D=D, chunk0=s["chunks"], tiles=tiles, proof_off=s["proof_bytes"],
                        b_off=s["b_scalars"], raw_off=s["raw_rows"], tab_off=s["tab_scalars"], part_off=s["part_scalars"], b0_off=s["b0_scalars"],
                        dyn=s["dyn_points"]))
        s["proof_bytes"] += count * 32 * (2 * k + 3); s["b_scalars"] += count * n; s["raw_rows"] += count * (k + 2); s["tab_scalars"] += count * tab_size(k)
        s["part_scalars"] += nch * n; s["b0_scalars"] += tiles * count; s["dyn_points"] += count * D; s["chunks"] += nch
        s["nmax"] = max(s["nmax"], n)
        first += count
    s["terms"] = s["nmax"] + 2 + s["dyn_points"] if classes else 0
    return out, s


def model(proofs, ns, set_n):
    codes, members, ks = [], {}, {}
    for j, (p, n) in enumerate(zip(proofs, ns)):
        code, k = model_code(p, n, set_n)
        codes.append(code)
        if code == OK:
            members.setdefault(n, []).append(j); ks[n] = k
    order = [j for n in members for j in members[n]]
    cls, sums = model_layout([(n, ks[n], len(m)) for n, m in members.items()])
    return codes, order, cls, sums


def test_parameter_codes_and_their_order(E):
    cases = [  # (proof, n, set_n, code)
        (proof_bytes(3, length=32 * 9 - 1), 8, 100, FORMAT_ERROR),                     # not whole scalars
        (proof_bytes(0)[:64], 1, 100, FORMAT_ERROR),                                   # fewer than 3 scalars
        (proof_bytes(3) + bytes(32), 8, 100, FORMAT_ERROR),                            # an even number of scalars
        (bytes(32 * (3 + 64)), 1 << 20, 100, FORMAT_ERROR),                            # 32 rounds
        (proof_bytes(3, a=l), 8, 2, FORMAT_ERROR),                                     # a non-canonical before the generators' length
        (proof_bytes(3, r=l + 5), 9, 100, FORMAT_ERROR),                               # r non-canonical before n != 2^k
        (proof_bytes(3, a=2**256 - 1), 0, 100, FORMAT_ERROR),                          # ... and before n = 0
        (proof_bytes(3), 8, 9, INVALID_GENERATORS_LENGTH),                             # set of n + 1 points
        (proof_bytes(3), 9, 10, INVALID_GENERATORS_LENGTH),                            # before n != 2^k
        (proof_bytes(3), 4, 100, VERIFICATION_ERROR),                                  # n != 2^k
        (proof_bytes(0), 0, 100, VERIFICATION_ERROR),                                  # n = 0 with no rounds
        (proof_bytes(3), 0, 100, VERIFICATION_ERROR),                                  # n = 0
        (proof_bytes(0), 0, 1, INVALID_GENERATORS_LENGTH),                             # n = 0 over a set of one point
        (proof_bytes(3), 8, 10, OK),                                                   # exactly n + 2 points
        (proof_bytes(0, a=l - 1, r=l - 1), 1, 3, OK),
    ]
    for p, n, set_n, code in cases:
        assert model_code(p, n, set_n)[0] == code
        got = run(E, [p], [n], set_n)
        assert got is not None and got[0] == [code], (n, set_n, code, got)
        assert len(got[2]) == (1 if code == OK else 0)


def test_classes_offsets_and_terms_against_python(E):
    rnd = random.Random(5)
    ks = [rnd.choice([0, 1, 2, 3, 5, 7, 10]) for _ in range(300)]
    proofs, ns = [], []
    for j, k in enumerate(ks):
        p, n = proof_bytes(k), 1 << k
        if j % 17 == 3:
            n = n + 1                                                  # VerificationError
        if j % 29 == 5:
            p = proof_bytes(k, a=l)                                    # FormatError
        if j % 31 == 7:
            n = 2048                                                   # beyond the set: InvalidGeneratorsLength
        proofs.append(p); ns.append(n)
    set_n = 1024 + 2
    got = run(E, proofs, ns, set_n)
    want = model(proofs, ns, set_n)
    assert got[0] == want[0]
    assert INVALID_GENERATORS_LENGTH in got[0] and VERIFICATION_ERROR in got[0] and FORMAT_ERROR in got[0]
    assert got[1] == want[1]
    assert got[2] == want[2]
    assert got[3] == want[3]
    # classes in the order of their first proof; within one, input order
    firsts = [next(j for j in range(len(ks)) if got[0][j] == OK and ns[j] == c["n"]) for c in got[2]]
    assert firsts == sorted(firsts) and len(got[2]) == 7
    for c in got[2]:
        members = got[1][c["first"]:c["first"] + c["count"]]
        assert members == sorted(members) and all(ns[j] == c["n"] for j in members)
    # the dynamic-term base of every admitted proof: Nmax + 2 + its class's dyn + its rank times D, every term once
    s = got[3]
    spans = [(s["nmax"] + 2 + c["dyn"] + r * c["D"], c["D"]) for c in got[2] for r in range(c["count"])]
    assert len(spans) == len(got[1]) and spans[0][0] == s["nmax"] + 2 == 1024 + 2
    assert all(b0 + D == b1 for (b0, D), (b1, _) in zip(spans, spans[1:])) and spans[-1][0] + spans[-1][1] == s["terms"]


def test_single_length_is_one_class(E):
    proofs = [proof_bytes(6)] * 100
    codes, order, cls, sums = run(E, proofs, [64] * 100, 66)
    assert codes == [OK] * 100 and order == list(range(100)) and len(cls) == 1
    c = cls[0]
    assert (c["first"], c["count"], c["chunk0"], c["dyn"], c["tiles"]) == (0, 100, 0, 0, 1)
    assert sums["terms"] == 64 + 2 + 100 * 14 and sums["chunks"] == 4


def test_every_proof_rejected_leaves_no_class(E):
    codes, order, cls, sums = run(E, [proof_bytes(2)] * 3, [5, 0, 7], 8)
    assert codes == [VERIFICATION_ERROR, VERIFICATION_ERROR, INVALID_GENERATORS_LENGTH] and order == [] and cls == [] and sums["terms"] == 0


def test_refusals(E):
    p = proof_bytes(1)
    assert run(E, [], [], 10) is None
    assert run(E, [p, p], [2, 2], 10, offsets=lambda po, bo: ([1] + po[1:], bo)) is None
    assert run(E, [p, p], [2, 2], 10, offsets=lambda po, bo: (po, [1] + bo[1:])) is None
    assert run(E, [p, p], [2, 2], 10, offsets=lambda po, bo: (po[:1] + [po[2], po[1]], bo)) is None
    assert run(E, [p, p], [2, 2], 10, offsets=lambda po, bo: (po, bo[:1] + [bo[2], bo[1]])) is None
    assert run(E, [p], [(1 << 20) + 1], 1 << 22) is None                     # n above 2^20, whatever else
    assert run(E, [p], [1 << 20], 10) is not None                              # 2^20 itself is a parameter code
    # more than 2^20 proofs
    many = (1 << 20) + 1
    po = (U64 * (many + 1))(*range(0, 96 * (many + 1), 96)); bo = (U64 * (many + 1))(*range(many + 1))
    buf = proof_bytes(0) * many
    out = ctypes.create_string_buffer(many); order = (ctypes.c_uint32 * many)(); cls = (U64 * (len(FIELDS) * 21))(); sums = (U64 * len(SUMS))()
    assert E.emul_linm_plan(many, buf, po, bo, 3, out, order, cls, sums) == -1
    assert E.emul_linm_plan(many - 1, buf, po, bo, 3, out, order, cls, sums) == 1


@pytest.mark.parametrize("k,count,ok", [(20, (1 << 31) // 42 - 25000, True), (20, (1 << 31) // 42 + 1, False), (0, (1 << 30) - 2, True), (0, (1 << 30) - 1, False)])
def test_layout_refuses_2_31_terms(E, k, count, ok):
    """a layout beyond what a call may hold, so that the term limit itself is reached: Nmax + 2 + count (2 + 2k) < 2^31"""
    cls = (U64 * len(FIELDS))(); sums = (U64 * len(SUMS))()
    rc = E.emul_linm_layout(1, (ctypes.c_uint32 * 1)(k), (ctypes.c_uint32 * 1)(count), cls, sums)
    terms = (1 << k) + 2 + count * (2 + 2 * k)
    assert (terms < 1 << 31) == ok
    assert rc == (1 if ok else -1)
    if ok:
        assert dict(zip(SUMS, sums)) == model_layout([(1 << k, k, count)])[1]


def test_layout_of_many_classes_against_python(E):
    rnd = random.Random(9)
    ks = rnd.sample(range(21), 21)
    counts = [rnd.randrange(1, 3000) for _ in ks]
    cls = (U64 * (len(FIELDS) * 21))(); sums = (U64 * len(SUMS))()
    assert E.emul_linm_layout(21, (ctypes.c_uint32 * 21)(*ks), (ctypes.c_uint32 * 21)(*counts), cls, sums) == 21
    want_cls, want_sums = model_layout([(1 << k, k, c) for k, c in zip(ks, counts)])
    assert [dict(zip(FIELDS, cls[len(FIELDS) * c:len(FIELDS) * (c + 1)])) for c in range(21)] == want_cls
    assert dict(zip(SUMS, sums)) == want_sums
