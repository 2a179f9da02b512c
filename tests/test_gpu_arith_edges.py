"""The arithmetic core (fe.cuh carry chains, sc.cuh Montgomery and lazy reductions, ge.cuh point formulas and Ristretto maps) on
structured operands, against Python integers and tests/pyref.py.  A uniformly random operand almost never puts an all-ones limb next
to an incoming carry, a product where a second fold fires, or an Elligator input on a zero denominator; the generator below does,
and the CPU-tier tests first show, with a Python model of each limb algorithm's fold and borrow decisions, that the operand sets
reach those branches a few hundred times each.  The same sets then run through the test hooks on the device (-m gpu: the PTX
branches) and through tests/host_emul on the host (the portable branches, among them the CIOS sc_mont_mul the C++ host mirror uses)."""
import ctypes
import os
import random

import numpy as np
import pytest

import pyref
from oracle_binding import L_ORDER as l, P_FIELD as p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 2**256
M256 = R - 1
R_INV = pow(R, -1, l)
L_PRIME = -pow(l, -1, R) % R
N_PAIRS = 2**18
I = pyref.SQRT_M1
gpu = pytest.mark.gpu


def le(x, n=32):
    return x.to_bytes(n, "little")


def ints(raw, w=32):
    return [int.from_bytes(raw[w * i:w * i + w], "little") for i in range(len(raw) // w)]


def pack(vals, w=32):
    return b"".join(v.to_bytes(w, "little") for v in vals)


# ---------------------------------------------------------------------------------------------- the structured operand generator
LIMBS = (0, 1, 2, 19, 38, 0x7fffffff, 0x80000000, 0xffffffed, 0xfffffffe, 0xffffffff)


def limb_pattern(rnd, n):
    """n values whose eight 32-bit limbs are each one of LIMBS or a uniformly random limb (one choice in 11)"""
    g = np.random.default_rng(rnd.getrandbits(64))
    idx = g.integers(0, len(LIMBS) + 1, size=(n, 8))
    limbs = np.where(idx == len(LIMBS), g.integers(0, 2**32, size=(n, 8), dtype=np.uint64), np.array(LIMBS + (0,), dtype=np.uint64)[idx])
    return ints(limbs.astype("<u4").tobytes())


def sparse(bits):
    """single bits 2^j, two-bit values, and runs 2^a - 2^b that cross limb boundaries, all below 2^bits"""
    single = [1 << j for j in range(bits)]
    two = [(1 << i) | (1 << j) for i in range(0, bits, 3) for j in range(i + 1, bits, 5)]
    runs = [(1 << a) - (1 << b) for a in range(1, bits + 1, 3) for b in range(0, a, 7)]
    return sorted(set(single + two + runs))


def near(centres, delta=40, lo=0, hi=R):
    return sorted({c + d for c in centres for d in range(-delta, delta + 1) if lo <= c + d < hi})


FE_HOT = near([0, p, 2 * p, R, 2**255])                  # k*p + delta, 2^256 - delta, 2^255 +- delta
SC_RAW_HOT = sorted(set(near([k * l for k in range(16)] + [R])) | {l - 1, l, l + 1})     # every k with k*l < 2^256
SC_LOW_HOT = near([0, l, 2**252], hi=l)                  # below l: delta, l - delta, 2^252 +- delta


def sc_low_pattern(rnd, n):
    """limb patterns below l that keep their limbs: bits 252..255 cleared (the top limb becomes 0x0fffffff, 0x07ffffff, ...), and
    one value in eight 2^252 + a 128-bit limb pattern below l - 2^252 (limbs 4..6 zero, as in l itself)"""
    out = []
    for v in limb_pattern(rnd, n):
        if v & 7 == 0 and (v & (2**128 - 1)) < l - 2**252:
            out.append(2**252 + (v & (2**128 - 1)))
        else:
            out.append(v & (2**252 - 1))
    return out


def make_pairs(rnd, a_hot, b_hot, a_sparse, b_sparse, a_pool, b_pool, extra=(), n=N_PAIRS):
    """hot x hot (sampled down to half the set when larger), sparse values paired with shuffled sparse values, the extra pairs, and
    the rest drawn from the pools (limb patterns mixed with every structured value)"""
    cross = [(a, b) for a in a_hot for b in b_hot]
    if len(cross) > n // 2:
        cross = rnd.sample(cross, n // 2)
    ps = cross + list(zip(a_sparse, rnd.sample(b_sparse, len(b_sparse)))) + list(extra)
    ps += [(rnd.choice(a_pool), rnd.choice(b_pool)) for _ in range(n - len(ps))]
    return [a for a, _ in ps], [b for _, b in ps]


def sq_row6_operands(rnd, n=2000):
    """values whose square takes the carry into o13 in row 6 of fe_sq_wide (m_sq_row6_carry): a7 * a6 = -1 mod 2^32 with a6 odd,
    high a4 and a5 so that the earlier odd-aligned rows leave o12 = 1, and limb patterns below"""
    out = []
    while len(out) < n:
        for v in limb_pattern(rnd, 4 * n):
            a6 = ((v >> 192) & 0xffffffff) | 1
            v = (v & (2**128 - 1)) | rnd.choice(LIMBS[5:]) << 128 | rnd.choice(LIMBS[5:]) << 160 | a6 << 192 | (-pow(a6, -1, 2**32) % 2**32) << 224
            if m_sq_row6_carry(v) and len(out) < n:
                out.append(v)
    return out


def fe_operands(seed=1):
    rnd = random.Random(seed)
    sp = sparse(256)
    structured = FE_HOT + sp
    pool = limb_pattern(rnd, N_PAIRS) + structured
    sq6 = sq_row6_operands(rnd)
    # (v, 0) and (0, v): fe_add(v, 0) and fe_sub(v, 0) hand v to fe_canon unchanged
    extra = [(v, 0) for v in structured] + [(0, v) for v in FE_HOT] + [(v, rnd.choice(pool)) for v in sq6]
    return make_pairs(rnd, FE_HOT, FE_HOT, sp, sp, pool, pool, extra)


def sc_operands(kind, seed=2):
    """pairs for the scalar ops: "mont" a any 256-bit value, b < l (op 0); "raw" both any 256-bit value (ops 1, 5, 6); "low" both
    below l (ops 2, 3, 4, 7, 8), with complement pairs (x, l - x) whose sum is exactly l, and equal pairs"""
    rnd = random.Random(seed * 10 + ("mont", "raw", "low").index(kind))
    raw_sp, low_sp = sparse(256), sparse(252)
    raw_pool = limb_pattern(rnd, N_PAIRS // 2) + SC_RAW_HOT + raw_sp
    low_pool = sc_low_pattern(rnd, N_PAIRS // 2) + SC_LOW_HOT + low_sp
    if kind == "mont":
        return make_pairs(rnd, SC_RAW_HOT, SC_LOW_HOT, raw_sp, low_sp, raw_pool, low_pool)
    if kind == "raw":
        return make_pairs(rnd, SC_RAW_HOT, SC_RAW_HOT, raw_sp, raw_sp, raw_pool, raw_pool)
    comp = [x for x in rnd.sample(low_pool, 2000) if x > 0]
    extra = [(x, l - x) for x in comp] + [(x, x) for x in comp[:500]]
    return make_pairs(rnd, SC_LOW_HOT, SC_LOW_HOT, low_sp, low_sp, low_pool, low_pool, extra)


def sum32_operands(seed=3):
    """2^18 pairs in groups of 32 (op 8): a quarter of the groups from values within a structured distance of l, where the lazy
    reduction ends between 2l and 3l, the rest from the "low" pairs"""
    rnd = random.Random(seed)
    A, B = sc_operands("low", seed)
    high = [x for x in SC_LOW_HOT + sc_low_pattern(rnd, 20000) if x >= 2**251 + 2**250]
    for g in range(0, len(A) // 32, 4):
        for j in range(32 * g, 32 * g + 32):
            A[j], B[j] = rnd.choice(high), rnd.choice(high)
    return A, B


# ---------------------------------------------------------------------------------------------- Python models of the limb algorithms
def m_fe_add(a, b):
    """fe_add: a + b, the carry c folded as 38c; a second carry c2 (the wrapped value was within 38 of 2^256) folds once more"""
    s = a + b
    s2 = (s & M256) + 38 * (s >> 256)
    c2 = s2 >> 256
    return (s2 & M256) + 38 * c2, c2


def m_fe_sub(a, b):
    """fe_sub: a - b, a borrow takes 38 more; a second borrow b2 (the wrapped value was below 38) takes 38 once more"""
    d = a - b
    d2 = (d & M256) - 38 * (d < 0)
    b2 = d2 < 0
    return (d2 & M256) - 38 * b2, b2


def m_fe_reduce_wide(t):
    """fe_reduce_wide: c8 = carry of t_lo + 38 t_hi, folded as 38 c8; a carry c2 out of that fold adds a last 38"""
    s = (t & M256) + 38 * (t >> 256)
    c8 = s >> 256
    s2 = (s & M256) + 38 * c8
    c2 = s2 >> 256
    return (s2 & M256) + 38 * c2, c8, c2


def m_sq_row6_carry(a):
    """fe_sq_wide row 6 forms (o12, o13) = a7*a6 + o12.  o12 <= 1 is what the earlier rows left above limb 11 of the odd-aligned
    accumulator, which holds the exact sum of the products a_i a_j, i < j, i + j odd, at limb i + j - 1; the carry from the low word
    into o13 fires only when lo(a7*a6) + o12 >= 2^32, i.e. a7*a6 = -1 mod 2^32 and o12 = 1"""
    L = [(a >> (32 * k)) & 0xffffffff for k in range(8)]
    O = sum(L[i] * L[j] << (32 * (i + j - 1)) for i in range(8) for j in range(i + 1, 8) if (i + j) % 2 and (i, j) != (6, 7))
    return (L[6] * L[7] & 0xffffffff) + (O >> 384) >= 2**32


def m_sc_redc(T):
    """REDC(T) = (T + M l) / R before the conditional subtractions, M = T_lo * (-l^-1) mod R"""
    return (T + (T * L_PRIME % R) * l) >> 256


def fe_branch_counts(A, B):
    add = [m_fe_add(a, b) for a, b in zip(A, B)]
    sub = [m_fe_sub(a, b) for a, b in zip(A, B)]
    red = [m_fe_reduce_wide(a * b) for a, b in zip(A, B)] + [m_fe_reduce_wide(a * a) for a in A]
    canon_in = [r for r, _ in add] + [r for r, _ in sub] + [r for r, _, _ in red]
    return {"fe_add c2": sum(c for _, c in add), "fe_sub b2": sum(b for _, b in sub),
            "fe_reduce_wide c2": sum(c for _, _, c in red), "fe_reduce_wide max c8": max(c for _, c, _ in red),
            "fe_sq_wide row-6 carry": sum(map(m_sq_row6_carry, A)),
            "fe_canon [p, 2p)": sum(p <= v < 2 * p for v in canon_in), "fe_canon [2p, 2^256)": sum(v >= 2 * p for v in canon_in),
            "fe_canon = p": canon_in.count(p), "fe_canon = 2p": canon_in.count(2 * p)}


@pytest.fixture(scope="module")
def fe_set():
    return fe_operands()


@pytest.fixture(scope="module")
def sc_sets():
    return {"mont": sc_operands("mont"), "raw": sc_operands("raw"), "low": sc_operands("low"), "sum32": sum32_operands()}


# ---------------------------------------------------------------------------------------------- 1. the operand sets reach the branches
def test_field_operands_reach_the_fold_and_borrow_branches(fe_set):
    """Every branch of fe_add, fe_sub, fe_reduce_wide and fe_canon, and the rarest carry of fe_sq_wide, a few hundred times.
    The largest c8 of fe_reduce_wide is 38, reached by (2^256 - 76)^2: t_lo + 38 t_hi < 39 * 2^256 for any 512-bit t, so 38 is
    also the bound."""
    A, B = fe_set
    assert len(A) == N_PAIRS
    n = fe_branch_counts(A, B)
    for k in ("fe_add c2", "fe_sub b2", "fe_reduce_wide c2", "fe_sq_wide row-6 carry", "fe_canon [p, 2p)", "fe_canon [2p, 2^256)",
              "fe_canon = p", "fe_canon = 2p"):
        assert n[k] >= 300, (k, n)
    assert n["fe_reduce_wide max c8"] == 38, n
    assert (M256 + 38 * M256) >> 256 == 38
    assert m_fe_reduce_wide((R - 76) ** 2)[1] == 38


def test_scalar_operands_reach_the_reduction_branches(sc_sets):
    """sc_wide_redc ends in [2l, 3l) (both conditional subtractions fire) for hundreds of sum32 groups and never reaches 3l;
    sc_cond_sub_l sees exactly l through sc_add; sc_mont_mul sees t = a*b with t_lo = 0 and t != 0, the no-carry side of the
    (t_lo != 0) trick, for hundreds of pairs"""
    A, B = sc_sets["sum32"]
    red = [m_sc_redc(sum(x * y for x, y in zip(A[j:j + 32], B[j:j + 32]))) for j in range(0, len(A), 32)]
    assert sum(r >= 2 * l for r in red) >= 300 and max(red) < 3 * l
    A, B = sc_sets["low"]
    assert all(a < l and b < l for a, b in zip(A, B))
    assert sum(a + b == l for a, b in zip(A, B)) >= 300
    A, B = sc_sets["mont"]
    assert all(b < l for b in B)
    assert sum(a * b % R == 0 and a * b != 0 for a, b in zip(A, B)) >= 300


# ---------------------------------------------------------------------------------------------- 2. bulk differential runs
def sqrt_ref(u, v):
    ok, r = pyref.sqrt_ratio_i(u, v)
    return r | (int(ok) << 255)


FE_REF = {0: lambda a, b: (a + b) % p, 1: lambda a, b: (a - b) % p, 2: lambda a, b: a * b % p, 3: lambda a, b: pow(a, p - 2, p),
          4: lambda a, b: pow(a, (p - 5) // 8, p), 5: lambda a, b: -a % p, 6: lambda a, b: a * a % p,
          7: lambda a, b: (a + b) * (a - b) % p, 8: lambda a, b: 2 * a % p,
          9: lambda a, b: int(a % p == 0) | (a % p & 1) << 8 | int((a - b) % p == 0) << 16, 10: sqrt_ref}
SC_REF = {0: ("mont", lambda a, b: a * b * R_INV % l), 1: ("raw", lambda a, b: a * b % l), 2: ("low", lambda a, b: (a + b) % l),
          3: ("low", lambda a, b: (a - b) % l), 4: ("low", lambda a, b: -a % l), 5: ("raw", lambda a, b: (a + (b << 256)) * R % l),
          6: ("raw", lambda a, b: (a + (b << 256)) * R % l), 7: ("low", lambda a, b: pow(a * R_INV % l, l - 2, l) * R % l)}


def check_fe_op(run, op, A, B):
    got = ints(run(op, pack(A), pack(B)))
    f = FE_REF[op]
    bad = [(hex(a), hex(b), hex(g)) for a, b, g in zip(A, B, got) if g != f(a, b)]
    assert not bad, (op, len(bad), bad[:3])


def check_sc_op(run, op, sets):
    if op == 8:
        A, B = sets["sum32"]
        got = ints(run(8, pack(A), pack(B)))
        want = [sum(x * y for x, y in zip(A[j:j + 32], B[j:j + 32])) * R_INV % l for j in range(0, len(A), 32)]
        bad = [j for j, (g, w) in enumerate(zip(got, want)) if g != w]
        assert len(got) == len(A) // 32 and not bad, (len(bad), bad[:3])
        return
    kind, f = SC_REF[op]
    A, B = sets[kind]
    got = ints(run(op, pack(A), pack(B)))
    bad = [(hex(a), hex(b), hex(g)) for a, b, g in zip(A, B, got) if g != f(a, b)]
    assert not bad, (op, len(bad), bad[:3])


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    for name in ("emul_debug_fe_op", "emul_debug_sc_op", "emul_debug_ge_op"):
        getattr(E, name).argtypes = [ctypes.c_int, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p]
    return E


def host_runner(E, name, w=32):
    def run(op, a, b):
        n = len(a) // w
        out = ctypes.create_string_buffer(w * (n // 32 if name == "emul_debug_sc_op" and op == 8 else n))
        getattr(E, name)(op, a, b, n, out)
        return out.raw
    return run


# the exponentiations (field ops 3, 4 and 10, scalar op 7) take every 32nd pair on the host: the same mix in a thirty-second of the time
HOST_STRIDE = 32


@pytest.mark.parametrize("op", range(11))
def test_host_field_ops_on_structured_operands(E, fe_set, op):
    A, B = fe_set
    s = HOST_STRIDE if op in (3, 4, 10) else 1
    check_fe_op(host_runner(E, "emul_debug_fe_op"), op, A[::s], B[::s])


@pytest.mark.parametrize("op", range(9))
def test_host_scalar_ops_on_structured_operands(E, sc_sets, op):
    sets = {k: (A[::HOST_STRIDE], B[::HOST_STRIDE]) if op == 7 else (A, B) for k, (A, B) in sc_sets.items()}
    check_sc_op(host_runner(E, "emul_debug_sc_op"), op, sets)


@gpu
@pytest.mark.parametrize("op", range(11))
def test_device_field_ops_on_structured_operands(gpu_ctx, fe_set, op):
    """2^18 structured pairs per op, one device call each"""
    check_fe_op(gpu_ctx.debug_fe_op, op, *fe_set)


@gpu
@pytest.mark.parametrize("op", range(9))
def test_device_scalar_ops_on_structured_operands(gpu_ctx, sc_sets, op):
    check_sc_op(gpu_ctx.debug_sc_op, op, sc_sets)


# ---------------------------------------------------------------------------------------------- 3. sqrt_ratio_i and the hook's arguments
def sqrt_branch(u, v):
    """which comparison of fe_sqrt_ratio_i matches: v r^2 = u ("ok"), = -u ("flip"), = -u i ("flip_i"), or none"""
    u %= p; v %= p
    v3 = v * v * v % p; v7 = v3 * v3 * v % p
    r = u * v3 * pow(u * v7, (p - 5) // 8, p) % p
    chk = v * r * r % p
    return "ok" if chk == u else "flip" if chk == -u % p else "flip_i" if chk == -u * I % p else "none"


def sqrt_cases(seed=4):
    """u = 0, v = 0, u/v = -1, u/v a square, a non-square, i times a square, each also with u and v as their +p and +2p
    representatives where those are below 2^256"""
    rnd = random.Random(seed)
    nonsq = next(x for x in range(2, 100) if pow(x, (p - 1) // 2, p) == p - 1)
    cases = [(0, 0), (p, 0), (0, p), (p, p), (2 * p, 0), (1, 0)]
    for _ in range(60):
        v, w = rnd.randrange(1, p), rnd.randrange(1, p)
        for u in (0, v * w * w % p, -v % p, -v * w * w % p, nonsq * v * w * w % p, I * v * w * w % p, -I * v * w * w % p, rnd.randrange(p)):
            cases += [(u, v), (u, 0)]
    out = []
    for u, v in cases:
        for du in (0, p, 2 * p):
            for dv in (0, p, 2 * p):
                if u + du < R and v + dv < R:
                    out.append((u + du, v + dv))
    return out


def test_sqrt_ratio_i_cases_reach_every_comparison():
    seen = {sqrt_branch(u, v) for u, v in sqrt_cases()}
    assert seen == {"ok", "flip", "flip_i", "none"}
    assert any(v % p == 0 and u % p for u, v in sqrt_cases()) and any(u + p < R and u % p == 0 for u, _ in sqrt_cases())


def test_host_sqrt_ratio_i_edges(E):
    A, B = zip(*sqrt_cases())
    check_fe_op(host_runner(E, "emul_debug_fe_op"), 10, list(A), list(B))


@gpu
def test_device_sqrt_ratio_i_edges(gpu_ctx):
    A, B = zip(*sqrt_cases())
    check_fe_op(gpu_ctx.debug_fe_op, 10, list(A), list(B))


@gpu
def test_hooks_reject_bad_arguments(gpu_ctx):
    import bulletproofs_b200 as bp
    for op in (-1, 11, 1000):
        with pytest.raises(bp.BpError) as e:
            gpu_ctx.debug_fe_op(op, bytes(32), bytes(32))
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
    for op in (-1, 4):
        with pytest.raises(bp.BpError) as e:
            gpu_ctx.debug_ge_op(op, bytes(128), bytes(128))
        assert e.value.code == bp.ERR_INVALID_ARGUMENT


# ---------------------------------------------------------------------------------------------- 4. point formulas on any representative
E4 = [(0, 1, 1, 0), (0, p - 1, 1, 0), (I, 0, 1, 0), (p - I, 0, 1, 0)]       # the 4-torsion: (0, +-1) and (+-i, 0)
LAMBDAS = [1, 2, p - 1, 19, 2**255 - 20, 2**128 + 1, (2**255 - 1) // 3, 0xffffffff, 2**224 - 2**32]


def neg(P_):
    X, Y, Z, T = P_
    return (-X % p, Y, Z, -T % p)


def scale(P_, lam):
    return tuple(c * lam % p for c in P_)


def rep(rnd, c):
    """c (< p) or one of its representatives c + p, c + 2p below 2^256"""
    return rnd.choice([c + k * p for k in range(3) if c + k * p < R])


def reps(rnd, P_):
    return tuple(rep(rnd, c) for c in P_)


def dbl_ref(P_):
    """ge_dbl's formula (HWCD dbl-2008-hwcd, a = -1) with Python integers"""
    X, Y, Z, _ = P_
    A, B, C = X * X % p, Y * Y % p, 2 * Z * Z % p
    H = (A + B) % p; E_ = ((X + Y) ** 2 - H) % p; G = (B - A) % p; F = (G - C) % p; Hn = -H % p
    return (E_ * F % p, G * Hn % p, F * G % p, E_ * Hn % p)


def on_curve(P_):
    X, Y, Z, T = P_
    return Z % p != 0 and X * Y % p == Z * T % p and (-X * X + Y * Y - Z * Z - pyref.D * T * T) % p == 0


def same_point(P_, Q):
    return all((a * Q[2] - b * P_[2]) % p == 0 for a, b in ((P_[0], Q[0]), (P_[1], Q[1]), (P_[3], Q[3])))


@pytest.fixture(scope="module")
def points(orc):
    """points decoded from oracle-made encodings (with their encodings)"""
    rnd = random.Random(5)
    encs = [orc.from_uniform(rnd.randbytes(64)) for _ in range(16)]
    return [(enc, pyref.decode(enc)) for enc in encs]


def ge_cases(points, seed=6):
    """(a, b) pairs of extended points: each point and the identity shifted by every E[4] element, scaled by structured lambda, with
    +p / +2p coordinates; then P + P, P + (-P), P + (P + T4) and random pairs among them"""
    rnd = random.Random(seed)
    base = [pt for _, pt in points] + [pyref.IDENT]
    forms = [scale(pyref.add(P_, T4), lam) for P_ in base for T4 in E4 for lam in rnd.sample(LAMBDAS, 3)]
    A, B = [], []
    for P_ in forms:
        for Q in (P_, neg(P_), scale(P_, rnd.choice(LAMBDAS))) + tuple(pyref.add(P_, T4) for T4 in E4) + (rnd.choice(forms),):
            A.append(reps(rnd, P_)); B.append(reps(rnd, Q))
    return A, B


def affine(rnd, Q):
    zi = pow(Q[2], p - 2, p)
    x, y = Q[0] * zi % p, Q[1] * zi % p
    return (rep(rnd, x), rep(rnd, y), 0, 0)


def check_ge_ops(run, points):
    A, B = ge_cases(points)
    pa, pb = b"".join(pack(P_) for P_ in A), b"".join(pack(Q) for Q in B)
    points_of = lambda raw: [tuple(ints(raw[128 * i:128 * i + 128])) for i in range(len(A))]
    assert points_of(run(0, pa, pb)) == [pyref.add(a, b) for a, b in zip(A, B)]
    assert points_of(run(3, pa, pb)) == [dbl_ref(a) for a in A]
    rnd = random.Random(7)
    Baff = [affine(rnd, Q) for Q in B]
    pq = b"".join(pack(Q) for Q in Baff)
    for op, sign in ((1, 1), (2, -1)):
        raw = run(op, pa, pq)
        for i, (a, q) in enumerate(zip(A, Baff)):
            x, y = q[0] % p, q[1] % p
            want = pyref.add(a, (sign * x % p, y, 1, sign * x * y % p))
            r = tuple(ints(raw[128 * i:128 * i + 128]))
            assert on_curve(r) and same_point(r, want), (op, i)


def test_host_point_formulas_on_any_representative(E, points):
    check_ge_ops(host_runner(E, "emul_debug_ge_op", 128), points)


@gpu
def test_device_point_formulas_on_any_representative(gpu_ctx, points):
    """ge_add and ge_dbl equal the HWCD formulas coordinate by coordinate; ge_madd / ge_msub give the same projective point, on the
    curve, for the identity and E[4]-shifted points in every representative"""
    check_ge_ops(gpu_ctx.debug_ge_op, points)


# ---------------------------------------------------------------------------------------------- 5. the public Ristretto maps
def encode_branches(pt):
    """(rot, y negated) of pyref.encode / ge_encode"""
    X, Y, Z, T = pt
    u1 = (Z + Y) * (Z - Y) % p; u2 = X * Y % p
    _, Ii = pyref.sqrt_ratio_i(1, u1 * u2 * u2 % p)
    zi = Ii * u1 % p * (Ii * u2 % p) % p * T % p
    rot = pyref.is_neg(T * zi % p)
    x = Y * I % p if rot else X
    return rot, pyref.is_neg(x * zi % p)


def compress_cases(points, seed=8):
    rnd = random.Random(seed)
    cases = []
    for enc, P_ in points + [(bytes(32), pyref.IDENT)]:
        for T4 in E4:
            for lam in LAMBDAS:
                cases.append((enc, reps(rnd, scale(pyref.add(P_, T4), lam))))
    return cases


def test_compress_cases_take_both_rotations_and_negations(points):
    cases = compress_cases(points)
    assert {encode_branches(pt) for _, pt in cases} == {(0, 0), (0, 1), (1, 0), (1, 1)}
    assert all(pyref.encode(pt) == enc for enc, pt in cases)


@gpu
def test_compress_on_every_coset_representative(gpu_ctx, points):
    """bp_compress_batch loads raw limbs: P + T for every T in E[4], scaled and weakly reduced, compresses to P's encoding"""
    cases = compress_cases(points)
    got = gpu_ctx.compress(b"".join(pack(pt) for _, pt in cases))
    assert [got[32 * i:32 * i + 32] for i in range(len(cases))] == [enc for enc, _ in cases]


def decode_reason(s_bytes):
    """why pyref.decode rejects (or "ok"), in the order the checks are made"""
    s = int.from_bytes(s_bytes, "little")
    if s >= p:
        return "non-canonical"
    if s & 1:
        return "odd"
    ss = s * s % p; u1 = (1 - ss) % p; u2 = (1 + ss) % p; u2s = u2 * u2 % p
    v = (-pyref.D * u1 % p * u1 - u2s) % p
    ok, Ii = pyref.sqrt_ratio_i(1, v * u2s % p)
    if not ok:
        return "u2 = 0" if u2 == 0 else "not square"
    dx = Ii * u2 % p; dy = Ii * dx % p * v % p
    x = pyref.fabs(2 * s * dx % p); y = u1 * dy % p
    return "negative t" if pyref.is_neg(x * y % p) else "y = 0" if y == 0 else "ok"


def decompress_families(points, seed=9):
    rnd = random.Random(seed)
    encs = [enc for enc, _ in points]
    even_i = I if I % 2 == 0 else p - I
    fam = {"non-canonical": [le(p + k) for k in range(19)],
           "bit 255": [le(int.from_bytes(e, "little") | 1 << 255) for e in encs],
           "odd": [le(int.from_bytes(e, "little") + 1) for e in encs] + [le(rnd.randrange(p) | 1) for _ in range(20)],
           "not square": [], "negative t": [], "y = 0": [le(p - 1)], "u2 = 0": [le(even_i)], "ok": encs + [bytes(32)]}
    while len(fam["not square"]) < 40 or len(fam["negative t"]) < 40:
        s = le(rnd.randrange(p) & ~1)
        r = decode_reason(s)
        if r in ("not square", "negative t") and len(fam[r]) < 40:
            fam[r].append(s)
    return fam


def test_decompress_families_have_their_reasons(points, orc):
    """each family non-empty, every member rejected (or accepted) by pyref for the family's reason, and by the oracle alike"""
    for family, members in decompress_families(points).items():
        assert members and all(decode_reason(s) == {"bit 255": "non-canonical"}.get(family, family) for s in members), family
        assert all(orc.point_is_valid(s) == (family == "ok") for s in members), family


@gpu
def test_decompress_rejects_each_reason(gpu_ctx, points):
    """ok flags and coordinates against pyref.decode, one family per rejection reason"""
    fam = decompress_families(points)
    cand = [s for members in fam.values() for s in members]
    want = [pyref.decode(s) for s in cand]
    assert gpu_ctx.decompress_check(b"".join(cand)) == [int(w is not None) for w in want]
    xyzt, ok = gpu_ctx.decompress(b"".join(cand))
    for i, w in enumerate(want):
        assert ok[i] == int(w is not None), i
        assert tuple(ints(xyzt[i])) == (w if w is not None else pyref.IDENT), i


def uniform_halves():
    """both roots r0 of each zero Elligator denominator D = (-1 - d r)(r + d), r = i r0^2 (r = -d and r = -1/d), plus 0, 1, p - 1
    and the non-canonical p .. 2^255 - 1"""
    halves = []
    for r in (-pyref.D % p, -pow(pyref.D, -1, p) % p):
        ok, r0 = pyref.sqrt_ratio_i(-r * I % p, 1)
        assert ok and (-1 - pyref.D * (I * r0 * r0)) * (I * r0 * r0 + pyref.D) % p == 0
        halves += [r0, p - r0]
    return halves + [0, 1, p - 1] + list(range(p, 2**255))


def test_uniform_halves_hit_zero_denominators():
    H = uniform_halves()
    zero_d = [r0 for r0 in H if (-1 - pyref.D * I * r0 * r0) * (I * r0 * r0 + pyref.D) % p == 0]
    assert len(zero_d) == 4 and len(set(zero_d)) == 4 and len(H) == 4 + 3 + 19
    # there sqrt_ratio_i(N, 0) returns s = 0 whichever way the square/non-square selects go, so w0 = 2 s D = 0: the identity
    for r0 in zero_d:
        X, Y, Z, T = pyref.elligator(r0)
        assert X == 0 and T == 0 and Y == Z != 0


@gpu
def test_from_uniform_at_zero_denominators(gpu_ctx, orc):
    """every pairing of the halves, against pyref.from_uniform and the oracle"""
    H = uniform_halves()
    uni = [le(a) + le(b) for a in H for b in H]
    got = gpu_ctx.from_uniform_bytes(b"".join(uni))
    got = [got[32 * i:32 * i + 32] for i in range(len(uni))]
    assert got == [pyref.encode(pyref.from_uniform(u)) for u in uni]
    assert got == [orc.from_uniform(u) for u in uni]
