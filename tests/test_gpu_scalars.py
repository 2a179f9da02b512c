"""GPU tier (-m gpu): the device scalar arithmetic of sc.cuh / rp.cuh (bp_debug_sc_op) against Python integers.  On the device
sc_mont_mul is three passes through the PTX multiplier of fe.cuh with a carry of (t_lo != 0), a different algorithm from the host
CIOS branch test_host_emul.py checks, and the lazy reduction of up to 32 products ends in two conditional subtractions of l.  Both
are driven at their edges here: zero operands, raw operands up to 2^256 - 1, challenges >= l and sums of near-maximal products."""
import random

import pytest

from oracle_binding import L_ORDER as l

pytestmark = pytest.mark.gpu

R = 2**256
R_INV = pow(R, -1, l)
EDGE = [0, 1, 2, l - 1, l - 2, 2**252, 2**252 - 1]          # below l
RAW_EDGE = EDGE + [l, l + 1, 2**255, 2**256 - 1]            # any 256-bit value, where the operation takes one


def le(x, n=32):
    return x.to_bytes(n, "little")


def _ints(raw):
    return [int.from_bytes(raw[32 * i:32 * i + 32], "little") for i in range(len(raw) // 32)]


def _pairs(rnd, a_vals, b_vals, n_rand, a_bits=None):
    """every edge pair, then random pairs: a below l, or any a_bits-bit value"""
    A = [a for a in a_vals for _ in b_vals]; B = [b for _ in a_vals for b in b_vals]
    for _ in range(n_rand):
        A.append(rnd.getrandbits(a_bits) if a_bits else rnd.randrange(l)); B.append(rnd.randrange(l))
    return A, B


def _run(ctx, op, A, B):
    return _ints(ctx.debug_sc_op(op, b"".join(le(x) for x in A), b"".join(le(x) for x in B)))


def _check(op, A, B, got, want):
    bad = [(hex(a), hex(b), hex(g)) for a, b, g in zip(A, B, got) if g != want(a, b)]
    assert not bad, (op, len(bad), bad[:4])


def test_mont_mul_raw(gpu_ctx):
    """sc_mont_mul(a, b) = a*b/R mod l for any 256-bit a and b < l, canonical out; zero operands and a*b = 0 mod 2^256 take the
    no-carry side of the (t_lo != 0) trick"""
    rnd = random.Random(71)
    A, B = _pairs(rnd, RAW_EDGE, EDGE, 4000, a_bits=256)
    A += [2**255, 2**255, 2**254 * 3]; B += [2, 2**252, 4]         # t = a*b a multiple of 2^256, t != 0
    _check(0, A, B, _run(gpu_ctx, 0, A, B), lambda a, b: a * b * R_INV % l)


def test_mont_round_trip(gpu_ctx):
    """from_mont(mont_mul(to_mont a, to_mont b)) = a*b mod l, a and b any 256-bit values (to_mont reduces)"""
    rnd = random.Random(72)
    A, B = _pairs(rnd, RAW_EDGE, RAW_EDGE, 4000, a_bits=256)
    _check(1, A, B, _run(gpu_ctx, 1, A, B), lambda a, b: a * b % l)


@pytest.mark.parametrize("op,f", [(2, lambda a, b: (a + b) % l), (3, lambda a, b: (a - b) % l), (4, lambda a, b: -a % l)])
def test_add_sub_neg(gpu_ctx, op, f):
    rnd = random.Random(73 + op)
    A, B = _pairs(rnd, EDGE, EDGE, 4000)
    _check(op, A, B, _run(gpu_ctx, op, A, B), f)


@pytest.mark.parametrize("op", [5, 6])
def test_wide_reduction(gpu_ctx, op):
    """sc_mont_from_wide / rp_wide (every challenge: 64 transcript bytes, usually >= l) = (a + 2^256 b)*R mod l"""
    rnd = random.Random(75 + op)
    A = [a for a in RAW_EDGE for _ in RAW_EDGE]; B = [b for _ in RAW_EDGE for b in RAW_EDGE]
    for _ in range(4000):
        A.append(rnd.getrandbits(256)); B.append(rnd.getrandbits(256))
    _check(op, A, B, _run(gpu_ctx, op, A, B), lambda a, b: (a + (b << 256)) * R % l)


def test_mont_invert(gpu_ctx):
    """sc_mont_invert: a Montgomery-form value in, its inverse in Montgomery form out (0 -> 0)"""
    rnd = random.Random(77)
    A = EDGE + [rnd.randrange(l) for _ in range(600)]
    _check(7, A, A, _run(gpu_ctx, 7, A, A), lambda a, b: pow(a * R_INV % l, l - 2, l) * R % l)


def test_sum32_lazy_reduction(gpu_ctx):
    """sum32 through one sc_wide accumulator (k_rp_scalars_sum: 32 proofs per chunk; k_ippx_inner: 16 products) and one REDC.  32 and
    31 products of (l-1)^2 leave the reduction between 2l and 3l, so both conditional subtractions matter; shorter sums are padded
    with zero products."""
    rnd = random.Random(78)
    groups = [([l - 1] * 32, [l - 1] * 32),
              ([l - 1] * 31 + [0], [l - 1] * 31 + [0]),
              ([l - 1] * 16 + [0] * 16, [l - 1] * 16 + [0] * 16),
              ([l - 1] + [0] * 31, [l - 1] + [0] * 31),
              ([0] * 32, [l - 1] * 32),
              ([l - 2] * 32, [l - 1] * 32)]
    assert (32 * (l - 1) ** 2 + ((-32 * (l - 1) ** 2 * pow(l, -1, R)) % R) * l) // R >= 2 * l        # the edge really is above 2l
    for _ in range(200):
        groups.append(([l - 1 - rnd.getrandbits(100) for _ in range(32)], [l - 1 - rnd.getrandbits(100) for _ in range(32)]))
    for _ in range(300):
        k = rnd.choice([1, 16, 31, 32])
        groups.append(([rnd.randrange(l) for _ in range(k)] + [0] * (32 - k), [rnd.randrange(l) for _ in range(k)] + [0] * (32 - k)))
    A = [x for a, _ in groups for x in a]; B = [y for _, b in groups for y in b]
    got = _run(gpu_ctx, 8, A, B)
    assert len(got) == len(groups)
    for i, (a, b) in enumerate(groups):
        assert got[i] == sum(x * y for x, y in zip(a, b)) * R_INV % l, (i, hex(got[i]))


def test_hook_rejects_bad_arguments(gpu_ctx):
    import bulletproofs_b200 as bp
    with pytest.raises(bp.BpError) as e:
        gpu_ctx.debug_sc_op(8, bytes(32 * 31), bytes(32 * 31))      # sum32 needs whole groups of 32
    assert e.value.code == bp.ERR_INVALID_ARGUMENT
    with pytest.raises(bp.BpError):
        gpu_ctx.debug_sc_op(9, bytes(32), bytes(32))
