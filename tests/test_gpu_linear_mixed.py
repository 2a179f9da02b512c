"""GPU tier (-m gpu): LinearProofs of different lengths in one call, bp_linear_verify_mixed (bp.linear_verify_mixed,
LinearVerifier.verify_mixed).  Every verdict must be what the single path (bp.linear_verify) and the oracle (orc.linear_verify) return for
that proof alone with G = the set's prefix of its length, and what bp_linear_verify_batch gives it alone; proofs rejected on their
parameters get their codes and leave the others alone.  Covered: every power-of-two length from 1 to 1024 in one call, bad proofs in each
class and of every damage kind, parameter codes, the fixed form's verdicts on one-length calls, a reject path over several slices,
proofs of different lengths whose errors cancel under weights blind to a || r, seeds, refusals, launches that do not grow with the
classes or the proofs, and the reserved LinearProof and range-proof graphs on the same context.  (The refusal at 2^31 MSM terms is past
what 2^20 proofs of n <= 2^20 can reach; tests/test_linear_mixed_cpu.py checks it on the layout.)"""
import ctypes
import json
import os
import random

import pytest

from oracle_binding import L_ORDER as l
from test_gpu_linear_device import run as device_run
from test_linear_verify_batch import (FORMAT_ERROR, INVALID_GENERATORS_LENGTH, KINDS, OK, VERIFICATION_ERROR, _damaged, _gens, _replay_python,
                                      gpu_proofs, le, lg, rng_bytes, single)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NS = [1 << k for k in range(11)]                    # 1 .. 1024
SEED = bytes(range(32))


@pytest.fixture(scope="module")
def bp():
    import bulletproofs_b200
    return bulletproofs_b200


@pytest.fixture(scope="module")
def V(bp, gpu_ctx, orc):
    """a verifier over [B, F, G_0 .. G_1023]"""
    v = bp.LinearVerifier(gpu_ctx, *_gens(orc, 1024))
    yield v
    v.close()


def pools(bp, ctx, orc, per, ns=NS):
    return {n: gpu_proofs(bp, ctx, orc, n, per)[0] for n in ns}


def expected(bp, ctx, orc, V, items, seed=SEED):
    """each item's verdict on its own: the single path and the oracle over G = the set's prefix of its length (for a proof whose length the
    set holds), and bp_linear_verify_batch with count 1"""
    G, F, B = _gens(orc, V.n)
    memo, out = {}, []
    for p in items:
        if id(p) not in memo:
            n = len(p.b) // 32
            alone = bp.linear_verify_batch(ctx, V.points, n, [p.item(bp)], seed)[0]
            if 1 <= n and n + 2 <= V.points.n:
                assert single(bp, ctx, orc, (G[:32 * n], F, B), p) == alone
            memo[id(p)] = alone
        out.append(memo[id(p)])
    return out


def mixed(bp, V, items, seed=SEED):
    return V.verify_mixed([p.item(bp) for p in items], seed=seed)


def launches(bp, ctx, V, items):
    l0 = ctx.launches
    got = mixed(bp, V, items)
    return got, ctx.launches - l0


def damage(p, kind, n, G):
    """_damaged's kinds where n has them, and zero L / R, undecodable C / S"""
    k = lg(n)
    pr = bytearray(p.proof)
    if kind == "zero L":
        pr[0:32] = bytes(32)
    elif kind == "zero R":
        pr[64 * (k - 1) + 32:64 * k] = bytes(32)
    elif kind == "undecodable C":
        return p.replace(C=b"\xff" * 32)
    elif kind == "undecodable S":
        pr[64 * k:64 * k + 32] = b"\xff" * 32
    else:
        return _damaged(p, kind, n, G)
    return p.replace(proof=bytes(pr))


# damage the front end rejects before the combined MSM (host parameter check, undecodable or zero point): no reject path runs; damage
# that reaches it: the reject path runs.  ("R" flips a bit of an encoding, which may or may not still decode.)
PRE_REJECTED = {"a non-canonical", "r non-canonical", "undecodable C", "undecodable S", "zero L", "zero R"}
REACHES_MSM = {"L", "S", "C", "b_i", "label", "a flipped", "r flipped"}


def kinds_for(n):
    """the damage kinds a proof of length n can take: L and R need a round, b_i needs six entries"""
    out = [x for x in KINDS if (x not in ("L", "R") or n > 1) and (x != "b_i" or n > 5)] + ["undecodable C", "undecodable S"]
    return out + (["zero L", "zero R"] if n > 1 else [])


def test_every_length_in_one_call(bp, gpu_ctx, orc, V):
    P = pools(bp, gpu_ctx, orc, 5)
    items = [p for n in NS for p in P[n]]
    random.Random(1).shuffle(items)
    assert expected(bp, gpu_ctx, orc, V, items) == [OK] * len(items)
    got, nl = launches(bp, gpu_ctx, V, items)
    assert got == [OK] * len(items)
    # over a set larger than the longest proof
    big = bp.LinearVerifier(gpu_ctx, *_gens(orc, 1500))
    assert big.verify_mixed([p.item(bp) for p in items], seed=SEED) == [OK] * len(items)
    big.close()


def test_launches_do_not_grow_with_classes_or_proofs(bp, gpu_ctx, orc, V):
    P = pools(bp, gpu_ctx, orc, 5)
    two = [P[16][j % 5] if j % 2 else P[1024][j % 5] for j in range(64)]
    eleven = [P[NS[j % 11]][j % 5] for j in range(64)]
    many = [P[NS[j % 11]][j % 5] for j in range(1024)]
    counts = []
    for items in (two, eleven, many):
        got, nl = launches(bp, gpu_ctx, V, items)
        assert got == [OK] * len(items)
        counts.append(nl)
    assert len(set(counts)) == 1 and counts[0] > 0, counts


def test_one_bad_proof_in_each_class_in_turn(bp, gpu_ctx, orc, V):
    P = pools(bp, gpu_ctx, orc, 4)
    G = _gens(orc, 1024)[0]
    base = [P[NS[j % 11]][(j // 11) % 4] for j in range(66)]
    ok_launches = launches(bp, gpu_ctx, V, base)[1]
    for c, n in enumerate(NS):
        at = next(j for j, p in enumerate(base) if len(p.b) == 32 * n)
        kind = kinds_for(n)[c % len(kinds_for(n))]
        items = list(base)
        items[at] = damage(base[at], kind, n, G)
        want = expected(bp, gpu_ctx, orc, V, items)
        assert want[at] != OK and want[:at] + want[at + 1:] == [OK] * 65, (n, kind)
        got, nl = launches(bp, gpu_ctx, V, items)
        assert got == want, (n, kind, got)
        if kind in REACHES_MSM or kind in PRE_REJECTED:
            assert (nl > ok_launches) == (kind in REACHES_MSM), (n, kind, nl, ok_launches)


def test_every_damage_kind_and_many_bad_proofs(bp, gpu_ctx, orc, V):
    P = pools(bp, gpu_ctx, orc, 4, [1, 2, 16, 64, 256])
    G = _gens(orc, 1024)[0]
    items = []
    for n in P:
        for j, kind in enumerate(kinds_for(n)):
            items.append(damage(P[n][j % 4], kind, n, G))
        items += P[n]
    # records no transcript can hold, at two lengths
    recs = {}
    for n in (2, 64):
        p = P[n][1].replace(label=P[n][1].label)
        recs[id(p)] = bp.Transcript(p.label).to_bytes()[:200] + bytes([166, 0, 0])
        items.append(p)
    random.Random(3).shuffle(items)
    tuples = [(bp.Transcript(state=recs[id(p)]) if id(p) in recs else bp.Transcript(p.label), p.proof, p.C, p.b) for p in items]
    want = [FORMAT_ERROR if id(p) in recs else w for p, w in zip(items, expected(bp, gpu_ctx, orc, V, items))]
    for j, p in enumerate(items):
        if id(p) in recs:
            assert bp.linear_verify_batch(gpu_ctx, V.points, len(p.b) // 32, [tuples[j]], SEED) == [FORMAT_ERROR]
    assert want.count(OK) == 4 * len(P) and VERIFICATION_ERROR in want and FORMAT_ERROR in want
    assert V.verify_mixed(tuples, seed=SEED) == want


def test_parameter_codes_among_valid_proofs(bp, gpu_ctx, orc, V):
    P = pools(bp, gpu_ctx, orc, 3, [4, 8, 64])
    G = _gens(orc, 1024)[0]
    params = [
        P[8][0].replace(proof=P[8][0].proof[:-32]),                            # no proof has this length: FormatError
        P[8][1].replace(proof=P[8][1].proof + bytes(1)),                       # not whole scalars
        P[8][2].replace(b=P[4][0].b),                                          # n = 4 against 3 rounds: VerificationError
        _damaged(P[8][2].replace(b=P[4][0].b), "a non-canonical", 8, G),       # ... FormatError first
        P[4][1].replace(b=P[64][0].b),                                         # n = 64 against 2 rounds
        P[64][1].replace(b=bytes(32 * 2048)),                                  # n + 2 beyond the set: InvalidGeneratorsLength
        _damaged(P[64][1].replace(b=bytes(32 * 2048)), "r non-canonical", 64, G),
        P[4][2].replace(b=b""),                                                # n = 0: VerificationError
    ]
    want_params = [FORMAT_ERROR, FORMAT_ERROR, VERIFICATION_ERROR, FORMAT_ERROR, VERIFICATION_ERROR, INVALID_GENERATORS_LENGTH, FORMAT_ERROR,
                   VERIFICATION_ERROR]
    assert expected(bp, gpu_ctx, orc, V, params) == want_params
    valid = [p for n in P for p in P[n]]
    items = valid + params
    random.Random(4).shuffle(items)
    want = expected(bp, gpu_ctx, orc, V, items)
    assert mixed(bp, V, items) == want and want.count(OK) == len(valid)
    # with a bad admitted proof beside them
    items[items.index(valid[4])] = _damaged(valid[4], "S", 8, G)
    want = expected(bp, gpu_ctx, orc, V, items)
    assert mixed(bp, V, items) == want and want.count(OK) == len(valid) - 1
    # only rejected proofs: no kernel runs
    l0 = gpu_ctx.launches
    assert mixed(bp, V, params) == want_params and gpu_ctx.launches == l0


@pytest.mark.parametrize("n", [1, 64, 1024])
def test_one_length_gives_verify_batchs_verdicts(bp, gpu_ctx, orc, V, n):
    proofs, (G, F, B) = gpu_proofs(bp, gpu_ctx, orc, n, 40)
    items = list(proofs)
    items[7] = _damaged(items[7], "r flipped", n, G)
    items[33] = _damaged(items[33], "C", n, _gens(orc, 1024)[0])
    fixed = bp.LinearVerifier(gpu_ctx, G, F, B)
    for its in (proofs, items):
        want = fixed.verify_batch([p.item(bp) for p in its], seed=SEED)
        assert mixed(bp, V, its) == want
        assert fixed.verify_mixed([p.item(bp) for p in its], seed=SEED) == want
    fixed.close()


def test_reject_path_over_several_slices(bp, gpu_ctx, orc):
    """300 proofs at n = 4096 are re-checked in slices of 254 (rows of 4096 + 2 + 26 terms in 2^20), beside shorter proofs"""
    n = 4096
    big, (G, F, B) = gpu_proofs(bp, gpu_ctx, orc, n, 4)
    V4 = bp.LinearVerifier(gpu_ctx, G, F, B)
    short = pools(bp, gpu_ctx, orc, 4, [16, 256])
    bad = _damaged(big[2], "a flipped", n, G)
    items = [big[j % 4] for j in range(300)] + short[16] * 10 + short[256] * 5
    items[280] = bad
    random.Random(6).shuffle(items)
    want = expected(bp, gpu_ctx, orc, V4, items)
    assert want.count(VERIFICATION_ERROR) == 1 and want.count(OK) == len(items) - 1
    assert mixed(bp, V4, items) == want
    V4.close()


def test_errors_that_cancel_across_lengths_are_rejected(bp, gpu_ctx, orc, V):
    """Proof P (n = 16) with r + d and proof Q (n = 256) with r + e, e = -rho_P d / rho_Q, rho the weights a verifier blind to a || r would
    draw from each transcript and the seed: under those weights the two B errors cancel.  Both must be rejected."""
    G, F, B = _gens(orc, 1024)
    p16, q256 = gpu_proofs(bp, gpu_ctx, orc, 16, 1)[0][0], gpu_proofs(bp, gpu_ctx, orc, 256, 1)[0][0]
    blind = []
    for p, n in ((p16, 16), (q256, 256)):
        _, wire = _replay_python(bp, p, n, G[:32 * n], F, B)
        blind.append(int.from_bytes(rng_bytes(wire, SEED, 64), "little") % l)
    d = 12345
    e = (-blind[0] * d * pow(blind[1], l - 2, l)) % l

    def with_r(p, n, delta):
        k, pr = lg(n), bytearray(p.proof)
        pr[64 * k + 64:64 * k + 96] = le((int.from_bytes(pr[64 * k + 64:64 * k + 96], "little") + delta) % l)
        return p.replace(proof=bytes(pr))

    P, Q = with_r(p16, 16, d), with_r(q256, 256, e)
    assert (blind[0] * d + blind[1] * e) % l == 0
    items = [P, Q] + gpu_proofs(bp, gpu_ctx, orc, 64, 3)[0]
    want = expected(bp, gpu_ctx, orc, V, items)
    assert want == [VERIFICATION_ERROR] * 2 + [OK] * 3
    assert mixed(bp, V, items) == want


def test_seeds(bp, gpu_ctx, orc, V):
    P = pools(bp, gpu_ctx, orc, 3, [2, 32, 512])
    items = [p for n in P for p in P[n]]
    items[4] = _damaged(items[4], "label", 32, None)
    want = expected(bp, gpu_ctx, orc, V, items)
    assert want == [OK] * 4 + [VERIFICATION_ERROR] + [OK] * 4
    for seed in (bytes(32), bytes([0xA5]) * 32, None):
        assert mixed(bp, V, items, seed) == want


def test_refusals_and_non_canonical_b(bp, gpu_ctx, orc, V):
    P = pools(bp, gpu_ctx, orc, 2, [4, 16])
    items = P[4] + P[16]
    L = bp.lib()
    INV = bp.ERR_INVALID_ARGUMENT
    t, pr, C, b = bp.pack_linear([p.item(bp) for p in items])
    po, bo = bp.linear_offsets([p.item(bp) for p in items])
    U = lambda xs: (ctypes.c_uint64 * len(xs))(*xs)
    vd = ctypes.create_string_buffer(len(items))

    def call(c=gpu_ctx, set=V.points._h, count=len(items), t=t, pr=pr, po=po, C=C, b=b, bo=bo, v=vd):
        return L.bp_linear_verify_mixed(c._h, set, count, t, pr, U(po) if po is not None else None, C, b, U(bo) if bo is not None else None, SEED, v)

    assert call() == bp.OK and list(vd.raw) == [OK] * 4
    for kw in (dict(count=0), dict(set=None), dict(t=None), dict(pr=None), dict(po=None), dict(C=None), dict(b=None), dict(bo=None), dict(v=None)):
        assert call(**kw) == INV, kw
    assert call(po=[1] + po[1:]) == INV and call(bo=[1] + bo[1:]) == INV
    assert call(po=po[:2] + [po[1] - 1] + po[3:]) == INV and call(bo=bo[:3] + [bo[2] - 1] + bo[4:]) == INV
    assert call(count=1, bo=[0, (1 << 20) + 1]) == INV                          # an n above 2^20
    many = (1 << 20) + 1
    assert call(count=many, po=list(range(many + 1)), bo=[0] * (many + 1)) == INV
    assert "2^20" in L.bp_last_error(gpu_ctx._h).decode()
    G, F, B = _gens(orc, 16)
    other = bp.Context(0)
    oset = bp.PointSet(other, B + F + G)
    assert call(set=oset._h) == INV
    oset.close(); other.close()
    # a b entry >= l: of an admitted proof, and of a proof rejected on its parameters
    bad_b = bytearray(P[16][0].b); bad_b[32 * 7:32 * 8] = le(l)
    rejected = P[4][0].replace(b=bytes(32 * 2) + le(l + 1))
    for bad in (P[16][0].replace(b=bytes(bad_b)), rejected):
        with pytest.raises(bp.BpError) as e:
            mixed(bp, V, P[4] + [bad] + P[16])
        assert e.value.code == bp.ERR_NONCANONICAL_SCALAR
    # a pending range-proof begin
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "range_proof_v1.json")))
    gens = bp.Gens(gpu_ctx, 64, 1)
    rp = bytes.fromhex([q for q in golden["proofs"] if q["n"] == 64 and q["m"] == 1][0]["proof"])
    vc = bytes.fromhex(golden["value_commitments"][0])
    bv = bp.BatchVerifier(gpu_ctx, gens, bp.Transcript(golden["transcript_label"].encode()), 64, 1, 1, reserve=False)
    pbuf, cbuf = ctypes.create_string_buffer(rp, len(rp)), ctypes.create_string_buffer(vc, 32)
    bv.begin(ctypes.addressof(pbuf), ctypes.addressof(cbuf))
    assert call() == INV
    assert list(bv.finish()) == [OK]
    assert call() == bp.OK and list(vd.raw) == [OK] * 4
    gens.close()
    assert mixed(bp, V, items) == [OK] * 4


def test_beside_reserved_linear_and_range_proof_graphs(bp, orc):
    c = bp.Context(0)
    n = 16
    proofs, gfb = gpu_proofs(bp, c, orc, n, 16)
    R = bp.LinearVerifier(c, *gfb, capacity=16)
    reserved_items = proofs[:9] + [_damaged(proofs[9], "R", n, gfb[0])] + proofs[10:]
    first = device_run(bp, R, reserved_items, bytes([1]) * 32)
    assert first[0] == [OK] * 9 + [VERIFICATION_ERROR] + [OK] * 6
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "range_proof_v1.json")))
    gens = bp.Gens(c, 64, 1)
    rp = bytes.fromhex([q for q in golden["proofs"] if q["n"] == 64 and q["m"] == 1][0]["proof"])
    vc = bytes.fromhex(golden["value_commitments"][0])
    bv = bp.BatchVerifier(c, gens, bp.Transcript(golden["transcript_label"].encode()), 64, 1, 1)
    pbuf, cbuf = ctypes.create_string_buffer(rp, len(rp)), ctypes.create_string_buffer(vc, 32)

    def range_call():
        l0 = c.launches
        bv.begin(ctypes.addressof(pbuf), ctypes.addressof(cbuf))
        assert list(bv.finish()) == [OK]
        return c.launches - l0

    r0 = range_call()
    # mixed calls large enough to regrow the context's LinearProof arenas, one with the reject path
    M = bp.LinearVerifier(c, *_gens(orc, 1024))
    P = pools(bp, c, orc, 4)
    items = [P[NS[j % 11]][j % 4] for j in range(400)]
    assert M.verify_mixed([p.item(bp) for p in items], seed=SEED) == [OK] * 400
    items[123] = _damaged(items[123], "a flipped", len(items[123].b) // 32, None)
    assert M.verify_mixed([p.item(bp) for p in items], seed=SEED) == [OK] * 123 + [VERIFICATION_ERROR] + [OK] * 276
    assert device_run(bp, R, reserved_items, bytes([1]) * 32) == first
    assert range_call() == r0
    assert M.verify_mixed([p.item(bp) for p in items[:50]], seed=SEED) == [OK] * 50
    assert device_run(bp, R, reserved_items, bytes([1]) * 32) == first
    M.close(); gens.close(); R.close(); c.close()
