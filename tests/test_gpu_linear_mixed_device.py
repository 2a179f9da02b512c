"""GPU tier (-m gpu): LinearProofs of mixed lengths from device-resident buffers, bp.LinearVerifier(..., mix={n: capacity}).run_device_mixed
(bp_linear_verify_mixed_reserve + bp_linear_verify_mixed_device).  The inputs are CUDA tensors at odd byte offsets.  Every device verdict
must be what the blocking bp_linear_verify_mixed gives that proof with the same seed, or the documented code: VERDICT_UNPLACED for an
admitted proof of an unreserved length or past its class's capacity, VERDICT_NONCANONICAL_B for a placed proof with a b entry >= l.
Covered: every length 1..1024 in one call, partial fills and stale slots, over-full and unreserved classes, one bad proof per class, every
damage kind, every proof bad, a reject loop of several iterations, errors that cancel across lengths, parameter codes, non-canonical b,
launch counts, queued calls, coexistence with the other LinearProof and range-proof paths on one context, refusals and PointSet.close."""
import ctypes
import json
import os
import random
import struct

import pytest

from oracle_binding import L_ORDER as l
from test_gpu_linear_device import run as fixed_run
from test_gpu_linear_mixed import NS, damage, kinds_for
from test_linear_verify_batch import (FORMAT_ERROR, INVALID_GENERATORS_LENGTH, OK, VERIFICATION_ERROR, _damaged, _gens, _replay_python, gpu_proofs, le,
                                      lg, rng_bytes)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = bytes(range(32))
UNPLACED, NONCANON = 0xFFFFFFFF, 0xFFFFFFFE


@pytest.fixture(scope="module")
def bp():
    import bulletproofs_b200
    return bulletproofs_b200


@pytest.fixture(scope="module")
def ctx(bp):
    c = bp.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def V(bp, ctx, orc):
    """a verifier over [B, F, G_0 .. G_1023] with a mix of every length"""
    v = bp.LinearVerifier(ctx, *_gens(orc, 1024), mix={n: 6 for n in NS})
    yield v
    v.close()


@pytest.fixture(scope="module")
def P(bp, ctx, orc):
    return {n: gpu_proofs(bp, ctx, orc, n, 5)[0] for n in NS}


def _dev(data, front):
    import torch
    t = torch.frombuffer(bytearray(bytes(front) + data + bytes(16)), dtype=torch.uint8).cuda()
    return t, t.data_ptr() + front


class Call:
    """one queued device call over the items (Proof objects, or item tuples): every input at byte `front` of its allocation, proof offsets
    from `base`; inputs and outputs stay alive until result()"""

    def __init__(self, bp, V, items, seed=SEED, front=1, base=0):
        import torch
        tuples = [p if isinstance(p, tuple) else p.item(bp) for p in items]
        self.ctx, self.count = V.ctx, len(items)
        t, pr, C, b, _, bo = bp.pack_linear_mixed(tuples)
        po, _ = bp.linear_offsets(tuples)
        po = struct.pack(f"<{len(po)}Q", *[base + x for x in po])
        bufs = [_dev(x, front + j) for j, x in enumerate((t, bytes(base) + pr, po, C, b, bo))]
        self.keep = [x for x, _ in bufs]
        pt, pp, ppo, pC, pb, pbo = (a for _, a in bufs)
        self.args = (pt, pp, base + len(pr), ppo, pC, pb, len(b) // 32, pbo)       # the call's inputs, as bp_linear_verify_mixed_device takes them
        self.verd = torch.full((self.count + 1,), 77, dtype=torch.int32, device="cuda")
        self.ok = torch.full((1,), 9, dtype=torch.int32).pin_memory()
        torch.cuda.synchronize()
        l0 = self.ctx.launches
        V.run_device_mixed(*self.args, self.count, self.verd.data_ptr(), self.ok.data_ptr(), seed)
        self.launches = self.ctx.launches - l0

    def result(self):
        self.ctx.synchronize()
        v = [x & 0xFFFFFFFF for x in self.verd.cpu().tolist()]
        assert v[self.count] == 77                  # nothing written past the call's proofs
        return v[:self.count], self.ok.item()


def run(bp, V, items, seed=SEED, **kw):
    c = Call(bp, V, items, seed, **kw)
    return (*c.result(), c.launches)


def blocking(bp, V, items, seed=SEED):
    return V.verify_mixed([p.item(bp) for p in items], seed=seed)


def check(bp, V, items, seed=SEED, unplaced=(), **kw):
    """the device call agrees with the blocking call over the same items and seed, the `unplaced` indices excepted; returns (verdicts,
    h_ok, launches)"""
    got, ok, nl = run(bp, V, items, seed, **kw)
    want = blocking(bp, V, items, seed)
    for i in unplaced:
        want[i] = UNPLACED
    assert got == want, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w][:10]
    if all(w in (OK, UNPLACED) for w in want):
        assert ok == 1
    return got, ok, nl


def test_every_length_in_one_call(bp, V, P):
    items = [p for n in NS for p in P[n]]
    random.Random(1).shuffle(items)
    got, ok, _ = check(bp, V, items)
    assert got == [OK] * len(items) and ok == 1


def test_partial_fill_and_stale_slots(bp, orc, P):
    """a full call with a bad proof, then smaller calls: the slots they leave inert give no stale verdicts and no reject path"""
    c = bp.Context(0)                   # a context holds one mix: the module's stays reserved on its own
    Vm = bp.LinearVerifier(c, *_gens(orc, 1024), mix={64: 5, 256: 4, 1024: 2})
    G = _gens(orc, 1024)[0]
    full = P[64] + P[256][:4] + P[1024][:2]
    full[3] = _damaged(full[3], "a flipped", 64, G)
    got, ok, nl = check(bp, Vm, full)
    assert got.count(VERIFICATION_ERROR) == 1 and ok == 0
    for small in ([P[64][0], P[1024][1]], [P[256][2]], P[64][:2] + P[256][:1]):
        got, ok, nl2 = check(bp, Vm, small)
        assert got == [OK] * len(small) and ok == 1 and nl2 == nl
    Vm.close(); c.close()


def test_overfull_and_unreserved_classes(bp, orc, P):
    """the later proofs of over-full classes and every proof of an unreserved length are unplaced; the others are verified"""
    c = bp.Context(0)
    Vm = bp.LinearVerifier(c, *_gens(orc, 1024), mix={64: 3, 256: 2})
    G = _gens(orc, 1024)[0]
    items = P[64] + P[256][:3] + P[16][:2] + [_damaged(P[256][3], "S", 256, G)]
    order = list(range(len(items)))
    random.Random(2).shuffle(order)
    items = [items[i] for i in order]
    seen, unplaced = {}, []
    for i, p in enumerate(items):
        n = len(p.b) // 32
        seen[n] = seen.get(n, 0) + 1
        if n not in (64, 256) or seen[n] > {64: 3, 256: 2}[n]:
            unplaced.append(i)
    got, _, _ = check(bp, Vm, items, unplaced=unplaced)
    assert got.count(UNPLACED) == len(unplaced) == 6
    # resubmitting exactly the unplaced proofs of the reserved lengths places them
    again = [items[i] for i in unplaced if len(items[i].b) // 32 in (64, 256)]
    check(bp, Vm, again[:3])
    Vm.close(); c.close()


def test_one_bad_proof_in_each_class_in_turn(bp, V, P, orc):
    G = _gens(orc, 1024)[0]
    base = [P[NS[j % 11]][(j // 11) % 5] for j in range(55)]
    _, _, ok_launches = check(bp, V, base)
    for c, n in enumerate(NS):
        at = next(j for j, p in enumerate(base) if len(p.b) == 32 * n)
        kind = kinds_for(n)[c % len(kinds_for(n))]
        items = list(base)
        items[at] = damage(base[at], kind, n, G)
        got, _, nl = check(bp, V, items)
        assert got[at] != OK and got[:at] + got[at + 1:] == [OK] * 54, (n, kind)
        assert nl == ok_launches


def test_every_damage_kind(bp, V, P, orc):
    G = _gens(orc, 1024)[0]
    items = []
    for n in (1, 2, 16, 64, 256):
        kinds = kinds_for(n)
        items += [damage(P[n][j % 5], kinds[j], n, G) for j in range(min(len(kinds), 5))]
        items += P[n][:1]
    got, ok, _ = check(bp, V, items)
    assert got.count(OK) >= 5 and FORMAT_ERROR in got and VERIFICATION_ERROR in got and ok == 0
    rest = kinds_for(64)[5:]
    for j0 in range(0, len(rest), 5):                        # a class holds 6: five damaged proofs and a valid one per call
        got, _, _ = check(bp, V, [damage(P[64][j % 5], rest[j], 64, G) for j in range(j0, min(j0 + 5, len(rest)))] + P[64][:1])
        assert got[-1] == OK and OK not in got[:-1]


def test_every_proof_bad(bp, V, P, orc):
    G = _gens(orc, 1024)[0]
    items = [_damaged(P[n][j], "a flipped", n, G) for n in NS for j in range(3)]
    got, ok, _ = check(bp, V, items)
    assert got == [VERIFICATION_ERROR] * len(items) and ok == 0


def test_reject_loop_of_several_iterations(bp, ctx, orc):
    """300 proofs at n = 4096 are re-checked 254 per iteration (rows of 4096 + 2 + 26 terms in 2^20): a bad proof in the second slice"""
    n = 4096
    big, (G, F, B) = gpu_proofs(bp, ctx, orc, n, 4)
    short = gpu_proofs(bp, ctx, orc, 16, 4)[0]
    c = bp.Context(0)
    Vm = bp.LinearVerifier(c, G, F, B, mix={16: 8, n: 300})
    items = [big[j % 4] for j in range(300)] + short
    items[280] = _damaged(big[2], "a flipped", n, G)
    items[302] = _damaged(short[2], "S", 16, G)
    got, ok, _ = check(bp, Vm, items)
    assert [i for i, v in enumerate(got) if v != OK] == [280, 302] and ok == 0
    Vm.close(); c.close()


def test_errors_that_cancel_across_lengths(bp, ctx, V, orc):
    """P (n = 16) with r + d and Q (n = 256) with r + e, e = -rho_P d / rho_Q under weights blind to a || r: both rejected"""
    G, F, B = _gens(orc, 1024)
    p16, q256 = gpu_proofs(bp, ctx, orc, 16, 1)[0][0], gpu_proofs(bp, ctx, orc, 256, 1)[0][0]
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

    items = [with_r(p16, 16, d), with_r(q256, 256, e)] + gpu_proofs(bp, ctx, orc, 64, 3)[0]
    got, _, _ = check(bp, V, items)
    assert got == [VERIFICATION_ERROR] * 2 + [OK] * 3


def test_parameter_codes_among_valid_proofs(bp, V, P, orc):
    G = _gens(orc, 1024)[0]
    params = [
        P[8][0].replace(proof=P[8][0].proof[:-32]),                            # no proof has this length: FormatError
        P[8][1].replace(proof=P[8][1].proof + bytes(1)),                       # not whole scalars
        P[8][2].replace(b=P[4][0].b),                                          # n = 4 against 3 rounds: VerificationError
        _damaged(P[8][2].replace(b=P[4][0].b), "a non-canonical", 8, G),       # ... FormatError first
        P[64][1].replace(b=bytes(32 * 2048)),                                  # n + 2 beyond the set: InvalidGeneratorsLength
        P[4][2].replace(b=b""),                                                # n = 0: VerificationError
    ]
    items = [p for n in (4, 8, 64) for p in P[n]] + params
    random.Random(4).shuffle(items)
    got, _, _ = check(bp, V, items)
    assert got.count(OK) == 15 and INVALID_GENERATORS_LENGTH in got and got.count(FORMAT_ERROR) == 3


def test_non_canonical_b(bp, V, P):
    """a placed proof with a b entry >= l gets VERDICT_NONCANONICAL_B and stays out of the combination; the blocking form refuses it"""
    bad_b = bytearray(P[16][0].b); bad_b[32 * 7:32 * 8] = le(l)
    bad = P[16][0].replace(b=bytes(bad_b))
    items = P[4] + [bad] + P[16][1:]
    got, ok, _ = run(bp, V, items)
    assert got == [OK] * 5 + [NONCANON] + [OK] * 4 and ok == 1
    with pytest.raises(bp.BpError) as e:
        blocking(bp, V, items)
    assert e.value.code == bp.ERR_NONCANONICAL_SCALAR


def test_launches_do_not_depend_on_fill_or_bad_proofs(bp, V, P, orc):
    G = _gens(orc, 1024)[0]
    calls = [[P[1024][0]], [p for n in NS for p in P[n]], [_damaged(P[n][0], "C", n, G) for n in NS], P[64] + P[64] + P[2],
             [P[32][0].replace(proof=b"")]]
    counts = {run(bp, V, items)[2] for items in calls}
    assert len(counts) == 1 and counts.pop() > 0


def test_queued_calls(bp, V, P, orc):
    """4 calls with different inputs and seeds queued, then one synchronise: each gets its own verdicts"""
    G = _gens(orc, 1024)[0]
    sets = []
    for j in range(4):
        items = [P[NS[(j + i) % 11]][i % 5] for i in range(20 + 7 * j)]
        items[j * 3] = _damaged(items[j * 3], "r flipped", len(items[j * 3].b) // 32, G)
        sets.append((items, bytes([j + 1]) * 32))
    calls = [Call(bp, V, items, seed, front=j + 1) for j, (items, seed) in enumerate(sets)]
    for c, (items, seed) in zip(calls, sets):
        got, ok = c.result()
        assert got == blocking(bp, V, items, seed) and ok == 0


def test_beside_other_paths_on_one_context(bp, orc):
    """a fixed LinearProof reservation, blocking LinearProof calls, a reserved range-proof graph and the mix on one context"""
    c = bp.Context(0)
    n = 16
    proofs, gfb = gpu_proofs(bp, c, orc, n, 16)
    R = bp.LinearVerifier(c, *gfb, capacity=16)
    reserved_items = proofs[:9] + [_damaged(proofs[9], "R", n, gfb[0])] + proofs[10:]
    first = fixed_run(bp, R, reserved_items, bytes([1]) * 32)
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "range_proof_v1.json")))
    gens = bp.Gens(c, 64, 1)
    rp = bytes.fromhex([q for q in golden["proofs"] if q["n"] == 64 and q["m"] == 1][0]["proof"])
    vc = bytes.fromhex(golden["value_commitments"][0])
    bv = bp.BatchVerifier(c, gens, bp.Transcript(golden["transcript_label"].encode()), 64, 1, 1)
    pbuf, cbuf = ctypes.create_string_buffer(rp, len(rp)), ctypes.create_string_buffer(vc, 32)

    def range_call():
        bv.begin(ctypes.addressof(pbuf), ctypes.addressof(cbuf))
        assert list(bv.finish()) == [OK]

    range_call()
    M = bp.LinearVerifier(c, *_gens(orc, 1024), mix={16: 8, 256: 8, 1024: 4})
    Pm = {k: gpu_proofs(bp, c, orc, k, 4)[0] for k in (16, 256, 1024)}
    items = Pm[16] + Pm[256] + Pm[1024][:2]
    items[5] = _damaged(items[5], "a flipped", 256, None)
    mixed_first = check(bp, M, items)[0]
    big = [Pm[(16, 256, 1024)[j % 3]][j % 4] for j in range(300)]
    assert M.verify_mixed([p.item(bp) for p in big], seed=SEED) == [OK] * 300        # regrows the blocking arenas
    assert fixed_run(bp, R, reserved_items, bytes([1]) * 32) == first
    range_call()
    assert check(bp, M, items)[0] == mixed_first
    assert R.verify_mixed([p.item(bp) for p in proofs[:4]], seed=SEED) == [OK] * 4
    assert fixed_run(bp, R, reserved_items, bytes([1]) * 32) == first
    M.close(); gens.close(); R.close(); c.close()


def test_refusals_queue_nothing(bp, ctx, V, P, orc):
    L, INV = bp.lib(), bp.ERR_INVALID_ARGUMENT
    items = P[4][:2] + P[64][:2]
    call = Call(bp, V, items)
    assert call.result()[0] == [OK] * 4
    pt, pp, pbytes, ppo, pC, pb, nb, pbo = call.args

    def raw(set=V.points._h, count=4, t=pt, pr=pp, po=ppo, C=pC, b=pb, bo=pbo, v=call.verd.data_ptr(), c=ctx):
        return L.bp_linear_verify_mixed_device(c._h, set, count, t, pr, pbytes, po, C, b, nb, bo, SEED, v, None)

    other = bp.LinearVerifier(ctx, *_gens(orc, 16))            # a set with no mix on this context
    l0 = ctx.launches
    for kw in (dict(set=None), dict(t=None), dict(pr=None), dict(po=None), dict(C=None), dict(b=None), dict(bo=None), dict(v=None), dict(count=0),
               dict(count=1 << 24), dict(v=call.verd.data_ptr() + 2)):
        assert raw(**kw) == INV, kw
    assert raw(set=other.points._h) == INV
    assert ctx.launches == l0
    # reserve refusals leave the mix in place
    U = lambda xs: (ctypes.c_uint32 * max(len(xs), 1))(*xs)
    h = V.points._h
    for ns, caps in (([], []), ([1 << k for k in range(11)] * 2, [1] * 22), ([64, 64], [1, 1]), ([48], [1]), ([0], [1]), ([1 << 21], [1]), ([2048], [1]),
                     ([64], [0]), ([64], [(1 << 20) + 1])):
        assert L.bp_linear_verify_mixed_reserve(ctx._h, h, len(ns), U(ns), U(caps)) == INV, ns
    assert L.bp_linear_verify_mixed_reserve(ctx._h, None, 1, U([4]), U([1])) == INV
    c2 = bp.Context(0)
    assert L.bp_linear_verify_mixed_reserve(c2._h, h, 1, U([4]), U([1])) == INV
    c2.close()
    # a pending range-proof begin
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "range_proof_v1.json")))
    gens = bp.Gens(ctx, 64, 1)
    rp = bytes.fromhex([q for q in golden["proofs"] if q["n"] == 64 and q["m"] == 1][0]["proof"])
    vc = bytes.fromhex(golden["value_commitments"][0])
    bv = bp.BatchVerifier(ctx, gens, bp.Transcript(golden["transcript_label"].encode()), 64, 1, 1, reserve=False)
    pbuf, cbuf = ctypes.create_string_buffer(rp, len(rp)), ctypes.create_string_buffer(vc, 32)
    bv.begin(ctypes.addressof(pbuf), ctypes.addressof(cbuf))
    l0 = ctx.launches
    assert raw() == INV and L.bp_linear_verify_mixed_reserve(ctx._h, h, 1, U([4]), U([1])) == INV and ctx.launches == l0
    assert list(bv.finish()) == [OK]
    gens.close()
    assert call.result()[0] == [OK] * 4                         # the queued-nothing calls wrote nothing
    assert run(bp, V, items)[0] == [OK] * 4                     # the mix is still reserved
    other.close()


def test_point_set_close_ends_the_mix(bp, orc, P):
    L = bp.lib()
    ctx = bp.Context(0)
    Vm = bp.LinearVerifier(ctx, *_gens(orc, 64), mix={4: 2, 64: 2})
    items = P[4][:2] + P[64][:1]
    assert run(bp, Vm, items)[0] == [OK] * 3
    call = Call(bp, Vm, items)
    call.result()
    h = Vm.points._h.value
    Vm.close()
    l0 = ctx.launches
    rc = L.bp_linear_verify_mixed_device(ctx._h, h, 3, *call.args, SEED, call.verd.data_ptr(), None)
    assert rc == bp.ERR_INVALID_ARGUMENT and ctx.launches == l0
    assert "no LinearProof mix" in L.bp_last_error(ctx._h).decode()
    ctx.close()
