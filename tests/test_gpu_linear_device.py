"""GPU tier (-m gpu): reserved LinearProof verification on device-resident inputs, bp.LinearVerifier(..., capacity=C).run_device
(bp_linear_verify_reserve + bp_linear_verify_device).  Every device verdict must be the blocking form's (verify_batch, the same seed) and
the single path's and the oracle's for that proof alone, whatever the pattern of bad proofs and whatever the fill of the reservation; a
proof with a non-canonical b gets VERDICT_NONCANONICAL_B.  Calls queue back to back without mixing their parameters, launch the same
kernels whatever the number of bad proofs, and the graph keeps working beside blocking LinearProof calls and a reserved range-proof
verifier on the same context."""
import ctypes
import json
import os

import pytest

from oracle_binding import L_ORDER as l
from test_linear_verify_batch import FORMAT_ERROR, KINDS, OK, VERIFICATION_ERROR, _damaged, gpu_proofs, le, lg, single

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def upload(bp, proofs, front=1):
    """pack_linear's four buffers of the proofs in device memory, each from byte `front` of its allocation (any alignment): (tensors,
    addresses)"""
    import torch
    bufs = [torch.frombuffer(bytearray(bytes(front) + x + bytes(16)), dtype=torch.uint8).cuda() for x in bp.pack_linear([p.item(bp) for p in proofs])]
    return bufs, [t.data_ptr() + front for t in bufs]


class Call:
    """one queued device call: its inputs and outputs stay alive until result()"""

    def __init__(self, bp, V, items, seed, front=1):
        import torch
        self.ctx, self.count = V.ctx, len(items)
        self.bufs, ptrs = upload(bp, items, front)
        self.verd = torch.full((self.count + 1,), 77, dtype=torch.int32, device="cuda")
        self.ok = torch.full((1,), 9, dtype=torch.int32).pin_memory()
        torch.cuda.synchronize()
        l0 = self.ctx.launches
        V.run_device(*ptrs, self.count, self.verd.data_ptr(), self.ok.data_ptr(), seed)
        self.launches = self.ctx.launches - l0

    def result(self):
        self.ctx.synchronize()
        v = [x & 0xFFFFFFFF for x in self.verd.cpu().tolist()]
        assert v[self.count] == 77                  # nothing written past the call's proofs
        return v[:self.count], self.ok.item()


def run(bp, V, items, seed):
    c = Call(bp, V, items, seed)
    return (*c.result(), c.launches)


def check(bp, V, items, seed, want=None):
    """the device call agrees with the blocking call with the same seed (and with `want`); returns (verdicts, h_ok, launches)"""
    got, ok, nl = run(bp, V, items, seed)
    host = V.verify_batch([p.item(bp) for p in items], seed=seed)
    assert got == host, [(i, g, h) for i, (g, h) in enumerate(zip(got, host)) if g != h][:10]
    if want is not None:
        assert got == want
    if all(v == OK for v in got):
        assert ok == 1
    return got, ok, nl


@pytest.fixture(scope="module")
def ctx():
    import bulletproofs_b200 as bp
    c = bp.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("n", [1, 2, 16, 64, 1024])
def test_all_valid_at_every_fill(ctx, orc, n):
    import bulletproofs_b200 as bp
    cap = 40
    proofs, gfb = gpu_proofs(bp, ctx, orc, n, cap)
    assert [single(bp, ctx, orc, gfb, p) for p in proofs[:2]] == [OK, OK]
    V = bp.LinearVerifier(ctx, *gfb, capacity=cap)
    for fill in (1, 31, 32, 33, cap):
        got, ok, _ = check(bp, V, proofs[:fill], bytes([fill]) * 32, [OK] * fill)
        assert ok == 1
    V.close()


@pytest.mark.parametrize("kind", KINDS)
def test_one_bad_proof_among_64(ctx, orc, kind):
    import bulletproofs_b200 as bp
    n = 16
    proofs, gfb = gpu_proofs(bp, ctx, orc, n, 64)
    bad = _damaged(proofs[17], kind, n, gfb[0])
    code = single(bp, ctx, orc, gfb, bad)
    V = bp.LinearVerifier(ctx, *gfb, capacity=64)
    items = proofs[:17] + [bad] + proofs[18:]
    _, ok, _ = check(bp, V, items, bytes(32), [OK] * 17 + [code] + [OK] * 46)
    if kind != "R":                                     # the flipped R bit may leave a point that does not decode: left out as well
        assert ok == (1 if code == FORMAT_ERROR else 0)  # a FormatError proof is left out before the combination
    V.close()


def test_every_proof_bad(ctx, orc):
    import bulletproofs_b200 as bp
    n = 64
    proofs, gfb = gpu_proofs(bp, ctx, orc, n, 40)
    items = [_damaged(p, KINDS[j % len(KINDS)], n, gfb[0]) for j, p in enumerate(proofs)]
    want = [single(bp, ctx, orc, gfb, p) for p in items]
    assert OK not in want
    V = bp.LinearVerifier(ctx, *gfb, capacity=48)
    check(bp, V, items, bytes([3]) * 32, want)
    V.close()


def test_bad_proofs_in_both_reject_iterations(ctx, orc):
    """n = 1024, capacity 1030: the reject loop checks 1000 proofs per iteration, so [0, 1000) and [1000, 1030) are two iterations"""
    import bulletproofs_b200 as bp
    n, count = 1024, 1030
    proofs, gfb = gpu_proofs(bp, ctx, orc, n, 4)
    bads = [_damaged(proofs[j], kind, n, gfb[0]) for j, kind in enumerate(("a flipped", "R", "C", "b_i"))]
    want_bad = [single(bp, ctx, orc, gfb, p) for p in bads]
    bad_at = {5, 500, 999, 1000, 1017, 1029}
    items = [bads[i % 4] if i in bad_at else proofs[i % 4] for i in range(count)]
    want = [want_bad[i % 4] if i in bad_at else OK for i in range(count)]
    V = bp.LinearVerifier(ctx, *gfb, capacity=count)
    _, ok, _ = check(bp, V, items, bytes(range(32)), want)
    assert ok == 0
    V.close()


def test_non_canonical_b_and_malformed_records(ctx, orc):
    import bulletproofs_b200 as bp
    n = 16
    proofs, gfb = gpu_proofs(bp, ctx, orc, n, 24)
    V = bp.LinearVerifier(ctx, *gfb, capacity=24)
    bad_b = bytearray(proofs[4].b); bad_b[32 * 3:32 * 4] = le(l)
    items = proofs[:4] + [proofs[4].replace(b=bytes(bad_b))] + proofs[5:]
    got, ok, _ = run(bp, V, items, bytes(32))
    assert got == [OK] * 4 + [bp.VERDICT_NONCANONICAL_B] + [OK] * 19 and ok == 1
    with pytest.raises(bp.BpError) as e:
        V.verify_batch([p.item(bp) for p in items], seed=bytes(32))
    assert e.value.code == bp.ERR_NONCANONICAL_SCALAR
    # the same with a bad proof beside it: the reject path leaves the non-canonical proof's code alone
    items[9] = _damaged(items[9], "r flipped", n, gfb[0])
    got, ok, _ = run(bp, V, items, bytes(32))
    assert got == [OK] * 4 + [bp.VERDICT_NONCANONICAL_B] + [OK] * 4 + [VERIFICATION_ERROR] + [OK] * 14 and ok == 0
    # records no transcript can hold: FormatError, in the blocking form as well
    items = list(proofs)
    recs = [bp.Transcript(p.label).to_bytes() for p in items]
    for j, (pos, pb) in zip((2, 7, 20), ((166, 0), (255, 1), (10, 11))):
        recs[j] = recs[j][:200] + bytes([pos, pb, 0])
    import torch
    tr, pr, C, b = bp.pack_linear([p.item(bp) for p in items])
    tr = b"".join(recs)
    bufs = [torch.frombuffer(bytearray(x + bytes(16)), dtype=torch.uint8).cuda() for x in (tr, pr, C, b)]
    verd = torch.zeros(24, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    V.run_device(*[t.data_ptr() for t in bufs], 24, verd.data_ptr())
    ctx.synchronize()
    want = [FORMAT_ERROR if j in (2, 7, 20) else OK for j in range(24)]
    assert verd.cpu().tolist() == want
    host = V.verify_batch([(bp.Transcript(state=recs[j]), p.proof, p.C, p.b) for j, p in enumerate(items)], seed=bytes(32))
    assert host == want
    V.close()


def test_inert_slots_after_a_full_call(ctx, orc):
    import bulletproofs_b200 as bp
    n = 64
    proofs, gfb = gpu_proofs(bp, ctx, orc, n, 40)
    V = bp.LinearVerifier(ctx, *gfb, capacity=40)
    full = proofs[:30] + [_damaged(p, k, n, gfb[0]) for p, k in zip(proofs[30:], KINDS)]
    got, ok, _ = check(bp, V, full, bytes([5]) * 32)
    assert got[:30] == [OK] * 30 and OK not in got[30:] and ok == 0
    for fill in (1, 17, 30):
        got, ok, _ = check(bp, V, proofs[:fill], bytes([5]) * 32, [OK] * fill)
        assert ok == 1
    V.close()


def test_four_calls_queued_then_one_synchronise(ctx, orc):
    import bulletproofs_b200 as bp
    n = 16
    proofs, gfb = gpu_proofs(bp, ctx, orc, n, 64)
    V = bp.LinearVerifier(ctx, *gfb, capacity=64)
    plans = [(proofs[:64], {}), (proofs[:7], {3: "S"}), (proofs[:33], {0: "label", 32: "C"}), (proofs[:50], {})]
    specs = []
    for j, (base, bad) in enumerate(plans):
        items = [_damaged(p, bad[i], n, gfb[0]) if i in bad else p for i, p in enumerate(base)]
        specs.append((items, bytes([j + 40]) * 32))
    calls = [Call(bp, V, items, seed, front=j) for j, (items, seed) in enumerate(specs)]
    results = [c.result() for c in calls]              # the first result() synchronises the context once for all four
    for (items, seed), (got, ok) in zip(specs, results):
        want = V.verify_batch([p.item(bp) for p in items], seed=seed)
        assert got == want and ok == (1 if all(v == OK for v in want) else 0)
    V.close()


def test_launches_do_not_depend_on_bad_proofs(ctx, orc):
    import bulletproofs_b200 as bp
    n = 16
    proofs, gfb = gpu_proofs(bp, ctx, orc, n, 32)
    V = bp.LinearVerifier(ctx, *gfb, capacity=32)
    bad = [_damaged(p, "a flipped", n, gfb[0]) for p in proofs]
    counts = [check(bp, V, items, bytes(32))[2] for items in (proofs, proofs[:5] + bad[5:6] + proofs[6:], bad)]
    assert len(set(counts)) == 1 and counts[0] > 0
    V.close()


def test_beside_blocking_and_range_proof_graphs(orc):
    import bulletproofs_b200 as bp
    n = 16
    c = bp.Context(0)
    proofs, gfb = gpu_proofs(bp, c, orc, n, 96)
    V = bp.LinearVerifier(c, *gfb, capacity=16)
    items = proofs[:12] + [_damaged(proofs[12], "R", n, gfb[0])] + proofs[13:16]
    first = check(bp, V, items, bytes([1]) * 32)
    # a larger blocking call regrows the context's own arenas; the reservation's are its own
    big = proofs[:60] + [_damaged(proofs[60], "S", n, gfb[0])] + proofs[61:96]
    assert V.verify_batch([p.item(bp) for p in big], seed=bytes(32)) == [OK] * 60 + [VERIFICATION_ERROR] + [OK] * 35
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
    assert check(bp, V, items, bytes([1]) * 32) == first
    assert range_call() == r0
    assert V.verify_batch([p.item(bp) for p in big[:40]], seed=bytes(32)) == [OK] * 40
    assert check(bp, V, items, bytes([1]) * 32) == first
    gens.close(); V.close(); c.close()


def test_refusals(orc):
    import torch
    import bulletproofs_b200 as bp
    n = 16
    c = bp.Context(0)
    L = bp.lib()
    INV = bp.ERR_INVALID_ARGUMENT
    proofs, (G, F, B) = gpu_proofs(bp, c, orc, n, 8)
    bufs, ptrs = upload(bp, proofs[:8])
    verd = torch.zeros(9, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    plen = len(proofs[0].proof)
    V = bp.LinearVerifier(c, G, F, B)                   # no reservation yet
    dev = lambda **kw: L.bp_linear_verify_device(c._h, kw.get("set", V.points._h), kw.get("n", n), kw.get("count", 8), kw.get("t", ptrs[0]), kw.get("p", ptrs[1]),
                                                 kw.get("plen", plen), kw.get("C", ptrs[2]), kw.get("b", ptrs[3]), None, kw.get("v", verd.data_ptr()), None)
    assert dev() == INV
    # reserve refusals
    other = bp.Context(0)
    oset = bp.PointSet(other, B + F + G)
    small = bp.PointSet(c, B + F + G[:32 * (n - 1)])
    for args in ((oset._h, n, 8), (small._h, n, 8), (V.points._h, 12, 8), (V.points._h, 0, 8), (V.points._h, 1 << 21, 8), (V.points._h, n, 0),
                 (V.points._h, n, (1 << 20) + 1), (None, n, 8)):
        assert L.bp_linear_verify_reserve(c._h, *args) == INV, args
    assert L.bp_linear_verify_reserve(c._h, V.points._h, n, 8) == bp.OK
    assert dev() == bp.OK
    c.synchronize()
    assert verd.cpu().tolist()[:8] == [OK] * 8
    # device-call refusals, nothing queued
    l0 = c.launches
    for kw in (dict(set=small._h), dict(n=8), dict(count=0), dict(count=9), dict(t=None), dict(p=None), dict(C=None), dict(b=None), dict(v=None),
               dict(v=verd.data_ptr() + 2), dict(plen=plen - 32), dict(plen=plen + 1), dict(set=None)):
        assert dev(**kw) == INV, kw
    assert c.launches == l0
    # a pending range-proof begin
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "range_proof_v1.json")))
    gens = bp.Gens(c, 64, 1)
    rp = bytes.fromhex([q for q in golden["proofs"] if q["n"] == 64 and q["m"] == 1][0]["proof"])
    vc = bytes.fromhex(golden["value_commitments"][0])
    bv = bp.BatchVerifier(c, gens, bp.Transcript(golden["transcript_label"].encode()), 64, 1, 1, reserve=False)
    pbuf, cbuf = ctypes.create_string_buffer(rp, len(rp)), ctypes.create_string_buffer(vc, 32)
    bv.begin(ctypes.addressof(pbuf), ctypes.addressof(cbuf))
    assert dev() == INV
    assert L.bp_linear_verify_reserve(c._h, V.points._h, n, 8) == INV
    assert list(bv.finish()) == [OK]
    assert dev() == bp.OK
    # destroying the reserved set ends the reservation, even for a new set at the same address
    V.points.close()
    again = bp.PointSet(c, B + F + G)
    assert dev(set=again._h) == INV
    assert L.bp_linear_verify_reserve(c._h, again._h, n, 8) == bp.OK
    assert dev(set=again._h) == bp.OK
    c.synchronize()
    assert verd.cpu().tolist()[:8] == [OK] * 8
    again.close(); small.close(); oset.close(); gens.close(); other.close(); c.close()
