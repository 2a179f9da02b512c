"""GPU tier (-m gpu): the exact device-resident verifiers, bp.BatchVerifier(..., exact=True).run_device_exact,
bp.verify_group_device_exact_each and bp.MixedVerifier(..., exact=True).run_device_exact(_each).  Their device verdicts must be the host
forms' (group begin + finish, verify_mixed) with the same seed and the oracle's verdict of each proof alone, whatever the pattern of bad
proofs; their flags must be the plain device call's; and the plain graphs keep working beside them."""
import random

import pytest

from test_gpu_geometry import _cell, _damage
from test_gpu_group_check import LABEL, _bad
from test_gpu_mixed_device import Call, KEYS
from test_gpu_mixed_service import FULL, MIX, _damaged, oracle, tx
from test_gpu_per_proof_transcripts import malformed_record

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def og(orc):
    return orc.gens(64, 32)


def _tile(orc, og, m, total):
    """`total` (64, m) oracle proofs tiled from the cell: (bytearray proofs, bytearray commitments, proof length)"""
    proofs, Vs, plen = _cell(orc, og, 64, m)
    per = len(proofs) // plen
    reps = -(-total // per)
    return bytearray((proofs * reps)[:total * plen]), bytearray((Vs * reps)[:total * 32 * m]), plen


def _items(pb, vb, plen, m, total):
    return [(bytes(pb[i * plen:(i + 1) * plen]), bytes(vb[32 * m * i:32 * m * (i + 1)]), 64) for i in range(total)]


class Fixed:
    """a context of its own with (64, m) x count x nb reserved with the exact graph"""

    def __init__(self, m, count, nb):
        import bulletproofs_b200 as bp
        self.m, self.count, self.nb = m, count, nb
        self.ctx = bp.Context(0)
        self.gens = bp.Gens(self.ctx, 64, 32)
        self.v = bp.BatchVerifier(self.ctx, self.gens, bp.Transcript(LABEL), 64, m, count, nb, exact=True)

    def prep(self, pb, vb, records=None):
        """one call's device inputs and outputs, uploaded"""
        import torch
        dev = lambda b: torch.frombuffer(bytearray(bytes(b) + bytes(16)), dtype=torch.uint8).cuda()
        d_p, d_v = dev(pb), dev(vb)
        d_t = dev(b"".join(records)) if records else None
        verd = torch.full((self.count * self.nb,), 77, dtype=torch.int32, device="cuda")
        ok = torch.full((self.nb,), 9, dtype=torch.int32).pin_memory()
        torch.cuda.synchronize()
        return (d_p, d_v, d_t, verd, ok, records)

    def launch(self, h, seed, exact=True):
        """queue one device call without synchronising"""
        import bulletproofs_b200 as bp
        d_p, d_v, d_t, verd, ok, records = h
        if records:
            bp.verify_group_device_exact_each(self.ctx, self.gens, d_t.data_ptr(), d_p.data_ptr(), d_v.data_ptr(), 64, self.m, self.count, self.nb,
                                              verd.data_ptr(), ok.data_ptr(), seed)
        elif exact:
            self.v.run_device_exact(d_p.data_ptr(), d_v.data_ptr(), verd.data_ptr(), ok.data_ptr(), seed)
        else:
            self.v.run_device(d_p.data_ptr(), d_v.data_ptr(), verd.data_ptr(), ok.data_ptr(), seed)
        return h

    def result(self, h):
        self.ctx.synchronize()
        return [x & 0xFFFFFFFF for x in h[3].cpu().tolist()], h[4].tolist()

    def run(self, pb, vb, seed, **kw):
        l0 = self.ctx.launches
        h = self.launch(self.prep(pb, vb, kw.pop("records", None)), seed, **kw)
        dl = self.ctx.launches - l0
        return (*self.result(h), dl)

    def host(self, pb, vb, seed, records=None):
        """the host form on the same context: (verdicts, batch flags)"""
        import bulletproofs_b200 as bp
        if records:
            return bp.verify_group_each(self.ctx, self.gens, b"".join(records), bytes(pb), bytes(vb), 64, self.m, self.count, self.nb, seed=seed)
        return bp.verify_group(self.ctx, self.gens, bp.Transcript(LABEL), bytes(pb), bytes(vb), 64, self.m, self.count, self.nb, seed=seed)

    def close(self):
        self.gens.close()
        self.ctx.close()


@pytest.fixture(scope="module")
def fx():
    f = Fixed(1, 100, 3)
    yield f
    f.close()


def _want(orc, og, pb, vb, plen, m, total, records=None):
    return oracle(orc, og, _items(pb, vb, plen, m, total), records)


def _check(orc, og, f, pb, vb, plen, seed, records=None):
    total = f.count * f.nb
    got, ok, dl = f.run(pb, vb, seed, records=records)
    hv, hok = f.host(pb, vb, seed, records)
    want = _want(orc, og, pb, vb, plen, f.m, total, records)
    assert got == hv == want, [(i, g, h, w) for i, (g, h, w) in enumerate(zip(got, hv, want)) if not g == h == w][:20]
    assert ok == hok
    return got, ok, dl


PATTERNS = {
    "none": [],
    "one": [150],
    "several_in_one_chunk": [200, 201, 203, 207, 231],
    "one_in_each_of_seven_chunks": [0, 40, 70, 110, 140, 180, 250],
    "last_batch_only": [200, 299],
    "every_proof": list(range(300)),
}


@pytest.mark.parametrize("name", list(PATTERNS))
def test_fixed_bad_patterns(orc, og, fx, name):
    pb, vb, plen = _tile(orc, og, 1, 300)
    for i in PATTERNS[name]:
        _bad(pb, plen, i)
    got, ok, _ = _check(orc, og, fx, pb, vb, plen, bytes([5]) * 32)
    assert [i for i, v in enumerate(got) if v] == PATTERNS[name]
    assert ok == [int(not any(b * 100 <= i < b * 100 + 100 for i in PATTERNS[name])) for b in range(3)]


def test_fixed_damage_next_to_malformed(orc, og, fx):
    """the six damage kinds (non-canonical scalar and undecodable point among them) in batch 1, one invalid proof in batch 2"""
    pb, vb, plen = _tile(orc, og, 1, 300)
    at = _damage(pb, vb, plen, 64, 1, base=100)
    _bad(pb, plen, 260)
    got, ok, _ = _check(orc, og, fx, pb, vb, plen, bytes([6]) * 32)
    assert [i for i, v in enumerate(got) if v] == at + [260] and ok == [1, 0, 0]
    assert 2 in got and 1 in got


def test_fixed_records_with_malformed_ones(orc, og, fx):
    rnd = random.Random(7)
    pb, vb, plen = _tile(orc, og, 1, 300)
    for i in (3, 77, 120):
        _bad(pb, plen, i)
    records = [orc.transcript(LABEL)[:203]] * 300
    for i, kind in ((5, 0), (130, 1), (299, 0)):
        records[i] = malformed_record(rnd, kind)
    got, ok, _ = _check(orc, og, fx, pb, vb, plen, bytes([7]) * 32, records=records)
    assert [i for i, v in enumerate(got) if v] == [3, 5, 77, 120, 130, 299]


def test_fixed_launches_do_not_depend_on_bad_proofs(orc, og, fx):
    pb, vb, plen = _tile(orc, og, 1, 300)
    launches = []
    for bad in ([], [42], list(range(300))):
        b = bytearray(pb)
        for i in bad:
            _bad(b, plen, i)
        launches.append(_check(orc, og, fx, b, vb, plen, bytes([8]) * 32)[2])
    assert len(set(launches)) == 1 and launches[0] > 0


def test_queued_calls_and_the_plain_graph(orc, og, fx):
    """four exact calls with their own bad sets and a plain one, queued without synchronising: each exact call is exact, the plain call
    still marks its failing batch's well-formed proofs VerificationError"""
    pb, vb, plen = _tile(orc, og, 1, 300)
    sets = [[], [1, 2, 3], [99, 100, 101, 250], list(range(0, 300, 7))]
    bufs = []
    for bad in sets:
        b = bytearray(pb)
        for i in bad:
            _bad(b, plen, i)
        bufs.append(b)
    hs = [fx.prep(b, vb) for b in bufs] + [fx.prep(bufs[1], vb)]
    calls = [fx.launch(h, bytes([10 + k]) * 32) for k, h in enumerate(hs[:4])]
    plain = fx.launch(hs[4], bytes([20]) * 32, exact=False)
    for k, (bad, h) in enumerate(zip(sets, calls)):
        got, ok = fx.result(h)
        assert got == _want(orc, og, bufs[k], vb, plen, 1, 300) and [i for i, v in enumerate(got) if v] == bad
    got, ok = fx.result(plain)
    assert got == [1] * 100 + [0] * 200 and ok == [0, 1, 1]


def test_refusals(orc, og, fx):
    import torch
    import bulletproofs_b200 as bp
    pb, vb, plen = _tile(orc, og, 1, 300)
    d_p = torch.frombuffer(bytearray(bytes(pb)), dtype=torch.uint8).cuda(); d_v = torch.frombuffer(bytearray(bytes(vb)), dtype=torch.uint8).cuda()
    verd = torch.zeros(300, dtype=torch.int32, device="cuda")
    L = bp.lib()
    t = bp.Transcript(LABEL).to_bytes()

    def call(ctx, gens, count, nb):
        return L.bp_rangeproof_verify_group_device_exact(ctx._h, gens._h, t, d_p.data_ptr(), plen, d_v.data_ptr(), 64, 1, count, nb, None, verd.data_ptr(), None)

    assert call(fx.ctx, fx.gens, 100, 3) == 0
    assert call(fx.ctx, fx.gens, 50, 2) == bp.ERR_INVALID_ARGUMENT            # a geometry not reserved
    other = bp.Gens(fx.ctx, 64, 32)
    assert call(fx.ctx, other, 100, 3) == bp.ERR_INVALID_ARGUMENT             # another table
    other.close()
    assert L.bp_rangeproof_verify_group_begin(fx.ctx._h, fx.gens._h, t, bytes(pb[:plen]), plen, bytes(vb[:32]), 64, 1, 1, 1, None) == 0
    assert call(fx.ctx, fx.gens, 100, 3) == bp.ERR_INVALID_ARGUMENT           # a begin pending
    import ctypes
    v1 = ctypes.create_string_buffer(1)
    assert L.bp_rangeproof_verify_group_finish(fx.ctx._h, v1, None) == 0 and v1.raw == b"\x00"
    assert call(fx.ctx, fx.gens, 100, 3) == 0
    plain = bp.Context(0)
    pg = bp.Gens(plain, 64, 32)
    bp.BatchVerifier(plain, pg, bp.Transcript(LABEL), 64, 1, 100, 3)           # reserved with the plain call only
    assert call(plain, pg, 100, 3) == bp.ERR_INVALID_ARGUMENT
    assert "reserve_exact" in L.bp_last_error(plain._h).decode()
    pg.close(); plain.close()
    fx.ctx.synchronize()


def test_larger_geometry_runs_several_iterations(orc, og):
    """(64, 16): P = 2^18 // 2090 = 125 proofs per level-2 iteration, so 210 bad proofs take two"""
    f = Fixed(16, 70, 3)
    try:
        pb, vb, plen = _tile(orc, og, 16, 210)
        for bad in ([69], list(range(210))):
            b = bytearray(pb)
            for i in bad:
                _bad(b, plen, i)
            got, _, _ = _check(orc, og, f, b, vb, plen, bytes([9]) * 32)
            assert [i for i, v in enumerate(got) if v] == bad
    finally:
        f.close()


def test_two_iterations_at_the_bench_geometry(orc, og):
    """(64, 1), 2 x 1000 proofs, every one bad: P = 1783, two level-2 iterations"""
    f = Fixed(1, 1000, 2)
    try:
        pb, vb, plen = _tile(orc, og, 1, 2000)
        for i in range(0, 2000, 1):
            _bad(pb, plen, i)
        got, ok, _ = _check(orc, og, f, pb, vb, plen, bytes([4]) * 32)
        assert got == [1] * 2000 and ok == [0, 0]
    finally:
        f.close()


class Mix:
    def __init__(self):
        import bulletproofs_b200 as bp
        self.ctx = bp.Context(0)
        self.gens = bp.Gens(self.ctx, 64, 32)
        self.v = bp.MixedVerifier(self.ctx, self.gens, MIX, exact=True)

    def run(self, items, seed, records=None, exact=True):
        import bulletproofs_b200 as bp
        call = Call(items, records)
        l0 = self.ctx.launches
        args = (call.proofs, call.proof_bytes, call.poff, call.n, call.commitments, call.n_commitments, call.coff, call.count, call.verdicts.data_ptr(),
                call.flags.data_ptr())
        if records is not None and exact:
            self.v.run_device_exact_each(call.records, *args, seed=seed)
        elif exact:
            self.v.run_device_exact(bp.Transcript(LABEL), *args, seed=seed)
        else:
            self.v.run_device(bp.Transcript(LABEL), *args, seed=seed)
        dl = self.ctx.launches - l0
        self.ctx.synchronize()
        return (*call.result(), dl)

    def close(self):
        self.gens.close()
        self.ctx.close()


@pytest.fixture(scope="module")
def mx():
    x = Mix()
    yield x
    x.close()


def _mix_expect(bp, orc, og, ref_ctx, ref_gens, items, seed, records=None):
    if records:
        host = bp.verify_mixed_each(ref_ctx, ref_gens, [(bp.Transcript(state=t), p, V, n) for t, (p, V, n) in zip(records, items)], seed=seed)
    else:
        host = bp.verify_mixed(ref_ctx, ref_gens, bp.Transcript(LABEL), items, seed=seed)
    want = oracle(orc, og, items, records)
    assert host == want
    return want


@pytest.fixture(scope="module")
def ref(gpu_ctx):
    import bulletproofs_b200 as bp
    g = bp.Gens(gpu_ctx, 64, 32)
    yield gpu_ctx, g
    g.close()


def test_mix_damage_in_two_classes(orc, og, mx, ref):
    import bulletproofs_b200 as bp
    rnd = random.Random(11)
    items, bad = _damaged(orc, og, (1, 4), rnd)
    got, flags, dl = mx.run(items, bytes([1]) * 32)
    assert got == _mix_expect(bp, orc, og, *ref, items, bytes([1]) * 32)
    assert [i for i, v in enumerate(got) if v] == [i for i, b in enumerate(bad) if b]
    assert flags == [0, 1, 0, 1]
    pgot, pflags, pdl = mx.run(items, bytes([1]) * 32, exact=False)         # the plain graph on the same context: flagged classes coarse
    assert pflags == flags and pdl < dl
    assert all(pgot[i] == got[i] for i, it in enumerate(items) if flags[KEYS.index((64, len(it[1]) // 32))])
    clean = mx.run(tx(orc, og, FULL, rnd), bytes([2]) * 32)
    assert clean[0] == [0] * sum(FULL.values()) and clean[2] == dl


def test_mix_inert_unplaced_and_records(orc, og, mx, ref):
    """a partial fill (inert slots), proofs of a class outside the mix and over capacity (unplaced), damage in two classes, and per-proof
    records, one of them malformed"""
    import bulletproofs_b200 as bp
    rnd = random.Random(12)
    items = tx(orc, og, {1: 20, 2: 40, 8: 5})
    for j in (3, 17, 25, 55):                      # (64, 1) twice, (64, 2) twice
        p, V, n = items[j]
        pb = bytearray(p); _bad(pb, len(p), 0)
        items[j] = (bytes(pb), V, n)
    proofs, Vs, plen = _cell(orc, og, 32, 2)
    items += [(proofs[i * plen:(i + 1) * plen], Vs[64 * i:64 * (i + 1)], 32) for i in range(3)]
    rnd.shuffle(items)
    got, flags, _ = mx.run(items, bytes([3]) * 32)
    seen, unplaced = {}, []
    for i, (p, V, n) in enumerate(items):
        key = (n, len(V) // 32)
        seen[key] = seen.get(key, 0) + 1
        if key not in MIX or seen[key] > MIX[key]:
            unplaced.append(i)
    assert [i for i, v in enumerate(got) if v == bp.VERDICT_UNPLACED] == unplaced and len(unplaced) == 3 + 7
    want = _mix_expect(bp, orc, og, *ref, items, bytes([3]) * 32)
    assert [g for i, g in enumerate(got) if i not in unplaced] == [w for i, w in enumerate(want) if i not in unplaced]
    assert flags[0] == 0 and flags[2:] == [1, 1]
    records = [orc.transcript(LABEL)[:203]] * len(items)
    records[rnd.randrange(len(items))] = malformed_record(rnd, 1)
    got, flags, _ = mx.run(items, bytes([4]) * 32, records=records)
    want = _mix_expect(bp, orc, og, *ref, items, bytes([4]) * 32, records)
    assert [g for i, g in enumerate(got) if i not in unplaced] == [w for i, w in enumerate(want) if i not in unplaced]


def test_mix_refused_without_exact_reservation(orc, og):
    import bulletproofs_b200 as bp
    ctx = bp.Context(0)
    gens = bp.Gens(ctx, 64, 32)
    try:
        v = bp.MixedVerifier(ctx, gens, MIX)
        call = Call(tx(orc, og, {1: 3}))
        with pytest.raises(bp.BpError) as e:
            v.run_device_exact(bp.Transcript(LABEL), call.proofs, call.proof_bytes, call.poff, call.n, call.commitments, call.n_commitments, call.coff,
                               call.count, call.verdicts.data_ptr())
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
    finally:
        gens.close()
        ctx.close()
