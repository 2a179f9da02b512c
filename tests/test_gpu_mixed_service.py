"""GPU tier (-m gpu): bp.MixedVerifier, mixed-geometry verification on a reserved mix (captured graph, begin / finish).  Every verdict list
is checked against bp.verify_mixed (or verify_mixed_each) on a context without a reserved mix, i.e. the direct launches, and against the
oracle's verdict of each proof alone.  The mix is that of a block of confidential transactions, (64, m) for m in 1, 2, 4, 8.  A clean call
that fits advances ctx.launches by one gather launch plus the graph's launches whatever the fill, which shows that the graph ran and that
no reject path did."""
import random

import pytest

from oracle_binding import L_ORDER as l
from test_batch_soundness import cancelling_set
from test_gpu_geometry import LABEL, _cell, _damage
from test_gpu_group_check import _malformed
from test_gpu_per_proof_transcripts import _contexts, _prove, malformed_record

pytestmark = pytest.mark.gpu

MIX = {(64, 1): 66, (64, 2): 33, (64, 4): 33, (64, 8): 33}
FULL = {m: c for (_, m), c in MIX.items()}


@pytest.fixture(scope="module")
def og(orc):
    return orc.gens(64, 32)


@pytest.fixture(scope="module")
def gens(gpu_ctx):
    import bulletproofs_b200 as bp
    g = bp.Gens(gpu_ctx, 64, 32)
    yield g
    g.close()


class Service:
    """a context of its own with the mix reserved; clean = the launch delta of a clean fitting call"""

    def __init__(self, mix=MIX):
        import bulletproofs_b200 as bp
        self.ctx = bp.Context(0)
        self.gens = bp.Gens(self.ctx, 64, 32)
        self.v = bp.MixedVerifier(self.ctx, self.gens, mix)
        self.clean = None

    def run(self, items, seed, each=False):
        """(verdicts, launch delta) of one begin / finish"""
        import bulletproofs_b200 as bp
        l0 = self.ctx.launches
        if each:
            self.v.begin_each(items, seed=seed)
        else:
            self.v.begin(bp.Transcript(LABEL), items, seed=seed)
        return self.v.finish(), self.ctx.launches - l0

    def close(self):
        self.gens.close()
        self.ctx.close()


@pytest.fixture(scope="module")
def svc(orc, og):
    s = Service()
    _, s.clean = s.run(tx(orc, og, FULL), bytes([1]) * 32)
    yield s
    s.close()


def tx(orc, og, counts, rnd=None):
    """items of (64, m) proofs, counts[m] of each, tiled from the oracle cells; shuffled when rnd is given"""
    items = []
    for m, c in counts.items():
        proofs, Vs, plen = _cell(orc, og, 64, m)
        per = len(proofs) // plen
        items += [(proofs[(i % per) * plen:(i % per + 1) * plen], Vs[32 * m * (i % per):32 * m * (i % per + 1)], 64) for i in range(c)]
    if rnd is not None:
        rnd.shuffle(items)
    return items


_alone = {}


def oracle(orc, og, items, records=None):
    """the oracle's verdict of each proof alone: verify_many over one proof of the proof's own geometry, the parameter code for a proof
    whose parameters are rejected, FormatError for a record no transcript can hold"""
    out = []
    for j, (p, V, n) in enumerate(items):
        ts = records[j] if records else orc.transcript(LABEL)[:203]
        key = (p, V, n, ts)
        if key not in _alone:
            m = len(V) // 32
            k = (n * m).bit_length() - 1
            if records and (ts[200] >= 166 or ts[201] > ts[200]):
                _alone[key] = 2
            elif n in (8, 16, 32, 64) and m in (1, 2, 4, 8, 16, 32) and len(p) == 32 * (9 + 2 * k):
                _alone[key] = orc.verify_many(og, ts if records else orc.transcript(LABEL), p, len(p), V, n, m, 1)[0]
            else:
                _alone[key] = orc.rangeproof_verify(og, ts if records else orc.transcript(LABEL), p, V, m, n)
        out.append(_alone[key])
    return out


def check(bp, orc, og, ref_ctx, ref_gens, s, items, seed, want_launches=None, records=None):
    """the service's verdicts == verify_mixed(_each) on the unreserved context == the oracle's; returns (verdicts, launch delta)"""
    if records:
        each = [(bp.Transcript(state=t), p, V, n) for t, (p, V, n) in zip(records, items)]
        got, dl = s.run(each, seed, each=True)
        direct = bp.verify_mixed_each(ref_ctx, ref_gens, each, seed=seed)
    else:
        got, dl = s.run(items, seed)
        direct = bp.verify_mixed(ref_ctx, ref_gens, bp.Transcript(LABEL), items, seed=seed)
    want = oracle(orc, og, items, records)
    assert got == direct == want, [(i, g, d, w) for i, (g, d, w) in enumerate(zip(got, direct, want)) if not g == d == w]
    if want_launches is not None:
        assert dl == want_launches
    return got, dl


def test_fill_levels_replay_the_graph(gpu_ctx, orc, og, gens, svc):
    """full, partial, one class empty, a single proof: every clean fitting call costs the same launches; a call that does not fit costs
    others"""
    import bulletproofs_b200 as bp
    rnd = random.Random(1)
    for counts in (FULL, {1: 40, 2: 7, 4: 33, 8: 1}, {1: 66, 2: 0, 4: 5, 8: 33}, {4: 1}, {1: 1}):
        got, _ = check(bp, orc, og, gpu_ctx, gens, svc, tx(orc, og, counts, rnd), bytes([2]) * 32, want_launches=svc.clean)
        assert got == [0] * sum(counts.values())
    _, dl = check(bp, orc, og, gpu_ctx, gens, svc, tx(orc, og, {1: 67}, rnd), bytes([2]) * 32)
    assert dl != svc.clean


def _damaged(orc, og, ms, rnd):
    """a full mix with the six damage kinds of test_gpu_geometry in the classes ms: (items, bad flags)"""
    items, bad = [], []
    for m, c in FULL.items():
        proofs, Vs, plen = _cell(orc, og, 64, m)
        pb, vb = bytearray(proofs), bytearray(Vs)
        at = _damage(pb, vb, plen, 64, m) if m in ms else []
        for i in range(c):
            q = i % 33
            items.append((bytes(pb[q * plen:(q + 1) * plen]), bytes(vb[32 * m * q:32 * m * (q + 1)]), 64))
            bad.append(q in at)
    perm = list(range(len(items)))
    rnd.shuffle(perm)
    return [items[i] for i in perm], [bad[i] for i in perm]


def test_damage_in_one_and_in_several_classes(gpu_ctx, orc, og, gens, svc):
    import bulletproofs_b200 as bp
    rnd = random.Random(2)
    for ms in ((4,), (1, 2, 8)):
        items, bad = _damaged(orc, og, ms, rnd)
        got, dl = check(bp, orc, og, gpu_ctx, gens, svc, items, bytes([3]) * 32)
        assert [v != 0 for v in got] == bad and dl > svc.clean
    check(bp, orc, og, gpu_ctx, gens, svc, tx(orc, og, FULL, rnd), bytes([3]) * 32, want_launches=svc.clean)


def test_cancelling_pair_in_one_class(gpu_ctx, orc, og, gens, svc):
    """P with a + d and P with a - d in the (64, 1) class: both rejected, everything else accepted"""
    import bulletproofs_b200 as bp
    k = 6
    items = tx(orc, og, {1: 20, 2: 10, 8: 5})
    P, V, _ = items[0]
    members, _ = cancelling_set(P, 224 + 64 * k, "a+-d", random.Random(7).randrange(1, l))
    items[3] = (members[0], V, 64)
    items[7] = (members[1], V, 64)
    got, _ = check(bp, orc, og, gpu_ctx, gens, svc, items, bytes([4]) * 32)
    assert [i for i, v in enumerate(got) if v] == [3, 7] and got[3] == got[7] == bp.PROOF_VERIFICATION_ERROR


def test_stale_slots_have_no_effect(gpu_ctx, orc, og, gens, svc):
    """call 1 fills (64, 2) to capacity with an invalid proof in its last slot; call 2 gives that class fewer proofs, all valid: every
    one is accepted, at the launches of a clean call (no reject path ran)"""
    import bulletproofs_b200 as bp
    items = tx(orc, og, {1: 10, 2: 33, 4: 2})
    p, V, n = items[10 + 32]
    pb = bytearray(p)
    pb[128] ^= 1                                                   # t_x changed: well-formed, invalid
    items[10 + 32] = (bytes(pb), V, n)
    got, _ = check(bp, orc, og, gpu_ctx, gens, svc, items, bytes([5]) * 32)
    assert [i for i, v in enumerate(got) if v] == [42]
    got, _ = check(bp, orc, og, gpu_ctx, gens, svc, tx(orc, og, {1: 10, 2: 20, 4: 2}), bytes([5]) * 32, want_launches=svc.clean)
    assert got == [0] * 32


def test_calls_that_do_not_fit(gpu_ctx, orc, og, gens, svc):
    """an unreserved class, one proof over a capacity and another generator table take the direct launches and give the same verdicts; a
    fitting call after them still replays the graph"""
    import bulletproofs_b200 as bp
    rnd = random.Random(6)
    proofs, Vs, plen = _cell(orc, og, 32, 2)
    other = [(proofs[i * plen:(i + 1) * plen], Vs[64 * i:64 * (i + 1)], 32) for i in range(5)]
    for items in (tx(orc, og, {1: 3, 2: 3}) + other, tx(orc, og, {1: 5, 2: 34}), tx(orc, og, {8: 34})):
        rnd.shuffle(items)
        _, dl = check(bp, orc, og, gpu_ctx, gens, svc, items, bytes([6]) * 32)
        assert dl != svc.clean
    g2 = bp.Gens(svc.ctx, 64, 32)
    try:
        items = tx(orc, og, {1: 4, 4: 4}, rnd)
        l0 = svc.ctx.launches
        got = bp.verify_mixed(svc.ctx, g2, bp.Transcript(LABEL), items, seed=bytes([6]) * 32)
        assert svc.ctx.launches - l0 != svc.clean and got == oracle(orc, og, items)
    finally:
        g2.close()
    check(bp, orc, og, gpu_ctx, gens, svc, tx(orc, og, {1: 30, 2: 30}, rnd), bytes([6]) * 32, want_launches=svc.clean)


def test_per_proof_transcripts(gpu_ctx, orc, og, gens, svc):
    """distinct records per proof, and malformed records, which give FormatError"""
    import bulletproofs_b200 as bp
    rnd = random.Random(8)
    ctxs = _contexts(orc)
    records, items = [], []
    for c, m in enumerate((1, 1, 2, 4, 8, 1, 2)):
        t = ctxs[c % len(ctxs)]
        proofs, Vs = _prove(orc, og, t, 64, m, 2, 800 + c)
        plen = len(proofs) // 2
        for i in range(2):
            records.append(t)
            items.append((proofs[i * plen:(i + 1) * plen], Vs[32 * m * i:32 * m * (i + 1)], 64))
    records[3] = malformed_record(rnd, 0)
    records[8] = malformed_record(rnd, 1)
    records[5] = next(x for x in ctxs if x != records[5])                    # the wrong transcript: VerificationError
    perm = list(range(len(items)))
    rnd.shuffle(perm)
    items, records = [items[i] for i in perm], [records[i] for i in perm]
    got, _ = check(bp, orc, og, gpu_ctx, gens, svc, items, bytes([7]) * 32, records=records)
    assert sorted(v for v in got if v) == [1, 2, 2]


def test_per_proof_parameter_codes(gpu_ctx, orc, og, gens, svc):
    """parameter-rejected proofs between valid ones of the mix: the call still fits, and each keeps its code"""
    import bulletproofs_b200 as bp
    valid = tx(orc, og, {1: 4, 4: 4})
    p81, V81, _ = tx(orc, og, {1: 1})[0]
    p84, V84, _ = tx(orc, og, {4: 1})[0]
    bad_tx = bytearray(p84)
    _malformed(bad_tx, len(p84), 0)
    rejected = [((p81, V81, 12), bp.PROOF_INVALID_BITSIZE), ((p81[:-32], V81, 64), bp.PROOF_FORMAT_ERROR),
                ((p84, V84[:96], 64), bp.PROOF_VERIFICATION_ERROR), ((bytes(bad_tx), V84[:96], 64), bp.PROOF_FORMAT_ERROR)]
    items = []
    for i, (it, _) in enumerate(rejected):
        items += [valid[i], it]
    items += valid[len(rejected):]
    got, _ = check(bp, orc, og, gpu_ctx, gens, svc, items, bytes([8]) * 32, want_launches=svc.clean)
    assert got[1::2][:len(rejected)] == [c for _, c in rejected]
    only = [it for it, _ in rejected]
    got, dl = check(bp, orc, og, gpu_ctx, gens, svc, only, bytes([8]) * 32)
    assert dl == 0                                                           # every proof rejected: no kernel runs


def test_pending_rules(orc, og, svc):
    """between a mixed begin and its finish the context refuses everything else, group finish included; a group begin blocks the mixed
    calls and the mixed finish; a failed begin leaves nothing pending"""
    import bulletproofs_b200 as bp
    ctx, gens, v = svc.ctx, svc.gens, svc.v
    items = tx(orc, og, {1: 3, 2: 2})
    v.begin(bp.Transcript(LABEL), items, seed=bytes([9]) * 32)
    for call in (lambda: bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), items),
                 lambda: bp.verify_batch(ctx, gens, bp.Transcript(LABEL), items[0][0], items[0][1], 64, 1, 1),
                 lambda: bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), 64, 1, 4, 1),
                 lambda: bp.MixedVerifier(ctx, gens, MIX),
                 lambda: ctx._check(bp.lib().bp_rangeproof_verify_group_finish(ctx._h, bytes(8), None))):
        with pytest.raises(bp.BpError) as e:
            call()
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
    assert v.finish() == [0] * 5
    with pytest.raises(bp.BpError):
        v.finish()
    proofs, Vs, plen = _cell(orc, og, 64, 1)
    b = bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), 64, 1, 4, 1, reserve=False)
    b.begin(proofs[:4 * plen], Vs[:4 * 32])
    for call in (lambda: v.begin(bp.Transcript(LABEL), items), lambda: ctx._check(bp.lib().bp_rangeproof_verify_mixed_finish(ctx._h, bytes(8)))):
        with pytest.raises(bp.BpError) as e:
            call()
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
    assert list(b.finish()) == [0] * 4
    with pytest.raises(bp.BpError) as e:                                     # a failed begin: offsets that do not start at 0
        ctx._check(bp.lib().bp_rangeproof_verify_mixed_begin(ctx._h, gens._h, bp.Transcript(LABEL).to_bytes(), 1, items[0][0],
                                                             (bp._c.c_uint64 * 2)(32, 32 + len(items[0][0])), (bp._c.c_uint32 * 1)(64), items[0][1],
                                                             (bp._c.c_uint64 * 2)(0, 1), None))
    assert e.value.code == bp.ERR_INVALID_ARGUMENT
    assert bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), items) == [0] * 5          # nothing was left pending


def test_reserved_batch_verifier_and_mix_on_one_context(orc, og):
    """alternating calls of a reserved BatchVerifier and a reserved MixedVerifier: each keeps its verdicts and its launch delta"""
    import bulletproofs_b200 as bp
    s = Service()
    try:
        N, M, count, nb = 64, 1, 16, 2
        proofs, Vs, plen = _cell(orc, og, N, M)
        pb, vb = bytearray(proofs[:plen * 16] * 2), bytearray(Vs[:32 * 16] * 2)
        bv = bp.BatchVerifier(s.ctx, s.gens, bp.Transcript(LABEL), N, M, count, nb)
        items = tx(orc, og, {1: 20, 2: 10, 4: 3, 8: 2}, random.Random(10))
        want = oracle(orc, og, items)
        deltas = set()
        bdeltas = set()
        for _ in range(3):
            l0 = s.ctx.launches
            bv.begin(bytes(pb), bytes(vb), bytes([11]) * 32)
            assert list(bv.finish()) == [0] * (count * nb) and bv.batch_ok == [1, 1]
            bdeltas.add(s.ctx.launches - l0)
            got, dl = s.run(items, bytes([11]) * 32)
            assert got == want
            deltas.add(dl)
        assert len(deltas) == 1 and len(bdeltas) == 1
    finally:
        s.close()


def test_two_contexts_in_flight(gpu_ctx, orc, og, gens):
    """begin on two contexts before either finish"""
    import bulletproofs_b200 as bp
    a, b = Service(), Service({(64, 8): 33, (64, 1): 66})
    try:
        ia = tx(orc, og, {1: 30, 2: 12, 4: 5, 8: 3}, random.Random(12))
        ib, bad = _damaged(orc, og, (8,), random.Random(13))
        ib = [it for it in ib if len(it[1]) in (32, 256)]
        a.v.begin(bp.Transcript(LABEL), ia, seed=bytes([12]) * 32)
        b.v.begin(bp.Transcript(LABEL), ib, seed=bytes([12]) * 32)
        gb, ga = b.v.finish(), a.v.finish()
        assert ga == oracle(orc, og, ia) == bp.verify_mixed(gpu_ctx, gens, bp.Transcript(LABEL), ia, seed=bytes([12]) * 32)
        assert gb == oracle(orc, og, ib) == bp.verify_mixed(gpu_ctx, gens, bp.Transcript(LABEL), ib, seed=bytes([12]) * 32)
    finally:
        a.close()
        b.close()
