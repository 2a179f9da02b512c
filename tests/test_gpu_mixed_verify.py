"""GPU tier (-m gpu): bp.verify_mixed, range proofs of any (n, m) in one call.  Every verdict list is checked per proof against the oracle
(RangeProof::verify_multiple of that proof alone) and against bp.verify_batch of that proof alone (count = 1, same transcript).  The
cases: the whole 64 x 32 grid in one shuffled call; damage in three classes of 33 proofs (a full chunk and a ragged one, so both levels of
the reject path run) beside undamaged classes; per-proof parameter codes next to valid proofs; a one-class call against verify_batch; a
permutation of the items; a cancelling pair in one class; and a context shared with a reserved BatchVerifier."""
import random

import pytest

from oracle_binding import L_ORDER as l
from test_batch_soundness import cancelling_set
from test_gpu_geometry import COUNT, GRID, LABEL, _cell, _damage
from test_gpu_group_check import _malformed

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def og(orc):
    return orc.gens(64, 32)


@pytest.fixture(scope="module")
def gens(gpu_ctx):
    import bulletproofs_b200 as bp
    g = bp.Gens(gpu_ctx, 64, 32)
    yield g
    g.close()


def _items(orc, og, n, m, count=COUNT):
    """the cell's proofs as verify_mixed items (proof, commitments, n)"""
    proofs, Vs, plen = _cell(orc, og, n, m)
    return [(proofs[i * plen:(i + 1) * plen], Vs[32 * m * i:32 * m * (i + 1)], n) for i in range(count)]


def _check(bp, orc, ctx, gens, ogens, items, seed, want=None):
    """verify_mixed's verdicts == the oracle's and verify_batch's, proof by proof (each distinct item verified once)"""
    got = bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), items, seed=seed)
    ot, alone = orc.transcript(LABEL), {}
    for p, V, n in items:
        if (p, V, n) not in alone:
            m = len(V) // 32
            ref = orc.rangeproof_verify(ogens, ot, p, V, m, n)
            dev = bp.verify_batch(ctx, gens, bp.Transcript(LABEL), p, V, n, m, 1, proof_len=len(p), seed=seed)[0]
            assert ref == dev, (n, m, len(p), ref, dev)
            alone[(p, V, n)] = ref
    ref = [alone[it] for it in items]
    assert got == ref, [(i, g, w) for i, (g, w) in enumerate(zip(got, ref)) if g != w]
    if want is not None:
        assert got == want
    return got


def test_whole_grid_in_one_call(gpu_ctx, orc, og, gens):
    import bulletproofs_b200 as bp
    items = [it for n, m in GRID for it in _items(orc, og, n, m, 5)]
    random.Random(1).shuffle(items)
    _check(bp, orc, gpu_ctx, gens, og, items, bytes([1]) * 32, want=[0] * len(items))


def _damaged_mix(orc, og):
    """(items, indices of the damaged ones): the six damage kinds of test_gpu_geometry in three classes of COUNT proofs each, beside two
    undamaged classes, shuffled"""
    items, bad = [], []
    for n, m, damage in ((64, 1, True), (16, 4, True), (64, 2, False), (8, 32, True), (32, 8, False)):
        proofs, Vs, plen = _cell(orc, og, n, m)
        pb, vb = bytearray(proofs), bytearray(Vs)
        at = _damage(pb, vb, plen, n, m) if damage else []
        for i in range(COUNT):
            items.append((bytes(pb[i * plen:(i + 1) * plen]), bytes(vb[32 * m * i:32 * m * (i + 1)]), n))
            bad.append(i in at)
    perm = list(range(len(items)))
    random.Random(2).shuffle(perm)
    return [items[i] for i in perm], [bad[i] for i in perm]


def test_damage_in_several_classes(gpu_ctx, orc, og, gens):
    import bulletproofs_b200 as bp
    items, bad = _damaged_mix(orc, og)
    got = _check(bp, orc, gpu_ctx, gens, og, items, bytes([2]) * 32)
    assert [v != 0 for v in got] == bad


def test_permuting_the_items_permutes_the_verdicts(gpu_ctx, orc, og, gens):
    import bulletproofs_b200 as bp
    items, _ = _damaged_mix(orc, og)
    got = bp.verify_mixed(gpu_ctx, gens, bp.Transcript(LABEL), items, seed=bytes([3]) * 32)
    perm = list(range(len(items)))
    random.Random(3).shuffle(perm)
    assert bp.verify_mixed(gpu_ctx, gens, bp.Transcript(LABEL), [items[i] for i in perm], seed=bytes([4]) * 32) == [got[i] for i in perm]


def test_per_proof_parameter_codes(gpu_ctx, orc):
    """parameter-rejected proofs next to valid ones, on a 64 x 16 table: n = 12, m above the table's parties, a length that does not
    match n*m, a length that is no proof length, m = 3, and a non-canonical t_x in a proof with m = 3"""
    import bulletproofs_b200 as bp
    og = orc.gens(64, 32)
    g16, og16 = bp.Gens(gpu_ctx, 64, 16), orc.gens(64, 16)
    try:
        valid = _items(orc, og, 64, 1, 4) + _items(orc, og, 8, 4, 4)
        p81, V81, _ = _items(orc, og, 8, 1, 1)[0]
        p832, V832, _ = _items(orc, og, 8, 32, 1)[0]
        p84, V84, _ = _items(orc, og, 8, 4, 1)[0]
        p6432, V6432, _ = _items(orc, og, 64, 32, 1)[0]
        bad_tx = bytearray(p84)
        _malformed(bad_tx, len(p84), 0)
        rejected = [
            ((p81, V81, 12), bp.PROOF_INVALID_BITSIZE),
            ((p6432, V6432, 64), bp.PROOF_INVALID_GENERATORS_LENGTH),
            ((p832, V832[:32 * 16], 8), bp.PROOF_VERIFICATION_ERROR),
            ((p81[:-32], V81, 8), bp.PROOF_FORMAT_ERROR),
            ((p84, V84[:96], 8), bp.PROOF_VERIFICATION_ERROR),
            ((bytes(bad_tx), V84[:96], 8), bp.PROOF_FORMAT_ERROR),
        ]
        items = []
        for i, (it, _) in enumerate(rejected):
            items += [valid[i], it]
        items += valid[len(rejected):]
        got = _check(bp, orc, gpu_ctx, g16, og16, items, bytes([5]) * 32)
        assert got[1:2 * len(rejected):2] == [c for _, c in rejected] and got[0:2 * len(rejected):2] == [0] * len(rejected)
        # every proof rejected: no kernel runs, the codes come back all the same
        only = [it for it, _ in rejected]
        assert bp.verify_mixed(gpu_ctx, g16, bp.Transcript(LABEL), only) == [c for _, c in rejected]
    finally:
        g16.close()


def test_one_class_matches_verify_batch(gpu_ctx, orc, og, gens):
    import bulletproofs_b200 as bp
    proofs, Vs, plen = _cell(orc, og, 32, 2)
    pb, vb = bytearray(proofs), bytearray(Vs)
    _damage(pb, vb, plen, 32, 2)
    items = [(bytes(pb[i * plen:(i + 1) * plen]), bytes(vb[64 * i:64 * (i + 1)]), 32) for i in range(COUNT)]
    seed = bytes([6]) * 32
    want = bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), bytes(pb), bytes(vb), 32, 2, COUNT, seed=seed)
    assert bp.verify_mixed(gpu_ctx, gens, bp.Transcript(LABEL), items, seed=seed) == want
    assert want == orc.verify_many(og, orc.transcript(LABEL), bytes(pb), plen, bytes(vb), 32, 2, COUNT)


def test_cancelling_pair_in_one_class(gpu_ctx, orc, og, gens):
    """P with a + d and P with a - d: their errors cancel under weights that ignore a; both must be rejected, the other classes accepted"""
    import bulletproofs_b200 as bp
    n, m = 64, 1
    k = (n * m).bit_length() - 1
    P, V, _ = _items(orc, og, n, m, 1)[0]
    members, _ = cancelling_set(P, 224 + 64 * k, "a+-d", random.Random(7).randrange(1, l))
    items = _items(orc, og, n, m, 10) + _items(orc, og, 16, 2, 10) + _items(orc, og, 8, 8, 10)
    items[3] = (members[0], V, n)
    items[7] = (members[1], V, n)
    got = _check(bp, orc, gpu_ctx, gens, og, items, bytes([8]) * 32)
    assert [i for i, v in enumerate(got) if v] == [3, 7] and got[3] == got[7] == bp.PROOF_VERIFICATION_ERROR


def test_shared_context_with_a_reserved_verifier(orc, og):
    """reserved call -> mixed call -> reserved call on one context: the mixed call leaves the verifier graph's scratch alone.  A mixed
    call while a launch group is pending is refused."""
    import bulletproofs_b200 as bp
    N, M, count, nb = 64, 1, 16, 2
    ctx = bp.Context(0)
    gens = bp.Gens(ctx, 64, 32)
    try:
        proofs, Vs, plen = _cell(orc, og, N, M)
        pb, vb = bytearray(proofs[:plen * 16] * 2), bytearray(Vs[:32 * 16] * 2)
        pb[(count + 5) * plen + 128] ^= 1                                 # batch 1 fails
        want = orc.verify_many(orc.gens(N, M), orc.transcript(LABEL), bytes(pb), plen, bytes(vb), N, M, count * nb)
        assert [i for i, w in enumerate(want) if w] == [count + 5]
        bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), N, M, count, nb)       # reserve: arenas sized, graph captured
        seed = bytes([9]) * 32
        assert bp.verify_group(ctx, gens, bp.Transcript(LABEL), bytes(pb), bytes(vb), N, M, count, nb, seed=seed) == (want, [1, 0])
        items, bad = _damaged_mix(orc, og)
        got = _check(bp, orc, ctx, gens, og, items, seed)
        assert [v != 0 for v in got] == bad
        assert bp.verify_group(ctx, gens, bp.Transcript(LABEL), bytes(pb), bytes(vb), N, M, count, nb, seed=seed) == (want, [1, 0])
        v = bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), N, M, count, nb, reserve=False)
        v.begin(bytes(pb), bytes(vb), seed)
        with pytest.raises(bp.BpError) as e:
            bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), items[:4])
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
        assert list(v.finish()) == want and v.batch_ok == [1, 0]
        with pytest.raises(bp.BpError) as e:
            bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), [])
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
    finally:
        gens.close()
        ctx.close()
