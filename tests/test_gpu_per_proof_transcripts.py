"""GPU tier (-m gpu): range-proof verification where every proof starts from its own transcript (bp.verify_group_each,
bp.verify_group_device_each, bp.verify_mixed_each).  The proofs are made by the oracle's prover under distinct transcripts: different
labels, appended context that leaves the position below the 166-byte rate or wraps it (positions 0 to 165, 165 included), and a state
taken right after a challenge.  Records are interleaved so that the proofs of one warp start at different positions.  Every verdict is
checked against the oracle's RangeProof::verify_multiple with that proof's own transcript; a record no transcript can hold between
operations must give FormatError."""
import os
import random

import pytest

from oracle_binding import L_ORDER as l
from test_gpu_geometry import GRID
from test_gpu_group_check import _bad, _expected, _malformed
from test_gpu_parity import le

pytestmark = pytest.mark.gpu

REC = 203
CONTEXT_LENGTHS = (0, 3, 40, 97, 118, 119, 120, 140, 155, 250, 400)


def _contexts(orc):
    """oracle transcript states (their first 203 bytes are the wire state): one per label, with context of CONTEXT_LENGTHS appended, and
    one taken right after a challenge"""
    out = []
    for i, extra in enumerate(CONTEXT_LENGTHS):
        st = orc.transcript(b"tx %d" % i)
        if extra:
            st = orc.transcript_append(st, b"context", bytes([i]) * extra)
        out.append(st[:REC])
    st = orc.transcript_append(orc.transcript(b"session"), b"id", b"42")
    out.append(orc.transcript_challenge(st, b"nonce", 32)[0][:REC])
    return out


def _prove(orc, og, tstate, n, m, count, seed):
    rnd = random.Random(seed)
    values = [rnd.randrange(1 << n) for _ in range(count * m)]
    blind = b"".join(le(rnd.randrange(l)) for _ in range(count * m))
    seeds = b"".join(le(seed * 1000 + i, 8) + bytes(24) for i in range(count))
    return orc.prove_many(og, tstate, values, blind, n, m, seeds, nthreads=os.cpu_count() or 4)


class Pool:
    """`per` oracle proofs of (n, m) under each context: entry j = (record, proof, commitments)"""

    def __init__(self, orc, og, n, m, per, seed):
        self.n, self.m, self.entries = n, m, []
        for c, ts in enumerate(_contexts(orc)):
            proofs, Vs = _prove(orc, og, ts, n, m, per, seed + c)
            plen = len(proofs) // per
            self.entries += [(ts, proofs[i * plen:(i + 1) * plen], Vs[32 * m * i:32 * m * (i + 1)]) for i in range(per)]
        order = list(range(len(self.entries)))
        random.Random(seed).shuffle(order)                 # neighbours in a warp come from different contexts
        self.entries = [self.entries[i] for i in order]

    def tile(self, total):
        return [self.entries[i % len(self.entries)] for i in range(total)]


def malformed_record(rnd, kind):
    body = rnd.randbytes(200)
    if kind == 0:
        return body + bytes([rnd.randrange(166, 256), 0, 0])                         # pos at or beyond the rate
    pos = rnd.randrange(0, 165)
    return body + bytes([pos, rnd.randrange(pos + 1, 256), 0])                        # pos_begin above pos


_verdicts = {}


def _want(orc, og, n, m, items):
    """the oracle's verdict of every (record, proof, commitments); FormatError for a malformed record, which no transcript can hold (every
    case here has parameters the verifier admits)"""
    out = []
    for ts, p, V in items:
        key = (n, m, ts, p, V)
        if key not in _verdicts:
            _verdicts[key] = 2 if ts[200] >= 166 or ts[201] > ts[200] else orc.rangeproof_verify(og, ts, p, V, m, n)
        out.append(_verdicts[key])
    return out


def _flat(items):
    return b"".join(t for t, _, _ in items), b"".join(p for _, p, _ in items), b"".join(V for _, _, V in items)


def _dev(data: bytes, front: int = 0):
    import torch
    return torch.frombuffer(bytearray(bytes(front) + data + bytes(16)), dtype=torch.uint8).cuda()


def _device_each(bp, ctx, gens, n, m, count, nb, items, seed, front=1):
    """verify_group_device_each with the records at byte `front` of a torch CUDA tensor; (verdicts, batch flags)"""
    import torch
    recs, proofs, Vs = _flat(items)
    d_t, d_p, d_v = _dev(recs, front), _dev(proofs), _dev(Vs)
    d_verd = torch.full((count * nb,), 77, dtype=torch.int32, device="cuda"); h_ok = torch.full((nb,), 9, dtype=torch.int32).pin_memory()
    torch.cuda.synchronize()
    bp.verify_group_device_each(ctx, gens, d_t.data_ptr() + front, d_p.data_ptr(), d_v.data_ptr(), n, m, count, nb, d_verd.data_ptr(), h_ok.data_ptr(), seed)
    ctx.synchronize()
    return d_verd.cpu().tolist(), h_ok.tolist()


def _paths(bp, n, m, count, nb):
    """(name, context, gens): direct launches, and the geometry reserved (captured graph, arenas sized)"""
    for name in ("direct", "graph"):
        ctx = bp.Context(0)
        gens = bp.Gens(ctx, 64, 32)
        if name == "graph":
            ctx._check(bp.lib().bp_rangeproof_verify_reserve(ctx._h, gens._h, n, m, count, nb))
        yield name, ctx, gens
        gens.close(); ctx.close()


def _check_all(bp, orc, og, n, m, count, nb, items, failing, seed=bytes([3]) * 32):
    """all three entry points on both paths: per-proof verdicts of the host forms, per-batch flags everywhere, and the device form's
    verdicts (a batch whose combination fails marks its well-formed proofs VerificationError)"""
    want = _want(orc, og, n, m, items)
    ok_want, dev_want = _expected(want, count, nb, set(failing))
    recs, proofs, Vs = _flat(items)
    for name, ctx, gens in _paths(bp, n, m, count, nb):
        got, ok = bp.verify_group_each(ctx, gens, recs, proofs, Vs, n, m, count, nb, seed=seed)
        assert got == want, (name, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w][:20])
        assert ok == ok_want, (name, ok, ok_want)
        dgot, dok = _device_each(bp, ctx, gens, n, m, count, nb, items, seed)
        assert dgot == dev_want, (name, [(i, g, w) for i, (g, w) in enumerate(zip(dgot, dev_want)) if g != w][:20])
        assert dok == ok_want, (name, dok, ok_want)
    return want


@pytest.fixture(scope="module")
def og(orc):
    return orc.gens(64, 32)


@pytest.fixture(scope="module")
def pool64(orc, og):
    return Pool(orc, og, 64, 1, 4, 500)


@pytest.fixture(scope="module")
def gens(gpu_ctx):
    import bulletproofs_b200 as bp
    g = bp.Gens(gpu_ctx, 64, 32)
    yield g
    g.close()


def test_contexts_cover_the_positions(orc):
    """the records start below and just under the rate, after a wrap, and right after a challenge (pos_begin 0)"""
    pos = [ts[200] for ts in _contexts(orc)]
    assert len(set(_contexts(orc))) == len(CONTEXT_LENGTHS) + 1
    assert 165 in pos and min(pos) < 8 and any(0 < p < 64 for p in pos) and any(100 < p < 165 for p in pos)
    assert _contexts(orc)[-1][201] == 0


def test_every_kind_of_proof_and_record(orc, og, pool64):
    """valid proofs, a well-formed invalid proof, a non-canonical proof, a proof under another context's record, and malformed records
    of both kinds, over two batches; batch 0 fails its combination, batch 1 holds only rejections that are left out of it"""
    import bulletproofs_b200 as bp
    n, m, count, nb = 64, 1, 40, 2
    rnd = random.Random(11)
    items = pool64.tile(count * nb)
    pb = bytearray(items[5][1]); _bad(pb, len(pb), 0); items[5] = (items[5][0], bytes(pb), items[5][2])
    pb = bytearray(items[9][1]); _malformed(pb, len(pb), 0); items[9] = (items[9][0], bytes(pb), items[9][2])
    other = next(e[0] for e in pool64.entries if e[0] != items[33][0])
    items[33] = (other, items[33][1], items[33][2])                                     # another proof's transcript
    for i, kind in ((count + 2, 0), (count + 17, 1), (count + 31, 0)):
        items[i] = (malformed_record(rnd, kind), items[i][1], items[i][2])
    want = _check_all(bp, orc, og, n, m, count, nb, items, failing=[0])
    assert [(i, w) for i, w in enumerate(want) if w] == [(5, 1), (9, 2), (33, 1), (count + 2, 2), (count + 17, 2), (count + 31, 2)]


def test_each_verdict_is_the_single_proof_call(gpu_ctx, orc, og, pool64, gens):
    """verify_group_each of one batch == verify_batch of each proof alone with its record as the transcript"""
    import bulletproofs_b200 as bp
    n, m = 64, 1
    items = pool64.tile(len(pool64.entries))
    pb = bytearray(items[3][1]); _bad(pb, len(pb), 0); items[3] = (items[3][0], bytes(pb), items[3][2])
    items[7] = (next(e[0] for e in items if e[0] != items[7][0]), items[7][1], items[7][2])
    items[12] = (malformed_record(random.Random(12), 1), items[12][1], items[12][2])
    seed = bytes([4]) * 32
    recs, proofs, Vs = _flat(items)
    got, ok = bp.verify_group_each(gpu_ctx, gens, recs, proofs, Vs, n, m, len(items), seed=seed)
    alone = [bp.verify_batch(gpu_ctx, gens, bp.Transcript(state=t), p, V, n, m, 1, seed=seed)[0] for t, p, V in items if t[200] < 166 and t[201] <= t[200]]
    assert [g for g, (t, _, _) in zip(got, items) if t[200] < 166 and t[201] <= t[200]] == alone
    assert got == _want(orc, og, n, m, items) and ok == [0]
    assert got[12] == bp.PROOF_FORMAT_ERROR and got[3] == got[7] == bp.PROOF_VERIFICATION_ERROR


def test_swapped_records_and_one_proof_under_two_transcripts(orc, og, pool64):
    """swapping the records of two proofs fails exactly those two and only their batch; the same proof bytes under their own transcript
    and under another one get their own verdicts"""
    import bulletproofs_b200 as bp
    n, m, count, nb = 64, 1, 24, 4
    items = pool64.tile(count * nb)
    i, j = count + 3, count + 14
    assert items[i][0] != items[j][0]
    items[i], items[j] = (items[j][0], items[i][1], items[i][2]), (items[i][0], items[j][1], items[j][2])
    t, p, V = items[3 * count + 1]
    other = next(e[0] for e in pool64.entries if e[0] != t)
    items[3 * count + 5] = (other, p, V)
    want = _check_all(bp, orc, og, n, m, count, nb, items, failing=[1, 3])
    assert [k for k, w in enumerate(want) if w] == [i, j, 3 * count + 5] and want[3 * count + 1] == 0


def test_one_record_everywhere_equals_the_shared_call(gpu_ctx, orc, og, pool64, gens):
    """records all equal to the shared transcript: verdicts and batch flags of verify_group / verify_mixed on the same seed"""
    import bulletproofs_b200 as bp
    n, m, count, nb = 64, 1, 24, 3
    ts = pool64.entries[0][0]
    same = [e for e in pool64.entries if e[0] == ts]
    items = [same[k % len(same)] for k in range(count * nb)]
    pb = bytearray(items[count + 4][1]); _bad(pb, len(pb), 0); items[count + 4] = (ts, bytes(pb), items[count + 4][2])
    pb = bytearray(items[7][1]); _malformed(pb, len(pb), 0); items[7] = (ts, bytes(pb), items[7][2])
    recs, proofs, Vs = _flat(items)
    for seed in (bytes([5]) * 32, bytes(range(32))):
        shared = bp.verify_group(gpu_ctx, gens, bp.Transcript(state=ts), proofs, Vs, n, m, count, nb, seed=seed)
        assert bp.verify_group_each(gpu_ctx, gens, recs, proofs, Vs, n, m, count, nb, seed=seed) == shared
        assert shared[1] == [0, 0, 1]
        mixed = bp.verify_mixed(gpu_ctx, gens, bp.Transcript(state=ts), [(p, V, n) for _, p, V in items], seed=seed)
        assert bp.verify_mixed_each(gpu_ctx, gens, [(bp.Transcript(state=t), p, V, n) for t, p, V in items], seed=seed) == mixed == shared[0]


def test_group_of_8x1024_with_failing_batches(orc, og, pool64):
    """8 batches of 1024: a well-formed invalid proof in batch 2, swapped records in batch 5 (both levels of the reject path find them),
    malformed records in batch 6 (rejected, left out of the combination)"""
    import bulletproofs_b200 as bp
    n, m, count, nb = 64, 1, 1024, 8
    rnd = random.Random(13)
    items = pool64.tile(count * nb)
    k = 2 * count + 700
    pb = bytearray(items[k][1]); _bad(pb, len(pb), 0); items[k] = (items[k][0], bytes(pb), items[k][2])
    i, j = 5 * count + 31, 5 * count + 32                                                 # two chunks
    while items[i][0] == items[j][0]:
        j += 1
    items[i], items[j] = (items[j][0], items[i][1], items[i][2]), (items[i][0], items[j][1], items[j][2])
    for q in (6 * count, 6 * count + 511, 7 * count - 1):
        items[q] = (malformed_record(rnd, q % 2), items[q][1], items[q][2])
    want = _check_all(bp, orc, og, n, m, count, nb, items, failing=[2, 5])
    assert [q for q, w in enumerate(want) if w] == sorted([k, i, j, 6 * count, 6 * count + 511, 7 * count - 1])


def test_device_records_at_an_odd_offset_back_to_back(orc, og, pool64):
    """records at an odd address of a torch CUDA tensor, on a reserved geometry (graph replay) and an unreserved one; two device calls
    queued back to back on one context with different records keep their own verdicts; shared-transcript calls in between still replay
    the graph with the block's own state"""
    import torch
    import bulletproofs_b200 as bp
    n, m, count, nb = 64, 1, 32, 2
    items = pool64.tile(count * nb)
    swapped = list(items)
    swapped[3], swapped[40] = (items[40][0], items[3][1], items[3][2]), (items[3][0], items[40][1], items[40][2])
    assert items[3][0] != items[40][0]
    seed = bytes([6]) * 32
    for name, ctx, gens in _paths(bp, n, m, count, nb):
        tensors = []
        for its in (items, swapped, items):
            recs, proofs, Vs = _flat(its)
            tensors.append((_dev(recs, 3), _dev(proofs), _dev(Vs)))
        d_verd = torch.full((3, count * nb), 77, dtype=torch.int32, device="cuda"); h_ok = torch.full((3, nb), 9, dtype=torch.int32).pin_memory()
        torch.cuda.synchronize()
        for r, (d_t, d_p, d_v) in enumerate(tensors):
            bp.verify_group_device_each(ctx, gens, d_t.data_ptr() + 3, d_p.data_ptr(), d_v.data_ptr(), n, m, count, nb, d_verd[r].data_ptr(), h_ok[r].data_ptr(), seed)
        ctx.synchronize()
        got = d_verd.cpu().tolist()
        assert got[0] == got[2] == [0] * (count * nb), name
        assert got[1] == [1] * (count * nb), name                          # both batches fail: every well-formed proof is marked
        assert h_ok.tolist() == [[1, 1], [0, 0], [1, 1]], name
        assert _device_each(bp, ctx, gens, n, m, count, nb, swapped, seed, front=1) == ([1] * (count * nb), [0, 0]), name
        ts = items[0][0]
        same = [e for e in pool64.entries if e[0] == ts]
        shared_items = [same[q % len(same)] for q in range(count * nb)]
        _, proofs, Vs = _flat(shared_items)
        assert bp.verify_group(ctx, gens, bp.Transcript(state=ts), proofs, Vs, n, m, count, nb, seed=seed) == ([0] * (count * nb), [1, 1]), name
        assert bp.verify_group_each(ctx, gens, _flat(items)[0], _flat(items)[1], _flat(items)[2], n, m, count, nb, seed=seed) == ([0] * (count * nb), [1, 1]), name


def test_mixed_over_the_grid(gpu_ctx, orc, og, gens):
    """every (n, m) of the reference grid with per-proof transcripts in one shuffled call, with damage in three classes"""
    import bulletproofs_b200 as bp
    rnd = random.Random(14)
    ctxs = _contexts(orc)
    entries = []                                                             # (n, m, record, proof, commitments)
    for c, (n, m) in enumerate(GRID):
        for t in (ctxs[c % len(ctxs)], ctxs[(c * 5 + 3) % len(ctxs)]):
            proofs, Vs = _prove(orc, og, t, n, m, 1, 700 + c)
            entries.append((n, m, t, proofs, Vs))
    items = [entries[i % len(entries)] for i in range(3 * len(entries))]
    bad = {}
    for q in (4, 20, 61):
        n, m, t, p, V = items[q]
        pb = bytearray(p); _bad(pb, len(pb), 0); items[q] = (n, m, t, bytes(pb), V); bad[q] = 1
    n, m, t, p, V = items[30]
    items[30] = (n, m, malformed_record(rnd, 0), p, V); bad[30] = 2
    n, m, t, p, V = items[45]
    items[45] = (n, m, next(x for x in ctxs if x != t), p, V); bad[45] = 1
    perm = list(range(len(items)))
    rnd.shuffle(perm)
    items = [items[i] for i in perm]
    want = [_want(orc, og, n, m, [(t, p, V)])[0] for n, m, t, p, V in items]
    assert [(k, w) for k, w in enumerate(want) if w] == sorted((perm.index(q), c) for q, c in bad.items())
    got = bp.verify_mixed_each(gpu_ctx, gens, [(bp.Transcript(state=t), p, V, n) for n, m, t, p, V in items], seed=bytes([7]) * 32)
    assert got == want, [(k, g, w) for k, (g, w) in enumerate(zip(got, want)) if g != w]
