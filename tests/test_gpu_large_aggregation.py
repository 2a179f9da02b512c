"""GPU tier (-m gpu): range proofs past the reference grid, up to n m = 2^20 generator pairs (BP_MAX_LG_N), against the oracle.  One cell per
k = 12..20, with m up to 131072 commitments per proof: every k_rp_head_seq<k> instance above the grid, the transcript program with
thousands of V steps, k_rp_scalars_sum and k_rp_static_sum over S up to 2^21 + 2 terms, and k_rp_decompress with more commitments per proof
than one block decodes.  Then the reject path at k = 17 (both chunk levels and the whole-batch re-check), the launch group and device entry
point, a mixed call with two large classes, the prover's bytes, and a caller transcript that is not fresh.

Every verdict is the oracle's (verify_many, or rangeproof_verify of one proof), never the GPU's own.  Up to k = 17 the proofs come from the
oracle's prover; above it that prover is too slow for the suite, so they come from the GPU prover, and the cell tests are where both
verifiers must accept them and reject one-bit changes."""
import os
import random

import pytest

from oracle_binding import L_ORDER as l, P_FIELD as p
from test_gpu_geometry import _cell as _grid_cell
from test_gpu_group_check import LABEL, _check_case
from test_gpu_mixed_verify import _check as _check_mixed

pytestmark = pytest.mark.gpu

CELLS = [(64, 64), (8, 512), (8, 1024), (8, 2048), (16, 1024), (16, 2048), (32, 2048), (64, 1024), (64, 2048),   # k = 12 .. 17
         (64, 4096), (64, 8192), (64, 16384), (8, 131072)]                                                    # k = 18 .. 20
ORACLE_MAX_K = 17               # proofs above it come from the GPU prover
DISTINCT = {(64, 64): 2, (64, 2048): 4}         # valid proofs made per cell (default 1)
THREADS = os.cpu_count() or 4


def le(x, n=32):
    return x.to_bytes(n, "little")


def _k(n, m):
    return (n * m).bit_length() - 1


@pytest.fixture(scope="module")
def t64(gpu_ctx, orc):
    """one table for every cell with m <= 16384: its party and generator strides differ from the cell's (n, m) everywhere but (64, 16384)"""
    import bulletproofs_b200 as bp
    g = bp.Gens(gpu_ctx, 64, 16384)
    yield g, orc.gens(64, 16384)
    g.close()


@pytest.fixture(scope="module")
def t8(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    g = bp.Gens(gpu_ctx, 8, 131072)
    yield g, orc.gens(8, 131072)
    g.close()


def _tables(request, m):
    return request.getfixturevalue("t8" if m > 16384 else "t64")


_cells = {}


def _cell(bp, orc, ctx, tables, n, m):
    """(values, blindings, rng seeds, proofs, commitments) of DISTINCT valid proofs of the cell, all from the fresh LABEL transcript"""
    if (n, m) not in _cells:
        gens, ogens = tables
        count = DISTINCT.get((n, m), 1)
        rnd = random.Random(7000 + 3 * n + m)
        values = [rnd.randrange(1 << n) for _ in range(count * m)]
        blind = b"".join(le(rnd.randrange(l)) for _ in range(count * m))
        seeds = b"".join(le(500 + n + i, 8) + bytes(24) for i in range(count))
        if _k(n, m) <= ORACLE_MAX_K:
            proofs, Vs = orc.prove_many(ogens, orc.transcript(LABEL), values, blind, n, m, seeds, nthreads=THREADS)
        else:
            st, proofs, Vs = bp.prove_many(ctx, gens, bp.Transcript(LABEL), values, blind, n, m, seeds)
            assert st == [0] * count
        _cells[(n, m)] = (values, blind, seeds, proofs, Vs)
    return _cells[(n, m)]


def _plus_one(pb, off):
    pb[off:off + 32] = le((int.from_bytes(pb[off:off + 32], "little") + 1) % l)


def _double_v(orc, vb, j):
    vb[32 * j:32 * j + 32] = orc.point_double_encode(bytes(vb[32 * j:32 * j + 32]))


def _damaged(orc, P, V, n, m):
    """[(name, proof, commitments)]: the valid proof and one damage each"""
    k, plen = _k(n, m), len(P)
    out = [("valid", P, V)]

    def proof(name, f):
        pb = bytearray(P); f(pb); out.append((name, bytes(pb), V))

    def commits(name, f):
        vb = bytearray(V); f(vb); out.append((name, P, bytes(vb)))

    proof("t_x + 1", lambda pb: _plus_one(pb, 128))
    proof("b + l (non-canonical)", lambda pb: pb.__setitem__(slice(plen - 32, plen), le(int.from_bytes(P[plen - 32:], "little") + l)))
    proof("last R undecodable", lambda pb: pb.__setitem__(slice(256 + 64 * (k - 1), 288 + 64 * (k - 1)), le(p + 1)))
    commits("V_0 and V_{m-1} doubled", lambda vb: (_double_v(orc, vb, 0), _double_v(orc, vb, m - 1)))
    commits("V_{m/2} undecodable", lambda vb: vb.__setitem__(slice(32 * (m // 2), 32 * (m // 2) + 32), le(p + 1)))
    proof("A = identity", lambda pb: pb.__setitem__(slice(0, 32), bytes(32)))
    proof("one bit of e_blinding", lambda pb: pb.__setitem__(192, pb[192] ^ 1))
    return out


def _oracle(orc, ogens, pb, vb, plen, n, m, count, tstate=None):
    """the oracle's verdict of each proof, every distinct (proof, commitments) verified once"""
    keys = [(bytes(pb[i * plen:(i + 1) * plen]), bytes(vb[32 * m * i:32 * m * (i + 1)])) for i in range(count)]
    uniq = list(dict.fromkeys(keys))
    res = orc.verify_many(ogens, tstate or orc.transcript(LABEL), b"".join(u[0] for u in uniq), plen, b"".join(u[1] for u in uniq), n, m,
                          len(uniq), nthreads=THREADS)
    verdict = dict(zip(uniq, res))
    return [verdict[key] for key in keys]


def _diff(got, want):
    return [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w]


@pytest.mark.parametrize("n,m", CELLS)
def test_cell_matches_the_oracle(request, gpu_ctx, orc, n, m):
    """the valid proof alone (the group check passes), then the valid proof beside seven damaged ones in one batch (the reject path
    decides); at k >= 18 the valid proof is the GPU prover's"""
    import bulletproofs_b200 as bp
    tables = _tables(request, m)
    gens, ogens = tables
    _, _, _, proofs, Vs = _cell(bp, orc, gpu_ctx, tables, n, m)
    plen = bp.rangeproof_size(n, m)
    cases = _damaged(orc, proofs[:plen], Vs[:32 * m], n, m)
    pb, vb = b"".join(c[1] for c in cases), b"".join(c[2] for c in cases)
    want = _oracle(orc, ogens, pb, vb, plen, n, m, len(cases))
    assert want[0] == 0 and want[2] == bp.PROOF_FORMAT_ERROR and all(want[1:]), list(zip([c[0] for c in cases], want))
    assert bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), pb[:plen], vb[:32 * m], n, m, 1, seed=bytes([n]) * 32) == [0]
    got = bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), pb, vb, n, m, len(cases), seed=bytes([m % 251]) * 32)
    assert got == want, [(cases[i][0], g, w) for i, g, w in _diff(got, want)]


# ---------------------------------------------------------------------------------------------- batches at k = 17
N17, M17 = 64, 2048


def _tiled(bp, orc, ctx, tables, count, bad):
    """the cell's distinct proofs tiled to count; bad = {index: "t_x" | "V" | "R"}: t_x + 1, V_{m-1} doubled, last R undecodable"""
    _, _, _, proofs, Vs = _cell(bp, orc, ctx, tables, N17, M17)
    plen, d, k = bp.rangeproof_size(N17, M17), DISTINCT[(N17, M17)], _k(N17, M17)
    pb = bytearray(b"".join(proofs[(i % d) * plen:(i % d + 1) * plen] for i in range(count)))
    vb = bytearray(b"".join(Vs[(i % d) * 32 * M17:(i % d + 1) * 32 * M17] for i in range(count)))
    for i, kind in bad.items():
        if kind == "t_x":
            _plus_one(pb, i * plen + 128)
        elif kind == "V":
            _double_v(orc, vb, i * M17 + M17 - 1)
        else:
            r = i * plen + 256 + 64 * (k - 1)
            pb[r:r + 32] = le(p + 1)
    return pb, vb, plen


@pytest.mark.parametrize("count,bad", [
    (40, {5: "t_x", 20: "R", 37: "V"}),                                          # both chunks fail: the chunks' proofs one by one
    (160, {3: "t_x", 40: "V", 70: "t_x", 100: "V", 130: "t_x", 159: "V"}),      # all five chunks fail: the whole batch at once
])
def test_reject_path_at_k17(t64, gpu_ctx, orc, count, bad):
    import bulletproofs_b200 as bp
    gens, ogens = t64
    pb, vb, plen = _tiled(bp, orc, gpu_ctx, t64, count, bad)
    want = _oracle(orc, ogens, pb, vb, plen, N17, M17, count)
    assert [i for i, w in enumerate(want) if w] == sorted(bad), want
    got = bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), bytes(pb), bytes(vb), N17, M17, count, seed=bytes([count % 256]) * 32)
    assert got == want, _diff(got, want)


def test_launch_group_at_k17(t64, gpu_ctx, orc):
    """two batches of six on the direct path and through a reserved BatchVerifier (graph capture), host entry points (codes) and the device
    entry point (flags): batch 0 holds an undecodable proof only (its combination passes), batch 1 a well-formed invalid one"""
    import bulletproofs_b200 as bp
    count = 6
    pb, vb, plen = _tiled(bp, orc, gpu_ctx, t64, 2 * count, {1: "R", count + 2: "t_x"})
    want = _check_case(bp, orc, t64[1], N17, M17, count, 2, pb, vb, plen, failing=[1])
    assert [i for i, w in enumerate(want) if w] == [1, count + 2]


def test_mixed_call_with_large_classes(t64, gpu_ctx, orc):
    """one verify_mixed call: (64, 2048) and (8, 4096) classes with damage, beside three undamaged grid classes; every verdict equals the
    oracle's and verify_batch's on that proof alone"""
    import bulletproofs_b200 as bp
    gens, ogens = t64
    pb, vb, plen = _tiled(bp, orc, gpu_ctx, t64, 6, {1: "t_x", 4: "V"})
    items = [(bytes(pb[i * plen:(i + 1) * plen]), bytes(vb[32 * M17 * i:32 * M17 * (i + 1)]), N17) for i in range(6)]
    _, _, _, P8, V8 = _cell(bp, orc, gpu_ctx, t64, 8, 4096)
    items += [(P, V, 8) for _, P, V in _damaged(orc, P8, V8, 8, 4096)[:4]]        # valid, t_x + 1, b + l, last R undecodable
    bad = {1, 4, 7, 8, 9}
    for n, m in ((64, 1), (16, 4), (8, 32)):
        proofs, Vs, gplen = _grid_cell(orc, ogens, n, m)
        items += [(proofs[i * gplen:(i + 1) * gplen], Vs[32 * m * i:32 * m * (i + 1)], n) for i in range(5)]
    flags = [i in bad for i in range(len(items))]
    perm = list(range(len(items)))
    random.Random(17).shuffle(perm)
    items, flags = [items[i] for i in perm], [flags[i] for i in perm]
    got = _check_mixed(bp, orc, gpu_ctx, gens, ogens, items, bytes([17]) * 32)
    assert [v != 0 for v in got] == flags


# ---------------------------------------------------------------------------------------------- prover
@pytest.mark.parametrize("n,m", [(64, 64), (8, 1024), (8, 2048), (64, 1024), (64, 2048)])
def test_prover_bytes_match_the_oracle(t64, gpu_ctx, orc, n, m):
    """prove_many of the cell's first proof alone, and at (64, 64) of both proofs in one call, gives the oracle prover's bytes"""
    import bulletproofs_b200 as bp
    gens, _ = t64
    values, blind, seeds, proofs, Vs = _cell(bp, orc, gpu_ctx, t64, n, m)
    plen = bp.rangeproof_size(n, m)
    for count in (1, 2) if (n, m) == (64, 64) else (1,):
        st, got_p, got_V = bp.prove_many(gpu_ctx, gens, bp.Transcript(LABEL), values[:count * m], blind[:32 * count * m], n, m, seeds[:32 * count])
        assert st == [0] * count
        assert got_V == Vs[:32 * count * m]
        assert got_p == proofs[:count * plen]


@pytest.mark.parametrize("n,m", CELLS[-4:])
def test_prover_commitments_beyond_the_oracle_prover(request, gpu_ctx, orc, n, m):
    """k = 18..20, where only the GPU prover runs in the suite: its commitments are V_j = v_j B + r_j B_blinding (the oracle's MSM at j = 0,
    m/2, m-1); test_cell_matches_the_oracle checks its proofs with both verifiers"""
    import bulletproofs_b200 as bp
    values, blind, _, proofs, Vs = _cell(bp, orc, gpu_ctx, _tables(request, m), n, m)
    assert len(proofs) == bp.rangeproof_size(n, m) and len(Vs) == 32 * m
    B, Bb = orc.pedersen()
    for j in (0, m // 2, m - 1):
        assert orc.msm(le(values[j]) + blind[32 * j:32 * j + 32], B + Bb) == (0, Vs[32 * j:32 * j + 32]), j


# ---------------------------------------------------------------------------------------------- transcript
def test_caller_transcript_at_a_nonzero_position(t64, gpu_ctx, orc):
    """(64, 2048) proofs made and verified from a transcript that absorbed a message after Transcript::new: accepted from that transcript,
    rejected from a fresh one, by both verifiers; a t_x + 1 beside them is rejected"""
    import bulletproofs_b200 as bp
    gens, ogens = t64
    values, blind, seeds, _, _ = _cell(bp, orc, gpu_ctx, t64, N17, M17)
    t = bp.Transcript(LABEL)
    t.append_message(b"session", b"large aggregation")
    ot = orc.transcript_append(orc.transcript(LABEL), b"session", b"large aggregation")
    assert ot[:bp.TRANSCRIPT_BYTES] == t.to_bytes()
    st, proofs, Vs = bp.prove_many(gpu_ctx, gens, t, values[:2 * M17], blind[:64 * M17], N17, M17, seeds[:64])
    assert st == [0, 0]
    plen = bp.rangeproof_size(N17, M17)
    pb = bytearray(proofs)
    _plus_one(pb, plen + 128)
    want = _oracle(orc, ogens, pb, Vs, plen, N17, M17, 2, tstate=ot)
    assert want[0] == 0 and want[1] != 0
    assert bp.verify_batch(gpu_ctx, gens, t, bytes(pb), Vs, N17, M17, 2, seed=bytes([5]) * 32) == want
    fresh = orc.rangeproof_verify(ogens, orc.transcript(LABEL), proofs[:plen], Vs[:32 * M17], M17, N17)
    assert fresh != 0
    assert bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), proofs[:plen], Vs[:32 * M17], N17, M17, 1, seed=bytes([6]) * 32) == [fresh]
