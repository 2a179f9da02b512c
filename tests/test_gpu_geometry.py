"""GPU tier (-m gpu): the batch verifier at every (n, m) of the reference's range-proof benchmark grid, n in {8, 16, 32, 64} x m in
{1, 2, 4, 8, 16, 32}, against the oracle.  The geometry decides the verification-scalar tables (the split of the k index bits, see
rp.cuh: TL = 2^ceil(k/2) lies above n only at (8,16), (8,32) and (16,32)), the powers of z of the commitments (up to z^31), the
commitments k_rp_decompress stages per proof, the static rows of up to S = 4098 terms and the term -> generator map when the table
holds more generators or parties than the proofs use.  The second half checks the codes of calls whose parameters are rejected."""
import pytest

from oracle_binding import L_ORDER as l, P_FIELD as p
from test_gpu_group_check import LABEL, _bad, _check_case, _malformed
from test_gpu_parity import _workload, le

pytestmark = pytest.mark.gpu

GRID = [(n, m) for n in (8, 16, 32, 64) for m in (1, 2, 4, 8, 16, 32)]
TL_ABOVE_N = [(8, 16), (8, 32), (16, 32)]
COUNT = 33                      # one full chunk of 32 proofs and a ragged chunk of one
DISTINCT = 4                    # oracle proofs per cell, tiled to COUNT


def _k(n, m):
    return (n * m).bit_length() - 1


@pytest.fixture(scope="module")
def og(orc):
    return orc.gens(64, 32)


@pytest.fixture(scope="module")
def gens64x32(gpu_ctx):
    import bulletproofs_b200 as bp
    g = bp.Gens(gpu_ctx, 64, 32)
    yield g
    g.close()


_cells = {}


def _cell(orc, og, n, m):
    """DISTINCT oracle proofs of the cell tiled to COUNT: (proofs, commitments, proof length)"""
    if (n, m) not in _cells:
        proofs, Vs = _workload(orc, og, LABEL, n, m, DISTINCT, seed=9000 + 100 * n + m)
        reps = -(-COUNT // DISTINCT)
        plen = len(proofs) // DISTINCT
        _cells[(n, m)] = ((proofs * reps)[:COUNT * plen], (Vs * reps)[:COUNT * 32 * m], plen)
    return _cells[(n, m)]


def _damage(pb, vb, plen, n, m, base=0):
    """six damaged proofs in both chunks: a well-formed invalid one, a non-canonical b, an undecodable last R, an identity T_2, an
    identity last commitment (accepted by the transcript, the statement is false) and one flipped bit in a commitment; returns their indices"""
    k = _k(n, m)
    at = [base + i for i in (1, 8, 15, 22, 31, 32)]
    _bad(pb, plen, at[0])
    pb[(at[1] + 1) * plen - 32:(at[1] + 1) * plen] = le(l)
    r = at[2] * plen + 224 + 64 * (k - 1) + 32
    pb[r:r + 32] = le(p + 1)
    pb[at[3] * plen + 96:at[3] * plen + 128] = bytes(32)
    v = (at[4] * m + m - 1) * 32
    vb[v:v + 32] = bytes(32)
    vb[(at[5] * m + m // 2) * 32 + 3] ^= 0x40
    return at


def _verify(bp, orc, ctx, gens, ogens, n, m, pb, vb, plen, count, seed):
    want = orc.verify_many(ogens, orc.transcript(LABEL), bytes(pb), plen, bytes(vb), n, m, count)
    got = bp.verify_batch(ctx, gens, bp.Transcript(LABEL), bytes(pb), bytes(vb), n, m, count, seed=seed)
    assert got == want, (n, m, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w])
    return want


def test_grid_reaches_both_table_regimes():
    """the cells of TL_ABOVE_N are the ones whose low index group is wider than n (rp_kl: kl = ceil(k/2))"""
    above = [(n, m) for n, m in GRID if 1 << ((_k(n, m) + 1) // 2) > n]
    assert above == TL_ABOVE_N, above


@pytest.mark.parametrize("n,m", GRID)
def test_verify_every_grid_cell(gpu_ctx, orc, og, gens64x32, n, m):
    """Gens(64, 32) for every cell, so the table's generator and party strides differ from (n, m); the TL > n cells again with a
    table of exactly (n, m)"""
    import bulletproofs_b200 as bp
    proofs, Vs, plen = _cell(orc, og, n, m)
    tables = [(gens64x32, og)]
    if (n, m) in TL_ABOVE_N:
        tables.append((bp.Gens(gpu_ctx, n, m), orc.gens(n, m)))
    for gens, ogens in tables:
        assert _verify(bp, orc, gpu_ctx, gens, ogens, n, m, proofs, Vs, plen, COUNT, bytes([n + m]) * 32) == [0] * COUNT
        pb, vb = bytearray(proofs), bytearray(Vs)
        at = _damage(pb, vb, plen, n, m)
        want = _verify(bp, orc, gpu_ctx, gens, ogens, n, m, pb, vb, plen, COUNT, bytes([n ^ m]) * 32)
        assert [i for i, w in enumerate(want) if w] == at and want[at[1]] == 2, (n, m, want)
    if len(tables) > 1:
        tables[1][0].close()


@pytest.mark.parametrize("n,m", TL_ABOVE_N + [(64, 32)])
def test_group_check_on_grid_cells(orc, og, n, m):
    """two batches per launch group on the direct and the graph path, host (exact codes) and device (flags) entry points"""
    import bulletproofs_b200 as bp
    proofs, Vs, plen = _cell(orc, og, n, m)
    ogens = orc.gens(n, m)
    pb, vb = bytearray(proofs * 2), bytearray(Vs * 2)
    assert _check_case(bp, orc, ogens, n, m, COUNT, 2, pb, vb, plen) == [0] * (2 * COUNT)
    at = _damage(pb, vb, plen, n, m, base=COUNT)
    want = _check_case(bp, orc, ogens, n, m, COUNT, 2, pb, vb, plen, failing=[1])
    assert [i for i, w in enumerate(want) if w] == at


# ---------------------------------------------------------------------------------------------- rejected parameters
def _mixed(proofs, Vs, plen, m_have, m_use, count=6):
    """count proofs cycling through the given ones, with commitments cut to m_use per proof; proof 1 gets t_x = 2^256 - 1 and proof 4
    a = l (both rejected by RangeProof::from_bytes)"""
    have = len(proofs) // plen
    pb = bytearray(b"".join(proofs[(i % have) * plen:(i % have + 1) * plen] for i in range(count)))
    vb = b"".join(Vs[(i % have) * 32 * m_have:(i % have) * 32 * m_have + 32 * m_use] for i in range(count))
    _malformed(pb, plen, 1)
    k = (plen // 32 - 9) // 2
    a = 4 * plen + 224 + 64 * k
    pb[a:a + 32] = le(l)
    return bytes(pb), vb


def test_rejected_parameters_keep_the_reference_order(gpu_ctx, orc, og, gens64x32):
    """RangeProof::from_bytes runs before verify_multiple's parameter checks: in a call whose parameters are rejected, a proof with a
    non-canonical scalar gets FormatError (2) and the others the parameter's code, as in the oracle.  The last setup has parameters that
    pass and a length that matches, so the kernels run and must reject the false statement."""
    import bulletproofs_b200 as bp
    g64x16, g32x32 = bp.Gens(gpu_ctx, 64, 16), bp.Gens(gpu_ctx, 32, 32)
    og64x16, og32x32 = orc.gens(64, 16), orc.gens(32, 32)
    ot = orc.transcript(LABEL)
    setups = [  # (name, proofs made at (n0, m0), verified as (n, m), device gens, oracle gens, parameter code)
        ("n = 12", (8, 1), (12, 1), gens64x32, og, bp.PROOF_INVALID_BITSIZE),
        ("(64,32) with Gens(64,16)", (64, 32), (64, 32), g64x16, og64x16, bp.PROOF_INVALID_GENERATORS_LENGTH),
        ("(64,1) with Gens(32,32)", (64, 1), (64, 1), g32x32, og32x32, bp.PROOF_INVALID_GENERATORS_LENGTH),
        ("m = 3", (8, 4), (8, 3), gens64x32, og, bp.PROOF_VERIFICATION_ERROR),
        ("(8,32) as (8,16)", (8, 32), (8, 16), gens64x32, og, bp.PROOF_VERIFICATION_ERROR),
        ("(8,32) as (16,16)", (8, 32), (16, 16), gens64x32, og, bp.PROOF_VERIFICATION_ERROR),
    ]
    for name, (n0, m0), (n, m), gens, ogens, code in setups:
        proofs, Vs, plen = _cell(orc, og, n0, m0)
        pb, vb = _mixed(proofs, Vs, plen, m0, m)
        want = orc.verify_many(ogens, ot, pb, plen, vb, n, m, 6)
        assert want == [code, 2, code, code, 2, code], (name, want)
        assert [orc.rangeproof_verify(ogens, ot, pb[i * plen:(i + 1) * plen], vb[32 * m * i:32 * m * (i + 1)], m, n) for i in (0, 1, 4)] == want[:2] + want[4:5]
        got = bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), pb, vb, n, m, 6, proof_len=plen, seed=bytes([7]) * 32)
        assert got == want, (name, got, want)
    # a launch group with rejected parameters: the same per-proof codes, every batch flag cleared
    proofs, Vs, plen = _cell(orc, og, 64, 1)
    pb, vb = _mixed(proofs, Vs, plen, 1, 1, count=12)
    want = orc.verify_many(og32x32, ot, pb, plen, vb, 64, 1, 12)
    assert bp.verify_group(gpu_ctx, g32x32, bp.Transcript(LABEL), pb, vb, 64, 1, 6, 2) == (want, [0, 0])
    # the device entry point has no per-proof codes for rejected parameters: it refuses the call
    import torch
    d_p = torch.frombuffer(bytearray(pb), dtype=torch.uint8).cuda(); d_v = torch.frombuffer(bytearray(vb), dtype=torch.uint8).cuda()
    d_verd = torch.zeros(12, dtype=torch.int32, device="cuda")
    with pytest.raises(bp.BpError):
        bp.BatchVerifier(gpu_ctx, g32x32, bp.Transcript(LABEL), 64, 1, 6, 2, reserve=False).run_device(d_p.data_ptr(), d_v.data_ptr(), d_verd.data_ptr())
    g64x16.close(); g32x32.close()
