"""GPU tier (-m gpu): a reserved verifier graph and the scratch it bakes in.  The captured graph holds the addresses of the verifier's
buffers; a larger geometry on the same context regrows (moves) them.  Afterwards the reserved geometry must still verify correctly, on
the direct path until it is reserved again, and the recaptured graph must agree."""
import pytest

from test_gpu_group_check import LABEL, _bad, _expected
from test_gpu_parity import _workload

pytestmark = pytest.mark.gpu

N, M = 64, 1
A = (8, 2)          # (proofs per batch, batches) of the reserved geometry
B = (32, 4)         # 4x the proofs and 2x the batches: regrows every per-proof and per-batch buffer of the graph
SEED = bytes([5]) * 32


def test_reserved_graph_after_a_larger_geometry_regrew_its_scratch(orc):
    import torch
    import bulletproofs_b200 as bp
    og = orc.gens(N, M)
    proofs, Vs = _workload(orc, og, LABEL, N, M, 8, seed=4242)
    plen = len(proofs) // 8

    def case(geom, bad):
        count, nb = geom
        pb, vb = bytearray(proofs * (count * nb // 8)), bytearray(Vs * (count * nb // 8))
        for i in bad:
            _bad(pb, plen, i)
        want = orc.verify_many(og, orc.transcript(LABEL), bytes(pb), plen, bytes(vb), N, M, count * nb)
        assert [i for i, w in enumerate(want) if w] == list(bad)
        ok_want, dev_want = _expected(want, count, nb, {i // count for i in bad})
        return bytes(pb), bytes(vb), want, ok_want, dev_want

    # bad proofs at different positions in A and B: stale verdicts or flags of B cannot pass for A's
    a_pb, a_vb, a_want, a_ok, a_dev = case(A, [8 + 3])                   # A: batch 1 fails
    b_pb, b_vb, b_want, b_ok, b_dev = case(B, [5, 2 * 32 + 20])          # B: batches 0 and 2 fail
    assert a_ok == [1, 0] and b_ok == [0, 1, 0, 1]

    ctx = bp.Context(0)
    gens = bp.Gens(ctx, N, M)
    d_p = torch.frombuffer(bytearray(a_pb), dtype=torch.uint8).cuda(); d_v = torch.frombuffer(bytearray(a_vb), dtype=torch.uint8).cuda()
    d_verd = torch.full((A[0] * A[1],), 77, dtype=torch.int32, device="cuda"); h_ok = torch.full((A[1],), 9, dtype=torch.int32).pin_memory()
    torch.cuda.synchronize()

    def check_a(when):
        got, ok = bp.verify_group(ctx, gens, bp.Transcript(LABEL), a_pb, a_vb, N, M, *A, seed=SEED)
        assert got == a_want and ok == a_ok, (when, "host", got, ok)
        d_verd.fill_(77); h_ok.fill_(9); torch.cuda.synchronize()
        bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), N, M, *A, reserve=False).run_device(d_p.data_ptr(), d_v.data_ptr(), d_verd.data_ptr(),
                                                                                              h_ok.data_ptr(), SEED)
        ctx.synchronize()
        assert d_verd.cpu().tolist() == a_dev and h_ok.tolist() == a_ok, (when, "device", d_verd.cpu().tolist(), h_ok.tolist())

    try:
        bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), N, M, *A)      # reserve A: arenas sized, graph captured
        check_a("reserved")
        got, ok = bp.verify_group(ctx, gens, bp.Transcript(LABEL), b_pb, b_vb, N, M, *B, seed=SEED)
        assert got == b_want and ok == b_ok, ("B", got, ok)
        check_a("after B regrew the scratch")
        bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), N, M, *A)      # reserve A again: the graph is captured over the new buffers
        check_a("reserved again")
    finally:
        gens.close(); ctx.close()
