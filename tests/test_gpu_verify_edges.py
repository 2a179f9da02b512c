"""GPU tier (-m gpu): the verifier at the bench geometry and at the edges of its reject path and its arguments, against the oracle's
per-proof verdicts.  Inputs are a few dozen oracle proofs tiled to size (each copy is an independent proof of the batch).  Every case
runs on the direct-launch path and on the reserved (graph) path, through the host and the device entry points (test_gpu_group_check).
The branch each test is about is shown to be reached with the selection rules of rp.cuh / msm_common.cuh built for the host."""
import ctypes
import os
import random

import pytest

from test_gpu_group_check import LABEL, _bad, _check_case, _expected, _malformed, _paths, _undecodable
from test_gpu_parity import _workload

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    E.emul_use_combine4.argtypes = [ctypes.c_uint32]
    E.emul_rp_recheck_whole_batch.argtypes = [ctypes.c_uint32]
    return E


@pytest.fixture(scope="module")
def bench_work(orc):
    """BASELINE config 2 in groups of 8: 8 batches of 1024 (64, 1) proofs, 64 oracle proofs tiled"""
    og = orc.gens(64, 1)
    proofs, Vs = _workload(orc, og, LABEL, 64, 1, 64, seed=8102)
    return og, proofs * 128, Vs * 128, len(proofs) // 64


def _failing_chunks(E, idx, count):
    chunk = E.emul_rp_chunk()
    return {(i % count) // chunk for i in idx}


def test_bench_geometry_all_valid(orc, bench_work):
    import bulletproofs_b200 as bp
    og, proofs, Vs, plen = bench_work
    want = _check_case(bp, orc, og, 64, 1, 1024, 8, bytearray(proofs), bytearray(Vs), plen)
    assert want == [0] * 8192


def test_bench_geometry_one_bad_proof(orc, bench_work, E):
    """one bad proof in batch 5: the group check fails, the per-batch pass flags batch 5, its one failing chunk is re-checked proof by proof"""
    import bulletproofs_b200 as bp
    og, proofs, Vs, plen = bench_work
    pb = bytearray(proofs); bad = 5 * 1024 + 333
    _bad(pb, plen, bad)
    assert not E.emul_rp_recheck_whole_batch(len(_failing_chunks(E, [bad], 1024)))
    want = _check_case(bp, orc, og, 64, 1, 1024, 8, pb, bytearray(Vs), plen, failing=[5])
    assert [i for i, w in enumerate(want) if w] == [bad]


def test_bench_geometry_whole_batch_recheck(orc, bench_work, E):
    """bad proofs in six chunks of batch 7: the batch is re-checked in one pass of 1024 MSMs (one per proof) that starts at proof
    7*1024 of the group, and those MSMs combine their windows with k_msm_combine"""
    import bulletproofs_b200 as bp
    og, proofs, Vs, plen = bench_work
    pb = bytearray(proofs)
    bad = [7 * 1024 + ch * 32 + off for ch, off in ((0, 0), (3, 17), (9, 31), (10, 2), (22, 9), (31, 31))]
    for i in bad:
        _bad(pb, plen, i)
    assert E.emul_rp_recheck_whole_batch(len(_failing_chunks(E, bad, 1024))), "six failing chunks no longer re-check the whole batch"
    assert not E.emul_use_combine4(1024)
    want = _check_case(bp, orc, og, 64, 1, 1024, 8, pb, bytearray(Vs), plen, failing=[7])
    assert [i for i, w in enumerate(want) if w] == bad


def test_single_batch_whole_recheck_with_malformed_proofs(orc, bench_work, E):
    """one batch of 1024 with a bad proof in every chunk of 32, and malformed and undecodable proofs that keep their own codes"""
    import bulletproofs_b200 as bp
    og, proofs, Vs, plen = bench_work
    pb, vb = bytearray(proofs[:1024 * plen]), bytearray(Vs[:1024 * 32])
    rnd = random.Random(1024)
    bad = [ch * 32 + rnd.randrange(32) for ch in range(32)]
    for i in bad:
        _bad(pb, plen, i)
    others = [i for i in range(1024) if i not in bad]
    malformed, undecodable = rnd.sample(others, 5), []
    for i in malformed:
        _malformed(pb, plen, i)
    for i in rnd.sample([i for i in others if i not in malformed], 5):
        _undecodable(pb, plen, i); undecodable.append(i)
    assert E.emul_rp_recheck_whole_batch(len(_failing_chunks(E, bad, 1024)))
    want = _check_case(bp, orc, og, 64, 1, 1024, 1, pb, vb, plen, failing=[0])
    assert sorted(i for i, w in enumerate(want) if w) == sorted(bad + malformed + undecodable)
    assert all(want[i] == bp.PROOF_FORMAT_ERROR for i in malformed) and all(want[i] == bp.PROOF_VERIFICATION_ERROR for i in bad + undecodable)


def test_group_of_256_batches_and_the_limit(orc, E):
    """256 batches of four (8, 1) proofs, the largest group: the per-batch pass after a failing group check runs 256 MSMs, the last
    count on k_msm_combine4.  257 batches are refused by the host entry point, the device entry point and reserve."""
    import torch
    import bulletproofs_b200 as bp
    n, m, count = 8, 1, 4
    og = orc.gens(n, m)
    proofs, Vs = _workload(orc, og, LABEL, n, m, 32, seed=256)
    plen = len(proofs) // 32
    pb, vb = bytearray(proofs * 33), bytearray(Vs * 33)            # 1056 proofs: enough for 257 batches
    assert E.emul_use_combine4(256)
    _bad(pb, plen, 200 * count + 3)
    want = _check_case(bp, orc, og, n, m, count, 256, pb[:256 * count * plen], vb[:256 * count * 32], plen, failing=[200])
    assert [i for i, w in enumerate(want) if w] == [200 * count + 3]
    ctx = bp.Context(0); gens = bp.Gens(ctx, n, m)
    try:
        t = bp.Transcript(LABEL)
        with pytest.raises(bp.BpError) as e:
            bp.verify_group(ctx, gens, t, bytes(pb[:257 * count * plen]), bytes(vb[:257 * count * 32]), n, m, count, 257)
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
        d_p = torch.frombuffer(bytearray(pb), dtype=torch.uint8).cuda(); d_v = torch.frombuffer(bytearray(vb), dtype=torch.uint8).cuda()
        d_verd = torch.zeros(257 * count, dtype=torch.int32, device="cuda")
        with pytest.raises(bp.BpError) as e:
            bp.BatchVerifier(ctx, gens, t, n, m, count, 257, reserve=False).run_device(d_p.data_ptr(), d_v.data_ptr(), d_verd.data_ptr())
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
        with pytest.raises(bp.BpError) as e:
            bp.BatchVerifier(ctx, gens, t, n, m, count, 257)
        assert e.value.code == bp.ERR_INVALID_ARGUMENT
        got, ok = bp.verify_group(ctx, gens, t, bytes(pb[:256 * count * plen]), bytes(vb[:256 * count * 32]), n, m, count, 256)
        assert got == want and ok == [int(b != 200) for b in range(256)]          # nothing was left pending by the refused calls
    finally:
        gens.close(); ctx.close()


@pytest.mark.parametrize("p_off,v_off", [(1, 8), (4, 8)])
def test_device_path_unaligned_inputs(orc, p_off, v_off):
    """Proof and commitment arrays at addresses that are not 16-byte aligned: k_rp_decompress stages them with a cooperative copy
    instead of the TMA bulk copy (which needs 16-byte alignment), and every other reader loads bytes.  Same verdicts and flags as
    from aligned buffers."""
    import torch
    import bulletproofs_b200 as bp
    n, m, count, nb = 64, 1, 24, 4
    og = orc.gens(n, m)
    proofs, Vs = _workload(orc, og, LABEL, n, m, 24, seed=7116)
    plen = len(proofs) // 24
    pb, vb = bytearray(proofs * nb), bytearray(Vs * nb)
    _bad(pb, plen, 2 * 24 + 5); _malformed(pb, plen, 2 * 24 + 11); _undecodable(pb, plen, 3 * 24 + 1)
    want = orc.verify_many(og, orc.transcript(LABEL), bytes(pb), plen, bytes(vb), n, m, count * nb)
    ok_want, dev_want = _expected(want, count, nb, {2})
    seed = bytes([5]) * 32
    for name, ctx, gens in _paths(bp, n, m, count, nb):
        runs = []
        for po, vo in ((0, 0), (p_off, v_off)):
            d_p = torch.zeros(len(pb) + 16, dtype=torch.uint8, device="cuda"); d_v = torch.zeros(len(vb) + 16, dtype=torch.uint8, device="cuda")
            d_p[po:po + len(pb)] = torch.frombuffer(bytearray(pb), dtype=torch.uint8).cuda()
            d_v[vo:vo + len(vb)] = torch.frombuffer(bytearray(vb), dtype=torch.uint8).cuda()
            pp, vp = d_p.data_ptr() + po, d_v.data_ptr() + vo
            assert (pp % 16 == 0) == (po == 0) and (vp % 16 == 0) == (vo == 0)
            d_verd = torch.full((count * nb,), 77, dtype=torch.int32, device="cuda"); h_ok = torch.full((nb,), 9, dtype=torch.int32).pin_memory()
            torch.cuda.synchronize()
            bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), n, m, count, nb, reserve=False).run_device(pp, vp, d_verd.data_ptr(), h_ok.data_ptr(), seed)
            ctx.synchronize()
            runs.append((d_verd.cpu().tolist(), h_ok.tolist()))
        assert runs[0] == (dev_want, ok_want), name
        assert runs[1] == runs[0], (name, [(i, a, b) for i, (a, b) in enumerate(zip(runs[1][0], runs[0][0])) if a != b])
