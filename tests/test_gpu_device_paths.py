"""GPU tier (-m gpu): the paths by which callers reach the MSM and verifier kernels, each result against the oracle per MSM or per proof.

1. Device buffers the kernels cannot read (a misaligned scalar, point, output, offset or verdict pointer) are refused with
   BP_ERR_INVALID_ARGUMENT before anything is queued, and the same context then computes correctly; proof and commitment
   buffers of any alignment stay accepted.
2. bp_msm_batch_device and bp_points_create_device / bp_msm_points_device: config 4's default shape (8 MSMs of 2^16 generator-chain
   points and ChaCha20 scalars), more than 2^22 terms in one call, device offsets around empty, poisoned and non-canonical MSMs,
   changing term counts over one resident point set, and argument errors.
3. Device calls queued without synchronising, then a call large enough to regrow the context's scratch.
4. Four contexts on four streams sharing one generator table (built once, imported into empty tables), graph and direct-launch
   verifiers mixed, driven from two threads: every call's verdicts and flags are its own.
5. Profiled verification (direct launches, decompression on the main stream) against unprofiled verification."""
import ctypes
import hashlib
import os
import random
import threading
from concurrent.futures import ThreadPoolExecutor

import pytest

from oracle_binding import L_ORDER as l
from test_gpu_group_check import LABEL, _bad, _expected, _identity_A, _malformed, _undecodable
from test_gpu_parity import _workload, le

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNDECODABLE = b"\x01" + bytes(31)          # s odd: not a canonical Ristretto encoding
NONCANONICAL = (l, 1 << 255, (1 << 256) - 1)


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    E.emul_pick_window.argtypes = [ctypes.c_uint64]
    E.emul_avg_terms.argtypes = [ctypes.c_uint64, ctypes.c_uint32]; E.emul_avg_terms.restype = ctypes.c_uint64
    E.emul_use_combine4.argtypes = [ctypes.c_uint32]
    return E


@pytest.fixture(scope="module")
def rp_work(orc):
    """24 distinct valid (64, 1) oracle proofs, the oracle's generators and the proof length"""
    og = orc.gens(64, 1)
    proofs, Vs = _workload(orc, og, LABEL, 64, 1, 24, seed=7100)
    plen = len(proofs) // 24
    assert orc.verify_many(og, orc.transcript(LABEL), proofs, plen, Vs, 64, 1, 24) == [0] * 24
    return og, proofs, Vs, plen


def _dev(data: bytes, front: int = 0):
    """device copy of `data` starting `front` bytes into a fresh allocation (so that data_ptr() + front holds it)"""
    import torch
    return torch.frombuffer(bytearray(bytes(front) + data + bytes(16)), dtype=torch.uint8).cuda()


def _offsets(sizes):
    offs = [0]
    for s in sizes:
        offs.append(offs[-1] + s)
    return offs


def _u32(values) -> bytes:
    return b"".join(v.to_bytes(4, "little") for v in values)


def _msm_device(ctx, d_sc, d_pts, d_off, n_msm, T, d_out, d_st):
    import bulletproofs_b200 as bp
    return bp.lib().bp_msm_batch_device(ctx._h, d_sc, d_pts, d_off, n_msm, T, d_out, d_st)


def _rows(t, n):
    return [bytes(t[32 * j:32 * j + 32].cpu().numpy().tobytes()) for j in range(n)]


def _want_msms(orc, sc, pp, offs):
    """the oracle's (status, result) per MSM; an empty MSM is the identity, 32 zero bytes"""
    return [orc.msm(sc[32 * a:32 * b], pp[32 * a:32 * b]) for a, b in zip(offs, offs[1:])]


def _rand_points(orc, rnd, n):
    return [orc.from_uniform(rnd.randbytes(64)) for _ in range(n)]


# ------------------------------------------------------------------------------------------------ 1. misaligned device buffers
def test_misaligned_msm_buffers_are_refused(orc):
    """16-byte rule for scalars, points and outputs (offsets 1 and 8), 4-byte rule for the offsets (offset 2): BP_ERR_INVALID_ARGUMENT
    with a message, nothing launched; then aligned calls on the same context equal the oracle"""
    import torch
    import bulletproofs_b200 as bp
    ctx = bp.Context(0)
    rnd = random.Random(1601)
    base = _rand_points(orc, rnd, 32)
    offs = [0, 150, 300]
    sc = b"".join(le(rnd.randrange(l)) for _ in range(300)); pp = b"".join(rnd.choice(base) for _ in range(300))
    d_sc, d_pp, d_off = _dev(sc), _dev(pp), _dev(_u32(offs))
    d_out = torch.zeros(2 * 32 + 16, dtype=torch.uint8, device="cuda"); d_st = torch.full((2,), 9, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    good = dict(sc=d_sc.data_ptr(), pp=d_pp.data_ptr(), off=d_off.data_ptr(), out=d_out.data_ptr())
    launches = ctx.launches
    for arg, shifts in (("sc", (1, 8)), ("pp", (1, 8)), ("out", (1, 8)), ("off", (2,))):
        for s in shifts:
            a = dict(good); a[arg] += s
            assert _msm_device(ctx, a["sc"], a["pp"], a["off"], 2, 300, a["out"], d_st.data_ptr()) == bp.ERR_INVALID_ARGUMENT, (arg, s)
            assert "aligned" in bp.lib().bp_last_error(ctx._h).decode(), (arg, s)
    ps = None
    for s in (1, 8):
        with pytest.raises(bp.BpError) as ei:
            bp.PointSet(ctx, n=300, device_ptr=good["pp"] + s)
        assert ei.value.code == bp.ERR_INVALID_ARGUMENT and "aligned" in str(ei.value)
    ps = bp.PointSet(ctx, n=300, device_ptr=good["pp"])
    launches_ps = ctx.launches - launches                       # the point set's own decompression
    for arg, s in (("sc", 1), ("sc", 8), ("out", 1), ("out", 8)):
        a = dict(good); a[arg] += s
        with pytest.raises(bp.BpError) as ei:
            ps.msm_device(a["sc"], 2, 150, a["out"], d_st.data_ptr())
        assert ei.value.code == bp.ERR_INVALID_ARGUMENT and "aligned" in str(ei.value), (arg, s)
    assert ctx.launches - launches == launches_ps, "a refused call queued work"
    # the same context, aligned
    assert _msm_device(ctx, good["sc"], good["pp"], good["off"], 2, 300, good["out"], d_st.data_ptr()) == bp.OK
    ctx.synchronize()
    want = _want_msms(orc, sc, pp, offs)
    assert list(zip(d_st.cpu().tolist(), _rows(d_out, 2))) == want
    d_out.zero_(); torch.cuda.synchronize()
    ps.msm_device(good["sc"], 2, 150, good["out"], d_st.data_ptr())
    ctx.synchronize()
    assert _rows(d_out, 2) == [orc.msm(sc[32 * 150 * j:32 * 150 * (j + 1)], pp[:32 * 150])[1] for j in range(2)]
    ps.close(); ctx.close()


def test_misaligned_verdicts_are_refused_and_unaligned_proofs_accepted(orc, rp_work):
    """d_verdicts_u32 two bytes off: BP_ERR_INVALID_ARGUMENT from both device entry points.  Proofs one byte and commitments eight
    bytes off a 16-byte boundary take the kernels' unaligned staging and give the verdicts of aligned buffers"""
    import torch
    import bulletproofs_b200 as bp
    og, proofs, Vs, plen = rp_work
    n, m, count, nb = 64, 1, 4, 2
    pb = bytearray(proofs[:8 * plen]); _bad(pb, plen, 5)
    vb = Vs[:8 * 32]
    want = orc.verify_many(og, orc.transcript(LABEL), bytes(pb), plen, vb, n, m, 8)
    assert [i for i, w in enumerate(want) if w] == [5]
    ok_want, dev_want = _expected(want, count, nb, {1})
    ctx = bp.Context(0); gens = bp.Gens(ctx, n, m)
    t = bp.Transcript(LABEL).to_bytes()
    d_p, d_v = _dev(bytes(pb)), _dev(vb)
    d_p1, d_v8 = _dev(bytes(pb), front=1), _dev(vb, front=8)
    d_verd = torch.full((8 + 4,), 77, dtype=torch.int32, device="cuda"); h_ok = torch.full((nb,), 9, dtype=torch.int32).pin_memory()
    torch.cuda.synchronize()
    L, launches = bp.lib(), ctx.launches
    mis = d_verd.data_ptr() + 2
    assert L.bp_rangeproof_verify_batch_device(ctx._h, gens._h, t, d_p.data_ptr(), plen, d_v.data_ptr(), n, m, 8, None, mis, None) == bp.ERR_INVALID_ARGUMENT
    assert L.bp_rangeproof_verify_group_device(ctx._h, gens._h, t, d_p.data_ptr(), plen, d_v.data_ptr(), n, m, count, nb, None, mis, h_ok.data_ptr()) == bp.ERR_INVALID_ARGUMENT
    assert "aligned" in L.bp_last_error(ctx._h).decode() and ctx.launches == launches
    ver = bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), n, m, count, nb, reserve=False)
    for dp, dv in ((d_p, d_v), (d_p, d_v8), (d_p1, d_v), (d_p1, d_v8)):
        d_verd.fill_(77); torch.cuda.synchronize()
        ptr_p = dp.data_ptr() + (1 if dp is d_p1 else 0); ptr_v = dv.data_ptr() + (8 if dv is d_v8 else 0)
        ver.run_device(ptr_p, ptr_v, d_verd.data_ptr(), h_ok.data_ptr(), bytes([3]) * 32)
        ctx.synchronize()
        assert d_verd[:8].cpu().tolist() == dev_want and h_ok.tolist() == ok_want, (ptr_p % 16, ptr_v % 16)
    gens.close(); ctx.close()


# ------------------------------------------------------------------------------------------------ 2. device-buffer MSM calls
@pytest.fixture(scope="module")
def chain16(orc):
    """config 4's points: the first 2^16 outputs of the party-0 G generator chain through from_uniform_bytes"""
    n = 1 << 16
    uni = hashlib.shake_256(b"GeneratorsChain" + b"G" + (0).to_bytes(4, "little")).digest(64 * n)
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        pts = b"".join(ex.map(lambda i: orc.from_uniform(uni[64 * i:64 * i + 64]), range(n), chunksize=4096))
    return uni, pts


def test_config4_shape_both_device_forms_every_msm(orc, E, chain16):
    """8 MSMs of 2^16 terms, as bench's msm workload runs them: decompressing every call (bp_msm_batch_device over 8 copies of the
    points) and over a resident point set (bp_msm_points_device); all 8 results of each form equal the oracle's"""
    import torch
    import bulletproofs_b200 as bp
    n, M = 1 << 16, 8
    c = E.emul_pick_window(E.emul_avg_terms(M * n, M))
    assert E.emul_avg_terms(M * n, M) == n and E.emul_use_combine4(M) and 1 << (c - 1) >= 4096, "config 4 no longer takes the wide-window, four-lane-combine pass"
    uni, pts = chain16
    sc = orc.scalars_from_chacha(bytes([0x2a]) * 32, M * n)
    want = [orc.msm(sc[32 * n * j:32 * n * (j + 1)], pts) for j in range(M)]
    assert all(rc == 0 for rc, _ in want)
    ctx = bp.Context(0)
    assert ctx.from_uniform_bytes(uni[:64 * 512]) == pts[:32 * 512]          # the device derives the same chain (bench's form)
    d_sc, d_pts, d_off = _dev(sc), _dev(pts * M), _dev(_u32(range(0, (M + 1) * n, n)))
    d_out = torch.zeros((2, M * 32), dtype=torch.uint8, device="cuda"); d_st = torch.full((2, M), 9, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert _msm_device(ctx, d_sc.data_ptr(), d_pts.data_ptr(), d_off.data_ptr(), M, M * n, d_out[0].data_ptr(), d_st[0].data_ptr()) == bp.OK
    ps = bp.PointSet(ctx, n=n, device_ptr=d_pts.data_ptr())
    ps.msm_device(d_sc.data_ptr(), M, n, d_out[1].data_ptr(), d_st[1].data_ptr())
    ctx.synchronize()
    for form in range(2):
        got = list(zip(d_st[form].cpu().tolist(), _rows(d_out[form], M)))
        assert got == want, (form, [j for j in range(M) if got[j] != want[j]])
    ps.close(); ctx.close()


def test_more_than_2_22_terms_folded(orc, E):
    """8 MSMs of 2^20 terms (2^23 in one call) over 1024 tiled bases, through both device forms: sum_i s_i P_(i mod b) must equal the
    b-term oracle MSM over the folded scalars"""
    import numpy as np
    import torch
    import bulletproofs_b200 as bp
    n, M, b = 1 << 20, 8, 1024
    assert M * n > 1 << 22 and 1 << (E.emul_pick_window(n) - 1) >= 4096
    rnd = random.Random(2023)
    base = b"".join(_rand_points(orc, rnd, b))
    sc = orc.scalars_from_chacha(bytes([0x17]) * 32, M * n)
    limbs = np.frombuffer(sc, dtype=np.uint16).reshape(M, n // b, b, 16).sum(axis=1, dtype=np.uint64)      # per MSM, per base, per 16-bit limb
    want = []
    for j in range(M):
        folded = b"".join(le(sum(int(v) << (16 * k) for k, v in enumerate(limbs[j, i])) % l) for i in range(b))
        want.append(orc.msm(folded, base))
    ctx = bp.Context(0)
    d_base = torch.frombuffer(bytearray(base), dtype=torch.uint8).cuda()
    d_pts = d_base.repeat(M * n // b)
    d_sc = torch.from_numpy(np.frombuffer(sc, dtype=np.uint8).copy()).cuda()
    d_off = _dev(_u32(range(0, (M + 1) * n, n)))
    d_out = torch.zeros((2, M * 32), dtype=torch.uint8, device="cuda"); d_st = torch.full((2, M), 9, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert _msm_device(ctx, d_sc.data_ptr(), d_pts.data_ptr(), d_off.data_ptr(), M, M * n, d_out[0].data_ptr(), d_st[0].data_ptr()) == bp.OK
    ps = bp.PointSet(ctx, n=n, device_ptr=d_pts.data_ptr())
    ps.msm_device(d_sc.data_ptr(), M, n, d_out[1].data_ptr(), d_st[1].data_ptr())
    ctx.synchronize()
    for form in range(2):
        assert list(zip(d_st[form].cpu().tolist(), _rows(d_out[form], M))) == want, form
    ps.close(); ctx.close()


def test_device_offsets_empty_poisoned_and_noncanonical_msms(orc):
    """u32 device offsets with empty MSMs first, in the middle and last (32 zero bytes, status 0); an undecodable point poisons only its
    own MSM (status 1); scalars l, 2^255 and 2^256 - 1, each in an MSM of its own, give status 3, and so does 2^256 - 1 beside an
    undecodable point in the same MSM (k_msm_status: 3 wins over 1); d_status = NULL is accepted and changes no result"""
    import torch
    import bulletproofs_b200 as bp
    sizes = [0, 40, 33, 0, 41, 39, 35, 44, 27, 0]
    offs = _offsets(sizes); T, M = offs[-1], len(sizes)
    rnd = random.Random(909)
    base = _rand_points(orc, rnd, 24)
    sc = [le(rnd.randrange(l)) for _ in range(T)]; pp = [rnd.choice(base) for _ in range(T)]
    pp[offs[2] + 7] = UNDECODABLE
    sc[offs[4] + 40] = le(NONCANONICAL[0])
    sc[offs[5] + 20] = le(NONCANONICAL[2])
    sc[offs[6]] = le(NONCANONICAL[1])
    pp[offs[7] + 3] = UNDECODABLE; sc[offs[7] + 30] = le(NONCANONICAL[2])          # the point comes first: the scalar's code still wins
    assert not orc.point_is_valid(UNDECODABLE) and all(v >= l for v in NONCANONICAL)
    sc, pp = b"".join(sc), b"".join(pp)
    status_want = [0, 0, 1, 0, 3, 3, 3, 3, 0, 0]
    ctx = bp.Context(0)
    d_sc, d_pp, d_off = _dev(sc), _dev(pp), _dev(_u32(offs))
    d_out = torch.full((2, M * 32), 0x5a, dtype=torch.uint8, device="cuda"); d_st = torch.full((M,), 9, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert _msm_device(ctx, d_sc.data_ptr(), d_pp.data_ptr(), d_off.data_ptr(), M, T, d_out[0].data_ptr(), d_st.data_ptr()) == bp.OK
    assert _msm_device(ctx, d_sc.data_ptr(), d_pp.data_ptr(), d_off.data_ptr(), M, T, d_out[1].data_ptr(), None) == bp.OK
    ctx.synchronize()
    assert d_st.cpu().tolist() == status_want
    want = _want_msms(orc, sc, pp, offs)
    outs = _rows(d_out[0], M)
    for j in range(M):
        if sizes[j] == 0:
            assert outs[j] == bytes(32), j
        elif status_want[j] == 0:
            assert want[j] == (0, outs[j]), j
        else:
            assert want[j][0] != 0, j                       # the oracle rejects it too
    assert _rows(d_out[1], M) == outs
    ctx.close()


def test_point_set_calls_with_changing_term_counts(orc):
    """bp_msm_points_device over the first `terms` of 1000 resident points, calls queued without synchronising with (n_msm, terms) =
    (1, 1000), (8, 500), (3, 1000), (2, 7), (4, 1000): the cached term -> point map follows every change of `terms`"""
    import torch
    import bulletproofs_b200 as bp
    rnd = random.Random(1000)
    pts = b"".join(_rand_points(orc, rnd, 1000))
    calls = [(1, 1000), (8, 500), (3, 1000), (2, 7), (4, 1000)]
    scal = [b"".join(le(rnd.randrange(l)) for _ in range(k * t)) for k, t in calls]
    ctx = bp.Context(0)
    d_pts = _dev(pts); d_sc = [_dev(s) for s in scal]
    d_out = torch.zeros((len(calls), 8 * 32), dtype=torch.uint8, device="cuda"); d_st = torch.full((len(calls), 8), 9, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ps = bp.PointSet(ctx, n=1000, device_ptr=d_pts.data_ptr())
    for r, (k, t) in enumerate(calls):
        ps.msm_device(d_sc[r].data_ptr(), k, t, d_out[r].data_ptr(), d_st[r].data_ptr())
    ctx.synchronize()
    for r, (k, t) in enumerate(calls):
        want = [orc.msm(scal[r][32 * t * j:32 * t * (j + 1)], pts[:32 * t]) for j in range(k)]
        assert list(zip(d_st[r, :k].cpu().tolist(), _rows(d_out[r], k))) == want, (r, k, t)
    ps.close(); ctx.close()


def test_device_msm_argument_errors(orc):
    """n_msm = 0, total_terms = 0 or >= 2^31, terms above the set size, n_msm * terms >= 2^31: BP_ERR_INVALID_ARGUMENT, nothing
    launched; the context then computes correctly"""
    import torch
    import bulletproofs_b200 as bp
    rnd = random.Random(31)
    pts = b"".join(_rand_points(orc, rnd, 64)); sc = b"".join(le(rnd.randrange(l)) for _ in range(64))
    ctx = bp.Context(0)
    d_sc, d_pp, d_off = _dev(sc), _dev(pts), _dev(_u32([0, 64]))
    d_out = torch.zeros(32, dtype=torch.uint8, device="cuda"); d_st = torch.full((1,), 9, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ps = bp.PointSet(ctx, n=64, device_ptr=d_pp.data_ptr())
    launches = ctx.launches
    for n_msm, T in ((0, 64), (1, 0), (1, 1 << 31)):
        assert _msm_device(ctx, d_sc.data_ptr(), d_pp.data_ptr(), d_off.data_ptr(), n_msm, T, d_out.data_ptr(), d_st.data_ptr()) == bp.ERR_INVALID_ARGUMENT, (n_msm, T)
    for n_msm, terms in ((0, 64), (1, 0), (1, 65), (1 << 25, 64)):
        with pytest.raises(bp.BpError) as ei:
            ps.msm_device(d_sc.data_ptr(), n_msm, terms, d_out.data_ptr(), d_st.data_ptr())
        assert ei.value.code == bp.ERR_INVALID_ARGUMENT, (n_msm, terms)
    assert ctx.launches == launches, "a refused call queued work"
    ps.msm_device(d_sc.data_ptr(), 1, 64, d_out.data_ptr(), d_st.data_ptr())
    ctx.synchronize()
    assert (int(d_st[0]), _rows(d_out, 1)[0]) == orc.msm(sc, pts)
    ps.close(); ctx.close()


# ------------------------------------------------------------------------------------------------ 3. queued calls, then a regrow
def test_queued_calls_then_a_call_that_regrows_the_scratch(orc):
    """four device MSM calls queued on a fresh context, then without synchronising one of 2^17 terms: its scratch (decompressed points,
    Pippenger arenas) is many times what the queued calls grew, so the context frees and reallocates buffers those calls read.  Every
    output equals the oracle's.  This pins the results of the sequence; it does not show that the queued calls were still running when
    the buffers were freed, so it would not catch a regrow without its stream synchronisation (cudaFree itself usually waits)"""
    import torch
    import bulletproofs_b200 as bp
    rnd = random.Random(17)
    base = _rand_points(orc, rnd, 256)
    shapes = [[700, 0, 900], [1500, 1500], [64] * 30, [2000, 13, 400]] + [[1 << 16, 1 << 16]]
    assert sum(shapes[-1]) > 8 * max(sum(s) for s in shapes[:-1])
    calls = []
    for sizes in shapes:
        offs = _offsets(sizes); T = offs[-1]
        sc = b"".join(le(rnd.randrange(l)) for _ in range(T)); pp = b"".join(base[(7 * i + T) % 256] for i in range(T))
        calls.append((offs, sc, pp, _dev(sc), _dev(pp), _dev(_u32(offs))))
    d_out = torch.zeros((len(shapes), 30 * 32), dtype=torch.uint8, device="cuda"); d_st = torch.full((len(shapes), 30), 9, dtype=torch.uint8, device="cuda")
    ctx = bp.Context(0)
    torch.cuda.synchronize()
    for r, (offs, _, _, d_sc, d_pp, d_off) in enumerate(calls):
        assert _msm_device(ctx, d_sc.data_ptr(), d_pp.data_ptr(), d_off.data_ptr(), len(offs) - 1, offs[-1], d_out[r].data_ptr(), d_st[r].data_ptr()) == bp.OK
    ctx.synchronize()
    for r, (offs, sc, pp, *_) in enumerate(calls):
        k = len(offs) - 1
        assert list(zip(d_st[r, :k].cpu().tolist(), _rows(d_out[r], k))) == _want_msms(orc, sc, pp, offs), r
    ctx.close()


# ------------------------------------------------------------------------------------------------ 4. concurrent contexts
def _variants(orc, og, rp_work, count, nb):
    """inputs of one group: all valid; one bad proof in batch b for every b; malformed / undecodable proofs only.  Each with the
    oracle's per-proof verdicts (proof by proof for the damaged ones) and the set of batches whose combination fails"""
    _, proofs, Vs, plen = rp_work
    total = count * nb
    reps = total // 24 + 1
    base_p, base_v = (proofs * reps)[:total * plen], (Vs * reps)[:total * 32]
    t = orc.transcript(LABEL)

    def make(name, damage, failing):
        pb = bytearray(base_p)
        for fn, i in damage:
            fn(pb, plen, i)
        want = [0] * total
        for _, i in damage:
            want[i] = orc.verify_many(og, t, bytes(pb[i * plen:(i + 1) * plen]), plen, base_v[i * 32:(i + 1) * 32], 64, 1, 1)[0]
            assert want[i] != 0, (name, i)
        return name, bytes(pb), want, failing

    out = [make("valid", [], set())]
    out += [make(f"bad-in-{b}", [(_bad, b * count + (7 * b + 5) % count)], {b}) for b in range(nb)]
    out.append(make("malformed", [(_malformed, 3), (_identity_A, total // 2 + 1), (_undecodable, total - 1)], set()))
    return out, base_v, plen


@pytest.mark.parametrize("count,nb", [(1024, 8), (24, 4)], ids=["bench-geometry", "small"])
def test_concurrent_contexts_from_two_threads(orc, rp_work, count, nb):
    """bench's arrangement: 4 contexts on 4 torch streams, context 0 builds the table and the others import it into empty tables,
    contexts 0 and 2 reserved (captured graph) and 1 and 3 not (direct launches), two host threads, each driving one reserved and one
    unreserved context (thread 0: contexts 0, 1; thread 1: contexts 2, 3), so one thread alternates graph replays with direct launches.
    Each thread queues device calls over rotating inputs, each into its own verdict and flag row, then runs host-path begin / finish on
    its contexts.  Every row equals what that call's own inputs give"""
    import torch
    import bulletproofs_b200 as bp
    og = rp_work[0]
    n, m, S, R = 64, 1, 4, 6
    variants, vs, plen = _variants(orc, og, rp_work, count, nb)
    streams = [torch.cuda.Stream() for _ in range(S)]
    ctxs = [bp.Context(0, stream=s.cuda_stream) for s in streams]
    gens = [bp.Gens(ctxs[0], n, m)]
    _, table_bytes = gens[0].device_table()
    table = torch.empty(table_bytes, dtype=torch.uint8, device="cuda")
    gens[0].table_export(table.data_ptr())
    for c in ctxs[1:]:
        g = bp.Gens(c, n, m, empty=True); g.table_import(table.data_ptr()); gens.append(g)
    assert gens[3].G(0, 5) == orc.gens_get(og, 0, 0, 5) and gens[2].B_blinding == orc.pedersen()[1]
    t = bp.Transcript(LABEL)
    ver = [bp.BatchVerifier(ctxs[k], gens[k], t, n, m, count, nb, reserve=(k % 2 == 0)) for k in range(S)]
    d_in = [torch.frombuffer(bytearray(v[1]), dtype=torch.uint8).cuda() for v in variants]
    h_in = [torch.frombuffer(bytearray(v[1]), dtype=torch.uint8).pin_memory() for v in variants]
    d_vs = torch.frombuffer(bytearray(vs), dtype=torch.uint8).cuda(); h_vs = torch.frombuffer(bytearray(vs), dtype=torch.uint8).pin_memory()
    d_verd = torch.full((S, R, count * nb), 77, dtype=torch.int32, device="cuda")
    h_ok = torch.full((S, R, nb), 9, dtype=torch.int32).pin_memory()
    torch.cuda.synchronize()
    pick = lambda k, r: (r * S + k) % len(variants)                                # noqa: E731
    host_runs = lambda k: [0, 1 + k % nb, len(variants) - 1]                        # noqa: E731
    host_got, errors = {}, []

    def drive(th):
        try:
            mine = (2 * th, 2 * th + 1)                                           # one reserved, one unreserved context
            for r in range(R):
                for k in mine:
                    ver[k].run_device(d_in[pick(k, r)].data_ptr(), d_vs.data_ptr(), d_verd[k, r].data_ptr(), h_ok[k, r].data_ptr(), bytes([16 * k + r]) * 32)
            for k in mine:
                for v in host_runs(k):
                    ver[k].begin(h_in[v].data_ptr(), h_vs.data_ptr(), bytes([v]) * 32)
                    host_got[(k, v)] = (list(ver[k].finish()), ver[k].batch_ok)
        except Exception as e:          # re-raised in the main thread
            errors.append(e)

    threads = [threading.Thread(target=drive, args=(th,)) for th in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    for c in ctxs:
        c.synchronize()
    try:
        assert not errors, errors
        got_v, got_ok = d_verd.cpu().tolist(), h_ok.tolist()
        for k in range(S):
            for r in range(R):
                name, _, want, failing = variants[pick(k, r)]
                ok_want, dev_want = _expected(want, count, nb, failing)
                assert got_v[k][r] == dev_want, (k, r, name, [i for i, (g, w) in enumerate(zip(got_v[k][r], dev_want)) if g != w][:10])
                assert got_ok[k][r] == ok_want, (k, r, name, got_ok[k][r])
            for v in host_runs(k):
                name, _, want, _ = variants[v]
                assert host_got[(k, v)] == (want, _expected(want, count, nb, set())[0]), (k, name)
    finally:
        for g in gens:
            g.close()
        for c in ctxs:
            c.close()


# ------------------------------------------------------------------------------------------------ 5. profiled verification
def test_profiled_verification_matches_unprofiled(orc, rp_work):
    """With bp_prof_enable on, the verifier runs direct launches with the decompression on the main stream instead of its graph: a
    passing and a failing group give the same verdicts and flags as without profiling, through the device and the host entry points.
    The profile counts the decompression, transcript and bucket-accumulation kernels; once profiling is off again a call costs the
    launches of a graph call made before profiling"""
    import torch
    import bulletproofs_b200 as bp
    og = rp_work[0]
    n, m, count, nb = 64, 1, 24, 4
    variants, vs, plen = _variants(orc, og, rp_work, count, nb)
    cases = [variants[0], variants[2]]                                   # passing; batch 1 fails
    ctx = bp.Context(0); gens = bp.Gens(ctx, n, m)
    ver = bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), n, m, count, nb)      # reserved: unprofiled calls replay the graph
    d_in = [torch.frombuffer(bytearray(v[1]), dtype=torch.uint8).cuda() for v in cases]
    d_vs = torch.frombuffer(bytearray(vs), dtype=torch.uint8).cuda()
    d_verd = torch.full((count * nb,), 77, dtype=torch.int32, device="cuda"); h_ok = torch.full((nb,), 9, dtype=torch.int32).pin_memory()
    torch.cuda.synchronize()
    seed = bytes([5]) * 32

    def run(i):
        d_verd.fill_(77); torch.cuda.synchronize()
        l0 = ctx.launches
        ver.run_device(d_in[i].data_ptr(), d_vs.data_ptr(), d_verd.data_ptr(), h_ok.data_ptr(), seed)
        dl = ctx.launches - l0
        ctx.synchronize()
        got, ok = bp.verify_group(ctx, gens, bp.Transcript(LABEL), cases[i][1], vs, n, m, count, nb, seed=seed)
        return (d_verd.cpu().tolist(), h_ok.tolist(), got, ok), dl

    plain = [run(i) for i in range(2)]
    for i, (name, _, want, failing) in enumerate(cases):
        ok_want, dev_want = _expected(want, count, nb, failing)
        assert plain[i][0] == (dev_want, ok_want, want, ok_want), name
    ctx.prof_enable(True)
    profiled = [run(i) for i in range(2)]
    prof = ctx.prof_report()
    ctx.prof_enable(False)
    assert [p[0] for p in profiled] == [p[0] for p in plain]
    for k in ("k_rp_decompress", "k_rp_transcript", "k_msm_accumulate"):
        assert prof.get(k, (0, 0))[1] >= 4, (k, prof.get(k))                # two device and two host calls, each launched directly
    after = [run(i) for i in range(2)]
    assert [a[0] for a in after] == [p[0] for p in plain]
    assert [a[1] for a in after] == [p[1] for p in plain], "after profiling, a call no longer costs what a graph call cost before it"
    gens.close(); ctx.close()
