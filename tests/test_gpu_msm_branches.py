"""GPU tier (-m gpu): branches of the Pippenger pipeline that random MSMs of the usual sizes never take, each against the oracle's MSM.
Every test first shows that its inputs reach its branch, with the selection rules of csrc/msm_common.cuh (built for the host into
tests/host_emul) and bucket sizes from the kernels' own signed-digit recoding, so that a later change of a threshold makes the test
fail loudly instead of quietly testing something else."""
import ctypes
import os
import random

import pytest

from oracle_binding import L_ORDER as l

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def le(x, n=32):
    return x.to_bytes(n, "little")


@pytest.fixture(scope="module")
def E(built):
    E = ctypes.CDLL(os.path.join(ROOT, "tests", "host_emul", "libemul.so"))
    E.emul_pick_window.argtypes = [ctypes.c_uint64]
    E.emul_avg_terms.argtypes = [ctypes.c_uint64, ctypes.c_uint32]; E.emul_avg_terms.restype = ctypes.c_uint64
    E.emul_heavy_min.argtypes = [ctypes.c_uint64, ctypes.c_uint32]; E.emul_heavy_min.restype = ctypes.c_uint32
    E.emul_acc_split.argtypes = [ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint64]
    E.emul_use_combine4.argtypes = [ctypes.c_uint32]
    return E


def _plan(E, T, n_msm):
    """window, windows, buckets per window, heavy threshold and accumulate split of an automatic-window pass over T terms in n_msm MSMs"""
    avg = E.emul_avg_terms(T, n_msm)
    c = E.emul_pick_window(avg); W = E.emul_num_windows(c); nb = 1 << (c - 1)
    return c, W, nb, E.emul_heavy_min(avg, nb), E.emul_acc_split(avg, nb, n_msm * W * nb)


def _bucket_sizes(E, scalars, c, W):
    counts = (ctypes.c_uint32 * (W << (c - 1)))()
    assert E.emul_bucket_counts(scalars, len(scalars) // 32, c, counts) == 0
    return list(counts)


def _check_batch(ctx, orc, sc, pp, offsets):
    """every MSM of the batch == the oracle's; one the oracle rejects (an undecodable point) must have status ERR_INVALID_POINT"""
    import bulletproofs_b200 as bp
    status, outs = ctx.msm_batch(sc, pp, offsets)
    for j in range(len(offsets) - 1):
        a, b = offsets[j], offsets[j + 1]
        rc, want = orc.msm(sc[32 * a:32 * b], pp[32 * a:32 * b])
        assert (status[j], outs[j]) == ((bp.ERR_INVALID_POINT, outs[j]) if rc else (bp.OK, want)), j
    return status


@pytest.mark.parametrize("n_msm", [256, 257, 1000])
def test_msm_batch_beyond_256_msms(gpu_ctx, orc, E, n_msm):
    """More than 256 MSMs in one call combine their windows with k_msm_combine (one thread per MSM) instead of k_msm_combine4; exactly
    256 is the last count on the four-lane kernel.  Ragged sizes, empty MSMs, and an invalid point that poisons only its own MSM."""
    assert E.emul_use_combine4(n_msm) == (n_msm <= 256), "the combine4 limit moved: update the MSM counts of this test"
    assert E.emul_use_combine4(256) == 1 and E.emul_use_combine4(257) == 0
    rnd = random.Random(n_msm)
    base = [orc.from_uniform(rnd.randbytes(64)) for _ in range(48)]
    sizes = [rnd.choice([0, 1, 2, 3, 5, 8, 13, 40]) for _ in range(n_msm)]
    sizes[0], sizes[-1], sizes[n_msm // 2] = 0, 150, 0
    offsets = [0]
    for s in sizes:
        offsets.append(offsets[-1] + s)
    T = offsets[-1]
    sc = b"".join(le(rnd.randrange(l)) for _ in range(T)); pp = bytearray(b"".join(rnd.choice(base) for _ in range(T)))
    bad = next(j for j in range(n_msm // 3, n_msm) if sizes[j] >= 5)
    t = offsets[bad] + sizes[bad] // 2
    pp[32 * t:32 * t + 32] = b"\x01" + bytes(31)
    status = _check_batch(gpu_ctx, orc, sc, bytes(pp), offsets)
    assert [j for j, s in enumerate(status) if s] == [bad]


@pytest.mark.parametrize("n_msm", [8, 300])
def test_heavy_list_longer_than_the_heavy_grid(gpu_ctx, orc, E, n_msm):
    """MSMs of ~300 terms with one scalar repeated 280 times: one heavy bucket per (MSM, non-zero window), thousands in all, spread over
    many MSMs.  k_msm_accumulate has at most one heavy block per SM, so each heavy block walks the heavy list with a grid stride.
    With 8 MSMs the light buckets take the two-lane accumulate (SPLIT = 2) in the same launch."""
    import torch
    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    rnd = random.Random(500 + n_msm)
    base = [orc.from_uniform(rnd.randbytes(64)) for _ in range(64)]
    sc, offsets = b"", [0]
    for _ in range(n_msm):
        k = rnd.randrange(290, 311)
        terms = [le(rnd.randrange(l))] * 280 + [le(rnd.randrange(l)) for _ in range(k - 280)]
        rnd.shuffle(terms)
        sc += b"".join(terms); offsets.append(offsets[-1] + k)
    T = offsets[-1]
    c, W, nb, heavy_min, split = _plan(E, T, n_msm)
    n_heavy = sum(sum(1 for v in _bucket_sizes(E, sc[32 * offsets[j]:32 * offsets[j + 1]], c, W) if v >= heavy_min) for j in range(n_msm))
    assert n_heavy > sm_count, f"{n_heavy} heavy buckets (threshold {heavy_min}) fit in the {sm_count} heavy blocks: no grid-stride loop"
    if n_msm == 8:
        assert split == 2, "the light buckets no longer take the two-lane accumulate"
    pp = b"".join(rnd.choice(base) for _ in range(T))
    assert _check_batch(gpu_ctx, orc, sc, pp, offsets) == [0] * n_msm


def test_indexed_msm_undecodable_dynamic_point(gpu_ctx, orc):
    """bp_msm_indexed_batch over generator-table slots and dynamic points, one of which does not decode: it poisons exactly the MSMs
    that use it (ERR_INVALID_POINT), a non-canonical scalar in the same MSM takes precedence (ERR_NONCANONICAL_SCALAR), the MSM between
    them is exact, and a null status array leaves the outputs unchanged."""
    import bulletproofs_b200 as bp
    cap, D = 16, 0x80000000
    gens = bp.Gens(gpu_ctx, cap, 1); og = orc.gens(cap, 1)
    rnd = random.Random(77)
    dyn = [orc.from_uniform(rnd.randbytes(64)), b"\x01" + bytes(31), orc.from_uniform(rnd.randbytes(64))]
    assert [orc.point_is_valid(q) for q in dyn] == [1, 0, 1]
    G = lambda i: 2 + i; H = lambda i: 2 + cap + i
    idx = [G(3), D | 1, D | 0, H(5),          # (a) the undecodable point
           G(1), D | 0, H(2), D | 2, 1,       # (c) valid dynamic points only, and B
           D | 1, H(7), G(9)]                 # (b) the undecodable point and a non-canonical scalar
    offsets = [0, 4, 9, 12]
    sc = [le(rnd.randrange(l)) for _ in idx]
    sc[10] = le(l)
    scalars = b"".join(sc)

    def call(status):
        outs = ctypes.create_string_buffer(32 * 3)
        rc = bp.lib().bp_msm_indexed_batch(gpu_ctx._h, gens._h, scalars, (ctypes.c_uint32 * len(idx))(*idx), b"".join(dyn), len(dyn),
                                           (ctypes.c_uint64 * 4)(*offsets), 3, outs, status)
        gpu_ctx._check(rc)
        return outs.raw

    st = ctypes.create_string_buffer(3)
    outs = call(st)
    assert list(st.raw) == [bp.ERR_INVALID_POINT, bp.OK, bp.ERR_NONCANONICAL_SCALAR]
    pts = orc.gens_get(og, 0, 0, 1) + dyn[0] + orc.gens_get(og, 1, 0, 2) + dyn[2] + orc.pedersen()[0]
    assert (0, outs[32:64]) == orc.msm(b"".join(sc[4:9]), pts)
    assert call(None) == outs
    gens.close()


def test_heavy_threshold_edge(gpu_ctx, orc, E):
    """One MSM of 2000 terms (two-lane accumulate) with buckets of exactly heavy_min and heavy_min - 1 entries: k_msm_order lists a
    bucket for the heavy blocks and k_msm_accumulate leaves it to them on the same condition (size >= heavy_min), so the first is
    summed by a heavy block, the second by light lanes, and neither is summed twice or not at all."""
    rnd = random.Random(2000)
    T = 2000
    c, W, nb, heavy_min, split = _plan(E, T, 1)
    assert split == 2, "2000 terms no longer select the two-lane accumulate"
    s1, s2 = le(rnd.randrange(l)), le(rnd.randrange(l))
    terms = [s1] * heavy_min + [s2] * (heavy_min - 1) + [le(rnd.randrange(l)) for _ in range(40)]
    terms += [le(0)] * (T - len(terms))
    rnd.shuffle(terms)
    sc = b"".join(terms)
    sizes = _bucket_sizes(E, sc, c, W)
    assert heavy_min in sizes and heavy_min - 1 in sizes, (heavy_min, sorted(sizes)[-8:])
    base = [orc.from_uniform(rnd.randbytes(64)) for _ in range(64)]
    pp = b"".join(rnd.choice(base) for _ in range(T))
    assert gpu_ctx.msm(sc, pp) == orc.msm(sc, pp)
