"""GPU tier: the fused single-proof path of bp_rangeproof_verify_batch (k_rp_single, one thread-block cluster per proof, one launch).

Calls of at most ROUTE_COUNT proofs with lg(n m) <= ROUTE_K take it; every verdict must equal the oracle's per-proof verify_multiple and
what verify_group(count, 1) -- the launch-group pipeline in the same build -- returns on the same bytes."""
import ctypes
import random
import threading

import pytest

from oracle_binding import L_ORDER as l

pytestmark = pytest.mark.gpu

LABEL = b"single proof"
ROUTE_COUNT, ROUTE_K = 8, 6            # RP_ROUTE_MAX_COUNT, RP_ROUTE_MAX_K (bpmsm.cu)
ROUTED = [(8, 1), (16, 1), (32, 1), (64, 1), (8, 2), (16, 2), (32, 2), (16, 4), (8, 8)]
_W = {}


def le(x, n=32):
    return x.to_bytes(n, "little")


def lg(x):
    return x.bit_length() - 1


def work(orc, n, m, count, label=LABEL):
    """`count` valid oracle proofs at (n, m) under `label`, their commitments and the oracle's generators"""
    key = (n, m, count, label)
    if key not in _W:
        rnd = random.Random(1000 * n + m + count)
        og = orc.gens(n, m)
        vals = [rnd.randrange(1 << n) for _ in range(count * m)]
        blind = b"".join(le(rnd.randrange(l)) for _ in range(count * m))
        seeds = b"".join(le(i + 17, 8) + bytes(24) for i in range(count))
        proofs, Vs = orc.prove_many(og, orc.transcript(label), vals, blind, n, m, seeds, nthreads=8)
        _W[key] = (og, proofs, Vs)
    return _W[key]


def damaged(proof, n, m, V, rnd):
    """(proof, commitments) variants: one-bit damage in every proof field, a wrong commitment, non-canonical scalars and an undecodable
    encoding at every point position"""
    k = lg(n * m)
    fields = [0, 32, 64, 96, 128, 160, 192] + [224 + 32 * j for j in range(2 * k)] + [224 + 64 * k, 256 + 64 * k]
    out = []
    for off in fields:
        b = bytearray(proof); b[off + rnd.randrange(31)] ^= 1 << rnd.randrange(8); out.append((bytes(b), V))
    w = bytearray(V); w[32 * rnd.randrange(m)] ^= 2; out.append((proof, bytes(w)))
    for off in (128, 160, 192, 224 + 64 * k, 256 + 64 * k):          # scalar + l: same value mod l, not canonical
        s = int.from_bytes(proof[off:off + 32], "little") + l
        if s < 1 << 256:
            b = bytearray(proof); b[off:off + 32] = le(s); out.append((bytes(b), V))
    for off in [0, 32, 64, 96] + [224 + 32 * j for j in range(2 * k)]:
        b = bytearray(proof); b[off:off + 32] = b"\xff" * 32; out.append((bytes(b), V))      # s >= p: no point
    w = bytearray(V); w[0:32] = b"\xee" * 32; out.append((proof, bytes(w)))
    return out


def three_ways(bp, orc, ctx, gens, og, proofs, Vs, n, m, count, seed=None, t=None, ot=None):
    t = t or bp.Transcript(LABEL)
    ot = ot or orc.transcript(LABEL)
    plen = len(proofs) // count
    want = orc.verify_many(og, ot, proofs, plen, Vs, n, m, count)
    l0 = ctx.launches
    got = bp.verify_batch(ctx, gens, t, proofs, Vs, n, m, count, seed=seed)
    launches = ctx.launches - l0
    pipe, _ = bp.verify_group(ctx, gens, t, proofs, Vs, n, m, count, 1, seed=seed)
    return want, got, pipe, launches


@pytest.fixture(scope="module")
def gens_for(gpu_ctx):
    import bulletproofs_b200 as bp
    made = {}

    def get(n, m):
        if (n, m) not in made:
            made[(n, m)] = bp.Gens(gpu_ctx, n, m)
        return made[(n, m)]
    yield get
    for g in made.values():
        g.close()


@pytest.mark.parametrize("n,m", ROUTED)
def test_routed_geometry_matches_oracle_and_pipeline(gpu_ctx, orc, gens_for, n, m):
    import bulletproofs_b200 as bp
    og, proofs, Vs = work(orc, n, m, 1)
    rnd = random.Random(n * 131 + m)
    cases = [(proofs, Vs)] + damaged(proofs, n, m, Vs, rnd)
    for pb, vb in cases:
        want, got, pipe, launches = three_ways(bp, orc, gpu_ctx, gens_for(n, m), og, pb, vb, n, m, 1, seed=bytes([5]) * 32)
        assert got == want == pipe, (got, want, pipe)
        assert launches == 1
    assert orc.verify_many(og, orc.transcript(LABEL), proofs, len(proofs), Vs, n, m, 1) == [0]


@pytest.mark.parametrize("n,m", [(64, 1), (16, 4), (8, 8)])
def test_routed_counts_with_damage_in_every_slot(gpu_ctx, orc, gens_for, n, m):
    import bulletproofs_b200 as bp
    count = ROUTE_COUNT
    og, proofs, Vs = work(orc, n, m, count)
    plen, rnd = len(proofs) // count, random.Random(7 * n + m)
    for q in range(count):
        pb = bytearray(proofs)
        pb[q * plen + rnd.randrange(plen - 64)] ^= 1 << rnd.randrange(8)
        want, got, pipe, launches = three_ways(bp, orc, gpu_ctx, gens_for(n, m), og, bytes(pb), Vs, n, m, count)
        assert got == want == pipe and want[q] != 0 and launches == 1


def test_routing_edges(gpu_ctx, orc, gens_for):
    """C_max is routed (one launch) and C_max + 1 is not; lg(nm) = K_max is routed and K_max + 1 is not.  Same verdicts either way."""
    import bulletproofs_b200 as bp
    for (n, m, count, routed) in [(64, 1, ROUTE_COUNT, True), (64, 1, ROUTE_COUNT + 1, False), (64, 1 << (ROUTE_K - 6), 2, True),
                                  (64, 1 << (ROUTE_K - 5), 2, False), (8, 1 << (ROUTE_K - 3), 1, True), (8, 1 << (ROUTE_K - 2), 1, False)]:
        og, proofs, Vs = work(orc, n, m, count)
        plen = len(proofs) // count
        for q in range(count):
            pb = bytearray(proofs); pb[q * plen + 130] ^= 4
            want, got, pipe, launches = three_ways(bp, orc, gpu_ctx, gens_for(n, m), og, bytes(pb), Vs, n, m, count)
            assert got == want == pipe, (n, m, count, q)
            assert (launches == 1) == routed, (n, m, count, launches)


def test_seeds_and_parameter_errors(gpu_ctx, orc, gens_for):
    import bulletproofs_b200 as bp
    n, m = 32, 2
    og, proofs, Vs = work(orc, n, m, 4)
    pb = bytearray(proofs); pb[len(proofs) // 4 * 2 + 40] ^= 8
    gens = gens_for(n, m)
    first = None
    for seed in (bytes(32), bytes([0x5A]) * 32, None, None):
        got = bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), bytes(pb), Vs, n, m, 4, seed=seed)
        first = first or got
        assert got == first == [0, 0, 1, 0]
    # parameter verdicts are decided before routing, as before: wrong n for the length, too few generators
    assert bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), proofs, Vs, 16, m, 4) == [1] * 4
    small = gens_for(8, 1)
    assert bp.verify_batch(gpu_ctx, small, bp.Transcript(LABEL), proofs, Vs, n, m, 4) == [4] * 4
    with pytest.raises(bp.BpError):
        bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), proofs, Vs, n, m, 4, proof_len=len(proofs) // 4 - 1)


def test_transcript_with_earlier_messages(gpu_ctx, orc, gens_for):
    """a proof made under a transcript that absorbed a message verifies under that transcript and not under a fresh one"""
    import bulletproofs_b200 as bp
    n, m = 64, 1
    og = orc.gens(n, m)
    ot = orc.transcript_append(orc.transcript(LABEL), b"tx", b"hash of the transaction")
    rnd = random.Random(3)
    rc, proof, V = orc.rangeproof_prove(og, ot, [rnd.randrange(1 << n)], le(rnd.randrange(l)), n, seed=le(99))
    assert rc == 0
    t = bp.Transcript(LABEL); t.append_message(b"tx", b"hash of the transaction")
    assert bp.verify_batch(gpu_ctx, gens_for(n, m), t, proof, V, n, m, 1) == [0]
    assert bp.verify_batch(gpu_ctx, gens_for(n, m), bp.Transcript(LABEL), proof, V, n, m, 1) == [1]


@pytest.mark.parametrize("kind", ["a+-d", "a triple"])
def test_cancelling_sets_rejected_per_proof(gpu_ctx, orc, kind):
    """the cancelling constructions of test_batch_soundness, in a routed call of ROUTE_COUNT proofs"""
    import bulletproofs_b200 as bp
    from test_batch_soundness import rp_inputs, LABEL as SL
    n, m = 64, 1
    placed = (1, 4, 6) if kind == "a triple" else (2, 5)
    og, P, V, members, off, pb, vb, plen, want = rp_inputs(orc, n, m, ROUTE_COUNT, placed, kind=kind)
    gens = bp.Gens(gpu_ctx, n, m)
    l0 = gpu_ctx.launches
    got = bp.verify_batch(gpu_ctx, gens, bp.Transcript(SL), pb, vb, n, m, ROUTE_COUNT, seed=bytes(32))
    assert gpu_ctx.launches - l0 == 1
    assert got == want
    gens.close()


def test_reserved_graphs_keep_replaying(orc):
    """a reserved BatchVerifier and a reserved mix on the context replay their graphs at the same launch cost after routed calls"""
    import bulletproofs_b200 as bp
    ctx = bp.Context(0)
    try:
        gens = bp.Gens(ctx, 64, 4)
        og, proofs, Vs = work(orc, 64, 1, 16)
        bv = bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), 64, 1, 16)
        mix = bp.MixedVerifier(ctx, gens, {(64, 1): 4, (32, 2): 2})
        pbuf, vbuf = ctypes.create_string_buffer(proofs, len(proofs)), ctypes.create_string_buffer(Vs, len(Vs))
        items = [(proofs[672 * i:672 * (i + 1)], Vs[32 * i:32 * (i + 1)], 64) for i in range(4)]

        def batch():
            l0 = ctx.launches
            bv.begin(ctypes.addressof(pbuf), ctypes.addressof(vbuf), seed=bytes(32))
            v = bv.finish()
            return list(v), ctx.launches - l0

        def mixed():
            l0 = ctx.launches
            mix.begin(bp.Transcript(LABEL), items, seed=bytes(32))
            return mix.finish(), ctx.launches - l0

        b0, m0 = batch(), mixed()
        assert b0[0] == [0] * 16 and m0[0] == [0] * 4
        for _ in range(3):
            assert bp.verify_batch(ctx, gens, bp.Transcript(LABEL), proofs[:672 * 2], Vs[:64], 64, 1, 2) == [0, 0]
            assert batch() == b0 and mixed() == m0
        gens.close()
    finally:
        ctx.close()


def test_pending_begin_refuses_routed_calls(gpu_ctx, orc, gens_for):
    import bulletproofs_b200 as bp
    og, proofs, Vs = work(orc, 64, 1, 2)
    gens = gens_for(64, 1)
    pbuf, vbuf = ctypes.create_string_buffer(proofs, len(proofs)), ctypes.create_string_buffer(Vs, len(Vs))
    bv = bp.BatchVerifier(gpu_ctx, gens, bp.Transcript(LABEL), 64, 1, 2, reserve=False)
    bv.begin(ctypes.addressof(pbuf), ctypes.addressof(vbuf))
    with pytest.raises(bp.BpError):
        bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), proofs[:672], Vs[:32], 64, 1, 1)
    assert list(bv.finish()) == [0, 0]
    assert bp.verify_batch(gpu_ctx, gens, bp.Transcript(LABEL), proofs[:672], Vs[:32], 64, 1, 1) == [0]


def test_two_contexts_two_threads(orc):
    import bulletproofs_b200 as bp
    og, proofs, Vs = work(orc, 16, 4, 4)
    plen = len(proofs) // 4
    bad = bytearray(proofs); bad[plen + 10] ^= 1
    want = orc.verify_many(og, orc.transcript(LABEL), bytes(bad), plen, Vs, 16, 4, 4)
    errors = []

    def run(i):
        try:
            ctx = bp.Context(0); gens = bp.Gens(ctx, 16, 4)
            for r in range(20):
                got = bp.verify_batch(ctx, gens, bp.Transcript(LABEL), bytes(bad), Vs, 16, 4, 4, seed=bytes([i, r]) * 16)
                assert got == want, got
            gens.close(); ctx.close()
        except Exception as e:          # noqa: BLE001 - reported by the main thread
            errors.append(e)
    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors


def test_debug_hook_verifies_beyond_the_routing_rule(gpu_ctx, orc, gens_for):
    """the fused kernel at geometries and counts the rule leaves to the pipeline (the benchmark times it there) gives the same verdicts"""
    import bulletproofs_b200 as bp
    for n, m, count in [(64, 16, 2), (8, 128, 1), (64, 1, 24)]:
        og, proofs, Vs = work(orc, n, m, count)
        plen = len(proofs) // count
        pb = bytearray(proofs); pb[(count - 1) * plen + 150] ^= 2
        want = orc.verify_many(og, orc.transcript(LABEL), bytes(pb), plen, Vs, n, m, count)
        out = ctypes.create_string_buffer(count)
        gpu_ctx._check(bp.lib().bp_debug_rp_single_verify(gpu_ctx._h, gens_for(n, m)._h, bp.Transcript(LABEL).to_bytes(), bytes(pb), plen, Vs, n, m, count,
                                                            None, out))
        assert list(out.raw) == want
