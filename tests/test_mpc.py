"""Aggregated range-proof MPC API (src/range_proof/{party,dealer,messages}.rs): the oracle's restatement checks itself against
the golden-pinned prover/verifier on the CPU tier; on the GPU tier the host mirror (bulletproofs_b200/host/mpc.cpp, every point
operation on the device) must produce the oracle's bytes and verdicts, including the dealer's share audit
(ProofShare::audit_share, messages.rs:84-167).  Mirrors the reference's tests create_and_verify_n_*_m_*,
detect_dishonest_party_during_aggregation and detect_dishonest_dealer_during_aggregation (src/range_proof/mod.rs)."""
import random

import pytest

from oracle_binding import L_ORDER

LABEL = b"AggregatedRangeProofTest"


def le(x):
    return x.to_bytes(32, "little")


def witness(n, m, seed, values=None):
    rnd = random.Random(seed)
    vs = values or [rnd.randrange(1 << n) for _ in range(m)]
    return vs, [le(rnd.randrange(L_ORDER)) for _ in range(m)], [rnd.randbytes(32) for _ in range(m)]


def oracle_run(orc, g, n, m, vs, bls, seeds, tamper=None):
    """the three rounds through the oracle; returns every message"""
    t0 = orc.transcript(LABEL)
    bitc = b"".join(orc.mpc_bit_commitment(g, vs[j], bls[j], n, j, seeds[j])[1] for j in range(m))
    rc, t1, y, z = orc.mpc_bit_challenge(g, t0, n, m, bitc)
    assert rc == 0
    polyc = b"".join(orc.mpc_poly_commitment(g, vs[j], n, j, seeds[j], y, z)[1] for j in range(m))
    rc, t2, x = orc.mpc_poly_challenge(t1, m, polyc)
    assert rc == 0
    shares = b"".join(orc.mpc_proof_share(g, vs[j], bls[j], n, j, seeds[j], y, z, x)[1] for j in range(m))
    if tamper:
        shares = tamper(shares)
    return t0, bitc, polyc, shares, (y, z, x)


def test_oracle_single_party_equals_prove_multiple(orc):
    # with m = 1 the party's RNG stream is prove_multiple's stream: the MPC path must give the golden-pinned prover's bytes
    n, m = 32, 1
    g = orc.gens(n, m)
    vs, bls, seeds = witness(n, m, 1)
    t0, bitc, polyc, shares, _ = oracle_run(orc, g, n, m, vs, bls, seeds)
    rc, proof, bad = orc.mpc_dealer_run(g, t0, n, m, bitc, polyc, shares)
    rc2, want, V = orc.rangeproof_prove(g, t0, vs, bls[0], n, seeds[0])
    assert (rc, rc2, bad) == (0, 0, [0]) and proof == want and bitc[:32] == V


@pytest.mark.parametrize("n,m", [(8, 2), (32, 4), (64, 8)])
def test_oracle_aggregation_verifies_and_audits_clean(orc, n, m):
    g = orc.gens(n, m)
    vs, bls, seeds = witness(n, m, 10 * n + m)
    t0, bitc, polyc, shares, (y, z, x) = oracle_run(orc, g, n, m, vs, bls, seeds)
    rc, proof, bad = orc.mpc_dealer_run(g, t0, n, m, bitc, polyc, shares)
    assert rc == 0 and not any(bad)
    Vs = b"".join(bitc[96 * j:96 * j + 32] for j in range(m))
    assert orc.rangeproof_verify(g, t0, proof, Vs, m, n) == 0
    sl = 32 * (3 + 2 * n)
    for j in range(m):
        assert orc.mpc_audit_share(g, n, j, bitc[96 * j:96 * j + 96], y, z, polyc[64 * j:64 * j + 64], x, shares[sl * j:sl * j + sl]) == 0
    rc, trusted, _ = orc.mpc_dealer_run(g, t0, n, m, bitc, polyc, shares, trusted=True)
    assert rc == 0 and trusted == proof


def test_oracle_detects_dishonest_party(orc):
    # mod.rs test detect_dishonest_party_during_aggregation: party 1 commits to u32::MAX + 1 with n = 32
    n, m = 32, 2
    g = orc.gens(n, m)
    vs, bls, seeds = witness(n, m, 5, values=[1234567, (1 << 32)])
    t0, bitc, polyc, shares, _ = oracle_run(orc, g, n, m, vs, bls, seeds)
    rc, _, bad = orc.mpc_dealer_run(g, t0, n, m, bitc, polyc, shares)
    assert rc == 10 and bad == [0, 1]                      # MPCError::MalformedProofShares { bad_shares: [1] }
    rc, proof, _ = orc.mpc_dealer_run(g, t0, n, m, bitc, polyc, shares, trusted=True)      # receive_trusted_shares does not look
    assert rc == 0 and orc.rangeproof_verify(g, t0, proof, bitc[:32] + bitc[96:128], m, n) == 1


def test_oracle_detects_dishonest_dealer_and_parameter_errors(orc):
    n, m = 32, 2
    g = orc.gens(n, m)
    vs, bls, seeds = witness(n, m, 6)
    y, z = le(7), le(9)
    assert orc.mpc_proof_share(g, vs[0], bls[0], n, 0, seeds[0], y, z, le(0))[0] == 8       # MaliciousDealer (party.rs:282-284)
    assert orc.mpc_bit_commitment(g, 1, bls[0], 10, 0, seeds[0])[0] == 3                     # InvalidBitsize
    assert orc.mpc_bit_commitment(g, 1, bls[0], 64, 0, seeds[0])[0] == 4                     # gens_capacity < n
    assert orc.mpc_bit_commitment(g, 1, bls[0], n, 2, seeds[0])[0] == 4                      # party_capacity <= j
    bitc = b"".join(orc.mpc_bit_commitment(g, vs[j], bls[j], n, j, seeds[j])[1] for j in range(m))
    t0 = orc.transcript(LABEL)
    assert orc.mpc_bit_challenge(orc.gens(n, 4), t0, n, 3, bitc + bitc[:96])[0] == 5         # InvalidAggregation
    assert orc.mpc_bit_challenge(g, t0, n, 4, bitc + bitc)[0] == 4                           # party_capacity < m


# ---------------------------------------------------------------------------------------------- GPU tier: host mirror == oracle
def gpu_run(bp, ctx, gens, n, m, vs, bls, seeds):
    t = bp.Transcript(LABEL)
    bitc = b""
    for j in range(m):
        rc, b = bp.mpc_party_bit_commitment(ctx, gens, vs[j], bls[j], n, j, seeds[j])
        assert rc == 0
        bitc += b
    t1 = t.clone()
    rc, _, _, (y, z, _) = bp.mpc_dealer_run(ctx, gens, t1, n, m, bitc)
    assert rc == 0
    polyc = b""
    for j in range(m):
        rc, b = bp.mpc_party_poly_commitment(ctx, gens, vs[j], n, j, seeds[j], y, z)
        assert rc == 0
        polyc += b
    t2 = t.clone()
    rc, _, _, (y2, z2, x) = bp.mpc_dealer_run(ctx, gens, t2, n, m, bitc, polyc)
    assert rc == 0 and (y2, z2) == (y, z)
    shares = b""
    for j in range(m):
        rc, b = bp.mpc_party_proof_share(ctx, gens, vs[j], bls[j], n, j, seeds[j], y, z, x)
        assert rc == 0
        shares += b
    return t, bitc, polyc, shares, (y, z, x)


@pytest.mark.gpu
@pytest.mark.parametrize("n,m", [(32, 1), (8, 2), (64, 4), (8, 16)])
def test_gpu_mpc_messages_and_proof_match_oracle(gpu_ctx, orc, n, m):
    import bulletproofs_b200 as bp
    g = orc.gens(n, m); gens = bp.Gens(gpu_ctx, n, m)
    vs, bls, seeds = witness(n, m, 100 + n + m)
    t0, bitc, polyc, shares, ch = oracle_run(orc, g, n, m, vs, bls, seeds)
    t, gbitc, gpolyc, gshares, gch = gpu_run(bp, gpu_ctx, gens, n, m, vs, bls, seeds)
    assert (gbitc, gpolyc, gshares, gch) == (bitc, polyc, shares, ch)
    rc, want, bad = orc.mpc_dealer_run(g, t0, n, m, bitc, polyc, shares)
    tf = t.clone()
    grc, proof, gbad, _ = bp.mpc_dealer_run(gpu_ctx, gens, tf, n, m, gbitc, gpolyc, gshares)
    assert (grc, gbad) == (rc, bad) == (0, [0] * m) and proof == want
    Vs = b"".join(bitc[96 * j:96 * j + 32] for j in range(m))
    assert bp.verify_multiple(gpu_ctx, gens, t, proof, Vs, n) == 0
    sl = 32 * (3 + 2 * n)
    for j in range(m):
        assert bp.mpc_audit_share(gpu_ctx, gens, n, j, bitc[96 * j:96 * j + 96], ch[0], ch[1], polyc[64 * j:64 * j + 64], ch[2], shares[sl * j:sl * j + sl]) == 0
    gens.close()


@pytest.mark.gpu
def test_gpu_mpc_detects_dishonest_party_like_oracle(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    n, m = 32, 4
    g = orc.gens(n, m); gens = bp.Gens(gpu_ctx, n, m)
    vs, bls, seeds = witness(n, m, 77, values=[5, (1 << 32), 99, (1 << 40) + 3])
    t0, bitc, polyc, shares, ch = oracle_run(orc, g, n, m, vs, bls, seeds)
    rc, _, bad = orc.mpc_dealer_run(g, t0, n, m, bitc, polyc, shares)
    t = bp.Transcript(LABEL)
    grc, proof, gbad, _ = bp.mpc_dealer_run(gpu_ctx, gens, t, n, m, bitc, polyc, shares)
    assert (grc, gbad) == (rc, bad) == (bp.MPC_MALFORMED_PROOF_SHARES, [0, 1, 0, 1]) and proof is None
    # a share damaged in transit (one bit of r_vec), a non-canonical scalar, an undecodable T_1_j: audit verdicts equal the oracle's
    sl = 32 * (3 + 2 * n)
    vs2, bls2, seeds2 = witness(n, m, 78)
    t0, bitc, polyc, shares, (y, z, x) = oracle_run(orc, g, n, m, vs2, bls2, seeds2)
    for j, mutate in ((2, lambda s: s[:96 + 32 * n + 7] + bytes([s[96 + 32 * n + 7] ^ 4]) + s[96 + 32 * n + 8:]), (0, lambda s: b"\xff" * 32 + s[32:])):
        sh = bytearray(shares); sh[sl * j:sl * j + sl] = mutate(shares[sl * j:sl * j + sl]); sh = bytes(sh)
        rc, _, bad = orc.mpc_dealer_run(g, t0, n, m, bitc, polyc, sh)
        grc, _, gbad, _ = bp.mpc_dealer_run(gpu_ctx, gens, bp.Transcript(LABEL), n, m, bitc, polyc, sh)
        assert (grc, gbad) == (rc, bad) and bad[j] == 1 and sum(bad) == 1
    bad_poly = bytearray(polyc); bad_poly[64:96] = b"\x01" + bytes(31)        # not a Ristretto encoding
    args = (n, 1, bitc[96:192], y, z, bytes(bad_poly[64:128]), x, shares[sl:2 * sl])
    assert bp.mpc_audit_share(gpu_ctx, gens, *args) == orc.mpc_audit_share(g, *args) == 1
    gens.close()


@pytest.mark.gpu
def test_gpu_mpc_dishonest_dealer_and_parameter_errors(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    n, m = 32, 2
    gens = bp.Gens(gpu_ctx, n, m)
    vs, bls, seeds = witness(n, m, 6)
    assert bp.mpc_party_proof_share(gpu_ctx, gens, vs[0], bls[0], n, 0, seeds[0], le(7), le(9), le(0))[0] == bp.MPC_MALICIOUS_DEALER
    assert bp.mpc_party_bit_commitment(gpu_ctx, gens, 1, bls[0], 10, 0, seeds[0])[0] == bp.MPC_INVALID_BITSIZE
    assert bp.mpc_party_bit_commitment(gpu_ctx, gens, 1, bls[0], 64, 0, seeds[0])[0] == bp.MPC_INVALID_GENERATORS_LENGTH
    assert bp.mpc_party_bit_commitment(gpu_ctx, gens, 1, bls[0], n, 2, seeds[0])[0] == bp.MPC_INVALID_GENERATORS_LENGTH
    bitc = b"".join(bp.mpc_party_bit_commitment(gpu_ctx, gens, vs[j], bls[j], n, j, seeds[j])[1] for j in range(m))
    gens4 = bp.Gens(gpu_ctx, n, 4)
    assert bp.mpc_dealer_run(gpu_ctx, gens4, bp.Transcript(LABEL), n, 3, bitc + bitc[:96])[0] == bp.MPC_INVALID_AGGREGATION
    assert bp.mpc_dealer_run(gpu_ctx, gens, bp.Transcript(LABEL), n, 4, bitc + bitc)[0] == bp.MPC_INVALID_GENERATORS_LENGTH
    gens.close(); gens4.close()
