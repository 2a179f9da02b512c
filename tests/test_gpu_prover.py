"""GPU tier: the prover-side call sites (§8 rows A1, A3, A5) through the C++ mirror of the reference API.
Proof bytes must equal the oracle's for identical values, blindings, RNG stream and transcript (group elements
have one canonical encoding, so bytes are a pure function of those inputs — SURVEY.md §8c)."""
import random

import pytest

from oracle_binding import L_ORDER as l

pytestmark = pytest.mark.gpu


def le(x, n=32):
    return x.to_bytes(n, "little")


@pytest.mark.parametrize("n,m", [(32, 1), (8, 1), (64, 1), (16, 2), (64, 4), (32, 8)] + [(n, m) for m in (16, 32) for n in (8, 16, 32, 64)])
def test_rangeproof_prove_bytes_match_oracle(gpu_ctx, orc, n, m):
    """up to m = 32 parties: N = 2048 generator pairs, an inner-product argument of 11 rounds"""
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 64, max(8, m)); og = orc.gens(64, max(8, m))
    rnd = random.Random(n * 10 + m)
    label = b"AggregateRangeProofBenchmark"                       # benches/range_proof.rs:34
    values = [rnd.randrange(1 << n) for _ in range(m)]
    blind = b"".join(le(rnd.randrange(l)) for _ in range(m))
    seed = bytes([24]) * 32                                        # ChaChaRng::from_seed([24u8; 32]), tests/range_proof.rs:108
    t = bp.Transcript(label)
    rc, proof, V = bp.prove_multiple(gpu_ctx, gens, t, values, blind, n, seed)
    orc_rc, want_proof, want_V = orc.rangeproof_prove(og, orc.transcript(label), values, blind, n, seed=seed)
    assert rc == 0 and orc_rc == 0
    assert V == want_V
    assert proof == want_proof                                     # bit-exact proof bytes (config 1 for n=32, m=1: 608 bytes)
    assert len(proof) == 32 * (9 + 2 * ((n * m).bit_length() - 1))
    # and both verifiers accept it
    assert bp.verify_multiple(gpu_ctx, gens, bp.Transcript(label), proof, V, n) == 0
    assert orc.rangeproof_verify(og, orc.transcript(label), proof, V, m, n) == 0
    bad = bytearray(proof); bad[70] ^= 1
    assert bp.verify_multiple(gpu_ctx, gens, bp.Transcript(label), bytes(bad), V, n) == orc.rangeproof_verify(og, orc.transcript(label), bytes(bad), V, m, n) != 0
    gens.close()


def test_rangeproof_prove_parameter_errors(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 32, 2)
    t = bp.Transcript(b"x"); bl = le(5) * 4; seed = bytes(32)
    assert bp.prove_multiple(gpu_ctx, gens, t, [1], bl[:32], 24, seed)[0] == bp.PROOF_INVALID_BITSIZE
    assert bp.prove_multiple(gpu_ctx, gens, t, [1, 2, 3], bl[:96], 8, seed)[0] == bp.PROOF_INVALID_AGGREGATION
    assert bp.prove_multiple(gpu_ctx, gens, t, [1], bl[:32], 64, seed)[0] == bp.PROOF_INVALID_GENERATORS_LENGTH
    assert bp.prove_multiple(gpu_ctx, gens, t, [1, 2, 3, 4], bl, 8, seed)[0] == bp.PROOF_INVALID_GENERATORS_LENGTH
    # out-of-range value: a proof is produced but must not verify (tests/r1cs.rs-style negative case for range proofs)
    rc, proof, V = bp.prove_multiple(gpu_ctx, gens, bp.Transcript(b"x"), [1 << 9], bl[:32], 8, seed)
    assert rc == 0 and bp.verify_multiple(gpu_ctx, gens, bp.Transcript(b"x"), proof, V, 8) != 0
    gens.close()


@pytest.mark.parametrize("n", [1, 2, 4, 32, 64])
def test_ipp_create_and_verify_match_oracle(gpu_ctx, orc, n):
    """inner_product_proof.rs:433-534: create -> verify; proof bytes equal the oracle's."""
    import bulletproofs_b200 as bp
    rnd = random.Random(50 + n)
    og = orc.gens(64, 1)
    Q = orc.from_uniform(orc.sha3_512(b"test point"))
    G = b"".join(orc.gens_get(og, 0, 0, i) for i in range(n)); H = b"".join(orc.gens_get(og, 1, 0, i) for i in range(n))
    a = [rnd.randrange(l) for _ in range(n)]; b = [rnd.randrange(l) for _ in range(n)]
    y_inv = rnd.randrange(1, l)
    Gf = [1] * n; Hf = [pow(y_inv, i, l) for i in range(n)]
    enc = lambda xs: b"".join(le(x) for x in xs)
    c = sum(x * y for x, y in zip(a, b)) % l
    rc, P = orc.msm(enc(a) + enc([x * h % l for x, h in zip(b, Hf)]) + enc([c]), G + H + Q)
    assert rc == 0
    t = bp.Transcript(b"innerproducttest")
    proof = bp.ipp_create(gpu_ctx, t, Q, enc(Gf), enc(Hf), G, H, enc(a), enc(b))
    orc_rc, orc_t, want = orc.ipp_create(orc.transcript(b"innerproducttest"), Q, enc(Gf), enc(Hf), G, H, enc(a), enc(b), n)
    assert orc_rc == 0 and proof == want
    assert t.to_bytes() == orc_t[:bp.TRANSCRIPT_BYTES]             # same transcript state after proving
    assert bp.ipp_verify(gpu_ctx, bp.Transcript(b"innerproducttest"), n, enc(Gf), enc(Hf), P, Q, G, H, proof) == 0
    assert orc.ipp_verify(orc.transcript(b"innerproducttest"), n, enc(Gf), enc(Hf), P, Q, G, H, proof) == 0
    bad = bytearray(proof); bad[-33] ^= 2
    assert bp.ipp_verify(gpu_ctx, bp.Transcript(b"innerproducttest"), n, enc(Gf), enc(Hf), P, Q, G, H, bytes(bad)) != 0
    if n > 1:
        bad = bytearray(proof); bad[0:32] = b"\x01" + bytes(31)      # L_0 is not a valid point
        assert bp.ipp_verify(gpu_ctx, bp.Transcript(b"innerproducttest"), n, enc(Gf), enc(Hf), P, Q, G, H, bytes(bad)) == 1


def test_indexed_msm_uses_the_resident_table(gpu_ctx, orc):
    """PedersenGens::commit (generators.rs:39-41) and a mixed static/dynamic MSM via table slots."""
    import ctypes
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 16, 2); og = orc.gens(16, 2)
    B, Bb = orc.pedersen()
    rnd = random.Random(8)
    dyn = [orc.from_uniform(rnd.randbytes(64)) for _ in range(3)]
    v, r = rnd.randrange(1 << 64), rnd.randrange(l)
    s = [rnd.randrange(l) for _ in range(5)]
    scalars = le(v) + le(r) + b"".join(le(x) for x in s)
    idx = [1, 0, 2 + 1 * 16 + 3, 2 + 2 * 16 + 0 * 16 + 7, 0x80000000 | 0, 0x80000000 | 2, 1]
    offsets = [0, 2, 7]
    outs = ctypes.create_string_buffer(64); st = ctypes.create_string_buffer(2)
    rc = bp.lib().bp_msm_indexed_batch(gpu_ctx._h, gens._h, scalars, (ctypes.c_uint32 * 7)(*idx), b"".join(dyn), 3, (ctypes.c_uint64 * 3)(*offsets), 2, outs, st)
    assert rc == 0 and st.raw == b"\x00\x00"
    assert (0, outs.raw[:32]) == orc.msm(le(v) + le(r), B + Bb)
    pts = orc.gens_get(og, 0, 1, 3) + orc.gens_get(og, 1, 0, 7) + dyn[0] + dyn[2] + B
    assert (0, outs.raw[32:]) == orc.msm(b"".join(le(x) for x in s), pts)
    gens.close()


@pytest.mark.parametrize("n,m,count", [(32, 1, 1), (32, 1, 9), (64, 1, 16), (8, 2, 5), (64, 4, 3), (8, 32, 3), (64, 32, 2)])
def test_batched_prover_bytes_match_oracle(gpu_ctx, orc, n, m, count):
    """RangeProof::prove_many: B proofs with every group operation batched across the proofs (one device session for all inner-product
    arguments, generators never folded) must give exactly the bytes of B independent reference provers (oracle prove_many)."""
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 64, max(4, m)); og = orc.gens(64, max(4, m))
    rnd = random.Random(1000 * n + 10 * m + count)
    label = b"AggregateRangeProofBenchmark"
    values = [rnd.randrange(1 << n) for _ in range(count * m)]
    blind = b"".join(le(rnd.randrange(l)) for _ in range(count * m))
    seeds = b"".join(le(1000 + i, 8) + bytes(24) for i in range(count))
    st, proofs, V = bp.prove_many(gpu_ctx, gens, bp.Transcript(label), values, blind, n, m, seeds)
    want_proofs, want_V = orc.prove_many(og, orc.transcript(label), values, blind, n, m, seeds, nthreads=4)
    assert st == [0] * count and V == want_V
    plen = len(want_proofs) // count
    for i in range(count):
        assert proofs[i * plen:(i + 1) * plen] == want_proofs[i * plen:(i + 1) * plen], i
    assert bp.verify_batch(gpu_ctx, gens, bp.Transcript(label), proofs, V, n, m, count) == [0] * count
    gens.close()


def test_unfolded_ipp_session_rounds(gpu_ctx, orc):
    """bp_ippx_*: the device-resident inner-product prover state (no generator folding) round by round through the C ABI, two proofs side
    by side over arbitrary points; L, R, a, b == the oracle's InnerProductProof::create bytes."""
    import ctypes
    import bulletproofs_b200 as bp
    L = bp.lib(); rnd = random.Random(77)
    N, B = 16, 2
    G = b"".join(orc.from_uniform(rnd.randbytes(64)) for _ in range(N)); H = b"".join(orc.from_uniform(rnd.randbytes(64)) for _ in range(N))
    Q = [orc.from_uniform(rnd.randbytes(64)) for _ in range(B)]
    Gf = [b"".join(le(rnd.randrange(l)) for _ in range(N)) for _ in range(B)]; Hf = [b"".join(le(rnd.randrange(l)) for _ in range(N)) for _ in range(B)]
    a = [b"".join(le(rnd.randrange(l)) for _ in range(N)) for _ in range(B)]; b = [b"".join(le(rnd.randrange(l)) for _ in range(N)) for _ in range(B)]
    want = [orc.ipp_create(orc.transcript(b"ipp x"), Q[p], Gf[p], Hf[p], G, H, a[p], b[p], N)[2] for p in range(B)]
    sess = ctypes.c_void_p()
    gpu_ctx._check(L.bp_ippx_begin_points(gpu_ctx._h, G, H, N, B, b"".join(Q), b"".join(Gf), b"".join(Hf), b"".join(a), b"".join(b), ctypes.byref(sess)))
    ts = [bp.Transcript(b"ipp x") for _ in range(B)]
    for t in ts:
        t.append_message(b"dom-sep", b"ipp v1"); t.append_u64(b"n", N)
    got = [b"" for _ in range(B)]
    n = N
    while n > 1:
        assert L.bp_ippx_current_len(sess) == n
        lr = ctypes.create_string_buffer(64 * B)
        gpu_ctx._check(L.bp_ippx_round(sess, lr))
        us, uis = b"", b""
        for p in range(B):
            Lp, Rp = lr.raw[64 * p:64 * p + 32], lr.raw[64 * p + 32:64 * p + 64]
            got[p] += Lp + Rp
            ts[p].append_message(b"L", Lp); ts[p].append_message(b"R", Rp)
            u = int.from_bytes(ts[p].challenge_bytes(b"u", 64), "little") % l
            us += le(u); uis += le(pow(u, l - 2, l))
        gpu_ctx._check(L.bp_ippx_fold(sess, us, uis))
        n //= 2
    ab = ctypes.create_string_buffer(64 * B)
    gpu_ctx._check(L.bp_ippx_finish(sess, ab))
    L.bp_ippx_end(sess)
    for p in range(B):
        assert got[p] + ab.raw[64 * p:64 * p + 64] == want[p], p
