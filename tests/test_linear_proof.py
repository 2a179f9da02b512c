"""LinearProof (SURVEY.md §8f rank 4; src/linear_proof.rs).  CPU tier: the oracle round-trips on the reference's
test sizes (linear_proof.rs:413-487: n in {1, 16, 32, 64}).  GPU tier: the C++ mirror (B, F and G resident on the device as one point
set, never folded) gives the oracle's proof bytes and verdicts."""
import random

import pytest

from oracle_binding import L_ORDER as l


def le(x, n=32):
    return x.to_bytes(n, "little")


def _instance(orc, n, seed):
    rnd = random.Random(seed)
    g = orc.gens(max(n, 1), 1)
    G = b"".join(orc.gens_get(g, 0, 0, i) for i in range(n))
    F, B = orc.pedersen()                                           # F = pc_gens.B, B = pc_gens.B_blinding (linear_proof.rs:422-424)
    a = [rnd.randrange(l) for _ in range(n)]; b = [rnd.randrange(l) for _ in range(n)]; r = rnd.randrange(l)
    c = sum(x * y for x, y in zip(a, b)) % l
    rc, C = orc.msm(b"".join(map(le, a)) + le(r) + le(c), G + B + F)
    assert rc == 0
    return G, F, B, b"".join(map(le, a)), b"".join(map(le, b)), le(r), C


@pytest.mark.parametrize("n", [1, 2, 16, 32, 64])
def test_oracle_linear_proof_roundtrip(orc, n):
    G, F, B, a, b, r, C = _instance(orc, n, n)
    t = orc.transcript(b"linearprooftest")
    rc, t_after, proof = orc.linear_create(t, bytes([9]) * 32, C, r, a, b, G, F, B)
    assert rc == 0 and len(proof) == 32 * (2 * (n.bit_length() - 1) + 3)
    assert orc.linear_verify(t, proof, C, G, F, B, b) == 0
    bad = bytearray(proof); bad[-1] ^= 1
    assert orc.linear_verify(t, bytes(bad), C, G, F, B, b) != 0
    b2 = bytearray(b); b2[0] ^= 1
    assert orc.linear_verify(t, proof, C, G, F, B, bytes(b2)) != 0
    assert orc.linear_verify(t, proof[:-32], C, G, F, B, b) == 2      # FormatError


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 16, 64, 256])
def test_gpu_linear_proof_matches_oracle(gpu_ctx, orc, n):
    import bulletproofs_b200 as bp
    G, F, B, a, b, r, C = _instance(orc, n, 100 + n)
    seed = bytes([n % 251]) * 32
    t = bp.Transcript(b"linearprooftest")
    rc, proof = bp.linear_create(gpu_ctx, t, seed, C, r, a, b, G, F, B)
    orc_rc, orc_t, want = orc.linear_create(orc.transcript(b"linearprooftest"), seed, C, r, a, b, G, F, B)
    assert rc == 0 and orc_rc == 0 and proof == want and t.to_bytes() == orc_t[:bp.TRANSCRIPT_BYTES]
    assert bp.linear_verify(gpu_ctx, bp.Transcript(b"linearprooftest"), proof, C, G, F, B, b) == 0
    assert orc.linear_verify(orc.transcript(b"linearprooftest"), proof, C, G, F, B, b) == 0
    bad = bytearray(proof); bad[5] ^= 1
    assert bp.linear_verify(gpu_ctx, bp.Transcript(b"linearprooftest"), bytes(bad), C, G, F, B, b) == orc.linear_verify(orc.transcript(b"linearprooftest"), bytes(bad), C, G, F, B, b) != 0
    b2 = bytearray(b); b2[33 % len(b)] ^= 2
    assert bp.linear_verify(gpu_ctx, bp.Transcript(b"linearprooftest"), proof, C, G, F, B, bytes(b2)) != 0
