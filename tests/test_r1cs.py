"""R1CS (§8 rows A7, A8; the reference's `yoloproofs` module).  CPU tier: the oracle's prover and verifier round-trip on
the reference's own test cases (tests/r1cs.rs:146-224 shuffle, :350-364 example gadget, :366-453 range gadget).
GPU tier: the C++ mirror (every MSM on the GPU) produces the same proof bytes as the oracle for the same witness,
blindings and external randomness, and the two verifiers agree on accept/reject."""
import random

import pytest

from oracle_binding import L_ORDER as l

SHUFFLE, EXAMPLE, RANGE = 0, 1, 2


def le(x, n=32):
    return x.to_bytes(n, "little")


def shuffle_transcript_orc(orc, k):
    t = orc.transcript(b"ShuffleProofTest")
    t = orc.transcript_append(t, b"dom-sep", b"ShuffleProof")
    return orc.transcript_append(t, b"k", le(k, 8))


def test_oracle_example_gadget(orc):
    g = orc.gens(128, 1); rnd = random.Random(1)
    t = orc.transcript(b"R1CSExampleGadget")
    bl = b"".join(le(rnd.randrange(l)) for _ in range(5))
    rc, proof, V = orc.r1cs_prove(g, t, EXAMPLE, [3, 4, 6, 1, 40], bl, param=9)
    assert rc == 0 and proof[0] == 0 and len(proof) == 1 + 11 * 32 + 32 * 2           # one-phase proof; one multiplier -> padded_n = 1, IPP = (a, b)
    assert orc.r1cs_verify(g, t, EXAMPLE, V, proof, param=9) == 0
    assert orc.r1cs_verify(g, t, EXAMPLE, V, proof, param=10) != 0
    rc, proof, V = orc.r1cs_prove(g, t, EXAMPLE, [3, 4, 6, 1, 40], bl, param=10)       # (3+4)*(6+1) != 40+10
    assert rc == 0 and orc.r1cs_verify(g, t, EXAMPLE, V, proof, param=10) != 0


def test_oracle_range_gadget(orc):
    g = orc.gens(128, 1); rnd = random.Random(2)
    for n in (2, 10, 32, 63):
        t = orc.transcript(b"RangeProofTest")
        for v in [rnd.randrange(1 << n) for _ in range(2)] + [(1 << n) - 1, 0]:
            rc, proof, V = orc.r1cs_prove(g, t, RANGE, [v], le(rnd.randrange(l)), param=n, aux=v)
            assert rc == 0 and orc.r1cs_verify(g, t, RANGE, V, proof, param=n) == 0, (n, v)
        rc, proof, V = orc.r1cs_prove(g, t, RANGE, [1 << n], le(rnd.randrange(l)), param=n, aux=1 << n)
        assert rc == 0 and orc.r1cs_verify(g, t, RANGE, V, proof, param=n) != 0


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 6, 7, 24, 42])
def test_oracle_shuffle(orc, k):
    g = orc.gens(128, 1); rnd = random.Random(k)
    t = shuffle_transcript_orc(orc, k)
    inp = [rnd.randrange(1 << 64) for _ in range(k)]; out = inp[:]; rnd.shuffle(out)
    bl = b"".join(le(rnd.randrange(l)) for _ in range(2 * k))
    rc, proof, V = orc.r1cs_prove(g, t, SHUFFLE, inp + out, bl)
    assert rc == 0 and proof[0] == (0 if k == 1 else 1)
    assert orc.r1cs_verify(g, t, SHUFFLE, V, proof) == 0
    if k > 1:
        bad = out[:]; bad[0] = (bad[0] + 1) % (1 << 64)
        rc, p2, V2 = orc.r1cs_prove(g, t, SHUFFLE, inp + bad, bl)
        assert rc == 0 and orc.r1cs_verify(g, t, SHUFFLE, V2, p2) != 0
    b = bytearray(proof); b[40] ^= 1
    assert orc.r1cs_verify(g, t, SHUFFLE, V, bytes(b)) != 0
    assert orc.r1cs_verify(g, t, SHUFFLE, V, proof[:-1]) == 2                           # FormatError
    assert orc.r1cs_verify(g, shuffle_transcript_orc(orc, k + 1), SHUFFLE, V, proof) != 0


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 5, 8, 42, 300, 2049])        # 2049 inputs = 4096 multipliers: R1CSProof bytes still equal the oracle's
def test_gpu_shuffle_matches_oracle(gpu_ctx, orc, k):
    import bulletproofs_b200 as bp
    cap = max(128, 1 << (2 * k).bit_length())
    gens = bp.Gens(gpu_ctx, cap, 1); og = orc.gens(cap, 1)
    rnd = random.Random(100 + k)
    inp = [rnd.randrange(1 << 64) for _ in range(k)]; out = inp[:]; rnd.shuffle(out)
    bl = b"".join(le(rnd.randrange(l)) for _ in range(2 * k)); ext = bytes([k % 256]) * 32

    def tr():
        t = bp.Transcript(b"ShuffleProofTest"); t.append_message(b"dom-sep", b"ShuffleProof"); t.append_u64(b"k", k); return t

    rc, proof, V = bp.r1cs_prove(gpu_ctx, gens, tr(), bp.GADGET_SHUFFLE, inp + out, bl, ext_seed=ext)
    orc_rc, want, want_V = orc.r1cs_prove(og, shuffle_transcript_orc(orc, k), SHUFFLE, inp + out, bl, ext_seed=ext)
    assert rc == 0 and orc_rc == 0 and V == want_V
    assert proof == want                                                                # bit-exact R1CSProof bytes
    assert bp.r1cs_verify(gpu_ctx, gens, tr(), bp.GADGET_SHUFFLE, V, proof) == 0
    assert orc.r1cs_verify(og, shuffle_transcript_orc(orc, k), SHUFFLE, V, proof) == 0
    b = bytearray(proof); b[len(b) // 2] ^= 4
    assert bp.r1cs_verify(gpu_ctx, gens, tr(), bp.GADGET_SHUFFLE, V, bytes(b)) != 0
    if k > 1:
        bad = out[:]; bad[-1] ^= 1
        rc, p2, V2 = bp.r1cs_prove(gpu_ctx, gens, tr(), bp.GADGET_SHUFFLE, inp + bad, bl, ext_seed=ext)
        assert rc == 0 and bp.r1cs_verify(gpu_ctx, gens, tr(), bp.GADGET_SHUFFLE, V2, p2) == orc.r1cs_verify(og, shuffle_transcript_orc(orc, k), SHUFFLE, V2, p2) != 0
    gens.close()


@pytest.mark.gpu
def test_gpu_example_and_range_gadgets_match_oracle(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 128, 1); og = orc.gens(128, 1)
    rnd = random.Random(9)
    bl = b"".join(le(rnd.randrange(l)) for _ in range(5))
    for c2, ok in ((9, True), (10, False)):
        rc, proof, V = bp.r1cs_prove(gpu_ctx, gens, bp.Transcript(b"R1CSExampleGadget"), bp.GADGET_EXAMPLE, [3, 4, 6, 1, 40], bl, param=c2)
        _, want, _ = orc.r1cs_prove(og, orc.transcript(b"R1CSExampleGadget"), EXAMPLE, [3, 4, 6, 1, 40], bl, param=c2)
        assert rc == 0 and proof == want
        got = bp.r1cs_verify(gpu_ctx, gens, bp.Transcript(b"R1CSExampleGadget"), bp.GADGET_EXAMPLE, V, proof, param=c2)
        assert (got == 0) == ok and got == orc.r1cs_verify(og, orc.transcript(b"R1CSExampleGadget"), EXAMPLE, V, proof, param=c2)
    for n in (2, 10, 32, 63):
        for v in (rnd.randrange(1 << n), 1 << n):
            b1 = le(rnd.randrange(l))
            rc, proof, V = bp.r1cs_prove(gpu_ctx, gens, bp.Transcript(b"RangeProofTest"), bp.GADGET_RANGE, [v], b1, param=n, aux=v)
            _, want, _ = orc.r1cs_prove(og, orc.transcript(b"RangeProofTest"), RANGE, [v], b1, param=n, aux=v)
            assert rc == 0 and proof == want
            got = bp.r1cs_verify(gpu_ctx, gens, bp.Transcript(b"RangeProofTest"), bp.GADGET_RANGE, V, proof, param=n)
            assert (got == 0) == (v < (1 << n)) and got == orc.r1cs_verify(og, orc.transcript(b"RangeProofTest"), RANGE, V, proof, param=n)
    gens.close()


@pytest.mark.gpu
def test_gpu_shuffle_config5_full_size(gpu_ctx, orc):
    """BASELINE config 5: k-shuffle with 2^16 multipliers (k = 32769), prove + verify on one H100.  The oracle prover
    would take tens of seconds at this size, so parity is checked through the independent verifier: the proof made
    on the GPU path must be accepted by the oracle's verifier (a 196 655-term CPU MSM) and by the GPU verifier, and a
    damaged proof / a non-permutation must be rejected by both."""
    import bulletproofs_b200 as bp
    k = 32769                                                                           # 2(k-1) = 65 536 multipliers (benches/r1cs.rs:52-67)
    gens = bp.Gens(gpu_ctx, 65536, 1); og = orc.gens(65536, 1)
    rnd = random.Random(5)
    inp = [rnd.randrange(1 << 64) for _ in range(k)]; out = inp[:]; rnd.shuffle(out)
    bl = b"".join(le(rnd.randrange(l)) for _ in range(2 * k))

    def tr():
        t = bp.Transcript(b"ShuffleBenchmark"); t.append_message(b"dom-sep", b"ShuffleProof"); t.append_u64(b"k", k); return t

    def otr():
        t = orc.transcript(b"ShuffleBenchmark"); t = orc.transcript_append(t, b"dom-sep", b"ShuffleProof"); return orc.transcript_append(t, b"k", le(k, 8))

    rc, proof, V = bp.r1cs_prove(gpu_ctx, gens, tr(), bp.GADGET_SHUFFLE, inp + out, bl)
    assert rc == 0 and len(proof) == 1 + 32 * 14 + 32 * 34                              # 1537 bytes (SURVEY.md §8 table)
    assert bp.r1cs_verify(gpu_ctx, gens, tr(), bp.GADGET_SHUFFLE, V, proof) == 0
    assert orc.r1cs_verify(og, otr(), SHUFFLE, V, proof) == 0
    b = bytearray(proof); b[700] ^= 1
    assert bp.r1cs_verify(gpu_ctx, gens, tr(), bp.GADGET_SHUFFLE, V, bytes(b)) != 0
    Vb = bytearray(V); Vb[5 * 32 + 1] ^= 1                                              # a different committed input: no longer a permutation
    assert bp.r1cs_verify(gpu_ctx, gens, tr(), bp.GADGET_SHUFFLE, bytes(Vb), proof) != 0
    gens.close()
