"""GPU tier (-m gpu): the CUDA path through the C ABI against the oracle and the golden fixtures."""
import os
import random

import pytest

from oracle_binding import L_ORDER as l, P_FIELD as p

pytestmark = pytest.mark.gpu


def le(x, n=32):
    return x.to_bytes(n, "little")


def test_native_library_is_the_one_running(gpu_ctx):
    import bulletproofs_b200 as bp
    maps = open("/proc/self/maps").read()
    assert "libbpmsm.so" in maps
    before = gpu_ctx.launches
    gpu_ctx.decompress_check(bytes(32))
    assert gpu_ctx.launches > before


def test_field_ptx_against_bigints(gpu_ctx):
    rnd = random.Random(1)
    edge = [0, 1, 2, 19, 38, p - 1, p, p + 1, 2**255 - 1, 2**255, 2**256 - 1, 2**256 - 38, 2**256 - 39, 2**256 - 37, 2**32 - 1, 2**224, (2**256 - 1) ^ (2**128)]
    vals = edge + [rnd.getrandbits(256) for _ in range(2000)] + [rnd.getrandbits(256) | (2**256 - 2**200) for _ in range(200)] + [rnd.getrandbits(64) for _ in range(100)]
    A = [rnd.choice(vals) for _ in range(20000)] + [a for a in edge for _ in edge]
    B = [rnd.choice(vals) for _ in range(20000)] + [b for _ in edge for b in edge]
    a, b = b"".join(le(x) for x in A), b"".join(le(x) for x in B)
    fns = {0: lambda x, y: (x + y) % p, 1: lambda x, y: (x - y) % p, 2: lambda x, y: x * y % p, 5: lambda x, y: (-x) % p,
           6: lambda x, y: x * x % p, 7: lambda x, y: (x + y) * (x - y) % p}
    for op, f in fns.items():
        out = gpu_ctx.debug_fe_op(op, a, b)
        for i, (x, y) in enumerate(zip(A, B)):
            assert int.from_bytes(out[32 * i:32 * i + 32], "little") == f(x, y), (op, hex(x), hex(y))
    n = 300
    out3 = gpu_ctx.debug_fe_op(3, a[:32 * n], b[:32 * n]); out4 = gpu_ctx.debug_fe_op(4, a[:32 * n], b[:32 * n])
    for i in range(n):
        assert int.from_bytes(out3[32 * i:32 * i + 32], "little") == pow(A[i] % p, p - 2, p)
        assert int.from_bytes(out4[32 * i:32 * i + 32], "little") == pow(A[i] % p, (p - 5) // 8, p)


def test_from_uniform_and_decompress(gpu_ctx, orc):
    rnd = random.Random(2)
    uni = [rnd.randbytes(64) for _ in range(300)] + [bytes(64), b"\xff" * 64]
    got = gpu_ctx.from_uniform_bytes(b"".join(uni))
    pts = [got[32 * i:32 * i + 32] for i in range(len(uni))]
    assert pts == [orc.from_uniform(u) for u in uni]
    cand = list(pts)
    for i in range(3000):
        s = bytearray(rnd.randbytes(32))
        if i % 4 == 0: s[31] |= 0x80
        if i % 5 == 0:
            s = bytearray(rnd.choice(pts)); s[rnd.randrange(32)] ^= 1 << rnd.randrange(8)
        cand.append(bytes(s))
    cand += [bytes(32), le(p), le(p + 2), le(1), le(2**255 - 20), b"\xff" * 32]
    assert gpu_ctx.decompress_check(b"".join(cand)) == [orc.point_is_valid(c) for c in cand]


def test_generators_match_oracle(gpu_ctx, orc):
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 64, 8); og = orc.gens(64, 8)
    B, Bb = orc.pedersen()
    assert gens.B == B and gens.B_blinding == Bb
    assert gens.G(0, 0).hex() == "fc3b25801422672a6a8d3adb5d8457d4301fe92324b4fc56ae934c8713ddfe2d"
    for which in (0, 1):
        for party in (0, 3, 7):
            for i in (0, 1, 31, 63):
                assert gens.get(which, party, i) == orc.gens_get(og, which, party, i)
    gens.close()


@pytest.mark.parametrize("n", [1, 2, 3, 17, 147, 190, 1000, 4099])
def test_msm_matches_oracle(gpu_ctx, orc, n):
    rnd = random.Random(100 + n)
    base = [orc.from_uniform(rnd.randbytes(64)) for _ in range(min(n, 64))]
    sc = b"".join(le(rnd.randrange(l)) for _ in range(n))
    pp = b"".join(rnd.choice(base) for _ in range(n))
    assert gpu_ctx.msm(sc, pp) == orc.msm(sc, pp)


def test_msm_edge_cases(gpu_ctx, orc):
    rnd = random.Random(9)
    pts = [orc.from_uniform(rnd.randbytes(64)) for _ in range(8)]
    # special scalars: 0, 1, l-1, powers of two, all equal (one bucket gets everything)
    sc = b"".join(le(x) for x in (0, 1, l - 1, 2**252, 2**128, l - 2**200, 2**252 + 1, 5))
    assert gpu_ctx.msm(sc, b"".join(pts)) == orc.msm(sc, b"".join(pts))
    sc = le(12345) * 200; pp = b"".join(rnd.choice(pts) for _ in range(200))
    assert gpu_ctx.msm(sc, pp) == orc.msm(sc, pp)
    # P + (-P) = identity encodes as zeros; all-zero scalars
    assert gpu_ctx.msm(le(7) + le(l - 7), pts[0] * 2) == (0, bytes(32))
    assert gpu_ctx.msm(le(0) * 5, b"".join(pts[:5])) == (0, bytes(32))
    # identity point as input
    assert gpu_ctx.msm(le(3) + le(4), bytes(32) + pts[1]) == orc.msm(le(3) + le(4), bytes(32) + pts[1])
    # invalid point -> None; non-canonical scalar
    import bulletproofs_b200 as bp
    assert gpu_ctx.msm(le(1), b"\x01" + bytes(31))[0] == bp.ERR_INVALID_POINT
    assert gpu_ctx.msm(le(l), pts[0])[0] == bp.ERR_NONCANONICAL_SCALAR


@pytest.mark.parametrize("n,kind", [(4096, "uniform"), (5000, "equal"), (12290, "few"), (1 << 16, "uniform")])
def test_msm_heavy_buckets(gpu_ctx, orc, n, kind):
    """Buckets far above the mean size go through k_msm_accumulate_heavy (a block per bucket).  With uniform scalars
    < l and c*(W-1) = 252 half of all terms share the top window's bucket 0; equal / few distinct scalars put every
    term of a window in one or a handful of buckets."""
    rnd = random.Random(n)
    base = [orc.from_uniform(rnd.randbytes(64)) for _ in range(64)]
    if kind == "uniform":
        sc = b"".join(le(rnd.randrange(l)) for _ in range(n))
    elif kind == "equal":
        sc = le(rnd.randrange(l)) * n
    else:
        few = [le(rnd.randrange(l)) for _ in range(3)]
        sc = b"".join(rnd.choice(few) for _ in range(n))
    pp = b"".join(rnd.choice(base) for _ in range(n))
    assert gpu_ctx.msm(sc, pp) == orc.msm(sc, pp)


def test_msm_batch_ragged(gpu_ctx, orc):
    rnd = random.Random(10)
    base = [orc.from_uniform(rnd.randbytes(64)) for _ in range(32)]
    sizes = [1, 0, 5, 64, 2, 147, 33, 0, 9]
    offsets = [0]
    for s in sizes: offsets.append(offsets[-1] + s)
    T = offsets[-1]
    sc = b"".join(le(rnd.randrange(l)) for _ in range(T)); pp = b"".join(rnd.choice(base) for _ in range(T))
    status, outs = gpu_ctx.msm_batch(sc, pp, offsets)
    for j, s in enumerate(sizes):
        a, b = offsets[j], offsets[j + 1]
        assert (status[j], outs[j]) == orc.msm(sc[32 * a:32 * b], pp[32 * a:32 * b]), j
    # one bad point poisons only its own MSM
    bad = bytearray(pp); bad[32 * offsets[3]:32 * offsets[3] + 32] = b"\x01" + bytes(31)
    status, outs2 = gpu_ctx.msm_batch(sc, bytes(bad), offsets)
    assert status[3] == 1 and [s for j, s in enumerate(status) if j != 3] == [0] * 8
    assert [o for j, o in enumerate(outs2) if j != 3] == [o for j, o in enumerate(outs) if j != 3]


def test_golden_proofs_batch_verify(gpu_ctx, orc, golden):
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 64, 8)
    vc = b"".join(bytes.fromhex(v) for v in golden["value_commitments"])
    t = bp.Transcript(golden["transcript_label"].encode())
    for pr in golden["proofs"]:
        proof = bytes.fromhex(pr["proof"]); m, n = pr["m"], pr["n"]
        assert bp.verify_batch(gpu_ctx, gens, t, proof, vc[:32 * m], n, m, 1) == [0], (n, m)
        # the same proof three times with one corrupted copy in the middle: fallback path gives per-proof verdicts
        bad = bytearray(proof); bad[len(proof) // 2] ^= 0x10
        got = bp.verify_batch(gpu_ctx, gens, t, proof + bytes(bad) + proof, vc[:32 * m] * 3, n, m, 3, seed=bytes([n + m]) * 32)
        assert got[0] == 0 and got[2] == 0 and got[1] != 0, (n, m, got)
    gens.close()


def _workload(orc, og, label, n, m, count, seed):
    rnd = random.Random(seed)
    t = orc.transcript(label)
    values = [rnd.randrange(1 << n) for _ in range(count * m)]
    blind = b"".join(le(rnd.randrange(l)) for _ in range(count * m))
    seeds = b"".join(le(i, 8) + bytes(24) for i in range(count))
    proofs, Vs = orc.prove_many(og, t, values, blind, n, m, seeds, nthreads=os.cpu_count() or 4)
    return proofs, Vs


@pytest.mark.parametrize("n,m,count", [(64, 1, 96), (32, 1, 33), (64, 4, 16), (8, 2, 40), (64, 16, 8)])
def test_batch_verify_matches_oracle_per_proof(gpu_ctx, orc, n, m, count):
    """verdict[i] == reference verdict of proof i, for valid batches and for batches with assorted damage."""
    import bulletproofs_b200 as bp
    label = b"AggregateRangeProofBenchmark"
    og = orc.gens(64, 16); gens = bp.Gens(gpu_ctx, 64, 16)
    proofs, Vs = _workload(orc, og, label, n, m, count, seed=n * 100 + m)
    plen = len(proofs) // count
    t = bp.Transcript(label); ot = orc.transcript(label)
    assert bp.verify_batch(gpu_ctx, gens, t, proofs, Vs, n, m, count) == [0] * count
    rnd = random.Random(n + m)
    pb, vb = bytearray(proofs), bytearray(Vs)
    damaged = rnd.sample(range(count), max(3, count // 6))
    for j, i in enumerate(damaged):
        kind = j % 6
        if kind == 0: pb[i * plen + rnd.randrange(plen)] ^= 1 << rnd.randrange(8)          # random bit anywhere
        elif kind == 1: pb[i * plen:i * plen + 32] = bytes(32)                                  # A = identity encoding
        elif kind == 2: pb[i * plen + 128:i * plen + 160] = b"\xff" * 32                        # non-canonical t_x -> FormatError
        elif kind == 3: vb[i * 32 * m + 3] ^= 0x40                                              # wrong commitment
        elif kind == 4: pb[i * plen + 224:i * plen + 256] = le(p + 1)                           # L_0 not a canonical field element
        else: pb[(i + 1) * plen - 32:(i + 1) * plen] = le(l)                                    # b = l, non-canonical
    want = orc.verify_many(og, ot, bytes(pb), plen, bytes(vb), n, m, count)
    got = bp.verify_batch(gpu_ctx, gens, t, bytes(pb), bytes(vb), n, m, count)
    assert got == want
    assert all(want[i] != 0 for i in damaged) and sum(1 for w in want if w) == len(damaged)
    gens.close()


def test_verify_parameter_errors(gpu_ctx, orc, golden):
    """mod.rs:358-366 and the from_bytes length rules, same codes as the oracle."""
    import bulletproofs_b200 as bp
    gens = bp.Gens(gpu_ctx, 32, 2); og = orc.gens(32, 2)
    vc = b"".join(bytes.fromhex(v) for v in golden["value_commitments"])
    label = golden["transcript_label"].encode(); t = bp.Transcript(label); ot = orc.transcript(label)
    by = {(q["n"], q["m"]): bytes.fromhex(q["proof"]) for q in golden["proofs"]}
    cases = [(by[(64, 1)], 64, 1),      # gens_capacity 32 < n
             (by[(8, 4)], 8, 4),        # party_capacity 2 < m
             (by[(8, 1)], 12, 1),       # bitsize
             (by[(8, 1)], 16, 1),       # n*m != 2^k
             (by[(8, 1)][:-32], 8, 1),  # odd number of IPP elements
             (by[(8, 1)][:200], 8, 1),  # too short
             (by[(8, 2)], 8, 2)]        # fine
    for proof, n, m in cases:
        want = orc.rangeproof_verify(og, ot, proof, vc[:32 * m], m, n)
        got = bp.verify_batch(gpu_ctx, gens, t, proof, vc[:32 * m], n, m, 1, proof_len=len(proof))
        assert got == [want], (n, m, len(proof), got, want)
    # a launch group whose parameters are rejected: every proof gets the code, every batch flag is cleared
    want = orc.rangeproof_verify(og, ot, by[(64, 1)], vc[:32], 1, 64)
    got, ok = bp.verify_group(gpu_ctx, gens, t, by[(64, 1)] * 6, vc[:32] * 6, 64, 1, 2, 3)
    assert want != 0 and got == [want] * 6 and ok == [0, 0, 0]
    gens.close()


def test_full_size_batch_properties(gpu_ctx, orc):
    """BASELINE config 2 size (1024 x (64,1)) through size-independent properties: a batch built from 64
    oracle-made proofs repeated 16 times verifies; one flipped bit in any single proof is found exactly."""
    import bulletproofs_b200 as bp
    label = b"AggregateRangeProofBenchmark"
    og = orc.gens(64, 1); gens = bp.Gens(gpu_ctx, 64, 1)
    proofs, Vs = _workload(orc, og, label, 64, 1, 64, seed=4242)
    plen = len(proofs) // 64
    big_p, big_v = proofs * 16, Vs * 16
    t = bp.Transcript(label)
    assert bp.verify_batch(gpu_ctx, gens, t, big_p, big_v, 64, 1, 1024) == [0] * 1024
    rnd = random.Random(77)
    for _ in range(2):
        i = rnd.randrange(1024); pb = bytearray(big_p); pb[i * plen + rnd.randrange(plen)] ^= 2
        got = bp.verify_batch(gpu_ctx, gens, t, bytes(pb), big_v, 64, 1, 1024)
        assert [j for j, v in enumerate(got) if v] == [i]
    gens.close()


def test_differential_fuzz_against_oracle(gpu_ctx, orc):
    """Many random mutations of valid proofs (bit flips, byte stomps, swapped fields, swapped proofs, zeroed / maximal
    fields, commitments of other proofs) in batches: the GPU verdict list must equal the oracle's per-proof verdicts."""
    import bulletproofs_b200 as bp
    label = b"fuzz"
    n, m, count = 16, 2, 48
    og = orc.gens(16, 2); gens = bp.Gens(gpu_ctx, 16, 2)
    proofs, Vs = _workload(orc, og, label, n, m, count, seed=999)
    plen = len(proofs) // count
    t = bp.Transcript(label); ot = orc.transcript(label)
    rnd = random.Random(2024)
    for round_ in range(6):
        pb, vb = bytearray(proofs), bytearray(Vs)
        for i in rnd.sample(range(count), 20):
            kind = rnd.randrange(9); o = i * plen
            if kind == 0: pb[o + rnd.randrange(plen)] ^= 1 << rnd.randrange(8)
            elif kind == 1: pb[o + rnd.randrange(plen)] = rnd.randrange(256)
            elif kind == 2:                                           # swap two 32-byte fields of the proof
                a, b = rnd.sample(range(plen // 32), 2); pb[o + 32 * a:o + 32 * a + 32], pb[o + 32 * b:o + 32 * b + 32] = pb[o + 32 * b:o + 32 * b + 32], pb[o + 32 * a:o + 32 * a + 32]
            elif kind == 3:                                           # another proof's bytes with this proof's commitments
                j = rnd.randrange(count); pb[o:o + plen] = proofs[j * plen:(j + 1) * plen]
            elif kind == 4: f = rnd.randrange(plen // 32); pb[o + 32 * f:o + 32 * f + 32] = bytes(32)
            elif kind == 5: f = rnd.randrange(plen // 32); pb[o + 32 * f:o + 32 * f + 32] = bytes([255]) * 32
            elif kind == 6: vb[i * 32 * m + rnd.randrange(32 * m)] ^= 1 << rnd.randrange(8)
            elif kind == 7: f = rnd.randrange(plen // 32); pb[o + 32 * f:o + 32 * f + 32] = le(l - 1)      # canonical-boundary scalar / non-point
            else: f = rnd.randrange(plen // 32); pb[o + 32 * f:o + 32 * f + 32] = le(p - 1)                 # largest field element
        want = orc.verify_many(og, ot, bytes(pb), plen, bytes(vb), n, m, count)
        got = bp.verify_batch(gpu_ctx, gens, t, bytes(pb), bytes(vb), n, m, count, seed=bytes([round_]) * 32)
        assert got == want, (round_, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w])
    gens.close()


def test_back_to_back_device_calls_keep_their_own_parameters(gpu_ctx, orc):
    """bp_rangeproof_verify_batch_device returns without synchronising: calls queued back to back on one context must each use the
    transcript they were given (their parameter blocks travel through a pinned staging ring), not the last caller's."""
    import torch
    import bulletproofs_b200 as bp
    n, m, count = 32, 1, 16
    rnd = random.Random(31)
    og = orc.gens(n, m); gens = bp.Gens(gpu_ctx, n, m)
    vals = [rnd.randrange(1 << n) for _ in range(count)]; bl = b"".join(le(rnd.randrange(l)) for _ in range(count))
    seeds = b"".join(i.to_bytes(8, "little") + bytes(24) for i in range(count))
    proofs, Vs = orc.prove_many(og, orc.transcript(b"label A"), vals, bl, n, m, seeds, nthreads=2)
    d_proofs = torch.frombuffer(bytearray(proofs), dtype=torch.uint8).cuda(); d_vs = torch.frombuffer(bytearray(Vs), dtype=torch.uint8).cuda()
    rounds = 24                                     # more than the ring has slots
    d_verdicts = torch.full((rounds, count), 77, dtype=torch.int32, device="cuda")
    good = bp.BatchVerifier(gpu_ctx, gens, bp.Transcript(b"label A"), n, m, count)
    wrong = bp.BatchVerifier(gpu_ctx, gens, bp.Transcript(b"label B"), n, m, count)      # same proofs under another transcript: the combined check fails,
    torch.cuda.synchronize()                                                              # and the device path (no per-proof recheck) marks the whole batch
    for r in range(rounds):
        (good if r % 2 == 0 else wrong).run_device(d_proofs.data_ptr(), d_vs.data_ptr(), d_verdicts[r].data_ptr(), None)
    gpu_ctx.synchronize()
    got = d_verdicts.cpu().tolist()
    for r in range(rounds):
        assert got[r] == [0 if r % 2 == 0 else 1] * count, (r, got[r])
    gens.close()


def test_launch_groups_match_oracle_per_proof(gpu_ctx, orc):
    """Several independent batches in one launch group (bp_rangeproof_verify_group_*): per-proof verdicts == oracle, per-batch accept
    flags right, a damaged proof only sends its own batch through the per-proof recheck; the reserved (CUDA graph) path and the
    direct-launch path agree."""
    import bulletproofs_b200 as bp
    label = b"AggregateRangeProofBenchmark"
    n, m, count, nb = 64, 1, 40, 5
    og = orc.gens(64, 1); gens = bp.Gens(gpu_ctx, 64, 1)
    proofs, Vs = _workload(orc, og, label, n, m, count * nb, seed=515)
    plen = len(proofs) // (count * nb)
    t = bp.Transcript(label); ot = orc.transcript(label)
    got, ok = bp.verify_group(gpu_ctx, gens, t, proofs, Vs, n, m, count, nb)
    assert got == [0] * (count * nb) and ok == [1] * nb
    pb, vb = bytearray(proofs), bytearray(Vs)
    pb[(1 * count + 7) * plen + 300] ^= 1            # batch 1: one bad proof
    pb[(3 * count + 0) * plen: (3 * count + 0) * plen + 32] = bytes(32)     # batch 3: A = identity encoding (caught before the MSM: combined check still passes)
    vb[(3 * count + 39) * 32 + 5] ^= 8              # batch 3: wrong commitment on the last proof
    pb[(4 * count + 3) * plen + 224: (4 * count + 3) * plen + 256] = le(p + 1)      # batch 4: L_0 undecodable
    want = orc.verify_many(og, ot, bytes(pb), plen, bytes(vb), n, m, count * nb)
    for reserve in (False, True):
        if reserve:
            v = bp.BatchVerifier(gpu_ctx, gens, t, n, m, count, nb)          # reserves: the next calls with this geometry replay the captured graph
        got, ok = bp.verify_group(gpu_ctx, gens, t, bytes(pb), bytes(vb), n, m, count, nb, seed=bytes([9]) * 32)
        assert got == want, (reserve, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w])
        assert ok == [1, 0, 1, 0, 0]
        assert sum(1 for w in want if w) == 4
    # another geometry on the same (reserved) context takes the direct path and leaves the graph intact
    assert bp.verify_batch(gpu_ctx, gens, t, proofs[:3 * plen], Vs[:3 * 32], n, m, 3) == [0, 0, 0]
    got, ok = bp.verify_group(gpu_ctx, gens, t, proofs, Vs, n, m, count, nb)
    assert got == [0] * (count * nb) and ok == [1] * nb
    gens.close()


def test_other_calls_between_verifications_keep_the_point_map(gpu_ctx, orc):
    """An indexed MSM (prover, R1CS verifier, MPC audit) on a context must not disturb the verifier's cached term->point map: device-path
    verification, then prove_multiple on the same context, then device-path verification again, all accepted (round-1 ADVICE, high)."""
    import torch
    import bulletproofs_b200 as bp
    label = b"AggregateRangeProofBenchmark"
    n, m, count = 32, 1, 24
    og = orc.gens(n, m); gens = bp.Gens(gpu_ctx, n, m)
    proofs, Vs = _workload(orc, og, label, n, m, count, seed=808)
    d_p = torch.frombuffer(bytearray(proofs), dtype=torch.uint8).cuda(); d_v = torch.frombuffer(bytearray(Vs), dtype=torch.uint8).cuda()
    d_verd = torch.full((3, count), 9, dtype=torch.int32, device="cuda"); h_ok = torch.zeros(3, dtype=torch.int32).pin_memory()
    ver = bp.BatchVerifier(gpu_ctx, gens, bp.Transcript(label), n, m, count, reserve=False)
    ver.run_device(d_p.data_ptr(), d_v.data_ptr(), d_verd[0].data_ptr(), h_ok[0:].data_ptr()); gpu_ctx.synchronize()
    rc, proof, V = bp.prove_multiple(gpu_ctx, gens, bp.Transcript(label), [5], le(7), n, bytes(32))
    assert rc == 0
    ver.run_device(d_p.data_ptr(), d_v.data_ptr(), d_verd[1].data_ptr(), h_ok[1:].data_ptr()); gpu_ctx.synchronize()
    ver2 = bp.BatchVerifier(gpu_ctx, gens, bp.Transcript(label), n, m, count)       # reserved / graph path
    rc, proof, V = bp.prove_multiple(gpu_ctx, gens, bp.Transcript(label), [6], le(8), n, bytes(32))
    ver2.run_device(d_p.data_ptr(), d_v.data_ptr(), d_verd[2].data_ptr(), h_ok[2:].data_ptr()); gpu_ctx.synchronize()
    assert d_verd.cpu().tolist() == [[0] * count] * 3 and h_ok.tolist() == [1, 1, 1]
    gens.close()


def test_pending_verification_blocks_other_entry_points(gpu_ctx, orc):
    """Between verify_begin and verify_finish the context's arenas belong to the pending verification (its fallback reads them):
    other entry points fail with a clear error instead of clobbering them, and a failed begin leaves the context usable."""
    import bulletproofs_b200 as bp
    label = b"AggregateRangeProofBenchmark"
    n, m, count = 8, 1, 6
    og = orc.gens(n, m); gens = bp.Gens(gpu_ctx, n, m)
    proofs, Vs = _workload(orc, og, label, n, m, count, seed=11)
    pb = bytearray(proofs); pb[2 * (len(proofs) // count) + 140] ^= 1
    ver = bp.BatchVerifier(gpu_ctx, gens, bp.Transcript(label), n, m, count, reserve=False)
    import ctypes
    hp = ctypes.create_string_buffer(bytes(pb)); hv = ctypes.create_string_buffer(Vs)
    ver.begin(ctypes.addressof(hp), ctypes.addressof(hv))
    with pytest.raises(bp.BpError):
        gpu_ctx.msm(le(1), orc.from_uniform(bytes(64)))
    with pytest.raises(bp.BpError):
        ver.begin(ctypes.addressof(hp), ctypes.addressof(hv))
    got = list(ver.finish())
    assert [i for i, v in enumerate(got) if v] == [2]
    assert gpu_ctx.msm(le(1), orc.from_uniform(bytes(64)))[0] == 0
    gens.close()


def test_point_values_cross_the_boundary(gpu_ctx, orc):
    """bp_decompress_batch / bp_compress_batch: CompressedRistretto::decompress -> Option<RistrettoPoint> and back (SURVEY.md 8b)."""
    rnd = random.Random(21)
    pts = [orc.from_uniform(rnd.randbytes(64)) for _ in range(200)] + [bytes(32)]
    bad = [b"\x01" + bytes(31), le(p), le(p - 1), b"\xff" * 32]
    xyzt, ok = gpu_ctx.decompress(b"".join(pts + bad))
    assert ok == [orc.point_is_valid(q) for q in pts + bad] and ok[:len(pts)] == [1] * len(pts)
    for v in xyzt[:len(pts)]:
        X, Y, Z, T = (int.from_bytes(v[32 * i:32 * i + 32], "little") for i in range(4))
        d = (-121665 * pow(121666, p - 2, p)) % p
        assert Z == 1 and T == X * Y % p and (-X * X + Y * Y - 1 - d * X * X * Y * Y) % p == 0          # on the curve, extended coordinates consistent
    assert gpu_ctx.compress(b"".join(xyzt[:len(pts)])) == b"".join(pts)
    # any projective representative compresses to the same bytes
    lam = 0x1234567
    scaled = b"".join(le(int.from_bytes(v[32 * i:32 * i + 32], "little") * lam % p) for v in xyzt[:20] for i in range(4))
    assert gpu_ctx.compress(scaled) == b"".join(pts[:20])


@pytest.mark.parametrize("terms,n_msm", [(1, 3), (147, 5), (1000, 8), (4096, 2)])
def test_resident_point_set_msm(gpu_ctx, orc, terms, n_msm):
    """bp_points: bases decompressed once, many MSMs over them == the oracle's MSM on the same bytes."""
    import bulletproofs_b200 as bp
    rnd = random.Random(terms)
    base = [orc.from_uniform(rnd.randbytes(64)) for _ in range(min(terms, 64))]
    pts = b"".join(rnd.choice(base) for _ in range(terms + 3))
    ps = bp.PointSet(gpu_ctx, pts)
    sc = b"".join(le(rnd.randrange(l)) for _ in range(terms * n_msm))
    st, outs = ps.msm(sc, n_msm, terms)
    assert st == [0] * n_msm
    for j in range(n_msm):
        assert (0, outs[j]) == orc.msm(sc[32 * terms * j:32 * terms * (j + 1)], pts[:32 * terms]), j
    st, outs2 = ps.msm(sc[:32 * terms], 1, terms)            # another shape on the same set
    assert outs2[0] == outs[0]
    ps.close()
    with pytest.raises(bp.BpError):
        bp.PointSet(gpu_ctx, pts[:64] + b"\x01" + bytes(31))


@pytest.mark.parametrize("window", [2, 3, 5, 8, 9, 12, 13, 16, 17, 18])
def test_msm_every_window_geometry(gpu_ctx, orc, window):
    """The result of an MSM does not depend on the Pippenger window: pin it (bp_ctx_set_msm_window) and compare with the oracle, including the
    windows with c*(W-1) = 252 whose top window holds only the recoding carry (c = 9, 12), windows wider than the MSM is long, and the
    widest windows the context accepts (c = 17, 18: 2^16 and 2^17 buckets per window, which msm_pick_window never chooses)."""
    rnd = random.Random(300 + window)
    base = [orc.from_uniform(rnd.randbytes(64)) for _ in range(40)]
    try:
        gpu_ctx.set_msm_window(window)
        for n in (1, 37, 700):
            sc = b"".join(le(rnd.randrange(l)) for _ in range(n)); pp = b"".join(rnd.choice(base) for _ in range(n))
            assert gpu_ctx.msm(sc, pp) == orc.msm(sc, pp), (window, n)
        sc = b"".join(le(x) for x in (0, 1, l - 1, 2**252, 2**128, l - 2**200, 2**252 + 1, 5)); pp = b"".join(base[:8])
        assert gpu_ctx.msm(sc, pp) == orc.msm(sc, pp)
    finally:
        gpu_ctx.set_msm_window(0)
