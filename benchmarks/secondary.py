"""Secondary measurements on one GPU (SURVEY.md §8d; none of these is the bench line):
  config 1  (32,1) prove + verify latency, GPU-backed path vs the CPU oracle, proof bytes compared
  config 2  reject path: the 1024-proof batch with one corrupted proof (RLC fails -> per-proof recheck)
  config 3  256 x (64,16) aggregated proofs, single blocking call (the pipelined figure is `bench.py --m 16 --batch 256`)
  config 4  Ristretto MSM sweep (pageable host buffers through bp_msm_batch, decompression included; every first result compared
            byte-for-byte with the CPU oracle).  The sweep with resident inputs is `bench.py --workload msm`.
Prints one JSON object."""
import hashlib, json, os, random, statistics, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bulletproofs_b200 as bp
from oracle_binding import Oracle, L_ORDER

orc = Oracle(); ctx = bp.Context(0); rnd = random.Random(7); res = {}
LABEL = b"AggregateRangeProofBenchmark"
max_lg = int(sys.argv[1]) if len(sys.argv) > 1 else 20


def med(f, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); f(); ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


# ---- config 1: (32,1) prove and verify, one proof at a time
n, m = 32, 1
og = orc.gens(n, m); gens = bp.Gens(ctx, n, m)
v = [rnd.randrange(1 << n)]; bl = rnd.randrange(L_ORDER).to_bytes(32, "little"); seed = bytes([0x18]) * 32
rc, proof, V = bp.prove_multiple(ctx, gens, bp.Transcript(LABEL), v, bl, n, seed)
orc_rc, want, wantV = orc.rangeproof_prove(og, orc.transcript(LABEL), v, bl, n, seed)
assert rc == 0 and orc_rc == 0 and proof == want and V == wantV and len(proof) == 608
assert bp.verify_multiple(ctx, gens, bp.Transcript(LABEL), proof, V, n) == 0
res["config1_(32,1)"] = {
    "proof_bytes_equal_oracle": True,
    "gpu_backed_prove_us": round(1e6 * med(lambda: bp.prove_multiple(ctx, gens, bp.Transcript(LABEL), v, bl, n, seed), 20)),
    "gpu_backed_verify_us": round(1e6 * med(lambda: bp.verify_multiple(ctx, gens, bp.Transcript(LABEL), proof, V, n), 20)),
    "cpu_oracle_prove_us": round(1e6 * med(lambda: orc.rangeproof_prove(og, orc.transcript(LABEL), v, bl, n, seed), 20)),
    "cpu_oracle_verify_us": round(1e6 * med(lambda: orc.rangeproof_verify(og, orc.transcript(LABEL), proof, V, m, n), 20)),
    "note": "single proof = latency bound on the GPU (k dependent IPP rounds, one launch chain per round); reference README: 7.3 ms prove / 1.04 ms verify at (64,1)"}
gens.close()

# ---- config 2 reject path
n, m, count = 64, 1, 1024
og = orc.gens(n, m); gens = bp.Gens(ctx, n, m)
vals = [rnd.randrange(1 << n) for _ in range(count)]; bls = b"".join(rnd.randrange(L_ORDER).to_bytes(32, "little") for _ in range(count))
seeds = b"".join(i.to_bytes(8, "little") + bytes(24) for i in range(count))
proofs, Vs = orc.prove_many(og, orc.transcript(LABEL), vals, bls, n, m, seeds, nthreads=16)
plen = len(proofs) // count
bad = bytearray(proofs); bad[517 * plen + 32 * 4 + 3] ^= 0x10          # t_x of proof 517
bad = bytes(bad); t = bp.Transcript(LABEL)
assert bp.verify_batch(ctx, gens, t, proofs, Vs, n, m, count) == [0] * count
got = bp.verify_batch(ctx, gens, t, bad, Vs, n, m, count)
assert got == [0] * 517 + [1] + [0] * (count - 518)
res["config2_reject_path"] = {
    "accept_single_call_ms": round(1e3 * med(lambda: bp.verify_batch(ctx, gens, t, proofs, Vs, n, m, count), 10), 3),
    "one_bad_proof_single_call_ms": round(1e3 * med(lambda: bp.verify_batch(ctx, gens, t, bad, Vs, n, m, count), 10), 3),
    "note": "blocking bp_rangeproof_verify_batch with host buffers, one stream; on an RLC failure the batch is rechecked in two levels: 32 chunk MSMs, then the 32 proofs of the failing chunk (benchmarks/reject_path.py has more cases)"}
gens.close()

# ---- config 3: 256 x (64,16)
n, m, base, count = 64, 16, 16, 256
og = orc.gens(n, m); gens = bp.Gens(ctx, n, m)
vals = [rnd.randrange(1 << n) for _ in range(base * m)]; bls = b"".join(rnd.randrange(L_ORDER).to_bytes(32, "little") for _ in range(base * m))
proofs, Vs = orc.prove_many(og, orc.transcript(LABEL), vals, bls, n, m, seeds[:32 * base], nthreads=16)
P, Vv = proofs * (count // base), Vs * (count // base); t = bp.Transcript(LABEL)
assert bp.verify_batch(ctx, gens, t, P, Vv, n, m, count) == [0] * count
dt = med(lambda: bp.verify_batch(ctx, gens, t, P, Vv, n, m, count), 10)
t0 = time.perf_counter(); st = orc.verify_many(og, orc.transcript(LABEL), proofs, len(proofs) // base, Vs, n, m, base, nthreads=16); dtc = time.perf_counter() - t0
assert not any(st)
res["config3_256x(64,16)"] = {"gpu_single_call_ms": round(dt * 1e3, 3), "gpu_proofs_per_s_single_stream": round(count / dt), "values_per_s_single_stream": round(count * m / dt),
                              "cpu_oracle_proofs_per_s_16_threads": round(base / dtc, 1)}
gens.close()

# ---- config 4: MSM sweep
nmax = 1 << max_lg
uniform = hashlib.shake_256(b"GeneratorsChain" + b"G" + (0).to_bytes(4, "little")).digest(64 * nmax)
points = ctx.from_uniform_bytes(uniform)                         # the first nmax points of the party-0 G chain, compressed
assert points[:32] == bytes.fromhex("fc3b25801422672a6a8d3adb5d8457d4301fe92324b4fc56ae934c8713ddfe2d")    # SURVEY.md §8c (iii)
K = 8
scal = orc.random_scalars(bytes([0x2a]) * 32, K * nmax)          # ChaCha20 stream, 64 B wide-reduced per scalar
sweep = {}
for lg in range(10, max_lg + 1):
    nn = 1 << lg
    sc = scal[:32 * K * nn]; pp = points[:32 * nn] * K
    offs = [i * nn for i in range(K + 1)]
    status, outs = ctx.msm_batch(sc, pp, offs)
    assert not any(status)
    dt = med(lambda: ctx.msm_batch(sc, pp, offs), 3)
    t0 = time.perf_counter(); want = orc.msm(sc[:32 * nn], pp[:32 * nn]); dtc = time.perf_counter() - t0
    assert want == (0, outs[0]), lg
    sweep[f"2^{lg}"] = {"msms_per_call": K, "ms_per_call": round(dt * 1e3, 2), "terms_per_s": round(K * nn / dt), "cpu_oracle_1thread_terms_per_s": round(nn / dtc),
                        "first_result_equals_oracle": True}
res["config4_msm_sweep"] = sweep
print(json.dumps(res))
