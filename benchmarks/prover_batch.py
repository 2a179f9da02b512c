"""Prover timings on one GPU (BASELINE configs 1 and 5 are the parity configs; these are their speeds):
  (32,1) and (64,1) range proofs: one proof at a time (latency) and batches through RangeProof::prove_many (every group operation
  batched across the proofs, one unfolded inner-product session for all), against the CPU oracle on one thread and on all cores.
Prints one JSON object.  Usage: python benchmarks/prover_batch.py [batch sizes...]"""
import json, os, random, statistics, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bulletproofs_b200 as bp
import bench
from oracle_binding import Oracle, L_ORDER

batches = [int(x) for x in sys.argv[1:]] or [1, 16, 64, 256, 1024]
orc = Oracle(); orc.set_backend("auto"); ctx = bp.Context(0); rnd = random.Random(3); LABEL = bench.LABEL
cores = bench.effective_cores()
out = {"cpu_backend": orc.backend_name(), "cores": cores}
for n, m in ((32, 1), (64, 1)):
    og = orc.gens(n, m); gens = bp.Gens(ctx, n, m); res = {}
    for B in batches:
        vals = [rnd.randrange(1 << n) for _ in range(B * m)]; bl = b"".join(rnd.randrange(L_ORDER).to_bytes(32, "little") for _ in range(B * m))
        seeds = b"".join(i.to_bytes(8, "little") + bytes(24) for i in range(B))
        st, proofs, V = bp.prove_many(ctx, gens, bp.Transcript(LABEL), vals, bl, n, m, seeds)
        want, wantV = orc.prove_many(og, orc.transcript(LABEL), vals, bl, n, m, seeds, nthreads=cores)
        assert st == [0] * B and proofs == want and V == wantV
        ts = []
        for _ in range(5):
            t0 = time.perf_counter(); bp.prove_many(ctx, gens, bp.Transcript(LABEL), vals, bl, n, m, seeds); ts.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); orc.prove_many(og, orc.transcript(LABEL), vals, bl, n, m, seeds, nthreads=cores); cpu_all = time.perf_counter() - t0
        t0 = time.perf_counter(); orc.prove_many(og, orc.transcript(LABEL), vals[:min(B, 8) * m], bl[:32 * m * min(B, 8)], n, m, seeds[:32 * min(B, 8)], nthreads=1); cpu_1 = (time.perf_counter() - t0) / min(B, 8)
        res[f"batch_{B}"] = {"gpu_ms_per_call": round(1e3 * statistics.median(ts), 3), "gpu_us_per_proof": round(1e6 * statistics.median(ts) / B, 1),
                             "cpu_oracle_us_per_proof_1_thread": round(1e6 * cpu_1, 1), f"cpu_oracle_us_per_proof_{cores}_threads": round(1e6 * cpu_all / B, 1), "bytes_equal_oracle": True}
    out[f"({n},{m})"] = res
    gens.close()
print(json.dumps(out))
