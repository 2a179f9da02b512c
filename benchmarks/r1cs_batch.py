"""R1CS batch verification (bp.r1cs_verify_batch: one combined MSM per batch) against a loop of bp.r1cs_verify (one mega-check MSM per
proof) on the same proofs.  Workloads: 1024 x 8-shuffle, 256 x 64-bit range gadget, 8 x 2049-shuffle (4096 multipliers), 4 x the
BASELINE config-5 shuffle (2^16 multipliers).  Each batch holds a few distinct proofs, repeated; every proof of a batch has its own
batching weight.  Prints the device and its power limit, then one JSON line per workload: proofs/s of both forms, the host phase and
the engine call of the batch, the MSM terms of both forms, and whether the verdicts are identical.
    python benchmarks/r1cs_batch.py [--reps R] [--only NAME]"""
import argparse, json, os, random, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bulletproofs_b200 as bp

L_ORDER = 2**252 + 27742317777372353535851937790883648493


def pow2(n):
    p = 1
    while p < n:
        p <<= 1
    return p


def shuffle_tr(k):
    t = bp.Transcript(b"ShuffleBenchmark"); t.append_message(b"dom-sep", b"ShuffleProof"); t.append_u64(b"k", k); return t


def make_shuffles(ctx, gens, k, distinct, rnd):
    out = []
    for _ in range(distinct):
        inp = [rnd.randrange(1 << 64) for _ in range(k)]; o = inp[:]; rnd.shuffle(o)
        bl = b"".join(rnd.randrange(L_ORDER).to_bytes(32, "little") for _ in range(2 * k))
        rc, proof, V = bp.r1cs_prove(ctx, gens, shuffle_tr(k), bp.GADGET_SHUFFLE, inp + o, bl)
        assert rc == 0
        out.append((shuffle_tr(k), bp.GADGET_SHUFFLE, V, proof, 0))
    # other terms: A_I1, A_O1, S1, A_I2, A_O2, S2, 2k V, T_1, T_3..T_6, B, B~, lg(padded_n) L and R
    N = pow2(2 * (k - 1)); return out, N, 13 + 2 * k + 2 * (N.bit_length() - 1)


def make_ranges(ctx, gens, n, distinct, rnd):
    out = []
    for _ in range(distinct):
        v = rnd.randrange(1 << n)
        rc, proof, V = bp.r1cs_prove(ctx, gens, bp.Transcript(b"RangeProofBenchmark"), bp.GADGET_RANGE, [v], rnd.randrange(L_ORDER).to_bytes(32, "little"), param=n, aux=v)
        assert rc == 0
        out.append((bp.Transcript(b"RangeProofBenchmark"), bp.GADGET_RANGE, V, proof, n))
    N = pow2(n); return out, N, 14 + 2 * (N.bit_length() - 1)


WORKLOADS = [("shuffle8 x 1024", "shuffle", 8, 1024, 16), ("range64 x 256", "range", 64, 256, 16),
             ("shuffle2049 x 8", "shuffle", 2049, 8, 2), ("shuffle32769 x 4 (config 5)", "shuffle", 32769, 4, 1)]


def device_line():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "unknown"
    return {"device": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default=None)
    args = ap.parse_args()
    print(json.dumps(device_line()), flush=True)
    ctx = bp.Context(0); rnd = random.Random(1)
    for name, kind, size, count, distinct in WORKLOADS:
        if args.only and args.only not in name:
            continue
        cap = pow2(2 * (size - 1)) if kind == "shuffle" else pow2(size)
        gens = bp.Gens(ctx, max(cap, 16), 1)
        base, N, other = (make_shuffles if kind == "shuffle" else make_ranges)(ctx, gens, size, distinct, rnd)
        items = [base[i % distinct] for i in range(count)]
        seed = bytes(range(32))
        batch_t, prep_t, dev_t = [], [], []
        got = bp.r1cs_verify_batch(ctx, gens, items, ext_seed=seed)                          # warm-up: arenas, module load
        for _ in range(args.reps):
            tm = {}
            t0 = time.perf_counter(); got = bp.r1cs_verify_batch(ctx, gens, items, ext_seed=seed, timings=tm); batch_t.append(time.perf_counter() - t0)
            prep_t.append(tm["prepare"]); dev_t.append(tm["device"])
        loop_t = []
        for _ in range(max(1, args.reps - 1)):
            t0 = time.perf_counter()
            want = [bp.r1cs_verify(ctx, gens, it[0], it[1], it[2], it[3], param=it[4], ext_seed=seed) for it in items]
            loop_t.append(time.perf_counter() - t0)
        assert got == want == [0] * count, (got, want)
        tb, tl = statistics.median(batch_t), statistics.median(loop_t)
        print(json.dumps({"workload": name, "proofs": count, "padded_n": N, "batch_s": round(tb, 4), "loop_s": round(tl, 4),
                          "batch_proofs_per_s": round(count / tb, 1), "loop_proofs_per_s": round(count / tl, 1), "speedup": round(tl / tb, 2),
                          "batch_host_prepare_s": round(statistics.median(prep_t), 4), "batch_engine_s": round(statistics.median(dev_t), 4),
                          "batch_msm_terms": 2 * N + count * other, "loop_msm_terms": count * (2 * N + other), "verdicts_identical": got == want}), flush=True)
        gens.close()
    ctx.close()


if __name__ == "__main__":
    main()
