"""Single-proof latency: the fused single-proof kernel (k_rp_single, one cluster per proof, one launch) against the launch-group pipeline
in the same build (verify_group(count, 1)) and against one CPU core (the oracle's verify_multiple on its fastest field backend, the
cpu_baseline path of bench.py), for small calls at several geometries.  The table it prints sets the routing constants of
bp_rangeproof_verify_batch (RP_ROUTE_MAX_COUNT, RP_ROUTE_MAX_K in bpmsm.cu): route only where the fused column is the faster one.

    python benchmarks/single_proof.py [--reps 50] [--out results.json]

Every time is the wall time of one blocking call (inputs from host memory, verdicts back on the host), median and p99 over --reps calls
after warm-up.  Kernel time is from bp_prof (CUDA events around each launch) in a separate pass."""
import argparse
import ctypes
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

LABEL = b"single proof latency"


def le(x, n=32):
    return x.to_bytes(n, "little")


def stats(ts):
    ts = sorted(ts)
    return {"median_us": 1e6 * statistics.median(ts), "p99_us": 1e6 * ts[min(len(ts) - 1, int(0.99 * len(ts)))]}


def timed(fn, reps, warm=5):
    for _ in range(warm):
        fn()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); out.append(time.perf_counter() - t0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write every row as JSON to this file")
    a = ap.parse_args()
    import bulletproofs_b200 as bp
    from oracle_binding import Oracle, L_ORDER as l
    orc = Oracle()
    ctx = bp.Context(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    # the fastest single-thread CPU backend, as bench.py's cpu_baseline selects it
    backends = [b for b in ("ifma", "avx2", "u64") if orc.set_backend(b) == 0]
    geoms = [(n, m) for n in (8, 16, 32, 64) for m in (1, 2, 4, 8, 16, 32, 64, 128) if n * m <= 1024]
    counts = {(64, 1): (1, 2, 4, 8, 12, 16, 32), (64, 4): (1, 2, 4, 8, 16), (16, 16): (1, 2, 4, 8, 16), (64, 16): (1, 2, 4)}
    rows = []
    for n, m in geoms:
        og = orc.gens(n, m)
        gens = bp.Gens(ctx, n, m)
        for count in counts.get((n, m), (1,)):
            rnd = random.Random(n * 1000 + m * 10 + count)
            vals = [rnd.randrange(1 << n) for _ in range(count * m)]
            blind = b"".join(le(rnd.randrange(l)) for _ in range(count * m))
            seeds = b"".join(le(i + 1, 8) + bytes(24) for i in range(count))
            proofs, Vs = orc.prove_many(og, orc.transcript(LABEL), vals, blind, n, m, seeds, nthreads=8)
            plen = len(proofs) // count
            t = bp.Transcript(LABEL).to_bytes()
            out = ctypes.create_string_buffer(count)

            def fused():
                ctx._check(bp.lib().bp_debug_rp_single_verify(ctx._h, gens._h, t, proofs, plen, Vs, n, m, count, bytes(32), out))
                return list(out.raw)

            def pipe():
                return bp.verify_group(ctx, gens, bp.Transcript(LABEL), proofs, Vs, n, m, count, 1, seed=bytes(32))[0]

            def routed():
                return bp.verify_batch(ctx, gens, bp.Transcript(LABEL), proofs, Vs, n, m, count, seed=bytes(32))

            assert fused() == pipe() == routed() == [0] * count
            row = {"n": n, "m": m, "count": count}
            row["fused"], row["pipeline"], row["routed"] = (stats(timed(f, a.reps)) for f in (fused, pipe, routed))
            for name, f in (("fused", fused), ("pipeline", pipe), ("routed", routed)):
                l0 = ctx.launches; f(); row[name]["launches"] = ctx.launches - l0
            ctx.prof_enable(True)
            for _ in range(10):
                fused()
            rep = ctx.prof_report(); ctx.prof_enable(False)
            ms, cnt = rep.get("k_rp_single", (0.0, 0))
            row["fused"]["kernel_us"] = 1e3 * ms / max(cnt, 1)
            if count == 1:
                cpu = {}
                ot = orc.transcript(LABEL)
                for b in backends:
                    orc.set_backend(b)
                    cpu[b] = stats(timed(lambda: orc.verify_many(og, ot, proofs, plen, Vs, n, m, 1, nthreads=1), max(10, a.reps // 2), warm=2))
                best = min(cpu, key=lambda b: cpu[b]["median_us"])
                row["cpu_1core"] = dict(cpu[best], backend=best)
            rows.append(row)
            c = row.get("cpu_1core", {})
            print(f"({n:2},{m:3}) x{count:2}: fused {row['fused']['median_us']:8.1f} us (p99 {row['fused']['p99_us']:8.1f}, kernel "
                  f"{row['fused']['kernel_us']:7.1f}, {row['fused']['launches']} launch) | pipeline {row['pipeline']['median_us']:8.1f} us "
                  f"(p99 {row['pipeline']['p99_us']:8.1f}, {row['pipeline']['launches']} launches) | routed {row['routed']['median_us']:8.1f}"
                  + (f" | cpu 1 core ({c['backend']}) {c['median_us']:8.1f} us" if c else ""), flush=True)
        gens.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)
    print(json.dumps({"card": card, "n_rows": len(rows)}))
    ctx.close()


if __name__ == "__main__":
    main()
