"""LinearProof latency of small calls: the fused path (k_lin_single: host transcript replay, one thread-block cluster per proof, one launch)
against the pipeline in the same build (both forced through bp_debug_linear_verify_path, paths 1 and 2), the routed public call
(bp_linear_verify_batch), the C++ mirror's loop of bp.linear_verify (host transcript plus bp_msm per proof) and one CPU core (the
oracle's linear_verify, one proof after another).  The table it prints sets the routing constants LIN_ROUTE_MAX_COUNT and LIN_ROUTE_MAX_N
(linear_single.cuh): route only where the fused column is the faster one.

    python benchmarks/linear_single.py [--reps 40] [--out results.json]

Every time is the wall time of one blocking call (inputs from host memory, verdicts back on the host), median and p99 over --reps calls
after warm-up.  Kernel time is from bp_prof (CUDA events around each launch) in a separate pass."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ROWS = [(n, 1) for n in (2, 8, 64, 256, 1024)] + [(n, c) for n in (64, 1024) for c in (2, 4, 8, 16, 32)]


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
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--out", default=None, help="also write every row as JSON to this file")
    a = ap.parse_args()
    import bulletproofs_b200 as bp
    from oracle_binding import Oracle
    from test_linear_verify_batch import _gens, gpu_proofs
    orc = Oracle()
    ctx = bp.Context(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(card, flush=True)
    backends = [b for b in ("ifma", "avx2", "u64") if orc.set_backend(b) == 0]
    rows, verifiers = [], {}
    for n, count in ROWS:
        if n not in verifiers:
            verifiers[n] = bp.LinearVerifier(ctx, *_gens(orc, n))
        V = verifiers[n]
        G, F, B = _gens(orc, n)
        proofs, _ = gpu_proofs(bp, ctx, orc, n, count, tag="bench")
        items = [p.item(bp) for p in proofs]
        seed = bytes(32)

        def fused():
            return ctx.debug_linear_verify_path(V.points, n, items, 1, seed)

        def pipe():
            return ctx.debug_linear_verify_path(V.points, n, items, 2, seed)

        def routed():
            return bp.linear_verify_batch(ctx, V.points, n, items, seed)

        def mirror():
            return [bp.linear_verify(ctx, bp.Transcript(p.label), p.proof, p.C, G, F, B, p.b) for p in proofs]

        def cpu():
            return [orc.linear_verify(orc.transcript(p.label), p.proof, p.C, G, F, B, p.b) for p in proofs]

        assert fused() == pipe() == routed() == mirror() == cpu() == [0] * count
        row = {"n": n, "count": count}
        for name, f in (("fused", fused), ("pipeline", pipe), ("routed", routed), ("mirror", mirror)):
            row[name] = stats(timed(f, a.reps))
            l0 = ctx.launches; f(); row[name]["launches"] = ctx.launches - l0
        ctx.prof_enable(True)
        for _ in range(10):
            fused()
        rep = ctx.prof_report(); ctx.prof_enable(False)
        ms, cnt = rep.get("k_lin_single", (0.0, 0))
        row["fused"]["kernel_us"] = 1e3 * ms / max(cnt, 1)
        best = None
        for b in backends:
            orc.set_backend(b)
            s = stats(timed(cpu, max(10, a.reps // 4), warm=2))
            if best is None or s["median_us"] < best["median_us"]:
                best = dict(s, backend=b)
        row["cpu_1core"] = best
        rows.append(row)
        f_, p_, r_, m_, c_ = (row[k] for k in ("fused", "pipeline", "routed", "mirror", "cpu_1core"))
        print(f"n {n:5} x{count:3}: fused {f_['median_us']:8.1f} us (p99 {f_['p99_us']:8.1f}, kernel {f_['kernel_us']:8.1f}) | pipeline "
              f"{p_['median_us']:8.1f} (p99 {p_['p99_us']:8.1f}, {p_['launches']} launches) | routed {r_['median_us']:8.1f} ({r_['launches']}) | "
              f"mirror {m_['median_us']:8.1f} (p99 {m_['p99_us']:8.1f}) | cpu 1 core ({c_['backend']}) {c_['median_us']:9.1f}", flush=True)
    for V in verifiers.values():
        V.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)
    print(json.dumps({"card": card, "n_rows": len(rows)}))
    ctx.close()


if __name__ == "__main__":
    main()
