"""Mixed-geometry verification as a service: a reserved mix (bp.MixedVerifier: captured graph, begin / finish) against the blocking
bp.verify_mixed loop, with a fixed-geometry bp.BatchVerifier over the same number of (64, 1) proofs as the ceiling.

Workloads (the proofs of benchmarks/mixed_verify.py):
  tx-1024, tx-8192  n = 64, m in {1, 2, 4, 8} in proportions 8 : 4 : 2 : 1, each reserved at exactly its class sizes
  tx-8192-half      the tx-8192 mix reserved, each call filling half of every class (inert slots)
  grid-24x33        every (n, m) of the reference grid, 33 proofs each
Forms, proofs/s over the same calls (median of alternating repetitions):
  blocking          bp.verify_mixed on a context without a reserved mix (direct launches, synchronised)
  service_1/4/8     bp.MixedVerifier on 1, 4 or 8 contexts: begin on every context, then finish on each in turn
  fixed_64x1        bp.BatchVerifier(64, 1) reserved at the same number of proofs (8 batches when it divides by 8), begin / finish
Prints the device and its power limit, then one JSON line per workload, with whether every form returned the same verdicts, and one line
breaking one blocking tx-8192 call down into Python packing, the host side of a reserved begin (planning, staging, queueing), the H2D copy
of its input bytes, per-kernel time (bp_prof_report, a run of its own) and the rest (launch gaps and synchronisation).
Usage: python benchmarks/mixed_service.py [repetitions]"""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import bulletproofs_b200 as bp
from mixed_verify import LABEL, class_items

SEED = bytes(range(32))


def workloads(ctx, gens):
    out = {}
    for total in (1024, 8192):
        unit = total // 15
        sizes = {1: total - 7 * unit, 2: 4 * unit, 4: 2 * unit, 8: unit}
        by_class = {(64, m): class_items(ctx, gens, 64, m, c, 100 + m) for m, c in sizes.items()}
        out[f"tx-{total}"] = ({k: len(v) for k, v in by_class.items()}, [it for v in by_class.values() for it in v])
        if total == 8192:
            out["tx-8192-half"] = ({k: len(v) for k, v in by_class.items()}, [it for v in by_class.values() for it in v[:len(v) // 2]])
    grid = {(n, m): class_items(ctx, gens, n, m, 33, 1000 + 64 * n + m) for n in (8, 16, 32, 64) for m in (1, 2, 4, 8, 16, 32)}
    out["grid-24x33"] = ({k: 33 for k in grid}, [it for v in grid.values() for it in v])
    return out


def timed(fn, calls):
    t0 = time.perf_counter()
    out = fn()
    return out, calls / (time.perf_counter() - t0)


def main():
    nums = [a for a in sys.argv[1:] if a.isdigit()]
    reps = int(nums[0]) if nums else 7
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    base = bp.Context(0)
    gens = bp.Gens(base, 64, 32)
    import random
    for name, (mix, items) in workloads(base, gens).items():
        random.Random(7).shuffle(items)
        N = len(items)
        svcs = []
        for _ in range(8):
            c = bp.Context(0)
            g = bp.Gens(c, 64, 32)
            svcs.append((c, g, bp.MixedVerifier(c, g, mix)))
        one = [it for it in items if len(it[1]) == 32 and it[2] == 64][:1] or [class_items(base, gens, 64, 1, 1, 5)[0]]
        nb = 8 if N % 8 == 0 else 1
        fixed = bp.BatchVerifier(base, gens, bp.Transcript(LABEL), 64, 1, N // nb, nb)
        fproofs, fV = one[0][0] * N, one[0][1] * N

        def blocking():
            return bp.verify_mixed(base, gens, bp.Transcript(LABEL), items, seed=SEED)

        def service(k):
            def run():
                for c, g, v in svcs[:k]:
                    v.begin(bp.Transcript(LABEL), items, seed=SEED)
                return [v.finish() for _, _, v in svcs[:k]]
            return run

        def fixed_run():
            fixed.begin(fproofs, fV, SEED)
            return fixed.finish()

        forms = {"blocking": (blocking, 1), "service_1": (service(1), 1), "service_4": (service(4), 4), "service_8": (service(8), 8), "fixed_64x1": (fixed_run, 1)}
        ref = blocking()
        same = True
        for f, (fn, calls) in forms.items():          # warm every form, check its verdicts
            out = fn()
            if f.startswith("service"):
                same &= all(o == ref for o in out)
        rates = {f: [] for f in forms}
        for _ in range(reps):
            for f, (fn, calls) in forms.items():
                _, r = timed(fn, calls)
                rates[f].append(r * N)
        launches = {}
        for f in ("blocking", "service_1"):
            c = base if f == "blocking" else svcs[0][0]
            l0 = c.launches; forms[f][0](); launches[f] = c.launches - l0
        print(json.dumps({"workload": name, "proofs": N, "classes": len(mix),
                          "proofs_per_s": {f: round(statistics.median(v)) for f, v in rates.items()},
                          "proofs_per_s_range": {f: [round(min(v)), round(max(v))] for f, v in rates.items()},
                          "launches_per_call": launches, "verdicts_identical": same, "all_accepted": ref == [0] * N}), flush=True)
        if name == "tx-8192":
            breakdown(base, gens, svcs[0], items, reps)
        del fixed
        for c, g, v in svcs:
            g.close(); c.close()
    gens.close()
    base.close()


def breakdown(base, gens, svc, items, reps):
    """one blocking verify_mixed call at tx-8192, in parts (median over reps, each measured in its own loop)"""
    import torch
    wall, pack, begin_host, h2d = [], [], [], []
    blob_p = b"".join(p for p, _, _ in items)
    blob_c = b"".join(V for _, V, _ in items)
    c, g, v = svc
    for _ in range(reps):
        t0 = time.perf_counter(); bp.verify_mixed(base, gens, bp.Transcript(LABEL), items, seed=SEED); wall.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); bp._mixed_args(items); pack.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); v.begin(bp.Transcript(LABEL), items, seed=SEED); begin_host.append(time.perf_counter() - t0); v.finish()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        torch.frombuffer(bytearray(blob_p), dtype=torch.uint8).cuda(); torch.frombuffer(bytearray(blob_c), dtype=torch.uint8).cuda()
        torch.cuda.synchronize(); h2d.append(time.perf_counter() - t0)
    base.prof_enable(True)
    bp.verify_mixed(base, gens, bp.Transcript(LABEL), items, seed=SEED)
    prof = base.prof_report()
    base.prof_enable(False)
    kern = sum(t for t, _ in prof.values())
    med = lambda xs: round(statistics.median(xs) * 1e3, 3)
    print(json.dumps({"breakdown": "tx-8192 blocking verify_mixed", "wall_ms": med(wall), "python_pack_ms": med(pack),
                      "reserved_begin_host_ms": med(begin_host), "h2d_input_copy_ms_torch": med(h2d), "kernel_sum_ms": round(kern, 3),
                      "rest_ms": round(med(wall) - med(pack) - med(h2d) - kern, 3),
                      "kernels_ms": {k: [round(t, 3), n] for k, (t, n) in sorted(prof.items(), key=lambda kv: -kv[1][0])}}), flush=True)


if __name__ == "__main__":
    main()
