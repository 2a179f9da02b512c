"""One bp.verify_mixed call against what a caller does without it: sort the proofs by (n, m), one bp.verify_batch per class, and put
the verdicts back in input order (the sort and the un-permute are timed).  Same seeded proofs, same batching seed for both forms.

Workloads:
  tx-1024, tx-8192  n = 64, m in {1, 2, 4, 8} in proportions 8 : 4 : 2 : 1.  This stands for a block of confidential transactions where
                    most transactions have one or two outputs; the proportions are an assumption, not a measured distribution.
  grid-24x33        every (n, m) of the reference grid, n in {8, 16, 32, 64} x m in {1, 2, 4, 8, 16, 32}, 33 proofs each: many small
                    classes.
Prints the device and its power limit, then one JSON line per workload: proofs/s of both forms (median of alternating repetitions), MSM
terms and kernel launches per call of both forms, and whether the verdicts are identical.  The proofs are made with bp.prove_many from
DISTINCT witnesses per class, tiled.  Usage: python benchmarks/mixed_verify.py [repetitions] [--profile]"""
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bulletproofs_b200 as bp

LABEL = b"AggregateRangeProofBenchmark"
DISTINCT = 4
L_ORDER = 2 ** 252 + 27742317777372353535851937790883648493


def class_items(ctx, gens, n, m, count, seed):
    rnd = random.Random(seed)
    vals = [rnd.randrange(1 << n) for _ in range(DISTINCT * m)]
    bl = b"".join(rnd.randrange(L_ORDER).to_bytes(32, "little") for _ in range(DISTINCT * m))
    seeds = b"".join(rnd.randrange(1 << 256).to_bytes(32, "little") for _ in range(DISTINCT))
    st, proofs, V = bp.prove_many(ctx, gens, bp.Transcript(LABEL), vals, bl, n, m, seeds)
    assert st == [0] * DISTINCT
    plen = len(proofs) // DISTINCT
    return [(proofs[(i % DISTINCT) * plen:(i % DISTINCT + 1) * plen], V[(i % DISTINCT) * 32 * m:(i % DISTINCT + 1) * 32 * m], n) for i in range(count)]


def per_class(ctx, gens, items, seed):
    """today's form: sort by (n, m), one verify_batch per class, verdicts back in input order"""
    order = sorted(range(len(items)), key=lambda i: (items[i][2], len(items[i][1])))
    out = [0] * len(items)
    j = 0
    while j < len(order):
        n, m = items[order[j]][2], len(items[order[j]][1]) // 32
        e = j
        while e < len(order) and items[order[e]][2] == n and len(items[order[e]][1]) // 32 == m:
            e += 1
        idx = order[j:e]
        got = bp.verify_batch(ctx, gens, bp.Transcript(LABEL), b"".join(items[i][0] for i in idx), b"".join(items[i][1] for i in idx), n, m, len(idx), seed=seed)
        for i, v in zip(idx, got):
            out[i] = v
        j = e
    return out


def terms(items):
    classes = {}
    for p, V, n in items:
        classes.setdefault((n, len(V) // 32), []).append(p)
    t = 0
    for (n, m), ps in classes.items():
        k = (n * m).bit_length() - 1
        t += 2 + 2 * n * m + len(ps) * (4 + 2 * k + m)
    return t


def main():
    nums = [a for a in sys.argv[1:] if a.isdigit()]
    reps = int(nums[0]) if nums else 15
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    ctx = bp.Context(0)
    gens = bp.Gens(ctx, 64, 32)
    workloads = {}
    for total in (1024, 8192):
        unit = total // 15
        sizes = {1: total - 7 * unit, 2: 4 * unit, 4: 2 * unit, 8: unit}         # 8 : 4 : 2 : 1, the remainder in m = 1
        workloads[f"tx-{total}"] = [it for m, c in sizes.items() for it in class_items(ctx, gens, 64, m, c, 100 + m)]
    workloads["grid-24x33"] = [it for n in (8, 16, 32, 64) for m in (1, 2, 4, 8, 16, 32) for it in class_items(ctx, gens, n, m, 33, 1000 + 64 * n + m)]
    seed = bytes(range(32))
    for name, items in workloads.items():
        random.Random(7).shuffle(items)
        mixed_v = bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), items, seed=seed)
        loop_v = per_class(ctx, gens, items, seed)
        l0 = ctx.launches; bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), items, seed=seed); mixed_l = ctx.launches - l0
        l0 = ctx.launches; per_class(ctx, gens, items, seed); loop_l = ctx.launches - l0
        tm, tl = [], []
        for _ in range(reps):           # alternating
            t0 = time.perf_counter(); bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), items, seed=seed); tm.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); per_class(ctx, gens, items, seed); tl.append(time.perf_counter() - t0)
        mm, ml = statistics.median(tm), statistics.median(tl)
        print(json.dumps({"workload": name, "proofs": len(items), "classes": len({(n, len(V)) for _, V, n in items}),
                          "mixed_proofs_per_s": round(len(items) / mm), "per_class_proofs_per_s": round(len(items) / ml),
                          "mixed_ms": round(mm * 1e3, 3), "per_class_ms": round(ml * 1e3, 3),
                          "mixed_ms_range": [round(min(tm) * 1e3, 3), round(max(tm) * 1e3, 3)], "per_class_ms_range": [round(min(tl) * 1e3, 3), round(max(tl) * 1e3, 3)],
                          "msm_terms": {"mixed": terms(items), "per_class": terms(items)},      # both: one static row per class, every dynamic term
                          "launches": {"mixed": mixed_l, "per_class": loop_l},
                          "verdicts_identical": mixed_v == loop_v, "all_accepted": mixed_v == [0] * len(items)}), flush=True)
        if "--profile" in sys.argv:     # per-kernel times (CUDA events) of one call of each form, in a run of their own
            ctx.prof_enable(True)
            bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), items, seed=seed)
            pm = ctx.prof_report()
            per_class(ctx, gens, items, seed)
            pl = ctx.prof_report()
            ctx.prof_enable(False)
            print(json.dumps({"workload": name, "profile_ms": {"mixed": {k: round(v[0], 3) for k, v in pm.items()},
                                                               "per_class": {k: round(v[0], 3) for k, v in pl.items()}}}), flush=True)
    gens.close()
    ctx.close()


if __name__ == "__main__":
    main()
