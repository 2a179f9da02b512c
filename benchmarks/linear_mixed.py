"""LinearProofs of different lengths: one bp_linear_verify_mixed call (bp.linear_verify_mixed) against what a caller does without it, sort
the proofs by n, make one bp_linear_verify_batch call per length over the same resident set and put the verdicts back in input order
(the sort and the un-permute are inside the timed region).

Workloads, 1024 proofs each, over one set of 1024 + 2 points, 16 distinct valid proofs per length tiled and shuffled:
  mix_4_2_1     lengths {64, 256, 1024} in proportion 4 : 2 : 1
  mix_all_11    every power-of-two length from 1 to 1024, about 93 proofs each
  mix_4_2_1_bad mix_4_2_1 with one proof flipped ("a"), so both forms run their reject paths
  single_256    one length, n = 256: the mixed call against verify_batch, the cost of the mixed path where the loop is one call
Each form is timed as the median of REPS alternating blocking calls (host clock around the call, which synchronises).  Prints the device and
its power limit, then one JSON line per workload: ms per call for both forms and their ratio, whether the verdicts agree, launches per call,
the combined MSM's terms, and the per-kernel time of one mixed call (bp_prof_report, in a profiled call of its own).
Usage: python benchmarks/linear_mixed.py [repetitions]"""
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

SEED = bytes(range(32))
L_ORDER = 2**252 + 27742317777372353535851937790883648493
COUNT = 1024


def le(x):
    return x.to_bytes(32, "little")


def make_proofs(ctx, G, F, B, n, distinct=16):
    rnd = random.Random(n)
    out = []
    for j in range(distinct):
        a = [rnd.randrange(L_ORDER) for _ in range(n)]; b = [rnd.randrange(L_ORDER) for _ in range(n)]; r = rnd.randrange(L_ORDER)
        Gn = G[:32 * n]
        rc, C = ctx.msm(b"".join(map(le, a)) + le(r) + le(sum(x * y for x, y in zip(a, b)) % L_ORDER), Gn + B + F)
        assert rc == 0
        label = b"linear mixed bench %d %d" % (n, j)
        rc, proof = bp.linear_create(ctx, bp.Transcript(label), le(j + 1), C, le(r), b"".join(map(le, a)), b"".join(map(le, b)), Gn, F, B)
        assert rc == 0
        out.append((label, proof, C, b"".join(map(le, b))))
    return out


def workload(pool, counts, seed):
    raw = [pool[n][j % len(pool[n])] for n, c in counts.items() for j in range(c)]
    random.Random(seed).shuffle(raw)
    return raw


def per_length(ctx, points, items):
    """what a caller does without the mixed call: sort by n, one blocking call per length, verdicts back in input order"""
    groups = {}
    for j, it in enumerate(items):
        groups.setdefault(len(it[3]) // 32, []).append(j)
    out = [None] * len(items)
    for n in sorted(groups):
        idx = groups[n]
        for j, v in zip(idx, bp.linear_verify_batch(ctx, points, n, [items[j] for j in idx], SEED)):
            out[j] = v
    return out


def main():
    nums = [a for a in sys.argv[1:] if a.isdigit()]
    reps = int(nums[0]) if nums else 9
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    ctx = bp.Context(0)
    gens = bp.Gens(ctx, 1024, 1)
    G = b"".join(gens.get(0, 0, i) for i in range(1024))
    F, B = gens.get(2), gens.get(3)                   # F = pc_gens.B, B = pc_gens.B_blinding
    gens.close()
    points = bp.PointSet(ctx, B + F + G)
    ns = [1 << k for k in range(11)]
    pool = {n: make_proofs(ctx, G, F, B, n) for n in ns}
    per = COUNT // 11
    loads = {
        "mix_4_2_1": workload(pool, {64: 585, 256: 293, 1024: 146}, 1),
        "mix_all_11": workload(pool, {n: per + (1 if j < COUNT - 11 * per else 0) for j, n in enumerate(ns)}, 2),
        "single_256": workload(pool, {256: COUNT}, 3),
    }
    bad = list(loads["mix_4_2_1"])
    label, proof, C, b = bad[500]
    k = (len(b) // 32).bit_length() - 1
    pr = bytearray(proof); pr[64 * k + 32] ^= 1
    bad[500] = (label, bytes(pr), C, b)
    loads["mix_4_2_1_bad"] = bad
    for name, raw in loads.items():
        items = [(bp.Transcript(lab), p, C, b) for lab, p, C, b in raw]
        assert len(items) == COUNT
        forms = {"mixed": lambda: bp.linear_verify_mixed(ctx, points, items, SEED), "per_length": lambda: per_length(ctx, points, items)}
        ref = {f: fn() for f, fn in forms.items()}                  # warm both, and their verdicts
        same = ref["mixed"] == ref["per_length"]
        assert same, name
        assert ref["mixed"].count(0) == COUNT - (1 if name.endswith("_bad") else 0)
        times = {f: [] for f in forms}
        for _ in range(reps):
            for f, fn in forms.items():
                t0 = time.perf_counter(); fn(); times[f].append(time.perf_counter() - t0)
        launches = {}
        for f, fn in forms.items():
            l0 = ctx.launches; fn(); launches[f] = ctx.launches - l0
        ctx.prof_enable(True)
        forms["mixed"]()
        prof = ctx.prof_report()
        ctx.prof_enable(False)
        med = {f: statistics.median(v) for f, v in times.items()}
        ks = sorted({(len(it[3]) // 32).bit_length() - 1 for it in items})
        terms = (1 << ks[-1]) + 2 + sum(2 + 2 * ((len(it[3]) // 32).bit_length() - 1) for it in items)
        print(json.dumps({"workload": name, "proofs": COUNT, "lengths": [1 << k for k in ks], "verdicts_identical": same,
                          "ms_per_call": {f: round(v * 1e3, 3) for f, v in med.items()},
                          "ms_range": {f: [round(min(v) * 1e3, 3), round(max(v) * 1e3, 3)] for f, v in times.items()},
                          "per_length_over_mixed": round(med["per_length"] / med["mixed"], 3),
                          "launches_per_call": launches, "mixed_msm_terms": terms,
                          "mixed_kernel_ms": {k_: [round(t, 3), n_] for k_, (t, n_) in sorted(prof.items(), key=lambda x: -x[1][0])}}), flush=True)
    points.close()
    ctx.close()


if __name__ == "__main__":
    main()
