"""LinearProof verification: bp.LinearVerifier.verify_batch (one device call, transcripts replayed on the device, one combined MSM) against a
loop of bp.linear_verify (the single-proof path: host transcript, one bp_msm per proof) over the same proofs.

For n in {64, 256, 1024} and count in {1, 64, 1024}: proofs from bp.linear_create with fixed seeds (a pool of distinct proofs, each under
its own transcript label, repeated up to count), the median of --reps synchronised calls of each form, and a check that both return the
same verdicts.  Prints the device, its power limit and the per-kernel times of one profiled batch call.

    python benchmarks/linear_verify_batch.py [--reps 5] [--pool 64]
"""
import argparse
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

import bulletproofs_b200 as bp  # noqa: E402
from oracle_binding import L_ORDER as l, Oracle  # noqa: E402


def le(x, n=32):
    return x.to_bytes(n, "little")


def device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception as e:                                          # noqa: BLE001
        return f"unknown ({e})"


def make_proofs(ctx, orc, n, pool):
    g = orc.gens(n, 1)
    G = b"".join(orc.gens_get(g, 0, 0, i) for i in range(n)); F, B = orc.pedersen()
    out = []
    for j in range(pool):
        rnd = random.Random(1000 * n + j)
        a = [rnd.randrange(l) for _ in range(n)]; b = [rnd.randrange(l) for _ in range(n)]; r = rnd.randrange(l)
        rc, C = ctx.msm(b"".join(map(le, a)) + le(r) + le(sum(x * y for x, y in zip(a, b)) % l), G + B + F)
        assert rc == 0
        label = b"linear bench %d %d" % (n, j)
        rc, proof = bp.linear_create(ctx, bp.Transcript(label), le(j + 1), C, le(r), b"".join(map(le, a)), b"".join(map(le, b)), G, F, B)
        assert rc == 0
        out.append((label, proof, C, b"".join(map(le, b))))
    return (G, F, B), out


def median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); res = fn(); ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pool", type=int, default=64, help="distinct proofs per n (repeated up to count)")
    args = ap.parse_args()
    print(f"device: {device_info()}", flush=True)
    ctx = bp.Context(0); orc = Oracle()
    for n in (64, 256, 1024):
        (G, F, B), pool = make_proofs(ctx, orc, n, args.pool)
        V = bp.LinearVerifier(ctx, G, F, B)
        for count in (1, 64, 1024):
            sel = [pool[i % len(pool)] for i in range(count)]

            def batch():
                v = V.verify_batch([(bp.Transcript(lb), p, C, b) for lb, p, C, b in sel], seed=bytes(32)); ctx.synchronize(); return v

            def loop():
                v = [bp.linear_verify(ctx, bp.Transcript(lb), p, C, G, F, B, b) for lb, p, C, b in sel]; ctx.synchronize(); return v

            batch()                                                   # warm-up: arenas grown
            tb, vb = median_ms(batch, args.reps)
            tl, vl = median_ms(loop, args.reps if count < 1024 else max(1, args.reps // 2 + 1))
            assert vb == vl == [0] * count, (n, count)
            print(f"n={n:5d} count={count:5d}  batch {tb:9.2f} ms  loop {tl:9.2f} ms  speed-up {tl / tb:6.2f}x  verdicts equal: {vb == vl}", flush=True)
            if count == 1024:
                ctx.prof_enable(True); batch(); rep = ctx.prof_report(); ctx.prof_enable(False)
                print("    per-kernel (ms, launches): " + ", ".join(f"{k} {ms:.3f}/{c}" for k, (ms, c) in sorted(rep.items(), key=lambda kv: -kv[1][0])), flush=True)
        V.close()
    ctx.close()


if __name__ == "__main__":
    main()
