"""LinearProof batches from device-resident inputs (bp.LinearVerifier(..., capacity).run_device: the reserved graph, the reject path on the
device) against the blocking call (bp.LinearVerifier.verify_batch: host packing, pageable copies, a host-driven reject path).

Workloads: n in {64, 256, 1024} x count in {64, 1024} x {0, 1, 64} bad proofs ("a flipped": each fails its own equation, so the reject
path runs for every bad proof).  The proofs are 16 distinct valid proofs per n, tiled.  Inputs are packed once (bp.pack_linear) and
uploaded once as CUDA tensors for the device forms; the blocking form is given the same items every call.
Forms, wall time of CALLS calls per context (median of alternating repetitions), reported as ms per call and proofs/s:
  blocking_1 / blocking_4   verify_batch on 1 or 4 contexts (one Python thread per context), CALLS calls each
  device_1 / device_4       run_device on 1 or 4 contexts, CALLS calls queued on each, then one synchronise per context
Prints the device and its power limit, then one JSON line per workload with the rates, whether every device call returned the blocking
call's verdicts (same seed), and the launches per device call.
Usage: python benchmarks/linear_device.py [repetitions]"""
import json
import os
import statistics
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bulletproofs_b200 as bp

CALLS = 4          # calls per context and repetition
SEED = bytes(range(32))
L_ORDER = 2**252 + 27742317777372353535851937790883648493


def le(x):
    return x.to_bytes(32, "little")


def make_proofs(ctx, n, distinct=16):
    """`distinct` valid proofs at n over the generators (G, F, B) of the oracle's layout, from bp.linear_create; returns (items, G, F, B)"""
    import random
    gens = bp.Gens(ctx, n, 1)
    G = b"".join(gens.get(0, 0, i) for i in range(n))
    F, B = gens.get(2), gens.get(3)                   # F = pc_gens.B, B = pc_gens.B_blinding
    gens.close()
    rnd = random.Random(n)
    items = []
    for j in range(distinct):
        a = [rnd.randrange(L_ORDER) for _ in range(n)]; b = [rnd.randrange(L_ORDER) for _ in range(n)]; r = rnd.randrange(L_ORDER)
        rc, C = ctx.msm(b"".join(map(le, a)) + le(r) + le(sum(x * y for x, y in zip(a, b)) % L_ORDER), G + B + F)
        assert rc == 0
        label = b"linear device bench %d %d" % (n, j)
        rc, proof = bp.linear_create(ctx, bp.Transcript(label), le(j + 1), C, le(r), b"".join(map(le, a)), b"".join(map(le, b)), G, F, B)
        assert rc == 0
        items.append((label, proof, C, b"".join(map(le, b))))
    return items, G, F, B


def flipped(it, n):
    label, proof, C, b = it
    k = n.bit_length() - 1
    pr = bytearray(proof); pr[64 * k + 32] ^= 1
    return (label, bytes(pr), C, b)


def main():
    import torch
    nums = [a for a in sys.argv[1:] if a.isdigit()]
    reps = int(nums[0]) if nums else 5
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    base = bp.Context(0)
    pool = ThreadPoolExecutor(4)
    for n in (64, 256, 1024):
        distinct, G, F, B = make_proofs(base, n)
        ctxs = [bp.Context(0) for _ in range(4)]
        for count in (64, 1024):
            Vs = [bp.LinearVerifier(c, G, F, B, capacity=count) for c in ctxs]
            for nbad in (0, 1, 64):
                raw = [distinct[i % len(distinct)] for i in range(count)]
                bad_at = set(range(0, count, max(1, count // nbad))) if nbad else set()
                bad_at = set(sorted(bad_at)[:nbad])
                raw = [flipped(it, n) if i in bad_at else it for i, it in enumerate(raw)]
                items = [(bp.Transcript(lab), p, C, b) for lab, p, C, b in raw]
                packed = bp.pack_linear(items)
                d_in = [torch.frombuffer(bytearray(x), dtype=torch.uint8).cuda() for x in packed]
                outs = [[torch.zeros(count, dtype=torch.int32, device="cuda") for _ in range(CALLS)] for _ in Vs]
                torch.cuda.synchronize()
                ptrs = [t.data_ptr() for t in d_in]

                def blocking(k):
                    def one(V):
                        return [V.verify_batch(items, seed=SEED) for _ in range(CALLS)]
                    return lambda: list(pool.map(one, Vs[:k]))

                def device(k):
                    def run():
                        for j in range(CALLS):
                            for s, V in enumerate(Vs[:k]):
                                V.run_device(*ptrs, count, outs[s][j].data_ptr(), None, SEED)
                        for V in Vs[:k]:
                            V.ctx.synchronize()
                    return run

                forms = {"blocking_1": (blocking(1), 1), "blocking_4": (blocking(4), 4), "device_1": (device(1), 1), "device_4": (device(4), 4)}
                ref = Vs[0].verify_batch(items, seed=SEED)
                same = True
                for f, (fn, k) in forms.items():          # warm every form, check its verdicts
                    out = fn()
                    if f.startswith("blocking"):
                        same &= all(v == ref for per in out for v in per)
                    else:
                        same &= all([x & 0xFFFFFFFF for x in outs[s][j].cpu().tolist()] == ref for s in range(k) for j in range(CALLS))
                assert same, (n, count, nbad)
                assert sum(v != 0 for v in ref) == nbad
                times = {f: [] for f in forms}
                for _ in range(reps):
                    for f, (fn, k) in forms.items():
                        t0 = time.perf_counter(); fn(); times[f].append(time.perf_counter() - t0)
                l0 = Vs[0].ctx.launches
                Vs[0].run_device(*ptrs, count, outs[0][0].data_ptr(), None, SEED)
                launches = Vs[0].ctx.launches - l0
                Vs[0].ctx.synchronize()
                med = {f: statistics.median(v) for f, v in times.items()}
                print(json.dumps({"n": n, "count": count, "bad": nbad, "calls_per_context": CALLS, "verdicts_identical": same,
                                  "ms_per_call": {f: round(med[f] * 1e3 / CALLS, 3) for f in forms},
                                  "proofs_per_s": {f: round(count * CALLS * forms[f][1] / med[f]) for f in forms},
                                  "ms_per_call_range": {f: [round(min(v) * 1e3 / CALLS, 3), round(max(v) * 1e3 / CALLS, 3)] for f, v in times.items()},
                                  "device_launches_per_call": launches}), flush=True)
                del d_in, outs
            for V in Vs:
                V.close()
        for c in ctxs:
            c.close()
    pool.shutdown()
    base.close()


if __name__ == "__main__":
    main()
