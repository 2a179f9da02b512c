"""Mixed-geometry verification from device-resident inputs (bp.MixedVerifier.run_device: the proofs placed in the reserved mix by device
kernels) against the host-packed service (bp.MixedVerifier begin / finish), with a fixed-geometry bp.BatchVerifier over the same number
of (64, 1) proofs as the ceiling.

Workloads: those of benchmarks/mixed_service.py (tx-1024, tx-8192, tx-8192-half, grid-24x33).  Each workload's inputs are packed once
(bp.pack_mixed) and uploaded once as CUDA tensors.
Forms, proofs/s over the same calls (median of alternating repetitions):
  service_1/4/8     bp.MixedVerifier on 1, 4 or 8 contexts, host packing per call: begin on every context, then finish on each
  device_1/4/8      bp.MixedVerifier.run_device on 1, 4 or 8 contexts, CALLS calls queued on each, then one synchronise per context
  fixed_64x1        bp.BatchVerifier(64, 1) reserved at the same number of proofs (8 batches when it divides by 8), begin / finish
  fixed_device      the same BatchVerifier through run_device on inputs uploaded once, CALLS calls queued, then one synchronise: the
                    device-resident fixed-geometry ceiling
Prints the device and its power limit, then one JSON line per workload: the rates, whether every form returned the verdicts of the
blocking bp.verify_mixed, the host time of one run_device enqueue, and the planner kernels' time (bp_prof_report, a run of its own).
Usage: python benchmarks/mixed_device.py [repetitions]"""
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import bulletproofs_b200 as bp
from mixed_service import SEED, timed, workloads
from mixed_verify import LABEL, class_items

CALLS = 4          # calls queued per context by the device forms


class Inputs:
    """a workload's five arrays uploaded once as CUDA tensors"""

    def __init__(self, items):
        import torch
        proofs, poff, ns, commitments, coff = bp.pack_mixed(items)
        up = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
        self.t = [up(proofs), up(poff.tobytes()), up(ns.tobytes()), up(commitments), up(coff.tobytes())]
        self.count, self.proof_bytes, self.n_commitments = len(items), len(proofs), len(commitments) // 32
        torch.cuda.synchronize()

    def run(self, v, d_verdicts):
        p, po, n, c, co = (t.data_ptr() for t in self.t)
        v.run_device(bp.Transcript(LABEL), p, self.proof_bytes, po, n, c, self.n_commitments, co, self.count, d_verdicts.data_ptr(), None, seed=SEED)


def main():
    import torch
    nums = [a for a in sys.argv[1:] if a.isdigit()]
    reps = int(nums[0]) if nums else 7
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    base = bp.Context(0)
    gens = bp.Gens(base, 64, 32)
    for name, (mix, items) in workloads(base, gens).items():
        random.Random(7).shuffle(items)
        N = len(items)
        svcs = []
        for _ in range(8):
            c = bp.Context(0)
            g = bp.Gens(c, 64, 32)
            svcs.append((c, g, bp.MixedVerifier(c, g, mix)))
        inp = Inputs(items)
        outs = [[torch.zeros(N, dtype=torch.int32, device="cuda") for _ in range(CALLS)] for _ in svcs]
        one = [it for it in items if len(it[1]) == 32 and it[2] == 64][:1] or [class_items(base, gens, 64, 1, 1, 5)[0]]
        nb = 8 if N % 8 == 0 else 1
        fixed = bp.BatchVerifier(base, gens, bp.Transcript(LABEL), 64, 1, N // nb, nb)
        fproofs, fV = one[0][0] * N, one[0][1] * N
        d_fproofs, d_fV = (torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() for b in (fproofs, fV))
        fouts = [torch.zeros(N, dtype=torch.int32, device="cuda") for _ in range(CALLS)]
        torch.cuda.synchronize()            # torch's stream has filled every tensor the contexts' streams read or write

        def service(k):
            def run():
                for c, g, v in svcs[:k]:
                    v.begin(bp.Transcript(LABEL), items, seed=SEED)
                return [v.finish() for _, _, v in svcs[:k]]
            return run

        def device(k):
            def run():
                for j in range(CALLS):
                    for s, (c, g, v) in enumerate(svcs[:k]):
                        inp.run(v, outs[s][j])
                for c, _, _ in svcs[:k]:
                    c.synchronize()
            return run

        def fixed_run():
            fixed.begin(fproofs, fV, SEED)
            return fixed.finish()

        def fixed_device():
            for o in fouts:
                fixed.run_device(d_fproofs.data_ptr(), d_fV.data_ptr(), o.data_ptr(), None, SEED)
            base.synchronize()

        forms = {"service_1": (service(1), 1), "service_4": (service(4), 4), "service_8": (service(8), 8), "device_1": (device(1), CALLS),
                 "device_4": (device(4), 4 * CALLS), "device_8": (device(8), 8 * CALLS), "fixed_64x1": (fixed_run, 1),
                 "fixed_device": (fixed_device, CALLS)}
        ref = bp.verify_mixed(base, gens, bp.Transcript(LABEL), items, seed=SEED)
        same = True
        for f, (fn, calls) in forms.items():          # warm every form, check its verdicts
            out = fn()
            if f.startswith("service"):
                same &= all(o == ref for o in out)
            elif f.startswith("device"):
                k = calls // CALLS
                same &= all([x & 0xFFFFFFFF for x in outs[s][j].cpu().tolist()] == ref for s in range(k) for j in range(CALLS))
        rates = {f: [] for f in forms}
        for _ in range(reps):
            for f, (fn, calls) in forms.items():
                _, r = timed(fn, calls)
                rates[f].append(r * N)
        c0, _, v0 = svcs[0]
        enqueue = []
        for _ in range(reps):
            c0.synchronize()
            t0 = time.perf_counter(); inp.run(v0, outs[0][0]); enqueue.append(time.perf_counter() - t0)
            c0.synchronize()
        l0 = c0.launches; inp.run(v0, outs[0][0]); launches = c0.launches - l0
        c0.synchronize()
        c0.prof_enable(True)
        inp.run(v0, outs[0][0])
        c0.synchronize()
        prof = c0.prof_report()
        c0.prof_enable(False)
        print(json.dumps({"workload": name, "proofs": N, "classes": len(mix), "calls_queued_per_context": CALLS,
                          "proofs_per_s": {f: round(statistics.median(v)) for f, v in rates.items()},
                          "proofs_per_s_range": {f: [round(min(v)), round(max(v))] for f, v in rates.items()},
                          "verdicts_identical": same, "all_accepted": ref == [0] * N, "device_enqueue_host_ms": round(statistics.median(enqueue) * 1e3, 3),
                          "device_launches_per_call": launches,
                          "planner_kernels_ms": {k: [round(t, 4), n] for k, (t, n) in prof.items() if k in ("k_mix_plan", "small_kernels")}}), flush=True)
        del fixed
        for c, g, v in svcs:
            g.close(); c.close()
    gens.close()
    base.close()


if __name__ == "__main__":
    main()
