"""LinearProofs of mixed lengths from device-resident buffers: LinearVerifier(..., mix=).run_device_mixed (bp_linear_verify_mixed_device)
against the blocking bp_linear_verify_mixed call on the same proofs, and, on the one-length workload, against the fixed-length
LinearVerifier(..., capacity=).run_device.

Workloads, 1024 proofs each, over one set of 1024 + 2 points, 16 distinct valid proofs per length tiled and shuffled (those of
benchmarks/linear_mixed.py):
  mix_4_2_1        lengths {64, 256, 1024} in proportion 4 : 2 : 1
  mix_all_11       every power-of-two length from 1 to 1024
  mix_4_2_1_bad1   mix_4_2_1 with one proof's a flipped: the reject path runs
  mix_4_2_1_bad64  mix_4_2_1 with 64 such proofs
  single_256       one length, n = 256
Forms, each the median of REPS rounds (host clock):
  blocking         one bp_linear_verify_mixed call (host packing, pageable copies, a synchronise)
  device_1ctx      4 calls queued on one context over inputs already on the device, then one synchronise: time / 4
  device_4ctx      4 calls queued on each of 4 contexts, then one synchronise per context: time / 16
  fixed_device     (single_256 only) the fixed-length device form, queued as device_1ctx
Each mix is reserved with the workload's own counts per length.  Prints the device and its power limit, then one JSON line per workload:
ms per call of each form, whether every device verdict equals the blocking call's, and launches per call.
Usage: python benchmarks/linear_mixed_device.py [repetitions]"""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import torch

import bulletproofs_b200 as bp
from linear_mixed import COUNT, SEED, make_proofs, workload

QUEUE, CONTEXTS = 4, 4


def flip_a(raw, at):
    label, proof, C, b = raw[at]
    k = (len(b) // 32).bit_length() - 1
    pr = bytearray(proof); pr[64 * k + 32] ^= 1
    raw[at] = (label, bytes(pr), C, b)


class Setup:
    """one context: the resident set with the workload's mix reserved, and the packed inputs on the device"""

    def __init__(self, G, F, B, items, counts, fixed_n=None):
        self.ctx = bp.Context(0)
        self.V = bp.LinearVerifier(self.ctx, G, F, B, mix=counts)
        self.F = bp.LinearVerifier(self.ctx, G[:32 * fixed_n], F, B, capacity=COUNT) if fixed_n else None
        bufs = bp.pack_linear_mixed(items)
        self.t = [torch.frombuffer(bytearray(x + bytes(16)), dtype=torch.uint8).cuda() for x in bufs]
        self.sizes = [len(x) for x in bufs]
        self.verd = [torch.zeros(COUNT, dtype=torch.int32, device="cuda") for _ in range(QUEUE)]
        torch.cuda.synchronize()

    def mixed(self, j):
        t, pr, C, b, po, bo = (x.data_ptr() for x in self.t)
        self.V.run_device_mixed(t, pr, self.sizes[1], po, C, b, self.sizes[3] // 32, bo, COUNT, self.verd[j].data_ptr(), seed=SEED)

    def fixed(self, j):
        t, pr, C, b = (x.data_ptr() for x in self.t[:4])
        self.F.run_device(t, pr, C, b, COUNT, self.verd[j].data_ptr(), seed=SEED)

    def verdicts(self):
        self.ctx.synchronize()
        return [[x & 0xFFFFFFFF for x in v.cpu().tolist()] for v in self.verd]

    def close(self):
        self.V.close()
        if self.F:
            self.F.close()
        self.ctx.close()


def queued(setups, call):
    t0 = time.perf_counter()
    for j in range(QUEUE):
        for s in setups:
            call(s, j)
    for s in setups:
        s.ctx.synchronize()
    return (time.perf_counter() - t0) / (QUEUE * len(setups))


def main():
    nums = [a for a in sys.argv[1:] if a.isdigit()]
    reps = int(nums[0]) if nums else 9
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    ctx = bp.Context(0)
    gens = bp.Gens(ctx, 1024, 1)
    G = b"".join(gens.get(0, 0, i) for i in range(1024))
    F, B = gens.get(2), gens.get(3)
    gens.close()
    ns = [1 << k for k in range(11)]
    pool = {n: make_proofs(ctx, G, F, B, n) for n in ns}
    per = COUNT // 11
    c421, c11 = {64: 585, 256: 293, 1024: 146}, {n: per + (1 if j < COUNT - 11 * per else 0) for j, n in enumerate(ns)}
    loads = {"mix_4_2_1": (workload(pool, c421, 1), c421), "mix_all_11": (workload(pool, c11, 2), c11)}
    for name, nbad in (("mix_4_2_1_bad1", 1), ("mix_4_2_1_bad64", 64)):
        raw = list(loads["mix_4_2_1"][0])
        for j in range(nbad):
            flip_a(raw, (500 + 16 * j) % COUNT)
        loads[name] = (raw, c421)
    loads["single_256"] = (workload(pool, {256: COUNT}, 3), {256: COUNT})
    points = bp.PointSet(ctx, B + F + G)
    for name, (raw, counts) in loads.items():
        items = [(bp.Transcript(lab), p, C, b) for lab, p, C, b in raw]
        fixed_n = 256 if name == "single_256" else None
        one = [Setup(G, F, B, items, counts, fixed_n)]
        four = one + [Setup(G, F, B, items, counts) for _ in range(CONTEXTS - 1)]
        ref = bp.linear_verify_mixed(ctx, points, items, SEED)
        forms = {"blocking": lambda: bp.linear_verify_mixed(ctx, points, items, SEED),
                 "device_1ctx": lambda: queued(one, Setup.mixed),
                 "device_4ctx": lambda: queued(four, Setup.mixed)}
        if fixed_n:
            forms["fixed_device"] = lambda: queued(one, Setup.fixed)
        same = True
        for f, fn in forms.items():                                   # warm every form, and check its verdicts
            fn()
            if f != "blocking":
                same = same and all(v == ref for s in (four if f == "device_4ctx" else one) for v in s.verdicts())
        times = {f: [] for f in forms}
        for _ in range(reps):
            for f, fn in forms.items():
                t0 = time.perf_counter(); r = fn(); dt = time.perf_counter() - t0
                times[f].append(dt if f == "blocking" else r)
        launches = {}
        for f, fn in (("blocking", forms["blocking"]), ("device", lambda: one[0].mixed(0))) + ((("fixed_device", lambda: one[0].fixed(0)),) if fixed_n else ()):
            l0 = one[0].ctx.launches if f != "blocking" else ctx.launches
            fn()
            launches[f] = (one[0].ctx.launches if f != "blocking" else ctx.launches) - l0
        one[0].ctx.synchronize()
        med = {f: statistics.median(v) for f, v in times.items()}
        print(json.dumps({"workload": name, "proofs": COUNT, "counts": counts, "bad": ref.count(1), "device_verdicts_identical": same,
                          "ms_per_call": {f: round(v * 1e3, 3) for f, v in med.items()},
                          "ms_range": {f: [round(min(v) * 1e3, 3), round(max(v) * 1e3, 3)] for f, v in times.items()},
                          "blocking_over_device": {f: round(med["blocking"] / med[f], 2) for f in med if f != "blocking"},
                          "launches_per_call": launches}), flush=True)
        for s in four:
            s.close()
    points.close()
    ctx.close()


if __name__ == "__main__":
    main()
