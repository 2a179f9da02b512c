"""The exact device-resident verifiers (bp.BatchVerifier(..., exact=True).run_device_exact, bp.MixedVerifier(..., exact=True).run_device_exact)
against the plain device forms and against what a caller of the plain forms does with a damaged batch today.

Workloads: the bench geometry (8 batches x 1024 (64, 1) proofs per call, 8 contexts in flight, CALLS calls queued on each) and tx-8192
(benchmarks/mixed_service.py, one context, CALLS calls queued).
  clean     plain device call against exact device call on valid proofs, proofs/s
  bad_B     B in {1, 8, 64} invalid proofs spread over the call: the exact call (one context, CALLS queued, one synchronise) against the
            plain device call followed by what its flags ask for: each flagged batch (bp_rangeproof_verify_group_begin + finish) or class
            (bp.verify_mixed) copied back to the host and verified again.  The copy and the rerun are part of that time.  ms per call.
Every number is the median of alternating repetitions; the exact verdicts are checked against the rerun's.  Prints the device name and
power limit, then one JSON line per workload.
Usage: python benchmarks/device_reject.py [repetitions]"""
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
from mixed_service import SEED, workloads
from mixed_verify import LABEL, class_items

CALLS = 4
COUNT, NB, CTXS = 1024, 8, 8


def damage(buf, plen, idx):
    """t_x + 1 in each listed proof: well-formed, invalid"""
    for i in idx:
        o = i * plen + 128
        buf[o] ^= 1


def spread(total, b):
    return sorted(random.Random(b).sample(range(total), b))


def dev(b):
    import torch
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()


class Fixed:
    def __init__(self, gens_of, items):
        import torch
        self.ctx = bp.Context(0)
        self.gens = gens_of(self.ctx)
        self.v = bp.BatchVerifier(self.ctx, self.gens, bp.Transcript(LABEL), 64, 1, COUNT, NB, exact=True)
        self.verd = torch.zeros(COUNT * NB, dtype=torch.int32, device="cuda")
        self.ok = torch.zeros(NB, dtype=torch.int32).pin_memory()
        self.set(items)

    def set(self, proofs):
        self.proofs = bytes(proofs)
        self.d_p = dev(self.proofs)

    def queue(self, d_v, exact):
        (self.v.run_device_exact if exact else self.v.run_device)(self.d_p.data_ptr(), d_v.data_ptr(), self.verd.data_ptr(), self.ok.data_ptr(), seed=SEED)

    def redo(self, V, host_ctx, host_gens):
        """the plain caller's follow-up: every flagged batch copied back and verified again on the host form (on a context of its own, so
        that the reserved one keeps its geometry)"""
        out = [x & 0xFFFFFFFF for x in self.verd.cpu().tolist()]
        plen = len(self.proofs) // (COUNT * NB)
        for b, f in enumerate(self.ok.tolist()):
            if not f:
                p = self.d_p[b * COUNT * plen:(b + 1) * COUNT * plen].cpu().numpy().tobytes()
                got, _ = bp.verify_group(host_ctx, host_gens, bp.Transcript(LABEL), p, V[b * COUNT * 32:(b + 1) * COUNT * 32], 64, 1, COUNT, 1, seed=SEED)
                out[b * COUNT:(b + 1) * COUNT] = got
        return out


def time_it(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def fixed_workload(reps):
    import torch
    base = bp.Context(0)
    g0 = bp.Gens(base, 64, 32)
    items = class_items(base, g0, 64, 1, COUNT * NB, 1)
    proofs = b"".join(p for p, _, _ in items)
    V = b"".join(v for _, v, _ in items)
    plen = len(items[0][0])
    fx = [Fixed(lambda c: bp.Gens(c, 64, 32), proofs) for _ in range(CTXS)]
    d_v = dev(V)
    torch.cuda.synchronize()

    def run_all(exact):
        for _ in range(CALLS):
            for f in fx:
                f.queue(d_v, exact)
        for f in fx:
            f.ctx.synchronize()

    res = {"workload": f"bench {NB}x{COUNT}x(64,1), {CTXS} contexts"}
    for ex in (False, True):
        run_all(ex)
    rate = {False: [], True: []}
    for _ in range(reps):
        for ex in (False, True):
            rate[ex].append(CALLS * CTXS * COUNT * NB / time_it(lambda: run_all(ex)))
    res["clean_plain_proofs_per_s"] = statistics.median(rate[False])
    res["clean_exact_proofs_per_s"] = statistics.median(rate[True])
    f = fx[0]
    for B in (1, 8, 64):
        b = bytearray(proofs)
        damage(b, plen, spread(COUNT * NB, B))
        f.set(b)
        f.queue(d_v, True); f.ctx.synchronize()
        exact_v = [x & 0xFFFFFFFF for x in f.verd.cpu().tolist()]
        f.queue(d_v, False); f.ctx.synchronize()
        redo_v = f.redo(V, base, g0)
        ms = {False: [], True: []}
        for _ in range(reps):
            ms[True].append(1e3 * time_it(lambda: ([f.queue(d_v, True) for _ in range(CALLS)], f.ctx.synchronize())) / CALLS)

            def plain():
                for _ in range(CALLS):
                    f.queue(d_v, False)
                    f.ctx.synchronize()
                    f.redo(V, base, g0)
            ms[False].append(1e3 * time_it(plain) / CALLS)
        res[f"bad_{B}"] = {"exact_ms": statistics.median(ms[True]), "plain_then_host_rerun_ms": statistics.median(ms[False]),
                           "verdicts_match": exact_v == redo_v, "bad_found": sum(1 for v in exact_v if v)}
        f.set(proofs)
    for x in fx:
        x.gens.close(); x.ctx.close()
    g0.close(); base.close()
    return res


def mixed_workload(reps):
    import torch
    base = bp.Context(0)
    g0 = bp.Gens(base, 64, 32)
    mix, items = workloads(base, g0)["tx-8192"]
    random.Random(7).shuffle(items)
    ctx = bp.Context(0)
    gens = bp.Gens(ctx, 64, 32)
    v = bp.MixedVerifier(ctx, gens, mix, exact=True)
    n = len(items)
    verd = torch.zeros(n, dtype=torch.int32, device="cuda")
    flags = torch.zeros(len(mix), dtype=torch.int32).pin_memory()
    keys = list(mix)

    def upload(its):
        proofs, poff, ns, commitments, coff = bp.pack_mixed(its)
        t = [dev(proofs), dev(poff.tobytes()), dev(ns.tobytes()), dev(commitments), dev(coff.tobytes())]
        torch.cuda.synchronize()
        return t, len(proofs), len(commitments) // 32

    def queue(inp, exact):
        t, pbytes, nc = inp
        p, po, ns, c, co = (x.data_ptr() for x in t)
        (v.run_device_exact if exact else v.run_device)(bp.Transcript(LABEL), p, pbytes, po, ns, c, nc, co, n, verd.data_ptr(), flags.data_ptr(), seed=SEED)

    def redo(its):
        out = [x & 0xFFFFFFFF for x in verd.cpu().tolist()]
        fl = flags.tolist()
        sel = [i for i, (p, V, nn) in enumerate(its) if not fl[keys.index((nn, len(V) // 32))]]
        if sel:
            got = bp.verify_mixed(base, g0, bp.Transcript(LABEL), [its[i] for i in sel], seed=SEED)
            for i, g in zip(sel, got):
                out[i] = g
        return out

    res = {"workload": "tx-8192, 1 context"}
    inp = upload(items)
    rate = {False: [], True: []}
    for ex in (False, True):
        queue(inp, ex); ctx.synchronize()
    for _ in range(reps):
        for ex in (False, True):
            rate[ex].append(CALLS * n / time_it(lambda: ([queue(inp, ex) for _ in range(CALLS)], ctx.synchronize())))
    res["clean_plain_proofs_per_s"] = statistics.median(rate[False])
    res["clean_exact_proofs_per_s"] = statistics.median(rate[True])
    for B in (1, 8, 64):
        its = list(items)
        for i in spread(n, B):
            p, V, nn = its[i]
            pb = bytearray(p); pb[128] ^= 1
            its[i] = (bytes(pb), V, nn)
        inp = upload(its)
        queue(inp, True); ctx.synchronize()
        exact_v = [x & 0xFFFFFFFF for x in verd.cpu().tolist()]
        queue(inp, False); ctx.synchronize()
        redo_v = redo(its)
        ms = {False: [], True: []}
        for _ in range(reps):
            ms[True].append(1e3 * time_it(lambda: ([queue(inp, True) for _ in range(CALLS)], ctx.synchronize())) / CALLS)

            def plain():
                for _ in range(CALLS):
                    queue(inp, False)
                    ctx.synchronize()
                    redo(its)
            ms[False].append(1e3 * time_it(plain) / CALLS)
        res[f"bad_{B}"] = {"exact_ms": statistics.median(ms[True]), "plain_then_host_rerun_ms": statistics.median(ms[False]),
                           "verdicts_match": exact_v == redo_v, "bad_found": sum(1 for x in exact_v if x)}
    gens.close(); ctx.close(); g0.close(); base.close()
    return res


def main():
    nums = [a for a in sys.argv[1:] if a.isdigit()]
    reps = int(nums[0]) if nums else 5
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    print(json.dumps(fixed_workload(reps)), flush=True)
    print(json.dumps(mixed_workload(reps)), flush=True)


if __name__ == "__main__":
    main()
