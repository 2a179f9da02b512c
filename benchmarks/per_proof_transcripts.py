"""Cost of giving every range proof its own transcript.  The device launch-group path at 8 batches x 1024 proofs x (n, m) = (64, 1), on one
context with the geometry reserved (one captured graph serves every mode), in three modes timed alternately:
  shared     one transcript for every proof (bp.BatchVerifier.run_device, what bench.py runs)
  same-pos   one record per proof (bp.verify_group_device_each); 32 transcripts whose labels have one length, so every record starts
             at the same position and the lanes of a warp take the same branches
  mixed-pos  one record per proof; 32 transcripts with appended context of 32 lengths, so the 32 lanes of a warp start at 32 different
             positions and diverge where an operation header crosses the rate
The records are 203 bytes back to back, so the replay loads them byte-wise.  Then one bp.verify_mixed_each call against one
bp.verify_mixed call over the same proofs (n = 64, m in {1, 2, 4, 8} in proportions 8 : 4 : 2 : 1, 1024 proofs).
Prints the device and its power limit, then JSON lines: proofs/s per mode (median of alternating repetitions, each of CALLS groups queued
back to back and one synchronise), the verdicts of every mode (all proofs are valid), and in a run of its own with per-kernel CUDA events
(direct launches, no graph) the k_rp_transcript time per group.  Usage: python benchmarks/per_proof_transcripts.py [repetitions]"""
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

import torch

N, M, COUNT, NB = 64, 1, 1024, 8
CALLS = 16                 # groups per timed window
DISTINCT = 4               # proofs per transcript, tiled
LANES = 32
L_ORDER = 2 ** 252 + 27742317777372353535851937790883648493
LABEL = b"AggregateRangeProofBenchmark"


def prove(ctx, gens, t, n, m, count, seed):
    rnd = random.Random(seed)
    vals = [rnd.randrange(1 << n) for _ in range(count * m)]
    bl = b"".join(rnd.randrange(L_ORDER).to_bytes(32, "little") for _ in range(count * m))
    seeds = b"".join(rnd.randrange(1 << 256).to_bytes(32, "little") for _ in range(count))
    st, proofs, V = bp.prove_many(ctx, gens, t.clone(), vals, bl, n, m, seeds)
    assert st == [0] * count
    plen = len(proofs) // count
    return [(proofs[i * plen:(i + 1) * plen], V[i * 32 * m:(i + 1) * 32 * m]) for i in range(count)]


def transcripts(kind):
    out = []
    for i in range(LANES):
        t = bp.Transcript(b"tx %04d" % i)
        if kind == "mixed-pos":
            t.append_message(b"context", bytes([i]) * (5 * i + 1))
        out.append(t)
    return out


def workload(ctx, gens, kind):
    """(records, proofs, commitments) of NB*COUNT proofs: proof q comes from transcript q % LANES"""
    ts = [bp.Transcript(LABEL)] * LANES if kind == "shared" else transcripts(kind)
    pool = [prove(ctx, gens, t, N, M, DISTINCT, 100 * i + len(kind)) for i, t in enumerate(ts)]
    recs, proofs, Vs = [], [], []
    for q in range(NB * COUNT):
        lane, rep = q % LANES, (q // LANES) % DISTINCT
        recs.append(ts[lane].to_bytes()); proofs.append(pool[lane][rep][0]); Vs.append(pool[lane][rep][1])
    pos = sorted({r[200] for r in recs[:LANES]})
    return b"".join(recs), b"".join(proofs), b"".join(Vs), pos


def dev(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()


def main():
    nums = [a for a in sys.argv[1:] if a.isdigit()]
    reps = int(nums[0]) if nums else 9
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"device": q}), flush=True)
    ctx = bp.Context(0)
    gens = bp.Gens(ctx, 64, 32)
    modes = ("shared", "same-pos", "mixed-pos")
    work = {k: workload(ctx, gens, k) for k in modes}
    ver = bp.BatchVerifier(ctx, gens, bp.Transcript(LABEL), N, M, COUNT, NB)            # reserves the geometry: arenas, graph
    d = {k: tuple(dev(x) for x in w[:3]) for k, w in work.items()}
    d_verd = torch.full((CALLS, NB * COUNT), 77, dtype=torch.int32, device="cuda")
    h_ok = torch.zeros((CALLS, NB), dtype=torch.int32).pin_memory()
    seed = bytes(range(32))

    def call(kind, r):
        d_t, d_p, d_v = d[kind]
        if kind == "shared":
            ver.run_device(d_p.data_ptr(), d_v.data_ptr(), d_verd[r].data_ptr(), h_ok[r].data_ptr(), seed)
        else:
            bp.verify_group_device_each(ctx, gens, d_t.data_ptr(), d_p.data_ptr(), d_v.data_ptr(), N, M, COUNT, NB, d_verd[r].data_ptr(), h_ok[r].data_ptr(), seed)

    verdicts_ok = {}
    for kind in modes:                                   # warm-up, and the outputs of each mode
        for r in range(CALLS):
            call(kind, r)
        ctx.synchronize()
        verdicts_ok[kind] = bool((d_verd == 0).all().item()) and bool((h_ok == 1).all().item())
    times = {k: [] for k in modes}
    for _ in range(reps):                                # alternating
        for kind in modes:
            ctx.synchronize()
            t0 = time.perf_counter()
            for r in range(CALLS):
                call(kind, r)
            ctx.synchronize()
            times[kind].append(time.perf_counter() - t0)
    ctx.prof_enable(True)                                # per-kernel CUDA events: direct launches, in a run of their own
    ctx.prof_report()
    tr_ms = {}
    for kind in modes:
        for r in range(4):
            call(kind, r)
        rep = ctx.prof_report()
        tr_ms[kind] = round(rep["k_rp_transcript"][0] / rep["k_rp_transcript"][1], 4)
    ctx.prof_enable(False)
    total = NB * COUNT * CALLS
    shared = statistics.median(times["shared"])
    print(json.dumps({"workload": f"group {NB}x{COUNT}x({N},{M}) device path, reserved", "calls_per_window": CALLS, "repetitions": reps,
                      "proofs_per_s": {k: round(total / statistics.median(v)) for k, v in times.items()},
                      "window_ms_range": {k: [round(min(v) * 1e3, 2), round(max(v) * 1e3, 2)] for k, v in times.items()},
                      "vs_shared": {k: round(shared / statistics.median(v), 4) for k, v in times.items()},
                      "record_positions_in_a_warp": {k: work[k][3] for k in modes},
                      "k_rp_transcript_ms_per_group": tr_ms, "all_accepted": verdicts_ok}), flush=True)

    # mixed call: per-proof transcripts against one shared transcript, the same proofs
    sizes = {1: 1024 - 7 * 68, 2: 4 * 68, 4: 2 * 68, 8: 68}
    shared_items, each_items = [], []
    ts = transcripts("mixed-pos")
    for m, c in sizes.items():
        base = prove(ctx, gens, bp.Transcript(LABEL), 64, m, DISTINCT, 7 + m)
        own = [prove(ctx, gens, ts[i], 64, m, 1, 50 * m + i)[0] for i in range(LANES)]
        shared_items += [(base[i % DISTINCT][0], base[i % DISTINCT][1], 64) for i in range(c)]
        each_items += [(ts[i % LANES], own[i % LANES][0], own[i % LANES][1], 64) for i in range(c)]
    perm = list(range(len(shared_items)))
    random.Random(7).shuffle(perm)
    shared_items = [shared_items[i] for i in perm]; each_items = [each_items[i] for i in perm]
    vm = bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), shared_items, seed=seed)
    ve = bp.verify_mixed_each(ctx, gens, each_items, seed=seed)
    tm, te = [], []
    for _ in range(reps):
        t0 = time.perf_counter(); bp.verify_mixed(ctx, gens, bp.Transcript(LABEL), shared_items, seed=seed); tm.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); bp.verify_mixed_each(ctx, gens, each_items, seed=seed); te.append(time.perf_counter() - t0)
    n = len(shared_items)
    print(json.dumps({"workload": f"mixed call, {n} proofs, n = 64, m in 1/2/4/8 (8:4:2:1)", "repetitions": reps,
                      "proofs_per_s": {"verify_mixed": round(n / statistics.median(tm)), "verify_mixed_each": round(n / statistics.median(te))},
                      "ms_range": {"verify_mixed": [round(min(tm) * 1e3, 2), round(max(tm) * 1e3, 2)],
                                   "verify_mixed_each": [round(min(te) * 1e3, 2), round(max(te) * 1e3, 2)]},
                      "all_accepted": vm == [0] * n and ve == [0] * n}), flush=True)
    gens.close()
    ctx.close()


if __name__ == "__main__":
    main()
