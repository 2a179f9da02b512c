"""LinearProof::create (bp.linear_create) timed at n in {64, 256, 1024}, the reference's linear-proof bench range (BASELINE.md).
Each instance is built as tests/test_linear_proof.py builds it, and the proof bytes are checked once against the oracle at each size.
One warm-up call, then the median of --reps timed calls; every call ends in a device synchronise.  Prints the device and its power
limit, then one JSON line per size.
    python benchmarks/linear_proof.py [--reps R] [--lib-dir DIR]
--lib-dir loads libbpmsm.so and libbulletproofs_host.so from another build (e.g. the parent commit's), so the same script times both."""
import argparse, json, os, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bulletproofs_b200 as bp
from oracle_binding import Oracle
from test_linear_proof import _instance

SIZES = (64, 256, 1024)
LABEL = b"linearproofbench"


def device_line():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "unknown"
    return {"device": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--lib-dir", default=None)
    args = ap.parse_args()
    if args.reps < 20:
        ap.error("--reps must be at least 20")
    if args.lib_dir:
        bp.LIB_PATH = os.path.abspath(os.path.join(args.lib_dir, "libbpmsm.so"))
        bp.HOST_LIB_PATH = os.path.abspath(os.path.join(args.lib_dir, "libbulletproofs_host.so"))
    print(json.dumps(dict(device_line(), lib=os.path.dirname(bp.LIB_PATH))), flush=True)
    orc = Oracle()
    ctx = bp.Context(0)
    for n in SIZES:
        G, F, B, a, b, r, C = _instance(orc, n, 100 + n)
        seed = bytes([n % 251]) * 32
        rc, proof = bp.linear_create(ctx, bp.Transcript(LABEL), seed, C, r, a, b, G, F, B)          # warm-up
        orc_rc, _, want = orc.linear_create(orc.transcript(LABEL), seed, C, r, a, b, G, F, B)
        assert rc == 0 and orc_rc == 0 and proof == want, f"n = {n}: proof bytes differ from the oracle's"
        ms = []
        for _ in range(args.reps):
            t = bp.Transcript(LABEL)
            t0 = time.perf_counter()
            bp.linear_create(ctx, t, seed, C, r, a, b, G, F, B)
            ctx.synchronize()
            ms.append(1e3 * (time.perf_counter() - t0))
        print(json.dumps({"n": n, "reps": args.reps, "median_ms": round(statistics.median(ms), 3), "min_ms": round(min(ms), 3),
                          "max_ms": round(max(ms), 3), "proof_matches_oracle": True}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
