"""Front end of one launch group at the bench geometry (1024-proof batches of 64-bit single-party range proofs, 8 batches per group):
solo duration of each per-proof kernel (library-side bp_prof_* events, one group at a time), its mean duration with 8 groups in
flight (benchmarks/timeline.py), and its register-time = registers/thread x threads/group x contended duration.  reg_file_share
divides that by the whole register file over one group's share of the steady-state time (registers per SM x SMs x G x us per
batch): the part of the GPU's register file-seconds the kernel holds, i.e. takes away from the MSM kernels that run beside it.
front_end_reg_file_share adds up the per-proof kernels that run beside the wide ones: k_rp_transcript, k_rp_head and
k_rp_scalars_sum.  pipe_bound_us is the kernel's wide multiplies per group (counted from the shapes below) at the measured
IMAD.WIDE rate: the least time its multiplies take when they have the whole GPU; solo_us over it is how far the kernel is
from its integer-pipe floor.
(A kernel whose grid is larger than what fits on the GPU at once, as k_rp_decompress's, is over-counted; the per-proof front-end
kernels, 256 warps each, are resident all at once.)  Registers come from the built library's resource table (cuobjdump).  Prints
one JSON line.
Usage: python benchmarks/front_end.py [groups in flight] [rounds] [libbpmsm.so to measure instead of the package's, e.g. another build]"""
import contextlib, io, json, os, re, runpy, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bulletproofs_b200 as bp

S = sys.argv[1] if len(sys.argv) > 1 else "8"
ROUNDS = sys.argv[2] if len(sys.argv) > 2 else "6"
LIB = sys.argv[3] if len(sys.argv) > 3 else None
G, BATCH, N, M = 8, 1024, 64, 1
K = (N * M).bit_length() - 1
D, PROOFS = 4 + 2 * K + M, G * BATCH
# profiling label -> (kernel symbol, threads per group), from the launches in bpmsm.cu (rp_front_end)
KERNELS = {"k_rp_transcript": ("k_rp_transcript", PROOFS),
           "k_rp_head": ("k_rp_head_seq", PROOFS),
           "k_rp_decompress": ("k_rp_decompress", -(-PROOFS * D // 128) * 128),
           "k_rp_scalars_sum": ("k_rp_scalars_sum", G * (BATCH // 32) * 64)}
# IMAD.WIDE.U32 thread-level multiply-adds/s (bench.py INT_PEAK, benchmarks/imad_microbench.cu on an H100 80GB HBM3)
INT_PEAK = 8.33e12
CHUNK = 32
# wide multiplies per group: a Montgomery product is 3 x 64 IMAD.WIDE, a 512-bit product-sum term 64 and its reduction 128
WIDE = {"k_rp_transcript": 0,                                                              # Keccak: no wide multiplies
        "k_rp_head": PROOFS * (D * 3 + 170) * 192,                                         # bench.py's per-proof head count
        "k_rp_decompress": PROOFS * D * (257 * 44 + 29 * 72),                              # bench.py's per-point count
        "k_rp_scalars_sum": PROOFS * N * M * 3 * 64 + G * (BATCH // CHUNK) * N * M * 3 * 128}


def registers(lib):
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    out = subprocess.run([cuobjdump, "--dump-resource-usage", lib], check=True, capture_output=True, text=True).stdout
    regs = {}
    for fn, body in re.findall(r"Function (\S+):\s*\n?\s*(REG:\d+ STACK:\d+[^\n]*)", out):
        for label, (sym, _) in KERNELS.items():
            # k_rp_head_seq has one instance per k (k_rp_head_seq<K>): take the bench's
            if re.match(r"_Z\d+" + sym + r"[^a-z_]", fn) and (not fn.startswith(f"_Z{len(sym)}{sym}ILj") or fn.startswith(f"_Z{len(sym)}{sym}ILj{K}E")):
                regs[label] = {"reg": int(re.search(r"REG:(\d+)", body).group(1)), "stack": int(re.search(r"STACK:(\d+)", body).group(1))}
    return regs


def main():
    if LIB:
        bp.LIB_PATH = os.path.abspath(LIB)
    regs = registers(bp.LIB_PATH)
    buf = io.StringIO()
    sys.argv = [os.path.join(ROOT, "benchmarks", "timeline.py"), S, ROUNDS, str(G)]
    with contextlib.redirect_stdout(buf):
        runpy.run_path(sys.argv[0], run_name="__main__")
    tl = json.loads(buf.getvalue().strip().splitlines()[-1])
    out = {"groups_in_flight": int(S), "batches_per_group": G, "us_per_batch": round(tl["us_per_batch"], 2), "kernels": {}}
    total = 0.0
    for label, (sym, threads) in KERNELS.items():
        k = tl["kernels"].get(label)
        if not k or label not in regs:
            continue
        rt = regs[label]["reg"] * threads * k["mean_us_contended"] * 1e-6          # register-seconds per group
        total += rt
        out["kernels"][label] = {"solo_us": k["solo_us"], "pipe_bound_us": round(WIDE[label] / INT_PEAK * 1e6, 2) if WIDE[label] else None,
                                 "contended_us": k["mean_us_contended"], "registers": regs[label]["reg"],
                                 "stack_bytes": regs[label]["stack"], "threads_per_group": threads, "reg_seconds_per_group": rt}
    prop = torch.cuda.get_device_properties(0)
    file_s = getattr(prop, "regs_per_multiprocessor", 65536) * prop.multi_processor_count * G * tl["us_per_batch"] * 1e-6
    out["register_file_seconds_per_group"] = round(file_s, 4)
    for v in out["kernels"].values():
        v["share_of_these_kernels"] = round(v["reg_seconds_per_group"] / total, 3) if total else None
        v["reg_file_share"] = round(v["reg_seconds_per_group"] / file_s, 3)
        v["reg_seconds_per_group"] = round(v["reg_seconds_per_group"], 4)
    fe = [out["kernels"][k] for k in ("k_rp_transcript", "k_rp_head", "k_rp_scalars_sum") if k in out["kernels"]]
    out["front_end_reg_file_share"] = round(sum(v["reg_file_share"] for v in fe), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
