"""bench.py --workload msm: BASELINE config 4, Ristretto multiscalar multiplication of 2^lg terms (SURVEY.md section 8d).

Points = the first n outputs of the party-0 'G' generator chain (SHAKE256("GeneratorsChain" || 'G' || LE32(0)), 64 bytes per
point through from_uniform_bytes, src/generators.rs:62-104), scalars = ChaCha20(seed 0x2a x 32) 64-byte blocks wide-reduced.
Every rank runs its own `--msms` independent MSMs per call ("per-GPU batch shard", weak scaling, no collective).

One step = one call = `--msms` MSMs of n terms.  Numbers on the JSON line:
  value            : terms/s, scalars resident in HBM, bases resident as a decompressed point set (bp_points / bp_msm_points_device)
  with_decompress  : terms/s, scalars AND 32-byte compressed points resident in HBM, every point decompressed inside the call
                     (bp_msm_batch_device) -- the form the verifier's mega-MSM has (points arrive compressed)
  e2e              : terms/s through the host-buffer C-ABI call with pinned buffers: bp_msm_points (scalars H2D, results D2H)
  e2e_compressed   : the same through bp_msm_batch (scalars + compressed points H2D, decompression, results D2H)
The first MSM of every call set is compared byte for byte with the CPU oracle up to 2^--check-lg terms."""
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))


def g_chain_uniform(n):
    return hashlib.shake_256(b"GeneratorsChain" + b"G" + (0).to_bytes(4, "little")).digest(64 * n)


def main(args, rank, world, local, local_world):
    import bench
    from oracle_binding import Oracle
    n = 1 << args.lg
    M = args.msms
    metric = f"Ristretto MSM terms/sec (n = 2^{args.lg}, {M} MSMs per call per GPU)"
    config = {"workload": f"Ristretto MSM size sweep: {M} independent MSMs of 2^{args.lg} terms per call per GPU (G-chain points, ChaCha20 scalars)",
              "lg_n": args.lg, "msms_per_call": M, "l2": "scalar sets rotate through a pool larger than L2 (>= 160 MiB of scalars)",
              "parallelism": f"whole MSMs per rank x{world}, no collective"}
    orc = Oracle()
    orc.set_backend("auto")
    seed = bytes([0x2a]) * 32
    if args.impl == "reference":
        if rank != 0:
            return
        from concurrent.futures import ThreadPoolExecutor
        import ctypes
        cores = bench.effective_cores()
        pts = b"".join(orc.from_uniform(g_chain_uniform(n)[64 * i:64 * i + 64]) for i in range(n)) if n <= (1 << 14) else None
        if pts is None:                      # large n: derive the points once with the oracle in threads
            uni = g_chain_uniform(n)
            with ThreadPoolExecutor(cores) as ex:
                pts = b"".join(ex.map(lambda i: orc.from_uniform(uni[64 * i:64 * i + 64]), range(n), chunksize=4096))
        per_step = max(1, min(M, cores))
        sc = [orc.scalars_from_chacha(seed, n, skip=j * n) for j in range(per_step)]
        def one(j):
            return orc.msm(sc[j], pts)
        with ThreadPoolExecutor(per_step) as ex:
            for _ in range(args.warmup):
                list(ex.map(one, range(per_step)))
            t0 = time.perf_counter()
            for _ in range(args.steps):
                list(ex.map(one, range(per_step)))
            dt = time.perf_counter() - t0
        value = per_step * n * args.steps / dt
        print(json.dumps({"impl": "reference", "metric": metric, "value": value, "unit": "terms/s", "n_gpus": 0, "steps": args.steps, "warmup": args.warmup,
                          "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": orc.backend_name() + " (CPU)",
                          "data": "synthetic (generator-chain points, ChaCha20 scalars)", "config": config,
                          "cpu_baseline": {"value": value, "unit": "terms/s", "cores": per_step, "kind": "port", "backend": orc.backend_name(),
                                           "sample": f"{per_step} of the step's {M} MSMs per step, one MSM per thread (Pippenger w = 8)"},
                          "e2e": {"value": value, "unit": "terms/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))
        return

    import numpy as np
    import torch
    import torch.distributed as dist
    import bulletproofs_b200 as bp
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs an H100: there is no CPU fallback on the MSM path")
    torch.cuda.set_device(local)
    pin = bench.pin_to_gpu_numa_node(local, local_world)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    stream = torch.cuda.Stream(device=local)
    ctx = bp.Context(local, stream=stream.cuda_stream)
    if getattr(args, "window", 0):
        ctx.set_msm_window(args.window)
    points = ctx.from_uniform_bytes(g_chain_uniform(n))                      # n x 32 B compressed, derived on the GPU
    # scalar pool: at least one call's worth, and more than L2
    T = M * n
    pool_scalars = max(T, (160 << 20) // 32)
    pool_scalars = (pool_scalars + T - 1) // T * T
    sets = pool_scalars // T
    h_sc = torch.frombuffer(bytearray(orc.scalars_from_chacha(seed, pool_scalars, skip=rank * pool_scalars)), dtype=torch.uint8).pin_memory()
    h_pts = torch.frombuffer(bytearray(points * M), dtype=torch.uint8).pin_memory()       # M copies: bp_msm_batch takes one point per term
    d_sc = h_sc.cuda(); d_pts = h_pts.cuda()
    d_off = torch.arange(0, (M + 1) * n, n, dtype=torch.int32, device="cuda")
    d_out = torch.zeros((sets, M, 32), dtype=torch.uint8, device="cuda"); d_st = torch.zeros((M,), dtype=torch.uint8, device="cuda")
    pset = bp.PointSet(ctx, n=n, device_ptr=d_pts.data_ptr())
    torch.cuda.synchronize()
    L = bp.lib()

    def call_cached(i):
        j = i % sets
        pset.msm_device(d_sc.data_ptr() + 32 * T * j, M, n, d_out[j].data_ptr(), d_st.data_ptr())

    def call_decomp(i):
        j = i % sets
        ctx._check(L.bp_msm_batch_device(ctx._h, d_sc.data_ptr() + 32 * T * j, d_pts.data_ptr(), d_off.data_ptr(), M, T, d_out[j].data_ptr(), d_st.data_ptr()))

    import ctypes
    h_out = torch.zeros((M, 32), dtype=torch.uint8).pin_memory(); h_st = torch.zeros((M,), dtype=torch.uint8).pin_memory()
    off64 = (ctypes.c_uint64 * (M + 1))(*[j * n for j in range(M + 1)])

    def call_e2e(i):
        j = i % sets
        ctx._check(L.bp_msm_points(ctx._h, pset._h, h_sc.data_ptr() + 32 * T * j, M, n, h_out.data_ptr(), h_st.data_ptr()))

    def call_e2e_comp(i):
        j = i % sets
        ctx._check(L.bp_msm_batch(ctx._h, ctypes.cast(h_sc.data_ptr() + 32 * T * j, ctypes.c_char_p), ctypes.cast(h_pts.data_ptr(), ctypes.c_char_p), off64, M,
                                  ctypes.cast(h_out.data_ptr(), ctypes.c_char_p), ctypes.cast(h_st.data_ptr(), ctypes.c_char_p)))

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier(); torch.cuda.synchronize()

    def timed(fn, steps, warmup):
        for i in range(warmup):
            fn(i)
        barrier()
        l0 = ctx.launches
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        a.record(stream)
        for i in range(warmup, warmup + steps):
            fn(i)
        b.record(stream); b.synchronize()
        wall = time.perf_counter() - t0
        tt = torch.tensor([a.elapsed_time(b) * 1e-3, wall], device="cuda", dtype=torch.float64)
        if world > 1:
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        return float(tt[0]), float(tt[1]), ctx.launches - l0

    # parity before timing: first MSM of set 0 against the oracle (byte for byte)
    call_cached(0); ctx.synchronize()
    got_cached = bytes(d_out[0].cpu().numpy().tobytes())
    call_decomp(0); ctx.synchronize()
    got_decomp = bytes(d_out[0].cpu().numpy().tobytes())
    assert got_cached == got_decomp and int(d_st.max()) == 0
    checked = None
    if args.lg <= args.check_lg and rank == 0:
        rc, want = orc.msm(bytes(h_sc[:32 * n].numpy().tobytes()), points)
        assert rc == 0 and want == got_cached[:32], "GPU MSM differs from the oracle"
        checked = "first MSM == oracle (32 bytes)"

    clk = None
    if rank == 0:
        clk = bench.ClockSampler(range(local_world)); clk.start(); time.sleep(0.3); clk.mark_begin()
    s_dev, _, launches = timed(call_cached, args.steps, args.warmup)
    if args.dump_outputs:          # the compressed results of the last timed call, one row of 32 bytes per MSM
        bench.dump_outputs(args.dump_outputs, rank, world, msm_results=d_out[(args.warmup + args.steps - 1) % sets].cpu().numpy())
    s_dec, _, _ = timed(call_decomp, args.steps, args.warmup)
    if clk:
        clk.mark_end(); clk.mark_begin()
    s_e2e, w_e2e, _ = timed(call_e2e, args.steps, args.warmup)
    s_e2c, w_e2c, _ = timed(call_e2e_comp, args.steps, args.warmup)
    clocks = None
    if clk:
        clk.mark_end(); clocks = clk.stop()
    terms_step = world * T
    value = terms_step * args.steps / s_dev
    # roofline: HBM on 64 B per term (SURVEY.md 8d) and the integer-multiply pipe (W windows x 7 field multiplications x 72 wide multiplies per term)
    ctx.prof_enable(True)
    for i in range(3):
        call_cached(i)
    prof = ctx.prof_report(); ctx.prof_enable(False)
    dom = "k_msm_accumulate"
    dom_ms = prof[dom][0] / prof[dom][1]
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = peaks.get("hbm_gbs", bench.HBM_PEAK_GBS)
    alg = M * (64 * n + 32)
    cwin = getattr(args, "window", 0) or {10: 8, 11: 8, 12: 10, 13: 10, 14: 11, 15: 11, 16: 13, 17: 13, 18: 13, 19: 15, 20: 15}.get(args.lg, 13)
    W = (255 + cwin - 1) // cwin
    wide = T * W * 7 * 72 + M * W * (1 << (cwin - 1)) * 3 * 9 * 72
    roofline = {"bound": "hbm", "kernel": dom, "achieved": alg / (dom_ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s", "frac": alg / (dom_ms * 1e-3) / 1e9 / peak, "traffic": None,
                "peak_source": "measured (MEASURED_PEAKS.json)" if peaks else "data sheet (H100 SXM)", "algorithmic_bytes_per_launch": alg,
                "units_per_launch": f"{M} MSMs x ({n} terms x 64 B + 32 B)", "kernel_ms": dom_ms, "kernel_share_of_step": prof[dom][0] / sum(v[0] for v in prof.values()),
                "whole_call": {"achieved_GBps_at_value": alg * args.steps / s_dev / 1e9, "hbm_frac_at_value": alg * args.steps / s_dev / 1e9 / peak},
                "int_pipe": {"window_bits": cwin, "wide_multiplies_per_call": wide, "achieved": wide * args.steps / s_dev, "peak": bench.INT_PEAK, "frac": wide * args.steps / s_dev / bench.INT_PEAK},
                "per_kernel_ms_per_call": {k: round(v[0] / 3, 4) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0])}}
    out = {"metric": metric, "value": value, "unit": "terms/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * s_dev / args.steps,
           "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u32x8 (mod 2^255-19)", "data": "synthetic (generator-chain points, ChaCha20 scalars)",
           "config": config, "with_decompress": {"value": terms_step * args.steps / s_dec, "unit": "terms/s", "ms_per_step": 1e3 * s_dec / args.steps},
           "e2e": {"value": terms_step * args.steps / max(s_e2e, w_e2e), "unit": "terms/s", "h2d_bytes_per_step": 32 * T, "d2h_bytes_per_step": 33 * M, "ms_per_step": 1e3 * max(s_e2e, w_e2e) / args.steps},
           "e2e_compressed": {"value": terms_step * args.steps / max(s_e2c, w_e2c), "unit": "terms/s", "h2d_bytes_per_step": 64 * T, "d2h_bytes_per_step": 33 * M, "ms_per_step": 1e3 * max(s_e2c, w_e2c) / args.steps},
           "gpu_launches": launches, "clocks": clocks, "roofline": roofline, "parity": checked, "diag": {"numa": pin, "scalar_sets": sets}}
    if rank == 0:
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()
