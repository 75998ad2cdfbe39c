#!/usr/bin/env python
"""Throughput + roofline of EVERY BASELINE.json config (the headline bench.py covers configs[1] only).

  python bench_configs.py [--iters K] [--json out.json]
  torchrun --nproc-per-node N bench_configs.py   (configs 3/4 shard their batch over the N ranks; config 4 adds
                                                  the one NCCL sum of the batch log-density)

Per config: device-resident CUDA-event timing (max over ranks), samples/s, algorithmic bytes per launch and the
achieved fraction of the measured HBM roofline for (a) the fused chain launch and (b) one launch per layer.
Inputs are larger than L2 or the buffers are rotated so that no iteration re-reads a cached batch.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

f32 = np.float32


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"]), "measured"
    return 3350.0, "fallback: H100 SXM data-sheet HBM3 bandwidth"


def time_ms(fn, iters, warmup=3, world=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
        torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda", dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    return float(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default="")
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    import bijectors_jl_b200 as B
    from bijectors_jl_b200.distributed import Communicator, shard_columns

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    comm = None
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        comm = Communicator()
    peak, peak_src = peaks()
    out = {"n_gpus": world, "hbm_peak_gbs": peak, "peak_source": peak_src, "configs": {}}
    gen = torch.Generator(device="cuda").manual_seed(7 + rank)

    def batch(D, N, scale=1.0):
        return (torch.randn((N, D), device="cuda", generator=gen) * scale).t()

    def report(name, N_total, ms, bytes_per_launch_fused, launches_layerwise=None, ms_layerwise=None, bytes_layerwise=None,
               extra=None):
        r = {"samples_per_s": N_total / (ms * 1e-3), "ms": ms, "fused_gbs": bytes_per_launch_fused / (ms * 1e-3) / 1e9,
             "fused_frac": bytes_per_launch_fused / (ms * 1e-3) / 1e9 / peak / world}
        if ms_layerwise is not None:
            r.update({"layerwise_ms": ms_layerwise, "layerwise_launches": launches_layerwise,
                      "layerwise_gbs": bytes_layerwise / (ms_layerwise * 1e-3) / 1e9,
                      "layerwise_frac": bytes_layerwise / (ms_layerwise * 1e-3) / 1e9 / peak / world})
        if extra:
            r.update(extra)
        out["configs"][name] = r
        if rank == 0:
            print(name, json.dumps(r), flush=True)

    def layerwise(layers, x, y, lj):
        B.run_chain(layers[0], x, y=y, logjac=lj)
        for lay in layers[1:]:
            B.run_chain(lay, y, y=y, logjac=lj, accumulate=True)

    want = set(args.only.split(",")) if args.only else None

    # ---- C2: 8 x Planar, D=128, N=2^20 per GPU ------------------------------------------------------------
    if not want or "C2" in want:
        D, N, L = 128, 1 << 20, 8
        ls = []
        for l in range(L):
            r = np.random.Generator(np.random.PCG64(100 + l))
            ls.append(B.PlanarLayer((r.standard_normal(D) / np.sqrt(D)).astype(f32), (r.standard_normal(D) / np.sqrt(D)).astype(f32),
                                    r.standard_normal(1).astype(f32)))
        flow = B.Composed(*ls)
        x, y, lj = batch(D, N), B.colmajor_empty(D, N), torch.empty(N, device="cuda")
        ms = time_ms(lambda: B.run_chain(flow, x, y=y, logjac=lj), args.iters, world=world)
        msl = time_ms(lambda: layerwise(ls, x, y, lj), args.iters, world=world)
        report("C2_planar8_D128_fwd", world * N, ms, world * N * 4 * (2 * D + 1), L, msl, world * N * 4 * (L * (2 * D + 1) + L - 1))
        inv = B.inverse(flow)
        ms = time_ms(lambda: B.run_chain(inv, y, y=x, logjac=lj), max(args.iters // 2, 3), world=world)
        report("C2_planar8_D128_inverse", world * N, ms, world * N * 4 * (2 * D + 1))
        # logpdf(transformed(MvNormal, flow), y) + batch sum: inverse chain + base density, no D x N store
        r = np.random.Generator(np.random.PCG64(199))
        td = B.transformed(B.MvNormal(D, (r.standard_normal(D) * 0.1).astype(f32), r.uniform(0.5, 2.0, D).astype(f32)), flow)
        B.run_chain(flow, x, y=y, logjac=lj)
        ms = time_ms(lambda: B.logpdf_sum(td, y), max(args.iters // 2, 3), world=world)
        report("C2_planar8_D128_logpdf_sum", world * N, ms, world * N * 4 * (D + 1),
               extra={"accounting": "read column + write logpdf: 4*(D+1) B/sample"})
        del x, y

    # ---- C3: 6 x Radial, D=64, N=2^20 per GPU, forward + inverse ------------------------------------------
    if not want or "C3" in want:
        D, N, L = 64, 1 << 20, 6
        ls = []
        for l in range(L):
            r = np.random.Generator(np.random.PCG64(200 + l))
            ls.append(B.RadialLayer(r.standard_normal(1).astype(f32), r.standard_normal(1).astype(f32), r.standard_normal(D).astype(f32)))
        flow = B.Composed(*ls)
        x, y, lj = batch(D, N), B.colmajor_empty(D, N), torch.empty(N, device="cuda")
        ms = time_ms(lambda: B.run_chain(flow, x, y=y, logjac=lj), args.iters, world=world)
        msl = time_ms(lambda: layerwise(ls, x, y, lj), args.iters, world=world)
        report("C3_radial6_D64_fwd", world * N, ms, world * N * 4 * (2 * D + 1), L, msl, world * N * 4 * (L * (2 * D + 1) + L - 1))
        B.run_chain(flow, x, y=y, logjac=lj)
        inv = B.inverse(flow)
        x2 = B.colmajor_empty(D, N)
        ms = time_ms(lambda: B.run_chain(inv, y, y=x2, logjac=lj), args.iters, world=world)
        report("C3_radial6_D64_inverse", world * N, ms, world * N * 4 * (2 * D + 1))
        del x, y, x2

    # ---- C4: RQS K=8, D=32, N=2^19 TOTAL, sharded over the ranks -------------------------------------------
    if not want or "C4" in want:
        D, Ntot, K = 32, 1 << 19, 8
        lo, hi = shard_columns(Ntot, rank, world)
        N = hi - lo
        r = np.random.Generator(np.random.PCG64(300))
        rqs = B.RationalQuadraticSpline(r.standard_normal((D, K)).astype(f32), r.standard_normal((D, K)).astype(f32),
                                        r.standard_normal((D, K - 1)).astype(f32), 3.0)
        # the 64 MiB batch is of the order of L2 (50 MB): rotate over 4 buffer pairs (> L2 in total) between iterations
        nbuf = 4 if world == 1 else 16
        xs = [batch(D, N, 1.5) for _ in range(nbuf)]
        ys = [B.colmajor_empty(D, N) for _ in range(nbuf)]
        lj = torch.empty(N, device="cuda")
        it = [0]

        def step():
            i = it[0] % nbuf
            it[0] += 1
            B.run_chain(rqs, xs[i], y=ys[i], logjac=lj)

        ms = time_ms(step, args.iters * 2, world=world)
        report("C4_rqs_K8_D32_fwd", Ntot, ms, Ntot * 4 * (2 * D + 1), extra={"l2": f"rotating {nbuf} buffer pairs"})
        irqs = B.inverse(rqs)

        def stepi():
            i = it[0] % nbuf
            it[0] += 1
            B.run_chain(irqs, ys[i], y=xs[i], logjac=lj)

        ms = time_ms(stepi, args.iters * 2, world=world)
        report("C4_rqs_K8_D32_inverse", Ntot, ms, Ntot * 4 * (2 * D + 1), extra={"l2": f"rotating {nbuf} buffer pairs"})
        del xs, ys

    # ---- C5: RealNVP 4 x (Coupling + BatchNorm), D=256, N=2^22 TOTAL sharded; logpdf + NCCL sum ---------
    if not want or "C5" in want:
        D, Ntot = 256, 1 << 22
        lo, hi = shard_columns(Ntot, rank, world)
        N = hi - lo
        if world == 1:
            N = Ntot // 8  # the per-GPU share of the 8-GPU config (4 GiB total would still fit; keep the bench short)
        r = np.random.Generator(np.random.PCG64(400))
        ls = []
        for l in range(4):
            first = l % 2 == 0
            idx1 = list(range(1, 129)) if first else list(range(129, 257))
            idx2 = list(range(129, 257)) if first else list(range(1, 129))
            W = (r.standard_normal((256, 128)) * 0.05 / np.sqrt(128)).astype(f32)
            ls.append(B.Coupling(B.AffineConditioner(W, np.zeros(256, f32)), B.PartitionMask(D, idx1, idx2)))
            ls.append(B.InvertibleBatchNorm(b=(r.standard_normal(D) * 0.1).astype(f32), logs=(r.standard_normal(D) * 0.1).astype(f32),
                                            m=(r.standard_normal(D) * 0.1).astype(f32), v=r.uniform(0.5, 1.5, D).astype(f32)))
        flow = B.Composed(*ls)
        td = B.transformed(B.MvNormal(D), flow)
        yb = batch(D, N)
        xb, lj = B.colmajor_empty(D, N), torch.empty(N, device="cuda")
        ms = time_ms(lambda: B.run_chain(flow, yb, y=xb, logjac=lj), args.iters, world=world)
        launches = B.lib().b2b_last_launch_count()
        Neff = N * world
        # BatchNorm layers are folded into the coupling launches: 4 data passes, each reads D, writes D + logjac
        # (the unfolded reference structure would be 8 passes)
        report("C5_realnvp_D256_fwd", Neff, ms, Neff * 4 * (4 * (2 * D + 1) + 3),
               extra={"launches": launches, "cols_per_gpu": N, "data_passes": 4,
                      "unfolded_8pass_equiv_frac": Neff * 4 * (8 * (2 * D + 1) + 7) / (ms * 1e-3) / 1e9 / peak / world})
        cpl = ls[0]
        ms1 = time_ms(lambda: B.run_chain(cpl, yb, y=xb, logjac=lj), args.iters, world=world)
        report("C5_coupling_tc_single", Neff, ms1, Neff * 4 * (2 * D + 1), extra={"launches": B.lib().b2b_last_launch_count()})
        B.lib().b2b_set_kernel_variant(10)
        ms2 = time_ms(lambda: B.run_chain(cpl, yb, y=xb, logjac=lj), max(args.iters // 4, 3), world=world)
        B.lib().b2b_set_kernel_variant(0)
        report("C5_coupling_fp32_single", Neff, ms2, Neff * 4 * (2 * D + 1))
        total = torch.zeros((), dtype=torch.float64, device="cuda")

        def logpdf_step():
            B.logpdf_sum(td, yb, out=total)
            if comm is not None:
                comm.allreduce_sum_(total.reshape(1))

        ms = time_ms(logpdf_step, args.iters, world=world)
        # inverse chain: 4 coupling passes with every BatchNorm folded in + the MvNormal pass (reads D + logjac, writes 1)
        report("C5_realnvp_logpdf_sum", Neff, ms, Neff * 4 * (4 * (2 * D + 1) + 3 + (D + 2)),
               extra={"collective": "one ncclAllReduce(sum) of 8 bytes per step" if world > 1 else "none (1 GPU)",
                      "total_logpdf": float(total)})

    if rank == 0 and args.json:
        json.dump(out, open(args.json, "w"), indent=1)
    if comm is not None:
        comm.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
