"""Times the fused planar chain kernel against the device copy rate of the same bytes.

  python tools/bench_planar_chain.py [--iters 300] [--warmup 5] [--json OUT]

At D = 128, N = 2^20, Float32 it reports, with CUDA events (launches back to back, one event between consecutive
launches, median over --iters launches after --warmup untimed ones):
  copy        a device-to-device copy of the 512 MiB batch plus a 4 MiB write (the logjac vector): the same bytes as one
              fused chain launch, 4*(2D+1) B/sample, moved by the copy engine path of torch (cudaMemcpyAsync)
  fwd[L]      with_logabsdet_jacobian through L = 1..8 PlanarLayers, device-resident parameters (one launch)
  host_fwd8   the same 8-layer chain with host-resident parameters (kernel-argument block)
  inv8        the inverse of the 8-layer chain
  logpdf_sum8 logpdf(transformed(MvNormal, flow), y) + batch sum (inverse chain + base density, no D x N store)
The card name and power limit are read with nvidia-smi in the same run, and the SM clock and board power are sampled
every 20 ms during every timed window (median of the samples inside it): a card held at its power limit lowers its SM
clock, which a rate at a fixed byte count does not show by itself.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bijectors_jl_b200 as B  # noqa: E402

D, N, LMAX = 128, 1 << 20, 8
f32 = np.float32


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.strip().split(",")]))
    except Exception as ex:  # the numbers below still stand; the card is then named by torch only
        return {"name": torch.cuda.get_device_name(), "error": str(ex)[:200]}


class Sampler:
    """nvidia-smi SM clock and board power every 20 ms, host-timestamped so that samples can be assigned to windows."""

    def __init__(self):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        try:
            self.p = subprocess.Popen(["nvidia-smi", "--query-gpu=timestamp,clocks.sm,power.draw",
                                       "--format=csv,noheader,nounits", "-lms", "20", "-i", str(torch.cuda.current_device())],
                                      stdout=self.f, stderr=subprocess.DEVNULL)
        except Exception:
            self.p = None

    def stop(self):
        rows = []
        if self.p is not None:
            self.p.terminate()
            try:
                self.p.wait(timeout=5)
            except Exception:
                self.p.kill()
                self.p.wait()
            self.f.flush()
            for r in open(self.f.name):
                try:
                    ts, mhz, w = [v.strip() for v in r.split(",")]
                    rows.append((time.mktime(time.strptime(ts[:19], "%Y/%m/%d %H:%M:%S")) + float("0" + ts[19:]),
                                 float(mhz), float(w)))
                except Exception:
                    continue
        os.unlink(self.f.name)
        return rows


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(iters + 1)]
    ev[0].record()
    for i in range(iters):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    t1 = time.time()
    ts = [ev[i].elapsed_time(ev[i + 1]) for i in range(iters)]
    return float(np.median(ts)), float(min(ts)), float(max(ts)), (t1 - sum(ts) * 1e-3, t1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_planar_chain.py needs a GPU"
    iters, warmup = max(args.iters, 20), max(args.warmup, 3)

    layers = []
    for l in range(LMAX):  # the parameters of bench.py's headline chain
        r = np.random.Generator(np.random.PCG64(100 + l))
        layers.append(B.PlanarLayer((r.standard_normal(D) / np.sqrt(D)).astype(f32),
                                    (r.standard_normal(D) / np.sqrt(D)).astype(f32), r.standard_normal(1).astype(f32)))
    gen = torch.Generator(device="cuda").manual_seed(1234)
    x = torch.randn((N, D), device="cuda", generator=gen).t()
    y, lj = B.colmajor_empty(D, N), torch.empty(N, device="cuda")
    bytes_launch = N * 4 * (2 * D + 1)
    res = {"card": card(), "D": D, "N": N, "iters": iters, "warmup": warmup, "bytes_per_launch": bytes_launch, "ms": {}}

    windows = {}

    def put(name, t):
        med, lo, hi, windows[name] = t
        res["ms"][name] = {"median": med, "min": lo, "max": hi, "gbs": bytes_launch / (med * 1e-3) / 1e9}
        print(f"{name:12s} {med:.4f} ms (min {lo:.4f}, max {hi:.4f})  {bytes_launch / (med * 1e-3) / 1e9:7.1f} GB/s",
              flush=True)

    sampler = Sampler()

    try:
        # the copy ceiling: same bytes read + written as one fused launch
        src_lj, dst_lj = torch.zeros(N, device="cuda"), torch.empty(N, device="cuda")

        def copy():
            y.copy_(x)
            dst_lj.copy_(src_lj)

        put("copy", median_ms(copy, iters, warmup))
        for L in range(1, LMAX + 1):
            flow = B.Composed(*layers[:L])
            put(f"fwd{L}", median_ms(lambda: B.run_chain(flow, x, y=y, logjac=lj), iters, warmup))
        flow = B.Composed(*layers)
        host_flow = B.Composed(*[lay.to("cpu") for lay in layers])
        put("host_fwd8", median_ms(lambda: B.run_chain(host_flow, x, y=y, logjac=lj), iters, warmup))
        B.run_chain(flow, x, y=y, logjac=lj)
        x2, lj2 = B.colmajor_empty(D, N), torch.empty(N, device="cuda")
        inv = B.inverse(flow)
        put("inv8", median_ms(lambda: B.run_chain(inv, y, y=x2, logjac=lj2), iters, warmup))
        r = np.random.Generator(np.random.PCG64(199))
        td = B.transformed(B.MvNormal(D, (r.standard_normal(D) * 0.1).astype(f32), r.uniform(0.5, 2.0, D).astype(f32)), flow)
        total = torch.zeros((), dtype=torch.float64, device="cuda")
        put("logpdf_sum8", median_ms(lambda: B.logpdf_sum(td, y, out=total), iters, warmup))
        res["ms"]["logpdf_sum8"]["gbs"] = N * 4 * (D + 1) / (res["ms"]["logpdf_sum8"]["median"] * 1e-3) / 1e9
        time.sleep(0.1)
    finally:
        samples = sampler.stop()
    for name, (t0, t1) in windows.items():
        inside = [(mhz, w) for (t, mhz, w) in samples if t0 <= t <= t1]
        res["ms"][name]["sm_mhz"] = float(np.median([m for m, _ in inside])) if inside else None
        res["ms"][name]["power_w"] = float(np.median([w for _, w in inside])) if inside else None
        res["ms"][name]["clock_samples"] = len(inside)
        print(f"{name:12s} SM clock {res['ms'][name]['sm_mhz']} MHz, board power {res['ms'][name]['power_w']} W "
              f"({len(inside)} samples)")
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
