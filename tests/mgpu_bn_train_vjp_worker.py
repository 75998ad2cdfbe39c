"""torchrun worker: reverse mode of the training-mode InvertibleBatchNorm over a column-sharded batch (one all-reduce of
4D+2 doubles inside b2b_batchnorm_train_vjp_f32).  Launched by tests/test_batchnorm_train_vjp.py:
torchrun --nproc-per-node 2 tests/mgpu_bn_train_vjp_worker.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def main():
    import bijectors_jl_b200 as B
    from bijectors_jl_b200.distributed import Communicator, shard_columns
    from oracle import oracle_np as O
    import bn_train_vjp_oracle as BO

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    comm = Communicator()
    assert comm.handle is not None, "libb2b NCCL communicator was not created"
    f32 = np.float32
    rng = np.random.default_rng(21)  # identical on every rank
    D, N = 200, 30_001
    b, logs = (rng.standard_normal(D) * 0.3).astype(f32), (rng.standard_normal(D) * 0.3).astype(f32)
    x = (rng.standard_normal((D, N)) * 1.7 + 0.3).astype(f32)
    ybar, ljbar = rng.standard_normal((D, N)).astype(f32), rng.standard_normal(N).astype(f32)
    lo, hi = shard_columns(N, rank, world)
    bn = B.InvertibleBatchNorm(b=b, logs=logs, training=True)
    xbar, g = B.batchnorm_train_vjp(bn, B.from_numpy(x[:, lo:hi]), B.from_numpy(ybar[:, lo:hi]),
                                    torch.from_numpy(np.ascontiguousarray(ljbar[lo:hi])).cuda(), comm=comm)
    bn64 = O.BatchNormParams(b.astype(np.float64), logs.astype(np.float64), np.zeros(D), np.ones(D), np.float64(f32(1e-5)),
                             np.float64(f32(0.1)))
    xo, bo, lo_ = BO.batchnorm_train_vjp(bn64, x.astype(np.float64), ybar.astype(np.float64), ljbar.astype(np.float64))
    xs, bs, ls = BO.batchnorm_train_vjp_shard(bn64, x.astype(np.float64), ybar.astype(np.float64), ljbar.astype(np.float64),
                                              lo, hi)

    def rel(a, b_):
        return np.linalg.norm(np.asarray(a, np.float64) - b_) / np.linalg.norm(b_)

    # x̄ of this rank's columns is the full-batch x̄ there (global statistics and sums)
    assert rel(B.to_numpy(xbar), xo[:, lo:hi]) <= 1e-5, rel(B.to_numpy(xbar), xo[:, lo:hi])
    # b̄ / l̄ogs are this rank's share ...
    floor = 2e-5 * np.sqrt(hi - lo)
    assert np.all(np.abs(B.to_numpy(g["b"]) - bs) <= np.maximum(2e-5 * np.abs(bs), floor))
    assert np.all(np.abs(B.to_numpy(g["logs"]) - ls) <= np.maximum(2e-5 * np.abs(ls), floor))
    # ... and one float64 all-reduce gives the full-batch cotangents
    buf = torch.cat([g["b"].double(), g["logs"].double()])
    comm.allreduce_sum_(buf)
    tot = buf.cpu().numpy()
    floor = 2e-5 * np.sqrt(N)
    assert np.all(np.abs(tot[:D] - bo) <= np.maximum(2e-5 * np.abs(bo), floor))
    assert np.all(np.abs(tot[D:] - lo_) <= np.maximum(2e-5 * np.abs(lo_), floor))
    comm.close()
    dist.barrier()
    if rank == 0:
        print(f"bn train vjp ok: world={world} rel_err x̄={rel(B.to_numpy(xbar), xo[:, lo:hi]):.2e}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
