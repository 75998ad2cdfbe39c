"""Launch counts of b2b_chain_run_f32, one chain per forward launch class and path: the fused planar constant-bank run,
the v1 and v0 interpreters, the specialised RQS and radial programs, the tensor-core affine coupling (alone, with folded
BatchNorm neighbours, with a ragged tail), the fp32 affine coupling, the spline, neural spline, MLP and deep MLP
couplings, dense Scale both ways, the TRIL and diagonal MvNormal terminals with and without a batch sum, a chain of
several launches without y, and a terminal batch sum without logjac.  Each call must succeed with the launch count of
LAUNCHES, and every output it was asked for must be finite.

LAUNCHES was recorded on an H100 from a trusted build:  python tests/test_chain_run_launches.py"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

f32 = np.float32


def _chains(B, rng):
    """(name, transform, base, D, N, kernel variant, outputs): outputs names the buffers the call gets, of "y", "lj"
    (log-Jacobian, or logpdf with a base) and "sum" (the batch sum)."""
    def planar(D, s=0.2):
        return B.PlanarLayer((rng.standard_normal(D) * s / np.sqrt(D)).astype(f32),
                             (rng.standard_normal(D) * s / np.sqrt(D)).astype(f32), rng.standard_normal(1).astype(f32))

    def radial(D):
        return B.RadialLayer(rng.standard_normal(1).astype(f32), rng.standard_normal(1).astype(f32),
                             (rng.standard_normal(D) * 0.1).astype(f32))

    def rqs(D, K=8):
        return B.RationalQuadraticSpline(rng.standard_normal((D, K)).astype(f32), rng.standard_normal((D, K)).astype(f32),
                                         rng.standard_normal((D, K - 1)).astype(f32), 3.0)

    def bn(D):
        return B.InvertibleBatchNorm(b=(rng.standard_normal(D) * 0.1).astype(f32),
                                     logs=(rng.standard_normal(D) * 0.1).astype(f32),
                                     m=(rng.standard_normal(D) * 0.1).astype(f32), v=rng.uniform(0.5, 1.5, D).astype(f32))

    def mask(D, n1, lists):
        if lists:
            sel = sorted(rng.choice(np.arange(1, D + 1), n1, replace=False).tolist())
            return B.PartitionMask(D, sel, [i for i in range(1, D + 1) if i not in set(sel)])
        return B.PartitionMask(D, list(range(1, n1 + 1)), list(range(n1 + 1, D + 1)))

    def affine(D, n1, lists=False):
        n2 = D - n1
        return B.Coupling(B.AffineConditioner((rng.standard_normal((2 * n1, n2)) * 0.02).astype(f32),
                                              (rng.standard_normal(2 * n1) * 0.1).astype(f32)), mask(D, n1, lists))

    def spline(D, n1, K=4):
        n2, J = D - n1, 3 * K - 1
        return B.Coupling(B.SplineConditioner((rng.standard_normal((J * n1, n2)) * 0.05).astype(f32),
                                              (rng.standard_normal(J * n1) * 0.1).astype(f32), K=K, B=3.0),
                          mask(D, n1, True))

    def nspline(D, n1, H, K=4):
        n2, J = D - n1, 3 * K - 1
        return B.Coupling(B.MLPSplineConditioner((rng.standard_normal((H, n2)) * 0.1).astype(f32),
                                                 (rng.standard_normal(H) * 0.1).astype(f32),
                                                 (rng.standard_normal((J * n1, H)) * 0.05).astype(f32),
                                                 (rng.standard_normal(J * n1) * 0.1).astype(f32), K=K, B=3.0,
                                                 activation="leaky_relu", slope=0.1), mask(D, n1, True))

    def mlp(D, n1, H, lists=False):
        n2 = D - n1
        return B.Coupling(B.MLPConditioner((rng.standard_normal((H, n2)) * 0.1).astype(f32),
                                           (rng.standard_normal(H) * 0.1).astype(f32),
                                           (rng.standard_normal((2 * n1, H)) * 0.05).astype(f32),
                                           (rng.standard_normal(2 * n1) * 0.1).astype(f32)), mask(D, n1, lists))

    def deep(D, n1, H, M):
        n2 = D - n1
        ws = ([(rng.standard_normal((H, n2)) * 0.1).astype(f32)] +
              [(rng.standard_normal((H, H)) * 0.1).astype(f32) for _ in range(M - 1)] +
              [(rng.standard_normal((2 * n1, H)) * 0.05).astype(f32)])
        cs = [(rng.standard_normal(H) * 0.1).astype(f32) for _ in range(M)] + [(rng.standard_normal(2 * n1) * 0.1).astype(f32)]
        return B.Coupling(B.DeepMLPConditioner(ws, cs), mask(D, n1, True))

    def dense(D):
        return B.Scale((np.eye(D) + rng.standard_normal((D, D)) * 0.1 / np.sqrt(D)).astype(f32))

    def diag(D):
        return B.MvNormal(D, mu=(rng.standard_normal(D) * 0.1).astype(f32), sigma=rng.uniform(0.5, 1.5, D).astype(f32))

    def tril(D):
        L = np.tril(rng.standard_normal((D, D)) * 0.1 / np.sqrt(D)) + np.diag(rng.uniform(0.8, 1.2, D))
        return B.MvNormal(D, mu=(rng.standard_normal(D) * 0.1).astype(f32), scale_tril=L.astype(f32))

    C = B.Composed
    y_lj, all3 = ("y", "lj"), ("y", "lj", "sum")
    fused = C(planar(64), radial(64), bn(64), B.Shift(0.1))
    return [
        ("planar-const", C(*[planar(64) for _ in range(4)]), None, 64, 3000, 0, y_lj),
        ("planar-const-diag-sum", B.inverse(C(planar(64), planar(64))), diag(64), 64, 3000, 0, all3),
        ("fused-v1", fused, None, 64, 3000, 2, y_lj),
        ("fused-v0", fused, None, 64, 3000, 1, y_lj),
        ("fused-v0-diag-sum", C(planar(100), B.Shift(0.2)), diag(100), 100, 3000, 0, all3),
        ("rqs-unrolled", rqs(32), None, 32, 3000, 0, y_lj),
        ("radial-unrolled", B.inverse(C(radial(64), radial(64), radial(64))), None, 64, 3000, 0, y_lj),
        ("coupling-tc", affine(128, 64), None, 128, 4096, 0, y_lj),
        ("coupling-tc-ragged", affine(128, 64), None, 128, 4096 + 13, 0, y_lj),
        ("coupling-tc-fold", C(bn(128), affine(128, 64), bn(128)), None, 128, 4096 + 13, 0, y_lj),
        ("coupling-tc-fold-pre", C(bn(128), affine(128, 64), planar(128)), None, 128, 4096, 0, y_lj),
        ("coupling-fp32", affine(128, 64), None, 128, 4096 + 13, 10, y_lj),
        ("coupling-fp32-fold", C(bn(128), affine(128, 64), bn(128)), None, 128, 4096 + 13, 10, y_lj),
        ("coupling-lists", B.inverse(affine(64, 20, True)), None, 64, 3000, 0, y_lj),
        ("spline-coupling", spline(64, 16), None, 64, 3000, 0, y_lj),
        ("mlp-spline-coupling", B.inverse(nspline(64, 16, 32)), None, 64, 3000, 0, y_lj),
        ("mlp-coupling", mlp(64, 32, 64), None, 64, 3000, 0, y_lj),
        ("deep-mlp-coupling", B.inverse(deep(64, 24, 32, 3)), None, 64, 3000, 0, y_lj),
        ("scale", dense(48), None, 48, 3000, 0, y_lj),
        ("scale-inv", B.inverse(dense(48)), None, 48, 3000, 0, y_lj),
        ("scale-no-y", B.inverse(dense(48)), None, 48, 3000, 0, ("lj",)),
        ("tril", C(), tril(48), 48, 3000, 0, y_lj),
        ("tril-sum", C(planar(48)), tril(48), 48, 3000, 0, all3),
        ("diag", C(B.Shift(0.3)), diag(40), 40, 3000, 0, y_lj),
        ("diag-sum", C(B.Shift(0.3)), diag(40), 40, 3000, 0, all3),
        ("no-y", C(planar(64), affine(64, 32), radial(64), spline(64, 16), mlp(64, 32, 32), dense(64)), None, 64, 3000, 0,
         ("lj",)),
        ("sum-no-logjac", C(affine(64, 32), B.Shift(0.1), mlp(64, 32, 32, True)), diag(64), 64, 3000, 0, ("sum",)),
        ("sum-no-logjac-tril", C(spline(64, 16), dense(64)), tril(64), 64, 3000, 0, ("y", "sum")),
    ]


def _run_case(B, t, base, D, N, variant, outputs, rng):
    """(status, launches, y, logjac, batch sum) of one call; the outputs not asked for are None."""
    import torch

    from bijectors_jl_b200 import _lib
    from bijectors_jl_b200.interface import _desc_array, _stream

    L_ = _lib.lib()
    descs = t._descs(False, D) + ([base._terminal_desc()] if base is not None else [])
    arr = _desc_array(descs)
    x = torch.from_numpy((rng.standard_normal((D, N)) * 0.5).astype(f32)).cuda().t().contiguous().t()
    y = torch.full((N, D), float("nan"), device="cuda").t() if "y" in outputs else None
    lj = torch.full((N,), float("nan"), device="cuda") if "lj" in outputs else None
    s = torch.full((1,), float("nan"), dtype=torch.float64, device="cuda") if "sum" in outputs else None
    need = L_.b2b_chain_workspace_bytes(arr, len(descs), D, N, int(y is not None), int(s is not None))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device="cuda")
    assert L_.b2b_set_kernel_variant(variant) == 0
    try:
        st = L_.b2b_chain_run_f32(arr, len(descs), x.data_ptr(), y.data_ptr() if y is not None else None,
                                  lj.data_ptr() if lj is not None else None, s.data_ptr() if s is not None else None,
                                  D, N, D, D, 0, ws.data_ptr(), need, _stream())
        n = L_.b2b_last_launch_count()
    finally:
        L_.b2b_set_kernel_variant(0)
    torch.cuda.synchronize()
    return st, n, y, lj, s


def measure_all(B):
    rng = np.random.default_rng(2025)
    return {name: _run_case(B, t, base, D, N, variant, outputs, rng)
            for name, t, base, D, N, variant, outputs in _chains(B, rng)}


# b2b_last_launch_count() by chain
LAUNCHES = {
    "planar-const": 1,
    "planar-const-diag-sum": 2,
    "fused-v1": 1,
    "fused-v0": 1,
    "fused-v0-diag-sum": 2,
    "rqs-unrolled": 1,
    "radial-unrolled": 1,
    "coupling-tc": 2,
    "coupling-tc-ragged": 3,
    "coupling-tc-fold": 4,
    "coupling-tc-fold-pre": 4,
    "coupling-fp32": 1,
    "coupling-fp32-fold": 2,
    "coupling-lists": 1,
    "spline-coupling": 1,
    "mlp-spline-coupling": 1,
    "mlp-coupling": 1,
    "deep-mlp-coupling": 1,
    "scale": 2,
    "scale-inv": 3,
    "scale-no-y": 2,
    "tril": 1,
    "tril-sum": 3,
    "diag": 1,
    "diag-sum": 2,
    "no-y": 7,
    "sum-no-logjac": 5,
    "sum-no-logjac-tril": 5,
}


@pytest.fixture(scope="module")
def results():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return measure_all(B)


CASES = tuple(LAUNCHES)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_launches(results, name):
    import torch

    st, n, y, lj, s = results[name]
    assert st == 0, (name, st)
    assert n == LAUNCHES[name], (name, n)
    for what, v in (("y", y), ("logjac", lj), ("sum", s)):
        assert v is None or bool(torch.isfinite(v).all()), (name, what)


if __name__ == "__main__":
    import json

    import bijectors_jl_b200 as B

    got = measure_all(B)
    print(json.dumps({name: v[1] for name, v in got.items()}, indent=1))
    print(json.dumps({name: v[0] for name, v in got.items()}))
