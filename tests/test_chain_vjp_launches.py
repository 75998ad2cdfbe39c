"""Launch counts and cotangent routing of b2b_chain_vjp_f32, one chain per reverse-mode segment class (planar run, radial
run, RQS, affine coupling, eval BatchNorm, elementwise run, TRIL terminal, spline coupling, dense Scale, MLP coupling) and a
mixed chain.  Each chain runs with ȳ given and NULL, and with every cotangent, a subset and none requested.  Each call must
succeed with the launch count of LAUNCHES.  A subset must give the same bits in its slots as the full request, and x̄ must
not depend on which cotangents are requested.

LAUNCHES was recorded on an H100 from a trusted build:  python tests/test_chain_vjp_launches.py"""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

f32 = np.float32
REQUESTS = ("all", "subset", "none")


def _chains(B, rng):
    """(name, transform, D, N, input layout): x at an offset of `xoff` floats with leading dimensions ldx, ldȳ, ldx̄."""
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

    def affine(D, n1, lists):
        n2 = D - n1
        return B.Coupling(B.AffineConditioner((rng.standard_normal((2 * n1, n2)) * 0.02).astype(f32),
                                              (rng.standard_normal(2 * n1) * 0.1).astype(f32)), mask(D, n1, lists))

    def spline(D, n1, K=4):
        n2, J = D - n1, 3 * K - 1
        return B.Coupling(B.SplineConditioner((rng.standard_normal((J * n1, n2)) * 0.05).astype(f32),
                                              (rng.standard_normal(J * n1) * 0.1).astype(f32), K=K, B=3.0),
                          mask(D, n1, True))

    def mlp(D, n1, H, lists):
        n2 = D - n1
        return B.Coupling(B.MLPConditioner((rng.standard_normal((H, n2)) * 0.1).astype(f32),
                                           (rng.standard_normal(H) * 0.1).astype(f32),
                                           (rng.standard_normal((2 * n1, H)) * 0.05).astype(f32),
                                           (rng.standard_normal(2 * n1) * 0.1).astype(f32)), mask(D, n1, lists))

    def dense(D):
        return B.Scale((np.eye(D) + rng.standard_normal((D, D)) * 0.1 / np.sqrt(D)).astype(f32))

    def diag(D):
        return B.MvNormal(D, mu=(rng.standard_normal(D) * 0.1).astype(f32), sigma=rng.uniform(0.5, 1.5, D).astype(f32))

    def tril(D):
        L = np.tril(rng.standard_normal((D, D)) * 0.1 / np.sqrt(D)) + np.diag(rng.uniform(0.8, 1.2, D))
        return B.MvNormal(D, mu=(rng.standard_normal(D) * 0.1).astype(f32), scale_tril=L.astype(f32))

    dense_io = (0, 0, 0, 0)  # xoff, extra ldx, extra ldȳ, extra ldx̄
    return [
        ("planar", B.Composed(*[planar(64) for _ in range(3)]), None, 64, 3000, dense_io),
        ("planar-embedded", B.inverse(B.Composed(planar(36), planar(36))), None, 36, 3000, dense_io),
        ("planar-misaligned", B.Composed(planar(64), planar(64)), None, 64, 3000, (1, 3, 1, 1)),
        ("radial", B.Composed(radial(48), B.inverse(radial(48)), radial(48)), None, 48, 3000, dense_io),
        ("rqs", rqs(32), None, 32, 3000, dense_io),
        ("coupling-rows", affine(64, 24, False), None, 64, 3000, dense_io),
        ("coupling-lists", B.inverse(affine(64, 20, True)), None, 64, 3000, dense_io),
        ("batchnorm", bn(96), None, 96, 3000, dense_io),
        ("elementwise", B.Composed(B.Shift(0.3), B.Permute((rng.permutation(40) + 1).tolist()), B.LeakyReLU(0.2)),
         diag(40), 40, 3000, dense_io),
        ("tril", B.Composed(), tril(48), 48, 3000, dense_io),
        ("spline-coupling", spline(64, 16), None, 64, 3000, dense_io),
        ("scale", dense(48), None, 48, 3000, dense_io),
        ("mlp-coupling-rows", mlp(64, 32, 64, False), None, 64, 3000, dense_io),
        ("mlp-coupling-lists", B.inverse(mlp(64, 24, 32, True)), None, 64, 3000, dense_io),
        ("mixed", B.Composed(planar(64), bn(64), affine(64, 32, False), radial(64), rqs(64), spline(64, 16), dense(64),
                             mlp(64, 32, 32, True), B.Shift(0.1)), diag(64), 64, 3000, (1, 3, 1, 1)),
    ]


def _slots(descs, D):
    from bijectors_jl_b200.interface import _SLOTS

    out = []
    for l, d in enumerate(descs):
        if d.kind in _SLOTS:
            for i, shape in enumerate(_SLOTS[d.kind][1](d, D)):
                out.append((l, i, shape))
    return out


def _run_case(B, name, t, base, D, N, io, rng):
    """{(ȳ given, request): (status, launches, x̄, {slot: cotangent})} for one chain."""
    import torch

    from bijectors_jl_b200 import _lib
    from bijectors_jl_b200.interface import _desc_array, _stream

    L_ = _lib.lib()
    descs = t._descs(False, D) + ([base._terminal_desc()] if base is not None else [])
    arr = _desc_array(descs)
    xoff, dx, dy, dxb = io
    ldx, ldyb, ldxb = D + dx, D + dy, D + dxb
    xbuf = torch.zeros(N * ldx + xoff, device="cuda")
    x = xbuf[xoff:].view(N, ldx).t()
    x[:D] = torch.from_numpy((rng.standard_normal((D, N)) * 0.5).astype(f32)).cuda()
    yb = torch.from_numpy(rng.standard_normal((ldyb, N)).astype(f32)).cuda().t().contiguous().t()
    lb = torch.from_numpy(rng.standard_normal(N).astype(f32)).cuda()
    need = L_.b2b_chain_vjp_workspace_bytes(arr, len(descs), D, N)
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device="cuda")
    slots = _slots(descs, D)
    assert slots, name
    out = {}
    for given in (True, False):
        for req in REQUESTS:
            chosen = slots if req == "all" else slots[::2] if req == "subset" else []
            bars = (ctypes.c_void_p * (4 * len(descs)))()
            got = {}
            for l, i, shape in chosen:
                got[(l, i)] = torch.full(shape, float("nan"), device="cuda")
                bars[4 * l + i] = got[(l, i)].data_ptr()
            xb = torch.full((N, ldxb), float("nan"), device="cuda").t()
            st = L_.b2b_chain_vjp_f32(arr, len(descs), x.data_ptr(), yb.data_ptr() if given else None, lb.data_ptr(),
                                      xb.data_ptr(), ctypes.cast(bars, ctypes.c_void_p) if chosen else None, D, N, ldx,
                                      ldyb, ldxb, ws.data_ptr(), need, _stream())
            n = L_.b2b_last_launch_count()
            torch.cuda.synchronize()
            out[(given, req)] = (st, n, xb[:D].clone(), got)
    return out


def measure_all(B):
    rng = np.random.default_rng(2024)
    return {name: _run_case(B, name, t, base, D, N, io, rng) for name, t, base, D, N, io in _chains(B, rng)}


# b2b_last_launch_count() by chain and call: ybar / noybar, then the cotangents requested
LAUNCHES = {
    "planar": {"ybar-all": 8, "ybar-subset": 8, "ybar-none": 1, "noybar-all": 9, "noybar-subset": 9, "noybar-none": 2},
    "planar-embedded": {"ybar-all": 14, "ybar-subset": 14, "ybar-none": 7, "noybar-all": 13, "noybar-subset": 13, "noybar-none": 6},
    "planar-misaligned": {"ybar-all": 11, "ybar-subset": 11, "ybar-none": 4, "noybar-all": 11, "noybar-subset": 11, "noybar-none": 4},
    "radial": {"ybar-all": 3, "ybar-subset": 3, "ybar-none": 2, "noybar-all": 4, "noybar-subset": 4, "noybar-none": 3},
    "rqs": {"ybar-all": 2, "ybar-subset": 2, "ybar-none": 2, "noybar-all": 3, "noybar-subset": 3, "noybar-none": 3},
    "coupling-rows": {"ybar-all": 2, "ybar-subset": 2, "ybar-none": 2, "noybar-all": 3, "noybar-subset": 3, "noybar-none": 3},
    "coupling-lists": {"ybar-all": 2, "ybar-subset": 2, "ybar-none": 2, "noybar-all": 3, "noybar-subset": 3, "noybar-none": 3},
    "batchnorm": {"ybar-all": 2, "ybar-subset": 2, "ybar-none": 2, "noybar-all": 3, "noybar-subset": 3, "noybar-none": 3},
    "elementwise": {"ybar-all": 2, "ybar-subset": 2, "ybar-none": 1, "noybar-all": 2, "noybar-subset": 2, "noybar-none": 1},
    "tril": {"ybar-all": 3, "ybar-subset": 3, "ybar-none": 1, "noybar-all": 3, "noybar-subset": 3, "noybar-none": 1},
    "spline-coupling": {"ybar-all": 2, "ybar-subset": 2, "ybar-none": 2, "noybar-all": 2, "noybar-subset": 2, "noybar-none": 2},
    "scale": {"ybar-all": 6, "ybar-subset": 6, "ybar-none": 1, "noybar-all": 5, "noybar-subset": 5, "noybar-none": 1},
    "mlp-coupling-rows": {"ybar-all": 2, "ybar-subset": 2, "ybar-none": 1, "noybar-all": 2, "noybar-subset": 2, "noybar-none": 1},
    "mlp-coupling-lists": {"ybar-all": 2, "ybar-subset": 2, "ybar-none": 1, "noybar-all": 2, "noybar-subset": 2, "noybar-none": 1},
    "mixed": {"ybar-all": 40, "ybar-subset": 35, "ybar-none": 25, "noybar-all": 40, "noybar-subset": 35, "noybar-none": 25},
}


@pytest.fixture(scope="module")
def results():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return measure_all(B)


CASES = ("planar", "planar-embedded", "planar-misaligned", "radial", "rqs", "coupling-rows", "coupling-lists", "batchnorm",
         "elementwise", "tril", "spline-coupling", "scale", "mlp-coupling-rows", "mlp-coupling-lists", "mixed")


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_launches_and_routing(results, name):
    import torch

    res = results[name]
    for given in (True, False):
        st, n, xb_all, all_bars = res[(given, "all")]
        for req in REQUESTS:
            st_r, n_r, xb_r, bars_r = res[(given, req)]
            assert st_r == 0, (name, given, req, st_r)
            assert n_r == LAUNCHES[name][f"{'ybar' if given else 'noybar'}-{req}"], (name, given, req, n_r)
            assert torch.equal(xb_r, xb_all), (name, given, req)
            assert not torch.isnan(xb_r).any(), (name, given, req)
            for key, v in bars_r.items():
                assert torch.equal(v, all_bars[key]), (name, given, req, key)
                assert not torch.isnan(v).any(), (name, given, req, key)


if __name__ == "__main__":
    import json

    import bijectors_jl_b200 as B

    got = measure_all(B)
    table = {name: {f"{'ybar' if g else 'noybar'}-{r}": v[(g, r)][1] for g in (True, False) for r in REQUESTS}
             for name, v in got.items()}
    status = {name: sorted({v[k][0] for k in v}) for name, v in got.items()}
    print(json.dumps(table, indent=1))
    print(json.dumps(status))
