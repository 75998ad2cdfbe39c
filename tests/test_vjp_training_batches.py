"""Reverse mode at training batch sizes (N = 2²² + 13 columns) against float64, one chain per segment class of
b2b_chain_vjp_f32 (planar run at D = 128 and through the padded embedding at D = 36, radial run, RQS, affine coupling,
eval BatchNorm, elementwise run with the diagonal MvNormal, TRIL terminal, spline coupling, dense Scale, MLP coupling),
one Float64 chain through b2b_chain_vjp_f64, and autograd.Flow on a mixed chain.

At small N every CTA of a VJP kernel sees one or two column tiles; at these sizes each CTA walks hundreds of tiles
round-robin, wraps its staging ring many times, and accumulates its parameter partials over thousands of columns.

Periodic batches.  x, ȳ and l̄ repeat M = 4099 columns (prime, no divisor of any tile width): column n is column n mod M.
The VJP is linear in (ȳ, l̄) and the parameter cotangents are column sums, so with N = qM + r the exact parameter
cotangent is q·P(M columns) + P(first r columns), and x̄ₙ = x̄_ref[n mod M]: two float64 oracle calls on at most M columns.

Probes.  ȳ and l̄ are zero except on probe columns placed from each kernel's launch geometry (GEOMETRY), x dense and
periodic.  The parameter sums then have a few dozen nonzero terms, so the device's fp32 accumulation is essentially exact:
a dropped probe is an O(1) error and a duplicated one doubles its term.

Inputs are built and columns compared on the device; only the M reference columns and the probe columns reach the host."""
import os
import re

import numpy as np
import pytest

import chain_vjp_oracle as V
import test_mixed_chains as MC

f32, f64 = np.float32, np.float64
M = 4099
N_BIG = (1 << 22) + 13
N_MLP = (1 << 21) + 13  # the MLP coupling's workspace holds per-CTA slices of H x N activations: half the batch
U32 = 2.0 ** -24

# x̄, per column:  ‖x̄ₙ − refₙ‖ ≤ max(XRTOL·‖refₙ‖, 4·‖ref32ₘ − refₘ‖) + max(XFLOOR·rms‖ref‖, 4·rms‖ref32 − ref‖).
# XRTOL is the norm-wise gate of the small-batch tests applied to one column; 4·‖ref32ₘ − refₘ‖ admits a column whose
# float32 evaluation is itself ill-conditioned (the device evaluates the same formulas in float32).  The floor admits the
# period's typical float32 error in any column: the device and the float32 reference round in different orders, so in a
# column where the reference happens to round well (a spline coupling's knots come from n₂-term dot products) the device
# can be a few times further off; XFLOOR·rms‖ref‖, a few float32 ulps of a typical column, covers x̄ near zero.  A stale or
# misplaced column is off by O(‖refₙ‖), and the bit-for-bit copy check catches it whatever its size.
XRTOL, XFLOOR = 1e-5, 1e-6
# parameter cotangents, norm-wise:  rel ≤ max(PRTOL, 2·rel(ref32, ref64) on the M columns), the gate of the small-batch
# tests (tests/test_mixed_chains.py), with the reference's own float32 error measured on one period.
PRTOL = 1e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bijectors.jl_b200", "csrc")


# ---- launch geometry ----------------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


def _outer_chunks(N):
    """(P, clen) of b2b_mvnormal_tril.cu chunk_len: P = min(⌈N / kChunk⌉, kMaxChunks) chunks of ⌈N / P⌉ columns rounded
    up to kBK."""
    P = max(1, min(_cdiv(N, 4096), 64))
    return P, _cdiv(_cdiv(N, P), 16) * 16


# kernel: (chains of CHAINS that run it, layouts(sms, N) -> [(G, T, S)], [(file, constant, value)], [(file, source line)]).
# Every layout is a round-robin walk: CTA b handles tiles b, b + G, b + 2G, ... of T columns and a ring of depth S reuses
# stage k mod S.  A kernel that gives each CTA one contiguous range of ⌈N / G⌉ columns is the layout (G, ⌈N / G⌉, 1).
# Where the grid depends on how many CTAs the shared memory lets an SM hold, every possible count is a layout of its
# own.  test_geometry_matches_source reads every constant and line back from the source, so a change to one fails there
# instead of silently moving the probes.
GEOMETRY = {
    # VJP_PG_GRID = 592 CTAs, PGB_CH = 16 columns per chunk, PGB_STAGES = 4 mbarrier stages
    "planar_pgrad_bulk_kernel": (("planar128", "planar36-inverse"), lambda sms, N: [(592, 16, 4)],
                                 [("b2b_planar_vjp.cu", "VJP_PG_GRID", 592), ("b2b_planar_vjp.cu", "PGB_CH", 16),
                                  ("b2b_planar_vjp.cu", "PGB_STAGES", 4)],
                                 [("b2b_planar_vjp.cu", "kernel<<<VJP_PG_GRID, PG_THREADS, smem, stream>>>")]),
    # VJP_SS_GRID = 296 CTAs of SS_THREADS = 128 threads, one column per thread
    "planar_sstat_kernel": (("planar128", "planar36-inverse"), lambda sms, N: [(296, 128, 1)],
                            [("b2b_planar_vjp.cu", "VJP_SS_GRID", 296), ("b2b_planar_vjp.cu", "SS_THREADS", 128)],
                            [("b2b_planar_vjp.cu", "planar_sstat_kernel<8><<<VJP_SS_GRID, SS_THREADS, 0, stream>>>")]),
    # grid = min(4·SMs, RV_GRID_MAX = 592); RV_THREADS / tpc column groups per CTA, tpc = 8 threads per column at D = 48
    "radial_vjp_kernel": (("radial",), lambda sms, N: [(min(4 * sms, 592), 256 // 8, 1)],
                          [("b2b_radial_vjp.cu", "RV_GRID_MAX", 592), ("b2b_radial_vjp.cu", "RV_THREADS", 256)],
                          [("b2b_radial_vjp.cu", "int grid = sms * 4;"),
                           ("b2b_radial_vjp.cu", "if (grid > RV_GRID_MAX) grid = RV_GRID_MAX;"),
                           ("b2b_radial_vjp.cu", "const int tpc = D <= 32 ? 4 : D <= 64 ? 8 : 16;")]),
    # grid = SMs, CV_TC = 32 columns per tile
    "coupling_vjp_kernel": (("coupling", "coupling-inverse"), lambda sms, N: [(sms, 32, 1)],
                            [("b2b_coupling_vjp.cu", "CV_TC", 32)],
                            [("b2b_coupling_vjp.cu", "long long grid = b2b_sm_count();"),
                             ("b2b_coupling_vjp.cu", "for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {")]),
    # crv_grid: SMs × (1 … 8 CTAs per SM, from the shared memory), CRV_TN = 64 columns per tile
    "coupling_rqs_vjp_kernel": (("spline-coupling", "spline-coupling-inverse"),
                                lambda sms, N: [(sms * k, 64, 1) for k in range(1, 9)],
                                [("b2b_coupling_rqs_vjp.cu", "CRV_TN", 64)],
                                [("b2b_coupling_rqs_vjp.cu", "per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);"),
                                 ("b2b_coupling_rqs_vjp.cu", "long long g = (long long)sms * per_sm;"),
                                 ("b2b_coupling_rqs_vjp.cu", "for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {")]),
    # cmv_grid: SMs; groups of 32·nsub columns, nsub ∈ {4, 2, 1} from the shared memory
    "coupling_mlp_vjp_kernel": (("mlp-coupling", "mlp-coupling-inverse"), lambda sms, N: [(sms, 32 * s, 1) for s in (1, 2, 4)],
                                [],
                                [("b2b_coupling_mlp_vjp.cu", "long long g = sms;"),
                                 ("b2b_coupling_mlp_vjp.cu", "for (int s = 4; s > 1; s >>= 1)"),
                                 ("b2b_coupling_mlp_vjp.cu", "TG = 32 * P.nsub"),
                                 ("b2b_coupling_mlp_vjp.cu", "for (long long g = blockIdx.x; g < groups; g += gridDim.x) {")]),
    # rqv_shape: SMs × (1 … 3 CTAs per SM); one contiguous range of ⌈N / grid⌉ columns per CTA
    "rqs_vjp_kernel": (("rqs", "rqs-inverse"), lambda sms, N: [(sms * k, _cdiv(N, sms * k), 1) for k in (1, 2, 3)],
                       [],
                       [("b2b_rqs_vjp.cu", "if (per_sm > 3) per_sm = 3;"), ("b2b_rqs_vjp.cu", "s.grid_max = sms * per_sm;"),
                        ("b2b_rqs_vjp.cu", "const long long per = (P.N + gridDim.x - 1) / gridDim.x;")]),
    # ev_grid_max = 8·SMs; one contiguous range of ⌈N / grid⌉ columns per CTA
    "ew_vjp_kernel": (("elementwise-diag", "tril"), lambda sms, N: [(8 * sms, _cdiv(N, 8 * sms), 1)],
                      [],
                      [("b2b_ew_vjp.cu", "static int ev_grid_max() { return b2b_sm_count() * 8; }"),
                       ("b2b_ew_vjp.cu", "const long long per = (P.N + gridDim.x - 1) / gridDim.x;")]),
    # outer_kernel (L̄ and μ̄ of the TRIL terminal, Ā of dense Scale): P fixed column chunks (_outer_chunks)
    "outer_kernel": (("tril", "scale", "scale-inverse"), lambda sms, N: [_outer_chunks(N) + (1,)],
                     [("b2b_mvnormal_tril.cu", "kChunk", 4096), ("b2b_mvnormal_tril.cu", "kMaxChunks", 64),
                      ("b2b_mvnormal_tril.cu", "kBK", 16)],
                     [("b2b_mvnormal_tril.cu", "long long P = (N + kChunk - 1) / kChunk;"),
                      ("b2b_mvnormal_tril.cu", "return (c + kBK - 1) / kBK * kBK;"),
                      ("b2b_scale_matrix.cu", "b2b_launch_outer_chunks(ybar, ldyb, x, ldx, part, nullptr, D, N, false, stream)")]),
}


def _source_constant(fname, name):
    src = open(os.path.join(CSRC, fname)).read()
    m = re.search(r"constexpr\s+int\s+(?:[A-Za-z_0-9]+\s*=\s*\d+\s*,\s*)*" + name + r"\s*=\s*(\d+)\s*[;,]", src)
    assert m, (fname, name)
    return int(m.group(1))


def test_geometry_matches_source():
    for kernel, (_, _, consts, lines) in GEOMETRY.items():
        for fname, name, value in consts:
            assert _source_constant(fname, name) == value, (kernel, fname, name, value)
        for fname, line in lines:
            assert line in open(os.path.join(CSRC, fname)).read(), (kernel, fname, line)


def probe_columns(G, T, S, N, tail):
    """Columns at the schedule's edges: for CTAs 0, 1 and G − 1 the first and last column of the tile in round-robin
    slots 0, S − 1, S, 2S − 1 and 2S and of the CTA's last tile; N − 1, N − 2 and the first column of the ragged tail.
    For a contiguous-range layout (one tile per CTA) these are the boundaries of ranges 0, 1 and G − 1."""
    tiles = _cdiv(N, T)
    cols = {N - 1, N - 2, tail}
    for c in (0, 1, G - 1):
        mine = (tiles - c + G - 1) // G
        for k in sorted({0, S - 1, S, 2 * S - 1, 2 * S, mine - 1}):
            t = c + k * G
            if 0 <= k < mine:
                cols.update((t * T, min(t * T + T - 1, N - 1)))
    return sorted(cols)


def test_probe_columns_cover_the_walk():
    """The probe placement itself, at 132 SMs: every round-robin CTA of the table walks more than 2S tiles, so slot 2S
    (the second wrap of a ring of depth S) exists for CTAs 0, 1 and G − 1 and gets both its columns; every contiguous
    range layout puts both ends of ranges 0, 1 and G − 1 among the probes."""
    for kernel, (chains, layouts, _, _) in GEOMETRY.items():
        for name in chains:
            N = CHAINS[name][1]
            for G, T, S in layouts(132, N):
                cols = set(probe_columns(G, T, S, N, M * (N // M)))
                assert {0, N - 1, N - 2} <= cols, kernel
                if T * G >= N:  # one contiguous range per CTA
                    for c in (0, 1, G - 1):
                        assert {c * T, min(c * T + T - 1, N - 1)} <= cols, (kernel, c)
                    continue
                assert _cdiv(N, T) // G > 2 * S, kernel
                for c in (0, 1, G - 1):
                    t = c + 2 * S * G
                    assert {t * T, t * T + T - 1} <= cols, (kernel, c)


# ---- the chains ---------------------------------------------------------------------------------------------------------------
# name: (D, N, [(kind, inverse, options)], base or None).  A chain with a base runs logpdf_vjp, the others chain_vjp with ȳ.
CHAINS = {
    "planar128": (128, N_BIG, [("planar", 0, {})] * 4, None),
    "planar36-inverse": (36, N_BIG, [("planar", 1, {})] * 2, None),
    "radial": (48, N_BIG, [("radial", 0, {}), ("radial", 1, {}), ("radial", 0, {})], None),
    "rqs": (32, N_BIG, [("rqs", 0, {})], None),
    "rqs-inverse": (32, N_BIG, [("rqs", 1, {})], None),
    "coupling": (64, N_BIG, [("cpl", 0, dict(n1=24, n2=40))], None),
    "coupling-inverse": (64, N_BIG, [("cpl", 1, dict(n1=20, n2=44, lists=True))], None),
    "batchnorm": (96, N_BIG, [("bn", 0, {})], None),
    "batchnorm-inverse": (96, N_BIG, [("bn", 1, {})], None),
    "elementwise-diag": (40, N_BIG, [("stacked", 0, {}), ("perm", 0, {})], "diag"),
    "tril": (48, N_BIG, [("perm", 0, {})], "tril"),
    "spline-coupling": (64, N_BIG, [("spl", 0, dict(n1=16, n2=48))], None),
    "spline-coupling-inverse": (64, N_BIG, [("spl", 1, dict(n1=24, n2=40, K=4))], None),
    "scale": (48, N_BIG, [("scale", 0, {})], None),
    "scale-inverse": (48, N_BIG, [("scale", 1, {})], None),
    "mlp-coupling": (64, N_MLP, [("mlp", 0, dict(n1=32, n2=32, H=64, lists=False))], None),
    "mlp-coupling-inverse": (64, N_MLP, [("mlp", 1, dict(n1=24, n2=40, H=32))], None),
}


@pytest.fixture(scope="module")
def B():
    import torch

    assert torch.cuda.is_available()
    import bijectors_jl_b200 as B

    return B


def _build(B, name):
    D, N, spec, base = CHAINS[name]
    rng = np.random.default_rng(len(name) * 7919 + D)
    dev, ora, flags = [], [], []
    for kind, inv, o in spec:
        d, r = MC._layer(B, rng, D, kind, o)
        dev.append(B.inverse(d) if inv else d)
        ora.append(r)
        flags.append(bool(inv))
    bd, kw = MC.base_of(B, rng, D, base) if base else (None, {})
    return D, N, dev, ora, flags, bd, kw


def _need_memory(nbytes):
    import torch

    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + (1 << 30):
        pytest.skip(f"needs {nbytes / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free (shared device)")


def _periodic(a, N, dtype):
    """Device Julia-layout (D, N) batch (or length-N vector) whose column n is column n mod M of the host array `a`."""
    import torch

    t = torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype).T)).cuda()
    reps = -(-N // a.shape[-1])
    if t.dim() == 1:
        return t.repeat(reps)[:N]
    return t.repeat(reps, 1)[:N].t()


def _run(B, dev, bd, x, ybar, lb):
    """(x̄, [grads per layer in application order], base grads) of the device chain (logpdf_vjp when there is a base)."""
    if bd is not None:
        xbar, flow_g, base_g = B.logpdf_vjp(B.transformed(bd, B.inverse(B.Composed(*dev))), x, lb)
        return xbar, flow_g[::-1], base_g
    xbar, grads = B.chain_vjp(B.Composed(*dev), x, ybar, lb)
    return xbar, grads, {}


def rel(a, b):
    a, b = np.asarray(a, f64), np.asarray(b, f64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(a), np.linalg.norm(b), 1e-300))


def _items(res):
    """{name: array} of every parameter and base cotangent of an oracle result or a device result."""
    _, grads, base = res
    out = {(l, k): v for l, g in enumerate(grads) for k, v in g.items()}
    out.update({("base", k): v for k, v in base.items()})
    return out


def check_columns(xbar, ref64, ref32, rtol=XRTOL, floor=XFLOOR, what=""):
    """Every column of the device x̄ against the tiled float64 reference (gate in the module notes), and every copy of a
    reference column bit for bit equal to the first period's: columns with the same n mod M have the same inputs, and no
    kernel's per-column arithmetic depends on the column's position, so a stale-stage or wrong-offset read shows up as a
    changed bit.  ref32 None: no float32 term (the Float64 path)."""
    import torch

    D, Mc = ref64.shape
    N = xbar.shape[1]
    q, r = divmod(N, Mc)
    xt = xbar.t()
    assert xt.is_contiguous()
    ref = torch.from_numpy(np.ascontiguousarray(ref64.T)).cuda()
    rn = ref.norm(dim=1)
    fl = floor * float(rn.square().mean().sqrt())
    tol = rtol * rn
    if ref32 is not None:
        e32 = np.linalg.norm(np.asarray(ref32, f64) - ref64, axis=0)
        tol = torch.maximum(tol, 4 * torch.from_numpy(e32).cuda())
        fl = max(fl, 4 * float(np.sqrt(np.mean(e32 ** 2))))
    tol = tol + fl
    bits = torch.int32 if xt.dtype == torch.float32 else torch.int64
    first = xt[:Mc].view(bits)
    worst, at, copies_bad = 0.0, -1, []
    chunk = max(1, (1 << 27) // (Mc * D))
    for p0 in range(0, q, chunk):
        p1 = min(q, p0 + chunk)
        blk = xt[p0 * Mc:p1 * Mc].view(p1 - p0, Mc, D)
        ratio = ((blk.double() - ref).norm(dim=2) / tol).view(-1)
        v, i = ratio.max(0)
        if float(v) > worst or not np.isfinite(float(v)):
            worst, at = float(v), p0 * Mc + int(i)
        same = (blk.view(bits) == first).all(dim=2).view(-1)
        if not bool(same.all()):
            copies_bad.append(p0 * Mc + int((~same).nonzero()[0]))
    if r:
        tail = xt[q * Mc:]
        ratio = (tail.double() - ref[:r]).norm(dim=1) / tol[:r]
        v, i = ratio.max(0)
        if float(v) > worst or not np.isfinite(float(v)):
            worst, at = float(v), q * Mc + int(i)
        same = (tail.view(bits) == first[:r]).all(dim=1)
        if not bool(same.all()):
            copies_bad.append(q * Mc + int((~same).nonzero()[0]))
    assert worst <= 1.0, (what, "worst x̄ column", at, "error / gate", worst)
    assert not copies_bad, (what, "x̄ column differs in its bits from the same column of the first period", copies_bad)


def planar_b_sums(ora, flags, X, Y, Lb, kw):
    """{(l, "b"): (Σₙ |gₙ|, Σₙ |g32ₙ − g64ₙ|)} over the columns of X for every planar layer l, from the float64 and
    float32 oracles' column terms of b̄."""
    t64, t32 = {}, {}
    V.chain_vjp(ora, flags, X.astype(f64), Y, Lb, b_terms=t64, **kw)
    V.chain_vjp(ora, flags, X, Y, Lb, dtype=f32, b_terms=t32, **kw)
    return {(l, "b"): (float(np.abs(t64[l]).sum()), float(np.abs(np.asarray(t32[l], f64) - t64[l]).sum())) for l in t64}


def sstat_chain_length(N):
    """Longest chain of float32 additions behind a planar b̄ (b2b_planar_vjp.cu): planar_sstat_kernel's thread adds
    ⌈N / (296·128)⌉ columns in sequence, a 5-level shuffle tree and 4 warp sums follow, then planar_psum_kernel's lane
    adds ⌈296 / 32⌉ CTA partials and a 5-level shuffle tree."""
    return -(-N // (296 * 128)) + 5 + 4 + -(-296 // 32) + 5


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CHAINS))
def test_periodic_batch(B, name):
    """Every column of x̄, every copy bit for bit, and every parameter and base cotangent over N = qM + r periodic columns
    against q·P(M) + P(r) in float64.

    Gates: x̄ per column as in the notes above XRTOL.  Parameters norm-wise: max(1e-5, 2 × the float32 reference's relative
    error on the M columns).  Planar b̄ is one sum of N scalars gₙ that may cancel, so its relative error is not bounded by
    the above; the float32 error model gives
        |b̄ − b̄₆₄| ≤ 2·Σₙ |g32ₙ − g64ₙ| + h·u·Σₙ |gₙ|,
    the first term the per-column error of forming gₙ in float32 (twice the float32 reference's, column by column), the
    second the first-order bound of float32 summation with longest addition chain h (sstat_chain_length) and u = 2⁻²⁴.
    Both sums are q·(sum over the M columns) + (sum over the first r), from the oracles' column terms of b̄."""
    import torch

    D, N, dev, ora, flags, bd, kw = _build(B, name)
    _need_memory(3 * D * N * 4 + N * 4 * 16)
    rng = np.random.default_rng(N % 1009 + D)
    q, r = divmod(N, M)
    X = MC.inputs(rng, D, M)
    Y = None if bd is not None else rng.standard_normal((D, M)).astype(f32)
    Lb = rng.standard_normal(M).astype(f32)
    x = _periodic(X, N, f32)
    yb = None if Y is None else _periodic(Y, N, f32)
    lb = _periodic(Lb, N, f32)
    got = _run(B, dev, bd, x, yb, lb)
    torch.cuda.synchronize()
    del x, yb

    o64 = V.chain_vjp(ora, flags, X.astype(f64), Y, Lb, **kw)
    o32 = V.chain_vjp(ora, flags, X, Y, Lb, dtype=f32, **kw)
    o64r = V.chain_vjp(ora, flags, X[:, :r].astype(f64), None if Y is None else Y[:, :r], Lb[:r], **kw)
    check_columns(got[0], np.asarray(o64[0]), np.asarray(o32[0]), what=name)

    dv, p64, p32, p64r = _items(got), _items(o64), _items(o32), _items(o64r)
    assert set(dv) == set(p64), (name, set(dv) ^ set(p64))
    sums, sums_r = {}, {}
    if any(lay.kind == "planar" for lay in ora):
        sums = planar_b_sums(ora, flags, X, Y, Lb, kw)
        sums_r = planar_b_sums(ora, flags, X[:, :r], None if Y is None else Y[:, :r], Lb[:r], kw)
    h = sstat_chain_length(N)
    for k in sorted(dv, key=str):
        d = np.asarray(B.to_numpy(dv[k]), f64).ravel()
        ref = (q * np.asarray(p64[k], f64) + np.asarray(p64r[k], f64)).ravel()
        tol = max(PRTOL, 2 * rel(p32[k], p64[k]))
        if k in sums:
            bound = 2 * (q * sums[k][1] + sums_r[k][1]) + h * U32 * (q * sums[k][0] + sums_r[k][0])
            assert abs(d[0] - ref[0]) <= max(tol * abs(ref[0]), bound), (name, k, d[0], ref[0], bound)
            continue
        assert rel(d, ref) <= tol, (name, k, rel(d, ref), tol)


# ---- probes -------------------------------------------------------------------------------------------------------------------
PROBE_CHAINS = sorted({c for g in GEOMETRY.values() for c in g[0]} | {"batchnorm"})


@pytest.mark.gpu
@pytest.mark.parametrize("name", PROBE_CHAINS)
def test_probe_columns(B, name):
    """ȳ and l̄ zero except on the probe columns of every GEOMETRY kernel the chain runs (plus N − 1, N − 2 and the first
    column of the ragged tail), x dense and periodic.  Every parameter and base cotangent element i must satisfy
        |dev_i − Σₚ pₚ,ᵢ| ≤ 1e-5 · Σₚ |pₚ,ᵢ| + 4 · Σₚ |p32ₚ,ᵢ − pₚ,ᵢ| + 1e-30
    against the float64 terms pₚ of the probes (one oracle call per probe): a few dozen float32 terms sum essentially
    exactly, 1e-5 (~170 float32 ulps) covers forming each term in float32, and the second term covers a probe whose
    float32 evaluation is ill-conditioned (four times the float32 reference's own error on that term), while a dropped or
    duplicated probe is off by its whole term.  x̄ at each probe column is gated as in check_columns (ȳ elsewhere is zero, so it depends on the
    probe's own cotangents only), and every other column of x̄ must be exactly zero."""
    import torch

    D, N, dev, ora, flags, bd, kw = _build(B, name)
    _need_memory(3 * D * N * 4 + N * 4 * 16)
    rng = np.random.default_rng(D + 31)
    q = N // M
    X = MC.inputs(rng, D, M)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cols = {N - 1, N - 2, q * M}
    for kernel, (chains, layouts, _, _) in GEOMETRY.items():
        if name in chains:
            for G, T, S in layouts(sms, N):
                cols.update(probe_columns(G, T, S, N, q * M))
    cols = np.array(sorted(cols), dtype=np.int64)
    P = len(cols)
    Yp = None if bd is not None else rng.standard_normal((D, P)).astype(f32)
    Lp = rng.standard_normal(P).astype(f32)
    x = _periodic(X, N, f32)
    ci = torch.from_numpy(cols).cuda()
    yb = None
    if Yp is not None:
        yb = torch.zeros((N, D), device="cuda")
        yb[ci] = torch.from_numpy(np.ascontiguousarray(Yp.T)).cuda()
        yb = yb.t()
    lb = torch.zeros(N, device="cuda")
    lb[ci] = torch.from_numpy(Lp).cuda()
    got = _run(B, dev, bd, x, yb, lb)
    torch.cuda.synchronize()
    del x, yb

    Xp = X[:, cols % M]
    o64 = V.chain_vjp(ora, flags, Xp.astype(f64), Yp, Lp, **kw)
    o32 = V.chain_vjp(ora, flags, Xp, Yp, Lp, dtype=f32, **kw)
    xt = got[0].t()
    xp = xt[ci].double().cpu().numpy().T
    rn = np.linalg.norm(o64[0], axis=0)
    e32 = np.linalg.norm(np.asarray(o32[0], f64) - o64[0], axis=0)
    fl = max(XFLOOR * np.sqrt(np.mean(rn ** 2)), 4 * np.sqrt(np.mean(e32 ** 2)))
    tol = np.maximum(XRTOL * rn, 4 * e32) + fl
    err = np.linalg.norm(xp - o64[0], axis=0)
    assert (err <= tol).all(), (name, "probe x̄", cols[np.argmax(err / tol)], float(np.max(err / tol)))
    nz = (xt != 0).any(dim=1)
    nz[ci] = False
    assert not bool(nz.any()), (name, "x̄ nonzero off the probes at column", int(nz.nonzero()[0]))

    dv = _items(got)
    absum, err32, ref = {}, {}, _items(o64)
    for p in range(P):
        yp = None if Yp is None else Yp[:, p:p + 1]
        it = _items(V.chain_vjp(ora, flags, Xp[:, p:p + 1].astype(f64), yp, Lp[p:p + 1], **kw))
        it32 = _items(V.chain_vjp(ora, flags, Xp[:, p:p + 1], yp, Lp[p:p + 1], dtype=f32, **kw))
        for k in dv:
            absum[k] = absum.get(k, 0.0) + np.abs(np.asarray(it[k], f64))
            err32[k] = err32.get(k, 0.0) + np.abs(np.asarray(it32[k], f64) - it[k])
    assert set(dv) == set(ref)
    for k in sorted(dv, key=str):
        d = np.asarray(B.to_numpy(dv[k]), f64).reshape(np.shape(ref[k]))
        bad = np.abs(d - ref[k]) > 1e-5 * absum[k] + 4 * err32[k] + 1e-30
        assert not bad.any(), (name, k, "element", np.argwhere(bad)[0].tolist(), float(np.ravel(d[bad])[0]),
                               float(np.ravel(np.asarray(ref[k])[bad])[0]))


# ---- Float64 and the training module ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_periodic_batch_f64(B):
    """Planar, planar and radial at D = 32 through b2b_chain_vjp_f64 at N = 2²² + 13: every x̄ column within 1e-10 of the
    tiled reference (plus 1e-12 · rms‖ref‖), every copy bit for bit, every parameter cotangent within 1e-10 norm-wise of
    q·P(M) + P(r): float64 evaluation and summation of ~4·10⁶ terms stay far inside 1e-10."""
    import torch

    D, N = 32, N_BIG
    _need_memory(3 * D * N * 8)
    rng = np.random.default_rng(64)
    t64 = torch.float64
    dev, ora = [], []
    for kind in ("planar", "planar", "radial"):
        _, r = MC._layer(B, rng, D, kind, {})
        p = r.params
        dev.append(B.PlanarLayer(p["w"], p["u"], p["b"], dtype=t64) if kind == "planar"
                   else B.RadialLayer(p["alpha_raw"], p["beta"], p["z0"], dtype=t64))
        ora.append(r)
    flags = [False, True, False]
    dev[1] = B.inverse(dev[1])
    q, r = divmod(N, M)
    X = MC.inputs(rng, D, M).astype(f64)
    Y, Lb = rng.standard_normal((D, M)), rng.standard_normal(M)
    xbar, grads = B.chain_vjp(B.Composed(*dev), _periodic(X, N, f64), _periodic(Y, N, f64), _periodic(Lb, N, f64))
    torch.cuda.synchronize()
    o64 = V.chain_vjp(ora, flags, X, Y, Lb)
    o64r = V.chain_vjp(ora, flags, X[:, :r], Y[:, :r], Lb[:r])
    check_columns(xbar, np.asarray(o64[0]), None, rtol=1e-10, floor=1e-12, what="f64")
    dv, p64, p64r = _items((xbar, grads, {})), _items(o64), _items(o64r)
    assert set(dv) == set(p64)
    for k in dv:
        ref = q * np.asarray(p64[k], f64) + np.asarray(p64r[k], f64)
        d = B.to_numpy(dv[k])
        assert str(dv[k].dtype) == "torch.float64"
        assert rel(np.ravel(d), np.ravel(ref)) <= 1e-10, (k, rel(np.ravel(d), np.ravel(ref)))


@pytest.mark.gpu
def test_flow_training_gradients(B):
    """autograd.Flow over BatchNorm, affine coupling, radial, RQS, spline coupling, dense Scale and MLP coupling at D = 64
    with a full-covariance base, N = 2²² + 13 periodic columns: every .grad of -Σ logpdf against q·P(M) + P(r) in float64,
    gated norm-wise as in test_periodic_batch (max(1e-5, 2 × the float32 reference's error on the M columns))."""
    import torch

    D, N = 64, N_BIG
    _need_memory(6 * D * N * 4)
    spec = [("bn", 0, {}), ("cpl", 0, dict(n1=32, n2=32)), ("radial", 0, {}), ("rqs", 0, {}),
            ("spl", 0, dict(n1=16, n2=24)), ("scale", 0, {}), ("mlp", 0, dict(n1=20, n2=24, H=32))]
    rng = np.random.default_rng(4242)
    pairs = [MC._layer(B, rng, D, k, o) for k, _, o in spec]
    dev, ora = [p for p, _ in pairs], [o for _, o in pairs]
    flags = [False] * len(ora)
    bd, kw = MC.base_of(B, rng, D, "tril")
    q, r = divmod(N, M)
    X = MC.inputs(rng, D, M)
    F = B.autograd.Flow(B.inverse(B.Composed(*dev)), base=bd)
    F.nll(_periodic(X, N, f32)).backward()
    torch.cuda.synchronize()
    lb = -np.ones(M)  # the cotangent of -Σ logpdf
    o64 = V.chain_vjp(ora, flags, X.astype(f64), None, lb, **kw)
    o32 = V.chain_vjp(ora, flags, X, None, lb.astype(f32), dtype=f32, **kw)
    o64r = V.chain_vjp(ora, flags, X[:, :r].astype(f64), None, lb[:r], **kw)
    got = {p.data_ptr(): p.grad for p in F.params}
    assert all(g is not None for g in got.values())

    def chk(g, k64, k32, k64r, what):
        ref = q * np.asarray(k64, f64) + np.asarray(k64r, f64)
        tol = max(PRTOL, 2 * rel(k32, k64))
        assert rel(np.ravel(g), np.ravel(ref)) <= tol, (what, rel(np.ravel(g), np.ravel(ref)), tol)

    chk(got[bd.mu.data_ptr()].cpu().numpy(), o64[2]["μ"], o32[2]["μ"], o64r[2]["μ"], "μ")
    chk(got[bd._tril.data_ptr()].t().cpu().numpy(), o64[2]["L"], o32[2]["L"], o64r[2]["L"], "L")
    checked = 2
    for l, d in enumerate(dev):
        # the trainable tensors of a leaf come in the order of the reference's cotangent dict; matrices are stored
        # column-major (transposed)
        for key, t in zip(o64[1][l], B.autograd._trainable_tensors(d)):
            g = got[t.data_ptr()]
            g = (g.t() if g.dim() == 2 else g).cpu().numpy()
            chk(g.reshape(np.shape(o64[1][l][key])), o64[1][l][key], o32[1][l][key], o64r[1][l][key], (l, key))
            checked += 1
    assert checked == len(F.params)
