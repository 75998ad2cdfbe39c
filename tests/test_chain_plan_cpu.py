"""Chain planning pinned on the host: workspace sizes, status codes and launch counts of the chain entry points for a sweep
of descriptor chains, against tests/golden/chain_plan.json (and, for the neural spline and deep network couplings, chain_plan_couplings.json).  No GPU needed: the workspace queries are pure host functions,
and so is b2b_chain_vjp_f32 / _f64 at N = 0 without parameter cotangents (it validates, plans and returns before any CUDA
call).  The descriptors carry a fake non-NULL address for every parameter; nothing is ever read through it.

Never pass a cotangent pointer here: at N = 0 an accepted slot is zeroed on the device.

The fixture is recorded by hand from a trusted build:  python tests/test_chain_plan_cpu.py [path/to/libb2b.so]"""
import ctypes
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "chain_plan.json")
GOLDEN_COUPLINGS = os.path.join(ROOT, "tests", "golden", "chain_plan_couplings.json")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bijectors_jl_b200 import _lib  # noqa: E402

P = 0x10000  # a fake device address
NS = (1000, 1 << 20)
DS = (1, 32, 36, 128, 129, 256, 257, 747, 748, 1024, 1025, 2048, 2049)
VALID_KINDS = {1, 2, 3, 4, 5, 6, 7, 8, 9, 11, 12, 13, 14, 15}


def planar(inv=0):
    return dict(kind=_lib.PLANAR, inverse=inv, p0=P, p1=P, p2=P)


def radial(inv=0):
    return dict(kind=_lib.RADIAL, inverse=inv, p0=P, p1=P, p2=P)


def rqs(inv=0, K1=9):
    return dict(kind=_lib.RQS, inverse=inv, p0=P, p1=P, p2=P, n0=K1)


def cpl(n1, n2, inv=0, lists=False, c=True):
    d = dict(kind=_lib.COUPLING_AFFINE, inverse=inv, p0=P, n0=n1, n1=n2)
    if c:
        d["p1"] = P
    if lists:
        d.update(i0=P, i1=P, n2=-1, n3=-1)
    else:
        d.update(n2=0, n3=n1)
    return d


def bn(inv=0):
    return dict(kind=_lib.BATCHNORM, inverse=inv, p0=P, p1=P, p2=P, p3=P, f0=1e-5)


def perm(inv=0):
    return dict(kind=_lib.PERMUTE, inverse=inv, i0=P)


def ew(inv=0):
    return dict(kind=_lib.STACKED_EW, inverse=inv, i0=P, p0=P, p1=P)


def diag(inv=0, mu=True, sigma=True):
    d = dict(kind=_lib.MVNORMAL_DIAG, inverse=inv)
    if mu:
        d["p0"] = P
    if sigma:
        d["p1"] = P
    return d


def tril(inv=0):
    return dict(kind=_lib.MVNORMAL_TRIL, inverse=inv, p0=P, p1=P)


def srqs(n1, n2, K=8, inv=0):
    return dict(kind=_lib.COUPLING_RQS, inverse=inv, p0=P, p1=P, i0=P, i1=P, n0=n1, n1=n2, n2=K, f0=3.0)


def scale(inv=0):
    return dict(kind=_lib.SCALE_MATRIX, inverse=inv, p0=P)


def mlp(n1, n2, H, inv=0, act=None):
    act = _lib.ACT_TANH if act is None else act
    return dict(kind=_lib.COUPLING_MLP, inverse=inv, p0=P, p1=P, p2=P, p3=P, i0=P, i1=P, n0=n1, n1=n2, n2=H, n3=act,
                f0=0.01)


def nrqs(n1, n2, H, K=8, inv=0, act=None, B=3.0):
    act = _lib.ACT_TANH if act is None else act
    return dict(kind=_lib.COUPLING_MLP_RQS, inverse=inv, p0=P, p1=P, p2=P, p3=P, i0=P, i1=P, n0=n1, n1=n2, n2=H,
                n3=act | K << 8, f0=0.01, f1=B)


def deep(n1, n2, H, M=2, inv=0, act=None):
    act = _lib.ACT_TANH if act is None else act
    return dict(kind=_lib.COUPLING_DEEP_MLP, inverse=inv, p0=P, p1=P, p2=P, p3=P, i0=P, i1=P, n0=n1, n1=n2, n2=H,
                n3=act | M << 8, f0=0.01)


def cases():
    """(name, chain, D): every chain the sweep queries, each under a unique name."""
    out = []

    def add(name, chain, Ds=DS):
        for D in Ds:
            out.append((f"{name}@{D}", chain, D))

    alone = {"planar": planar, "radial": radial, "rqs": rqs, "bn": bn, "perm": perm, "ew": ew, "scale": scale}
    for name, f in alone.items():
        for inv in (0, 1):
            add(f"{name}{'-inv' if inv else ''}", [f(inv)])
    add("diag", [diag()])
    add("diag-nomu", [diag(mu=False)])
    add("diag-nosigma", [diag(sigma=False)])
    add("diag-inv", [diag(1)])
    add("tril", [tril()])
    add("tril-inv", [tril(1)])
    add("kind10", [dict(kind=10, p0=P, p1=P, p2=P, p3=P, i0=P, i1=P)])
    for K1 in (1, 2, 33, 64, 65):
        add(f"rqs-K{K1}", [rqs(K1=K1)], (32, 128, 256, 257, 1024))
    for n1, n2 in ((1, 1), (32, 32), (64, 64), (128, 64), (128, 128), (129, 64), (64, 129), (300, 300), (383, 383),
                   (384, 384), (1000, 1000)):
        for inv in (0, 1):
            for lists in (False, True):
                add(f"cpl{n1}x{n2}{'-inv' if inv else ''}{'-lists' if lists else ''}", [cpl(n1, n2, inv, lists)],
                    (36, 256, 257, 747, 748, 1024, 1025, 2048, 2049))
    add("cpl-noc", [cpl(32, 32, c=False)], (64, 256))
    for n1, n2, K in ((32, 32, 8), (128, 128, 16), (129, 64, 8), (64, 129, 8), (64, 64, 17), (64, 64, 2), (64, 64, 1),
                      (16, 16, 16)):
        for inv in (0, 1):
            add(f"srqs{n1}x{n2}K{K}{'-inv' if inv else ''}", [srqs(n1, n2, K, inv)], (36, 256, 257, 1024, 1025))
    for n1, n2, H in ((1, 1, 1), (32, 32, 64), (128, 128, 256), (129, 64, 64), (64, 129, 64), (64, 64, 257),
                      (16, 16, 0)):
        for inv in (0, 1):
            add(f"mlp{n1}x{n2}H{H}{'-inv' if inv else ''}", [mlp(n1, n2, H, inv)], (36, 256, 257, 1024, 1025))
    add("mlp-leaky", [mlp(32, 32, 64, act=_lib.ACT_LEAKY_RELU)], (64, 1024))
    add("mlp-act9", [mlp(32, 32, 64, act=9)], (64,))
    # BatchNorm neighbours folded into coupling launches
    add("bn-cpl-bn", [bn(), cpl(32, 32), bn()], (64, 256, 1024))
    add("bn-cpl", [bn(), cpl(32, 32)], (64, 1024))
    add("cpl-bn", [cpl(32, 32, lists=True), bn(1)], (64, 1024))
    add("bn-cpl-cpl-bn", [bn(), cpl(32, 32), cpl(32, 32, 1), bn()], (64, 256))
    add("bn-cpl-bn-cpl-bn", [bn(), cpl(64, 64), bn(), cpl(64, 64), bn()], (128, 256, 1024))
    add("bn-srqs-bn", [bn(), srqs(32, 32), bn()], (64, 256))
    add("realnvp", [bn(), cpl(64, 64), perm(), bn(), cpl(64, 64, 1), perm(1), diag()], (128, 256, 257, 748))
    # mixed chains ending in a terminal
    add("planar4-diag", [planar()] * 4 + [diag()])
    add("planar4-inv-tril", [planar(1)] * 4 + [tril()])
    add("radial-planar-ew-tril", [radial(), planar(), ew(), perm(), tril()])
    add("scale-planar-tril", [scale(), planar(1), tril()])
    add("srqs-scale-diag", [srqs(32, 32), scale(1), ew(), diag()], (64, 256, 257))
    add("mixed-all", [planar(), radial(1), rqs(), bn(), perm(), ew(1), cpl(16, 16), srqs(16, 16), scale(), tril()],
        (32, 64, 128, 256))
    add("planar-bn-mlp-diag", [planar(), bn(), mlp(32, 32, 64), bn(1), diag()], (64, 128, 1024, 1025))
    add("mlp-inv-planar-tril", [mlp(64, 64, 128, 1), planar(1), tril()], (128, 256, 257))
    add("ew9-diag", [ew()] * 9 + [diag()], (32, 1024, 1025))
    # a batch sum without logjac over a DIAG-terminated chain of several launches (N floats of log-Jacobian workspace)
    add("cpl-diag", [cpl(32, 32), diag()], (64, 256, 1024))
    add("mlp-ew-diag", [mlp(32, 32, 64), ew(), diag()], (64, 256, 1024))
    add("bn-cpl-bn-diag", [bn(), cpl(32, 32), bn(), diag()], (64, 256))
    add("srqs-diag", [srqs(32, 32), diag()], (64, 256))
    add("scale-diag", [scale(1), diag()], (64, 256))
    add("planar9-radial9", [planar()] * 9 + [radial()] * 9, (32, 100, 128))
    add("planar-dirs", [planar(), planar(1), planar(), planar()], (32, 100))
    # runs split at the fused kernels' shared-memory budget
    add("bn24", [bn()] * 24, (256, 1024))
    add("bn13-diag", [bn()] * 12 + [diag()], (1024,))
    add("rqs-K64x4", [rqs(K1=64)] * 4, (32, 64, 128))
    add("planar-rqs33x3-bn", [planar(), rqs(K1=33), rqs(K1=33), rqs(K1=33), bn()], (128, 256))
    add("perm-rqs17x3-diag", [perm(), rqs(K1=17), rqs(K1=17), rqs(K1=17), diag()], (256, 512))
    # chain length
    add("planar24", [planar()] * 24, (32, 128))
    add("planar25", [planar()] * 25, (32, 128))
    add("mixed24", ([planar(), bn(), cpl(16, 16)] * 8)[:23] + [diag()], (64, 256))
    add("mixed25", ([planar(), bn(), cpl(16, 16)] * 9)[:24] + [diag()], (64,))
    # terminals that are not last
    add("diag-planar", [diag(), planar()], (32, 300))
    add("tril-planar", [tril(), planar()], (32, 300))
    add("tril-tril", [tril(), tril()], (32, 300))
    add("planar-kind10-diag", [planar(), dict(kind=10), diag()], (32,))
    # each required pointer set to NULL in turn (an optional one too)
    for name, d in (("planar", planar()), ("radial", radial()), ("rqs", rqs()), ("cpl", cpl(16, 16)),
                    ("cpl-lists", cpl(16, 16, lists=True)), ("bn", bn()), ("perm", perm()), ("ew", ew()),
                    ("diag", diag()), ("tril", tril()), ("srqs", srqs(16, 16)), ("scale", scale()),
                    ("mlp", mlp(16, 16, 32))):
        for f in ("p0", "p1", "p2", "p3", "i0", "i1"):
            if f in d:
                e = dict(d)
                del e[f]
                add(f"null-{name}-{f}", [e], (64, 300))
                add(f"planar-then-null-{name}-{f}", [planar(), e], (64,))
        add(f"{name}-then-null-planar", [d, dict(planar(), p1=0)], (64, 300, 2048))
    return out


def coupling_cases():
    """(name, chain, D) for the neural spline (B2B_COUPLING_MLP_RQS) and deep network (B2B_COUPLING_DEEP_MLP) couplings:
    both sides of every limit, the descriptor rules, both directions, and chains mixing them with other kinds."""
    out = []

    def add(name, chain, Ds):
        for D in Ds:
            out.append((f"{name}@{D}", chain, D))

    # n1, n2, H, K or M and D each on both sides of their limits.  K = 1 is a valid descriptor past the envelope
    # (B2B_EUNSUPPORTED), M = 1 and H = 0 are invalid descriptors (B2B_EINVAL).
    for kind, f, depths in (("nrqs", lambda n1, n2, H, k, inv=0: nrqs(n1, n2, H, k, inv), (16, 17, 1, 0)),
                            ("deep", lambda n1, n2, H, k, inv=0: deep(n1, n2, H, k, inv), (4, 5, 1, 0))):
        top, past, low, zero = depths
        for n1, n2, H, k in ((1, 1, 1, 2), (128, 128, 128, top), (129, 64, 64, 2), (64, 129, 64, 2), (64, 64, 129, 2),
                             (64, 64, 0, 2), (64, 64, 64, past), (64, 64, 64, low), (64, 64, 64, zero)):
            add(f"{kind}{n1}x{n2}H{H}k{k}", [f(n1, n2, H, k)], (36, 1024, 1025))
        add(f"{kind}-inv", [f(32, 32, 64, 3, 1)], (64, 1024, 1025))
        base = f(16, 16, 32, 2)
        for field in ("p0", "p1", "p2", "p3", "i0", "i1"):
            e = dict(base)
            del e[field]
            add(f"null-{kind}-{field}", [e], (64,))
            add(f"planar-then-null-{kind}-{field}", [planar(), e], (64,))
        add(f"{kind}-then-null-planar", [base, dict(planar(), p1=0)], (64,))
        # with planar, BatchNorm and both terminals
        add(f"planar-bn-{kind}-bn-diag", [planar(), bn(), f(32, 32, 64, 3), bn(1), diag()], (64, 1025))
        add(f"{kind}-inv-planar-tril", [f(64, 64, 128, 4, 1), planar(1), tril()], (128, 257))
        add(f"{kind}-ew-diag", [f(32, 32, 64, 2), ew(), diag()], (64, 1024))
    add("nrqs-leaky", [nrqs(32, 32, 64, act=_lib.ACT_LEAKY_RELU)], (64,))
    add("nrqs-act9", [nrqs(32, 32, 64, act=9)], (64,))
    add("nrqs-B0", [nrqs(32, 32, 64, B=0.0)], (64,))
    add("nrqs-Bneg", [nrqs(32, 32, 64, B=-1.0)], (64,))
    add("deep-leaky", [deep(32, 32, 64, act=_lib.ACT_LEAKY_RELU)], (64,))
    add("deep-act9", [deep(32, 32, 64, act=9)], (64,))
    add("nrqs-deep-mlp-srqs", [nrqs(16, 16, 32), deep(16, 16, 32, 2, 1), mlp(16, 16, 32), srqs(16, 16)], (32, 64))
    return out


def _arr(chain, t):
    ds = []
    for spec in chain:
        d = t()
        for k, v in spec.items():
            setattr(d, k, v)
        ds.append(d)
    return (t * len(ds))(*ds)


def measure(L_, chain, D):
    """Every quantity the fixture pins for one chain at depth D."""
    L = len(chain)
    a32 = _arr(chain, _lib.LayerDesc)
    a64 = _arr(chain, _lib.LayerDesc64)
    valid = all(s["kind"] in VALID_KINDS for s in chain)
    fwd = [L_.b2b_chain_workspace_bytes(a32, L, D, N, wy, ws) if (wy or valid) else None
           for N in NS for wy in (0, 1) for ws in (0, 1)]
    op = [L_.b2b_workspace_bytes(a32, D, N) for N in NS]
    vjp = [L_.b2b_chain_vjp_workspace_bytes(a32, L, D, N) for N in NS]
    vjp64 = [L_.b2b_chain_vjp_workspace_bytes_f64(a64, L, D, N) for N in NS]
    st = L_.b2b_chain_vjp_f32(a32, L, None, None, None, None, None, D, 0, D, D, D, None, 0, None)
    n = L_.b2b_last_launch_count()
    st64 = L_.b2b_chain_vjp_f64(a64, L, None, None, None, None, None, D, 0, D, D, D, None, 0, None)
    n64 = L_.b2b_last_launch_count()
    return dict(fwd=fwd, op=op, vjp=vjp, vjp64=vjp64, status=[st, n, st64, n64])


def _load(path):
    handle = ctypes.CDLL(path)
    for name, (res, args) in _lib._SIGS.items():
        fn = getattr(handle, name)
        fn.restype, fn.argtypes = res, args
    return handle


def all_cases():
    return cases() + coupling_cases()


def record(path=_lib.LIB_PATH):
    L_ = _load(path)
    for golden, sweep in ((GOLDEN, cases), (GOLDEN_COUPLINGS, coupling_cases)):
        data = {name: measure(L_, chain, D) for name, chain, D in sweep()}
        with open(golden, "w") as f:
            if golden == GOLDEN:
                json.dump(data, f, separators=(",", ":"), sort_keys=True)
            else:  # one chain per line
                f.write("{\n" + ",\n".join(f"{json.dumps(k)}:{json.dumps(data[k], separators=(',', ':'))}"
                                             for k in sorted(data)) + "\n}")
            f.write("\n")
        print(f"{len(data)} chains -> {golden}")


@pytest.fixture(scope="module")
def expected():
    out = {}
    for golden in (GOLDEN, GOLDEN_COUPLINGS):
        with open(golden) as f:
            out.update(json.load(f))
    return out


def test_sweep_covers_the_fixture(expected):
    names = [name for name, _, _ in all_cases()]
    assert len(names) == len(set(names))
    assert set(names) == set(expected)


def test_chain_plan_matches_fixture(expected):
    L_ = _lib.lib()
    bad = []
    for name, chain, D in all_cases():
        got = measure(L_, chain, D)
        if got != expected[name]:
            bad.append((name, got, expected[name]))
    assert not bad, f"{len(bad)} chains differ, first: {bad[:3]}"


def test_invalid_kind_needs_no_intermediate():
    """A chain with a kind include/b2b.h does not define has no launch plan: the workspace query returns at once, sizing
    no D x N intermediate whether or not y is wanted."""
    L_ = _lib.lib()
    for name, chain, D in all_cases():
        if all(s["kind"] in VALID_KINDS for s in chain):
            continue
        a = _arr(chain, _lib.LayerDesc)
        for N in NS:
            for ws in (0, 1):
                assert (L_.b2b_chain_workspace_bytes(a, len(chain), D, N, 0, ws) ==
                        L_.b2b_chain_workspace_bytes(a, len(chain), D, N, 1, ws)), name


if __name__ == "__main__":
    record(*sys.argv[1:])
