"""bijectors.jl_b200 -- H100-native batched bijector evaluation path behind Bijectors.jl's Transform API.

Import name: ``bijectors_jl_b200`` (the directory name contains a dot; ``bijectors_jl_b200.py`` at the
repository root registers this package under that name).
"""
from ._lib import B2BError, LIB_PATH, exported_symbols, lib  # noqa: F401
from .interface import (  # noqa: F401
    Bijector, Columnwise, Composed, ComposedFunction, GraphedCalls, Inverse, Transform, chain_vjp, colmajor_empty, columnwise, compose, flatten,
    from_numpy,
    inverse, isclosedform, isinvertible, logabsdetjac, logabsdetjac_, planar_chain_vjp, radial_chain_vjp, coupling_vjp, batchnorm_vjp, batchnorm_train_vjp, rqs_vjp, run_chain, to_numpy, transform, transform_,
    with_logabsdet_jacobian, with_logabsdet_jacobian_,
)
from .layers import (  # noqa: F401
    AffineConditioner, Coupling, Elementwise, InvertibleBatchNorm, LeakyReLU, Logit, MLPConditioner, MLPSplineConditioner, DeepMLPConditioner, DeepMLPSplineConditioner, PartitionMask, Permute, PlanarLayer, RadialLayer,
    RationalQuadraticSpline, Scale, Shift, SplineConditioner, Stacked, TruncatedBijector, coupling, elementwise,
    LowerTriangular, UpperTriangular, UnitLowerTriangular, UnitUpperTriangular, LULinear, MaskedAutoregressive,
)
from .transformed_distribution import (  # noqa: F401
    MvNormal, PosDefException, TransformedDistribution, logpdf, logpdf_sum, logpdf_vjp, rand, rand_logpdf, rand_vjp,
    transformed,
)
from . import autograd, distributed  # noqa: F401

lib()  # fail loudly at import time when libb2b.so has not been built
