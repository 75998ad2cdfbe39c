/*
 * b2b.h -- C ABI of libb2b.so: the H100-native batched bijector evaluation path.
 *
 * This is the drop-in boundary for the hot path of TuringLang/Bijectors.jl (v0.16.2): batched
 * `with_logabsdet_jacobian` / `transform` / `logabsdetjac` / `logpdf` of normalising-flow layers over a
 * (D x N) Float32 column-batch.  The reference has no FFI for this path -- "plugging in" means adding
 * more specific Julia methods of its generic functions (src/interface.jl:144,156,183,265) that `ccall`
 * the entry points below; INTEGRATION.md shows that binding (julia/B200Bijectors.jl).
 *
 * Conventions
 *   - Batches are Julia column-major D x N Float32 matrices: column n (one sample) is D contiguous
 *     floats at  x + n*ldx  (ldx >= D, in elements).  Outputs: y (D x N, column stride ldy) and a
 *     length-N vector `logjac` with logjac[n] = log|det J| of the map at column n -- exactly what the
 *     reference's matrix methods return (planar_layer.jl:102-110, radial_layer.jl:58-72,
 *     normalise.jl:41-69); for layers the reference only defines on vectors it equals mapping over
 *     eachcol (SURVEY.md §8).
 *   - ALL pointers are DEVICE pointers unless the name says `host`.  The caller owns every buffer;
 *     the library never allocates or frees device memory on the hot path (b2b_host_ctx_create is the
 *     one explicit allocation site, for the host-buffer entry point).
 *   - `y` may alias `x` (in place; mirrors transform!/with_logabsdet_jacobian!, interface.jl:175-176,
 *     212-218).  `accumulate_logjac != 0` adds into `logjac` (mirrors `logjac + logjac_`,
 *     interface.jl:217); otherwise `logjac` is overwritten.  `y == NULL` skips the D x N store
 *     (logabsdetjac / logpdf only).
 *   - Layer parameters are passed as device pointers to the RAW reference struct fields (e.g.
 *     PlanarLayer.w/u/b, planar_layer.jl:13-18); derived quantities (û, wᵀû, softplus terms) are
 *     computed on the device so no host synchronisation is needed when parameters change every step.
 *   - Index arguments are 0-based.
 *   - `stream` is a cudaStream_t (CUstream) passed as void*.  All work is enqueued on it; no entry
 *     point synchronises the host except b2b_chain_run_host_f32 and b2b_host_ctx_* .
 *   - Return value: 0 = success; negative = argument error (B2B_E*); 1 .. 99999 = the cudaError_t of the failing
 *     runtime call passed through; 100000 + r = NCCL call failed with ncclResult_t r (the two enums overlap, hence the
 *     offset).  Never aborts, never throws.  The Julia shim turns non-zero into
 *     `error(b2b_status_string(rc))`, matching the reference's error sites (interface.jl:160,186;
 *     normalise.jl:43; stacked.jl:158; permute.jl:109-119; rational_quadratic_spline.jl:84-85).
 *   - There is NO CPU fallback anywhere in this library.
 */
#ifndef B2B_H_
#define B2B_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2B_VERSION 100 /* 0.1.0 */

/* status codes */
#define B2B_OK 0
#define B2B_EINVAL (-1)       /* NULL / shape / alignment / range error                         */
#define B2B_EUNSUPPORTED (-2) /* valid request the device path does not implement (e.g. D > 1024) */
#define B2B_EWORKSPACE (-3)   /* workspace too small: see b2b_chain_workspace_bytes              */
#define B2B_ENONCCL (-4)      /* libnccl.so.2 could not be loaded                                */

/* layer kinds (b2b_layer_desc.kind) */
#define B2B_PLANAR 1          /* PlanarLayer                src/bijectors/planar_layer.jl            */
#define B2B_RADIAL 2          /* RadialLayer                src/bijectors/radial_layer.jl            */
#define B2B_RQS 3             /* RationalQuadraticSpline    src/bijectors/rational_quadratic_spline.jl */
#define B2B_COUPLING_AFFINE 4 /* Coupling, θ = Shift(t)∘Scale(exp.(s)), [s;t]=W·x₂+c  coupling.jl    */
#define B2B_BATCHNORM 5       /* InvertibleBatchNorm (eval) src/bijectors/normalise.jl               */
#define B2B_PERMUTE 6         /* Permute                    src/bijectors/permute.jl                 */
#define B2B_STACKED_EW 7      /* Stacked of elementwise laws on row ranges  src/bijectors/stacked.jl */
#define B2B_MVNORMAL_DIAG 8   /* terminal op: logpdf of MvNormal(mu, Diagonal(sigma.^2)) + logjac    */
#define B2B_MVNORMAL_TRIL 9   /* terminal op: logpdf of MvNormal(mu, L*L') (L lower Cholesky factor) + logjac */
/* 10 is not a layer kind: it stays invalid (B2B_EINVAL) so that callers and tests have one fixed invalid value. */
#define B2B_COUPLING_RQS 11   /* Coupling, θ = x₂ -> RationalQuadraticSpline(reshape(W·x₂+c), B)  coupling.jl      */

/* Envelope of B2B_COUPLING_RQS (every entry point, forward, inverse and reverse mode): n1, n2 <= 128, 2 <= K <= 16,
 * D <= 1024.  A layer past it returns B2B_EUNSUPPORTED with nothing launched, and the workspace queries return 0. */
#define B2B_COUPLING_RQS_MAX_N 128
#define B2B_COUPLING_RQS_MAX_K 16
#define B2B_COUPLING_RQS_MAX_D 1024

#define B2B_SCALE_MATRIX 12   /* Scale(A), A a trainable D x D matrix: y = A*x, logjac = logabsdet(A)  scale.jl:14,17,35-36 */
/* Envelope of B2B_SCALE_MATRIX: Float32, D <= 256.  Beyond it every entry point returns B2B_EUNSUPPORTED with nothing
 * launched and the workspace queries return 0; the Float64 entry points refuse the kind the same way. */
#define B2B_SCALE_MATRIX_MAX_D 256

#define B2B_COUPLING_MLP 13   /* Coupling, θ = x₂ -> Shift(t) ∘ Scale(exp.(s)), [s; t] = W₂·σ.(W₁·x₂+c₁)+c₂   coupling.jl */
/* Envelope of B2B_COUPLING_MLP (every entry point, forward, inverse and reverse mode): n1, n2 <= 128, 1 <= H <= 256,
 * D <= 1024.  A layer past it returns B2B_EUNSUPPORTED with nothing launched, and the workspace queries return 0. */
#define B2B_COUPLING_MLP_MAX_N 128
#define B2B_COUPLING_MLP_MAX_H 256
#define B2B_COUPLING_MLP_MAX_D 1024
#define B2B_COUPLING_MLP_RQS 14 /* Coupling, θ = x₂ -> RationalQuadraticSpline(reshape(W₂·σ.(W₁·x₂+c₁)+c₂), B)  coupling.jl */
/* Envelope of B2B_COUPLING_MLP_RQS (every entry point, forward, inverse and reverse mode): n1, n2 <= 128, 1 <= H <= 128,
 * 2 <= K <= 16, D <= 1024.  A layer past it returns B2B_EUNSUPPORTED with nothing launched, and the workspace queries
 * return 0; the Float64 entry points refuse the kind the same way. */
#define B2B_COUPLING_MLP_RQS_MAX_N 128
#define B2B_COUPLING_MLP_RQS_MAX_H 128
#define B2B_COUPLING_MLP_RQS_MAX_K 16
#define B2B_COUPLING_MLP_RQS_MAX_D 1024
#define B2B_COUPLING_DEEP_MLP 15 /* Coupling, θ = x₂ -> Shift(t) ∘ Scale(exp.(s)), [s; t] from an MLP with M hidden layers   coupling.jl */
/* Envelope of B2B_COUPLING_DEEP_MLP (every entry point, forward, inverse and reverse mode): n1, n2 <= 128,
 * 1 <= H <= 128, 2 <= M <= 4 hidden layers, D <= 1024.  A layer past it returns B2B_EUNSUPPORTED with nothing launched,
 * and the workspace queries return 0; the Float64 entry points refuse the kind the same way. */
#define B2B_COUPLING_DEEP_MLP_MAX_N 128
#define B2B_COUPLING_DEEP_MLP_MAX_H 128
#define B2B_COUPLING_DEEP_MLP_MAX_DEPTH 4
#define B2B_COUPLING_DEEP_MLP_MAX_D 1024
#define B2B_COUPLING_DEEP_MLP_RQS 16 /* Coupling, θ = x₂ -> RationalQuadraticSpline(…, B), raw knots from an MLP with M hidden layers   coupling.jl */
/* Envelope of B2B_COUPLING_DEEP_MLP_RQS (every entry point, forward, inverse and reverse mode): n1, n2 <= 128,
 * 1 <= H <= 128, 2 <= K <= 16, 2 <= M <= 4 hidden layers, D <= 1024.  A layer past it returns B2B_EUNSUPPORTED with
 * nothing launched, and the workspace queries return 0; the Float64 entry points refuse the kind the same way. */
#define B2B_COUPLING_DEEP_MLP_RQS_MAX_N 128
#define B2B_COUPLING_DEEP_MLP_RQS_MAX_H 128
#define B2B_COUPLING_DEEP_MLP_RQS_MAX_K 16
#define B2B_COUPLING_DEEP_MLP_RQS_MAX_DEPTH 4
#define B2B_COUPLING_DEEP_MLP_RQS_MAX_D 1024
#define B2B_ELEMENTWISE_VEC 17 /* Shift(a) / Scale(a) / LeakyReLU(a) with a trainable vector a[D]   shift.jl, scale.jl:16,31-32, leaky_relu.jl:25-29 */
#define B2B_SCALE_TRIANGULAR 18 /* Scale(T), T triangular (Lower/Upper/UnitLower/UnitUpperTriangular): y = T*x, logjac = Σ log|Tᵢᵢ|  scale.jl:14,17,35-36 */
/* Envelope of B2B_SCALE_TRIANGULAR: Float32 D <= 256 (the Float64 entry points: D <= 2048).  Beyond it every entry point
 * returns B2B_EUNSUPPORTED with nothing launched and the workspace queries return 0. */
#define B2B_SCALE_TRIANGULAR_MAX_D 256
#define B2B_SCALE_LU 19 /* LULinear: y = P*L*U*x, L, U packed in F as lu(A).factors, P from lu(A).p; logjac = Σ log|Uᵢᵢ|  (Glow's invertible 1x1 convolution) */
/* Envelope of B2B_SCALE_LU: Float32 D <= 256 (the Float64 entry points: D <= 2048).  Beyond it every entry point returns
 * B2B_EUNSUPPORTED with nothing launched and the workspace queries return 0. */
#define B2B_SCALE_LU_MAX_D 256
#define B2B_AUTOREGRESSIVE_MLP 20 /* MaskedAutoregressive: y = x ⊙ exp.(s) + t, [s; t] from a MADE of x₁..x_{i−1} for row i  (MAF / IAF) */
/* Envelope of B2B_AUTOREGRESSIVE_MLP (every Float32 entry point, both directions and reverse mode): D <= 128,
 * 1 <= H <= 256.  Beyond it every entry point returns B2B_EUNSUPPORTED with nothing launched and the workspace queries
 * return 0; the Float64 entry points refuse the kind the same way. */
#define B2B_AUTOREGRESSIVE_MLP_MAX_D 128
#define B2B_AUTOREGRESSIVE_MLP_MAX_H 256
/* hidden-layer activation σ of B2B_COUPLING_MLP, B2B_COUPLING_MLP_RQS, B2B_COUPLING_DEEP_MLP,
 * B2B_COUPLING_DEEP_MLP_RQS and B2B_AUTOREGRESSIVE_MLP (descriptor field n3) */
#define B2B_ACT_TANH 0
#define B2B_ACT_LEAKY_RELU 1 /* v >= 0 ? v : a*v with a = f0 (a = 0: ReLU), the convention of B2B_EW_LEAKY_RELU */

/* elementwise law codes for B2B_STACKED_EW (one code per row) */
#define B2B_EW_IDENTITY 0
#define B2B_EW_EXP 1   /* elementwise(exp): y=exp(x), logjac += x          exp_log.jl:5-6  */
#define B2B_EW_LOG 2   /* elementwise(log): y=log(x), logjac -= log(x)     exp_log.jl:8-9  */
#define B2B_EW_SHIFT 3 /* Shift(a): y = a + x                              shift.jl:14,21  */
#define B2B_EW_SCALE 4 /* Scale(a): y = a * x, logjac += log|a|            scale.jl:13,26  */
#define B2B_EW_LEAKY_RELU 5 /* LeakyReLU(a): y = x >= 0 ? x : a*x, logjac += x < 0 ? log|a| : 0   leaky_relu.jl:18-29 */
#define B2B_EW_LOGIT 6      /* Logit(a, b): y = logit((x-a)/(b-a)), logjac -= log((x-a)(b-x)/(b-a))        logit.jl:15-29 */
#define B2B_EW_TRUNCATED 7  /* TruncatedBijector(lb=a, ub=b) (either may be ±Inf): clamp, then logit / log(x-lb) /
                               log(ub-x) / identity; closed-form inverse log-Jacobian                    truncated.jl:15-91 */

/*
 * One element of a chain.  `inverse != 0` evaluates Inverse(layer) and its log-Jacobian
 * (interface.jl:276-281) in one fused pass.
 *
 * kind               p0          p1          p2          p3       i0              i1            n0    n1   f0
 * PLANAR             w[D]        u[D]        b[1]        -        -               -             -     -    -
 * RADIAL             α_[1]       β[1]        z_0[D]      -        -               -             -     -    -
 * RQS                widths      heights     derivatives -        -               -             K1    -    -
 *                    (each D x K1 column-major = the struct fields of rational_quadratic_spline.jl:75-79)
 * COUPLING_AFFINE    W[2n1 x n2] c[2n1]|NULL -           -        idx1[n1]        idx2[n2]      n1    n2   -
 *                    (W column-major; rows 0..n1-1 give s, rows n1..2n1-1 give t; idx = PartitionMask rows.
 *                     n2 / n3 = first row of idx1 / idx2 when that list is the contiguous range
 *                     first..first+len-1 (then the pointer may be NULL), else -1.  Contiguous masks with
 *                     n1 <= 128 and n2 in {64,128} run on the tensor cores (wgmma) when workspace is given.)
 * BATCHNORM          b[D]        logs[D]     m[D]        v[D]     -               -             -     -    eps
 * PERMUTE            -           -           -           -        dst_of_src[D]   -             -     -    -
 *                    (y[dst_of_src[i]] = x[i], i.e. Permute(indices) of permute.jl:90-100, 0-based)
 * STACKED_EW         a[D]        b[D]|NULL   -           -        code[D]         -             -     -    -
 *                    (a = the law's parameter: Shift / Scale / LeakyReLU value, Logit / Truncated lower bound;
 *                     b = second parameter: Logit / Truncated upper bound)
 * MVNORMAL_DIAG      mu[D]|NULL  sigma[D]|NULL -         -        -               -             -     -    -
 * MVNORMAL_TRIL      mu[D]|NULL  L[D x D]    -           -        -               -             -     -    -
 *                    (Distributions' FullNormal MvNormal(mu, Σ) with Σ = L Lᵀ: L column-major, required; only its lower
 *                     triangle is read, the strictly upper entries are ignored.  Lᵢᵢ > 0 is the caller's contract -- what
 *                     `cholesky` guarantees; nothing on the device checks it, and a non-positive diagonal gives NaN / −Inf.
 *                     Like MVNORMAL_DIAG it must be the last element with inverse == 0, else B2B_EINVAL.  Float32:
 *                     D <= 256, Float64 (b2b_layer_desc_f64, L read through L2): D <= 2048; B2B_EUNSUPPORTED beyond.)
 * COUPLING_RQS       W           c|NULL      -           -        idx1[n1]        idx2[n2]      n1    n2   B
 *                    (n2 of the descriptor = K bins, n3 = 0; W is ((3K−1)·n1 x n2) column-major, c has (3K−1)·n1 entries
 *                     (NULL = 0); both index lists are required.  Per column, v = W·x₂ + c; transformed row i (0-based) takes
 *                     raw widths v[i + n1·k] (k < K), raw heights v[n1·K + i + n1·k] (k < K) and raw derivatives
 *                     v[2·n1·K + i + n1·k] (k < K−1), normalised as rational_quadratic_spline.jl:109-123 does (row softmax,
 *                     a leading 0, cumsum, 2B·(…) − B; log1pexp derivatives with unit end slopes), then the spline of
 *                     :317-357 (inverse :183-220) maps x₁; outside [−B, B] an element is the identity with log-Jacobian 0.
 *                     Float32 only, exact fp32 on the CUDA cores, its own launch (no BatchNorm folding).  Envelope:
 *                     B2B_COUPLING_RQS_MAX_*; the Float64 entry points return B2B_EUNSUPPORTED for this kind.)
 * SCALE_MATRIX       A[D x D]    -           -           -        -               -             -     -    -
 *                    (A column-major, required.  Per column y = A x with logjac = log|det A|; inverse != 0 gives
 *                     y = A⁻¹ x with −log|det A|.  The sign of det A does not matter (logabsdet).  log|det A| and A⁻¹ come
 *                     from an fp64 LU with partial pivoting computed on the device at every call (A may change between
 *                     calls; nothing synchronises the host); the map is exact fp32 FMA.  An invertible A is the caller's
 *                     contract, as Lᵢᵢ > 0 is for MVNORMAL_TRIL: for a singular A the forward gives y = A x and −Inf, the
 *                     inverse non-finite values; nothing on the device checks it.  Float32 only, D <= B2B_SCALE_MATRIX_MAX_D,
 *                     its own launch; the Float64 entry points return B2B_EUNSUPPORTED for this kind.)
 * COUPLING_MLP       W₁[H x n2]  c₁[H]|NULL  W₂[2n1 x H] c₂[2n1]|NULL idx1[n1]    idx2[n2]      n1    n2   a
 *                    (n2 of the descriptor = H hidden units, n3 = the activation σ: B2B_ACT_TANH or B2B_ACT_LEAKY_RELU
 *                     with slope a = f0 (ignored for tanh); any other n3 returns B2B_EINVAL.  W₁ and W₂ are column-major
 *                     and required, c₁ / c₂ may be NULL (= 0); both index lists are required.  Per column
 *                     [s; t] = W₂·σ.(W₁·x₂ + c₁) + c₂, rows 0..n1-1 of W₂ give s and rows n1..2n1-1 give t as for
 *                     COUPLING_AFFINE, whose law, log-Jacobian ±Σ s and inverse (the network evaluated on y₂ = x₂) the
 *                     layer shares.  Float32 only, exact fp32 FMA on the CUDA cores, its own launch (no BatchNorm
 *                     folding).  Envelope: B2B_COUPLING_MLP_MAX_*; the Float64 entry points return B2B_EUNSUPPORTED.)
 * COUPLING_MLP_RQS   W₁[H x n2]  c₁[H]|NULL  W₂[J x H]   c₂[J]|NULL idx1[n1]      idx2[n2]      n1    n2   a
 *                    (J = (3K−1)·n1; n2 of the descriptor = H hidden units, n3 = σ | (K << 8) with σ = B2B_ACT_TANH or
 *                     B2B_ACT_LEAKY_RELU (slope a = f0) and K bins, f1 = B > 0.  W₁ and W₂ are column-major and required,
 *                     c₁ / c₂ may be NULL (= 0); both index lists are required.  Per column h = σ.(W₁·x₂ + c₁) and
 *                     v = W₂·h + c₂; transformed row i takes its raw widths, heights and derivatives from v as COUPLING_RQS
 *                     does (v[i + n1·k], v[n1·K + i + n1·k], v[2·n1·K + i + n1·k]), with that layer's normalisation, spline,
 *                     inverse (the network evaluated on y₂ = x₂) and identity outside [−B, B].  n1, n2, H >= 1,
 *                     n1 + n2 <= D, K >= 1, a known σ and B > 0, else B2B_EINVAL.  Float32 only, exact fp32 on the CUDA
 *                     cores, its own launch.  Envelope: B2B_COUPLING_MLP_RQS_MAX_*; the Float64 entry points return
 *                     B2B_EUNSUPPORTED.)
 * COUPLING_DEEP_MLP  W_in[H x n2] W_hid     W_out[2n1 x H] c|NULL  idx1[n1]        idx2[n2]      n1    n2   a
 *                    (n2 of the descriptor = H hidden units, n3 = σ | (M << 8) with σ = B2B_ACT_TANH or
 *                     B2B_ACT_LEAKY_RELU (slope a = f0) and M >= 2 hidden layers.  W_hid holds the M − 1 hidden-to-hidden
 *                     matrices W_2 .. W_M, each H x H, back to back (W_l at offset (l − 2)·H²).  c packs every bias,
 *                     [c_1 (H) | … | c_M (H) | c_out (2n1)], or is NULL for none.  All matrices are column-major; W_in,
 *                     W_hid, W_out and both index lists are required.  Per column h_1 = σ.(W_in·x₂ + c_1),
 *                     h_l = σ.(W_l·h_{l−1} + c_l) for l = 2..M and [s; t] = W_out·h_M + c_out, rows 0..n1-1 of W_out
 *                     giving s and rows n1..2n1-1 giving t; law, log-Jacobian ±Σ s and inverse (the network evaluated on
 *                     y₂ = x₂) as for COUPLING_MLP.  n1, n2, H >= 1, n1 + n2 <= D, M >= 2 and a known σ, else B2B_EINVAL.
 *                     Float32 only, exact fp32 FMA on the CUDA cores, its own launch.  Envelope:
 *                     B2B_COUPLING_DEEP_MLP_MAX_*; the Float64 entry points return B2B_EUNSUPPORTED.)
 * COUPLING_DEEP_MLP_RQS W_in[H x n2] W_hid  W_out[J x H] c|NULL    idx1[n1]        idx2[n2]      n1    n2   a
 *                    (J = (3K−1)·n1; n2 of the descriptor = H hidden units, n3 = σ | (K << 8) | (M << 16) with
 *                     σ = B2B_ACT_TANH or B2B_ACT_LEAKY_RELU (slope a = f0), K bins and M >= 2 hidden layers, f1 = B > 0.
 *                     W_hid holds W_2 .. W_M, each H x H, back to back (W_l at offset (l − 2)·H²); c packs every bias,
 *                     [c_1 (H) | … | c_M (H) | c_out (J)], or is NULL for none.  All matrices are column-major; W_in,
 *                     W_hid, W_out and both index lists are required.  Per column h_1 = σ.(W_in·x₂ + c_1),
 *                     h_l = σ.(W_l·h_{l−1} + c_l) for l = 2..M and v = W_out·h_M + c_out; transformed row i takes its raw
 *                     widths, heights and derivatives from v, with the normalisation, spline, inverse (the network
 *                     evaluated on y₂ = x₂) and identity outside [−B, B] of COUPLING_RQS and COUPLING_MLP_RQS.
 *                     n1, n2, H >= 1, n1 + n2 <= D, K >= 1, M >= 2, a known σ and B > 0, else B2B_EINVAL.  Float32 only,
 *                     exact fp32 on the CUDA cores, its own launch.  Envelope: B2B_COUPLING_DEEP_MLP_RQS_MAX_*; the
 *                     Float64 entry points return B2B_EUNSUPPORTED.)
 * ELEMENTWISE_VEC    a[D]        -           -           -        -               -             law   -    -
 *                    (one law on every row, n0 = B2B_EW_SHIFT, B2B_EW_SCALE or B2B_EW_LEAKY_RELU (any other value returns
 *                     B2B_EINVAL), with the row's own parameter a = p0[r] (required): the map and log-Jacobian of that law of
 *                     STACKED_EW, and inverse != 0 its inverse on the same a.  A STACKED_EW layer with code[r] = n0 and the
 *                     same a gives the same bits.  It fuses into column-local launches like STACKED_EW (same 3Dp staging,
 *                     D <= 1024), runs in both precisions, and trains a: slot 0 of b2b_chain_vjp_f32 / _f64.  a > 0 for
 *                     LeakyReLU is the caller's contract; nothing on the device checks it.)
 * SCALE_TRIANGULAR   T[D x D]    -           -           -        -               -             tri   unit -
 *                    (T column-major, required.  n0 = 0: lower, 1: upper -- only that triangle is read; n1 = 0: the stored
 *                     diagonal, 1: a unit diagonal, taken as 1 and not read.  Any other n0 / n1 returns B2B_EINVAL.  Entries
 *                     outside what is read may hold anything, NaN included.  Per column y = T x with logjac = Σᵢ log|Tᵢᵢ|,
 *                     summed in fp64 in row order and rounded once (0 for the unit forms); inverse != 0 gives y = T⁻¹ x
 *                     with the negated log-Jacobian.  A zero diagonal is the caller's contract, as an invertible A is for
 *                     SCALE_MATRIX.  A prep launch writes the triangle of T (forward) or of T⁻¹ (inverse, D independent
 *                     fp64 substitutions rounded to fp32) with zeros elsewhere; the map is exact fp32 FMA over the
 *                     triangle only.  Float32 D <= B2B_SCALE_TRIANGULAR_MAX_D, its own launches; Float64 D <= 2048, one
 *                     warp per column with T read through L2.  Trains T: slot 0 of b2b_chain_vjp_f32 / _f64.)
 * SCALE_LU           F[D x D]    -           -           -        dst_of_src[D]   -             -     -    -
 *                    (F column-major, required (NULL: B2B_EINVAL); i0 NULL is the identity permutation.  F packs two
 *                     factors as LAPACK getrf and Julia's lu(A).factors do: the strict lower triangle is L, whose unit
 *                     diagonal is implied and not read, and the upper triangle with the diagonal is U.  Per column
 *                     y = P·L·U·x with y[i0[r]] = (L U x)[r] (PERMUTE's index semantics), so F = lu(A).factors with
 *                     i0 = lu(A).p .- 1 is y = A x; logjac = Σᵢ log|Uᵢᵢ|, summed in fp64 in row order and rounded once.
 *                     inverse != 0 gives y = U⁻¹ L⁻¹ Pᵀ x with the negated log-Jacobian.  The map of the composition
 *                     PERMUTE(i0) ∘ SCALE_TRIANGULAR(F, unit lower) ∘ SCALE_TRIANGULAR(F, upper) in one layer.  A
 *                     permutation in i0 and a non-zero Uᵢᵢ are the caller's contract.  A prep launch writes M = P·L·U or
 *                     U⁻¹ L⁻¹ Pᵀ (each entry in fp64, rounded once to fp32); the map is SCALE_MATRIX's.  Float32
 *                     D <= B2B_SCALE_LU_MAX_D, its own launches; Float64 D <= 2048, one warp per column with F read
 *                     through L2.  Trains F: slot 0 of b2b_chain_vjp_f32 / _f64, packed like F.)
 * AUTOREGRESSIVE_MLP W₁[H x D]  c₁[H]|NULL  W₂[2D x H] c₂[2D]|NULL m[H]           -             -     -    H    σ   a
 *                    (a MADE layer: i0 holds the hidden units' integer degrees m_k (int32, any value), n2 = H hidden
 *                     units, n3 = σ: B2B_ACT_TANH or B2B_ACT_LEAKY_RELU with slope a = f0; any other n3 returns
 *                     B2B_EINVAL.  W₁, W₂ and m are required, c₁ / c₂ may be NULL (= 0); W₁ and W₂ are column-major.
 *                     With 1-based rows r and masks M₁[k, r] = (r <= m_k), M₂[i, k] = M₂[D+i, k] = (m_k < i), per column
 *                     [s; t] = (M₂⊙W₂)·σ.((M₁⊙W₁)·x + c₁) + c₂ and y = x ⊙ exp.(s) + t, logjac = Σ s: sᵢ and tᵢ depend
 *                     on x₁..x_{i−1} only, so the Jacobian is lower triangular for any degrees.  Entries outside the
 *                     masks are not read and may hold anything, NaN included.  inverse != 0 recovers x row by row,
 *                     xᵢ = (yᵢ − tᵢ)/exp(sᵢ) with sᵢ, tᵢ from the rows already recovered, logjac = −Σ s(x).  The forward
 *                     direction (IAF sampling, MAF's logpdf through inverse) is one network evaluation, exact fp32 FMA
 *                     on the CUDA cores; the inverse is sequential over the D rows.  Float32 only, its own launches.
 *                     Envelope: B2B_AUTOREGRESSIVE_MLP_MAX_*.  Trains W₁ c₁ W₂ c₂: slots 0-3 of b2b_chain_vjp_f32.)
 * Any other kind value returns B2B_EINVAL.
 */
typedef struct b2b_layer_desc {
  int32_t kind;
  int32_t inverse;
  int32_t n0, n1, n2, n3;
  float f0, f1;
  const float* p0;
  const float* p1;
  const float* p2;
  const float* p3;
  const int32_t* i0;
  const int32_t* i1;
} b2b_layer_desc;

#define B2B_MAX_CHAIN 24

int b2b_version(void);
const char* b2b_status_string(int status);

/* ---- chain evaluation: Composed / ComposedFunction (src/bijectors/composed.jl:4,11-14 and the
 * ChangesOfVariables rule for ComposedFunction) ----------------------------------------------------
 * Applies layers[0], layers[1], ... in order (inner-most first), accumulating per-column log-Jacobians.
 * Consecutive column-local layers are fused into ONE kernel launch (each column is read once and
 * written once for the whole fused run); COUPLING_AFFINE layers run in their own GEMM kernel, which also
 * absorbs a BATCHNORM layer directly before and/or after it as a per-row affine (needs workspace).
 * Limits.  Column-local layers need D <= 1024.  A fused launch stages the derived parameters of its layers in
 * 200 KB of shared memory, in floats at the padded depth Dp = D rounded up to 32, 64, 128, 256, 512 or 1024:
 * PLANAR 2Dp+4, RADIAL Dp+4, BATCHNORM 4Dp+4, STACKED_EW and ELEMENTWISE_VEC 3Dp, MVNORMAL_DIAG 2Dp+4, PERMUTE Dp (plus, once per launch
 * that permutes, 8192 floats of column scratch), RQS (2·KP + 8·K1)·Dp with KP = K1 rounded up
 * to a power of two -- so an RQS layer takes K1 <= 64 knots for D <= 64, K1 <= 34 for D <= 128, K1 <= 17 for D <= 256,
 * K1 <= 8 for D <= 512 and K1 <= 4 for D <= 1024 (the default K = 8 bins, K1 = 9, up to D = 256).  A run of column-local
 * layers that does not fit is split into several launches (the terminal MVNORMAL_DIAG stays in the last one).
 * COUPLING_AFFINE takes any N, and any D while 264·(n1 + n2) + 4·ceil(D/32) + 2048 <= 204800 bytes (the rows it stages
 * and a bit per row); up to D = 1024 that is n1 + n2 <= 767.  COUPLING_RQS runs in its own launch (any N, the envelope of
 * B2B_COUPLING_RQS_MAX_*; a batch sum needs the chain to end in a fused launch).  SCALE_MATRIX runs in its own launches
 * (D <= B2B_SCALE_MATRIX_MAX_D, any N): a one-CTA fp64 LU of A, for the inverse direction a second launch forming A⁻¹,
 * then the per-column GEMM y = M x, which reads each column once and writes it once (y may alias x).  Like COUPLING_RQS,
 * a batch sum needs the chain to end in a fused launch (a logpdf chain ends in its MvNormal terminal).  The layer needs
 * workspace for its factor: b2b_chain_workspace_bytes adds 12·D² + 4·D + 8 bytes, each of the four parts rounded up to
 * 256 bytes, plus 256, for a chain with any SCALE_MATRIX layer (the layers share it; they run one after another).
 * SCALE_TRIANGULAR runs the same way (D <= B2B_SCALE_TRIANGULAR_MAX_D, any N, y may alias x) in two launches: a prep
 * launch, parallel over columns, writing M = T or T⁻¹ (fp32, zero outside the triangle) and log|det T|, then the map
 * y = M x, which skips the k-blocks that are zero for all rows a warp owns (about D(D+1)/2 FMA per column).  With y == NULL
 * the second launch writes the log-Jacobians only.  Its workspace is 4·D² + 8 bytes, each part rounded up to 256 bytes,
 * plus 256; a chain holding both Scale kinds shares one region of the larger of the two sizes.
 * SCALE_LU runs in two launches the same way (D <= B2B_SCALE_LU_MAX_D, any N, y may alias x): a prep launch, parallel
 * over columns, writing M = P·L·U or U⁻¹ L⁻¹ Pᵀ (fp32) and log|det U|, then SCALE_MATRIX's map y = M x (D² FMA per
 * column).  With y == NULL the second launch writes the log-Jacobians only.  Its workspace is SCALE_TRIANGULAR's,
 * 4·D² + 8 bytes, each part rounded up to 256 bytes, plus 256; a chain holding several Scale kinds (SCALE_MATRIX,
 * SCALE_TRIANGULAR, SCALE_LU) shares one region of the larger of the sizes.
 * COUPLING_MLP runs in its own launch (any N, any ld >= D, scattered index lists, y may alias x; the envelope of
 * B2B_COUPLING_MLP_MAX_*; no workspace); like COUPLING_RQS, a batch sum needs the chain to end in a fused launch.
 * COUPLING_MLP_RQS runs in its own launch the same way (any N, any ld >= D, scattered index lists, y may alias x; the
 * envelope of B2B_COUPLING_MLP_RQS_MAX_*; no workspace; a batch sum needs the chain to end in a fused launch).
 * COUPLING_DEEP_MLP runs in its own launch the same way (any N, any ld >= D, scattered index lists, y may alias x; the
 * envelope of B2B_COUPLING_DEEP_MLP_MAX_*; no workspace; a batch sum needs the chain to end in a fused launch).
 * COUPLING_DEEP_MLP_RQS runs in its own launch the same way (any N, any ld >= D, scattered index lists, y may alias x;
 * the envelope of B2B_COUPLING_DEEP_MLP_RQS_MAX_*; no workspace; a batch sum needs the chain to end in a fused launch).
 * AUTOREGRESSIVE_MLP runs in two launches (D <= B2B_AUTOREGRESSIVE_MLP_MAX_D, H <= B2B_AUTOREGRESSIVE_MLP_MAX_H, any
 * N, any ld >= D, y may alias x): a prep launch writing the masked weights M₁⊙W₁, M₂⊙W₂ (zeros outside the masks) and
 * a row-paired copy of M₂⊙W₂, then the forward network over 64-column tiles or, for inverse != 0, the sequential
 * recovery, one warp per four columns.  Its workspace is 5·H·D floats in three parts (H·D, 2·H·D, 2·H·D), each rounded
 * up to 256 bytes, plus 256, shared with the Scale layers' region (one region of the largest; the layers run one after
 * another); a batch sum needs the chain to end in a fused launch.
 * The whole chain is planned before anything is enqueued: a
 * layer that fits no kernel returns B2B_EUNSUPPORTED with nothing launched and no output written.
 * If the last element is B2B_MVNORMAL_DIAG, `logjac` receives logpdf[n] = logpdf(MvNormal)(x_n) +
 * accumulated logjac (transformed_distribution.jl:165-169 when the preceding layers are the inverse
 * chain) and, when sum_out != NULL, *sum_out (device double) receives Σ_n logpdf[n] (fixed summation
 * order, deterministic).
 * B2B_MVNORMAL_TRIL as the last element does the same for MvNormal(mu, L Lᵀ).  It runs as its own launch after the
 * preceding layers (which write the recovered x to y, or to the D x N scratch of the workspace when y == NULL), so it costs
 * 8·D B/sample more HBM traffic than a terminal fused into the last column-local launch; the launch stages the packed lower
 * triangle of L in shared memory (Float32 D <= 256, B2B_EUNSUPPORTED beyond, nothing launched) and is bound by the
 * D(D+1)/2 FP32 FMA per sample of the whitening solve L⁻¹(x − mu).
 * A batch sum without `logjac` (sum_out != NULL, logjac == NULL) needs the chain to end in either terminal.  When such a
 * chain takes more than one launch, the log-Jacobians of the launches before the last travel through an N-float slice of
 * the workspace, which b2b_chain_workspace_bytes includes when want_sum != 0 (align_up(4·N, 1024) bytes); the first
 * launch writes that slice, so accumulate_logjac has no effect, as everywhere `logjac` is NULL.
 * With a batch sum, a BatchNorm that is the chain's last launch on its own is not folded into the coupling before it.
 * workspace: device scratch of at least b2b_chain_workspace_bytes(...) bytes (may be NULL when 0).
 */
int b2b_chain_run_f32(const b2b_layer_desc* layers, int32_t L, const float* x, float* y, float* logjac,
                      double* sum_out, int32_t D, int64_t N, int64_t ldx, int64_t ldy,
                      int accumulate_logjac, void* workspace, size_t workspace_bytes, void* stream);

size_t b2b_chain_workspace_bytes(const b2b_layer_desc* layers, int32_t L, int32_t D, int64_t N,
                                 int want_y, int want_sum);
/* Workspace of ONE operation (SURVEY §8(b) `b2b_workspace_bytes(op, D, N)`): what b2b_chain_workspace_bytes returns for
 * the one-element chain {*op} with the D x N store and without the batch sum.  The specialised queries below
 * (b2b_coupling_workspace_bytes, b2b_batchnorm_train_workspace_bytes, b2b_*_vjp_workspace_bytes) remain for entry
 * points that are not chain elements.  With y == NULL a chain of several launches (a coupling layer, or a split run)
 * needs a D x N scratch matrix, which is included. */
size_t b2b_workspace_bytes(const b2b_layer_desc* op, int32_t D, int64_t N);

/* Number of kernel launches the previous b2b_chain_run_f32 call on this thread enqueued. */
int b2b_last_launch_count(void);

/* Select kernel implementations (testing / profiling); the selection is PER CALLING THREAD (thread-local, default 0),
 * so concurrent callers cannot disturb each other.  Ones digit -- fused column-local kernel: 0 = auto
 * (default), 1 = lane-group direct-global kernel (v0), 2 = TMA-staged thread-per-column interpreter (v1) only,
 * 3 = unrolled planar-chain kernel only (segments of <= 8 PlanarLayers, D in {32,64,128}; else B2B_EUNSUPPORTED).
 * Tens digit -- coupling: 0 = auto (tensor cores when the mask is contiguous and workspace is given),
 * 1 = always the exact-fp32 CUDA-core kernel.  Hundreds digit -- 1 = do not fold BatchNorm layers into neighbouring coupling launches.
 * No entry point uses library-owned device state (everything is launch-only on the caller's stream), and the library
 * keeps no mutable process-global state: the only host-side state is this thread-local selector, the thread-local
 * launch counter and the lazily resolved driver / NCCL entry points (write-once). */
int b2b_set_kernel_variant(int variant);

/* ---- single layers (thin wrappers over a 1-element chain) --------------------------------------- */
/* PlanarLayer: planar_layer.jl:102-110 (fwd), :112-127 + find_alpha :160-185 (inverse) */
int b2b_planar_fwd_f32(const float* x, float* y, float* logjac, const float* w, const float* u,
                       const float* b, int32_t D, int64_t N, int64_t ldx, int64_t ldy,
                       int accumulate_logjac, void* stream);
int b2b_planar_inv_f32(const float* x, float* y, float* logjac, const float* w, const float* u,
                       const float* b, int32_t D, int64_t N, int64_t ldx, int64_t ldy,
                       int accumulate_logjac, void* stream);
/* A ∘-chain of L PlanarLayers whose parameters live in HOST memory -- which is where the reference keeps them
 * (PlanarLayer's fields are host Arrays, planar_layer.jl:13-18; a flow that was never moved with fmap(cu, .)).
 * `w_host`, `u_host` are L x D (layer l at offset l*D, application order), `b_host` has L entries.  û = get_u_hat
 * (planar_layer.jl:65-70) is derived on the host; the derived parameters travel as KERNEL ARGUMENTS (constant bank),
 * so the kernel spends no shared-memory bandwidth on them.  `inverse` != 0 applies inverse(layer l) for every l in
 * the given order (the caller passes the layers reversed, as inverse(f∘g) = inverse(g)∘inverse(f)).
 * `x`, `y`, `logjac` are DEVICE pointers as everywhere else.  D in {32, 64, 128}; B2B_EUNSUPPORTED otherwise (use
 * b2b_chain_run_f32 with device-resident parameters). */
int b2b_planar_chain_hostparams_f32(const float* w_host, const float* u_host, const float* b_host, int32_t L,
                                    int inverse, const float* x, float* y, float* logjac, int32_t D, int64_t N,
                                    int64_t ldx, int64_t ldy, int accumulate_logjac, void* stream);
/* Reverse mode (vector-Jacobian product) of with_logabsdet_jacobian through a ∘-chain of L <= 8 PlanarLayers, forward
 * direction -- the computation the reference obtains from its AD rules when a flow is trained
 * (docs/src/flows.md:93-100; ext/BijectorsChainRulesCoreExt.jl; get_u_hat planar_layer.jl:65-70 is differentiated
 * through).  Inputs: the batch `x` the chain was applied to, the cotangents `ybar` (D x N, of the transformed batch)
 * and `ljbar` (N, of the accumulated logjac; NULL = zeros).  Outputs: `xbar` (D x N cotangent of x, required) and --
 * when all three are non-NULL -- the parameter cotangents `wbar`, `ubar` (L x D, layer l at offset l*D) and `bbar` (L),
 * summed over the N columns (a multi-GPU caller all-reduces them, see b2b_allreduce_sum_f64).  D in {32, 64, 128};
 * `layers` are B2B_PLANAR descriptors in application order, either all with inverse == 0 (the forward chain) or all
 * with inverse == 1 (the chain inverse(flow) that logpdf(td, y) evaluates, docs/src/flows.md:66-100: `x` is then the
 * observed batch y, `ybar` the cotangent of the recovered x; find_alpha is differentiated with the reference's
 * implicit-function rule, ext/BijectorsChainRulesCoreExt.jl:42-46); cotangent l of wbar/ubar/bbar belongs to layers[l].  `xbar` may alias `ybar` (or `x`) only when no parameter cotangents
 * are requested: with them the parameter pass re-reads `x` and `ybar` after `xbar` has been written, and any overlap
 * of the xbar range with either returns B2B_EINVAL.  Workspace: b2b_planar_chain_vjp_workspace_bytes. */
size_t b2b_planar_chain_vjp_workspace_bytes(int32_t L, int32_t D, int64_t N);
int b2b_planar_chain_vjp_f32(const b2b_layer_desc* layers, int32_t L, const float* x, const float* ybar,
                             const float* ljbar, float* xbar, float* wbar, float* ubar, float* bbar, int32_t D,
                             int64_t N, int64_t ldx, int64_t ldybar, int64_t ldxbar, void* workspace,
                             size_t workspace_bytes, void* stream);
/* Reverse mode of with_logabsdet_jacobian through a ∘-chain of L <= 8 RadialLayers, each layer forward or Inverse
 * (radial_layer.jl:43-53,58-72 / :88-102,124-129 differentiated as the reference's AD does; compute_r by the
 * implicit-function rule; directions may be mixed): inputs as for b2b_planar_chain_vjp_f32;
 * outputs `xbar` (D x N, may alias `ybar`) and the parameter cotangents summed over the columns: `alpha_bar`, `beta_bar`
 * (L each, w.r.t. the RAW parameters α_, β: the log1pexp transforms of :44-45 are differentiated through) and `z0_bar`
 * (L x D).  Any D <= 128.  Workspace: b2b_radial_chain_vjp_workspace_bytes. */
size_t b2b_radial_chain_vjp_workspace_bytes(int32_t L, int32_t D);
int b2b_radial_chain_vjp_f32(const b2b_layer_desc* layers, int32_t L, const float* x, const float* ybar,
                             const float* ljbar, float* xbar, float* alpha_bar, float* beta_bar, float* z0_bar,
                             int32_t D, int64_t N, int64_t ldx, int64_t ldybar, int64_t ldxbar, void* workspace,
                             size_t workspace_bytes, void* stream);
/* Reverse mode of ONE affine coupling layer (either direction) -- with the eval-mode BatchNorm VJP below it makes a
 * RealNVP flow (BASELINE config 5) trainable on the device.  What the reference's AD computes for coupling.jl:206-228
 * with the law Shift(t)∘Scale(exp.(s)); the pullback of `combine` (ext/BijectorsChainRulesCoreExt.jl:48-62) is the row
 * scatter of the three cotangent blocks.  `layer`: a B2B_COUPLING_AFFINE descriptor (n1, n2 <= 128, any index lists;
 * the kernel stages all D rows of the input and the cotangent: D <= 747 at n1 = n2 = 128, else B2B_EUNSUPPORTED);
 * `x`: the batch the layer was applied to (for inverse != 0 the observed y); `ybar` (D x N) / `ljbar` (N, NULL = zeros):
 * cotangents of the layer's two outputs.  Outputs: `xbar` (D x N; may alias `ybar`), `Wbar` (2n1 x n2, column-major like
 * W) and `cbar` (2n1), summed over the N columns (a multi-GPU caller all-reduces them).  Exact fp32 on the CUDA cores,
 * deterministic.  Workspace: b2b_coupling_affine_vjp_workspace_bytes. */
size_t b2b_coupling_affine_vjp_workspace_bytes(int32_t n1, int32_t n2);
int b2b_coupling_affine_vjp_f32(const b2b_layer_desc* layer, const float* x, const float* ybar, const float* ljbar,
                                float* xbar, float* Wbar, float* cbar, int32_t D, int64_t N, int64_t ldx, int64_t ldybar,
                                int64_t ldxbar, void* workspace, size_t workspace_bytes, void* stream);
/* Reverse mode of the eval-mode InvertibleBatchNorm (normalise.jl:61-67 / :74-86) w.r.t. its input and its trainable
 * fields b, logs (Functors.@functor InvertibleBatchNorm (b, logs); m, v are statistics): `bbar`, `logsbar` (D each) are
 * summed over the columns; arguments as above.  D <= 1024. */
size_t b2b_batchnorm_eval_vjp_workspace_bytes(int32_t D);
int b2b_batchnorm_eval_vjp_f32(const b2b_layer_desc* layer, const float* x, const float* ybar, const float* ljbar,
                               float* xbar, float* bbar, float* logsbar, int32_t D, int64_t N, int64_t ldx, int64_t ldybar,
                               int64_t ldxbar, void* workspace, size_t workspace_bytes, void* stream);
/* Reverse mode of ONE RationalQuadraticSpline layer (either direction): what the reference's AD computes through
 * rational_quadratic_spline.jl:317-357 (forward) / :183-220 (inverse, by the inverse-function theorem at the recovered
 * point).  `layer`: a B2B_RQS descriptor (K1 = n0 <= 64 knots, D <= 256); `x`: the batch the layer was applied to (the
 * observed y for inverse != 0).  Outputs: `xbar` (D x N; may alias `ybar`) and the cotangents of the PROCESSED knot arrays
 * `widths_bar`, `heights_bar`, `derivs_bar` (D x K1 each, laid out like the descriptor's p0/p1/p2), summed over the N
 * columns; elements outside the box pass `ybar` through.  The map from the raw (softmax / softplus) parameters to the
 * processed arrays is the caller's (constructor :47-76), as in the reference.  Deterministic (no atomics).
 * Workspace: b2b_rqs_vjp_workspace_bytes (0 = unsupported shape). */
size_t b2b_rqs_vjp_workspace_bytes(int32_t K1, int32_t D);
int b2b_rqs_vjp_f32(const b2b_layer_desc* layer, const float* x, const float* ybar, const float* ljbar, float* xbar,
                    float* widths_bar, float* heights_bar, float* derivs_bar, int32_t D, int64_t N, int64_t ldx,
                    int64_t ldybar, int64_t ldxbar, void* workspace, size_t workspace_bytes, void* stream);
/* Reverse mode of b2b_chain_run_f32: the vector-Jacobian product through ANY chain it accepts -- layers in application
 * order with their `inverse` flags, optionally ending in the terminal B2B_MVNORMAL_DIAG / _TRIL (then the logjac output is
 * logpdf).  What the reference's reverse-mode AD computes for `with_logabsdet_jacobian(flow, x)` or
 * `logpdf(transformed(base, flow), y)` (docs/src/flows.md:93-100).
 * Inputs: `x`, the batch the chain was applied to; `ybar` (D x N) the cotangent of the y that b2b_chain_run_f32 writes
 * for the same chain (NULL = zeros, the usual case for logpdf); `ljbar` (N) the cotangent of logjac / logpdf (NULL =
 * zeros).  Outputs: `xbar` (D x N, required, must not overlap `x` or `ybar`: B2B_EINVAL) and, when `param_bars` != NULL,
 * 4*L pointers: entry 4l+i receives the cotangent of layers[l].p<i> in the shape and layout of p<i> (NULL entries are not
 * computed), summed over the N columns in a fixed order (deterministic; a multi-GPU caller all-reduces them).
 * Trainable slots: PLANAR w u b; RADIAL α_ β z_0 (raw); RQS widths heights derivatives (processed); COUPLING W c (also
 * COUPLING_RQS, whose W̄ is ((3K−1)·n1 x n2) column-major like W; a c̄ request with c == NULL returns B2B_EINVAL);
 * COUPLING_MLP and COUPLING_MLP_RQS W₁ c₁ W₂ c₂ (column-major like the parameters; a c̄₁ / c̄₂ request whose c is NULL
 * returns B2B_EINVAL); COUPLING_DEEP_MLP W_in W_hid W_out c (in the layouts of p0 .. p3: W̄_hid packs the M − 1 matrices
 * like W_hid, c̄ every bias like c; a c̄ request with c == NULL returns B2B_EINVAL); COUPLING_DEEP_MLP_RQS W_in W_hid
 * W_out c the same way (W̄_out ((3K−1)·n1 x H) column-major like W_out);
 * SCALE_MATRIX a (Ā, D x D column-major like A: G + (Σ l̄)·A⁻ᵀ, or −A⁻ᵀ G A⁻ᵀ − (Σ l̄)·A⁻ᵀ for the inverse layer, with
 * G = Σₙ ȳₙ uₙᵀ over the layer's inputs u; slots 1-3 return B2B_EUNSUPPORTED);
 * SCALE_TRIANGULAR a (T̄, D x D column-major like T: the dense Ā projected on the triangle 𝒫 that T's parameters occupy --
 * strictly below / above the diagonal for the unit forms, the diagonal included otherwise -- and exactly 0 outside 𝒫:
 * 𝒫(G) + (Σ l̄)·diag(1/Tᵢᵢ), or −𝒫(T⁻ᵀ G T⁻ᵀ) − (Σ l̄)·diag(1/Tᵢᵢ) for the inverse layer, no diagonal term for the unit
 * forms; slots 1-3 return B2B_EUNSUPPORTED);
 * SCALE_LU a (F̄, D x D column-major and packed like F: with M̄ = G for the forward layer or −M⁻ᵀ G M⁻ᵀ for the inverse
 * one, M = P·L·U, the strict lower triangle is L̄ = 𝒮(Pᵀ M̄ Uᵀ) and the upper one with the diagonal is
 * Ū = 𝒰(Lᵀ Pᵀ M̄) + (Σ l̄)·diag(1/Uᵢᵢ), − (Σ l̄)·diag(1/Uᵢᵢ) for the inverse layer; the permutation has no cotangent;
 * slots 1-3 return B2B_EUNSUPPORTED);
 * AUTOREGRESSIVE_MLP W₁ c₁ W₂ c₂ (column-major like the parameters, the W̄ entries outside the masks exactly 0; a c̄₁ /
 * c̄₂ request whose c is NULL returns B2B_EINVAL);
 * ELEMENTWISE_VEC a (ā[D], Σₙ of ḡ·∂y/∂a + l̄·∂ℓ/∂a at the layer's output cotangent ḡ; slots 1-3 return
 * B2B_EUNSUPPORTED); BATCHNORM b logs; MVNORMAL_DIAG μ σ (only where the parameter pointer is non-NULL, else B2B_EINVAL); MVNORMAL_TRIL μ
 * (B2B_EINVAL when p0 is NULL) and L (D x D column-major, its upper triangle exactly zero).  Any other non-NULL entry
 * (BatchNorm m / v, PERMUTE, STACKED_EW, MVNORMAL_TRIL slots 2-3) returns B2B_EUNSUPPORTED.
 * The chain is cut into segments that existing kernels differentiate -- planar runs of one direction (<= 8 layers; D not
 * in {32, 64, 128} is embedded in the next of them with zero rows), radial runs (<= 8), single RQS / coupling / spline coupling /
 * dense Scale (factor, x̄ by the transposed map, G over column chunks, an fp64 finalize; workspace: the factor of
 * b2b_chain_run_f32 plus P·D² floats, P <= 64 chunks, and 2·D² + 1 doubles) / triangular Scale (the prep launch, x̄ by
 * the transposed triangular map; with T̄ requested G over column chunks -- on 𝒫 only, by the lower-triangle tiles, for the
 * forward layer -- Σ l̄, and a masked fp64 finalize: 3 launches more for the forward layer, 5 for the inverse; workspace:
 * its factor storage of b2b_chain_run_f32 plus P·D² floats and 2·D² + 1 doubles, each part rounded up to 256 bytes) /
 * LU Scale (the prep launch, x̄ by the transposed dense map; with F̄ requested G over column chunks, Σ l̄, the dense
 * finalize into an fp64 M̄ and one launch taking M̄ through the factors: 4 launches more for the forward layer, 6 for the
 * inverse; workspace as for the triangular Scale) /
 * eval-BatchNorm layers -- and runs of <= 8 STACKED_EW / ELEMENTWISE_VEC / PERMUTE layers (with the terminal MvNormal),
 * which one kernel differentiates (with ā requested, a second instantiation that also sweeps the run backwards, plus
 * G·V·D floats of per-CTA partials for the V ELEMENTWISE_VEC layers of the run, G <= 8 per SM); a terminal MVNORMAL_TRIL is a segment of its own (D <= 256).  It writes x̄ = ȳ − l̄·L⁻ᵀL⁻¹(x − μ) in one
 * launch; with μ̄ / L̄ requested it also stores r = L⁻¹(x − μ) and l̄·L⁻ᵀr (2·D·N floats of workspace), and two more
 * launches form L̄ = tril(Σ l̄ s rᵀ) over at most 64 column chunks (P·D·(D+1) floats of chunk partials, P = min(ceil(N /
 * 4096), 64)) and reduce the chunks in order.  The forward is recomputed once to checkpoint each segment's input, then the segments are
 * differentiated last to first.  Limits are the kernels': planar and radial D <= 128, RQS D <= 256 and K1 <= 64, coupling
 * n1, n2 <= 128 and D <= 747 at n1 = n2 = 128 (see b2b_coupling_affine_vjp_f32), BatchNorm and elementwise runs D <= 1024,
 * and the forward recompute those of b2b_chain_run_f32; an unsupported chain returns B2B_EUNSUPPORTED before anything
 * is launched.  N == 0 zeroes the requested parameter
 * cotangents.  Launch-only on `stream`, no allocation (CUDA-graph capturable).  workspace: b2b_chain_vjp_workspace_bytes
 * (0 = unsupported chain); b2b_last_launch_count counts every kernel, copy and fill enqueued. */
size_t b2b_chain_vjp_workspace_bytes(const b2b_layer_desc* layers, int32_t L, int32_t D, int64_t N);
int b2b_chain_vjp_f32(const b2b_layer_desc* layers, int32_t L, const float* x, const float* ybar, const float* ljbar,
                      float* xbar, float* const* param_bars, int32_t D, int64_t N, int64_t ldx, int64_t ldybar,
                      int64_t ldxbar, void* workspace, size_t workspace_bytes, void* stream);
/* RadialLayer: radial_layer.jl:58-72 (fwd), :88-102,124-129 (inverse) */
int b2b_radial_fwd_f32(const float* x, float* y, float* logjac, const float* alpha_raw,
                       const float* beta, const float* z0, int32_t D, int64_t N, int64_t ldx,
                       int64_t ldy, int accumulate_logjac, void* stream);
int b2b_radial_inv_f32(const float* x, float* y, float* logjac, const float* alpha_raw,
                       const float* beta, const float* z0, int32_t D, int64_t N, int64_t ldx,
                       int64_t ldy, int accumulate_logjac, void* stream);
/* RationalQuadraticSpline: rational_quadratic_spline.jl:317-357 (fwd), :183-220 (inverse) */
int b2b_rqs_fwd_f32(const float* x, float* y, float* logjac, const float* widths,
                    const float* heights, const float* derivs, int32_t K1, int32_t D, int64_t N,
                    int64_t ldx, int64_t ldy, int accumulate_logjac, void* stream);
int b2b_rqs_inv_f32(const float* x, float* y, float* logjac, const float* widths,
                    const float* heights, const float* derivs, int32_t K1, int32_t D, int64_t N,
                    int64_t ldx, int64_t ldy, int accumulate_logjac, void* stream);
/* Coupling with the affine law: coupling.jl:206-215 (fwd), :217-228 (inverse).
 * row1 / row2: first row of idx1 / idx2 when the list is a contiguous range (pointer may then be NULL), else -1.
 * workspace: b2b_coupling_workspace_bytes(n1, n2) bytes, 1024-byte aligned, enables the tensor-core path
 * (may be NULL: the exact-fp32 CUDA-core kernel is used). */
int b2b_coupling_affine_fwd_f32(const float* x, float* y, float* logjac, const int32_t* idx1, int32_t n1,
                                int32_t row1, const int32_t* idx2, int32_t n2, int32_t row2, const float* W,
                                const float* c, int32_t D, int64_t N, int64_t ldx, int64_t ldy,
                                int accumulate_logjac, void* workspace, size_t workspace_bytes, void* stream);
int b2b_coupling_affine_inv_f32(const float* x, float* y, float* logjac, const int32_t* idx1, int32_t n1,
                                int32_t row1, const int32_t* idx2, int32_t n2, int32_t row2, const float* W,
                                const float* c, int32_t D, int64_t N, int64_t ldx, int64_t ldy,
                                int accumulate_logjac, void* workspace, size_t workspace_bytes, void* stream);
size_t b2b_coupling_workspace_bytes(int32_t n1, int32_t n2);
/* InvertibleBatchNorm, eval mode: normalise.jl:61-67 (fwd), :74-86 (inverse) */
int b2b_batchnorm_eval_fwd_f32(const float* x, float* y, float* logjac, const float* b,
                               const float* logs, const float* m, const float* v, float eps,
                               int32_t D, int64_t N, int64_t ldx, int64_t ldy, int accumulate_logjac,
                               void* stream);
int b2b_batchnorm_eval_inv_f32(const float* x, float* y, float* logjac, const float* b,
                               const float* logs, const float* m, const float* v, float eps,
                               int32_t D, int64_t N, int64_t ldx, int64_t ldy, int accumulate_logjac,
                               void* stream);
/* InvertibleBatchNorm, TRAINING mode: normalise.jl:51-60 (the reference's global istraining() switch is this
 * separate entry point).  Batch mean / variance over the N columns -- over ALL ranks when comm != NULL, which costs
 * one all-reduce of 2D+1 doubles -- then the moving statistics m, v are updated IN PLACE (momentum mtm, n/(n-1)
 * correction) and y / logjac are computed with the batch statistics.  workspace: b2b_batchnorm_train_workspace_bytes(D). */
int b2b_batchnorm_train_fwd_f32(const float* x, float* y, float* logjac, const float* b, const float* logs,
                                float* m, float* v, float eps, float mtm, int32_t D, int64_t N, int64_t ldx,
                                int64_t ldy, int accumulate_logjac, struct b2b_comm* comm, void* workspace,
                                size_t workspace_bytes, void* stream);
size_t b2b_batchnorm_train_workspace_bytes(int32_t D);
/* Reverse mode of the TRAINING-mode InvertibleBatchNorm (normalise.jl:51-67 with istraining() == true): y and logjac
 * depend on the batch statistics, so the cotangents reach every column through m and v.  With n the number of columns
 * over all ranks, m, v the batch statistics exactly as b2b_batchnorm_train_fwd_f32 computes them on the same x, device and
 * communicator (bit-identical), σ² = v + eps, A = exp(logs)/σ and the global sums S1 = Σȳ, S2 = Σȳ(x − m), L̄ = Σl̄:
 *   x̄ = A ȳ − A S1/n − (x − m)(A S2 + L̄)/(n σ²),   b̄ = S1,   l̄ogs = A S2 + L̄.
 * `x` (D x N, the batch the forward saw), `xbar` and `logs` are required; `ybar` (D x N) and `ljbar` (N) may be NULL
 * (zeros).  `xbar` may be exactly `ybar` (same pointer and leading dimension); any other overlap of `xbar` with `x` or
 * `ybar` returns B2B_EINVAL.  `bbar` and `logsbar` (D each) are both given or both NULL (one alone: B2B_EINVAL).
 * Sharded batch (comm != NULL): x̄ uses the global statistics and sums -- one all-reduce of 4D+2 doubles -- while `bbar`
 * and `logsbar` are summed over THIS rank's columns only, like every other parameter cotangent of the library: a
 * data-parallel caller all-reduces them with the rest of its gradient.  The moving statistics are not touched (they have
 * no cotangent, and the function takes no pointer to them).  N < 2 (local) returns B2B_EINVAL, D > 1024
 * B2B_EUNSUPPORTED with nothing launched, as for the forward.  Deterministic (fixed-order fp64 sums, no atomics),
 * launch-only on `stream`, no allocation (CUDA-graph capturable).
 * workspace: b2b_batchnorm_train_vjp_workspace_bytes(D) (0 when D < 1 or D > 1024; independent of N). */
size_t b2b_batchnorm_train_vjp_workspace_bytes(int32_t D);
int b2b_batchnorm_train_vjp_f32(const float* x, const float* ybar, const float* ljbar, float* xbar, float* bbar,
                                float* logsbar, const float* logs, float eps, int32_t D, int64_t N, int64_t ldx,
                                int64_t ldybar, int64_t ldxbar, struct b2b_comm* comm, void* workspace,
                                size_t workspace_bytes, void* stream);
/* Permute rows (also serves PartitionMask / Stacked range movement): permute.jl:152-155. Bit-exact. */
int b2b_permute_rows_f32(const float* x, float* y, float* logjac, const int32_t* dst_of_src,
                         int inverse, int32_t D, int64_t N, int64_t ldx, int64_t ldy,
                         int accumulate_logjac, void* stream);
/* Stacked of elementwise laws on rows: stacked.jl:157-166,242-252 */
int b2b_stacked_elementwise_f32(const float* x, float* y, float* logjac, const int32_t* code,
                                const float* a, const float* b, int inverse, int32_t D, int64_t N, int64_t ldx,
                                int64_t ldy, int accumulate_logjac, void* stream);
/* logpdf(MvNormal(mu, Diagonal(sigma.^2)), x) + logjac_in  (Distributions/PDMats);
 * logpdf_out may alias logjac_in; sum_out (device double) optional; workspace as for chains. */
int b2b_mvnormal_diag_logpdf_f32(const float* x, const float* mu, const float* sigma,
                                 const float* logjac_in, float* logpdf_out, double* sum_out,
                                 int32_t D, int64_t N, int64_t ldx, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* ---- Float64 batches -------------------------------------------------------------------------------------------------
 * The reference is generic in its element type and its own tests run in Float64 (test/normalising_flows.jl:47-71 checks
 * find_alpha to 1e-14).  b2b_chain_run_f64 evaluates the same chains -- every layer kind but B2B_COUPLING_RQS,
 * B2B_COUPLING_MLP, B2B_COUPLING_MLP_RQS, B2B_COUPLING_DEEP_MLP, B2B_COUPLING_DEEP_MLP_RQS and B2B_AUTOREGRESSIVE_MLP
 * (Float32 only: the Float64
 * entry points and workspace
 * queries refuse them with B2B_EUNSUPPORTED / 0),
 * both directions, the terminal
 * MvNormal, the deterministic batch sum -- on D x N Float64 batches with Float64 parameters (b2b_layer_desc_f64: the
 * same fields with double pointers).  It is a straightforward double-precision restatement (one warp per column), NOT a
 * tuned kernel: Float64 is a correctness path, Float32 the hot path.  workspace: b2b_chain_workspace_bytes_f64.
 * b2b_chain_vjp_f64 is its reverse mode. */
typedef struct b2b_layer_desc_f64 {
  int32_t kind;
  int32_t inverse;
  int32_t n0, n1, n2, n3;
  double f0, f1;
  const double* p0;
  const double* p1;
  const double* p2;
  const double* p3;
  const int32_t* i0;
  const int32_t* i1;
} b2b_layer_desc_f64;
size_t b2b_chain_workspace_bytes_f64(int32_t L, int want_sum);
int b2b_chain_run_f64(const b2b_layer_desc_f64* layers, int32_t L, const double* x, double* y, double* logjac,
                      double* sum_out, int32_t D, int64_t N, int64_t ldx, int64_t ldy, int accumulate_logjac,
                      void* workspace, size_t workspace_bytes, void* stream);
/* Reverse mode of b2b_chain_run_f64: the contract of b2b_chain_vjp_f32 with double everywhere.  Any chain
 * b2b_chain_run_f64 accepts (every kind, either direction, mixed, L <= B2B_MAX_CHAIN, D <= 2048, optionally ending in
 * the terminal B2B_MVNORMAL_DIAG or B2B_MVNORMAL_TRIL, whose logjac output is then logpdf).  `xbar` (D x N, required) must not overlap `x` or
 * `ybar` (B2B_EINVAL); NULL `ybar` / `ljbar` are zeros; `param_bars` (NULL = x̄ only) holds 4*L pointers, entry 4l+i the
 * cotangent of layers[l].p<i> in its shape and layout, summed over the N columns.  Trainable slots as for Float32: PLANAR
 * w u b; RADIAL α_ β z_0 (raw, through log1pexp); RQS widths heights derivatives (processed); COUPLING W c; ELEMENTWISE_VEC
 * a; SCALE_TRIANGULAR a (T̄, zero outside 𝒫); SCALE_LU a (F̄, packed like F); BATCHNORM b logs; MVNORMAL_DIAG μ σ (only where the parameter pointer is non-NULL, else B2B_EINVAL); MVNORMAL_TRIL μ (B2B_EINVAL when
 * p0 is NULL) and L (D x D column-major, exactly zero above the diagonal); any other non-NULL entry returns
 * B2B_EUNSUPPORTED.  D > 2048 returns B2B_EUNSUPPORTED with nothing launched.  N == 0 zeroes the requested
 * parameter cotangents.  One warp per column recomputes the forward with the arithmetic of b2b_chain_run_f64, keeping
 * each layer's input in a tape, then differentiates the layers last to first; parameter cotangents accumulate in
 * per-warp slots that a second kernel sums in a fixed order (deterministic, no atomics) and a third turns into the
 * caller's arrays.  Launch-only on `stream`, no allocation (CUDA-graph capturable); b2b_last_launch_count counts the
 * kernels and fills enqueued (1, or 3 with parameter cotangents).
 * Workspace (b2b_chain_vjp_workspace_bytes_f64; 0 exactly when the call refuses the chain) is bounded independently of N:
 * W warp slots of 8·(T + P) bytes plus 8·P, with T = Lf·D (Lf: layers before the MvNormal) and P the accumulators, per
 * layer PLANAR 2D+2, RADIAL D+2, RQS 3·D·K1, COUPLING 2n1·n2 + 2n1, ELEMENTWISE_VEC D, BATCHNORM / MVNORMAL_DIAG 2D, MVNORMAL_TRIL
 * D + D(D+1)/2 (μ̄ and the packed lower triangle of L̄), SCALE_TRIANGULAR D(D+1)/2 (T̄'s packed triangle), SCALE_LU D² (F̄) doubles (each rounded up to 32); W = min(ceil(N / w), 528) CTAs of w warps (w = 4, or 3 for D > 1816), lowered so that the slots stay within
 * 256 MiB but never below one CTA -- so the bound exceeds 256 MiB only when one CTA's slots do (e.g. wide couplings with
 * 2n1·n2 in the millions).  The number of warps, and with it the summation order, depends only on the chain, D and N. */
size_t b2b_chain_vjp_workspace_bytes_f64(const b2b_layer_desc_f64* layers, int32_t L, int32_t D, int64_t N);
int b2b_chain_vjp_f64(const b2b_layer_desc_f64* layers, int32_t L, const double* x, const double* ybar,
                      const double* ljbar, double* xbar, double* const* param_bars, int32_t D, int64_t N,
                      int64_t ldx, int64_t ldybar, int64_t ldxbar, void* workspace, size_t workspace_bytes,
                      void* stream);

/* ---- sampling: rand(rng, td, n) (src/transformed_distribution.jl:212-224) -----------------------------------------
 * Base samples z ~ N(0, I) come from Philox4x32-10 (the counter-based generator of Random123 / cuRAND) + Box-Muller and
 * are generated INSIDE the kernel: the four normals of rows 4k..4k+3 of GLOBAL column n = column_offset + local column
 * use the counter (lo32(n), hi32(n), k, lo32(offset)) under the key (lo32(seed), hi32(seed)), so a sample depends only
 * on (seed, offset, n, row) -- column shards on different ranks draw disjoint parts of ONE stream, and a re-run with the
 * same arguments is bit-identical.  x = mu + sigma .* z (NULL = 0 / 1) is MvNormal(mu, Diagonal(sigma.^2)).
 * b2b_chain_sample_f32 pushes the samples through layers[0..L) in the forward direction (L = 0: the base samples);
 * `logjac` (optional) receives log|det J| of the chain at each sample.  Column-local chains with D in {32,64,128,256}
 * run as ONE launch whose only HBM traffic is the D x N store; other chains take two passes (b2b_randn_f32 into y, then
 * the chain in place; workspace as for b2b_chain_run_f32). */
int b2b_randn_f32(float* z, const float* mu, const float* sigma, uint64_t seed, uint64_t offset, int64_t column_offset,
                  int32_t D, int64_t N, int64_t ld, void* stream);
int b2b_chain_sample_f32(const b2b_layer_desc* layers, int32_t L, const float* mu, const float* sigma, uint64_t seed,
                         uint64_t offset, int64_t column_offset, float* y, float* logjac, int32_t D, int64_t N,
                         int64_t ldy, void* workspace, size_t workspace_bytes, void* stream);
/* rand(td, n) for the base MvNormal(mu, L Lᵀ) (B2B_MVNORMAL_TRIL): y = mu + L z (PDMats' unwhiten), z the SAME stream
 * b2b_randn_f32 draws for (seed, offset, global column, row) with mu = sigma = NULL, then layers[0..L) applied in place
 * (two passes; L = 0 returns the base samples and zeroes `logjac` when given).  `scale_tril` (D x D column-major, lower
 * triangle read) is required; `mu` may be NULL.  D <= 256 (B2B_EUNSUPPORTED beyond, nothing launched); a chain
 * b2b_chain_run_f32 refuses is refused before anything is launched.  workspace as for b2b_chain_run_f32 on the chain. */
int b2b_chain_sample_tril_f32(const b2b_layer_desc* layers, int32_t L, const float* mu, const float* scale_tril,
                              uint64_t seed, uint64_t offset, int64_t column_offset, float* y, float* logjac, int32_t D,
                              int64_t N, int64_t ldy, void* workspace, size_t workspace_bytes, void* stream);
/* ---- reparameterised sampling: rand(td, n) with log q, and its reverse mode (variational inference, the ELBO) ------
 * `base` is a descriptor of kind B2B_MVNORMAL_DIAG (p0 = mu or NULL, p1 = sigma or NULL) or B2B_MVNORMAL_TRIL (p0 = mu or
 * NULL, p1 = L, D x D column-major, lower triangle read), inverse == 0.  With z the stream of b2b_randn_f32 for (seed,
 * offset, global column, row), x = mu + sigma .* z or mu + L z, y = T(x) through layers[0..L) in the forward direction and
 * ℓ(x) its log|det J|, the samples' log-density is
 *   log q(y) = −½‖z‖² − Σᵢ log sigmaᵢ (or log Lᵢᵢ) − ½·D·log2π − ℓ(x).
 * b2b_chain_sample_logq_f32 writes y bit-identical to b2b_chain_sample_f32 / b2b_chain_sample_tril_f32 for the same
 * arguments, and log q (N floats) to `logq`.  A chain b2b_chain_sample_f32 runs as one launch stays one launch (‖z‖² is
 * summed while z is generated, the store is still 4·(D+1) B/sample); a two-pass chain adds one pass over the N floats of
 * logq (the diagonal base regenerates z per column; the TRIL sample launch emits the base term itself).
 * b2b_chain_sample_vjp_f32 is its reverse mode with z held fixed (the reparameterisation gradient): `ybar` (D x N,
 * leading dimension ldybar) and `lqbar` (N) are the cotangents of y and log q, NULL = zeros.  `param_bars` is NULL or
 * 4·(L+1) pointers: entries 0 .. 4L−1 as in b2b_chain_vjp_f32 (same slots, layouts and rules), entries 4L .. 4L+3 the base's:
 * μ̄ and σ̄ (DIAG; a request whose parameter is NULL returns B2B_EINVAL) or μ̄ (B2B_EINVAL when p0 is NULL) and L̄ (D x D
 * column-major, exactly zero above the diagonal); slots 4L+2, 4L+3 return B2B_EUNSUPPORTED.
 *   x̄ = b2b_chain_vjp_f32 at x with ybar and l̄ = −lqbar,   μ̄ = Σₙ x̄ₙ,
 *   σ̄ = Σₙ x̄ₙ ⊙ zₙ − (Σₙ q̄ₙ)/σ,   L̄ = tril(Σₙ x̄ₙ zₙᵀ) − (Σₙ q̄ₙ)·diag(1/Lᵢᵢ).
 * x (and for TRIL z) is regenerated into the workspace; every cotangent is summed over this call's N columns in a fixed
 * order (deterministic, no atomics): column shards pass their first global column as column_offset and all-reduce the
 * cotangents like any other.  N == 0 zeroes the requested cotangents.
 * Refusals, before anything is launched: a chain b2b_chain_vjp_f32 refuses (its status), a chain holding an MvNormal
 * terminal or a base of another kind (B2B_EINVAL), a TRIL base with D > 256 (B2B_EUNSUPPORTED).  Float32 only.
 * Launch-only on `stream`, no allocation (CUDA-graph capturable); both set b2b_last_launch_count.  The workspace queries
 * return 0 exactly when their call refuses the input, and depend on nothing else. */
size_t b2b_chain_sample_logq_workspace_bytes(const b2b_layer_desc* layers, int32_t L, const b2b_layer_desc* base,
                                             int32_t D, int64_t N);
int b2b_chain_sample_logq_f32(const b2b_layer_desc* layers, int32_t L, const b2b_layer_desc* base, uint64_t seed,
                              uint64_t offset, int64_t column_offset, float* y, float* logq, int32_t D, int64_t N,
                              int64_t ldy, void* workspace, size_t workspace_bytes, void* stream);
size_t b2b_chain_sample_vjp_workspace_bytes(const b2b_layer_desc* layers, int32_t L, const b2b_layer_desc* base,
                                            int32_t D, int64_t N);
int b2b_chain_sample_vjp_f32(const b2b_layer_desc* layers, int32_t L, const b2b_layer_desc* base, uint64_t seed,
                             uint64_t offset, int64_t column_offset, const float* ybar, int64_t ldybar,
                             const float* lqbar, float* const* param_bars, int32_t D, int64_t N, void* workspace,
                             size_t workspace_bytes, void* stream);

/* ---- host-buffer entry point (what a caller holding plain host Arrays uses; the bench's `e2e`) ----
 * Streams the batch through the device in column chunks: H2D copy, chain kernels and D2H copy of
 * successive chunks overlap on `n_streams` streams.  x_host / y_host / logjac_host are HOST pointers
 * (pinned memory gives full PCIe bandwidth; pageable memory works but is slower); layer parameter
 * pointers inside `layers` stay DEVICE pointers.  Synchronises before returning.
 */
typedef struct b2b_host_ctx b2b_host_ctx;
int b2b_host_ctx_create(b2b_host_ctx** ctx, int32_t D_max, int64_t chunk_cols, int32_t n_streams);
int b2b_host_ctx_destroy(b2b_host_ctx* ctx);
/* Orders the ctx's internal streams after the work enqueued so far on `stream` (parameters written on the caller's
 * stream -- an optimiser step -- are then visible to the next b2b_chain_run_host_f32). */
int b2b_host_ctx_wait_stream(b2b_host_ctx* ctx, void* stream);
int b2b_chain_run_host_f32(b2b_host_ctx* ctx, const b2b_layer_desc* layers, int32_t L,
                           const float* x_host, float* y_host, float* logjac_host, double* sum_host,
                           int32_t D, int64_t N);
/* cudaHostRegister / cudaHostUnregister passthroughs so a host runtime can pin its own arrays */
int b2b_host_register(void* ptr, size_t bytes);
int b2b_host_unregister(void* ptr);
/* Binds the CALLING THREAD (CPU affinity + preferred memory node) to the NUMA node of CUDA device `device`, so that
 * pinned host buffers allocated afterwards live on the socket whose PCIe root complex serves that GPU (on the 2-socket
 * HGX hosts a remote-socket buffer sends every H2D / D2H byte across the inter-socket link).  One process per GPU calls
 * it once before allocating its host batches.  Best effort: *node_out = -1 when the topology is not exposed
 * (/sys/bus/pci/devices/<bus id>/numa_node); *ncpus_out = CPUs in the new affinity mask.  Linux only. */
int b2b_numa_bind_to_device(int32_t device, int32_t* node_out, int32_t* ncpus_out);
/* NUMA node of the PCIe root complex that serves CUDA device `device` (-1 when not exposed).  A launcher that starts
 * fewer ranks than the box has GPUs can use it to spread the ranks over the sockets: the host-buffer path is bound by
 * host DRAM bandwidth per socket. */
int b2b_device_numa_node(int32_t device, int32_t* node_out);

/* ---- multi-GPU: the ONE collective of the path (SURVEY §8(e)) -----------------------------------
 * Columns shard across ranks with no data-path collective; the batch log-density Σ_n logpdf[n] is
 * summed across ranks with a single ncclAllReduce(sum) of one double.  NCCL is loaded with
 * dlopen("libnccl.so.2") so the library has no link-time NCCL dependency.
 */
typedef struct b2b_comm b2b_comm;
int b2b_comm_unique_id(char id_out[128]);
int b2b_comm_init_rank(b2b_comm** comm, int nranks, int rank, const char id[128]);
int b2b_allreduce_sum_f64(b2b_comm* comm, double* dev_values, int32_t count, void* stream);
/* ONE process driving several GPUs (e.g. a single Julia session that holds all 8 devices): a clique of `ndev`
 * communicators over the CUDA devices devs[0..ndev) (NULL = 0..ndev-1) made with ncclCommInitAll, and the sum issued for
 * all of them inside one NCCL group: dev_values[i] (a device pointer on devs[i], `count` doubles, reduced in place) and
 * streams[i] belong to devs[i]. */
int b2b_comm_init_all(b2b_comm** comm, int ndev, const int* devs);
int b2b_allreduce_sum_f64_all(b2b_comm* comm, double* const* dev_values, int32_t count, void* const* streams);
int b2b_comm_destroy(b2b_comm* comm);

#ifdef __cplusplus
}
#endif
#endif /* B2B_H_ */
