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
 * If the last element is B2B_MVNORMAL_DIAG, `logjac` receives logpdf[n] = logpdf(MvNormal)(x_n) +
 * accumulated logjac (transformed_distribution.jl:165-169 when the preceding layers are the inverse
 * chain) and, when sum_out != NULL, *sum_out (device double) receives Σ_n logpdf[n] (fixed summation
 * order, deterministic).
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
 * points that are not chain elements. */
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
 * scatter of the three cotangent blocks.  `layer`: a B2B_COUPLING_AFFINE descriptor (n1, n2 <= 128, any index lists);
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
 * find_alpha to 1e-14).  b2b_chain_run_f64 evaluates the same chains -- every layer kind, both directions, the terminal
 * MvNormal, the deterministic batch sum -- on D x N Float64 batches with Float64 parameters (b2b_layer_desc_f64: the
 * same fields with double pointers).  It is a straightforward double-precision restatement (one warp per column), NOT a
 * tuned kernel: Float64 is a correctness path, Float32 the hot path.  workspace: b2b_chain_workspace_bytes_f64. */
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
