// Internal declarations shared by the translation units of libb2b.so (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b2b.h"

// Kernel argument block of the fused column-local chain kernels (passed by value, < 4 KB).
struct B2BChainParams {
  const float* x;
  float* y;          // may be NULL (no D x N store)
  float* logjac;     // N (or logpdf when the chain ends in MVNORMAL_DIAG); may be NULL
  double* partials;  // per-CTA partial sums of the last op's output (NULL unless a batch sum is wanted)
  long long N, ldx, ldy;
  int D, L, accumulate;
  int scratch_off;  // float offset of the per-warp permute scratch in dynamic smem, -1 if unused
  int soff[B2B_MAX_CHAIN];  // float offset of layer l's staged parameters in dynamic smem
  b2b_layer_desc layers[B2B_MAX_CHAIN];
};

#ifdef __CUDACC__
// Element-wise float2 arithmetic of the paired-column kernels.  sm_90 has no packed FP32 instruction, so each is two
// scalar operations; the _rn intrinsics keep every product and sum individually rounded (no contraction).
__device__ __forceinline__ float2 b2b_ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 b2b_fadd2(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 b2b_fmul2(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
#endif

// number of floats of staged (derived) parameters a layer needs for padded depth Dp
static inline int b2b_layer_smem_floats(const b2b_layer_desc& d, int Dp) {
  switch (d.kind) {
    case B2B_PLANAR: return 2 * Dp + 4;
    case B2B_RADIAL: return Dp + 4;
    case B2B_BATCHNORM: return 4 * Dp + 4;
    case B2B_RQS: {
      int kp = 2;
      while (kp < d.n0) kp <<= 1;  // knots padded to a power of two (rqs_kp)
      return (2 * kp + 8 * d.n0) * Dp;
    }
    case B2B_PERMUTE: return Dp;
    case B2B_STACKED_EW:
    case B2B_ELEMENTWISE_VEC: return 3 * Dp;  // staged as the STACKED_EW table
    case B2B_MVNORMAL_DIAG: return 2 * Dp + 4;
    default: return 0;
  }
}

// ---- launchers (each returns a cudaError_t as int, or a negative B2B_E* code) ---------------------
// v0: lane-group direct-global fused interpreter (any D <= 1024 whose staged parameters fit B2B_V0_SMEM_MAX)
int b2b_launch_chain_v0(const B2BChainParams& p, cudaStream_t stream);
// Dynamic shared memory v0 stages for the fused run layers[0..L) at D (SIZE_MAX when D is out of range).  Every other
// fused kernel stages at least as much for the runs it accepts, so a run within B2B_V0_SMEM_MAX always has a kernel:
// the chain orchestrator ends a fused segment before the layer that would cross the budget.
#define B2B_V0_SMEM_MAX (200 * 1024)
size_t b2b_chain_v0_smem_bytes(const b2b_layer_desc* layers, int L, int D);
// Launch segments b2b_chain_run_f32 cuts a chain into (before BatchNorm neighbours are folded into coupling launches), or
// a negative B2B_E* code when a layer fits no kernel.  With y == NULL a chain of more than one segment needs a D x N
// intermediate between them (b2b_api.cu).
int b2b_chain_segment_count(const b2b_layer_desc* layers, int32_t L, int32_t D);
// v1: TMA-staged thread-per-column fused interpreter (D in {32,64,128}); returns B2B_EUNSUPPORTED otherwise
int b2b_launch_chain_v1(const B2BChainParams& p, cudaStream_t stream);
// fused planar chains (b2b_planar_const.cu).  hostparams: `L` in 1..8 layers, derived parameters packed
// w[L][D] | û[L][D] | c[L] | b[L] in HOST memory, bit l of invmask = inverse of layer l.
int b2b_launch_planar_hostparams(const B2BChainParams& p, int L, const float* packed, int invmask,
                                 cudaStream_t stream);
// device-resident parameters: p.layers must be 1..8 PLANAR layers; B2B_EUNSUPPORTED when not applicable
int b2b_launch_planar_chain_const(const B2BChainParams& p, cudaStream_t stream);
int b2b_planar_const_grid_size(const B2BChainParams& p);
// number of planar layers when the fused planar chain kernel applies to the segment `p`, else 0
int b2b_planar_const_layers(const B2BChainParams& p);
// reverse mode of a forward radial chain (b2b_radial_vjp.cu)
size_t b2b_radial_vjp_workspace(int L, int D);
// 1..8 radial layers of one direction as a specialised program (b2b_radial_unrolled.cu)
int b2b_radial_unrolled_applicable(const B2BChainParams& p);
int b2b_launch_radial_unrolled(const B2BChainParams& p, cudaStream_t stream);
// a single RQS layer with 9 knots as a specialised program (b2b_rqs_unrolled.cu)
int b2b_rqs_unrolled_applicable(const B2BChainParams& p);
int b2b_launch_rqs_unrolled(const B2BChainParams& p, cudaStream_t stream);
// reverse mode of a forward planar chain (b2b_planar_vjp.cu)
size_t b2b_planar_vjp_workspace(int L, int D, long long N);
// reverse mode of one affine coupling layer (b2b_coupling_vjp.cu): whether its kernel takes the layer at D (n1, n2 <= 128
// and the D-row input / cotangent tiles within shared memory: D <= 747 at n1 = n2 = 128)
bool b2b_coupling_affine_vjp_fits(const b2b_layer_desc& d, int D);
// reverse mode of an elementwise run (b2b_ew_vjp.cu): <= 8 STACKED_EW / ELEMENTWISE_VEC / PERMUTE layers, optionally closed
// by the terminal MVNORMAL_DIAG.  ybar, ljbar may be NULL (zeros); mubar / sigmabar (D, or NULL) and the ā of the run's
// `vec_layers` ELEMENTWISE_VEC layers need b2b_ew_vjp_workspace(D, 1, vec_layers) bytes (0 for a run with neither).
size_t b2b_ew_vjp_workspace(int D, int want_mvn_params, int vec_layers);
// one launch copying up to 24 small device vectors: dst[k][0, len[k]) = src[k][0, len[k]), zero up to dst_len[k]
int b2b_launch_copy_list(int n, const float* const* src, float* const* dst, const int* len, const int* dst_len,
                         cudaStream_t stream);
// deterministic final sum of per-CTA partials into *sum_out
int b2b_launch_sum_partials(const double* partials, int n, double* sum_out, cudaStream_t stream);
// affine coupling, tensor-core path (B2B_EUNSUPPORTED when the shape / workspace does not fit)
size_t b2b_coupling_tc_workspace_bytes(int n1, int n2);
// `fold` (device, 4*D+1 floats, or NULL): folded BatchNorm neighbours, see bn_fold_prep_kernel
int b2b_launch_coupling_affine_tc(const b2b_layer_desc& d, const float* fold, const float* x, float* y,
                                  float* logjac, int D, long long N, long long ldx, long long ldy, int accumulate,
                                  void* workspace, size_t workspace_bytes, int* launches, cudaStream_t stream);
int b2b_launch_bn_fold_prep(const b2b_layer_desc* pre, const b2b_layer_desc* post, int D, float* out,
                            cudaStream_t stream);
// affine coupling, exact-fp32 CUDA-core kernel (any index lists; it stages the n1 + n2 rows it reads, so the limit is
// b2b_coupling_affine_fits, independent of D and N)
bool b2b_coupling_affine_fits(int n1, int n2, int D);
int b2b_launch_coupling_affine(const b2b_layer_desc& d, const float* fold, const float* x, float* y,
                               float* logjac, int D, long long N, long long ldx, long long ldy, int accumulate,
                               cudaStream_t stream);
// full-covariance MvNormal terminal (b2b_mvnormal_tril.cu).  Float32 stages the packed lower triangle of L in shared
// memory: D <= B2B_TRIL_MAX_D.
#define B2B_TRIL_MAX_D 256
// reverse mode: μ̄ / L̄ need b2b_tril_vjp_workspace(D, N) bytes
size_t b2b_tril_vjp_workspace(int D, long long N);
// Σₙ S[:, n] R[:, n]ᵀ over column chunks (b2b_mvnormal_tril.cu): CTA (tile, p) writes its 64 x 64 tile of chunk p's sum
// to part[p] (D x D, column-major; fp32 FMA within a chunk, which the caller sums over p in a fixed order).  `lower`:
// only the tiles on and below the diagonal, elements i >= j, and (when mup != NULL) chunk row sums of S to mup[p].
// b2b_outer_chunk_len(N) columns per chunk, at most 64 chunks.
long long b2b_outer_chunk_len(long long N);
int b2b_launch_outer_chunks(const float* S, long long lds, const float* R, long long ldr, float* part, float* mup, int D,
                            long long N, bool lower, cudaStream_t stream);
// dense, triangular and LU Scale (b2b_scale_matrix.cu), SCALE_MATRIX, SCALE_TRIANGULAR or SCALE_LU `kind` at D <= 256:
// the factor storage of its forward launches (0 beyond the envelope)
size_t b2b_scale_workspace(int kind, int D);
// reverse mode: b2b_scale_vjp_workspace(kind, D, N) bytes (0 beyond the envelope)
size_t b2b_scale_vjp_workspace(int kind, int D, long long N);
// masked autoregressive layer (b2b_autoregressive.cu): whether its kernels take `d` at D (the
// B2B_AUTOREGRESSIVE_MLP_MAX_* envelope), the masked-weight storage of its forward launches and the workspace of its
// reverse mode (0 outside the envelope; bounded independently of N)
bool b2b_ar_fits(const b2b_layer_desc& d, int D);
size_t b2b_ar_workspace(const b2b_layer_desc& d, int D);
size_t b2b_ar_vjp_workspace(const b2b_layer_desc& d, int D, long long N);
// spline coupling, reverse mode (b2b_coupling_rqs_vjp.cu): b2b_coupling_rqs_vjp_workspace(d, D, N) bytes (0 outside the
// envelope, bounded independently of N)
size_t b2b_coupling_rqs_vjp_workspace(const b2b_layer_desc& d, int D, long long N);
// neural-network coupling, reverse mode (b2b_coupling_mlp_vjp.cu): with any parameter cotangent
// b2b_coupling_mlp_vjp_workspace(d, D, N) bytes (0 outside the envelope, bounded independently of N) and two launches,
// else one launch and no workspace
size_t b2b_coupling_mlp_vjp_workspace(const b2b_layer_desc& d, int D, long long N);
// B2B_OK when b2b_chain_run_f32 accepts `layers` at D (every descriptor valid, every segment planned), else its status
int b2b_chain_check_f32(const b2b_layer_desc* layers, int32_t L, int32_t D);
// The one-launch form of rand (b2b_sample.cu), shared by b2b_chain_sample_f32 and b2b_chain_sample_logq_f32 (logq: `out`
// receives log q instead of ℓ): *launched = false, with nothing enqueued, when the chain does not fuse.
int b2b_launch_sample_fused(const b2b_layer_desc* layers, int L, const float* mu, const float* sigma, uint64_t seed,
                            uint64_t offset, int64_t column_offset, float* y, float* out, int D, long long N,
                            long long ldy, bool logq, bool* launched, cudaStream_t stream);
// B2B_OK when b2b_chain_vjp_f32 accepts `layers` at D (L >= 1), else the status it returns before launching anything
int b2b_chain_vjp_check_f32(const b2b_layer_desc* layers, int32_t L, int32_t D);
// The TRIL base of the reparameterised sampler (b2b_mvnormal_tril.cu, D <= B2B_TRIL_MAX_D).  b2b_tril_sample: y = μ + L z
// with z the b2b_randn_f32 stream, and with logq != NULL logq[n] = qsign·(−½·D·log2π − Σ log Lᵢᵢ − ½‖zₙ‖²), one launch.
// b2b_tril_base_vjp: μ̄ = Σ x̄ₙ and L̄ = tril(Σ x̄ₙ zₙᵀ) − (*qsum)·diag(1/Lᵢᵢ) (qsum NULL: 0) over the chunked GEMM and
// its ordered reduce, two launches; workspace b2b_tril_base_vjp_workspace(D, N) bytes.
int b2b_tril_sample(const float* Lg, const float* mu, uint64_t seed, uint64_t offset, long long col0, float* y,
                    long long ldy, float* logq, float qsign, int D, long long N, cudaStream_t stream);
size_t b2b_tril_base_vjp_workspace(int D, long long N);
int b2b_tril_base_vjp(const float* xbar, long long ldxb, const float* z, const double* qsum, const float* Lg,
                      float* mubar, float* Lbar, int D, long long N, void* workspace, int* launches,
                      cudaStream_t stream);
// Float64 chains (b2b_chain_f64.cu): B2B_OK when b2b_chain_run_f64 accepts descriptor `d` at D (`last`: the chain's final
// element, the only place a MVNORMAL_DIAG may stand), else B2B_EINVAL (B2B_EUNSUPPORTED for the Float32-only
// COUPLING_RQS, SCALE_MATRIX, COUPLING_MLP, COUPLING_MLP_RQS, COUPLING_DEEP_MLP and COUPLING_DEEP_MLP_RQS).
int b2b_f64_validate_layer(const b2b_layer_desc_f64& d, int D, bool last);
// Sets what b2b_last_launch_count reports for the calling thread (entry points outside b2b_api.cu).
void b2b_set_last_launch_count(int n);
// SMs of the current device, or 132 (an H100 SXM) when the query fails, as in a host-only workspace query
int b2b_sm_count();
// `workspace` rounded up to 256 bytes (the workspace sizes include 256 bytes of slack for it)
inline char* b2b_align256(void* workspace) {
  char* p = static_cast<char*>(workspace);
  return p + ((256 - (reinterpret_cast<uintptr_t>(p) & 255)) & 255);
}

// ---- forward segment launchers ---------------------------------------------------------------------------------------
// One launch segment of b2b_chain_run_f32: `n` layers of one B2BLaunchClass from x to y (NULL: not stored), adding their
// log-Jacobians to logjac (may be NULL).  The rules of the reverse-mode launchers below hold: the caller has validated
// the descriptors, the launcher checks what its kernels need, and it adds the launches it enqueued to *launches.
// pre / post: BatchNorm layers folded into a coupling launch through the table `fold`; partials (NULL: no batch sum):
// per-CTA sums of the fused or TRIL launch, added into *sum_out; workspace: the class's slice (W image, Scale factor).
struct B2BFwdSeg {
  const b2b_layer_desc* layers;
  int n;
  const float* x;
  long long ldx;
  float* y;
  long long ldy;
  float* logjac;
  int accumulate;
  int D;
  long long N;
  const b2b_layer_desc *pre, *post;
  float* fold;
  double* partials;
  double* sum_out;
  void* workspace;
  size_t workspace_bytes;
  int* launches;
  cudaStream_t stream;
};
int b2b_fwd_spline(const B2BFwdSeg& s);  // b2b_coupling_rqs.cu: COUPLING_RQS, _MLP_RQS and _DEEP_MLP_RQS
int b2b_fwd_mlp(const B2BFwdSeg& s);     // b2b_coupling_mlp.cu: COUPLING_MLP and COUPLING_DEEP_MLP
int b2b_fwd_scale(const B2BFwdSeg& s);   // b2b_scale_matrix.cu: SCALE_MATRIX, _TRIANGULAR, _LU; y == NULL: log-Jacobians only
int b2b_fwd_tril(const B2BFwdSeg& s);    // b2b_mvnormal_tril.cu: copies x to y (when y != x), writes logpdf to logjac
int b2b_fwd_ar(const B2BFwdSeg& s);      // b2b_autoregressive.cu: AUTOREGRESSIVE_MLP; workspace: its masked weights

// ---- reverse-mode segment launchers ----------------------------------------------------------------------------------
// One segment of b2b_chain_vjp_f32: `n` layers of one B2BVjpClass, their input x, the cotangent ȳ of their output, l̄ (N
// floats, NULL: zero) and x̄ (written).  bars[4j + i] receives the cotangent of slot i of layer j (NULL: not wanted).
// Every launcher works to the same rules:
//   - the caller has validated the descriptors against vjp_envelope, N > 0, and ȳ is non-NULL for the classes of
//     vjp_needs_ybar (b2b_api.cu);
//   - the launcher checks what its kernels need: alignment, overlap, workspace size;
//   - a cotangent its kernels always form but nobody asked for goes to `scratch` (seg_param_floats of b2b_api.cu);
//   - it adds the exact number of launches it enqueued to *launches.
// Planar and radial runs form their cotangents as whole arrays (w̄, ū n x D, b̄ n; ᾱ, β̄ n, z̄₀ n x D) in scratch and copy
// the requested slots out in one launch; with scratch == NULL the bars are those arrays themselves (bars[i] is array i).
struct B2BVjpSeg {
  const b2b_layer_desc* layers;
  int n;
  const float* x;
  long long ldx;
  const float* ybar;
  long long ldyb;
  const float* ljbar;
  float* xbar;
  long long ldxb;
  int D;
  long long N;
  float* const* bars;
  float* scratch;
  void* workspace;
  size_t workspace_bytes;
  int* launches;
  cudaStream_t stream;
};
int b2b_vjp_planar(const B2BVjpSeg& s);    // b2b_planar_vjp.cu: <= 8 layers of one direction, D in {32, 64, 128}
int b2b_vjp_radial(const B2BVjpSeg& s);    // b2b_radial_vjp.cu: <= 8 layers
int b2b_vjp_rqs(const B2BVjpSeg& s);       // b2b_rqs_vjp.cu
int b2b_vjp_coupling(const B2BVjpSeg& s);  // b2b_coupling_vjp.cu
int b2b_vjp_batchnorm(const B2BVjpSeg& s); // b2b_coupling_vjp.cu: eval mode
int b2b_vjp_ew(const B2BVjpSeg& s);        // b2b_ew_vjp.cu: <= 8 STACKED_EW / ELEMENTWISE_VEC / PERMUTE, optionally closed by MVNORMAL_DIAG
int b2b_vjp_tril(const B2BVjpSeg& s);      // b2b_mvnormal_tril.cu
int b2b_vjp_spline(const B2BVjpSeg& s);    // b2b_coupling_rqs_vjp.cu: COUPLING_RQS, _MLP_RQS and _DEEP_MLP_RQS
int b2b_vjp_scale(const B2BVjpSeg& s);     // b2b_scale_matrix.cu: SCALE_MATRIX, SCALE_TRIANGULAR, SCALE_LU
int b2b_vjp_mlp(const B2BVjpSeg& s);       // b2b_coupling_mlp_vjp.cu: COUPLING_MLP and COUPLING_DEEP_MLP
int b2b_vjp_ar(const B2BVjpSeg& s);        // b2b_autoregressive.cu: AUTOREGRESSIVE_MLP
// One launch copying slot i of layer j from base[i] + j·step[i] to bars[4j + i], for the requested slots of a run of
// n <= 8 layers at D (nothing is launched when none is requested).
int b2b_copy_run_bars(const b2b_layer_desc* layers, int n, float* const* bars, const float* const base[3],
                      const size_t step[3], int D, int* launches, cudaStream_t stream);

// ---- layer kinds ---------------------------------------------------------------------------------------------------
// What the chain orchestration knows about each kind of include/b2b.h.  A new kind enters the host code as one row of
// the table in b2b_kind, its limits in the envelope functions of b2b_api.cu, its slot lengths in b2b_slot_len, one
// B2BFwdSeg launcher plus one case of the forward switch in b2b_chain_run_f32, and for reverse mode one B2BVjpSeg
// launcher plus one case of the sweep's switch in b2b_chain_vjp_f32 (and its scratch and workspace sizes in
// seg_param_floats / seg_kernel_bytes).  A coupling instead gives its shape fields and the slot of each parameter role
// in b2b_coupling, which b2b_slot_len and the coupling launchers read, and a row of b2b_coupling_fits.

// Forward launch class: a run of fused column-local layers, or a launch of its own.
enum B2BLaunchClass { B2B_LC_FUSED, B2B_LC_COUPLING, B2B_LC_SPLINE, B2B_LC_SCALE, B2B_LC_TRIL, B2B_LC_MLP, B2B_LC_AR };
// Reverse-mode segment class of b2b_chain_vjp_f32 (B2B_VC_EW: runs of STACKED_EW / ELEMENTWISE_VEC / PERMUTE, with
// MVNORMAL_DIAG).
enum B2BVjpClass {
  B2B_VC_PLANAR, B2B_VC_RADIAL, B2B_VC_RQS, B2B_VC_COUPLING, B2B_VC_BN, B2B_VC_EW, B2B_VC_TRIL, B2B_VC_SPLINE, B2B_VC_SCALE, B2B_VC_MLP,
  B2B_VC_AR
};
// descriptor pointer fields as bits
enum { B2B_F_P0 = 1, B2B_F_P1 = 2, B2B_F_P2 = 4, B2B_F_P3 = 8, B2B_F_I0 = 16, B2B_F_I1 = 32 };

struct B2BKind {
  int kind;
  int required;   // B2B_F_* fields that must be non-NULL
  bool terminal;  // must be the chain's last element, with inverse == 0
  int launch;     // B2BLaunchClass
  int vjp;        // B2BVjpClass
  int slots;      // trainable slots: param_bars entries 4l + i for i < slots (p<i>'s cotangent)
  int optional;   // B2B_F_* bits of the slots that have a cotangent only when their parameter is given
  bool f64;       // the Float64 entry points accept the kind
};

// the row of `kind`, NULL for a value include/b2b.h does not define
inline const B2BKind* b2b_kind(int kind) {
  // function-local, so that only the host compilation sees the table (at namespace scope the device pass does too)
  constexpr int P012 = B2B_F_P0 | B2B_F_P1 | B2B_F_P2;
  static const B2BKind kinds[] = {
      // kind              required                     terminal launch        vjp              slots optional  f64
      {B2B_PLANAR,          P012,                        false, B2B_LC_FUSED,    B2B_VC_PLANAR,   3, 0,        true},
      {B2B_RADIAL,          P012,                        false, B2B_LC_FUSED,    B2B_VC_RADIAL,   3, 0,        true},
      {B2B_RQS,             P012,                        false, B2B_LC_FUSED,    B2B_VC_RQS,      3, 0,        true},
      {B2B_COUPLING_AFFINE, B2B_F_P0,                    false, B2B_LC_COUPLING, B2B_VC_COUPLING, 2, B2B_F_P1, true},
      {B2B_BATCHNORM,       P012 | B2B_F_P3,             false, B2B_LC_FUSED,    B2B_VC_BN,       2, 0,        true},
      {B2B_PERMUTE,         B2B_F_I0,                    false, B2B_LC_FUSED,    B2B_VC_EW,       0, 0,        true},
      {B2B_STACKED_EW,      B2B_F_I0,                    false, B2B_LC_FUSED,    B2B_VC_EW,       0, 0,        true},
      {B2B_MVNORMAL_DIAG,   0,                           true,  B2B_LC_FUSED,    B2B_VC_EW,       2, B2B_F_P0 | B2B_F_P1, true},
      {B2B_MVNORMAL_TRIL,   B2B_F_P1,                    true,  B2B_LC_TRIL,     B2B_VC_TRIL,     2, B2B_F_P0, true},
      {B2B_COUPLING_RQS,    B2B_F_P0 | B2B_F_I0 | B2B_F_I1, false, B2B_LC_SPLINE, B2B_VC_SPLINE,   2, B2B_F_P1, false},
      {B2B_SCALE_MATRIX,    B2B_F_P0,                    false, B2B_LC_SCALE,    B2B_VC_SCALE,    1, 0,        false},
      {B2B_COUPLING_MLP,    B2B_F_P0 | B2B_F_P2 | B2B_F_I0 | B2B_F_I1, false, B2B_LC_MLP, B2B_VC_MLP, 4, B2B_F_P1 | B2B_F_P3, false},
      {B2B_COUPLING_MLP_RQS, B2B_F_P0 | B2B_F_P2 | B2B_F_I0 | B2B_F_I1, false, B2B_LC_SPLINE, B2B_VC_SPLINE, 4, B2B_F_P1 | B2B_F_P3, false},
      {B2B_COUPLING_DEEP_MLP, P012 | B2B_F_I0 | B2B_F_I1, false, B2B_LC_MLP, B2B_VC_MLP, 4, B2B_F_P3, false},
      {B2B_COUPLING_DEEP_MLP_RQS, P012 | B2B_F_I0 | B2B_F_I1, false, B2B_LC_SPLINE, B2B_VC_SPLINE, 4, B2B_F_P3, false},
      {B2B_ELEMENTWISE_VEC, B2B_F_P0,                    false, B2B_LC_FUSED,    B2B_VC_EW,       1, 0,        true},
      {B2B_SCALE_TRIANGULAR, B2B_F_P0,                   false, B2B_LC_SCALE,    B2B_VC_SCALE,    1, 0,        true},
      {B2B_SCALE_LU,        B2B_F_P0,                    false, B2B_LC_SCALE,    B2B_VC_SCALE,    1, 0,        true},
      {B2B_AUTOREGRESSIVE_MLP, B2B_F_P0 | B2B_F_P2 | B2B_F_I0, false, B2B_LC_AR,   B2B_VC_AR,       4, B2B_F_P1 | B2B_F_P3, false},
  };
  for (const B2BKind& k : kinds)
    if (k.kind == kind) return &k;
  return nullptr;
}

inline bool b2b_chain_has_launch(const b2b_layer_desc* layers, int L, int launch) {
  for (int l = 0; l < L; ++l) {
    const B2BKind* k = b2b_kind(layers[l].kind);
    if (k && k->launch == launch) return true;
  }
  return false;
}

// ---- coupling descriptors ------------------------------------------------------------------------------------------
// Parameter roles of a coupling's conditioner: the network's first layer (W_in, and c_in = [c_1 | … | c_M], every hidden
// layer's bias), its hidden-to-hidden layers (W_hid = W_2 … W_M back to back) and the last layer (W_out, c_out: all a
// linear conditioner has).  Each kind keeps each role in one descriptor slot p0 .. p3, the roles of a slot back to back
// in this order, so the slot table of b2b_coupling fixes every role's offset and every slot's length.
enum B2BRole { B2B_W_IN, B2B_C_IN, B2B_W_HID, B2B_W_OUT, B2B_C_OUT, B2B_NROLES };

// A COUPLING_AFFINE / _RQS / _MLP / _MLP_RQS / _DEEP_MLP / _DEEP_MLP_RQS or AUTOREGRESSIVE_MLP descriptor decoded: the one
// place that knows how include/b2b.h packs each kind's shape, law and parameters.  Desc is b2b_layer_desc or
// b2b_layer_desc_f64.  AUTOREGRESSIVE_MLP is the network of COUPLING_MLP with n1 = n2 = D (the batch's rows, which
// b2b_coupling takes as its second argument) and no index lists, plus the hidden units' degrees.
template <class Desc>
struct B2BCoupling {
  using Ptr = decltype(Desc::p0);
  int n1, n2;        // rows of x₁ (transformed) and of x₂ (conditioning)
  int H, M, K;       // hidden units and hidden layers (0, 0: a linear conditioner); spline bins (0: the affine law)
  bool net, spline;  // the conditioner is a network (H, M, act, slope apply); the law is the spline (K, B apply)
  int act;
  decltype(Desc::f0) slope, B;
  int slot[B2B_NROLES];                     // descriptor slot of each role (-1: the kind has none)
  size_t off[B2B_NROLES], len[B2B_NROLES];  // its offset in the slot and its elements
  Ptr W_in, c_in, W_hid, W_out, c_out;      // the roles in the descriptor (NULL: absent)
  const int32_t *idx1, *idx2;
  const int32_t* degrees;  // AUTOREGRESSIVE_MLP: the hidden units' degrees m[H] (NULL for the couplings)
  int row1, row2;    // affine law: first rows of idx1 / idx2 when they are contiguous ranges (< 0: use the list)

  // role r within the arrays p[0..3] of the four slots (NULL when the kind has no role r or its slot's array is NULL)
  template <class T>
  T* role(T* const* p, int r) const {
    return slot[r] < 0 || !p[slot[r]] ? nullptr : p[slot[r]] + off[r];
  }
};

inline bool b2b_is_coupling(int kind) {
  return kind == B2B_COUPLING_AFFINE || kind == B2B_COUPLING_RQS || kind == B2B_COUPLING_MLP ||
         kind == B2B_COUPLING_MLP_RQS || kind == B2B_COUPLING_DEEP_MLP || kind == B2B_COUPLING_DEEP_MLP_RQS;
}

template <class Desc>
B2BCoupling<Desc> b2b_coupling(const Desc& d, int D = 0) {
  const int k = d.kind;
  const bool deep_rqs = k == B2B_COUPLING_DEEP_MLP_RQS, deep = k == B2B_COUPLING_DEEP_MLP || deep_rqs;
  const bool ar = k == B2B_AUTOREGRESSIVE_MLP;
  B2BCoupling<Desc> c{};
  c.n1 = ar ? D : d.n0;
  c.n2 = ar ? D : d.n1;
  c.net = k == B2B_COUPLING_MLP || k == B2B_COUPLING_MLP_RQS || deep || ar;
  c.spline = k == B2B_COUPLING_RQS || k == B2B_COUPLING_MLP_RQS || deep_rqs;
  // MLP_RQS: n3 = σ | K << 8; DEEP_MLP: n3 = σ | M << 8; DEEP_MLP_RQS: n3 = σ | K << 8 | M << 16
  c.K = k == B2B_COUPLING_RQS ? d.n2 : k == B2B_COUPLING_MLP_RQS ? d.n3 >> 8 : deep_rqs ? (d.n3 >> 8) & 255 : 0;
  c.M = deep_rqs ? d.n3 >> 16 : deep ? d.n3 >> 8 : c.net ? 1 : 0;
  c.B = k == B2B_COUPLING_RQS ? d.f0 : k == B2B_COUPLING_MLP_RQS || deep_rqs ? d.f1 : 0;
  c.idx1 = ar ? nullptr : d.i0;
  c.idx2 = ar ? nullptr : d.i1;
  c.degrees = ar ? d.i0 : nullptr;
  c.row1 = k == B2B_COUPLING_AFFINE ? d.n2 : -1;
  c.row2 = k == B2B_COUPLING_AFFINE ? d.n3 : -1;
  if (c.net) {
    c.H = d.n2;
    c.act = k == B2B_COUPLING_MLP || ar ? d.n3 : d.n3 & 255;
    c.slope = d.f0;
  }
  // the slot of each role: W_in, c_in, W_hid, W_out, c_out
  static constexpr int linear[B2B_NROLES] = {-1, -1, -1, 0, 1};  // AFFINE, RQS: p0 = W, p1 = c
  static constexpr int one[B2B_NROLES] = {0, 1, -1, 2, 3};       // MLP, MLP_RQS: p0 = W₁, p1 = c₁, p2 = W₂, p3 = c₂
  static constexpr int many[B2B_NROLES] = {0, 3, 1, 2, 3};       // DEEP_*: p3 = [c_1 | … | c_M | c_out]
  const int* slot = deep ? many : c.net ? one : linear;
  const size_t J = c.spline ? (size_t)(3 * c.K - 1) * c.n1 : (size_t)2 * c.n1;  // rows of W_out
  const size_t H = c.H, M = c.M;
  const size_t len[B2B_NROLES] = {H * c.n2, M * H, M > 1 ? (M - 1) * H * H : 0, J * (c.net ? H : c.n2), J};
  const typename B2BCoupling<Desc>::Ptr p[4] = {d.p0, d.p1, d.p2, d.p3};
  for (int r = 0; r < B2B_NROLES; ++r) {
    c.slot[r] = slot[r];
    c.len[r] = len[r];
    for (int q = 0; q < r; ++q)
      if (slot[q] == slot[r]) c.off[r] += len[q];
  }
  c.W_in = c.role(p, B2B_W_IN);
  c.c_in = c.role(p, B2B_C_IN);
  c.W_hid = c.role(p, B2B_W_HID);
  c.W_out = c.role(p, B2B_W_OUT);
  c.c_out = c.role(p, B2B_C_OUT);
  return c;
}

// Float32 kernel envelope of a COUPLING_RQS / _MLP / _MLP_RQS / _DEEP_MLP / _DEEP_MLP_RQS layer at D: the B2B_COUPLING_*_MAX_* limits
// of include/b2b.h (the affine coupling's limits are shared-memory budgets, b2b_coupling_affine_fits).  Defined in
// b2b_api.cu: inline here, it changes the SASS nvcc 12.9 emits for the neural-spline reverse-mode kernels.
bool b2b_coupling_fits(const b2b_layer_desc& d, int D);

// whether the chain ends in its MvNormal terminal (its logjac output is then logpdf)
template <class Desc>
bool b2b_ends_in_terminal(const Desc* layers, int L) {
  const B2BKind* k = b2b_kind(layers[L - 1].kind);
  return k && k->terminal;
}

// B2B_EINVAL when `d` breaks the pointer and shape rules of include/b2b.h at D (`last`: the chain's final element),
// else B2B_OK.  The rules of both precisions; the envelopes are the caller's.
template <class Desc>
int b2b_check_desc(const Desc& d, int D, bool last) {
  const B2BKind* k = b2b_kind(d.kind);
  if (!k) return B2B_EINVAL;
  const void* const field[6] = {d.p0, d.p1, d.p2, d.p3, d.i0, d.i1};
  for (int f = 0; f < 6; ++f)
    if ((k->required >> f & 1) && !field[f]) return B2B_EINVAL;
  if (k->terminal && (!last || d.inverse)) return B2B_EINVAL;
  if (d.kind == B2B_RQS) return d.n0 >= 2 ? B2B_OK : B2B_EINVAL;
  if (d.kind == B2B_ELEMENTWISE_VEC)
    return d.n0 == B2B_EW_SHIFT || d.n0 == B2B_EW_SCALE || d.n0 == B2B_EW_LEAKY_RELU ? B2B_OK : B2B_EINVAL;
  if (d.kind == B2B_SCALE_TRIANGULAR)  // n0: lower / upper, n1: stored / unit diagonal
    return (d.n0 == 0 || d.n0 == 1) && (d.n1 == 0 || d.n1 == 1) ? B2B_OK : B2B_EINVAL;
  if (d.kind == B2B_AUTOREGRESSIVE_MLP)  // n2: H, n3: σ
    return d.n2 >= 1 && (d.n3 == B2B_ACT_TANH || d.n3 == B2B_ACT_LEAKY_RELU) ? B2B_OK : B2B_EINVAL;
  if (!b2b_is_coupling(d.kind)) return B2B_OK;
  const B2BCoupling<Desc> c = b2b_coupling(d);
  bool ok = c.n1 >= 1 && c.n2 >= 1 && c.n1 + c.n2 <= D;
  if (c.net) ok = ok && c.H >= 1 && (c.act == B2B_ACT_TANH || c.act == B2B_ACT_LEAKY_RELU);
  if (c.spline) ok = ok && c.K >= 1 && c.B > 0;
  if (d.kind == B2B_COUPLING_DEEP_MLP || d.kind == B2B_COUPLING_DEEP_MLP_RQS) ok = ok && c.M >= 2;
  // an index list may be NULL when n2 / n3 gives the first row of its contiguous range
  if (d.kind == B2B_COUPLING_AFFINE) ok = ok && (c.idx1 || c.row1 >= 0) && (c.idx2 || c.row2 >= 0);
  return ok ? B2B_OK : B2B_EINVAL;
}

// elements of trainable slot i of `d` (its cotangent has the parameter's shape)
template <class Desc>
size_t b2b_slot_len(const Desc& d, int i, int D) {
  if (b2b_is_coupling(d.kind) || d.kind == B2B_AUTOREGRESSIVE_MLP) {  // the sum of the slot's roles
    const B2BCoupling<Desc> c = b2b_coupling(d, D);
    size_t n = 0;
    for (int r = 0; r < B2B_NROLES; ++r)
      if (c.slot[r] == i) n += c.len[r];
    return n;
  }
  switch (d.kind) {
    case B2B_PLANAR: return i == 2 ? 1 : D;
    case B2B_RADIAL: return i == 2 ? D : 1;
    case B2B_RQS: return (size_t)D * d.n0;
    case B2B_MVNORMAL_TRIL: return i == 1 ? (size_t)D * D : D;
    case B2B_SCALE_MATRIX:
    case B2B_SCALE_TRIANGULAR:
    case B2B_SCALE_LU: return (size_t)D * D;
    default: return D;  // BATCHNORM b / logs, MVNORMAL_DIAG μ / σ, ELEMENTWISE_VEC a
  }
}

// ---- checks shared by b2b_chain_vjp_f32 and b2b_chain_vjp_f64 (valid descriptors; each entry point keeps its order) ----
// The requested cotangents (non-NULL param_bars entries): B2B_EUNSUPPORTED for a slot the kind does not train,
// B2B_EINVAL for an optional parameter that is absent.  *want gets bit l for every layer with a request.
template <class Desc, class T>
int b2b_vjp_check_slots(const Desc* layers, int L, T* const* param_bars, unsigned* want) {
  *want = 0;
  for (int l = 0; l < L && param_bars; ++l)
    for (int i = 0; i < 4; ++i) {
      if (!param_bars[4 * l + i]) continue;
      const B2BKind& k = *b2b_kind(layers[l].kind);
      const void* const p[4] = {layers[l].p0, layers[l].p1, layers[l].p2, layers[l].p3};
      if (i >= k.slots) return B2B_EUNSUPPORTED;
      if ((k.optional >> i & 1) && !p[i]) return B2B_EINVAL;
      *want |= 1u << l;
    }
  return B2B_OK;
}

// N == 0: zeroes the requested cotangents, which is the whole call.  Otherwise checks the batch arguments: x̄ is written
// while x and ȳ are still being read, so it must not overlap either.
template <class Desc, class T>
int b2b_vjp_check_batch(const Desc* layers, int L, T* const* param_bars, const T* x, const T* ybar, T* xbar, int D,
                        long long N, long long ldx, long long ldybar, long long ldxbar, cudaStream_t stream) {
  if (N == 0) {
    int launches = 0;
    for (int l = 0; l < L && param_bars; ++l)
      for (int i = 0; i < 4; ++i)
        if (T* bar = param_bars[4 * l + i]) {
          const cudaError_t e = cudaMemsetAsync(bar, 0, b2b_slot_len(layers[l], i, D) * sizeof(T), stream);
          if (e != cudaSuccess) return (int)e;
          ++launches;
        }
    b2b_set_last_launch_count(launches);
    return B2B_OK;
  }
  if (!x || !xbar || ldx < D || ldxbar < D || (ybar && ldybar < D)) return B2B_EINVAL;
  const size_t span = ((size_t)(N - 1) * (size_t)ldxbar + (size_t)D) * sizeof(T);
  auto overlaps = [&](const T* p, long long ld) {
    const char *a = reinterpret_cast<const char*>(p), *b = reinterpret_cast<const char*>(xbar);
    return b < a + ((size_t)(N - 1) * (size_t)ld + (size_t)D) * sizeof(T) && a < b + span;
  };
  if (overlaps(x, ldx) || (ybar && overlaps(ybar, ldybar))) return B2B_EINVAL;
  return B2B_OK;
}
