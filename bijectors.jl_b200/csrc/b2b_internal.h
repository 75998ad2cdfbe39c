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
    case B2B_STACKED_EW: return 3 * Dp;
    case B2B_MVNORMAL_DIAG: return 2 * Dp + 4;
    default: return 0;
  }
}

// ---- launchers (each returns a cudaError_t as int, or a negative B2B_E* code) ---------------------
// v0: lane-group direct-global fused interpreter (any D <= 1024)
int b2b_launch_chain_v0(const B2BChainParams& p, cudaStream_t stream);
// v1: TMA-staged thread-per-column fused interpreter (D in {32,64,128}); returns B2B_EUNSUPPORTED otherwise
int b2b_launch_chain_v1(const B2BChainParams& p, cudaStream_t stream);
// constant-bank planar chains (b2b_planar_const.cu).  hostparams: `L` in {1,2,4,8} layers, derived parameters packed
// w[L][D] | û[L][D] | c[L] | b[L] in HOST memory, bit l of invmask = inverse of layer l.
int b2b_launch_planar_hostparams(const B2BChainParams& p, int L, const float* packed, int invmask,
                                 cudaStream_t stream);
// device-resident parameters: p.layers must be 1..8 PLANAR layers; B2B_EUNSUPPORTED when not applicable
int b2b_launch_planar_chain_const(const B2BChainParams& p, cudaStream_t stream);
int b2b_planar_const_grid_size(const B2BChainParams& p);
// number of planar layers when the constant-bank path applies to the segment `p`, else 0
int b2b_planar_const_layers(const B2BChainParams& p);
// reverse mode of a forward radial chain (b2b_radial_vjp.cu)
size_t b2b_radial_vjp_workspace(int L, int D);
int b2b_launch_radial_chain_vjp(const B2BChainParams& p, const float* ybar, long long ldyb, const float* ljbar,
                                float* xbar, long long ldxb, float* alpha_bar, float* beta_bar, float* z0_bar,
                                void* workspace, size_t workspace_bytes, int* launches, cudaStream_t stream);
// 1..8 radial layers of one direction as a specialised program (b2b_radial_unrolled.cu)
int b2b_radial_unrolled_applicable(const B2BChainParams& p);
int b2b_launch_radial_unrolled(const B2BChainParams& p, cudaStream_t stream);
// a single RQS layer with 9 knots as a specialised program (b2b_rqs_unrolled.cu)
int b2b_rqs_unrolled_applicable(const B2BChainParams& p);
int b2b_launch_rqs_unrolled(const B2BChainParams& p, cudaStream_t stream);
// reverse mode of a forward planar chain (b2b_planar_const.cu)
size_t b2b_planar_vjp_workspace(int L, int D, long long N);
int b2b_launch_planar_chain_vjp(const B2BChainParams& p, const float* ybar, long long ldyb, const float* ljbar,
                                float* xbar, long long ldxb, float* wbar, float* ubar, float* bbar, void* workspace,
                                size_t workspace_bytes, int* launches, cudaStream_t stream);
// number of CTAs the v0/v1 launch of `p` will use (size of the partials array)
int b2b_chain_grid_size(const B2BChainParams& p);
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
// affine coupling, exact-fp32 CUDA-core kernel (any index lists)
int b2b_launch_coupling_affine(const b2b_layer_desc& d, const float* fold, const float* x, float* y,
                               float* logjac, int D, long long N, long long ldx, long long ldy, int accumulate,
                               cudaStream_t stream);
