// Shared by b2b_planar_const.cu (forward / inverse evaluation) and b2b_planar_vjp.cu (reverse mode): the in-kernel
// get_u_hat derivation into shared memory, the stand-alone preparation kernel and the launch shapes.
#pragma once
#include <cstring>

#include "b2b_v1_pipeline.cuh"

namespace b2b {

constexpr int HP_MAX_L = 8;
constexpr int HP_MAX_D = 128;

// get_u_hat (planar_layer.jl:65-70) of the layers P.layers[0..nreal) into shared memory, packed for (D, L):
// w[L][D] | û[L][D] | c[L] | b[L]; layers nreal..L-1 are identity padding.  One warp per layer.
template <int D>
__device__ __forceinline__ void planar_derive_smem(const B2BChainParams& P, int nreal, int L, float* params, int warp,
                                                   int lane, int nw) {
  for (int l = warp; l < L; l += nw) {
    float* w_out = params + l * D;
    float* u_out = params + L * D + l * D;
    if (l >= nreal) {
      for (int i = lane; i < D; i += 32) w_out[i] = u_out[i] = 0.f;
      if (lane == 0) params[2 * L * D + l] = params[2 * L * D + L + l] = 0.f;
      continue;
    }
    const b2b_layer_desc& d = P.layers[l];
    float s = 0.f, q = 0.f;
    for (int i = lane; i < D; i += 32) {
      const float w = d.p0[i], u = d.p1[i];
      s = fmaf(w, u, s);
      q = fmaf(w, w, q);
    }
    s = warp_sum(s);
    q = warp_sum(q);
    const float k = (softplus(-s) - 1.0f) / q;  // planar_layer.jl:67
    for (int i = lane; i < D; i += 32) {
      const float w = d.p0[i];
      w_out[i] = w;
      u_out[i] = fmaf(k, w, d.p1[i]);
    }
    if (lane == 0) {
      params[2 * L * D + l] = softplus(s) - 1.0f;  // wᵀû, planar_layer.jl:68
      params[2 * L * D + L + l] = d.p2[0];          // first(flow.b), :75
    }
  }
}

// get_u_hat (planar_layer.jl:65-70) for Lp layers (the last Lp - L are identity padding), one warp per layer,
// packed for (D, Lp) into `out`.
static __global__ void __launch_bounds__(HP_MAX_L * 32)
    planar_prep_kernel(const __grid_constant__ B2BChainParams P, int L, int Lp, float* __restrict__ out) {
  const int lane = threadIdx.x & 31, l = threadIdx.x >> 5, D = P.D;
  if (l >= Lp) return;
  auto put = [&](int idx, float v) { out[idx] = v; };
  const int wo = l * D, uo = Lp * D + l * D;
  if (l >= L) {
    for (int i = lane; i < D; i += 32) {
      put(wo + i, 0.f);
      put(uo + i, 0.f);
    }
    if (lane == 0) {
      put(2 * Lp * D + l, 0.f);
      put(2 * Lp * D + Lp + l, 0.f);
    }
    return;
  }
  const b2b_layer_desc& d = P.layers[l];
  float s = 0.f, q = 0.f;
  for (int i = lane; i < D; i += 32) {
    const float w = d.p0[i], u = d.p1[i];
    s = fmaf(w, u, s);
    q = fmaf(w, w, q);
  }
  s = warp_sum(s);
  q = warp_sum(q);
  const float k = (softplus(-s) - 1.0f) / q;  // planar_layer.jl:67
  for (int i = lane; i < D; i += 32) {
    const float w = d.p0[i];
    put(wo + i, w);
    put(uo + i, fmaf(k, w, d.p1[i]));
  }
  if (lane == 0) {
    put(2 * Lp * D + l, softplus(s) - 1.0f);  // wᵀû, planar_layer.jl:68
    put(2 * Lp * D + Lp + l, d.p2[0]);        // first(flow.b), :75
  }
}

// ---- host side: launch shapes -------------------------------------------------------------------------------
// warps per CTA as in the interpreter (register budget)
static int hp_warps(int D) { return D == 128 ? 8 : (D == 64 ? 12 : 16); }

}  // namespace b2b
