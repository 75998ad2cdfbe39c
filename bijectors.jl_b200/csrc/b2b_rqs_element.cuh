// RQS element reverse mode shared by the RationalQuadraticSpline VJP (b2b_rqs_vjp.cu) and the spline coupling VJP
// (b2b_coupling_rqs_vjp.cu): the cotangents of one element's input and of the processed knots of its bin, with the
// knot-accurate numerics described at the top of b2b_rqs_vjp.cu.  The knots are read through an accessor, so the caller
// decides where they live (a per-row table, or a per-thread table of knots computed on the device).
#pragma once
#include <cuda_runtime.h>

namespace b2b {

struct RqvCot {
  float xk, xk1, yk, yk1, dk, dk1;
  int k;
};

// The row's knots: W | H | Dv tables with this thread's row offset folded in; `stride` floats between consecutive knots.
template <bool INV, bool STAB>
struct RqvKnots {
  const float *W, *H, *Dv;
  int stride;
  __device__ __forceinline__ float ld(const float* p) const { return STAB ? *p : __ldg(p); }
  __device__ __forceinline__ float w(int k) const { return ld(W + k * stride); }
  __device__ __forceinline__ float h(int k) const { return ld(H + k * stride); }
  __device__ __forceinline__ float d(int k) const { return ld(Dv + k * stride); }
  __device__ __forceinline__ float s(int k) const { return INV ? h(k) : w(k); }
};

__device__ __forceinline__ float rqv_rcp(float x) { return __fdividef(1.0f, x); }  // MUFU.RCP, <= 1 ulp

// One element (v inside the box; elements outside arrive as v = 0 with zero cotangents): returns the input cotangent, fills the
// knot cotangents of its bin.  Branch-free: the k == 0 / k == K1−1 cases are selects.
template <bool INV, bool STAB>
__device__ __forceinline__ float rqv_element(const RqvKnots<INV, STAB>& T, int K1, int k, float Wl, float Hl, float v, float cb,
                                              float lb, RqvCot& c) {
  const int km = k > 0 ? k - 1 : 0;
  const float wa = T.w(km), ha = T.h(km), da = T.d(km), db = T.d(k);
  const float xk = k == 0 ? -Wl : wa, xk1 = T.w(k);
  const float yk = k == 0 ? -Hl : ha, yk1 = T.h(k);
  const float dk = k == 0 ? 1.0f : da;
  const float dk1 = k == K1 - 1 ? 1.0f : db;
  const float w = xk1 - xk, dyv = yk1 - yk, iw = rqv_rcp(w), s = dyv * iw;
  const float dsv = dk1 + dk - 2.0f * s;
  float xi, o;
  if (INV) {
    const float lo = v - yk, hi = yk1 - v;
    const bool lower = lo < hi;
    const float yh = lower ? lo : hi, dd = lower ? dk : dk1;  // solve from the nearer knot
    const float a1 = fmaf(dyv, s - dd, yh * dsv), a2 = fmaf(dyv, dd, -yh * dsv), a3 = -s * yh;
    const float r = -2.0f * a3 * rqv_rcp(a2 + sqrtf(fmaf(a2, a2, -4.0f * a1 * a3)));
    xi = lower ? r : 1.0f - r;
    o = lower ? 1.0f - r : r;
  } else {
    xi = (v - xk) * iw;
    o = (xk1 - v) * iw;
  }
  const float p = xi * o;
  const float den = fmaf(s, 1.0f - 2.0f * p, (dk1 + dk) * p), iden = rqv_rcp(den);
  const float a = fmaf(s * xi, xi, dk * p), num = dyv * a;
  const float b = fmaf(dk1 * xi, xi, fmaf(2.0f * s, p, dk * o * o));
  const float ib = rqv_rcp(b);
  float yb_ = cb, lb_ = lb, ystar = 0.f;
  if (INV) {
    const float if_x = den * den * rqv_rcp(s * s * b);
    const float b_xi = 2.0f * fmaf(dk1 - s, xi, (s - dk) * o);
    const float den_xi = dsv * (o - xi);
    const float lj_x = (b_xi * ib - 2.0f * den_xi * iden) * iw;
    ystar = (cb - lb * lj_x) * if_x;
    yb_ = -ystar;
    lb_ = -lb;
  }
  // reverse sweep (oracle_np.rqs_vjp)
  const float num_b = yb_ * iden;
  const float den_b = -(num_b * num + 2.0f * lb_) * iden;
  const float b_b = lb_ * ib;
  float s_b = 2.0f * lb_ * rqv_rcp(s);
  float dyv_b = num_b * a;
  const float a_b = num_b * dyv;
  s_b = fmaf(a_b * xi, xi, s_b);
  float xi_b = a_b * 2.0f * s * xi;
  float dk_b = a_b * p;
  float p_b = a_b * dk;
  float dk1_b = b_b * xi * xi;
  xi_b = fmaf(b_b * 2.0f * dk1, xi, xi_b);
  s_b = fmaf(b_b * 2.0f, p, s_b);
  p_b = fmaf(b_b * 2.0f, s, p_b);
  dk_b = fmaf(b_b * o, o, dk_b);
  float o_b = b_b * 2.0f * dk * o;
  s_b += den_b;
  const float ds_b = den_b * p;
  p_b = fmaf(den_b, dsv, p_b);
  dk1_b += ds_b;
  dk_b += ds_b;
  s_b -= 2.0f * ds_b;
  xi_b = fmaf(p_b, o, xi_b);
  o_b = fmaf(p_b, xi, o_b);
  xi_b -= o_b;
  const float x_b = xi_b * iw;
  float w_b = -x_b * xi;
  dyv_b = fmaf(s_b, iw, dyv_b);
  w_b = fmaf(-s_b * s, iw, w_b);
  // k == 0: x_k = −widths[end], y_k = −heights[end] (negated, scattered to the last knot), d_k = 1 (no cotangent);
  // k == K1−1: d_{k+1} = 1
  const float xk_b = -x_b - w_b, yk_b = yb_ - dyv_b;
  c.xk = k == 0 ? -xk_b : xk_b;
  c.xk1 = w_b;
  c.yk = k == 0 ? -yk_b : yk_b;
  c.yk1 = dyv_b;
  c.dk = k == 0 ? 0.f : dk_b;
  c.dk1 = k == K1 - 1 ? 0.f : dk1_b;
  c.k = k;
  return INV ? ystar : x_b;
}

}  // namespace b2b
