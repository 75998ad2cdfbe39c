// Reverse mode (vector-Jacobian product) of the RationalQuadraticSpline layer, either direction: cotangents of the input
// and of the PROCESSED knot arrays widths / heights / derivatives (D x K1) -- what the reference's reverse-mode AD computes
// through rational_quadratic_spline.jl:317-357 (forward) / :183-220 (inverse).  Restated and finite-difference-checked in
// oracle/oracle_np.py (rqs_vjp), whose reverse sweep this kernel follows line by line:
//   w = x_{k+1} − x_k, Δ = y_{k+1} − y_k, s = Δ/w, ξ = (x − x_k)/w, o = 1 − ξ, p = ξo, ds = d_{k+1} + d_k − 2s,
//   den = s + ds·p, a = sξ² + d_k p, y = y_k + Δ·a/den, b = d_{k+1}ξ² + 2sp + d_k o², lj = 2 log s + log b − 2 log den.
// Inverse: inverse-function theorem at the recovered point: f_x = s²b/den², lj_x = (b_ξ/b − 2 den_ξ/den)/w,
// ȳ* = (x̄ − l̄·lj_x)/f_x is the input cotangent, the knot cotangents are the forward sweep's with (ȳ, l̄) -> (−ȳ*, −l̄).
//
// Numerics.  Cotangents blow up next to a knot of a steep bin, where o = 1 − ξ (or ξ) is tiny; the float32 reference
// loses them there (1e-4 .. 1e-3 of the batch maximum).  This kernel keeps BOTH ξ and o to relative accuracy:
//   forward   o = (x_{k+1} − x)/w (an exact difference) instead of 1 − ξ;
//   inverse   the quadratic of :205-214 is solved from the NEARER knot -- by the reflection symmetry of the rational
//             quadratic, 1 − ξ is the root of the same quadratic with d_k <-> d_{k+1} and y − y_k -> y_{k+1} − y;
//   den = s(1 − 2p) + (d_k + d_{k+1})p, all terms positive (p <= 1/4).
// Measured against the float64 oracle this is 1e-7 .. 1e-5 where the float32 restatement of the reference has 1e-5 .. 2e-3.
//
// Mapping: a thread owns ONE ROW of a slab of columns (threads of a warp = consecutive rows of one column: coalesced) and
// walks its columns in a fixed order, U at a time for memory-level parallelism; the 3·K1 knot cotangents of its row
// accumulate in shared-memory slots of its own ([slot][thread]: conflict-free), the row's knots sit in a shared table
// ([knot][row]: conflict-free for any bin pattern).  Slabs are summed inside the CTA, CTAs by a second kernel, both in a
// fixed order -- deterministic, no atomics.
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_internal.h"

namespace b2b {

constexpr int RQV_THREADS = 256;
constexpr int RQV_U = 4;
constexpr size_t RQV_SMEM_MAX = 200 * 1024;

struct RqvParams {
  const float* x;
  const float* ybar;
  const float* ljbar;
  float* xbar;
  const float *W, *H, *Dv;
  float* part;  // [grid][3][K1][D]
  long long N, ldx, ldyb, ldxb;
  int D, K1;
};

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

// K1T / DPT: 0 = knot count / padded row count at run time, else the exact values (table offsets, accumulator slots and the
// bin search become constants and a fully unrolled loop).
template <bool INV, bool STAB, int K1T, int DPT>
__global__ void __launch_bounds__(RQV_THREADS, 3) rqs_vjp_kernel(const __grid_constant__ RqvParams P) {
  extern __shared__ float rqv_sm[];
  const int D = P.D, K1 = K1T ? K1T : P.K1, Dp = DPT ? DPT : ((D + 31) & ~31), nslab = RQV_THREADS / Dp;
  const int tid = threadIdx.x, slab = tid / Dp, i = tid - slab * Dp;
  float* acc = rqv_sm;                          // [3*K1][RQV_THREADS]
  float* tab = rqv_sm + 3 * K1 * RQV_THREADS;   // [3][K1][Dp] when STAB
  for (int k = 0; k < 3 * K1; ++k) acc[k * RQV_THREADS + tid] = 0.f;
  if (STAB) {
    for (int e = tid; e < 3 * K1 * Dp; e += RQV_THREADS) {
      const int kk = e / Dp, ii = e - kk * Dp, arr = kk / K1, k = kk - arr * K1;
      const float* src = arr == 0 ? P.W : arr == 1 ? P.H : P.Dv;
      tab[e] = ii < D ? src[(size_t)k * D + ii] : 0.f;
    }
  }
  __syncthreads();
  const bool active = slab < nslab && i < D;
  // contiguous column range of this CTA, columns dealt round-robin to its slabs
  const long long per = (P.N + gridDim.x - 1) / gridDim.x;
  const long long c0 = (long long)blockIdx.x * per, c1 = (c0 + per < P.N) ? c0 + per : P.N;
  if (active) {
    RqvKnots<INV, STAB> T;
    T.W = (STAB ? tab : P.W) + i;
    T.H = (STAB ? tab + K1 * Dp : P.H) + i;
    T.Dv = (STAB ? tab + 2 * K1 * Dp : P.Dv) + i;
    T.stride = STAB ? Dp : D;
    const float Wl = T.w(K1 - 1), Hl = T.h(K1 - 1);
    const float Bs = INV ? Hl : Wl;
    float* my = acc + tid;
    const int K1s = K1 * RQV_THREADS;
    for (long long n0 = c0 + slab; n0 < c1; n0 += (long long)RQV_U * nslab) {
      float v[RQV_U], cb[RQV_U], lb[RQV_U], raw[RQV_U];
      bool in[RQV_U];
      int kb[RQV_U];
#pragma unroll
      for (int u = 0; u < RQV_U; ++u) {
        const long long n = n0 + (long long)u * nslab;
        const bool ok = n < c1;  // columns past the range run on zeros (zero cotangents, nothing stored)
        raw[u] = ok ? __ldcs(P.x + n * P.ldx + i) : 0.f;
        cb[u] = ok ? __ldcs(P.ybar + n * P.ldyb + i) : 0.f;
        lb[u] = ok && P.ljbar ? P.ljbar[n] : 0.f;
        kb[u] = 0;
      }
#pragma unroll
      for (int u = 0; u < RQV_U; ++u) {
        // identity outside the box (:322 / :188): the element is evaluated at 0 (inside every box, in a bin of positive
        // width) with zero cotangents, so that every knot cotangent it adds is an exact 0; its own cotangent passes through
        in[u] = raw[u] > -Bs && raw[u] < Bs;
        v[u] = in[u] ? raw[u] : 0.f;
      }
      // bin = number of knots < v (searchsortedfirst − 1); one pass over the row's knots serves the U columns
#pragma unroll
      for (int j = 0; j < K1 - 1; ++j) {
        const float sj = T.s(j);
#pragma unroll
        for (int u = 0; u < RQV_U; ++u) kb[u] += sj < v[u] ? 1 : 0;
      }
      RqvCot c[RQV_U];
#pragma unroll
      for (int u = 0; u < RQV_U; ++u) {
        const long long n = n0 + (long long)u * nslab;
        const float out = rqv_element<INV, STAB>(T, K1, kb[u], Wl, Hl, v[u], in[u] ? cb[u] : 0.f, in[u] ? lb[u] : 0.f, c[u]);
        if (n < c1) __stcs(P.xbar + n * P.ldxb + i, in[u] ? out : cb[u]);
      }
      // scatter into this thread's own slots: W | H | Dv
#pragma unroll
      for (int u = 0; u < RQV_U; ++u) {
        const int k = c[u].k;
        float* pa = my + (k > 0 ? k - 1 : K1 - 1) * RQV_THREADS;
        float* pb = my + k * RQV_THREADS;
        pa[0] += c[u].xk;
        pa[K1s] += c[u].yk;
        pa[2 * K1s] += c[u].dk;
        pb[0] += c[u].xk1;
        pb[K1s] += c[u].yk1;
        pb[2 * K1s] += c[u].dk1;
      }
    }
  }
  __syncthreads();
  // slabs summed in order; per-CTA partial laid out [3][K1][D] like the parameter arrays
  float* out = P.part + (size_t)blockIdx.x * 3 * K1 * D;
  for (int e = tid; e < 3 * K1 * D; e += RQV_THREADS) {
    const int kk = e / D, ii = e - kk * D;
    float t = 0.f;
    for (int sl = 0; sl < nslab; ++sl) t += acc[kk * RQV_THREADS + sl * Dp + ii];
    out[e] = t;
  }
}

// Sums the per-CTA partials: 8 strided sub-sums per element, then those in order.
__global__ void __launch_bounds__(256) rqs_vjp_reduce_kernel(const float* __restrict__ part, int nparts, int len, int per,
                                                             float* __restrict__ Wb, float* __restrict__ Hb,
                                                             float* __restrict__ Db) {
  __shared__ float sub[8][32];
  const int e = blockIdx.x * 32 + threadIdx.x;
  float t = 0.f;
  if (e < len)
    for (int p = threadIdx.y; p < nparts; p += 8) t += part[(size_t)p * len + e];
  sub[threadIdx.y][threadIdx.x] = t;
  __syncthreads();
  if (threadIdx.y == 0 && e < len) {
    float r = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) r += sub[q][threadIdx.x];
    if (e < per) Wb[e] = r;
    else if (e < 2 * per) Hb[e - per] = r;
    else Db[e - 2 * per] = r;
  }
}

struct RqvShape {
  size_t smem;
  bool stab;
  int grid_max;
};

static RqvShape rqv_shape(int K1, int D) {
  const int Dp = (D + 31) & ~31;
  RqvShape s;
  const size_t acc = (size_t)3 * K1 * RQV_THREADS * sizeof(float), tab = (size_t)3 * K1 * Dp * sizeof(float);
  s.stab = acc + tab <= RQV_SMEM_MAX;
  s.smem = acc + (s.stab ? tab : 0);
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sms <= 0) sms = 132;
  int per_sm = (int)((size_t)(227 * 1024) / (s.smem + 1024));
  if (per_sm > 3) per_sm = 3;  // 80 registers x 256 threads: three CTAs per SM
  if (per_sm < 1) per_sm = 1;
  s.grid_max = sms * per_sm;
  return s;
}

}  // namespace b2b

extern "C" size_t b2b_rqs_vjp_workspace_bytes(int32_t K1, int32_t D) {
  if (K1 < 2 || K1 > 64 || D < 1 || D > 256) return 0;
  return (size_t)b2b::rqv_shape(K1, D).grid_max * 3 * (size_t)K1 * D * sizeof(float) + 256;
}

extern "C" int b2b_rqs_vjp_f32(const b2b_layer_desc* layer, const float* x, const float* ybar, const float* ljbar, float* xbar,
                               float* widths_bar, float* heights_bar, float* derivs_bar, int32_t D, int64_t N, int64_t ldx,
                               int64_t ldybar, int64_t ldxbar, void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b2b;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!layer || layer->kind != B2B_RQS || D < 1 || N < 0 || !widths_bar || !heights_bar || !derivs_bar) return B2B_EINVAL;
  const b2b_layer_desc& d = *layer;
  const int K1 = d.n0;
  if (!d.p0 || !d.p1 || !d.p2 || K1 < 2) return B2B_EINVAL;
  if (K1 > 64 || D > 256) return B2B_EUNSUPPORTED;
  const size_t per = (size_t)K1 * D;
  if (N == 0) {
    cudaMemsetAsync(widths_bar, 0, per * sizeof(float), stream);
    cudaMemsetAsync(heights_bar, 0, per * sizeof(float), stream);
    return (int)cudaMemsetAsync(derivs_bar, 0, per * sizeof(float), stream);
  }
  if (!x || !ybar || !xbar || ldx < D || ldybar < D || ldxbar < D) return B2B_EINVAL;
  if (!workspace || workspace_bytes < b2b_rqs_vjp_workspace_bytes(K1, D)) return B2B_EWORKSPACE;
  char* wsb = static_cast<char*>(workspace);
  wsb += (256 - (reinterpret_cast<uintptr_t>(wsb) & 255)) & 255;
  RqvParams P;
  P.x = x;
  P.ybar = ybar;
  P.ljbar = ljbar;
  P.xbar = xbar;
  P.W = d.p0;
  P.H = d.p1;
  P.Dv = d.p2;
  P.part = reinterpret_cast<float*>(wsb);
  P.N = N;
  P.ldx = ldx;
  P.ldyb = ldybar;
  P.ldxb = ldxbar;
  P.D = D;
  P.K1 = K1;
  const RqvShape sh = rqv_shape(K1, D);
  const int Dp = (D + 31) & ~31, nslab = RQV_THREADS / Dp;
  int grid = sh.grid_max;
  const long long want = (N + (long long)nslab * RQV_U - 1) / ((long long)nslab * RQV_U);
  if (grid > want) grid = (int)want;
  void (*kernel)(const RqvParams) = nullptr;
#define B2B_RQV_EXACT(KK, DD)                                                                        \
  if (sh.stab && K1 == KK && Dp == DD)                                                               \
    kernel = d.inverse ? rqs_vjp_kernel<true, true, KK, DD> : rqs_vjp_kernel<false, true, KK, DD>;
  B2B_RQV_EXACT(5, 32) B2B_RQV_EXACT(9, 32) B2B_RQV_EXACT(17, 32) B2B_RQV_EXACT(33, 32)
  B2B_RQV_EXACT(5, 64) B2B_RQV_EXACT(9, 64) B2B_RQV_EXACT(17, 64) B2B_RQV_EXACT(33, 64)
#undef B2B_RQV_EXACT
  if (!kernel)
    kernel = d.inverse ? (sh.stab ? rqs_vjp_kernel<true, true, 0, 0> : rqs_vjp_kernel<true, false, 0, 0>)
                       : (sh.stab ? rqs_vjp_kernel<false, true, 0, 0> : rqs_vjp_kernel<false, false, 0, 0>);
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<grid, RQV_THREADS, sh.smem, stream>>>(P);
  e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  const int len = (int)(3 * per);
  rqs_vjp_reduce_kernel<<<(len + 31) / 32, dim3(32, 8), 0, stream>>>(P.part, grid, len, (int)per, widths_bar, heights_bar,
                                                                     derivs_bar);
  return (int)cudaGetLastError();
}
