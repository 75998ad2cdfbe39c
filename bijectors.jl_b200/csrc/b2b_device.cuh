// Device-side math and parameter staging shared by the chain kernels.
// Every function cites the reference lines (Bijectors.jl v0.16.2) whose arithmetic it restates.
#pragma once
#include "b2b_internal.h"

namespace b2b {

// ---- scalar math ---------------------------------------------------------------------------------

// LogExpFunctions.log1pexp (softplus), used only on per-layer scalars / small tables
// (planar_layer.jl:67-68, radial_layer.jl:44-45,91-92).
__device__ __forceinline__ float softplus(float x) {
  return x > 0.f ? x + log1pf(expf(-x)) : log1pf(expf(x));
}

// tanh(a) and sech(a)^2 from ONE exponential: e = exp(-2|a|), tanh = (1-e)/(1+e), sech^2 = 4e/(1+e)^2.
// sech^2 has no cancellation for large |a| (the reference evaluates abs2(sech(a)), planar_layer.jl:107);
// for |a| < 0.25 an odd polynomial keeps tanh accurate to ~1 ulp where (1-e) would cancel.
__device__ __forceinline__ void tanh_sech2(float a, float& t, float& s2) {
  const float ax = fabsf(a);
  const float e = __expf(-2.0f * ax);
  const float r = __frcp_rn(1.0f + e);
  float tb = (1.0f - e) * r;
  const float a2 = a * a;
  float p = fmaf(a2, 0.021869488f, -0.053968254f);  // 62/2835, -17/315
  p = fmaf(a2, p, 0.13333334f);                      // 2/15
  p = fmaf(a2, p, -0.33333334f);                     // -1/3
  const float ts = fmaf(ax * a2, p, ax);
  tb = ax < 0.25f ? ts : tb;
  t = copysignf(tb, a);
  s2 = 4.0f * e * r * r;
}

// find_alpha (planar_layer.jl:160-185): root of f(α) = α + c·tanh(α+b) − t in [t−2|c|, t+2|c|]; also returns
// tanh(α+b) and sech²(α+b), which the inverse needs next (planar_layer.jl:122-124, interface.jl:276-281).
// The reference narrows a bracket with Roots.A42; results are pinned by the equation residual
// (test/normalising_flows.jl:47-71), so any bracketed iteration on the monotone f is admissible.  Here:
//  * start from one fixed-point step x0 = t − c·tanh(t+b) (always inside the bracket since |tanh| < 1);
//  * Chebyshev steps x ← x − N(1 + N·A), N = f/f1, A = f2/(2·f1) (cubic; tanh and sech² give f and its first three
//    derivatives f1, f2, f3 for free), falling back to Newton when the series is not trustworthy and to bisection
//    when a step leaves the bracket;
//  * stop as soon as the PREDICTED error of the new iterate, |2A² − f3/(6·f1)|·|N|³ (+ a quartic bound), is below
//    one ulp of the bracket's magnitude -- no extra evaluation just to observe a tiny step;
//  * tanh / sech² at the final iterate come from their second-order expansion around the last evaluation point
//    (the last step d satisfies |d|³ ≲ tol), so the caller does not re-evaluate them.
// Typical cost: 3 exponentials per root (the Newton version with re-evaluation needed 5-6).
__device__ __forceinline__ float find_alpha_ts(float t, float c, float b, float& th, float& s2) {
  const float delta = 2.0f * fabsf(c);
  float lo = t - delta, hi = t + delta;
  tanh_sech2(t + b, th, s2);
  if (lo == hi) return lo;  // empty bracket, planar_layer.jl:171-173
  const float tol = 1.2e-7f * (fabsf(t) + delta) + 1e-30f;
  float x = fminf(fmaxf(fmaf(-c, th, t), lo), hi);
  float d = 0.0f;  // x − (point at which th, s2 were evaluated)
  bool stale = true;
#pragma unroll 1
  for (int it = 0; it < 64; ++it) {
    tanh_sech2(x + b, th, s2);
    const float f = fmaf(c, th, x) - t;
    stale = false;
    if (f == 0.0f) break;
    if (f < 0.0f) lo = x; else hi = x;
    const float r = __frcp_rn(fmaf(c, s2, 1.0f));  // 1/f1 (f1 > 0: wᵀû > −1)
    const float n = f * r;
    const float cs = c * s2 * r;
    const float a = -cs * th;                                          // f2/(2 f1)
    const float b3 = -cs * fmaf(-2.0f * th, th, s2) * (1.0f / 3.0f);   // f3/(6 f1)
    const float na = n * a;
    const bool series_ok = fabsf(na) <= 0.25f;
    float xn = series_ok ? fmaf(-n, 1.0f + na, x) : x - n;
    // predicted error of xn: the cubic term of the Chebyshev iteration plus a bound of the quartic one
    // (|d⁴tanh| <= 4.1); only trusted for steps well inside tanh's unit length scale (far out in the saturated
    // region all local derivatives vanish although the root is elsewhere)
    const float n2 = n * n;
    const float err = fmaf(fabsf(fmaf(2.0f * a, a, -b3)), fabsf(n2 * n), 0.2f * fabsf(c) * r * n2 * n2);
    const bool inside = xn > lo && xn < hi;
    if (inside && series_ok && fabsf(n) <= 0.25f && err <= tol) {  // converged: accept without re-evaluating
      d = xn - x;
      x = xn;
      break;
    }
    if (!inside) {
      xn = 0.5f * (lo + hi);
      if (!(xn > lo && xn < hi)) break;  // bracket is adjacent floats
    }
    x = xn;
    stale = true;
  }
  if (stale) {  // iteration cap reached (never observed): th, s2 must match the returned point
    tanh_sech2(x + b, th, s2);
  } else {
    const float ts = th * s2;                       // d/dx tanh = sech², d²/dx² tanh = −2·tanh·sech²
    const float q = s2 * fmaf(-2.0f * th, th, s2);  // −(d²/dx² sech²)/2 = sech²(sech² − 2tanh²)
    th = fmaf(d, fmaf(-d, ts, s2), th);
    s2 = fmaf(-d, fmaf(d, q, 2.0f * ts), s2);
  }
  return x;
}

// Table-driven find_alpha for the fused planar chain kernels.  With u = α + b and s = t + b the equation reads
// u + c·tanh(u) = s, so the root is a ONE-dimensional function u = G_c(s) of the column's scalar s for a fixed layer.
// Every CTA tabulates G_c on [−R, R] (R = 9.5 + |c|; beyond it tanh is ±1 in fp32 and u = s ∓ c exactly) as PT_N cubic
// Hermite pieces (nodes solved with find_alpha_ts, slope 1/(1 + c·sech²u)) in its prologue; a column then takes
//   lookup (one LDS.128 + Horner) -> ONE Newton step (one tanh evaluation) -> tanh / sech² at the root by expansion,
// about a third of the instructions and half the dependent latency of the safeguarded iteration, which the whole warp
// falls back to (warp vote) whenever some lane's step is not tiny or its predicted error exceeds the tolerance of
// find_alpha_ts -- e.g. for c -> −1, where G_c has an infinite slope at 0.  Results are pinned by the residual of the
// equation exactly as before (test/normalising_flows.jl:47-71).
constexpr int PT_N = 128;                 // Hermite pieces per layer
constexpr int PT_FLOATS = PT_N * 4 + 4;   // coefficients + {R, PT_N/(2R), -, -}

// piece `i` of layer constant c: coefficients of u(τ), τ in [0, 1], on [−R + i·h, −R + (i+1)·h]
__device__ inline void planar_table_piece(float c, int i, float* tab) {
  const float R = 9.5f + fabsf(c), h = 2.0f * R / PT_N;
  const float s0 = fmaf((float)i, h, -R), s1 = fmaf((float)(i + 1), h, -R);
  float th, q0, q1;
  const float u0 = find_alpha_ts(s0, c, 0.0f, th, q0);
  const float u1 = find_alpha_ts(s1, c, 0.0f, th, q1);
  const float g0 = h / fmaf(c, q0, 1.0f), g1 = h / fmaf(c, q1, 1.0f);  // h·G'(s) = h/(1 + c·sech²u)
  const float d = u1 - u0;
  reinterpret_cast<float4*>(tab)[i] = make_float4(u0, g0, 3.0f * d - 2.0f * g0 - g1, g0 + g1 - 2.0f * d);
  if (i == 0) reinterpret_cast<float4*>(tab)[PT_N] = make_float4(R, (float)PT_N / (2.0f * R), 0.f, 0.f);
}

// the safeguarded iteration as an out-of-line call: the planar layer loop would otherwise carry an inlined copy of a
// loop it almost never runs in its hot body (inlined into each layer of the former unrolled 8-layer program, it made
// the kernel instruction-cache bound)
static __device__ __noinline__ float find_alpha_ts_call(float t, float c, float b, float* th, float* s2) {
  float th_, s2_;
  const float x = find_alpha_ts(t, c, b, th_, s2_);
  *th = th_;
  *s2 = s2_;
  return x;
}

__device__ __forceinline__ float find_alpha_tab(float t, float c, float b, const float* __restrict__ tab, float& th, float& s2) {
  const float4 meta = reinterpret_cast<const float4*>(tab)[PT_N];
  const float s = t + b;
  const float pos = fminf(fmaxf(fmaf(s, meta.y, meta.x * meta.y), 0.0f), (float)PT_N - 0.0078125f);
  const float fi = floorf(pos), tau = pos - fi;
  const float4 q = reinterpret_cast<const float4*>(tab)[(int)fi];
  float u0 = fmaf(fmaf(fmaf(q.w, tau, q.z), tau, q.y), tau, q.x);
  u0 = fabsf(s) < meta.x ? u0 : s - copysignf(c, s);
  tanh_sech2(u0, th, s2);
  const float f = fmaf(c, th, u0) - s;
  const float r = __frcp_rn(fmaf(c, s2, 1.0f));
  const float n = f * r;                 // Newton step
  const float a = c * s2 * r * th;       // −f''/(2f')
  const float tol = 1.2e-7f * (fabsf(t) + 2.0f * fabsf(c)) + 1e-30f;
  const bool ok = fabsf(n) <= 4e-3f && fabsf(a) * n * n <= tol;
  if (__all_sync(0xffffffffu, ok)) {
    const float d = -n;
    const float ts = th * s2;
    const float qq = s2 * fmaf(-2.0f * th, th, s2);
    th = fmaf(d, fmaf(-d, ts, s2), th);
    s2 = fmaf(-d, fmaf(d, qq, 2.0f * ts), s2);
    return (u0 - n) - b;
  }
  float th_, s2_;
  const float x = find_alpha_ts_call(t, c, b, &th_, &s2_);
  th = th_;
  s2 = s2_;
  return x;
}

__device__ __forceinline__ float find_alpha(float t, float c, float b) {
  float th, s2;
  return find_alpha_ts(t, c, b, th, s2);
}

// One RQS element (rational_quadratic_spline.jl:317-357 forward, :183-220 inverse + the forward
// log-Jacobian at the recovered point, interface.jl:276-281).
// Staged tables (see stage_layer), ROW-major so that lanes that work on the same row but land in different bins
// hit different banks: knots Sw[row][KP] (widths) and Sh[row][KP] (heights), padded with +inf up to KP = the next
// power of two >= K1 (a branch-free binary search needs no bound checks), and per (row, bin) the eight per-bin
// constants the reference recomputes for every element:
//   {w_k, 1/w, w, h_k | Δy, s = Δy/w, d_k, d_{k+1} + d_k − 2s}
// Bin k is the reference's 1-based index (searchsortedfirst − 1); bin 0 is the k == 0 branch (:331-343) that
// only raw three-argument-constructor knots can reach.
__host__ __device__ constexpr inline int rqs_kp(int K1) {
  int kp = 2;
  while (kp < K1) kp <<= 1;
  return kp;
}

// K1C > 0: the knot count is a compile-time constant (the common K = 8 bins -> K1 = 9): the bin search unrolls into
// four compare/select steps with immediate offsets and all table addresses fold into constants.
template <bool INV, int K1C = 0>
__device__ __forceinline__ void rqs_element(const float* __restrict__ tab, int K1rt, int KPrt, int Dp, int row, float v,
                                            float& out, float& lj) {
  const int K1 = K1C ? K1C : K1rt;
  const int KP = K1C ? rqs_kp(K1C) : KPrt;
  const float* S = tab + (INV ? Dp * KP : 0) + row * KP;  // heights for the inverse (:191), widths otherwise (:328)
  const float Bs = S[K1 - 1];
  const bool outside = (v <= -Bs) || (v >= Bs);  // identity outside the box, :322-324 / :186-188
  // k = number of knots < v  (searchsortedfirst − 1): branch-free binary search over the padded knots
  int k = 0;
  if constexpr (K1C != 0) {
#pragma unroll
    for (int st = rqs_kp(K1C) >> 1; st >= 1; st >>= 1) k += (S[k + st - 1] < v) ? st : 0;
  } else {
    for (int st = KP >> 1; st >= 1; st >>= 1) k += (S[k + st - 1] < v) ? st : 0;
  }
  k = min(k, K1 - 1);
  const float4* cf = reinterpret_cast<const float4*>(tab + 2 * Dp * KP) + (size_t)(row * K1 + k) * 2;
  const float4 c0 = cf[0], c1 = cf[1];
  const float w_k = c0.x, inv_w = c0.y, w = c0.z, h_k = c0.w;
  const float dy = c1.x, sl = c1.y, d_k = c1.z, ds = c1.w;
  const float d_k1 = ds - d_k + 2.0f * sl;
  float xi, res;
  if (INV) {
    const float yh = v - h_k;
    const float a1 = fmaf(dy, sl - d_k, yh * ds);   // :208
    const float a2 = fmaf(dy, d_k, -yh * ds);       // :210
    const float a3 = -sl * yh;                      // :212
    xi = __fdividef(-2.0f * a3, a2 + sqrtf(fmaf(a2, a2, -4.0f * a1 * a3)));  // :215-217
    res = fmaf(xi, w, w_k);                         // :219
  } else {
    xi = (v - w_k) * inv_w;  // :340
  }
  const float omx = 1.0f - xi, xo = xi * omx;
  const float den = fmaf(ds, xo, sl);               // :346
  const float rden = __fdividef(1.0f, den);
  const float num = sl * sl * fmaf(d_k1 * xi, xi, fmaf(2.0f * sl, xo, d_k * omx * omx));  // :349
  const float l = __logf(num * rden * rden);        // = log(num) − 2·log(den), :350
  if (!INV) res = fmaf(dy * fmaf(sl * xi, xi, d_k * xo), rden, h_k);  // :353-354
  out = outside ? v : res;
  lj = outside ? 0.0f : (INV ? -l : l);
}

// One element of a Stacked block of elementwise laws (stacked.jl:157-166,242-252): code `op` with per-row parameters
// (a, b); `inverse` evaluates Inverse(law) and ITS log-Jacobian.  Returns the transformed value, adds to `lj`.
//   EXP / LOG    exp_log.jl:5-9          SHIFT shift.jl:12-24        SCALE scale.jl:13-31
//   LEAKY_RELU   leaky_relu.jl:16-29 (inverse(b) = LeakyReLU(inv(α)))
//   LOGIT        logit.jl:15-29: y = logit((x−a)/(b−a)), logjac = −log((x−a)(b−x)/(b−a)); the inverse has no method of
//                its own for the log-Jacobian, so it is −logjac at the recovered x (interface.jl:276-281)
//   TRUNCATED    truncated.jl:15-91: x is clamped to [lb, ub] first (Bijectors.jl:95-100); finite/infinite bounds pick
//                logit / log(x−lb) / log(ub−x) / identity; the inverse has its own closed form (:62-76)
__device__ __forceinline__ float ew_apply(int op, bool inverse, float a, float b, float xv, float& lj) {
  switch (op) {
    case B2B_EW_EXP:
    case B2B_EW_LOG: {
      const bool is_exp = (op == B2B_EW_EXP) != inverse;  // inverse(exp) = log
      if (is_exp) {
        lj += xv;
        return expf(xv);
      }
      const float lg = logf(xv);
      lj -= lg;
      return lg;
    }
    case B2B_EW_SHIFT: return inverse ? xv - a : a + xv;
    case B2B_EW_SCALE: {
      const float la = logf(fabsf(a));
      lj += inverse ? -la : la;
      return inverse ? xv / a : a * xv;
    }
    case B2B_EW_LEAKY_RELU: {
      const float al = inverse ? 1.0f / a : a;
      if (xv < 0.f) {
        lj += logf(fabsf(al));
        return al * xv;
      }
      return xv;
    }
    case B2B_EW_LOGIT: {
      if (!inverse) {
        const float z = (xv - a) / (b - a);
        lj -= logf((xv - a) * (b - xv) / (b - a));      // logit.jl:24
        return logf(z / (1.0f - z));                      // LogExpFunctions.logit
      }
      const float sg = 1.0f / (1.0f + expf(-xv));         // LogExpFunctions.logistic
      const float x = fmaf(b - a, sg, a);                 // logit.jl:19
      lj += logf((x - a) * (b - x) / (b - a));
      return x;
    }
    case B2B_EW_TRUNCATED: {
      const bool lo = !isinf(a), hi = !isinf(b);
      if (!inverse) {
        const float x = xv < a ? a : (xv > b ? b : xv);   // _clamp, Bijectors.jl:95-100
        if (lo && hi) {
          lj -= logf((x - a) * (b - x) / (b - a));        // truncated.jl:55
          return logf(((x - a) / (b - a)) / (1.0f - (x - a) / (b - a)));
        }
        if (lo) {
          const float lg = logf(x - a);
          lj -= lg;
          return lg;
        }
        if (hi) {
          const float lg = logf(b - x);
          lj -= lg;
          return lg;
        }
        return x;
      }
      float x = xv;
      if (lo && hi) {
        const float ay = fabsf(xv);
        lj += logf(b - a) - ay - 2.0f * softplus(-ay);    // truncated.jl:70
        x = fmaf(b - a, 1.0f / (1.0f + expf(-xv)), a);
      } else if (lo) {
        lj += xv;
        x = expf(xv) + a;
      } else if (hi) {
        lj += xv;
        x = b - expf(xv);
      }
      return x < a ? a : (x > b ? b : x);
    }
    default: return xv;
  }
}

// ---- parameter staging (once per CTA) --------------------------------------------------------------
// Layout of the staged block of one layer (floats, Dp = padded depth, rows >= D are zero):
//   PLANAR    : w[Dp] | û[Dp] | {c = wᵀû, b, -, -}                      (get_u_hat, planar_layer.jl:65-70)
//   RADIAL    : z0[Dp] | {α, β̂, α+β̂, -}                                 (radial_layer.jl:44-45,91-92)
//   BATCHNORM : A[Dp] | C[Dp] | iA[Dp] | iC[Dp] | {Σ(logs − log(v+eps)/2)}   y = A·x + C, x = iA·y + iC
//   RQS       : Sw[Dp][KP] | Sh[Dp][KP] | per-(row,bin) constants float4 x 2 [Dp][K1]  ((2·KP + 8·K1)·Dp floats)
//   PERMUTE   : src_of_dst[Dp] (int)
//   STACKED_EW: code[Dp] (int) | a[Dp] | b[Dp]   (ELEMENTWISE_VEC: the same table, code = n0 and b = 0 on every row)
//   MVNORMAL  : mu[Dp] | 1/sigma[Dp] | {−(D·log2π + Σ log σ²)/2}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// RQS tables staged by ALL threads of the CTA, one (row, knot) pair per thread: the per-warp version below walks the
// KP knots of a row serially (KP x ~8 dependent-latency global loads and two divisions, with the other warps
// idle at the barrier).  Same table layout as stage_layer(B2B_RQS).
__device__ inline void stage_rqs_cta(const b2b_layer_desc& d, float* sm, int D, int Dp, int tid, int nthreads) {
  const int K1 = d.n0, KP = rqs_kp(K1);
  float* Sw = sm;
  float* Sh = sm + Dp * KP;
  float4* cf = reinterpret_cast<float4*>(sm + 2 * Dp * KP);
  const float inf = __int_as_float(0x7f800000);
  for (int idx = tid; idx < Dp * KP; idx += nthreads) {
    const int k = idx / Dp, i = idx - k * Dp;  // consecutive threads -> consecutive rows (coalesced parameter reads)
    const bool in = i < D, kin = k < K1;
    Sw[i * KP + k] = kin ? (in ? d.p0[(size_t)k * D + i] : 0.f) : inf;
    Sh[i * KP + k] = kin ? (in ? d.p1[(size_t)k * D + i] : 0.f) : inf;
    if (!kin) continue;
    float w_k = 0.f, w = 1.f, h_k = 0.f, dy = 1.f, d_k = 1.f, d_k1 = 1.f;
    if (in) {
      const float Wl = d.p0[(size_t)(K1 - 1) * D + i], Hl = d.p1[(size_t)(K1 - 1) * D + i];
      w_k = k == 0 ? -Wl : d.p0[(size_t)(k - 1) * D + i];              // rational_quadratic_spline.jl:331
      w = d.p0[(size_t)k * D + i] - w_k;                               // :332
      h_k = k == 0 ? -Hl : d.p1[(size_t)(k - 1) * D + i];              // :335
      dy = d.p1[(size_t)k * D + i] - h_k;                              // :336
      d_k = k == 0 ? 1.0f : d.p2[(size_t)(k - 1) * D + i];             // :342
      d_k1 = k == K1 - 1 ? 1.0f : d.p2[(size_t)k * D + i];             // :343
    }
    const float sl = dy / w;                                           // :339
    cf[(size_t)(i * K1 + k) * 2 + 0] = make_float4(w_k, 1.0f / w, w, h_k);
    cf[(size_t)(i * K1 + k) * 2 + 1] = make_float4(dy, sl, d_k, d_k1 + d_k - 2.0f * sl);
  }
}

// Executed by ONE warp per layer (different warps stage different layers concurrently).
__device__ inline void stage_layer(const b2b_layer_desc& d, float* sm, int D, int Dp, int lane) {
  switch (d.kind) {
    case B2B_PLANAR: {
      float s = 0.f, q = 0.f;
      for (int i = lane; i < D; i += 32) {
        const float w = d.p0[i], u = d.p1[i];
        s = fmaf(w, u, s);
        q = fmaf(w, w, q);
      }
      s = warp_sum(s);
      q = warp_sum(q);
      const float k = (softplus(-s) - 1.0f) / q;  // planar_layer.jl:67
      for (int i = lane; i < Dp; i += 32) {
        const bool in = i < D;
        const float w = in ? d.p0[i] : 0.f;
        sm[i] = w;
        sm[Dp + i] = in ? fmaf(k, w, d.p1[i]) : 0.f;
      }
      if (lane == 0) {
        sm[2 * Dp + 0] = softplus(s) - 1.0f;  // wᵀû, planar_layer.jl:68
        sm[2 * Dp + 1] = d.p2[0];             // first(flow.b), :75
      }
    } break;
    case B2B_RADIAL: {
      for (int i = lane; i < Dp; i += 32) sm[i] = i < D ? d.p2[i] : 0.f;
      if (lane == 0) {
        const float alpha = softplus(d.p0[0]);  // radial_layer.jl:44
        const float apb = softplus(d.p1[0]);    // α + β̂, :45,:92
        sm[Dp + 0] = alpha;
        sm[Dp + 1] = apb - alpha;
        sm[Dp + 2] = apb;
      }
    } break;
    case B2B_BATCHNORM: {
      // y = s·(x − m)/sqrt(v+eps) + b = A·x + C  (normalise.jl:66);  x = (y − b)/s·sqrt(v+eps) + m = iA·y + iC (:84)
      float lj = 0.f;
      for (int i = lane; i < Dp; i += 32) {
        const bool in = i < D;
        float A = 0.f, iA = 0.f, Cc = 0.f, iC = 0.f;
        if (in) {
          const float ve = d.p3[i] + d.f0;
          const float sd = sqrtf(ve);
          const float sc = expf(d.p1[i]);
          A = sc / sd;
          iA = sd / sc;
          Cc = fmaf(-d.p2[i], A, d.p0[i]);
          iC = fmaf(-d.p0[i], iA, d.p2[i]);
          lj += d.p1[i] - logf(ve) * 0.5f;  // normalise.jl:67
        }
        sm[i] = A;
        sm[Dp + i] = Cc;
        sm[2 * Dp + i] = iA;
        sm[3 * Dp + i] = iC;
      }
      lj = warp_sum(lj);
      if (lane == 0) sm[4 * Dp] = lj;
    } break;
    case B2B_RQS: {
      // row-major knots (padded with +inf) for the bin search + per-(row,bin) constants (see rqs_element); padded
      // rows get a zero-width box, i.e. the identity with zero log-Jacobian
      const int K1 = d.n0, KP = rqs_kp(K1);
      float* Sw = sm;
      float* Sh = sm + Dp * KP;
      float4* cf = reinterpret_cast<float4*>(sm + 2 * Dp * KP);
      const float inf = __int_as_float(0x7f800000);
      for (int i = lane; i < Dp; i += 32) {
        const bool in = i < D;
        for (int k = 0; k < KP; ++k) {
          const bool kin = k < K1;
          Sw[i * KP + k] = kin ? (in ? d.p0[(size_t)k * D + i] : 0.f) : inf;
          Sh[i * KP + k] = kin ? (in ? d.p1[(size_t)k * D + i] : 0.f) : inf;
          if (!kin) continue;
          float w_k = 0.f, w = 1.f, h_k = 0.f, dy = 1.f, d_k = 1.f, d_k1 = 1.f;
          if (in) {
            const float Wl = d.p0[(size_t)(K1 - 1) * D + i], Hl = d.p1[(size_t)(K1 - 1) * D + i];
            w_k = k == 0 ? -Wl : d.p0[(size_t)(k - 1) * D + i];              // :331
            w = d.p0[(size_t)k * D + i] - w_k;                               // :332
            h_k = k == 0 ? -Hl : d.p1[(size_t)(k - 1) * D + i];              // :335
            dy = d.p1[(size_t)k * D + i] - h_k;                              // :336
            d_k = k == 0 ? 1.0f : d.p2[(size_t)(k - 1) * D + i];             // :342
            d_k1 = k == K1 - 1 ? 1.0f : d.p2[(size_t)k * D + i];             // :343
          }
          const float sl = dy / w;                                           // :339
          cf[(size_t)(i * K1 + k) * 2 + 0] = make_float4(w_k, 1.0f / w, w, h_k);
          cf[(size_t)(i * K1 + k) * 2 + 1] = make_float4(dy, sl, d_k, d_k1 + d_k - 2.0f * sl);
        }
      }
    } break;
    case B2B_PERMUTE: {
      int* sp = reinterpret_cast<int*>(sm);
      for (int i = lane; i < Dp; i += 32) {
        if (i >= D) sp[i] = i;
        else if (d.inverse) sp[i] = d.i0[i];  // inverse: y[i] = x[dst[i]]  (Permute(transpose(A)), permute.jl:153)
      }
      if (!d.inverse)
        for (int i = lane; i < D; i += 32) sp[d.i0[i]] = i;  // y[dst[i]] = x[i], permute.jl:95-97,152
    } break;
    case B2B_STACKED_EW: {
      int* sc = reinterpret_cast<int*>(sm);
      for (int i = lane; i < Dp; i += 32) {
        sc[i] = i < D ? d.i0[i] : B2B_EW_IDENTITY;
        sm[Dp + i] = (i < D && d.p0) ? d.p0[i] : 0.f;
        sm[2 * Dp + i] = (i < D && d.p1) ? d.p1[i] : 0.f;
      }
    } break;
    case B2B_ELEMENTWISE_VEC: {
      int* sc = reinterpret_cast<int*>(sm);
      for (int i = lane; i < Dp; i += 32) {
        sc[i] = i < D ? d.n0 : B2B_EW_IDENTITY;
        sm[Dp + i] = i < D ? d.p0[i] : 0.f;
        sm[2 * Dp + i] = 0.f;
      }
    } break;
    case B2B_MVNORMAL_DIAG: {
      float ls = 0.f;
      for (int i = lane; i < Dp; i += 32) {
        const bool in = i < D;
        const float sg = (in && d.p1) ? d.p1[i] : 1.0f;
        sm[i] = (in && d.p0) ? d.p0[i] : 0.f;
        sm[Dp + i] = in ? 1.0f / sg : 0.f;
        if (in) ls += logf(sg * sg);
      }
      ls = warp_sum(ls);
      if (lane == 0) sm[2 * Dp] = -0.5f * (D * 1.8378770664093453f + ls);
    } break;
    default: break;
  }
}

}  // namespace b2b
