// Reverse mode of Float64 chains (include/b2b.h: b2b_chain_vjp_f64).
//
// The Float64 counterpart of b2b_chain_vjp_f32, laid out like the Float64 forward (b2b_chain_f64.cu): one warp per column,
// the column in shared memory, lanes over rows, row reductions by warp shuffles.  A correctness path, not a tuned one.
//
// A fixed number of resident warps walks the columns, each warp taking columns gw, gw + W, gw + 2W, ...  Per column:
//   1. forward recompute with f64_layer_forward (the forward kernel's own arithmetic), storing every layer's input
//      column in the warp's tape (L·D doubles of the workspace);
//   2. the terminal MvNormal, if any, adds its x-cotangent to ȳ;
//   3. the reverse sweep, last layer to first, moves the cotangent ȳ → x̄ in shared memory; l̄ is shared by every layer.
// Parameter cotangents accumulate in the warp's slot of the workspace: entries of row i are owned by lane i mod 32
// (coupling W̄ / c̄: lane j mod 32 of the row j of [s; t]), per-column scalars by lane 0, so every address has one writer
// and a fixed summation order.  A reduce kernel then sums the warps in order, and a finalize kernel writes the caller's
// arrays, applying the chain rules that are linear in the sums: get_u_hat for planar w̄ / ū (planar_layer.jl:65-70) and
// log1pexp for radial α_, β (radial_layer.jl:44-45).
//
// Reverse rules (the float64 restatements in oracle/oracle_np.py and tests/chain_vjp_oracle.py): planar inverse by the
// implicit-function rule of find_alpha (ext/BijectorsChainRulesCoreExt.jl:42-46); radial inverse differentiates compute_r
// implicitly (radial_layer.jl:124-129); RQS through the knots of the bin, with the k = 0 / k = K edges and pass-through
// outside the box; coupling through the pullback of `combine` (ext/BijectorsChainRulesCoreExt.jl:48-62).
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "b2b_f64_device.cuh"

namespace b2b {
namespace {

constexpr int V64_WARPS = 4;                         // warps per CTA (fewer when 4·D doubles per warp do not fit)
// CTAs walking the columns at most: 4 per SM of the H100 SXM (132 SMs).  A constant rather than the device's SM count, so
// the workspace query needs no device and the warp count -- hence the order in which parameter cotangents are summed and
// the bits of the result -- does not depend on the GPU that runs the call.  Another SM count changes occupancy only.
constexpr int V64_MAX_CTAS = 132 * 4;
constexpr size_t V64_BUDGET = (size_t)256 << 20;     // bytes of per-warp slots above which fewer warps are used
constexpr int V64_SMEM_MAX = 227 * 1024;             // dynamic shared memory of one CTA on sm_90
constexpr int V64_FIN_THREADS = 256;

struct V64Params {
  const double* x;
  const double* ybar;
  const double* ljbar;
  double* xbar;
  double* ws;                    // warp slots: [tape: T doubles][accumulators: P doubles], `stride` doubles apart
  long long N, ldx, ldyb, ldxb, stride, T;
  int D, L, Lf, wpc;             // Lf: layers before the terminal MvNormal (L or L - 1)
  unsigned want;                 // bit l: accumulate the parameter cotangents of layer l
  long long off[B2B_MAX_CHAIN];  // offset of layer l's accumulators in the accumulator area
  b2b_layer_desc_f64 layers[B2B_MAX_CHAIN];
};

struct V64Fin {
  const double* red;  // the accumulator area summed over the warps
  double* bars[4 * B2B_MAX_CHAIN];
  long long off[B2B_MAX_CHAIN];
  int D;
  b2b_layer_desc_f64 layers[B2B_MAX_CHAIN];
};

// (f′, ∂log|f′|/∂x) of one Stacked law at x, including _clamp's zero derivative outside [lb, ub] (Bijectors.jl:95-100)
__device__ __forceinline__ void law_deriv64(int op, bool inverse, double a, double b, double x, double& f, double& dl) {
  f = 1.0;
  dl = 0.0;
  switch (op) {
    case B2B_EW_EXP:
    case B2B_EW_LOG:
      if ((op == B2B_EW_EXP) != inverse) {
        f = exp(x);
        dl = 1.0;
      } else {
        f = 1.0 / x;
        dl = -1.0 / x;
      }
      break;
    case B2B_EW_SCALE: f = inverse ? 1.0 / a : a; break;
    case B2B_EW_LEAKY_RELU: f = x < 0.0 ? (inverse ? 1.0 / a : a) : 1.0; break;
    case B2B_EW_LOGIT:
      if (!inverse) {
        f = 1.0 / (x - a) + 1.0 / (b - x);
        dl = 1.0 / (b - x) - 1.0 / (x - a);
      } else {
        const double s = 1.0 / (1.0 + exp(-x));
        f = (b - a) * s * (1.0 - s);
        dl = 1.0 - 2.0 * s;
      }
      break;
    case B2B_EW_TRUNCATED: {
      const bool lo = !isinf(a), hi = !isinf(b);
      if (!inverse) {
        if (!(x >= a && x <= b)) {
          f = 0.0;
        } else if (lo && hi) {
          f = 1.0 / (x - a) + 1.0 / (b - x);
          dl = 1.0 / (b - x) - 1.0 / (x - a);
        } else if (lo) {
          f = 1.0 / (x - a);
          dl = -f;
        } else if (hi) {
          f = -1.0 / (b - x);
          dl = 1.0 / (b - x);
        }
        break;
      }
      double xo = x;
      if (lo && hi) {
        const double s = 1.0 / (1.0 + exp(-x));
        xo = (b - a) * s + a;
        f = (b - a) * s * (1.0 - s);
        dl = 1.0 - 2.0 * s;
      } else if (lo || hi) {
        const double e = exp(x);
        xo = lo ? e + a : b - e;
        f = lo ? e : -e;
        dl = 1.0;
      }
      if (xo < a || xo > b) f = 0.0;
    } break;
    default: break;  // IDENTITY, SHIFT
  }
}

// v := Tᵀ v in place for a triangular T (column k of T read coalesced, a warp sum per entry): for an upper T entry k reads
// the v_i with i < k, so k runs downwards; for a lower T upwards.
__device__ __forceinline__ void f64_tri_tmul(const double* Tm, bool up, bool unit, int D, int lane, double* v) {
  for (int kk = 0; kk < D; ++kk) {
    const int k = up ? D - 1 - kk : kk;
    double p = 0.0;
    for (int i = (up ? 0 : k + 1) + lane; i < (up ? k : D); i += 32) p += Tm[(size_t)k * D + i] * v[i];
    p = wsum(p);
    if (lane == 0) v[k] = p + (unit ? v[k] : Tm[(size_t)k * D + k] * v[k]);
    __syncwarp();
  }
}

// v := T⁻ᵀ v in place for a triangular T: Tᵀ v̄ = v, v̄ᵢ = (vᵢ − Σ_k T(k, i)·v̄_k)/Tᵢᵢ over the finished k of column i
__device__ __forceinline__ void f64_tri_tsolve(const double* Tm, bool up, bool unit, int D, int lane, double* v) {
  for (int ii = 0; ii < D; ++ii) {
    const int i = up ? ii : D - 1 - ii;
    double p = 0.0;
    for (int k = (up ? 0 : i + 1) + lane; k < (up ? i : D); k += 32) p += Tm[(size_t)i * D + k] * v[k];
    p = wsum(p);
    if (lane == 0) v[i] = (v[i] - p) / (unit ? 1.0 : Tm[(size_t)i * D + i]);
    __syncwarp();
  }
}

// acc(i, j) += sg·a_i·b_j on the strict lower triangle (lower) or on the upper one with the diagonal, where the diagonal
// also takes dsg/F(j, j); acc and F are D x D column-major.  Entry (i, j) has one writer lane, (i − i₀(j)) mod 32.
__device__ __forceinline__ void f64_lu_acc(double* acc, bool lower, const double* a, const double* b, double sg,
                                           const double* F, double dsg, int D, int lane) {
  for (int j = 0; j < D; ++j) {
    double* Ac = acc + (size_t)j * D;
    const double bj = sg * b[j];
    for (int i = (lower ? j + 1 : 0) + lane; i < (lower ? D : j + 1); i += 32)
      Ac[i] += i == j ? a[i] * bj + dsg / F[(size_t)j * D + j] : a[i] * bj;
  }
  __syncwarp();  // a and b were read with a lane mapping that shifts with j
}

// Reverse mode of one layer at its input column `col`: g (the cotangent of the layer's output) becomes the cotangent of
// its input; `acc` (NULL: not wanted) receives this column's parameter cotangents.  All 32 lanes call it; ends synced.
// LU = false leaves SCALE_LU out (chain_vjp_f64_kernel<false>: the chains without the layer).
template <bool LU>
__device__ __forceinline__ void layer_vjp(const b2b_layer_desc_f64& d, int D, int lane, const double* col, double* g,
                                          double* t1, double* t2, double lb, double* acc) {
  const bool inv = d.inverse != 0;
  switch (d.kind) {
    case B2B_PLANAR: {  // accumulators: Σ ȳ·∂y/∂û [D] | direct w̄ [D] | c̄ | b̄
      double s = 0.0, q = 0.0, wz = 0.0;
      for (int i = lane; i < D; i += 32) {
        const double w = d.p0[i];
        s += w * d.p1[i];
        q += w * w;
        wz += w * col[i];
      }
      s = wsum(s);
      q = wsum(q);
      wz = wsum(wz);
      const double kk = (softplus64(-s) - 1.0) / q;
      const double c = softplus64(s) - 1.0, b = d.p2[0];
      double ug = 0.0;
      for (int i = lane; i < D; i += 32) ug += (d.p1[i] + kk * d.p0[i]) * g[i];
      ug = wsum(ug);  // ûᵀȳ
      double th, s2, ga, tc, cb;  // ga: cotangent of wᵀx; y = x + û·tc; cb: c̄
      if (!inv) {
        tanh_sech2_64(wz + b, th, s2);
        const double den = 1.0 + c * s2;
        ga = s2 * ug - lb * (2.0 * c * th * s2 / den);
        cb = lb * s2 / den;
        tc = th;
      } else {
        find_alpha64(wz, c, b, th, s2);
        const double X = 1.0 / (1.0 + c * s2);  // ∂α/∂(wᵀy); ∂α/∂c = −tanh·X, ∂α/∂b = X − 1
        const double abar = -s2 * ug + lb * (2.0 * c * th * s2 * X);
        cb = -lb * s2 * X - abar * th * X;
        ga = abar * X;
        tc = -th;
      }
      if (acc) {
        for (int i = lane; i < D; i += 32) {
          acc[i] += g[i] * tc;
          acc[D + i] += col[i] * ga;
        }
        if (lane == 0) {
          acc[2 * D] += cb;
          acc[2 * D + 1] += ga;  // b̄: a = wᵀx + b (forward), a = α + b with ∂α/∂b = X − 1 (inverse)
        }
      }
      for (int i = lane; i < D; i += 32) g[i] += d.p0[i] * ga;
    } break;
    case B2B_RADIAL: {  // accumulators: z̄_0 [D] | Σ ∂/∂α | Σ ∂/∂β̂
      const double alpha = softplus64(d.p0[0]), A = softplus64(d.p1[0]), bh = A - alpha;
      double r2 = 0.0, dg = 0.0;
      for (int i = lane; i < D; i += 32) {
        const double dd = col[i] - d.p2[i];
        r2 += dd * dd;
        dg += dd * g[i];
      }
      const double nrm = sqrt(wsum(r2));
      dg = wsum(dg);
      double r = nrm;
      if (inv) {
        const double a = A - nrm;
        const double sq = sqrt(a * a + 4.0 * alpha * nrm);
        r = a > 0.0 ? (2.0 * alpha * nrm) / (sq + a) : 0.5 * (sq - a);
      }
      const double h = 1.0 / (alpha + r), sv = bh * h, qv = bh * r * h * h;
      const double Fs = (double)(D - 1) / (1.0 + sv) + 1.0 / (1.0 + sv - qv), Fq = -1.0 / (1.0 + sv - qv);
      double alpha_bar, bh_bar, scale, kappa;  // new g = g·scale + δ·kappa
      if (!inv) {
        const double s_tot = dg + lb * Fs, q_bar = lb * Fq;
        bh_bar = s_tot * h + q_bar * r * h * h;
        const double h_bar = s_tot * bh + q_bar * 2.0 * bh * r * h;
        const double r_bar = q_bar * bh * h * h - h_bar * h * h;
        alpha_bar = -h_bar * h * h;
        kappa = r > 0.0 ? r_bar / r : 0.0;
        scale = 1.0 + sv;
      } else {
        const double Ar = A + r, h3 = h * h * h, F_bar = -lb;
        const double dF_dr = Fs * (-bh * h * h) + Fq * (bh * h * h - 2.0 * bh * r * h3);
        const double dF_da = Fs * (-bh * h * h) + Fq * (-2.0 * bh * r * h3);
        const double dF_db = Fs * h + Fq * (r * h * h);
        const double r_bar = dg * bh / (Ar * Ar) + F_bar * dF_dr;
        const double m = 2.0 * r + A - nrm;  // ∂/∂r of r² + (A − γ)r − αγ
        const double A_bar = dg * (-(alpha + r) / (Ar * Ar)) + r_bar * (-r / m);
        alpha_bar = dg / Ar + F_bar * dF_da + r_bar * nrm / m + A_bar;
        bh_bar = F_bar * dF_db + A_bar;
        const double gam_bar = r_bar * (alpha + r) / m;
        kappa = nrm > 0.0 ? gam_bar / nrm : 0.0;
        scale = (alpha + r) / Ar;
      }
      for (int i = lane; i < D; i += 32) {
        const double dd = col[i] - d.p2[i], ng = g[i] * scale + dd * kappa;
        if (acc) acc[i] += g[i] - ng;  // z_0 enters as x − z_0 and (inverse) z = z_0 + ρ(y − z_0)
        g[i] = ng;
      }
      if (acc && lane == 0) {
        acc[D] += alpha_bar;
        acc[D + 1] += bh_bar;
      }
    } break;
    case B2B_RQS: {  // accumulators: W̄ | H̄ | D̄, each D x K1 like the knot arrays
      const int K1 = d.n0;
      const double *Wd = d.p0, *Hd = d.p1, *Dv = d.p2;
      for (int i = lane; i < D; i += 32) {
        const double v = col[i];
        const double* S = inv ? Hd : Wd;
        const double Bs = S[(size_t)(K1 - 1) * D + i];
        if (v <= -Bs || v >= Bs) continue;  // identity outside the box: ȳ passes through
        int k = 0;
        while (k < K1 && S[(size_t)k * D + i] < v) ++k;
        if (k > K1 - 1) k = K1 - 1;
        const double xk = k == 0 ? -Wd[(size_t)(K1 - 1) * D + i] : Wd[(size_t)(k - 1) * D + i];
        const double xk1 = Wd[(size_t)k * D + i];
        const double yk = k == 0 ? -Hd[(size_t)(K1 - 1) * D + i] : Hd[(size_t)(k - 1) * D + i];
        const double yk1 = Hd[(size_t)k * D + i];
        const double dk = k == 0 ? 1.0 : Dv[(size_t)(k - 1) * D + i];
        const double dk1 = k == K1 - 1 ? 1.0 : Dv[(size_t)k * D + i];
        const double w = xk1 - xk, dyv = yk1 - yk, s = dyv / w, dsv = dk1 + dk - 2.0 * s;
        double xi;
        if (inv) {
          const double yh = v - yk;
          const double a1 = dyv * (s - dk) + yh * dsv, a2 = dyv * dk - yh * dsv, a3 = -s * yh;
          xi = -2.0 * a3 / (a2 + sqrt(a2 * a2 - 4.0 * a1 * a3));
        } else {
          xi = (v - xk) / w;
        }
        const double o = 1.0 - xi, p = xi * o, den = s + dsv * p, a = s * xi * xi + dk * p, num = dyv * a;
        const double bq = dk1 * xi * xi + 2.0 * s * p + dk * o * o;
        double yb = g[i], lbe = lb, ystar = 0.0;
        if (inv) {  // inverse-function theorem at the recovered x
          const double f_x = s * s * bq / (den * den);
          const double b_xi = 2.0 * dk1 * xi + 2.0 * s * (1.0 - 2.0 * xi) - 2.0 * dk * o;
          const double den_xi = dsv * (1.0 - 2.0 * xi);
          const double lj_x = (b_xi / bq - 2.0 * den_xi / den) / w;
          ystar = (g[i] - lb * lj_x) / f_x;
          yb = -ystar;
          lbe = -lb;
        }
        const double num_b = yb / den;
        const double den_b = -yb * num / (den * den) - 2.0 * lbe / den;
        double yk_b = yb;
        const double b_b = lbe / bq;
        double s_b = 2.0 * lbe / s;
        double dyv_b = num_b * a;
        const double a_b = num_b * dyv;
        s_b += a_b * xi * xi;
        double xi_b = a_b * 2.0 * s * xi;
        double dk_b = a_b * p;
        double p_b = a_b * dk;
        double dk1_b = b_b * xi * xi;
        xi_b += b_b * 2.0 * dk1 * xi;
        s_b += b_b * 2.0 * p;
        p_b += b_b * 2.0 * s;
        dk_b += b_b * o * o;
        double o_b = b_b * 2.0 * dk * o;
        s_b += den_b;
        const double ds_b = den_b * p;
        p_b += den_b * dsv;
        dk1_b += ds_b;
        dk_b += ds_b;
        s_b -= 2.0 * ds_b;
        xi_b += p_b * o;
        o_b += p_b * xi;
        xi_b -= o_b;
        const double x_b = xi_b / w;
        double xk_b = -xi_b / w;
        double w_b = -xi_b * xi / w;
        dyv_b += s_b / w;
        w_b -= s_b * s / w;
        const double yk1_b = dyv_b;
        yk_b -= dyv_b;
        const double xk1_b = w_b;
        xk_b -= w_b;
        g[i] = inv ? ystar : x_b;
        if (acc) {
          double *Wb = acc, *Hb = acc + (size_t)D * K1, *Db = acc + 2 * (size_t)D * K1;
          if (k >= 1) {
            Wb[(size_t)(k - 1) * D + i] += xk_b;
            Hb[(size_t)(k - 1) * D + i] += yk_b;
            Db[(size_t)(k - 1) * D + i] += dk_b;
          } else {  // x_0 = −widths[end], y_0 = −heights[end]; d_0 = 1 is a constant
            Wb[(size_t)(K1 - 1) * D + i] -= xk_b;
            Hb[(size_t)(K1 - 1) * D + i] -= yk_b;
          }
          Wb[(size_t)k * D + i] += xk1_b;
          Hb[(size_t)k * D + i] += yk1_b;
          if (k < K1 - 1) Db[(size_t)k * D + i] += dk1_b;  // d_K = 1 is a constant
        }
      }
    } break;
    case B2B_COUPLING_AFFINE: {  // accumulators: W̄ [2n1 x n2, column-major] | c̄ [2n1]
      const int n1 = d.n0, n2 = d.n1;
      for (int j = lane; j < n1; j += 32) {  // s̄ → t1, t̄ → t2; x̄₁ in place
        double sv = d.p1 ? d.p1[j] : 0.0, tv = d.p1 ? d.p1[n1 + j] : 0.0;
        for (int k = 0; k < n2; ++k) {
          const double xk = col[d.i1 ? d.i1[k] : d.n3 + k];
          sv += d.p0[(size_t)k * (2 * n1) + j] * xk;
          tv += d.p0[(size_t)k * (2 * n1) + n1 + j] * xk;
        }
        const int r = d.i0 ? d.i0[j] : d.n2 + j;
        const double yb1 = g[r];
        if (!inv) {  // y₁ = e^s x₁ + t, lj = Σ s
          const double e = exp(sv);
          t1[j] = yb1 * e * col[r] + lb;
          t2[j] = yb1;
          g[r] = e * yb1;
        } else {  // x₁ = (y₁ − t) e^−s, lj = −Σ s
          const double em = exp(-sv);
          t1[j] = -((col[r] - tv) * em) * yb1 - lb;
          t2[j] = -em * yb1;
          g[r] = em * yb1;
        }
      }
      __syncwarp();
      for (int k = lane; k < n2; k += 32) {  // x̄₂ = ȳ₂ + Wᵀ[s̄; t̄]; rows outside both index lists pass through
        const double* Wk = d.p0 + (size_t)k * (2 * n1);
        double a = 0.0;
        for (int j = 0; j < n1; ++j) a += Wk[j] * t1[j] + Wk[n1 + j] * t2[j];
        g[d.i1 ? d.i1[k] : d.n3 + k] += a;
      }
      if (acc) {
        for (int j = lane; j < 2 * n1; j += 32) {
          const double sb = j < n1 ? t1[j] : t2[j - n1];
          for (int k = 0; k < n2; ++k) acc[(size_t)k * (2 * n1) + j] += sb * col[d.i1 ? d.i1[k] : d.n3 + k];
          acc[(size_t)2 * n1 * n2 + j] += sb;
        }
      }
    } break;
    case B2B_BATCHNORM: {  // accumulators: b̄ [D] | logs̄ [D]
      for (int i = lane; i < D; i += 32) {
        const double ve = d.p3[i] + d.f0, sc = exp(d.p1[i]), A = sc / sqrt(ve), gi = g[i];
        if (!inv) {  // y = A(x − m) + b
          g[i] = A * gi;
          if (acc) {
            acc[i] += gi;
            acc[D + i] += gi * (sc * (col[i] - d.p2[i]) / sqrt(ve)) + lb;
          }
        } else {  // x = (y − b)/A + m
          g[i] = gi / A;
          if (acc) {
            acc[i] -= gi / A;
            acc[D + i] -= gi * ((col[i] - d.p0[i]) / sc * sqrt(ve)) + lb;
          }
        }
      }
    } break;
    case B2B_STACKED_EW: {
      for (int i = lane; i < D; i += 32) {
        double f, dl;
        law_deriv64(d.i0[i], inv, d.p0 ? d.p0[i] : 0.0, d.p1 ? d.p1[i] : 0.0, col[i], f, dl);
        g[i] = g[i] * f + lb * dl;
      }
    } break;
    case B2B_ELEMENTWISE_VEC: {  // accumulators: ā [D]; ∂y/∂a, ∂ℓ/∂a as in b2b_ew_vjp.cu:ew_vec_dparam
      for (int i = lane; i < D; i += 32) {
        const double a = d.p0[i], x = col[i];
        double f, dl;
        law_deriv64(d.n0, inv, a, 0.0, x, f, dl);
        if (acc) {
          double dy = 0.0, da = 0.0;
          if (d.n0 == B2B_EW_SHIFT) {
            dy = inv ? -1.0 : 1.0;
          } else if (d.n0 == B2B_EW_SCALE || x < 0.0) {
            dy = inv ? -x / (a * a) : x;
            da = inv ? -1.0 / a : 1.0 / a;
          }
          acc[i] += g[i] * dy + lb * da;
        }
        g[i] = g[i] * f + lb * dl;
      }
    } break;
    case B2B_SCALE_TRIANGULAR: {  // accumulators: T̄ on 𝒫 packed by columns (column j: rows j..D-1 lower, 0..j upper)
      const double* Tm = d.p0;
      const bool up = d.n0 != 0, unit = d.n1 != 0;
      const double* u = col;  // forward: T̄ += ȳ xᵀ on 𝒫 (+ l̄/Tᵢᵢ);  inverse: T̄ −= x̄ yᵀ on 𝒫 (+ l̄/Tᵢᵢ), y = T⁻¹x in t2
      if (!inv) {
        for (int k = 0; k < D; ++k) {  // x̄_k = Σᵢ T(i, k)·ȳᵢ over column k of T: a coalesced read and a warp sum
          double p = 0.0;
          for (int i = (up ? 0 : k + 1) + lane; i < (up ? k : D); i += 32) p += Tm[(size_t)k * D + i] * g[i];
          p = wsum(p);
          if (lane == 0) t1[k] = p + (unit ? g[k] : Tm[(size_t)k * D + k] * g[k]);
        }
      } else {
        for (int i = lane; i < D; i += 32) t2[i] = col[i];
        __syncwarp();
        f64_tri_solve(d, D, lane, t2);
        for (int ii = 0; ii < D; ++ii) {  // Tᵀ x̄ = ȳ: x̄ᵢ = (ȳᵢ − Σ_k T(k, i)·x̄_k)/Tᵢᵢ over the finished k of column i
          const int i = up ? ii : D - 1 - ii;
          double p = 0.0;
          for (int k = (up ? 0 : i + 1) + lane; k < (up ? i : D); k += 32) p += Tm[(size_t)i * D + k] * t1[k];
          p = wsum(p);
          if (lane == 0) t1[i] = (g[i] - p) / (unit ? 1.0 : Tm[(size_t)i * D + i]);
          __syncwarp();
        }
        u = t2;
      }
      __syncwarp();
      if (acc) {
        const double* gl = inv ? t1 : g;  // the outer product's left factor: ȳ, or −x̄ for the inverse layer
        const double sg = inv ? -1.0 : 1.0;
        for (int j = 0; j < D; ++j) {
          double* Ac = acc + (up ? (size_t)j * (j + 1) / 2 : (size_t)j * D - (size_t)j * (j + 1) / 2);  // T̄(i, j) at Ac[i]
          const double uj = sg * u[j];
          const int i0 = up ? 0 : (unit ? j + 1 : j), i1 = up ? (unit ? j : j + 1) : D;
          for (int i = i0 + lane; i < i1; i += 32) Ac[i] += gl[i] * uj;
          if (!unit && lane == 0) Ac[j] += sg * lb / Tm[(size_t)j * D + j];
        }
      }
      __syncwarp();  // the outer product reads g with a lane mapping that shifts with j: every lane is done with it
      for (int i = lane; i < D; i += 32) g[i] = t1[i];
    } break;
    case B2B_SCALE_LU:  // accumulators: F̄ (D x D column-major, packed like F: L̄ below the diagonal, Ū on and above it)
      if constexpr (LU) {
        const double* F = d.p0;
        const b2b_layer_desc_f64 Uf = f64_lu_factor(d, true), Lf = f64_lu_factor(d, false);
        if (!inv) {  // y = P v, v = L u, u = U x:  v̄ = Pᵀȳ, L̄ += v̄ uᵀ, ū = Lᵀv̄, Ū += ū xᵀ + l̄·diag(1/Uᵢᵢ), x̄ = Uᵀū
          for (int i = lane; i < D; i += 32) t2[i] = col[i];
          __syncwarp();
          f64_tri_forward(Uf, D, lane, t2, t1);
          for (int i = lane; i < D; i += 32) t1[i] = d.i0 ? g[d.i0[i]] : g[i];
          __syncwarp();
          if (acc) f64_lu_acc(acc, true, t1, t2, 1.0, F, 0.0, D, lane);
          f64_tri_tmul(F, false, true, D, lane, t1);
          if (acc) f64_lu_acc(acc, false, t1, col, 1.0, F, lb, D, lane);
          f64_tri_tmul(F, true, false, D, lane, t1);
          for (int i = lane; i < D; i += 32) g[i] = t1[i];
        } else {  // z = U⁻¹ v, v = L⁻¹ w, w = Pᵀ y:  v̄ = U⁻ᵀz̄, Ū −= v̄ zᵀ + l̄·diag(1/Uᵢᵢ), w̄ = L⁻ᵀv̄, L̄ −= w̄ vᵀ, ȳ = P w̄
          for (int i = lane; i < D; i += 32) t2[i] = d.i0 ? col[d.i0[i]] : col[i];
          __syncwarp();
          f64_tri_solve(Lf, D, lane, t2);
          for (int i = lane; i < D; i += 32) t1[i] = t2[i];
          __syncwarp();
          f64_tri_solve(Uf, D, lane, t1);
          f64_tri_tsolve(F, true, false, D, lane, g);
          if (acc) f64_lu_acc(acc, false, g, t1, -1.0, F, -lb, D, lane);
          f64_tri_tsolve(F, false, true, D, lane, g);
          if (acc) f64_lu_acc(acc, true, g, t2, -1.0, F, 0.0, D, lane);
          if (d.i0) f64_lu_permute(d.i0, false, D, lane, g, t1);
        }
      }
      break;
    case B2B_PERMUTE: {
      for (int i = lane; i < D; i += 32) t1[i] = g[i];
      __syncwarp();
      for (int i = lane; i < D; i += 32) {
        if (inv) g[d.i0[i]] = t1[i];  // x[i] = y[dst[i]]
        else g[i] = t1[d.i0[i]];      // y[dst[i]] = x[i]
      }
    } break;
    default: break;
  }
  __syncwarp();
}

// LU: the chain holds a SCALE_LU layer (f64_layer_forward and layer_vjp with its case)
template <bool LU>
__global__ void __launch_bounds__(V64_WARPS * 32) chain_vjp_f64_kernel(const __grid_constant__ V64Params P) {
  extern __shared__ double smv[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, D = P.D;
  double* col = smv + (size_t)warp * 4 * D;  // the layer input
  double* g = col + D;                       // the cotangent
  double* t1 = g + D;                        // scratch (permute, s̄ of coupling)
  double* t2 = t1 + D;                       // scratch (t̄ of coupling)
  const long long gw = (long long)blockIdx.x * P.wpc + warp, W = (long long)gridDim.x * P.wpc;
  double* tape = P.ws + gw * P.stride;
  double* acc = tape + P.T;
  if (P.want)
    for (long long k = lane; k < P.stride - P.T; k += 32) acc[k] = 0.0;
  __syncwarp();
  for (long long n = gw; n < P.N; n += W) {
    for (int i = lane; i < D; i += 32) col[i] = P.x[n * P.ldx + i];
    __syncwarp();
    double lj = 0.0;
    for (int l = 0; l < P.Lf; ++l) {
      for (int i = lane; i < D; i += 32) tape[(size_t)l * D + i] = col[i];
      f64_layer_forward<true, LU>(P.layers[l], D, lane, col, t1, lj);
    }
    const double lb = P.ljbar ? P.ljbar[n] : 0.0;
    for (int i = lane; i < D; i += 32) g[i] = P.ybar ? P.ybar[n * P.ldyb + i] : 0.0;
    if (P.Lf < P.L && P.layers[P.Lf].kind == B2B_MVNORMAL_TRIL) {
      // full-covariance terminal at y = col: r = L⁻¹(y − μ), s = L⁻ᵀr; ȳ −= l̄·s, μ̄ += l̄·s, L̄(i, j) += l̄·sᵢ·r_j (i ≥ j) and
      // L̄(i, i) −= l̄/Lᵢᵢ.  Accumulators: μ̄ [D] | L̄ packed by columns (column j holds rows j..D-1).  The lane writing
      // L̄(i, j) is (i − j) mod 32, the same for every column.
      const b2b_layer_desc_f64& d = P.layers[P.Lf];
      double* a = (P.want >> P.Lf) & 1u ? acc + P.off[P.Lf] : nullptr;
      __syncwarp();
      f64_tril_solve(d, D, lane, col, t1);
      f64_tril_back(d, D, lane, t1, t2);
      for (int i = lane; i < D; i += 32) {
        const double gs = lb * t2[i];
        g[i] -= gs;
        if (a) a[i] += gs;
      }
      if (a && lb != 0.0)
        for (int j = 0; j < D; ++j) {
          double* Lc = a + D + (size_t)j * D - (size_t)j * (j + 1) / 2;  // L̄(i, j) at Lc[i]
          const double rj = lb * t1[j];
          for (int i = j + lane; i < D; i += 32) Lc[i] += t2[i] * rj;
          if (lane == 0) Lc[j] -= lb / d.p1[(size_t)j * D + j];
        }
    } else if (P.Lf < P.L) {  // terminal MvNormal at y = col: q = (y − μ)/σ, ȳ −= l̄·q/σ, μ̄ += l̄·q/σ, σ̄ += l̄·(q² − 1)/σ
      const b2b_layer_desc_f64& d = P.layers[P.Lf];
      double* a = (P.want >> P.Lf) & 1u ? acc + P.off[P.Lf] : nullptr;
      for (int i = lane; i < D; i += 32) {
        const double sg = d.p1 ? d.p1[i] : 1.0, q = (col[i] - (d.p0 ? d.p0[i] : 0.0)) / sg, gq = lb * q / sg;
        g[i] -= gq;
        if (a) {
          a[i] += gq;
          a[D + i] += lb * (q * q - 1.0) / sg;
        }
      }
    }
    __syncwarp();
    for (int l = P.Lf - 1; l >= 0; --l) {
      for (int i = lane; i < D; i += 32) col[i] = tape[(size_t)l * D + i];
      __syncwarp();
      layer_vjp<LU>(P.layers[l], D, lane, col, g, t1, t2, lb, (P.want >> l) & 1u ? acc + P.off[l] : nullptr);
    }
    for (int i = lane; i < D; i += 32) P.xbar[n * P.ldxb + i] = g[i];
    __syncwarp();
  }
}

// red[p] = Σ_w acc_w[p] over the warps in order
__global__ void vjp_f64_reduce_kernel(const double* __restrict__ ws, long long stride, long long T, long long P, int warps,
                                      double* __restrict__ red) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int w = 0; w < warps; ++w) s += ws[(size_t)w * stride + T + p];
    red[p] = s;
  }
}

__device__ double block_sum(double v, double* sh) {  // fixed-order sum over the CTA
  const int t = threadIdx.x;
  sh[t] = v;
  __syncthreads();
  for (int o = V64_FIN_THREADS / 2; o > 0; o >>= 1) {
    if (t < o) sh[t] += sh[t + o];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

// one CTA per layer: the caller's cotangent arrays from the warp sums
__global__ void __launch_bounds__(V64_FIN_THREADS) vjp_f64_finalize_kernel(const __grid_constant__ V64Fin F) {
  __shared__ double sh[V64_FIN_THREADS];
  const int l = blockIdx.x, t = threadIdx.x, D = F.D;
  const b2b_layer_desc_f64& d = F.layers[l];
  const double* r = F.red + F.off[l];
  double* const* bars = F.bars + 4 * l;
  auto copy = [&](double* dst, const double* src, size_t n) {
    if (dst)
      for (size_t i = t; i < n; i += V64_FIN_THREADS) dst[i] = src[i];
  };
  switch (d.kind) {
    case B2B_PLANAR: {
      if (!bars[0] && !bars[1] && !bars[2]) return;
      // get_u_hat: û = u + k(s, q)·w, k = (log1pexp(−s) − 1)/q, s = wᵀu, q = wᵀw; c = log1pexp(s) − 1
      double s = 0.0, q = 0.0, uw = 0.0;
      for (int i = t; i < D; i += V64_FIN_THREADS) {
        s += d.p0[i] * d.p1[i];
        q += d.p0[i] * d.p0[i];
        uw += r[i] * d.p0[i];
      }
      s = block_sum(s, sh);
      q = block_sum(q, sh);
      uw = block_sum(uw, sh);
      const double kk = (softplus64(-s) - 1.0) / q, sig = 1.0 / (1.0 + exp(-s));
      const double dk_ds = -(1.0 / (1.0 + exp(s))) / q, dk_dq = -kk / q, cb = r[2 * D];
      for (int i = t; i < D; i += V64_FIN_THREADS) {
        const double ub = r[i], w = d.p0[i], u = d.p1[i];
        if (bars[1]) bars[1][i] = ub + (uw * dk_ds + cb * sig) * w;
        if (bars[0]) bars[0][i] = r[D + i] + kk * ub + uw * (dk_ds * u + dk_dq * 2.0 * w) + cb * sig * u;
      }
      if (bars[2] && t == 0) bars[2][0] = r[2 * D + 1];
    } break;
    case B2B_RADIAL:  // α = log1pexp(α_), β̂ = log1pexp(β) − α
      if (t == 0) {
        const double bh = r[D + 1];
        if (bars[0]) bars[0][0] = (r[D] - bh) / (1.0 + exp(-d.p0[0]));
        if (bars[1]) bars[1][0] = bh / (1.0 + exp(-d.p1[0]));
      }
      copy(bars[2], r, D);
      break;
    case B2B_RQS:
      for (int i = 0; i < 3; ++i) copy(bars[i], r + (size_t)i * D * d.n0, (size_t)D * d.n0);
      break;
    case B2B_ELEMENTWISE_VEC: copy(bars[0], r, D); break;
    case B2B_COUPLING_AFFINE:
      copy(bars[0], r, (size_t)2 * d.n0 * d.n1);
      copy(bars[1], r + (size_t)2 * d.n0 * d.n1, (size_t)2 * d.n0);
      break;
    case B2B_BATCHNORM:
    case B2B_MVNORMAL_DIAG:
      copy(bars[0], r, D);
      copy(bars[1], r + D, D);
      break;
    case B2B_MVNORMAL_TRIL:  // L̄ unpacked to D x D column-major, zero above the diagonal
      copy(bars[0], r, D);
      if (bars[1])
        for (size_t k = t; k < (size_t)D * D; k += V64_FIN_THREADS) {
          const size_t j = k / D, i = k - j * D;
          bars[1][k] = i >= j ? r[D + j * D - j * (j + 1) / 2 + i] : 0.0;
        }
      break;
    case B2B_SCALE_TRIANGULAR:  // T̄ unpacked to D x D column-major, zero outside 𝒫
      if (bars[0])
        for (size_t k = t; k < (size_t)D * D; k += V64_FIN_THREADS) {
          const size_t j = k / D, i = k - j * D;
          const bool in = d.n0 ? (d.n1 ? i < j : i <= j) : (d.n1 ? i > j : i >= j);
          bars[0][k] = in ? r[(d.n0 ? j * (j + 1) / 2 : j * D - j * (j + 1) / 2) + i] : 0.0;
        }
      break;
    case B2B_SCALE_LU: copy(bars[0], r, (size_t)D * D); break;  // F̄ is accumulated in F's own layout
    default: break;
  }
}

// doubles of parameter-cotangent accumulators of one layer, rounded to 32 (256 bytes)
long long acc_len(const b2b_layer_desc_f64& d, int D) {
  long long n = 0;
  switch (d.kind) {
    case B2B_PLANAR: n = 2LL * D + 2; break;
    case B2B_RADIAL: n = (long long)D + 2; break;
    case B2B_ELEMENTWISE_VEC: n = D; break;
    case B2B_RQS: n = 3LL * D * d.n0; break;
    case B2B_COUPLING_AFFINE: n = 2LL * d.n0 * d.n1 + 2LL * d.n0; break;
    case B2B_BATCHNORM:
    case B2B_MVNORMAL_DIAG: n = 2LL * D; break;
    case B2B_MVNORMAL_TRIL: n = (long long)D + (long long)D * (D + 1) / 2; break;
    case B2B_SCALE_TRIANGULAR: n = (long long)D * (D + 1) / 2; break;
    case B2B_SCALE_LU: n = (long long)D * D; break;
    default: break;
  }
  return (n + 31) & ~31LL;
}

struct V64Plan {
  int Lf, wpc, warps;  // warps: the number the call uses (the workspace holds that many slots)
  long long T, P, stride;
  long long off[B2B_MAX_CHAIN];
  size_t smem, bytes;
};

// Layout of a valid chain (descriptors already validated) for N columns; B2B_EUNSUPPORTED when D > 2048.  The warps are
// one per column up to V64_MAX_CTAS CTAs, fewer when their slots would pass V64_BUDGET, never fewer than one CTA: the
// workspace grows with N only up to that bound.
int v64_plan(const b2b_layer_desc_f64* layers, int L, int D, long long N, V64Plan& p) {
  if (D > 2048) return B2B_EUNSUPPORTED;
  p.Lf = b2b_ends_in_terminal(layers, L) ? L - 1 : L;
  p.T = ((long long)p.Lf * D + 31) & ~31LL;
  p.P = 0;
  for (int l = 0; l < L; ++l) {
    p.off[l] = p.P;
    p.P += acc_len(layers[l], D);
  }
  p.stride = p.T + p.P;
  p.wpc = V64_WARPS;
  while (p.wpc > 1 && (size_t)p.wpc * 4 * D * sizeof(double) > (size_t)V64_SMEM_MAX) --p.wpc;
  p.smem = (size_t)p.wpc * 4 * D * sizeof(double);
  const size_t slot = (size_t)p.stride * sizeof(double);
  long long ctas = (N + p.wpc - 1) / p.wpc;
  if (ctas > V64_MAX_CTAS) ctas = V64_MAX_CTAS;
  long long w = slot ? (long long)(V64_BUDGET / slot) : ctas * p.wpc;
  if (w > ctas * p.wpc) w = ctas * p.wpc;
  w -= w % p.wpc;
  if (w < p.wpc) w = p.wpc;  // one CTA at least, whatever its slots cost
  p.warps = (int)w;
  p.bytes = (size_t)w * slot + (size_t)p.P * sizeof(double) + 256;
  return B2B_OK;
}

}  // namespace
}  // namespace b2b

extern "C" size_t b2b_chain_vjp_workspace_bytes_f64(const b2b_layer_desc_f64* layers, int32_t L, int32_t D, int64_t N) {
  using namespace b2b;
  if (!layers || L < 1 || L > B2B_MAX_CHAIN || D < 1 || N < 0) return 0;
  for (int l = 0; l < L; ++l)
    if (b2b_f64_validate_layer(layers[l], D, l == L - 1) != B2B_OK) return 0;
  V64Plan p;
  if (v64_plan(layers, L, D, N, p) != B2B_OK) return 0;
  return p.bytes;
}

extern "C" int b2b_chain_vjp_f64(const b2b_layer_desc_f64* layers, int32_t L, const double* x, const double* ybar,
                                 const double* ljbar, double* xbar, double* const* param_bars, int32_t D, int64_t N,
                                 int64_t ldx, int64_t ldybar, int64_t ldxbar, void* workspace, size_t workspace_bytes,
                                 void* stream_) {
  using namespace b2b;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  b2b_set_last_launch_count(0);
  if (!layers || L < 1 || L > B2B_MAX_CHAIN || D < 1 || N < 0) return B2B_EINVAL;
  for (int l = 0; l < L; ++l) {
    const int rc = b2b_f64_validate_layer(layers[l], D, l == L - 1);
    if (rc != B2B_OK) return rc;
  }
  V64Plan plan;
  int rc = v64_plan(layers, L, D, N, plan);
  if (rc != B2B_OK) return rc;
  unsigned want;
  if ((rc = b2b_vjp_check_slots(layers, L, param_bars, &want)) != B2B_OK) return rc;
  rc = b2b_vjp_check_batch(layers, L, param_bars, x, ybar, xbar, D, N, ldx, ldybar, ldxbar, stream);
  if (rc != B2B_OK || N == 0) return rc;
  int launches = 0;
  if (!workspace || workspace_bytes < plan.bytes) return B2B_EWORKSPACE;
  char* ws = b2b_align256(workspace);
  double* slots = reinterpret_cast<double*>(ws);
  double* red = slots + (size_t)plan.warps * plan.stride;

  V64Params P;
  memset(&P, 0, sizeof(P));
  P.x = x;
  P.ybar = ybar;
  P.ljbar = ljbar;
  P.xbar = xbar;
  P.ws = slots;
  P.N = N;
  P.ldx = ldx;
  P.ldyb = ybar ? ldybar : D;
  P.ldxb = ldxbar;
  P.stride = plan.stride;
  P.T = plan.T;
  P.D = D;
  P.L = L;
  P.Lf = plan.Lf;
  P.wpc = plan.wpc;
  P.want = want;
  for (int l = 0; l < L; ++l) {
    P.off[l] = plan.off[l];
    P.layers[l] = layers[l];
  }
  const long long ctas = plan.warps / plan.wpc;
  bool lu = false;
  for (int l = 0; l < L; ++l) lu = lu || layers[l].kind == B2B_SCALE_LU;
  const auto kernel = lu ? chain_vjp_f64_kernel<true> : chain_vjp_f64_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<(int)ctas, plan.wpc * 32, plan.smem, stream>>>(P);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++launches;
  if (want) {
    long long blocks = (plan.P + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    vjp_f64_reduce_kernel<<<(int)blocks, 256, 0, stream>>>(slots, plan.stride, plan.T, plan.P, (int)(ctas * plan.wpc), red);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    ++launches;
    V64Fin F;
    memset(&F, 0, sizeof(F));
    F.red = red;
    F.D = D;
    for (int l = 0; l < L; ++l) {
      F.off[l] = plan.off[l];
      F.layers[l] = layers[l];
      for (int i = 0; i < 4; ++i) F.bars[4 * l + i] = param_bars ? param_bars[4 * l + i] : nullptr;
    }
    vjp_f64_finalize_kernel<<<L, V64_FIN_THREADS, 0, stream>>>(F);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    ++launches;
  }
  b2b_set_last_launch_count(launches);
  return B2B_OK;
}
