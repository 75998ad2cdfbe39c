// Float64 device arithmetic shared by the forward (b2b_chain_f64.cu) and the reverse mode (b2b_chain_vjp_f64.cu) of
// Float64 chains: one warp per column, the column in shared memory, lanes over rows, row reductions by warp shuffles.
// The reverse mode recomputes the forward with f64_layer_forward, so both entry points evaluate the same arithmetic.
//
// Reference semantics: planar_layer.jl:65-127,160-185; radial_layer.jl:36-129; rational_quadratic_spline.jl:183-220,
// 317-357; coupling.jl:206-228; normalise.jl:61-86; permute.jl:152-155; stacked.jl:157-166; transformed_distribution.jl:165-169.
#pragma once
#include <cuda_runtime.h>

#include "b2b_internal.h"

namespace b2b {

static __device__ __forceinline__ double wsum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

static __device__ __forceinline__ double softplus64(double x) { return x > 0.0 ? x + log1p(exp(-x)) : log1p(exp(x)); }

static __device__ __forceinline__ void tanh_sech2_64(double a, double& t, double& s2) {
  const double e = exp(-2.0 * fabs(a));
  t = tanh(a);
  const double r = 1.0 / (1.0 + e);
  s2 = 4.0 * e * r * r;  // abs2(sech(a)) without cancellation, planar_layer.jl:107
}

// find_alpha (planar_layer.jl:160-185) in double: bracketed Newton on the monotone f(α) = α + c·tanh(α+b) − t
static __device__ double find_alpha64(double t, double c, double b, double& th, double& s2) {
  const double delta = 2.0 * fabs(c);
  double lo = t - delta, hi = t + delta;
  if (lo == hi) {  // empty bracket, :171-173
    tanh_sech2_64(lo + b, th, s2);
    return lo;
  }
  tanh_sech2_64(t + b, th, s2);
  double x = fmin(fmax(t - c * th, lo), hi);
  for (int it = 0; it < 200; ++it) {
    tanh_sech2_64(x + b, th, s2);
    const double f = x + c * th - t;
    if (f == 0.0) break;
    if (f < 0.0) lo = x; else hi = x;
    double xn = x - f / (1.0 + c * s2);
    if (!(xn > lo && xn < hi)) {
      xn = 0.5 * (lo + hi);
      if (!(xn > lo && xn < hi)) break;  // adjacent doubles
    }
    if (fabs(xn - x) <= 2.3e-16 * (fabs(t) + delta)) {
      x = xn;
      tanh_sech2_64(x + b, th, s2);
      break;
    }
    x = xn;
  }
  return x;
}

static __device__ __forceinline__ double ew_apply64(int op, bool inverse, double a, double b, double xv, double& lj) {
  switch (op) {
    case B2B_EW_EXP:
    case B2B_EW_LOG: {
      const bool is_exp = (op == B2B_EW_EXP) != inverse;
      if (is_exp) {
        lj += xv;
        return exp(xv);
      }
      const double lg = log(xv);
      lj -= lg;
      return lg;
    }
    case B2B_EW_SHIFT: return inverse ? xv - a : a + xv;
    case B2B_EW_SCALE: {
      const double la = log(fabs(a));
      lj += inverse ? -la : la;
      return inverse ? xv / a : a * xv;
    }
    case B2B_EW_LEAKY_RELU: {
      const double al = inverse ? 1.0 / a : a;
      if (xv < 0.0) {
        lj += log(fabs(al));
        return al * xv;
      }
      return xv;
    }
    case B2B_EW_LOGIT: {
      if (!inverse) {
        const double z = (xv - a) / (b - a);
        lj -= log((xv - a) * (b - xv) / (b - a));
        return log(z / (1.0 - z));
      }
      const double x = (b - a) / (1.0 + exp(-xv)) + a;
      lj += log((x - a) * (b - x) / (b - a));
      return x;
    }
    case B2B_EW_TRUNCATED: {
      const bool lo = !isinf(a), hi = !isinf(b);
      if (!inverse) {
        const double x = xv < a ? a : (xv > b ? b : xv);
        if (lo && hi) {
          const double z = (x - a) / (b - a);
          lj -= log((x - a) * (b - x) / (b - a));
          return log(z / (1.0 - z));
        }
        if (lo) {
          const double lg = log(x - a);
          lj -= lg;
          return lg;
        }
        if (hi) {
          const double lg = log(b - x);
          lj -= lg;
          return lg;
        }
        return x;
      }
      double x = xv;
      if (lo && hi) {
        const double ay = fabs(xv);
        lj += log(b - a) - ay - 2.0 * softplus64(-ay);
        x = (b - a) / (1.0 + exp(-xv)) + a;
      } else if (lo) {
        lj += xv;
        x = exp(xv) + a;
      } else if (hi) {
        lj += xv;
        x = b - exp(xv);
      }
      return x < a ? a : (x > b ? b : x);
    }
    default: return xv;
  }
}

// one RQS element straight from the knot arrays (D x K1, column-major); forward :317-357, inverse :183-220
static __device__ double rqs64(const b2b_layer_desc_f64& d, int D, int i, double v, bool inv, double& lj) {
  const int K1 = d.n0;
  const double* Wd = d.p0;
  const double* Hd = d.p1;
  const double* Dv = d.p2;
  const double* S = inv ? Hd : Wd;
  const double Bs = S[(size_t)(K1 - 1) * D + i];
  if (v <= -Bs || v >= Bs) return v;
  int k = 0;  // searchsortedfirst − 1 = number of knots < v
  while (k < K1 && S[(size_t)k * D + i] < v) ++k;
  if (k > K1 - 1) k = K1 - 1;
  const double Wl = Wd[(size_t)(K1 - 1) * D + i], Hl = Hd[(size_t)(K1 - 1) * D + i];
  const double w_k = k == 0 ? -Wl : Wd[(size_t)(k - 1) * D + i];
  const double w = Wd[(size_t)k * D + i] - w_k;
  const double h_k = k == 0 ? -Hl : Hd[(size_t)(k - 1) * D + i];
  const double dy = Hd[(size_t)k * D + i] - h_k;
  const double s = dy / w;
  const double d_k = k == 0 ? 1.0 : Dv[(size_t)(k - 1) * D + i];
  const double d_k1 = k == K1 - 1 ? 1.0 : Dv[(size_t)k * D + i];
  const double ds = d_k1 + d_k - 2.0 * s;
  double xi, res;
  if (inv) {
    const double yh = v - h_k;
    const double a1 = dy * (s - d_k) + yh * ds;
    const double a2 = dy * d_k - yh * ds;
    const double a3 = -s * yh;
    xi = -2.0 * a3 / (a2 + sqrt(a2 * a2 - 4.0 * a1 * a3));
    res = xi * w + w_k;
  } else {
    xi = (v - w_k) / w;
  }
  const double omx = 1.0 - xi;
  const double den = s + ds * xi * omx;
  const double l = log(s * s * (d_k1 * xi * xi + 2.0 * s * xi * omx + d_k * omx * omx)) - 2.0 * log(den);
  if (!inv) res = h_k + dy * (s * xi * xi + d_k * xi * omx) / den;
  lj += inv ? -l : l;
  return res;
}

// r := L⁻¹(col − μ) for the terminal MVNORMAL_TRIL (p0 = μ or NULL, p1 = L column-major, read through L2), by forward
// substitution: r_j is final once the steps before j have run, then rows i > j subtract L(i, j)·r_j.  Returns, in every
// lane, −Σ log Lᵢᵢ − ½‖r‖².  `r` may not alias `col`.
static __device__ double f64_tril_solve(const b2b_layer_desc_f64& d, int D, int lane, const double* col, double* r) {
  const double* Lm = d.p1;
  for (int i = lane; i < D; i += 32) r[i] = col[i] - (d.p0 ? d.p0[i] : 0.0);
  __syncwarp();
  for (int j = 0; j < D; ++j) {
    const double rj = r[j] / Lm[(size_t)j * D + j];
    __syncwarp();  // every lane has read r[j]
    if (lane == 0) r[j] = rj;
    for (int i = j + 1 + lane; i < D; i += 32) r[i] = fma(-Lm[(size_t)j * D + i], rj, r[i]);
    __syncwarp();
  }
  double q = 0.0, ls = 0.0;
  for (int i = lane; i < D; i += 32) {
    q += r[i] * r[i];
    ls += log(Lm[(size_t)i * D + i]);
  }
  return -wsum(ls) - 0.5 * wsum(q);
}

// s := L⁻ᵀ r by left-looking back substitution, s_i = (r_i − Σ_{k>i} L(k, i)·s_k)/Lᵢᵢ: column i of L is contiguous, so the
// dot product is a coalesced read and a warp sum.  `s` may not alias `r`.
static __device__ void f64_tril_back(const b2b_layer_desc_f64& d, int D, int lane, const double* r, double* s) {
  const double* Lm = d.p1;
  for (int i = D - 1; i >= 0; --i) {
    double p = 0.0;
    for (int k = i + 1 + lane; k < D; k += 32) p += Lm[(size_t)i * D + k] * s[k];
    p = wsum(p);
    if (lane == 0) s[i] = (r[i] - p) / Lm[(size_t)i * D + i];
    __syncwarp();
  }
}

// v := T⁻¹ v in place for SCALE_TRIANGULAR (p0 = T column-major, read through L2; n0: upper, n1: unit diagonal): forward
// substitution for a lower T, back substitution for an upper one, v_j final once the steps before it have run, then the
// rest of column j of T is subtracted.  Reads only the triangle (not the diagonal of a unit T).
static __device__ void f64_tri_solve(const b2b_layer_desc_f64& d, int D, int lane, double* v) {
  const double* Tm = d.p0;
  const bool up = d.n0 != 0, unit = d.n1 != 0;
  for (int jj = 0; jj < D; ++jj) {
    const int j = up ? D - 1 - jj : jj;
    const double vj = unit ? v[j] : v[j] / Tm[(size_t)j * D + j];
    __syncwarp();  // every lane has read v[j]
    if (lane == 0) v[j] = vj;
    for (int i = (up ? 0 : j + 1) + lane; i < (up ? j : D); i += 32) v[i] = fma(-Tm[(size_t)j * D + i], vj, v[i]);
    __syncwarp();
  }
}

// Σᵢ log|Tᵢᵢ| of SCALE_TRIANGULAR in every lane (0 for a unit diagonal)
static __device__ __forceinline__ double f64_tri_logdet(const b2b_layer_desc_f64& d, int D, int lane) {
  double p = 0.0;
  for (int i = lane; i < D && !d.n1; i += 32) p += log(fabs(d.p0[(size_t)i * D + i]));
  return wsum(p);
}

// y = T x (rows owned by lanes, k increasing; `tmp` holds x) or T⁻¹ x (substitution in place) for SCALE_TRIANGULAR;
// returns its log-Jacobian in every lane.
static __device__ double f64_tri_forward(const b2b_layer_desc_f64& d, int D, int lane, double* col,
                                                      double* tmp) {
  const double lp = f64_tri_logdet(d, D, lane);
  if (d.inverse) {
    f64_tri_solve(d, D, lane, col);
    return -lp;
  }
  const bool up = d.n0 != 0, unit = d.n1 != 0;
  for (int i = lane; i < D; i += 32) {
    tmp[i] = col[i];
    col[i] = unit ? col[i] : 0.0;
  }
  __syncwarp();
  for (int k = 0; k < D; ++k) {
    const double xk = tmp[k];
    const double* Tk = d.p0 + (size_t)k * D;
    for (int i = lane; i < D; i += 32)
      if (up ? (i < k || (i == k && !unit)) : (i > k || (i == k && !unit))) col[i] = fma(Tk[i], xk, col[i]);
  }
  __syncwarp();
  return lp;
}

// v := P v (y[dst[r]] = v[r]) or, `inv`, Pᵀ v (v[r] = y[dst[r]]) in place through `tmp`, for dst = i0 of SCALE_LU
static __device__ __forceinline__ void f64_lu_permute(const int32_t* dst, bool inv, int D, int lane, double* v,
                                                      double* tmp) {
  for (int i = lane; i < D; i += 32) tmp[i] = v[i];
  __syncwarp();
  for (int i = lane; i < D; i += 32) {
    if (inv) v[i] = tmp[dst[i]];
    else v[dst[i]] = tmp[i];
  }
  __syncwarp();
}

// The SCALE_TRIANGULAR descriptor of one factor of a SCALE_LU layer `d` (F in p0): U (upper) or L (unit lower)
static __device__ __forceinline__ b2b_layer_desc_f64 f64_lu_factor(const b2b_layer_desc_f64& d, bool upper) {
  b2b_layer_desc_f64 t = d;
  t.kind = B2B_SCALE_TRIANGULAR;
  t.n0 = upper ? 1 : 0;
  t.n1 = upper ? 0 : 1;
  return t;
}

// y = P·L·U x or U⁻¹ L⁻¹ Pᵀ x for SCALE_LU (p0 = F: L strictly below the diagonal with a unit diagonal, U on and above it;
// i0 = dst or NULL): the steps of PERMUTE ∘ SCALE_TRIANGULAR(unit lower) ∘ SCALE_TRIANGULAR(upper) on F, by the
// triangular layer's own functions.  Returns the log-Jacobian, ±Σ log|Uᵢᵢ|, in every lane.
static __device__ double f64_lu_forward(const b2b_layer_desc_f64& d, int D, int lane, double* col, double* tmp) {
  const b2b_layer_desc_f64 U = f64_lu_factor(d, true), L = f64_lu_factor(d, false);
  if (d.inverse) {
    if (d.i0) f64_lu_permute(d.i0, true, D, lane, col, tmp);
    f64_tri_forward(L, D, lane, col, tmp);
    return f64_tri_forward(U, D, lane, col, tmp);
  }
  const double lp = f64_tri_forward(U, D, lane, col, tmp);
  f64_tri_forward(L, D, lane, col, tmp);
  if (d.i0) f64_lu_permute(d.i0, false, D, lane, col, tmp);
  return lp;
}

// Applies one layer to the column `col` (D doubles in shared memory; `tmp`: D more, scratch) and adds its log-Jacobian
// (for MVNORMAL_DIAG: the log-density) to `lj`.  Called by all 32 lanes of a warp; ends with __syncwarp.  TRI = false
// leaves SCALE_TRIANGULAR out: compiled in, that case costs the Float64 forward kernel registers (80 instead of 96, and a
// spill), so b2b_chain_run_f64 uses that instantiation only for chains that hold the layer.  LU = false leaves SCALE_LU
// out the same way: only chains that hold it run an instantiation with that case.
template <bool TRI = true, bool LU = false>
static __device__ __forceinline__ void f64_layer_forward(const b2b_layer_desc_f64& d, int D, int lane, double* col,
                                                         double* tmp, double& lj) {
  const bool inv = d.inverse != 0;
  switch (d.kind) {
    case B2B_PLANAR: {
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
      const double kk = (softplus64(-s) - 1.0) / q;  // get_u_hat, planar_layer.jl:65-70
      const double c = softplus64(s) - 1.0, b = d.p2[0];
      double t, s2;
      if (!inv) {
        tanh_sech2_64(wz + b, t, s2);
        lj += log1p(c * s2);
      } else {
        find_alpha64(wz, c, b, t, s2);
        lj -= log1p(c * s2);
        t = -t;
      }
      for (int i = lane; i < D; i += 32) col[i] += (d.p1[i] + kk * d.p0[i]) * t;
    } break;
    case B2B_RADIAL: {
      const double alpha = softplus64(d.p0[0]), apb = softplus64(d.p1[0]), bhat = apb - alpha;
      double r2 = 0.0;
      for (int i = lane; i < D; i += 32) {
        const double dd = col[i] - d.p2[i];
        r2 += dd * dd;
      }
      const double nrm = sqrt(wsum(r2));
      double r = nrm;
      if (inv) {
        const double a = apb - nrm;  // radial_layer.jl:126-127
        const double sq = sqrt(a * a + 4.0 * alpha * nrm);
        r = a > 0.0 ? (2.0 * alpha * nrm) / (sq + a) : 0.5 * (sq - a);  // the same root without cancellation
      }
      const double hh = 1.0 / (alpha + r);
      const double ljf = (double)(D - 1) * log1p(bhat * hh) + log1p(bhat * hh - bhat * hh * hh * r);
      const double g = inv ? (alpha + r) / (apb + r) - 1.0 : bhat * hh;
      lj += inv ? -ljf : ljf;
      for (int i = lane; i < D; i += 32) col[i] += g * (col[i] - d.p2[i]);
    } break;
    case B2B_RQS: {
      double p = 0.0;
      for (int i = lane; i < D; i += 32) col[i] = rqs64(d, D, i, col[i], inv, p);
      lj += wsum(p);
    } break;
    case B2B_BATCHNORM: {
      double p = 0.0;
      for (int i = lane; i < D; i += 32) {
        const double ve = d.p3[i] + d.f0, sc = exp(d.p1[i]);
        col[i] = inv ? (col[i] - d.p0[i]) / sc * sqrt(ve) + d.p2[i] : sc * (col[i] - d.p2[i]) / sqrt(ve) + d.p0[i];
        p += d.p1[i] - 0.5 * log(ve);
      }
      p = wsum(p);
      lj += inv ? -p : p;
    } break;
    case B2B_ELEMENTWISE_VEC:  // the law n0 on every row, a = p0 (b unused)
    case B2B_STACKED_EW: {
      const bool vec = d.kind == B2B_ELEMENTWISE_VEC;
      double p = 0.0;
      for (int i = lane; i < D; i += 32)
        col[i] = ew_apply64(vec ? d.n0 : d.i0[i], inv, d.p0 ? d.p0[i] : 0.0, d.p1 && !vec ? d.p1[i] : 0.0, col[i], p);
      lj += wsum(p);
    } break;
    case B2B_PERMUTE: {
      for (int i = lane; i < D; i += 32) tmp[i] = col[i];
      __syncwarp();
      for (int i = lane; i < D; i += 32) {
        if (inv) col[i] = tmp[d.i0[i]];       // Permute(transpose(A)), permute.jl:153
        else col[d.i0[i]] = tmp[i];           // y[dst[i]] = x[i], :95-97,152
      }
    } break;
    case B2B_COUPLING_AFFINE: {
      const int n1 = d.n0, n2 = d.n1;
      double p = 0.0;
      for (int j = lane; j < n1; j += 32) {
        double sv = d.p1 ? d.p1[j] : 0.0, tv = d.p1 ? d.p1[n1 + j] : 0.0;
        for (int k = 0; k < n2; ++k) {
          const double xk = col[d.i1 ? d.i1[k] : d.n3 + k];
          sv += d.p0[(size_t)k * (2 * n1) + j] * xk;
          tv += d.p0[(size_t)k * (2 * n1) + n1 + j] * xk;
        }
        const int r = d.i0 ? d.i0[j] : d.n2 + j;
        tmp[j] = inv ? (col[r] - tv) * exp(-sv) : exp(sv) * col[r] + tv;  // scale.jl:13,16; shift.jl:12,14
        p += sv;
      }
      __syncwarp();  // every lane has read its x₂ rows before x₁ rows are overwritten (disjoint row sets anyway)
      for (int j = lane; j < n1; j += 32) col[d.i0 ? d.i0[j] : d.n2 + j] = tmp[j];
      p = wsum(p);
      lj += inv ? -p : p;
    } break;
    case B2B_MVNORMAL_DIAG: {
      double q = 0.0, ls = 0.0;
      for (int i = lane; i < D; i += 32) {
        const double sg = d.p1 ? d.p1[i] : 1.0, z = (col[i] - (d.p0 ? d.p0[i] : 0.0)) / sg;
        q += z * z;
        ls += log(sg * sg);
      }
      q = wsum(q);
      ls = wsum(ls);
      lj += -0.5 * ((double)D * 1.8378770664093453 + ls) - 0.5 * q;
    } break;
    case B2B_SCALE_TRIANGULAR:
      if constexpr (TRI) lj += f64_tri_forward(d, D, lane, col, tmp);
      break;
    case B2B_SCALE_LU:
      if constexpr (LU) lj += f64_lu_forward(d, D, lane, col, tmp);
      break;
    case B2B_MVNORMAL_TRIL:  // the column is left as it is (the terminal's y is its input); r goes to tmp
      lj += -0.5 * (double)D * 1.8378770664093453 + f64_tril_solve(d, D, lane, col, tmp);
      break;
    default: break;
  }
  __syncwarp();
}

}  // namespace b2b
