// Float64 evaluation of the same chains (include/b2b.h: b2b_chain_run_f64).
//
// The reference is generic in its element type and its own tests run in Float64 (e.g. the find_alpha residual grid with
// atol = 1e-14, test/normalising_flows.jl:47-71); this kernel is the device counterpart for those element types.  It is a
// plain, layer-by-layer restatement in double precision -- one warp per column, the column staged in shared memory,
// lanes over rows, row reductions by warp shuffles -- NOT a tuned kernel: Float64 batches are a correctness path, the
// Float32 kernels are the hot path.  Every layer kind of the Float32 path is
// covered, including affine coupling (a per-column matrix-vector product) and the terminal MvNormal.
//
// Reference semantics: planar_layer.jl:65-127,160-185; radial_layer.jl:36-129; rational_quadratic_spline.jl:183-220,
// 317-357; coupling.jl:206-228; normalise.jl:61-86; permute.jl:152-155; stacked.jl:157-166; transformed_distribution.jl:165-169.
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_internal.h"

namespace b2b {

constexpr int F64_WARPS = 4;

struct F64Params {
  const double* x;
  double* y;
  double* logjac;
  double* partials;
  long long N, ldx, ldy;
  int D, L, accumulate;
  b2b_layer_desc_f64 layers[B2B_MAX_CHAIN];
};

__device__ __forceinline__ double wsum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double softplus64(double x) { return x > 0.0 ? x + log1p(exp(-x)) : log1p(exp(x)); }

__device__ __forceinline__ void tanh_sech2_64(double a, double& t, double& s2) {
  const double e = exp(-2.0 * fabs(a));
  t = tanh(a);
  const double r = 1.0 / (1.0 + e);
  s2 = 4.0 * e * r * r;  // abs2(sech(a)) without cancellation, planar_layer.jl:107
}

// find_alpha (planar_layer.jl:160-185) in double: bracketed Newton on the monotone f(α) = α + c·tanh(α+b) − t
__device__ double find_alpha64(double t, double c, double b, double& th, double& s2) {
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

__device__ __forceinline__ double ew_apply64(int op, bool inverse, double a, double b, double xv, double& lj) {
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
__device__ double rqs64(const b2b_layer_desc_f64& d, int D, int i, double v, bool inv, double& lj) {
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

__global__ void __launch_bounds__(F64_WARPS * 32) chain_f64_kernel(const __grid_constant__ F64Params P) {
  extern __shared__ double sm64[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, D = P.D;
  double* col = sm64 + (size_t)warp * 2 * D;  // the column
  double* tmp = col + D;                       // scratch (permute, coupling)
  double dsum = 0.0;
  for (long long n = (long long)blockIdx.x * F64_WARPS + warp; n < P.N; n += (long long)gridDim.x * F64_WARPS) {
    for (int i = lane; i < D; i += 32) col[i] = P.x[n * P.ldx + i];
    double lj = (P.accumulate && P.logjac) ? P.logjac[n] : 0.0;
    __syncwarp();
    for (int l = 0; l < P.L; ++l) {
      const b2b_layer_desc_f64& d = P.layers[l];
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
        case B2B_STACKED_EW: {
          double p = 0.0;
          for (int i = lane; i < D; i += 32)
            col[i] = ew_apply64(d.i0[i], inv, d.p0 ? d.p0[i] : 0.0, d.p1 ? d.p1[i] : 0.0, col[i], p);
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
        default: break;
      }
      __syncwarp();
    }
    if (P.y)
      for (int i = lane; i < D; i += 32) P.y[n * P.ldy + i] = col[i];
    if (lane == 0) {
      if (P.logjac) P.logjac[n] = lj;
      dsum += lj;
    }
    __syncwarp();
  }
  if (P.partials) {
    __shared__ double red[F64_WARPS];
    if (lane == 0) red[warp] = dsum;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < F64_WARPS; ++w) t += red[w];
      P.partials[blockIdx.x] = t;
    }
  }
}

}  // namespace b2b

extern "C" size_t b2b_chain_workspace_bytes_f64(int32_t L, int want_sum) { return (L > 0 && want_sum) ? 4096 * sizeof(double) : 0; }

extern "C" int b2b_chain_run_f64(const b2b_layer_desc_f64* layers, int32_t L, const double* x, double* y, double* logjac,
                                 double* sum_out, int32_t D, int64_t N, int64_t ldx, int64_t ldy, int accumulate_logjac,
                                 void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b2b;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!layers || L < 1 || L > B2B_MAX_CHAIN || D < 1 || N < 0 || ldx < D) return B2B_EINVAL;
  if (D > 2048) return B2B_EUNSUPPORTED;
  if (N == 0) {
    if (sum_out) return (int)cudaMemsetAsync(sum_out, 0, sizeof(double), stream);
    return B2B_OK;
  }
  if (!x || (y && ldy < D) || (!y && !logjac && !sum_out)) return B2B_EINVAL;
  F64Params P;
  memset(&P, 0, sizeof(P));
  for (int l = 0; l < L; ++l) {
    const b2b_layer_desc_f64& d = layers[l];
    switch (d.kind) {
      case B2B_PLANAR:
      case B2B_RADIAL:
        if (!d.p0 || !d.p1 || !d.p2) return B2B_EINVAL;
        break;
      case B2B_RQS:
        if (!d.p0 || !d.p1 || !d.p2 || d.n0 < 2) return B2B_EINVAL;
        break;
      case B2B_COUPLING_AFFINE:
        if (!d.p0 || d.n0 < 1 || d.n1 < 1 || d.n0 + d.n1 > D || (!d.i0 && d.n2 < 0) || (!d.i1 && d.n3 < 0)) return B2B_EINVAL;
        break;
      case B2B_BATCHNORM:
        if (!d.p0 || !d.p1 || !d.p2 || !d.p3) return B2B_EINVAL;
        break;
      case B2B_PERMUTE:
      case B2B_STACKED_EW:
        if (!d.i0) return B2B_EINVAL;
        break;
      case B2B_MVNORMAL_DIAG:
        if (l != L - 1 || d.inverse) return B2B_EINVAL;
        break;
      default: return B2B_EINVAL;
    }
    P.layers[l] = d;
  }
  if (sum_out && !logjac && layers[L - 1].kind != B2B_MVNORMAL_DIAG) return B2B_EINVAL;
  P.x = x;
  P.y = y;
  P.logjac = logjac;
  P.N = N;
  P.ldx = ldx;
  P.ldy = y ? ldy : D;
  P.D = D;
  P.L = L;
  P.accumulate = accumulate_logjac ? 1 : 0;
  long long grid = (N + F64_WARPS - 1) / F64_WARPS;
  if (grid > 132 * 8) grid = 132 * 8;
  if (sum_out) {
    if (!workspace || workspace_bytes < 4096 * sizeof(double)) return B2B_EWORKSPACE;
    P.partials = static_cast<double*>(workspace);
  }
  const size_t smem = (size_t)F64_WARPS * 2 * D * sizeof(double);
  cudaError_t e = cudaFuncSetAttribute(chain_f64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  chain_f64_kernel<<<(int)grid, F64_WARPS * 32, smem, stream>>>(P);
  e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  if (sum_out) return b2b_launch_sum_partials(P.partials, (int)grid, sum_out, stream);
  return B2B_OK;
}
