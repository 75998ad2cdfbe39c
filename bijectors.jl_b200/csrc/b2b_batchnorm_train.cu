// InvertibleBatchNorm, TRAINING mode (src/bijectors/normalise.jl:51-60): batch statistics over the N columns
// (over all ranks when a communicator is given: the path's second, 2·D+1-double all-reduce), moving-average
// update of the layer's m / v in place (with the n/(n-1) correction of :60), then the forward map and the
// log-Jacobian with the BATCH statistics (:66-67).
//
//   pass 1  bn_stats_kernel     reads x once: per-row Σx and Σx² in fp64, per-CTA partials (deterministic)
//           bn_reduce_kernel    fixed-order sum of the partials -> acc[2D+1] = {Σx, Σx², n}
//           (ncclAllReduce of acc when sharded)
//           bn_finalize_kernel  m = Σx/n, v = Σx²/n − m² (= sum((x−m)²)/n, :55), moving update, batch m/v as float
//   pass 2  the eval-mode BatchNorm op of the chain kernels with the batch statistics
// Algorithmic traffic: 3 passes over D x N floats (read, read, write).
//
// Reverse mode (b2b_batchnorm_train_vjp_f32; the output and the log-Jacobian both depend on the batch statistics, so x̄ of
// one column depends on sums over every column of every rank):
//   pass 1  bn_stats_kernel<BWD>  reads x, ȳ (and l̄) once: Σx, Σx² in the forward's order, Σȳ, Σȳx per row, Σl̄
//           bn_reduce_kernel      -> acc[4D+2] = {Σx, Σx², n, Σȳ, Σȳx, Σl̄} (+ a copy of this rank's sums when sharded)
//           (one all-reduce of acc when sharded)
//           bn_vjp_coef_kernel    m, v; per-row A, C, B; this rank's b̄ = Σȳ, l̄ogs = A Σȳ(x − m) + Σl̄
//   pass 2  bn_vjp_apply_kernel   reads x, ȳ, writes x̄ = A ȳ + C (x − m) + B,
//           C = −(A S2 + L̄)/(n σ²), B = −A S1/n  (S1 = Σȳ, S2 = Σȳ(x − m), L̄ = Σl̄ over all columns, σ² = v + eps)
// Algorithmic traffic: 4·(5D + 1) bytes per column.
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_internal.h"

namespace b2b {

constexpr int BNT_THREADS = 256;

// Each warp walks columns; lane l owns the float4 chunks {l + 32 v} of the CTA's row slice.  Rows are accumulated in fp64
// registers.  BWD (the reverse mode) also accumulates Σȳ and Σȳ·x per row and Σl̄ per column, and splits the rows over
// blockIdx.y slices of 128·V rows to bound its registers.  A row's sums see the same columns in the same order whatever the
// slicing (same grid, same warp-to-column walk, same warp-then-CTA combine), so Σx and Σx² are bit-identical to the
// forward's on the same x.
template <int V, bool VEC, bool BWD>
__global__ void __launch_bounds__(BNT_THREADS) bn_stats_kernel(const float* __restrict__ x, int D, long long N,
                                                               long long ldx, const float* __restrict__ ybar,
                                                               long long ldyb, const float* __restrict__ ljbar,
                                                               double* __restrict__ partials) {
  extern __shared__ double sred[];  // [K][Dp] (+ Σl̄ when BWD) per CTA
  constexpr int K = BWD ? 4 : 2;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = BNT_THREADS / 32;
  const int Dp = 128 * V, base = Dp * blockIdx.y;
  for (int i = threadIdx.x; i < K * Dp + (BWD ? 1 : 0); i += BNT_THREADS) sred[i] = 0.0;
  __syncthreads();
  double s1[V][4], s2[V][4], s3[V][4], s4[V][4], sl = 0.0;
#pragma unroll
  for (int v = 0; v < V; ++v)
#pragma unroll
    for (int e = 0; e < 4; ++e) s1[v][e] = s2[v][e] = s3[v][e] = s4[v][e] = 0.0;
  const long long gw = (long long)blockIdx.x * nwarps + warp, stride = (long long)gridDim.x * nwarps;
  for (long long col = gw; col < N; col += stride) {
    const float* xc = x + col * ldx;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int r0 = base + 4 * (lane + 32 * v);
      float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
      if (VEC) {
        if (r0 < D) q = __ldcs(reinterpret_cast<const float4*>(xc + r0));
      } else {
        if (r0 + 0 < D) q.x = xc[r0 + 0];
        if (r0 + 1 < D) q.y = xc[r0 + 1];
        if (r0 + 2 < D) q.z = xc[r0 + 2];
        if (r0 + 3 < D) q.w = xc[r0 + 3];
      }
      const double a = q.x, b = q.y, c = q.z, d = q.w;
      s1[v][0] += a; s2[v][0] = fma(a, a, s2[v][0]);
      s1[v][1] += b; s2[v][1] = fma(b, b, s2[v][1]);
      s1[v][2] += c; s2[v][2] = fma(c, c, s2[v][2]);
      s1[v][3] += d; s2[v][3] = fma(d, d, s2[v][3]);
      if (BWD && ybar) {
        const float* yc = ybar + col * ldyb;
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
        if (VEC) {
          if (r0 < D) g = __ldcs(reinterpret_cast<const float4*>(yc + r0));
        } else {
          if (r0 + 0 < D) g.x = yc[r0 + 0];
          if (r0 + 1 < D) g.y = yc[r0 + 1];
          if (r0 + 2 < D) g.z = yc[r0 + 2];
          if (r0 + 3 < D) g.w = yc[r0 + 3];
        }
        const double ga = g.x, gb = g.y, gc = g.z, gd = g.w;
        s3[v][0] += ga; s4[v][0] = fma(ga, a, s4[v][0]);
        s3[v][1] += gb; s4[v][1] = fma(gb, b, s4[v][1]);
        s3[v][2] += gc; s4[v][2] = fma(gc, c, s4[v][2]);
        s3[v][3] += gd; s4[v][3] = fma(gd, d, s4[v][3]);
      }
    }
    if (BWD && ljbar && lane == 0 && blockIdx.y == 0) sl += (double)ljbar[col];
  }
  // combine the warps of the CTA in a fixed order (warp 0 first, ...) for determinism
  for (int w = 0; w < nwarps; ++w) {
    if (warp == w) {
#pragma unroll
      for (int v = 0; v < V; ++v)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int r = 4 * (lane + 32 * v) + e;
          sred[r] += s1[v][e];
          sred[Dp + r] += s2[v][e];
          if (BWD) {
            sred[2 * Dp + r] += s3[v][e];
            sred[3 * Dp + r] += s4[v][e];
          }
        }
      if (BWD && lane == 0) sred[4 * Dp] += sl;
    }
    __syncthreads();
  }
  // per-CTA partials: {Σx, Σx²} (2D) forward, {Σx, Σx², Σȳ, Σȳx, Σl̄} (4D + 1) reverse
  const size_t len = BWD ? 4 * (size_t)D + 1 : 2 * (size_t)D;
  double* part = partials + (size_t)blockIdx.x * len;
  for (int i = threadIdx.x; i < Dp; i += BNT_THREADS) {
    if (base + i >= D) break;
#pragma unroll
    for (int k = 0; k < K; ++k) part[(size_t)k * D + base + i] = sred[k * Dp + i];
  }
  if (BWD && blockIdx.y == 0 && threadIdx.x == 0) part[4 * (size_t)D] = sred[4 * Dp];
}

// acc[0..2D) = Σ of the first 2D partial entries, acc[2D] = n, acc[2D+1..len+1) = the rest (reverse mode).  Blocks are
// summed in index order.  `loc` (reverse mode on a sharded batch) keeps this rank's Σȳ, Σȳx, Σl̄ from the all-reduce.
__global__ void __launch_bounds__(256) bn_reduce_kernel(const double* __restrict__ partials, int nblk, int D, int len,
                                                        long long N, double* __restrict__ acc, double* __restrict__ loc) {
  for (int i = blockIdx.x * 256 + threadIdx.x; i < len; i += gridDim.x * 256) {
    double t = 0.0;
    for (int b = 0; b < nblk; ++b) t += partials[(size_t)b * len + i];
    acc[i < 2 * D ? i : i + 1] = t;
    if (loc && i >= 2 * D) loc[i - 2 * D] = t;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) acc[2 * D] = (double)N;
}

__global__ void __launch_bounds__(256) bn_finalize_kernel(const double* __restrict__ acc, int D, float mtm,
                                                          float* __restrict__ mov_m, float* __restrict__ mov_v,
                                                          float* __restrict__ batch_m, float* __restrict__ batch_v) {
  const double n = acc[2 * D];
  for (int i = blockIdx.x * 256 + threadIdx.x; i < D; i += gridDim.x * 256) {
    const double mean = acc[i] / n;                       // mean(x; dims), normalise.jl:54
    double var = acc[D + i] / n - mean * mean;            // sum((x .- m).^2) ./ n, :55
    var = var > 0.0 ? var : 0.0;
    batch_m[i] = (float)mean;
    batch_v[i] = (float)var;
    // moving statistics, :59-60  (T.(…) rounds the batch statistic to the parameter eltype first)
    const float mf = (float)mean, vf = (float)var;
    mov_m[i] = (1.0f - mtm) * mov_m[i] + mtm * mf;
    mov_v[i] = (1.0f - mtm) * mov_v[i] + (float)((double)mtm * n / (n - 1.0)) * vf;
  }
}

// Reverse mode, between the passes: batch m / v exactly as bn_finalize_kernel rounds them (no moving update), the per-row
// coefficients of x̄ = A ȳ + C (x − m) + B, and this rank's b̄ / l̄ogs from its own sums (`loc`, with the global m).
__global__ void __launch_bounds__(256) bn_vjp_coef_kernel(const double* __restrict__ acc, const double* __restrict__ loc,
                                                          const float* __restrict__ logs, float eps, int D,
                                                          float* __restrict__ coef, float* __restrict__ bbar,
                                                          float* __restrict__ logsbar) {
  const double n = acc[2 * D], L = acc[4 * D + 1];
  for (int i = blockIdx.x * 256 + threadIdx.x; i < D; i += gridDim.x * 256) {
    const double mean = acc[i] / n;
    double var = acc[D + i] / n - mean * mean;
    var = var > 0.0 ? var : 0.0;
    const float mf = (float)mean, s2 = (float)var + eps;  // m and σ² = v + eps as the forward holds them
    const float A = expf(logs[i]) / sqrtf(s2);
    const double S1 = acc[2 * D + 1 + i], S2 = acc[3 * D + 1 + i] - (double)mf * S1;  // Σȳ, Σȳ(x − m)
    coef[i] = A;
    coef[D + i] = (float)(-((double)A * S2 + L) / (n * (double)s2));
    coef[2 * D + i] = (float)(-(double)A * S1 / n);
    coef[3 * D + i] = mf;
    if (bbar) {
      bbar[i] = (float)loc[i];
      logsbar[i] = (float)((double)A * (loc[D + i] - (double)mf * loc[i]) + loc[2 * D]);
    }
  }
}

template <int W>
__device__ __forceinline__ void bnt_load(const float* p, float (&v)[W]) {
  if constexpr (W == 4) {
    const float4 q = __ldcs(reinterpret_cast<const float4*>(p));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
    v[0] = __ldcs(p);
  }
}

// Reverse mode, pass 2: x̄ = A ȳ + C (x − m) + B.  A thread owns one unit (W = 4: a float4, W = 1: a float) of rows -- RPT
// units 256 apart when a column has more than 256 units -- in a slab of columns; U columns are loaded before any is stored,
// so `xbar` may be `ybar` itself.  (x − m) is kept as the forward forms it: folding C·m into B cancels when |m| ≫ σ.
template <int RPT, int W>
__global__ void __launch_bounds__(256) bn_vjp_apply_kernel(const float* __restrict__ x, const float* ybar, float* xbar,
                                                           const float* __restrict__ coef, int D, long long N,
                                                           long long ldx, long long ldyb, long long ldxb) {
  constexpr int U = RPT == 1 ? 4 : 8 / RPT;  // columns in flight per thread
  const int Du = D / W, Dp = RPT == 1 ? ((Du + 31) & ~31) : 256, nslab = 256 / Dp;
  const int slab = threadIdx.x / Dp, i = threadIdx.x - slab * Dp;
  if (slab >= nslab) return;
  float A[RPT][W], C[RPT][W], B[RPT][W], M[RPT][W];
#pragma unroll
  for (int j = 0; j < RPT; ++j)
#pragma unroll
    for (int e = 0; e < W; ++e) {
      const int r = (i + 256 * j) * W + e;
      const bool ok = i + 256 * j < Du;
      A[j][e] = ok ? coef[r] : 0.f;
      C[j][e] = ok ? coef[D + r] : 0.f;
      B[j][e] = ok ? coef[2 * D + r] : 0.f;
      M[j][e] = ok ? coef[3 * D + r] : 0.f;
    }
  const long long per = (N + gridDim.x - 1) / gridDim.x;
  const long long c0 = (long long)blockIdx.x * per, c1 = (c0 + per < N) ? c0 + per : N;
  for (long long n0 = c0 + slab; n0 < c1; n0 += (long long)U * nslab) {
    float xv[U][RPT][W], gv[U][RPT][W];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long n = n0 + (long long)u * nslab;
#pragma unroll
      for (int j = 0; j < RPT; ++j) {
        const int r = (i + 256 * j) * W;
        const bool ok = n < c1 && i + 256 * j < Du;
#pragma unroll
        for (int e = 0; e < W; ++e) xv[u][j][e] = gv[u][j][e] = 0.f;
        if (ok) bnt_load<W>(x + n * ldx + r, xv[u][j]);
        if (ok && ybar) bnt_load<W>(ybar + n * ldyb + r, gv[u][j]);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long n = n0 + (long long)u * nslab;
#pragma unroll
      for (int j = 0; j < RPT; ++j) {
        if (!(n < c1 && i + 256 * j < Du)) continue;
        float o[W];
#pragma unroll
        for (int e = 0; e < W; ++e) o[e] = fmaf(A[j][e], gv[u][j][e], fmaf(C[j][e], xv[u][j][e] - M[j][e], B[j][e]));
        float* dst = xbar + n * ldxb + (i + 256 * j) * W;
        if constexpr (W == 4) __stcs(reinterpret_cast<float4*>(dst), make_float4(o[0], o[1], o[2], o[3]));
        else __stcs(dst, o[0]);
      }
    }
  }
}

static int stats_grid(long long N) {
  const int sms = b2b_sm_count();
  int grid = sms * 4;
  if (grid > 1184) grid = 1184;
  const long long want = (N + 7) / 8;
  if (grid > want) grid = (int)want;
  if (grid < 1) grid = 1;
  return grid;
}

}  // namespace b2b

extern "C" size_t b2b_batchnorm_train_workspace_bytes(int32_t D) {
  // per-CTA partials (<= 1184 CTAs) + acc[2D+1] + batch m / v
  return (size_t)1184 * 2 * D * sizeof(double) + (size_t)(2 * D + 2) * sizeof(double) + (size_t)2 * D * sizeof(float) + 256;
}

extern "C" int b2b_batchnorm_train_fwd_f32(const float* x, float* y, float* logjac, const float* b, const float* logs,
                                           float* m, float* v, float eps, float mtm, int32_t D, int64_t N,
                                           int64_t ldx, int64_t ldy, int accumulate_logjac, b2b_comm* comm,
                                           void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b2b;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !b || !logs || !m || !v || D < 1 || N < 2 || ldx < D || (y && ldy < D)) return B2B_EINVAL;
  if (D > 1024) return B2B_EUNSUPPORTED;
  if (!workspace || workspace_bytes < b2b_batchnorm_train_workspace_bytes(D)) return B2B_EWORKSPACE;
  const int grid = stats_grid(N);
  char* ws = b2b_align256(workspace);
  double* partials = reinterpret_cast<double*>(ws);
  double* acc = partials + (size_t)1184 * 2 * D;
  float* batch_m = reinterpret_cast<float*>(acc + 2 * D + 2);
  float* batch_v = batch_m + D;
  const bool vec = (D % 4 == 0) && (ldx % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  const int V = (D + 127) / 128 <= 1 ? 1 : ((D + 127) / 128 <= 2 ? 2 : ((D + 127) / 128 <= 4 ? 4 : 8));
  const size_t smem = (size_t)2 * 128 * V * sizeof(double);
#define B2B_BNT_LAUNCH(VV)                                                                      \
  if (vec) bn_stats_kernel<VV, true, false><<<grid, BNT_THREADS, smem, stream>>>(x, D, N, ldx, nullptr, 0, nullptr, partials); \
  else bn_stats_kernel<VV, false, false><<<grid, BNT_THREADS, smem, stream>>>(x, D, N, ldx, nullptr, 0, nullptr, partials);
  if (V == 1) { B2B_BNT_LAUNCH(1) } else if (V == 2) { B2B_BNT_LAUNCH(2) } else if (V == 4) { B2B_BNT_LAUNCH(4) } else { B2B_BNT_LAUNCH(8) }
#undef B2B_BNT_LAUNCH
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  bn_reduce_kernel<<<(2 * D + 255) / 256, 256, 0, stream>>>(partials, grid, D, 2 * D, N, acc, nullptr);
  if (comm) {  // sharded batch: one all-reduce of {Σx, Σx², n}
    const int rc = b2b_allreduce_sum_f64(comm, acc, 2 * D + 1, stream);
    if (rc != B2B_OK) return rc;
  }
  bn_finalize_kernel<<<(D + 255) / 256, 256, 0, stream>>>(acc, D, mtm, m, v, batch_m, batch_v);
  e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  if (!y && !logjac) return B2B_OK;
  b2b_layer_desc d;
  memset(&d, 0, sizeof(d));
  d.kind = B2B_BATCHNORM;
  d.p0 = b;
  d.p1 = logs;
  d.p2 = batch_m;
  d.p3 = batch_v;
  d.f0 = eps;
  return b2b_chain_run_f32(&d, 1, x, y, logjac, nullptr, D, N, ldx, ldy, accumulate_logjac, nullptr, 0, stream_);
}

static bool overlaps(const float* a, long long lda, const float* b, long long ldb, int D, long long N) {
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), a1 = a0 + (size_t)((N - 1) * lda + D) * sizeof(float);
  const uintptr_t b0 = reinterpret_cast<uintptr_t>(b), b1 = b0 + (size_t)((N - 1) * ldb + D) * sizeof(float);
  return a0 < b1 && b0 < a1;
}

extern "C" size_t b2b_batchnorm_train_vjp_workspace_bytes(int32_t D) {
  if (D < 1 || D > 1024) return 0;
  // per-CTA partials (<= 1184 CTAs) + acc[4D+2] + this rank's sums[2D+1] + coefficients A, C, B, m
  return (size_t)1184 * (4 * D + 1) * sizeof(double) + (size_t)(6 * D + 3) * sizeof(double) + (size_t)4 * D * sizeof(float) + 256;
}

extern "C" int b2b_batchnorm_train_vjp_f32(const float* x, const float* ybar, const float* ljbar, float* xbar, float* bbar,
                                           float* logsbar, const float* logs, float eps, int32_t D, int64_t N, int64_t ldx,
                                           int64_t ldybar, int64_t ldxbar, b2b_comm* comm, void* workspace,
                                           size_t workspace_bytes, void* stream_) {
  using namespace b2b;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!x || !xbar || !logs || D < 1 || N < 2 || ldx < D || ldxbar < D || (ybar && ldybar < D)) return B2B_EINVAL;
  if ((bbar == nullptr) != (logsbar == nullptr)) return B2B_EINVAL;
  if (overlaps(xbar, ldxbar, x, ldx, D, N)) return B2B_EINVAL;
  if (ybar && overlaps(xbar, ldxbar, ybar, ldybar, D, N) && !(xbar == ybar && ldxbar == ldybar)) return B2B_EINVAL;
  if (D > 1024) return B2B_EUNSUPPORTED;
  if (!workspace || workspace_bytes < b2b_batchnorm_train_vjp_workspace_bytes(D)) return B2B_EWORKSPACE;
  const int grid = stats_grid(N);
  char* ws = b2b_align256(workspace);
  double* partials = reinterpret_cast<double*>(ws);
  double* acc = partials + (size_t)1184 * (4 * D + 1);
  double* loc = acc + 4 * D + 2;
  float* coef = reinterpret_cast<float*>(loc + 2 * D + 1);
  // pass 1: the forward's walk, slices of 128 rows
  const bool vec = (D % 4 == 0) && (ldx % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
                   (!ybar || ((ldybar % 4 == 0) && (reinterpret_cast<uintptr_t>(ybar) & 15) == 0));
  const dim3 g1(grid, (D + 127) / 128);
  const size_t smem = (size_t)(4 * 128 + 1) * sizeof(double);
  if (vec) bn_stats_kernel<1, true, true><<<g1, BNT_THREADS, smem, stream>>>(x, D, N, ldx, ybar, ldybar, ljbar, partials);
  else bn_stats_kernel<1, false, true><<<g1, BNT_THREADS, smem, stream>>>(x, D, N, ldx, ybar, ldybar, ljbar, partials);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  bn_reduce_kernel<<<(4 * D + 1 + 255) / 256, 256, 0, stream>>>(partials, grid, D, 4 * D + 1, N, acc, comm ? loc : nullptr);
  if (comm) {  // sharded batch: one all-reduce of {Σx, Σx², n, Σȳ, Σȳx, Σl̄}
    const int rc = b2b_allreduce_sum_f64(comm, acc, 4 * D + 2, stream);
    if (rc != B2B_OK) return rc;
  }
  bn_vjp_coef_kernel<<<(D + 255) / 256, 256, 0, stream>>>(acc, comm ? loc : acc + 2 * D + 1, logs, eps, D, coef, bbar, logsbar);
  e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  // pass 2
  const bool vec2 = (D % 4 == 0) && (ldx % 4 == 0) && (ldxbar % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
                    ((reinterpret_cast<uintptr_t>(xbar) & 15) == 0) &&
                    (!ybar || ((ldybar % 4 == 0) && (reinterpret_cast<uintptr_t>(ybar) & 15) == 0));
  const int Du = vec2 ? D / 4 : D, rpt = (Du + 255) / 256, Dp = rpt == 1 ? ((Du + 31) & ~31) : 256, nslab = 256 / Dp;
  const int U = rpt == 1 ? 4 : 8 / rpt;
  const int sms = b2b_sm_count();
  long long grid2 = (long long)sms * 4;
  const long long want = (N + (long long)nslab * U - 1) / ((long long)nslab * U);
  if (grid2 > want) grid2 = want;
  void (*apply)(const float*, const float*, float*, const float*, int, long long, long long, long long, long long);
  if (vec2) apply = bn_vjp_apply_kernel<1, 4>;
  else apply = rpt == 1 ? bn_vjp_apply_kernel<1, 1> : rpt == 2 ? bn_vjp_apply_kernel<2, 1> : bn_vjp_apply_kernel<4, 1>;
  apply<<<(int)grid2, 256, 0, stream>>>(x, ybar, xbar, coef, D, N, ldx, ldybar, ldxbar);
  return (int)cudaGetLastError();
}
