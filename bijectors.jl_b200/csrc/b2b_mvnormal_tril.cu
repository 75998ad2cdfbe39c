// Full-covariance MvNormal base, B2B_MVNORMAL_TRIL (include/b2b.h): MvNormal(μ, Σ) with Σ = L Lᵀ given by its lower
// Cholesky factor L -- Distributions' FullNormal, whose PDMat holds exactly that factor.  Third-party arithmetic
// (Distributions / PDMats), restated:
//   logpdf(x) = −½·D·log2π − Σᵢ log Lᵢᵢ − ½·‖r‖²,   r = L⁻¹(x − μ)      (logdet Σ = 2 Σ log Lᵢᵢ; invquad = ‖L⁻¹δ‖²)
//   rand      = μ + L z,  z ~ N(0, I)                                      (PDMats' unwhiten)
//   reverse   s = L⁻ᵀ r,  x̄ = ȳ − l̄·s,  μ̄ = Σₙ l̄ₙ sₙ,  L̄ = tril(Σₙ l̄ₙ sₙ rₙᵀ) − (Σₙ l̄ₙ)·diag(1/Lᵢᵢ)
//
// Mapping (all three kernels).  The packed lower triangle of L (column j holds rows j..D-1, contiguous) is staged once
// per CTA in shared memory, with 1/Lᵢᵢ and μ.  A warp works on 2·C columns: lanes form two groups of 16, group g takes
// C columns and lane t of a group owns rows t, t+16, t+32, ... (R = ceil(D/16) rows per lane, C columns each, all in
// registers).  The substitution steps over j: the owner lane's value is broadcast by a shuffle, and every lane updates
// its rows i > j with L(i, j), read ONCE from shared memory and used for C columns.  The 16 lanes of a group read 16
// consecutive words of column j and the two groups read the same words, so the reads are conflict-free.  Per sample and
// step that is ~R/2 loads per C FMAs and one shuffle per 2 columns; the solve is FP32-FMA bound, not HBM bound
// (D(D+1)/2 FMA for 4·(D+1) B per sample).
//
// Determinism: the grid depends only on D and N; each warp accumulates its columns in a fixed order, each CTA combines
// its warps in order, and every cross-CTA reduction reads per-CTA partials in index order.  No atomics.
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_internal.h"
#include "b2b_v1_pipeline.cuh"  // philox_normal4, V1Gen: the sampling stream of b2b_randn_f32

namespace b2b_tril {

constexpr int kLPG = 16;     // lanes per column group
constexpr int kWarps = 16;   // warps per CTA
constexpr int kMaxGrid = 264;  // fixed (not device-derived), so the partial-sum order depends only on D and N
constexpr unsigned kFull = 0xffffffffu;

// packed column-major lower triangle: L(i, j) (i >= j) at colb(j) + i
__host__ __device__ __forceinline__ int colb(int j, int D) { return j * D - j * (j + 1) / 2; }

size_t smem_bytes(int D) {
  return sizeof(float) * ((size_t)D * (D + 1) / 2 + 2 * (size_t)D) + sizeof(double) * kWarps + 16;
}

// Stages packed L, 1/Lᵢᵢ, μ; returns (in every thread) c0 = −½·D·log2π − Σ log Lᵢᵢ.
__device__ float stage(const float* __restrict__ Lg, const float* __restrict__ mu, int D, float* sL, float* rinv,
                       float* smu, float* sc0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < D; j += kWarps) {
    const int b = colb(j, D);
    for (int i = j + lane; i < D; i += 32) sL[b + i] = __ldg(Lg + (size_t)j * D + i);
  }
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    rinv[i] = 1.0f / __ldg(Lg + (size_t)i * D + i);
    smu[i] = mu ? __ldg(mu + i) : 0.f;
  }
  if (warp == 0) {
    float ls = 0.f;
    for (int i = lane; i < D; i += 32) ls += logf(__ldg(Lg + (size_t)i * D + i));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ls += __shfl_xor_sync(kFull, ls, o);
    if (lane == 0) *sc0 = -0.5f * (D * 1.8378770664093453f) - ls;
  }
  __syncthreads();
  return *sc0;
}

// r := L⁻¹ r (forward substitution, right-looking)
template <int R, int C>
__device__ __forceinline__ void solve_lower(float (&r)[R][C], const float* sL, const float* rinv, int D, int t, int g0) {
#pragma unroll
  for (int kb = 0; kb < R; ++kb) {
#pragma unroll 2
    for (int jj = 0; jj < kLPG; ++jj) {
      const int j = kb * kLPG + jj;
      if (j >= D) break;
      const float ri = rinv[j];
      float v[C];
#pragma unroll
      for (int c = 0; c < C; ++c) {
        v[c] = __shfl_sync(kFull, r[kb][c], g0 + jj) * ri;
        if (t == jj) r[kb][c] = v[c];
      }
      const float* Lc = sL + colb(j, D) + t;
#pragma unroll
      for (int k = kb; k < R; ++k) {
        const int i = t + kLPG * k;
        if ((k != kb || t > jj) && i < D) {
          const float l = Lc[kLPG * k];
#pragma unroll
          for (int c = 0; c < C; ++c) r[k][c] = fmaf(-l, v[c], r[k][c]);
        }
      }
    }
  }
}

// s := L⁻ᵀ s (back substitution, right-looking from the last row): L(j, i) for i < j is read from column i
template <int R, int C>
__device__ __forceinline__ void solve_upper(float (&s)[R][C], const float* sL, const float* rinv, const int (&cb)[R],
                                            int D, int t, int g0) {
#pragma unroll
  for (int kb = R - 1; kb >= 0; --kb) {
#pragma unroll 2
    for (int jj = kLPG - 1; jj >= 0; --jj) {
      const int j = kb * kLPG + jj;
      if (j >= D) continue;
      const float ri = rinv[j];
      float v[C];
#pragma unroll
      for (int c = 0; c < C; ++c) {
        v[c] = __shfl_sync(kFull, s[kb][c], g0 + jj) * ri;
        if (t == jj) s[kb][c] = v[c];
      }
#pragma unroll
      for (int k = 0; k <= kb; ++k) {
        if (k != kb || t < jj) {
          const float l = sL[cb[k] + j];
#pragma unroll
          for (int c = 0; c < C; ++c) s[k][c] = fmaf(-l, v[c], s[k][c]);
        }
      }
    }
  }
}

// column-group sum over the 16 lanes of a group (fixed butterfly order)
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = kLPG / 2; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

__device__ __forceinline__ void cta_partial(double acc, double* red, double* partials) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += red[w];
    partials[blockIdx.x] = s;
  }
}

struct Smem {
  float *L, *rinv, *mu, *c0;
  double* red;
};
__device__ __forceinline__ Smem carve(int D) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem s;
  s.red = reinterpret_cast<double*>(smem_raw);
  s.c0 = reinterpret_cast<float*>(smem_raw + sizeof(double) * kWarps);
  s.rinv = s.c0 + 4;
  s.mu = s.rinv + D;
  s.L = s.mu + D;
  return s;
}

// logpdf[n] (+ logjac[n] when accumulate) into logjac (may be NULL), optional copy of x into y, per-CTA batch sums
template <int R, int C>
__global__ void __launch_bounds__(kWarps * 32, 1)
    logpdf_kernel(const float* __restrict__ x, long long ldx, float* __restrict__ y, long long ldy, float* logjac,
                  int accumulate, double* __restrict__ partials, const float* __restrict__ Lg,
                  const float* __restrict__ mu, int D, long long N) {
  const Smem sm = carve(D);
  const float c0 = stage(Lg, mu, D, sm.L, sm.rinv, sm.mu, sm.c0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = lane & (kLPG - 1), g0 = lane & kLPG;
  double acc = 0.0;
  const long long chunks = (N + 2 * C - 1) / (2 * C);
  for (long long ch = (long long)blockIdx.x * kWarps + warp; ch < chunks; ch += (long long)gridDim.x * kWarps) {
    const long long col0 = ch * 2 * C + (g0 ? C : 0);
    float r[R][C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const long long n = col0 + c;
#pragma unroll
      for (int k = 0; k < R; ++k) {
        const int i = t + kLPG * k;
        float v = 0.f;
        if (n < N && i < D) {
          const float xv = x[n * ldx + i];
          if (y) y[n * ldy + i] = xv;
          v = xv - sm.mu[i];
        }
        r[k][c] = v;
      }
    }
    solve_lower<R, C>(r, sm.L, sm.rinv, D, t, g0);
#pragma unroll
    for (int c = 0; c < C; ++c) {
      float q = 0.f;
#pragma unroll
      for (int k = 0; k < R; ++k) q = fmaf(r[k][c], r[k][c], q);
      q = group_sum(q);
      const long long n = col0 + c;
      if (t == c && n < N) {
        float lp = fmaf(-0.5f, q, c0);
        if (accumulate && logjac) lp += logjac[n];
        if (logjac) logjac[n] = lp;
        acc += (double)lp;
      }
    }
  }
  if (partials) cta_partial(acc, sm.red, partials);
}

// reverse mode, per column: x̄ = ȳ − l̄·s; with want_params, r and l̄·s go to Rw / Sw (D x N, ld = D) for the L̄ GEMM,
// and every CTA writes its Σ l̄ to ljp[blockIdx.x]
template <int R, int C>
__global__ void __launch_bounds__(kWarps * 32, 1)
    vjp_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ ybar, long long ldyb,
               const float* __restrict__ ljbar, float* __restrict__ xbar, long long ldxb, float* __restrict__ Rw,
               float* __restrict__ Sw, double* __restrict__ ljp, const float* __restrict__ Lg,
               const float* __restrict__ mu, int D, long long N) {
  const Smem sm = carve(D);
  stage(Lg, mu, D, sm.L, sm.rinv, sm.mu, sm.c0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = lane & (kLPG - 1), g0 = lane & kLPG;
  int cb[R];
#pragma unroll
  for (int k = 0; k < R; ++k) {
    const int i = t + kLPG * k;
    cb[k] = i < D ? colb(i, D) : 0;
  }
  double acc = 0.0;
  const long long chunks = (N + 2 * C - 1) / (2 * C);
  for (long long ch = (long long)blockIdx.x * kWarps + warp; ch < chunks; ch += (long long)gridDim.x * kWarps) {
    const long long col0 = ch * 2 * C + (g0 ? C : 0);
    float r[R][C], s[R][C], lb[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const long long n = col0 + c;
      lb[c] = (n < N && ljbar) ? ljbar[n] : 0.f;
#pragma unroll
      for (int k = 0; k < R; ++k) {
        const int i = t + kLPG * k;
        r[k][c] = (n < N && i < D) ? x[n * ldx + i] - sm.mu[i] : 0.f;
      }
      if (t == c && n < N) acc += (double)lb[c];
    }
    solve_lower<R, C>(r, sm.L, sm.rinv, D, t, g0);
#pragma unroll
    for (int k = 0; k < R; ++k)
#pragma unroll
      for (int c = 0; c < C; ++c) s[k][c] = r[k][c];
    solve_upper<R, C>(s, sm.L, sm.rinv, cb, D, t, g0);
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const long long n = col0 + c;
      if (n >= N) continue;
#pragma unroll
      for (int k = 0; k < R; ++k) {
        const int i = t + kLPG * k;
        if (i >= D) continue;
        const float ls = lb[c] * s[k][c];
        xbar[n * ldxb + i] = (ybar ? ybar[n * ldyb + i] : 0.f) - ls;
        if (Rw) {
          Rw[n * D + i] = r[k][c];
          Sw[n * D + i] = ls;
        }
      }
    }
  }
  if (ljp) cta_partial(acc, sm.red, ljp);
}

// y = μ + L z with z the Philox stream of b2b_randn_f32 (rows 4k..4k+3 of global column n from one counter).
// LOGQ: also logq[n] = qsign·(c0 − ½‖zₙ‖²), the base log-density of the sample from the z it holds in registers.
template <int R, int C, bool LOGQ>
__device__ __forceinline__ void sample_body(float* __restrict__ y, long long ldy, const b2b::V1Gen& gen,
                                            const float* __restrict__ Lg, const float* __restrict__ mu, int D, long long N,
                                            float* __restrict__ logq, float qsign) {
  const Smem sm = carve(D);
  const float c0 = stage(Lg, mu, D, sm.L, sm.rinv, sm.mu, sm.c0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = lane & (kLPG - 1), g0 = lane & kLPG;
  const long long chunks = (N + 2 * C - 1) / (2 * C);
  for (long long ch = (long long)blockIdx.x * kWarps + warp; ch < chunks; ch += (long long)gridDim.x * kWarps) {
    const long long col0 = ch * 2 * C + (g0 ? C : 0);
    float z[R][C], acc[R][C];
    // Each Philox call gives the four normals of rows 4p..4p+3.  Lane t draws quads p = t + 16·kk, so each quad is drawn
    // once; row i = t + 16k (quad 4k + t/4, element t mod 4) is then fetched from lane 4·(k mod 4) + t/4 of its group.
    constexpr int KQ = (R + 3) / 4;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const long long n = col0 + c;
      float4 q[KQ];
#pragma unroll
      for (int kk = 0; kk < KQ; ++kk)
        q[kk] = (n < N && 4 * (t + kLPG * kk) < D) ? b2b::philox_normal4(gen, gen.col0 + n, t + kLPG * kk)
                                                     : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int k = 0; k < R; ++k) {
        const int i = t + kLPG * k, src = g0 + 4 * (k & 3) + (t >> 2), e = t & 3;
        const float4 w = q[k >> 2];
        const float a0 = __shfl_sync(kFull, w.x, src), a1 = __shfl_sync(kFull, w.y, src);
        const float a2 = __shfl_sync(kFull, w.z, src), a3 = __shfl_sync(kFull, w.w, src);
        const float v = e == 0 ? a0 : e == 1 ? a1 : e == 2 ? a2 : a3;
        z[k][c] = (n < N && i < D) ? v : 0.f;
        acc[k][c] = i < D ? sm.mu[i] : 0.f;
      }
    }
#pragma unroll
    for (int kb = 0; kb < R; ++kb) {
#pragma unroll 2
      for (int jj = 0; jj < kLPG; ++jj) {
        const int j = kb * kLPG + jj;
        if (j >= D) break;
        float v[C];
#pragma unroll
        for (int c = 0; c < C; ++c) v[c] = __shfl_sync(kFull, z[kb][c], g0 + jj);
        const float* Lc = sm.L + colb(j, D) + t;
#pragma unroll
        for (int k = kb; k < R; ++k) {
          const int i = t + kLPG * k;
          if ((k != kb || t >= jj) && i < D) {
            const float l = Lc[kLPG * k];
#pragma unroll
            for (int c = 0; c < C; ++c) acc[k][c] = fmaf(l, v[c], acc[k][c]);
          }
        }
      }
    }
    if constexpr (LOGQ) {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < R; ++k) q = fmaf(z[k][c], z[k][c], q);
        q = group_sum(q);
        const long long n = col0 + c;
        if (t == c && n < N) logq[n] = qsign * fmaf(-0.5f, q, c0);
      }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const long long n = col0 + c;
      if (n >= N) continue;
#pragma unroll
      for (int k = 0; k < R; ++k) {
        const int i = t + kLPG * k;
        if (i < D) y[n * ldy + i] = acc[k][c];
      }
    }
  }
}

template <int R, int C>
__global__ void __launch_bounds__(kWarps * 32, 1)
    sample_kernel(float* __restrict__ y, long long ldy, const b2b::V1Gen gen, const float* __restrict__ Lg,
                  const float* __restrict__ mu, int D, long long N) {
  sample_body<R, C, false>(y, ldy, gen, Lg, mu, D, N, nullptr, 0.f);
}

template <int R, int C>
__global__ void __launch_bounds__(kWarps * 32, 1)
    sample_logq_kernel(float* __restrict__ y, long long ldy, const b2b::V1Gen gen, const float* __restrict__ Lg,
                       const float* __restrict__ mu, int D, long long N, float* __restrict__ logq, float qsign) {
  sample_body<R, C, true>(y, ldy, gen, Lg, mu, D, N, logq, qsign);
}

// ---- L̄ = tril(S Rᵀ) over column chunks: CTA (tile, p) writes the 64 x 64 tile of Σ_{n in chunk p} S[:, n] R[:, n]ᵀ
// to part[p] (D x D, column-major): with `lower` the lower-triangle tiles only, whose diagonal tiles also write the
// chunk's row sums of S (μ̄) to mup[p] when it is given; otherwise every tile (dense Scale's G = Σ ȳ uᵀ).  fp32 FMA over
// blocks of kFlush stages (16 384 columns), fp64 across the blocks of a chunk and across chunks (finalize_kernel): a chunk
// holds up to N / kMaxChunks columns (65 536 at N = 2²²), and one fp32 sum over all of them loses ~1e-5 relative.  Up to
// N = 2²⁰ a chunk is one block.
constexpr int kTile = 64, kBK = 16, kChunk = 4096, kMaxChunks = 64, kFlush = 1024;

__global__ void __launch_bounds__(256) outer_kernel(const float* __restrict__ S, long long lds, const float* __restrict__ Rm,
                                                    long long ldr, float* __restrict__ part, float* __restrict__ mup, int D,
                                                    long long N, long long clen, bool lower) {
  __shared__ __align__(16) float As[kBK][kTile];
  __shared__ __align__(16) float Bs[kBK][kTile];
  int ti = 0, tj = 0;
  if (lower) {  // lower-triangle tile (ti, tj), ti >= tj, in row order
    int rem = blockIdx.x;
    while (rem > ti) rem -= ++ti;
    tj = rem;
  } else {  // every tile, in row order
    const int T = (D + kTile - 1) / kTile;
    ti = blockIdx.x / T;
    tj = blockIdx.x - ti * T;
  }
  const bool diag = lower && ti == tj && mup;
  const int p = blockIdx.y, i0 = ti * kTile, j0 = tj * kTile;
  const long long n0 = (long long)p * clen, n1 = n0 + clen < N ? n0 + clen : N;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int lk = threadIdx.x >> 4, lr = (threadIdx.x & 15) * 4;  // loader: column lk of the stage, rows lr..lr+3
  double accd[4][4] = {};
  double msumd = 0.0;
  for (long long nf = n0; nf < n1; nf += (long long)kFlush * kBK) {
    const long long nf1 = nf + (long long)kFlush * kBK < n1 ? nf + (long long)kFlush * kBK : n1;
    float acc[4][4] = {};
    float msum = 0.f;
    for (long long nb = nf; nb < nf1; nb += kBK) {
      const long long n = nb + lk;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int ia = i0 + lr + q, ja = j0 + lr + q;
        As[lk][lr + q] = (n < nf1 && ia < D) ? S[n * lds + ia] : 0.f;
        Bs[lk][lr + q] = (n < nf1 && ja < D) ? Rm[n * ldr + ja] : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kBK; ++k) {
        const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int v = 0; v < 4; ++v) acc[u][v] = fmaf(av[u], bv[v], acc[u][v]);
      }
      if (diag && threadIdx.x < kTile) {
#pragma unroll
        for (int k = 0; k < kBK; ++k) msum += As[k][threadIdx.x];
      }
      __syncthreads();
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) accd[u][v] += (double)acc[u][v];
    msumd += (double)msum;
  }
  float* P = part + (size_t)p * D * D;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int i = i0 + ty * 4 + u, j = j0 + tx * 4 + v;
      if (i < D && j < D && (i >= j || !lower)) P[(size_t)j * D + i] = (float)accd[u][v];
    }
  if (diag && threadIdx.x < kTile && i0 + (int)threadIdx.x < D) mup[(size_t)p * D + i0 + threadIdx.x] = (float)msumd;
}

// L̄ (D x D column-major, exactly zero above the diagonal) and μ̄ from the chunk partials, in chunk order
__global__ void __launch_bounds__(256) finalize_kernel(const float* __restrict__ part, const float* __restrict__ mup,
                                                       int P, const double* __restrict__ ljp, int nljp,
                                                       const float* __restrict__ Lg, float* __restrict__ Lbar,
                                                       float* __restrict__ mubar, int D) {
  __shared__ double ljs;
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < nljp; ++k) s += ljp[k];
    ljs = s;
  }
  __syncthreads();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x, DD = (long long)D * D;
  if (idx < DD) {
    if (!Lbar) return;
    const int j = (int)(idx / D), i = (int)(idx - (long long)j * D);
    if (i < j) {
      Lbar[idx] = 0.f;
      return;
    }
    double a = 0.0;
    for (int p = 0; p < P; ++p) a += (double)part[(size_t)p * DD + idx];
    if (i == j) a -= ljs / (double)__ldg(Lg + idx);
    Lbar[idx] = (float)a;
  } else if (idx < DD + D) {
    if (!mubar) return;
    const int i = (int)(idx - DD);
    double a = 0.0;
    for (int p = 0; p < P; ++p) a += (double)mup[(size_t)p * D + i];
    mubar[i] = (float)a;
  }
}

int grid_for(int C, long long N) {
  const long long chunks = (N + 2 * C - 1) / (2 * C);
  const long long g = (chunks + kWarps - 1) / kWarps;
  return (int)(g < kMaxGrid ? (g > 0 ? g : 1) : kMaxGrid);
}

// rows per lane (compile-time) for D; C columns per lane for the solve and for the two-register-array kernels
int rows_per_lane(int D) { return D <= 16 ? 1 : D <= 32 ? 2 : D <= 64 ? 4 : D <= 128 ? 8 : 16; }
constexpr int c_logpdf(int R) { return R >= 16 ? 4 : 8; }
constexpr int c_two(int R) { return R >= 16 ? 2 : 4; }

template <class K>
int launch(K kernel, int grid, int D, cudaStream_t stream, auto... args) {
  const size_t smem = smem_bytes(D);
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<grid, kWarps * 32, smem, stream>>>(args...);
  return (int)cudaGetLastError();
}

long long chunk_len(long long N) {
  long long P = (N + kChunk - 1) / kChunk;
  if (P > kMaxChunks) P = kMaxChunks;
  if (P < 1) P = 1;
  const long long c = (N + P - 1) / P;
  return (c + kBK - 1) / kBK * kBK;
}

}  // namespace b2b_tril

using namespace b2b_tril;

long long b2b_outer_chunk_len(long long N) { return chunk_len(N); }

int b2b_launch_outer_chunks(const float* S, long long lds, const float* R, long long ldr, float* part, float* mup, int D,
                            long long N, bool lower, cudaStream_t stream) {
  const long long clen = chunk_len(N), P = (N + clen - 1) / clen;
  const int T = (D + kTile - 1) / kTile;
  outer_kernel<<<dim3(lower ? T * (T + 1) / 2 : T * T, (unsigned)P), 256, 0, stream>>>(S, lds, R, ldr, part, mup, D, N,
                                                                                        clen, lower);
  return (int)cudaGetLastError();
}

// logjac := logpdf of x, the recovered point (+ logjac when accumulate); with partials, their per-CTA sums as well
int b2b_fwd_tril(const B2BFwdSeg& s) {
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  const long long N = s.N;
  if (D < 1 || D > B2B_TRIL_MAX_D) return B2B_EUNSUPPORTED;
  float* const y = s.y == s.x ? nullptr : s.y;  // in place: nothing to copy
  const int R = rows_per_lane(D);
  const int grid = grid_for(c_logpdf(R), N);
  int rc = B2B_EUNSUPPORTED;
#define B2B_TRIL_LP(RR)                                                                                                \
  case RR:                                                                                                             \
    rc = launch(logpdf_kernel<RR, c_logpdf(RR)>, grid, D, s.stream, s.x, s.ldx, y, s.ldy, s.logjac, s.accumulate,     \
                s.partials, d.p1, d.p0, D, N);                                                                         \
    break;
  switch (R) {
    B2B_TRIL_LP(1) B2B_TRIL_LP(2) B2B_TRIL_LP(4) B2B_TRIL_LP(8) B2B_TRIL_LP(16)
  }
#undef B2B_TRIL_LP
  if (rc != B2B_OK) return rc;
  ++*s.launches;
  if (!s.partials) return B2B_OK;
  if ((rc = b2b_launch_sum_partials(s.partials, grid, s.sum_out, s.stream)) != B2B_OK) return rc;
  ++*s.launches;
  return B2B_OK;
}

// workspace: [r | l̄·s] (2 x D x N floats) [chunk partials of L̄ (P x D x D) and μ̄ (P x D)] [per-CTA Σ l̄ (kMaxGrid doubles)]
size_t b2b_tril_vjp_workspace(int D, long long N) {
  if (D < 1 || D > B2B_TRIL_MAX_D || N < 0) return 0;
  const long long clen = chunk_len(N), P = N > 0 ? (N + clen - 1) / clen : 1;
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  return 2 * al(sizeof(float) * (size_t)D * N) + al(sizeof(float) * (size_t)P * D * (D + 1)) +
         al(sizeof(double) * kMaxGrid);
}

int b2b_vjp_tril(const B2BVjpSeg& s) {
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  const long long N = s.N;
  float* const mubar = s.bars[0];
  float* const Lbar = s.bars[1];
  const cudaStream_t stream = s.stream;
  if (D < 1 || D > B2B_TRIL_MAX_D) return B2B_EUNSUPPORTED;
  const bool params = mubar || Lbar;
  if (params && s.workspace_bytes < b2b_tril_vjp_workspace(D, N)) return B2B_EWORKSPACE;
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  char* ws = static_cast<char*>(s.workspace);
  float* Rw = params ? reinterpret_cast<float*>(ws) : nullptr;
  float* Sw = params ? reinterpret_cast<float*>(ws + al(sizeof(float) * (size_t)D * N)) : nullptr;
  const long long clen = chunk_len(N), P = (N + clen - 1) / clen;
  float* part = params ? reinterpret_cast<float*>(ws + 2 * al(sizeof(float) * (size_t)D * N)) : nullptr;
  float* mup = part ? part + (size_t)P * D * D : nullptr;
  double* ljp = params ? reinterpret_cast<double*>(reinterpret_cast<char*>(part) + al(sizeof(float) * (size_t)P * D * (D + 1)))
                       : nullptr;
  const int R = rows_per_lane(D);
  int grid = 0, rc = B2B_EUNSUPPORTED;
#define B2B_TRIL_VJP(RR)                                                                                             \
  case RR:                                                                                                           \
    grid = grid_for(c_two(RR), N);                                                                                   \
    rc = launch(vjp_kernel<RR, c_two(RR)>, grid, D, stream, s.x, s.ldx, s.ybar, s.ldyb, s.ljbar, s.xbar, s.ldxb, Rw, Sw, \
                ljp, d.p1, d.p0, D, N);                                                                              \
    break;
  switch (R) {
    B2B_TRIL_VJP(1) B2B_TRIL_VJP(2) B2B_TRIL_VJP(4) B2B_TRIL_VJP(8) B2B_TRIL_VJP(16)
  }
#undef B2B_TRIL_VJP
  if (rc != B2B_OK) return rc;
  ++*s.launches;
  if (!params) return B2B_OK;
  if ((rc = b2b_launch_outer_chunks(Sw, D, Rw, D, part, mup, D, N, true, stream)) != B2B_OK) return rc;
  const long long tot = (long long)D * D + D;
  finalize_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(part, mup, (int)P, ljp, grid, d.p1, Lbar, mubar, D);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  *s.launches += 2;
  return B2B_OK;
}

extern "C" int b2b_chain_sample_tril_f32(const b2b_layer_desc* layers, int32_t L, const float* mu,
                                         const float* scale_tril, uint64_t seed, uint64_t offset, int64_t column_offset,
                                         float* y, float* logjac, int32_t D, int64_t N, int64_t ldy, void* workspace,
                                         size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  b2b_set_last_launch_count(0);
  if (L < 0 || L > B2B_MAX_CHAIN || (L > 0 && !layers) || D < 1 || N < 0 || ldy < D || !scale_tril) return B2B_EINVAL;
  if (D > B2B_TRIL_MAX_D) return B2B_EUNSUPPORTED;
  if (L > 0) {  // refuse an unsupported chain before the samples are drawn
    const int rc = b2b_chain_check_f32(layers, L, D);
    if (rc != B2B_OK) return rc;
  }
  if (N == 0) return B2B_OK;
  if (!y) return B2B_EINVAL;
  int launches = 0;
  if (L == 0 && logjac) {
    const cudaError_t e = cudaMemsetAsync(logjac, 0, (size_t)N * sizeof(float), stream);
    if (e != cudaSuccess) return (int)e;
    ++launches;
  }
  const b2b::V1Gen gen{seed, offset, column_offset, nullptr, nullptr};
  const int R = rows_per_lane(D);
  int rc = B2B_EUNSUPPORTED;
#define B2B_TRIL_SMP(RR)                                                                                          \
  case RR:                                                                                                        \
    rc = launch(sample_kernel<RR, c_two(RR)>, grid_for(c_two(RR), N), D, stream, y, (long long)ldy, gen, scale_tril, \
                mu, D, (long long)N);                                                                             \
    break;
  switch (R) {
    B2B_TRIL_SMP(1) B2B_TRIL_SMP(2) B2B_TRIL_SMP(4) B2B_TRIL_SMP(8) B2B_TRIL_SMP(16)
  }
#undef B2B_TRIL_SMP
  if (rc != B2B_OK) return rc;
  ++launches;
  if (L > 0) {  // the chain in place, as the two-pass path of b2b_chain_sample_f32
    rc = b2b_chain_run_f32(layers, L, y, y, logjac, nullptr, D, N, ldy, ldy, 0, workspace, workspace_bytes, stream_);
    if (rc != B2B_OK) return rc;
    launches += b2b_last_launch_count();
  }
  b2b_set_last_launch_count(launches);
  return B2B_OK;
}

// ---- the TRIL base of the reparameterised sampler (b2b_rsample.cu) ----------------------------------------------------
int b2b_tril_sample(const float* Lg, const float* mu, uint64_t seed, uint64_t offset, long long col0, float* y,
                    long long ldy, float* logq, float qsign, int D, long long N, cudaStream_t stream) {
  if (D < 1 || D > B2B_TRIL_MAX_D) return B2B_EUNSUPPORTED;
  const b2b::V1Gen gen{seed, offset, col0, nullptr, nullptr};
  const int R = rows_per_lane(D);
  int rc = B2B_EUNSUPPORTED;
#define B2B_TRIL_SMPQ(RR)                                                                                          \
  case RR:                                                                                                         \
    rc = logq ? launch(sample_logq_kernel<RR, c_two(RR)>, grid_for(c_two(RR), N), D, stream, y, ldy, gen, Lg, mu, D, \
                       N, logq, qsign)                                                                             \
              : launch(sample_kernel<RR, c_two(RR)>, grid_for(c_two(RR), N), D, stream, y, ldy, gen, Lg, mu, D, N); \
    break;
  switch (R) {
    B2B_TRIL_SMPQ(1) B2B_TRIL_SMPQ(2) B2B_TRIL_SMPQ(4) B2B_TRIL_SMPQ(8) B2B_TRIL_SMPQ(16)
  }
#undef B2B_TRIL_SMPQ
  return rc;
}

size_t b2b_tril_base_vjp_workspace(int D, long long N) {
  if (D < 1 || D > B2B_TRIL_MAX_D || N < 1) return 0;
  const long long clen = chunk_len(N), P = (N + clen - 1) / clen;
  return (sizeof(float) * (size_t)P * D * (D + 1) + 255) & ~(size_t)255;
}

int b2b_tril_base_vjp(const float* xbar, long long ldxb, const float* z, const double* qsum, const float* Lg,
                      float* mubar, float* Lbar, int D, long long N, void* workspace, int* launches,
                      cudaStream_t stream) {
  const long long clen = chunk_len(N), P = (N + clen - 1) / clen;
  float* part = static_cast<float*>(workspace);
  float* mup = mubar ? part + (size_t)P * D * D : nullptr;
  int rc = b2b_launch_outer_chunks(xbar, ldxb, z, D, part, mup, D, N, true, stream);
  if (rc != B2B_OK) return rc;
  const long long tot = (long long)D * D + D;
  finalize_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(part, mup, (int)P, qsum, qsum ? 1 : 0, Lg, Lbar,
                                                                     mubar, D);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  *launches += 2;
  return B2B_OK;
}
