// Dense linear layer, B2B_SCALE_MATRIX (include/b2b.h): Scale(A) with a D x D matrix A (scale.jl:14,17,35-36):
//   forward   y = A x,    logjac = log|det A|          inverse   y = A⁻¹ x,   logjac = −log|det A|
//   reverse   (u the layer's input, M = A or A⁻¹, G = Σₙ ȳₙ uₙᵀ, s = Σₙ l̄ₙ, B = A⁻ᵀ)
//             forward layer: x̄ = Aᵀ ȳ,    Ā = G + s·B
//             inverse layer: x̄ = A⁻ᵀ ȳ,   Ā = −B G B − s·B
//
// factor_kernel (one CTA of 512 threads): blocked right-looking LU with partial pivoting of the fp32 A in fp64 (what
// logabsdet computes through getrf), column-major in the workspace.  A panel of kNB columns is factored in shared
// memory (pivot search by one warp, first maximum wins as in idamax), its row swaps are applied to the other columns
// one column per thread, the block row U12 is solved against the unit lower L11, and the trailing matrix takes the
// rank-kNB update A22 −= L21·U12 in one read and one write per element.  log|det A| = Σ log|Uᵢᵢ| in row order.  A zero
// pivot leaves its column unscaled (getrf's convention), so a singular A gives −Inf and finite y = A x.
// inv_kernel: A⁻¹ column by column from P A = L U; a warp solves kInvC columns, lanes own rows, and both substitutions
// step over k reading column k of L / U once (coalesced) for all of them.  M = A⁻¹ is rounded to fp32.
// map_kernel<DP, BN, TRANS>: Y = M X (or Mᵀ X) in exact fp32 FFMA.  A CTA owns all D rows of BN columns: it stages the
// x tile (rows padded to DP) in shared memory before anything is stored -- so y may alias x -- streams M through
// shared memory in k-blocks of kBK (double buffered through registers), and each thread keeps an 8 x 8 register tile.
// Every output is one fmaf chain in increasing k: results do not depend on N, the tile or the launch.
// Reverse mode: x̄ by map_kernel with the transposed operand; G by the chunked outer-product kernel of the full-covariance
// base (all tiles), its chunks and Σ l̄ summed in a fixed order in fp64, and the two D x D products of the inverse layer
// in fp64.  No atomics; every launch is graph-capturable.
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>

#include "b2b_internal.h"

namespace b2b_scale {

constexpr int kFactorThreads = 512;
constexpr int kNB = 16;     // LU panel width
constexpr int kInvC = 4;    // columns of A⁻¹ per warp
constexpr int kInvWarps = 4;
constexpr int kBK = 16;     // k-block of the map GEMM
constexpr unsigned kFull = 0xffffffffu;

size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

// factor storage: [LU (D x D fp64, column-major)][M = A⁻¹ (D x D fp32)][perm (D int32)][log|det A| (fp64)]
struct Factor {
  double* lu;
  float* minv;
  int* perm;
  double* logdet;
};

size_t factor_bytes(int D) {
  return al256(sizeof(double) * (size_t)D * D) + al256(sizeof(float) * (size_t)D * D) + al256(sizeof(int) * (size_t)D) +
         al256(sizeof(double)) + 256;
}

Factor carve(void* ws, int D) {
  char* p = b2b_align256(ws);
  Factor f;
  f.lu = reinterpret_cast<double*>(p);
  p += al256(sizeof(double) * (size_t)D * D);
  f.minv = reinterpret_cast<float*>(p);
  p += al256(sizeof(float) * (size_t)D * D);
  f.perm = reinterpret_cast<int*>(p);
  p += al256(sizeof(int) * (size_t)D);
  f.logdet = reinterpret_cast<double*>(p);
  return f;
}

size_t factor_smem(int D) { return sizeof(double) * 2 * (size_t)kNB * D + sizeof(int) * ((size_t)D + kNB + 4); }

__global__ void __launch_bounds__(kFactorThreads, 1)
    factor_kernel(const float* __restrict__ A, int D, double* __restrict__ lu, int* __restrict__ perm_out,
                  double* __restrict__ logdet) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* Ps = reinterpret_cast<double*>(smem_raw);  // panel: Ps[c * D + i], column c of the panel, row i
  double* Us = Ps + (size_t)kNB * D;                 // block row U12: Us[r * D + j]
  int* perm = reinterpret_cast<int*>(Us + (size_t)kNB * D);
  int* pivs = perm + D;
  int* sp = pivs + kNB;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (long long idx = tid; idx < (long long)D * D; idx += kFactorThreads) lu[idx] = (double)__ldg(A + idx);
  for (int i = tid; i < D; i += kFactorThreads) perm[i] = i;
  double ld = 0.0;  // thread 0
  __syncthreads();
  for (int k0 = 0; k0 < D; k0 += kNB) {
    const int nb = D - k0 < kNB ? D - k0 : kNB;
    for (int idx = tid; idx < nb * D; idx += kFactorThreads) {
      const int c = idx / D, i = idx - c * D;
      if (i >= k0) Ps[c * D + i] = lu[(size_t)(k0 + c) * D + i];
    }
    __syncthreads();
    // unblocked LU of the panel (rows k0..D-1)
    for (int c = 0; c < nb; ++c) {
      const int kk = k0 + c;
      if (warp == 0) {
        double best = -1.0;
        int bi = D;
        for (int i = kk + lane; i < D; i += 32) {
          const double v = fabs(Ps[c * D + i]);
          if (v > best) {
            best = v;
            bi = i;
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const double ov = __shfl_xor_sync(kFull, best, o);
          const int oi = __shfl_xor_sync(kFull, bi, o);
          if (ov > best || (ov == best && oi < bi)) {
            best = ov;
            bi = oi;
          }
        }
        if (lane == 0) {
          *sp = bi < D ? bi : kk;  // NaN column: no swap
          pivs[c] = *sp;
        }
      }
      __syncthreads();
      const int p = *sp;
      if (p != kk && tid < nb) {
        const double t = Ps[tid * D + kk];
        Ps[tid * D + kk] = Ps[tid * D + p];
        Ps[tid * D + p] = t;
      }
      __syncthreads();
      const double piv = Ps[c * D + kk];
      if (tid == 0) ld += log(fabs(piv));
      for (int i = kk + 1 + tid; i < D; i += kFactorThreads)
        if (piv != 0.0) Ps[c * D + i] /= piv;
      __syncthreads();
      const int m = D - kk - 1;
      for (int idx = tid; idx < (nb - c - 1) * m; idx += kFactorThreads) {
        const int c2 = c + 1 + idx / m, i = kk + 1 + idx % m;
        Ps[c2 * D + i] = fma(-Ps[c * D + i], Ps[c2 * D + kk], Ps[c2 * D + i]);
      }
      __syncthreads();
    }
    // the panel back to global; its row swaps applied to every other column (one column per thread, in order)
    for (int idx = tid; idx < nb * D; idx += kFactorThreads) {
      const int c = idx / D, i = idx - c * D;
      if (i >= k0) lu[(size_t)(k0 + c) * D + i] = Ps[c * D + i];
    }
    for (int j = tid; j < D; j += kFactorThreads) {
      if (j >= k0 && j < k0 + nb) continue;
      double* col = lu + (size_t)j * D;
      for (int c = 0; c < nb; ++c) {
        const int p = pivs[c];
        if (p != k0 + c) {
          const double t = col[k0 + c];
          col[k0 + c] = col[p];
          col[p] = t;
        }
      }
    }
    if (tid == 0)
      for (int c = 0; c < nb; ++c) {
        const int p = pivs[c], t = perm[k0 + c];
        perm[k0 + c] = perm[p];
        perm[p] = t;
      }
    __syncthreads();
    const int j0 = k0 + nb;
    if (j0 >= D) break;
    // U12 = L11⁻¹ A12, one column per thread, worked on in shared memory
    for (int j = j0 + tid; j < D; j += kFactorThreads) {
      double* col = lu + (size_t)j * D + k0;
      for (int r = 0; r < nb; ++r) Us[r * D + j] = col[r];
      for (int r = 0; r < nb; ++r) {
        const double ur = Us[r * D + j];
        for (int r2 = r + 1; r2 < nb; ++r2) Us[r2 * D + j] = fma(-Ps[r * D + k0 + r2], ur, Us[r2 * D + j]);
        col[r] = ur;
      }
    }
    __syncthreads();
    // A22 −= L21 · U12
    const int m = D - j0;
    for (int idx = tid; idx < m * m; idx += kFactorThreads) {
      const int j = j0 + idx / m, i = j0 + idx % m;
      double* a = lu + (size_t)j * D + i;
      double v = *a;
      for (int r = 0; r < nb; ++r) v = fma(-Ps[r * D + i], Us[r * D + j], v);
      *a = v;
    }
    __syncthreads();
  }
  for (int i = tid; i < D; i += kFactorThreads) perm_out[i] = perm[i];
  if (tid == 0) *logdet = ld;
}

// columns of M = A⁻¹ (fp32, column-major): solve L U z = P e_j
template <int R>
__global__ void __launch_bounds__(kInvWarps * 32)
    inv_kernel(const double* __restrict__ lu, const int* __restrict__ perm, float* __restrict__ minv, int D) {
  const int lane = threadIdx.x & 31;
  const int col0 = (blockIdx.x * kInvWarps + (threadIdx.x >> 5)) * kInvC;
  if (col0 >= D) return;
  double z[R][kInvC];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int i = lane + 32 * r;
    const int pi = i < D ? perm[i] : -1;
#pragma unroll
    for (int c = 0; c < kInvC; ++c) z[r][c] = (pi == col0 + c) ? 1.0 : 0.0;
  }
  // forward substitution, unit lower L (right-looking)
#pragma unroll
  for (int kb = 0; kb < R; ++kb) {
    for (int jj = 0; jj < 32; ++jj) {
      const int k = kb * 32 + jj;
      if (k >= D) break;
      double v[kInvC];
#pragma unroll
      for (int c = 0; c < kInvC; ++c) v[c] = __shfl_sync(kFull, z[kb][c], jj);
      const double* Lk = lu + (size_t)k * D;
#pragma unroll
      for (int r = kb; r < R; ++r) {
        const int i = lane + 32 * r;
        if (i > k && i < D) {
          const double l = Lk[i];
#pragma unroll
          for (int c = 0; c < kInvC; ++c) z[r][c] = fma(-l, v[c], z[r][c]);
        }
      }
    }
  }
  // back substitution, upper U
#pragma unroll
  for (int kb = R - 1; kb >= 0; --kb) {
    for (int jj = 31; jj >= 0; --jj) {
      const int k = kb * 32 + jj;
      if (k >= D) continue;
      const double* Uk = lu + (size_t)k * D;
      const double ukk = Uk[k];
      double v[kInvC];
#pragma unroll
      for (int c = 0; c < kInvC; ++c) {
        v[c] = __shfl_sync(kFull, z[kb][c], jj) / ukk;
        if (lane == jj) z[kb][c] = v[c];
      }
#pragma unroll
      for (int r = 0; r <= kb; ++r) {
        const int i = lane + 32 * r;
        if (i < k) {
          const double u = Uk[i];
#pragma unroll
          for (int c = 0; c < kInvC; ++c) z[r][c] = fma(-u, v[c], z[r][c]);
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < kInvC; ++c) {
    const int j = col0 + c;
    if (j >= D) break;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int i = lane + 32 * r;
      if (i < D) minv[(size_t)j * D + i] = (float)z[r][c];
    }
  }
}

template <int DP, int BN>
__host__ __device__ constexpr int map_threads() {
  return (DP / 8) * (BN / 8);
}
template <int DP, int BN>
constexpr size_t map_smem() {
  return sizeof(float) * ((size_t)DP * (BN + 4) + 2 * (size_t)kBK * DP);
}

// Y = op(M) X with op(M) = M (TRANS = false) or Mᵀ; logjac[n] = lj (+ logjac[n]) when logjac != NULL
template <int DP, int BN, bool TRANS>
__global__ void __launch_bounds__(map_threads<DP, BN>(), 1)
    map_kernel(const float* __restrict__ M, const float* x, long long ldx, float* y, long long ldy, float* logjac,
               int accumulate, const double* __restrict__ logdet, float lj_sign, int D, long long N) {
  constexpr int T = map_threads<DP, BN>(), XS = BN + 4, PER = DP * kBK / T;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* Xs = reinterpret_cast<float*>(smem_raw);  // Xs[k * XS + n]
  float* Ms = Xs + (size_t)DP * XS;                // Ms[buf][kk * DP + i] = op(M)(i, k0 + kk)
  const int tid = threadIdx.x, ty = tid % (DP / 8), tx = tid / (DP / 8);
  const long long n0 = (long long)blockIdx.x * BN;
  const int Kp = (D + kBK - 1) / kBK * kBK, KB = Kp / kBK;
  float pre[PER];
  auto fetch = [&](int kb) {
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int idx = tid + e * T;
      int i, kk;
      if (TRANS) {
        kk = idx % kBK;
        i = idx / kBK;
      } else {
        i = idx % DP;
        kk = idx / DP;
      }
      const int k = kb * kBK + kk;
      float v = 0.f;
      if (i < D && k < D) v = TRANS ? __ldg(M + (size_t)i * D + k) : __ldg(M + (size_t)k * D + i);
      pre[e] = v;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int idx = tid + e * T;
      const int i = TRANS ? idx / kBK : idx % DP, kk = TRANS ? idx % kBK : idx / DP;
      Ms[buf * kBK * DP + kk * DP + i] = pre[e];
    }
  };
  fetch(0);
  // the whole x tile is read before any y of it is written (y may alias x)
  for (int idx = tid; idx < BN * Kp; idx += T) {
    const int n = idx / Kp, k = idx - n * Kp;
    const long long col = n0 + n;
    Xs[k * XS + n] = (col < N && k < D) ? x[col * ldx + k] : 0.f;
  }
  stash(0);
  __syncthreads();
  float acc[8][8];
#pragma unroll
  for (int u = 0; u < 8; ++u)
#pragma unroll
    for (int v = 0; v < 8; ++v) acc[u][v] = 0.f;
  for (int kb = 0; kb < KB; ++kb) {
    if (kb + 1 < KB) fetch(kb + 1);
    const float* Mb = Ms + (kb & 1) * kBK * DP;
    const float* Xb = Xs + (size_t)kb * kBK * XS;
#pragma unroll
    for (int kk = 0; kk < kBK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(Mb + kk * DP + ty * 4);
      const float4 a1 = *reinterpret_cast<const float4*>(Mb + kk * DP + DP / 2 + ty * 4);
      const float4 b0 = *reinterpret_cast<const float4*>(Xb + kk * XS + tx * 4);
      const float4 b1 = *reinterpret_cast<const float4*>(Xb + kk * XS + BN / 2 + tx * 4);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int v = 0; v < 8; ++v) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
    }
    if (kb + 1 < KB) stash((kb + 1) & 1);
    __syncthreads();
  }
#pragma unroll
  for (int v = 0; v < 8; ++v) {
    const long long col = n0 + (v < 4 ? tx * 4 + v : BN / 2 + tx * 4 + v - 4);
    if (col >= N) continue;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = u < 4 ? ty * 4 + u : DP / 2 + ty * 4 + u - 4;
      if (i < D) y[col * ldy + i] = acc[u][v];
    }
  }
  if (logjac) {
    const float lj = (float)(lj_sign * *logdet);
    for (int c = tid; c < BN && n0 + c < N; c += T) {
      const long long col = n0 + c;
      logjac[col] = accumulate ? logjac[col] + lj : lj;
    }
  }
}

// logjac only (y == NULL)
__global__ void logjac_kernel(float* __restrict__ logjac, int accumulate, const double* __restrict__ logdet,
                              float lj_sign, long long N) {
  const float lj = (float)(lj_sign * *logdet);
  for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += (long long)gridDim.x * blockDim.x)
    logjac[n] = accumulate ? logjac[n] + lj : lj;
}

// Σₙ l̄ₙ in fp64: strided per-thread sums, then a fixed tree over the block
__global__ void __launch_bounds__(1024) ljsum_kernel(const float* __restrict__ ljbar, long long N, double* __restrict__ out) {
  __shared__ double red[1024];
  double s = 0.0;
  if (ljbar)
    for (long long n = threadIdx.x; n < N; n += 1024) s += (double)ljbar[n];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = 512; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = red[0];
}

// forward layer: Ā = Σ_p part[p] + s·B;  inverse layer: Gd = Σ_p part[p] (fp64).  B(i, j) = A⁻¹(j, i) = minv[i·D + j].
__global__ void __launch_bounds__(256) gsum_kernel(const float* __restrict__ part, int P, const double* __restrict__ ljs,
                                                   const float* __restrict__ minv, int D, float* __restrict__ Abar,
                                                   double* __restrict__ Gd) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x, DD = (long long)D * D;
  if (idx >= DD) return;
  double a = 0.0;
  for (int p = 0; p < P; ++p) a += (double)part[(size_t)p * DD + idx];
  if (Gd) {
    Gd[idx] = a;
    return;
  }
  const int j = (int)(idx / D), i = (int)(idx - (long long)j * D);
  Abar[idx] = (float)(a + *ljs * (double)minv[(size_t)i * D + j]);
}

// T = Gd · B (fp64, column-major)
__global__ void __launch_bounds__(256) prod_gb_kernel(const double* __restrict__ Gd, const float* __restrict__ minv, int D,
                                                      double* __restrict__ Tm) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)D * D) return;
  const int j = (int)(idx / D), i = (int)(idx - (long long)j * D);
  double a = 0.0;
  for (int k = 0; k < D; ++k) a = fma(Gd[(size_t)k * D + i], (double)minv[(size_t)k * D + j], a);
  Tm[idx] = a;
}

// inverse layer: Ā = −B · T − s·B
__global__ void __launch_bounds__(256) final_inv_kernel(const double* __restrict__ Tm, const float* __restrict__ minv,
                                                        const double* __restrict__ ljs, int D, float* __restrict__ Abar) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)D * D) return;
  const int j = (int)(idx / D), i = (int)(idx - (long long)j * D);
  double a = 0.0;
  for (int k = 0; k < D; ++k) a = fma((double)minv[(size_t)i * D + k], Tm[(size_t)j * D + k], a);
  Abar[idx] = (float)(-a - *ljs * (double)minv[(size_t)i * D + j]);
}

int launch_factor(const b2b_layer_desc& d, const Factor& f, int D, bool want_inverse, int* launches, cudaStream_t stream) {
  const size_t smem = factor_smem(D);
  cudaError_t e = cudaFuncSetAttribute(factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  factor_kernel<<<1, kFactorThreads, smem, stream>>>(d.p0, D, f.lu, f.perm, f.logdet);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*launches;
  if (!want_inverse) return B2B_OK;
  const int grid = (D + kInvWarps * kInvC - 1) / (kInvWarps * kInvC);
  if (D <= 32) inv_kernel<1><<<grid, kInvWarps * 32, 0, stream>>>(f.lu, f.perm, f.minv, D);
  else if (D <= 64) inv_kernel<2><<<grid, kInvWarps * 32, 0, stream>>>(f.lu, f.perm, f.minv, D);
  else if (D <= 128) inv_kernel<4><<<grid, kInvWarps * 32, 0, stream>>>(f.lu, f.perm, f.minv, D);
  else inv_kernel<8><<<grid, kInvWarps * 32, 0, stream>>>(f.lu, f.perm, f.minv, D);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*launches;
  return B2B_OK;
}

template <int DP, int BN, bool TRANS>
int launch_map_t(const float* M, const float* x, long long ldx, float* y, long long ldy, float* logjac, int accumulate,
                 const double* logdet, float sign, int D, long long N, cudaStream_t stream) {
  constexpr size_t smem = map_smem<DP, BN>();
  auto k = map_kernel<DP, BN, TRANS>;
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  const long long grid = (N + BN - 1) / BN;
  k<<<(unsigned)grid, map_threads<DP, BN>(), smem, stream>>>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N);
  return (int)cudaGetLastError();
}

template <bool TRANS>
int launch_map(const float* M, const float* x, long long ldx, float* y, long long ldy, float* logjac, int accumulate,
               const double* logdet, float sign, int D, long long N, cudaStream_t stream) {
  if (D <= 32) return launch_map_t<32, 128, TRANS>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
  if (D <= 64) return launch_map_t<64, 128, TRANS>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
  if (D <= 128) return launch_map_t<128, 128, TRANS>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
  return launch_map_t<256, 64, TRANS>(M, x, ldx, y, ldy, logjac, accumulate, logdet, sign, D, N, stream);
}

}  // namespace b2b_scale

using namespace b2b_scale;

size_t b2b_scale_matrix_workspace(int D) {
  return D >= 1 && D <= B2B_SCALE_MATRIX_MAX_D ? factor_bytes(D) : 0;
}

int b2b_fwd_scale(const B2BFwdSeg& s) {
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  if (D < 1 || D > B2B_SCALE_MATRIX_MAX_D) return B2B_EUNSUPPORTED;
  if (!s.workspace || s.workspace_bytes < factor_bytes(D)) return B2B_EWORKSPACE;
  const Factor f = carve(s.workspace, D);
  const bool inv = d.inverse != 0;
  int rc = launch_factor(d, f, D, inv && s.y, s.launches, s.stream);
  if (rc != B2B_OK) return rc;
  const float sign = inv ? -1.f : 1.f;
  if (!s.y) {  // log-Jacobians only
    if (!s.logjac) return B2B_OK;
    long long g = (s.N + 255) / 256;
    logjac_kernel<<<(unsigned)(g < 1024 ? g : 1024), 256, 0, s.stream>>>(s.logjac, s.accumulate, f.logdet, sign, s.N);
    if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
    ++*s.launches;
    return B2B_OK;
  }
  rc = launch_map<false>(inv ? f.minv : d.p0, s.x, s.ldx, s.y, s.ldy, s.logjac, s.accumulate, f.logdet, sign, D, s.N,
                         s.stream);
  if (rc != B2B_OK) return rc;
  ++*s.launches;
  return B2B_OK;
}

// workspace: [factor storage][chunk partials of G (P x D x D fp32)][Gd, T (D x D fp64 each)][Σ l̄ (fp64)]
size_t b2b_scale_matrix_vjp_workspace(int D, long long N) {
  if (D < 1 || D > B2B_SCALE_MATRIX_MAX_D || N < 0) return 0;
  const long long clen = b2b_outer_chunk_len(N), P = N > 0 ? (N + clen - 1) / clen : 1;
  return factor_bytes(D) + al256(sizeof(float) * (size_t)P * D * D) + 2 * al256(sizeof(double) * (size_t)D * D) +
         al256(sizeof(double));
}

int b2b_vjp_scale(const B2BVjpSeg& s) {
  const b2b_layer_desc& d = s.layers[0];
  const float *x = s.x, *ybar = s.ybar, *ljbar = s.ljbar;
  const long long ldx = s.ldx, ldyb = s.ldyb, ldxb = s.ldxb, N = s.N;
  float* const xbar = s.xbar;
  float* const Abar = s.bars[0];
  void* const workspace = s.workspace;
  const int D = s.D;
  int* const launches = s.launches;
  const cudaStream_t stream = s.stream;
  if (D < 1 || D > B2B_SCALE_MATRIX_MAX_D) return B2B_EUNSUPPORTED;
  if (!workspace || s.workspace_bytes < b2b_scale_matrix_vjp_workspace(D, N)) return B2B_EWORKSPACE;
  const Factor f = carve(workspace, D);
  const bool inv = d.inverse != 0;
  char* ws = static_cast<char*>(workspace) + factor_bytes(D);
  const long long clen = b2b_outer_chunk_len(N), P = (N + clen - 1) / clen;
  float* part = reinterpret_cast<float*>(ws);
  ws += al256(sizeof(float) * (size_t)P * D * D);
  double* Gd = reinterpret_cast<double*>(ws);
  ws += al256(sizeof(double) * (size_t)D * D);
  double* Tm = reinterpret_cast<double*>(ws);
  ws += al256(sizeof(double) * (size_t)D * D);
  double* ljs = reinterpret_cast<double*>(ws);
  int rc = B2B_OK;
  if (inv || Abar) {
    rc = launch_factor(d, f, D, true, launches, stream);
    if (rc != B2B_OK) return rc;
  }
  // x̄ = op(M)ᵀ ȳ
  if (ybar) {
    rc = launch_map<true>(inv ? f.minv : d.p0, ybar, ldyb, xbar, ldxb, nullptr, 0, nullptr, 0.f, D, N, stream);
    if (rc != B2B_OK) return rc;
  } else {
    rc = (int)cudaMemset2DAsync(xbar, (size_t)ldxb * sizeof(float), 0, (size_t)D * sizeof(float), (size_t)N, stream);
    if (rc != cudaSuccess) return rc;
  }
  ++*launches;
  if (!Abar) return B2B_OK;
  if (ybar) {
    rc = b2b_launch_outer_chunks(ybar, ldyb, x, ldx, part, nullptr, D, N, false, stream);
    if (rc != B2B_OK) return rc;
    ++*launches;
  }
  ljsum_kernel<<<1, 1024, 0, stream>>>(ljbar, N, ljs);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  ++*launches;
  const long long DD = (long long)D * D;
  const unsigned g = (unsigned)((DD + 255) / 256);
  gsum_kernel<<<g, 256, 0, stream>>>(part, ybar ? (int)P : 0, ljs, f.minv, D, Abar, inv ? Gd : nullptr);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  ++*launches;
  if (!inv) return B2B_OK;
  prod_gb_kernel<<<g, 256, 0, stream>>>(Gd, f.minv, D, Tm);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  final_inv_kernel<<<g, 256, 0, stream>>>(Tm, f.minv, ljs, D, Abar);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  *launches += 2;
  return B2B_OK;
}
