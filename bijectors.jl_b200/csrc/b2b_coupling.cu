// Affine coupling layer, SIMT (fp32 CUDA-core) version.
//
// Reference: Coupling (src/bijectors/coupling.jl:206-228) with the law θ(x₂) = Shift(t) ∘ Scale(exp.(s)),
// [s; t] = W·x₂ + c  (scale.jl:13,31; shift.jl:14,21), mapped over the columns of a D x N batch:
//   forward : y₁ = exp(s) ⊙ x₁ + t,        logjac = Σ_j log|exp(s_j)| = Σ_j s_j
//   inverse : x₁ = inv.(exp(s)) ⊙ (y₁ − t), logjac = −Σ_j s_j
// x₂ (rows idx2) and x₃ (the remaining rows) pass through unchanged (combine, coupling.jl:125).
//
// A CTA owns a tile of TC columns.  The tile is transposed into shared memory ([row][col], padded), every thread
// computes a 4(j) x 2(s,t) x 2(col) register block of the conditioner GEMM reading W through the read-only path (uniform
// addresses -> one sector per request, W stays L1/L2 resident), the epilogue applies exp/FMA in place on the x₁ rows and
// the tile is written back.  Two programs: coupling_affine_full_kernel stages all D rows (coalesced reads and writes of
// whole columns) when they fit; coupling_affine_rows_kernel stages only the x₂ and x₁ rows and copies the pass-through
// rows x₃ global to global (through the folded BatchNorm affines when there are any; skipped in place without them), so
// its shared memory -- and the limit -- depends on n1 + n2 only, not on D.  This is the exact-fp32 path; the tensor-core
// path (fp16-split wgmma) lives in b2b_coupling_tc.cu and is cross-checked against this kernel.
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_coupling_tile.cuh"
#include "b2b_internal.h"

namespace b2b {

// Layers whose D rows fit shared memory (D <= 777 at n2 = 128) stage the whole tile: every row is read and written
// coalesced, column by column.
template <bool INV>
__global__ void __launch_bounds__(CP_THREADS) coupling_affine_full_kernel(
    const float* __restrict__ x, float* __restrict__ y, float* __restrict__ logjac,
    const int32_t* __restrict__ idx1, const int32_t* __restrict__ idx2, const float* __restrict__ W,
    const float* __restrict__ cvec, const float* __restrict__ fold, int D, int n1, int n2, int row1, int row2,
    long long N, long long ldx, long long ldy, int accumulate) {
  extern __shared__ float smem[];
  float* X = smem;                                    // [D][CP_LD]
  float* red = X + (size_t)D * CP_LD;                 // [8][CP_TC]
  int* sidx2 = reinterpret_cast<int*>(red + 8 * CP_TC);  // [n2]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = threadIdx.x; k < n2; k += CP_THREADS) sidx2[k] = idx2 ? idx2[k] : row2 + k;
  const bool wvec = ((n1 & 3) == 0) && ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
  const long long tiles = (N + CP_TC - 1) / CP_TC;

  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long col0 = tile * CP_TC;
    __syncthreads();  // previous tile fully written back / sidx2 visible
    // ---- load + transpose ----------------------------------------------------------------------
    for (int c = warp; c < CP_TC; c += CP_THREADS / 32) {
      const long long col = col0 + c;
      if (col < N) {
        const float* xc = x + col * ldx;
        if (fold) {
          for (int r = lane; r < D; r += 32) X[r * CP_LD + c] = fmaf(__ldcs(xc + r), fold[r], fold[D + r]);
        } else {
          for (int r = lane; r < D; r += 32) X[r * CP_LD + c] = __ldcs(xc + r);
        }
      } else {
        for (int r = lane; r < D; r += 32) X[r * CP_LD + c] = 0.f;
      }
    }
    __syncthreads();
    // ---- conditioner GEMM + epilogue -------------------------------------------------------------
    coupling_tile<INV>(X, X, [&](int k) { return sidx2[k]; }, [&](int j) { return idx1 ? __ldg(idx1 + j) : row1 + j; },
                       W, cvec, n1, n2, wvec, red);
    __syncthreads();
    // ---- write back --------------------------------------------------------------------------------
    if (y) {
      for (int c = warp; c < CP_TC; c += CP_THREADS / 32) {
        const long long col = col0 + c;
        if (col < N) {
          float* yc = y + col * ldy;
          if (fold) {
            for (int r = lane; r < D; r += 32) __stcs(yc + r, fmaf(X[r * CP_LD + c], fold[2 * D + r], fold[3 * D + r]));
          } else {
            for (int r = lane; r < D; r += 32) __stcs(yc + r, X[r * CP_LD + c]);
          }
        }
      }
    }
    if (logjac && threadIdx.x < CP_TC) {
      const long long col = col0 + threadIdx.x;
      if (col < N) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < CP_THREADS / 32; ++w) s += red[w * CP_TC + threadIdx.x];
        const float base = (accumulate ? logjac[col] : 0.f) + (fold ? fold[4 * D] : 0.f);
        logjac[col] = INV ? base - s : base + s;  // Σ log|exp(s)| = Σ s  (scale.jl:31)
      }
    }
  }
}

// Wider layers stage only the rows they read.  Three CTAs per SM leave 85 registers per thread: no spills.
template <bool INV>
__global__ void __launch_bounds__(CP_THREADS, 3) coupling_affine_rows_kernel(
    const float* __restrict__ x, float* __restrict__ y, float* __restrict__ logjac,
    const int32_t* __restrict__ idx1, const int32_t* __restrict__ idx2, const float* __restrict__ W,
    const float* __restrict__ cvec, const float* __restrict__ fold, int D, int n1, int n2, int row1, int row2,
    long long N, long long ldx, long long ldy, int accumulate) {
  // x and y may alias (in place): every element is read before it is written, by the same CTA
  extern __shared__ float smem[];
  float* X2 = smem;                                      // [n2][CP_LD]  conditioner input x₂ (folded)
  float* X1 = X2 + (size_t)n2 * CP_LD;                   // [n1][CP_LD]  x₁ (folded), transformed in place
  float* red = X1 + (size_t)n1 * CP_LD;                  // [8][CP_TC]
  int* sidx2 = reinterpret_cast<int*>(red + 8 * CP_TC);  // [n2]
  int* sidx1 = sidx2 + n2;                               // [n1]
  unsigned* coupled = reinterpret_cast<unsigned*>(sidx1 + n1);  // [ceil(D/32)] bit r: row r is in idx1 or idx2
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // pass-through rows exist when the two index lists do not cover the column; without a fold an in-place call leaves
  // them (and x₂) where they are
  const bool has_x3 = n1 + n2 < D;
  const bool copy_through = y && (fold || y != x);
  const int nwords = (D + 31) >> 5;
  if (has_x3 && copy_through)
    for (int k = threadIdx.x; k < nwords; k += CP_THREADS) coupled[k] = 0u;
  for (int k = threadIdx.x; k < n2; k += CP_THREADS) sidx2[k] = idx2 ? idx2[k] : row2 + k;
  for (int k = threadIdx.x; k < n1; k += CP_THREADS) sidx1[k] = idx1 ? idx1[k] : row1 + k;
  __syncthreads();
  if (has_x3 && copy_through) {
    for (int k = threadIdx.x; k < n2; k += CP_THREADS) atomicOr(&coupled[sidx2[k] >> 5], 1u << (sidx2[k] & 31));
    for (int k = threadIdx.x; k < n1; k += CP_THREADS) atomicOr(&coupled[sidx1[k] >> 5], 1u << (sidx1[k] & 31));
  }
  const bool wvec = ((n1 & 3) == 0) && ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
  const long long tiles = (N + CP_TC - 1) / CP_TC;

  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long col0 = tile * CP_TC;
    __syncthreads();  // previous tile fully written back / index tables visible
    // ---- load + transpose x₂ and x₁; pass-through rows go straight to y ---------------------------------------
    for (int c = warp; c < CP_TC; c += CP_THREADS / 32) {
      const long long col = col0 + c;
      if (col < N) {
        const float* xc = x + col * ldx;
        if (fold) {
          for (int k = lane; k < n2; k += 32) X2[k * CP_LD + c] = fmaf(__ldcs(xc + sidx2[k]), fold[sidx2[k]], fold[D + sidx2[k]]);
          if (y)  // the log-Jacobian needs x₂ only
            for (int k = lane; k < n1; k += 32) X1[k * CP_LD + c] = fmaf(__ldcs(xc + sidx1[k]), fold[sidx1[k]], fold[D + sidx1[k]]);
        } else {
          for (int k = lane; k < n2; k += 32) X2[k * CP_LD + c] = __ldcs(xc + sidx2[k]);
          if (y)
            for (int k = lane; k < n1; k += 32) X1[k * CP_LD + c] = __ldcs(xc + sidx1[k]);
        }
        if (has_x3 && copy_through) {
          float* yc = y + col * ldy;
          for (int r = lane; r < D; r += 32) {
            if ((coupled[r >> 5] >> (r & 31)) & 1u) continue;
            const float v = __ldcs(xc + r);
            // pre- then post-BatchNorm affine: exactly what the rows would get had they been staged
            __stcs(yc + r, fold ? fmaf(fmaf(v, fold[r], fold[D + r]), fold[2 * D + r], fold[3 * D + r]) : v);
          }
        }
      } else {
        for (int k = lane; k < n2; k += 32) X2[k * CP_LD + c] = 0.f;
        for (int k = lane; k < n1; k += 32) X1[k * CP_LD + c] = 0.f;
      }
    }
    __syncthreads();
    // ---- conditioner GEMM + epilogue -------------------------------------------------------------
    coupling_tile<INV>(X2, X1, [](int k) { return k; }, [](int j) { return j; }, W, cvec, n1, n2, wvec, red);
    __syncthreads();
    // ---- write back x₁ (and x₂ unless it is already in place) ---------------------------------------------------------
    if (y) {
      for (int c = warp; c < CP_TC; c += CP_THREADS / 32) {
        const long long col = col0 + c;
        if (col < N) {
          float* yc = y + col * ldy;
          if (fold) {
            for (int k = lane; k < n1; k += 32) {
              const int r = sidx1[k];
              __stcs(yc + r, fmaf(X1[k * CP_LD + c], fold[2 * D + r], fold[3 * D + r]));
            }
            for (int k = lane; k < n2; k += 32) {
              const int r = sidx2[k];
              __stcs(yc + r, fmaf(X2[k * CP_LD + c], fold[2 * D + r], fold[3 * D + r]));
            }
          } else {
            for (int k = lane; k < n1; k += 32) __stcs(yc + sidx1[k], X1[k * CP_LD + c]);
            if (copy_through)
              for (int k = lane; k < n2; k += 32) __stcs(yc + sidx2[k], X2[k * CP_LD + c]);
          }
        }
      }
    }
    if (logjac && threadIdx.x < CP_TC) {
      const long long col = col0 + threadIdx.x;
      if (col < N) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < CP_THREADS / 32; ++w) s += red[w * CP_TC + threadIdx.x];
        const float base = (accumulate ? logjac[col] : 0.f) + (fold ? fold[4 * D] : 0.f);
        logjac[col] = INV ? base - s : base + s;  // Σ log|exp(s)| = Σ s  (scale.jl:31)
      }
    }
  }
}

// Folded BatchNorm neighbours of a coupling layer (normalise.jl:61-67, :74-86): the per-row affine
// x' = preA·x + preC is applied on the way in, y' = postA·y + postC on the way out, and the (column-independent)
// log-Jacobian constants are summed into out[4D].  Layout: preA[D] | preC[D] | postA[D] | postC[D] | {lj}.
__global__ void __launch_bounds__(256) bn_fold_prep_kernel(b2b_layer_desc pre, int has_pre, b2b_layer_desc post,
                                                           int has_post, int D, float* __restrict__ out) {
  __shared__ float red[8];
  float lj = 0.f;
  for (int i = threadIdx.x; i < D; i += 256) {
    float A[2] = {1.f, 1.f}, C[2] = {0.f, 0.f};
    for (int w = 0; w < 2; ++w) {
      const b2b_layer_desc& d = w == 0 ? pre : post;
      if (!(w == 0 ? has_pre : has_post)) continue;
      const float ve = d.p3[i] + d.f0, sd = sqrtf(ve), sc = expf(d.p1[i]);
      const float l = d.p1[i] - logf(ve) * 0.5f;
      if (!d.inverse) {
        A[w] = sc / sd;
        C[w] = fmaf(-d.p2[i], A[w], d.p0[i]);
        lj += l;
      } else {
        A[w] = sd / sc;
        C[w] = fmaf(-d.p0[i], A[w], d.p2[i]);
        lj -= l;
      }
    }
    out[i] = A[0];
    out[D + i] = C[0];
    out[2 * D + i] = A[1];
    out[3 * D + i] = C[1];
  }
  for (int o = 16; o > 0; o >>= 1) lj += __shfl_xor_sync(0xffffffffu, lj, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lj;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    out[4 * D] = t;
  }
}

// coupling_affine_rows_kernel: x₂ and x₁ tiles, the column-sum slab, both index tables and the coupled-row bitmap
static size_t coupling_smem_bytes(int n1, int n2, int D) {
  return ((size_t)(n1 + n2) * CP_LD + 8 * CP_TC) * sizeof(float) + (size_t)(n1 + n2) * sizeof(int) +
         (size_t)((D + 31) / 32) * sizeof(unsigned);
}

}  // namespace b2b

bool b2b_coupling_affine_fits(int n1, int n2, int D) {
  return b2b::coupling_smem_bytes(n1, n2, D) <= 200 * 1024;
}

int b2b_launch_bn_fold_prep(const b2b_layer_desc* pre, const b2b_layer_desc* post, int D, float* out,
                            cudaStream_t stream) {
  b2b_layer_desc z;
  memset(&z, 0, sizeof(z));
  b2b::bn_fold_prep_kernel<<<1, 256, 0, stream>>>(pre ? *pre : z, pre != nullptr, post ? *post : z, post != nullptr, D, out);
  return (int)cudaGetLastError();
}

int b2b_launch_coupling_affine(const b2b_layer_desc& d, const float* fold, const float* x, float* y, float* logjac,
                               int D, long long N, long long ldx, long long ldy, int accumulate,
                               cudaStream_t stream) {
  using namespace b2b;
  const int n1 = d.n0, n2 = d.n1;  // a valid descriptor (b2b_check_desc)
  if (!b2b_coupling_affine_fits(n1, n2, D)) return B2B_EUNSUPPORTED;
  const size_t smem_full = ((size_t)D * CP_LD + 8 * CP_TC) * sizeof(float) + (size_t)n2 * sizeof(int);
  const bool full = smem_full <= 200 * 1024;
  const size_t smem = full ? smem_full : coupling_smem_bytes(n1, n2, D);
  auto kern = full ? (d.inverse ? coupling_affine_full_kernel<true> : coupling_affine_full_kernel<false>)
                   : (d.inverse ? coupling_affine_rows_kernel<true> : coupling_affine_rows_kernel<false>);
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  const int sms = b2b_sm_count();
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, CP_THREADS, smem);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < 1) per_sm = 1;
  const long long tiles = (N + CP_TC - 1) / CP_TC;
  long long grid = (long long)sms * per_sm;
  if (grid > tiles) grid = tiles;
  if (grid < 1) grid = 1;
  kern<<<(int)grid, CP_THREADS, smem, stream>>>(x, y, logjac, d.i0, d.i1, d.p0, d.p1, fold, D, n1, n2, d.n2, d.n3, N, ldx,
                                                ldy, accumulate);
  return (int)cudaGetLastError();
}
