// Affine coupling layer, SIMT (fp32 CUDA-core) version.
//
// Reference: Coupling (src/bijectors/coupling.jl:206-228) with the law θ(x₂) = Shift(t) ∘ Scale(exp.(s)),
// [s; t] = W·x₂ + c  (scale.jl:13,31; shift.jl:14,21), mapped over the columns of a D x N batch:
//   forward : y₁ = exp(s) ⊙ x₁ + t,        logjac = Σ_j log|exp(s_j)| = Σ_j s_j
//   inverse : x₁ = inv.(exp(s)) ⊙ (y₁ − t), logjac = −Σ_j s_j
// x₂ (rows idx2) and x₃ (the remaining rows) pass through unchanged (combine, coupling.jl:125).
//
// A CTA owns a tile of TC columns.  The tile is transposed into shared memory ([row][col], padded) with
// coalesced global reads, every thread computes a 4(j) x 2(s,t) x 2(col) register block of the
// conditioner GEMM reading W through the read-only path (uniform addresses -> one sector per request,
// W stays L1/L2 resident), the epilogue applies exp/FMA in place on the x₁ rows of the tile and the
// tile is written back coalesced.  This is the exact-fp32 path; the tensor-core path (fp16-split wgmma)
// lives in b2b_coupling_tc.cu and is cross-checked against this kernel.
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_internal.h"

namespace b2b {

constexpr int CP_TC = 64;       // columns per tile
constexpr int CP_LD = CP_TC + 1;  // padded row stride of the smem tile
constexpr int CP_THREADS = 256;

template <bool INV>
__global__ void __launch_bounds__(CP_THREADS) coupling_affine_kernel(
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
  const int ldw = 2 * n1;

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
    const int cA = lane, cB = lane + 32;
    float sumA = 0.f, sumB = 0.f;
    for (int jb = 4 * warp; jb < n1; jb += 4 * (CP_THREADS / 32)) {
      float sA[4] = {0.f, 0.f, 0.f, 0.f}, sB[4] = {0.f, 0.f, 0.f, 0.f};
      float tA[4] = {0.f, 0.f, 0.f, 0.f}, tB[4] = {0.f, 0.f, 0.f, 0.f};
      if (wvec) {
#pragma unroll 4
        for (int k = 0; k < n2; ++k) {
          const int r2 = sidx2[k];
          const float xa = X[r2 * CP_LD + cA], xb = X[r2 * CP_LD + cB];
          const float4 ws = __ldg(reinterpret_cast<const float4*>(W + (size_t)k * ldw + jb));
          const float4 wt = __ldg(reinterpret_cast<const float4*>(W + (size_t)k * ldw + n1 + jb));
          sA[0] = fmaf(ws.x, xa, sA[0]); sB[0] = fmaf(ws.x, xb, sB[0]);
          sA[1] = fmaf(ws.y, xa, sA[1]); sB[1] = fmaf(ws.y, xb, sB[1]);
          sA[2] = fmaf(ws.z, xa, sA[2]); sB[2] = fmaf(ws.z, xb, sB[2]);
          sA[3] = fmaf(ws.w, xa, sA[3]); sB[3] = fmaf(ws.w, xb, sB[3]);
          tA[0] = fmaf(wt.x, xa, tA[0]); tB[0] = fmaf(wt.x, xb, tB[0]);
          tA[1] = fmaf(wt.y, xa, tA[1]); tB[1] = fmaf(wt.y, xb, tB[1]);
          tA[2] = fmaf(wt.z, xa, tA[2]); tB[2] = fmaf(wt.z, xb, tB[2]);
          tA[3] = fmaf(wt.w, xa, tA[3]); tB[3] = fmaf(wt.w, xb, tB[3]);
        }
      } else {
        for (int k = 0; k < n2; ++k) {
          const int r2 = sidx2[k];
          const float xa = X[r2 * CP_LD + cA], xb = X[r2 * CP_LD + cB];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (jb + q < n1) {
              const float ws = __ldg(W + (size_t)k * ldw + jb + q);
              const float wt = __ldg(W + (size_t)k * ldw + n1 + jb + q);
              sA[q] = fmaf(ws, xa, sA[q]); sB[q] = fmaf(ws, xb, sB[q]);
              tA[q] = fmaf(wt, xa, tA[q]); tB[q] = fmaf(wt, xb, tB[q]);
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int j = jb + q;
        if (j < n1) {
          const float cs = cvec ? __ldg(cvec + j) : 0.f, ct = cvec ? __ldg(cvec + n1 + j) : 0.f;
          const int r1 = idx1 ? __ldg(idx1 + j) : row1 + j;
          const float s_a = sA[q] + cs, s_b = sB[q] + cs, t_a = tA[q] + ct, t_b = tB[q] + ct;
          const float xa = X[r1 * CP_LD + cA], xb = X[r1 * CP_LD + cB];
          if (!INV) {
            X[r1 * CP_LD + cA] = fmaf(expf(s_a), xa, t_a);  // exp(s)·x₁ + t  (scale.jl:13, shift.jl:14)
            X[r1 * CP_LD + cB] = fmaf(expf(s_b), xb, t_b);
          } else {
            X[r1 * CP_LD + cA] = (xa - t_a) / expf(s_a);  // inv.(a) .* (y₁ + (−t))  (scale.jl:16, shift.jl:12)
            X[r1 * CP_LD + cB] = (xb - t_b) / expf(s_b);
          }
          sumA += s_a;
          sumB += s_b;
        }
      }
    }
    red[warp * CP_TC + cA] = sumA;
    red[warp * CP_TC + cB] = sumB;
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

}  // namespace b2b

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
  const int n1 = d.n0, n2 = d.n1;
  if (n1 < 1 || n2 < 1 || n1 + n2 > D || !d.p0) return B2B_EINVAL;
  if ((!d.i0 && d.n2 < 0) || (!d.i1 && d.n3 < 0)) return B2B_EINVAL;
  const size_t smem = ((size_t)D * CP_LD + 8 * CP_TC) * sizeof(float) + (size_t)n2 * sizeof(int);
  if (smem > 200 * 1024) return B2B_EUNSUPPORTED;
  auto kern = d.inverse ? coupling_affine_kernel<true> : coupling_affine_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  int dev = 0, sms = 0, per_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
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
