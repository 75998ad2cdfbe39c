// The network pieces of the neural-network coupling kernels (b2b_coupling_mlp.cu, b2b_coupling_mlp_vjp.cu), shared with
// the masked autoregressive layer (b2b_autoregressive.cu): a hidden layer over a 64-column tile for the forward kernels,
// and the per-sub-tile hidden layer, transposed GEMM and outer-product sums of the reverse-mode kernels.
#pragma once
#include <cuda_runtime.h>

#include "b2b_coupling_mlp.cuh"
#include "b2b_coupling_tile.cuh"

namespace b2b {

// dst = σ(W·src + c) for one tile: W is H x nk column-major, src [nk][CP_LD], dst [H][CP_LD], c NULL = 0.  Eight
// hidden rows per warp and step.
__device__ __forceinline__ void cmlp_hidden(const float* src, int nk, const float* __restrict__ W,
                                            const float* __restrict__ c, bool vec, int H, int act, float slope,
                                            float* dst) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto same = [](int k) { return k; };
  for (int jb = 8 * warp; jb < H; jb += 8 * (CP_THREADS / 32)) {
    float va[4][2] = {}, vb[4][2] = {};
    coupling_gemm_block<2>(src, CP_LD, same, nk, W + jb, W + jb + 4, H, H - jb, H - jb - 4, vec, va, vb);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int m = jb + q;
      if (m < H) {
        const float cm = c ? __ldg(c + m) : 0.f;
        float dh;
#pragma unroll
        for (int u = 0; u < 2; ++u)
          mlp_act(act, slope, (q < 4 ? va[q & 3][u] : vb[q & 3][u]) + cm, dst[m * CP_LD + lane + 32 * u], dh);
      }
    }
  }
}

constexpr int CMV_THREADS = 256;
constexpr int CMV_SP = 33;  // pitch of the one-sub-tile scratch block

// acc[q] += Σ_k A[q·nk + k] · B[k·ld + lane] for the `rows` (<= 8) rows at A, each contiguous in k, k increasing
__device__ __forceinline__ void cmv_gemm_t(const float* B, int ld, int nk, const float* __restrict__ A, int rows, bool vec,
                                           float (&acc)[8]) {
  const int lane = threadIdx.x & 31;
  if (vec && rows >= 8) {
    for (int k = 0; k < nk; k += 4) {
      const float b0 = B[k * ld + lane], b1 = B[(k + 1) * ld + lane], b2 = B[(k + 2) * ld + lane], b3 = B[(k + 3) * ld + lane];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(A + (size_t)q * nk + k));
        acc[q] = fmaf(a.w, b3, fmaf(a.z, b2, fmaf(a.y, b1, fmaf(a.x, b0, acc[q]))));
      }
    }
  } else {
    for (int k = 0; k < nk; ++k) {
      const float b = B[k * ld + lane];
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if (q < rows) acc[q] = fmaf(__ldg(A + (size_t)q * nk + k), b, acc[q]);
    }
  }
}

// out[i + RA·j] += Σ_c A[i][c]·B[j][c] over the group's `cols` columns (A: RA rows, B: RB rows, pitch ld), and
// outc[i] += Σ_c A[i][c].  16 x 16 threads, a 4 x 4 block each, swept over 64 x 64 blocks of the matrix.
__device__ __forceinline__ void cmv_outer(const float* A, int RA, const float* B, int RB, int ld, int cols, float* out,
                                          float* outc) {
  const int ti = threadIdx.x & 15, tj = threadIdx.x >> 4;
  for (int bi = 0; bi < RA; bi += 64)
    for (int bj = 0; bj < RB; bj += 64) {
      float acc[4][4] = {};
      const float *pa[4], *pb[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {  // rows past the matrix read its last row; their sums are dropped below
        pa[q] = A + (size_t)min(bi + ti + 16 * q, RA - 1) * ld;
        pb[q] = B + (size_t)min(bj + tj + 16 * q, RB - 1) * ld;
      }
      for (int c = 0; c < cols; ++c) {
        float a[4], b[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          a[q] = pa[q][c];
          b[q] = pb[q][c];
        }
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int p = 0; p < 4; ++p) acc[q][p] = fmaf(a[q], b[p], acc[q][p]);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const int i = bi + ti + 16 * q, j = bj + tj + 16 * p;
          if (i < RA && j < RB) out[(size_t)i + (size_t)RA * j] += acc[q][p];
        }
    }
  for (int i = threadIdx.x; i < RA; i += CMV_THREADS) {
    float s = 0.f;
    for (int c = 0; c < cols; ++c) s += A[(size_t)i * ld + c];
    outc[i] += s;
  }
}

// One sub-tile's hidden layer: h = σ(W·src + c) and σ′ into hs / dv ([H][ld], column `lane`), W H x nk column-major
__device__ __forceinline__ void cmv_hidden(const float* src, int ld, int nk, const float* __restrict__ W,
                                           const float* __restrict__ c, bool vec, int H, int act, float slope, float* hs,
                                           float* dv) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto same = [](int k) { return k; };
  for (int jb = 8 * warp; jb < H; jb += 8 * (CMV_THREADS / 32)) {
    float va[4][1] = {}, vb[4][1] = {};
    coupling_gemm_block<1>(src, ld, same, nk, W + jb, W + jb + 4, H, H - jb, H - jb - 4, vec, va, vb);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int m = jb + q;
      if (m < H)
        mlp_act(act, slope, (q < 4 ? va[q & 3][0] : vb[q & 3][0]) + (c ? __ldg(c + m) : 0.f), hs[m * ld + lane],
                dv[m * ld + lane]);
    }
  }
}

// v̄ = (Wᵀ g) ⊙ σ′ in place over the σ′ block v ([H][ld]), W ng x H column-major, g [ng][ld]
__device__ __forceinline__ void cmv_back(const float* g, int ld, int ng, const float* __restrict__ W, bool vec, int H,
                                         float* v) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int mb = 8 * warp; mb < H; mb += 8 * (CMV_THREADS / 32)) {
    float acc[8] = {};
    cmv_gemm_t(g, ld, ng, W + (size_t)mb * ng, H - mb, vec, acc);
#pragma unroll
    for (int q = 0; q < 8; ++q)
      if (mb + q < H) v[(mb + q) * ld + lane] *= acc[q];
  }
}

}  // namespace b2b
