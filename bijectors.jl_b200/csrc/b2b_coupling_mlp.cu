// Neural-network coupling layers, B2B_COUPLING_MLP and B2B_COUPLING_DEEP_MLP (include/b2b.h): Coupling(θ, mask)
// (coupling.jl:206-228) with the affine law θ(x₂) = Shift(t) ∘ Scale(exp.(s)) whose parameters come from a network of
// M hidden layers (M = 1 for B2B_COUPLING_MLP),
//   h_0 = x₂,   h_l = σ.(W_l·h_{l−1} + c_l) (W_1 = W_in),   [s; t] = W_out·h_M + c_out,   σ = tanh or LeakyReLU(a),
// forward and inverse, in exact fp32 on the CUDA cores.
//
// Mapping.  A CTA owns a tile of 64 columns and stages the n1 + n2 rows it reads, [row][column] with pitch 65, as
// coupling_affine_rows_kernel does (pass-through rows go global to global and are skipped in place).  Phase 1 forms
// h_1 .. h_M with cmlp_hidden (coupling_gemm_block, eight hidden rows per warp and step): odd layers go to a third
// shared-memory block [H][65], even layers back to the x₂ block, which holds max(n2, H) rows when M >= 2 (x₂ has then
// been stored to y₂ as it was loaded).  At n1 = n2 = H = 128 any depth then needs the shared memory of M = 1, and two
// CTAs still fit an SM.  Phase 2 is coupling_tile of the affine kernel with X2 = h_M, n2 = H, W = W_out, cvec = c_out: the same
// GEMM, exp / FMA epilogue and per-warp Σ s.  Every output is a fixed-order fmaf chain over k, then over the hidden
// units, so it does not depend on N, the tile or the grid.
#include <cuda_runtime.h>

#include "b2b_coupling_mlp.cuh"
#include "b2b_coupling_net.cuh"
#include "b2b_coupling_tile.cuh"
#include "b2b_internal.h"

namespace b2b {

struct CmlpParams {
  const float* x;
  float* y;
  float* logjac;
  const float *W1, *c1, *W2, *c2;  // W_in, [c_1 | … | c_M] (or NULL), W_out, c_out
  const int *idx1, *idx2;
  long long N, ldx, ldy;
  int D, n1, n2, H, act, accumulate;
  float slope;
  const float* Wh;  // W_2 .. W_M, each H x H column-major, back to back
  int depth;        // M hidden layers
};

template <bool INV>
__global__ void __launch_bounds__(CP_THREADS, 2) coupling_mlp_kernel(const __grid_constant__ CmlpParams P) {
  // x and y may alias (in place): every element is read before it is written, by the same CTA
  extern __shared__ float smem[];
  const int D = P.D, n1 = P.n1, n2 = P.n2, H = P.H;
  float* X2 = smem;                                      // [n2][CP_LD]  x₂ (M >= 2: max(n2, H) rows, h_l of even l)
  float* X1 = X2 + (size_t)(P.depth > 1 ? max(n2, H) : n2) * CP_LD;  // [n1][CP_LD]  x₁, transformed in place
  float* Hs = X1 + (size_t)n1 * CP_LD;                   // [H][CP_LD]   h_l of odd l
  float* red = Hs + (size_t)H * CP_LD;                   // [8][CP_TC]
  int* sidx2 = reinterpret_cast<int*>(red + 8 * CP_TC);  // [n2]
  int* sidx1 = sidx2 + n2;                               // [n1]
  unsigned* coupled = reinterpret_cast<unsigned*>(sidx1 + n1);  // [ceil(D/32)] bit r: row r is in idx1 or idx2
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* x = P.x;
  float* y = P.y;
  const bool copy_through = y && y != x;  // in place, x₂ and x₃ stay where they are
  // y₂ = x₂ goes out with y₁ at M = 1 (measured faster at H = 128), and as x₂ is loaded at M >= 2, where the x₂ block
  // will hold h_2
  const bool y2_early = copy_through && P.depth > 1, y2_late = copy_through && P.depth == 1;
  const bool has_x3 = n1 + n2 < D;
  const int nwords = (D + 31) >> 5;
  if (has_x3 && copy_through)
    for (int k = threadIdx.x; k < nwords; k += CP_THREADS) coupled[k] = 0u;
  for (int k = threadIdx.x; k < n2; k += CP_THREADS) sidx2[k] = P.idx2[k];
  for (int k = threadIdx.x; k < n1; k += CP_THREADS) sidx1[k] = P.idx1[k];
  __syncthreads();
  if (has_x3 && copy_through) {
    for (int k = threadIdx.x; k < n2; k += CP_THREADS) atomicOr(&coupled[sidx2[k] >> 5], 1u << (sidx2[k] & 31));
    for (int k = threadIdx.x; k < n1; k += CP_THREADS) atomicOr(&coupled[sidx1[k] >> 5], 1u << (sidx1[k] & 31));
  }
  const bool vec1 = ((H & 7) == 0) && ((reinterpret_cast<uintptr_t>(P.W1) & 15) == 0);
  const bool vec2 = ((n1 & 3) == 0) && ((reinterpret_cast<uintptr_t>(P.W2) & 15) == 0);
  const bool vech = ((H & 7) == 0) && ((reinterpret_cast<uintptr_t>(P.Wh) & 15) == 0);
  const long long tiles = (P.N + CP_TC - 1) / CP_TC;
  auto same = [](int k) { return k; };

  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long col0 = tile * CP_TC;
    __syncthreads();  // previous tile fully written back / index tables visible
    // ---- load + transpose x₂ and x₁; pass-through rows go straight to y ---------------------------------------
    for (int c = warp; c < CP_TC; c += CP_THREADS / 32) {
      const long long col = col0 + c;
      if (col < P.N) {
        const float* xc = x + col * P.ldx;
        for (int k = lane; k < n2; k += 32) X2[k * CP_LD + c] = __ldcs(xc + sidx2[k]);
        if (y2_early)
          for (int k = lane; k < n2; k += 32) __stcs(y + col * P.ldy + sidx2[k], X2[k * CP_LD + c]);
        if (y)  // the log-Jacobian needs x₂ only
          for (int k = lane; k < n1; k += 32) X1[k * CP_LD + c] = __ldcs(xc + sidx1[k]);
        if (has_x3 && copy_through) {
          float* yc = y + col * P.ldy;
          for (int r = lane; r < D; r += 32)
            if (!((coupled[r >> 5] >> (r & 31)) & 1u)) __stcs(yc + r, __ldcs(xc + r));
        }
      } else {
        for (int k = lane; k < n2; k += 32) X2[k * CP_LD + c] = 0.f;
        for (int k = lane; k < n1; k += 32) X1[k * CP_LD + c] = 0.f;
      }
    }
    __syncthreads();
    // ---- phase 1: h_l = σ(W_l·h_{l−1} + c_l), l = 1..M ----------------------------------------------------------
    const float* hM = X2;  // h_{l−1}, read with W (nk columns)
    const float* W = P.W1;
    int nk = n2;
    for (int l = 1; l <= P.depth; ++l) {
      float* dst = (l & 1) ? Hs : X2;
      cmlp_hidden(hM, nk, W, P.c1 ? P.c1 + (size_t)(l - 1) * H : nullptr, l == 1 ? vec1 : vech, H, P.act, P.slope, dst);
      __syncthreads();
      hM = dst;
      W = P.Wh + (size_t)(l - 1) * H * H;
      nk = H;
    }
    // ---- phase 2: [s; t] = W_out·h_M + c_out and the affine law on x₁ --------------------------------------------
    coupling_tile<INV>(hM, X1, same, same, P.W2, P.c2, n1, H, vec2, red);
    __syncthreads();
    // ---- write back x₁ (and x₂ at M = 1) ---------------------------------------------------------------------------
    if (y) {
      for (int c = warp; c < CP_TC; c += CP_THREADS / 32) {
        const long long col = col0 + c;
        if (col < P.N) {
          float* yc = y + col * P.ldy;
          for (int k = lane; k < n1; k += 32) __stcs(yc + sidx1[k], X1[k * CP_LD + c]);
          if (y2_late)
            for (int k = lane; k < n2; k += 32) __stcs(yc + sidx2[k], X2[k * CP_LD + c]);
        }
      }
    }
    if (P.logjac && threadIdx.x < CP_TC) {
      const long long col = col0 + threadIdx.x;
      if (col < P.N) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < CP_THREADS / 32; ++w) s += red[w * CP_TC + threadIdx.x];
        const float base = P.accumulate ? P.logjac[col] : 0.f;
        P.logjac[col] = INV ? base - s : base + s;  // Σ log|exp(s)| = Σ s  (scale.jl:31)
      }
    }
  }
}

// x₂ (M >= 2: max(n2, H) rows), x₁ and h tiles, the column-sum slab, both index tables and the coupled-row bitmap
static size_t cmlp_smem_bytes(int n1, int n2, int H, int D, bool deep) {
  const int r2 = deep && H > n2 ? H : n2;
  return ((size_t)(n1 + r2 + H) * CP_LD + 8 * CP_TC) * sizeof(float) + (size_t)(n1 + n2) * sizeof(int) +
         (size_t)((D + 31) / 32) * sizeof(unsigned);
}

}  // namespace b2b

int b2b_fwd_mlp(const B2BFwdSeg& s) {
  using namespace b2b;
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  if (!b2b_coupling_fits(d, D)) return B2B_EUNSUPPORTED;
  const B2BCoupling<b2b_layer_desc> c = b2b_coupling(d);
  CmlpParams P;
  P.x = s.x;
  P.y = s.y;
  P.logjac = s.logjac;
  P.W1 = c.W_in;
  P.c1 = c.c_in;
  P.Wh = c.W_hid;
  P.W2 = c.W_out;
  P.c2 = c.c_out;
  P.idx1 = c.idx1;
  P.idx2 = c.idx2;
  P.N = s.N;
  P.ldx = s.ldx;
  P.ldy = s.ldy;
  P.D = D;
  P.n1 = c.n1;
  P.n2 = c.n2;
  P.H = c.H;
  P.act = c.act;
  P.accumulate = s.accumulate;
  P.slope = c.slope;
  P.depth = c.M;
  const size_t smem = cmlp_smem_bytes(c.n1, c.n2, c.H, D, c.M > 1);
  void (*kernel)(const CmlpParams) = d.inverse ? coupling_mlp_kernel<true> : coupling_mlp_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  const int sms = b2b_sm_count();
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, CP_THREADS, smem);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < 1) per_sm = 1;
  const long long tiles = (s.N + CP_TC - 1) / CP_TC;
  long long grid = (long long)sms * per_sm;
  if (grid > tiles) grid = tiles;
  kernel<<<(int)grid, CP_THREADS, smem, s.stream>>>(P);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*s.launches;
  return B2B_OK;
}
