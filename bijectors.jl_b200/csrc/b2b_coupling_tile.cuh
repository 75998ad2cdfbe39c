// The exact-fp32 conditioner GEMM of the coupling kernels and the affine law's epilogue, shared by the affine coupling
// kernels (b2b_coupling.cu) and the neural-network coupling kernels (b2b_coupling_mlp.cu, b2b_coupling_mlp_vjp.cu).
#pragma once
#include <cuda_runtime.h>

namespace b2b {

constexpr int CP_TC = 64;       // columns per tile
constexpr int CP_LD = CP_TC + 1;  // padded row stride of the smem tile
constexpr int CP_THREADS = 256;

// One register block of a column-major GEMM over a shared-memory tile: rows Wa[0..4) and Wb[0..4) of the matrix (two
// groups of four consecutive rows, leading dimension ldw) times NC columns per lane (lane, lane + 32, ...):
//   a[q][u] += Σ_k Wa[k·ldw + q] · X[row(k)·ld + lane + 32u],   the same for b with Wb,
// one fmaf per term with k increasing, so the result depends on nothing but the operands.  `vec`: both groups are whole
// and 16-byte aligned for every k; otherwise na / nb (may be <= 0) rows of each group exist.  W goes through the read-only
// path (uniform addresses -> one sector per request, W stays L1/L2 resident).
template <int NC, class Row>
__device__ __forceinline__ void coupling_gemm_block(const float* X, int ld, Row row, int nk, const float* __restrict__ Wa,
                                                    const float* __restrict__ Wb, int ldw, int na, int nb, bool vec,
                                                    float (&a)[4][NC], float (&b)[4][NC]) {
  const int lane = threadIdx.x & 31;
  if (vec) {
#pragma unroll 4
    for (int k = 0; k < nk; ++k) {
      const int r = row(k);
      float xv[NC];
#pragma unroll
      for (int u = 0; u < NC; ++u) xv[u] = X[r * ld + lane + 32 * u];
      const float4 wa = __ldg(reinterpret_cast<const float4*>(Wa + (size_t)k * ldw));
      const float4 wb = __ldg(reinterpret_cast<const float4*>(Wb + (size_t)k * ldw));
#pragma unroll
      for (int u = 0; u < NC; ++u) {
        a[0][u] = fmaf(wa.x, xv[u], a[0][u]);
        a[1][u] = fmaf(wa.y, xv[u], a[1][u]);
        a[2][u] = fmaf(wa.z, xv[u], a[2][u]);
        a[3][u] = fmaf(wa.w, xv[u], a[3][u]);
      }
#pragma unroll
      for (int u = 0; u < NC; ++u) {
        b[0][u] = fmaf(wb.x, xv[u], b[0][u]);
        b[1][u] = fmaf(wb.y, xv[u], b[1][u]);
        b[2][u] = fmaf(wb.z, xv[u], b[2][u]);
        b[3][u] = fmaf(wb.w, xv[u], b[3][u]);
      }
    }
  } else {
    for (int k = 0; k < nk; ++k) {
      const int r = row(k);
      float xv[NC];
#pragma unroll
      for (int u = 0; u < NC; ++u) xv[u] = X[r * ld + lane + 32 * u];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (q < na) {
          const float w = __ldg(Wa + (size_t)k * ldw + q);
#pragma unroll
          for (int u = 0; u < NC; ++u) a[q][u] = fmaf(w, xv[u], a[q][u]);
        }
        if (q < nb) {
          const float w = __ldg(Wb + (size_t)k * ldw + q);
#pragma unroll
          for (int u = 0; u < NC; ++u) b[q][u] = fmaf(w, xv[u], b[q][u]);
        }
      }
    }
  }
}

// Conditioner GEMM [s; t] = W·x₂ + c and the affine epilogue on x₁, in place in shared memory, for one 64-column tile;
// leaves the column sums of s of this warp in red[warp][*].  The callers stage rows differently: x₂ row k lives at
// X2 + row2(k)·CP_LD, x₁ row j at X1 + row1(j)·CP_LD.  Every thread computes a 4(j) x 2(s,t) x 2(col) register block.
template <bool INV, class Row2, class Row1>
__device__ __forceinline__ void coupling_tile(const float* X2, float* X1, Row2 row2, Row1 row1, const float* __restrict__ W,
                                              const float* __restrict__ cvec, int n1, int n2, bool wvec, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ldw = 2 * n1;
  const int cA = lane, cB = lane + 32;
  float sumA = 0.f, sumB = 0.f;
  for (int jb = 4 * warp; jb < n1; jb += 4 * (CP_THREADS / 32)) {
    float s[4][2] = {}, t[4][2] = {};
    coupling_gemm_block<2>(X2, CP_LD, row2, n2, W + jb, W + n1 + jb, ldw, n1 - jb, n1 - jb, wvec, s, t);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = jb + q;
      if (j < n1) {
        const float cs = cvec ? __ldg(cvec + j) : 0.f, ct = cvec ? __ldg(cvec + n1 + j) : 0.f;
        const int r1 = row1(j);
        const float s_a = s[q][0] + cs, s_b = s[q][1] + cs, t_a = t[q][0] + ct, t_b = t[q][1] + ct;
        const float xa = X1[r1 * CP_LD + cA], xb = X1[r1 * CP_LD + cB];
        if (!INV) {
          X1[r1 * CP_LD + cA] = fmaf(expf(s_a), xa, t_a);  // exp(s)·x₁ + t  (scale.jl:13, shift.jl:14)
          X1[r1 * CP_LD + cB] = fmaf(expf(s_b), xb, t_b);
        } else {
          X1[r1 * CP_LD + cA] = (xa - t_a) / expf(s_a);  // inv.(a) .* (y₁ + (−t))  (scale.jl:16, shift.jl:12)
          X1[r1 * CP_LD + cB] = (xb - t_b) / expf(s_b);
        }
        sumA += s_a;
        sumB += s_b;
      }
    }
  }
  red[warp * CP_TC + cA] = sumA;
  red[warp * CP_TC + cB] = sumB;
}

}  // namespace b2b
