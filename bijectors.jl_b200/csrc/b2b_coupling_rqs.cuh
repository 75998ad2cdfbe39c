// Device pieces shared by the spline coupling kernels (B2B_COUPLING_RQS): the conditioner GEMM v = W·x₂ + c of one
// transformed row and the normalising constructor of rational_quadratic_spline.jl:109-123 with its pullback.
//
// Raw parameter j of transformed row i is v[i + n1·j] (0-based): widths j < K, heights K <= j < 2K, derivatives
// 2K <= j < 3K − 1.  A kernel stages the row's block of W as Ws[m][j] (n2 x JP floats, JP = 3K − 1 rounded up to 8,
// padding zero) and the row's c as cs[JP]; every thread then forms the 3K − 1 raw parameters of its own column.
#pragma once
#include <cuda_runtime.h>

namespace b2b {

__host__ __device__ constexpr inline int crq_jp(int K) { return (3 * K - 1 + 7) & ~7; }

// Copies transformed row i's (3K − 1) x n2 block of W (column-major, (3K − 1)·n1 rows) into Ws[m][j] and its c into cs
// (zeros when c == NULL).  Called by all `nthreads` threads of the CTA.
__device__ __forceinline__ void crq_stage_row(const float* __restrict__ W, const float* __restrict__ c, int i, int n1, int n2,
                                              int K, float* Ws, float* cs, int tid, int nthreads) {
  const int J = 3 * K - 1, JP = crq_jp(K);
  const size_t R = (size_t)J * n1;
  for (int e = tid; e < n2 * JP; e += nthreads) {
    const int m = e / JP, j = e - m * JP;
    Ws[e] = j < J ? W[(size_t)(i + n1 * j) + R * m] : 0.f;
  }
  for (int j = tid; j < JP; j += nthreads) cs[j] = (j < J && c) ? c[i + n1 * j] : 0.f;
}

// The raw parameters of one column: P[j·ps] = cs[j] + Σ_m Ws[m][j]·xcol[m·xs] for j < 3K − 1, in exact fp32 with the
// sum over m in increasing order.  Eight parameters at a time share each x₂ load (two broadcast float4 reads of Ws).
__device__ __forceinline__ void crq_params(const float* Ws, const float* cs, const float* xcol, int xs, int n2, int K,
                                           float* P, int ps) {
  const int J = 3 * K - 1, JP = crq_jp(K);
  for (int jb = 0; jb < J; jb += 8) {
    float a[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) a[q] = cs[jb + q];
    for (int m = 0; m < n2; ++m) {
      const float xv = xcol[m * xs];
      const float4 w0 = *reinterpret_cast<const float4*>(Ws + m * JP + jb);
      const float4 w1 = *reinterpret_cast<const float4*>(Ws + m * JP + jb + 4);
      a[0] = fmaf(w0.x, xv, a[0]);
      a[1] = fmaf(w0.y, xv, a[1]);
      a[2] = fmaf(w0.z, xv, a[2]);
      a[3] = fmaf(w0.w, xv, a[3]);
      a[4] = fmaf(w1.x, xv, a[4]);
      a[5] = fmaf(w1.y, xv, a[5]);
      a[6] = fmaf(w1.z, xv, a[6]);
      a[7] = fmaf(w1.w, xv, a[7]);
    }
#pragma unroll
    for (int q = 0; q < 8; ++q)
      if (jb + q < J) P[(jb + q) * ps] = a[q];
  }
}

// The neural spline coupling's hidden pre-activation W₁·x₂ + c₁ of unit m for one column (x₂ at xcol[k·xs]): from c₁
// (NULL: 0), FMAs over k in increasing order, so the forward and reverse-mode kernels form bit-identical values.  W₁ is
// H x n2 column-major.
__device__ __forceinline__ float crq_hidden_pre(const float* __restrict__ W1, const float* __restrict__ c1, int H, int n2,
                                                const float* xcol, int xs, int m) {
  float a = c1 ? __ldg(c1 + m) : 0.f;
  for (int k = 0; k < n2; ++k) a = fmaf(__ldg(W1 + (size_t)k * H + m), xcol[k * xs], a);
  return a;
}

// K + 1 knots from K raw values (stride as): out[k·os] = 2B·cumsum([0; softmax(a)])[k] − B, the max-subtracted softmax of
// oracle_np.softmax_rows and a sequential cumsum, each product and difference rounded as the float32 restatement does.
__device__ __forceinline__ void crq_knots(const float* a, int as, int K, float B, float* out, int os) {
  float mx = a[0];
  for (int k = 1; k < K; ++k) mx = fmaxf(mx, a[k * as]);
  float S = 0.f;
  for (int k = 0; k < K; ++k) S += expf(a[k * as] - mx);
  const float twoB = 2.0f * B;
  float cum = 0.f;
  out[0] = -B;
  for (int k = 0; k < K; ++k) {
    cum += expf(a[k * as] - mx) / S;
    out[(k + 1) * os] = __fsub_rn(__fmul_rn(twoB, cum), B);
  }
}

// Pullback of crq_knots: g[k·gs] (k = 0..K) holds the knot cotangents and is overwritten; a[k·as] (the raw values) is
// replaced by their cotangents.  Knot k depends on s_j for j < k (reverse cumsum), and the softmax pullback is
// ā = s ⊙ (s̄ − ⟨s̄, s⟩).  Knot 0 (= −B) is a constant.
__device__ __forceinline__ void crq_knots_vjp(float* a, int as, int K, float B, float* g, int gs) {
  float mx = a[0];
  for (int k = 1; k < K; ++k) mx = fmaxf(mx, a[k * as]);
  float S = 0.f;
  for (int k = 0; k < K; ++k) S += expf(a[k * as] - mx);
  const float twoB = 2.0f * B;
  float acc = 0.f, dot = 0.f;
  for (int j = K - 1; j >= 0; --j) {
    acc += g[(j + 1) * gs];
    const float sb = twoB * acc;
    g[(j + 1) * gs] = sb;  // slot j + 1 is consumed: it now holds s̄_j
    dot = fmaf(sb, expf(a[j * as] - mx) / S, dot);
  }
  for (int j = 0; j < K; ++j) {
    const float s = expf(a[j * as] - mx) / S;
    a[j * as] = s * (g[(j + 1) * gs] - dot);
  }
}

}  // namespace b2b
