// Reverse mode (VJP) of with_logabsdet_jacobian through a ∘-chain of RadialLayers, each applied forward
// (src/bijectors/radial_layer.jl:43-53,58-72) or as Inverse(layer) (:88-102,124-129; compute_r differentiated with the
// implicit-function rule) -- what the reference's AD computes when a radial flow is trained, on the sampling path
// (forward chain), the logpdf / NLL path (inverse(flow)) or any mix.
//
// Per layer, with δ = z − z0, r = ‖δ‖, h = 1/(α+r), s = β̂h, q = β̂ r h²:   y = z + sδ,
// logjac = (D−1)·log(1+s) + log(1+s−q).  Given the cotangents ȳ (D x N) and l̄ (N):
//   s̄ = δᵀȳ + l̄·((D−1)/(1+s) + 1/(1+s−q)),  q̄ = −l̄/(1+s−q),
//   β̂̄ = s̄ h + q̄ r h²,  h̄ = s̄ β̂ + 2 q̄ β̂ r h,  r̄ = q̄ β̂ h² − h̄ h²,  ᾱ = −h̄ h²,  κ = r̄/r,
//   z̄ = (1+s) ȳ + κ δ,   z̄0 = −Σ_n (s ȳ + κ δ),   then α = log1pexp(α_raw), β̂ = log1pexp(β) − α.
//
// Layout: TPC = 4 / 8 / 16 threads share a column (D <= 32 / 64 / 128), thread t owns rows t + TPC·v, v < 8, in registers:
// the two row reductions per layer (‖δ‖², δᵀȳ) are log2(TPC) shuffle steps and the per-column scalar algebra is repeated
// by TPC lanes instead of 32 (the warp-per-column first version spent three quarters of its issue slots on that).  The
// per-layer δ stay in registers between the forward recompute and the reverse sweep; the z̄0 partial sums (L x D per
// column group) live in shared-memory slots owned by the group (bank-disjoint across the groups of a warp), ᾱ / β̂̄ in
// registers.  Deterministic: groups, then CTAs, are combined in a fixed order.
// Algorithmic traffic: read x, read ȳ, write x̄ (+ l̄).
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_device.cuh"

namespace b2b {

constexpr int RV_THREADS = 256;
constexpr int RV_GRID_MAX = 592;
constexpr int RV_V = 8;  // rows per thread

template <int TPC>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = TPC / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// slot stride of a column group: L·D rounded up to TPC mod 32, so that the 32 / TPC groups of a warp hit disjoint banks
__host__ __device__ inline int rv_slot_stride(int L, int D, int tpc) { return ((L * D + 31) / 32) * 32 + tpc; }

// DD: 0 = D at run time, else the exact D = 8·TPC (row guards and every shared-memory offset become constants: a sixth
// of the instructions); FWD: all layers forward (the Inverse branch and its per-layer γ are compiled out).
template <int TPC, int L, int DD, bool FWD>
__global__ void __launch_bounds__(RV_THREADS, 2)
    radial_vjp_kernel(const __grid_constant__ B2BChainParams P, const float* __restrict__ ybar, long long ldyb,
                      const float* __restrict__ ljbar, float* __restrict__ xbar, long long ldxb,
                      float* __restrict__ partials) {
  constexpr int V = RV_V, G = RV_THREADS / TPC;
  extern __shared__ float rsm[];
  const int D = DD ? DD : P.D, SL = rv_slot_stride(L, D, TPC);
  float* z0s = rsm;               // [L][D]
  float* slots = rsm + L * D;     // [G][SL]
  const int t = threadIdx.x % TPC, g = threadIdx.x / TPC;
  float alpha[L], bhat[L];
  bool inv[L];
#pragma unroll
  for (int l = 0; l < L; ++l) {
    const b2b_layer_desc& d = P.layers[l];
    inv[l] = !FWD && d.inverse != 0;          // Inverse(layer): radial_layer.jl:88-102,124-129
    alpha[l] = softplus(d.p0[0]);             // radial_layer.jl:44
    bhat[l] = softplus(d.p1[0]) - alpha[l];   // :45
    for (int r = threadIdx.x; r < D; r += RV_THREADS) z0s[l * D + r] = d.p2[r];
  }
  for (int e = threadIdx.x; e < G * SL; e += RV_THREADS) slots[e] = 0.f;
  __syncthreads();
  float* my = slots + (size_t)g * SL;
  float acc_a[L], acc_b[L];
#pragma unroll
  for (int l = 0; l < L; ++l) acc_a[l] = acc_b[l] = 0.f;
  const float dm1 = (float)(D - 1);
  // every group of the grid walks columns gg, gg + stride, ... (whole warps stay in the loop together)
  const long long gg = (long long)blockIdx.x * G + g, stride = (long long)gridDim.x * G;
  const long long iters = (P.N + stride - 1) / stride;
  for (long long it = 0; it < iters; ++it) {
    const long long c = gg + it * stride;
    const bool ok = c < P.N;
    float z[V], yb[V], dl[L][V], rr[L], gm[L];
    const float lb = (ok && ljbar) ? ljbar[c] : 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const bool in = ok && (t + TPC * v < D);
      z[v] = in ? __ldcs(P.x + c * P.ldx + t + TPC * v) : 0.f;
      yb[v] = in ? __ldcs(ybar + c * ldyb + t + TPC * v) : 0.f;
    }
    // forward recompute: δ_l, r_l
#pragma unroll
    for (int l = 0; l < L; ++l) {
      float r2 = 0.f, z0v[V];
#pragma unroll
      for (int v = 0; v < V; ++v) {
        z0v[v] = (t + TPC * v < D) ? z0s[l * D + t + TPC * v] : 0.f;
        dl[l][v] = z[v] - z0v[v];
        r2 = fmaf(dl[l][v], dl[l][v], r2);
      }
      r2 = group_sum<TPC>(r2);
      // LinearAlgebra.norm, radial_layer.jl:47-49.  MUFU-based sqrt / reciprocals (<= 2 ulp)
      const float nrm = r2 > 0.f ? r2 * rsqrtf(r2) : 0.f;
      gm[l] = nrm;
      if (!inv[l]) {
        rr[l] = nrm;
        const float s = bhat[l] * __fdividef(1.0f, alpha[l] + nrm);
#pragma unroll
        for (int v = 0; v < V; ++v) z[v] = fmaf(s, dl[l][v], z[v]);  // :51
      } else {
        // compute_r (:124-129): the positive root of r² + (A − γ) r − αγ, without cancellation
        const float A = alpha[l] + bhat[l], a = A - nrm;
        const float sq = sqrtf(fmaf(a, a, 4.0f * alpha[l] * nrm));
        const float r = a > 0.f ? __fdividef(2.0f * alpha[l] * nrm, sq + a) : 0.5f * (sq - a);
        rr[l] = r;
        const float rho = (alpha[l] + r) * __fdividef(1.0f, A + r);  // :96
#pragma unroll
        for (int v = 0; v < V; ++v) z[v] = fmaf(rho, dl[l][v], z0v[v]);
      }
    }
    // reverse sweep
#pragma unroll
    for (int l = L - 1; l >= 0; --l) {
      float dot = 0.f;
#pragma unroll
      for (int v = 0; v < V; ++v) dot = fmaf(dl[l][v], yb[v], dot);
      dot = group_sum<TPC>(dot);
      const float r = rr[l], h = __fdividef(1.0f, alpha[l] + r), s = bhat[l] * h, q = bhat[l] * r * h * h;
      const float i1 = __fdividef(1.0f, 1.0f + s), i2 = __fdividef(1.0f, 1.0f + s - q);
      if (inv[l]) {
        // Inverse(layer): z = z0 + ρ δy, lj = −F(r); r differentiated implicitly (m = 2r + A − γ):
        // ∂r/∂γ = (α+r)/m, ∂r/∂α = γ/m, ∂r/∂A = −r/m  (oracle: radial_chain_vjp_dir)
        const float A = alpha[l] + bhat[l], gam = gm[l];
        const float iAr = __fdividef(1.0f, A + r), rho = (alpha[l] + r) * iAr;
        const float Fs = fmaf(dm1, i1, i2), Fq = -i2, Fb = -lb;
        const float bh2 = bhat[l] * h * h, bh3r = 2.0f * bhat[l] * r * h * h * h;
        const float dF_dr = fmaf(Fs, -bh2, Fq * (bh2 - bh3r));
        const float dF_da = fmaf(Fs, -bh2, Fq * -bh3r);
        const float dF_db = fmaf(Fs, h, Fq * r * h * h);
        const float r_bar = fmaf(dot * bhat[l], iAr * iAr, Fb * dF_dr);
        const float im = __fdividef(1.0f, 2.0f * r + A - gam);
        const float A_bar = fmaf(-dot * (alpha[l] + r), iAr * iAr, -r_bar * r * im);
        acc_a[l] += fmaf(dot, iAr, fmaf(Fb, dF_da, r_bar * gam * im)) + A_bar;
        acc_b[l] += fmaf(Fb, dF_db, A_bar);
        const float gam_bar = r_bar * (alpha[l] + r) * im;
        const float kap = gam > 0.f ? gam_bar * __fdividef(1.0f, gam) : 0.f;
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const float dyb = fmaf(yb[v], rho, kap * dl[l][v]);
          if (t + TPC * v < D) my[l * D + t + TPC * v] += yb[v] - dyb;
          yb[v] = dyb;
        }
        continue;
      }
      const float s_tot = fmaf(lb, fmaf(dm1, i1, i2), dot);
      const float q_bar = -lb * i2;
      const float bh_bar = fmaf(s_tot, h, q_bar * r * h * h);
      const float h_bar = fmaf(s_tot, bhat[l], 2.0f * q_bar * bhat[l] * r * h);
      const float r_bar = (q_bar * bhat[l] - h_bar) * h * h;
      const float kappa = r > 0.f ? r_bar * __fdividef(1.0f, r) : 0.f;
      acc_a[l] -= h_bar * h * h;
      acc_b[l] += bh_bar;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        if (t + TPC * v < D) my[l * D + t + TPC * v] -= fmaf(s, yb[v], kappa * dl[l][v]);
        yb[v] = fmaf(yb[v], 1.0f + s, kappa * dl[l][v]);
      }
    }
#pragma unroll
    for (int v = 0; v < V; ++v)
      if (ok && t + TPC * v < D) __stcs(xbar + c * ldxb + t + TPC * v, yb[v]);
  }
  // CTA partials: the groups' slots in a fixed order; ᾱ, β̂̄ from lane 0 of every group (all TPC lanes hold the same).
  // Columns beyond N ran on zeros: ȳ = 0, l̄ = 0 -> s̄ = 0 and every cotangent term is exactly 0.
  __shared__ float ab[2 * 8][RV_THREADS / 4];
  if (t == 0) {
#pragma unroll
    for (int l = 0; l < L; ++l) {
      ab[l][g] = acc_a[l];
      ab[8 + l][g] = acc_b[l];
    }
  }
  __syncthreads();
  const int nred = L * D + 2 * L;
  for (int i = threadIdx.x; i < nred; i += RV_THREADS) {
    float tsum = 0.f;
    if (i < L * D) {
      for (int w = 0; w < G; ++w) tsum += slots[(size_t)w * SL + i];
    } else {
      const int k = i - L * D, row = k < L ? k : 8 + (k - L);
      for (int w = 0; w < G; ++w) tsum += ab[row][w];
    }
    partials[(size_t)blockIdx.x * nred + i] = tsum;
  }
}

// out[i] = Σ_b partials[b][i], one warp per output (lane-strided partial sums, then a shuffle tree: fixed order).  Block 0
// owns the 2L scalar outputs and the chain rule through the parameter transforms, α = log1pexp(α_raw),
// β̂ = log1pexp(β) − α (radial_layer.jl:44-45); blocks 1.. own 8 entries of z̄0 each.
__global__ void __launch_bounds__(256)
    radial_vjp_finalize_kernel(const __grid_constant__ B2BChainParams P, int L, const float* __restrict__ partials,
                               int nblk, float* __restrict__ alpha_bar, float* __restrict__ beta_bar,
                               float* __restrict__ z0_bar) {
  const int D = P.D, n = L * D + 2 * L, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ float sums[16];
  auto total = [&](int i) {
    float s = 0.f;
    for (int b = lane; b < nblk; b += 32) s += partials[(size_t)b * n + i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
  };
  if (blockIdx.x > 0) {
    const int i = (blockIdx.x - 1) * 8 + warp;
    if (i < L * D) {
      const float s = total(i);
      if (lane == 0) z0_bar[i] = s;
    }
    return;
  }
  for (int k = warp; k < 2 * L; k += 8) {
    const float s = total(L * D + k);
    if (lane == 0) sums[k] = s;
  }
  __syncthreads();
  if (threadIdx.x < L) {
    const int l = threadIdx.x;
    const float a_raw = P.layers[l].p0[0], b_raw = P.layers[l].p1[0];
    const float bh = sums[L + l], al = sums[l] - bh;
    alpha_bar[l] = al / (1.0f + expf(-a_raw));
    beta_bar[l] = bh / (1.0f + expf(-b_raw));
  }
}

template <int TPC, int DD, bool FWD>
static int launch_radial_vjp(int L, int grid, const B2BChainParams& p, const float* ybar, long long ldyb,
                             const float* ljbar, float* xbar, long long ldxb, float* partials, cudaStream_t stream) {
  const size_t smem = ((size_t)L * p.D + (size_t)(RV_THREADS / TPC) * rv_slot_stride(L, p.D, TPC)) * sizeof(float);
#define B2B_RV_CASE(LL)                                                                                                \
  case LL: {                                                                                                           \
    auto kernel = radial_vjp_kernel<TPC, LL, DD, FWD>;                                                                 \
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);              \
    if (e != cudaSuccess) return (int)e;                                                                               \
    kernel<<<grid, RV_THREADS, smem, stream>>>(p, ybar, ldyb, ljbar, xbar, ldxb, partials);                            \
    break;                                                                                                             \
  }
  switch (L) {
    B2B_RV_CASE(1) B2B_RV_CASE(2) B2B_RV_CASE(3) B2B_RV_CASE(4) B2B_RV_CASE(5) B2B_RV_CASE(6) B2B_RV_CASE(7) B2B_RV_CASE(8)
    default: return B2B_EUNSUPPORTED;
  }
#undef B2B_RV_CASE
  return (int)cudaGetLastError();
}

// exact D = 8·TPC: forward-only and any-direction programs; other D: the any-direction program with run-time D
template <int TPC>
static int dispatch_radial_vjp(bool exact, bool fwd, int L, int grid, const B2BChainParams& p, const float* ybar, long long ldyb,
                               const float* ljbar, float* xbar, long long ldxb, float* partials, cudaStream_t stream) {
  if (exact && fwd) return launch_radial_vjp<TPC, 8 * TPC, true>(L, grid, p, ybar, ldyb, ljbar, xbar, ldxb, partials, stream);
  if (exact) return launch_radial_vjp<TPC, 8 * TPC, false>(L, grid, p, ybar, ldyb, ljbar, xbar, ldxb, partials, stream);
  return launch_radial_vjp<TPC, 0, false>(L, grid, p, ybar, ldyb, ljbar, xbar, ldxb, partials, stream);
}

}  // namespace b2b

size_t b2b_radial_vjp_workspace(int L, int D) {
  return (size_t)b2b::RV_GRID_MAX * (size_t)(L * D + 2 * L) * sizeof(float) + 256;
}

int b2b_vjp_radial(const B2BVjpSeg& s) {
  using namespace b2b;
  const int L = s.n, D = s.D;
  if (L < 1 || L > 8 || D > 128) return B2B_EUNSUPPORTED;
  for (int l = 0; l < L; ++l)
    if (s.layers[l].kind != B2B_RADIAL) return B2B_EUNSUPPORTED;
  if (!s.workspace || s.workspace_bytes < b2b_radial_vjp_workspace(L, D)) return B2B_EWORKSPACE;
  float* partials = reinterpret_cast<float*>(b2b_align256(s.workspace));
  B2BChainParams p;
  memset(&p, 0, sizeof(p));
  p.x = s.x;
  p.N = s.N;
  p.ldx = s.ldx;
  p.D = D;
  p.L = L;
  for (int l = 0; l < L; ++l) p.layers[l] = s.layers[l];
  const int sms = b2b_sm_count();
  int grid = sms * 4;
  if (grid > RV_GRID_MAX) grid = RV_GRID_MAX;
  const int tpc = D <= 32 ? 4 : D <= 64 ? 8 : 16;
  const long long want = (p.N + RV_THREADS / tpc - 1) / (RV_THREADS / tpc);
  if (grid > want) grid = (int)want;
  if (grid < 1) grid = 1;
  bool fwd = true;
  for (int l = 0; l < L; ++l) fwd = fwd && !p.layers[l].inverse;
  const bool exact = D == 8 * tpc;
  int rc;
  if (tpc == 4) rc = dispatch_radial_vjp<4>(exact, fwd, L, grid, p, s.ybar, s.ldyb, s.ljbar, s.xbar, s.ldxb, partials, s.stream);
  else if (tpc == 8) rc = dispatch_radial_vjp<8>(exact, fwd, L, grid, p, s.ybar, s.ldyb, s.ljbar, s.xbar, s.ldxb, partials, s.stream);
  else rc = dispatch_radial_vjp<16>(exact, fwd, L, grid, p, s.ybar, s.ldyb, s.ljbar, s.xbar, s.ldxb, partials, s.stream);
  if (rc != B2B_OK) return rc;
  // ᾱ, β̄ (L) and z̄₀ (L x D), each array 64-float aligned in scratch
  const size_t r = 64 * (size_t)((L + 63) / 64);
  float* const ab = s.scratch ? s.scratch : s.bars[0];
  float* const bb = s.scratch ? s.scratch + r : s.bars[1];
  float* const zb = s.scratch ? s.scratch + 2 * r : s.bars[2];
  radial_vjp_finalize_kernel<<<1 + (L * D + 7) / 8, 256, 0, s.stream>>>(p, L, partials, grid, ab, bb, zb);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  *s.launches += 2;
  if (!s.scratch) return B2B_OK;
  const float* const base[3] = {ab, bb, zb};
  const size_t step[3] = {1, 1, (size_t)D};
  return b2b_copy_run_bars(s.layers, L, s.bars, base, step, D, s.launches, s.stream);
}
