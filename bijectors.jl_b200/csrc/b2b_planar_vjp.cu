// Reverse mode (VJP) of planar chains on the TMA pipeline (see b2b_planar_const.cu for the forward kernels); parameters
// are derived in the kernel prologue into shared memory, as in planar_dev_kernel -- no library-owned device state.
#include "b2b_planar_common.cuh"

namespace b2b {

// ---- reverse mode (VJP) of a forward planar chain ---------------------------------------------------------
// Reverse-mode AD of with_logabsdet_jacobian through L PlanarLayers is what the reference's training loop runs
// (docs/src/flows.md:93-100; rules in ext/BijectorsChainRulesCoreExt.jl).  With z_{l+1} = z_l + û_l t_l,
// a_l = w_lᵀz_l + b_l, t_l = tanh a_l, s_l = sech² a_l, logjac = Σ_l log1p(c_l s_l) and cotangents ȳ (D x N), l̄ (N):
//     d_l = û_lᵀ ȳ_{l+1},   g_l = s_l d_l − l̄ · 2 c_l t_l s_l / (1 + c_l s_l),   ȳ_l = ȳ_{l+1} + w_l g_l      (x̄ = ȳ_0)
//     û̄_l = Σ_n t_l ȳ_{l+1},  w̄_l(direct) = Σ_n g_l z_l,  b̄_l = Σ_n g_l,  c̄_l = Σ_n l̄ s_l / (1 + c_l s_l).
// Since ȳ_{l+1} = ȳ_L + Σ_{k>l} w_k g_k and z_l = z_0 + Σ_{k<l} û_k t_k, the two D x N reductions only need the
// ORIGINAL tensors:  û̄_l = T_l·Ȳ_Lᵀ + Σ_{k>l} S[k][l] w_k,  w̄_l = G_l·Z_0ᵀ + Σ_{k<l} S[l][k] û_k,  S[l][k] = Σ_n g_l t_k.
//   K1 planar_vjp_kernel   thread-per-column (same TMA pipeline, 2 input tensors): forward recompute of t, s from x,
//                          then the reverse sweep on ȳ in the SAME registers; writes x̄ and 3·L scalars per column
//   K2 planar_pgrad_kernel skinny reductions G·Z_0ᵀ and T·Ȳ_Lᵀ (L x D each), deterministic partials
//   K3 planar_sstat_kernel S, b̄, c̄ from the per-column scalars
//   K4 planar_vjp_finalize combines everything and applies the chain rule through get_u_hat (planar_layer.jl:65-70)
template <int L>
struct VjpState {
  float t[L], s2[L];
};

// DIR 0: forward layers; DIR 1: inverse layers in application order (the logpdf / NLL path): α from find_alpha,
// differentiated with the implicit-function rule ext/BijectorsChainRulesCoreExt.jl:42-46
// (∂α/∂(wᵀy) = X, ∂α/∂c = −tanh(α+b)·X, ∂α/∂b = X − 1, X = 1/(1 + c·sech²(α+b))):
//   u_{k+1} = u_k − û_k th_k,  g_k = X·(−s_k·û_kᵀζ_{k+1} + 2 c th_k·l̄ s_k X),  ζ_k = ζ_{k+1} + w_k g_k.
template <int D, int L, int DIR>
struct PlanarVjpProg {
  using State = VjpState<L>;
  const B2BChainParams& P;
  int nreal;
  float* scal;     // [N][3][L]: g | t | l̄·s/(1+c·s)
  long long N;
  __device__ __forceinline__ void stage(float* params, int warp, int lane, int nw) const {
    planar_derive_smem<D>(P, nreal, L, params, warp, lane, nw);
  }
  // forward recompute on the x fragment: t_l, s_l
  __device__ __forceinline__ void phase1(float2 (&x)[1][D / 2], const ColCtx<D, 1>&, const float* params,
                                         State& st) const {
#pragma unroll
    for (int l = 0; l < L; ++l) {
      const float4* w4 = reinterpret_cast<const float4*>(params + l * D);
      const float4* u4 = reinterpret_cast<const float4*>(params + L * D + l * D);
      float2 acc[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = make_float2(0.f, 0.f);
#pragma unroll
      for (int i = 0; i < D / 4; ++i) {
        const float4 w = w4[i];
        acc[(i & 1) * 2 + 0] = b2b_ffma2(make_float2(w.x, w.y), x[0][2 * i], acc[(i & 1) * 2 + 0]);
        acc[(i & 1) * 2 + 1] = b2b_ffma2(make_float2(w.z, w.w), x[0][2 * i + 1], acc[(i & 1) * 2 + 1]);
      }
      const float2 s = b2b_fadd2(b2b_fadd2(acc[0], acc[1]), b2b_fadd2(acc[2], acc[3]));
      const float cc_ = params[2 * L * D + l], bb = params[2 * L * D + L + l];
      if (DIR == 0) tanh_sech2(s.x + s.y + bb, st.t[l], st.s2[l]);
      else find_alpha_ts(s.x + s.y, cc_, bb, st.t[l], st.s2[l]);  // planar_layer.jl:121
      if (l + 1 < L) {  // the last layer's output is not needed
        const float tt = DIR == 0 ? st.t[l] : -st.t[l];
        const float2 t2 = make_float2(tt, tt);
#pragma unroll
        for (int i = 0; i < D / 4; ++i) {
          const float4 u = u4[i];
          x[0][2 * i] = b2b_ffma2(make_float2(u.x, u.y), t2, x[0][2 * i]);
          x[0][2 * i + 1] = b2b_ffma2(make_float2(u.z, u.w), t2, x[0][2 * i + 1]);
        }
      }
    }
  }
  // reverse sweep on the ȳ fragment; lj[0] = l̄ of this column
  __device__ __forceinline__ void apply(float2 (&x)[1][D / 2], const ColCtx<D, 1>&, const float* params,
                                        float (&lj)[1], const State& st, long long col) const {
    float g[L], cb[L];
#pragma unroll
    for (int l = L - 1; l >= 0; --l) {
      const float4* w4 = reinterpret_cast<const float4*>(params + l * D);
      const float4* u4 = reinterpret_cast<const float4*>(params + L * D + l * D);
      float2 acc[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = make_float2(0.f, 0.f);
#pragma unroll
      for (int i = 0; i < D / 4; ++i) {
        const float4 u = u4[i];
        acc[(i & 1) * 2 + 0] = b2b_ffma2(make_float2(u.x, u.y), x[0][2 * i], acc[(i & 1) * 2 + 0]);
        acc[(i & 1) * 2 + 1] = b2b_ffma2(make_float2(u.z, u.w), x[0][2 * i + 1], acc[(i & 1) * 2 + 1]);
      }
      const float2 s = b2b_fadd2(b2b_fadd2(acc[0], acc[1]), b2b_fadd2(acc[2], acc[3]));
      const float d = s.x + s.y;  // û_lᵀ ȳ_{l+1}
      const float c = params[2 * L * D + l], s2 = st.s2[l], t = st.t[l];
      const float rden = __frcp_rn(fmaf(c, s2, 1.0f));
      cb[l] = lj[0] * s2 * rden;
      if (DIR == 0) g[l] = fmaf(s2, d, -2.0f * c * t * cb[l]);
      else g[l] = rden * fmaf(-s2, d, 2.0f * c * t * cb[l]);
      const float2 g2 = make_float2(g[l], g[l]);
#pragma unroll
      for (int i = 0; i < D / 4; ++i) {
        const float4 w = w4[i];
        x[0][2 * i] = b2b_ffma2(make_float2(w.x, w.y), g2, x[0][2 * i]);
        x[0][2 * i + 1] = b2b_ffma2(make_float2(w.z, w.w), g2, x[0][2 * i + 1]);
      }
    }
    if (col < N) {
      float* o = scal + col * (3 * L);
#pragma unroll
      for (int l = 0; l < L; ++l) {
        o[l] = g[l];
        o[L + l] = st.t[l];
        o[2 * L + l] = cb[l];
      }
    }
  }
};

template <int D, int L, int NW, int DIR>
__global__ void __launch_bounds__(NW * 32, 1)
    planar_vjp_kernel(const __grid_constant__ B2BChainParams P, const __grid_constant__ V1Extra E,
                      const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_yb,
                      const __grid_constant__ CUtensorMap map_xb, float* scal, const int nreal) {
  const PlanarVjpProg<D, L, DIR> prog{P, nreal, scal, P.N};
  v1_run<D, 1, 1, NW, PlanarVjpProg<D, L, DIR>, 2>(P, E, map_x, map_xb, prog, &map_yb);
}

// K2: A1[l][r] = Σ_n g[l,n]·x[r,n],  A2[l][r] = Σ_n t[l,n]·ȳ[r,n].  A warp handles 128/D columns at a time (lane ->
// (sub-column, 4-row chunk)), private fp32 accumulators, CTA partials combined in a fixed order (deterministic).
constexpr int PG_THREADS = 256;
template <int D, int L>
__global__ void __launch_bounds__(PG_THREADS)
    planar_pgrad_kernel(const float* __restrict__ x, const float* __restrict__ yb, const float* __restrict__ scal,
                        long long N, long long ldx, long long ldyb, float* __restrict__ partials) {
  constexpr int LPCOL = D / 4;        // lanes per column
  constexpr int CPW = 32 / LPCOL;     // columns per warp step
  __shared__ float red[2 * L * D];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = PG_THREADS / 32;
  for (int i = threadIdx.x; i < 2 * L * D; i += PG_THREADS) red[i] = 0.f;
  __syncthreads();
  const int sub = lane / LPCOL, chunk = lane % LPCOL;
  float4 a1[L], a2[L];
#pragma unroll
  for (int l = 0; l < L; ++l) a1[l] = a2[l] = make_float4(0.f, 0.f, 0.f, 0.f);
  const long long gw = (long long)blockIdx.x * nwarps + warp, stride = (long long)gridDim.x * nwarps;
  // UNR column groups per iteration: all loads are issued before the FMAs (2·UNR 16-byte loads in flight per lane)
  constexpr int UNR = 4;
  for (long long c0 = gw * (CPW * UNR); c0 < N; c0 += stride * (CPW * UNR)) {
    float4 xv[UNR], yv[UNR];
    float g[UNR][L], t[UNR][L];
#pragma unroll
    for (int k = 0; k < UNR; ++k) {
      const long long col = c0 + k * CPW + sub;
      const bool ok = col < N;
      const long long cs = ok ? col : 0;
      xv[k] = __ldcs(reinterpret_cast<const float4*>(x + cs * ldx) + chunk);
      yv[k] = __ldcs(reinterpret_cast<const float4*>(yb + cs * ldyb) + chunk);
      const float* sc = scal + cs * (3 * L);
      if constexpr (L % 4 == 0) {
#pragma unroll
        for (int l = 0; l < L; l += 4) {
          const float4 gv = __ldg(reinterpret_cast<const float4*>(sc + l));
          const float4 tv = __ldg(reinterpret_cast<const float4*>(sc + L + l));
          g[k][l] = gv.x; g[k][l + 1] = gv.y; g[k][l + 2] = gv.z; g[k][l + 3] = gv.w;
          t[k][l] = tv.x; t[k][l + 1] = tv.y; t[k][l + 2] = tv.z; t[k][l + 3] = tv.w;
        }
      } else {
#pragma unroll
        for (int l = 0; l < L; ++l) {
          g[k][l] = __ldg(sc + l);
          t[k][l] = __ldg(sc + L + l);
        }
      }
      if (!ok) {
#pragma unroll
        for (int l = 0; l < L; ++l) g[k][l] = t[k][l] = 0.f;
      }
    }
#pragma unroll
    for (int k = 0; k < UNR; ++k) {
#pragma unroll
      for (int l = 0; l < L; ++l) {
        a1[l].x = fmaf(g[k][l], xv[k].x, a1[l].x); a1[l].y = fmaf(g[k][l], xv[k].y, a1[l].y);
        a1[l].z = fmaf(g[k][l], xv[k].z, a1[l].z); a1[l].w = fmaf(g[k][l], xv[k].w, a1[l].w);
        a2[l].x = fmaf(t[k][l], yv[k].x, a2[l].x); a2[l].y = fmaf(t[k][l], yv[k].y, a2[l].y);
        a2[l].z = fmaf(t[k][l], yv[k].z, a2[l].z); a2[l].w = fmaf(t[k][l], yv[k].w, a2[l].w);
      }
    }
  }
  // sub-columns of a warp -> lanes [0, LPCOL)
#pragma unroll
  for (int l = 0; l < L; ++l) {
#pragma unroll
    for (int o = LPCOL; o < 32; o <<= 1) {
      a1[l].x += __shfl_xor_sync(0xffffffffu, a1[l].x, o); a1[l].y += __shfl_xor_sync(0xffffffffu, a1[l].y, o);
      a1[l].z += __shfl_xor_sync(0xffffffffu, a1[l].z, o); a1[l].w += __shfl_xor_sync(0xffffffffu, a1[l].w, o);
      a2[l].x += __shfl_xor_sync(0xffffffffu, a2[l].x, o); a2[l].y += __shfl_xor_sync(0xffffffffu, a2[l].y, o);
      a2[l].z += __shfl_xor_sync(0xffffffffu, a2[l].z, o); a2[l].w += __shfl_xor_sync(0xffffffffu, a2[l].w, o);
    }
  }
  // warps add their sums in a fixed order (warp 0 first, ...): deterministic
  for (int w = 0; w < nwarps; ++w) {
    if (warp == w && lane < LPCOL) {
#pragma unroll
      for (int l = 0; l < L; ++l) {
        float4* r1 = reinterpret_cast<float4*>(&red[l * D + 4 * chunk]);
        float4* r2 = reinterpret_cast<float4*>(&red[L * D + l * D + 4 * chunk]);
        float4 v1 = *r1, v2 = *r2;
        v1.x += a1[l].x; v1.y += a1[l].y; v1.z += a1[l].z; v1.w += a1[l].w;
        v2.x += a2[l].x; v2.y += a2[l].y; v2.z += a2[l].z; v2.w += a2[l].w;
        *r1 = v1;
        *r2 = v2;
      }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < 2 * L * D; i += PG_THREADS) partials[(size_t)blockIdx.x * (2 * L * D) + i] = red[i];
}

// K2 for dense batches (ld == D): chunks of PGB_CH columns of x, ȳ and the per-column scalars are contiguous in global
// memory, so one elected thread streams them into a 4-stage shared-memory ring with three 1-D bulk copies per chunk
// (cp.async.bulk + mbarrier full/empty pairs); the 8 warps consume from shared memory.  This keeps ~100 KB in flight
// per SM -- the register-staged kernel above is bound by load latency.
constexpr int PGB_CH = 16;      // columns per chunk
constexpr int PGB_STAGES = 4;
template <int D, int L>
__global__ void __launch_bounds__(PG_THREADS)
    planar_pgrad_bulk_kernel(const float* __restrict__ x, const float* __restrict__ yb, const float* __restrict__ scal,
                             long long N, float* __restrict__ partials) {
  constexpr int LPCOL = D / 4, CPW = 32 / LPCOL, NWARPS = PG_THREADS / 32;
  constexpr int XB = PGB_CH * D * 4, SB = PGB_CH * 3 * L * 4, STAGE = 2 * XB + SB;
  extern __shared__ __align__(128) unsigned char pg_smem[];
  __shared__ uint64_t full[PGB_STAGES], empty[PGB_STAGES];
  __shared__ float red[2 * L * D];
  const int lane = threadIdx.x & 31, warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int sub = lane / LPCOL, chunk = lane % LPCOL;
  for (int i = threadIdx.x; i < 2 * L * D; i += PG_THREADS) red[i] = 0.f;
  if (threadIdx.x == 0) {
    for (int s = 0; s < PGB_STAGES; ++s) {
      mbar_init(smem_u32(&full[s]), 1);
      mbar_init(smem_u32(&empty[s]), NWARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const long long nchunks = (N + PGB_CH - 1) / PGB_CH;
  const long long mine = (nchunks - blockIdx.x + gridDim.x - 1) / gridDim.x;  // chunks blockIdx.x + k*gridDim.x
  auto issue = [&](long long k) {
    const int s = (int)(k % PGB_STAGES);
    const long long c0 = (blockIdx.x + k * gridDim.x) * PGB_CH;
    const int cols = (int)((N - c0 < PGB_CH) ? (N - c0) : PGB_CH);
    const uint32_t bar = smem_u32(&full[s]);
    unsigned char* st = pg_smem + (size_t)s * STAGE;
    // bulk copies move multiples of 16 bytes: the scalar block of a ragged last chunk is rounded up (the bytes past
    // it belong to the same workspace allocation and are never used)
    const uint32_t sbytes = ((uint32_t)cols * 3 * L * 4 + 15u) & ~15u;
    mbar_expect_tx(bar, (uint32_t)cols * (2 * D * 4) + sbytes);
    bulk_load_1d(smem_u32(st), x + c0 * D, (uint32_t)cols * D * 4, bar);
    bulk_load_1d(smem_u32(st + XB), yb + c0 * D, (uint32_t)cols * D * 4, bar);
    bulk_load_1d(smem_u32(st + 2 * XB), scal + c0 * (3 * L), sbytes, bar);
  };
  if (threadIdx.x == 0)
    for (long long k = 0; k < PGB_STAGES - 1 && k < mine; ++k) issue(k);

  float4 a1[L], a2[L];
#pragma unroll
  for (int l = 0; l < L; ++l) a1[l] = a2[l] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long k = 0; k < mine; ++k) {
    const int s = (int)(k % PGB_STAGES);
    // refill the stage that was consumed in the previous iteration with chunk k + STAGES − 1
    if (threadIdx.x == 0 && k + PGB_STAGES - 1 < mine) {
      const long long kn = k + PGB_STAGES - 1;
      if (kn >= PGB_STAGES) mbar_wait(smem_u32(&empty[kn % PGB_STAGES]), (uint32_t)(((kn / PGB_STAGES) - 1) & 1));
      issue(kn);
    }
    mbar_wait(smem_u32(&full[s]), (uint32_t)((k / PGB_STAGES) & 1));
    const long long c0 = (blockIdx.x + k * gridDim.x) * PGB_CH;
    const int cols = (int)((N - c0 < PGB_CH) ? (N - c0) : PGB_CH);
    const unsigned char* st = pg_smem + (size_t)s * STAGE;
    const float4* xs = reinterpret_cast<const float4*>(st);
    const float4* ys = reinterpret_cast<const float4*>(st + XB);
    const float* sc = reinterpret_cast<const float*>(st + 2 * XB);
#pragma unroll
    for (int cc = 0; cc < PGB_CH / (NWARPS * CPW) + (PGB_CH % (NWARPS * CPW) ? 1 : 0); ++cc) {
      const int col = (cc * NWARPS + warp) * CPW + sub;
      if (col < cols) {
        const float4 xv = xs[col * LPCOL + chunk], yv = ys[col * LPCOL + chunk];
        const float* sp = sc + col * (3 * L);
#pragma unroll
        for (int l = 0; l < L; ++l) {
          const float g = sp[l], t = sp[L + l];
          a1[l].x = fmaf(g, xv.x, a1[l].x); a1[l].y = fmaf(g, xv.y, a1[l].y);
          a1[l].z = fmaf(g, xv.z, a1[l].z); a1[l].w = fmaf(g, xv.w, a1[l].w);
          a2[l].x = fmaf(t, yv.x, a2[l].x); a2[l].y = fmaf(t, yv.y, a2[l].y);
          a2[l].z = fmaf(t, yv.z, a2[l].z); a2[l].w = fmaf(t, yv.w, a2[l].w);
        }
      }
    }
    // this warp is done with the stage: order its generic-proxy reads before the async refill, then release
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&empty[s]));
  }
#pragma unroll
  for (int l = 0; l < L; ++l) {
#pragma unroll
    for (int o = LPCOL; o < 32; o <<= 1) {
      a1[l].x += __shfl_xor_sync(0xffffffffu, a1[l].x, o); a1[l].y += __shfl_xor_sync(0xffffffffu, a1[l].y, o);
      a1[l].z += __shfl_xor_sync(0xffffffffu, a1[l].z, o); a1[l].w += __shfl_xor_sync(0xffffffffu, a1[l].w, o);
      a2[l].x += __shfl_xor_sync(0xffffffffu, a2[l].x, o); a2[l].y += __shfl_xor_sync(0xffffffffu, a2[l].y, o);
      a2[l].z += __shfl_xor_sync(0xffffffffu, a2[l].z, o); a2[l].w += __shfl_xor_sync(0xffffffffu, a2[l].w, o);
    }
  }
  for (int w = 0; w < NWARPS; ++w) {
    if (warp == w && lane < LPCOL) {
#pragma unroll
      for (int l = 0; l < L; ++l) {
        float4* r1 = reinterpret_cast<float4*>(&red[l * D + 4 * chunk]);
        float4* r2 = reinterpret_cast<float4*>(&red[L * D + l * D + 4 * chunk]);
        float4 v1 = *r1, v2 = *r2;
        v1.x += a1[l].x; v1.y += a1[l].y; v1.z += a1[l].z; v1.w += a1[l].w;
        v2.x += a2[l].x; v2.y += a2[l].y; v2.z += a2[l].z; v2.w += a2[l].w;
        *r1 = v1;
        *r2 = v2;
      }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < 2 * L * D; i += PG_THREADS) partials[(size_t)blockIdx.x * (2 * L * D) + i] = red[i];
}

// fixed-order sum of per-CTA partials: out[i] = Σ_b partials[b][i].  One warp per output: lane k adds the partials
// b ≡ k (mod 32) in increasing order, then a fixed shuffle tree combines the lanes (deterministic, and the nblk
// dependent loads of a serial sum become nblk/32).
__global__ void __launch_bounds__(256) planar_psum_kernel(const float* __restrict__ partials, int nblk, int n,
                                                          float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * 8 + (threadIdx.x >> 5); i < n; i += gridDim.x * 8) {
    float s = 0.f;
    for (int b = lane; b < nblk; b += 32) s += partials[(size_t)b * n + i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[i] = s;
  }
}

// K3: S[l][k] = Σ_n g[l,n]·t[k,n] (all L x L), gb[l] = Σ_n g[l,n], gc[l] = Σ_n cb[l,n]; thread per column.
constexpr int SS_THREADS = 128;
template <int L>
__global__ void __launch_bounds__(SS_THREADS)
    planar_sstat_kernel(const float* __restrict__ scal, long long N, float* __restrict__ partials) {
  constexpr int NS = L * L + 2 * L;
  __shared__ float red[SS_THREADS / 32][NS];
  float acc[NS];
#pragma unroll
  for (int i = 0; i < NS; ++i) acc[i] = 0.f;
  for (long long col = (long long)blockIdx.x * SS_THREADS + threadIdx.x; col < N; col += (long long)gridDim.x * SS_THREADS) {
    const float* sc = scal + col * (3 * L);
    float g[L], t[L];
#pragma unroll
    for (int l = 0; l < L; ++l) {
      g[l] = sc[l];
      t[l] = sc[L + l];
      acc[L * L + l] += g[l];
      acc[L * L + L + l] += sc[2 * L + l];
    }
#pragma unroll
    for (int l = 0; l < L; ++l)
#pragma unroll
      for (int k = 0; k < L; ++k) acc[l * L + k] = fmaf(g[l], t[k], acc[l * L + k]);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NS; ++i) {
    float v = acc[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NS; i += SS_THREADS) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < SS_THREADS / 32; ++w) s += red[w][i];
    partials[(size_t)blockIdx.x * NS + i] = s;
  }
}

// K4 (one CTA per layer): w̄, ū, b̄ of the `nreal` layers.  `packed` = the prep kernel's w | û | c | b for (D, Lp); A = A1 | A2
// (Lp x D each); SS = S | gb | gc.  Chain rule through get_u_hat: û = u + k·w, k = (log1pexp(−s) − 1)/q, s = wᵀu,
// q = wᵀw, c = log1pexp(s) − 1 (planar_layer.jl:65-70).
__device__ __forceinline__ float block_sum_256(float v, float* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += sh[w];
  return s;
}

__global__ void __launch_bounds__(256)
    planar_vjp_finalize_kernel(const __grid_constant__ B2BChainParams P, int nreal, int Lp, int dir, const float* __restrict__ packed,
                               const float* __restrict__ A, const float* __restrict__ SS, float* __restrict__ wbar,
                               float* __restrict__ ubar, float* __restrict__ bbar) {
  __shared__ float sh[8];
  const int D = P.D, i = threadIdx.x;
  const float* W = packed;
  const float* UH = packed + Lp * D;
  const float* S = SS;
  const float* gb = SS + Lp * Lp;
  const float* gc = gb + Lp;
  const int l = blockIdx.x;  // one CTA per layer
  {
    const b2b_layer_desc& d = P.layers[l];
    float uhb = 0.f, wdir = 0.f, w = 0.f, u = 0.f;
    if (i < D) {
      w = d.p0[i];
      u = d.p1[i];
      uhb = A[Lp * D + l * D + i];
      wdir = A[l * D + i];
#pragma unroll
      for (int k = 0; k < HP_MAX_L; ++k) {  // independent loads first, short FMA chains after
        const float s_kl = (k > l && k < nreal) ? S[k * Lp + l] : 0.f;
        const float w_k = (k > l && k < nreal) ? W[k * D + i] : 0.f;
        const float s_lk = (k < l) ? S[l * Lp + k] : 0.f;
        const float uh_k = (k < l) ? UH[k * D + i] : 0.f;
        uhb = fmaf(s_kl, w_k, uhb);
        wdir = fmaf(dir ? -s_lk : s_lk, uh_k, wdir);
      }
      if (dir) uhb = -uhb;  // inverse layers subtract û·tanh
    }
    const float s = block_sum_256(w * u, sh);
    const float q = block_sum_256(w * w, sh);
    const float uw = block_sum_256(uhb * w, sh);
    const float kk = (softplus(-s) - 1.0f) / q;
    const float sig_s = 1.0f / (1.0f + expf(-s)), sig_ms = 1.0f / (1.0f + expf(s));
    const float dk_ds = -sig_ms / q, dk_dq = -kk / q;
    const float cbar = dir ? -S[l * Lp + l] - gc[l] : gc[l];  // inverse: Σ(−th·g) − Σ l̄ s X
    if (i < D) {
      ubar[l * D + i] = fmaf(fmaf(uw, dk_ds, cbar * sig_s), w, uhb);
      wbar[l * D + i] = wdir + kk * uhb + uw * fmaf(dk_ds, u, dk_dq * 2.0f * w) + cbar * sig_s * u;
    }
    if (i == 0) bbar[l] = gb[l];
  }
}

}  // namespace b2b

// ---- reverse mode: host side ----------------------------------------------------------------------------
namespace b2b {

static inline size_t vjp_align(size_t v) { return (v + 255) & ~(size_t)255; }
constexpr int VJP_PG_GRID = 592;   // 4 CTAs per SM
constexpr int VJP_SS_GRID = 296;

struct VjpWs {
  float *scal, *pg_partials, *A, *ss_partials, *SS, *packed;
  size_t bytes;
};

static VjpWs vjp_carve(char* base, int Lp, int D, long long N) {
  VjpWs w;
  size_t off = 0;
  auto take = [&](size_t nfloats) {
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += vjp_align(nfloats * sizeof(float));
    return p;
  };
  w.scal = take((size_t)N * 3 * Lp);
  w.pg_partials = take((size_t)VJP_PG_GRID * 2 * Lp * D);
  w.A = take((size_t)2 * Lp * D);
  w.ss_partials = take((size_t)VJP_SS_GRID * (Lp * Lp + 2 * Lp));
  w.SS = take((size_t)Lp * Lp + 2 * Lp);
  w.packed = take((size_t)2 * Lp * D + 2 * Lp);
  w.bytes = off + 256;
  return w;
}

template <int D, int L, int NW>
static int launch_vjp_main(int dir, const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx, const CUtensorMap& myb,
                           const CUtensorMap& mxb, float* scal, int nreal, cudaStream_t stream) {
  auto kernel = dir ? planar_vjp_kernel<D, L, NW, 1> : planar_vjp_kernel<D, L, NW, 0>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<g.grid, NW * 32, g.smem, stream>>>(q, g.extra, mx, myb, mxb, scal, nreal);
  return (int)cudaGetLastError();
}

// NW8: the warps of the 8-layer program
template <int D, int NW, int NW8 = NW>
static int dispatch_vjp_main(int dir, int L, const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx,
                             const CUtensorMap& myb, const CUtensorMap& mxb, float* scal, int nreal,
                             cudaStream_t stream) {
  switch (L) {
    case 1: return launch_vjp_main<D, 1, NW>(dir, q, g, mx, myb, mxb, scal, nreal, stream);
    case 2: return launch_vjp_main<D, 2, NW>(dir, q, g, mx, myb, mxb, scal, nreal, stream);
    case 4: return launch_vjp_main<D, 4, NW>(dir, q, g, mx, myb, mxb, scal, nreal, stream);
    case 8: return launch_vjp_main<D, 8, NW8>(dir, q, g, mx, myb, mxb, scal, nreal, stream);
    default: return B2B_EUNSUPPORTED;
  }
}

template <int D, int L>
static int launch_pgrad_L(const float* x, const float* yb, const float* scal, long long N, long long ldx,
                          long long ldyb, float* partials, cudaStream_t stream) {
  const bool dense = ldx == D && ldyb == D && !((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(yb) |
                                                 reinterpret_cast<uintptr_t>(scal)) & 15);
  if (dense) {
    auto kernel = planar_pgrad_bulk_kernel<D, L>;
    const int smem = PGB_STAGES * (2 * PGB_CH * D * 4 + PGB_CH * 3 * L * 4);
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    kernel<<<VJP_PG_GRID, PG_THREADS, smem, stream>>>(x, yb, scal, N, partials);
  } else {
    planar_pgrad_kernel<D, L><<<VJP_PG_GRID, PG_THREADS, 0, stream>>>(x, yb, scal, N, ldx, ldyb, partials);
  }
  return (int)cudaGetLastError();
}

template <int D>
static int launch_pgrad(int L, const float* x, const float* yb, const float* scal, long long N, long long ldx,
                        long long ldyb, float* partials, cudaStream_t stream) {
  switch (L) {
    case 1: return launch_pgrad_L<D, 1>(x, yb, scal, N, ldx, ldyb, partials, stream);
    case 2: return launch_pgrad_L<D, 2>(x, yb, scal, N, ldx, ldyb, partials, stream);
    case 4: return launch_pgrad_L<D, 4>(x, yb, scal, N, ldx, ldyb, partials, stream);
    case 8: return launch_pgrad_L<D, 8>(x, yb, scal, N, ldx, ldyb, partials, stream);
    default: return B2B_EUNSUPPORTED;
  }
}

static int launch_sstat(int L, const float* scal, long long N, float* partials, cudaStream_t stream) {
  switch (L) {
    case 1: planar_sstat_kernel<1><<<VJP_SS_GRID, SS_THREADS, 0, stream>>>(scal, N, partials); break;
    case 2: planar_sstat_kernel<2><<<VJP_SS_GRID, SS_THREADS, 0, stream>>>(scal, N, partials); break;
    case 4: planar_sstat_kernel<4><<<VJP_SS_GRID, SS_THREADS, 0, stream>>>(scal, N, partials); break;
    case 8: planar_sstat_kernel<8><<<VJP_SS_GRID, SS_THREADS, 0, stream>>>(scal, N, partials); break;
    default: return B2B_EUNSUPPORTED;
  }
  return (int)cudaGetLastError();
}

}  // namespace b2b

size_t b2b_planar_vjp_workspace(int L, int D, long long N) {
  int Lp = 1;
  while (Lp < L) Lp <<= 1;
  return b2b::vjp_carve(nullptr, Lp, D, N).bytes;
}

int b2b_vjp_planar(const B2BVjpSeg& s) {
  using namespace b2b;
  const int n = s.n, D = s.D;
  if (n < 1 || n > HP_MAX_L || !(D == 32 || D == 64 || D == 128)) return B2B_EUNSUPPORTED;
  const int dir = s.layers[0].inverse ? 1 : 0;  // all layers forward, or all inverse (application order)
  for (int l = 0; l < n; ++l)
    if (s.layers[l].kind != B2B_PLANAR || (s.layers[l].inverse ? 1 : 0) != dir) return B2B_EUNSUPPORTED;
  bool want = false;
  for (int k = 0; k < 4 * n; ++k) want = want || s.bars[k];
  float *wbar = nullptr, *ubar = nullptr, *bbar = nullptr;
  const size_t r64 = ((size_t)n * D + 63) & ~(size_t)63;
  if (want && s.scratch) {
    wbar = s.scratch;
    ubar = s.scratch + r64;
    bbar = s.scratch + 2 * r64;
  } else if (want) {
    wbar = s.bars[0];
    ubar = s.bars[1];
    bbar = s.bars[2];
  }
  B2BChainParams p;
  memset(&p, 0, sizeof(p));
  p.x = s.x;
  p.N = s.N;
  p.ldx = s.ldx;
  p.D = D;
  p.L = n;
  for (int l = 0; l < n; ++l) p.layers[l] = s.layers[l];
  const float* ybar = s.ybar;
  const long long ldyb = s.ldyb;
  float* xbar = s.xbar;
  int Lp = 1;
  while (Lp < n) Lp <<= 1;
  B2BChainParams q = p;  // main kernel: x -> (fragment 1), ybar -> (fragment 2), xbar out, ljbar read-only
  q.L = 0;
  q.scratch_off = -1;
  q.y = xbar;
  q.ldy = s.ldxb;
  q.logjac = const_cast<float*>(s.ljbar);
  q.accumulate = 3;  // read ljbar, never write it
  q.partials = nullptr;
  if (v1_check_io(q) != 0) return B2B_EUNSUPPORTED;
  if ((ldyb % 4) || (reinterpret_cast<uintptr_t>(ybar) & 15) || !xbar) return B2B_EUNSUPPORTED;
  // the parameter pass re-reads x AND ybar after the main kernel has written xbar: xbar must not overlap either
  if (want) {
    auto overlaps = [&](const float* a, long long lda, const float* b, long long ldb) {
      const char* a0 = reinterpret_cast<const char*>(a);
      const char* a1 = a0 + ((size_t)(p.N - 1) * (size_t)lda + (size_t)D) * sizeof(float);
      const char* b0 = reinterpret_cast<const char*>(b);
      const char* b1 = b0 + ((size_t)(p.N - 1) * (size_t)ldb + (size_t)D) * sizeof(float);
      return a0 < b1 && b0 < a1;
    };
    if (overlaps(xbar, s.ldxb, ybar, ldyb) || overlaps(xbar, s.ldxb, p.x, p.ldx)) return B2B_EINVAL;
  }
  if (!s.workspace || s.workspace_bytes < b2b_planar_vjp_workspace(n, D, p.N)) return B2B_EWORKSPACE;
  const VjpWs ws = vjp_carve(b2b_align256(s.workspace), Lp, D, p.N);
  const cudaStream_t stream = s.stream;

  V1Geom g;
  // D = 128 x 8 layers: two-tensor slots are 32 KB; 7 warps leave room for 3 of them (8 warps: 2)
  int rc = v1_geometry(D, p.N, D == 128 && Lp == 8 ? 7 : hp_warps(D), 32, (size_t)((2 * Lp * D + 2 * Lp + 3) & ~3), g, 2);
  if (rc != 0) return rc;
  CUtensorMap mx, mxb, myb;
  if (!make_maps(q, g.cols, &mx, &mxb, &g.extra.tma3d)) return B2B_EUNSUPPORTED;
  if (!make_map(&myb, ybar, D, p.N, ldyb, g.cols, g.extra.tma3d != 0)) return B2B_EUNSUPPORTED;
  if (D == 128) rc = dispatch_vjp_main<128, 8, 7>(dir, Lp, q, g, mx, myb, mxb, ws.scal, n, stream);
  else if (D == 64) rc = dispatch_vjp_main<64, 12>(dir, Lp, q, g, mx, myb, mxb, ws.scal, n, stream);
  else rc = dispatch_vjp_main<32, 16>(dir, Lp, q, g, mx, myb, mxb, ws.scal, n, stream);
  if (rc != B2B_OK) return rc;
  ++*s.launches;
  if (!want) return B2B_OK;
  // parameter gradients: skinny reductions over the ORIGINAL x and ybar
  planar_prep_kernel<<<1, HP_MAX_L * 32, 0, stream>>>(p, n, Lp, ws.packed);  // w | û | c | b for the finalize kernel
  if (D == 128) rc = launch_pgrad<128>(Lp, p.x, ybar, ws.scal, p.N, p.ldx, ldyb, ws.pg_partials, stream);
  else if (D == 64) rc = launch_pgrad<64>(Lp, p.x, ybar, ws.scal, p.N, p.ldx, ldyb, ws.pg_partials, stream);
  else rc = launch_pgrad<32>(Lp, p.x, ybar, ws.scal, p.N, p.ldx, ldyb, ws.pg_partials, stream);
  if (rc != B2B_OK) return rc;
  planar_psum_kernel<<<(2 * Lp * D + 7) / 8, 256, 0, stream>>>(ws.pg_partials, VJP_PG_GRID, 2 * Lp * D, ws.A);
  rc = launch_sstat(Lp, ws.scal, p.N, ws.ss_partials, stream);
  if (rc != B2B_OK) return rc;
  const int ns = Lp * Lp + 2 * Lp;
  planar_psum_kernel<<<(ns + 7) / 8, 256, 0, stream>>>(ws.ss_partials, VJP_SS_GRID, ns, ws.SS);
  planar_vjp_finalize_kernel<<<n, 256, 0, stream>>>(p, n, Lp, dir, ws.packed, ws.A, ws.SS, wbar, ubar, bbar);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  *s.launches += 6;
  if (!s.scratch) return B2B_OK;
  const float* const base[3] = {wbar, ubar, bbar};
  const size_t step[3] = {(size_t)D, (size_t)D, 1};
  return b2b_copy_run_bars(s.layers, n, s.bars, base, step, D, s.launches, stream);
}
