// v0 fused column-local chain kernel: "lane group per column", direct coalesced global loads.
//
// Mapping: a column (one sample, D contiguous floats) is owned by a group of G lanes; lane j of the group
// holds the float4 chunks {v*G + j : v < V}.  A warp processes CPW = (32/G)*C columns per iteration
// (C columns per group, all loads issued before any use, so >= 4 KB are in flight per warp).  Every layer
// of the chain is applied to the register-resident fragments; the column is read ONCE and written ONCE
// for the whole fused run, and the per-column log|det J| is accumulated in a register.
//
// Row reductions (Planar dot, Radial norm, RQS / Stacked / MvNormal sums) for the C columns of a group
// are done together by a transposing butterfly: after log2(C) halving exchanges each lane owns ONE
// column's partial, so the C reductions cost C-1 + log2(G/C) shuffles instead of C*log2(G), and the
// per-column transcendental work (tanh, log1p, the find_alpha root-find) runs once per column per
// G/C lanes instead of once per lane.  The owner's scalar is broadcast back with one shuffle per column.
//
// Reference semantics: SURVEY.md §8(a) rows a3-a10, a13-a17 (file:line cited at each op).
#include <cuda_runtime.h>

#include "b2b_device.cuh"

namespace b2b {

template <int G, int C>
struct Own {
  // column (0..C-1) owned by lane j of a group after the transposing reduction
  static __device__ __forceinline__ int col(int j) {
    int own = 0;
#pragma unroll
    for (int half = C >> 1, off = G >> 1; half >= 1; half >>= 1, off >>= 1) own += (j & off) ? half : 0;
    return own;
  }
  // first lane (relative to the group) that owns column c
  static __device__ __forceinline__ int src(int c) {
    int s = 0;
#pragma unroll
    for (int half = C >> 1, off = G >> 1; half >= 1; half >>= 1, off >>= 1) s += (c & half) ? off : 0;
    return s;
  }
};

// Reduce p[0..C) over the G lanes of the group; returns the total of column Own::col(j).
template <int G, int C>
__device__ __forceinline__ float reduce_cols(float (&p)[C], int j) {
  int off = G >> 1;
#pragma unroll
  for (int half = C >> 1; half >= 1; half >>= 1) {
    const bool up = (j & off) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const float send = up ? p[i] : p[i + half];
      const float keep = up ? p[i + half] : p[i];
      p[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
    off >>= 1;
  }
  float v = p[0];
#pragma unroll
  for (; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

template <int G, int C>
__device__ __forceinline__ float bcast_col(float v, int c, int lane) {
  return __shfl_sync(0xffffffffu, v, (lane & ~(G - 1)) | Own<G, C>::src(c));
}

__device__ __forceinline__ float dot4(const float4& a, const float4& b, float acc) {
  acc = fmaf(a.x, b.x, acc);
  acc = fmaf(a.y, b.y, acc);
  acc = fmaf(a.z, b.z, acc);
  return fmaf(a.w, b.w, acc);
}

template <int G, int V, int C, bool VEC>
__global__ void __launch_bounds__(256) chain_v0_kernel(const __grid_constant__ B2BChainParams P) {
  constexpr int NG = 32 / G;
  constexpr int CPW = NG * C;
  constexpr int Dp = 4 * G * V;
  extern __shared__ float4 smem4[];
  float* sm = reinterpret_cast<float*>(smem4);

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int l = 0; l < P.L; ++l)  // RQS tables: all threads (see stage_rqs_cta)
    if (P.layers[l].kind == B2B_RQS) stage_rqs_cta(P.layers[l], sm + P.soff[l], P.D, Dp, threadIdx.x, blockDim.x);
  for (int l = warp; l < P.L; l += nwarps)
    if (P.layers[l].kind != B2B_RQS) stage_layer(P.layers[l], sm + P.soff[l], P.D, Dp, lane);
  __syncthreads();

  const int j = lane & (G - 1), gi = lane / G;
  const int own = Own<G, C>::col(j);
  const bool writer = (j & (G / C - 1)) == 0;
  const int D = P.D;
  const long long nIter = (P.N + CPW - 1) / CPW;
  const long long gw = (long long)blockIdx.x * nwarps + warp;
  const long long stride = (long long)gridDim.x * nwarps;
  float* scratch = P.scratch_off >= 0 ? sm + P.scratch_off + (size_t)warp * CPW * Dp : nullptr;
  double dsum = 0.0;

  for (long long it = gw; it < nIter; it += stride) {
    const long long base = it * CPW;
    float4 xr[C][V];
    // ---- load: all C*V requests of the lane are issued back to back ---------------------------------
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const long long col = base + c * NG + gi;
      const float* xc = P.x + col * P.ldx;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int vi = v * G + j;
        float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
        if (col < P.N) {
          if (VEC) {
            if (4 * vi < D) r = __ldcs(reinterpret_cast<const float4*>(xc) + vi);
          } else {
            const int r0 = 4 * vi;
            if (r0 + 0 < D) r.x = xc[r0 + 0];
            if (r0 + 1 < D) r.y = xc[r0 + 1];
            if (r0 + 2 < D) r.z = xc[r0 + 2];
            if (r0 + 3 < D) r.w = xc[r0 + 3];
          }
        }
        xr[c][v] = r;
      }
    }
    const long long col_own = base + own * NG + gi;
    float lj = (P.accumulate && P.logjac && col_own < P.N) ? P.logjac[col_own] : 0.0f;

    // ---- the layer program -----------------------------------------------------------------------
#pragma unroll 1
    for (int l = 0; l < P.L; ++l) {
      const b2b_layer_desc& d = P.layers[l];
      const float* sp = sm + P.soff[l];
      switch (d.kind) {
        case B2B_PLANAR: {
          // planar_layer.jl:73-80,102-110 (fwd); :112-127 (inverse)
          const float4* w4 = reinterpret_cast<const float4*>(sp);
          const float4* u4 = reinterpret_cast<const float4*>(sp + Dp);
          const float cc = sp[2 * Dp], bb = sp[2 * Dp + 1];
          float p[C];
#pragma unroll
          for (int c = 0; c < C; ++c) {
            float a = 0.f;
#pragma unroll
            for (int v = 0; v < V; ++v) a = dot4(xr[c][v], w4[v * G + j], a);
            p[c] = a;
          }
          const float wz = reduce_cols<G, C>(p, j);  // aT_b(w, z), utils.jl:2
          float t, s2;
          if (!d.inverse) {
            tanh_sech2(wz + bb, t, s2);
            lj += log1pf(cc * s2);  // :107
          } else {
            find_alpha_ts(wz, cc, bb, t, s2);  // :121; t = tanh(α+b), s2 = sech²(α+b)
            lj -= log1pf(cc * s2);  // interface.jl:276-281 with wᵀz + b = α + b
            t = -t;
          }
#pragma unroll
          for (int c = 0; c < C; ++c) {
            const float tc = bcast_col<G, C>(t, c, lane);
#pragma unroll
            for (int v = 0; v < V; ++v) {
              const float4 u = u4[v * G + j];
              xr[c][v].x = fmaf(u.x, tc, xr[c][v].x);  // z .+ û .* tanh.(…), :78 / y .- û .* tanh.(…), :124
              xr[c][v].y = fmaf(u.y, tc, xr[c][v].y);
              xr[c][v].z = fmaf(u.z, tc, xr[c][v].z);
              xr[c][v].w = fmaf(u.w, tc, xr[c][v].w);
            }
          }
        } break;
        case B2B_RADIAL: {
          // radial_layer.jl:43-53,58-72 (fwd); :88-102,124-129 (inverse)
          const float4* z4 = reinterpret_cast<const float4*>(sp);
          const float alpha = sp[Dp], bhat = sp[Dp + 1], apb = sp[Dp + 2];
          float p[C];
#pragma unroll
          for (int c = 0; c < C; ++c) {
            float a = 0.f;
#pragma unroll
            for (int v = 0; v < V; ++v) {
              const float4 z0 = z4[v * G + j];
              const float dx = xr[c][v].x - z0.x, dy = xr[c][v].y - z0.y, dz = xr[c][v].z - z0.z,
                          dw = xr[c][v].w - z0.w;
              a = fmaf(dx, dx, a);
              a = fmaf(dy, dy, a);
              a = fmaf(dz, dz, a);
              a = fmaf(dw, dw, a);
            }
            p[c] = a;
          }
          const float nrm = sqrtf(reduce_cols<G, C>(p, j));  // r (fwd, :49) or γ (inverse, :125)
          float g;   // fwd: x += g·(x − z0);  inverse: x = z0 + ρ·(x − z0) = x + (ρ−1)(x − z0)
          float r = nrm;
          if (d.inverse) {
            const float a = apb - nrm;                                      // :126
            const float sq = sqrtf(fmaf(a, a, 4.0f * alpha * nrm));
            r = a > 0.f ? (2.0f * alpha * nrm) / (sq + a) : 0.5f * (sq - a);  // :127 (stable form)
          }
          const float h = 1.0f / (alpha + r);  // h(α, r), :36
          const float bh = bhat * h;
          // (d−1)·log(1+β̂h) + log(1 + β̂h − β̂h²r),  1 − hr = αh   (:68-70)
          const float ljf = (float)(D - 1) * log1pf(bh) + log1pf(bh * alpha * h);
          if (!d.inverse) {
            g = bh;
            lj += ljf;
          } else {
            g = (alpha + r) / (apb + r) - 1.0f;  // γ of :96 minus one
            lj -= ljf;
          }
#pragma unroll
          for (int c = 0; c < C; ++c) {
            const float gc = bcast_col<G, C>(g, c, lane);
#pragma unroll
            for (int v = 0; v < V; ++v) {
              const float4 z0 = z4[v * G + j];
              xr[c][v].x = fmaf(gc, xr[c][v].x - z0.x, xr[c][v].x);
              xr[c][v].y = fmaf(gc, xr[c][v].y - z0.y, xr[c][v].y);
              xr[c][v].z = fmaf(gc, xr[c][v].z - z0.z, xr[c][v].z);
              xr[c][v].w = fmaf(gc, xr[c][v].w - z0.w, xr[c][v].w);
            }
          }
        } break;
        case B2B_BATCHNORM: {
          // normalise.jl:61-67 (fwd), :76-85 (inverse); eval mode, constants folded at staging time
          const float4* A4 = reinterpret_cast<const float4*>(sp + (d.inverse ? 2 * Dp : 0));
          const float4* C4 = reinterpret_cast<const float4*>(sp + (d.inverse ? 3 * Dp : Dp));
          const float ljc = sp[4 * Dp];
#pragma unroll
          for (int v = 0; v < V; ++v) {
            const float4 A = A4[v * G + j], K = C4[v * G + j];
#pragma unroll
            for (int c = 0; c < C; ++c) {
              xr[c][v].x = fmaf(xr[c][v].x, A.x, K.x);
              xr[c][v].y = fmaf(xr[c][v].y, A.y, K.y);
              xr[c][v].z = fmaf(xr[c][v].z, A.z, K.z);
              xr[c][v].w = fmaf(xr[c][v].w, A.w, K.w);
            }
          }
          lj += d.inverse ? -ljc : ljc;
        } break;
        case B2B_RQS: {
          const int K1 = d.n0, KP = rqs_kp(K1);
          float p[C];
#pragma unroll
          for (int c = 0; c < C; ++c) {
            float acc = 0.f;
#pragma unroll
            for (int v = 0; v < V; ++v) {
              const int r0 = 4 * (v * G + j);
              float* e = reinterpret_cast<float*>(&xr[c][v]);
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                float o = e[q], l1 = 0.f;
                if (d.inverse) rqs_element<true>(sp, K1, KP, Dp, r0 + q, e[q], o, l1);
                else rqs_element<false>(sp, K1, KP, Dp, r0 + q, e[q], o, l1);
                e[q] = o;
                acc += l1;
              }
            }
            p[c] = acc;
          }
          lj += reduce_cols<G, C>(p, j);  // sum over dimensions, :304-309
        } break;
        case B2B_ELEMENTWISE_VEC:  // staged as the STACKED_EW table
        case B2B_STACKED_EW: {
          // stacked.jl:157-166,242-252 with elementwise blocks (exp_log.jl, shift.jl, scale.jl)
          const int* code = reinterpret_cast<const int*>(sp);
          const float* av = sp + Dp;
          float p[C];
#pragma unroll
          for (int c = 0; c < C; ++c) p[c] = 0.f;
#pragma unroll
          for (int v = 0; v < V; ++v) {
            const int r0 = 4 * (v * G + j);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int op = code[r0 + q];
              const float a = av[r0 + q], b = av[Dp + r0 + q];
#pragma unroll
              for (int c = 0; c < C; ++c) {
                float* e = reinterpret_cast<float*>(&xr[c][v]);
                e[q] = ew_apply(op, d.inverse != 0, a, b, e[q], p[c]);
              }
            }
          }
          lj += reduce_cols<G, C>(p, j);
        } break;
        case B2B_PERMUTE: {
          // permute.jl:152 (A*x as index movement; bit-exact), logjac 0 (:155)
          const int* src = reinterpret_cast<const int*>(sp);
          __syncwarp();
#pragma unroll
          for (int c = 0; c < C; ++c)
#pragma unroll
            for (int v = 0; v < V; ++v)
              reinterpret_cast<float4*>(scratch + (size_t)(c * NG + gi) * Dp)[v * G + j] = xr[c][v];
          __syncwarp();
#pragma unroll
          for (int c = 0; c < C; ++c) {
            const float* sc = scratch + (size_t)(c * NG + gi) * Dp;
#pragma unroll
            for (int v = 0; v < V; ++v) {
              const int r0 = 4 * (v * G + j);
              xr[c][v] = make_float4(sc[src[r0]], sc[src[r0 + 1]], sc[src[r0 + 2]], sc[src[r0 + 3]]);
            }
          }
        } break;
        case B2B_MVNORMAL_DIAG: {
          // logpdf(MvNormal(μ, Diagonal(σ²)), x) + logjac  (transformed_distribution.jl:168)
          const float4* mu4 = reinterpret_cast<const float4*>(sp);
          const float4* is4 = reinterpret_cast<const float4*>(sp + Dp);
          const float cst = sp[2 * Dp];
          float p[C];
#pragma unroll
          for (int c = 0; c < C; ++c) {
            float a = 0.f;
#pragma unroll
            for (int v = 0; v < V; ++v) {
              const float4 mu = mu4[v * G + j], is = is4[v * G + j];
              const float zx = (xr[c][v].x - mu.x) * is.x, zy = (xr[c][v].y - mu.y) * is.y,
                          zz = (xr[c][v].z - mu.z) * is.z, zw = (xr[c][v].w - mu.w) * is.w;
              a = fmaf(zx, zx, a);
              a = fmaf(zy, zy, a);
              a = fmaf(zz, zz, a);
              a = fmaf(zw, zw, a);
            }
            p[c] = a;
          }
          lj += cst - 0.5f * reduce_cols<G, C>(p, j);
        } break;
        default: break;
      }
    }

    // ---- store ---------------------------------------------------------------------------------------
    if (P.y) {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const long long col = base + c * NG + gi;
        if (col < P.N) {
          float* yc = P.y + col * P.ldy;
#pragma unroll
          for (int v = 0; v < V; ++v) {
            const int vi = v * G + j;
            if (VEC) {
              if (4 * vi < D) __stcs(reinterpret_cast<float4*>(yc) + vi, xr[c][v]);
            } else {
              const int r0 = 4 * vi;
              if (r0 + 0 < D) yc[r0 + 0] = xr[c][v].x;
              if (r0 + 1 < D) yc[r0 + 1] = xr[c][v].y;
              if (r0 + 2 < D) yc[r0 + 2] = xr[c][v].z;
              if (r0 + 3 < D) yc[r0 + 3] = xr[c][v].w;
            }
          }
        }
      }
    }
    if (writer && col_own < P.N) {
      if (P.logjac) P.logjac[col_own] = lj;
      dsum += (double)lj;
    }
  }

  if (P.partials) {
    __shared__ double red[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
    if (lane == 0) red[warp] = dsum;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < nwarps; ++w) t += red[w];
      P.partials[blockIdx.x] = t;
    }
  }
}

__global__ void sum_partials_kernel(const double* __restrict__ partials, int n, double* __restrict__ out) {
  // single warp, fixed order: deterministic
  double t = 0.0;
  for (int i = threadIdx.x; i < n; i += 32) t += partials[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if (threadIdx.x == 0) *out = t;
}

struct V0Config {
  int G, V, C;
};

static V0Config pick_config(int D) {
  const int nvec = (D + 3) / 4;
  if (nvec <= 8) return {8, 1, 8};
  if (nvec <= 16) return {16, 1, 8};
  if (nvec <= 32) return {32, 1, 8};
  if (nvec <= 64) return {32, 2, 4};
  if (nvec <= 128) return {32, 4, 2};
  return {32, 8, 1};
}

typedef void (*v0_kernel_t)(const B2BChainParams);

template <bool VEC>
static v0_kernel_t pick_kernel(const V0Config& c) {
  if (c.G == 8) return chain_v0_kernel<8, 1, 8, VEC>;
  if (c.G == 16) return chain_v0_kernel<16, 1, 8, VEC>;
  if (c.V == 1) return chain_v0_kernel<32, 1, 8, VEC>;
  if (c.V == 2) return chain_v0_kernel<32, 2, 4, VEC>;
  if (c.V == 4) return chain_v0_kernel<32, 4, 2, VEC>;
  return chain_v0_kernel<32, 8, 1, VEC>;
}

struct V0Plan {
  v0_kernel_t kernel;
  int grid, block;
  size_t smem;
  int Dp, cpw;
  bool ok;
};

constexpr int V0_BLOCK = 256;

// Shared-memory layout of a v0 launch: every layer's derived parameters at padded depth Dp (soff[l], when given), then
// the per-warp permute scratch (*scratch_off, -1 when no layer permutes).  Returns the floats staged.
static size_t v0_layout(const b2b_layer_desc* layers, int L, int D, int* soff, int* scratch_off) {
  const V0Config cfg = pick_config(D);
  const int Dp = 4 * cfg.G * cfg.V;
  const int cpw = (32 / cfg.G) * cfg.C;
  size_t off = 0;
  bool need_scratch = false;
  for (int l = 0; l < L; ++l) {
    if (soff) soff[l] = (int)off;
    off += (b2b_layer_smem_floats(layers[l], Dp) + 3) & ~3;
    if (layers[l].kind == B2B_PERMUTE) need_scratch = true;
  }
  if (scratch_off) *scratch_off = need_scratch ? (int)off : -1;
  if (need_scratch) off += (size_t)(V0_BLOCK / 32) * cpw * Dp;
  return off;
}

static int plan_v0(B2BChainParams& p, V0Plan& plan) {
  if (p.D < 1 || p.D > 1024) return B2B_EUNSUPPORTED;
  const V0Config cfg = pick_config(p.D);
  const int Dp = 4 * cfg.G * cfg.V;
  const int cpw = (32 / cfg.G) * cfg.C;
  const bool vec = (p.D % 4 == 0) && (p.ldx % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.x) & 15) == 0) &&
                   (!p.y || ((p.ldy % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.y) & 15) == 0)));
  plan.kernel = vec ? pick_kernel<true>(cfg) : pick_kernel<false>(cfg);
  plan.block = V0_BLOCK;
  plan.smem = v0_layout(p.layers, p.L, p.D, p.soff, &p.scratch_off) * sizeof(float);
  if (plan.smem > B2B_V0_SMEM_MAX) return B2B_EUNSUPPORTED;
  plan.Dp = Dp;
  plan.cpw = cpw;
  cudaError_t e = cudaSuccess;
  if (plan.smem > 48 * 1024)
    e = cudaFuncSetAttribute(plan.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem);
  if (e != cudaSuccess) return (int)e;
  const int sms = b2b_sm_count();
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, plan.kernel, plan.block, plan.smem);
  if (e != cudaSuccess) return (int)e;
  if (per_sm < 1) per_sm = 1;
  const long long n_iter = (p.N + cpw - 1) / cpw;
  const long long want = (n_iter + (plan.block / 32) - 1) / (plan.block / 32);
  long long grid = (long long)sms * per_sm;
  if (grid > want) grid = want;
  if (grid < 1) grid = 1;
  plan.grid = (int)grid;
  return 0;
}

}  // namespace b2b

size_t b2b_chain_v0_smem_bytes(const b2b_layer_desc* layers, int L, int D) {
  if (D < 1 || D > 1024) return SIZE_MAX;
  return b2b::v0_layout(layers, L, D, nullptr, nullptr) * sizeof(float);
}

int b2b_chain_grid_size_v0(const B2BChainParams& p) {
  B2BChainParams q = p;
  b2b::V0Plan plan;
  if (b2b::plan_v0(q, plan) != 0) return 0;
  return plan.grid;
}

int b2b_launch_chain_v0(const B2BChainParams& p, cudaStream_t stream) {
  B2BChainParams q = p;
  b2b::V0Plan plan;
  const int rc = b2b::plan_v0(q, plan);
  if (rc != 0) return rc;
  plan.kernel<<<plan.grid, plan.block, plan.smem, stream>>>(q);
  return (int)cudaGetLastError();
}

int b2b_launch_sum_partials(const double* partials, int n, double* sum_out, cudaStream_t stream) {
  b2b::sum_partials_kernel<<<1, 32, 0, stream>>>(partials, n, sum_out);
  return (int)cudaGetLastError();
}
