// Chains of <= 8 PlanarLayers as ONE UNROLLED program on the TMA pipeline (b2b_v1_pipeline.cuh).
//
// Why: the layer interpreter (b2b_chain_v1.cu) pays for a rolled layer loop, a switch on the layer kind and a generic
// fragment mapping on the 8-layer D = 128 headline chain; specialising the program on (D, L, direction) and unrolling
// the layers removes that overhead.  Parameter operands:
//   device-resident parameters (DevSrc, every b2b_chain_run_f32 segment made of PlanarLayers): each CTA derives û /
//       wᵀû in its prologue into shared memory and all operands are warp-uniform LDS broadcasts -- one launch, no
//       library-owned device state;
//   host-resident parameters (ArgSrc, b2b_planar_chain_hostparams_f32): derived on the host, passed BY VALUE as kernel
//       arguments, i.e. CONSTANT-BANK operands (LDC -> FFMA operand: no LSU work).  The first-level
//       constant cache holds ~4 KB, so the 8 KB of an 8-layer D = 128 chain is split: w in shared memory, û in the
//       constant bank (MODE 2).
// A __constant__ slot filled per call from device parameters (prep kernel + copy) is not used: the extra
// launch + copy-engine hop costs more per call than constant operands gain over shared-memory ones at D >= 64.
//
// Reference semantics: planar_layer.jl:65-80 (get_u_hat, forward), :102-110 (logabsdetjac), :112-127 + :160-185
// (inverse through find_alpha).
#include "b2b_planar_common.cuh"

namespace b2b {

template <int D, int L>
struct PlanarHP {
  float v[2 * L * D + 2 * L];
};

template <int D, int L>
struct ArgSrc {
  static constexpr bool kDerive = false;
  const PlanarHP<D, L>& H;
  int invmask;
  __device__ __forceinline__ float w(int l, int i) const { return H.v[l * D + i]; }
  __device__ __forceinline__ float uh(int l, int i) const { return H.v[L * D + l * D + i]; }
  __device__ __forceinline__ float c(int l) const { return H.v[2 * L * D + l]; }
  __device__ __forceinline__ float b(int l) const { return H.v[2 * L * D + L + l]; }
  __device__ __forceinline__ bool inv(int l) const { return (invmask >> l) & 1; }
  __device__ __forceinline__ float raw(int i) const { return H.v[i]; }  // dynamic index: staging only
};

// MODE 0: w and û from the constant bank; MODE 1: û staged in shared memory (LDS broadcast), w from the constant
// bank; MODE 2: w in shared memory, û from the constant bank.
// DIR 0: every layer forward, 1: every layer inverse, 2: per-layer direction from the mask.  The unrolled program of
// 8 layers is large; carrying the (unused) root-finder of the other direction in the hot path costs a quarter of the
// forward throughput in instruction-cache misses, so the pure directions get their own kernels.
// Device-resident parameters: the kernel derives û / wᵀû itself (get_u_hat, planar_layer.jl:65-70, one warp per layer
// in the prologue of every CTA) into shared memory and runs the unrolled program on the shared-memory copy -- one
// launch, no library-owned device state.  (Measured: for the unrolled program the shared-memory operands are as fast
// as the constant-bank ones at D >= 64, and a separate preparation
// kernel + copy into a __constant__ slot costs more per call than it gains.)
template <int D, int L>
struct DevSrc {
  static constexpr bool kDerive = true;
  int invmask, nreal;
  __device__ __forceinline__ bool inv(int l) const { return (invmask >> l) & 1; }
};

// MVN: the chain ends in the base MvNormal log-density (descriptor P.layers[nreal]): logpdf(td, y).
template <int D, int L, int MODE, int DIR, bool MVN, class Src>
struct PlanarConstProg {
  using State = V1NoState;
  const Src src;
  const B2BChainParams& P;
  static constexpr bool DERIVE = Src::kDerive;
  static constexpr int NPK = 2 * L * D + 2 * L;                    // packed w | û | c | b
  static constexpr bool STAGED = MODE != 0 || DERIVE;
  static constexpr int MVN_OFF = STAGED ? ((NPK + 3) & ~3) : 0;
  // device-resident parameters, inverse layers: per-layer lookup tables of the root (find_alpha_tab)
  static constexpr bool TAB = DERIVE && DIR != 0;
  static constexpr int TAB_OFF = MVN_OFF + (MVN ? 2 * D + 4 : 0);
  static constexpr int SMEM_FLOATS = TAB_OFF + (TAB ? L * PT_FLOATS : 0);
  __device__ __forceinline__ void stage(float* params, int warp, int lane, int nw) const {
    if constexpr (DERIVE) {
      if (MVN && warp == nw - 1) stage_layer(P.layers[src.nreal], params + MVN_OFF, D, D, lane);
      planar_derive_smem<D, L>(P, src.nreal, params, warp, lane, nw);
      if constexpr (TAB) {
        __syncthreads();  // wᵀû of every layer is in shared memory
        for (int idx = warp * 32 + lane; idx < L * PT_N; idx += nw * 32) {
          const int l = idx / PT_N;
          if (DIR == 1 || src.inv(l)) planar_table_piece(params[2 * L * D + l], idx - l * PT_N, params + TAB_OFF + l * PT_FLOATS);
        }
      }
    } else if constexpr (STAGED) {
      for (int i = warp * 32 + lane; i < NPK; i += nw * 32) params[i] = src.raw(i);
    }
  }

  template <bool WS, bool US, bool SS>
  __device__ __forceinline__ void layers(float2 (&x)[1][D / 2], const float* params, float (&lj)[1]) const {
#pragma unroll
    for (int l = 0; l < L; ++l) {
      const float4* w4 = reinterpret_cast<const float4*>(params + l * D);
      const float4* u4 = reinterpret_cast<const float4*>(params + L * D + l * D);
      float2 acc[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = make_float2(0.f, 0.f);
#pragma unroll
      for (int i = 0; i < D / 4; ++i) {
        float4 w;
        if constexpr (WS) w = w4[i];
        else w = make_float4(src.w(l, 4 * i), src.w(l, 4 * i + 1), src.w(l, 4 * i + 2), src.w(l, 4 * i + 3));
        acc[(i & 1) * 2 + 0] = b2b_ffma2(make_float2(w.x, w.y), x[0][2 * i], acc[(i & 1) * 2 + 0]);
        acc[(i & 1) * 2 + 1] = b2b_ffma2(make_float2(w.z, w.w), x[0][2 * i + 1], acc[(i & 1) * 2 + 1]);
      }
      const float2 s = b2b_fadd2(b2b_fadd2(acc[0], acc[1]), b2b_fadd2(acc[2], acc[3]));
      const float wz = s.x + s.y;  // aT_b(w, z), utils.jl:2
      float cc_, bb;
      if constexpr (SS) {
        cc_ = params[2 * L * D + l];
        bb = params[2 * L * D + L + l];
      } else {
        cc_ = src.c(l);
        bb = src.b(l);
      }
      float t, s2;
      if (DIR == 0 || (DIR == 2 && !src.inv(l))) {
        tanh_sech2(wz + bb, t, s2);
        lj[0] += log1pf(cc_ * s2);  // planar_layer.jl:107
      } else {
        // planar_layer.jl:121; t = tanh(α+b), s2 = sech²(α+b)
        if constexpr (TAB) find_alpha_tab(wz, cc_, bb, params + TAB_OFF + l * PT_FLOATS, t, s2);
        else find_alpha_ts(wz, cc_, bb, t, s2);
        lj[0] -= log1pf(cc_ * s2);
        t = -t;
      }
      const float2 t2 = make_float2(t, t);
#pragma unroll
      for (int i = 0; i < D / 4; ++i) {
        float4 u;
        if constexpr (US) u = u4[i];
        else u = make_float4(src.uh(l, 4 * i), src.uh(l, 4 * i + 1), src.uh(l, 4 * i + 2), src.uh(l, 4 * i + 3));
        x[0][2 * i] = b2b_ffma2(make_float2(u.x, u.y), t2, x[0][2 * i]);  // planar_layer.jl:78 / :124
        x[0][2 * i + 1] = b2b_ffma2(make_float2(u.z, u.w), t2, x[0][2 * i + 1]);
      }
    }
  }

  __device__ __forceinline__ void apply(float2 (&x)[1][D / 2], const ColCtx<D, 1>& ctx, const float* params,
                                        float (&lj)[1]) const {
    if constexpr (DERIVE) layers<true, true, true>(x, params, lj);
    else layers<MODE == 2, MODE == 1, false>(x, params, lj);
    if (MVN) mvnormal_apply<D, 1, 1>(x, ctx, params + MVN_OFF, lj);
  }
};

template <int D, int L, int NW, int MODE, int DIR>
__global__ void __launch_bounds__(NW * 32, 1)
    planar_arg_kernel(const __grid_constant__ B2BChainParams P, const __grid_constant__ V1Extra E,
                      const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                      const __grid_constant__ PlanarHP<D, L> H, const int invmask) {
  const PlanarConstProg<D, L, MODE, DIR, false, ArgSrc<D, L>> prog{{H, invmask}, P};
  v1_run<D, 1, 1, NW>(P, E, map_x, map_y, prog);
}

template <int D, int L, int NW, int DIR, bool MVN>
__global__ void __launch_bounds__(NW * 32, 1)
    planar_dev_kernel(const __grid_constant__ B2BChainParams P, const __grid_constant__ V1Extra E,
                      const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                      const int invmask, const int nreal) {
  const PlanarConstProg<D, L, 0, DIR, MVN, DevSrc<D, L>> prog{{invmask, nreal}, P};
  v1_run<D, 1, 1, NW>(P, E, map_x, map_y, prog);
}

// ---- host side -----------------------------------------------------------------------------------------
template <int D, int L, int NW, int MODE, int DIR>
static int launch_arg(const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx, const CUtensorMap& my,
                      const float* packed, int invmask, cudaStream_t stream) {
  static PlanarHP<D, L> H;  // copied into the launch's argument buffer by <<<>>>
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  memcpy(H.v, packed, sizeof(H.v));
  auto kernel = planar_arg_kernel<D, L, NW, MODE, DIR>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<g.grid, NW * 32, g.smem, stream>>>(q, g.extra, mx, my, H, invmask);
  return (int)cudaGetLastError();
}

template <int D, int L, int NW, int DIR, bool MVN = false>
static int launch_dev(const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx, const CUtensorMap& my,
                      int nreal, int invmask, cudaStream_t stream) {
  auto kernel = planar_dev_kernel<D, L, NW, DIR, MVN>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<g.grid, NW * 32, g.smem, stream>>>(q, g.extra, mx, my, invmask, nreal);
  return (int)cudaGetLastError();
}

// ---- host-resident parameters: dispatch over (D, L, MODE, DIR) -------------------------------------------------
template <int D, int NW, int LL, int MM>
static int dispatch_arg_dir(const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx, const CUtensorMap& my,
                            const float* packed, int invmask, cudaStream_t stream) {
  const int all = (1 << LL) - 1;
  const int dir = (invmask & all) == 0 ? 0 : ((invmask & all) == all ? 1 : 2);
  if (dir == 0) return launch_arg<D, LL, NW, MM, 0>(q, g, mx, my, packed, invmask, stream);
  if (dir == 1) return launch_arg<D, LL, NW, MM, 1>(q, g, mx, my, packed, invmask, stream);
  return launch_arg<D, LL, NW, MM, 2>(q, g, mx, my, packed, invmask, stream);
}

template <int D, int NW>
static int dispatch_arg(int L, int mode, const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx,
                        const CUtensorMap& my, const float* packed, int invmask, cudaStream_t stream) {
  if (L == 1 && mode == 0) return dispatch_arg_dir<D, NW, 1, 0>(q, g, mx, my, packed, invmask, stream);
  if (L == 2 && mode == 0) return dispatch_arg_dir<D, NW, 2, 0>(q, g, mx, my, packed, invmask, stream);
  if (L == 4 && mode == 0) return dispatch_arg_dir<D, NW, 4, 0>(q, g, mx, my, packed, invmask, stream);
  if constexpr (2 * D * 8 * 4 > 4096) {
    if (L == 8 && mode == 2) return dispatch_arg_dir<D, NW, 8, 2>(q, g, mx, my, packed, invmask, stream);
  } else {
    if (L == 8 && mode == 0) return dispatch_arg_dir<D, NW, 8, 0>(q, g, mx, my, packed, invmask, stream);
  }
  return B2B_EUNSUPPORTED;
}

// ---- device-resident parameters: dispatch over (D, L, DIR, MVN) --------------------------------------------------
template <int D, int NW, int LL>
static int dispatch_dev_dir(const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx, const CUtensorMap& my,
                            int nreal, int invmask, bool mvn, cudaStream_t stream) {
  const int all = (1 << LL) - 1;
  const int dir = (invmask & all) == 0 ? 0 : ((invmask & all) == all ? 1 : 2);
  if (mvn) {  // terminal MvNormal: all-inverse chains only (= logpdf(td, y))
    if (dir == 1) return launch_dev<D, LL, NW, 1, true>(q, g, mx, my, nreal, invmask, stream);
    return B2B_EUNSUPPORTED;
  }
  if (dir == 0) return launch_dev<D, LL, NW, 0>(q, g, mx, my, nreal, invmask, stream);
  if (dir == 1) return launch_dev<D, LL, NW, 1>(q, g, mx, my, nreal, invmask, stream);
  return launch_dev<D, LL, NW, 2>(q, g, mx, my, nreal, invmask, stream);
}

template <int D, int NW>
static int dispatch_dev(int L, const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx, const CUtensorMap& my,
                        int nreal, int invmask, bool mvn, cudaStream_t stream) {
  switch (L) {
    case 1: return dispatch_dev_dir<D, NW, 1>(q, g, mx, my, nreal, invmask, mvn, stream);
    case 2: return dispatch_dev_dir<D, NW, 2>(q, g, mx, my, nreal, invmask, mvn, stream);
    case 3: return dispatch_dev_dir<D, NW, 3>(q, g, mx, my, nreal, invmask, mvn, stream);
    case 4: return dispatch_dev_dir<D, NW, 4>(q, g, mx, my, nreal, invmask, mvn, stream);
    case 5: return dispatch_dev_dir<D, NW, 5>(q, g, mx, my, nreal, invmask, mvn, stream);
    case 6: return dispatch_dev_dir<D, NW, 6>(q, g, mx, my, nreal, invmask, mvn, stream);
    case 7: return dispatch_dev_dir<D, NW, 7>(q, g, mx, my, nreal, invmask, mvn, stream);
    case 8: return dispatch_dev_dir<D, NW, 8>(q, g, mx, my, nreal, invmask, mvn, stream);
    default: return B2B_EUNSUPPORTED;
  }
}

// `packed` != NULL: host-resident parameters (kernel arguments); NULL: device-resident (p.layers[0..nreal), derived in
// the kernel; p.layers[nreal] = terminal MvNormal when `mvn`).  L = layer count of the program (host parameters: padded
// to 1, 2, 4, 8; device parameters: exact).
static int launch_planar_unrolled(const B2BChainParams& p, int L, const float* packed, int nreal, int invmask, bool mvn,
                                  cudaStream_t stream) {
  B2BChainParams q = p;
  q.scratch_off = -1;
  if (!(q.D == 32 || q.D == 64 || q.D == 128)) return B2B_EUNSUPPORTED;
  if (v1_check_io(q) != 0) return B2B_EUNSUPPORTED;
  const HPShape sh = hp_shape(q.D, L);
  V1Geom g;
  // shared memory: the packed parameter block when it is staged (MODE != 0, or device-resident parameters)
  const bool staged = sh.mode != 0 || !packed;
  const size_t pf = (staged ? (size_t)((2 * L * q.D + 2 * L + 3) & ~3) : 0) + (mvn ? 2 * q.D + 4 : 0) +
                    ((!packed && invmask != 0) ? (size_t)L * PT_FLOATS : 0);  // root lookup tables of inverse layers
  const int rc = v1_geometry(q.D, q.N, sh.nw, 32, pf, g);
  if (rc != 0) return rc;
  CUtensorMap mx, my;
  if (!make_maps(q, g.cols, &mx, &my, &g.extra.tma3d)) return B2B_EUNSUPPORTED;
  if (packed) {
    if (q.D == 128) return dispatch_arg<128, 8>(L, sh.mode, q, g, mx, my, packed, invmask, stream);
    if (q.D == 64) return dispatch_arg<64, 12>(L, sh.mode, q, g, mx, my, packed, invmask, stream);
    return dispatch_arg<32, 16>(L, sh.mode, q, g, mx, my, packed, invmask, stream);
  }
  if (q.D == 128) return dispatch_dev<128, 8>(L, q, g, mx, my, nreal, invmask, mvn, stream);
  if (q.D == 64) return dispatch_dev<64, 12>(L, q, g, mx, my, nreal, invmask, mvn, stream);
  return dispatch_dev<32, 16>(L, q, g, mx, my, nreal, invmask, mvn, stream);
}

}  // namespace b2b

int b2b_planar_const_grid_size(const B2BChainParams& p) {
  using namespace b2b;
  if (!(p.D == 32 || p.D == 64 || p.D == 128)) return 0;
  V1Geom g;
  const HPShape sh = hp_shape(p.D, 8);
  if (v1_geometry(p.D, p.N, sh.nw, 32, 0, g) != 0) return 0;
  return g.grid;
}

// `L` (1, 2, 4 or 8) planar layers, derived parameters packed for (D, L) in HOST memory -> kernel arguments
int b2b_launch_planar_hostparams(const B2BChainParams& p, int L, const float* packed, int invmask,
                                 cudaStream_t stream) {
  return b2b::launch_planar_unrolled(p, L, packed, L, invmask, false, stream);
}

// Applicability of the unrolled planar kernels to a fusable segment: 1..8 PlanarLayers, optionally followed by the
// terminal MvNormal when every planar layer is inverse (= logpdf(td, y)); D in {32,64,128}; 16-byte aligned batches.
// Returns the number of planar layers, 0 when not applicable.
int b2b_planar_const_layers(const B2BChainParams& p) {
  using namespace b2b;
  if (!(p.D == 32 || p.D == 64 || p.D == 128) || p.L < 1) return 0;
  const bool mvn = p.layers[p.L - 1].kind == B2B_MVNORMAL_DIAG;
  const int n = p.L - (mvn ? 1 : 0);
  if (n < 1 || n > HP_MAX_L) return 0;
  for (int l = 0; l < n; ++l) {
    if (p.layers[l].kind != B2B_PLANAR) return 0;
    if (mvn && !p.layers[l].inverse) return 0;
  }
  if (v1_check_io(p) != 0) return 0;
  return n;
}

// One launch of the unrolled kernel with in-kernel parameter derivation.  B2B_EUNSUPPORTED when not applicable.
int b2b_launch_planar_chain_const(const B2BChainParams& p, cudaStream_t stream) {
  using namespace b2b;
  const int n = b2b_planar_const_layers(p);
  if (n == 0) return B2B_EUNSUPPORTED;
  int invmask = 0;
  for (int l = 0; l < n; ++l)
    if (p.layers[l].inverse) invmask |= 1 << l;
  // device-resident parameters: a program of exactly n layers (every L in 1..8 is instantiated; only the host-parameter
  // family, whose programs are keyed by the packed argument block, pads to 1, 2, 4, 8)
  return launch_planar_unrolled(p, n, nullptr, n, invmask, p.L > n, stream);
}
