// Chains of <= 8 PlanarLayers as ONE program on the TMA pipeline (b2b_v1_pipeline.cuh).
//
// Why: the layer interpreter (b2b_chain_v1.cu) pays for a switch on the layer kind and a generic fragment mapping on the
// 8-layer D = 128 headline chain; specialising the program on (D, direction) and keeping every parameter in shared
// memory (warp-uniform LDS.128 broadcasts) removes that overhead.
// The layers run in a ROLLED loop; only the per-layer body (the D/4-step dot product and the û·t update) is unrolled.
// On sm_90 every float2 FMA is two scalar FFMAs, so one unrolled D = 128 layer is ~400 instructions (6.3 KB): eight of
// them made a ~56 KB hot loop that did not stay in the instruction cache and left the fused chain well below the HBM
// rate of a one-layer launch.  The rolled loop is one layer body (~1.9 K instructions for the whole kernel), costs a
// handful of instructions per layer for the run-time parameter offsets, and does the same float operations in the same
// order, so the results are bit-identical to the unrolled program.  The layer count is a run-time argument: one kernel
// per (D, direction[, MvNormal]) serves every L in 1..8.
// Parameter sources:
//   device-resident parameters (DevSrc, every b2b_chain_run_f32 segment made of PlanarLayers): each CTA derives û /
//       wᵀû in its prologue into shared memory -- one launch, no library-owned device state;
//   host-resident parameters (ArgSrc, b2b_planar_chain_hostparams_f32): derived on the host, passed BY VALUE as a kernel
//       argument block and copied into shared memory by every CTA in its prologue.
// A __constant__ slot filled per call from device parameters (prep kernel + copy) is not used: the extra
// launch + copy-engine hop costs more per call than constant operands could gain over shared-memory ones.
//
// Reference semantics: planar_layer.jl:65-80 (get_u_hat, forward), :102-110 (logabsdetjac), :112-127 + :160-185
// (inverse through find_alpha).
#include "b2b_planar_common.cuh"

namespace b2b {

// host-derived parameters of up to HP_MAX_L layers, packed for the launch's layer count L: w[L][D] | û[L][D] | c[L] | b[L]
template <int D>
struct PlanarHP {
  float v[2 * HP_MAX_L * D + 2 * HP_MAX_L];
};

template <int D>
struct ArgSrc {
  static constexpr bool kDerive = false;
  const PlanarHP<D>& H;
  int invmask;
  __device__ __forceinline__ bool inv(int l) const { return (invmask >> l) & 1; }
};

// Device-resident parameters: the kernel derives û / wᵀû itself (get_u_hat, planar_layer.jl:65-70, one warp per layer
// in the prologue of every CTA) into shared memory.
struct DevSrc {
  static constexpr bool kDerive = true;
  int invmask;
  __device__ __forceinline__ bool inv(int l) const { return (invmask >> l) & 1; }
};

// DIR 0: every layer forward, 1: every layer inverse, 2: per-layer direction from the mask.  Carrying the (unused)
// root-finder of the other direction in the forward program costs instruction-cache space, so the pure directions get
// their own kernels.
// MVN: the chain ends in the base MvNormal log-density (descriptor P.layers[L]): logpdf(td, y).
// Shared memory: w[L][D] | û[L][D] | c[L] | b[L] (| MvNormal μ, 1/σ, const) (| root tables of the inverse layers).
template <int D, int DIR, bool MVN, class Src>
struct PlanarProg {
  using State = V1NoState;
  const Src src;
  const B2BChainParams& P;
  const int L;  // layers of the program
  static constexpr bool DERIVE = Src::kDerive;
  // device-resident parameters, inverse layers: per-layer lookup tables of the root (find_alpha_tab)
  static constexpr bool TAB = DERIVE && DIR != 0;
  __device__ __forceinline__ int npk() const { return 2 * L * D + 2 * L; }
  __device__ __forceinline__ int mvn_off() const { return (npk() + 3) & ~3; }
  __device__ __forceinline__ int tab_off() const { return mvn_off() + (MVN ? 2 * D + 4 : 0); }

  __device__ __forceinline__ void stage(float* params, int warp, int lane, int nw) const {
    if constexpr (DERIVE) {
      if (MVN && warp == nw - 1) stage_layer(P.layers[L], params + mvn_off(), D, D, lane);
      planar_derive_smem<D>(P, L, L, params, warp, lane, nw);
      if constexpr (TAB) {
        __syncthreads();  // wᵀû of every layer is in shared memory
        for (int idx = warp * 32 + lane; idx < L * PT_N; idx += nw * 32) {
          const int l = idx / PT_N;
          if (DIR == 1 || src.inv(l)) planar_table_piece(params[2 * L * D + l], idx - l * PT_N, params + tab_off() + l * PT_FLOATS);
        }
      }
    } else {
      for (int i = warp * 32 + lane; i < npk(); i += nw * 32) params[i] = src.H.v[i];
    }
  }

  __device__ __forceinline__ void apply(float2 (&x)[1][D / 2], const ColCtx<D, 1>& ctx, const float* params,
                                        float (&lj)[1]) const {
    const float* cb = params + 2 * L * D;  // c[L] | b[L]
    const float* tab = params + tab_off();
#pragma unroll 1
    for (int l = 0; l < L; ++l) {
      const float4* w4 = reinterpret_cast<const float4*>(params + l * D);
      const float4* u4 = reinterpret_cast<const float4*>(params + (L + l) * D);
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
      const float wz = s.x + s.y;  // aT_b(w, z), utils.jl:2
      const float cc_ = cb[l], bb = cb[L + l];
      float t, s2;
      if (DIR == 0 || (DIR == 2 && !src.inv(l))) {
        tanh_sech2(wz + bb, t, s2);
        lj[0] += log1pf(cc_ * s2);  // planar_layer.jl:107
      } else {
        // planar_layer.jl:121; t = tanh(α+b), s2 = sech²(α+b)
        if constexpr (TAB) find_alpha_tab(wz, cc_, bb, tab + l * PT_FLOATS, t, s2);
        else find_alpha_ts(wz, cc_, bb, t, s2);
        lj[0] -= log1pf(cc_ * s2);
        t = -t;
      }
      const float2 t2 = make_float2(t, t);
#pragma unroll
      for (int i = 0; i < D / 4; ++i) {
        const float4 u = u4[i];
        x[0][2 * i] = b2b_ffma2(make_float2(u.x, u.y), t2, x[0][2 * i]);  // planar_layer.jl:78 / :124
        x[0][2 * i + 1] = b2b_ffma2(make_float2(u.z, u.w), t2, x[0][2 * i + 1]);
      }
    }
    if (MVN) mvnormal_apply<D, 1, 1>(x, ctx, params + mvn_off(), lj);
  }
};

template <int D, int NW, int DIR>
__global__ void __launch_bounds__(NW * 32, 1)
    planar_arg_kernel(const __grid_constant__ B2BChainParams P, const __grid_constant__ V1Extra E,
                      const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                      const __grid_constant__ PlanarHP<D> H, const int L, const int invmask) {
  const PlanarProg<D, DIR, false, ArgSrc<D>> prog{{H, invmask}, P, L};
  v1_run<D, 1, 1, NW>(P, E, map_x, map_y, prog);
}

template <int D, int NW, int DIR, bool MVN>
__global__ void __launch_bounds__(NW * 32, 1)
    planar_dev_kernel(const __grid_constant__ B2BChainParams P, const __grid_constant__ V1Extra E,
                      const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y,
                      const int L, const int invmask) {
  const PlanarProg<D, DIR, MVN, DevSrc> prog{{invmask}, P, L};
  v1_run<D, 1, 1, NW>(P, E, map_x, map_y, prog);
}

// ---- host side -----------------------------------------------------------------------------------------
template <int D, int NW, int DIR>
static int launch_arg(const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx, const CUtensorMap& my, int L,
                      const float* packed, int invmask, cudaStream_t stream) {
  static PlanarHP<D> H;  // copied into the launch's argument buffer by <<<>>>
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  memcpy(H.v, packed, sizeof(float) * (size_t)(2 * L * D + 2 * L));
  auto kernel = planar_arg_kernel<D, NW, DIR>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<g.grid, NW * 32, g.smem, stream>>>(q, g.extra, mx, my, H, L, invmask);
  return (int)cudaGetLastError();
}

template <int D, int NW, int DIR, bool MVN = false>
static int launch_dev(const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx, const CUtensorMap& my, int L,
                      int invmask, cudaStream_t stream) {
  auto kernel = planar_dev_kernel<D, NW, DIR, MVN>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<g.grid, NW * 32, g.smem, stream>>>(q, g.extra, mx, my, L, invmask);
  return (int)cudaGetLastError();
}

// dispatch over (DIR, MVN); `packed` != NULL: host-resident parameters
template <int D, int NW>
static int dispatch(int L, const B2BChainParams& q, const V1Geom& g, const CUtensorMap& mx, const CUtensorMap& my,
                    const float* packed, int invmask, bool mvn, cudaStream_t stream) {
  const int all = (1 << L) - 1;
  const int dir = (invmask & all) == 0 ? 0 : ((invmask & all) == all ? 1 : 2);
  if (packed) {
    if (dir == 0) return launch_arg<D, NW, 0>(q, g, mx, my, L, packed, invmask, stream);
    if (dir == 1) return launch_arg<D, NW, 1>(q, g, mx, my, L, packed, invmask, stream);
    return launch_arg<D, NW, 2>(q, g, mx, my, L, packed, invmask, stream);
  }
  if (mvn) {  // terminal MvNormal: all-inverse chains only (= logpdf(td, y))
    if (dir == 1) return launch_dev<D, NW, 1, true>(q, g, mx, my, L, invmask, stream);
    return B2B_EUNSUPPORTED;
  }
  if (dir == 0) return launch_dev<D, NW, 0>(q, g, mx, my, L, invmask, stream);
  if (dir == 1) return launch_dev<D, NW, 1>(q, g, mx, my, L, invmask, stream);
  return launch_dev<D, NW, 2>(q, g, mx, my, L, invmask, stream);
}

// `packed` != NULL: host-resident parameters of L layers, packed for L (kernel argument, staged into shared memory);
// NULL: device-resident (p.layers[0..L), derived in the kernel; p.layers[L] = terminal MvNormal when `mvn`).
static int launch_planar(const B2BChainParams& p, int L, const float* packed, int invmask, bool mvn,
                                  cudaStream_t stream) {
  B2BChainParams q = p;
  q.scratch_off = -1;
  if (!(q.D == 32 || q.D == 64 || q.D == 128) || L < 1 || L > HP_MAX_L) return B2B_EUNSUPPORTED;
  if (v1_check_io(q) != 0) return B2B_EUNSUPPORTED;
  V1Geom g;
  // shared memory: the packed parameter block (+ MvNormal) (+ root lookup tables of the inverse layers, device-resident
  // parameters only)
  const size_t pf = (size_t)((2 * L * q.D + 2 * L + 3) & ~3) + (mvn ? 2 * q.D + 4 : 0) +
                    ((!packed && invmask != 0) ? (size_t)L * PT_FLOATS : 0);
  const int rc = v1_geometry(q.D, q.N, hp_warps(q.D), 32, pf, g);
  if (rc != 0) return rc;
  CUtensorMap mx, my;
  if (!make_maps(q, g.cols, &mx, &my, &g.extra.tma3d)) return B2B_EUNSUPPORTED;
  if (q.D == 128) return dispatch<128, 8>(L, q, g, mx, my, packed, invmask, mvn, stream);
  if (q.D == 64) return dispatch<64, 12>(L, q, g, mx, my, packed, invmask, mvn, stream);
  return dispatch<32, 16>(L, q, g, mx, my, packed, invmask, mvn, stream);
}

}  // namespace b2b

int b2b_planar_const_grid_size(const B2BChainParams& p) {
  using namespace b2b;
  if (!(p.D == 32 || p.D == 64 || p.D == 128)) return 0;
  V1Geom g;
  if (v1_geometry(p.D, p.N, hp_warps(p.D), 32, 0, g) != 0) return 0;
  return g.grid;
}

// `L` (1..8; the host pads to 1, 2, 4 or 8) planar layers, derived parameters packed for (D, L) in HOST memory -> kernel
// argument
int b2b_launch_planar_hostparams(const B2BChainParams& p, int L, const float* packed, int invmask,
                                 cudaStream_t stream) {
  return b2b::launch_planar(p, L, packed, invmask, false, stream);
}

// Applicability of the planar chain kernels to a fusable segment: 1..8 PlanarLayers, optionally followed by the
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

// One launch of the planar chain kernel with in-kernel parameter derivation.  B2B_EUNSUPPORTED when not applicable.
int b2b_launch_planar_chain_const(const B2BChainParams& p, cudaStream_t stream) {
  using namespace b2b;
  const int n = b2b_planar_const_layers(p);
  if (n == 0) return B2B_EUNSUPPORTED;
  int invmask = 0;
  for (int l = 0; l < n; ++l)
    if (p.layers[l].inverse) invmask |= 1 << l;
  return launch_planar(p, n, nullptr, invmask, p.L > n, stream);
}
