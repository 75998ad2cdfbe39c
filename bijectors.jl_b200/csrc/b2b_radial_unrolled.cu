// INVERSE chains of <= 8 RadialLayers as ONE UNROLLED program on the TMA pipeline, specialised on (D, L) -- the radial
// counterpart of b2b_planar_const.cu (BASELINE config 3, inverse).  The forward direction stays in the layer
// interpreter: an unrolled forward program of this shape spills at 12 warps.
// Reference semantics: radial_layer.jl:43-72 (forward), :88-102,124-129 (inverse), see radial_apply.
#include "b2b_v1_pipeline.cuh"

namespace b2b {

template <int D, int L, bool INV>
struct RadialProg {
  using State = V1NoState;
  const B2BChainParams& P;
  static constexpr int STRIDE = D + 4;  // z0[D] | α, β̂, α+β̂, -
  __device__ __forceinline__ void stage(float* params, int warp, int lane, int nw) const {
    for (int l = warp; l < L; l += nw) stage_layer(P.layers[l], params + l * STRIDE, D, D, lane);
  }
  __device__ __forceinline__ void apply(float2 (&x)[1][D / 2], const ColCtx<D, 1>& ctx, const float* params,
                                        float (&lj)[1]) const {
#pragma unroll
    for (int l = 0; l < L; ++l) radial_apply<D, 1, 1>(x, ctx, params + l * STRIDE, INV, lj);
  }
};

template <int D, int L, int NW, bool INV>
__global__ void __launch_bounds__(NW * 32, 1)
    radial_unrolled_kernel(const __grid_constant__ B2BChainParams P, const __grid_constant__ V1Extra E,
                           const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y) {
  const RadialProg<D, L, INV> prog{P};
  v1_run<D, 1, 1, NW>(P, E, map_x, map_y, prog);
}

template <int D, int L, int NW>
static int launch_radial(const B2BChainParams& q, bool inv, cudaStream_t stream) {
  V1Geom g;
  const int rc = v1_geometry(D, q.N, NW, 32, (size_t)L * (D + 4), g);
  if (rc != 0) return rc;
  CUtensorMap mx, my;
  if (!make_maps(q, g.cols, &mx, &my, &g.extra.tma3d)) return B2B_EUNSUPPORTED;
  (void)inv;
  auto kernel = radial_unrolled_kernel<D, L, NW, true>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<g.grid, NW * 32, g.smem, stream>>>(q, g.extra, mx, my);
  return (int)cudaGetLastError();
}

template <int D, int NW>
static int dispatch_radial(const B2BChainParams& q, bool inv, cudaStream_t stream) {
  switch (q.L) {
    case 1: return launch_radial<D, 1, NW>(q, inv, stream);
    case 2: return launch_radial<D, 2, NW>(q, inv, stream);
    case 3: return launch_radial<D, 3, NW>(q, inv, stream);
    case 4: return launch_radial<D, 4, NW>(q, inv, stream);
    case 5: return launch_radial<D, 5, NW>(q, inv, stream);
    case 6: return launch_radial<D, 6, NW>(q, inv, stream);
    case 7: return launch_radial<D, 7, NW>(q, inv, stream);
    case 8: return launch_radial<D, 8, NW>(q, inv, stream);
    default: return B2B_EUNSUPPORTED;
  }
}

}  // namespace b2b

// p: a segment of 1..8 INVERSE RADIAL layers, D in {32, 64, 128}
int b2b_radial_unrolled_applicable(const B2BChainParams& p) {
  if (p.L < 1 || p.L > 8 || !(p.D == 32 || p.D == 64 || p.D == 128)) return 0;
  for (int l = 0; l < p.L; ++l)
    if (p.layers[l].kind != B2B_RADIAL || !p.layers[l].inverse) return 0;
  return b2b::v1_check_io(p) == 0;
}

int b2b_launch_radial_unrolled(const B2BChainParams& p, cudaStream_t stream) {
  using namespace b2b;
  if (!b2b_radial_unrolled_applicable(p)) return B2B_EUNSUPPORTED;
  B2BChainParams q = p;
  q.scratch_off = -1;
  const bool inv = p.layers[0].inverse != 0;
  if (q.D == 128) return dispatch_radial<128, 8>(q, inv, stream);
  if (q.D == 64) return dispatch_radial<64, 12>(q, inv, stream);
  return dispatch_radial<32, 16>(q, inv, stream);
}
