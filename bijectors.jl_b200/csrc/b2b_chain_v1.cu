// v1 fused column-local chain kernel: TMA-staged, THREAD-PER-COLUMN.
//
// Why: in the v0 (lane-group) kernel an 8-layer chain costs ~250 warp-instructions per column (cross-lane
// reductions, selects, broadcasts, redundant transcendental work) and the kernel is issue-bound well below
// the HBM roofline.  Here one thread owns one whole column in registers, so a row reduction is a private
// FFMA chain (no shuffles), per-column scalars (tanh, log1p, find_alpha) are computed exactly once, and
// every layer parameter read is a warp-uniform shared-memory broadcast.
//
// (For D >= 128 a column is split over TPC = 2 or 4 adjacent lanes -- 64 rows each -- so that 16 warps fit
// in the register file; the only cross-lane traffic is one or two shuffles per row reduction.)
//
// Data movement: the D x N batch is described by a 2-D TMA tensor map {D, N}.  A tile is 32/TPC columns;
// it is fetched as D/32 boxes of {32 floats, 32/TPC columns} with the 128-byte swizzle, i.e. box q holds rows
// [32q, 32q+32) of the tile's columns, one column per 128-byte line, and the 16-byte chunk k of line t lives
// at chunk slot k ^ (t & 7).  A thread therefore reads its rows with conflict-free LDS.128
// (the 8 lanes of a quarter-warp hit 8 different 16-byte bank groups) while the register <-> row mapping
// stays identical in all lanes (so parameters are warp-uniform).  Results go back through a per-warp
// staging buffer in the same layout and a TMA store.
//
// Pipeline (persistent CTA, one per SM): tiles j = 0,1,2,... of a CTA are consumed round-robin by its NW
// warps; tile j lands in input buffer j % P.  The warp that consumed tile j copies it to registers and
// IMMEDIATELY re-arms the same buffer with the load of tile j + P (its lane 0 issues the TMA), so P tiles
// (P*16 KB at D=128) are always in flight per SM with no producer warp and no empty-barriers: refills of a
// buffer are ordered by the consumption of its previous tile.
//
// Reference semantics per layer: see b2b_chain_v0.cu / b2b_device.cuh (file:line cited there).
#include "b2b_chain_v1_prog.cuh"

namespace b2b {

template <int D, int TPC, int CPT, int NW>
__global__ void __launch_bounds__(NW * 32, 1)
    chain_v1_kernel(const __grid_constant__ B2BChainParams P, const __grid_constant__ V1Extra E,
                    const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y) {
  const InterpProg<D, TPC, CPT> prog{P};
  v1_run<D, TPC, CPT, NW>(P, E, map_x, map_y, prog);
}

typedef void (*v1_kernel_t)(const B2BChainParams, const V1Extra, const CUtensorMap, const CUtensorMap);

struct V1Plan : V1Geom {
  v1_kernel_t kernel;
  int shape;  // which <D, TPC, CPT, NW> instantiation: D * 10000 + TPC * 1000 + CPT * 100 + NW
};

static int plan_v1(B2BChainParams& p, V1Plan& plan) {
  const int D = p.D;
  if (!(D == 32 || D == 64 || D == 128 || D == 256)) return B2B_EUNSUPPORTED;
  if (v1_check_io(p) != 0) return B2B_EUNSUPPORTED;
  int off = 0;
  for (int l = 0; l < p.L; ++l) {
    const int k = p.layers[l].kind;
    if (k == B2B_PERMUTE || k == B2B_COUPLING_AFFINE) return B2B_EUNSUPPORTED;
    p.soff[l] = off;
    off += (b2b_layer_smem_floats(p.layers[l], D) + 3) & ~3;
  }
  p.scratch_off = -1;
  bool per_row = false;  // RQS / Stacked are unrolled per row: only built for <= 64 rows per thread
  for (int l = 0; l < p.L; ++l) per_row |= p.layers[l].kind == B2B_RQS || p.layers[l].kind == B2B_STACKED_EW;
  // <D, lanes per column, columns per thread, warps>: warps are chosen so that the per-thread register budget
  // (65536 / threads) holds the fragment without spilling: 64 data registers need ~170 (12 warps), 128 need 255
  // (8 warps), 32 fit in 128 (16 warps).  B2B_V1_CFG selects alternative builds for experiments.
  static const int cfg = getenv("B2B_V1_CFG") ? atoi(getenv("B2B_V1_CFG")) : 0;
  int nw, tpc, cpt = 1;
  if (D == 256) { plan.kernel = chain_v1_kernel<256, 4, 1, 12>; nw = 12; tpc = 4; }
  else if (D == 128) {
    // default: one thread per column.  Chains with per-row layers
    // (RQS, Stacked) use two lanes per column.  B2B_V1_CFG=2218 selects the build with two lanes per column and
    // TWO columns per thread (every parameter load serves two columns: LDS wavefronts -36 %, but more scalar work
    // per warp), 2112 the 2-lane / 12-warp build.
    if (cfg == 2218 && !per_row) { plan.kernel = chain_v1_kernel<128, 2, 2, 8>; nw = 8; tpc = 2; cpt = 2; }
    else if (cfg == 2112 || per_row) { plan.kernel = chain_v1_kernel<128, 2, 1, 12>; nw = 12; tpc = 2; }
    else { plan.kernel = chain_v1_kernel<128, 1, 1, 8>; nw = 8; tpc = 1; }
  }
  else if (D == 64) {
    if (cfg == 1128 && !per_row) { plan.kernel = chain_v1_kernel<64, 1, 2, 8>; nw = 8; tpc = 1; cpt = 2; }
    else { plan.kernel = chain_v1_kernel<64, 1, 1, 12>; nw = 12; tpc = 1; }
  }
  else { plan.kernel = chain_v1_kernel<32, 1, 1, 16>; nw = 16; tpc = 1; }
  plan.shape = D * 10000 + tpc * 1000 + cpt * 100 + nw;
  return v1_geometry(D, p.N, nw, (32 / tpc) * cpt, (size_t)off, plan);
}

}  // namespace b2b

// geometry + staged-parameter offsets of the interpreter launch for `p` (shared with the sampling kernels of
// b2b_sample.cu, which instantiate the same program with a generator in place of the input ring)
int b2b_v1_plan(B2BChainParams& p, b2b::V1Geom& g, int* shape) {
  b2b::V1Plan plan;
  const int rc = b2b::plan_v1(p, plan);
  if (rc != 0) return rc;
  g = plan;
  *shape = plan.shape;
  return 0;
}

int b2b_chain_grid_size_v1(const B2BChainParams& p) {
  B2BChainParams q = p;
  b2b::V1Plan plan;
  if (b2b::plan_v1(q, plan) != 0) return 0;
  return plan.grid;
}

int b2b_launch_chain_v1(const B2BChainParams& p, cudaStream_t stream) {
  using namespace b2b;
  B2BChainParams q = p;
  V1Plan plan;
  const int rc = plan_v1(q, plan);
  if (rc != 0) return rc;
  CUtensorMap mx, my;
  if (!make_maps(q, plan.cols, &mx, &my, &plan.extra.tma3d)) return B2B_EUNSUPPORTED;
  cudaError_t e = cudaFuncSetAttribute(plan.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem);
  if (e != cudaSuccess) return (int)e;
  plan.kernel<<<plan.grid, plan.nw * 32, plan.smem, stream>>>(q, plan.extra, mx, my);
  return (int)cudaGetLastError();
}

