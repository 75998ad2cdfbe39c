// Sampling path: rand(rng, td, n) of the reference (src/transformed_distribution.jl:212-224) = base samples pushed
// through the FORWARD chain.  The reference draws the base samples on the host and maps the transform over the columns;
// here the normals are generated INSIDE the chain kernel (Philox4x32-10 + Box-Muller in the tile loop of the
// thread-per-column pipeline, b2b_v1_pipeline.cuh), so the D x N matrix of base samples never exists in HBM and a
// sampling pass moves 4·(D+1) B/sample (the store) instead of 4·(3D+1).
//   b2b_randn_f32        : the generator alone (any D, any ld) -- also the first pass of chains the fused kernel
//                          does not cover (coupling layers, Permute, D not in {32, 64, 128, 256})
//   b2b_chain_sample_f32 : generator + chain
// The stream is a pure function of (seed, offset, global column, row): see V1Gen.
#include "b2b_chain_v1_prog.cuh"

int b2b_v1_plan(B2BChainParams& p, b2b::V1Geom& g, int* shape);

namespace b2b {

// one thread per (column, group of four rows)
__global__ void __launch_bounds__(256) randn_kernel(float* __restrict__ z, const V1Gen g, int D, long long N, long long ld) {
  const int Dc = (D + 3) >> 2;
  const long long total = N * Dc;
  const bool vec = (D % 4 == 0) && (ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(z) & 15) == 0);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / Dc;
    const int k = (int)(i - n * Dc);
    float4 v = philox_normal4(g, g.col0 + n, k);
    float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int r = 4 * k + q;
      if (r < D) {
        if (g.sigma) e[q] *= g.sigma[r];
        if (g.mu) e[q] += g.mu[r];
      }
    }
    float* dst = z + n * ld + 4 * k;
    if (vec) {
      *reinterpret_cast<float4*>(dst) = make_float4(e[0], e[1], e[2], e[3]);
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (4 * k + q < D) dst[q] = e[q];
    }
  }
}

template <int D, int TPC, int CPT, int NW>
__global__ void __launch_bounds__(NW * 32, 1)
    chain_sample_kernel(const __grid_constant__ B2BChainParams P, const __grid_constant__ V1Extra E,
                        const __grid_constant__ CUtensorMap map_y, const __grid_constant__ V1Gen G) {
  const InterpProg<D, TPC, CPT> prog{P};
  v1_run<D, TPC, CPT, NW, InterpProg<D, TPC, CPT>, 1, true>(P, E, map_y, map_y, prog, nullptr, &G);
}

template <int D, int TPC, int CPT, int NW>
static int launch_sample(const B2BChainParams& q, const V1Geom& g, const CUtensorMap& my, const V1Gen& gen, cudaStream_t stream) {
  auto kernel = chain_sample_kernel<D, TPC, CPT, NW>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<g.grid, NW * 32, g.smem, stream>>>(q, g.extra, my, gen);
  return (int)cudaGetLastError();
}

}  // namespace b2b

static bool fusable_kind(int kind) {
  return kind == B2B_PLANAR || kind == B2B_RADIAL || kind == B2B_RQS || kind == B2B_BATCHNORM || kind == B2B_STACKED_EW;
}

extern "C" int b2b_randn_f32(float* z, const float* mu, const float* sigma, uint64_t seed, uint64_t offset,
                             int64_t column_offset, int32_t D, int64_t N, int64_t ld, void* stream_) {
  using namespace b2b;
  if (D < 1 || N < 0 || ld < D) return B2B_EINVAL;
  if (N == 0) return B2B_OK;
  if (!z) return B2B_EINVAL;
  V1Gen g{seed, offset, column_offset, mu, sigma};
  const long long total = N * ((D + 3) / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  randn_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream_)>>>(z, g, D, N, ld);
  return (int)cudaGetLastError();
}

extern "C" int b2b_chain_sample_f32(const b2b_layer_desc* layers, int32_t L, const float* mu, const float* sigma,
                                    uint64_t seed, uint64_t offset, int64_t column_offset, float* y, float* logjac,
                                    int32_t D, int64_t N, int64_t ldy, void* workspace, size_t workspace_bytes,
                                    void* stream_) {
  using namespace b2b;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (L < 0 || L > B2B_MAX_CHAIN || (L > 0 && !layers) || D < 1 || N < 0 || ldy < D) return B2B_EINVAL;
  if (N == 0) return B2B_OK;
  if (!y) return B2B_EINVAL;
  if (L == 0) {
    if (logjac) {
      cudaError_t e = cudaMemsetAsync(logjac, 0, (size_t)N * sizeof(float), stream);
      if (e != cudaSuccess) return (int)e;
    }
    return b2b_randn_f32(y, mu, sigma, seed, offset, column_offset, D, N, ldy, stream_);
  }
  // fused: one launch when the whole chain is column-local and the thread-per-column pipeline covers D
  bool fused = (D % 4 == 0) && (!mu || (reinterpret_cast<uintptr_t>(mu) & 15) == 0) &&
               (!sigma || (reinterpret_cast<uintptr_t>(sigma) & 15) == 0);
  for (int l = 0; l < L && fused; ++l) fused = fusable_kind(layers[l].kind);
  if (fused) {
    B2BChainParams p;
    memset(&p, 0, sizeof(p));
    p.x = y;  // geometry / alignment checks only: the sampling kernel never reads x
    p.y = y;
    p.logjac = logjac;
    p.N = N;
    p.ldx = ldy;
    p.ldy = ldy;
    p.D = D;
    p.L = L;
    for (int l = 0; l < L; ++l) p.layers[l] = layers[l];
    V1Geom g;
    int shape = 0;
    if (b2b_v1_plan(p, g, &shape) == 0) {
      CUtensorMap mx, my;
      if (make_maps(p, g.cols, &mx, &my, &g.extra.tma3d)) {
        V1Gen gen{seed, offset, column_offset, mu, sigma};
        switch (shape) {
          case 2564112: return launch_sample<256, 4, 1, 12>(p, g, my, gen, stream);
          case 1281108: return launch_sample<128, 1, 1, 8>(p, g, my, gen, stream);
          case 1282112: return launch_sample<128, 2, 1, 12>(p, g, my, gen, stream);
          case 641112: return launch_sample<64, 1, 1, 12>(p, g, my, gen, stream);
          case 321116: return launch_sample<32, 1, 1, 16>(p, g, my, gen, stream);
          default: break;  // experimental shapes (B2B_V1_CFG): two passes below
        }
      }
    }
  }
  // two passes: base samples into y, then the chain in place
  int rc = b2b_randn_f32(y, mu, sigma, seed, offset, column_offset, D, N, ldy, stream_);
  if (rc != B2B_OK) return rc;
  return b2b_chain_run_f32(layers, L, y, y, logjac, nullptr, D, N, ldy, ldy, 0, workspace, workspace_bytes, stream_);
}
