// Float64 evaluation of the same chains (include/b2b.h: b2b_chain_run_f64), including the full-covariance terminal
// MVNORMAL_TRIL up to D = 2048 (its factor read through L2).
//
// The reference is generic in its element type and its own tests run in Float64 (e.g. the find_alpha residual grid with
// atol = 1e-14, test/normalising_flows.jl:47-71); this kernel is the device counterpart for those element types.  It is a
// plain, layer-by-layer restatement in double precision -- one warp per column, the column staged in shared memory,
// lanes over rows, row reductions by warp shuffles -- NOT a tuned kernel: Float64 batches are a correctness path, the
// Float32 kernels are the hot path.  Every layer kind of the Float32 path is
// covered, including affine coupling (a per-column matrix-vector product) and the terminal MvNormal.  The per-layer
// arithmetic (f64_layer_forward) lives in b2b_f64_device.cuh, which the reverse mode (b2b_chain_vjp_f64.cu) shares.
//
// Reference semantics: planar_layer.jl:65-127,160-185; radial_layer.jl:36-129; rational_quadratic_spline.jl:183-220,
// 317-357; coupling.jl:206-228; normalise.jl:61-86; permute.jl:152-155; stacked.jl:157-166; transformed_distribution.jl:165-169.
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_f64_device.cuh"

namespace b2b {

constexpr int F64_WARPS = 4;

struct F64Params {
  const double* x;
  double* y;
  double* logjac;
  double* partials;
  long long N, ldx, ldy;
  int D, L, accumulate;
  b2b_layer_desc_f64 layers[B2B_MAX_CHAIN];
};

// TRI: the chain holds a SCALE_TRIANGULAR layer, LU: a SCALE_LU layer (f64_layer_forward<TRI, LU>)
template <bool TRI, bool LU>
__global__ void __launch_bounds__(F64_WARPS * 32) chain_f64_kernel(const __grid_constant__ F64Params P) {
  extern __shared__ double sm64[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, D = P.D;
  double* col = sm64 + (size_t)warp * 2 * D;  // the column
  double* tmp = col + D;                       // scratch (permute, coupling)
  double dsum = 0.0;
  for (long long n = (long long)blockIdx.x * F64_WARPS + warp; n < P.N; n += (long long)gridDim.x * F64_WARPS) {
    for (int i = lane; i < D; i += 32) col[i] = P.x[n * P.ldx + i];
    double lj = (P.accumulate && P.logjac) ? P.logjac[n] : 0.0;
    __syncwarp();
    for (int l = 0; l < P.L; ++l) f64_layer_forward<TRI, LU>(P.layers[l], D, lane, col, tmp, lj);
    if (P.y)
      for (int i = lane; i < D; i += 32) P.y[n * P.ldy + i] = col[i];
    if (lane == 0) {
      if (P.logjac) P.logjac[n] = lj;
      dsum += lj;
    }
    __syncwarp();
  }
  if (P.partials) {
    __shared__ double red[F64_WARPS];
    if (lane == 0) red[warp] = dsum;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < F64_WARPS; ++w) t += red[w];
      P.partials[blockIdx.x] = t;
    }
  }
}

}  // namespace b2b

int b2b_f64_validate_layer(const b2b_layer_desc_f64& d, int D, bool last) {
  const B2BKind* k = b2b_kind(d.kind);
  if (k && !k->f64) return B2B_EUNSUPPORTED;  // Float32 only (include/b2b.h)
  return b2b_check_desc(d, D, last);
}

extern "C" size_t b2b_chain_workspace_bytes_f64(int32_t L, int want_sum) { return (L > 0 && want_sum) ? 4096 * sizeof(double) : 0; }

extern "C" int b2b_chain_run_f64(const b2b_layer_desc_f64* layers, int32_t L, const double* x, double* y, double* logjac,
                                 double* sum_out, int32_t D, int64_t N, int64_t ldx, int64_t ldy, int accumulate_logjac,
                                 void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b2b;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!layers || L < 1 || L > B2B_MAX_CHAIN || D < 1 || N < 0 || ldx < D) return B2B_EINVAL;
  if (D > 2048) return B2B_EUNSUPPORTED;
  if (N == 0) {
    if (sum_out) return (int)cudaMemsetAsync(sum_out, 0, sizeof(double), stream);
    return B2B_OK;
  }
  if (!x || (y && ldy < D) || (!y && !logjac && !sum_out)) return B2B_EINVAL;
  F64Params P;
  memset(&P, 0, sizeof(P));
  for (int l = 0; l < L; ++l) {
    const int rc = b2b_f64_validate_layer(layers[l], D, l == L - 1);
    if (rc != B2B_OK) return rc;
    P.layers[l] = layers[l];
  }
  if (sum_out && !logjac && !b2b_ends_in_terminal(layers, L)) return B2B_EINVAL;
  P.x = x;
  P.y = y;
  P.logjac = logjac;
  P.N = N;
  P.ldx = ldx;
  P.ldy = y ? ldy : D;
  P.D = D;
  P.L = L;
  P.accumulate = accumulate_logjac ? 1 : 0;
  long long grid = (N + F64_WARPS - 1) / F64_WARPS;
  if (grid > 132 * 8) grid = 132 * 8;
  if (sum_out) {
    if (!workspace || workspace_bytes < 4096 * sizeof(double)) return B2B_EWORKSPACE;
    P.partials = static_cast<double*>(workspace);
  }
  const size_t smem = (size_t)F64_WARPS * 2 * D * sizeof(double);
  bool tri = false, lu = false;
  for (int l = 0; l < L; ++l) {
    tri = tri || layers[l].kind == B2B_SCALE_TRIANGULAR;
    lu = lu || layers[l].kind == B2B_SCALE_LU;
  }
  const auto kernel =
      lu ? chain_f64_kernel<true, true> : tri ? chain_f64_kernel<true, false> : chain_f64_kernel<false, false>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<(int)grid, F64_WARPS * 32, smem, stream>>>(P);
  e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  if (sum_out) return b2b_launch_sum_partials(P.partials, (int)grid, sum_out, stream);
  return B2B_OK;
}
