// Reparameterised sampling, the path variational inference trains through (ELBO / reverse KL; the reference keeps its
// non-in-place rand overloads for "differentiating sampling wrt. params of `td.dist` or params of `Bijector`",
// src/transformed_distribution.jl:210-213):
//   z ~ N(0, I) (the b2b_randn_f32 stream), x = μ + σ ⊙ z or μ + L z, y = T(x) with log-Jacobian ℓ(x),
//   log q(y) = −½‖z‖² − Σᵢ log σᵢ (or log Lᵢᵢ) − ½·D·log2π − ℓ(x).
// Reverse mode with z held fixed, given ȳ (D x N) and q̄ (N): x̄ is b2b_chain_vjp_f32 at x with l̄ = −q̄, which also
// forms every layer's cotangents; then μ̄ = Σₙ x̄ₙ and σ̄ = Σₙ x̄ₙ ⊙ zₙ − (Σₙ q̄ₙ)/σ, or L̄ = tril(Σₙ x̄ₙ zₙᵀ) −
// (Σₙ q̄ₙ)·diag(1/Lᵢᵢ).
//   b2b_chain_sample_logq_f32 : y exactly as b2b_chain_sample_f32 / _tril_f32, and log q per column.  A chain the
//                               thread-per-column pipeline fuses stays ONE launch (the LOGQ instantiation of v1_run);
//                               other chains add one pass over N floats, never over D x N
//   b2b_chain_sample_vjp_f32  : x (and z for L Lᵀ) regenerated into the workspace, the chain's reverse mode, and the
//                               base cotangents from fixed column chunks reduced in order (no atomics)
#include <cstring>

#include "b2b_v1_pipeline.cuh"  // philox_normal4, V1Gen: the sampling stream of b2b_randn_f32

namespace b2b {

// −½·D·log2π − Σᵢ log σᵢ from warp 0 of the CTA (σ NULL: 1)
__device__ __forceinline__ float base_const(const float* sigma, int D, float* slot) {
  if (threadIdx.x < 32) {
    float ls = 0.f;
    if (sigma)
      for (int i = threadIdx.x; i < D; i += 32) ls += logf(__ldg(sigma + i));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ls += __shfl_xor_sync(0xffffffffu, ls, o);
    if (threadIdx.x == 0) *slot = -0.5f * (D * 1.8378770664093453f) - ls;
  }
  __syncthreads();
  return *slot;
}

// two-pass chains: logq[n] := base(zₙ) − logq[n] (logq holds ℓ) or base(zₙ) (L = 0), zₙ regenerated per column
__global__ void __launch_bounds__(256) logq_finish_kernel(float* __restrict__ logq, const V1Gen g, int D, long long N,
                                                          bool have_lj) {
  __shared__ float c0s;
  const float c0 = base_const(g.sigma, D, &c0s);
  for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += (long long)gridDim.x * blockDim.x) {
    float q = 0.f;
    for (int k = 0; 4 * k < D; ++k) {
      const float4 z = philox_normal4(g, g.col0 + n, k);
      const float e[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (4 * k + i < D) q = fmaf(e[i], e[i], q);
    }
    const float b = fmaf(-0.5f, q, c0);
    logq[n] = have_lj ? b - logq[n] : b;
  }
}

__global__ void __launch_bounds__(256) negate_kernel(const float* src, float* dst, long long N) {
  for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += (long long)gridDim.x * blockDim.x)
    dst[n] = -src[n];
}

// *out = Σₙ q[n] in fp64, one CTA in a fixed order
__global__ void __launch_bounds__(1024) qsum_kernel(const float* __restrict__ q, long long N, double* out) {
  __shared__ double red[1024];
  double s = 0.0;
  for (long long n = threadIdx.x; n < N; n += 1024) s += (double)q[n];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = red[0];
}

// Diagonal base: CTA (p, b) sums chunk p (kBaseChunk columns) for rows 128b .. 128b+127: 32 lanes of four rows (one
// philox_normal4 each, the rows of one counter) x 8 column lanes.  part[p] = [Σ x̄ (D) | Σ x̄ ⊙ z (D)], fp64.
constexpr int kBaseChunk = 4096;

__global__ void __launch_bounds__(256) diag_base_partials_kernel(const float* __restrict__ xbar, long long ldxb,
                                                                 const V1Gen g, int D, long long N,
                                                                 double* __restrict__ part) {
  __shared__ double red[2][8][128];
  const int tq = threadIdx.x & 31, tc = threadIdx.x >> 5;
  const int k = blockIdx.y * 32 + tq;
  const long long p = blockIdx.x, n0 = p * kBaseChunk, n1 = n0 + kBaseChunk < N ? n0 + kBaseChunk : N;
  double sx[4] = {0.0, 0.0, 0.0, 0.0}, sxz[4] = {0.0, 0.0, 0.0, 0.0};
  if (xbar && 4 * k < D) {
    for (long long n = n0 + tc; n < n1; n += 8) {
      const float4 z = philox_normal4(g, g.col0 + n, k);
      const float ze[4] = {z.x, z.y, z.z, z.w};
      const float* xc = xbar + n * ldxb + 4 * k;
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (4 * k + i < D) {
          const double xb = (double)xc[i];
          sx[i] += xb;
          sxz[i] = fma(xb, (double)ze[i], sxz[i]);
        }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    red[0][tc][4 * tq + i] = sx[i];
    red[1][tc][4 * tq + i] = sxz[i];
  }
  __syncthreads();
  const int which = threadIdx.x >> 7, rr = threadIdx.x & 127, row = blockIdx.y * 128 + rr;
  if (row < D) {
    double s = 0.0;
    for (int c = 0; c < 8; ++c) s += red[which][c][rr];
    part[((size_t)p * 2 + which) * D + row] = s;
  }
}

// μ̄, σ̄ from the chunk partials, in chunk order
__global__ void __launch_bounds__(256) diag_base_finalize_kernel(const double* __restrict__ part, long long P,
                                                                 const double* qsum, const float* __restrict__ sigma,
                                                                 float* __restrict__ mubar, float* __restrict__ sigmabar,
                                                                 int D) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= D) return;
  if (mubar) {
    double s = 0.0;
    for (long long p = 0; p < P; ++p) s += part[(size_t)p * 2 * D + row];
    mubar[row] = (float)s;
  }
  if (sigmabar) {
    double s = 0.0;
    for (long long p = 0; p < P; ++p) s += part[((size_t)p * 2 + 1) * D + row];
    if (qsum) s -= *qsum / (double)__ldg(sigma + row);
    sigmabar[row] = (float)s;
  }
}

}  // namespace b2b

namespace {

size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

int grid_1d(long long n) {
  long long b = (n + 255) / 256;
  if (b > 132 * 16) b = 132 * 16;
  return (int)(b > 0 ? b : 1);
}

// Every refusal of both entry points, before anything is launched: the base (B2B_EINVAL for another kind), the chain
// (what b2b_chain_vjp_f32 returns for it; no MvNormal terminal inside), and D for a TRIL base
int rs_check(const b2b_layer_desc* layers, int32_t L, const b2b_layer_desc* base, int32_t D, int64_t N) {
  if (L < 0 || L > B2B_MAX_CHAIN || (L > 0 && !layers) || !base || D < 1 || N < 0) return B2B_EINVAL;
  if (base->kind != B2B_MVNORMAL_DIAG && base->kind != B2B_MVNORMAL_TRIL) return B2B_EINVAL;
  int rc = b2b_check_desc(*base, D, true);
  if (rc != B2B_OK) return rc;
  for (int l = 0; l < L; ++l) {
    const B2BKind* k = b2b_kind(layers[l].kind);
    if (k && k->terminal) return B2B_EINVAL;
  }
  if (L > 0 && (rc = b2b_chain_vjp_check_f32(layers, L, D)) != B2B_OK) return rc;
  if (base->kind == B2B_MVNORMAL_TRIL && D > B2B_TRIL_MAX_D) return B2B_EUNSUPPORTED;
  return B2B_OK;
}

// workspace of b2b_chain_sample_vjp_f32: [x, then z][x̄][−q̄][Σ q̄][base partials][chain VJP], each 256-aligned.  The
// chain reads x (L > 0) and the TRIL base reads z after it: they share one D x N buffer, reserved only when one of them
// is used; x̄ has its own only when the chain forms it or a TRIL base may need zeros in its place
struct RsLayout {
  size_t xz, xbar, nq, qsum, base, chain, total;
};

RsLayout rs_layout(const b2b_layer_desc* layers, int L, const b2b_layer_desc* base, int D, long long N) {
  RsLayout v{};
  const bool tril = base->kind == B2B_MVNORMAL_TRIL;
  const size_t m = al256((size_t)D * (size_t)N * sizeof(float));
  v.xz = L > 0 || tril ? m : 0;
  v.xbar = L > 0 || tril ? m : 0;
  v.nq = L > 0 ? al256((size_t)N * sizeof(float)) : 0;
  v.qsum = 256;
  const long long P = (N + b2b::kBaseChunk - 1) / b2b::kBaseChunk;
  v.base = tril ? b2b_tril_base_vjp_workspace(D, N) : al256((size_t)P * 2 * D * sizeof(double));
  v.chain = L > 0 ? al256(b2b_chain_vjp_workspace_bytes(layers, L, D, N)) : 0;
  v.total = v.xz + v.xbar + v.nq + v.qsum + v.base + v.chain + 256;
  return v;
}

}  // namespace

extern "C" size_t b2b_chain_sample_logq_workspace_bytes(const b2b_layer_desc* layers, int32_t L,
                                                        const b2b_layer_desc* base, int32_t D, int64_t N) {
  if (rs_check(layers, L, base, D, N) != B2B_OK) return 0;
  return (L > 0 ? b2b_chain_workspace_bytes(layers, L, D, N, 1, 0) : 0) + 256;
}

extern "C" int b2b_chain_sample_logq_f32(const b2b_layer_desc* layers, int32_t L, const b2b_layer_desc* base,
                                         uint64_t seed, uint64_t offset, int64_t column_offset, float* y, float* logq,
                                         int32_t D, int64_t N, int64_t ldy, void* workspace, size_t workspace_bytes,
                                         void* stream_) {
  using namespace b2b;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  b2b_set_last_launch_count(0);
  int rc = rs_check(layers, L, base, D, N);
  if (rc != B2B_OK) return rc;
  if (ldy < D) return B2B_EINVAL;
  if (N == 0) return B2B_OK;
  if (!y || !logq) return B2B_EINVAL;
  const float* mu = base->p0;
  int launches = 0;
  if (base->kind == B2B_MVNORMAL_TRIL) {
    // the sample launch writes the base term (negated when the chain's ℓ is added to it in place, then negated back)
    if ((rc = b2b_tril_sample(base->p1, mu, seed, offset, column_offset, y, ldy, logq, L > 0 ? -1.f : 1.f, D, N,
                              stream)) != B2B_OK)
      return rc;
    ++launches;
    if (L > 0) {
      rc = b2b_chain_run_f32(layers, L, y, y, logq, nullptr, D, N, ldy, ldy, 1, workspace, workspace_bytes, stream_);
      if (rc != B2B_OK) return rc;
      launches += b2b_last_launch_count();
      negate_kernel<<<grid_1d(N), 256, 0, stream>>>(logq, logq, N);
      if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
      ++launches;
    }
    b2b_set_last_launch_count(launches);
    return B2B_OK;
  }
  const float* sigma = base->p1;
  const V1Gen gen{seed, offset, column_offset, mu, sigma};
  // fused: one launch, the decision and geometry of b2b_chain_sample_f32
  bool launched = false;
  rc = b2b_launch_sample_fused(layers, L, mu, sigma, seed, offset, column_offset, y, logq, D, N, ldy, true, &launched,
                               stream);
  if (launched) {
    if (rc == B2B_OK) b2b_set_last_launch_count(1);
    return rc;
  }
  // two passes: base samples into y, the chain in place writing ℓ into logq, then the base term per column
  if ((rc = b2b_randn_f32(y, mu, sigma, seed, offset, column_offset, D, N, ldy, stream_)) != B2B_OK) return rc;
  ++launches;
  if (L > 0) {
    rc = b2b_chain_run_f32(layers, L, y, y, logq, nullptr, D, N, ldy, ldy, 0, workspace, workspace_bytes, stream_);
    if (rc != B2B_OK) return rc;
    launches += b2b_last_launch_count();
  }
  logq_finish_kernel<<<grid_1d(N), 256, 0, stream>>>(logq, gen, D, N, L > 0);
  if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;
  b2b_set_last_launch_count(launches + 1);
  return B2B_OK;
}

extern "C" size_t b2b_chain_sample_vjp_workspace_bytes(const b2b_layer_desc* layers, int32_t L,
                                                       const b2b_layer_desc* base, int32_t D, int64_t N) {
  if (rs_check(layers, L, base, D, N) != B2B_OK) return 0;
  return rs_layout(layers, L, base, D, N).total;
}

extern "C" int b2b_chain_sample_vjp_f32(const b2b_layer_desc* layers, int32_t L, const b2b_layer_desc* base,
                                        uint64_t seed, uint64_t offset, int64_t column_offset, const float* ybar,
                                        int64_t ldybar, const float* lqbar, float* const* param_bars, int32_t D,
                                        int64_t N, void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b2b;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  b2b_set_last_launch_count(0);
  int rc = rs_check(layers, L, base, D, N);
  if (rc != B2B_OK) return rc;
  if (ybar && ldybar < D) return B2B_EINVAL;
  // [layers | base]: the slot rules of b2b_chain_vjp_f32 then cover the base's entries 4L .. 4L+3 too
  b2b_layer_desc all[B2B_MAX_CHAIN + 1];
  for (int l = 0; l < L; ++l) all[l] = layers[l];
  all[L] = *base;
  unsigned want = 0;
  if ((rc = b2b_vjp_check_slots(all, L + 1, param_bars, &want)) != B2B_OK) return rc;
  if (N == 0)  // zeroes the requested cotangents
    return b2b_vjp_check_batch(all, L + 1, param_bars, (const float*)nullptr, (const float*)nullptr, (float*)nullptr, D,
                               0, D, D, D, stream);
  if (!want) return B2B_OK;
  const RsLayout lay = rs_layout(layers, L, base, D, N);
  if (!workspace || workspace_bytes < lay.total) return B2B_EWORKSPACE;
  char* ws = b2b_align256(workspace);
  float* const x = reinterpret_cast<float*>(ws);  // x for the chain, then z for a TRIL base
  float* const z = x;
  float* const xbuf = reinterpret_cast<float*>(ws + lay.xz);
  float* const nq = reinterpret_cast<float*>(ws + lay.xz + lay.xbar);
  double* const qsum = reinterpret_cast<double*>(ws + lay.xz + lay.xbar + lay.nq);
  char* const bws = ws + lay.xz + lay.xbar + lay.nq + lay.qsum;
  char* const cws = bws + lay.base;
  const bool tril = base->kind == B2B_MVNORMAL_TRIL, want_base = (want >> L) & 1;
  int launches = 0;
#define B2B_RS_LAUNCHED()                                                     \
  do {                                                                        \
    if ((rc = (int)cudaGetLastError()) != cudaSuccess) return rc;             \
    ++launches;                                                               \
  } while (0)
  // 1. the batch the chain saw (x)
  if (L > 0) {
    rc = tril ? b2b_tril_sample(base->p1, base->p0, seed, offset, column_offset, x, D, nullptr, 0.f, D, N, stream)
              : b2b_randn_f32(x, base->p0, base->p1, seed, offset, column_offset, D, N, D, stream_);
    if (rc != B2B_OK) return rc;
    ++launches;
  }
  // 2. x̄ and the layers' cotangents: the chain's reverse mode with l̄ = −q̄ (L = 0: x̄ = ȳ)
  const float* xb = ybar;
  long long ldxb = ldybar;
  if (L > 0) {
    const float* lb = nullptr;
    if (lqbar) {
      negate_kernel<<<grid_1d(N), 256, 0, stream>>>(lqbar, nq, N);
      B2B_RS_LAUNCHED();
      lb = nq;
    }
    float* const none[4 * B2B_MAX_CHAIN] = {};
    rc = b2b_chain_vjp_f32(layers, L, x, ybar, lb, xbuf, param_bars ? param_bars : none, D, N, D, ybar ? ldybar : D, D,
                           cws, lay.chain, stream_);
    if (rc != B2B_OK) return rc;
    launches += b2b_last_launch_count();
    xb = xbuf;
    ldxb = D;
  }
  // 3. the base's cotangents
  if (want_base) {
    const double* qs = nullptr;
    if (lqbar) {
      qsum_kernel<<<1, 1024, 0, stream>>>(lqbar, N, qsum);
      B2B_RS_LAUNCHED();
      qs = qsum;
    }
    float* const mubar = param_bars[4 * L];
    float* const pbar = param_bars[4 * L + 1];
    if (tril) {
      // z where the GEMM reads it from memory, over x (the chain's reverse mode, which read x, is enqueued before it)
      if ((rc = b2b_randn_f32(z, nullptr, nullptr, seed, offset, column_offset, D, N, D, stream_)) != B2B_OK) return rc;
      ++launches;
      if (!xb) {  // ȳ = 0 and no chain: x̄ = 0
        const cudaError_t e = cudaMemsetAsync(xbuf, 0, (size_t)D * N * sizeof(float), stream);
        if (e != cudaSuccess) return (int)e;
        ++launches;
        xb = xbuf;
        ldxb = D;
      }
      if ((rc = b2b_tril_base_vjp(xb, ldxb, z, qs, base->p1, mubar, pbar, D, N, bws, &launches, stream)) != B2B_OK)
        return rc;
    } else {
      const long long P = (N + kBaseChunk - 1) / kBaseChunk;
      const V1Gen g{seed, offset, column_offset, nullptr, nullptr};
      double* const part = reinterpret_cast<double*>(bws);
      diag_base_partials_kernel<<<dim3((unsigned)P, (unsigned)((D + 127) / 128)), 256, 0, stream>>>(xb, ldxb, g, D, N,
                                                                                                    part);
      B2B_RS_LAUNCHED();
      diag_base_finalize_kernel<<<(D + 255) / 256, 256, 0, stream>>>(part, P, qs, base->p1, mubar, pbar, D);
      B2B_RS_LAUNCHED();
    }
  }
#undef B2B_RS_LAUNCHED
  b2b_set_last_launch_count(launches);
  return B2B_OK;
}
