// Reverse mode (vector-Jacobian product) of the affine coupling layer and of the eval-mode InvertibleBatchNorm -- the two
// layer kinds of a RealNVP flow (BASELINE config 5) -- so that such a flow can be TRAINED on the device path.
//
// Reference: what the reference's reverse-mode AD computes for Coupling (src/bijectors/coupling.jl:206-228) with the law
// Shift(t) ∘ Scale(exp.(s)), [s; t] = W·x₂ + c; the pullback of `combine` (ext/BijectorsChainRulesCoreExt.jl:48-62) is
// the row scatter of the three cotangent blocks.  Restated and finite-difference-checked in oracle/oracle_np.py
// (coupling_affine_vjp, batchnorm_eval_vjp).
//   forward : y₁ = e^s x₁ + t,  lj = Σ s        x̄₁ = e^s ȳ₁,   s̄ = ȳ₁ e^s x₁ + l̄,   t̄ = ȳ₁
//   inverse : x₁ = (y₁ − t) e^−s, lj = −Σ s     ȳ₁ = e^−s x̄₁,  s̄ = −x₁ x̄₁ − l̄,    t̄ = −e^−s x̄₁
//   both    : x̄₂ = ȳ₂ + Wᵀ[s̄; t̄],  W̄ = Σ_n [s̄; t̄]_n x₂ₙᵀ,  c̄ = Σ_n [s̄; t̄]_n,  pass-through rows x̄₃ = ȳ₃
//
// Three GEMMs of the forward's size per tile (recompute [s; t], the x̄₂ product, the W̄ outer-product accumulation) in
// exact fp32 on the CUDA cores: a persistent CTA per SM, tiles of 32 columns transposed into shared memory, the CTA's
// partial W̄ (2·n1 x n2 <= 256 x 128 floats) lives in REGISTERS for the whole launch (128 accumulators per thread) and is
// written once; a second kernel sums the per-CTA partials in a fixed order (deterministic).  Two programs: the generic one
// below (any n1, n2 <= 128, scalar loads) and the float4 / float2-pair one for n1, n2 multiples of 4.  The tensor-core (fp16-split
// wgmma) form of the forward kernel has not been carried over to the reverse mode (DESIGN §8).
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_internal.h"

namespace b2b {

constexpr int CV_TC = 32;            // columns per tile
constexpr int CV_LD = CV_TC + 1;     // padded row stride of the shared-memory tiles
constexpr int CV_THREADS = 256;

struct CvParams {
  const float* x;
  const float* ybar;
  const float* ljbar;
  float* xbar;
  const float* W;
  const float* c;
  const int32_t* idx1;
  const int32_t* idx2;
  float* part;  // per-CTA partials: [grid][2n1*n2 + 2n1]
  long long N, ldx, ldyb, ldxb;
  int D, n1, n2, row1, row2;
};

template <bool INV>
__global__ void __launch_bounds__(CV_THREADS, 1) coupling_vjp_kernel(const __grid_constant__ CvParams P) {
  extern __shared__ float smem[];
  const int D = P.D, n1 = P.n1, n2 = P.n2, m2 = 2 * n1;
  float* X = smem;                         // [D][CV_LD]   the layer's input tile
  float* YB = X + (size_t)D * CV_LD;       // [D][CV_LD]   cotangent tile, turned into the input cotangent in place
  float* SB = YB + (size_t)D * CV_LD;      // [2n1][CV_LD] s̄ | t̄
  float* LB = SB + (size_t)m2 * CV_LD;     // [CV_TC]      l̄ of the tile's columns
  int* s1 = reinterpret_cast<int*>(LB + CV_TC);  // [n1] rows of x₁
  int* s2 = s1 + n1;                              // [n2] rows of x₂
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = threadIdx.x; k < n1; k += CV_THREADS) s1[k] = P.idx1 ? P.idx1[k] : P.row1 + k;
  for (int k = threadIdx.x; k < n2; k += CV_THREADS) s2[k] = P.idx2 ? P.idx2[k] : P.row2 + k;
  const long long tiles = (P.N + CV_TC - 1) / CV_TC;
  const int ldw = m2;
  // this thread's block of the W̄ partial: rows 32·warp .. +31 (of [s̄; t̄]), columns lane + 32·q (of x₂)
  float acc[32][4];
#pragma unroll
  for (int i = 0; i < 32; ++i)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[i][q] = 0.f;
  float cacc = 0.f;  // c̄ partial of row threadIdx.x

  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long col0 = tile * CV_TC;
    __syncthreads();  // previous tile fully consumed / index lists visible
    // ---- load + transpose x and ȳ (zero-filled beyond N: such columns contribute exactly 0 to every cotangent) ----
    for (int cidx = warp; cidx < CV_TC; cidx += CV_THREADS / 32) {
      const long long col = col0 + cidx;
      const bool ok = col < P.N;
      for (int r = lane; r < D; r += 32) {
        X[r * CV_LD + cidx] = ok ? __ldcs(P.x + col * P.ldx + r) : 0.f;
        YB[r * CV_LD + cidx] = ok ? __ldcs(P.ybar + col * P.ldyb + r) : 0.f;
      }
      if (lane == 0) LB[cidx] = (ok && P.ljbar) ? P.ljbar[col] : 0.f;
    }
    __syncthreads();
    // ---- [s; t] = W·x₂ + c, then the elementwise cotangents (thread: 4 rows j, column `lane`) -------------------
    for (int jb = 4 * warp; jb < n1; jb += 4 * (CV_THREADS / 32)) {
      float sv[4] = {0.f, 0.f, 0.f, 0.f}, tv[4] = {0.f, 0.f, 0.f, 0.f};
      for (int k = 0; k < n2; ++k) {
        const float xk = X[s2[k] * CV_LD + lane];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (jb + i < n1) {
            sv[i] = fmaf(__ldg(P.W + (size_t)k * ldw + jb + i), xk, sv[i]);
            tv[i] = fmaf(__ldg(P.W + (size_t)k * ldw + n1 + jb + i), xk, tv[i]);
          }
        }
      }
      const float lb = LB[lane];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = jb + i;
        if (j >= n1) break;
        const float s_ = sv[i] + (P.c ? P.c[j] : 0.f), t_ = tv[i] + (P.c ? P.c[n1 + j] : 0.f);
        const int r1 = s1[j];
        const float in1 = X[r1 * CV_LD + lane], cb1 = YB[r1 * CV_LD + lane];
        float sbar, tbar, out1;
        if (!INV) {
          const float e = expf(s_);
          out1 = e * cb1;                 // x̄₁ = e^s ȳ₁
          sbar = fmaf(cb1 * e, in1, lb);  // ȳ₁ e^s x₁ + l̄
          tbar = cb1;
        } else {
          const float em = expf(-s_);
          const float x1 = (in1 - t_) * em;  // the recovered x₁
          out1 = em * cb1;                   // ȳ₁ = e^−s x̄₁
          sbar = -fmaf(x1, cb1, lb);         // −x₁ x̄₁ − l̄
          tbar = -out1;
        }
        YB[r1 * CV_LD + lane] = out1;
        SB[j * CV_LD + lane] = sbar;
        SB[(n1 + j) * CV_LD + lane] = tbar;
      }
    }
    __syncthreads();
    // ---- x̄₂ = ȳ₂ + Wᵀ[s̄; t̄]  (thread: 4 rows k of x₂, column `lane`) ----------------------------------------------
    for (int kb = 4 * warp; kb < n2; kb += 4 * (CV_THREADS / 32)) {
      float a[4] = {0.f, 0.f, 0.f, 0.f};
      for (int j = 0; j < m2; ++j) {
        const float sb = SB[j * CV_LD + lane];
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (kb + i < n2) a[i] = fmaf(__ldg(P.W + (size_t)(kb + i) * ldw + j), sb, a[i]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (kb + i < n2) YB[s2[kb + i] * CV_LD + lane] += a[i];
    }
    // ---- W̄ += [s̄; t̄]·x₂ᵀ over the tile's columns; c̄ += Σ columns ---------------------------------------------------
    {
      const int rbase = 32 * warp;
      if (rbase < m2) {
#pragma unroll 4
        for (int cidx = 0; cidx < CV_TC; ++cidx) {
          float b[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) b[q] = (lane + 32 * q < n2) ? X[s2[lane + 32 * q] * CV_LD + cidx] : 0.f;
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const float av = (rbase + i < m2) ? SB[(rbase + i) * CV_LD + cidx] : 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][q] = fmaf(av, b[q], acc[i][q]);
          }
        }
      }
      if ((int)threadIdx.x < m2) {
        float t = 0.f;
        for (int cidx = 0; cidx < CV_TC; ++cidx) t += SB[threadIdx.x * CV_LD + cidx];
        cacc += t;
      }
    }
    __syncthreads();  // x̄₂ complete
    // ---- write the input cotangent tile back (coalesced) ---------------------------------------------------------
    for (int cidx = warp; cidx < CV_TC; cidx += CV_THREADS / 32) {
      const long long col = col0 + cidx;
      if (col < P.N)
        for (int r = lane; r < D; r += 32) __stcs(P.xbar + col * P.ldxb + r, YB[r * CV_LD + cidx]);
    }
  }
  // ---- this CTA's partial of W̄ (column-major like W) and c̄ -----------------------------------------------------------
  float* part = P.part + (size_t)blockIdx.x * ((size_t)m2 * n2 + m2);
  const int rbase = 32 * warp;
#pragma unroll
  for (int i = 0; i < 32; ++i)
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (rbase + i < m2 && lane + 32 * q < n2) part[(size_t)(lane + 32 * q) * m2 + rbase + i] = acc[i][q];
  if ((int)threadIdx.x < m2) part[(size_t)m2 * n2 + threadIdx.x] = cacc;
}

// ---- register-tiled version for n1, n2 multiples of 4 (the RealNVP shapes) -----------------------------------------------
// Same three GEMMs, FMA-bound instead of load-bound: every shared-memory operand is a float4,
//   [s; t]   thread = 4 s rows + the matching 4 t rows x 4 columns: per k two float4 of W (L1) + one float4 of x₂ -> 32 FMA
//   x̄₂       thread = 4 rows of x₂ x 4 columns: per 4 j four float4 of W + four float4 of [s̄; t̄]              -> 64 FMA
//   W̄        warp = 32 rows of [s̄; t̄], lane = 4 rows of x₂: per 4 columns 32 broadcast float4 + 4 float4     -> 512 FMA
// and every FMA is one half of a float2-pair b2b_ffma2 (row pairs of W / of [s̄; t̄] against a broadcast scalar, or even/odd-j
// partial sums).
// The tiles are 32 floats wide with the 16-byte chunks XOR-swizzled by the row (chunk ^ (row & 7)) instead of padded:
// conflict-free for the row-wise float4 reads, the lane-per-row reads of the W̄ product and the transposing stores alike,
// and the CTA stays under 100 KB of shared memory -- which leaves 156 KB of L1 for W (128 KB at n1 = n2 = 128), read
// through L1 by every tile; streaming W through shared memory with bulk
// copies was tried and was slower.
constexpr int CF_LD = CV_TC;

__device__ __forceinline__ float4 ld4s(const float* p) { return *reinterpret_cast<const float4*>(p); }
// W is swept once per tile by every warp and must stay in L1: its loads ask to be evicted last, the streamed batch
// (x, ȳ in, x̄ out) does not allocate in L1 at all.
__device__ __forceinline__ float4 ld4g(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::evict_last.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_stream(const float* p) {
  float v;
  asm volatile("ld.global.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream(float* p, float v) {
  asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void fma4(float (&a)[4], float w, const float4& x) {
  a[0] = fmaf(w, x.x, a[0]);
  a[1] = fmaf(w, x.y, a[1]);
  a[2] = fmaf(w, x.z, a[2]);
  a[3] = fmaf(w, x.w, a[3]);
}
// float offset of chunk `ch` (4 columns) of tile row `r`, and of the single element (r, c)
__device__ __forceinline__ int cf_chunk(int r, int ch) { return r * CF_LD + ((ch ^ (r & 7)) << 2); }
__device__ __forceinline__ int cf_elem(int r, int c) { return r * CF_LD + ((((c >> 2) ^ (r & 7)) << 2) | (c & 3)); }

// [s̄; t̄] tile: rows stored in interleaved PAIRS -- a 16-byte chunk holds {row 2p, row 2p+1} x {col 2h, col 2h+1} -- so that
// a float4 is two b2b_ffma2 operands (row pairs against a broadcast scalar).  Chunk h of pair p sits at h ^ (h >> 3).
__device__ __forceinline__ int sb_chunk(int p, int h) { return p * 64 + ((h ^ (h >> 3)) << 2); }
__device__ __forceinline__ int sb_elem(int row, int col) { return sb_chunk(row >> 1, col >> 1) + ((col & 1) << 1) + (row & 1); }
__device__ __forceinline__ float2 bc2(float v) { return make_float2(v, v); }

// CONTIG: x₂ is a contiguous row range (row2 >= 0).
template <bool INV, bool CONTIG>
__global__ void __launch_bounds__(CV_THREADS, 1) coupling_vjp_fast_kernel(const __grid_constant__ CvParams P) {
  extern __shared__ __align__(16) float smem_f[];
  const int D = P.D, n1 = P.n1, n2 = P.n2, m2 = 2 * n1;
  const int m2p = (m2 + 31) & ~31;
  float* X = smem_f;                          // [D + 1][32]    row D stays zero (x₂ rows beyond n2 in the W̄ tile)
  float* YB = X + (size_t)(D + 1) * CF_LD;    // [D][32]
  float* SB = YB + (size_t)D * CF_LD;         // [m2p / 2][64]  row pairs; rows beyond 2n1 stay zero
  float* LB = SB + (size_t)m2p * CF_LD;       // [CV_TC]
  int* s1 = reinterpret_cast<int*>(LB + CV_TC);
  int* s2 = s1 + n1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int rg = threadIdx.x >> 3, cg = threadIdx.x & 7;  // rows 4·rg + i, columns 4·cg + q
  for (int k = threadIdx.x; k < n1; k += CV_THREADS) s1[k] = P.idx1 ? P.idx1[k] : P.row1 + k;
  for (int k = threadIdx.x; k < n2; k += CV_THREADS) s2[k] = P.idx2 ? P.idx2[k] : P.row2 + k;
  for (int e = threadIdx.x; e < CF_LD; e += CV_THREADS) X[D * CF_LD + e] = 0.f;
  for (int e = threadIdx.x; e < (m2p - m2) * CF_LD; e += CV_THREADS) SB[m2 * CF_LD + e] = 0.f;
  const long long tiles = (P.N + CV_TC - 1) / CV_TC;
  const int ldw = m2, nrb = (D + 7) / 8;
  float2 acc[16][4];   // rows 32·warp + 2·ip (+1) of [s̄; t̄]  x  x₂ rows lane + 32·q
#pragma unroll
  for (int i = 0; i < 16; ++i)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[i][q] = make_float2(0.f, 0.f);
  float cacc = 0.f;  // c̄ partial: thread (rg, cg) owns row 4rg + cg of s̄ (cg < 4) or of t̄ (cg >= 4)

  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long col0 = tile * CV_TC;
    __syncthreads();
    // a warp moves 8 rows x 4 columns per step: whole 32-byte sectors in global memory, 32 distinct banks in the tiles
    for (int cb = warp; cb < CV_TC / 4; cb += CV_THREADS / 32) {
      const int cidx = 4 * cb + (lane >> 3);
      const long long col = col0 + cidx;
      const bool okc = col < P.N;
      for (int rb0 = 0; rb0 < nrb; rb0 += 8) {  // 16 loads in flight per lane
        float xv[8], yv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int r = 8 * (rb0 + u) + (lane & 7);
          const bool ok = okc && r < D;
          xv[u] = ok ? ld_stream(P.x + col * P.ldx + r) : 0.f;
          yv[u] = ok ? ld_stream(P.ybar + col * P.ldyb + r) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int r = 8 * (rb0 + u) + (lane & 7);
          if (r < D) {
            X[cf_elem(r, cidx)] = xv[u];
            YB[cf_elem(r, cidx)] = yv[u];
          }
        }
      }
    }
    if (threadIdx.x < CV_TC) LB[threadIdx.x] = (col0 + threadIdx.x < P.N && P.ljbar) ? P.ljbar[col0 + threadIdx.x] : 0.f;
    __syncthreads();
    // ---- [s; t] = W·x₂ + c ----------------------------------------------------------------------------------------------
    float2 sv[2][4], tv[2][4];  // [row pair][column]
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int q = 0; q < 4; ++q) sv[i][q] = tv[i][q] = make_float2(0.f, 0.f);
    if (4 * rg < n1) {
      const float* Wp = P.W + 4 * rg;
#pragma unroll 4
      for (int k = 0; k < n2; ++k) {
        const int xr = CONTIG ? P.row2 + k : s2[k];
        const float4 xv = ld4s(X + cf_chunk(xr, cg));
        const float4 ws = ld4g(Wp + (size_t)k * ldw), wt = ld4g(Wp + (size_t)k * ldw + n1);
        const float2 ws0 = make_float2(ws.x, ws.y), ws1 = make_float2(ws.z, ws.w);
        const float2 wt0 = make_float2(wt.x, wt.y), wt1 = make_float2(wt.z, wt.w);
        const float xq[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          sv[0][q] = b2b_ffma2(ws0, bc2(xq[q]), sv[0][q]);
          sv[1][q] = b2b_ffma2(ws1, bc2(xq[q]), sv[1][q]);
          tv[0][q] = b2b_ffma2(wt0, bc2(xq[q]), tv[0][q]);
          tv[1][q] = b2b_ffma2(wt1, bc2(xq[q]), tv[1][q]);
        }
      }
    }
    // ---- the elementwise cotangents ------------------------------------------------------------------------------------
    float rs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // row sums of s̄ (0..3) and t̄ (4..7) over the thread's 4 columns
    if (4 * rg < n1) {
      const float4 lb4 = ld4s(LB + 4 * cg);
      const float lbv[4] = {lb4.x, lb4.y, lb4.z, lb4.w};
      float sbar[4][4], tbar[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = 4 * rg + i;
        const float cs = P.c ? P.c[j] : 0.f, ct = P.c ? P.c[n1 + j] : 0.f;
        const int o1 = cf_chunk(s1[j], cg);
        const float4 in4 = ld4s(X + o1), cb4 = ld4s(YB + o1);
        const float in1[4] = {in4.x, in4.y, in4.z, in4.w}, cb1[4] = {cb4.x, cb4.y, cb4.z, cb4.w};
        float out1[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float s_ = ((i & 1) ? sv[i >> 1][q].y : sv[i >> 1][q].x) + cs;
          const float t_ = ((i & 1) ? tv[i >> 1][q].y : tv[i >> 1][q].x) + ct;
          if (!INV) {
            const float e = expf(s_);
            out1[q] = e * cb1[q];
            sbar[i][q] = fmaf(cb1[q] * e, in1[q], lbv[q]);
            tbar[i][q] = cb1[q];
          } else {
            const float em = expf(-s_);
            const float x1 = (in1[q] - t_) * em;
            out1[q] = em * cb1[q];
            sbar[i][q] = -fmaf(x1, cb1[q], lbv[q]);
            tbar[i][q] = -out1[q];
          }
        }
        *reinterpret_cast<float4*>(YB + o1) = make_float4(out1[0], out1[1], out1[2], out1[3]);
      }
#pragma unroll
      for (int pp = 0; pp < 2; ++pp) {  // row pairs (4rg + 2pp, +1) of s̄ and of t̄, chunks 2cg, 2cg + 1
        const int ps = 2 * rg + pp, pt = (n1 >> 1) + ps, i0 = 2 * pp, i1 = 2 * pp + 1;
        *reinterpret_cast<float4*>(SB + sb_chunk(ps, 2 * cg)) = make_float4(sbar[i0][0], sbar[i1][0], sbar[i0][1], sbar[i1][1]);
        *reinterpret_cast<float4*>(SB + sb_chunk(ps, 2 * cg + 1)) = make_float4(sbar[i0][2], sbar[i1][2], sbar[i0][3], sbar[i1][3]);
        *reinterpret_cast<float4*>(SB + sb_chunk(pt, 2 * cg)) = make_float4(tbar[i0][0], tbar[i1][0], tbar[i0][1], tbar[i1][1]);
        *reinterpret_cast<float4*>(SB + sb_chunk(pt, 2 * cg + 1)) = make_float4(tbar[i0][2], tbar[i1][2], tbar[i0][3], tbar[i1][3]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        rs[i] = (sbar[i][0] + sbar[i][1]) + (sbar[i][2] + sbar[i][3]);
        rs[4 + i] = (tbar[i][0] + tbar[i][1]) + (tbar[i][2] + tbar[i][3]);
      }
    }
    // c̄: the 8 column groups of a row group are 8 consecutive lanes (whole warps take part in the shuffles)
#pragma unroll
    for (int o = 1; o < 8; o <<= 1)
#pragma unroll
      for (int i = 0; i < 8; ++i) rs[i] += __shfl_xor_sync(0xffffffffu, rs[i], o);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (cg == i) cacc += rs[i];
    __syncthreads();
    // ---- x̄₂ = ȳ₂ + Wᵀ[s̄; t̄]: even-j and odd-j partial sums in the two halves of a packed accumulator -------------------
    if (4 * rg < n2) {
      float2 a[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int q = 0; q < 4; ++q) a[i][q] = make_float2(0.f, 0.f);
      const float* wr[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) wr[i] = P.W + (size_t)(4 * rg + i) * ldw;
      const int h0 = ((2 * cg) ^ (cg >> 2)) << 2, h1 = ((2 * cg + 1) ^ (cg >> 2)) << 2;
#pragma unroll 2
      for (int j = 0; j < m2; j += 4) {
        const float* sp = SB + (j >> 1) * 64;
        const float4 p00 = ld4s(sp + h0), p01 = ld4s(sp + h1);            // rows j, j+1: columns 0,1 | 2,3
        const float4 p10 = ld4s(sp + 64 + h0), p11 = ld4s(sp + 64 + h1);  // rows j+2, j+3
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float4 w = ld4g(wr[i] + j);
          const float2 w0 = make_float2(w.x, w.y), w1 = make_float2(w.z, w.w);
          a[i][0] = b2b_ffma2(w0, make_float2(p00.x, p00.y), a[i][0]);
          a[i][1] = b2b_ffma2(w0, make_float2(p00.z, p00.w), a[i][1]);
          a[i][2] = b2b_ffma2(w0, make_float2(p01.x, p01.y), a[i][2]);
          a[i][3] = b2b_ffma2(w0, make_float2(p01.z, p01.w), a[i][3]);
          a[i][0] = b2b_ffma2(w1, make_float2(p10.x, p10.y), a[i][0]);
          a[i][1] = b2b_ffma2(w1, make_float2(p10.z, p10.w), a[i][1]);
          a[i][2] = b2b_ffma2(w1, make_float2(p11.x, p11.y), a[i][2]);
          a[i][3] = b2b_ffma2(w1, make_float2(p11.z, p11.w), a[i][3]);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float* dst = YB + cf_chunk(s2[4 * rg + i], cg);
        const float4 o = ld4s(dst);
        *reinterpret_cast<float4*>(dst) = make_float4(o.x + (a[i][0].x + a[i][0].y), o.y + (a[i][1].x + a[i][1].y),
                                                      o.z + (a[i][2].x + a[i][2].y), o.w + (a[i][3].x + a[i][3].y));
      }
    }
    // ---- W̄ += [s̄; t̄]·x₂ᵀ over the tile's columns ----------------------------------------------------------------------
    {
      const int rbase = 32 * warp;
      if (rbase < m2) {
        const float* xr[4];
        int xs[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int r = (lane + 32 * q < n2) ? s2[lane + 32 * q] : D;
          xr[q] = X + r * CF_LD;
          xs[q] = r & 7;
        }
        const float* sbp = SB + (rbase >> 1) * 64;
#pragma unroll 2
        for (int ch = 0; ch < CV_TC / 4; ++ch) {
          float4 bq[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) bq[q] = ld4s(xr[q] + ((ch ^ xs[q]) << 2));
          const int g0 = ((2 * ch) ^ (ch >> 2)) << 2, g1 = ((2 * ch + 1) ^ (ch >> 2)) << 2;
#pragma unroll
          for (int ip = 0; ip < 16; ++ip) {
            const float4 a0 = ld4s(sbp + ip * 64 + g0), a1 = ld4s(sbp + ip * 64 + g1);  // columns 4ch, +1 | +2, +3
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              float2 t = acc[ip][q];
              t = b2b_ffma2(make_float2(a0.x, a0.y), bc2(bq[q].x), t);
              t = b2b_ffma2(make_float2(a0.z, a0.w), bc2(bq[q].y), t);
              t = b2b_ffma2(make_float2(a1.x, a1.y), bc2(bq[q].z), t);
              t = b2b_ffma2(make_float2(a1.z, a1.w), bc2(bq[q].w), t);
              acc[ip][q] = t;
            }
          }
        }
      }
    }
    __syncthreads();
    for (int blk = warp; blk < nrb * (CV_TC / 4); blk += CV_THREADS / 32) {
      const int r = 8 * (blk % nrb) + (lane & 7), cidx = 4 * (blk / nrb) + (lane >> 3);
      const long long col = col0 + cidx;
      if (col < P.N && r < D) st_stream(P.xbar + col * P.ldxb + r, YB[cf_elem(r, cidx)]);
    }
  }
  float* part = P.part + (size_t)blockIdx.x * ((size_t)m2 * n2 + m2);
  const int rbase = 32 * warp;
#pragma unroll
  for (int ip = 0; ip < 16; ++ip)
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (lane + 32 * q < n2) {
        if (rbase + 2 * ip < m2) part[(size_t)(lane + 32 * q) * m2 + rbase + 2 * ip] = acc[ip][q].x;
        if (rbase + 2 * ip + 1 < m2) part[(size_t)(lane + 32 * q) * m2 + rbase + 2 * ip + 1] = acc[ip][q].y;
      }
  if (4 * rg < n1) part[(size_t)m2 * n2 + (cg < 4 ? 4 * rg + cg : n1 + 4 * rg + cg - 4)] = cacc;
}

// out[e] = Σ_cta part[cta][e], fixed order
__global__ void __launch_bounds__(256) partial_sum_kernel(const float* __restrict__ part, int nparts, int len, float* __restrict__ out0,
                                                          int len0, float* __restrict__ out1) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < len; e += gridDim.x * blockDim.x) {
    float t = 0.f;
    for (int p = 0; p < nparts; ++p) t += part[(size_t)p * len + e];
    if (e < len0) out0[e] = t;
    else out1[e - len0] = t;
  }
}

// ---- eval-mode InvertibleBatchNorm -------------------------------------------------------------------------------------
// y = A(x − m) + b, A = e^logs / sqrt(v + eps) (normalise.jl:61-67).  forward: x̄ = A ȳ, b̄ = Σ ȳ, l̄ogs = Σ ȳ⊙(y − b) + Σ l̄;
// inverse: ȳ = x̄ / A, b̄ = −Σ x̄/A, l̄ogs = −Σ x̄⊙(x − m) − Σ l̄.
struct BvParams {
  const float* x;
  const float* ybar;
  const float* ljbar;
  float* xbar;
  const float *b, *logs, *m, *v;
  float eps;
  float* part;  // [grid][2D + 1]
  long long N, ldx, ldyb, ldxb;
  int D, inverse;
};

constexpr int BV_U = 8;

// Thread = one row (RPT rows 256 apart when D > 256) of a slab of columns, U columns at a time; the row's two partial sums
// stay in registers, slabs are summed in shared memory, CTAs by the finalize kernel -- fixed order throughout.
// U columns of one slab.  FULL: every column and every row of the group exists (no guards in the body).
template <int RPT, int U, bool INV, bool FULL>
__device__ __forceinline__ void bn_vjp_group(const BvParams& P, long long n0, long long c1, int nslab, int i, int D,
                                             const float (&A)[RPT], const float (&sh)[RPT], float (&gb)[RPT], float (&gl)[RPT],
                                             float& lsum) {
  float xv[U][RPT], cb[U][RPT];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const long long n = n0 + (long long)u * nslab;
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      const int r = i + 256 * j;
      const bool ok = FULL || (n < c1 && r < D);
      xv[u][j] = ok ? __ldcs(P.x + n * P.ldx + r) : sh[j];
      cb[u][j] = ok ? __ldcs(P.ybar + n * P.ldyb + r) : 0.f;
    }
    if (i == 0 && P.ljbar && (FULL || n < c1)) lsum += P.ljbar[n];
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const long long n = n0 + (long long)u * nslab;
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      const int r = i + 256 * j;
      // forward: x̄ = A ȳ, b̄ += ȳ, l̄ogs += ȳ·A(x − m);  inverse (A holds 1/A): ȳ = x̄/A, b̄ −= ȳ, l̄ogs −= ȳ (y − b)
      const float o = A[j] * cb[u][j];
      if (FULL || (n < c1 && r < D)) __stcs(P.xbar + n * P.ldxb + r, o);
      gb[j] += INV ? -o : cb[u][j];
      gl[j] = fmaf(INV ? -o : o, xv[u][j] - sh[j], gl[j]);
    }
  }
}

template <int RPT, bool INV>
__global__ void __launch_bounds__(256) bn_eval_vjp_kernel(const __grid_constant__ BvParams P) {
  extern __shared__ float bsm[];  // [nslab][2D + 1]
  constexpr int U = RPT == 1 ? BV_U : BV_U / 2;  // columns in flight per thread
  const int D = P.D, Dp = RPT == 1 ? ((D + 31) & ~31) : 256, nslab = 256 / Dp;
  const int slab = threadIdx.x / Dp, i = threadIdx.x - slab * Dp;
  float A[RPT], sh[RPT], gb[RPT], gl[RPT];
  bool rows = true;
#pragma unroll
  for (int j = 0; j < RPT; ++j) {
    const int r = i + 256 * j;
    gb[j] = gl[j] = 0.f;
    A[j] = 1.f;
    sh[j] = 0.f;
    rows = rows && r < D;
    if (r < D) {
      const float a = expf(P.logs[r]) / sqrtf(P.v[r] + P.eps);
      A[j] = INV ? 1.0f / a : a;
      sh[j] = INV ? P.b[r] : P.m[r];  // the shift removed before scaling: y − b (inverse) / x − m (forward)
    }
  }
  float lsum = 0.f;
  const long long per = (P.N + gridDim.x - 1) / gridDim.x;
  const long long c0 = (long long)blockIdx.x * per, c1 = (c0 + per < P.N) ? c0 + per : P.N;
  if (slab < nslab) {
    for (long long n0 = c0 + slab; n0 < c1; n0 += (long long)U * nslab) {
      if (rows && n0 + (long long)(U - 1) * nslab < c1) bn_vjp_group<RPT, U, INV, true>(P, n0, c1, nslab, i, D, A, sh, gb, gl, lsum);
      else bn_vjp_group<RPT, U, INV, false>(P, n0, c1, nslab, i, D, A, sh, gb, gl, lsum);
    }
    float* mine = bsm + (size_t)slab * (2 * D + 1);
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      const int r = i + 256 * j;
      if (r < D) {
        mine[r] = gb[j];
        mine[D + r] = gl[j];
      }
    }
    if (i == 0) mine[2 * D] = lsum;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 2 * D + 1; e += blockDim.x) {
    float t = 0.f;
    for (int w = 0; w < nslab; ++w) t += bsm[(size_t)w * (2 * D + 1) + e];
    P.part[(size_t)blockIdx.x * (2 * D + 1) + e] = t;
  }
}

// bbar[r] = Σ parts, logsbar[r] = Σ parts ± Σ l̄; block (32, 8): 8 strided sub-sums per element, then those in order
__global__ void __launch_bounds__(256) bn_vjp_finalize_kernel(const float* __restrict__ part, int nparts, int D, int inverse,
                                                              float* __restrict__ bbar, float* __restrict__ logsbar) {
  __shared__ float sub[8][32];
  __shared__ float lsm[256];
  const int len = 2 * D + 1, e = blockIdx.x * 32 + threadIdx.x, q = threadIdx.y * 32 + threadIdx.x;
  float t = 0.f, l = 0.f;
  if (e < 2 * D)
    for (int p = threadIdx.y; p < nparts; p += 8) t += part[(size_t)p * len + e];
  for (int p = q; p < nparts; p += 256) l += part[(size_t)p * len + 2 * D];
  sub[threadIdx.y][threadIdx.x] = t;
  lsm[q] = l;
  __syncthreads();
  if (threadIdx.y == 0 && e < 2 * D) {
    float r = 0.f, ls = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) r += sub[k][threadIdx.x];
    if (e < D) {
      bbar[e] = r;
    } else {
      for (int k = 0; k < 256; ++k) ls += lsm[k];
      logsbar[e - D] = r + (inverse ? -ls : ls);
    }
  }
}

// float4 path: n1, n2 multiples of 4 and a 16-byte aligned W (its leading dimension 2·n1 is then a multiple of 4 too)
static bool vjp_fast(const b2b_layer_desc& d) {
  return d.n0 % 4 == 0 && d.n1 % 4 == 0 && (reinterpret_cast<uintptr_t>(d.p0) & 15) == 0;
}

// both programs stage the layer's input and output cotangent tiles over all D rows
static size_t vjp_smem_bytes(const b2b_layer_desc& d, int D) {
  const int n1 = d.n0, n2 = d.n1;
  return vjp_fast(d) ? ((size_t)(2 * D + 1 + ((2 * n1 + 31) & ~31)) * CF_LD + CV_TC) * sizeof(float) + (size_t)(n1 + n2) * sizeof(int)
                     : ((size_t)2 * D * CV_LD + (size_t)2 * n1 * CV_LD + CV_TC) * sizeof(float) + (size_t)(n1 + n2) * sizeof(int);
}

}  // namespace b2b

bool b2b_coupling_affine_vjp_fits(const b2b_layer_desc& d, int D) {
  return d.n0 <= 128 && d.n1 <= 128 && b2b::vjp_smem_bytes(d, D) <= 220 * 1024;
}

extern "C" size_t b2b_coupling_affine_vjp_workspace_bytes(int32_t n1, int32_t n2) {
  if (n1 < 1 || n1 > 128 || n2 < 1 || n2 > 128) return 0;
  return (size_t)b2b_sm_count() * ((size_t)2 * n1 * n2 + 2 * n1) * sizeof(float) + 256;
}

int b2b_vjp_coupling(const B2BVjpSeg& s) {
  using namespace b2b;
  const b2b_layer_desc& d = s.layers[0];
  const int n1 = d.n0, n2 = d.n1, D = s.D;
  if (!s.workspace || s.workspace_bytes < b2b_coupling_affine_vjp_workspace_bytes(n1, n2)) return B2B_EWORKSPACE;
  const int len0 = 2 * n1 * n2, len = len0 + 2 * n1;
  // the kernel forms W̄ and c̄: those not asked for go to scratch
  float* const Wbar = s.bars[0] ? s.bars[0] : s.scratch;
  float* const cbar = s.bars[1] ? s.bars[1] : s.scratch + ((len0 + 63) & ~63);
  CvParams P;
  P.x = s.x;
  P.ybar = s.ybar;
  P.ljbar = s.ljbar;
  P.xbar = s.xbar;
  P.W = d.p0;
  P.c = d.p1;
  P.idx1 = d.i0;
  P.idx2 = d.i1;
  P.part = reinterpret_cast<float*>(b2b_align256(s.workspace));
  P.N = s.N;
  P.ldx = s.ldx;
  P.ldyb = s.ldyb;
  P.ldxb = s.ldxb;
  P.D = D;
  P.n1 = n1;
  P.n2 = n2;
  P.row1 = d.n2;
  P.row2 = d.n3;
  const long long tiles = (s.N + CV_TC - 1) / CV_TC;
  long long grid = b2b_sm_count();
  if (grid > tiles) grid = tiles;
  const bool fast = vjp_fast(d);
  const size_t smem = vjp_smem_bytes(d, D);
  void (*kernel)(const CvParams);
  if (!fast) kernel = d.inverse ? coupling_vjp_kernel<true> : coupling_vjp_kernel<false>;
  else if (d.n3 < 0) kernel = d.inverse ? coupling_vjp_fast_kernel<true, false> : coupling_vjp_fast_kernel<false, false>;
  else kernel = d.inverse ? coupling_vjp_fast_kernel<true, true> : coupling_vjp_fast_kernel<false, true>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  // the smallest carve-out that holds the CTA: the rest of the 256 KB stays L1 (W is re-read through it by every tile)
  cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)((smem + 1024) * 100 / (228 * 1024) + 1));
  kernel<<<(int)grid, CV_THREADS, smem, s.stream>>>(P);
  e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  partial_sum_kernel<<<(len + 255) / 256, 256, 0, s.stream>>>(P.part, (int)grid, len, Wbar, len0, cbar);
  *s.launches += 2;
  return (int)cudaGetLastError();
}

extern "C" int b2b_coupling_affine_vjp_f32(const b2b_layer_desc* layer, const float* x, const float* ybar, const float* ljbar,
                                           float* xbar, float* Wbar, float* cbar, int32_t D, int64_t N, int64_t ldx,
                                           int64_t ldybar, int64_t ldxbar, void* workspace, size_t workspace_bytes,
                                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!layer || layer->kind != B2B_COUPLING_AFFINE || D < 1 || N < 0 || !Wbar || !cbar) return B2B_EINVAL;
  const b2b_layer_desc& d = *layer;
  const int n1 = d.n0, n2 = d.n1;
  if (!d.p0 || n1 < 1 || n2 < 1 || n1 + n2 > D || (!d.i0 && d.n2 < 0) || (!d.i1 && d.n3 < 0)) return B2B_EINVAL;
  if (!b2b_coupling_affine_vjp_fits(d, D)) return B2B_EUNSUPPORTED;
  if (N == 0) {
    cudaMemsetAsync(Wbar, 0, sizeof(float) * (size_t)2 * n1 * n2, stream);
    return (int)cudaMemsetAsync(cbar, 0, sizeof(float) * 2 * n1, stream);
  }
  if (!x || !ybar || !xbar || ldx < D || ldybar < D || ldxbar < D) return B2B_EINVAL;
  float* const bars[4] = {Wbar, cbar, nullptr, nullptr};
  int launches = 0;
  return b2b_vjp_coupling({layer, 1, x, ldx, ybar, ldybar, ljbar, xbar, ldxbar, D, N, bars, nullptr, workspace,
                           workspace_bytes, &launches, stream});
}

extern "C" size_t b2b_batchnorm_eval_vjp_workspace_bytes(int32_t D) {
  if (D < 1 || D > 1024) return 0;
  return (size_t)b2b_sm_count() * 4 * (size_t)(2 * D + 1) * sizeof(float) + 256;
}

int b2b_vjp_batchnorm(const B2BVjpSeg& s) {
  using namespace b2b;
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  if (!s.workspace || s.workspace_bytes < b2b_batchnorm_eval_vjp_workspace_bytes(D)) return B2B_EWORKSPACE;
  // the kernel forms b̄ and log s̄: those not asked for go to scratch
  float* const bbar = s.bars[0] ? s.bars[0] : s.scratch;
  float* const logsbar = s.bars[1] ? s.bars[1] : s.scratch + ((D + 63) & ~63);
  BvParams P;
  P.x = s.x;
  P.ybar = s.ybar;
  P.ljbar = s.ljbar;
  P.xbar = s.xbar;
  P.b = d.p0;
  P.logs = d.p1;
  P.m = d.p2;
  P.v = d.p3;
  P.eps = d.f0;
  P.part = reinterpret_cast<float*>(b2b_align256(s.workspace));
  P.N = s.N;
  P.ldx = s.ldx;
  P.ldyb = s.ldyb;
  P.ldxb = s.ldxb;
  P.D = D;
  P.inverse = d.inverse ? 1 : 0;
  const int rpt = (D + 255) / 256, Dp = rpt == 1 ? ((D + 31) & ~31) : 256, nslab = 256 / Dp;
  long long grid = (long long)b2b_sm_count() * 4;
  const int bu = rpt == 1 ? BV_U : BV_U / 2;
  const long long want = (s.N + (long long)nslab * bu - 1) / ((long long)nslab * bu);
  if (grid > want) grid = want;
  const size_t smem = (size_t)nslab * (2 * D + 1) * sizeof(float);
  void (*kernel)(const BvParams);
  if (P.inverse) kernel = rpt == 1 ? bn_eval_vjp_kernel<1, true> : rpt == 2 ? bn_eval_vjp_kernel<2, true> : bn_eval_vjp_kernel<4, true>;
  else kernel = rpt == 1 ? bn_eval_vjp_kernel<1, false> : rpt == 2 ? bn_eval_vjp_kernel<2, false> : bn_eval_vjp_kernel<4, false>;
  kernel<<<(int)grid, 256, smem, s.stream>>>(P);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  bn_vjp_finalize_kernel<<<(2 * D + 31) / 32, dim3(32, 8), 0, s.stream>>>(P.part, (int)grid, D, P.inverse, bbar, logsbar);
  *s.launches += 2;
  return (int)cudaGetLastError();
}

extern "C" int b2b_batchnorm_eval_vjp_f32(const b2b_layer_desc* layer, const float* x, const float* ybar, const float* ljbar,
                                          float* xbar, float* bbar, float* logsbar, int32_t D, int64_t N, int64_t ldx,
                                          int64_t ldybar, int64_t ldxbar, void* workspace, size_t workspace_bytes,
                                          void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!layer || layer->kind != B2B_BATCHNORM || D < 1 || N < 0 || !bbar || !logsbar) return B2B_EINVAL;
  const b2b_layer_desc& d = *layer;
  if (!d.p0 || !d.p1 || !d.p2 || !d.p3) return B2B_EINVAL;
  if (D > 1024) return B2B_EUNSUPPORTED;
  if (N == 0) {
    cudaMemsetAsync(bbar, 0, sizeof(float) * D, stream);
    return (int)cudaMemsetAsync(logsbar, 0, sizeof(float) * D, stream);
  }
  if (!x || !ybar || !xbar || ldx < D || ldybar < D || ldxbar < D) return B2B_EINVAL;
  float* const bars[4] = {bbar, logsbar, nullptr, nullptr};
  int launches = 0;
  return b2b_vjp_batchnorm({layer, 1, x, ldx, ybar, ldybar, ljbar, xbar, ldxbar, D, N, bars, nullptr, workspace,
                            workspace_bytes, &launches, stream});
}
