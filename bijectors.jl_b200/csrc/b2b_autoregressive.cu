// Masked autoregressive layers, B2B_AUTOREGRESSIVE_MLP (include/b2b.h): MAF / IAF's affine layer y = x ⊙ exp.(s) + t
// whose row i takes sᵢ, tᵢ from a MADE network of rows 1..i−1,
//   u = (M₁⊙W₁)·x + c₁,   h = σ.(u),   [s; t] = (M₂⊙W₂)·h + c₂,   M₁[k, r] = (r <= m_k),   M₂[i, k] = M₂[D+i, k] = (m_k < i),
// forward, inverse and reverse mode, in exact fp32 on the CUDA cores.
//
// Masked weights.  Every launcher first runs ar_prep_kernel, which writes M₁⊙W₁ and M₂⊙W₂ into the workspace (a
// selected 0 outside the masks, which are never read), a row-paired copy W2p[i·H + k] = ((M₂⊙W₂)[i, k], (M₂⊙W₂)[D+i, k])
// for the sequential kernels, and for the inverse layer's reverse mode W1r = (M₁⊙W₁)·diag(Σᵢ (M₂⊙W₂)[i, :]).
//
// Forward (parallel): the MLP coupling's tile with x₁ = x₂ = x and the masked weights -- cmlp_hidden, then coupling_tile
// -- over 64-column tiles.  A masked weight is an exact 0, so fmaf(0, h, acc) = acc: sᵢ is bit for bit independent of
// rows >= i.
//
// Inverse (sequential): ar_recover, one warp per AR_C columns, lanes over the hidden units (k = lane + 32j, H/32 <= 8 per
// lane).  Each lane keeps the pre-activations u_k and the activations h_k of its units for each column in registers; h_k
// is 0 until unit k is final (after row m_k) and σ(u_k) from then on.  Row i: one warp reduction for sᵢ and one for tᵢ
// over the lane partials Σ W2p[i, k]·h_k, xᵢ = (yᵢ − tᵢ)/exp(sᵢ), then u_k += (M₁⊙W₁)[k, i]·xᵢ.  Each W load serves AR_C
// columns.  W (5·H·D floats with the paired copy, 640 KB at D = 128, H = 256) is read through L1 / L2.
//
// Reverse mode: coupling_mlp_vjp_kernel's structure (b2b_coupling_net.cuh), with M = 1, n1 = n2 = D and the masked
// weights.  Forward layer: v̄ = ȳ ⊙ eˢ + (M₁⊙W₁)ᵀū.  Inverse layer: the input v is recovered by ar_recover, then
// g = v̄ − l̄·W1rᵀσ′(u) and the upper-triangular solve Jᵀw̄ = g by ar_solve (one warp per AR_C columns, row D down to 1,
// the hidden cotangent accumulated as each row is finished); the parameter sums are the forward rule's at v with
// [s̄; t̄] = −[w̄ ⊙ v ⊙ eˢ + l̄; w̄].  Per-CTA slices and an ordered fp64 reduce that writes exact zeros outside the masks:
// deterministic, no atomics.
#include <cuda_runtime.h>

#include "b2b_coupling_mlp.cuh"
#include "b2b_coupling_net.cuh"
#include "b2b_coupling_tile.cuh"
#include "b2b_internal.h"

namespace b2b {

constexpr int AR_C = 4;          // columns per warp of the sequential kernels
constexpr int AR_UNITS = 8;      // hidden units per lane (H <= 256)
constexpr int AR_SEQ_THREADS = 128;

// the network of one layer as the kernels read it: the masked weights in the workspace, the descriptor's biases
struct ArNet {
  const float* W1;    // M₁⊙W₁, H x D column-major
  const float* c1;    // H or NULL
  const float* W2;    // M₂⊙W₂, 2D x H column-major
  const float* c2;    // 2D or NULL
  const float2* W2p;  // row pairs of M₂⊙W₂, D x H
  const float* W1r;   // (M₁⊙W₁)·diag(Σᵢ (M₂⊙W₂)[i, :]), H x D column-major (reverse mode of the inverse layer)
  const int* deg;     // m[H]
  int D, H, act;
  float slope;
};

static size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

// the workspace regions: W1 | W2 | W2p (| W1r)
struct ArWs {
  float *W1, *W2, *W1r;
  float2* W2p;
  size_t bytes;
};
static ArWs ar_ws(void* base, int D, int H, bool w1r) {
  ArWs w{};
  char* p = base ? b2b_align256(base) : nullptr;
  const size_t hd = (size_t)H * D * sizeof(float);
  size_t off = 0;
  w.W1 = reinterpret_cast<float*>(p + off);
  off += al256(hd);
  w.W2 = reinterpret_cast<float*>(p + off);
  off += al256(2 * hd);
  w.W2p = reinterpret_cast<float2*>(p + off);
  off += al256(2 * hd);
  if (w1r) {
    w.W1r = reinterpret_cast<float*>(p + off);
    off += al256(hd);
  }
  w.bytes = off + 256;
  return w;
}

// The masked copies, one element per thread (grid-stride).  W1r's column sums run over i in increasing order.
__global__ void __launch_bounds__(256) ar_prep_kernel(const float* __restrict__ W1, const float* __restrict__ W2,
                                                      const int* __restrict__ deg, int D, int H, float* __restrict__ oW1,
                                                      float* __restrict__ oW2, float2* __restrict__ oW2p,
                                                      float* __restrict__ oW1r) {
  const long long hd = (long long)H * D, stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < 4 * hd; e += stride) {
    if (e < hd) {  // M₁⊙W₁ (and W1r) at (k, i), e = k + H·i
      const int k = (int)(e % H), i = (int)(e / H);
      const bool on = i + 1 <= deg[k];
      const float w = on ? W1[e] : 0.f;
      oW1[e] = w;
      if (oW1r) {
        float r = 0.f;
        for (int j = 0; j < D && on; ++j)
          if (deg[k] < j + 1) r += W2[(size_t)j + (size_t)2 * D * k];
        oW1r[e] = on ? w * r : 0.f;
      }
    } else if (e < 3 * hd) {  // M₂⊙W₂ at (j, k), e − hd = j + 2D·k
      const long long f = e - hd;
      const int j = (int)(f % (2 * D)), k = (int)(f / (2 * D));
      oW2[f] = deg[k] < j % D + 1 ? W2[f] : 0.f;
    } else {  // the pair of row i at k, e − 3hd = k + H·i
      const long long f = e - 3 * hd;
      const int k = (int)(f % H), i = (int)(f / H);
      const bool on = deg[k] < i + 1;
      const size_t col = (size_t)2 * D * k;
      oW2p[f] = on ? make_float2(W2[col + i], W2[col + D + i]) : make_float2(0.f, 0.f);
    }
  }
}

static int ar_prep(const B2BCoupling<b2b_layer_desc>& c, const ArWs& w, int D, cudaStream_t stream) {
  const long long n = 4LL * c.H * D;
  const int grid = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
  ar_prep_kernel<<<grid, 256, 0, stream>>>(c.W_in, c.W_out, c.degrees, D, c.H, w.W1, w.W2, w.W2p, w.W1r);
  return (int)cudaGetLastError();
}

__device__ __forceinline__ float ar_warp_sum(float v) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);  // every lane ends with the same bits
  return v;
}

// Recovers x from y for AR_C columns, row by row (the inverse layer's map).  load(c, r) gives y of column c, row r;
// store(c, r, v) receives x; both are called by lane r % 32 for 32-row blocks.  ssum[c] = Σ s of column c.
template <class Load, class Store>
__device__ __forceinline__ void ar_recover(const ArNet& net, Load load, Store store, float (&ssum)[AR_C]) {
  const int lane = threadIdx.x & 31, D = net.D, H = net.H, nj = (H + 31) >> 5;
  float u[AR_C][AR_UNITS], h[AR_C][AR_UNITS];
  int mk[AR_UNITS];
#pragma unroll
  for (int j = 0; j < AR_UNITS; ++j) {
    const int k = lane + 32 * j;
    const bool unit = j < nj && k < H;
    mk[j] = unit ? net.deg[k] : -1;
    const float ck = unit && net.c1 ? __ldg(net.c1 + k) : 0.f;
    float hk = 0.f, dh;
    if (unit && mk[j] <= 0) mlp_act(net.act, net.slope, ck, hk, dh);  // final from the start
#pragma unroll
    for (int c = 0; c < AR_C; ++c) {
      u[c][j] = ck;
      h[c][j] = hk;
    }
  }
#pragma unroll
  for (int c = 0; c < AR_C; ++c) ssum[c] = 0.f;
  for (int b = 0; b < D; b += 32) {
    float yv[AR_C], xv[AR_C];
#pragma unroll
    for (int c = 0; c < AR_C; ++c) {
      yv[c] = b + lane < D ? load(c, b + lane) : 0.f;
      xv[c] = 0.f;
    }
    const int nr = min(32, D - b);
    for (int q = 0; q < nr; ++q) {
      const int i = b + q;
      float ps[AR_C] = {}, pt[AR_C] = {};
#pragma unroll
      for (int j = 0; j < AR_UNITS; ++j)
        if (j < nj) {
          const int k = lane + 32 * j;
          const float2 w = k < H ? __ldg(net.W2p + (size_t)i * H + k) : make_float2(0.f, 0.f);
#pragma unroll
          for (int c = 0; c < AR_C; ++c) {
            ps[c] = fmaf(w.x, h[c][j], ps[c]);
            pt[c] = fmaf(w.y, h[c][j], pt[c]);
          }
        }
      const float cs = net.c2 ? __ldg(net.c2 + i) : 0.f, ct = net.c2 ? __ldg(net.c2 + D + i) : 0.f;
      float xi[AR_C];
#pragma unroll
      for (int c = 0; c < AR_C; ++c) {
        const float s = ar_warp_sum(ps[c]) + cs, t = ar_warp_sum(pt[c]) + ct;
        xi[c] = (__shfl_sync(0xffffffffu, yv[c], q) - t) / expf(s);  // the inverse law of coupling_tile
        ssum[c] += s;
        if (lane == q) xv[c] = xi[c];
      }
#pragma unroll
      for (int j = 0; j < AR_UNITS; ++j)
        if (j < nj) {
          const int k = lane + 32 * j;
          const float w = k < H ? __ldg(net.W1 + (size_t)i * H + k) : 0.f;
#pragma unroll
          for (int c = 0; c < AR_C; ++c) {
            u[c][j] = fmaf(w, xi[c], u[c][j]);
            if (mk[j] == i + 1) {  // unit k is final once row m_k is known
              float dh;
              mlp_act(net.act, net.slope, u[c][j], h[c][j], dh);
            }
          }
        }
    }
#pragma unroll
    for (int c = 0; c < AR_C; ++c)
      if (b + lane < D) store(c, b + lane, xv[c]);
  }
}

struct ArParams {
  const float* x;
  float* y;
  float* logjac;
  ArNet net;
  long long N, ldx, ldy;
  int accumulate;
};

// the forward layer over 64-column tiles: x staged twice, the network's input and the rows the law transforms in place
__global__ void __launch_bounds__(CP_THREADS, 2) ar_forward_kernel(const __grid_constant__ ArParams P) {
  extern __shared__ float smem[];
  const int D = P.net.D, H = P.net.H;
  float* X = smem;                    // [D][CP_LD] x
  float* Y = X + (size_t)D * CP_LD;   // [D][CP_LD] x, transformed in place
  float* Hs = Y + (size_t)D * CP_LD;  // [H][CP_LD] h
  float* red = Hs + (size_t)H * CP_LD;  // [8][CP_TC]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool vec1 = ((H & 7) == 0) && ((reinterpret_cast<uintptr_t>(P.net.W1) & 15) == 0);
  const bool vec2 = ((D & 3) == 0) && ((reinterpret_cast<uintptr_t>(P.net.W2) & 15) == 0);
  const long long tiles = (P.N + CP_TC - 1) / CP_TC;
  auto same = [](int k) { return k; };
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long col0 = tile * CP_TC;
    __syncthreads();  // the previous tile is written back
    for (int c = warp; c < CP_TC; c += CP_THREADS / 32) {
      const long long col = col0 + c;
      for (int k = lane; k < D; k += 32) {
        const float v = col < P.N ? __ldcs(P.x + col * P.ldx + k) : 0.f;
        X[k * CP_LD + c] = v;
        Y[k * CP_LD + c] = v;
      }
    }
    __syncthreads();
    cmlp_hidden(X, D, P.net.W1, P.net.c1, vec1, H, P.net.act, P.net.slope, Hs);
    __syncthreads();
    coupling_tile<false>(Hs, Y, same, same, P.net.W2, P.net.c2, D, H, vec2, red);
    __syncthreads();
    if (P.y)  // x and y may alias: every element of the tile was read above
      for (int c = warp; c < CP_TC; c += CP_THREADS / 32) {
        const long long col = col0 + c;
        if (col < P.N)
          for (int k = lane; k < D; k += 32) __stcs(P.y + col * P.ldy + k, Y[k * CP_LD + c]);
      }
    if (P.logjac && threadIdx.x < CP_TC) {
      const long long col = col0 + threadIdx.x;
      if (col < P.N) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < CP_THREADS / 32; ++w) s += red[w * CP_TC + threadIdx.x];
        P.logjac[col] = (P.accumulate ? P.logjac[col] : 0.f) + s;
      }
    }
  }
}

// the inverse layer: AR_C columns per warp, recovered row by row
__global__ void __launch_bounds__(AR_SEQ_THREADS) ar_inverse_kernel(const __grid_constant__ ArParams P) {
  const long long warps = (long long)gridDim.x * (AR_SEQ_THREADS / 32);
  const long long groups = (P.N + AR_C - 1) / AR_C;
  for (long long g = blockIdx.x * (AR_SEQ_THREADS / 32) + (threadIdx.x >> 5); g < groups; g += warps) {
    const long long col0 = g * AR_C;
    auto load = [&](int c, int r) { return col0 + c < P.N ? __ldcs(P.x + (col0 + c) * P.ldx + r) : 0.f; };
    auto store = [&](int c, int r, float v) {
      if (P.y && col0 + c < P.N) __stcs(P.y + (col0 + c) * P.ldy + r, v);
    };
    float ssum[AR_C];
    ar_recover(P.net, load, store, ssum);  // in place: a 32-row block of y is read before its x is stored
    const int lane = threadIdx.x & 31;
    if (P.logjac && lane < AR_C && col0 + lane < P.N) {
      float s = ssum[0];
#pragma unroll
      for (int c = 1; c < AR_C; ++c)
        if (lane == c) s = ssum[c];
      P.logjac[col0 + lane] = (P.accumulate ? P.logjac[col0 + lane] : 0.f) - s;
    }
  }
}

// ---- reverse mode ---------------------------------------------------------------------------------------------------
struct ArvParams {
  const float* x;
  const float* ybar;
  const float* ljbar;
  float* xbar;
  ArNet net;
  float* part;  // [grid][slice], NULL: no parameter cotangents
  long long N, ldx, ldyb, ldxb, slice;
  long long soff[4];  // offsets of W̄₁, c̄₁, W̄₂, c̄₂ in the slice
  int nsub;
};

// Solves Jᵀw̄ = g for AR_C columns of one sub-tile, rows D..1 (w̄ᵢ needs rows j > i only).  σ′ [H][ld], s and g
// [D][CMV_SP] each, v [D][ld]; w̄ overwrites g.  a_k = σ′_k·Σⱼ ((M₂⊙W₂)[j, k]·vⱼ e^{sⱼ} w̄ⱼ + (M₂⊙W₂)[D+j, k]·w̄ⱼ) over
// the finished rows.
__device__ __forceinline__ void ar_solve(const ArNet& net, const float* dv, const float* v, int ld, float* S, float* G,
                                         int c0) {
  const int lane = threadIdx.x & 31, D = net.D, H = net.H, nj = (H + 31) >> 5;
  float sp[AR_C][AR_UNITS], a[AR_C][AR_UNITS];
#pragma unroll
  for (int j = 0; j < AR_UNITS; ++j) {
    const int k = lane + 32 * j;
#pragma unroll
    for (int c = 0; c < AR_C; ++c) {
      sp[c][j] = j < nj && k < H ? dv[k * ld + c0 + c] : 0.f;
      a[c][j] = 0.f;
    }
  }
  for (int i = D - 1; i >= 0; --i) {
    float dot[AR_C] = {};
#pragma unroll
    for (int j = 0; j < AR_UNITS; ++j)
      if (j < nj) {
        const int k = lane + 32 * j;
        const float w = k < H ? __ldg(net.W1 + (size_t)i * H + k) : 0.f;
#pragma unroll
        for (int c = 0; c < AR_C; ++c) dot[c] = fmaf(w, a[c][j], dot[c]);
      }
    float al[AR_C], wb[AR_C];
#pragma unroll
    for (int c = 0; c < AR_C; ++c) {
      const float e = expf(S[i * CMV_SP + c0 + c]);
      wb[c] = (G[i * CMV_SP + c0 + c] - ar_warp_sum(dot[c])) / e;
      al[c] = v[i * ld + c0 + c] * e * wb[c];
    }
    __syncwarp();
    if (lane < AR_C) {
      float w = wb[0];
#pragma unroll
      for (int c = 1; c < AR_C; ++c)
        if (lane == c) w = wb[c];
      G[i * CMV_SP + c0 + lane] = w;
    }
#pragma unroll
    for (int j = 0; j < AR_UNITS; ++j)
      if (j < nj) {
        const int k = lane + 32 * j;
        const float2 w = k < H ? __ldg(net.W2p + (size_t)i * H + k) : make_float2(0.f, 0.f);
#pragma unroll
        for (int c = 0; c < AR_C; ++c) a[c][j] = fmaf(sp[c][j], fmaf(w.x, al[c], w.y * wb[c]), a[c][j]);
      }
  }
}

template <bool INV>
__global__ void __launch_bounds__(CMV_THREADS, 1) ar_vjp_kernel(const __grid_constant__ ArvParams P) {
  extern __shared__ float arv_sm[];
  const ArNet& net = P.net;
  const int D = net.D, H = net.H, TG = 32 * P.nsub, FP = TG + 1;
  float* V = arv_sm;                   // [D][FP]   v, the layer's input (recovered for the inverse layer)
  float* ST = V + (size_t)D * FP;      // [2D][FP]  ȳ, then s̄ | t̄
  float* Hs = ST + (size_t)2 * D * FP; // [H][FP]   h
  float* Vb = Hs + (size_t)H * FP;     // [H][FP]   σ′(u), then ū
  float* Sc = Vb + (size_t)H * FP;     // [2D][CMV_SP] one sub-tile: x̄ (forward); s, then g -> w̄ (inverse)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float* slice = P.part ? P.part + (size_t)blockIdx.x * P.slice : nullptr;
  if (slice)
    for (long long e = tid; e < P.slice; e += CMV_THREADS) slice[e] = 0.f;
  const bool vec1 = ((H & 7) == 0) && ((reinterpret_cast<uintptr_t>(net.W1) & 15) == 0);
  const bool vec2 = ((D & 3) == 0) && ((reinterpret_cast<uintptr_t>(net.W2) & 15) == 0);
  const bool vec1t = ((H & 3) == 0) && ((reinterpret_cast<uintptr_t>(net.W1) & 15) == 0);
  const bool vec1rt = ((H & 3) == 0) && ((reinterpret_cast<uintptr_t>(net.W1r) & 15) == 0);
  const bool vec2t = ((D & 1) == 0) && ((reinterpret_cast<uintptr_t>(net.W2) & 15) == 0);
  auto same = [](int k) { return k; };

  const long long groups = (P.N + TG - 1) / TG;
  for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
    const long long n0 = g * TG;
    const int gcols = (int)min((long long)TG, P.N - n0);
    for (int co = 0; co < gcols; co += 32) {
      __syncthreads();  // Sc and the previous group's factors are no longer read
      // ---- stage ȳ (and x for the forward layer); the inverse layer recovers x from its input ------------------------
      for (int c = warp; c < 32; c += CMV_THREADS / 32) {
        const long long col = n0 + co + c;
        const bool ok = col < P.N;
        const float* yb = P.ybar && ok ? P.ybar + col * P.ldyb : nullptr;
        for (int k = lane; k < D; k += 32) {
          ST[k * FP + co + c] = yb ? __ldcs(yb + k) : 0.f;
          if (!INV) V[k * FP + co + c] = ok ? __ldcs(P.x + col * P.ldx + k) : 0.f;
        }
      }
      if (INV) {
        const long long col0 = n0 + co + warp * AR_C;
        auto load = [&](int c, int r) { return col0 + c < P.N ? __ldcs(P.x + (col0 + c) * P.ldx + r) : 0.f; };
        auto store = [&](int c, int r, float v) { V[r * FP + co + warp * AR_C + c] = v; };
        float ssum[AR_C];
        ar_recover(net, load, store, ssum);
      }
      __syncthreads();
      // ---- h = σ(u), σ′(u) ---------------------------------------------------------------------------------------
      cmv_hidden(V + co, FP, D, net.W1, net.c1, vec1, H, net.act, net.slope, Hs + co, Vb + co);
      __syncthreads();
      const long long mycol = n0 + co + lane;
      const float lb = P.ljbar && mycol < P.N ? P.ljbar[mycol] : 0.f;
      // ---- s (and t); forward: x̄ of the law, s̄, t̄.  inverse: s, and g = v̄ − l̄·W1rᵀσ′ ------------------------------
      for (int jb = 4 * warp; jb < D; jb += 4 * (CMV_THREADS / 32)) {
        float sv[4][1] = {}, tv[4][1] = {};
        coupling_gemm_block<1>(Hs + co, FP, same, H, net.W2 + jb, net.W2 + D + jb, 2 * D, D - jb, D - jb, vec2, sv, tv);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int j = jb + q;
          if (j < D) {
            const float s_ = sv[q][0] + (net.c2 ? __ldg(net.c2 + j) : 0.f);
            if (!INV) {
              const float e = expf(s_), in = V[j * FP + co + lane], cb = ST[j * FP + co + lane];
              Sc[j * CMV_SP + lane] = e * cb;                // ȳ e^s
              ST[j * FP + co + lane] = fmaf(cb * e, in, lb);  // s̄ = ȳ e^s x + l̄
              ST[(D + j) * FP + co + lane] = cb;             // t̄ = ȳ
            } else {
              Sc[j * CMV_SP + lane] = s_;
            }
          }
        }
      }
      if (INV)
        for (int kb = 8 * warp; kb < D; kb += 8 * (CMV_THREADS / 32)) {
          float acc[8] = {};
          cmv_gemm_t(Vb + co, FP, H, net.W1r + (size_t)kb * H, D - kb, vec1rt, acc);
#pragma unroll
          for (int q = 0; q < 8; ++q)
            if (kb + q < D) Sc[(D + kb + q) * CMV_SP + lane] = fmaf(-lb, acc[q], ST[(kb + q) * FP + co + lane]);
        }
      __syncthreads();
      if (!INV) {
        // ---- ū = ((M₂⊙W₂)ᵀ[s̄; t̄]) ⊙ σ′, then x̄ = ȳ e^s + (M₁⊙W₁)ᵀū -------------------------------------------------
        cmv_back(ST + co, FP, 2 * D, net.W2, vec2t, H, Vb + co);
        __syncthreads();
        for (int kb = 8 * warp; kb < D; kb += 8 * (CMV_THREADS / 32)) {
          float acc[8] = {};
          cmv_gemm_t(Vb + co, FP, H, net.W1 + (size_t)kb * H, D - kb, vec1t, acc);
#pragma unroll
          for (int q = 0; q < 8; ++q)
            if (kb + q < D) Sc[(kb + q) * CMV_SP + lane] += acc[q];
        }
        __syncthreads();
        for (int c = warp; c < 32; c += CMV_THREADS / 32) {
          const long long col = n0 + co + c;
          if (col < P.N)
            for (int k = lane; k < D; k += 32) __stcs(P.xbar + col * P.ldxb + k, Sc[k * CMV_SP + c]);
        }
      } else {
        // ---- w̄ = J⁻ᵀ g, row by row; x̄ = w̄ ----------------------------------------------------------------------
        ar_solve(net, Vb + co, V + co, FP, Sc, Sc + D * CMV_SP, warp * AR_C);
        __syncthreads();
        for (int c = warp; c < 32; c += CMV_THREADS / 32) {
          const long long col = n0 + co + c;
          if (col < P.N)
            for (int k = lane; k < D; k += 32) __stcs(P.xbar + col * P.ldxb + k, Sc[(D + k) * CMV_SP + c]);
        }
        if (slice) {  // [s̄; t̄] = −[w̄ ⊙ v ⊙ eˢ + l̄; w̄], then ū = ((M₂⊙W₂)ᵀ[s̄; t̄]) ⊙ σ′
          for (int j = warp; j < D; j += CMV_THREADS / 32) {
            const float wb = Sc[(D + j) * CMV_SP + lane], e = expf(Sc[j * CMV_SP + lane]);
            ST[j * FP + co + lane] = -fmaf(wb * e, V[j * FP + co + lane], lb);
            ST[(D + j) * FP + co + lane] = -wb;
          }
          __syncthreads();
          cmv_back(ST + co, FP, 2 * D, net.W2, vec2t, H, Vb + co);
        }
      }
    }
    if (slice) {  // the group's parameter sums, added to the CTA's slice
      __syncthreads();
      cmv_outer(Vb, H, V, D, FP, gcols, slice + P.soff[0], slice + P.soff[1]);
      cmv_outer(ST, 2 * D, Hs, H, FP, gcols, slice + P.soff[2], slice + P.soff[3]);
    }
  }
}

// The slices summed in order, in fp64; W̄ entries outside the masks are written as exact zeros.  Slice layout: W̄₁ (H·D),
// c̄₁ (H), W̄₂ (2D·H), c̄₂ (2D).
__global__ void __launch_bounds__(256) ar_vjp_reduce_kernel(const float* __restrict__ part, int nparts, long long slice,
                                                            const int* __restrict__ deg, int D, int H,
                                                            float* __restrict__ o0, float* __restrict__ o1,
                                                            float* __restrict__ o2, float* __restrict__ o3) {
  const long long l0 = (long long)H * D, l1 = H, l2 = 2LL * D * H, l3 = 2LL * D;
  const long long e0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e0 >= l0 + l1 + l2 + l3) return;
  long long e = e0;
  float* o;
  bool on = true;
  if (e < l0) {
    o = o0;
    on = e / H + 1 <= deg[e % H];
  } else if ((e -= l0) < l1) {
    o = o1;
  } else if ((e -= l1) < l2) {
    o = o2;
    on = deg[e / (2 * D)] < (e % (2 * D)) % D + 1;
  } else {
    e -= l2;
    o = o3;
  }
  if (!o) return;
  double t = 0.0;
  for (int g = 0; g < nparts && on; ++g) t += (double)part[(size_t)g * slice + e0];
  o[e] = on ? (float)t : 0.f;
}

static long long arv_slice_floats(int D, int H) { return (3LL * H * D + H + 2LL * D + 63) & ~63LL; }

static size_t arv_smem_bytes(int D, int H, int nsub) {
  return ((size_t)(3 * D + 2 * H) * (32 * nsub + 1) + (size_t)2 * D * CMV_SP) * sizeof(float);
}

// sub-tiles per group: the most whose factors fit the 227 KB a CTA may use
static int arv_nsub(int D, int H) {
  for (int s = 4; s > 1; s >>= 1)
    if (arv_smem_bytes(D, H, s) <= 227 * 1024) return s;
  return 1;
}

static int arv_grid(int D, int H, long long N) {
  long long g = b2b_sm_count();
  const long long groups = (N + 32 * arv_nsub(D, H) - 1) / (32 * arv_nsub(D, H));
  if (g > groups) g = groups;
  return g < 1 ? 1 : (int)g;
}

static ArNet ar_net(const B2BCoupling<b2b_layer_desc>& c, const ArWs& w, int D) {
  ArNet n;
  n.W1 = w.W1;
  n.c1 = c.c_in;
  n.W2 = w.W2;
  n.c2 = c.c_out;
  n.W2p = w.W2p;
  n.W1r = w.W1r;
  n.deg = c.degrees;
  n.D = D;
  n.H = c.H;
  n.act = c.act;
  n.slope = c.slope;
  return n;
}

}  // namespace b2b

bool b2b_ar_fits(const b2b_layer_desc& d, int D) {
  return D >= 1 && D <= B2B_AUTOREGRESSIVE_MLP_MAX_D && d.n2 >= 1 && d.n2 <= B2B_AUTOREGRESSIVE_MLP_MAX_H;
}

size_t b2b_ar_workspace(const b2b_layer_desc& d, int D) {
  return b2b_ar_fits(d, D) ? b2b::ar_ws(nullptr, D, d.n2, false).bytes : 0;
}

size_t b2b_ar_vjp_workspace(const b2b_layer_desc& d, int D, long long N) {
  using namespace b2b;
  if (!b2b_ar_fits(d, D)) return 0;
  const int H = d.n2;
  return ar_ws(nullptr, D, H, true).bytes + (size_t)arv_grid(D, H, N) * (size_t)arv_slice_floats(D, H) * sizeof(float);
}

int b2b_fwd_ar(const B2BFwdSeg& s) {
  using namespace b2b;
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  if (!b2b_ar_fits(d, D)) return B2B_EUNSUPPORTED;
  if (!s.workspace || s.workspace_bytes < b2b_ar_workspace(d, D)) return B2B_EWORKSPACE;
  const B2BCoupling<b2b_layer_desc> c = b2b_coupling(d, D);
  const ArWs w = ar_ws(s.workspace, D, c.H, false);
  int rc = ar_prep(c, w, D, s.stream);
  if (rc != B2B_OK) return rc;
  ++*s.launches;
  ArParams P;
  P.x = s.x;
  P.y = s.y;
  P.logjac = s.logjac;
  P.net = ar_net(c, w, D);
  P.N = s.N;
  P.ldx = s.ldx;
  P.ldy = s.ldy;
  P.accumulate = s.accumulate;
  void (*kernel)(const ArParams) = d.inverse ? ar_inverse_kernel : ar_forward_kernel;
  const int threads = d.inverse ? AR_SEQ_THREADS : CP_THREADS;
  const size_t smem = d.inverse ? 0 : ((size_t)(2 * D + c.H) * CP_LD + 8 * CP_TC) * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  int per_sm = 0;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem)) != cudaSuccess) return (int)e;
  if (per_sm < 1) per_sm = 1;
  const long long cols = d.inverse ? AR_C * (AR_SEQ_THREADS / 32) : CP_TC;  // columns per CTA and step
  const long long blocks = (s.N + cols - 1) / cols;
  long long grid = (long long)b2b_sm_count() * per_sm;
  if (grid > blocks) grid = blocks;
  kernel<<<(int)grid, threads, smem, s.stream>>>(P);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*s.launches;
  return B2B_OK;
}

int b2b_vjp_ar(const B2BVjpSeg& s) {  // the four sums come from one kernel: those not asked for are dropped
  using namespace b2b;
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  const long long N = s.N;
  float* const* bars = s.bars;
  if (!b2b_ar_fits(d, D)) return B2B_EUNSUPPORTED;
  const B2BCoupling<b2b_layer_desc> c = b2b_coupling(d, D);
  const int H = c.H;
  const bool want = bars[0] || bars[1] || bars[2] || bars[3];
  if (!s.workspace || s.workspace_bytes < b2b_ar_vjp_workspace(d, D, N)) return B2B_EWORKSPACE;
  const ArWs w = ar_ws(s.workspace, D, H, d.inverse != 0);
  int rc = ar_prep(c, w, D, s.stream);
  if (rc != B2B_OK) return rc;
  ++*s.launches;
  ArvParams P;
  P.x = s.x;
  P.ybar = s.ybar;
  P.ljbar = s.ljbar;
  P.xbar = s.xbar;
  P.net = ar_net(c, w, D);
  P.part = want ? reinterpret_cast<float*>(reinterpret_cast<char*>(b2b_align256(s.workspace)) + w.bytes - 256) : nullptr;
  P.N = N;
  P.ldx = s.ldx;
  P.ldyb = s.ldyb;
  P.ldxb = s.ldxb;
  P.slice = arv_slice_floats(D, H);
  P.soff[0] = 0;
  P.soff[1] = (long long)H * D;
  P.soff[2] = P.soff[1] + H;
  P.soff[3] = P.soff[2] + 2LL * D * H;
  P.nsub = arv_nsub(D, H);
  const int grid = arv_grid(D, H, N);
  const size_t smem = arv_smem_bytes(D, H, P.nsub);
  void (*kernel)(const ArvParams) = d.inverse ? ar_vjp_kernel<true> : ar_vjp_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<grid, CMV_THREADS, smem, s.stream>>>(P);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*s.launches;
  if (want) {
    const long long total = P.soff[3] + 2LL * D;
    ar_vjp_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s.stream>>>(P.part, grid, P.slice, c.degrees, D, H,
                                                                                 bars[0], bars[1], bars[2], bars[3]);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    ++*s.launches;
  }
  return B2B_OK;
}
