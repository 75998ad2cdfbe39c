// Reverse mode of the neural-network coupling layers, B2B_COUPLING_MLP and B2B_COUPLING_DEEP_MLP, either direction:
// cotangents of the input and of every weight and bias -- what the reference's reverse-mode AD computes through
// coupling.jl:206-228 with the law Shift(t) ∘ Scale(exp.(s)) and the network of b2b_coupling_mlp.cu, M hidden layers
// (M = 1 for B2B_COUPLING_MLP), h_0 = x₂, W_1 = W_in.  With h_l = σ(v_l) and the affine law's s̄, t̄, x̄₁ (formed as
// b2b_coupling_vjp.cu forms them):
//   v̄_M = (W_outᵀ[s̄; t̄]) ⊙ σ′_M     v̄_{l−1} = (W_lᵀ v̄_l) ⊙ σ′_{l−1}     x̄₂ = ȳ₂ + W_inᵀ v̄_1     x̄₃ = ȳ₃
//   W̄_out = Σₙ [s̄; t̄] h_Mᵀ   c̄_out = Σₙ [s̄; t̄]   W̄_l = Σₙ v̄_l h_{l−1}ᵀ   c̄_l = Σₙ v̄_l
//
// Mapping.  A fixed grid of at most one CTA per SM walks groups of 32·S columns round-robin (S = 4, 2 or 1 sub-tiles,
// the most whose factors fit shared memory: S = 2 at n1 = n2 = 128, H = 256, M = 1).  Each sub-tile of 32 columns (one
// per lane) runs the network forward and backward with coupling_gemm_block and its transposed counterpart, leaving x₂,
// [s̄; t̄] and h_l, v̄_l of every layer of its columns in shared memory.  After the group's last sub-tile the CTA forms the
// parameter sums of the whole group, a 4 x 4 register block per thread swept over the matrices, and adds them to its
// private slice of the workspace (the descriptor's four slots back to back, each role at the offset the host gives it;
// every element always by the same thread): one read-modify-write of the slice per 32·S columns.  A second kernel sums
// the slices in order, in fp64, into the caller's arrays.  Deterministic, no atomics; the workspace depends on the
// grid, not on N.
#include <cuda_runtime.h>

#include "b2b_coupling_mlp.cuh"
#include "b2b_coupling_net.cuh"
#include "b2b_coupling_tile.cuh"
#include "b2b_internal.h"

namespace b2b {

struct CmvParams {
  const float* x;
  const float* ybar;
  const float* ljbar;
  float* xbar;
  const float *W1, *c1, *W2, *c2;  // W_in, [c_1 | … | c_M] (or NULL), W_out, c_out
  const int *idx1, *idx2;
  float* part;  // [grid][slice], NULL: no parameter cotangents
  long long N, ldx, ldyb, ldxb, slice;
  long long soff[B2B_NROLES];  // offset of each B2BRole's sums in the slice
  int D, n1, n2, H, act, nsub;
  float slope;
  const float* Wh;  // W_2 .. W_M, each H x H column-major, back to back
  int depth;        // M hidden layers
};

template <bool INV>
__global__ void __launch_bounds__(CMV_THREADS, 1) coupling_mlp_vjp_kernel(const __grid_constant__ CmvParams P) {
  extern __shared__ float cmv_sm[];
  const int D = P.D, n1 = P.n1, n2 = P.n2, H = P.H, TG = 32 * P.nsub, FP = TG + 1, nmax = max(n1, n2);
  const int M = P.depth;
  const size_t HB = (size_t)H * FP;     // one hidden block
  float* X2 = cmv_sm;                   // [n2][FP]   x₂
  float* ST = X2 + (size_t)n2 * FP;     // [2n1][FP]  ȳ₁, then s̄ | t̄
  float* Hs = ST + (size_t)2 * n1 * FP; // [M][H][FP] h_l
  float* Vb = Hs + M * HB;              // [M][H][FP] σ′(v_l), then v̄_l
  float* Sc = Vb + M * HB;              // [max(n1, n2)][33]  one sub-tile: x₁ -> x̄₁, then W₁ᵀ v̄
  const float* hM = Hs + (M - 1) * HB;  // h_M, the input of W_out
  int* sidx1 = reinterpret_cast<int*>(Sc + (size_t)nmax * CMV_SP);  // [n1]
  int* sidx2 = sidx1 + n1;                                          // [n2]
  unsigned char* kind = reinterpret_cast<unsigned char*>(sidx2 + n2);  // [D]: 0 = a pass-through row
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float* slice = P.part ? P.part + (size_t)blockIdx.x * P.slice : nullptr;

  for (int r = tid; r < D; r += CMV_THREADS) kind[r] = 0;
  if (slice)
    for (long long e = tid; e < P.slice; e += CMV_THREADS) slice[e] = 0.f;
  __syncthreads();
  for (int i = tid; i < n1; i += CMV_THREADS) kind[sidx1[i] = P.idx1[i]] = 1;
  for (int k = tid; k < n2; k += CMV_THREADS) kind[sidx2[k] = P.idx2[k]] = 2;
  const bool vec1 = ((H & 7) == 0) && ((reinterpret_cast<uintptr_t>(P.W1) & 15) == 0);
  const bool vec2 = ((n1 & 3) == 0) && ((reinterpret_cast<uintptr_t>(P.W2) & 15) == 0);
  const bool vec1t = ((H & 3) == 0) && ((reinterpret_cast<uintptr_t>(P.W1) & 15) == 0);
  const bool vec2t = ((n1 & 1) == 0) && ((reinterpret_cast<uintptr_t>(P.W2) & 15) == 0);
  const bool vech = ((H & 7) == 0) && ((reinterpret_cast<uintptr_t>(P.Wh) & 15) == 0);
  const bool vecht = ((H & 3) == 0) && ((reinterpret_cast<uintptr_t>(P.Wh) & 15) == 0);
  auto same = [](int k) { return k; };

  const long long groups = (P.N + TG - 1) / TG;
  for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
    const long long n0 = g * TG;
    const int gcols = (int)min((long long)TG, P.N - n0);
    for (int co = 0; co < gcols; co += 32) {
      __syncthreads();  // index tables visible; Sc and the factors of the previous group are no longer read
      // ---- stage x₂, x₁, ȳ₁ of the sub-tile; x̄₃ = ȳ₃ goes straight out --------------------------------------------
      for (int c = warp; c < 32; c += CMV_THREADS / 32) {
        const long long col = n0 + co + c;
        const bool ok = col < P.N;
        const float* xc = P.x + col * P.ldx;
        const float* yb = P.ybar ? P.ybar + col * P.ldyb : nullptr;
        for (int k = lane; k < n2; k += 32) X2[k * FP + co + c] = ok ? __ldcs(xc + sidx2[k]) : 0.f;
        for (int k = lane; k < n1; k += 32) {
          Sc[k * CMV_SP + c] = ok ? __ldcs(xc + sidx1[k]) : 0.f;
          ST[k * FP + co + c] = ok && yb ? __ldcs(yb + sidx1[k]) : 0.f;
        }
        if (ok && n1 + n2 < D)
          for (int r = lane; r < D; r += 32)
            if (!kind[r]) __stcs(P.xbar + col * P.ldxb + r, yb ? __ldcs(yb + r) : 0.f);
      }
      __syncthreads();
      // ---- h_l = σ(W_l h_{l−1} + c_l) and σ′_l, l = 1..M ---------------------------------------------------------
      for (int l = 1; l <= M; ++l) {
        cmv_hidden(l == 1 ? X2 + co : Hs + (l - 2) * HB + co, FP, l == 1 ? n2 : H,
                   l == 1 ? P.W1 : P.Wh + (size_t)(l - 2) * H * H, P.c1 ? P.c1 + (size_t)(l - 1) * H : nullptr,
                   l == 1 ? vec1 : vech, H, P.act, P.slope, Hs + (l - 1) * HB + co, Vb + (l - 1) * HB + co);
        __syncthreads();
      }
      // ---- [s; t] = W_out h_M + c_out, then x̄₁, s̄, t̄ of the affine law --------------------------------------------
      const long long mycol = n0 + co + lane;
      const float lb = P.ljbar && mycol < P.N ? P.ljbar[mycol] : 0.f;
      for (int jb = 4 * warp; jb < n1; jb += 4 * (CMV_THREADS / 32)) {
        float sv[4][1] = {}, tv[4][1] = {};
        coupling_gemm_block<1>(hM + co, FP, same, H, P.W2 + jb, P.W2 + n1 + jb, 2 * n1, n1 - jb, n1 - jb, vec2, sv, tv);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int j = jb + q;
          if (j < n1) {
            const float s_ = sv[q][0] + (P.c2 ? __ldg(P.c2 + j) : 0.f), t_ = tv[q][0] + (P.c2 ? __ldg(P.c2 + n1 + j) : 0.f);
            const float in1 = Sc[j * CMV_SP + lane], cb1 = ST[j * FP + co + lane];
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
            Sc[j * CMV_SP + lane] = out1;
            ST[j * FP + co + lane] = sbar;
            ST[(n1 + j) * FP + co + lane] = tbar;
          }
        }
      }
      __syncthreads();
      for (int c = warp; c < 32; c += CMV_THREADS / 32) {
        const long long col = n0 + co + c;
        if (col < P.N)
          for (int k = lane; k < n1; k += 32) __stcs(P.xbar + col * P.ldxb + sidx1[k], Sc[k * CMV_SP + c]);
      }
      // ---- v̄_M = (W_outᵀ[s̄; t̄]) ⊙ σ′_M, then v̄_{l−1} = (W_lᵀ v̄_l) ⊙ σ′_{l−1}, l = M..2 ---------------------------
      cmv_back(ST + co, FP, 2 * n1, P.W2, vec2t, H, Vb + (M - 1) * HB + co);
      __syncthreads();
      for (int l = M - 1; l >= 1; --l) {
        cmv_back(Vb + l * HB + co, FP, H, P.Wh + (size_t)(l - 1) * H * H, vecht, H, Vb + (l - 1) * HB + co);
        __syncthreads();
      }
      // ---- x̄₂ = ȳ₂ + W_inᵀ v̄_1 ------------------------------------------------------------------------------------
      for (int kb = 8 * warp; kb < n2; kb += 8 * (CMV_THREADS / 32)) {
        float acc[8] = {};
        cmv_gemm_t(Vb + co, FP, H, P.W1 + (size_t)kb * H, n2 - kb, vec1t, acc);
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (kb + q < n2) Sc[(kb + q) * CMV_SP + lane] = acc[q];
      }
      __syncthreads();
      for (int c = warp; c < 32; c += CMV_THREADS / 32) {
        const long long col = n0 + co + c;
        if (col < P.N)
          for (int k = lane; k < n2; k += 32) {
            const float yb = P.ybar ? __ldcs(P.ybar + col * P.ldyb + sidx2[k]) : 0.f;
            __stcs(P.xbar + col * P.ldxb + sidx2[k], yb + Sc[k * CMV_SP + c]);
          }
      }
    }
    if (slice) {  // the group's parameter sums, added to the CTA's slice
      __syncthreads();
      float* const sc = slice + P.soff[B2B_C_IN];  // c̄_1 .. c̄_M
      cmv_outer(Vb, H, X2, n2, FP, gcols, slice + P.soff[B2B_W_IN], sc);
      for (int l = 1; l < M; ++l)
        cmv_outer(Vb + l * HB, H, Hs + (l - 1) * HB, H, FP, gcols, slice + P.soff[B2B_W_HID] + (size_t)(l - 1) * H * H,
                  sc + (size_t)l * H);
      cmv_outer(ST, 2 * n1, hM, H, FP, gcols, slice + P.soff[B2B_W_OUT], slice + P.soff[B2B_C_OUT]);
    }
  }
}

// the `nparts` slices summed in order; element e of the slice layout (the four slots back to back, of lengths l0 .. l3)
// goes to its array (NULL: dropped)
__global__ void __launch_bounds__(256) coupling_mlp_vjp_reduce_kernel(const float* __restrict__ part, int nparts, long long slice,
                                                                      long long l0, long long l1, long long l2, long long l3,
                                                                      float* __restrict__ o0, float* __restrict__ o1,
                                                                      float* __restrict__ o2, float* __restrict__ o3) {
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= l0 + l1 + l2 + l3) return;
  double t = 0.0;
  for (int g = 0; g < nparts; ++g) t += (double)part[(size_t)g * slice + e];
  float* o = o0;
  if (e >= l0) { e -= l0; o = o1;
    if (e >= l1) { e -= l1; o = o2;
      if (e >= l2) { e -= l2; o = o3; } } }
  if (o) o[e] = (float)t;
}

static long long cmv_param_floats(const b2b_layer_desc& d) {
  long long n = 0;
  for (int i = 0; i < 4; ++i) n += (long long)b2b_slot_len(d, i, 0);
  return n;
}
static long long cmv_slice_floats(const b2b_layer_desc& d) { return (cmv_param_floats(d) + 63) & ~63LL; }

// the kernel keeps the factors of every hidden layer
static size_t cmv_smem_bytes(const b2b_layer_desc& d, int D, int nsub) {
  const B2BCoupling<b2b_layer_desc> c = b2b_coupling(d);
  const size_t f = (size_t)(c.n2 + 2 * c.n1 + 2 * c.M * c.H) * (32 * nsub + 1) + (size_t)(c.n1 > c.n2 ? c.n1 : c.n2) * CMV_SP;
  return (f * sizeof(float) + (size_t)(c.n1 + c.n2) * sizeof(int) + D + 15) & ~(size_t)15;
}

// sub-tiles per group: the most whose factors fit the 227 KB a CTA may use
static int cmv_nsub(const b2b_layer_desc& d, int D) {
  for (int s = 4; s > 1; s >>= 1)
    if (cmv_smem_bytes(d, D, s) <= 227 * 1024) return s;
  return 1;
}

static int cmv_grid(const b2b_layer_desc& d, int D, long long N) {
  const int sms = b2b_sm_count();
  long long g = sms;
  const long long groups = (N + 32 * cmv_nsub(d, D) - 1) / (32 * cmv_nsub(d, D));
  if (g > groups) g = groups;
  const long long cap = (256LL << 20) / (cmv_slice_floats(d) * (long long)sizeof(float));
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

}  // namespace b2b

size_t b2b_coupling_mlp_vjp_workspace(const b2b_layer_desc& d, int D, long long N) {
  using namespace b2b;
  if (!b2b_coupling_fits(d, D)) return 0;
  return (size_t)cmv_grid(d, D, N) * (size_t)cmv_slice_floats(d) * sizeof(float) + 256;
}

int b2b_vjp_mlp(const B2BVjpSeg& s) {  // the four sums come from one kernel: those not asked for are dropped
  using namespace b2b;
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  const long long N = s.N;
  float* const* bars = s.bars;
  if (!b2b_coupling_fits(d, D)) return B2B_EUNSUPPORTED;
  const B2BCoupling<b2b_layer_desc> c = b2b_coupling(d);
  const bool want = bars[0] || bars[1] || bars[2] || bars[3];
  if (want && (!s.workspace || s.workspace_bytes < b2b_coupling_mlp_vjp_workspace(d, D, N))) return B2B_EWORKSPACE;
  char* wsb = b2b_align256(s.workspace);
  CmvParams P;
  P.x = s.x;
  P.ybar = s.ybar;
  P.ljbar = s.ljbar;
  P.xbar = s.xbar;
  P.W1 = c.W_in;
  P.c1 = c.c_in;
  P.Wh = c.W_hid;
  P.W2 = c.W_out;
  P.c2 = c.c_out;
  P.depth = c.M;
  P.act = c.act;
  P.idx1 = c.idx1;
  P.idx2 = c.idx2;
  P.part = want ? reinterpret_cast<float*>(wsb) : nullptr;
  P.N = N;
  P.ldx = s.ldx;
  P.ldyb = s.ldyb;
  P.ldxb = s.ldxb;
  P.slice = cmv_slice_floats(d);
  long long l[4], so[4] = {};  // the slots' lengths and offsets in the slice
  for (int i = 0; i < 4; ++i) {
    l[i] = (long long)b2b_slot_len(d, i, D);
    if (i) so[i] = so[i - 1] + l[i - 1];
  }
  for (int r = 0; r < B2B_NROLES; ++r) P.soff[r] = c.slot[r] < 0 ? 0 : so[c.slot[r]] + (long long)c.off[r];
  P.D = D;
  P.n1 = c.n1;
  P.n2 = c.n2;
  P.H = c.H;
  P.nsub = cmv_nsub(d, D);
  P.slope = c.slope;
  const int grid = cmv_grid(d, D, N);
  const size_t smem = cmv_smem_bytes(d, D, P.nsub);
  void (*kernel)(const CmvParams) = d.inverse ? coupling_mlp_vjp_kernel<true> : coupling_mlp_vjp_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<grid, CMV_THREADS, smem, s.stream>>>(P);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*s.launches;
  if (want) {
    float* o[4] = {bars[0], bars[1], bars[2], bars[3]};
    coupling_mlp_vjp_reduce_kernel<<<(unsigned)((l[0] + l[1] + l[2] + l[3] + 255) / 256), 256, 0, s.stream>>>(
        P.part, grid, P.slice, l[0], l[1], l[2], l[3], o[0], o[1], o[2], o[3]);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    ++*s.launches;
  }
  return B2B_OK;
}
