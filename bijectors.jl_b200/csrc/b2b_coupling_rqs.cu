// Spline coupling layer, B2B_COUPLING_RQS (include/b2b.h): Coupling(x₂ -> RationalQuadraticSpline(…, B), mask)
// (coupling.jl:206-228 with the normalising constructor rational_quadratic_spline.jl:109-123), forward and inverse, in
// exact fp32 on the CUDA cores.
//
// Mapping.  A CTA owns a tile of CRQ_TN columns, one thread per column.  It stages the tile's x₂ rows in shared memory
// ([m][column], padded pitch: conflict-free both ways), then walks the n1 transformed rows in order.  For each row i it
// streams that row's (3K − 1) x n2 block of W through shared memory (W itself is up to 1.5 MB), and every thread forms its
// column's 3K − 1 raw parameters with an FMA GEMM over x₂, normalises them into K + 1 knots, builds the per-bin constants
// of rqs_element in a table row of its own, and evaluates the element with rqs_element (b2b_device.cuh), the same element
// function the fused RQS programs use.  The log-Jacobian is summed over the rows in increasing order by the column's
// thread, so it is deterministic.  x₂ and x₃ rows are copied bit-exactly (nothing is copied in place).
//
// The neural spline couplings, B2B_COUPLING_MLP_RQS and B2B_COUPLING_DEEP_MLP_RQS, are the instantiation NET = true:
// v = W_out·h_M + c_out with M hidden layers h_l = σ(W_l·h_{l−1} + c_l), h_0 = x₂, W_1 = W_in (M = 1 for
// B2B_COUPLING_MLP_RQS).  Each thread forms the layers of its own column before the row loop, which runs unchanged
// with (x₂, n2, W, c) := (h_M, H, W_out, c_out).  The layers alternate between the [H][XP] h block the row loop reads
// and the table region, where the rqs_element table and W's row block will be (neither is written before the row loop;
// x₂ spills past them only when they are smaller than x₂, at small K).  x₂ is staged in the table region when M is odd
// and in the h block when M is even, so that h_M lands in the h block.  For M >= 2 both blocks hold max(n2, H) rows,
// so the shared memory is that of M = 1 with n2 := max(n2, H).
#include <cuda_runtime.h>

#include "b2b_coupling_mlp.cuh"
#include "b2b_coupling_rqs.cuh"
#include "b2b_device.cuh"
#include "b2b_internal.h"

namespace b2b {

constexpr int CRQ_TN = 128;

struct CrqParams {
  const float* x;
  float* y;
  float* logjac;
  const float *W, *c;  // NET: W_out, c_out
  const int *idx1, *idx2;
  long long N, ldx, ldy;
  int D, n1, n2, K, accumulate;
  float B;
  const float *W1, *c1;  // NET only: W_in, [c_1 | … | c_M] (or NULL)
  int H, act;
  float slope;
  const float* Wh;  // NET: W_2 .. W_M, each H x H column-major, back to back
  int M;            // NET: hidden layers
};

// floats of the per-thread rqs_element table: Sw[KP] | Sh[KP] | 2 float4 per bin
static __host__ __device__ inline int crq_tab_floats(int K) { return 2 * rqs_kp(K + 1) + 8 * (K + 1); }

// float offset of the conditioning block Xs: after the table, W's row block and c; with the network (n2x = n2 rows of x₂
// staged from offset 0) at least past x₂
static __host__ __device__ inline int crq_xs_off(int nc, int K, int n2x) {
  const int off = crq_tab_floats(K) * CRQ_TN + nc * crq_jp(K) + crq_jp(K);
  return off > n2x * (CRQ_TN + 1) ? off : n2x * (CRQ_TN + 1);
}

template <bool INV, bool NET>
__global__ void __launch_bounds__(CRQ_TN) coupling_rqs_kernel(const __grid_constant__ CrqParams P) {
  extern __shared__ __align__(16) float crq_sm[];
  constexpr int TN = CRQ_TN, XP = CRQ_TN + 1;
  // nc: rows of the conditioning block the row loop reads (x₂, or the hidden layer h)
  const int tid = threadIdx.x, n1 = P.n1, n2 = P.n2, nc = NET ? P.H : n2, K = P.K, K1 = K + 1, KP = rqs_kp(K1);
  const int J = 3 * K - 1, JP = crq_jp(K), D = P.D;
  float* tab = crq_sm;                              // rqs_element table, one row per thread (Dp = TN)
  float* Ws = tab + crq_tab_floats(K) * TN;         // [nc][JP]
  float* cs = Ws + nc * JP;                         // [JP]
  const bool deep = NET && P.M > 1;                // h_l and x₂ alternate between Xs and the table region
  const int nxs = deep ? max(n2, nc) : nc;          // rows of the Xs block
  float* Xs = NET ? crq_sm + crq_xs_off(nc, K, deep ? nxs : n2) : cs + JP;  // [nc][XP]
  float* X2 = NET && P.M % 2 == 1 ? crq_sm : Xs;   // [n2][XP] x₂
  float* Pr = Xs + nxs * XP;                        // [J][TN] raw parameters
  unsigned char* x1row = reinterpret_cast<unsigned char*>(Pr + J * TN);  // [D]: 1 = a transformed row
  const long long n0 = (long long)blockIdx.x * TN, n = n0 + tid;
  const int cols = (int)min((long long)TN, P.N - n0);
  const bool active = tid < cols;

  for (int r = tid; r < D; r += TN) x1row[r] = 0;
  __syncthreads();
  for (int i = tid; i < n1; i += TN) x1row[P.idx1[i]] = 1;
  for (int e = tid; e < n2 * TN; e += TN) {
    const int c = e / n2, m = e - c * n2;
    X2[m * XP + c] = c < cols ? P.x[(n0 + c) * P.ldx + P.idx2[m]] : 0.f;
  }
  __syncthreads();
  if (NET) {  // h_1 .. h_M of this thread's column, alternating between the two blocks and ending in Xs
    const int H = P.H;
    float* in = X2;
    for (int l = 1; l <= P.M; ++l) {
      float* out = in == Xs ? crq_sm : Xs;
      const float* W = l == 1 ? P.W1 : P.Wh + (size_t)(l - 2) * H * H;
      const float* c = P.c1 ? P.c1 + (size_t)(l - 1) * H : nullptr;
      for (int m = 0; m < H; ++m) {
        float dh;
        mlp_act(P.act, P.slope, crq_hidden_pre(W, c, H, l == 1 ? n2 : H, in + tid, XP, m), out[m * XP + tid], dh);
      }
      in = out;
    }
  }
  if (P.y && (P.y != P.x || P.ldy != P.ldx))  // x₂ and x₃ pass through
    for (int e = tid; e < cols * D; e += TN) {
      const int c = e / D, r = e - c * D;
      if (!x1row[r]) P.y[(n0 + c) * P.ldy + r] = P.x[(n0 + c) * P.ldx + r];
    }

  float* Sw = tab + tid * KP;
  float* Sh = tab + TN * KP + tid * KP;
  float4* cf = reinterpret_cast<float4*>(tab + 2 * TN * KP) + tid * K1 * 2;
  const float inf = __int_as_float(0x7f800000);
  float lj = 0.f;
  for (int i = 0; i < n1; ++i) {
    __syncthreads();  // the previous row's block of W is no longer read
    crq_stage_row(P.W, P.c, i, n1, nc, K, Ws, cs, tid, TN);
    __syncthreads();
    crq_params(Ws, cs, Xs + tid, XP, nc, K, Pr + tid, TN);
    crq_knots(Pr + tid, TN, K, P.B, Sw, 1);
    crq_knots(Pr + K * TN + tid, TN, K, P.B, Sh, 1);
    for (int k = K1; k < KP; ++k) Sw[k] = Sh[k] = inf;
    // per-bin constants, as stage_layer(B2B_RQS) computes them from the processed arrays (derivatives: 1, log1pexp, 1)
    const float Wl = Sw[K], Hl = Sh[K];
    float dprev = 1.f;
    for (int k = 0; k < K1; ++k) {
      const float dcur = (k == 0 || k == K) ? 1.0f : softplus(Pr[(2 * K + k - 1) * TN + tid]);
      const float w_k = k == 0 ? -Wl : Sw[k - 1], w = Sw[k] - w_k;
      const float h_k = k == 0 ? -Hl : Sh[k - 1], dy = Sh[k] - h_k;
      const float d_k = k == 0 ? 1.0f : dprev, d_k1 = dcur;
      const float sl = dy / w;
      cf[2 * k + 0] = make_float4(w_k, 1.0f / w, w, h_k);
      cf[2 * k + 1] = make_float4(dy, sl, d_k, d_k1 + d_k - 2.0f * sl);
      dprev = dcur;
    }
    if (active) {
      const int row = P.idx1[i];
      float out, l;
      rqs_element<INV>(tab, K1, KP, TN, tid, P.x[n * P.ldx + row], out, l);
      if (P.y) P.y[n * P.ldy + row] = out;
      lj += l;
    }
  }
  if (active && P.logjac) P.logjac[n] = P.accumulate ? P.logjac[n] + lj : lj;
}

// nc conditioning rows; with the network, n2x = n2 rows of x₂ staged before the row loop; nxs rows of the Xs block
static size_t crq_smem_bytes(int nc, int K, int D, int n2x, int nxs) {
  const size_t f = (size_t)crq_xs_off(nc, K, n2x) + (size_t)nxs * (CRQ_TN + 1) + (size_t)(3 * K - 1) * CRQ_TN;
  return (f * sizeof(float) + D + 15) & ~(size_t)15;
}

}  // namespace b2b

int b2b_fwd_spline(const B2BFwdSeg& s) {
  using namespace b2b;
  const b2b_layer_desc& d = s.layers[0];
  if (!b2b_coupling_fits(d, s.D)) return B2B_EUNSUPPORTED;
  const B2BCoupling<b2b_layer_desc> c = b2b_coupling(d);
  CrqParams P = {};
  P.x = s.x;
  P.y = s.y;
  P.logjac = s.logjac;
  P.W = c.W_out;
  P.c = c.c_out;
  P.W1 = c.W_in;
  P.c1 = c.c_in;
  P.idx1 = c.idx1;
  P.idx2 = c.idx2;
  P.N = s.N;
  P.ldx = s.ldx;
  P.ldy = s.ldy;
  P.D = s.D;
  P.n1 = c.n1;
  P.n2 = c.n2;
  P.K = c.K;
  P.H = c.H;
  P.act = c.act;
  P.accumulate = s.accumulate;
  P.B = c.B;
  P.slope = c.slope;
  P.Wh = c.W_hid;
  P.M = c.M;
  const int nd = c.n2 > c.H ? c.n2 : c.H;  // M >= 2: max(n2, H)
  const size_t smem = c.M > 1 ? crq_smem_bytes(c.H, c.K, s.D, nd, nd)
                      : c.net ? crq_smem_bytes(c.H, c.K, s.D, c.n2, c.H)
                              : crq_smem_bytes(c.n2, c.K, s.D, 0, c.n2);
  void (*kernel)(const CrqParams) = c.net ? (d.inverse ? coupling_rqs_kernel<true, true> : coupling_rqs_kernel<false, true>)
                                          : (d.inverse ? coupling_rqs_kernel<true, false> : coupling_rqs_kernel<false, false>);
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  const long long tiles = (s.N + CRQ_TN - 1) / CRQ_TN;
  kernel<<<(unsigned)tiles, CRQ_TN, smem, s.stream>>>(P);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*s.launches;
  return B2B_OK;
}
