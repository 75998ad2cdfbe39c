// Reverse mode of the spline coupling layer, B2B_COUPLING_RQS, either direction: cotangents of the input and of the
// conditioner's W and c -- what the reference's reverse-mode AD computes through coupling.jl:206-228 with the law
// RationalQuadraticSpline(reshape(W·x₂ + c, …)..., B) (rational_quadratic_spline.jl:109-123, :317-357 / :183-220).
//
// Per column and transformed row i, the kernel recomputes the raw parameters v (crq_params) and the knots (crq_knots),
// takes the processed-knot cotangents of the element from rqv_element (b2b_rqs_element.cuh, the RQS VJP's own element
// function, knot-accurate in both directions) and pulls them back through the normaliser: a reverse cumsum and the
// softmax pullback for widths and heights (crq_knots_vjp), r̄ = d̄·σ(r) for the derivatives.  With r̄ the (3K − 1)
// cotangents of row i:  x̄₂ += W_iᵀ r̄,  c̄_i += Σ_n r̄,  W̄_i += Σ_n r̄ x₂ᵀ;  x̄₁ comes from the element, x̄₃ = ȳ₃.
//
// Mapping.  A fixed grid of G CTAs (at most one wave, fewer when the W̄ slices would pass 256 MiB) walks the column tiles
// round-robin, one thread per column, the rows in order as the forward kernel does.  x̄₂ accumulates in shared memory
// in fp64 (each element sums (3K − 1)·n1 products, which cancel).
// After each row the CTA forms the (3K − 1) x n2 block Σ_n r̄ x₂ᵀ of its tile and adds it to a private slice of the
// workspace ([n1][3K − 1][n2] then [n1][3K − 1] for c̄), owned element by element by one thread.  A second kernel sums
// the G slices in order into W̄ (column-major like W) and c̄.  Deterministic, no atomics, workspace independent of N.
//
// The neural spline couplings, B2B_COUPLING_MLP_RQS and B2B_COUPLING_DEEP_MLP_RQS, are the instantiation NET = true,
// with the network of b2b_coupling_rqs.cu (M hidden layers, M = 1 for B2B_COUPLING_MLP_RQS).  Each thread forms
// h_1 .. h_M of its column from a staged x₂ tile before the row loop, alternating between Xs and one more [H][XP] block
// E so that h_M lands in Xs, and the row loop runs on h_M with W_out and c_out, so its fp64 accumulator holds h̄_M.  The
// kernel then walks back l = M .. 2: each thread recomputes h_{l−1} of its column from x₂ (again through Xs and E: the
// hidden layers cost (M − 1)·H² FMAs per column against (3K − 1)·n1·H for the row loop, so recomputing them is cheap and
// keeps the workspace independent of N), forms v̄_l = h̄_l ⊙ σ′_l in the other block and h̄_{l−1} = W_lᵀv̄_l into the
// accumulator, and the CTA adds Σ v̄_l h_{l−1}ᵀ and Σ v̄_l to its slice.  Last, each thread recomputes W_in·x₂ + c_1 for
// σ′_1, turns h̄_1 into v̄_1 and forms x̄₂ = ȳ₂ + W_inᵀv̄_1 in a fixed order, and the CTA adds Σ v̄_1 x₂ᵀ and Σ v̄_1.  The
// slice is laid out [W̄_out | c̄_out | W̄_in ([H][n2]) | c̄_1 ([H]) | W̄_2 … W̄_M ([H][H] each) | c̄_2 … c̄_M ([H] each)],
// and coupling_rqs_vjp_reduce_kernel sums the slices into the arrays of each parameter role.
#include <cuda_runtime.h>

#include "b2b_coupling_mlp.cuh"
#include "b2b_coupling_rqs.cuh"
#include "b2b_device.cuh"
#include "b2b_internal.h"
#include "b2b_rqs_element.cuh"

namespace b2b {

constexpr int CRV_TN = 64;

struct CrvParams {
  const float* x;
  const float* ybar;
  const float* ljbar;
  float* xbar;
  const float *W, *c;  // NET: W_out, c_out
  const int *idx1, *idx2;
  float* part;  // [G][slice]
  long long N, ldx, ldyb, ldxb, slice;
  int D, n1, n2, K;
  float B;
  const float *W1, *c1;  // NET only: W_in, [c_1 | … | c_M] (or NULL)
  int H, act;
  float slope;
  const float* Wh;  // NET: W_2 .. W_M, each H x H column-major, back to back
  int M;            // NET: hidden layers
};

// NET: layer l (1-based) of the network on this thread's column, from `in` (n_in rows) to `out` ([H] rows), stride XP
template <int XP>
__device__ __forceinline__ void crv_layer(const CrvParams& P, int l, const float* in, int n_in, float* out, int tid) {
  const int H = P.H;
  const float* W = l == 1 ? P.W1 : P.Wh + (size_t)(l - 2) * H * H;
  const float* c = P.c1 ? P.c1 + (size_t)(l - 1) * H : nullptr;
  for (int m = 0; m < H; ++m) {
    float dh;
    mlp_act(P.act, P.slope, crq_hidden_pre(W, c, H, n_in, in + tid, XP, m), out[m * XP + tid], dh);
  }
}

// NET: the second [H][XP] block E, after the D row kinds.  The launcher allocates it for M >= 2 only; at M = 1 the
// pointer lies past the allocation and is never dereferenced (see the forward walk).
__device__ __forceinline__ float* crv_deep_block(unsigned char* kind, int D) {
  return reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(kind + D) + 15) & ~(uintptr_t)15);
}

template <bool INV, bool NET>
__global__ void __launch_bounds__(CRV_TN, 1) coupling_rqs_vjp_kernel(const __grid_constant__ CrvParams P) {
  extern __shared__ __align__(16) float crv_sm[];
  constexpr int TN = CRV_TN, XP = CRV_TN + 1;
  // nc: rows of the conditioning block the row loop reads (x₂, or the hidden layer h)
  const int tid = threadIdx.x, n1 = P.n1, n2 = P.n2, nc = NET ? P.H : n2, K = P.K, K1 = K + 1, J = 3 * K - 1;
  const int JP = crq_jp(K), D = P.D;
  float* Ws = crv_sm;               // [nc][JP]
  float* cs = Ws + nc * JP;         // [JP]
  float* KT = cs + JP;              // knots W | H | Dv, [3][K1][TN]
  float* G = KT + 3 * K1 * TN;      // their cotangents, same layout
  float* Xs = G + 3 * K1 * TN;      // x₂ (NET: h) [nc][XP]
  float* Pr = Xs + nc * XP;         // raw parameters, then their cotangents [J][XP]
  double* XB = reinterpret_cast<double*>(crv_sm) + ((size_t)(nc * JP + JP + 6 * K1 * TN + nc * XP + J * XP) + 1) / 2;
  // x̄₂ (NET: h̄) [nc][XP] in fp64: it sums (3K − 1)·n1 products per element
  float* X2 = reinterpret_cast<float*>(XB + nc * XP);  // NET: x₂ [n2][XP]
  // [D]: 1 = x₁ row, 2 = x₂ row, 0 = x₃ row
  unsigned char* kind = reinterpret_cast<unsigned char*>(NET ? reinterpret_cast<void*>(X2 + n2 * XP) : XB + n2 * XP);
  float* slice = P.part + (size_t)blockIdx.x * P.slice;
  float* cslice = slice + (size_t)n1 * J * nc;
  float* w1slice = cslice + (size_t)n1 * J;  // NET: W̄_in [H][n2], c̄_1 [H], W̄_2 .. W̄_M, c̄_2 .. c̄_M
  const long long slen = NET ? (long long)n1 * J * (nc + 1) + (long long)nc * (n2 + 1) + (long long)(P.M - 1) * nc * (nc + 1)
                             : (long long)n1 * J * (n2 + 1);

  for (int r = tid; r < D; r += TN) kind[r] = 0;
  for (long long e = tid; e < slen; e += TN) slice[e] = 0.f;
  __syncthreads();
  for (int i = tid; i < n1; i += TN) kind[P.idx1[i]] = 1;
  for (int m = tid; m < n2; m += TN) kind[P.idx2[m]] = 2;

  RqvKnots<INV, true> T;
  T.W = KT + tid;
  T.H = KT + K1 * TN + tid;
  T.Dv = KT + 2 * K1 * TN + tid;
  T.stride = TN;
  float* dv = KT + 2 * K1 * TN + tid;
  float* gw = G + tid;
  float* gh = G + K1 * TN + tid;
  float* gd = G + 2 * K1 * TN + tid;
  const long long tiles = (P.N + TN - 1) / TN;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const long long n0 = t * TN, n = n0 + tid;
    const int cols = (int)min((long long)TN, P.N - n0);
    const bool active = tid < cols;
    __syncthreads();  // the previous tile's x̄₂ has been stored
    for (int e = tid; e < n2 * TN; e += TN) {
      const int c = e / n2, m = e - c * n2;
      const bool ok = c < cols;
      (NET ? X2 : Xs)[m * XP + c] = ok ? P.x[(n0 + c) * P.ldx + P.idx2[m]] : 0.f;
      if (!NET) XB[m * XP + c] = ok && P.ybar ? P.ybar[(n0 + c) * P.ldyb + P.idx2[m]] : 0.0;
    }
    if constexpr (NET) {  // h_1 .. h_M of this thread's column (as the forward kernel forms them), h_M in Xs
      __syncthreads();
      float* const E = crv_deep_block(kind, D);
      const float* in = X2;
      // layer l goes to Xs when M − l is even: at M = 1 the only layer lands in Xs and E is untouched, as it is by the
      // walk back l = M .. 2 below, which is then empty
      for (int l = 1; l <= P.M; ++l) {
        float* out = (P.M - l) % 2 == 0 ? Xs : E;
        crv_layer<XP>(P, l, in, l == 1 ? n2 : nc, out, tid);
        in = out;
      }
      for (int m = 0; m < nc; ++m) XB[m * XP + tid] = 0.0;  // h̄_M starts at 0
    }
    const float lb = active && P.ljbar ? P.ljbar[n] : 0.f;
    for (int i = 0; i < n1; ++i) {
      __syncthreads();  // Ws and every column's r̄ of the previous row are no longer read
      crq_stage_row(P.W, P.c, i, n1, nc, K, Ws, cs, tid, TN);
      __syncthreads();
      crq_params(Ws, cs, Xs + tid, XP, nc, K, Pr + tid, XP);
      crq_knots(Pr + tid, XP, K, P.B, KT + tid, TN);
      crq_knots(Pr + K * XP + tid, XP, K, P.B, KT + K1 * TN + tid, TN);
      dv[0] = 1.0f;
      dv[K * TN] = 1.0f;
      for (int j = 1; j < K; ++j) dv[j * TN] = softplus(Pr[(2 * K + j - 1) * XP + tid]);
      for (int k = 0; k < K1; ++k) gw[k * TN] = gh[k * TN] = gd[k * TN] = 0.f;
      if (active) {
        const int row = P.idx1[i];
        const float v = P.x[n * P.ldx + row];
        const float cb = P.ybar ? P.ybar[n * P.ldyb + row] : 0.f;
        const float Wl = T.w(K), Hl = T.h(K), Bs = INV ? Hl : Wl;
        // identity outside the box: evaluated at 0 with zero cotangents, so every knot cotangent is an exact 0
        const bool in = v > -Bs && v < Bs;
        const float ve = in ? v : 0.f;
        int kb = 0;
        for (int j = 0; j < K; ++j) kb += T.s(j) < ve ? 1 : 0;
        RqvCot c;
        const float out = rqv_element<INV, true>(T, K1, kb, Wl, Hl, ve, in ? cb : 0.f, in ? lb : 0.f, c);
        P.xbar[n * P.ldxb + row] = in ? out : cb;
        const int ka = kb > 0 ? kb - 1 : K1 - 1;
        gw[ka * TN] += c.xk;
        gh[ka * TN] += c.yk;
        gd[ka * TN] += c.dk;
        gw[kb * TN] += c.xk1;
        gh[kb * TN] += c.yk1;
        gd[kb * TN] += c.dk1;
      }
      // pull the knot cotangents back to the raw parameters (zero for columns past the batch)
      crq_knots_vjp(Pr + tid, XP, K, P.B, gw, TN);
      crq_knots_vjp(Pr + K * XP + tid, XP, K, P.B, gh, TN);
      for (int j = 0; j < K - 1; ++j) {
        float* r = Pr + (2 * K + j) * XP + tid;
        *r = gd[(j + 1) * TN] / (1.0f + expf(-*r));
      }
      for (int m = 0; m < nc; ++m) {
        float s = 0.f;
        for (int j = 0; j < J; ++j) s = fmaf(Ws[m * JP + j], Pr[j * XP + tid], s);
        XB[m * XP + tid] += (double)s;
      }
      __syncthreads();
      // this tile's Σ_n r̄ x₂ᵀ and Σ_n r̄ for row i, added to the CTA's slice (each element always by the same thread)
      float* sl = slice + (size_t)i * J * nc;
      for (int e = tid; e < J * nc; e += TN) {
        const int j = e / nc, m = e - j * nc;
        const float* pr = Pr + j * XP;
        const float* xs = Xs + m * XP;
        float s = 0.f;
        for (int c = 0; c < cols; ++c) s = fmaf(pr[c], xs[c], s);
        sl[e] += s;
      }
      for (int j = tid; j < J; j += TN) {
        const float* pr = Pr + j * XP;
        float s = 0.f;
        for (int c = 0; c < cols; ++c) s += pr[c];
        cslice[(size_t)i * J + j] += s;
      }
    }
    __syncthreads();
    if constexpr (NET) {
      float* const E = crv_deep_block(kind, D);
      float* const whslice = w1slice + (size_t)nc * (n2 + 1);  // W̄_2 .. W̄_M ([H][H] each), then c̄_2 .. c̄_M
      for (int l = P.M; l >= 2; --l) {
        // h_{l−1} of this thread's column, recomputed from x₂ through E and Xs (the previous step's reads are done)
        const float* hin = X2;
        for (int j = 1; j < l; ++j) {
          float* out = (l - 1 - j) % 2 == 0 ? Xs : E;
          crv_layer<XP>(P, j, hin, j == 1 ? n2 : nc, out, tid);
          hin = out;
        }
        // v̄_l = h̄_l ⊙ σ′(W_l·h_{l−1} + c_l) into E, then h̄_{l−1} = W_lᵀv̄_l (the sum over the units in increasing
        // order) into the accumulator: both this thread's column only
        const float* Wl = P.Wh + (size_t)(l - 2) * nc * nc;
        const float* cl = P.c1 ? P.c1 + (size_t)(l - 1) * nc : nullptr;
        for (int m = 0; m < nc; ++m) {
          float h, dh;
          mlp_act(P.act, P.slope, crq_hidden_pre(Wl, cl, nc, nc, hin + tid, XP, m), h, dh);
          E[m * XP + tid] = (float)XB[m * XP + tid] * dh;
        }
        for (int k = 0; k < nc; ++k) {
          float s = 0.f;
          for (int m = 0; m < nc; ++m) s = fmaf(__ldg(Wl + (size_t)k * nc + m), E[m * XP + tid], s);
          XB[k * XP + tid] = (double)s;
        }
        __syncthreads();
        // this tile's Σ_n v̄_l h_{l−1}ᵀ and Σ_n v̄_l, added to the CTA's slice (each element always by the same thread)
        float* wsl = whslice + (size_t)(l - 2) * nc * nc;
        for (int e = tid; e < nc * nc; e += TN) {
          const int m = e / nc, k = e - m * nc;
          const float* vb = E + m * XP;
          const float* hs = hin + k * XP;
          float s = 0.f;
          for (int c = 0; c < cols; ++c) s = fmaf(vb[c], hs[c], s);
          wsl[e] += s;
        }
        float* csl = whslice + (size_t)(P.M - 1) * nc * nc + (size_t)(l - 2) * nc;
        for (int m = tid; m < nc; m += TN) {
          const float* vb = E + m * XP;
          float s = 0.f;
          for (int c = 0; c < cols; ++c) s += vb[c];
          csl[m] += s;
        }
        __syncthreads();
      }
    }
    if (NET) {
      // v̄_1 = h̄_1 ⊙ σ′(W_in·x₂ + c_1) of this thread's column into Xs (h_1 is no longer read)
      for (int m = 0; m < nc; ++m) {
        float h, dh;
        mlp_act(P.act, P.slope, crq_hidden_pre(P.W1, P.c1, nc, n2, X2 + tid, XP, m), h, dh);
        Xs[m * XP + tid] = (float)XB[m * XP + tid] * dh;
      }
      __syncthreads();
      // this tile's Σ_n v̄_1 x₂ᵀ and Σ_n v̄_1, added to the CTA's slice (each element always by the same thread)
      for (int e = tid; e < nc * n2; e += TN) {
        const int m = e / n2, k = e - m * n2;
        const float* vb = Xs + m * XP;
        const float* xs = X2 + k * XP;
        float s = 0.f;
        for (int c = 0; c < cols; ++c) s = fmaf(vb[c], xs[c], s);
        w1slice[e] += s;
      }
      for (int m = tid; m < nc; m += TN) {
        const float* vb = Xs + m * XP;
        float s = 0.f;
        for (int c = 0; c < cols; ++c) s += vb[c];
        w1slice[(size_t)nc * n2 + m] += s;
      }
      __syncthreads();
      // W_inᵀv̄_1 of this thread's column into X2 (x₂ is no longer read), the sum over the hidden units in increasing order
      for (int k = 0; k < n2; ++k) {
        float s = 0.f;
        for (int m = 0; m < nc; ++m) s = fmaf(__ldg(P.W1 + (size_t)k * nc + m), Xs[m * XP + tid], s);
        X2[k * XP + tid] = s;
      }
      __syncthreads();
    }
    for (int e = tid; e < n2 * TN; e += TN) {
      const int c = e / n2, m = e - c * n2;
      if (c < cols)  // NET: x̄₂ = ȳ₂ + W_inᵀv̄_1
        P.xbar[(n0 + c) * P.ldxb + P.idx2[m]] =
            NET ? (P.ybar ? P.ybar[(n0 + c) * P.ldyb + P.idx2[m]] : 0.f) + X2[m * XP + c] : (float)XB[m * XP + c];
    }
    for (int e = tid; e < cols * D; e += TN) {  // x̄₃ = ȳ₃
      const int c = e / D, r = e - c * D;
      if (!kind[r]) P.xbar[(n0 + c) * P.ldxb + r] = P.ybar ? P.ybar[(n0 + c) * P.ldyb + r] : 0.f;
    }
  }
}

// The G slices summed in order (in T: float, or double for the deep network) and scattered from the slice layout
// [W̄_out | c̄_out | W̄_in | c̄_1 | W̄_2 .. W̄_M | c̄_2 .. c̄_M] to the arrays of the parameter roles (NULL: not wanted).  nc:
// the conditioning rows (n2, or H); H, nl: the network's hidden units and hidden-to-hidden layers (0, 0: none).  W_out is
// J x nc column-major (J = (3K − 1)·n1), W_in H x n2, W_hid nl H x H blocks, cin = [c_1 | … | c_M].
template <class T>
__global__ void __launch_bounds__(256) coupling_rqs_vjp_reduce_kernel(const float* __restrict__ part, int nparts,
                                                                      long long slice, int n1, int nc, int K, int H,
                                                                      int n2, int nl, float* __restrict__ Wout,
                                                                      float* __restrict__ cout, float* __restrict__ Win,
                                                                      float* __restrict__ cin, float* __restrict__ Whid) {
  const long long J = (long long)(3 * K - 1) * n1, hh = (long long)H * H;
  const long long nw = J * nc, nwc = nw + J, nw1 = nwc + (long long)H * n2, nc1 = nw1 + H, nwh = nc1 + nl * hh;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nwh + (long long)nl * H) return;
  T t = 0;
  for (int g = 0; g < nparts; ++g) t += part[(size_t)g * slice + e];
  if (e < nw) {  // [i][j][m] -> W_out row i + n1·j, column m
    const long long i = e / ((3 * K - 1) * (long long)nc), rem = e - i * (3 * K - 1) * nc, j = rem / nc, m = rem - j * nc;
    if (Wout) Wout[(size_t)(i + n1 * j) + (size_t)J * m] = (float)t;
  } else if (e < nwc) {  // [i][j] -> c_out[i + n1·j]
    const long long f = e - nw, i = f / (3 * K - 1), j = f - i * (3 * K - 1);
    if (cout) cout[(size_t)(i + n1 * j)] = (float)t;
  } else if (e < nw1) {  // [m][k] -> W_in row m, column k
    const long long f = e - nwc, m = f / n2, k = f - m * n2;
    if (Win) Win[(size_t)(m + H * k)] = (float)t;
  } else if (e < nc1) {
    if (cin) cin[e - nw1] = (float)t;
  } else if (e < nwh) {  // [l − 2][m][k] -> W_l row m, column k
    const long long f = e - nc1, l = f / hh, m = (f - l * hh) / H, k = f - l * hh - m * H;
    if (Whid) Whid[(size_t)(l * hh + m + H * k)] = (float)t;
  } else if (cin) {  // c̄_2 .. c̄_M
    cin[(size_t)H + (size_t)(e - nwh)] = (float)t;
  }
}

using Cpl = B2BCoupling<b2b_layer_desc>;
// the kernels' nc conditioning rows (x₂, or the network's H hidden units) and nx rows of x₂ under the network (0: none)
static int crv_nc(const Cpl& c) { return c.net ? c.H : c.n2; }
static int crv_nx(const Cpl& c) { return c.net ? c.n2 : 0; }

// the deep network's hidden-to-hidden layers W_2 .. W_M (0: none)
static int crv_nl(const Cpl& c) { return c.M > 1 ? c.M - 1 : 0; }

static size_t crv_smem_bytes(const Cpl& c, int D) {
  const int nc = crv_nc(c), K = c.K, J = 3 * K - 1, JP = crq_jp(K), K1 = K + 1;
  const size_t f = (size_t)nc * JP + JP + (size_t)6 * K1 * CRV_TN + (size_t)nc * (CRV_TN + 1) + (size_t)J * (CRV_TN + 1);
  const size_t e = crv_nl(c) ? (size_t)c.H * (CRV_TN + 1) * sizeof(float) : 0;  // the deep network's block E
  return ((((f + 1) / 2 + (size_t)nc * (CRV_TN + 1)) * sizeof(double) + (size_t)crv_nx(c) * (CRV_TN + 1) * sizeof(float) +
           D + 15) & ~(size_t)15) + e;
}

// floats of the slice's sums: W̄ / c̄ of the spline's conditioner, then W̄₁ / c̄₁ of the network, then W̄_2 .. W̄_M and
// c̄_2 .. c̄_M of the deep network
static long long crv_sum_floats(const Cpl& c) {
  return (long long)c.n1 * (3 * c.K - 1) * (crv_nc(c) + 1) + (long long)c.H * (crv_nx(c) + 1) +
         (long long)crv_nl(c) * c.H * (c.H + 1);
}

static long long crv_slice_floats(const b2b_layer_desc& d) { return (crv_sum_floats(b2b_coupling(d)) + 63) & ~63LL; }

static int crv_grid(const b2b_layer_desc& d, int D, long long N) {
  const int sms = b2b_sm_count();
  int per_sm = (int)((size_t)(227 * 1024) / (crv_smem_bytes(b2b_coupling(d), D) + 1024));
  per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
  long long g = (long long)sms * per_sm;
  const long long tiles = (N + CRV_TN - 1) / CRV_TN;
  if (g > tiles) g = tiles;
  const long long cap = (256LL << 20) / (crv_slice_floats(d) * (long long)sizeof(float));
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

}  // namespace b2b

size_t b2b_coupling_rqs_vjp_workspace(const b2b_layer_desc& d, int D, long long N) {
  using namespace b2b;
  if (!b2b_coupling_fits(d, D)) return 0;
  return (size_t)crv_grid(d, D, N) * (size_t)crv_slice_floats(d) * sizeof(float) + 256;
}

int b2b_vjp_spline(const B2BVjpSeg& s) {
  using namespace b2b;
  const b2b_layer_desc& d = s.layers[0];
  const int D = s.D;
  const long long N = s.N;
  if (!b2b_coupling_fits(d, D)) return B2B_EUNSUPPORTED;
  if (!s.workspace || s.workspace_bytes < b2b_coupling_rqs_vjp_workspace(d, D, N)) return B2B_EWORKSPACE;
  const Cpl c = b2b_coupling(d);
  // The network's sums are written only where they are asked for.  Without the network, W̄ always goes somewhere (the
  // kernel forms it anyway), and c̄ when the layer has a c.
  float* const Wbar = c.net || s.bars[0] ? c.role(s.bars, B2B_W_OUT) : s.scratch;
  float* const cbar = c.net || !c.c_out || s.bars[1] ? c.role(s.bars, B2B_C_OUT)
                                                     : s.scratch + ((b2b_slot_len(d, 0, D) + 63) & ~(size_t)63);
  CrvParams P = {};
  P.x = s.x;
  P.ybar = s.ybar;
  P.ljbar = s.ljbar;
  P.xbar = s.xbar;
  P.W = c.W_out;
  P.c = c.c_out;
  P.W1 = c.W_in;
  P.c1 = c.c_in;
  P.idx1 = c.idx1;
  P.idx2 = c.idx2;
  P.part = reinterpret_cast<float*>(b2b_align256(s.workspace));
  P.N = N;
  P.ldx = s.ldx;
  P.ldyb = s.ldyb;
  P.ldxb = s.ldxb;
  P.slice = crv_slice_floats(d);
  P.D = D;
  P.n1 = c.n1;
  P.n2 = c.n2;
  P.K = c.K;
  P.H = c.H;
  P.act = c.act;
  P.B = c.B;
  P.slope = c.slope;
  P.Wh = c.W_hid;
  P.M = c.M;
  const int grid = crv_grid(d, D, N);
  const size_t smem = crv_smem_bytes(c, D);
  void (*kernel)(const CrvParams) = c.net ? (d.inverse ? coupling_rqs_vjp_kernel<true, true> : coupling_rqs_vjp_kernel<false, true>)
                                          : (d.inverse ? coupling_rqs_vjp_kernel<true, false> : coupling_rqs_vjp_kernel<false, false>);
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<grid, CRV_TN, smem, s.stream>>>(P);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  const unsigned blocks = (unsigned)((crv_sum_floats(c) + 255) / 256);
  (crv_nl(c) ? coupling_rqs_vjp_reduce_kernel<double> : coupling_rqs_vjp_reduce_kernel<float>)<<<blocks, 256, 0, s.stream>>>(
      P.part, grid, P.slice, c.n1, crv_nc(c), c.K, c.H, c.n2, crv_nl(c), Wbar, cbar, c.role(s.bars, B2B_W_IN),
      c.role(s.bars, B2B_C_IN), c.role(s.bars, B2B_W_HID));
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  *s.launches += 2;
  return B2B_OK;
}
