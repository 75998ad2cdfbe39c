// Reverse mode of an "elementwise run": up to 8 STACKED_EW / PERMUTE layers (either direction), optionally closed by the
// terminal MvNormal of logpdf -- the layers b2b_chain_vjp_f32 hands to this kernel.  What the reference's reverse-mode AD
// computes through stacked.jl:157-166,242-252 (the laws of b2b_device.cuh:ew_apply, restated below with their
// derivatives), permute.jl:152-155 and logpdf(MvNormal(μ, Diagonal(σ²))).
//
// Every element of such a run is independent: input row r follows the fixed path r_0 = r, r_k = π_k(r_{k−1}) through the
// permutations, and along it the value goes through one scalar law per Stacked layer.  One thread owns one input row
// and a slab of columns (like the eval-BatchNorm VJP); it resolves its path and the laws on it once, in the prologue.
// The backward sweep ḡ ← ḡ·f′_k(x_{k−1}) + l̄·∂log|f′_k|/∂x is linear in ḡ, so it is evaluated during the forward sweep:
//   P = Π_k f′_k,   Q = Σ_k ∂log|f′_k|/∂x · Π_{j<k} f′_j,   x̄ = ḡ_K·P + l̄·Q
// with ḡ_K = ȳ[r_K] (or 0) − l̄·(x_K − μ)/σ² when the run ends in the MvNormal.  No forward value has to be kept, so the
// layer loop stays rolled and the kernel is a pure stream over x, ȳ and x̄.  μ̄ and σ̄ of row r_K belong to exactly one
// thread per slab (the path is a permutation); slabs are summed in shared memory and CTAs by a fixed-order finalize,
// so the result is bitwise deterministic.
//
// ELEMENTWISE_VEC layers run as the STACKED_EW layer they equal: code[r] = the law (a row of the constant table
// ew_vec_codes), a = p0, b = 0 -- so x̄ is the same stream with the same bits.  Their ā needs the cotangent ḡ_k at each
// such layer's output, which the forward-only sweep does not have: when ā is requested, the SLOTS instantiation also runs
// the run backwards per column, recomputing each layer's input from x (O(Ls²) law evaluations for Ls laws, no tape):
//   ā_k[r_k] += ḡ_k·∂y/∂a + l̄·∂ℓ/∂a,   ḡ_{k−1} = ḡ_k·f′_k + l̄·∂log|f′_k|/∂x
// Row r_k at layer k belongs to one thread per slab, so ā goes through the same slab / CTA / finalize path as μ̄ and σ̄.
#include <cuda_runtime.h>

#include <cstring>

#include "b2b_internal.h"

namespace b2b {

constexpr int EV_MAXL = 8;  // STACKED_EW / PERMUTE layers per launch

struct EvParams {
  const float* x;
  const float* ybar;   // NULL = zeros
  const float* ljbar;  // NULL = zeros
  float* xbar;
  const float* mu;     // terminal MvNormal (mvn != 0): NULL = 0
  const float* sigma;  //                               NULL = 1
  float* part;         // [grid][2D] per-CTA partials of μ̄ | σ̄ (NULL: not wanted)
  long long N, ldx, ldyb, ldxb;
  int D, L, mvn;
  b2b_layer_desc layers[EV_MAXL];
  // SLOTS instantiation only (the fields after `layers` leave the other instantiations' parameter offsets as they were)
  int width;            // floats per CTA in `part`: [μ̄ | σ̄] (2D, when the run ends in the MvNormal) | ā of each vec layer (D)
  int mw;               // 2D or 0: where the ā blocks start
  int vlo;              // first Stacked layer with an ā block
  int vslot[EV_MAXL];   // per Stacked layer: its ā block, -1 for none
};

// The law column of an ELEMENTWISE_VEC layer seen as STACKED_EW: ew_vec_codes.c[law − B2B_EW_SHIFT][r] = law.
static_assert(B2B_EW_SCALE == B2B_EW_SHIFT + 1 && B2B_EW_LEAKY_RELU == B2B_EW_SHIFT + 2, "law codes");
struct EwVecCodes {
  int32_t c[3][1024];
};
constexpr EwVecCodes ew_vec_codes_init() {
  EwVecCodes t{};
  for (int k = 0; k < 3; ++k)
    for (int r = 0; r < 1024; ++r) t.c[k][r] = B2B_EW_SHIFT + k;
  return t;
}
__device__ const EwVecCodes ew_vec_codes = ew_vec_codes_init();

// One law of ew_apply at input xv: returns the value (the formulas of ew_apply) together with f′ and ∂log|f′|/∂x, the
// derivatives of exactly those formulas.  Value and derivatives share their transcendentals; reciprocals are the
// correctly rounded __frcp_rn (the same value as 1.0f / t without the division routine).
__device__ __forceinline__ float ew_step(int op, bool inverse, float a, float b, float xv, float& f1, float& dl) {
  f1 = 1.0f;
  dl = 0.0f;
  switch (op) {
    case B2B_EW_EXP:
    case B2B_EW_LOG:
      if ((op == B2B_EW_EXP) != inverse) {  // y = e^x, logjac += x
        f1 = expf(xv);
        dl = 1.0f;
        return f1;
      }
      f1 = __frcp_rn(xv);  // y = log x, logjac −= log x
      dl = -f1;
      return logf(xv);
    case B2B_EW_SHIFT: return inverse ? xv - a : a + xv;
    case B2B_EW_SCALE:
      f1 = inverse ? 1.0f / a : a;
      return inverse ? xv / a : a * xv;
    case B2B_EW_LEAKY_RELU: {  // x = 0 takes the identity branch
      const float al = inverse ? 1.0f / a : a;
      if (xv < 0.f) {
        f1 = al;
        return al * xv;
      }
      return xv;
    }
    case B2B_EW_LOGIT:
      if (!inverse) {  // y = logit((x−a)/(b−a)): f′ = 1/(x−a) + 1/(b−x), logjac = −log((x−a)(b−x)/(b−a))
        const float rp = __frcp_rn(xv - a), rq = __frcp_rn(b - xv);
        f1 = rp + rq;
        dl = rq - rp;
        const float z = (xv - a) / (b - a);
        return logf(z / (1.0f - z));
      } else {  // x = a + (b−a)·σ(y): f′ = (b−a)σ(1−σ); logjac = log((x−a)(b−x)/(b−a)) has derivative 1 − 2σ
        const float sg = __frcp_rn(1.0f + expf(-xv));
        f1 = (b - a) * sg * (1.0f - sg);
        dl = 1.0f - 2.0f * sg;
        return fmaf(b - a, sg, a);
      }
    case B2B_EW_TRUNCATED: {
      const bool lo = !isinf(a), hi = !isinf(b);
      if (!inverse) {
        // _clamp (Bijectors.jl:95-100) returns x itself inside [lb, ub] and a constant outside: AD gives 0 there
        const bool in = !(xv < a) && !(xv > b);
        const float x = xv < a ? a : (xv > b ? b : xv);
        float y = x;
        if (lo && hi) {
          const float rp = __frcp_rn(x - a), rq = __frcp_rn(b - x);
          f1 = rp + rq;
          dl = rq - rp;
          y = logf(((x - a) / (b - a)) / (1.0f - (x - a) / (b - a)));
        } else if (lo) {  // y = log(x − lb)
          f1 = __frcp_rn(x - a);
          dl = -f1;
          y = logf(x - a);
        } else if (hi) {  // y = log(ub − x)
          dl = __frcp_rn(b - x);
          f1 = -dl;
          y = logf(b - x);
        }
        if (!in) f1 = dl = 0.0f;
        return y;
      }
      // inverse (truncated.jl:62-76): the closed-form log-Jacobian does not go through the final clamp, the value does
      float xo = xv;
      if (lo && hi) {  // logjac = log(b−a) − |y| − 2·log1pexp(−|y|): derivative 1 − 2σ(y)
        const float sg = __frcp_rn(1.0f + expf(-xv));
        xo = fmaf(b - a, sg, a);
        f1 = (b - a) * sg * (1.0f - sg);
        dl = 1.0f - 2.0f * sg;
      } else if (lo || hi) {  // x = lb + e^y or ub − e^y, logjac = y
        const float e = expf(xv);
        xo = lo ? e + a : b - e;
        f1 = lo ? e : -e;
        dl = 1.0f;
      }
      if (xo < a || xo > b) f1 = 0.0f;
      return xo < a ? a : (xo > b ? b : xo);
    }
    default: return xv;  // IDENTITY
  }
}

// ∂y/∂a and ∂ℓ/∂a of an ELEMENTWISE_VEC law at input xv (the row's a; the laws of ew_step):
//   Shift 1, 0 (inverse −1, 0); Scale xv, 1/a (inverse −xv/a², −1/a); LeakyReLU those of Scale where xv < 0, else 0, 0
__device__ __forceinline__ void ew_vec_dparam(int op, bool inverse, float a, float xv, float& dy, float& dl) {
  dy = 0.0f;
  dl = 0.0f;
  if (op == B2B_EW_SHIFT) {
    dy = inverse ? -1.0f : 1.0f;
  } else if (op == B2B_EW_SCALE || xv < 0.f) {
    const float ra = 1.0f / a;
    dy = inverse ? -(xv * ra) * ra : xv;
    dl = inverse ? -ra : ra;
  }
}

// blockDim.x = max(256, Dp) threads: nslab = blockDim.x / Dp slabs of Dp rows.  Dynamic shared memory:
//   nxt [L][Dp] (int)    next row of each PERMUTE layer
//   law [Ls][T] (int)    per-thread law code | inverse << 8 of the thread's row at the s-th Stacked layer
//   pa, pb [Ls][T]       its parameters
//   red [nslab][2D]      slab partials of μ̄ | σ̄
// TMAX: the block size bound (256 for D <= 256, else 1024, which caps the registers at 64); U: columns in flight per thread.
template <int TMAX, int U>
__global__ void __launch_bounds__(TMAX) ew_vjp_kernel(const __grid_constant__ EvParams P) {
  extern __shared__ __align__(16) int esm[];
  const int D = P.D, L = P.L, Dp = (D + 31) & ~31, T = blockDim.x, nslab = T / Dp, tid = threadIdx.x;
  int Ls = 0;
  for (int l = 0; l < L; ++l) Ls += P.layers[l].kind == B2B_STACKED_EW;
  int* nxt = esm;
  int* law = nxt + L * Dp;
  float* pa = reinterpret_cast<float*>(law + Ls * T);
  float* pb = pa + Ls * T;
  float* red = pb + Ls * T;
  for (int l = 0; l < L; ++l) {
    const b2b_layer_desc& d = P.layers[l];
    if (d.kind != B2B_PERMUTE) continue;
    for (int i = tid; i < D; i += T) {  // y[dst[i]] = x[i]; the inverse reads y[i] = x[dst[i]]
      const int j = d.i0[i];
      if (d.inverse) nxt[l * Dp + j] = i;
      else nxt[l * Dp + i] = j;
    }
  }
  __syncthreads();
  const int slab = tid / Dp, r0 = tid - slab * Dp;
  const bool active = slab < nslab && r0 < D;
  int rK = r0;
  if (active) {
    int s = 0;
    for (int l = 0; l < L; ++l) {
      const b2b_layer_desc& d = P.layers[l];
      if (d.kind == B2B_PERMUTE) {
        rK = nxt[l * Dp + rK];
      } else {
        law[s * T + tid] = d.i0[rK] | (d.inverse ? 256 : 0);
        pa[s * T + tid] = d.p0 ? d.p0[rK] : 0.f;
        pb[s * T + tid] = d.p1 ? d.p1[rK] : 0.f;
        ++s;
      }
    }
  }
  float mu = 0.f, is = 1.f;
  if (P.mvn && active) {
    mu = P.mu ? P.mu[rK] : 0.f;
    is = P.sigma ? 1.0f / P.sigma[rK] : 1.0f;
  }
  float gmu = 0.f, gsg = 0.f;
  const long long per = (P.N + gridDim.x - 1) / gridDim.x;
  const long long c0 = (long long)blockIdx.x * per, c1 = (c0 + per < P.N) ? c0 + per : P.N;
  if (active) {
    for (long long n0 = c0 + slab; n0 < c1; n0 += (long long)U * nslab) {
      float v[U], g[U], lb[U], Pp[U], Q[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long n = n0 + (long long)u * nslab;
        const bool ok = n < c1;
        v[u] = ok ? __ldcs(P.x + n * P.ldx + r0) : 0.f;
        g[u] = (ok && P.ybar) ? __ldcs(P.ybar + n * P.ldyb + rK) : 0.f;
        lb[u] = (ok && P.ljbar) ? __ldcs(P.ljbar + n) : 0.f;
        Pp[u] = 1.0f;
        Q[u] = 0.0f;
      }
#pragma unroll 1
      for (int s = 0; s < Ls; ++s) {
        const int c = law[s * T + tid];
        const int op = c & 255;
        const bool inv = c >> 8;
        const float a = pa[s * T + tid], b = pb[s * T + tid];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          float f1, dl;
          v[u] = ew_step(op, inv, a, b, v[u], f1, dl);
          Q[u] = fmaf(Pp[u], dl, Q[u]);
          Pp[u] *= f1;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long n = n0 + (long long)u * nslab;
        if (n >= c1) continue;
        float gk = g[u];
        if (P.mvn) {  // logpdf = −(D·log2π + Σ log σ²)/2 − Σ q²/2, q = (x − μ)/σ
          const float q = (v[u] - mu) * is;
          const float w = lb[u] * q * is;
          gk -= w;
          gmu += w;
          gsg = fmaf(lb[u] * is, fmaf(q, q, -1.0f), gsg);
        }
        __stcs(P.xbar + n * P.ldxb + r0, fmaf(gk, Pp[u], lb[u] * Q[u]));
      }
    }
  }
  if (!P.part) return;
  if (active) {
    red[slab * 2 * D + rK] = gmu;
    red[slab * 2 * D + D + rK] = gsg;
  }
  __syncthreads();
  for (int e = tid; e < 2 * D; e += T) {
    float t = 0.f;
    for (int w = 0; w < nslab; ++w) t += red[w * 2 * D + e];
    P.part[(size_t)blockIdx.x * 2 * D + e] = t;
  }
}


// ew_vjp_kernel with the ā of the run's ELEMENTWISE_VEC layers, for any D <= 1024 (T = max(256, Dp) threads, two columns
// in flight).  A kernel of its own so that the x̄-only instantiations above keep their code.  Shared memory as above,
// with acc [V][T] (the thread's ā sums of the V vec layers) before red [nslab][P.width] (μ̄ | σ̄ | ā).  x̄, μ̄ and σ̄
// are computed exactly as above.
__global__ void __launch_bounds__(1024) ew_vjp_slots_kernel(const __grid_constant__ EvParams P) {
  constexpr int U = 2;
  extern __shared__ __align__(16) int esm[];
  const int D = P.D, L = P.L, Dp = (D + 31) & ~31, T = blockDim.x, nslab = T / Dp, tid = threadIdx.x, W = P.width;
  int Ls = 0;
  for (int l = 0; l < L; ++l) Ls += P.layers[l].kind == B2B_STACKED_EW;
  int* nxt = esm;
  int* law = nxt + L * Dp;
  float* pa = reinterpret_cast<float*>(law + Ls * T);
  float* pb = pa + Ls * T;
  float* acc = pb + Ls * T;
  float* red = acc + (W - P.mw) / D * T;
  for (int l = 0; l < L; ++l) {
    const b2b_layer_desc& d = P.layers[l];
    if (d.kind != B2B_PERMUTE) continue;
    for (int i = tid; i < D; i += T) {
      const int j = d.i0[i];
      if (d.inverse) nxt[l * Dp + j] = i;
      else nxt[l * Dp + i] = j;
    }
  }
  __syncthreads();
  const int slab = tid / Dp, r0 = tid - slab * Dp;
  const bool active = slab < nslab && r0 < D;
  int rK = r0;
  if (active) {
    int s = 0;
    for (int l = 0; l < L; ++l) {
      const b2b_layer_desc& d = P.layers[l];
      if (d.kind == B2B_PERMUTE) {
        rK = nxt[l * Dp + rK];
      } else {
        law[s * T + tid] = d.i0[rK] | (d.inverse ? 256 : 0);
        pa[s * T + tid] = d.p0 ? d.p0[rK] : 0.f;
        pb[s * T + tid] = d.p1 ? d.p1[rK] : 0.f;
        if (P.vslot[s] >= 0) acc[P.vslot[s] * T + tid] = 0.f;
        ++s;
      }
    }
  }
  float mu = 0.f, is = 1.f;
  if (P.mvn && active) {
    mu = P.mu ? P.mu[rK] : 0.f;
    is = P.sigma ? 1.0f / P.sigma[rK] : 1.0f;
  }
  float gmu = 0.f, gsg = 0.f;
  const long long per = (P.N + gridDim.x - 1) / gridDim.x;
  const long long c0 = (long long)blockIdx.x * per, c1 = (c0 + per < P.N) ? c0 + per : P.N;
  if (active) {
    for (long long n0 = c0 + slab; n0 < c1; n0 += (long long)U * nslab) {
      float v[U], g[U], lb[U], Pp[U], Q[U], x0[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long n = n0 + (long long)u * nslab;
        const bool ok = n < c1;
        v[u] = x0[u] = ok ? __ldcs(P.x + n * P.ldx + r0) : 0.f;
        g[u] = (ok && P.ybar) ? __ldcs(P.ybar + n * P.ldyb + rK) : 0.f;
        lb[u] = (ok && P.ljbar) ? __ldcs(P.ljbar + n) : 0.f;
        Pp[u] = 1.0f;
        Q[u] = 0.0f;
      }
#pragma unroll 1
      for (int s = 0; s < Ls; ++s) {
        const int c = law[s * T + tid];
        const int op = c & 255;
        const bool inv = c >> 8;
        const float a = pa[s * T + tid], b = pb[s * T + tid];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          float f1, dl;
          v[u] = ew_step(op, inv, a, b, v[u], f1, dl);
          Q[u] = fmaf(Pp[u], dl, Q[u]);
          Pp[u] *= f1;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long n = n0 + (long long)u * nslab;
        if (n >= c1) continue;
        float gk = g[u];
        if (P.mvn) {
          const float q = (v[u] - mu) * is;
          const float w = lb[u] * q * is;
          gk -= w;
          gmu += w;
          gsg = fmaf(lb[u] * is, fmaf(q, q, -1.0f), gsg);
        }
        __stcs(P.xbar + n * P.ldxb + r0, fmaf(gk, Pp[u], lb[u] * Q[u]));
        // the backward sweep from the run's output down to the first vec layer, each layer's input recomputed from x
#pragma unroll 1
        for (int k = Ls - 1; k >= P.vlo; --k) {
          float xin = x0[u], f1, dl;
#pragma unroll 1
          for (int s = 0; s < k; ++s) {
            const int c = law[s * T + tid];
            xin = ew_step(c & 255, c >> 8, pa[s * T + tid], pb[s * T + tid], xin, f1, dl);
          }
          const int c = law[k * T + tid];
          const int op = c & 255;
          const bool inv = c >> 8;
          const float a = pa[k * T + tid];
          ew_step(op, inv, a, pb[k * T + tid], xin, f1, dl);
          const int j = P.vslot[k];
          if (j >= 0) {
            float dy, da;
            ew_vec_dparam(op, inv, a, xin, dy, da);
            acc[j * T + tid] = fmaf(gk, dy, fmaf(lb[u], da, acc[j * T + tid]));
          }
          gk = fmaf(gk, f1, lb[u] * dl);
        }
      }
    }
  }
  if (active) {
    if (P.mvn) {
      red[slab * W + rK] = gmu;
      red[slab * W + D + rK] = gsg;
    }
    int r = r0, s = 0;  // the thread's row at each Stacked layer, walked again
    for (int l = 0; l < L; ++l) {
      if (P.layers[l].kind == B2B_PERMUTE) {
        r = nxt[l * Dp + r];
        continue;
      }
      if (P.vslot[s] >= 0) red[slab * W + P.mw + P.vslot[s] * D + r] = acc[P.vslot[s] * T + tid];
      ++s;
    }
  }
  __syncthreads();
  for (int e = tid; e < W; e += T) {
    float t = 0.f;
    for (int w = 0; w < nslab; ++w) t += red[w * W + e];
    P.part[(size_t)blockIdx.x * W + e] = t;
  }
}

// The per-CTA partials summed in a fixed order: out[e] = Σ_cta part[cta][e], e < width, then μ̄ = out[0, D),
// σ̄ = out[D, 2D) (mw = 2D), ā of vec layer j = out[mw + jD, mw + (j+1)D)
struct EvFin {
  const float* part;
  int nparts, D, width, mw;
  float* mubar;
  float* sigmabar;
  float* abar[EV_MAXL];
};

__global__ void __launch_bounds__(256) ew_vjp_finalize_kernel(const __grid_constant__ EvFin F) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x, D = F.D;
  if (e >= F.width) return;
  float t = 0.f;
  for (int p = 0; p < F.nparts; ++p) t += F.part[(size_t)p * F.width + e];
  if (e >= F.mw) {
    if (float* a = F.abar[(e - F.mw) / D]) a[(e - F.mw) % D] = t;
  } else if (e < D) {
    if (F.mubar) F.mubar[e] = t;
  } else if (F.sigmabar) {
    F.sigmabar[e - D] = t;
  }
}

struct CopyList {
  int n;
  const float* src[3 * EV_MAXL];
  float* dst[3 * EV_MAXL];
  int len[3 * EV_MAXL];      // elements copied
  int dst_len[3 * EV_MAXL];  // elements written (the tail beyond len is zero-filled)
};

__global__ void __launch_bounds__(128) copy_list_kernel(const __grid_constant__ CopyList c) {
  const int k = blockIdx.y;
  for (int e = threadIdx.x; e < c.dst_len[k]; e += blockDim.x) c.dst[k][e] = e < c.len[k] ? c.src[k][e] : 0.f;
}

static int ev_threads(int D) {
  const int Dp = (D + 31) & ~31;
  return Dp > 256 ? Dp : 256;
}

static int ev_grid_max() { return b2b_sm_count() * 8; }

}  // namespace b2b

size_t b2b_ew_vjp_workspace(int D, int want_mvn_params, int vec_layers) {
  const size_t width = (want_mvn_params ? 2 * (size_t)D : 0) + (size_t)vec_layers * D;
  if (!width) return 0;
  return (size_t)b2b::ev_grid_max() * width * sizeof(float) + 256;
}

int b2b_vjp_ew(const B2BVjpSeg& s) {
  using namespace b2b;
  const b2b_layer_desc* layers = s.layers;
  const int L = s.n, D = s.D;
  const bool mvn = L > 0 && layers[L - 1].kind == B2B_MVNORMAL_DIAG;
  float* const mubar = mvn ? s.bars[4 * (L - 1)] : nullptr;
  float* const sigmabar = mvn ? s.bars[4 * (L - 1) + 1] : nullptr;
  if (D < 1 || D > 1024 || L < 0) return B2B_EUNSUPPORTED;
  EvParams P;
  memset(&P, 0, sizeof(P));
  float* abar[EV_MAXL] = {};
  const int32_t* codes = nullptr;
  int Ls = 0, V = 0;
  bool want_a = false;
  for (int l = 0; l < L; ++l) {
    const b2b_layer_desc& d = layers[l];
    if (d.kind == B2B_MVNORMAL_DIAG && l == L - 1) {
      P.mvn = 1;
      P.mu = d.p0;
      P.sigma = d.p1;
    } else if (d.kind == B2B_STACKED_EW || d.kind == B2B_PERMUTE || d.kind == B2B_ELEMENTWISE_VEC) {
      if (P.L == EV_MAXL) return B2B_EUNSUPPORTED;
      b2b_layer_desc& e = P.layers[P.L++] = d;
      if (d.kind == B2B_PERMUTE) continue;
      P.vslot[Ls] = -1;
      if (d.kind == B2B_ELEMENTWISE_VEC) {  // the STACKED_EW layer it equals
        if (!codes) {
          const EwVecCodes* t;
          cudaError_t err = cudaGetSymbolAddress((void**)&t, ew_vec_codes);
          if (err != cudaSuccess) return (int)err;
          codes = &t->c[0][0];
        }
        e.kind = B2B_STACKED_EW;
        e.i0 = codes + (size_t)(d.n0 - B2B_EW_SHIFT) * 1024;
        e.p1 = nullptr;
        abar[V] = s.bars[4 * l];
        want_a |= abar[V] != nullptr;
        if (V == 0) P.vlo = Ls;
        P.vslot[Ls] = V++;
      }
      ++Ls;
    } else {
      return B2B_EUNSUPPORTED;
    }
  }
  const bool want = (P.mvn && (mubar || sigmabar)) || want_a;
  if (want && (!s.workspace || s.workspace_bytes < b2b_ew_vjp_workspace(D, P.mvn, V))) return B2B_EWORKSPACE;
  P.x = s.x;
  P.ybar = s.ybar;
  P.ljbar = s.ljbar;
  P.xbar = s.xbar;
  P.N = s.N;
  P.ldx = s.ldx;
  P.ldyb = s.ldyb;
  P.ldxb = s.ldxb;
  P.D = D;
  P.mw = P.mvn ? 2 * D : 0;
  P.width = want_a ? P.mw + V * D : 2 * D;
  const int T = ev_threads(D), Dp = (D + 31) & ~31, nslab = T / Dp;
  long long grid = ev_grid_max();
  const int U = want_a || T > 256 ? 2 : 4;  // columns in flight per thread of the instantiation launched below
  const long long need = (s.N + (long long)nslab * U - 1) / ((long long)nslab * U);
  if (grid > need) grid = need;
  if (grid < 1) grid = 1;
  if (want) P.part = reinterpret_cast<float*>(b2b_align256(s.workspace));
  size_t smem = ((size_t)P.L * Dp + (size_t)3 * Ls * T) * sizeof(int) + (want ? (size_t)nslab * P.width * sizeof(float) : 0);
  void (*kernel)(const EvParams) = T <= 256 ? ew_vjp_kernel<256, 4> : ew_vjp_kernel<1024, 2>;
  if (want_a) {
    kernel = ew_vjp_slots_kernel;
    smem += (size_t)V * T * sizeof(float);
  }
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<(int)grid, T, smem, s.stream>>>(P);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  ++*s.launches;
  if (want) {
    EvFin F;
    memset(&F, 0, sizeof(F));
    F.part = P.part;
    F.nparts = (int)grid;
    F.D = D;
    F.width = P.width;
    F.mw = want_a ? P.mw : 2 * D;
    F.mubar = mubar;
    F.sigmabar = sigmabar;
    for (int j = 0; j < V; ++j) F.abar[j] = abar[j];
    ew_vjp_finalize_kernel<<<(F.width + 255) / 256, 256, 0, s.stream>>>(F);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    ++*s.launches;
  }
  return B2B_OK;
}

int b2b_launch_copy_list(int n, const float* const* src, float* const* dst, const int* len, const int* dst_len,
                         cudaStream_t stream) {
  using namespace b2b;
  if (n < 1) return B2B_OK;
  if (n > 3 * EV_MAXL) return B2B_EUNSUPPORTED;
  CopyList c;
  memset(&c, 0, sizeof(c));
  c.n = n;
  for (int k = 0; k < n; ++k) {
    c.src[k] = src[k];
    c.dst[k] = dst[k];
    c.len[k] = len[k];
    c.dst_len[k] = dst_len[k];
  }
  copy_list_kernel<<<dim3(1, n), 128, 0, stream>>>(c);
  return (int)cudaGetLastError();
}

int b2b_copy_run_bars(const b2b_layer_desc* layers, int n, float* const* bars, const float* const base[3],
                      const size_t step[3], int D, int* launches, cudaStream_t stream) {
  const float* src[24];
  float* dst[24];
  int len[24], dlen[24], c = 0;
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < 3; ++i)
      if (float* d = bars[4 * j + i]) {
        src[c] = base[i] + j * step[i];
        dst[c] = d;
        len[c] = dlen[c] = (int)b2b_slot_len(layers[j], i, D);
        ++c;
      }
  if (!c) return B2B_OK;
  const int rc = b2b_launch_copy_list(c, src, dst, len, dlen, stream);
  if (rc == B2B_OK) ++*launches;
  return rc;
}
