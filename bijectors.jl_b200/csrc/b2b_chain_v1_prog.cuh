// The layer-descriptor interpreter of the thread-per-column pipeline (b2b_chain_v1.cu; also instantiated by the
// sampling kernels of b2b_sample.cu): per-layer maps on register fragments + the program that walks a descriptor list.
// Reference semantics per layer: see b2b_chain_v0.cu / b2b_device.cuh (file:line cited there).
#pragma once
#include "b2b_v1_pipeline.cuh"

namespace b2b {

template <int D, int TPC, int CPT>
__device__ __forceinline__ void planar_apply(float2 (&x)[CPT][D / TPC / 2], const ColCtx<D, TPC>& c, const float* sp,
                                             bool inverse, float (&lj)[CPT]) {
  using C = ColCtx<D, TPC>;
  const float4* w4 = reinterpret_cast<const float4*>(sp);
  const float4* u4 = reinterpret_cast<const float4*>(sp + D);
  const float cc_ = sp[2 * D], bb = sp[2 * D + 1];
  float2 acc[CPT][4];
  B2B_FOR_COLS {
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[cc][i] = make_float2(0.f, 0.f);
  }
  B2B_FOR_SLOTS {
    const float4 w = w4[c.prm(ql, r)];
    const int i = (ql * 8 + r) * 2;
    B2B_FOR_COLS {
      acc[cc][(r & 1) * 2 + 0] = b2b_ffma2(make_float2(w.x, w.y), x[cc][i], acc[cc][(r & 1) * 2 + 0]);
      acc[cc][(r & 1) * 2 + 1] = b2b_ffma2(make_float2(w.z, w.w), x[cc][i + 1], acc[cc][(r & 1) * 2 + 1]);
    }
  }
  float2 t2[CPT];
  B2B_FOR_COLS {
    const float2 s = b2b_fadd2(b2b_fadd2(acc[cc][0], acc[cc][1]), b2b_fadd2(acc[cc][2], acc[cc][3]));
    const float wz = part_sum<TPC>(s.x + s.y);  // aT_b(w, z), utils.jl:2
    float t, s2;
    if (!inverse) {
      tanh_sech2(wz + bb, t, s2);
      lj[cc] += log1pf(cc_ * s2);  // planar_layer.jl:107
    } else {
      find_alpha_ts(wz, cc_, bb, t, s2);  // planar_layer.jl:121; t = tanh(α+b), s2 = sech²(α+b)
      lj[cc] -= log1pf(cc_ * s2);
      t = -t;
    }
    t2[cc] = make_float2(t, t);
  }
  B2B_FOR_SLOTS {
    const float4 u = u4[c.prm(ql, r)];
    const int i = (ql * 8 + r) * 2;
    B2B_FOR_COLS {
      x[cc][i] = b2b_ffma2(make_float2(u.x, u.y), t2[cc], x[cc][i]);  // planar_layer.jl:78 / :124
      x[cc][i + 1] = b2b_ffma2(make_float2(u.z, u.w), t2[cc], x[cc][i + 1]);
    }
  }
}

template <int D, int TPC, int CPT>
__device__ __forceinline__ void batchnorm_apply(float2 (&x)[CPT][D / TPC / 2], const ColCtx<D, TPC>& c,
                                                const float* sp, bool inverse, float (&lj)[CPT]) {
  using C = ColCtx<D, TPC>;
  // staged as y = A·x + C (fwd) / x = iA·y + iC (inverse): normalise.jl:66 / :84 with the constants folded
  const float4* A4 = reinterpret_cast<const float4*>(sp + (inverse ? 2 * D : 0));
  const float4* C4 = reinterpret_cast<const float4*>(sp + (inverse ? 3 * D : D));
  B2B_FOR_SLOTS {
    const float4 a = A4[c.prm(ql, r)], k = C4[c.prm(ql, r)];
    const int i = (ql * 8 + r) * 2;
    B2B_FOR_COLS {
      x[cc][i] = b2b_ffma2(x[cc][i], make_float2(a.x, a.y), make_float2(k.x, k.y));
      x[cc][i + 1] = b2b_ffma2(x[cc][i + 1], make_float2(a.z, a.w), make_float2(k.z, k.w));
    }
  }
  const float ljc = sp[4 * D];
  B2B_FOR_COLS lj[cc] += inverse ? -ljc : ljc;
}

template <int D, int TPC, int CPT>
__device__ __forceinline__ void rqs_apply(float2 (&x)[CPT][D / TPC / 2], const ColCtx<D, TPC>& c, const float* sp,
                                          int K1, bool inverse, float (&lj)[CPT]) {
  using C = ColCtx<D, TPC>;
  const int KP = rqs_kp(K1);
  float acc[CPT];
  B2B_FOR_COLS acc[cc] = 0.f;
  B2B_FOR_SLOTS {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int row = c.row(ql, r, e);
      B2B_FOR_COLS {
        float& xe = (e & 1) ? x[cc][(ql * 8 + r) * 2 + (e >> 1)].y : x[cc][(ql * 8 + r) * 2 + (e >> 1)].x;
        float o = xe, l1 = 0.f;
        if (inverse) rqs_element<true>(sp, K1, KP, D, row, xe, o, l1);
        else rqs_element<false>(sp, K1, KP, D, row, xe, o, l1);
        xe = o;
        acc[cc] += l1;
      }
    }
  }
  B2B_FOR_COLS lj[cc] += part_sum<TPC>(acc[cc]);  // sum over dimensions, rational_quadratic_spline.jl:304-309
}

template <int D, int TPC, int CPT>
__device__ __forceinline__ void stacked_apply(float2 (&x)[CPT][D / TPC / 2], const ColCtx<D, TPC>& c, const float* sp,
                                              bool inverse, float (&lj)[CPT]) {
  using C = ColCtx<D, TPC>;
  const int* code = reinterpret_cast<const int*>(sp);
  const float* av = sp + D;
  float acc[CPT];
  B2B_FOR_COLS acc[cc] = 0.f;
  B2B_FOR_SLOTS {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int row = c.row(ql, r, e);
      const int op = code[row];
      const float a = av[row], b = av[D + row];
      B2B_FOR_COLS {
        float& xe = (e & 1) ? x[cc][(ql * 8 + r) * 2 + (e >> 1)].y : x[cc][(ql * 8 + r) * 2 + (e >> 1)].x;
        xe = ew_apply(op, inverse, a, b, xe, acc[cc]);
      }
    }
  }
  B2B_FOR_COLS lj[cc] += part_sum<TPC>(acc[cc]);
}

// Program 1: the layer-descriptor interpreter (parameters staged in shared memory from DEVICE pointers).
template <int D, int TPC, int CPT>
struct InterpProg {
  using State = V1NoState;
  const B2BChainParams& P;
  __device__ __forceinline__ void stage(float* params, int warp, int lane, int nw) const {
    // RQS tables are large: all threads of the CTA build them; every other layer is staged by one warp
    for (int l = 0; l < P.L; ++l)
      if (P.layers[l].kind == B2B_RQS) stage_rqs_cta(P.layers[l], params + P.soff[l], D, D, warp * 32 + lane, nw * 32);
    for (int l = warp; l < P.L; l += nw)
      if (P.layers[l].kind != B2B_RQS) stage_layer(P.layers[l], params + P.soff[l], D, D, lane);
  }
  __device__ __forceinline__ void apply(float2 (&x)[CPT][D / TPC / 2], const ColCtx<D, TPC>& ctx, const float* params,
                                        float (&lj)[CPT]) const {
    using C = ColCtx<D, TPC>;
#pragma unroll 1
    for (int l = 0; l < P.L; ++l) {
      const b2b_layer_desc& d = P.layers[l];
      const float* sp = params + P.soff[l];
      switch (d.kind) {
        case B2B_PLANAR: planar_apply<D, TPC, CPT>(x, ctx, sp, d.inverse != 0, lj); break;
        case B2B_RADIAL: radial_apply<D, TPC, CPT>(x, ctx, sp, d.inverse != 0, lj); break;
        case B2B_BATCHNORM: batchnorm_apply<D, TPC, CPT>(x, ctx, sp, d.inverse != 0, lj); break;
        case B2B_RQS:
          if constexpr (C::EPT * CPT <= 64) rqs_apply<D, TPC, CPT>(x, ctx, sp, d.n0, d.inverse != 0, lj);
          break;
        case B2B_ELEMENTWISE_VEC:  // staged as the STACKED_EW table
        case B2B_STACKED_EW:
          if constexpr (C::EPT * CPT <= 64) stacked_apply<D, TPC, CPT>(x, ctx, sp, d.inverse != 0, lj);
          break;
        case B2B_MVNORMAL_DIAG: mvnormal_apply<D, TPC, CPT>(x, ctx, sp, lj); break;
        default: break;
      }
    }
  }
};

}  // namespace b2b
