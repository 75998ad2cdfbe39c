// A single RationalQuadraticSpline layer with K <= 32 bins (K1 = K + 1 knots; K = 8 is the BASELINE configuration) as a
// program specialised on (D, table size, direction) on the TMA pipeline; table sizes 5 / 9 / 17 / 33 knots, a layer with
// another knot count runs in the next larger table (padded with +inf probes: same number of search steps).
//
// Reference semantics: rational_quadratic_spline.jl:317-357 (forward), :183-220 (inverse) + the forward log-Jacobian
// at the recovered point (interface.jl:276-281).
//
// Per element the work is a bin search plus ~25 flops, i.e. the layer is bound by instruction issue and by
// shared-memory wavefronts, not by HBM.  What this program does about it:
//   * ONE 48-byte record per (row, bin): {w_k, 1/w | w, h_k, Δy | s}{d_k, d_k1}{probe knot, aux} -- one LDS.128 + one
//     LDS.64 (6 wavefronts, the minimum for six lane-divergent numbers) fetch everything the element needs; with a
//     48-byte stride the nine bins of a row start in nine different 16-byte bank groups, so the lane-divergent fetch is
//     conflict-free (a 32-byte stride is 2-3-way conflicted);
//   * the bin search walks the K - 1 INTERIOR knots only (log2(K) dependent probes instead of log2(2K)), the probes live
//     in the records themselves so the running bin index IS the byte offset of the record (no index -> address
//     arithmetic, no clamp), and the first knot is compared separately (only raw three-argument-constructor knots can
//     put a point left of it, :331-343);
//   * rcp / lg2 / sqrt through the .approx.ftz forms (one MUFU each; the default forms carry 4 extra instructions of
//     denormal handling per call), log-Jacobian accumulated in log2 units and scaled once per column.
#include "b2b_v1_pipeline.cuh"

namespace b2b {

constexpr int RQS_REC = 12;  // floats per (row, bin) record

__host__ __device__ constexpr int rqs2_steps(int K1) {
  int s = 0;
  while ((1 << s) < K1 - 1) ++s;
  return s;
}
__host__ __device__ constexpr bool rqs2_supported(int K1) { return K1 >= 2 && K1 <= 33; }  // padded to 5 / 9 / 17 / 33
__host__ __device__ constexpr int rqs2_row_floats(int K1) { return (K1 + 1) * RQS_REC; }

__device__ __forceinline__ float rcp_ftz(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float lg2_ftz(float x) {
  float r;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float sqrt_ftz(float x) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// Records of one layer, built by the whole CTA (one (row, record) pair per thread and step).
// Record c < K1 of row i is bin c (= the reference's k = searchsortedfirst − 1, :328 / :191; c == 0 is the k == 0 branch):
//   [0] w_k  [1] 1/w (forward) | w (inverse)  [2] h_k  [3] Δy (forward) | s = Δy/w (inverse)  [4] d_k  [5] d_k1
//   [8] probe: interior knot S[c+1] for c <= K1-3; the record of the FIRST probe (c = (K1-1)/2 - 1) also holds
//       {S[0], S[K1-1]} in [9], [10]
// with S = widths (forward search on x, :328) or heights (inverse search on y, :191).  Record K1 is padding (v = +inf
// counts every knot; the element is outside the box and its result is discarded).
// K1 is the program's (padded) knot count, 5 / 9 / 17 / 33; the layer has K1r = d.n0 <= K1 knots.  Probe slots beyond the
// layer's interior knots hold +inf (never "< v"), so the bisection over the padded table returns the layer's own bin.
template <int K1, bool INV>
__device__ inline void stage_rqs_records(const b2b_layer_desc& d, float* sm, int D, int tid, int nthreads) {
  constexpr int NR = K1 + 1;
  const int K1r = d.n0;
  const float* S = INV ? d.p1 : d.p0;
  for (int idx = tid; idx < D * NR; idx += nthreads) {
    const int c = idx / D, i = idx - c * D;  // consecutive threads -> consecutive rows (coalesced parameter reads)
    float* rec = sm + (size_t)(i * NR + c) * RQS_REC;
    float w_k = 0.f, w = 1.f, h_k = 0.f, dy = 1.f, d_k = 1.f, d_k1 = 1.f;
    if (c < K1r) {
      const float Wl = d.p0[(size_t)(K1r - 1) * D + i], Hl = d.p1[(size_t)(K1r - 1) * D + i];
      w_k = c == 0 ? -Wl : d.p0[(size_t)(c - 1) * D + i];   // rational_quadratic_spline.jl:331
      w = d.p0[(size_t)c * D + i] - w_k;                    // :332
      h_k = c == 0 ? -Hl : d.p1[(size_t)(c - 1) * D + i];   // :335
      dy = d.p1[(size_t)c * D + i] - h_k;                   // :336
      d_k = c == 0 ? 1.0f : d.p2[(size_t)(c - 1) * D + i];  // :342
      d_k1 = c == K1r - 1 ? 1.0f : d.p2[(size_t)c * D + i]; // :343
    }
    const float sl = dy / w;                                // :339
    float4* r4 = reinterpret_cast<float4*>(rec);
    r4[0] = INV ? make_float4(w_k, w, h_k, sl) : make_float4(w_k, 1.0f / w, h_k, dy);
    r4[1] = make_float4(d_k, d_k1, 0.f, 0.f);
    float p8 = __int_as_float(0x7f800000), p9 = 0.f, p10 = 0.f;  // +inf: not an interior knot of this layer
    if (c <= K1r - 3) p8 = S[(size_t)(c + 1) * D + i];
    if (c == (1 << (rqs2_steps(K1) - 1)) - 1) {  // the record of the first (lane-uniform) probe also carries the end knots
      p9 = S[i];
      p10 = S[(size_t)(K1r - 1) * D + i];
    }
    r4[2] = make_float4(p8, p9, p10, 0.f);
  }
}

// Shared-memory loads by 32-bit shared-space address: the running record offset is then ONE register that the search
// updates with predicated adds and every load uses directly (generic addressing cost an extra three-input add per
// dependent probe and a select + add per step).  NOT volatile: volatile asm statements keep their program order, which
// serialises the 32 elements of a column.
__device__ __forceinline__ float lds_f32(uint32_t a) {
  float v;
  asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ float2 lds_f32x2(uint32_t a) {
  float2 v;
  asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a));
  return v;
}
__device__ __forceinline__ float4 lds_f32x4(uint32_t a) {
  float4 v;
  asm("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
// addr += (probe < v) ? BYTES : 0 as one compare and one predicated add
template <int BYTES>
__device__ __forceinline__ void step_if_less(uint32_t& addr, float probe, float v) {
  asm("{\n .reg .pred p;\n setp.lt.f32 p, %1, %2;\n @p add.u32 %0, %0, %3;\n}" : "+r"(addr) : "f"(probe), "f"(v), "n"(BYTES));
}

template <int K1, int ST>
struct RqsSearch {
  static __device__ __forceinline__ void run(uint32_t& addr, float v) {
    constexpr int RB = RQS_REC * 4;
    step_if_less<ST * RB>(addr, lds_f32(addr + (ST - 1) * RB + 32), v);
    RqsSearch<K1, ST / 2>::run(addr, v);
  }
};
template <int K1>
struct RqsSearch<K1, 0> {
  static __device__ __forceinline__ void run(uint32_t&, float) {}
};

// One element.  `row` is the shared-space address of the records of the element's row; `lg` receives log2 of the
// spline's derivative at the element (0 outside the box), `out` the transformed value.
template <int K1, bool INV>
__device__ __forceinline__ void rqs2_element(uint32_t row, float v, float& out, float& lg) {
  constexpr int STEPS = rqs2_steps(K1);
  constexpr int RB = RQS_REC * 4;  // record stride in bytes
  // the first probe is the same for every lane: one LDS.128 also brings the two end knots
  const float4 head = lds_f32x4(row + ((1 << (STEPS - 1)) - 1) * RB + 32);  // {S[2^(STEPS-1)], S[0], S[K1-1], -}
  const bool outside = fabsf(v) >= head.z;  // x <= -B or x >= B: identity, :322-324 / :186-188 (NaN goes through the spline)
  // number of knots < v (searchsortedfirst − 1): interior knots by bisection, the first knot on its own
  uint32_t addr = row;
  step_if_less<(1 << (STEPS - 1)) * RB>(addr, head.x, v);
  RqsSearch<K1, (1 << (STEPS - 1)) / 2>::run(addr, v);
  step_if_less<RB>(addr, head.y, v);
  const float4 c0 = lds_f32x4(addr);
  const float2 c1 = lds_f32x2(addr + 16);
  const float w_k = c0.x, h_k = c0.z;
  const float d_k = c1.x, d_k1 = c1.y;
  // the record holds 6 numbers (LDS.128 + LDS.64 = 6 shared-memory wavefronts; the kernel is bound by them): Δy or s
  // is rebuilt from the other with one multiplication, d_k1 + d_k − 2s with two more instructions
  const float sl = INV ? c0.w : c0.w * c0.y;   // s = Δy/w, :339
  const float dy = INV ? c0.w * c0.y : c0.w;   // Δy = s·w
  const float ds = fmaf(-2.0f, sl, d_k1 + d_k);  // :205 / :346
  float xi, res;
  if (INV) {
    const float w = c0.y;
    const float yh = v - h_k;
    const float t = yh * ds;
    const float a1 = fmaf(dy, sl - d_k, t);   // :208
    const float a2 = fmaf(dy, d_k, -t);       // :210
    const float a3n = sl * yh;                // −a3, :212
    const float disc = fmaf(4.0f * a1, a3n, a2 * a2);               // a2² − 4·a1·a3
    xi = (a3n + a3n) * rcp_ftz(a2 + sqrt_ftz(disc));                // :215-217
    res = fmaf(xi, w, w_k);                                         // :219
  } else {
    xi = (v - w_k) * c0.y;                                          // :340
  }
  const float omx = 1.0f - xi, xo = xi * omx;
  const float rden = rcp_ftz(fmaf(ds, xo, sl));                     // 1/den, :346
  const float inner = fmaf(sl + sl, xo, fmaf(d_k1 * xi, xi, d_k * omx * omx));  // :349 without the s² factor
  const float q = sl * rden;
  const float arg = q * q * inner;                                  // s²·inner/den² = exp(lj), :349-350
  if (!INV) res = fmaf(dy * fmaf(sl * xi, xi, d_k * xo), rden, h_k);  // :353-354
  out = outside ? v : res;
  lg = lg2_ftz(outside ? 1.0f : arg);
}

template <int D, int K1, bool INV>
struct RqsProg {
  using State = V1NoState;
  const B2BChainParams& P;
  __device__ __forceinline__ void stage(float* params, int warp, int lane, int nw) const {
    stage_rqs_records<K1, INV>(P.layers[0], params, D, warp * 32 + lane, nw * 32);
  }
  __device__ __forceinline__ void apply(float2 (&x)[1][D / 2], const ColCtx<D, 1>&, const float* params,
                                        float (&lj)[1]) const {
    constexpr int RF = rqs2_row_floats(K1);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    // the record loads below are plain (non-volatile) asm so that the scheduler can interleave the elements freely;
    // routing the base address through this statement keeps them behind the tile's barrier wait
    uint32_t pbase = smem_u32(params);
    asm volatile("" : "+r"(pbase));
#pragma unroll
    for (int i = 0; i < D / 2; ++i) {
      float o, l1;
      rqs2_element<K1, INV>(pbase + (2 * i) * RF * 4, x[0][i].x, o, l1);
      x[0][i].x = o;
      acc[(2 * i) & 3] += l1;
      rqs2_element<K1, INV>(pbase + (2 * i + 1) * RF * 4, x[0][i].y, o, l1);
      x[0][i].y = o;
      acc[(2 * i + 1) & 3] += l1;
    }
    const float s = ((acc[0] + acc[1]) + (acc[2] + acc[3])) * 0.6931471805599453f;  // log2 -> ln
    lj[0] += INV ? -s : s;  // sum over dimensions, rational_quadratic_spline.jl:304-309; inverse: interface.jl:278-281
  }
};

template <int D, int K1, int NW, bool INV>
__global__ void __launch_bounds__(NW * 32, 1)
    rqs_unrolled_kernel(const __grid_constant__ B2BChainParams P, const __grid_constant__ V1Extra E,
                        const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_y) {
  const RqsProg<D, K1, INV> prog{P};
  v1_run<D, 1, 1, NW>(P, E, map_x, map_y, prog);
}

template <int D, int K1, int NW>
static int launch_rqs(const B2BChainParams& q, cudaStream_t stream) {
  V1Geom g;
  const int rc = v1_geometry(D, q.N, NW, 32, (size_t)D * rqs2_row_floats(K1), g);
  if (rc != 0) return rc;
  CUtensorMap mx, my;
  if (!make_maps(q, g.cols, &mx, &my, &g.extra.tma3d)) return B2B_EUNSUPPORTED;
  auto kernel = q.layers[0].inverse ? rqs_unrolled_kernel<D, K1, NW, true> : rqs_unrolled_kernel<D, K1, NW, false>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<g.grid, NW * 32, g.smem, stream>>>(q, g.extra, mx, my);
  return (int)cudaGetLastError();
}

template <int D, int NW>
static int dispatch_rqs(const B2BChainParams& q, cudaStream_t stream) {
  const int K1r = q.layers[0].n0;  // the program of the next table size 5 / 9 / 17 / 33 (same number of search steps)
  if (K1r < 2 || K1r > 33) return B2B_EUNSUPPORTED;
  if (K1r <= 5) return launch_rqs<D, 5, NW>(q, stream);
  if (K1r <= 9) return launch_rqs<D, 9, NW>(q, stream);
  if (K1r <= 17) return launch_rqs<D, 17, NW>(q, stream);
  return launch_rqs<D, 33, NW>(q, stream);
}

}  // namespace b2b

// p: a segment that is exactly one RQS layer with 2..33 knots, D in {32, 64}; B2B_EUNSUPPORTED otherwise
int b2b_rqs_unrolled_applicable(const B2BChainParams& p) {
  return p.L == 1 && p.layers[0].kind == B2B_RQS && b2b::rqs2_supported(p.layers[0].n0) && (p.D == 32 || p.D == 64) &&
         b2b::v1_check_io(p) == 0;
}

int b2b_rqs_unrolled_warps(int D) { return D == 64 ? 12 : 16; }

int b2b_launch_rqs_unrolled(const B2BChainParams& p, cudaStream_t stream) {
  using namespace b2b;
  if (!b2b_rqs_unrolled_applicable(p)) return B2B_EUNSUPPORTED;
  B2BChainParams q = p;
  q.scratch_off = -1;
  if (q.D == 64) return dispatch_rqs<64, 12>(q, stream);
  return dispatch_rqs<32, 16>(q, stream);
}
