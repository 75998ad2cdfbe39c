// Affine coupling layer on the Hopper tensor cores (wgmma, accumulators in registers).
//
// Reference: Coupling (src/bijectors/coupling.jl:206-228) with θ(x₂) = Shift(t) ∘ Scale(exp.(s)),
// [s; t] = W·x₂ + c (scale.jl:13,31; shift.jl:14,21) mapped over the columns of the batch; see
// b2b_coupling.cu for the exact-fp32 SIMT version this kernel is cross-checked against.
//
// The conditioner is a GEMM  [s;t](2·n1 x T) = W(2·n1 x n2) · X₂(n2 x T)  per tile of T = 64 columns:
// 65.5 kFLOP per 2 KB sample at D = 256 (AI ≈ 32 FLOP/B), i.e. compute-bound on the fp32 CUDA cores,
// hence tensor cores.  Plain TF32/BF16 cannot hold the 1e-5 parity bar, so both
// operands are split into an fp16 "hi" and an fp16 "lo" half (22 mantissa bits together) after an EXACT
// power-of-two rescale (W by one global 2^k, every x₂ column by its own 2^k, undone in the epilogue), and
// three products hi·hi + hi·lo + lo·hi are accumulated in fp32 (the dropped lo·lo term is 2^-22).
//
// Warp roles of the persistent CTA (512 threads = 4 warpgroups, one CTA per SM):
//   warpgroups 0-1  consumers: warpgroup g issues the wgmma.mma_async m64n64k16 chain (48 per tile at n2 = 128) for
//                         rows 64g..64g+63 of both the s and the t block, so the s and t value of one (row, column)
//                         sit in the same accumulator slot of the same thread.  x₁ of the tile is requested before
//                         the MMAs are issued; the epilogue then adds c, forms y₁ = exp(s)·x₁ + t (or the inverse)
//                         and stores -- each warp store covers 16 rows (64 B) of each of 8 columns
//   warpgroups 2-3  producers: coalesced float4 loads of the x₂ rows (prefetched one tile ahead), per-column scale
//                         (REDUX max of the float bit patterns), hi/lo split, store into the K-major 128B-swizzled
//                         wgmma operand layout, logjac = wsum·x₂ + Σc in fp32 (Σ_j s_j = (Σ_j W_j)·x₂ + Σ_j c_j),
//                         pass-through rows when y != x
// W (both halves, both M tiles) stays resident in shared memory for the lifetime of the CTA (128 KB at
// n2 = 128, loaded once by bulk copies); x₂ operand stages are double buffered and handed over with mbarriers.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdlib>

#include "b2b_internal.h"

namespace b2b {

constexpr int TC_T = 64;              // batch columns per tile == wgmma N
constexpr int TC_STAGES = 2;          // x₂ operand stages in shared memory
constexpr int TC_SCALE_SLOTS = 4;     // per-column scale slots (producer may run 4 tiles ahead of the epilogue)
constexpr int TC_ABLK = 128 * 128;    // one [128 rows x 64 k] fp16 block, 128B-swizzled, 16 KB
constexpr int TC_BBLK = TC_T * 128;   // one [64 rows x 64 k] fp16 block, 8 KB
constexpr int TC_THREADS = 512;
constexpr int TC_PROD_WARPS = 8, TC_EPI_WARPS = 8;  // consumers are warps 0-7, producers warps 8-15

struct TcParams {
  const float* x;
  float* y;
  float* logjac;
  const unsigned char* wimg;  // prepared fp16 hi/lo operand image of W (see coupling_prep_kernel)
  const float* wsum;          // [n2]  Σ_j W[j, k] over the s rows
  const float* meta;          // {1/scaleW, Σ_j c_j}
  const float* fold;          // folded neighbouring BatchNorm layers: preA[D] | preC[D] | postA[D] | postC[D] | {Σ logjac}; or NULL
  const float* cvec;          // [2 n1] or NULL
  long long N, ldx, ldy, tiles;
  int D, n1, n2, nkb, row1, row2, accumulate, inverse;
};

// ---- PTX wrappers ----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sm_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void bar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void bar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "TC_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra TC_DONE;\n"
      "bra TC_WAIT;\n"
      "TC_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of the accumulators across the wgmma fence / wait
__device__ __forceinline__ void wg_fence_acc(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D(64 x 64, fp32) (+)= A(64 x 16) · B(16 x 64), fp16 operands K-major in shared memory; `accumulate` = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// wgmma shared-memory matrix descriptor: K-major operand, 128-byte swizzle, 8-row groups 1024 B apart:
// start>>4 | LBO(=1, unused for swizzled K-major)<<16 | SBO(1024>>4)<<32 | SW128(1)<<62
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

// byte offset of the 8-byte group holding k' .. k'+3 of row `row` inside one 128B-swizzled [rows x 64] fp16 block
__device__ __forceinline__ int sw128_off(int row, int kprime) {
  return (row >> 3) * 1024 + (row & 7) * 128 + ((((kprime >> 3) ^ (row & 7)) & 7) << 4) + (kprime & 7) * 2;
}

// ---- W preparation (once per call, ~µs): global power-of-two scale, hi/lo fp16 split in operand layout --------
// image blocks (16 KB each) are ordered [mt (0: s rows, 1: t rows)][part (0: hi, 1: lo)][kb]
__global__ void __launch_bounds__(1024) coupling_prep_kernel(const float* __restrict__ W, const float* __restrict__ c,
                                                             int n1, int n2, unsigned char* __restrict__ wimg,
                                                             float* __restrict__ wsum, float* __restrict__ meta) {
  __shared__ float red[32];
  __shared__ float s_scale;
  const int tid = threadIdx.x;
  const int total = 2 * n1 * n2;
  float m = 0.f;
  for (int i = tid; i < total; i += 1024) m = fmaxf(m, fabsf(W[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((tid & 31) == 0) red[tid >> 5] = m;
  __syncthreads();
  if (tid < 32) {
    float v = red[tid];
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (tid == 0) {
      int e = (int)((__float_as_uint(v) >> 23) & 0xffu) - 127;  // floor(log2(max|W|))
      e = max(-100, min(100, e));
      s_scale = __uint_as_float((uint32_t)(127 + 9 - e) << 23);  // max|W|·scale in [2^9, 2^10)
      meta[0] = __uint_as_float((uint32_t)(127 - 9 + e) << 23);  // 1/scale (exact)
      float cs = 0.f;
      if (c)
        for (int j = 0; j < n1; ++j) cs += c[j];
      meta[1] = cs;
    }
  }
  __syncthreads();
  const float scale = s_scale;
  const int nkb = n2 / 64;
  // one thread per (mt, m, group of 4 k)
  const int groups = 2 * 128 * (n2 / 4);
  for (int g = tid; g < groups; g += 1024) {
    const int k4 = g % (n2 / 4), m_ = (g / (n2 / 4)) % 128, mt = g / ((n2 / 4) * 128);
    __half hi[4], lo[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = 4 * k4 + e;
      const float w = m_ < n1 ? W[(size_t)k * (2 * n1) + mt * n1 + m_] * scale : 0.f;
      hi[e] = __float2half_rn(w);
      lo[e] = __float2half_rn(w - __half2float(hi[e]));
    }
    const int kb = (4 * k4) / 64, kp = (4 * k4) % 64;
    const int off = sw128_off(m_, kp);
    *reinterpret_cast<uint2*>(wimg + (size_t)((mt * 2 + 0) * nkb + kb) * TC_ABLK + off) = *reinterpret_cast<uint2*>(hi);
    *reinterpret_cast<uint2*>(wimg + (size_t)((mt * 2 + 1) * nkb + kb) * TC_ABLK + off) = *reinterpret_cast<uint2*>(lo);
  }
  for (int k = tid; k < n2; k += 1024) {
    float s = 0.f;
    for (int j = 0; j < n1; ++j) s += W[(size_t)k * (2 * n1) + j];
    wsum[k] = s;
  }
}

// ---- main kernel -------------------------------------------------------------------------------------------
// Template parameters: LD > 0 = compile-time leading dimension of BOTH x and y (the dense D = 256 batches of the
// BASELINE configuration: every per-column address becomes an immediate offset), 0 = run-time strides; FOLD = a
// neighbouring BatchNorm is folded in (per-row affine before / after); INV = inverse law.
// Per-column bounds tests, clamps, 64-bit address products and run-time mode flags make a kernel like this one issue /
// instruction-cache bound, so this kernel only ever sees WHOLE tiles (the
// launcher hands the < 64 ragged columns at the end of a batch to the exact-fp32 kernel), so there is no bounds logic
// at all, and addresses are a per-tile pointer plus immediates.
template <int LD, bool FOLD, bool INV>
__global__ void __launch_bounds__(TC_THREADS, 1) coupling_tc_kernel(const __grid_constant__ TcParams P) {
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* base = smem_dyn + ((1024u - (sm_u32(smem_dyn) & 1023u)) & 1023u);
  const int nkb = P.nkb;
  const int a_bytes = 4 * nkb * TC_ABLK;            // W image: 2 M tiles x {hi, lo} x nkb blocks
  const int b_stage = 2 * nkb * TC_BBLK;            // x₂ stage: {hi, lo} x nkb blocks
  unsigned char* sA = base;
  unsigned char* sB = base + a_bytes;
  float* colscale = reinterpret_cast<float*>(sB + TC_STAGES * b_stage);   // [TC_SCALE_SLOTS][TC_T]
  uint64_t* bars = reinterpret_cast<uint64_t*>(colscale + TC_SCALE_SLOTS * TC_T);
  // bars: [0..1] b_full, [2..3] b_empty, [4] w_ready
  const long long ldx = LD ? LD : P.ldx, ldy = LD ? LD : P.ldy;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < TC_STAGES; ++s) {
      bar_init(sm_u32(&bars[0 + s]), TC_PROD_WARPS);
      bar_init(sm_u32(&bars[2 + s]), TC_EPI_WARPS);  // every consumer warp, once its MMAs have read the stage
    }
    bar_init(sm_u32(&bars[4]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const long long my_tiles = (P.tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;

  if (warp >= TC_EPI_WARPS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 112;" ::: "memory");  // registers go to the consumers
    // ================================ producers ================================
    // Warp p converts columns [8p, 8p+8) of every tile.  Lane l holds the float4 #l of a column (rows
    // row2+4l..+3).  The per-column maximum (operand scale) is ONE redux.sync on the float bit patterns (monotonic
    // for non-negative floats); the 8 dots with wsum (log-Jacobian) are reduced together by a transposing butterfly
    // (7+2 shuffles), after which lane l owns column (l>>2)&7.  The NEXT tile's eight columns are requested at the top
    // of the loop, so a whole tile of conversion work hides their DRAM latency.
    constexpr int CW = TC_T / TC_PROD_WARPS;  // 8 columns per producer warp
    const int p = warp - TC_EPI_WARPS;
    const bool active = 4 * lane < P.n2;
    const int lrow = active ? 4 * lane : 0;  // inactive lanes read a valid address, result unused
    const float4 one4 = make_float4(1.f, 1.f, 1.f, 1.f), zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 ws = active ? *reinterpret_cast<const float4*>(P.wsum + 4 * lane) : zero4;
    const float cs_mul = 6.103515625e-05f * P.meta[0];  // 2^-14 / scaleW: undoes both operand scales
    const float csum = P.meta[1] * (INV ? -1.f : 1.f) + (FOLD ? P.fold[4 * P.D] : 0.f);
    float4 preA = one4, preC = zero4, postA = one4, postC = zero4;
    if (FOLD && active) {
      preA = *reinterpret_cast<const float4*>(P.fold + P.row2 + 4 * lane);
      preC = *reinterpret_cast<const float4*>(P.fold + P.D + P.row2 + 4 * lane);
      postA = *reinterpret_cast<const float4*>(P.fold + 2 * P.D + P.row2 + 4 * lane);
      postC = *reinterpret_cast<const float4*>(P.fold + 3 * P.D + P.row2 + 4 * lane);
    }
    const bool write_y2 = P.y != nullptr && (P.y != P.x || FOLD);
    const bool rest_rows = write_y2 && P.n1 + P.n2 < P.D;
    const int own = (lane >> 2) & 7;  // column owned by this lane after the transposing reduction
    // operand-layout offset of this lane's 8-byte group in row (8p + c): sw128_off(8p + c, kp) = st_base ^ (c<<4 | c<<7)
    const int kb = (4 * lane) / 64, kp = (4 * lane) % 64;
    const int st_base = p * 1024 + ((kp >> 3) << 4) + (kp & 7) * 2 + kb * TC_BBLK;
    const int lo_off = nkb * TC_BBLK;
    const long long tstride = (long long)gridDim.x * TC_T;  // columns between two tiles of this CTA
    long long col0 = (long long)blockIdx.x * TC_T + p * CW;  // first column of this warp in the current tile
    const float* xt = P.x + P.row2 + lrow + col0 * ldx;
    float* yt = write_y2 ? P.y + P.row2 + lrow + col0 * ldy : nullptr;

    float4 cur[CW];
    if (my_tiles > 0) {
#pragma unroll
      for (int c = 0; c < CW; ++c) cur[c] = __ldcs(reinterpret_cast<const float4*>(xt + c * ldx));
    }
    for (long long i = 0; i < my_tiles; ++i) {
      const int s = (int)(i & 1);
      const uint32_t ph = (uint32_t)((i >> 1) & 1);
      // x₂ registers are refilled column by column with the NEXT tile while the current one is converted (the last
      // tile re-reads itself: harmless, keeps the loop free of branches)
      const float* xn = (i + 1 < my_tiles) ? xt + tstride * ldx : xt;
      float dt[CW];
      unsigned emax[CW];
#pragma unroll
      for (int c = 0; c < CW; ++c) {
        float4 vc = cur[c];
        if (FOLD)
          vc = make_float4(fmaf(vc.x, preA.x, preC.x), fmaf(vc.y, preA.y, preC.y), fmaf(vc.z, preA.z, preC.z),
                           fmaf(vc.w, preA.w, preC.w));
        if (!active) vc = zero4;
        cur[c] = vc;
        const float mx = fmaxf(fmaxf(fabsf(vc.x), fabsf(vc.y)), fmaxf(fabsf(vc.z), fabsf(vc.w)));
        emax[c] = __reduce_max_sync(0xffffffffu, __float_as_uint(mx));  // bits of max|x₂ column|
        dt[c] = fmaf(vc.x, ws.x, fmaf(vc.y, ws.y, fmaf(vc.z, ws.z, vc.w * ws.w)));
      }
      // transposing butterfly: 8 dots over 32 lanes -> lane owns column `own`
#pragma unroll
      for (int half = CW / 2, off = 16; half >= 1; half >>= 1, off >>= 1) {
        const bool up = (lane & off) != 0;
#pragma unroll
        for (int q = 0; q < half; ++q) {
          const float sd_ = up ? dt[q] : dt[q + half], kd = up ? dt[q + half] : dt[q];
          dt[q] = kd + __shfl_xor_sync(0xffffffffu, sd_, off);
        }
      }
      float cdot = dt[0] + __shfl_xor_sync(0xffffffffu, dt[0], 2);
      cdot += __shfl_xor_sync(0xffffffffu, cdot, 1);
      if ((lane & 3) == 0 && P.logjac) {
        // Σ_j s_j = (Σ_j W_j)·x₂ + Σ_j c_j  (scale.jl:31); csum also carries the folded BatchNorm constants
        float* lp = P.logjac + col0 + own;
        const float b0 = P.accumulate ? *lp : 0.f;
        *lp = b0 + (INV ? -cdot : cdot) + csum;
      }
      bar_wait(sm_u32(&bars[2 + s]), ph ^ 1);  // stage free (MMAs that read it have completed)
      float* cslot = colscale + (int)(i & (TC_SCALE_SLOTS - 1)) * TC_T + p * CW;
#pragma unroll
      for (int c = 0; c < CW; ++c) {
        // power of two of the column maximum, clamped to [2^-100, 2^100]; operand scale 2^14 / that (exact)
        const float p2 = fminf(fmaxf(__uint_as_float(emax[c] & 0x7f800000u), 7.888609052210118e-31f), 1.2676506002282294e30f);
        const float scale = __uint_as_float(0x86000000u - __float_as_uint(p2));  // 2^(14 - e): max|x₂ col|·scale in [2^14, 2^15)
        if (lane == 0) cslot[c] = p2 * cs_mul;
        const float4 vc = cur[c];
        cur[c] = __ldcs(reinterpret_cast<const float4*>(xn + c * ldx));  // refill with the next tile's column
        if (active) {
          const float q0 = vc.x * scale, q1 = vc.y * scale, q2 = vc.z * scale, q3 = vc.w * scale;
          const __half2 h01 = __floats2half2_rn(q0, q1), h23 = __floats2half2_rn(q2, q3);
          const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
          const __half2 l01 = __floats2half2_rn(q0 - f01.x, q1 - f01.y), l23 = __floats2half2_rn(q2 - f23.x, q3 - f23.y);
          const int off = c * 128 + (c << 4);  // = (c<<4 | c<<7): XORed into the (disjoint) bits of st_base
          uint2 hi2, lo2;
          hi2.x = *reinterpret_cast<const unsigned*>(&h01);
          hi2.y = *reinterpret_cast<const unsigned*>(&h23);
          lo2.x = *reinterpret_cast<const unsigned*>(&l01);
          lo2.y = *reinterpret_cast<const unsigned*>(&l23);
          unsigned char* dst = sB + s * b_stage + (st_base ^ off);
          *reinterpret_cast<uint2*>(dst) = hi2;
          *reinterpret_cast<uint2*>(dst + lo_off) = lo2;
          if (write_y2) {  // x₂ passes through (plus the folded affines)
            float4 o = vc;
            if (FOLD)
              o = make_float4(fmaf(vc.x, postA.x, postC.x), fmaf(vc.y, postA.y, postC.y), fmaf(vc.z, postA.z, postC.z),
                              fmaf(vc.w, postA.w, postC.w));
            __stcs(reinterpret_cast<float4*>(yt + c * ldy), o);
          }
        }
      }
      // rows that belong to neither x₁ nor x₂ pass through when y != x
      if (rest_rows) {
        for (int c = 0; c < CW; ++c) {
          const long long col = col0 + c;
          for (int r = lane; r < P.D; r += 32) {
            const bool in1 = r >= P.row1 && r < P.row1 + P.n1, in2 = r >= P.row2 && r < P.row2 + P.n2;
            if (!in1 && !in2) {
              float xv = P.x[col * ldx + r];
              if (FOLD) xv = fmaf(fmaf(xv, P.fold[r], P.fold[P.D + r]), P.fold[2 * P.D + r], P.fold[3 * P.D + r]);
              P.y[col * ldy + r] = xv;
            }
          }
        }
      }
      fence_async_smem();  // generic-proxy smem writes -> visible to the tensor-core (async) proxy
      __syncwarp();
      if (lane == 0) bar_arrive(sm_u32(&bars[0 + s]));
      col0 += tstride;
      xt += tstride * ldx;
      if (write_y2) yt += tstride * ldy;
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 144;" ::: "memory");  // 64 accumulators + 32 x₁ values per thread
    // ================================ consumers ================================
    // Warpgroup g owns rows 64g..64g+63 of s and of t.  In the m64n64 accumulator layout, thread (warp w, lane l) of
    // the warpgroup holds rows j0 = 64g + 16(w%4) + l/4 and j0 + 8, columns 8i + 2(l%4) + {0, 1} (i = 0..7):
    // slot 4i + 2h + e is (row j0 + 8h, column 8i + 2(l%4) + e), identically for s and t.
    const int g = warp >> 2;
    const int j0 = 64 * g + 16 * (warp & 3) + (lane >> 2);
    const int cq = 2 * (lane & 3);  // first of this thread's two columns in every group of 8
    float cs_j[2], ct_j[2], preA_j[2], preC_j[2], postA_j[2], postC_j[2];
    bool store_j[2];
    int jr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = j0 + 8 * h;
      const bool rowok = j < P.n1;
      jr[h] = rowok ? j : 0;  // clamp: loads stay in bounds, stores are predicated
      store_j[h] = P.y != nullptr && rowok;
      cs_j[h] = (rowok && P.cvec) ? P.cvec[j] : 0.f;
      ct_j[h] = (rowok && P.cvec) ? P.cvec[P.n1 + j] : 0.f;
      preA_j[h] = 1.f, preC_j[h] = 0.f, postA_j[h] = 1.f, postC_j[h] = 0.f;
      if (FOLD && rowok) {
        preA_j[h] = P.fold[P.row1 + j];
        preC_j[h] = P.fold[P.D + P.row1 + j];
        postA_j[h] = P.fold[2 * P.D + P.row1 + j];
        postC_j[h] = P.fold[3 * P.D + P.row1 + j];
      }
    }
    const long long tstride = (long long)gridDim.x * TC_T;
    const float* xr = P.x + P.row1 + (long long)blockIdx.x * TC_T * ldx + cq * ldx;
    float* yr = P.y ? P.y + P.row1 + (long long)blockIdx.x * TC_T * ldy + cq * ldy : nullptr;
    const uint32_t wbar = sm_u32(&bars[4]);
    if (threadIdx.x == 0) {
      bar_expect_tx(wbar, (uint32_t)a_bytes);
      for (int off = 0; off < a_bytes; off += TC_ABLK) bulk_g2s(sm_u32(sA + off), P.wimg + off, TC_ABLK, wbar);
    }
    bar_wait(wbar, 0);
    const uint32_t aW = sm_u32(sA) + (uint32_t)(g * 64 * 128);  // rows 64g.. of a 128-row block: 8 swizzle atoms in

    for (long long i = 0; i < my_tiles; ++i) {
      const int s = (int)(i & 1);
      const uint32_t ph = (uint32_t)((i >> 1) & 1);
      // x₁ of this tile: requested first, in flight while the stage fills and the MMAs run
      float xv[32];
#pragma unroll
      for (int q = 0; q < 8; ++q)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) xv[4 * q + 2 * h + e] = __ldcs(xr + (8 * q + e) * ldx + jr[h]);
      float accs[32], acct[32];
      bar_wait(sm_u32(&bars[0 + s]), ph);  // x₂ operand stage filled
      const uint32_t bB = sm_u32(sB + s * b_stage);
      wg_fence_acc(accs);
      wg_fence_acc(acct);
      wg_fence();
      // smallest terms first: lo·hi, hi·lo, hi·hi
#pragma unroll
      for (int prod = 0; prod < 3; ++prod) {
        const int pa = prod == 0 ? 1 : 0, pb = prod == 1 ? 1 : 0;
        for (int kb = 0; kb < nkb; ++kb) {  // nkb is left rolled: unrolled, the chain spills in every variant
          const uint32_t as = aW + (uint32_t)(((0 * 2 + pa) * nkb + kb) * TC_ABLK);
          const uint32_t at = aW + (uint32_t)(((1 * 2 + pa) * nkb + kb) * TC_ABLK);
          const uint32_t baddr = bB + (uint32_t)((pb * nkb + kb) * TC_BBLK);
          const uint32_t first = prod == 0 && kb == 0;
#pragma unroll
          for (int j = 0; j < 4; ++j) {  // 4 K-steps of 16 fp16 (32 B) inside the 128-byte swizzle atom
            const uint64_t bd = gmma_desc_k_sw128(baddr + 32 * j);
            wgmma_m64n64k16(accs, gmma_desc_k_sw128(as + 32 * j), bd, first && j == 0 ? 0u : 1u);
            wgmma_m64n64k16(acct, gmma_desc_k_sw128(at + 32 * j), bd, first && j == 0 ? 0u : 1u);
          }
        }
      }
      wg_commit();
      wg_wait0();
      wg_fence_acc(accs);
      wg_fence_acc(acct);
      __syncwarp();
      if (lane == 0) bar_arrive(sm_u32(&bars[2 + s]));  // operand stage may be refilled

      const float* cs = colscale + (int)(i & (TC_SCALE_SLOTS - 1)) * TC_T + cq;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float2 f2 = *reinterpret_cast<const float2*>(cs + 8 * q);
        const float ff[2] = {f2.x, f2.y};
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = 4 * q + 2 * h + e;
            const float sv = fmaf(accs[n], ff[e], cs_j[h]);
            const float tv = fmaf(acct[n], ff[e], ct_j[h]);
            const float x1 = FOLD ? fmaf(xv[n], preA_j[h], preC_j[h]) : xv[n];
            float out;
            if (!INV) out = fmaf(__expf(sv), x1, tv);  // exp(s)·x₁ + t  (scale.jl:13, shift.jl:14)
            else out = (x1 - tv) * __expf(-sv);         // inv.(a) .* (y₁ + (−t))  (scale.jl:16, shift.jl:12)
            if (store_j[h]) __stcs(yr + (8 * q + e) * ldy + jr[h], FOLD ? fmaf(out, postA_j[h], postC_j[h]) : out);
          }
      }
      xr += tstride * ldx;
      if (yr) yr += tstride * ldy;
    }
  }
}

}  // namespace b2b

size_t b2b_coupling_tc_workspace_bytes(int n1, int n2) {
  if (n1 < 1 || n1 > 128 || (n2 != 64 && n2 != 128)) return 0;
  return (size_t)4 * (n2 / 64) * b2b::TC_ABLK + (size_t)n2 * sizeof(float) + 64;
}

// Returns B2B_EUNSUPPORTED when the layer shape does not fit the tensor-core path (the caller then uses the
// SIMT kernel).  The mask must be declared contiguous through desc.n2 / desc.n3 (first rows of idx1 / idx2).
int b2b_launch_coupling_affine_tc(const b2b_layer_desc& d, const float* fold, const float* x, float* y,
                                  float* logjac, int D, long long N, long long ldx, long long ldy, int accumulate,
                                  void* workspace, size_t workspace_bytes, int* launches, cudaStream_t stream) {
  using namespace b2b;
  const int n1 = d.n0, n2 = d.n1;
  const size_t need = b2b_coupling_tc_workspace_bytes(n1, n2);
  if (need == 0 || !workspace || workspace_bytes < need) return B2B_EUNSUPPORTED;
  const int row1 = d.n2, row2 = d.n3;
  if (row1 < 0 || row2 < 0 || row1 + n1 > D || row2 + n2 > D) return B2B_EUNSUPPORTED;
  if (fold && ((D % 4) || (reinterpret_cast<uintptr_t>(fold) & 15))) return B2B_EUNSUPPORTED;
  if ((row2 % 4) || (ldx % 4) || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(d.p0) & 15))
    return B2B_EUNSUPPORTED;
  if (y && ((ldy % 4) || (reinterpret_cast<uintptr_t>(y) & 15))) return B2B_EUNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(workspace) & 1023)) return B2B_EUNSUPPORTED;
  // the tensor-core kernel takes whole tiles of 64 columns; the ragged tail (< 64 columns) goes to the exact-fp32
  // kernel -- a disjoint column range, so in-place operation and logjac accumulation are unaffected
  const long long n_full = N / TC_T * TC_T;
  if (n_full < N) {
    const int rc = b2b_launch_coupling_affine(d, fold, x + n_full * ldx, y ? y + n_full * ldy : nullptr,
                                              logjac ? logjac + n_full : nullptr, D, N - n_full, ldx, ldy, accumulate, stream);
    if (rc != B2B_OK) return rc;
  }
  if (launches) *launches = (n_full < N ? 1 : 0) + (n_full > 0 ? 2 : 0);
  if (n_full == 0) return B2B_OK;
  N = n_full;
  const int nkb = n2 / 64;
  unsigned char* wimg = static_cast<unsigned char*>(workspace);
  float* wsum = reinterpret_cast<float*>(wimg + (size_t)4 * nkb * TC_ABLK);
  float* meta = wsum + n2;
  coupling_prep_kernel<<<1, 1024, 0, stream>>>(d.p0, d.p1, n1, n2, wimg, wsum, meta);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  TcParams P;
  P.x = x;
  P.y = y;
  P.logjac = logjac;
  P.wimg = wimg;
  P.wsum = wsum;
  P.meta = meta;
  P.fold = fold;
  P.cvec = d.p1;
  P.N = N;
  P.nkb = nkb;
  P.ldx = ldx;
  P.ldy = ldy;
  P.tiles = N / TC_T;
  P.D = D;
  P.n1 = n1;
  P.n2 = n2;
  P.row1 = row1;
  P.row2 = row2;
  P.accumulate = accumulate;
  P.inverse = d.inverse;
  const size_t smem = (size_t)4 * nkb * TC_ABLK + (size_t)TC_STAGES * 2 * nkb * TC_BBLK +
                      TC_SCALE_SLOTS * TC_T * sizeof(float) + 8 * sizeof(uint64_t) + 1024;
  const bool dense256 = ldx == 256 && (!y || ldy == 256);
  const bool inv = d.inverse != 0, fd = fold != nullptr;
  typedef void (*kernel_t)(const TcParams);
  kernel_t kernel;
  if (dense256) {
    kernel = fd ? (inv ? coupling_tc_kernel<256, true, true> : coupling_tc_kernel<256, true, false>)
                : (inv ? coupling_tc_kernel<256, false, true> : coupling_tc_kernel<256, false, false>);
  } else {
    kernel = fd ? (inv ? coupling_tc_kernel<0, true, true> : coupling_tc_kernel<0, true, false>)
                : (inv ? coupling_tc_kernel<0, false, true> : coupling_tc_kernel<0, false, false>);
  }
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  const int sms = b2b_sm_count();
  long long grid = sms;
  if (grid > P.tiles) grid = P.tiles;
  if (grid < 1) grid = 1;
  kernel<<<(int)grid, TC_THREADS, smem, stream>>>(P);
  return (int)cudaGetLastError();
}
