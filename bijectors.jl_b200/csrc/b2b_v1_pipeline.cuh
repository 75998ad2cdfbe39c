// TMA tile pipeline shared by the thread-per-column kernels (b2b_chain_v1.cu: layer interpreter,
// b2b_planar_const.cu: constant-bank planar chains).  See b2b_chain_v1.cu for the design notes.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdlib>
#include <mutex>

#include "b2b_device.cuh"

namespace b2b {

// ---- PTX wrappers ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "B2B_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra B2B_DONE;\n"
      "bra B2B_WAIT;\n"
      "B2B_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int c0, int c1, uint32_t src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(c0), "r"(c1), "r"(src)
               : "memory");
}
// 3-D forms: the tensor map views a batch as {32 floats, N columns, D/32 row-blocks} so that ONE instruction moves
// a whole [row-block][column][32 floats] tile (the 128-byte swizzle limits the innermost box extent to 32 floats)
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, int c0, int c1, int c2, uint32_t src) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(c0), "r"(c1), "r"(c2), "r"(src)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// 1-D bulk copy global -> shared (bytes % 16 == 0, both addresses 16-byte aligned), completion on an mbarrier
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void flag_store_release(int* p, int v) {
  asm volatile("st.release.cta.shared::cta.s32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ int flag_load_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.cta.shared::cta.s32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
  return v;
}

struct V1Extra {
  int n_in;        // input ring depth P
  int param_off;   // byte offset of the staged parameters in dynamic smem
  int bar_off;     // byte offset of the mbarriers
  int nwarps;
  int tma3d;       // 1: the tensor maps are 3-D (one TMA instruction per tile), 0: 2-D (one per 32-row block)
  long long tiles;
};

// Register layout of one thread: it owns rows [h*EPT, (h+1)*EPT) (h = part index, TPC parts per column) of CPT
// columns, as float2 pairs (b2b_ffma2 and friends: two scalar fp32 operations each on sm_90) that do
// the per-row work.  Every layer parameter that is loaded from shared memory is used for all CPT columns of the
// thread: at D = 128 (TPC = 2, CPT = 2) that halves the LDS wavefronts per column, which is what bounds the
// one-column-per-thread mapping.  Box ql (of NQT = EPT/32 boxes) slot r holds the LOGICAL 16-byte chunk r ^ rot
// (rot = h * 8/TPC keeps the TPC parts of a quarter-warp on different bank groups); pair index =
// (ql*8 + r)*2 + {0,1}.  prm() returns the float4 index of the parameters matching slot (ql, r).
template <int D, int TPC>
struct ColCtx {
  static constexpr int EPT = D / TPC;
  static constexpr int NQT = EPT / 32;
  int h, rot;
  __device__ __forceinline__ int prm(int ql, int r) const { return (h * NQT + ql) * 8 + (r ^ rot); }
  __device__ __forceinline__ int row(int ql, int r, int e) const { return prm(ql, r) * 4 + e; }
};

template <int TPC>
__device__ __forceinline__ float part_sum(float v) {
#pragma unroll
  for (int o = 1; o < TPC; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

#define B2B_FOR_SLOTS                        \
  _Pragma("unroll") for (int ql = 0; ql < C::NQT; ++ql) _Pragma("unroll") for (int r = 0; r < 8; ++r)
#define B2B_FOR_COLS _Pragma("unroll") for (int cc = 0; cc < CPT; ++cc)

// RadialLayer on register fragments (radial_layer.jl:43-72 forward, :88-102,124-129 inverse); parameters staged by
// stage_layer(B2B_RADIAL): z0[D] | α, β̂, α+β̂.
template <int D, int TPC, int CPT>
__device__ __forceinline__ void radial_apply(float2 (&x)[CPT][D / TPC / 2], const ColCtx<D, TPC>& c, const float* sp,
                                             bool inverse, float (&lj)[CPT]) {
  using C = ColCtx<D, TPC>;
  const float4* z4 = reinterpret_cast<const float4*>(sp);
  const float alpha = sp[D], bhat = sp[D + 1], apb = sp[D + 2];
  const float2 m1 = make_float2(-1.f, -1.f);
  float2 acc[CPT][4];
  B2B_FOR_COLS {
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[cc][i] = make_float2(0.f, 0.f);
  }
  B2B_FOR_SLOTS {
    const float4 z0 = z4[c.prm(ql, r)];
    const int i = (ql * 8 + r) * 2;
    B2B_FOR_COLS {
      const float2 d0 = b2b_ffma2(make_float2(z0.x, z0.y), m1, x[cc][i]);
      const float2 d1 = b2b_ffma2(make_float2(z0.z, z0.w), m1, x[cc][i + 1]);
      acc[cc][(r & 1) * 2 + 0] = b2b_ffma2(d0, d0, acc[cc][(r & 1) * 2 + 0]);
      acc[cc][(r & 1) * 2 + 1] = b2b_ffma2(d1, d1, acc[cc][(r & 1) * 2 + 1]);
    }
  }
  float2 g2[CPT];
  B2B_FOR_COLS {
    const float2 s = b2b_fadd2(b2b_fadd2(acc[cc][0], acc[cc][1]), b2b_fadd2(acc[cc][2], acc[cc][3]));
    const float nrm = sqrtf(part_sum<TPC>(s.x + s.y));  // radial_layer.jl:49 / :125
    float r_ = nrm;
    if (inverse) {
      const float a = apb - nrm;  // radial_layer.jl:126-127
      const float sq = sqrtf(fmaf(a, a, 4.0f * alpha * nrm));
      r_ = a > 0.f ? (2.0f * alpha * nrm) / (sq + a) : 0.5f * (sq - a);
    }
    const float hh = 1.0f / (alpha + r_);
    const float bh = bhat * hh;
    const float ljf = (float)(D - 1) * log1pf(bh) + log1pf(bh * alpha * hh);  // radial_layer.jl:68-70
    float g;
    if (!inverse) {
      g = bh;
      lj[cc] += ljf;
    } else {
      g = -bhat / (apb + r_);  // (α+r)/(α+β̂+r) − 1, radial_layer.jl:96
      lj[cc] -= ljf;
    }
    g2[cc] = make_float2(g, g);
  }
  B2B_FOR_SLOTS {
    const float4 z0 = z4[c.prm(ql, r)];
    const int i = (ql * 8 + r) * 2;
    B2B_FOR_COLS {
      const float2 d0 = b2b_ffma2(make_float2(z0.x, z0.y), m1, x[cc][i]);
      const float2 d1 = b2b_ffma2(make_float2(z0.z, z0.w), m1, x[cc][i + 1]);
      x[cc][i] = b2b_ffma2(g2[cc], d0, x[cc][i]);
      x[cc][i + 1] = b2b_ffma2(g2[cc], d1, x[cc][i + 1]);
    }
  }
}

// Terminal op of logpdf(td, y): lj += const − ½·Σ((x−μ)/σ)² (transformed_distribution.jl:165-169 + MvNormal logpdf);
// parameters staged by stage_layer(B2B_MVNORMAL_DIAG): μ | 1/σ | const.
template <int D, int TPC, int CPT>
__device__ __forceinline__ void mvnormal_apply(const float2 (&x)[CPT][D / TPC / 2], const ColCtx<D, TPC>& c,
                                               const float* sp, float (&lj)[CPT]) {
  using C = ColCtx<D, TPC>;
  const float4* mu4 = reinterpret_cast<const float4*>(sp);
  const float4* is4 = reinterpret_cast<const float4*>(sp + D);
  const float2 m1 = make_float2(-1.f, -1.f);
  float2 acc[CPT][2];
  B2B_FOR_COLS acc[cc][0] = acc[cc][1] = make_float2(0.f, 0.f);
  B2B_FOR_SLOTS {
    const float4 mu = mu4[c.prm(ql, r)], is = is4[c.prm(ql, r)];
    const int i = (ql * 8 + r) * 2;
    B2B_FOR_COLS {
      const float2 z0 = b2b_fmul2(b2b_ffma2(make_float2(mu.x, mu.y), m1, x[cc][i]), make_float2(is.x, is.y));
      const float2 z1 = b2b_fmul2(b2b_ffma2(make_float2(mu.z, mu.w), m1, x[cc][i + 1]), make_float2(is.z, is.w));
      acc[cc][0] = b2b_ffma2(z0, z0, acc[cc][0]);
      acc[cc][1] = b2b_ffma2(z1, z1, acc[cc][1]);
    }
  }
  B2B_FOR_COLS {
    const float2 s = b2b_fadd2(acc[cc][0], acc[cc][1]);
    lj[cc] += sp[2 * D] - 0.5f * part_sum<TPC>(s.x + s.y);
  }
}

// ---- sampling source: Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11; the
// counter-based generator of Random123 / cuRAND) + Box-Muller.  The four normals of rows 4k..4k+3 of GLOBAL column n
// come from the counter (lo32(n), hi32(n), k, lo32(offset)) under the key (lo32(seed), hi32(seed)): a sample depends
// only on (seed, offset, n, row), not on the launch geometry, so column shards on different ranks draw disjoint parts
// of one stream.  Restated for the tests in oracle/oracle_np.py (philox4x32_10, philox_normals), which also checks the
// three known-answer vectors of Random123.
struct V1Gen {
  unsigned long long seed, offset;
  long long col0;       // global index of column 0 of this launch
  const float* mu;      // base distribution MvNormal(mu, Diagonal(sigma.^2)): x = mu + sigma .* z; NULL = 0 / 1
  const float* sigma;
};

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                                              uint32_t (&out)[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c0;
  out[1] = c1;
  out[2] = c2;
  out[3] = c3;
}

// two standard normals from two 32-bit words: u = x·2^-32 + 2^-33 in (0, 1] (fp32), Box-Muller
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  const float u1 = fmaf(__uint2float_rn(a), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
  const float u2 = fmaf(__uint2float_rn(b), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
  // special-function-unit forms (lg2, sqrt, sin, cos: one MUFU each): the library-accurate logf / sincospif cost several
  // times the instructions; their absolute error (~2^-21) is far below the 1e-5 parity bar
  const float r = sqrtf(-1.3862943611198906f * __log2f(u1));  // sqrt(−2·ln u1)
  const float ang = 6.283185307179586f * u2 - 3.141592653589793f;  // 2π·u2 − π in (−π, π]: the accurate range of MUFU.SIN/COS
  z0 = -r * __cosf(ang);                                            // cos(2π u2) = −cos(2π u2 − π)
  z1 = -r * __sinf(ang);
}

// the four normals of rows 4k..4k+3 of global column n (optionally mapped through mu + sigma .* z)
__device__ __forceinline__ float4 philox_normal4(const V1Gen& g, long long n, int k) {
  uint32_t o[4];
  philox4x32_10((uint32_t)n, (uint32_t)((unsigned long long)n >> 32), (uint32_t)k, (uint32_t)g.offset, (uint32_t)g.seed,
                (uint32_t)(g.seed >> 32), o);
  float4 z;
  box_muller(o[0], o[1], z.x, z.y);
  box_muller(o[2], o[3], z.z, z.w);
  return z;
}

// The pipeline (TMA tile ring, register-resident fragments, per-warp TMA store) is independent of WHAT is applied
// to the fragments: `prog.stage()` prepares per-CTA state, `prog.apply()` maps the fragments and accumulates logjac.
//
// NIN = 2 (reverse-mode kernels): every input slot holds the tile of a SECOND D x N tensor (map_x2) behind the first.
// The program first consumes the fragment of the first tensor (`prog.phase1`), then the SAME registers are reloaded
// with the second tensor's fragment for `prog.apply` -- the register budget stays that of one column.  Per-tile
// program state travels in `Prog::State`; `apply` also receives the tile's first column index.
struct V1NoState {};

// GEN = true (sampling, rand(td, n)): there is no input batch -- every thread GENERATES the fragment of its column
// (philox_normal4), the input ring is unused and the kernel's only HBM traffic is the D x N store: 4·(D+1) B/sample.
template <int D, int TPC, int CPT, int NW, class Prog, int NIN = 1, bool GEN = false>
__device__ __forceinline__ void v1_run(const B2BChainParams& P, const V1Extra& E, const CUtensorMap& map_x,
                                       const CUtensorMap& map_y, const Prog& prog,
                                       const CUtensorMap* map_x2 = nullptr, const V1Gen* gen = nullptr) {
  using C = ColCtx<D, TPC>;
  constexpr int NQ = D / 32;                 // boxes per tile
  constexpr int LPC = 32 / TPC;              // lane groups per warp
  constexpr int COLS = LPC * CPT;            // columns per tile (= per warp)
  constexpr int BOX_BYTES = COLS * 128;      // COLS lines of 128 B
  constexpr int TILE_BYTES = NQ * BOX_BYTES;
  constexpr int SLOT_BYTES = NIN * TILE_BYTES;  // one input slot
  extern __shared__ unsigned char smem_dyn[];
  // the 128-byte swizzle pattern repeats every 1024 B: align the tile area by hand (1 KB of slack is allocated)
  unsigned char* smem_raw = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  unsigned char* in_base = smem_raw;                                    // n_in tiles
  unsigned char* out_base = smem_raw + (size_t)E.n_in * SLOT_BYTES;     // NW tiles
  float* params = reinterpret_cast<float*>(smem_raw + E.param_off);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + E.bar_off);
  // armed[b] = index j of the tile whose load has been issued into input buffer b.  A warp may only wait on
  // bars[b] for tile j once armed[b] == j: an mbarrier parity wait is only meaningful one phase ahead, and
  // with P < NW a warp could otherwise be two phases ahead of the buffer it shares with another warp.
  // (flag hand-off between warps: st.release / ld.acquire at CTA scope; compute-sanitizer's racecheck reports the
  // polling load against the releasing store -- that pairing is the synchronisation itself)
  int* armed = reinterpret_cast<int*>(bars + 8);

  // the warp index is made provably warp-uniform: tile / buffer / barrier addresses then live in uniform registers
  // and the TMA instructions take them directly (no per-instruction R2UR + BRA.U.ANY uniformisation loop)
  const int lane = threadIdx.x & 31, warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  auto load_tile = [&](uint32_t dst, int col0, uint32_t bar) {
    if (E.tma3d) {
      tma_load_3d(dst, &map_x, 0, col0, 0, bar);
      if (NIN == 2) tma_load_3d(dst + TILE_BYTES, map_x2, 0, col0, 0, bar);
    } else {
#pragma unroll
      for (int q = 0; q < NQ; ++q) tma_load_2d(dst + q * BOX_BYTES, &map_x, q * 32, col0, bar);
      if (NIN == 2) {
#pragma unroll
        for (int q = 0; q < NQ; ++q) tma_load_2d(dst + TILE_BYTES + q * BOX_BYTES, map_x2, q * 32, col0, bar);
      }
    }
  };
  // tiles of this CTA: global tile id = blockIdx.x + j * gridDim.x
  const long long my_tiles = (E.tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;
  // The first P tile loads are issued BEFORE the parameters are staged: the DRAM latency of the first tiles overlaps the prologue arithmetic (get_u_hat, spline records).
  if (threadIdx.x == 0 && !GEN) {
    for (int i = 0; i < E.n_in; ++i) mbar_init(smem_u32(&bars[i]), 1);
    fence_mbar_init();
    for (int j = 0; j < E.n_in && j < my_tiles; ++j) {
      const uint32_t bar = smem_u32(&bars[j]);
      mbar_expect_tx(bar, SLOT_BYTES);
      const long long tile = blockIdx.x + (long long)j * gridDim.x;
      load_tile(smem_u32(in_base + (size_t)j * SLOT_BYTES), (int)(tile * COLS), bar);
      flag_store_release(&armed[j], j);
    }
  }
  prog.stage(params, warp, lane, NW);
  __syncthreads();

  C ctx;
  const int t = lane / TPC;  // lane group: columns t, t + LPC, ... of the tile
  ctx.h = lane % TPC;
  ctx.rot = ctx.h * (8 / TPC);
  unsigned char* my_out = out_base + (size_t)warp * TILE_BYTES;
  // byte XOR: physical slot = r ^ rot ^ (line & 7); LPC is a multiple of 8, so it is the same for all CPT columns
  const int sw = (((t & 7) ^ ctx.rot) & 7) * 16;
  const int line = t * 128 + ctx.h * C::NQT * BOX_BYTES;  // this thread's first line inside its first box
  double dsum = 0.0;
  bool store_pending = false;

  for (long long j = warp; j < my_tiles; j += NW) {
    const int buf = (int)(j % E.n_in);
    const uint32_t parity = (uint32_t)((j / E.n_in) & 1);
    const long long tile = blockIdx.x + j * gridDim.x;
    const long long col = tile * COLS + t;
    if constexpr (!GEN) {
      while (flag_load_acquire(&armed[buf]) != (int)j) __nanosleep(20);
      mbar_wait(smem_u32(&bars[buf]), parity);
    }

    float2 x[CPT][C::EPT / 2];
    auto load_fragment = [&](const unsigned char* src) {
      B2B_FOR_COLS {
        B2B_FOR_SLOTS {
          const float4 v =
              *reinterpret_cast<const float4*>(src + cc * (LPC * 128) + ql * BOX_BYTES + ((r * 16) ^ sw));
          x[cc][(ql * 8 + r) * 2] = make_float2(v.x, v.y);
          x[cc][(ql * 8 + r) * 2 + 1] = make_float2(v.z, v.w);
        }
      }
    };
    if constexpr (GEN) {
      B2B_FOR_COLS {
        const long long n = gen->col0 + col + cc * LPC;
        B2B_FOR_SLOTS {
          const int row0 = ctx.row(ql, r, 0);
          float4 z = philox_normal4(*gen, n, row0 >> 2);
          if (gen->sigma) {
            const float4 sg = __ldg(reinterpret_cast<const float4*>(gen->sigma + row0));
            z = make_float4(z.x * sg.x, z.y * sg.y, z.z * sg.z, z.w * sg.w);
          }
          if (gen->mu) {
            const float4 m = __ldg(reinterpret_cast<const float4*>(gen->mu + row0));
            z = make_float4(z.x + m.x, z.y + m.y, z.z + m.z, z.w + m.w);
          }
          x[cc][(ql * 8 + r) * 2] = make_float2(z.x, z.y);
          x[cc][(ql * 8 + r) * 2 + 1] = make_float2(z.z, z.w);
        }
      }
    } else {
      load_fragment(in_base + (size_t)buf * SLOT_BYTES + line);
    }
    typename Prog::State st;
    if constexpr (NIN == 2) {
      prog.phase1(x, ctx, params, st);
      load_fragment(in_base + (size_t)buf * SLOT_BYTES + TILE_BYTES + line);
    }
    // The slot is about to be overwritten through the ASYNC proxy (TMA) after having been read through the generic
    // proxy (LDS): every lane orders its reads before later async-proxy accesses, then the warp converges.  Without
    // the proxy fence the refill can overtake reads that are still in flight (observed with the two-tensor slots:
    // torn tiles in the first refilled slot).
    if constexpr (!GEN) fence_proxy_async();
    __syncwarp();
    // re-arm this input buffer with the tile P steps ahead
    if (!GEN && lane == 0 && j + E.n_in < my_tiles) {
      const uint32_t bar = smem_u32(&bars[buf]);
      mbar_expect_tx(bar, SLOT_BYTES);
      const long long nt = blockIdx.x + (j + E.n_in) * gridDim.x;
      load_tile(smem_u32(in_base + (size_t)buf * SLOT_BYTES), (int)(nt * COLS), bar);
      flag_store_release(&armed[buf], (int)(j + E.n_in));
    }

    float lj[CPT];
    B2B_FOR_COLS {
      const long long cl = col + cc * LPC;
      lj[cc] = (P.accumulate && P.logjac && cl < P.N) ? P.logjac[cl] : 0.0f;
    }
    if constexpr (NIN == 2) prog.apply(x, ctx, params, lj, st, col);
    else prog.apply(x, ctx, params, lj);

    if (P.y) {
      if (store_pending) {
        if (lane == 0) tma_wait_read0();  // previous store of this warp has finished reading my_out
        __syncwarp();
      }
      unsigned char* dst = my_out + line;
      B2B_FOR_COLS {
        B2B_FOR_SLOTS {
          const float2 a = x[cc][(ql * 8 + r) * 2], b = x[cc][(ql * 8 + r) * 2 + 1];
          *reinterpret_cast<float4*>(dst + cc * (LPC * 128) + ql * BOX_BYTES + ((r * 16) ^ sw)) =
              make_float4(a.x, a.y, b.x, b.y);
        }
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) {
        if (E.tma3d) {
          tma_store_3d(&map_y, 0, (int)(tile * COLS), 0, smem_u32(my_out));
        } else {
#pragma unroll
          for (int q = 0; q < NQ; ++q)
            tma_store_2d(&map_y, q * 32, (int)(tile * COLS), smem_u32(my_out + q * BOX_BYTES));
        }
        tma_commit();
      }
      store_pending = true;
    }
    if (ctx.h == 0) {
      B2B_FOR_COLS {
        const long long cl = col + cc * LPC;
        if (cl < P.N) {
          if (P.logjac && !(P.accumulate & 2)) P.logjac[cl] = lj[cc];  // accumulate bit 1: logjac is read-only
          dsum += (double)lj[cc];
        }
      }
    }
  }
  if (lane == 0 && store_pending) tma_wait_all0();  // smem must stay valid until the stores have drained

  if (P.partials) {
    __shared__ double red[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
    if (lane == 0) red[warp] = dsum;
    __syncthreads();
    if (threadIdx.x == 0) {
      double tt = 0.0;
      for (int w = 0; w < NW; ++w) tt += red[w];
      P.partials[blockIdx.x] = tt;
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------------
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline encode_tiled_fn get_encode() {
  static encode_tiled_fn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<encode_tiled_fn>(p);
  });
  return fn;
}

static inline bool make_map(CUtensorMap* m, const float* base, int D, long long N, long long ld, int cols, bool three_d) {
  encode_tiled_fn enc = get_encode();
  if (!enc) return false;
  const cuuint32_t estr[3] = {1, 1, 1};
  if (three_d) {
    // {32 floats, N columns, D/32 row-blocks}: the row-block stride (128 B) is SMALLER than the column stride
    const cuuint64_t dims[3] = {32, (cuuint64_t)N, (cuuint64_t)(D / 32)};
    const cuuint64_t strides[2] = {(cuuint64_t)ld * sizeof(float), 128};
    const cuuint32_t box[3] = {32, (cuuint32_t)cols, (cuuint32_t)(D / 32)};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)D, (cuuint64_t)N};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
  const cuuint32_t box[2] = {32, (cuuint32_t)cols};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Both maps of a launch; 3-D when the driver accepts them (B2B_V1_TMA=2 forces the 2-D form)
static inline bool make_maps(const B2BChainParams& q, int cols, CUtensorMap* mx, CUtensorMap* my, int* tma3d) {
  static const int force2d = getenv("B2B_V1_TMA") && atoi(getenv("B2B_V1_TMA")) == 2;
  for (int three_d = force2d ? 0 : 1; three_d >= 0; --three_d) {
    if (three_d && q.D == 32) continue;  // one row-block: the 2-D form already is one instruction
    bool ok = make_map(mx, q.x, q.D, q.N, q.ldx, cols, three_d != 0);
    if (ok && q.y) ok = make_map(my, q.y, q.D, q.N, q.ldy, cols, three_d != 0);
    if (ok) {
      if (!q.y) *my = *mx;
      *tma3d = three_d;
      return true;
    }
  }
  return false;
}

// Shared-memory / grid geometry of one launch: NW per-warp output tiles, as many input tiles as fit (<= 8),
// `param_floats` floats of staged parameters, the mbarriers and flags.
struct V1Geom {
  int nw, grid, cols;
  size_t smem;
  V1Extra extra;
};

static inline int v1_check_io(const B2BChainParams& p) {
  if (p.N >= (1ll << 31) - 64) return B2B_EUNSUPPORTED;
  if ((p.ldx % 4) || (reinterpret_cast<uintptr_t>(p.x) & 15)) return B2B_EUNSUPPORTED;
  if (p.y && ((p.ldy % 4) || (reinterpret_cast<uintptr_t>(p.y) & 15))) return B2B_EUNSUPPORTED;
  return 0;
}

static inline int v1_geometry(int D, long long N, int nw, int cols, size_t param_floats, V1Geom& g,
                              int in_tiles = 1) {
  const int tile_bytes = D * 4 * cols;
  const size_t param_bytes = param_floats * sizeof(float);
  const size_t budget = 225 * 1024;
  const size_t fixed = (size_t)nw * tile_bytes + ((param_bytes + 15) & ~(size_t)15) + 16 * sizeof(uint64_t) + 1024;
  const size_t slot_bytes = (size_t)in_tiles * tile_bytes;
  if (fixed + 2 * slot_bytes > budget) return B2B_EUNSUPPORTED;
  int n_in = (int)((budget - fixed) / slot_bytes);
  if (n_in > 8) n_in = 8;
  g.nw = nw;
  g.cols = cols;
  g.extra.n_in = n_in;
  g.extra.nwarps = nw;
  g.extra.tma3d = 0;
  g.extra.param_off = n_in * (int)slot_bytes + nw * tile_bytes;
  g.extra.bar_off = g.extra.param_off + (int)((param_bytes + 15) & ~(size_t)15);
  g.extra.tiles = (N + cols - 1) / cols;
  g.smem = (size_t)g.extra.bar_off + 16 * sizeof(uint64_t) + 1024;  // +1024: base alignment slack
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long grid = sms;
  const long long want = (g.extra.tiles + nw - 1) / nw;
  if (grid > want) grid = want;
  if (grid < 1) grid = 1;
  g.grid = (int)grid;
  return 0;
}

}  // namespace b2b
