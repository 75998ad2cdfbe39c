// C ABI of libb2b.so (include/b2b.h): argument validation, chain segmentation, launch bookkeeping.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "b2b_internal.h"

int b2b_chain_grid_size_v0(const B2BChainParams& p);
int b2b_chain_grid_size_v1(const B2BChainParams& p);

static thread_local int g_last_launches = 0;
// kernel selection of b2b_set_kernel_variant: per calling thread (no mutable process-global state)
static thread_local int g_variant = 0;           // fused chain kernel: 0 auto, 1 v0, 2 v1 interpreter, 3 planar chain
static thread_local int g_fold_bn = 1;            // fold BatchNorm neighbours into coupling launches (hundreds digit 1 disables)
static thread_local int g_coupling_variant = 0;  // coupling: 0 auto (tensor cores when possible), 1 force the fp32 CUDA-core kernel

extern "C" int b2b_version(void) { return B2B_VERSION; }

extern "C" const char* b2b_status_string(int status) {
  switch (status) {
    case B2B_OK: return "ok";
    case B2B_EINVAL: return "b2b: invalid argument (null pointer, shape, range or alignment)";
    case B2B_EUNSUPPORTED: return "b2b: not implemented on the device path (no CPU fallback exists)";
    case B2B_EWORKSPACE: return "b2b: workspace too small (see b2b_chain_workspace_bytes)";
    case B2B_ENONCCL: return "b2b: libnccl.so.2 could not be loaded";
    default: break;
  }
  if (status >= 100000) return "b2b: NCCL error (status - 100000 is the ncclResult_t)";
  switch (status) {
    default: break;
  }
  if (status > 0) return cudaGetErrorString(static_cast<cudaError_t>(status));
  return "b2b: unknown status";
}

extern "C" int b2b_last_launch_count(void) { return g_last_launches; }

extern "C" int b2b_set_kernel_variant(int variant) {
  // low decimal digit: fused chain kernel variant; tens digit: coupling variant (10 = force fp32 CUDA cores)
  const int chain = variant % 10, cpl = (variant / 10) % 10, nofold = variant / 100;
  if (variant < 0 || chain > 3 || cpl > 1 || nofold > 1) return B2B_EINVAL;
  g_variant = chain;
  g_coupling_variant = cpl;
  g_fold_bn = nofold ? 0 : 1;
  return B2B_OK;
}

static bool fusable(int kind) {
  return kind == B2B_PLANAR || kind == B2B_RADIAL || kind == B2B_RQS || kind == B2B_BATCHNORM ||
         kind == B2B_PERMUTE || kind == B2B_STACKED_EW || kind == B2B_MVNORMAL_DIAG;
}

static int validate_layer(const b2b_layer_desc& d, int D, bool last) {
  switch (d.kind) {
    case B2B_PLANAR:
      if (!d.p0 || !d.p1 || !d.p2) return B2B_EINVAL;
      break;
    case B2B_RADIAL:
      if (!d.p0 || !d.p1 || !d.p2) return B2B_EINVAL;
      break;
    case B2B_RQS:
      if (!d.p0 || !d.p1 || !d.p2 || d.n0 < 2) return B2B_EINVAL;
      if (d.n0 > 64) return B2B_EUNSUPPORTED;
      break;
    case B2B_COUPLING_AFFINE:
      if (!d.p0 || d.n0 < 1 || d.n1 < 1 || d.n0 + d.n1 > D) return B2B_EINVAL;
      if ((!d.i0 && d.n2 < 0) || (!d.i1 && d.n3 < 0)) return B2B_EINVAL;
      break;
    case B2B_BATCHNORM:
      if (!d.p0 || !d.p1 || !d.p2 || !d.p3) return B2B_EINVAL;
      break;
    case B2B_PERMUTE:
      if (!d.i0) return B2B_EINVAL;
      break;
    case B2B_STACKED_EW:
      if (!d.i0) return B2B_EINVAL;
      break;
    case B2B_MVNORMAL_DIAG:
      if (!last || d.inverse) return B2B_EINVAL;
      break;
    default:
      return B2B_EINVAL;
  }
  return B2B_OK;
}

// number of kernel launches the last launch_fused enqueued (the constant-bank path adds a prep kernel and a copy)
static thread_local int g_fused_launches = 1;

static int launch_fused(B2BChainParams& p, cudaStream_t stream) {
  int rc = B2B_EUNSUPPORTED;
  g_fused_launches = 1;
  // segments made of <= 8 PlanarLayers: the fused planar chain kernel (variant 3 forces, 1 / 2 disable)
  if (g_variant == 0 || g_variant == 3) {
    rc = b2b_launch_planar_chain_const(p, stream);
    if (rc == B2B_OK) {
      g_fused_launches = 1;
      return rc;
    }
    if (g_variant == 3 || rc != B2B_EUNSUPPORTED) return rc;
  }
  if (g_variant == 0 && b2b_radial_unrolled_applicable(p)) {  // inverse radial chains: specialised program
    rc = b2b_launch_radial_unrolled(p, stream);
    if (rc != B2B_EUNSUPPORTED) return rc;
  }
  if (g_variant == 0 && b2b_rqs_unrolled_applicable(p)) {  // one RQS layer, K = 8 bins: specialised program
    rc = b2b_launch_rqs_unrolled(p, stream);
    if (rc != B2B_EUNSUPPORTED) return rc;
  }
  if (g_variant != 1) {
    rc = b2b_launch_chain_v1(p, stream);
    if (rc == B2B_OK) return rc;
    if (g_variant == 2 || rc != B2B_EUNSUPPORTED) return rc;
  }
  return b2b_launch_chain_v0(p, stream);
}

static int fused_grid(const B2BChainParams& p) {
  if ((g_variant == 0 || g_variant == 3) && b2b_planar_const_layers(p) > 0) {
    const int g = b2b_planar_const_grid_size(p);
    if (g > 0 || g_variant == 3) return g;
  }
  if (g_variant == 0 && (b2b_rqs_unrolled_applicable(p) || b2b_radial_unrolled_applicable(p))) {  // same warps-per-D table as the planar kernels
    const int g = b2b_planar_const_grid_size(p);
    if (g > 0) return g;
  }
  if (g_variant != 1) {
    const int g = b2b_chain_grid_size_v1(p);
    if (g > 0) return g;
  }
  return b2b_chain_grid_size_v0(p);
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// workspace layout: [tensor-core W image (shared by all coupling layers; they run one after another)]
//                   [D x N scratch when y == NULL and the chain has several segments] [batch-sum partials]
static size_t fold_bytes(int D) { return align_up((size_t)(4 * D + 4) * sizeof(float), 1024); }

static bool chain_has_fold(const b2b_layer_desc* layers, int32_t L) {
  for (int l = 0; l < L; ++l)
    if (layers[l].kind == B2B_COUPLING_AFFINE &&
        ((l > 0 && layers[l - 1].kind == B2B_BATCHNORM) || (l + 1 < L && layers[l + 1].kind == B2B_BATCHNORM)))
      return true;
  return false;
}

// [BatchNorm fold table (only when a BatchNorm neighbours a coupling)][tensor-core W image], each 1024-aligned,
// + 1024 of alignment slack
static size_t chain_tc_bytes(const b2b_layer_desc* layers, int32_t L, int D) {
  size_t tc = 0;
  for (int l = 0; l < L; ++l)
    if (layers[l].kind == B2B_COUPLING_AFFINE && layers[l].n2 >= 0 && layers[l].n3 >= 0) {
      const size_t b = b2b_coupling_tc_workspace_bytes(layers[l].n0, layers[l].n1);
      if (b > tc) tc = b;
    }
  const size_t fb = chain_has_fold(layers, L) ? fold_bytes(D) : 0;
  if (!tc && !fb) return 0;
  return fb + (tc ? align_up(tc, 1024) : 0) + 1024;
}

extern "C" size_t b2b_coupling_workspace_bytes(int32_t n1, int32_t n2) {
  const size_t b = b2b_coupling_tc_workspace_bytes(n1, n2);
  return b ? align_up(b, 1024) + 1024 : 0;
}

extern "C" size_t b2b_chain_workspace_bytes(const b2b_layer_desc* layers, int32_t L, int32_t D, int64_t N,
                                            int want_y, int want_sum) {
  size_t bytes = chain_tc_bytes(layers, L, D);
  bool has_coupling = false;
  for (int l = 0; l < L; ++l) has_coupling |= layers[l].kind == B2B_COUPLING_AFFINE;
  // a D x N scratch matrix is needed only when y == NULL but the chain has more than one segment
  if (!want_y && has_coupling && L > 1) bytes += align_up((size_t)D * (size_t)N * sizeof(float), 1024);
  if (want_sum) bytes += 4096 * sizeof(double);
  return bytes;
}

extern "C" size_t b2b_workspace_bytes(const b2b_layer_desc* op, int32_t D, int64_t N) {
  return op ? b2b_chain_workspace_bytes(op, 1, D, N, 1, 0) : 0;
}

extern "C" int b2b_chain_run_f32(const b2b_layer_desc* layers, int32_t L, const float* x, float* y,
                                 float* logjac, double* sum_out, int32_t D, int64_t N, int64_t ldx,
                                 int64_t ldy, int accumulate_logjac, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  g_last_launches = 0;
  if (!layers || L < 1 || L > B2B_MAX_CHAIN || D < 1 || N < 0 || ldx < D) return B2B_EINVAL;
  if (N == 0) {  // empty batch: nothing to launch (pointers may be NULL)
    if (sum_out) return (int)cudaMemsetAsync(sum_out, 0, sizeof(double), stream);
    return B2B_OK;
  }
  if (!x) return B2B_EINVAL;
  if (y && ldy < D) return B2B_EINVAL;
  if (!y && !logjac && !sum_out) return B2B_EINVAL;
  for (int l = 0; l < L; ++l) {
    const int rc = validate_layer(layers[l], D, l == L - 1);
    if (rc != B2B_OK) return rc;
  }
  if (N == 0) {
    if (sum_out) return (int)cudaMemsetAsync(sum_out, 0, sizeof(double), stream);
    return B2B_OK;
  }
  const bool terminal = layers[L - 1].kind == B2B_MVNORMAL_DIAG;
  if (sum_out && !logjac && !terminal) return B2B_EINVAL;

  // segments: maximal runs of fusable layers, and single coupling layers
  struct Seg {
    int begin, end;
    bool coupling;
    int pre, post;  // layer index of a BatchNorm folded into this coupling launch (-1: none)
  };
  std::vector<Seg> segs;
  for (int l = 0; l < L;) {
    if (layers[l].kind == B2B_COUPLING_AFFINE) {
      segs.push_back({l, l + 1, true, -1, -1});
      ++l;
    } else {
      int e = l;
      while (e < L && fusable(layers[e].kind)) ++e;
      segs.push_back({l, e, false, -1, -1});
      l = e;
    }
  }
  // workspace carve-up
  char* ws = static_cast<char*>(workspace);
  size_t ws_left = workspace ? workspace_bytes : 0;
  void* tc_ws = nullptr;
  size_t tc_bytes = 0;
  float* fold_ws = nullptr;
  {
    const size_t want = chain_tc_bytes(layers, L, D);
    if (want && ws_left >= want) {
      const size_t pad = (1024 - (reinterpret_cast<uintptr_t>(ws) & 1023)) & 1023;
      const size_t fb = chain_has_fold(layers, L) ? fold_bytes(D) : 0;
      if (fb) fold_ws = reinterpret_cast<float*>(ws + pad);
      if (want > fb + 1024) {
        tc_ws = ws + pad + fb;
        tc_bytes = want - pad - fb;
      }
      ws += want;
      ws_left -= want;
    }
  }
  // fold BatchNorm neighbours (a per-row affine) into the coupling launches: removes their own pass over HBM
  if (fold_ws && g_fold_bn) {
    for (size_t s = 0; s < segs.size(); ++s) {
      if (!segs[s].coupling) continue;
      if (s + 1 < segs.size() && !segs[s + 1].coupling && segs[s + 1].end > segs[s + 1].begin &&
          layers[segs[s + 1].begin].kind == B2B_BATCHNORM)
        segs[s].post = segs[s + 1].begin++;
      if (s > 0 && !segs[s - 1].coupling && segs[s - 1].end > segs[s - 1].begin &&
          layers[segs[s - 1].end - 1].kind == B2B_BATCHNORM)
        segs[s].pre = --segs[s - 1].end;
    }
    std::vector<Seg> kept;
    for (const Seg& g : segs)
      if (g.coupling || g.end > g.begin) kept.push_back(g);
    segs.swap(kept);
  }
  float* scratch = nullptr;
  if (!y && segs.size() > 1) {
    const size_t need = align_up((size_t)D * (size_t)N * sizeof(float), 1024);
    if (ws_left < need) return B2B_EWORKSPACE;
    scratch = reinterpret_cast<float*>(ws);
    ws += need;
    ws_left -= need;
  }
  double* partials = nullptr;
  if (sum_out) {
    if (segs.back().coupling) return B2B_EUNSUPPORTED;  // batch sum needs a fusable last segment
    if (ws_left < 4096 * sizeof(double)) return B2B_EWORKSPACE;
    partials = reinterpret_cast<double*>(ws);
  }

  const float* cur = x;
  long long cur_ld = ldx;
  bool lj_started = accumulate_logjac != 0;
  for (size_t s = 0; s < segs.size(); ++s) {
    const bool last_seg = s + 1 == segs.size();
    // destination of this segment: y when given, else scratch for intermediates, nothing for the last
    float* dst = y ? y : (last_seg ? nullptr : scratch);
    const long long dst_ld = y ? ldy : D;
    int rc;
    if (segs[s].coupling) {
      float* cdst = dst;
      // logjac-only call with a trailing coupling layer still needs no store
      const float* fold = nullptr;
      if (segs[s].pre >= 0 || segs[s].post >= 0) {
        rc = b2b_launch_bn_fold_prep(segs[s].pre >= 0 ? &layers[segs[s].pre] : nullptr,
                                     segs[s].post >= 0 ? &layers[segs[s].post] : nullptr, D, fold_ws, stream);
        if (rc != B2B_OK) return rc;
        ++g_last_launches;
        fold = fold_ws;
      }
      rc = B2B_EUNSUPPORTED;
      if (tc_ws && g_coupling_variant != 1) {
        int n_launch = 0;
        rc = b2b_launch_coupling_affine_tc(layers[segs[s].begin], fold, cur, cdst, logjac, D, N, cur_ld, dst_ld,
                                           lj_started ? 1 : 0, tc_ws, tc_bytes, &n_launch, stream);
        if (rc == B2B_OK) g_last_launches += n_launch;  // W preparation + main kernel (+ fp32 kernel on a ragged tail)
      }
      if (rc == B2B_EUNSUPPORTED) {
        rc = b2b_launch_coupling_affine(layers[segs[s].begin], fold, cur, cdst, logjac, D, N, cur_ld, dst_ld,
                                        lj_started ? 1 : 0, stream);
        if (rc == B2B_OK) ++g_last_launches;
      }
      if (rc != B2B_OK) return rc;
    } else {
      B2BChainParams p;
      memset(&p, 0, sizeof(p));
      p.x = cur;
      p.y = dst;
      p.logjac = logjac;
      p.N = N;
      p.ldx = cur_ld;
      p.ldy = dst_ld;
      p.D = D;
      p.L = segs[s].end - segs[s].begin;
      p.accumulate = lj_started ? 1 : 0;
      for (int l = 0; l < p.L; ++l) p.layers[l] = layers[segs[s].begin + l];
      int grid = 0;
      if (sum_out && last_seg) {
        grid = fused_grid(p);
        if (grid <= 0 || grid > 4096) return B2B_EUNSUPPORTED;
        p.partials = partials;
      }
      rc = launch_fused(p, stream);
      if (rc != B2B_OK) return rc;
      g_last_launches += g_fused_launches;
      if (sum_out && last_seg) {
        rc = b2b_launch_sum_partials(partials, grid, sum_out, stream);
        if (rc != B2B_OK) return rc;
        ++g_last_launches;
      }
    }
    if (dst) {
      cur = dst;
      cur_ld = dst_ld;
    }
    lj_started = true;
  }
  return B2B_OK;
}

// ---- single-layer wrappers -------------------------------------------------------------------------
static int run1(const b2b_layer_desc& d, const float* x, float* y, float* logjac, int32_t D, int64_t N,
                int64_t ldx, int64_t ldy, int acc, void* stream) {
  return b2b_chain_run_f32(&d, 1, x, y, logjac, nullptr, D, N, ldx, ldy, acc, nullptr, 0, stream);
}

static b2b_layer_desc mk(int kind, int inverse) {
  b2b_layer_desc d;
  memset(&d, 0, sizeof(d));
  d.kind = kind;
  d.inverse = inverse;
  return d;
}

#define B2B_PLANAR_IMPL(NAME, INV)                                                                       \
  extern "C" int NAME(const float* x, float* y, float* logjac, const float* w, const float* u,           \
                      const float* b, int32_t D, int64_t N, int64_t ldx, int64_t ldy, int acc,           \
                      void* stream) {                                                                    \
    b2b_layer_desc d = mk(B2B_PLANAR, INV);                                                              \
    d.p0 = w;                                                                                            \
    d.p1 = u;                                                                                            \
    d.p2 = b;                                                                                            \
    return run1(d, x, y, logjac, D, N, ldx, ldy, acc, stream);                                           \
  }
B2B_PLANAR_IMPL(b2b_planar_fwd_f32, 0)
B2B_PLANAR_IMPL(b2b_planar_inv_f32, 1)

#define B2B_RADIAL_IMPL(NAME, INV)                                                                       \
  extern "C" int NAME(const float* x, float* y, float* logjac, const float* alpha_raw,                   \
                      const float* beta, const float* z0, int32_t D, int64_t N, int64_t ldx,             \
                      int64_t ldy, int acc, void* stream) {                                              \
    b2b_layer_desc d = mk(B2B_RADIAL, INV);                                                              \
    d.p0 = alpha_raw;                                                                                    \
    d.p1 = beta;                                                                                         \
    d.p2 = z0;                                                                                           \
    return run1(d, x, y, logjac, D, N, ldx, ldy, acc, stream);                                           \
  }
B2B_RADIAL_IMPL(b2b_radial_fwd_f32, 0)
B2B_RADIAL_IMPL(b2b_radial_inv_f32, 1)

#define B2B_RQS_IMPL(NAME, INV)                                                                          \
  extern "C" int NAME(const float* x, float* y, float* logjac, const float* widths,                      \
                      const float* heights, const float* derivs, int32_t K1, int32_t D, int64_t N,       \
                      int64_t ldx, int64_t ldy, int acc, void* stream) {                                 \
    b2b_layer_desc d = mk(B2B_RQS, INV);                                                                 \
    d.p0 = widths;                                                                                       \
    d.p1 = heights;                                                                                      \
    d.p2 = derivs;                                                                                       \
    d.n0 = K1;                                                                                           \
    return run1(d, x, y, logjac, D, N, ldx, ldy, acc, stream);                                           \
  }
B2B_RQS_IMPL(b2b_rqs_fwd_f32, 0)
B2B_RQS_IMPL(b2b_rqs_inv_f32, 1)

#define B2B_COUPLING_IMPL(NAME, INV)                                                                     \
  extern "C" int NAME(const float* x, float* y, float* logjac, const int32_t* idx1, int32_t n1, int32_t row1, \
                      const int32_t* idx2, int32_t n2, int32_t row2, const float* W, const float* c,        \
                      int32_t D, int64_t N, int64_t ldx, int64_t ldy, int acc, void* workspace,             \
                      size_t workspace_bytes, void* stream) {                                               \
    b2b_layer_desc d = mk(B2B_COUPLING_AFFINE, INV);                                                     \
    d.p0 = W;                                                                                            \
    d.p1 = c;                                                                                            \
    d.i0 = idx1;                                                                                         \
    d.i1 = idx2;                                                                                         \
    d.n0 = n1;                                                                                           \
    d.n1 = n2;                                                                                           \
    d.n2 = row1;                                                                                         \
    d.n3 = row2;                                                                                         \
    return b2b_chain_run_f32(&d, 1, x, y, logjac, nullptr, D, N, ldx, ldy, acc, workspace, workspace_bytes, \
                             stream);                                                                    \
  }
B2B_COUPLING_IMPL(b2b_coupling_affine_fwd_f32, 0)
B2B_COUPLING_IMPL(b2b_coupling_affine_inv_f32, 1)

#define B2B_BN_IMPL(NAME, INV)                                                                           \
  extern "C" int NAME(const float* x, float* y, float* logjac, const float* b, const float* logs,        \
                      const float* m, const float* v, float eps, int32_t D, int64_t N, int64_t ldx,      \
                      int64_t ldy, int acc, void* stream) {                                              \
    b2b_layer_desc d = mk(B2B_BATCHNORM, INV);                                                           \
    d.p0 = b;                                                                                            \
    d.p1 = logs;                                                                                         \
    d.p2 = m;                                                                                            \
    d.p3 = v;                                                                                            \
    d.f0 = eps;                                                                                          \
    return run1(d, x, y, logjac, D, N, ldx, ldy, acc, stream);                                           \
  }
B2B_BN_IMPL(b2b_batchnorm_eval_fwd_f32, 0)
B2B_BN_IMPL(b2b_batchnorm_eval_inv_f32, 1)

extern "C" int b2b_permute_rows_f32(const float* x, float* y, float* logjac, const int32_t* dst_of_src,
                                    int inverse, int32_t D, int64_t N, int64_t ldx, int64_t ldy, int acc,
                                    void* stream) {
  b2b_layer_desc d = mk(B2B_PERMUTE, inverse ? 1 : 0);
  d.i0 = dst_of_src;
  return run1(d, x, y, logjac, D, N, ldx, ldy, acc, stream);
}

extern "C" int b2b_stacked_elementwise_f32(const float* x, float* y, float* logjac, const int32_t* code,
                                           const float* a, const float* b, int inverse, int32_t D, int64_t N,
                                           int64_t ldx, int64_t ldy, int acc, void* stream) {
  b2b_layer_desc d = mk(B2B_STACKED_EW, inverse ? 1 : 0);
  d.i0 = code;
  d.p0 = a;
  d.p1 = b;
  return run1(d, x, y, logjac, D, N, ldx, ldy, acc, stream);
}

extern "C" int b2b_mvnormal_diag_logpdf_f32(const float* x, const float* mu, const float* sigma,
                                            const float* logjac_in, float* logpdf_out, double* sum_out,
                                            int32_t D, int64_t N, int64_t ldx, void* workspace,
                                            size_t workspace_bytes, void* stream) {
  if (!logpdf_out && !sum_out) return B2B_EINVAL;
  b2b_layer_desc d = mk(B2B_MVNORMAL_DIAG, 0);
  d.p0 = mu;
  d.p1 = sigma;
  int acc = 0;
  if (logjac_in) {
    if (!logpdf_out) return B2B_EINVAL;
    if (logjac_in != logpdf_out) {
      cudaError_t e = cudaMemcpyAsync(logpdf_out, logjac_in, (size_t)N * sizeof(float),
                                      cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream));
      if (e != cudaSuccess) return (int)e;
    }
    acc = 1;
  }
  return b2b_chain_run_f32(&d, 1, x, nullptr, logpdf_out, sum_out, D, N, ldx, D, acc, workspace,
                           workspace_bytes, stream);
}

// ---- planar chains with HOST-resident parameters ---------------------------------------------------------
// get_u_hat (planar_layer.jl:65-70) on the host: û = u + (m(wᵀu) − wᵀu)·w/‖w‖², m(x) = −1 + softplus(x); c = wᵀû.
static float softplus_host(float x) { return x > 0.f ? x + log1pf(expf(-x)) : log1pf(expf(x)); }

static void planar_derive_host(const float* w, const float* u, int D, float* uh, float* c) {
  double wu = 0.0, ww = 0.0;
  for (int i = 0; i < D; ++i) {
    wu += (double)w[i] * u[i];
    ww += (double)w[i] * w[i];
  }
  const float s = (float)wu;
  const float k = (softplus_host(-s) - 1.0f) / (float)ww;  // (m(wᵀu) − wᵀu)/‖w‖², planar_layer.jl:67
  for (int i = 0; i < D; ++i) uh[i] = fmaf(k, w[i], u[i]);
  *c = softplus_host(s) - 1.0f;  // wᵀû = m(wᵀu), planar_layer.jl:68
}

extern "C" int b2b_planar_chain_hostparams_f32(const float* w_host, const float* u_host, const float* b_host,
                                               int32_t L, int inverse, const float* x, float* y, float* logjac,
                                               int32_t D, int64_t N, int64_t ldx, int64_t ldy,
                                               int accumulate_logjac, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  g_last_launches = 0;
  if (L < 1 || D < 1 || N < 0) return B2B_EINVAL;
  if (N == 0) return B2B_OK;
  if (!w_host || !u_host || !b_host || !x || (!y && !logjac) || ldx < D || (y && ldy < D)) return B2B_EINVAL;
  if (!(D == 32 || D == 64 || D == 128)) return B2B_EUNSUPPORTED;
  if (!y && L > 8) return B2B_EUNSUPPORTED;  // several launches need the D x N intermediate
  // launches take 1, 2, 4 or 8 layers: the tail is padded with identity layers (w = û = 0: y = x, logjac += 0),
  // which costs a little arithmetic but no extra pass over the batch
  std::vector<float> uh((size_t)L * D), c(L), packed;
  for (int l = 0; l < L; ++l) planar_derive_host(w_host + (size_t)l * D, u_host + (size_t)l * D, D, &uh[(size_t)l * D], &c[l]);
  B2BChainParams p;
  memset(&p, 0, sizeof(p));
  p.D = D;
  p.N = N;
  p.logjac = logjac;
  p.scratch_off = -1;
  int done = 0;
  while (done < L) {
    int n = 1;
    while (n < L - done && n < 8) n <<= 1;
    const int real = L - done < n ? L - done : n;
    packed.assign((size_t)2 * n * D + 2 * n, 0.f);  // w[n][D] | û[n][D] | c[n] | b[n]
    memcpy(&packed[0], w_host + (size_t)done * D, sizeof(float) * (size_t)real * D);
    memcpy(&packed[(size_t)n * D], &uh[(size_t)done * D], sizeof(float) * (size_t)real * D);
    memcpy(&packed[(size_t)2 * n * D], &c[done], sizeof(float) * real);
    memcpy(&packed[(size_t)2 * n * D + n], b_host + done, sizeof(float) * real);
    p.x = done == 0 ? x : y;
    p.ldx = done == 0 ? ldx : ldy;
    p.y = y;
    p.ldy = ldy;
    p.accumulate = (done == 0) ? (accumulate_logjac != 0) : 1;
    const int rc = b2b_launch_planar_hostparams(p, n, packed.data(), inverse ? (1 << n) - 1 : 0, stream);
    if (rc != B2B_OK) return rc;
    ++g_last_launches;
    done += n;
  }
  return B2B_OK;
}

// ---- reverse mode of forward planar chains ----------------------------------------------------------------
extern "C" size_t b2b_planar_chain_vjp_workspace_bytes(int32_t L, int32_t D, int64_t N) {
  if (L < 1 || L > 8 || D < 1 || N < 0) return 0;
  return b2b_planar_vjp_workspace(L, D, N);
}

extern "C" int b2b_planar_chain_vjp_f32(const b2b_layer_desc* layers, int32_t L, const float* x, const float* ybar,
                                        const float* ljbar, float* xbar, float* wbar, float* ubar, float* bbar,
                                        int32_t D, int64_t N, int64_t ldx, int64_t ldybar, int64_t ldxbar,
                                        void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  g_last_launches = 0;
  if (!layers || L < 1 || D < 1 || N < 0) return B2B_EINVAL;
  if (L > 8) return B2B_EUNSUPPORTED;
  const bool want_params = wbar || ubar || bbar;
  if (want_params && !(wbar && ubar && bbar)) return B2B_EINVAL;
  if (N == 0) {
    if (want_params) {
      cudaMemsetAsync(wbar, 0, sizeof(float) * (size_t)L * D, stream);
      cudaMemsetAsync(ubar, 0, sizeof(float) * (size_t)L * D, stream);
      return (int)cudaMemsetAsync(bbar, 0, sizeof(float) * L, stream);
    }
    return B2B_OK;
  }
  if (!x || !ybar || !xbar || ldx < D || ldybar < D || ldxbar < D) return B2B_EINVAL;
  for (int l = 0; l < L; ++l) {
    if (layers[l].kind != B2B_PLANAR) return B2B_EUNSUPPORTED;
    const int rc = validate_layer(layers[l], D, false);
    if (rc != B2B_OK) return rc;
    if ((layers[l].inverse != 0) != (layers[0].inverse != 0)) return B2B_EUNSUPPORTED;  // one direction per call
  }
  B2BChainParams p;
  memset(&p, 0, sizeof(p));
  p.x = x;
  p.N = N;
  p.ldx = ldx;
  p.D = D;
  p.L = L;
  for (int l = 0; l < L; ++l) p.layers[l] = layers[l];
  int launches = 0;
  const int rc = b2b_launch_planar_chain_vjp(p, ybar, ldybar, ljbar, xbar, ldxbar, wbar, ubar, bbar, workspace,
                                             workspace_bytes, &launches, stream);
  if (rc == B2B_OK) g_last_launches = launches;
  return rc;
}

extern "C" size_t b2b_radial_chain_vjp_workspace_bytes(int32_t L, int32_t D) {
  if (L < 1 || L > 8 || D < 1 || D > 128) return 0;
  return b2b_radial_vjp_workspace(L, D);
}

extern "C" int b2b_radial_chain_vjp_f32(const b2b_layer_desc* layers, int32_t L, const float* x, const float* ybar,
                                        const float* ljbar, float* xbar, float* alpha_bar, float* beta_bar,
                                        float* z0_bar, int32_t D, int64_t N, int64_t ldx, int64_t ldybar,
                                        int64_t ldxbar, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  g_last_launches = 0;
  if (!layers || L < 1 || D < 1 || N < 0 || !alpha_bar || !beta_bar || !z0_bar) return B2B_EINVAL;
  if (L > 8 || D > 128) return B2B_EUNSUPPORTED;
  if (N == 0) {
    cudaMemsetAsync(alpha_bar, 0, sizeof(float) * L, stream);
    cudaMemsetAsync(beta_bar, 0, sizeof(float) * L, stream);
    return (int)cudaMemsetAsync(z0_bar, 0, sizeof(float) * (size_t)L * D, stream);
  }
  if (!x || !ybar || !xbar || ldx < D || ldybar < D || ldxbar < D) return B2B_EINVAL;
  for (int l = 0; l < L; ++l) {
    if (layers[l].kind != B2B_RADIAL) return B2B_EUNSUPPORTED;
    const int rc = validate_layer(layers[l], D, false);
    if (rc != B2B_OK) return rc;
  }
  B2BChainParams p;
  memset(&p, 0, sizeof(p));
  p.x = x;
  p.N = N;
  p.ldx = ldx;
  p.D = D;
  p.L = L;
  for (int l = 0; l < L; ++l) p.layers[l] = layers[l];
  int launches = 0;
  const int rc = b2b_launch_radial_chain_vjp(p, ybar, ldybar, ljbar, xbar, ldxbar, alpha_bar, beta_bar, z0_bar,
                                             workspace, workspace_bytes, &launches, stream);
  if (rc == B2B_OK) g_last_launches = launches;
  return rc;
}
