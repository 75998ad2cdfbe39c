// C ABI of libb2b.so (include/b2b.h): argument validation, chain segmentation, launch bookkeeping.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <algorithm>
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
void b2b_set_last_launch_count(int n) { g_last_launches = n; }

int b2b_sm_count() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 132;
}

extern "C" int b2b_set_kernel_variant(int variant) {
  // low decimal digit: fused chain kernel variant; tens digit: coupling variant (10 = force fp32 CUDA cores)
  const int chain = variant % 10, cpl = (variant / 10) % 10, nofold = variant / 100;
  if (variant < 0 || chain > 3 || cpl > 1 || nofold > 1) return B2B_EINVAL;
  g_variant = chain;
  g_coupling_variant = cpl;
  g_fold_bn = nofold ? 0 : 1;
  return B2B_OK;
}

// one row of limits per kind of b2b_coupling
bool b2b_coupling_fits(const b2b_layer_desc& d, int D) {
  struct Limits { int kind, n, h_lo, h_hi, k_lo, k_hi, m_lo, m_hi, d; };
  static const Limits rows[] = {  // kind, n1 and n2, H, K, M, D
      {B2B_COUPLING_RQS, B2B_COUPLING_RQS_MAX_N, 0, 0, 2, B2B_COUPLING_RQS_MAX_K, 0, 0, B2B_COUPLING_RQS_MAX_D},
      {B2B_COUPLING_MLP, B2B_COUPLING_MLP_MAX_N, 1, B2B_COUPLING_MLP_MAX_H, 0, 0, 1, 1, B2B_COUPLING_MLP_MAX_D},
      {B2B_COUPLING_MLP_RQS, B2B_COUPLING_MLP_RQS_MAX_N, 1, B2B_COUPLING_MLP_RQS_MAX_H, 2, B2B_COUPLING_MLP_RQS_MAX_K,
       1, 1, B2B_COUPLING_MLP_RQS_MAX_D},
      {B2B_COUPLING_DEEP_MLP, B2B_COUPLING_DEEP_MLP_MAX_N, 1, B2B_COUPLING_DEEP_MLP_MAX_H, 0, 0,
       2, B2B_COUPLING_DEEP_MLP_MAX_DEPTH, B2B_COUPLING_DEEP_MLP_MAX_D},
      {B2B_COUPLING_DEEP_MLP_RQS, B2B_COUPLING_DEEP_MLP_RQS_MAX_N, 1, B2B_COUPLING_DEEP_MLP_RQS_MAX_H, 2,
       B2B_COUPLING_DEEP_MLP_RQS_MAX_K, 2, B2B_COUPLING_DEEP_MLP_RQS_MAX_DEPTH, B2B_COUPLING_DEEP_MLP_RQS_MAX_D},
  };
  const B2BCoupling<b2b_layer_desc> c = b2b_coupling(d);
  auto in = [](int v, int lo, int hi) { return v >= lo && v <= hi; };
  for (const Limits& r : rows)
    if (r.kind == d.kind)
      return in(c.n1, 1, r.n) && in(c.n2, 1, r.n) && in(c.H, r.h_lo, r.h_hi) && in(c.K, r.k_lo, r.k_hi) &&
             in(c.M, r.m_lo, r.m_hi) && D <= r.d;
  return false;
}

// Float32 envelope of a valid layer at D: B2B_EUNSUPPORTED when its forward kernel does not take it, else B2B_OK.  The
// fused kinds are also bound by their run's shared-memory budget, which plan_segments checks.
static int fwd_envelope(const b2b_layer_desc& d, int D) {
  bool ok = true;
  switch (d.kind) {
    case B2B_RQS: ok = d.n0 <= 64; break;
    case B2B_COUPLING_AFFINE: ok = b2b_coupling_affine_fits(d.n0, d.n1, D); break;
    case B2B_SCALE_MATRIX: ok = D <= B2B_SCALE_MATRIX_MAX_D; break;
    case B2B_SCALE_TRIANGULAR: ok = D <= B2B_SCALE_TRIANGULAR_MAX_D; break;
    case B2B_SCALE_LU: ok = D <= B2B_SCALE_LU_MAX_D; break;
    case B2B_MVNORMAL_TRIL: ok = D <= B2B_TRIL_MAX_D; break;
    case B2B_AUTOREGRESSIVE_MLP: ok = b2b_ar_fits(d, D); break;
    default: ok = !b2b_is_coupling(d.kind) || b2b_coupling_fits(d, D); break;  // the other couplings' table
  }
  return ok ? B2B_OK : B2B_EUNSUPPORTED;
}

// The same for the kernels of b2b_chain_vjp_f32.
static int vjp_envelope(const b2b_layer_desc& d, int D) {
  bool ok;
  switch (d.kind) {
    case B2B_PLANAR:
    case B2B_RADIAL: ok = D <= 128; break;
    case B2B_RQS: ok = D <= 256 && d.n0 <= 64; break;
    case B2B_COUPLING_AFFINE: ok = b2b_coupling_affine_vjp_fits(d, D); break;
    case B2B_BATCHNORM:
    case B2B_PERMUTE:
    case B2B_STACKED_EW:
    case B2B_ELEMENTWISE_VEC:
    case B2B_MVNORMAL_DIAG: ok = D <= 1024; break;  // BatchNorm and the elementwise-run kernel
    default: return fwd_envelope(d, D);
  }
  return ok ? B2B_OK : B2B_EUNSUPPORTED;
}

// The descriptor rules, then the envelope -- but a coupling's kernel limit and the terminal's D are refused only when
// the chain is planned, after the batch-sum and cotangent-slot checks of the entry points.
static int validate_layer(const b2b_layer_desc& d, int D, bool last) {
  const int rc = b2b_check_desc(d, D, last);
  if (rc != B2B_OK) return rc;
  const int launch = b2b_kind(d.kind)->launch;
  return launch == B2B_LC_COUPLING || launch == B2B_LC_TRIL ? B2B_OK : fwd_envelope(d, D);
}

static int launch_fused(B2BChainParams& p, cudaStream_t stream) {
  int rc = B2B_EUNSUPPORTED;
  // segments made of <= 8 PlanarLayers: the fused planar chain kernel (variant 3 forces, 1 / 2 disable)
  if (g_variant == 0 || g_variant == 3) {
    rc = b2b_launch_planar_chain_const(p, stream);
    if (rc == B2B_OK) return rc;
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

// A run of fused column-local layers: one launch of the kernel launch_fused picks (with a batch sum, a second adding its
// per-CTA partials)
static int fwd_fused(const B2BFwdSeg& s) {
  B2BChainParams p;
  memset(&p, 0, sizeof(p));
  p.x = s.x;
  p.y = s.y;
  p.logjac = s.logjac;
  p.N = s.N;
  p.ldx = s.ldx;
  p.ldy = s.ldy;
  p.D = s.D;
  p.L = s.n;
  p.accumulate = s.accumulate;
  for (int l = 0; l < p.L; ++l) p.layers[l] = s.layers[l];
  int grid = 0;
  if (s.partials) {
    grid = fused_grid(p);
    if (grid <= 0 || grid > 4096) return B2B_EUNSUPPORTED;
    p.partials = s.partials;
  }
  int rc = launch_fused(p, s.stream);
  if (rc != B2B_OK) return rc;
  ++*s.launches;
  if (!s.partials) return B2B_OK;
  if ((rc = b2b_launch_sum_partials(s.partials, grid, s.sum_out, s.stream)) != B2B_OK) return rc;
  ++*s.launches;
  return B2B_OK;
}

// An affine coupling, with the BatchNorm neighbours folded into it: the fold table's preparation, then the tensor-core
// kernel when the layer and the workspace fit it (and b2b_set_kernel_variant does not rule it out), else the exact-fp32
// kernel
static int fwd_coupling(const B2BFwdSeg& s) {
  const b2b_layer_desc& d = s.layers[0];
  const float* fold = nullptr;
  int rc;
  if (s.pre || s.post) {
    if ((rc = b2b_launch_bn_fold_prep(s.pre, s.post, s.D, s.fold, s.stream)) != B2B_OK) return rc;
    ++*s.launches;
    fold = s.fold;
  }
  rc = B2B_EUNSUPPORTED;
  if (s.workspace && g_coupling_variant != 1) {
    int n = 0;  // W preparation + main kernel (+ fp32 kernel on a ragged tail)
    rc = b2b_launch_coupling_affine_tc(d, fold, s.x, s.y, s.logjac, s.D, s.N, s.ldx, s.ldy, s.accumulate, s.workspace,
                                       s.workspace_bytes, &n, s.stream);
    if (rc == B2B_OK) *s.launches += n;
  }
  if (rc == B2B_EUNSUPPORTED) {
    rc = b2b_launch_coupling_affine(d, fold, s.x, s.y, s.logjac, s.D, s.N, s.ldx, s.ldy, s.accumulate, s.stream);
    if (rc == B2B_OK) ++*s.launches;
  }
  return rc;
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

// A launch of the chain: a run of fused layers, or one layer of another launch class (a coupling with the BatchNorm
// neighbours folded into it).
struct Seg {
  int begin, end;
  int launch;     // B2BLaunchClass
  int pre, post;  // layer index of a BatchNorm folded into this coupling launch (-1: none)
};

// Cuts the chain into launches before anything is enqueued: single layers of their own launch class, and maximal runs of
// fused layers whose staged parameters fit one fused kernel (a run is ended before the layer that would cross the
// shared-memory budget, so the terminal MvNormal stays in the last segment).  B2B_EUNSUPPORTED when one layer alone does
// not fit, B2B_EINVAL for a kind include/b2b.h does not define.
static int plan_segments(const b2b_layer_desc* layers, int32_t L, int32_t D, std::vector<Seg>& segs) {
  segs.clear();
  auto launch = [&](int l) {
    const B2BKind* k = b2b_kind(layers[l].kind);
    return k ? k->launch : -1;
  };
  for (int l = 0; l < L;) {
    if (launch(l) < 0) return B2B_EINVAL;
    if (launch(l) != B2B_LC_FUSED) {
      if (fwd_envelope(layers[l], D) != B2B_OK) return B2B_EUNSUPPORTED;
      segs.push_back({l, l + 1, launch(l), -1, -1});
      ++l;
      continue;
    }
    int e = l;
    while (e < L && launch(e) == B2B_LC_FUSED) ++e;
    for (int b = l; b < e;) {
      if (b2b_chain_v0_smem_bytes(layers + b, 1, D) > B2B_V0_SMEM_MAX) return B2B_EUNSUPPORTED;
      int k = b + 1;
      while (k < e && b2b_chain_v0_smem_bytes(layers + b, k + 1 - b, D) <= B2B_V0_SMEM_MAX) ++k;
      segs.push_back({b, k, B2B_LC_FUSED, -1, -1});
      b = k;
    }
    l = e;
  }
  return B2B_OK;
}

int b2b_chain_segment_count(const b2b_layer_desc* layers, int32_t L, int32_t D) {
  std::vector<Seg> segs;
  const int rc = plan_segments(layers, L, D, segs);
  return rc != B2B_OK ? rc : (int)segs.size();
}

int b2b_chain_check_f32(const b2b_layer_desc* layers, int32_t L, int32_t D) {
  for (int l = 0; l < L; ++l) {
    const int rc = validate_layer(layers[l], D, l == L - 1);
    if (rc != B2B_OK) return rc;
  }
  const int n = b2b_chain_segment_count(layers, L, D);
  return n < 0 ? n : B2B_OK;
}

// A batch sum without `logjac` over a terminal-ended chain of several launches: the launches before the last hand their
// log-Jacobians to it through N floats of workspace (`nsegs`: the plan's launch count before BatchNorm folding, which
// never changes whether a terminal-ended chain has more than one)
static bool sum_needs_logjac_ws(const b2b_layer_desc* layers, int32_t L, int nsegs) {
  return layers && L >= 1 && b2b_ends_in_terminal(layers, L) && nsegs > 1;
}

// factor storage of the dense, triangular and LU Scale layers and masked weights of the autoregressive layers (one
// region of the largest: they run one after another); 0 for a chain without one
static size_t chain_scale_bytes(const b2b_layer_desc* layers, int32_t L, int D) {
  size_t bytes = 0;
  for (int l = 0; layers && l < L; ++l) {
    const B2BKind* k = b2b_kind(layers[l].kind);
    if (k && (k->launch == B2B_LC_SCALE || k->launch == B2B_LC_AR)) {
      const size_t b = k->launch == B2B_LC_AR ? b2b_ar_workspace(layers[l], D) : b2b_scale_workspace(layers[l].kind, D);
      if (b > bytes) bytes = b;
    }
  }
  return bytes;
}

extern "C" size_t b2b_chain_workspace_bytes(const b2b_layer_desc* layers, int32_t L, int32_t D, int64_t N,
                                            int want_y, int want_sum) {
  // 0 for a layer past the envelopes include/b2b.h states (the call refuses the chain); a coupling past its kernel's
  // limit, or a descriptor the call finds invalid, is still sized
  for (int l = 0; layers && l < L; ++l) {
    const B2BKind* k = b2b_kind(layers[l].kind);
    if (k && (k->launch == B2B_LC_SPLINE || k->launch == B2B_LC_SCALE || k->launch == B2B_LC_MLP || k->launch == B2B_LC_AR ||
              (k->launch == B2B_LC_TRIL && l == L - 1)) &&
        fwd_envelope(layers[l], D) != B2B_OK)
      return 0;
  }
  size_t bytes = chain_scale_bytes(layers, L, D) + chain_tc_bytes(layers, L, D);
  // a D x N scratch matrix is needed only when y == NULL but the chain has more than one segment
  if (!want_y && b2b_chain_segment_count(layers, L, D) > 1)
    bytes += align_up((size_t)D * (size_t)N * sizeof(float), 1024);
  if (want_sum) bytes += 4096 * sizeof(double);
  if (want_sum && sum_needs_logjac_ws(layers, L, b2b_chain_segment_count(layers, L, D)))
    bytes += align_up((size_t)N * sizeof(float), 1024);
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
  if (sum_out && !logjac && !b2b_ends_in_terminal(layers, L)) return B2B_EINVAL;

  std::vector<Seg> segs;
  {
    const int rc = plan_segments(layers, L, D, segs);
    if (rc != B2B_OK) return rc;
  }
  const bool lj_ws = sum_out && !logjac && sum_needs_logjac_ws(layers, L, (int)segs.size());
  // workspace carve-up
  char* ws = static_cast<char*>(workspace);
  size_t ws_left = workspace ? workspace_bytes : 0;
  void* scale_ws = nullptr;
  const size_t scale_bytes = chain_scale_bytes(layers, L, D);
  if (scale_bytes) {
    if (ws_left < scale_bytes) return B2B_EWORKSPACE;
    scale_ws = ws;
    ws += scale_bytes;
    ws_left -= scale_bytes;
  }
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
  // fold BatchNorm neighbours (a per-row affine) into the coupling launches: removes their own pass over HBM.  With a
  // batch sum, the chain's last fused launch is never emptied: the sum comes from it.
  if (fold_ws && g_fold_bn) {
    for (size_t s = 0; s < segs.size(); ++s) {
      if (segs[s].launch != B2B_LC_COUPLING) continue;
      const bool keeps_sum = sum_out && s + 2 == segs.size() && segs[s + 1].end - segs[s + 1].begin == 1;
      if (s + 1 < segs.size() && segs[s + 1].launch != B2B_LC_COUPLING && segs[s + 1].end > segs[s + 1].begin &&
          layers[segs[s + 1].begin].kind == B2B_BATCHNORM && !keeps_sum)
        segs[s].post = segs[s + 1].begin++;
      if (s > 0 && segs[s - 1].launch != B2B_LC_COUPLING && segs[s - 1].end > segs[s - 1].begin &&
          layers[segs[s - 1].end - 1].kind == B2B_BATCHNORM)
        segs[s].pre = --segs[s - 1].end;
    }
    std::vector<Seg> kept;
    for (const Seg& g : segs)
      if (g.end > g.begin) kept.push_back(g);
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
  if (lj_ws) {
    // the launches before the last hand their log-Jacobians to it through N floats of workspace
    const size_t need = align_up((size_t)N * sizeof(float), 1024);
    if (ws_left < need) return B2B_EWORKSPACE;
    logjac = reinterpret_cast<float*>(ws);
    ws += need;
    ws_left -= need;
  }
  double* partials = nullptr;
  if (sum_out) {
    if (segs.back().launch != B2B_LC_FUSED && segs.back().launch != B2B_LC_TRIL)
      return B2B_EUNSUPPORTED;  // the batch sum comes from a fused or the terminal's launch
    if (ws_left < 4096 * sizeof(double)) return B2B_EWORKSPACE;
    partials = reinterpret_cast<double*>(ws);
  }

  const float* cur = x;
  long long cur_ld = ldx;
  // accumulate_logjac adds onto the caller's logjac; the workspace slice is written by the first launch
  bool lj_started = accumulate_logjac != 0 && !lj_ws;
  for (size_t s = 0; s < segs.size(); ++s) {
    const Seg& g = segs[s];
    const bool last_seg = s + 1 == segs.size();
    // destination of this segment: y when given, else scratch for intermediates, nothing for the last
    float* dst = y ? y : (last_seg ? nullptr : scratch);
    const long long dst_ld = y ? ldy : D;
    // the classes with a workspace slice
    const bool cpl = g.launch == B2B_LC_COUPLING, sc = g.launch == B2B_LC_SCALE || g.launch == B2B_LC_AR;
    const B2BFwdSeg a{layers + g.begin, g.end - g.begin, cur, cur_ld, dst, dst_ld, logjac, lj_started ? 1 : 0, D, N,
                      g.pre >= 0 ? &layers[g.pre] : nullptr, g.post >= 0 ? &layers[g.post] : nullptr, fold_ws,
                      last_seg ? partials : nullptr, sum_out, cpl ? tc_ws : sc ? scale_ws : nullptr,
                      cpl ? tc_bytes : sc ? scale_bytes : 0, &g_last_launches, stream};
    int rc;
    switch (g.launch) {
      case B2B_LC_COUPLING: rc = fwd_coupling(a); break;
      case B2B_LC_SPLINE: rc = b2b_fwd_spline(a); break;
      case B2B_LC_MLP: rc = b2b_fwd_mlp(a); break;
      case B2B_LC_SCALE: rc = b2b_fwd_scale(a); break;
      case B2B_LC_TRIL: rc = b2b_fwd_tril(a); break;  // always the last segment
      case B2B_LC_AR: rc = b2b_fwd_ar(a); break;
      default: rc = fwd_fused(a); break;
    }
    if (rc != B2B_OK) return rc;
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
  float* const bars[4 * 8] = {wbar, ubar, bbar};
  int launches = 0;
  const int rc = b2b_vjp_planar({layers, L, x, ldx, ybar, ldybar, ljbar, xbar, ldxbar, D, N, bars, nullptr, workspace,
                                 workspace_bytes, &launches, stream});
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
  float* const bars[4 * 8] = {alpha_bar, beta_bar, z0_bar};
  int launches = 0;
  const int rc = b2b_vjp_radial({layers, L, x, ldx, ybar, ldybar, ljbar, xbar, ldxbar, D, N, bars, nullptr, workspace,
                                 workspace_bytes, &launches, stream});
  if (rc == B2B_OK) g_last_launches = launches;
  return rc;
}

// ---- reverse mode of any chain ------------------------------------------------------------------------------------------
// The chain is cut into VJP segments, each differentiated by an existing per-kind kernel or by the elementwise-run kernel:
// planar runs of one direction (<= 8), radial runs (<= 8, mixed directions), single RQS / coupling / eval-BatchNorm layers,
// and runs of <= 8 STACKED_EW / ELEMENTWISE_VEC / PERMUTE layers optionally closed by the terminal MVNORMAL_DIAG.  The forward is recomputed
// once, segment by segment, storing each segment's input (at ld = D); then the segments are differentiated last to first,
// the cotangent moving between two D x N buffers.  Every segment sees the same l̄ (the log-Jacobians add up).
namespace {

struct VSeg {
  int kind, begin, end;
  int Dk;  // rows the segment's kernel runs at: planar runs at D not in {32, 64, 128} are embedded in the next of them
};

size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }
size_t mat_bytes(int D, long long N) { return al256((size_t)D * (size_t)N * sizeof(float)); }

int vjp_segments(const b2b_layer_desc* layers, int L, int D, std::vector<VSeg>& segs) {  // valid descriptors
  segs.clear();
  for (int l = 0; l < L;) {
    if (vjp_envelope(layers[l], D) != B2B_OK) return B2B_EUNSUPPORTED;
    VSeg s{b2b_kind(layers[l].kind)->vjp, l, l + 1, D};
    int& e = s.end;
    if (s.kind == B2B_VC_PLANAR) {
      while (e < L && e - l < 8 && layers[e].kind == B2B_PLANAR && (layers[e].inverse != 0) == (layers[l].inverse != 0)) ++e;
      s.Dk = D <= 32 ? 32 : D <= 64 ? 64 : 128;
    } else if (s.kind == B2B_VC_RADIAL) {
      while (e < L && e - l < 8 && layers[e].kind == B2B_RADIAL) ++e;
    } else if (s.kind == B2B_VC_EW) {  // PERMUTE / STACKED_EW / ELEMENTWISE_VEC layers and the terminal MVNORMAL_DIAG after
      e = l;                           // them, or alone
      while (e < L && e - l < 8 && layers[e].kind != B2B_MVNORMAL_DIAG && b2b_kind(layers[e].kind)->vjp == B2B_VC_EW) ++e;
      if (e < L && layers[e].kind == B2B_MVNORMAL_DIAG) ++e;
    }
    segs.push_back(s);
    l = e;
  }
  // the forward recompute runs every segment but the last through b2b_chain_run_f32: it must accept them, so that the
  // workspace query and the call refuse the same chains, before anything is launched
  std::vector<Seg> fwd;
  for (size_t k = 0; k + 1 < segs.size(); ++k) {
    const int rc = plan_segments(layers + segs[k].begin, segs[k].end - segs[k].begin, D, fwd);
    if (rc != B2B_OK) return rc;
  }
  return B2B_OK;
}

// floats of parameter-cotangent scratch (each array rounded up to 64 floats) and bytes of kernel workspace of a segment
size_t seg_param_floats(const b2b_layer_desc* layers, const VSeg& s, int D) {
  const size_t n = (size_t)(s.end - s.begin);
  auto r = [](size_t f) { return (f + 63) & ~(size_t)63; };
  const b2b_layer_desc& d = layers[s.begin];
  switch (s.kind) {
    case B2B_VC_PLANAR: return 4 * r(n * s.Dk) + r(n);  // w̄, ū, b̄ as the kernel writes them (+ padded w, u)
    case B2B_VC_RADIAL: return 2 * r(n) + r(n * D);
    case B2B_VC_RQS: return 3 * r((size_t)D * d.n0);
    case B2B_VC_COUPLING: return r((size_t)2 * d.n0 * d.n1) + r((size_t)2 * d.n0);
    case B2B_VC_BN: return 2 * r(D);
    case B2B_VC_SPLINE: return r(b2b_slot_len(d, 0, D)) + r(b2b_slot_len(d, 1, D));  // W̄ / c̄ sent to scratch
    default: return 0;
  }
}

size_t seg_kernel_bytes(const b2b_layer_desc* layers, const VSeg& s, int D, long long N) {
  const int n = s.end - s.begin;
  const b2b_layer_desc& d = layers[s.begin];
  switch (s.kind) {
    case B2B_VC_PLANAR: return b2b_planar_vjp_workspace(n, s.Dk, N);
    case B2B_VC_RADIAL: return b2b_radial_vjp_workspace(n, D);
    case B2B_VC_RQS: return b2b_rqs_vjp_workspace_bytes(d.n0, D);
    case B2B_VC_COUPLING: return b2b_coupling_affine_vjp_workspace_bytes(d.n0, d.n1);
    case B2B_VC_BN: return b2b_batchnorm_eval_vjp_workspace_bytes(D);
    case B2B_VC_TRIL: return b2b_tril_vjp_workspace(D, N);
    case B2B_VC_SPLINE: return b2b_coupling_rqs_vjp_workspace(d, D, N);
    case B2B_VC_MLP: return b2b_coupling_mlp_vjp_workspace(d, D, N);
    case B2B_VC_SCALE: return b2b_scale_vjp_workspace(d.kind, D, N);  // also holds the factor of the forward recompute
    case B2B_VC_AR: return b2b_ar_vjp_workspace(d, D, N);  // also holds the masked weights of the forward recompute
    default: {
      int vec = 0;
      for (int l = s.begin; l < s.end; ++l) vec += layers[l].kind == B2B_ELEMENTWISE_VEC;
      return b2b_ew_vjp_workspace(D, layers[s.end - 1].kind == B2B_MVNORMAL_DIAG, vec);
    }
  }
}

// workspace: [checkpoints of segments 1..S-1][2 cotangent buffers][staged x][3 padded planar buffers][parameter scratch]
//            [kernel workspace], each 256-aligned, + 256 of alignment slack
struct VLayout {
  size_t ckpt, ncot, stage, pad, param, kern, total;
  int Dk_pad;  // rows of the padded planar buffers (0: none)
};

VLayout vjp_layout(const b2b_layer_desc* layers, const std::vector<VSeg>& segs, int D, long long N) {
  VLayout v{};
  const size_t S = segs.size(), m = mat_bytes(D, N);
  v.ckpt = (S - 1) * m;
  v.ncot = (S == 1 && (segs[0].kind == B2B_VC_EW || segs[0].kind == B2B_VC_TRIL)) ? 0 : 2;
  // the planar kernels read x through TMA: an x they cannot read is copied (into a free checkpoint when there is one)
  v.stage = (S == 1 && segs[0].kind == B2B_VC_PLANAR && segs[0].Dk == D) ? m : 0;
  size_t pf = 0;
  for (const VSeg& s : segs) {
    if (s.kind == B2B_VC_PLANAR && s.Dk != D) v.Dk_pad = s.Dk;
    pf = std::max(pf, seg_param_floats(layers, s, D));
    v.kern = std::max(v.kern, al256(seg_kernel_bytes(layers, s, D, N)));
  }
  v.pad = v.Dk_pad ? 3 * mat_bytes(v.Dk_pad, N) : 0;
  v.param = al256(pf * sizeof(float));
  v.total = v.ckpt + v.ncot * m + v.stage + v.pad + v.param + v.kern + 256;
  return v;
}

bool tma_ok(const float* p, long long ld) { return p && (reinterpret_cast<uintptr_t>(p) & 15) == 0 && ld % 4 == 0; }

// the classes whose kernels read ȳ: a NULL ȳ is staged as zeros for them (the others take NULL as zero)
bool vjp_needs_ybar(int vc) {
  return vc == B2B_VC_RADIAL || vc == B2B_VC_RQS || vc == B2B_VC_COUPLING || vc == B2B_VC_BN;
}

// ȳ := zeros (ȳ == NULL) or a copy of ȳ at ld = D, in `buf`
int stage_ybar(B2BVjpSeg& a, float* buf) {
  const size_t F = sizeof(float);
  const cudaError_t e =
      a.ybar ? cudaMemcpy2DAsync(buf, (size_t)a.D * F, a.ybar, (size_t)a.ldyb * F, (size_t)a.D * F, a.N, cudaMemcpyDeviceToDevice, a.stream)
             : cudaMemsetAsync(buf, 0, (size_t)a.D * a.N * F, a.stream);
  if (e != cudaSuccess) return (int)e;
  ++*a.launches;
  a.ybar = buf;
  a.ldyb = a.D;
  return B2B_OK;
}

// A planar run: its kernels read x and ȳ and write x̄ through TMA, at D in {32, 64, 128}.  At another D the run is
// embedded in the next of them, Dk rows (pad[0..2]; w and u padded with zeros in scratch, after the kernel's w̄, ū, b̄
// arrays).  Otherwise an operand TMA cannot address is staged: x into `xst`, ȳ into `yst`, x̄ through `xbst`.
int vjp_planar_run(B2BVjpSeg a, int Dk, float* const pad[3], float* xst, float* yst, float* xbst) {
  const int n = a.n, D = a.D;
  const long long N = a.N;
  const size_t F = sizeof(float);
  const b2b_layer_desc* const layers = a.layers;
  float* const* const bars = a.bars;
  float* const scratch = a.scratch;
  float* const xbar = a.xbar;
  const long long ldxb = a.ldxb;
  cudaError_t e;
  int rc;
#define B2B_VJP_CUDA(call)                          \
  do {                                              \
    if ((e = (call)) != cudaSuccess) return (int)e; \
    ++*a.launches;                                  \
  } while (0)
  const size_t r64 = ((size_t)n * Dk + 63) & ~(size_t)63;
  b2b_layer_desc lp[8];
  float* kbars[4 * 8] = {};
  if (Dk != D) {
    // w, u padded with zeros give the same map on the first D rows (wᵀz, wᵀu, ‖w‖² and those rows of û are unchanged)
    // and leave the zero rows of x at zero.  The kernel writes its w̄, ū, b̄ arrays at Dk; the requested rows go out below.
    float* wp = scratch + 2 * r64 + 64;
    float* up = wp + r64;
    const float* src[16];
    float* dst[16];
    int len[16], dlen[16];
    for (int j = 0; j < n; ++j) {
      lp[j] = a.layers[j];
      src[2 * j] = a.layers[j].p0;
      dst[2 * j] = wp + (size_t)j * Dk;
      src[2 * j + 1] = a.layers[j].p1;
      dst[2 * j + 1] = up + (size_t)j * Dk;
      len[2 * j] = len[2 * j + 1] = D;
      dlen[2 * j] = dlen[2 * j + 1] = Dk;
      lp[j].p0 = dst[2 * j];
      lp[j].p1 = dst[2 * j + 1];
    }
    if ((rc = b2b_launch_copy_list(2 * n, src, dst, len, dlen, a.stream)) != B2B_OK) return rc;
    ++*a.launches;
    const size_t pitch = (size_t)Dk * F, zrows = (size_t)(Dk - D) * F;
    B2B_VJP_CUDA(cudaMemcpy2DAsync(pad[0], pitch, a.x, (size_t)a.ldx * F, (size_t)D * F, N, cudaMemcpyDeviceToDevice, a.stream));
    B2B_VJP_CUDA(cudaMemset2DAsync(pad[0] + D, pitch, 0, zrows, N, a.stream));
    if (a.ybar) {
      B2B_VJP_CUDA(cudaMemcpy2DAsync(pad[1], pitch, a.ybar, (size_t)a.ldyb * F, (size_t)D * F, N, cudaMemcpyDeviceToDevice, a.stream));
      B2B_VJP_CUDA(cudaMemset2DAsync(pad[1] + D, pitch, 0, zrows, N, a.stream));
    } else {
      B2B_VJP_CUDA(cudaMemsetAsync(pad[1], 0, (size_t)Dk * N * F, a.stream));
    }
    for (int k = 0; k < 4 * n; ++k)
      if (bars[k]) {
        kbars[0] = scratch;
        kbars[1] = scratch + r64;
        kbars[2] = scratch + 2 * r64;
      }
    a.layers = lp;
    a.x = pad[0];
    a.ybar = pad[1];
    a.xbar = pad[2];
    a.ldx = a.ldyb = a.ldxb = a.D = Dk;
    a.bars = kbars;
    a.scratch = nullptr;
  } else {
    if (!tma_ok(a.x, a.ldx)) {
      B2B_VJP_CUDA(cudaMemcpy2DAsync(xst, (size_t)D * F, a.x, (size_t)a.ldx * F, (size_t)D * F, N, cudaMemcpyDeviceToDevice, a.stream));
      a.x = xst;
      a.ldx = D;
    }
    if (!tma_ok(a.ybar, a.ldyb) && (rc = stage_ybar(a, yst)) != B2B_OK) return rc;
    if (!tma_ok(a.xbar, a.ldxb)) {
      a.xbar = xbst;
      a.ldxb = D;
    }
  }
  if ((rc = b2b_vjp_planar(a)) != B2B_OK) return rc;
  if (a.xbar != xbar)
    B2B_VJP_CUDA(cudaMemcpy2DAsync(xbar, (size_t)ldxb * F, a.xbar, (size_t)a.ldxb * F, (size_t)D * F, N, cudaMemcpyDeviceToDevice, a.stream));
#undef B2B_VJP_CUDA
  if (Dk == D) return B2B_OK;
  const float* const base[3] = {scratch, scratch + r64, scratch + 2 * r64};
  const size_t step[3] = {(size_t)Dk, (size_t)Dk, 1};
  return b2b_copy_run_bars(layers, n, bars, base, step, D, a.launches, a.stream);
}

}  // namespace

// The chain checks of the reverse mode that need no batch: descriptors, then segments.  b2b_chain_vjp_f32 makes the same
// checks with the slot requests between them, so that its status for a bad request keeps its precedence.
static int vjp_chain_check(const b2b_layer_desc* layers, int32_t L, int32_t D, std::vector<VSeg>& segs) {
  if (!layers || L < 1 || L > B2B_MAX_CHAIN || D < 1) return B2B_EINVAL;
  for (int l = 0; l < L; ++l) {
    const int rc = validate_layer(layers[l], D, l == L - 1);
    if (rc != B2B_OK) return rc;
  }
  return vjp_segments(layers, L, D, segs);
}

int b2b_chain_vjp_check_f32(const b2b_layer_desc* layers, int32_t L, int32_t D) {
  std::vector<VSeg> segs;
  return vjp_chain_check(layers, L, D, segs);
}

extern "C" size_t b2b_chain_vjp_workspace_bytes(const b2b_layer_desc* layers, int32_t L, int32_t D, int64_t N) {
  std::vector<VSeg> segs;
  if (N < 0 || vjp_chain_check(layers, L, D, segs) != B2B_OK) return 0;
  return vjp_layout(layers, segs, D, N).total;
}


extern "C" int b2b_chain_vjp_f32(const b2b_layer_desc* layers, int32_t L, const float* x, const float* ybar,
                                 const float* ljbar, float* xbar, float* const* param_bars, int32_t D, int64_t N,
                                 int64_t ldx, int64_t ldybar, int64_t ldxbar, void* workspace, size_t workspace_bytes,
                                 void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  g_last_launches = 0;
  if (!layers || L < 1 || L > B2B_MAX_CHAIN || D < 1 || N < 0) return B2B_EINVAL;
  for (int l = 0; l < L; ++l) {
    const int rc = validate_layer(layers[l], D, l == L - 1);
    if (rc != B2B_OK) return rc;
  }
  unsigned want;
  int rc = b2b_vjp_check_slots(layers, L, param_bars, &want);
  if (rc != B2B_OK) return rc;
  std::vector<VSeg> segs;
  if ((rc = vjp_segments(layers, L, D, segs)) != B2B_OK) return rc;
  rc = b2b_vjp_check_batch(layers, L, param_bars, x, ybar, xbar, D, N, ldx, ldybar, ldxbar, stream);
  if (rc != B2B_OK || N == 0) return rc;
  float* const none[4 * B2B_MAX_CHAIN] = {};
  float* const* bars = param_bars ? param_bars : none;
  int launches = 0;
  const VLayout lay = vjp_layout(layers, segs, D, N);
  if (!workspace || workspace_bytes < lay.total) return B2B_EWORKSPACE;
  const int S = (int)segs.size();
  const size_t m = mat_bytes(D, N);
  char* ws = b2b_align256(workspace);
  std::vector<float*> ckpt(S, nullptr);
  for (int s = 1; s < S; ++s) ckpt[s] = reinterpret_cast<float*>(ws + (size_t)(s - 1) * m);
  ws += lay.ckpt;
  float* G[2] = {nullptr, nullptr};
  for (size_t k = 0; k < lay.ncot; ++k) G[k] = reinterpret_cast<float*>(ws + k * m);
  ws += lay.ncot * m;
  float* stage = lay.stage ? reinterpret_cast<float*>(ws) : nullptr;
  ws += lay.stage;
  float* pad[3] = {nullptr, nullptr, nullptr};
  for (int k = 0; k < 3 && lay.Dk_pad; ++k) pad[k] = reinterpret_cast<float*>(ws + (size_t)k * mat_bytes(lay.Dk_pad, N));
  ws += lay.pad;
  float* scratch = reinterpret_cast<float*>(ws);
  ws += lay.param;
  void* kws = ws;
  const size_t kws_bytes = lay.kern;
  // 1. forward recompute: the input of every segment after the first (a Scale keeps its factor, an autoregressive layer
  // its masked weights in the kernel workspace, free until the reverse sweep)
  for (int s = 0; s + 1 < S; ++s) {
    const bool sc = segs[s].kind == B2B_VC_SCALE || segs[s].kind == B2B_VC_AR;
    rc = b2b_chain_run_f32(layers + segs[s].begin, segs[s].end - segs[s].begin, s == 0 ? x : ckpt[s], ckpt[s + 1],
                           nullptr, nullptr, D, N, s == 0 ? ldx : D, D, 0, sc ? kws : nullptr, sc ? kws_bytes : 0, stream);
    if (rc != B2B_OK) return rc;
    launches += g_last_launches;
  }
  // 2. reverse sweep: the cotangent moves between G[0] and G[1]; the one a segment does not write is free while it runs
  for (int s = S - 1; s >= 0; --s) {
    const VSeg& sg = segs[s];
    B2BVjpSeg a{layers + sg.begin, sg.end - sg.begin, s == 0 ? x : ckpt[s], s == 0 ? ldx : D,
                s == S - 1 ? ybar : G[(s + 1) & 1], s == S - 1 ? ldybar : D, ljbar, s == 0 ? xbar : G[s & 1],
                s == 0 ? ldxbar : D, D, N, bars + 4 * sg.begin, scratch, kws, kws_bytes, &launches, stream};
    float* const free_cot = G[(s + 1) & 1];
    if (!a.ybar && vjp_needs_ybar(sg.kind) && (rc = stage_ybar(a, free_cot)) != B2B_OK) return rc;
    switch (sg.kind) {  // segment 1's checkpoint is no longer needed when a planar run stages its x there
      case B2B_VC_PLANAR: rc = vjp_planar_run(a, sg.Dk, pad, S >= 2 ? ckpt[1] : stage, free_cot, G[s & 1]); break;
      case B2B_VC_RADIAL: rc = b2b_vjp_radial(a); break;
      case B2B_VC_RQS: rc = b2b_vjp_rqs(a); break;
      case B2B_VC_COUPLING: rc = b2b_vjp_coupling(a); break;
      case B2B_VC_BN: rc = b2b_vjp_batchnorm(a); break;
      case B2B_VC_EW: rc = b2b_vjp_ew(a); break;
      case B2B_VC_TRIL: rc = b2b_vjp_tril(a); break;
      case B2B_VC_SPLINE: rc = b2b_vjp_spline(a); break;
      case B2B_VC_SCALE: rc = b2b_vjp_scale(a); break;
      case B2B_VC_AR: rc = b2b_vjp_ar(a); break;
      default: rc = b2b_vjp_mlp(a); break;
    }
    if (rc != B2B_OK) return rc;
  }
  g_last_launches = launches;
  return B2B_OK;
}
