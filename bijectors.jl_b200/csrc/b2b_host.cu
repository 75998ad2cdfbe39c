// Host-buffer entry point (chunked H2D / compute / D2H pipeline) and the NCCL call site.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstdlib>
#include <cstring>
#include <vector>

#include "b2b_internal.h"

// ---------------------------------------------------------------------------------------------------
// b2b_host_ctx: per-stream device staging buffers, allocated ONCE (not on the hot path).
// ---------------------------------------------------------------------------------------------------
struct b2b_host_ctx {
  int D_max;
  long long chunk_cols;
  int n_streams;
  std::vector<cudaStream_t> streams;
  std::vector<float*> dx;      // D_max * chunk_cols floats each (y is produced in place)
  std::vector<float*> dlj;     // chunk_cols floats each
  std::vector<char*> dws;      // workspace for the batch-sum partials (ws_bytes each)
  size_t ws_bytes;
  std::vector<double*> dsum;   // one device double per stream
  double* hsum;                // pinned, one slot per chunk (grown on demand)
  long long hsum_cap;
};

static const size_t kWsBytes = 512 * 1024;  // batch-sum partials + tensor-core W image of a coupling layer

// A chain with a dense, triangular or LU Scale also needs its factor storage, and one with an autoregressive layer its
// masked weights, before the partials: the staging workspace grows to hold the larger of the dense Scale's and the
// widest autoregressive layer's at D_max, and only such chains are handed the larger size (every other chain sees
// kWsBytes, as before).
static size_t ctx_ws_bytes(int D_max) {
  const int d = D_max < B2B_SCALE_MATRIX_MAX_D ? D_max : B2B_SCALE_MATRIX_MAX_D;
  size_t scale = b2b_scale_workspace(B2B_SCALE_MATRIX, d);
  b2b_layer_desc ar{};
  ar.kind = B2B_AUTOREGRESSIVE_MLP;
  ar.n2 = B2B_AUTOREGRESSIVE_MLP_MAX_H;
  const size_t arb = b2b_ar_workspace(ar, D_max < B2B_AUTOREGRESSIVE_MLP_MAX_D ? D_max : B2B_AUTOREGRESSIVE_MLP_MAX_D);
  if (arb > scale) scale = arb;
  scale += 4096 * sizeof(double) + 1024;
  return scale > kWsBytes ? scale : kWsBytes;
}

extern "C" int b2b_host_ctx_create(b2b_host_ctx** out, int32_t D_max, int64_t chunk_cols, int32_t n_streams) {
  if (!out || D_max < 1 || chunk_cols < 1 || n_streams < 1 || n_streams > 16) return B2B_EINVAL;
  b2b_host_ctx* c = new b2b_host_ctx();
  c->D_max = D_max;
  c->chunk_cols = chunk_cols;
  c->n_streams = n_streams;
  c->hsum = nullptr;
  c->hsum_cap = 0;
  c->ws_bytes = ctx_ws_bytes(D_max);
  cudaError_t e = cudaSuccess;
  for (int s = 0; s < n_streams && e == cudaSuccess; ++s) {
    cudaStream_t st = nullptr;
    float *dx = nullptr, *dlj = nullptr;
    char* ws = nullptr;
    double* ds = nullptr;
    e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMalloc(&dx, (size_t)D_max * (size_t)chunk_cols * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&dlj, (size_t)chunk_cols * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&ws, c->ws_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&ds, sizeof(double));
    c->streams.push_back(st);
    c->dx.push_back(dx);
    c->dlj.push_back(dlj);
    c->dws.push_back(ws);
    c->dsum.push_back(ds);
  }
  if (e != cudaSuccess) {
    b2b_host_ctx_destroy(c);
    return (int)e;
  }
  *out = c;
  return B2B_OK;
}

// Orders the ctx's internal (non-blocking) streams after everything enqueued so far on `stream` -- e.g. an optimiser
// step on the caller's stream that has just rewritten the layer parameters the next b2b_chain_run_host_f32 will read.
extern "C" int b2b_host_ctx_wait_stream(b2b_host_ctx* c, void* stream) {
  if (!c) return B2B_EINVAL;
  cudaEvent_t ev;
  cudaError_t e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
  if (e != cudaSuccess) return (int)e;
  e = cudaEventRecord(ev, static_cast<cudaStream_t>(stream));
  for (size_t s = 0; s < c->streams.size() && e == cudaSuccess; ++s) e = cudaStreamWaitEvent(c->streams[s], ev, 0);
  cudaEventDestroy(ev);
  return (int)e;
}

extern "C" int b2b_host_ctx_destroy(b2b_host_ctx* c) {
  if (!c) return B2B_OK;
  for (size_t s = 0; s < c->streams.size(); ++s) {
    if (c->streams[s]) cudaStreamSynchronize(c->streams[s]);
    if (c->dx[s]) cudaFree(c->dx[s]);
    if (c->dlj[s]) cudaFree(c->dlj[s]);
    if (c->dws[s]) cudaFree(c->dws[s]);
    if (c->dsum[s]) cudaFree(c->dsum[s]);
    if (c->streams[s]) cudaStreamDestroy(c->streams[s]);
  }
  if (c->hsum) cudaFreeHost(c->hsum);
  delete c;
  return B2B_OK;
}

// ---------------------------------------------------------------------------------------------------
// NUMA placement of the calling thread next to a GPU.  On the 2-socket HGX hosts every GPU hangs off one socket's PCIe
// root complexes; a pinned host buffer that lives on the OTHER socket makes every H2D / D2H copy cross the inter-socket
// link, which caps the host-buffer throughput when several ranks share a box.  This binds the
// calling thread (CPU affinity + preferred memory node) to the NUMA node of `device`, so that pinned buffers allocated
// afterwards (cudaHostAlloc / torch pin_memory from this thread) and the host ctx's staging land on the local node.
// Linux only; every step is best effort (returns B2B_OK with *node_out = -1 when the topology is not exposed).
// ---------------------------------------------------------------------------------------------------
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <cctype>
#include <cstdio>

static int read_small_file(const char* path, char* buf, size_t cap) {
  FILE* f = fopen(path, "r");
  if (!f) return -1;
  const size_t n = fread(buf, 1, cap - 1, f);
  fclose(f);
  buf[n] = 0;
  return (int)n;
}

extern "C" int b2b_device_numa_node(int32_t device, int32_t* node_out) {
  if (!node_out) return B2B_EINVAL;
  *node_out = -1;
  char bus[64] = {0};
  cudaError_t e = cudaDeviceGetPCIBusId(bus, sizeof(bus), device);
  if (e != cudaSuccess) return (int)e;
  for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
  char path[256], buf[64];
  snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
  if (read_small_file(path, buf, sizeof(buf)) <= 0) return B2B_OK;
  *node_out = atoi(buf);
  return B2B_OK;
}

extern "C" int b2b_numa_bind_to_device(int32_t device, int32_t* node_out, int32_t* ncpus_out) {
  if (node_out) *node_out = -1;
  if (ncpus_out) *ncpus_out = 0;
  int32_t node = -1;
  const int rc = b2b_device_numa_node(device, &node);
  if (rc != B2B_OK) return rc;
  if (node < 0) return B2B_OK;
  char path[256], buf[4096];
  snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
  if (read_small_file(path, buf, sizeof(buf)) <= 0) return B2B_OK;
  // cpulist: "0-31,64-95"
  cpu_set_t set;
  CPU_ZERO(&set);
  int ncpu = 0;
  for (char* p = buf; *p;) {
    while (*p && !isdigit((unsigned char)*p)) ++p;
    if (!*p) break;
    long a = strtol(p, &p, 10), b = a;
    if (*p == '-') b = strtol(p + 1, &p, 10);
    for (long c = a; c <= b && c < CPU_SETSIZE; ++c) {
      CPU_SET((int)c, &set);
      ++ncpu;
    }
  }
  if (ncpu == 0) return B2B_OK;
  // intersect with what the process may use (cgroup / taskset); keep the old mask when the intersection is empty
  cpu_set_t cur, both;
  if (sched_getaffinity(0, sizeof(cur), &cur) == 0) {
    CPU_AND(&both, &set, &cur);
    if (CPU_COUNT(&both) > 0) set = both;
  }
  if (sched_setaffinity(0, sizeof(set), &set) != 0) return B2B_OK;
  // set_mempolicy(MPOL_PREFERRED, {node}): allocations of this thread come from the local node when it has room
  // (needs no privilege for the calling thread; ignored when the kernel / sandbox refuses)
  unsigned long mask[16] = {0};
  if (node < (int)(sizeof(mask) * 8)) {
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    (void)syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, sizeof(mask) * 8);
  }
  if (node_out) *node_out = node;
  if (ncpus_out) *ncpus_out = CPU_COUNT(&set);
  return B2B_OK;
}

extern "C" int b2b_host_register(void* ptr, size_t bytes) {
  return (int)cudaHostRegister(ptr, bytes, cudaHostRegisterDefault);
}
extern "C" int b2b_host_unregister(void* ptr) { return (int)cudaHostUnregister(ptr); }

extern "C" int b2b_chain_run_host_f32(b2b_host_ctx* c, const b2b_layer_desc* layers, int32_t L,
                                      const float* x_host, float* y_host, float* logjac_host,
                                      double* sum_host, int32_t D, int64_t N) {
  if (!c || !layers || !x_host || D < 1 || D > c->D_max || N < 0) return B2B_EINVAL;
  if (!y_host && !logjac_host && !sum_host) return B2B_EINVAL;
  const long long chunk = c->chunk_cols;
  const long long nchunks = (N + chunk - 1) / chunk;
  if (sum_host && nchunks > c->hsum_cap) {
    if (c->hsum) cudaFreeHost(c->hsum);
    c->hsum = nullptr;
    cudaError_t e = cudaMallocHost(&c->hsum, (size_t)nchunks * sizeof(double));
    if (e != cudaSuccess) return (int)e;
    c->hsum_cap = nchunks;
  }
  int launches = 0;
  // a logjac-only call still needs the D x N intermediate when the chain runs as several launches (a coupling layer, or
  // a run of layers split at the fused kernels' shared-memory budget): the staging buffer doubles as that scratch
  const int nseg = b2b_chain_segment_count(layers, L, D);
  if (nseg < 0) return nseg;
  const bool stage_y = y_host != nullptr || nseg > 1;
  const size_t ws_bytes =
      b2b_chain_has_launch(layers, L, B2B_LC_SCALE) || b2b_chain_has_launch(layers, L, B2B_LC_AR) ? c->ws_bytes : kWsBytes;
  for (long long k = 0; k < nchunks; ++k) {
    const int s = (int)(k % c->n_streams);
    cudaStream_t st = c->streams[s];
    const long long c0 = k * chunk;
    const long long n = (N - c0 < chunk) ? (N - c0) : chunk;
    cudaError_t e = cudaMemcpyAsync(c->dx[s], x_host + (size_t)c0 * D, (size_t)n * D * sizeof(float),
                                    cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return (int)e;
    const bool terminal = b2b_ends_in_terminal(layers, L);
    const bool want_lj = logjac_host != nullptr || (sum_host && !terminal);
    const int rc = b2b_chain_run_f32(layers, L, c->dx[s], stage_y ? c->dx[s] : nullptr,  // in place
                                     (want_lj || terminal) ? c->dlj[s] : nullptr,
                                     sum_host ? c->dsum[s] : nullptr, D, n, D, D, 0, c->dws[s], ws_bytes, st);
    if (rc != B2B_OK) return rc;
    launches += b2b_last_launch_count();
    if (y_host) {
      e = cudaMemcpyAsync(y_host + (size_t)c0 * D, c->dx[s], (size_t)n * D * sizeof(float),
                          cudaMemcpyDeviceToHost, st);
      if (e != cudaSuccess) return (int)e;
    }
    if (logjac_host) {
      e = cudaMemcpyAsync(logjac_host + c0, c->dlj[s], (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, st);
      if (e != cudaSuccess) return (int)e;
    }
    if (sum_host) {
      e = cudaMemcpyAsync(c->hsum + k, c->dsum[s], sizeof(double), cudaMemcpyDeviceToHost, st);
      if (e != cudaSuccess) return (int)e;
    }
  }
  for (int s = 0; s < c->n_streams; ++s) {
    cudaError_t e = cudaStreamSynchronize(c->streams[s]);
    if (e != cudaSuccess) return (int)e;
  }
  if (sum_host) {
    double t = 0.0;
    for (long long k = 0; k < nchunks; ++k) t += c->hsum[k];
    *sum_host = t;
  }
  (void)launches;
  return B2B_OK;
}

// ---------------------------------------------------------------------------------------------------
// NCCL: the single collective of the path (SURVEY §8(e)): all-reduce(sum) of the batch log-density.
// libnccl.so.2 is resolved at run time so that libb2b.so has no link-time NCCL dependency (inside a
// torch process this resolves to the NCCL torch already loaded; inside Julia to the system library).
// ---------------------------------------------------------------------------------------------------
typedef struct {
  char internal[128];
} b2b_nccl_uid;  // layout of ncclUniqueId (NCCL_UNIQUE_ID_BYTES = 128)
typedef void* b2b_nccl_comm_t;
typedef int (*fn_get_uid)(b2b_nccl_uid*);
typedef int (*fn_init_rank)(b2b_nccl_comm_t*, int, b2b_nccl_uid, int);
typedef int (*fn_allreduce)(const void*, void*, size_t, int, int, b2b_nccl_comm_t, cudaStream_t);
typedef int (*fn_destroy)(b2b_nccl_comm_t);
typedef int (*fn_init_all)(b2b_nccl_comm_t*, int, const int*);
typedef int (*fn_group)(void);

static struct {
  void* handle;
  fn_get_uid get_uid;
  fn_init_rank init_rank;
  fn_allreduce allreduce;
  fn_destroy destroy;
  fn_init_all init_all;
  fn_group group_start, group_end;
} g_nccl = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};

static int load_nccl() {
  if (g_nccl.handle) return B2B_OK;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return B2B_ENONCCL;
  g_nccl.get_uid = (fn_get_uid)dlsym(h, "ncclGetUniqueId");
  g_nccl.init_rank = (fn_init_rank)dlsym(h, "ncclCommInitRank");
  g_nccl.allreduce = (fn_allreduce)dlsym(h, "ncclAllReduce");
  g_nccl.destroy = (fn_destroy)dlsym(h, "ncclCommDestroy");
  g_nccl.init_all = (fn_init_all)dlsym(h, "ncclCommInitAll");
  g_nccl.group_start = (fn_group)dlsym(h, "ncclGroupStart");
  g_nccl.group_end = (fn_group)dlsym(h, "ncclGroupEnd");
  if (!g_nccl.get_uid || !g_nccl.init_rank || !g_nccl.allreduce || !g_nccl.destroy || !g_nccl.init_all ||
      !g_nccl.group_start || !g_nccl.group_end)
    return B2B_ENONCCL;
  g_nccl.handle = h;
  return B2B_OK;
}

struct b2b_comm {
  b2b_nccl_comm_t comm;  // this process's rank (one process per GPU), or rank 0 of an in-process clique
  int nranks, rank;
  std::vector<b2b_nccl_comm_t> all;  // b2b_comm_init_all: one communicator per device of the calling process
  std::vector<int> devs;
};

extern "C" int b2b_comm_unique_id(char id_out[128]) {
  int rc = load_nccl();
  if (rc != B2B_OK) return rc;
  b2b_nccl_uid uid;
  rc = g_nccl.get_uid(&uid);
  if (rc != 0) return 100000 + rc;
  memcpy(id_out, uid.internal, 128);
  return B2B_OK;
}

extern "C" int b2b_comm_init_rank(b2b_comm** out, int nranks, int rank, const char id[128]) {
  if (!out || nranks < 1 || rank < 0 || rank >= nranks || !id) return B2B_EINVAL;
  int rc = load_nccl();
  if (rc != B2B_OK) return rc;
  b2b_nccl_uid uid;
  memcpy(uid.internal, id, 128);
  b2b_comm* c = new b2b_comm();
  c->nranks = nranks;
  c->rank = rank;
  rc = g_nccl.init_rank(&c->comm, nranks, uid, rank);
  if (rc != 0) {
    delete c;
    return 100000 + rc;
  }
  *out = c;
  return B2B_OK;
}

extern "C" int b2b_allreduce_sum_f64(b2b_comm* c, double* dev_values, int32_t count, void* stream) {
  if (!c || !dev_values || count < 1) return B2B_EINVAL;
  const int kNcclDouble = 8, kNcclSum = 0;  // ncclFloat64, ncclSum (nccl.h)
  const int rc = g_nccl.allreduce(dev_values, dev_values, (size_t)count, kNcclDouble, kNcclSum, c->comm,
                                  static_cast<cudaStream_t>(stream));
  return rc == 0 ? B2B_OK : 100000 + rc;
}

// ONE process driving several GPUs (a single Julia session holding all 8 devices of a box; SURVEY §8(b)): a clique of
// `ndev` communicators created with ncclCommInitAll, and the log-density sum issued for all of them inside one NCCL
// group.  values[i] / streams[i] belong to device devs[i].
extern "C" int b2b_comm_init_all(b2b_comm** out, int ndev, const int* devs) {
  if (!out || ndev < 1 || ndev > 64) return B2B_EINVAL;
  int rc = load_nccl();
  if (rc != B2B_OK) return rc;
  b2b_comm* c = new b2b_comm();
  c->nranks = ndev;
  c->rank = 0;
  c->all.resize(ndev);
  c->devs.resize(ndev);
  for (int i = 0; i < ndev; ++i) c->devs[i] = devs ? devs[i] : i;
  rc = g_nccl.init_all(c->all.data(), ndev, c->devs.data());
  if (rc != 0) {
    delete c;
    return 100000 + rc;
  }
  c->comm = c->all[0];
  *out = c;
  return B2B_OK;
}

extern "C" int b2b_allreduce_sum_f64_all(b2b_comm* c, double* const* dev_values, int32_t count, void* const* streams) {
  if (!c || c->all.empty() || !dev_values || !streams || count < 1) return B2B_EINVAL;
  const int kNcclDouble = 8, kNcclSum = 0;
  int prev = 0;
  cudaGetDevice(&prev);
  int rc = g_nccl.group_start();
  for (size_t i = 0; i < c->all.size() && rc == 0; ++i) {
    cudaSetDevice(c->devs[i]);
    rc = g_nccl.allreduce(dev_values[i], dev_values[i], (size_t)count, kNcclDouble, kNcclSum, c->all[i],
                          static_cast<cudaStream_t>(streams[i]));
  }
  const int rc2 = g_nccl.group_end();
  cudaSetDevice(prev);
  if (rc == 0) rc = rc2;
  return rc == 0 ? B2B_OK : 100000 + rc;
}

extern "C" int b2b_comm_destroy(b2b_comm* c) {
  if (!c) return B2B_OK;
  int rc = 0;
  if (!c->all.empty()) {
    for (b2b_nccl_comm_t h : c->all) {
      const int r = g_nccl.destroy(h);
      if (r != 0) rc = r;
    }
  } else {
    rc = g_nccl.destroy(c->comm);
  }
  delete c;
  return rc == 0 ? B2B_OK : 100000 + rc;
}
