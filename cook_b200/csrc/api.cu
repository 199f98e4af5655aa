// api.cu — lifetime and error surface of libcookgpu.so (include/cook_gpu.h).
#include <dlfcn.h>

#include "common.cuh"

extern "C" {

const char* cook_gpu_version(void) { return "cook_b200 0.1 sm_90a"; }

// Replaces per-pool make-fenzo-state (scheduler/scheduler.clj:2301-2324):
// called once at takeLeadership (mesos.clj:193).  Fails (no CPU fallback) when
// no CUDA device is visible.
int32_t cook_gpu_init(const cook_gpu_config* cfg, cook_ctx** out) {
  if (!out) return COOK_E_BADARG;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) return COOK_E_NO_DEVICE;
  cook_ctx* c = new cook_ctx();
  if (cfg && cfg->n_devices > 0 && cfg->device_ids) {
    for (int i = 0; i < cfg->n_devices; i++) {
      if (cfg->device_ids[i] < 0 || cfg->device_ids[i] >= n) { delete c; return COOK_E_BADARG; }
      c->devices.push_back(cfg->device_ids[i]);
    }
  } else {
    int cur = 0;
    cudaGetDevice(&cur);
    c->devices.push_back(cur);
  }
  *out = c;
  return COOK_OK;
}

int32_t cook_gpu_shutdown(cook_ctx* ctx) {
  if (!ctx) return COOK_E_BADARG;
  delete ctx;
  return COOK_OK;
}

int32_t cook_pool_open(cook_ctx* ctx, const char* pool_name, int32_t dru_mode, int32_t device,
                       cook_pool** out) {
  if (!ctx || !out || dru_mode < 0 || dru_mode > 1) return COOK_E_BADARG;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return COOK_E_NO_DEVICE;
  if (device < 0 || device >= n) return COOK_E_BADARG;
  cook_pool* p = new cook_pool();
  p->ctx = ctx;
  p->name = pool_name ? pool_name : "";
  p->dru_mode = dru_mode;
  p->device = device;
  if (cudaSetDevice(device) != cudaSuccess) { delete p; return COOK_E_CUDA; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete p; return COOK_E_CUDA; }
  p->sm_count = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking) != cudaSuccess) { delete p; return COOK_E_CUDA; }
  for (auto& e : p->ev)
    if (cudaEventCreate(&e) != cudaSuccess) { delete p; return COOK_E_CUDA; }
  *out = p;
  return COOK_OK;
}

int32_t cook_pool_close(cook_pool* p) {
  if (!p) return COOK_E_BADARG;
  cudaSetDevice(p->device);
  if (p->stream) cudaStreamSynchronize(p->stream);
  p->arena.release();
  if (p->xchg) cudaFree(p->xchg);
  if (p->match_plan && p->match_plan_free) p->match_plan_free(p->match_plan);
  if (p->state && p->state_free) p->state_free(p->state);
  for (auto& e : p->ev)
    if (e) cudaEventDestroy(e);
  if (p->stream) cudaStreamDestroy(p->stream);
  delete p;
  return COOK_OK;
}

int32_t cook_last_error(cook_pool* p, char* buf, int32_t len) {
  if (!p || !buf || len <= 0) return COOK_E_BADARG;
  strncpy(buf, p->err, (size_t)len - 1);
  buf[len - 1] = 0;
  return COOK_OK;
}

int32_t cook_last_stats(cook_pool* p, int32_t phase, cook_phase_stats* out) {
  if (!p || !out || phase < 0 || phase > COOK_PHASE_AUDIT) return COOK_E_BADARG;
  *out = p->phase[phase];
  return COOK_OK;
}

// §8e: the one exchange step.  NCCL is resolved at run time (dlopen) so the
// library loads on hosts without it and shares the process's NCCL (torch's
// bundled copy when the host is Python).
typedef int (*nccl_allgather_fn)(const void*, void*, size_t, int, void*, void*);
int32_t cook_allgather_usage(void* comm, void* stream, const double* local_dev, double* out_dev,
                             int64_t n_doubles) {
  if (!comm || !local_dev || !out_dev || n_doubles <= 0) return COOK_E_BADARG;
  static nccl_allgather_fn fn = nullptr;
  if (!fn) {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return COOK_E_NCCL;
    fn = (nccl_allgather_fn)dlsym(h, "ncclAllGather");
    if (!fn) return COOK_E_NCCL;
  }
  const int ncclFloat64 = 8;  // ncclDataType_t: ncclDouble
  int rc = fn(local_dev, out_dev, (size_t)n_doubles, ncclFloat64, comm, stream);
  return rc == 0 ? COOK_OK : COOK_E_NCCL;
}

static void* nccl_sym(const char* name) {
  static void* h = nullptr;
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  return h ? dlsym(h, name) : nullptr;
}
struct nccl_uid { char b[128]; };
int32_t cook_comm_unique_id(uint8_t out_id[128]) {
  if (!out_id) return COOK_E_BADARG;
  typedef int (*fn_t)(nccl_uid*);
  fn_t fn = (fn_t)nccl_sym("ncclGetUniqueId");
  if (!fn) return COOK_E_NCCL;
  nccl_uid u;
  if (fn(&u) != 0) return COOK_E_NCCL;
  memcpy(out_id, u.b, 128);
  return COOK_OK;
}
int32_t cook_comm_init(const uint8_t id[128], int32_t rank, int32_t world, int32_t device, void** out_comm) {
  if (!id || !out_comm || rank < 0 || world <= 0 || rank >= world) return COOK_E_BADARG;
  typedef int (*fn_t)(void**, int, nccl_uid, int);
  fn_t fn = (fn_t)nccl_sym("ncclCommInitRank");
  if (!fn) return COOK_E_NCCL;
  if (cudaSetDevice(device) != cudaSuccess) return COOK_E_CUDA;
  nccl_uid u;
  memcpy(u.b, id, 128);
  void* comm = nullptr;
  if (fn(&comm, world, u, rank) != 0) return COOK_E_NCCL;
  *out_comm = comm;
  return COOK_OK;
}
int32_t cook_comm_destroy(void* comm) {
  if (!comm) return COOK_E_BADARG;
  typedef int (*fn_t)(void*);
  fn_t fn = (fn_t)nccl_sym("ncclCommDestroy");
  if (!fn) return COOK_E_NCCL;
  return fn(comm) == 0 ? COOK_OK : COOK_E_NCCL;
}

}  // extern "C"
