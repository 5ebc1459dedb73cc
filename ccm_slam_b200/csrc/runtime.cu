// runtime.cu — process-level state of libccm_b200.so: device selection, error string, launch counter,
// and the NCCL communicator used by landmark-sharded global BA (one process per GPU).
#include <dlfcn.h>

#include <mutex>

#include "common.cuh"

namespace ccm {

static thread_local std::string t_last_error;
void set_last_error(const std::string& s) { t_last_error = s; }
std::atomic<uint64_t> g_launches{0};

static std::atomic<int> g_device{0};
static std::atomic<int> g_sm_count{0};

int current_device() { return g_device.load(); }

void ensure_device() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    cudaGetLastError();
    throw Error(CCM_ERR_NO_DEVICE, "no CUDA device: libccm_b200 has no CPU fallback");
  }
  CCM_CUDA(cudaSetDevice(g_device.load()));
}

int sm_count() {
  int v = g_sm_count.load();
  if (v == 0) {
    cudaDeviceProp prop;
    CCM_CUDA(cudaGetDeviceProperties(&prop, g_device.load()));
    v = prop.multiProcessorCount;
    g_sm_count.store(v);
  }
  return v;
}

// ---- pooled device memory --------------------------------------------------------------------------------------
static std::mutex g_alloc_mu;
static cudaStream_t g_alloc_stream[64] = {nullptr};
static bool g_pool_ready[64] = {false};

static cudaStream_t alloc_stream(int dev) {
  std::lock_guard<std::mutex> lk(g_alloc_mu);
  if (!g_pool_ready[dev]) {
    CCM_CUDA(cudaStreamCreateWithFlags(&g_alloc_stream[dev], cudaStreamNonBlocking));
    cudaMemPool_t pool;
    CCM_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev));
    unsigned long long thr = ~0ull;  // never hand cached memory back to the driver
    CCM_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    g_pool_ready[dev] = true;
  }
  return g_alloc_stream[dev];
}

// second stream (+ its event) of the current device for host-to-device copies that overlap kernels of a handle's own stream
static cudaStream_t g_copy_stream[64] = {nullptr};
static cudaEvent_t g_copy_event[64] = {nullptr};
void copy_stream(cudaStream_t* cs, cudaEvent_t* ev) {
  int dev = 0;
  CCM_CUDA(cudaGetDevice(&dev));
  dev &= 63;
  std::lock_guard<std::mutex> lk(g_alloc_mu);
  if (!g_copy_stream[dev]) {
    CCM_CUDA(cudaStreamCreateWithFlags(&g_copy_stream[dev], cudaStreamNonBlocking));
    CCM_CUDA(cudaEventCreateWithFlags(&g_copy_event[dev], cudaEventDisableTiming));
  }
  *cs = g_copy_stream[dev];
  *ev = g_copy_event[dev];
}

void* dev_alloc(size_t bytes) {
  int dev = 0;
  CCM_CUDA(cudaGetDevice(&dev));
  cudaStream_t s = alloc_stream(dev & 63);
  void* p = nullptr;
  CCM_CUDA(cudaMallocAsync(&p, bytes, s));
  CCM_CUDA(cudaStreamSynchronize(s));  // the block is usable from any stream afterwards
  return p;
}

void dev_free(void* p) {
  // callers synchronise the stream that used the block before releasing it (handle destructors do)
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return;
  if (!g_pool_ready[dev & 63]) { cudaFree(p); return; }
  cudaFreeAsync(p, g_alloc_stream[dev & 63]);
}

// ---- per-thread staging of the batched entry points -------------------------------------------------------------------------------
Staging::~Staging() {
  if (h_in) cudaFreeHost(h_in);
  if (h_out) cudaFreeHost(h_out);
  if (stream) cudaStreamDestroy(stream);
}

void Staging::use_current_device() {
  if (device != current_device()) {
    if (stream) { cudaStreamDestroy(stream); stream = nullptr; }
    in.release(); out.release();
    device = current_device();
  }
  if (!stream) CCM_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
}

void Staging::reserve(size_t d_in, size_t d_out, size_t p_in, size_t p_out) {
  auto pinned = [](uint8_t** p, size_t* cap, size_t bytes) {
    if (*cap >= bytes) return;
    if (*p) cudaFreeHost(*p);
    *p = nullptr; *cap = 0;
    CCM_CUDA(cudaMallocHost((void**)p, bytes + bytes / 4));
    *cap = bytes + bytes / 4;
  };
  pinned(&h_in, &h_in_cap, p_in);
  pinned(&h_out, &h_out_cap, p_out);
  if (in.n < d_in) in.alloc(d_in + d_in / 4);
  if (out.n < d_out) out.alloc(d_out + d_out / 4);
}

// ---- NCCL through dlopen: the single-GPU path has no link-time dependency on it ----
typedef struct { char internal[128]; } ncclUniqueId_t;
typedef int (*fn_ncclGetUniqueId)(ncclUniqueId_t*);
typedef int (*fn_ncclCommInitRank)(void**, int, ncclUniqueId_t, int);
typedef int (*fn_ncclCommDestroy)(void*);
typedef int (*fn_ncclAllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef const char* (*fn_ncclGetErrorString)(int);

static struct {
  void* lib = nullptr;
  fn_ncclGetUniqueId GetUniqueId = nullptr;
  fn_ncclCommInitRank CommInitRank = nullptr;
  fn_ncclCommDestroy CommDestroy = nullptr;
  fn_ncclAllReduce AllReduce = nullptr;
  fn_ncclGetErrorString GetErrorString = nullptr;
} g_nccl;
static std::mutex g_nccl_mu;
static Comm g_comm;
Comm& comm() { return g_comm; }

static void load_nccl() {
  std::lock_guard<std::mutex> lk(g_nccl_mu);
  if (g_nccl.lib) return;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    g_nccl.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.lib) break;
  }
  if (!g_nccl.lib) throw Error(CCM_ERR_NCCL, std::string("dlopen(libnccl.so.2) failed: ") + dlerror());
  g_nccl.GetUniqueId = (fn_ncclGetUniqueId)dlsym(g_nccl.lib, "ncclGetUniqueId");
  g_nccl.CommInitRank = (fn_ncclCommInitRank)dlsym(g_nccl.lib, "ncclCommInitRank");
  g_nccl.CommDestroy = (fn_ncclCommDestroy)dlsym(g_nccl.lib, "ncclCommDestroy");
  g_nccl.AllReduce = (fn_ncclAllReduce)dlsym(g_nccl.lib, "ncclAllReduce");
  g_nccl.GetErrorString = (fn_ncclGetErrorString)dlsym(g_nccl.lib, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.AllReduce)
    throw Error(CCM_ERR_NCCL, "libnccl.so.2 lacks a required symbol");
}

#define CCM_NCCL(call)                                                                     \
  do {                                                                                     \
    int r__ = (call);                                                                      \
    if (r__ != 0) {                                                                        \
      std::string m__ = std::string(#call) + " -> ";                                       \
      m__ += g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "nccl error";            \
      throw Error(CCM_ERR_NCCL, m__);                                                      \
    }                                                                                      \
  } while (0)

// op: ncclSum = 0, ncclMax = 2 ; datatype ncclFloat64 = 8
void allreduce_f64(double* buf, size_t count, int op, cudaStream_t s) {
  if (!g_comm.active() || count == 0) return;
  CCM_NCCL(g_nccl.AllReduce(buf, buf, count, 8, op, g_comm.nccl, s));
}

}  // namespace ccm

using namespace ccm;

extern "C" int ccm_version(void) { return 100; }
extern "C" const char* ccm_last_error(void) { return t_last_error.c_str(); }
extern "C" uint64_t ccm_kernel_launches(void) { return g_launches.load(); }

extern "C" int ccm_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

extern "C" int ccm_init(int device) {
  return guarded([&] {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      throw Error(CCM_ERR_NO_DEVICE, "no CUDA device: libccm_b200 has no CPU fallback");
    }
    CCM_REQUIRE(device >= 0 && device < n, "ccm_init: device index out of range");
    g_device.store(device);
    g_sm_count.store(0);
    CCM_CUDA(cudaSetDevice(device));
    CCM_CUDA(cudaFree(0));
  });
}

extern "C" int ccm_shutdown(void) {
  return guarded([&] {
    if (g_comm.nccl) {
      g_nccl.CommDestroy(g_comm.nccl);
      g_comm = Comm{};
    }
  });
}

extern "C" int ccm_comm_unique_id(uint8_t id[128]) {
  return guarded([&] {
    load_nccl();
    ncclUniqueId_t u;
    CCM_NCCL(g_nccl.GetUniqueId(&u));
    memcpy(id, u.internal, 128);
  });
}

extern "C" int ccm_comm_init(int rank, int nranks, const uint8_t id[128]) {
  return guarded([&] {
    CCM_REQUIRE(nranks >= 1 && rank >= 0 && rank < nranks, "ccm_comm_init: bad rank/nranks");
    ensure_device();
    if (g_comm.nccl) {
      g_nccl.CommDestroy(g_comm.nccl);
      g_comm = Comm{};
    }
    if (nranks == 1) return;
    load_nccl();
    ncclUniqueId_t u;
    memcpy(u.internal, id, 128);
    void* c = nullptr;
    CCM_NCCL(g_nccl.CommInitRank(&c, nranks, u, rank));
    g_comm.rank = rank; g_comm.nranks = nranks; g_comm.nccl = c;
  });
}

extern "C" int ccm_comm_destroy(void) { return ccm_shutdown(); }
extern "C" int ccm_comm_rank(void) { return g_comm.rank; }
extern "C" int ccm_comm_size(void) { return g_comm.nranks; }

extern "C" int ccm_l2_flush(void) {
  return guarded([&] {
    ensure_device();
    static void* buf = nullptr;
    const size_t n = 256ull << 20;
    if (!buf) CCM_CUDA(cudaMalloc(&buf, n));
    CCM_CUDA(cudaMemset(buf, 0x5a, n));
    CCM_CUDA(cudaDeviceSynchronize());
  });
}

extern "C" int ccm_host_register(void* ptr, uint64_t bytes) {
  return guarded([&] {
    ensure_device();
    CCM_CUDA(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
  });
}

extern "C" int ccm_host_unregister(void* ptr) {
  return guarded([&] { CCM_CUDA(cudaHostUnregister(ptr)); });
}
