// common.cuh — error handling, device buffers, launch accounting for libccm_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/ccm_b200.h"

namespace ccm {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

void set_last_error(const std::string& s);
extern std::atomic<uint64_t> g_launches;

#define CCM_CUDA(call)                                                                              \
  do {                                                                                              \
    cudaError_t e__ = (call);                                                                       \
    if (e__ != cudaSuccess) {                                                                       \
      char buf__[512];                                                                              \
      snprintf(buf__, sizeof buf__, "%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      throw ::ccm::Error(e__ == cudaErrorMemoryAllocation ? CCM_ERR_OOM : CCM_ERR_CUDA, buf__);     \
    }                                                                                               \
  } while (0)

#define CCM_REQUIRE(cond, msg)                                           \
  do {                                                                   \
    if (!(cond)) throw ::ccm::Error(CCM_ERR_INVALID, std::string(msg)); \
  } while (0)

// counts our launches (bench.py reports the number as gpu_launches) and checks the launch itself
#define CCM_LAUNCHED()                \
  do {                                \
    ::ccm::g_launches.fetch_add(1);   \
    CCM_CUDA(cudaGetLastError());     \
  } while (0)

// device allocations go through the stream-ordered allocator with an unbounded release threshold: repeated
// create/solve/destroy cycles (LocalBA runs once per keyframe) reuse cached memory instead of paying cudaMalloc/cudaFree
void* dev_alloc(size_t bytes);
void dev_free(void* p);
void copy_stream(cudaStream_t* cs, cudaEvent_t* ev);   // process-wide copy stream and event of the current device (runtime.cu)

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  void release() {
    if (p) dev_free(p);
    p = nullptr; n = 0;
  }
  void alloc(size_t count) {
    release();
    n = count;
    if (count) p = static_cast<T*>(dev_alloc(count * sizeof(T)));
  }
  void alloc_zero(size_t count, cudaStream_t s) {
    alloc(count);
    if (count) CCM_CUDA(cudaMemsetAsync(p, 0, count * sizeof(T), s));
  }
  void upload(const T* h, size_t count, cudaStream_t s) {
    if (n < count) alloc(count);
    if (count) CCM_CUDA(cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, s));
  }
  void download(T* h, size_t count, cudaStream_t s) const {
    if (count) CCM_CUDA(cudaMemcpyAsync(h, p, count * sizeof(T), cudaMemcpyDeviceToHost, s));
  }
  size_t bytes() const { return n * sizeof(T); }
};

inline int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Lays arrays out in one block at 16-byte boundaries, for a single upload (new_points.cu, fuse_neighbours.cu).  Without a host block it
// only measures; with one it copies each array in and answers the address the array will have on the device.
struct Packer {
  size_t at = 0;
  uint8_t* host = nullptr;
  const uint8_t* dev = nullptr;
  size_t reserve(size_t bytes) {
    const size_t off = at;
    at = (at + bytes + 15) & ~size_t(15);
    return off;
  }
  template <typename T>
  const T* put(const T* src, size_t count) {
    const size_t off = reserve(count * sizeof(T));
    if (!host) return nullptr;
    if (count) memcpy(host + off, src, count * sizeof(T));
    return reinterpret_cast<const T*>(dev + off);
  }
};

int current_device();      // device chosen by ccm_init (default 0)
int sm_count();
void ensure_device();      // throws CCM_ERR_NO_DEVICE when there is none

// ---- NCCL communicator (dlopen'ed) ----
struct Comm {
  int rank = 0, nranks = 1;
  void* nccl = nullptr;  // ncclComm_t
  bool active() const { return nranks > 1; }
};
Comm& comm();
void allreduce_f64(double* buf, size_t count, int op, cudaStream_t s);  // op: 0 sum, 2 max

// match.cu: nA x nB Hamming distances of 32-byte descriptors (host in, pinned thread-local host out, one k_hamming launch)
const uint16_t* hamming_matrix_host(const uint8_t* A, int nA, const uint8_t* B, int nB);

// catch-all used by every extern "C" entry point
template <typename F>
int guarded(F&& f) {
  try {
    f();
    return CCM_OK;
  } catch (const Error& e) {
    set_last_error(e.what());
    return e.code;
  } catch (const std::exception& e) {
    set_last_error(e.what());
    return CCM_ERR_INVALID;
  }
}

}  // namespace ccm
