// common.cuh — error handling, device buffers, launch accounting for libccm_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
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
  ~DevBuf() {
    // on an error path work queued on the caller's stream may still use the block: dev_free's contract wants it finished
    if (p && std::uncaught_exceptions()) cudaDeviceSynchronize();
    release();
  }
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

int sm_count();

// blocks for n items at per_cta items a block, at most eight per SM (the kernels loop over the rest), at least one
inline int grid_size(long long n, int per_cta) { return std::max(1, std::min(div_up(n, per_cta), sm_count() * 8)); }

// a non-blocking stream for the length of one call
struct CallStream {
  cudaStream_t s = nullptr;
  CallStream() { CCM_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); }
  CallStream(const CallStream&) = delete;
  CallStream& operator=(const CallStream&) = delete;
  ~CallStream() { cudaStreamDestroy(s); }
};

// Lays arrays out in one block at 16-byte boundaries, for a single upload (Staging::upload).  Without a host block it
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

// The staging of one batched entry point, which keeps its own thread_local instance: a stream, a pinned block and a device block each
// way.  A block too small for a call grows to 1.25x what the call needs.  The stream and the device blocks belong to the device they
// were made on: the first call after ccm_init picks another device releases them.  The pinned output holds a call's results until the
// thread's next call that uses the same instance.
struct Staging {
  cudaStream_t stream = nullptr;
  int device = -1;
  uint8_t* h_in = nullptr;
  uint8_t* h_out = nullptr;
  size_t h_in_cap = 0, h_out_cap = 0;
  DevBuf<uint8_t> in, out;
  Staging() = default;
  Staging(const Staging&) = delete;
  Staging& operator=(const Staging&) = delete;
  ~Staging();
  // blocks of at least these sizes in bytes: device input, device output, pinned input, pinned output
  void reserve(size_t d_in, size_t d_out, size_t p_in, size_t p_out);
  // pack(Packer&) lays the upload out; it runs twice, to measure and then to fill the pinned input.  The device output grows to
  // out_bytes, of which the first down_bytes come back through the pinned output.  Queues the upload on `stream`.
  template <typename F>
  void upload(F&& pack, size_t out_bytes, size_t down_bytes) {
    Packer measure;
    pack(measure);
    const size_t bytes = measure.at;
    reserve(bytes, out_bytes, bytes, down_bytes);
    Packer pk;
    pk.host = h_in; pk.dev = in.p;
    pack(pk);
    CCM_CUDA(cudaMemcpyAsync(in.p, h_in, bytes, cudaMemcpyHostToDevice, stream));
  }
  // runs a call's device work, f(), on the current device's stream; if f throws, the stream is drained before the exception leaves,
  // so no copy of the call still reads the pinned blocks or writes the caller's arrays
  template <typename F>
  void run(F&& f) {
    use_current_device();
    struct Drain {
      cudaStream_t s;
      ~Drain() { if (std::uncaught_exceptions()) cudaStreamSynchronize(s); }
    } drain{stream};
    f();
  }

 private:
  void use_current_device();
};

int current_device();      // device chosen by ccm_init (default 0)
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
