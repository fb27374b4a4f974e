// What the C-ABI translation units (api.cu and db_api.cu: Spiral, dpir_api.cu and dpir_server_api.cu: DoublePIR) share:
// device buffers, the error plumbing of the entry points and the device check.
#pragma once
#include "../../include/b200pir.h"
#include "kernels.h"
#include <exception>
#include <string>

namespace b200pir {

// what b200pir_last_error() returns: the message of the calling thread's last failed call (defined in api.cu)
extern thread_local std::string g_last_error;

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() {}
  explicit DevBuf(size_t count) { alloc(count); }
  void alloc(size_t count) {
    release();
    n = count;
    if (count) B200_CUDA(cudaMalloc(&p, count * sizeof(T)));
  }
  void ensure(size_t count) { if (count > n) alloc(count); }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
  ~DevBuf() { release(); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
};

// records e as the last error and returns its code
int fail(const std::exception& e);

// `device` must exist (there is no CPU path); it becomes the calling thread's current device
inline void use_device(int device) {
  int ndev = 0;
  B200_CUDA(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) throw Error(B200PIR_E_BADARG, "no such CUDA device (this library has no CPU path)");
  B200_CUDA(cudaSetDevice(device));
}

}  // namespace b200pir

#define API_BEGIN try {
#define API_END                                                 \
  }                                                             \
  catch (const std::exception& e) { return ::b200pir::fail(e); } \
  return 0;
