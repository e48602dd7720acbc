// Host-side plumbing shared by the library's translation units: the error string, device buffers, launch shapes and
// the one rule that decides whether a kernel may use a caller's pointer in place.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/derp_b200.h"

// The calling thread's last error message (derp_last_error); defined in derp_b200.cu
extern thread_local std::string g_err;

inline int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define CU(call)                                                                                     \
  do {                                                                                               \
    cudaError_t e_ = (call);                                                                         \
    if (e_ != cudaSuccess)                                                                           \
      return fail(DERP_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_) + " (" + __FILE__ + ":" + \
                                  std::to_string(__LINE__) + ")");                                   \
  } while (0)

// Grow-only device buffer on the device that was current when it was allocated.  ensure() on another device frees the
// old block on its own device and allocates on the current one, so a thread_local scratch follows its thread from GPU to
// GPU without a list of buffers to release.
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  int device = -1;
  ~DevBuf() { release(); }
  void release() {
    if (p) {
      int cur = device;
      cudaGetDevice(&cur);
      if (cur != device) cudaSetDevice(device);
      cudaFree(p);
      if (cur != device) cudaSetDevice(cur);
    }
    p = nullptr;
    n = 0;
  }
  cudaError_t ensure(size_t count) {
    int cur = 0;
    cudaError_t e = cudaGetDevice(&cur);
    if (e != cudaSuccess) return e;
    if (count <= n && p && device == cur) return cudaSuccess;
    release();
    e = cudaMalloc(&p, std::max<size_t>(count, 1) * sizeof(T));
    if (e == cudaSuccess) {
      n = count;
      device = cur;
    }
    return e;
  }
};

// The CTA of the 2-D per-pixel kernels: derp::kBlockX x derp::kBlockY (derp_kernels.cuh; derp_b200.cu asserts they agree)
constexpr int kBlock2X = 32, kBlock2Y = 8;
inline dim3 grid2(int W, int H, int z = 1) { return dim3((W + kBlock2X - 1) / kBlock2X, (H + kBlock2Y - 1) / kBlock2Y, z); }
inline dim3 block2() { return dim3(kBlock2X, kBlock2Y, 1); }
inline unsigned grid1(size_t n, int t = 256) { return (unsigned)((n + t - 1) / t); }

inline int floorD(double v) {
  int i = (int)v;
  return i - (i > v);
}
// INTER_NEAREST source index of each of dn destination samples (resize.cpp resizeNN)
inline void nearestAxis(int sn, int dn, std::vector<int>& ofs) {
  const double inv = (double)dn / sn, ifx = 1. / inv;
  ofs.resize(dn);
  for (int d = 0; d < dn; ++d) ofs[d] = std::min(floorD(d * ifx), sn - 1);
}

// ---- caller pointers ----------------------------------------------------------------------------------------------
// The device whose memory p is, or -1 for host, managed and unknown pointers
inline int deviceOf(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    (void)cudaGetLastError();
    return -1;
  }
  return a.type == cudaMemoryTypeDevice ? a.device : -1;
}

// The rule for a caller's pointer: a kernel uses it in place only when it is device memory of the current device and
// aligned to `align` bytes (16 where the kernel moves float4 or uint4).  Anything else (host, managed or another GPU's
// memory, or a misaligned pointer) is staged through scratch with cudaMemcpyDefault.
inline bool inPlace(const void* p, size_t align) {
  int cur = -1;
  return (uintptr_t)p % align == 0 && cudaGetDevice(&cur) == cudaSuccess && deviceOf(p) == cur;
}

// Points p at count elements a kernel on the current device can read: p itself, or a copy in scratch made on stream st
template <typename T>
int stageIn(const T*& p, size_t count, DevBuf<T>& scratch, size_t align = alignof(T), cudaStream_t st = nullptr) {
  if (inPlace(p, align)) return DERP_OK;
  CU(scratch.ensure(count));
  CU(cudaMemcpyAsync(scratch.p, p, count * sizeof(T), cudaMemcpyDefault, st));
  p = scratch.p;
  return DERP_OK;
}

// Points p at count elements a kernel on the current device can write: p itself, or scratch (see stageOut)
template <typename T>
int outBuffer(T*& p, size_t count, DevBuf<T>& scratch, size_t align = alignof(T)) {
  if (inPlace(p, align)) return DERP_OK;
  CU(scratch.ensure(count));
  p = scratch.p;
  return DERP_OK;
}

// Copies what a kernel wrote to `written` (from outBuffer) to the caller's dst, when the two differ
template <typename T>
int stageOut(T* dst, const T* written, size_t count) {
  if (written != dst) CU(cudaMemcpy(dst, written, count * sizeof(T), cudaMemcpyDefault));
  return DERP_OK;
}

// Enables the current device's direct access to `other`'s memory where the two have a peer path (NVLink)
inline int enablePeer(int device, int other) {
  int can = 0;
  CU(cudaDeviceCanAccessPeer(&can, device, other));
  if (can) {
    const cudaError_t e = cudaDeviceEnablePeerAccess(other, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CU(e);
    (void)cudaGetLastError();
  }
  return DERP_OK;
}
