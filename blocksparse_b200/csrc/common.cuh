// Shared device/host helpers for libbsmm_b200.so (sm_90a only).
#pragma once
#include <stdlib.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>

#include "../../include/bsmm_b200.h"

namespace bsmm {

// ---- error plumbing (thread-local, no exceptions cross the C ABI) ----------------
inline char* err_buf() { static thread_local char buf[512] = ""; return buf; }
inline const char*& kernel_name_slot() { static thread_local const char* k = ""; return k; }

inline int fail(int code, const char* fmt, ...) {
  va_list ap; va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}
inline int check_launch(const char* what) {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail((int)e, "%s: %s", what, cudaGetErrorString(e));
  }
  kernel_name_slot() = what;
  return 0;
}

// ---- dtype helpers --------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__host__ __device__ inline int dtype_size(int dt) { return dt == BSMM_F32 ? 4 : 2; }

// Dispatch a dtype code to a template type.  Usage: DISPATCH_DTYPE(code, T, { body using T; })
#define BSMM_DISPATCH_DTYPE(code, T, ...)                               \
  switch (code) {                                                       \
    case BSMM_F32:  { using T = float;          __VA_ARGS__; break; }   \
    case BSMM_F16:  { using T = __half;         __VA_ARGS__; break; }   \
    case BSMM_BF16: { using T = __nv_bfloat16;  __VA_ARGS__; break; }   \
    default: return bsmm::fail(BSMM_E_DTYPE, "unsupported dtype code %d", (int)(code)); \
  }

#define BSMM_DISPATCH_BSIZE(bs, BS, ...)                                \
  switch (bs) {                                                         \
    case 8:  { constexpr int BS = 8;  __VA_ARGS__; break; }             \
    case 16: { constexpr int BS = 16; __VA_ARGS__; break; }             \
    case 32: { constexpr int BS = 32; __VA_ARGS__; break; }             \
    case 64: { constexpr int BS = 64; __VA_ARGS__; break; }             \
    default: return bsmm::fail(BSMM_E_BSIZE, "unsupported block size %d", (int)(bs)); \
  }

// sm_grid = sm_count minus BSMM_SM_MARGIN (environment, default 0): the SMs host-side schedules are balanced for, so that
// a margin stays free for a concurrent NCCL kernel.
struct DeviceInfo { int sm_count, cc_major, cc_minor; bool ok; int sm_grid; };
inline int sm_margin() {
  static const int margin = [] {
    const char* e = getenv("BSMM_SM_MARGIN");
    const int v = e ? atoi(e) : 0;
    return v < 0 ? 0 : v;
  }();
  return margin;
}
inline const DeviceInfo& device_info() {
  static thread_local DeviceInfo info = {0, 0, 0, false, 0};
  static thread_local int cached_dev = -1;
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess) { info.ok = false; return info; }
  if (dev != cached_dev) {
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) == cudaSuccess) {
      const int usable = p.multiProcessorCount - sm_margin();
      info = {p.multiProcessorCount, p.major, p.minor, true, usable > 0 ? usable : 1};
      cached_dev = dev;
    } else {
      info.ok = false;
    }
  }
  return info;
}

// cudaFuncSetAttribute is per device: `mask` (one static per kernel instantiation) remembers the device ordinals a
// kernel has already been configured on, so a host thread that moves between GPUs configures each of them once.
template <typename K>
inline int ensure_dyn_smem(K kern, size_t smem, uint64_t& mask) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return fail(BSMM_E_NODEV, "no CUDA device");
  const uint64_t bit = 1ull << (dev & 63);
  if (mask & bit) return 0;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e));
  mask |= bit;
  return 0;
}

}  // namespace bsmm
