// Shared helpers for the bbdm_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/bbdm_b200.h"

namespace bbdm {

// ---- host-side error plumbing ------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);
// device fault word (mbarrier wait timeouts etc.); lives in cabi.cu
unsigned long long* device_fault_ptr();

#define BBDM_CUDA_CHECK(expr)                                                   \
  do {                                                                          \
    cudaError_t _e = (expr);                                                    \
    if (_e != cudaSuccess) return ::bbdm::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)

#define BBDM_REQUIRE(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      ::bbdm::set_error(__VA_ARGS__);      \
      return BBDM_E_INVALID;               \
    }                                      \
  } while (0)

#define BBDM_LAUNCH_CHECK() BBDM_CUDA_CHECK(cudaGetLastError())

// Head dims of the mma.sync attention forward (attention_split.cuh) and the flash backward (attention_bwd.cu): every
// multiple of 8 up to 128.  A multiple of 8 keeps each head's columns 16-byte aligned in the bf16 planes, as the
// 16-byte cp.async chunks need; past 128 these kernels' tiles do not fit in shared memory.  The forward instantiates
// the multiples of 16 in attention_split.cu and the padded sizes in attention_split_padded.cu.
#define BBDM_ATTN_POW2_HEAD_DIMS(X) X(16) X(32) X(64) X(128)
#define BBDM_ATTN_PADDED_HEAD_DIMS(X) X(8) X(24) X(40) X(48) X(56) X(72) X(80) X(88) X(96) X(104) X(112) X(120)
#define BBDM_FOR_ATTN_HEAD_DIMS(X) BBDM_ATTN_POW2_HEAD_DIMS(X) BBDM_ATTN_PADDED_HEAD_DIMS(X)
// Head dims 136 to 256 (multiples of 8) run on kernels of their own (attention_split_wide.cu, attention_bwd_wide.cu),
// instantiated per padded width: D runs at the next multiple of 32, zero past D.
#define BBDM_ATTN_WIDE_PADDED_DIMS(X) X(160) X(192) X(224) X(256)

// Everything cached on the host is cached PER DEVICE (the reference's single-GPU launcher puts the
// model on cuda:N without cudaSetDevice-ing the process default; cabi.py guards the device per call).
constexpr int kMaxDevices = 64;
inline int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}

inline int num_sms() {
  static int n[kMaxDevices] = {0};
  const int dev = current_device();
  if (!n[dev]) {
    cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
    if (n[dev] <= 0) n[dev] = 132;
  }
  return n[dev];
}

// one-time-per-device latch for cudaFuncSetAttribute (function attributes are per device)
struct DeviceOnce {
  bool done[kMaxDevices] = {false};
  bool need() { return !done[current_device()]; }
  void mark() { done[current_device()] = true; }
};

// ---- device helpers ----------------------------------------------------------------------
__device__ __forceinline__ float silu_f(float x) {
  // x * sigmoid(x) = x / (1 + exp(-x)); expf (not __expf) keeps ~1 ulp like torch's CPU path
  return x / (1.0f + expf(-x));
}

// hi = bf16(x) (round-to-nearest-even), lo = bf16(x - hi)
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

// two floats -> packed (hi, lo) bf16x2 words with ONE cvt.rn.bf16x2.f32 per plane (the scalar
// conversions run on the quarter-rate XU pipe and were the attention kernel's top stall)
__device__ __forceinline__ void split2x(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);          // .x = a (low half), .y = b
  const float2 hf = __bfloat1622float2(h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// split 4 floats -> two uint2 (4 bf16 each)
__device__ __forceinline__ void split4(const float4 v, uint2& hi, uint2& lo) {
  split2x(v.x, v.y, hi.x, lo.x);
  split2x(v.z, v.w, hi.y, lo.y);
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float4 ld_f4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st_f4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

}  // namespace bbdm
