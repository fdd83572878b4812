// C-ABI plumbing: error state, device info, device fault word.
#include "common.cuh"
#include <string.h>

namespace bbdm {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
  return BBDM_E_CUDA;
}

__device__ unsigned long long g_device_fault = 0ull;

unsigned long long* device_fault_ptr() {
  static unsigned long long* p[kMaxDevices] = {nullptr};   // the symbol has one instance per device
  const int dev = current_device();
  if (!p[dev]) cudaGetSymbolAddress((void**)&p[dev], g_device_fault);
  return p[dev];
}

}  // namespace bbdm

extern "C" {

int bbdm_abi_version(void) { return BBDM_ABI_VERSION; }

const char* bbdm_last_error(void) { return bbdm::g_err; }

int bbdm_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  BBDM_CUDA_CHECK(cudaGetDevice(&dev));
  cudaDeviceProp p;
  BBDM_CUDA_CHECK(cudaGetDeviceProperties(&p, dev));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (cc_major) *cc_major = p.major;
  if (cc_minor) *cc_minor = p.minor;
  return BBDM_OK;
}

int bbdm_check_device_fault(void* stream, unsigned long long* fault_word) {
  unsigned long long* p = bbdm::device_fault_ptr();
  BBDM_REQUIRE(p != nullptr, "device fault word unavailable");
  unsigned long long h = 0, zero = 0;
  cudaStream_t s = (cudaStream_t)stream;
  BBDM_CUDA_CHECK(cudaMemcpyAsync(&h, p, sizeof(h), cudaMemcpyDeviceToHost, s));
  BBDM_CUDA_CHECK(cudaStreamSynchronize(s));
  if (h) BBDM_CUDA_CHECK(cudaMemcpyAsync(p, &zero, sizeof(zero), cudaMemcpyHostToDevice, s));
  if (fault_word) *fault_word = h;
  if (h) {
    if ((h >> 28) == 0xBull)
      bbdm::set_error("device fault word 0x%llx: timestep index out of range (the reference's gather raises IndexError)", h);
    else if ((h >> 28) == 0xCull)
      bbdm::set_error("device fault word 0x%llx: Winograd F(6x6,3x3) input transform of a %llu-channel conv left the "
                      "fp16 range (activations above ~290, or non-finite)", h, h & 0xFFFFFFFull);
    else
      bbdm::set_error("device fault word 0x%llx (kernel-side wait timeout)", h);
    return BBDM_E_DEVICE;
  }
  return BBDM_OK;
}

}  // extern "C"
