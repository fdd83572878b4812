// Multi-tensor optimizer / EMA updates: ONE launch over all 248 UNet parameter tensors
// instead of ~10 elementwise launches per tensor.
//
//   adam_multi_kernel  torch.optim.Adam's single-tensor update (runners/utils.py:48-57 creates it; step at
//                      runners/BaseRunner.py:413): grad (+ wd * p), exp_avg.lerp_(grad, 1-b1),
//                      exp_avg_sq = b2*exp_avg_sq + (1-b2)*grad^2, p -= step_size * exp_avg / (sqrt(exp_avg_sq)/bc2s + eps),
//                      optionally followed IN THE SAME PASS by the EMA update of the freshly written parameter.
//   adam_multi_dev_kernel  the same update with step and lr in device memory (bbdm_adam_multi_dev: capturable).
//   ema_multi_kernel   shadow = (1-d)*p + d*shadow  (runners/base/EMA.py:21-29), or shadow = p (with_decay=False).
//
// Parameters and gradients stay the separate nn.Parameter / .grad tensors of the module (pointer table); the optimizer
// state and the EMA shadow live in flat buffers addressed through per-tensor offsets.  HBM-bound: Adam 16 B read +
// 12 B written per element (+ 4 + 4 with the fused EMA); EMA alone 8 B read + 4 B written.
#include "common.cuh"

namespace bbdm {

constexpr int OPT_CHUNK = 4096;      // elements per CTA pass (256 threads x 4 x float4)

struct AdamScalars {
  float lr_over_bc1, beta1, beta2, eps, weight_decay, inv_bc2_sqrt, one_minus_beta1, one_minus_beta2;
  float ema_decay, ema_one_minus;      // ema_decay < 0: no fused EMA
};

__device__ __forceinline__ float ema_lerp(float p, float s, float d, float one_minus_d) {
  // the reference's expression: (1.0 - d) * param + d * shadow with the python scalars (1.0 - d) and d each
  // rounded to fp32 once (torch multiplies an fp32 tensor by a python float in fp32), one rounding per op
  return __fadd_rn(__fmul_rn(one_minus_d, p), __fmul_rn(d, s));
}

// the scalar preparation of torch.optim.adam._single_tensor_adam (python floats = fp64), each scalar rounded to fp32
// once at the end.  The hyper-parameters must arrive as doubles: 1 - beta2 of an fp32-rounded beta2 0.999 is 1.3e-5
// off, and with it exp_avg_sq and the bias correction.  Host (bbdm_adam_multi) and device (bbdm_adam_multi_dev, step
// and lr read from device memory) run the same expressions.
__host__ __device__ inline AdamScalars adam_scalars(double lr, double beta1, double beta2, double eps, double weight_decay,
                                                    double step, bool ema, double ema_decay) {
  const double bc1 = 1.0 - pow(beta1, step), bc2 = 1.0 - pow(beta2, step);
  AdamScalars a;
  a.lr_over_bc1 = (float)(lr / bc1);
  a.beta1 = (float)beta1; a.beta2 = (float)beta2; a.eps = (float)eps; a.weight_decay = (float)weight_decay;
  a.inv_bc2_sqrt = (float)(1.0 / sqrt(bc2));
  a.one_minus_beta1 = (float)(1.0 - beta1);
  a.one_minus_beta2 = (float)(1.0 - beta2);
  a.ema_decay = ema ? (float)ema_decay : -1.0f;
  a.ema_one_minus = (float)(1.0 - ema_decay);
  return a;
}

__device__ __forceinline__ void adam_chunk(float* const* __restrict__ params, const float* const* __restrict__ grads,
                                           const int64_t* __restrict__ numel, const int64_t* __restrict__ state_off,
                                           const int32_t* __restrict__ chunk_tensor, const int32_t* __restrict__ chunk_index,
                                           float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                           float* __restrict__ ema_shadow, const AdamScalars& a) {
  const int t = chunk_tensor[blockIdx.x];
  const int64_t n = numel[t], start = (int64_t)chunk_index[blockIdx.x] * OPT_CHUNK;
  float* __restrict__ p = params[t];
  const float* __restrict__ g = grads[t];
  if (g == nullptr) return;                       // parameter without a gradient this step: untouched, like torch
  float* __restrict__ m = exp_avg + state_off[t];
  float* __restrict__ v = exp_avg_sq + state_off[t];
  float* __restrict__ s = ema_shadow ? ema_shadow + state_off[t] : nullptr;
  const int64_t end = start + OPT_CHUNK < n ? start + OPT_CHUNK : n;
  for (int64_t i = start + threadIdx.x; i < end; i += 256) {
    float gi = g[i];
    const float pi = p[i];
    if (a.weight_decay != 0.f) gi = fmaf(a.weight_decay, pi, gi);
    const float mi = fmaf(a.one_minus_beta1, gi - m[i], m[i]);
    const float vi = fmaf(a.one_minus_beta2 * gi, gi, a.beta2 * v[i]);
    const float denom = sqrtf(vi) * a.inv_bc2_sqrt + a.eps;
    const float pn = pi - a.lr_over_bc1 * (mi / denom);
    m[i] = mi;
    v[i] = vi;
    p[i] = pn;
    if (s && a.ema_decay >= 0.f) s[i] = ema_lerp(pn, s[i], a.ema_decay, a.ema_one_minus);
  }
}

__global__ void __launch_bounds__(256)
adam_multi_kernel(float* const* __restrict__ params, const float* const* __restrict__ grads,
                  const int64_t* __restrict__ numel, const int64_t* __restrict__ state_off,
                  const int32_t* __restrict__ chunk_tensor, const int32_t* __restrict__ chunk_index,
                  float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, float* __restrict__ ema_shadow,
                  const AdamScalars a) {
  adam_chunk(params, grads, numel, state_off, chunk_tensor, chunk_index, exp_avg, exp_avg_sq, ema_shadow, a);
}

// step += 1 on the device, ahead of the update launch that reads it (stream order: every CTA sees the new count)
__global__ void adam_step_increment_kernel(float* step) { *step += 1.0f; }

// the capturable form: step (fp32, already incremented) and lr (fp64) in device memory, so a captured graph
// replays with the counter advancing and the learning rate its owner last wrote; the bias corrections are formed
// once per CTA from them
__global__ void __launch_bounds__(256)
adam_multi_dev_kernel(float* const* __restrict__ params, const float* const* __restrict__ grads,
                      const int64_t* __restrict__ numel, const int64_t* __restrict__ state_off,
                      const int32_t* __restrict__ chunk_tensor, const int32_t* __restrict__ chunk_index,
                      float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, float* __restrict__ ema_shadow,
                      const float* __restrict__ step, const double* __restrict__ lr, double beta1, double beta2,
                      double eps, double weight_decay, double ema_decay) {
  __shared__ AdamScalars sa;
  if (threadIdx.x == 0)
    sa = adam_scalars(*lr, beta1, beta2, eps, weight_decay, (double)*step, ema_shadow != nullptr, ema_decay);
  __syncthreads();
  const AdamScalars a = sa;
  adam_chunk(params, grads, numel, state_off, chunk_tensor, chunk_index, exp_avg, exp_avg_sq, ema_shadow, a);
}

__global__ void __launch_bounds__(256)
ema_multi_kernel(const float* const* __restrict__ params, const int64_t* __restrict__ numel,
                 const int64_t* __restrict__ state_off, const int32_t* __restrict__ chunk_tensor,
                 const int32_t* __restrict__ chunk_index, float* __restrict__ shadow, float decay, float one_minus,
                 int with_decay) {
  const int t = chunk_tensor[blockIdx.x];
  const int64_t n = numel[t], start = (int64_t)chunk_index[blockIdx.x] * OPT_CHUNK;
  const float* __restrict__ p = params[t];
  float* __restrict__ s = shadow + state_off[t];
  const int64_t end = start + OPT_CHUNK < n ? start + OPT_CHUNK : n;
  for (int64_t i = start + threadIdx.x; i < end; i += 256) s[i] = with_decay ? ema_lerp(p[i], s[i], decay, one_minus) : p[i];
}

}  // namespace bbdm

using namespace bbdm;

extern "C" {

int bbdm_optim_chunk_elems(void) { return OPT_CHUNK; }

int bbdm_adam_multi(void* const* params, const void* const* grads, const int64_t* numel, const int64_t* state_off,
                    const int32_t* chunk_tensor, const int32_t* chunk_index, int n_chunks, float* exp_avg,
                    float* exp_avg_sq, double lr, double beta1, double beta2, double eps, double weight_decay, int64_t step,
                    float* ema_shadow, double ema_decay, void* stream) {
  BBDM_REQUIRE(params && grads && numel && state_off && chunk_tensor && chunk_index && exp_avg && exp_avg_sq,
               "adam_multi: null pointer");
  BBDM_REQUIRE(n_chunks > 0 && step >= 1, "adam_multi: need n_chunks > 0 and step >= 1");
  const AdamScalars a = adam_scalars(lr, beta1, beta2, eps, weight_decay, (double)step, ema_shadow != nullptr, ema_decay);
  adam_multi_kernel<<<n_chunks, 256, 0, (cudaStream_t)stream>>>((float* const*)params, (const float* const*)grads, numel,
                                                               state_off, chunk_tensor, chunk_index, exp_avg, exp_avg_sq,
                                                               ema_shadow, a);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

int bbdm_adam_multi_dev(void* const* params, const void* const* grads, const int64_t* numel, const int64_t* state_off,
                        const int32_t* chunk_tensor, const int32_t* chunk_index, int n_chunks, float* exp_avg,
                        float* exp_avg_sq, float* step, const double* lr, double beta1, double beta2, double eps,
                        double weight_decay, float* ema_shadow, double ema_decay, void* stream) {
  BBDM_REQUIRE(params && grads && numel && state_off && chunk_tensor && chunk_index && exp_avg && exp_avg_sq && step && lr,
               "adam_multi_dev: null pointer");
  BBDM_REQUIRE(n_chunks > 0, "adam_multi_dev: need n_chunks > 0");
  adam_step_increment_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step);
  BBDM_LAUNCH_CHECK();
  adam_multi_dev_kernel<<<n_chunks, 256, 0, (cudaStream_t)stream>>>((float* const*)params, (const float* const*)grads,
                                                                   numel, state_off, chunk_tensor, chunk_index, exp_avg,
                                                                   exp_avg_sq, ema_shadow, step, lr, beta1, beta2, eps,
                                                                   weight_decay, ema_decay);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

int bbdm_ema_multi(const void* const* params, const int64_t* numel, const int64_t* state_off,
                   const int32_t* chunk_tensor, const int32_t* chunk_index, int n_chunks, float* shadow, double decay,
                   int with_decay, void* stream) {
  BBDM_REQUIRE(params && numel && state_off && chunk_tensor && chunk_index && shadow && n_chunks > 0, "ema_multi: bad args");
  ema_multi_kernel<<<n_chunks, 256, 0, (cudaStream_t)stream>>>((const float* const*)params, numel, state_off, chunk_tensor,
                                                              chunk_index, shadow, (float)decay, (float)(1.0 - decay), with_decay);
  BBDM_LAUNCH_CHECK();
  return BBDM_OK;
}

}  // extern "C"
