// common.cuh -- shared helpers of librgnn (error plumbing, activations, vector loads).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <float.h>
#include <math.h>
#include <stdlib.h>

#include "../../include/rgnn.h"

namespace rgnn {

// ---- error plumbing (thread-local message, never throws across the ABI) ----
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define RGNN_CHECK_CUDA(expr)                                                              \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      rgnn::set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, \
                      cudaGetErrorString(_e));                                             \
      return RGNN_E_CUDA;                                                                  \
    }                                                                                      \
  } while (0)

#define RGNN_REQUIRE(cond, ...)                                                            \
  do {                                                                                     \
    if (!(cond)) {                                                                         \
      rgnn::set_error(__VA_ARGS__);                                                        \
      return RGNN_E_INVALID;                                                               \
    }                                                                                      \
  } while (0)

#define RGNN_PROPAGATE(expr)                                                               \
  do {                                                                                     \
    int _r = (expr);                                                                       \
    if (_r != RGNN_OK) return _r;                                                          \
  } while (0)

// SMs of an H100 SXM: the grid-shape heuristics (GEMM tile width, split-K, segment-kernel splits) aim at one wave of
// this many CTAs; persistent grids use the SM count of the device they run on.
constexpr int RGNN_WAVE_SMS = 132;

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- device-side activations: utils/utils.py:36-58 ----
// The transcendental activations are kept OUT of line: inlining tanhf/erff/expm1f at every use site
// (4 components x rows in flight x 2 sites) makes the segment kernels many times larger and instruction-fetch
// bound.  relu / linear / leaky_relu stay inline.
// Each translation unit gets its own copy (static), so no relocatable device code is needed.
// tanh is the default activation of GGNN / RGAT / the scaffold and sits in GEMM epilogues (GRU candidate state):
// 1 - 2 / (exp(2x) + 1) with the SFU exponential -- absolute error < 1e-6 (the parity metric is max-norm, 1e-4),
// exact limits at +-inf, 6 instructions instead of the ~40 of tanhf (the GRU output GEMM was epilogue-bound on it).
__device__ __forceinline__ float fast_tanh(float x) {
  const float e = __expf(2.0f * x);
  return 1.0f - __fdividef(2.0f, e + 1.0f);
}
static __device__ __noinline__ float slow_act(float x, int act) {
  switch (act) {
    case RGNN_ACT_TANH: return fast_tanh(x);
    case RGNN_ACT_ELU: return x > 0.0f ? x : expm1f(x);
    case RGNN_ACT_SELU: return 1.0507009873554805f * (x > 0.0f ? x : 1.6732632423543772f * expm1f(x));
    case RGNN_ACT_GELU: return x * (0.5f * (1.0f + erff(x * 0.70710678118654752f)));  // exact-erf form
    default: return x;
  }
}
__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == RGNN_ACT_LINEAR) return x;
  if (act == RGNN_ACT_RELU) return fmaxf(x, 0.0f);
  if (act == RGNN_ACT_LEAKY_RELU) return x > 0.0f ? x : 0.2f * x;        // tf.nn.leaky_relu alpha=0.2
  if (act == RGNN_ACT_TANH) return fast_tanh(x);
  return slow_act(x, act);
}
__device__ __forceinline__ float hard_sigmoid(float x) {                 // Keras hard_sigmoid (TF1 GRU default)
  return fminf(fmaxf(0.2f * x + 0.5f, 0.0f), 1.0f);
}
static __device__ __noinline__ float4 slow_act4(float4 v, int act) {     // one call per 4 elements, every activation
  switch (act) {
    case RGNN_ACT_RELU: return make_float4(fmaxf(v.x, 0.0f), fmaxf(v.y, 0.0f), fmaxf(v.z, 0.0f), fmaxf(v.w, 0.0f));
    case RGNN_ACT_TANH: return make_float4(fast_tanh(v.x), fast_tanh(v.y), fast_tanh(v.z), fast_tanh(v.w));
    case RGNN_ACT_LEAKY_RELU:
      return make_float4(v.x > 0.0f ? v.x : 0.2f * v.x, v.y > 0.0f ? v.y : 0.2f * v.y, v.z > 0.0f ? v.z : 0.2f * v.z,
                         v.w > 0.0f ? v.w : 0.2f * v.w);
    case RGNN_ACT_GELU:
      return make_float4(v.x * (0.5f * (1.0f + erff(v.x * 0.70710678118654752f))), v.y * (0.5f * (1.0f + erff(v.y * 0.70710678118654752f))),
                         v.z * (0.5f * (1.0f + erff(v.z * 0.70710678118654752f))), v.w * (0.5f * (1.0f + erff(v.w * 0.70710678118654752f))));
    default: return make_float4(slow_act(v.x, act), slow_act(v.y, act), slow_act(v.z, act), slow_act(v.w, act));
  }
}
// Hot per-message path: linear / relu inline, everything else one out-of-line call per float4.
__device__ __forceinline__ float4 act4(float4 v, int act) {
  if (act == RGNN_ACT_LINEAR) return v;
  if (act == RGNN_ACT_RELU) return make_float4(fmaxf(v.x, 0.0f), fmaxf(v.y, 0.0f), fmaxf(v.z, 0.0f), fmaxf(v.w, 0.0f));
  return slow_act4(v, act);
}
// Cold path (row epilogues): nothing inline, to keep these kernels small enough for the instruction cache.
__device__ __forceinline__ float4 act4_cold(float4 v, int act) {
  if (act == RGNN_ACT_LINEAR) return v;
  return slow_act4(v, act);
}
// d act(x) / dx from the pre-activation x (utils/utils.py:36-58); transcendental cases out of line, as above
static __device__ __noinline__ float act_grad_slow(float x, int act) {
  switch (act) {
    case RGNN_ACT_TANH: { const float y = fast_tanh(x); return 1.0f - y * y; }
    case RGNN_ACT_ELU: return x > 0.0f ? 1.0f : expf(x);
    case RGNN_ACT_SELU: return x > 0.0f ? 1.0507009873554805f : 1.0507009873554805f * 1.6732632423543772f * expf(x);
    case RGNN_ACT_GELU: return 0.5f * (1.0f + erff(x * 0.70710678118654752f)) + x * 0.3989422804014327f * expf(-0.5f * x * x);
    default: return 1.0f;
  }
}
__device__ __forceinline__ float act_grad(float x, int act) {
  if (act == RGNN_ACT_LINEAR) return 1.0f;
  if (act == RGNN_ACT_RELU) return x > 0.0f ? 1.0f : 0.0f;
  if (act == RGNN_ACT_LEAKY_RELU) return x > 0.0f ? 1.0f : 0.2f;
  return act_grad_slow(x, act);
}

// Programmatic dependent launch (sm_90+): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may
// become resident while its predecessor in the stream is still running; pdl_wait() blocks until the predecessor grid has
// COMPLETED and its writes are visible (no-op for a normal launch), so everything before it (barrier init,
// reads of per-batch plan arrays) overlaps the predecessor's tail.  pdl_launch_dependents() lets the successor start.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Launch `kernel<<<grid, block, smem, stream>>>(params)` as a programmatic dependent of the previous kernel in the stream.
// Only for kernels that call pdl_wait() before touching anything an earlier kernel produced or still reads.
template <typename Params>
static inline cudaError_t launch_pdl(void (*kernel)(Params), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, const Params& params) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, params);
}

// read-only 128-bit load through the non-coherent path (tables written by a previous kernel)
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace rgnn
