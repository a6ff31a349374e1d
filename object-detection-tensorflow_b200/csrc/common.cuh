// Shared helpers for the sm_90a kernels behind include/odt_b200.h.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/odt_b200.h"

namespace odt {

void set_error(const char* fmt, ...);

#define ODT_CHECK_ARG(cond, msg)                                   \
  do {                                                             \
    if (!(cond)) {                                                 \
      odt::set_error("%s: invalid argument: %s", __func__, msg);   \
      return ODT_ERR_INVALID;                                      \
    }                                                              \
  } while (0)

#define ODT_CUDA_OK(expr)                                                        \
  do {                                                                           \
    cudaError_t e__ = (expr);                                                    \
    if (e__ != cudaSuccess) {                                                    \
      odt::set_error("%s: %s -> %s", __func__, #expr, cudaGetErrorString(e__));  \
      return ODT_ERR_CUDA;                                                       \
    }                                                                            \
  } while (0)

#define ODT_LAUNCH_OK()                                                          \
  do {                                                                           \
    cudaError_t e__ = cudaGetLastError();                                        \
    if (e__ != cudaSuccess) {                                                    \
      odt::set_error("%s: launch failed: %s", __func__, cudaGetErrorString(e__)); \
      return ODT_ERR_CUDA;                                                       \
    }                                                                            \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

template <typename T>
struct Elem;
template <>
struct Elem<float> {
  static __host__ __device__ __forceinline__ float ld(const float* p) { return *p; }
  static __host__ __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
template <>
struct Elem<__half> {
  static __host__ __device__ __forceinline__ float ld(const __half* p) { return __half2float(*p); }
  static __host__ __device__ __forceinline__ void st(__half* p, float v) { *p = __float2half_rn(v); }
};

__host__ __device__ __forceinline__ float apply_act(float v, int act) {
  if (act == ODT_ACT_RELU) return fmaxf(v, 0.f);
  if (act == ODT_ACT_LEAKY) return fmaxf(v, 0.1f * v);
  return v;
}

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// Programmatic dependent launch (PDL).  Every kernel of the library signals its
// dependents at entry; kernels launched with the programmatic-serialisation
// attribute (the tensor-core convolutions) run their prologue early and block in
// pdl_wait() until the preceding grid has completed and flushed its writes.
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Launch with the programmatic-serialisation attribute.  For kernels that call pdl_wait() before they touch what the
// previous kernel in the stream wrote.
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kern)(KArgs...), unsigned grid, int block, int smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

// The per-kernel convolution switches, read on every call (api.cu): 0 = never, 1 = where the kernel's planner or
// cost model takes the layer (the default, also when the variable is unset), 2 = wherever the layer qualifies.  They
// stay because the tests need both ends: mode 2 pins a kernel onto shapes small enough to test, mode 0 gives the
// bit-exact reference the kernel is compared with.  One function per kernel, so that the CPU harnesses of
// tests/native/ can pin their kernel by defining its function alone.
int pw_mode();    // ODT_TC_PW: narrow 1x1 / stride-1 layers on the staged pointwise kernel of conv_pw.cu (tried first)
int thin_mode();  // ODT_TC_THIN: very thin layers (Cin, Cout <= 32, few multiply-adds per pixel) on conv_thin.cu
int tapn_mode();  // ODT_TC_TAPN: narrow 3x3 halo layers with the horizontal taps folded into N (conv_tapn.cu)
int swap_mode();  // ODT_TC_SWAP: narrow 3x3 halo layers (Cout_pad 64 / 128, fp16 out0 alone) on the transposed
                  // 64-cout x 256-pixel tiles of conv_tc_swap.cu
int wide_mode();  // ODT_TC_WIDE: conv_tc's 128 x 256 im2col tile (mode 2: wherever Cout_pad % 256 == 0)

// debug: name of the convolution kernel the last odt_conv2d_* call launched (a string literal; see
// odt_debug_last_conv_kernel), so that tests can name the path a layer took without a profiler.  An inline variable:
// one instance in the library, and a definition in any program that includes a kernel source on its own.
inline const char* g_last_conv_kernel = "";
}  // namespace odt
