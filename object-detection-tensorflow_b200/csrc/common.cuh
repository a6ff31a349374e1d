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
  static __device__ __forceinline__ float ld(const float* p) { return *p; }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
template <>
struct Elem<__half> {
  static __device__ __forceinline__ float ld(const __half* p) { return __half2float(*p); }
  static __device__ __forceinline__ void st(__half* p, float v) { *p = __float2half_rn(v); }
};

__device__ __forceinline__ float apply_act(float v, int act) {
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
bool pdl_enabled();   // ODT_PDL=0 disables the launch attribute (api.cu)
bool flat_enabled();  // ODT_TC_FLAT=0 disables the halo-flat 3x3 path (A/B measurements)
bool kskip_enabled();  // ODT_TC_KSKIP=1: do not issue the all-zero 16-deep K steps of thin layers (Cin padded to 64)
int thin_mode();       // ODT_TC_THIN: 1 = very thin layers (Cin, Cout <= 32, few multiply-adds per pixel) go through the
                       // CUDA-core kernel of conv_thin.cu, 2 = wherever the layer qualifies, 0 / unset = never
int tapn_mode();       // ODT_TC_TAPN: 1 = narrow 3x3 halo layers go through conv_tapn.cu (taps folded into N) where its
                       // cost model predicts a gain, 2 = wherever the layer qualifies, 0 / unset = never
int pw_mode();         // ODT_TC_PW: 1 = narrow 1x1 / stride-1 layers go through the staged pointwise kernel of conv_pw.cu
                       // (tried before conv_thin.cu), 2 = wherever the layer qualifies, 0 = never
bool wres_enabled();  // ODT_TC_WRES=0 disables shared-memory-resident filter banks in the flat path

}  // namespace odt
