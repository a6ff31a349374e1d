// Fused convolution epilogue shared by the tensor-core and the CUDA-core
// convolution kernels.  v = act(acc*scale[c]+shift[c]) (+residual) -> out0 ;
// out1 = act2(v*scale2[c]+shift2[c]), out2 = act3(v*scale3[c]+shift3[c]) (consumer pre-activations).
// ref: bias_add+ReLU SSD300.py:520-521; BN(+act) SSD300.py:534-537,
// YOLOv3.py:504-507; pre-activation BN+ReLU RetinaNet.py:594-597;
// residual adds RetinaNet.py:643, YOLOv3.py:491.
#pragma once
#include "common.cuh"

namespace odt {

struct Epi {
  const float* scale;
  const float* shift;
  int act;
  const void* residual;
  void* out0;
  int out0_dtype;
  long long out0_img_stride;
  int out0_pix_stride;
  int out0_group, out0_group_stride;
  const float* scale2;
  const float* shift2;
  int act2;
  void* out1;
  long long out1_img_stride;
  int out1_pix_stride;
  const float* scale3;
  const float* shift3;
  int act3;
  void* out2;
  long long out2_img_stride;
  int out2_pix_stride;
  int Cout;
  int out1_halo, out2_halo, OW;  // extra outputs stored with a zero 1-pixel border (row length OW + 2)
};

int check_conv_params(const odt_conv_params* p);
}  // namespace odt
// internal: tensor-core stem; ODT_ERR_UNSUPPORTED when no variant matches
int odt_conv2d_stem_tc_try(const float* images, const float* mean3_host, const void* weights,
                           const odt_conv_params* p, void* stream);
namespace odt {

inline Epi make_epi(const odt_conv_params& p) {
  Epi e;
  e.scale = p.scale;
  e.shift = p.shift;
  e.act = p.act;
  e.residual = p.residual;
  e.out0 = p.out0;
  e.out0_dtype = p.out0_dtype;
  e.out0_img_stride = p.out0_img_stride;
  e.out0_pix_stride = p.out0_pix_stride;
  e.out0_group = p.out0_group;
  e.out0_group_stride = p.out0_group_stride;
  e.scale2 = p.scale2;
  e.shift2 = p.shift2;
  e.act2 = p.act2;
  e.out1 = p.out1;
  e.out1_img_stride = p.out1_img_stride;
  e.out1_pix_stride = p.out1_pix_stride;
  e.scale3 = p.scale3;
  e.shift3 = p.shift3;
  e.act3 = p.act3;
  e.out2 = p.out2;
  e.out2_img_stride = p.out2_img_stride;
  e.out2_pix_stride = p.out2_pix_stride;
  e.Cout = p.Cout;
  e.out1_halo = p.out1_halo;
  e.out2_halo = p.out2_halo;
  e.OW = p.OW;
  return e;
}

// element offset of pixel (image b, linear pixel `pix` = oy*OW + ox) in an extra output (dense or halo layout)
__host__ __device__ __forceinline__ long long aux_row(long long img_stride, int pix_stride, int halo, int OW, int b,
                                                      int pix) {
  if (halo) {
    const int oy = pix / OW, ox = pix - oy * OW;
    return (long long)b * img_stride + (long long)((oy + 1) * (OW + 2) + ox + 1) * pix_stride;
  }
  return (long long)b * img_stride + (long long)pix * pix_stride;
}

__device__ __forceinline__ int regroup(const Epi& e, int n) {
  return e.out0_group > 0 ? (n / e.out0_group) * e.out0_group_stride + (n % e.out0_group) : n;
}

// scalar path: one output element (image b, pixel `pix` inside the image, channel n)
template <typename T>
__device__ __forceinline__ void epi_store_one(const Epi& e, int b, int pix, int n, float acc) {
  float sc = e.scale ? __ldg(e.scale + n) : 1.f;
  float sh = e.shift ? __ldg(e.shift + n) : 0.f;
  float v = apply_act(fmaf(acc, sc, sh), e.act);
  const long long o0 = (long long)b * e.out0_img_stride + (long long)pix * e.out0_pix_stride +
                       regroup(e, n);
  if (e.residual) v += Elem<T>::ld(reinterpret_cast<const T*>(e.residual) + o0);
  if (e.out0) {
    if (e.out0_dtype == ODT_F32) {
      reinterpret_cast<float*>(e.out0)[o0] = v;
    } else {
      reinterpret_cast<__half*>(e.out0)[o0] = __float2half_rn(v);
      // the consumer of the fp16 tensor sees the rounded value
      if (sizeof(T) == 2) v = __half2float(__float2half_rn(v));
    }
  }
  if (e.out1) {
    float s2 = e.scale2 ? __ldg(e.scale2 + n) : 1.f;
    float h2 = e.shift2 ? __ldg(e.shift2 + n) : 0.f;
    float w = apply_act(fmaf(v, s2, h2), e.act2);
    const long long o1 = aux_row(e.out1_img_stride, e.out1_pix_stride, e.out1_halo, e.OW, b, pix) + n;
    Elem<T>::st(reinterpret_cast<T*>(e.out1) + o1, w);
  }
  if (e.out2) {
    float s3 = e.scale3 ? __ldg(e.scale3 + n) : 1.f;
    float h3 = e.shift3 ? __ldg(e.shift3 + n) : 0.f;
    float w = apply_act(fmaf(v, s3, h3), e.act3);
    const long long o2 = aux_row(e.out2_img_stride, e.out2_pix_stride, e.out2_halo, e.OW, b, pix) + n;
    Elem<T>::st(reinterpret_cast<T*>(e.out2) + o2, w);
  }
}

}  // namespace odt
