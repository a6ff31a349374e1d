// Fused convolution epilogue shared by the tensor-core and the CUDA-core
// convolution kernels.  v = act(acc*scale[c]+shift[c]) (+residual) -> out0 ;
// out1 = act2(v*scale2[c]+shift2[c]), out2 = act3(v*scale3[c]+shift3[c]) (consumer pre-activations).
// One definition, callable on host and device: epi_param (the staged parameters), epi_act_f16 / epi_store_f16
// (the fp16 vector step of conv_tc, conv_tapn, conv_thin and conv_pw) and epi_store_one (one element, conv_direct).
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

// host: a 16-byte aligned fp16 tensor whose pixel rows are whole 16-byte sectors and hold at least `need` channels
inline bool f16_rows_aligned(const void* ptr, long long img_stride, int pix_stride, int need) {
  return ((uintptr_t)ptr & 15) == 0 && img_stride % 8 == 0 && pix_stride % 8 == 0 && pix_stride >= need;
}

// host: the outputs can be stored in whole 16-byte sectors of `need` channels per pixel (conv_thin, conv_pw).  The
// residual shares out0's addressing (strides / halo), whether or not out0 itself is stored.
inline bool f16_sector_outputs_ok(const odt_conv_params* p, int need) {
  return (!p->out0 || (p->out0_dtype == ODT_F16 && f16_rows_aligned(p->out0, p->out0_img_stride, p->out0_pix_stride, need))) &&
         (!p->out1 || f16_rows_aligned(p->out1, p->out1_img_stride, p->out1_pix_stride, need)) &&
         (!p->out2 || f16_rows_aligned(p->out2, p->out2_img_stride, p->out2_pix_stride, need)) &&
         (!p->residual || (f16_rows_aligned(p->residual, p->out0_img_stride, p->out0_pix_stride, need) &&
                           (p->out0 || p->out0_dtype == ODT_F16)));
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

__host__ __device__ __forceinline__ int regroup(const Epi& e, int n) {
  return e.out0_group > 0 ? (n / e.out0_group) * e.out0_group_stride + (n % e.out0_group) : n;
}

// read-only global load; a plain load where the same source runs on the CPU (the kernels' test harnesses)
#ifdef __CUDA_ARCH__
#define ODT_LDG(p) __ldg(p)
#else
#define ODT_LDG(p) (*(p))
#endif

// Parameter row `row` at channel n: 0 scale, 1 shift, 2 scale2, 3 shift2, 4 scale3, 5 shift3.  A missing pointer, or
// a channel at or past Cout, gives the identity (scale 1, shift 0).  The kernels stage these rows in this order.
__host__ __device__ __forceinline__ float epi_param(const Epi& e, int row, int n) {
  const float* src = row == 0 ? e.scale : row == 1 ? e.shift : row == 2 ? e.scale2 : row == 3 ? e.shift2
                     : row == 4 ? e.scale3 : e.shift3;
  return (n < e.Cout && src) ? ODT_LDG(src + n) : ((row & 1) ? 0.f : 1.f);
}

// ---- vector step: a run of NV 16-byte sectors (8*NV channels) of one pixel row, fp16 outputs ----
// `par` points at the run's first channel in the staged parameter rows (row stride `ps` floats); both are multiples
// of 4 floats, so parameters are read 128 bits at a time.

template <int NV>
__host__ __device__ __forceinline__ void epi_affine(float* v, const float* par, int ps, int act) {
#pragma unroll
  for (int i = 0; i < 2 * NV; ++i) {
    const float4 sc = reinterpret_cast<const float4*>(par)[i], sh = reinterpret_cast<const float4*>(par + ps)[i];
    v[4 * i + 0] = apply_act(fmaf(v[4 * i + 0], sc.x, sh.x), act);
    v[4 * i + 1] = apply_act(fmaf(v[4 * i + 1], sc.y, sh.y), act);
    v[4 * i + 2] = apply_act(fmaf(v[4 * i + 2], sc.z, sh.z), act);
    v[4 * i + 3] = apply_act(fmaf(v[4 * i + 3], sc.w, sh.w), act);
  }
}

template <int NV>
__host__ __device__ __forceinline__ void epi_round_f16(const float* v, uint4* out) {
  __half2* h = reinterpret_cast<__half2*>(out);
#pragma unroll
  for (int i = 0; i < 4 * NV; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
}

// v = act(v * par[0] + par[1]), rounded to fp16 into `out` (the pooled paths take their maximum of these)
template <int NV>
__host__ __device__ __forceinline__ void epi_act_f16(float* v, const float* par, int ps, int act, uint4* out) {
  epi_affine<NV>(v, par, ps, act);
  epi_round_f16<NV>(v, out);
}

// the fragment form of epi_act_f16: one pair of adjacent columns of an accumulator row (a wgmma fragment register
// pair), act(v * sc + sh) rounded to one half2 -- the same operations, element by element, as epi_act_f16
__host__ __device__ __forceinline__ __half2 epi_act_f16x2(float a, float b, float2 sc, float2 sh, int act) {
  return __floats2half2_rn(apply_act(fmaf(a, sc.x, sh.x), act), apply_act(fmaf(b, sc.y, sh.y), act));
}

// a consumer's pre-activation act(x * par[0] + par[1]) of the rounded fp16 values x
template <int NV>
__host__ __device__ __forceinline__ void epi_pre_f16(const uint4* x, const float* par, int ps, int act, uint4* out) {
  const __half2* h = reinterpret_cast<const __half2*>(x);
  __half2* o = reinterpret_cast<__half2*>(out);
#pragma unroll
  for (int i = 0; i < 2 * NV; ++i) {
    const float4 sc = reinterpret_cast<const float4*>(par)[i], sh = reinterpret_cast<const float4*>(par + ps)[i];
    const float2 fa = __half22float2(h[2 * i]), fb = __half22float2(h[2 * i + 1]);
    o[2 * i] = __floats2half2_rn(apply_act(fmaf(fa.x, sc.x, sh.x), act), apply_act(fmaf(fa.y, sc.y, sh.y), act));
    o[2 * i + 1] = __floats2half2_rn(apply_act(fmaf(fb.x, sc.z, sh.z), act), apply_act(fmaf(fb.y, sc.w, sh.w), act));
  }
}

// The fused output of the run: v = act(acc*scale + shift) (+ the residual where e.residual is set), rounded to fp16
// and stored to out0; out1 / out2 are computed from the ROUNDED value, which is what the consumer of out0 sees, and
// stay the same when out0 is not stored (epi_store_one and conv_tc's scalar column path follow the same rule).
// res(q) yields the residual's sector q of the run: a load issued right there (after the affine step, which keeps
// the loaded values' live range short) or a value the caller loaded earlier.  o0 / o1 / o2: element offsets of the
// run in out0 (= residual) / out1 / out2.
template <int NV, typename Res>
__host__ __device__ __forceinline__ void epi_store_f16(const Epi& e, float* v, const float* par, int ps, Res res,
                                                       long long o0, long long o1, long long o2) {
  epi_affine<NV>(v, par, ps, e.act);
  if (e.residual) {
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      const uint4 t = res(q);
      const __half2* r = reinterpret_cast<const __half2*>(&t);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(r[i]);
        v[8 * q + 2 * i] += f.x;
        v[8 * q + 2 * i + 1] += f.y;
      }
    }
  }
  uint4 packed[NV];
  epi_round_f16<NV>(v, packed);
  if (e.out0) {
    uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out0) + o0);
#pragma unroll
    for (int q = 0; q < NV; ++q) op[q] = packed[q];
  }
  if (e.out1) {
    uint4 p1[NV];
    epi_pre_f16<NV>(packed, par + 2 * ps, ps, e.act2, p1);
    uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out1) + o1);
#pragma unroll
    for (int q = 0; q < NV; ++q) op[q] = p1[q];
  }
  if (e.out2) {
    uint4 p2[NV];
    epi_pre_f16<NV>(packed, par + 4 * ps, ps, e.act3, p2);
    uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out2) + o2);
#pragma unroll
    for (int q = 0; q < NV; ++q) op[q] = p2[q];
  }
}

// scalar path: one output element (image b, pixel `pix` inside the image, channel n)
template <typename T>
__host__ __device__ __forceinline__ void epi_store_one(const Epi& e, int b, int pix, int n, float acc) {
  float sc = e.scale ? ODT_LDG(e.scale + n) : 1.f;
  float sh = e.shift ? ODT_LDG(e.shift + n) : 0.f;
  float v = apply_act(fmaf(acc, sc, sh), e.act);
  const long long o0 = (long long)b * e.out0_img_stride + (long long)pix * e.out0_pix_stride +
                       regroup(e, n);
  if (e.residual) v += Elem<T>::ld(reinterpret_cast<const T*>(e.residual) + o0);
  if (e.out0 && e.out0_dtype == ODT_F32) {
    reinterpret_cast<float*>(e.out0)[o0] = v;
  } else {
    const __half hv = __float2half_rn(v);
    if (e.out0) reinterpret_cast<__half*>(e.out0)[o0] = hv;
    // out1 / out2 of an fp16 layer take the rounded value, as the vector step does, whether or not out0 is stored
    if (sizeof(T) == 2) v = __half2float(hv);
  }
  if (e.out1) {
    float s2 = e.scale2 ? ODT_LDG(e.scale2 + n) : 1.f;
    float h2 = e.shift2 ? ODT_LDG(e.shift2 + n) : 0.f;
    float w = apply_act(fmaf(v, s2, h2), e.act2);
    const long long o1 = aux_row(e.out1_img_stride, e.out1_pix_stride, e.out1_halo, e.OW, b, pix) + n;
    Elem<T>::st(reinterpret_cast<T*>(e.out1) + o1, w);
  }
  if (e.out2) {
    float s3 = e.scale3 ? ODT_LDG(e.scale3 + n) : 1.f;
    float h3 = e.shift3 ? ODT_LDG(e.shift3 + n) : 0.f;
    float w = apply_act(fmaf(v, s3, h3), e.act3);
    const long long o2 = aux_row(e.out2_img_stride, e.out2_pix_stride, e.out2_halo, e.OW, b, pix) + n;
    Elem<T>::st(reinterpret_cast<T*>(e.out2) + o2, w);
  }
}

}  // namespace odt
