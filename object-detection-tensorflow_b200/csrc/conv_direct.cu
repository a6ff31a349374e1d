// CUDA-core implicit-GEMM convolution: any filter / stride / dilation / channel
// count, fp32 accumulate.  Used for (i) the reference-precision fp32 path that
// backs the 1e-4 box parity claim, (ii) the Cin=3 stems (mean subtraction fused
// into the operand load) and (iii) as the on-device cross-check of the wgmma
// kernel.  ref: tf.nn.conv2d SSD300.py:519, tf.layers.conv2d SSD300.py:524.
#include "epilogue.cuh"

namespace odt {

constexpr int DM = 64, DN = 64, DK = 16, DTHREADS = 256;

struct DirectGeom {
  int B, H, W, Cin, in_ld, OH, OW, Cout, R, S, stride, dil, pad_t, pad_l, w_ld;
  float mean[3];
};

template <typename T, bool STEM>
__global__ void __launch_bounds__(DTHREADS)
    conv_direct_kernel(const void* __restrict__ in_, const T* __restrict__ wgt,
                       const __grid_constant__ DirectGeom g, const __grid_constant__ Epi e) {
  pdl_launch_dependents();
  __shared__ float As[DK][DM + 4];
  __shared__ float Bs[DK][DN + 4];
  const int tid = threadIdx.x;
  const long long M = (long long)g.B * g.OH * g.OW;
  const int K = g.R * g.S * g.Cin;
  const long long m0 = (long long)blockIdx.x * DM;
  const int n0 = blockIdx.y * DN;

  // loader mapping: row = tid/4 (0..63), k sub-block = (tid%4)*4 .. +3
  const int lrow = tid >> 2, lk = (tid & 3) * 4;
  const long long lm = m0 + lrow;
  const bool lm_ok = lm < M;
  int lb = 0, loy = 0, lox = 0;
  if (lm_ok) {
    lox = (int)(lm % g.OW);
    loy = (int)((lm / g.OW) % g.OH);
    lb = (int)(lm / ((long long)g.OW * g.OH));
  }
  const int ln = n0 + lrow;
  const bool ln_ok = ln < g.Cout;

  // compute mapping: 16x16 threads, 4x4 micro tile
  const int tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += DK) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + lk + j;
      float av = 0.f, bv = 0.f;
      if (k < K) {
        const int tap = k / g.Cin, c = k - tap * g.Cin;
        if (lm_ok) {
          const int r = tap / g.S, s = tap - r * g.S;
          const int iy = loy * g.stride - g.pad_t + r * g.dil;
          const int ix = lox * g.stride - g.pad_l + s * g.dil;
          if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) {
            const long long off = (((long long)lb * g.H + iy) * g.W + ix) * g.in_ld + c;
            if (STEM)
              av = __fsub_rn(reinterpret_cast<const float*>(in_)[off], g.mean[c]);
            else
              av = Elem<T>::ld(reinterpret_cast<const T*>(in_) + off);
          }
        }
        if (ln_ok) bv = Elem<T>::ld(wgt + ((long long)ln * g.R * g.S + tap) * g.w_ld + c);
      }
      As[lk + j][lrow] = av;
      Bs[lk + j][lrow] = bv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < DK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }

  const int ohw = g.OH * g.OW;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const int b = (int)(m / ohw), pix = (int)(m - (long long)b * ohw);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < g.Cout) epi_store_one<T>(e, b, pix, n, acc[i][j]);
    }
  }
}


// ---------------------------------------------------------------------------
// Specialised stems (Cin = 3): one thread = one output pixel x all COUT channels.
// The KS*KS*3 mean-subtracted inputs live in registers, the weights in shared
// memory as [k][COUT] fp32 and are read as warp-broadcast 128-bit loads, so the
// inner loop is 4 FFMA per LDS.128.  HBM traffic = image read + output write.
// ref: conv1_1 SSD300.py:193-200 (3x3 s1 -> 64), YOLOv3.py:388 (3x3 s1 -> 32),
// RetinaNet.py:260-265 / FCOS.py:73-78 (7x7 s2 -> 16), input mean SSD300.py:52-66.
template <typename T, int COUT, int KS, int STRIDE>
__global__ void __launch_bounds__(128)
    conv_stem_kernel(const float* __restrict__ img, const T* __restrict__ wgt,
                     const __grid_constant__ DirectGeom g, const __grid_constant__ Epi e) {
  pdl_launch_dependents();
  constexpr int KK = KS * KS * 3;
  __shared__ __align__(16) float ws[KK][COUT];
  __shared__ float s_scale[COUT], s_shift[COUT];
  for (int i = threadIdx.x; i < KK * COUT; i += blockDim.x) {
    const int k = i / COUT, c = i - k * COUT;  // wgt is [COUT][KS][KS][w_ld]
    const int tap = k / 3, ch = k - tap * 3;
    ws[k][c] = Elem<T>::ld(wgt + ((long long)c * KS * KS + tap) * g.w_ld + ch);
  }
  for (int c = threadIdx.x; c < COUT; c += blockDim.x) {
    s_scale[c] = e.scale ? e.scale[c] : 1.f;
    s_shift[c] = e.shift ? e.shift[c] : 0.f;
  }
  __syncthreads();
  const long long M = (long long)g.B * g.OH * g.OW;
  const int ohw = g.OH * g.OW;
  for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < M;
       m += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(m / ohw);
    const int pix = (int)(m - (long long)b * ohw);
    const int oy = pix / g.OW, ox = pix - oy * g.OW;
    float x[KK];
#pragma unroll
    for (int r = 0; r < KS; ++r) {
      const int iy = oy * STRIDE - g.pad_t + r;
#pragma unroll
      for (int s = 0; s < KS; ++s) {
        const int ix = ox * STRIDE - g.pad_l + s;
        const bool ok = iy >= 0 && iy < g.H && ix >= 0 && ix < g.W;
        const float* p = img + (((long long)b * g.H + iy) * g.W + ix) * 3;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch)
          x[(r * KS + s) * 3 + ch] = ok ? __fsub_rn(__ldg(p + ch), g.mean[ch]) : 0.f;
      }
    }
    float acc[COUT];
#pragma unroll
    for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
#pragma unroll
    for (int k = 0; k < KK; ++k) {
#pragma unroll
      for (int c4 = 0; c4 < COUT / 4; ++c4) {
        const float4 w4 = *reinterpret_cast<const float4*>(&ws[k][c4 * 4]);
        acc[c4 * 4 + 0] = fmaf(x[k], w4.x, acc[c4 * 4 + 0]);
        acc[c4 * 4 + 1] = fmaf(x[k], w4.y, acc[c4 * 4 + 1]);
        acc[c4 * 4 + 2] = fmaf(x[k], w4.z, acc[c4 * 4 + 2]);
        acc[c4 * 4 + 3] = fmaf(x[k], w4.w, acc[c4 * 4 + 3]);
      }
    }
    T* o = reinterpret_cast<T*>(e.out0) + (long long)b * e.out0_img_stride +
           (long long)pix * e.out0_pix_stride;
    constexpr int V = 16 / sizeof(T);
#pragma unroll
    for (int c0 = 0; c0 < COUT; c0 += V) {
      float v[V];
#pragma unroll
      for (int q = 0; q < V; ++q)
        v[q] = apply_act(fmaf(acc[c0 + q], s_scale[c0 + q], s_shift[c0 + q]), e.act);
      if (sizeof(T) == 2) {
        uint4 t;
        __half2* h = reinterpret_cast<__half2*>(&t);
#pragma unroll
        for (int q = 0; q < 4; ++q) h[q] = __floats2half2_rn(v[2 * q], v[2 * q + 1]);
        *reinterpret_cast<uint4*>(o + c0) = t;
      } else {
        *reinterpret_cast<float4*>(o + c0) = make_float4(v[0], v[1], v[2], v[3]);
      }
    }
  }
}

template <typename T, int COUT, int KS, int STRIDE>
static void launch_stem(const float* img, const void* w, const DirectGeom& g, const Epi& e,
                        cudaStream_t st) {
  long long M = (long long)g.B * g.OH * g.OW;
  long long blocks = (M + 127) / 128;
  long long cap = (long long)kNumSMs * 16;
  conv_stem_kernel<T, COUT, KS, STRIDE>
      <<<(unsigned)(blocks < cap ? blocks : cap), 128, 0, st>>>(img, (const T*)w, g, e);
}

template <bool STEM>
static int launch_direct(const void* in, const void* w, int dtype, const odt_conv_params* p,
                         const float* mean, cudaStream_t st) {
  DirectGeom g;
  g.B = p->B; g.H = p->H; g.W = p->W; g.Cin = p->Cin; g.in_ld = p->in_ld;
  g.OH = p->OH; g.OW = p->OW; g.Cout = p->Cout; g.R = p->R; g.S = p->S;
  g.stride = p->stride; g.dil = p->dil; g.pad_t = p->pad_t; g.pad_l = p->pad_l; g.w_ld = p->w_ld;
  g.mean[0] = mean ? mean[0] : 0.f;
  g.mean[1] = mean ? mean[1] : 0.f;
  g.mean[2] = mean ? mean[2] : 0.f;
  Epi e = make_epi(*p);
  long long M = (long long)p->B * p->OH * p->OW;
  dim3 grid((unsigned)((M + DM - 1) / DM), (unsigned)((p->Cout + DN - 1) / DN));
  if (dtype == ODT_F16)
    conv_direct_kernel<__half, STEM><<<grid, DTHREADS, 0, st>>>(in, (const __half*)w, g, e);
  else
    conv_direct_kernel<float, STEM><<<grid, DTHREADS, 0, st>>>(in, (const float*)w, g, e);
  return ODT_OK;
}

}  // namespace odt

using namespace odt;

extern "C" int odt_conv2d_direct(const void* in, const void* weights, int dtype,
                                 const odt_conv_params* p, void* stream) {
  int rc = check_conv_params(p);
  if (rc) return rc;
  ODT_CHECK_ARG(in && weights, "null tensor");
  ODT_CHECK_ARG(dtype == ODT_F16 || dtype == ODT_F32, "dtype");
  ODT_CHECK_ARG(p->in_halo == 0 && p->out0_halo == 0 && p->out0_pool == 0,
                "halo layouts / fused pooling are tensor-core-path only");
  launch_direct<false>(in, weights, dtype, p, nullptr, (cudaStream_t)stream);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_conv2d_stem(const float* images, const float* mean3_host, const void* weights,
                               int dtype, const odt_conv_params* p, void* stream) {
  int rc = check_conv_params(p);
  if (rc) return rc;
  ODT_CHECK_ARG(images && weights && mean3_host, "null tensor");
  ODT_CHECK_ARG(p->Cin == 3, "stem expects Cin == 3");
  ODT_CHECK_ARG(dtype == ODT_F16 || dtype == ODT_F32, "dtype");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == ODT_F16) {  // tensor-core stem first (conv_stem_tc.cu)
    int trc = odt_conv2d_stem_tc_try(images, mean3_host, weights, p, stream);
    if (trc != ODT_ERR_UNSUPPORTED) return trc;
  }
  ODT_CHECK_ARG(p->out0_halo == 0 && p->in_halo == 0 && p->out0_pool == 0,
                "halo output needs the tensor-core stem");
  const bool simple = p->out0 && !p->out1 && !p->out2 && !p->residual && p->out0_group == 0 && p->R == p->S &&
                      p->dil == 1 && p->in_ld == 3 &&
                      p->out0_dtype == (dtype == ODT_F16 ? ODT_F16 : ODT_F32) &&
                      ((uintptr_t)p->out0 % 16) == 0 &&
                      (p->out0_pix_stride * (dtype == ODT_F16 ? 2 : 4)) % 16 == 0 &&
                      (p->out0_img_stride * (dtype == ODT_F16 ? 2 : 4)) % 16 == 0;
  int variant = 0;
  if (simple && p->R == 3 && p->stride == 1 && p->Cout == 64) variant = 1;
  if (simple && p->R == 3 && p->stride == 1 && p->Cout == 32) variant = 2;
  if (simple && p->R == 7 && p->stride == 2 && p->Cout == 16) variant = 3;
  if (variant) {
    DirectGeom g;
    g.B = p->B; g.H = p->H; g.W = p->W; g.Cin = 3; g.in_ld = 3;
    g.OH = p->OH; g.OW = p->OW; g.Cout = p->Cout; g.R = p->R; g.S = p->S;
    g.stride = p->stride; g.dil = 1; g.pad_t = p->pad_t; g.pad_l = p->pad_l; g.w_ld = p->w_ld;
    g.mean[0] = mean3_host[0]; g.mean[1] = mean3_host[1]; g.mean[2] = mean3_host[2];
    Epi e = make_epi(*p);
    if (dtype == ODT_F16) {
      if (variant == 1) launch_stem<__half, 64, 3, 1>(images, weights, g, e, st);
      if (variant == 2) launch_stem<__half, 32, 3, 1>(images, weights, g, e, st);
      if (variant == 3) launch_stem<__half, 16, 7, 2>(images, weights, g, e, st);
    } else {
      if (variant == 1) launch_stem<float, 64, 3, 1>(images, weights, g, e, st);
      if (variant == 2) launch_stem<float, 32, 3, 1>(images, weights, g, e, st);
      if (variant == 3) launch_stem<float, 16, 7, 2>(images, weights, g, e, st);
    }
  } else {
    launch_direct<true>(images, weights, dtype, p, mean3_host, st);
  }
  ODT_LAUNCH_OK();
  return ODT_OK;
}
