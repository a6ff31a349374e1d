// HBM-bound glue kernels between the convolutions (NHWC, fp16 or fp32 storage,
// fp32 math): input normalisation, SAME max-pool, channel L2-norm, per-channel
// affine+activation, legacy bilinear / nearest up-sampling, GroupNorm.
// 128-bit vectorised along C whenever C and the channel stride allow it.
#include "common.cuh"

namespace odt {

// ---- 16-byte vector access helpers ---------------------------------------
template <typename T, int V>
struct VecIO;
template <>
struct VecIO<float, 1> {
  static __device__ __forceinline__ void ld(const float* p, float* v) { v[0] = *p; }
  static __device__ __forceinline__ void st(float* p, const float* v) { *p = v[0]; }
};
template <>
struct VecIO<__half, 1> {
  static __device__ __forceinline__ void ld(const __half* p, float* v) { v[0] = __half2float(*p); }
  static __device__ __forceinline__ void st(__half* p, const float* v) { *p = __float2half_rn(v[0]); }
};
template <>
struct VecIO<float, 4> {
  static __device__ __forceinline__ void ld(const float* p, float* v) {
    float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  static __device__ __forceinline__ void st(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <>
struct VecIO<__half, 8> {
  static __device__ __forceinline__ void ld(const __half* p, float* v) {
    uint4 t = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 f = __half22float2(h[i]);
      v[2 * i] = f.x;
      v[2 * i + 1] = f.y;
    }
  }
  static __device__ __forceinline__ void st(__half* p, const float* v) {
    uint4 t;
    __half2* h = reinterpret_cast<__half2*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = t;
  }
};
template <typename T>
struct FullVec;
template <>
struct FullVec<float> {
  static constexpr int V = 4;
};
template <>
struct FullVec<__half> {
  static constexpr int V = 8;
};

static inline bool can_vec(const void* a, const void* b, int C, int ld, int V, int esize) {
  return C % V == 0 && ld % V == 0 && ((uintptr_t)a % 16) == 0 && ((uintptr_t)b % 16) == 0 &&
         V * esize == 16;
}

static inline int grid_for(long long work, int threads) {
  long long b = (work + threads - 1) / threads;
  long long cap = (long long)kNumSMs * 16;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

// ---- input normalisation (a1) ---------------------------------------------
template <typename T>
__global__ void normalize_kernel(const float* __restrict__ img, T* __restrict__ out,
                                 long long pixels, int ld, float m0, float m1, float m2) {
  pdl_launch_dependents();
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < pixels;
       p += (long long)gridDim.x * blockDim.x) {
    const float* s = img + p * 3;
    T* d = out + p * ld;
    Elem<T>::st(d + 0, __fsub_rn(s[0], m0));
    Elem<T>::st(d + 1, __fsub_rn(s[1], m1));
    Elem<T>::st(d + 2, __fsub_rn(s[2], m2));
    for (int c = 3; c < ld; ++c) Elem<T>::st(d + c, 0.f);
  }
}

// images - mean -> fp16 RGBX with a zero border of `pad` pixels (the border is never written: the caller zero-fills
// the buffer once).  One thread = 4 pixels: 3 x LDG.128 in, 2 x STG.128 out.
__global__ void pack_rgbx_kernel(const float* __restrict__ img, __half* __restrict__ out, int B, int H, int W,
                                 int pad, float m0, float m1, float m2, int vec) {
  pdl_launch_dependents();
  const int PW = W + 2 * pad, PH = H + 2 * pad;
  if (vec) {
    const int wq = W >> 2;
    const long long total = (long long)B * H * wq;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
      const int xq = (int)(i % wq);
      const long long row = i / wq;  // b*H + y
      const int y = (int)(row % H), b = (int)(row / H);
      const float4* s = reinterpret_cast<const float4*>(img + (row * W + 4 * xq) * 3);
      const float4 a = __ldcs(s), c = __ldcs(s + 1), d = __ldcs(s + 2);
      uint4 o0, o1;
      __half2* h0 = reinterpret_cast<__half2*>(&o0);
      __half2* h1 = reinterpret_cast<__half2*>(&o1);
      h0[0] = __floats2half2_rn(__fsub_rn(a.x, m0), __fsub_rn(a.y, m1));
      h0[1] = __floats2half2_rn(__fsub_rn(a.z, m2), 0.f);
      h0[2] = __floats2half2_rn(__fsub_rn(a.w, m0), __fsub_rn(c.x, m1));
      h0[3] = __floats2half2_rn(__fsub_rn(c.y, m2), 0.f);
      h1[0] = __floats2half2_rn(__fsub_rn(c.z, m0), __fsub_rn(c.w, m1));
      h1[1] = __floats2half2_rn(__fsub_rn(d.x, m2), 0.f);
      h1[2] = __floats2half2_rn(__fsub_rn(d.y, m0), __fsub_rn(d.z, m1));
      h1[3] = __floats2half2_rn(__fsub_rn(d.w, m2), 0.f);
      __half* dst = out + (((long long)b * PH + y + pad) * PW + 4 * xq + pad) * 4;
      if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        reinterpret_cast<uint4*>(dst)[0] = o0;
        reinterpret_cast<uint4*>(dst)[1] = o1;
      } else {  // odd pad: 8-byte aligned rows
        uint2* d2 = reinterpret_cast<uint2*>(dst);
        d2[0] = make_uint2(o0.x, o0.y);
        d2[1] = make_uint2(o0.z, o0.w);
        d2[2] = make_uint2(o1.x, o1.y);
        d2[3] = make_uint2(o1.z, o1.w);
      }
    }
  } else {
    const long long total = (long long)B * H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
      const int x = (int)(i % W);
      const long long row = i / W;
      const int y = (int)(row % H), b = (int)(row / H);
      const float* s = img + i * 3;
      uint2 o;
      __half2* h = reinterpret_cast<__half2*>(&o);
      h[0] = __floats2half2_rn(__fsub_rn(s[0], m0), __fsub_rn(s[1], m1));
      h[1] = __floats2half2_rn(__fsub_rn(s[2], m2), 0.f);
      *reinterpret_cast<uint2*>(out + (((long long)b * PH + y + pad) * PW + x + pad) * 4) = o;
    }
  }
}

// Flat element index -> (first channel of the vector, pixel, x, y, image).  `small` (uniform: the whole index space fits
// 31 bits) selects 32-bit unsigned divisions: the 64-bit ones cost ~100 instructions each, and five of them per vector
// made these kernels instruction-bound (upsample_add at the 100x100 FPN level: 0.105 ms for 246 MB of traffic).
struct PixelIndex {
  int c, x, y, b;
  long long pix;
};
template <int V>
__device__ __forceinline__ PixelIndex split_index(long long i, int cv, int W, int H, bool small) {
  PixelIndex r;
  if (small) {
    const unsigned u = (unsigned)i, p = u / (unsigned)cv;
    const unsigned row = p / (unsigned)W, b = row / (unsigned)H;
    r.c = (int)(u - p * (unsigned)cv) * V;
    r.x = (int)(p - row * (unsigned)W);
    r.y = (int)(row - b * (unsigned)H);
    r.b = (int)b;
    r.pix = (long long)p;
  } else {
    r.c = (int)(i % cv) * V;
    r.pix = i / cv;
    r.x = (int)(r.pix % W);
    r.y = (int)((r.pix / W) % H);
    r.b = (int)(r.pix / ((long long)W * H));
  }
  return r;
}
// V per-channel parameters starting at channel c (16-byte aligned when V is a multiple of 4: checked at the launch)
template <int V>
__device__ __forceinline__ void ld_params(const float* __restrict__ p, int c, float dflt, float* o) {
  if (!p) {
#pragma unroll
    for (int q = 0; q < V; ++q) o[q] = dflt;
  } else if (V % 4 == 0) {
#pragma unroll
    for (int q = 0; q < V; q += 4) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(p + c + q));
      o[q] = t.x, o[q + 1] = t.y, o[q + 2] = t.z, o[q + 3] = t.w;
    }
  } else {
#pragma unroll
    for (int q = 0; q < V; ++q) o[q] = __ldg(p + c + q);
  }
}

// ---- max pool, TF SAME (a4) -------------------------------------------------
template <typename T, int V>
__global__ void maxpool_kernel(const T* __restrict__ in, T* __restrict__ out, int B, int H, int W,
                               int OH, int OW, int C, int ld, int k, int stride, int pt, int pl,
                               int ih, int oh) {
  pdl_launch_dependents();
  // ih / oh: 1-pixel halo of the stored input / output tensor (0 or 1)
  const int IW = W + 2 * ih, IH = H + 2 * ih, PW = OW + 2 * oh, PH = OH + 2 * oh;
  const int cv = C / V;
  const long long total = (long long)B * OH * OW * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % cv) * V;
    long long pix = i / cv;
    int ox = (int)(pix % OW);
    int oy = (int)((pix / OW) % OH);
    int b = (int)(pix / ((long long)OW * OH));
    float m[V];
#pragma unroll
    for (int q = 0; q < V; ++q) m[q] = -INFINITY;
    for (int r = 0; r < k; ++r) {
      int iy = oy * stride - pt + r;
      if (iy < 0 || iy >= H) continue;
      for (int s = 0; s < k; ++s) {
        int ix = ox * stride - pl + s;
        if (ix < 0 || ix >= W) continue;
        float v[V];
        VecIO<T, V>::ld(in + (((long long)b * IH + iy + ih) * IW + ix + ih) * ld + c, v);
#pragma unroll
        for (int q = 0; q < V; ++q) m[q] = fmaxf(m[q], v[q]);
      }
    }
    VecIO<T, V>::st(out + (((long long)b * PH + oy + oh) * PW + ox + oh) * ld + c, m);
  }
}

// The two pooling shapes of the SSD backbones (2x2 / stride 2 and 3x3 / stride 1, SSD300.py:539-547) on fp16 tensors
// with 8-channel vectors: compile-time window, 32-bit index arithmetic, no bounds branches (a tap that falls into the
// SAME padding is clamped onto the nearest valid row / column, which lies inside the same window, so the maximum is
// unchanged) and all K*K 16-byte loads of a thread in flight before the first __hmax2.  Bit-identical to
// maxpool_kernel (max is exact in fp16); 1.5-2x faster: the generic kernel spends four 64-bit divisions per output
// and issues its loads one dependent iteration at a time.
template <int K, int S>
__global__ void __launch_bounds__(256)
    maxpool_h8_kernel(const __half* __restrict__ in, __half* __restrict__ out, int total, int H, int W, int OH, int OW,
                      int cv, int ld, int pt, int pl, int ih, int oh) {
  pdl_launch_dependents();
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= total) return;
  const int IW = W + 2 * ih, IH = H + 2 * ih, PW = OW + 2 * oh, PH = OH + 2 * oh;
  const int pix = i / cv, c = (i - pix * cv) * 8;
  const int row = pix / OW, ox = pix - row * OW;
  const int b = row / OH, oy = row - b * OH;
  uint4 v[K * K];
#pragma unroll
  for (int r = 0; r < K; ++r) {
    const int iy = min(max(oy * S - pt + r, 0), H - 1);
#pragma unroll
    for (int q = 0; q < K; ++q) {
      const int ix = min(max(ox * S - pl + q, 0), W - 1);
      v[r * K + q] = __ldg(reinterpret_cast<const uint4*>(in + ((long long)(b * IH + iy + ih) * IW + ix + ih) * ld + c));
    }
  }
  uint4 m = v[0];
  __half2* mh = reinterpret_cast<__half2*>(&m);
#pragma unroll
  for (int t = 1; t < K * K; ++t) {
    const __half2* h = reinterpret_cast<const __half2*>(&v[t]);
#pragma unroll
    for (int j = 0; j < 4; ++j) mh[j] = __hmax2(mh[j], h[j]);
  }
  *reinterpret_cast<uint4*>(out + ((long long)(b * PH + oy + oh) * PW + ox + oh) * ld + c) = m;
}

// max pool + up to two per-channel affine+activation outputs of the pooled value (RetinaNet / FCOS: the pooled stem
// feeds the two pre-activation BN+ReLU of block1_unit1, RetinaNet.py:594-597,634-643): one pass instead of three.
// `out` (the raw pooled tensor) may be NULL; out1 / out2 are dense [B][OH][OW][ld].
template <typename T, int V>
__global__ void maxpool_affine_kernel(const T* __restrict__ in, T* __restrict__ out, int B, int H, int W,
                                      int OH, int OW, int C, int ld, int k, int stride, int pt, int pl,
                                      int ih, int oh, const float* __restrict__ s1, const float* __restrict__ h1,
                                      int act1, T* __restrict__ out1, int halo1, const float* __restrict__ s2,
                                      const float* __restrict__ h2, int act2, T* __restrict__ out2, int halo2) {
  pdl_launch_dependents();
  const int IW = W + 2 * ih, IH = H + 2 * ih, PW = OW + 2 * oh, PH = OH + 2 * oh;
  const int cv = C / V;
  const long long total = (long long)B * OH * OW * cv;
  const bool small = total < (1ll << 31);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const PixelIndex ix0 = split_index<V>(i, cv, OW, OH, small);
    const int c = ix0.c, ox = ix0.x, oy = ix0.y, b = ix0.b;
    const long long pix = ix0.pix;
    float m[V];
#pragma unroll
    for (int q = 0; q < V; ++q) m[q] = -INFINITY;
    for (int r = 0; r < k; ++r) {
      int iy = oy * stride - pt + r;
      if (iy < 0 || iy >= H) continue;
      for (int s = 0; s < k; ++s) {
        int ix = ox * stride - pl + s;
        if (ix < 0 || ix >= W) continue;
        float v[V];
        VecIO<T, V>::ld(in + (((long long)b * IH + iy + ih) * IW + ix + ih) * ld + c, v);
#pragma unroll
        for (int q = 0; q < V; ++q) m[q] = fmaxf(m[q], v[q]);
      }
    }
    if (out) VecIO<T, V>::st(out + (((long long)b * PH + oy + oh) * PW + ox + oh) * ld + c, m);
    // (the maximum of stored values is itself a stored value: no rounding between the pool and the affine)
    if (out1) {
      float v[V], sc[V], sh[V];
      ld_params<V>(s1, c, 1.f, sc);
      ld_params<V>(h1, c, 0.f, sh);
#pragma unroll
      for (int q = 0; q < V; ++q) v[q] = apply_act(fmaf(m[q], sc[q], sh[q]), act1);
      const long long o = halo1 ? ((long long)b * (OH + 2) + oy + 1) * (OW + 2) + ox + 1 : pix;
      VecIO<T, V>::st(out1 + o * ld + c, v);
    }
    if (out2) {
      float v[V], sc[V], sh[V];
      ld_params<V>(s2, c, 1.f, sc);
      ld_params<V>(h2, c, 0.f, sh);
#pragma unroll
      for (int q = 0; q < V; ++q) v[q] = apply_act(fmaf(m[q], sc[q], sh[q]), act2);
      const long long o = halo2 ? ((long long)b * (OH + 2) + oy + 1) * (OW + 2) + ox + 1 : pix;
      VecIO<T, V>::st(out2 + o * ld + c, v);
    }
  }
}

// ---- conv4_3 L2 normalisation x learned scale (a5) -------------------------
template <typename T>
__global__ void l2norm_kernel(const T* __restrict__ in, T* __restrict__ out, long long pixels,
                              int C, int ld, float gamma) {
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long p = warp; p < pixels; p += nwarps) {
    const T* s = in + p * ld;
    float acc = 0.f;
    for (int c = lane; c < C; c += 32) {
      float v = Elem<T>::ld(s + c);
      acc = fmaf(v, v, acc);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    float rs = __frsqrt_rn(fmaxf(acc, 1e-12f));
    T* d = out + p * ld;
    for (int c = lane; c < C; c += 32)
      Elem<T>::st(d + c, __fmul_rn(gamma, __fmul_rn(Elem<T>::ld(s + c), rs)));
  }
}

// ---- y = act(x*scale[c]+shift[c]) ------------------------------------------
template <typename T, int V>
__global__ void affine_act_kernel(const T* __restrict__ in, T* __restrict__ out, long long pixels,
                                  int C, int ld, const float* __restrict__ scale,
                                  const float* __restrict__ shift, int act) {
  pdl_launch_dependents();
  const int cv = C / V;
  const long long total = pixels * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % cv) * V;
    long long p = i / cv;
    float v[V];
    VecIO<T, V>::ld(in + p * ld + c, v);
#pragma unroll
    for (int q = 0; q < V; ++q) {
      float sc = scale ? __ldg(scale + c + q) : 1.f;
      float sh = shift ? __ldg(shift + c + q) : 0.f;
      v[q] = apply_act(fmaf(v[q], sc, sh), act);
    }
    VecIO<T, V>::st(out + p * ld + c, v);
  }
}

// ---- FPN: out = a + legacy bilinear(top) (a16) ------------------------------
template <typename T, int V>
__global__ void upsample_bilinear_add_kernel(const T* __restrict__ top, const T* __restrict__ a,
                                             T* __restrict__ out, int B, int TH, int TW, int H,
                                             int W, int C, int ld, float hs, float ws,
                                             const float* __restrict__ scale2,
                                             const float* __restrict__ shift2, int act2,
                                             T* __restrict__ out1) {
  pdl_launch_dependents();
  const int cv = C / V;
  const long long total = (long long)B * H * W * cv;
  const bool small = total < (1ll << 31);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const PixelIndex ix0 = split_index<V>(i, cv, W, H, small);
    const int c = ix0.c, x = ix0.x, y = ix0.y, b = ix0.b;
    const long long pix = ix0.pix;
    // TF1 resize_bilinear, align_corners=False: src = dst*scale (App. A.6)
    float sy = __fmul_rn((float)y, hs), sx = __fmul_rn((float)x, ws);
    int y0 = (int)floorf(sy), x0 = (int)floorf(sx);
    int y1 = min((int)ceilf(sy), TH - 1), x1 = min((int)ceilf(sx), TW - 1);
    float ly = __fsub_rn(sy, (float)y0), lx = __fsub_rn(sx, (float)x0);
    float tl[V], tr[V], bl[V], br[V], av[V], o[V];
    const T* tb = top + (long long)b * TH * TW * ld + c;
    VecIO<T, V>::ld(tb + ((long long)y0 * TW + x0) * ld, tl);
    VecIO<T, V>::ld(tb + ((long long)y0 * TW + x1) * ld, tr);
    VecIO<T, V>::ld(tb + ((long long)y1 * TW + x0) * ld, bl);
    VecIO<T, V>::ld(tb + ((long long)y1 * TW + x1) * ld, br);
    VecIO<T, V>::ld(a + pix * ld + c, av);
#pragma unroll
    for (int q = 0; q < V; ++q) {
      float t = __fadd_rn(tl[q], __fmul_rn(__fsub_rn(tr[q], tl[q]), lx));
      float bt = __fadd_rn(bl[q], __fmul_rn(__fsub_rn(br[q], bl[q]), lx));
      float r = __fadd_rn(t, __fmul_rn(__fsub_rn(bt, t), ly));
      o[q] = __fadd_rn(av[q], r);
    }
    VecIO<T, V>::st(out + pix * ld + c, o);
    if (out1) {
      float sc[V], sh[V];
      ld_params<V>(scale2, c, 1.f, sc);
      ld_params<V>(shift2, c, 0.f, sh);
#pragma unroll
      for (int q = 0; q < V; ++q) {
        // the consumer sees the stored (rounded) sum: round in registers instead of reading the element back
        const float stored = sizeof(T) == 2 ? __half2float(__float2half_rn(o[q])) : o[q];
        o[q] = apply_act(fmaf(stored, sc[q], sh[q]), act2);
      }
      VecIO<T, V>::st(out1 + pix * ld + c, o);
    }
  }
}

// ---- YOLOv3: concat([a, nearest(b)]) (a18) ----------------------------------
template <typename T, int V>
__global__ void upsample_nearest_concat_kernel(const T* __restrict__ a, const T* __restrict__ bsrc,
                                               T* __restrict__ out, int B, int H, int W, int Ca,
                                               int lda, int BH, int BW, int Cb, int ldb, int ldo,
                                               float hs, float ws) {
  pdl_launch_dependents();
  const int cv = (Ca + Cb) / V;
  const long long total = (long long)B * H * W * cv;
  const bool small = total < (1ll << 31);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const PixelIndex ix0 = split_index<V>(i, cv, W, H, small);
    const int c = ix0.c, x = ix0.x, y = ix0.y, b = ix0.b;
    const long long pix = ix0.pix;
    float v[V];
    if (c < Ca) {
      VecIO<T, V>::ld(a + pix * lda + c, v);
    } else {
      int sy = min((int)floorf(__fmul_rn((float)y, hs)), BH - 1);
      int sx = min((int)floorf(__fmul_rn((float)x, ws)), BW - 1);
      VecIO<T, V>::ld(bsrc + (((long long)b * BH + sy) * BW + sx) * ldb + (c - Ca), v);
    }
    VecIO<T, V>::st(out + pix * ldo + c, v);
  }
}

// ---- GroupNorm (a19) --------------------------------------------------------
// stats[b][g] = (mean, rsqrt(var+eps)); two-pass like tf.nn.moments.
template <typename T>
__global__ void groupnorm_stats_kernel(const T* __restrict__ in, float* __restrict__ stats,
                                       long long hw, int C, int ld, int groups, float eps) {
  pdl_launch_dependents();
  const int g = blockIdx.x, b = blockIdx.y;
  const int cpg = C / groups;
  const T* base = in + (long long)b * hw * ld + g * cpg;
  const long long n = hw * cpg;
  __shared__ float red[32], red2[32];
  __shared__ float s_mean;
  float acc = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x)
    acc += Elem<T>::ld(base + (i / cpg) * ld + (i % cpg));
#pragma unroll
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) s_mean = v / (float)n;
  }
  __syncthreads();
  const float mean = s_mean;
  // sum (x - mean)^2 and sum (x - mean): the second corrects for the rounding of `mean` (corrected two-pass)
  acc = 0.f;
  float accd = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    float d = Elem<T>::ld(base + (i / cpg) * ld + (i % cpg)) - mean;
    accd += d;
    acc = fmaf(d, d, acc);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
    accd += __shfl_xor_sync(0xffffffffu, accd, o);
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  if ((threadIdx.x & 31) == 0) red2[threadIdx.x >> 5] = accd;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    float vd = threadIdx.x < (blockDim.x >> 5) ? red2[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      v += __shfl_xor_sync(0xffffffffu, v, o);
      vd += __shfl_xor_sync(0xffffffffu, vd, o);
    }
    if (threadIdx.x == 0) {
      const double sd = vd, m2 = (double)v - sd * sd / (double)n;
      const float var = (float)(m2 > 0.0 ? m2 / (double)n : 0.0);
      stats[((long long)b * groups + g) * 2 + 0] = (float)((double)mean + sd / (double)n);
      stats[((long long)b * groups + g) * 2 + 1] = __frsqrt_rn(var + eps);
    }
  }
}

// Statistics of the two-launch path (odt_groupnorm_act), fixed-order and batch-invariant.  Every image is cut into
// slices of kGnThreads * kGnSliceVecs channel vectors (the partition depends on hw and C only, never on B); one CTA per
// (slice, image).  A thread owns one channel vector (so its group(s) are fixed) and kGnSliceVecs pixels, kept in
// registers; the slice is reduced twice in a fixed order, no float atomics: the slice mean m, then sum (x - m)^2 and
// sum (x - m) (which corrects for the rounding of m), giving (mean_s, M2_s) per group in fp64, stored to the slice's
// slot.  The last CTA of an image to arrive (threadfence + an integer counter, which it resets) merges the image's
// slots in a fixed order in fp64 about the first slice's mean, and writes (mean, rstd) for groupnorm_apply_kernel.
constexpr int kGnThreads = 256, kGnSliceVecs = 8, kGnMaxGroups = 64;

// pixels per slice for C channels in vectors of V
static inline long long gn_slice_pixels(int C, int V) { return (long long)(kGnThreads / (C / V)) * kGnSliceVecs; }

// GPV: groups per channel vector (1 when a group spans whole vectors)
template <typename T, int V, int GPV>
__global__ void __launch_bounds__(kGnThreads)
    groupnorm_slice_kernel(const T* __restrict__ in, double* __restrict__ slots, float* __restrict__ stats,
                           unsigned* __restrict__ arrivals, long long hw, int C, int ld, int groups, int pps,
                           float eps) {
  pdl_launch_dependents();
  constexpr int NG = GPV, QPG = V / GPV;  // (QPG: channels of one group in a vector when GPV > 1)
  __shared__ float s_a[kGnThreads][NG], s_b[kGnThreads][NG];
  __shared__ double s_mean[kGnMaxGroups];
  __shared__ double s_m[kGnThreads][2];
  __shared__ bool s_last;
  const int S = gridDim.x, s = blockIdx.x, b = blockIdx.y;
  const int cv = C / V, cpg = C / groups;
  const int cvi = threadIdx.x % cv, pl = threadIdx.x / cv, pstep = kGnThreads / cv;
  const long long p0 = (long long)s * pps, p1 = min(hw, p0 + pps);
  const T* base = in + (long long)b * hw * ld + cvi * V;
  uint4 raw[kGnSliceVecs];
  int nv = 0;  // valid pixels of this thread: a prefix of j
#pragma unroll
  for (int j = 0; j < kGnSliceVecs; ++j) {
    const long long p = p0 + pl + (long long)j * pstep;
    if (p < p1) {
      raw[j] = __ldg(reinterpret_cast<const uint4*>(base + p * ld));
      nv = j + 1;
    }
  }
  // pass 1: slice mean per group
  float acc[NG], acc2[NG];
#pragma unroll
  for (int q = 0; q < NG; ++q) acc[q] = 0.f;
#pragma unroll
  for (int j = 0; j < kGnSliceVecs; ++j) {
    if (j < nv) {
      float v[V];
      VecIO<T, V>::ld(reinterpret_cast<const T*>(&raw[j]), v);
#pragma unroll
      for (int q = 0; q < V; ++q) acc[GPV == 1 ? 0 : q / QPG] += v[q];
    }
  }
#pragma unroll
  for (int q = 0; q < NG; ++q) s_a[threadIdx.x][q] = acc[q];
  __syncthreads();
  // the threads of group g, in a fixed order: (pixel lane, channel vector[, group within the vector])
  const int vpg = GPV == 1 ? cpg / V : 1;
  const double n_s = (double)(p1 - p0) * cpg;
  if (threadIdx.x < groups) {
    const int g = threadIdx.x;
    const int c0 = GPV == 1 ? g * vpg : g / GPV, gq = GPV == 1 ? 0 : g % GPV;
    double a = 0.0;
    for (int l = 0; l < pstep; ++l)
      for (int k = 0; k < vpg; ++k) a += s_a[l * cv + c0 + k][gq];
    s_mean[g] = a / n_s;
  }
  __syncthreads();
  // pass 2 (from registers): sum (x - m) and sum (x - m)^2 about the fp32 slice mean m
  const int g0 = cvi * V / cpg;
  float m[NG];
#pragma unroll
  for (int q = 0; q < NG; ++q) {
    m[q] = (float)s_mean[g0 + q];
    acc[q] = acc2[q] = 0.f;
  }
#pragma unroll
  for (int j = 0; j < kGnSliceVecs; ++j) {
    if (j < nv) {
      float v[V];
      VecIO<T, V>::ld(reinterpret_cast<const T*>(&raw[j]), v);
#pragma unroll
      for (int q = 0; q < V; ++q) {
        const int gl = GPV == 1 ? 0 : q / QPG;
        const float d = v[q] - m[gl];
        acc[gl] += d;
        acc2[gl] = fmaf(d, d, acc2[gl]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < NG; ++q) {
    s_a[threadIdx.x][q] = acc[q];
    s_b[threadIdx.x][q] = acc2[q];
  }
  __syncthreads();
  if (threadIdx.x < groups) {
    const int g = threadIdx.x;
    const int c0 = GPV == 1 ? g * vpg : g / GPV, gq = GPV == 1 ? 0 : g % GPV;
    double sd = 0.0, sq = 0.0;
    for (int l = 0; l < pstep; ++l)
      for (int k = 0; k < vpg; ++k) {
        sd += s_a[l * cv + c0 + k][gq];
        sq += s_b[l * cv + c0 + k][gq];
      }
    const double m2 = sq - sd * sd / n_s;
    double* slot = slots + (((long long)b * S + s) * groups + g) * 2;
    slot[0] = (double)(float)s_mean[g] + sd / n_s;
    slot[1] = m2 > 0.0 ? m2 : 0.0;
  }
  // the last CTA of this image merges its S slots
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(arrivals + b, 1u) == (unsigned)S - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int L = kGnThreads / groups;  // lanes per group; lane l takes slices l, l + L, ...
  const int g = threadIdx.x % groups, l = threadIdx.x / groups;
  const double* sl = slots + (long long)b * S * groups * 2;
  const double K = __ldcg(sl + g * 2);  // shift: the first slice's mean
  if (l < L) {
    double A = 0.0, Q = 0.0;
    for (int t = l; t < S; t += L) {
      const double mt = __ldcg(sl + ((long long)t * groups + g) * 2), m2t = __ldcg(sl + ((long long)t * groups + g) * 2 + 1);
      const long long q0 = (long long)t * pps;
      const double nt = (double)(min(hw, q0 + pps) - q0) * cpg, d = mt - K;
      A = fma(nt, d, A);
      Q += fma(nt * d, d, m2t);
    }
    s_m[threadIdx.x][0] = A;
    s_m[threadIdx.x][1] = Q;
  }
  __syncthreads();
  if (threadIdx.x < groups) {
    double A = 0.0, Q = 0.0;
    for (int k = 0; k < L; ++k) {
      A += s_m[k * groups + g][0];
      Q += s_m[k * groups + g][1];
    }
    const double N = (double)hw * cpg;
    // sum over the image of (x - mean)^2 = Q - N (mean - K)^2, with N (mean - K) = A
    const double m2 = Q - A * A / N, var = m2 > 0.0 ? m2 / N : 0.0;
    stats[((long long)b * groups + g) * 2] = (float)(K + A / N);
    stats[((long long)b * groups + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
  if (threadIdx.x == 0) arrivals[b] = 0u;
}

template <typename T, int V>
__global__ void groupnorm_apply_kernel(const T* __restrict__ in, T* __restrict__ out,
                                       const float* __restrict__ stats, int B, long long hw, int C,
                                       int ld, int groups, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, int act) {
  pdl_launch_dependents();
  const int cv = C / V;
  const int cpg = C / groups;
  const long long total = (long long)B * hw * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % cv) * V;
    long long pix = i / cv;
    int b = (int)(pix / hw);
    float v[V];
    VecIO<T, V>::ld(in + pix * ld + c, v);
#pragma unroll
    for (int q = 0; q < V; ++q) {
      int g = (c + q) / cpg;
      float mean = __ldg(stats + ((long long)b * groups + g) * 2);
      float rstd = __ldg(stats + ((long long)b * groups + g) * 2 + 1);
      // tf.contrib group_norm: gain = rstd*gamma; offset = -mean*gain + beta
      float gm = gamma ? __ldg(gamma + c + q) : 1.f;
      float bt = beta ? __ldg(beta + c + q) : 0.f;
      float gain = __fmul_rn(rstd, gm);
      float off = __fadd_rn(__fmul_rn(-mean, gain), bt);
      v[q] = apply_act(__fadd_rn(__fmul_rn(v[q], gain), off), act);
    }
    VecIO<T, V>::st(out + pix * ld + c, v);
  }
}

// apply of the two-launch path: every block first copies the (mean, rstd) of all (image, group) pairs that
// groupnorm_slice_kernel wrote into shared memory
template <typename T, int V>
__global__ void __launch_bounds__(256)
    groupnorm_apply_acc_kernel(const T* __restrict__ in, T* __restrict__ out, const float* __restrict__ stats,
                               int B, long long hw, int C, int ld, int groups,
                               const float* __restrict__ gamma, const float* __restrict__ beta, int act) {
  pdl_launch_dependents();
  extern __shared__ float s_stat[];  // [B*groups][2]
  for (int i = threadIdx.x; i < B * groups * 2; i += blockDim.x) s_stat[i] = stats[i];
  __syncthreads();
  const int cv = C / V;
  const int cpg = C / groups;
  const long long total = (long long)B * hw * cv;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * V;
    const long long pix = i / cv;
    const int b = (int)(pix / hw);
    float v[V];
    VecIO<T, V>::ld(in + pix * ld + c, v);
#pragma unroll
    for (int q = 0; q < V; ++q) {
      const int g = (c + q) / cpg;
      const float mean = s_stat[(b * groups + g) * 2], rstd = s_stat[(b * groups + g) * 2 + 1];
      const float gm = gamma ? __ldg(gamma + c + q) : 1.f;
      const float bt = beta ? __ldg(beta + c + q) : 0.f;
      const float gain = __fmul_rn(rstd, gm);
      const float off = __fadd_rn(__fmul_rn(-mean, gain), bt);
      v[q] = apply_act(__fadd_rn(__fmul_rn(v[q], gain), off), act);
    }
    VecIO<T, V>::st(out + pix * ld + c, v);
  }
}

}  // namespace odt

using namespace odt;

#define DISPATCH_DTYPE(dtype, ...)              \
  if ((dtype) == ODT_F16) {                     \
    using T = __half;                           \
    __VA_ARGS__                                 \
  } else if ((dtype) == ODT_F32) {              \
    using T = float;                            \
    __VA_ARGS__                                 \
  } else {                                      \
    odt::set_error("%s: bad dtype", __func__);  \
    return ODT_ERR_INVALID;                     \
  }

extern "C" int odt_normalize_input(const float* images, void* out, int out_dtype, int B, int H,
                                   int W, int out_ld, const float* mean3_host, void* stream) {
  ODT_CHECK_ARG(images && out && mean3_host && B > 0 && H > 0 && W > 0 && out_ld >= 3, "args");
  cudaStream_t st = (cudaStream_t)stream;
  long long pixels = (long long)B * H * W;
  DISPATCH_DTYPE(out_dtype, {
    normalize_kernel<T><<<grid_for(pixels, 256), 256, 0, st>>>(
        images, (T*)out, pixels, out_ld, mean3_host[0], mean3_host[1], mean3_host[2]);
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_pack_input_rgbx(const float* images, void* out_f16, int B, int H, int W, int pad,
                                   const float* mean3_host, void* stream) {
  ODT_CHECK_ARG(images && out_f16 && mean3_host && B > 0 && H > 0 && W > 0 && pad >= 0 && pad <= 8, "args");
  ODT_CHECK_ARG(((uintptr_t)out_f16 & 15) == 0, "out must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int vec = ((W & 3) == 0 && ((uintptr_t)images & 15) == 0) ? 1 : 0;
  const long long work = (long long)B * H * (vec ? W / 4 : W);
  pack_rgbx_kernel<<<grid_for(work, 256), 256, 0, st>>>(images, (__half*)out_f16, B, H, W, pad, mean3_host[0],
                                                        mean3_host[1], mean3_host[2], vec);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_maxpool(const void* in, void* out, int dtype, int B, int H, int W, int C,
                           int ld, int k, int stride, int in_halo, int out_halo, void* stream) {
  ODT_CHECK_ARG(in && out && B > 0 && H > 0 && W > 0 && C > 0 && ld >= C && k > 0 && stride > 0,
                "args");
  ODT_CHECK_ARG((in_halo == 0 || in_halo == 1) && (out_halo == 0 || out_halo == 1), "halo must be 0/1");
  int OH, OW, pt, pl, pa;
  odt_same_pad(H, k, stride, 1, &OH, &pt, &pa);
  odt_same_pad(W, k, stride, 1, &OW, &pl, &pa);
  cudaStream_t st = (cudaStream_t)stream;
  {
    const long long work = (long long)B * OH * OW * (C / 8);
    const bool shape = (k == 2 && stride == 2) || (k == 3 && stride == 1);
    if (dtype == ODT_F16 && shape && can_vec(in, out, C, ld, 8, 2) && work < (1ll << 31) - 256 &&
        (long long)B * (H + 2) * (W + 2) < (1ll << 31)) {
      const int blocks = (int)((work + 255) / 256);
      const __half* ip = (const __half*)in;
      __half* op = (__half*)out;
      if (k == 2)
        maxpool_h8_kernel<2, 2><<<blocks, 256, 0, st>>>(ip, op, (int)work, H, W, OH, OW, C / 8, ld, pt, pl, in_halo, out_halo);
      else
        maxpool_h8_kernel<3, 1><<<blocks, 256, 0, st>>>(ip, op, (int)work, H, W, OH, OW, C / 8, ld, pt, pl, in_halo, out_halo);
      ODT_LAUNCH_OK();
      return ODT_OK;
    }
  }
  DISPATCH_DTYPE(dtype, {
    constexpr int V = FullVec<T>::V;
    if (can_vec(in, out, C, ld, V, sizeof(T))) {
      long long work = (long long)B * OH * OW * (C / V);
      maxpool_kernel<T, V><<<grid_for(work, 256), 256, 0, st>>>((const T*)in, (T*)out, B, H, W, OH,
                                                               OW, C, ld, k, stride, pt, pl, in_halo, out_halo);
    } else {
      long long work = (long long)B * OH * OW * C;
      maxpool_kernel<T, 1><<<grid_for(work, 256), 256, 0, st>>>((const T*)in, (T*)out, B, H, W, OH,
                                                               OW, C, ld, k, stride, pt, pl, in_halo, out_halo);
    }
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_maxpool_affine(const void* in, void* out, int dtype, int B, int H, int W, int C, int ld, int k,
                                  int stride, int in_halo, int out_halo, const float* scale1, const float* shift1,
                                  int act1, void* out1, int out1_halo, const float* scale2, const float* shift2,
                                  int act2, void* out2, int out2_halo, void* stream) {
  ODT_CHECK_ARG(in && (out || out1 || out2) && B > 0 && H > 0 && W > 0 && C > 0 && ld >= C && k > 0 && stride > 0,
                "args");
  ODT_CHECK_ARG((in_halo == 0 || in_halo == 1) && (out_halo == 0 || out_halo == 1), "halo must be 0/1");
  ODT_CHECK_ARG(act1 >= 0 && act1 <= 2 && act2 >= 0 && act2 <= 2, "activation code");
  ODT_CHECK_ARG((out1_halo == 0 || out1_halo == 1) && (out2_halo == 0 || out2_halo == 1), "out halo must be 0/1");
  int OH, OW, pt, pl, pa;
  odt_same_pad(H, k, stride, 1, &OH, &pt, &pa);
  odt_same_pad(W, k, stride, 1, &OW, &pl, &pa);
  cudaStream_t st = (cudaStream_t)stream;
  DISPATCH_DTYPE(dtype, {
    constexpr int V = FullVec<T>::V;
    const bool vec = can_vec(in, out ? out : in, C, ld, V, sizeof(T)) && ((uintptr_t)out1 % 16) == 0 &&
                     ((uintptr_t)out2 % 16) == 0 &&
                     (((uintptr_t)scale1 | (uintptr_t)shift1 | (uintptr_t)scale2 | (uintptr_t)shift2) & 15) == 0;
    if (vec) {
      long long work = (long long)B * OH * OW * (C / V);
      maxpool_affine_kernel<T, V><<<grid_for(work, 256), 256, 0, st>>>(
          (const T*)in, (T*)out, B, H, W, OH, OW, C, ld, k, stride, pt, pl, in_halo, out_halo, scale1, shift1, act1,
          (T*)out1, out1_halo, scale2, shift2, act2, (T*)out2, out2_halo);
    } else {
      long long work = (long long)B * OH * OW * C;
      maxpool_affine_kernel<T, 1><<<grid_for(work, 256), 256, 0, st>>>(
          (const T*)in, (T*)out, B, H, W, OH, OW, C, ld, k, stride, pt, pl, in_halo, out_halo, scale1, shift1, act1,
          (T*)out1, out1_halo, scale2, shift2, act2, (T*)out2, out2_halo);
    }
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_l2norm_scale(const void* in, void* out, int dtype, long long pixels, int C,
                                int ld, float gamma, void* stream) {
  ODT_CHECK_ARG(in && out && pixels > 0 && C > 0 && ld >= C, "args");
  cudaStream_t st = (cudaStream_t)stream;
  DISPATCH_DTYPE(dtype, {
    l2norm_kernel<T><<<grid_for(pixels * 32, 256), 256, 0, st>>>((const T*)in, (T*)out, pixels, C,
                                                               ld, gamma);
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_affine_act(const void* in, void* out, int dtype, long long pixels, int C, int ld,
                              const float* scale, const float* shift, int act, void* stream) {
  ODT_CHECK_ARG(in && out && pixels > 0 && C > 0 && ld >= C, "args");
  cudaStream_t st = (cudaStream_t)stream;
  DISPATCH_DTYPE(dtype, {
    constexpr int V = FullVec<T>::V;
    if (can_vec(in, out, C, ld, V, sizeof(T))) {
      affine_act_kernel<T, V><<<grid_for(pixels * (C / V), 256), 256, 0, st>>>(
          (const T*)in, (T*)out, pixels, C, ld, scale, shift, act);
    } else {
      affine_act_kernel<T, 1><<<grid_for(pixels * C, 256), 256, 0, st>>>(
          (const T*)in, (T*)out, pixels, C, ld, scale, shift, act);
    }
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_upsample_bilinear_add(const void* top, const void* a, void* out, int dtype,
                                         int B, int TH, int TW, int H, int W, int C, int ld,
                                         const float* scale2, const float* shift2, int act2,
                                         void* out1, void* stream) {
  ODT_CHECK_ARG(top && a && out && B > 0 && TH > 0 && TW > 0 && H > 0 && W > 0 && C > 0 && ld >= C,
                "args");
  cudaStream_t st = (cudaStream_t)stream;
  float hs = (float)TH / (float)H, ws = (float)TW / (float)W;
  DISPATCH_DTYPE(dtype, {
    constexpr int V = FullVec<T>::V;
    bool vec = can_vec(top, a, C, ld, V, sizeof(T)) && can_vec(out, out1 ? out1 : out, C, ld, V, sizeof(T)) &&
               (((uintptr_t)scale2 | (uintptr_t)shift2) & 15) == 0;
    if (vec) {
      long long work = (long long)B * H * W * (C / V);
      upsample_bilinear_add_kernel<T, V><<<grid_for(work, 256), 256, 0, st>>>(
          (const T*)top, (const T*)a, (T*)out, B, TH, TW, H, W, C, ld, hs, ws, scale2, shift2, act2,
          (T*)out1);
    } else {
      long long work = (long long)B * H * W * C;
      upsample_bilinear_add_kernel<T, 1><<<grid_for(work, 256), 256, 0, st>>>(
          (const T*)top, (const T*)a, (T*)out, B, TH, TW, H, W, C, ld, hs, ws, scale2, shift2, act2,
          (T*)out1);
    }
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_upsample_nearest_concat(const void* a, const void* b, void* out, int dtype,
                                           int B, int H, int W, int Ca, int lda, int BH, int BW,
                                           int Cb, int ldb, int ldo, void* stream) {
  ODT_CHECK_ARG(a && b && out && B > 0 && H > 0 && W > 0 && Ca > 0 && Cb > 0 && lda >= Ca &&
                    ldb >= Cb && ldo >= Ca + Cb,
                "args");
  cudaStream_t st = (cudaStream_t)stream;
  float hs = (float)BH / (float)H, ws = (float)BW / (float)W;
  DISPATCH_DTYPE(dtype, {
    constexpr int V = FullVec<T>::V;
    const bool vec = Ca % V == 0 && Cb % V == 0 && lda % V == 0 && ldb % V == 0 && ldo % V == 0 &&
                     ((uintptr_t)a % 16) == 0 && ((uintptr_t)b % 16) == 0 && ((uintptr_t)out % 16) == 0;
    if (vec) {
      long long work = (long long)B * H * W * ((Ca + Cb) / V);
      upsample_nearest_concat_kernel<T, V><<<grid_for(work, 256), 256, 0, st>>>(
          (const T*)a, (const T*)b, (T*)out, B, H, W, Ca, lda, BH, BW, Cb, ldb, ldo, hs, ws);
    } else {
      long long work = (long long)B * H * W * (Ca + Cb);
      upsample_nearest_concat_kernel<T, 1><<<grid_for(work, 256), 256, 0, st>>>(
          (const T*)a, (const T*)b, (T*)out, B, H, W, Ca, lda, BH, BW, Cb, ldb, ldo, hs, ws);
    }
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_groupnorm_stats(const void* in, float* stats, int dtype, int B, long long hw,
                                   int C, int ld, int groups, float eps, void* stream) {
  ODT_CHECK_ARG(in && stats && B > 0 && B <= 65535 && hw > 0 && C > 0 && ld >= C && groups > 0 && C % groups == 0,
                "args");
  cudaStream_t st = (cudaStream_t)stream;
  DISPATCH_DTYPE(dtype, {
    groupnorm_stats_kernel<T><<<dim3(groups, B), 1024, 0, st>>>((const T*)in, stats, hw, C, ld, groups, eps);
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_groupnorm_apply(const void* in, void* out, const float* stats, int dtype, int B,
                                   long long hw, int C, int ld, int groups, const float* gamma,
                                   const float* beta, int act, void* stream) {
  ODT_CHECK_ARG(in && out && stats && B > 0 && hw > 0 && C > 0 && ld >= C && groups > 0 &&
                    C % groups == 0,
                "args");
  cudaStream_t st = (cudaStream_t)stream;
  DISPATCH_DTYPE(dtype, {
    constexpr int V = FullVec<T>::V;
    if (can_vec(in, out, C, ld, V, sizeof(T))) {
      long long work = (long long)B * hw * (C / V);
      groupnorm_apply_kernel<T, V><<<grid_for(work, 256), 256, 0, st>>>(
          (const T*)in, (T*)out, stats, B, hw, C, ld, groups, gamma, beta, act);
    } else {
      long long work = (long long)B * hw * C;
      groupnorm_apply_kernel<T, 1><<<grid_for(work, 256), 256, 0, st>>>(
          (const T*)in, (T*)out, stats, B, hw, C, ld, groups, gamma, beta, act);
    }
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

// ---- GroupNorm + activation in two launches -----------------------------------
// workspace: slots [B][S][groups] x (mean_s, M2_s) doubles | stats [B][groups] x (mean, rstd) floats | B arrival counters
static bool gn_fused_shape(int V, int B, int C, int groups) {
  return B > 0 && B <= 65535 && C > 0 && groups > 0 && (C & (C - 1)) == 0 && (groups & (groups - 1)) == 0 &&
         C % groups == 0 && C % V == 0 && C / V <= kGnThreads && groups <= kGnMaxGroups &&
         (long long)B * groups * 2 * sizeof(float) <= 48 * 1024;  // the apply kernel's shared-memory copy of the stats
}

static long long gn_slices(long long hw, int C, int V) {
  const long long pps = gn_slice_pixels(C, V);
  return (hw + pps - 1) / pps;
}

static long long gn_workspace_bytes(int V, int B, long long hw, int C, int groups) {
  return (long long)sizeof(double) * B * gn_slices(hw, C, V) * groups * 2 + (long long)sizeof(float) * B * groups * 2 +
         (long long)sizeof(unsigned) * B;
}

extern "C" long long odt_groupnorm_act_workspace_bytes(int dtype, int B, long long hw, int C, int groups) {
  const int V = dtype == ODT_F16 ? FullVec<__half>::V : dtype == ODT_F32 ? FullVec<float>::V : 0;
  if (V == 0 || hw <= 0 || !gn_fused_shape(V, B, C, groups)) return 0;
  return gn_workspace_bytes(V, B, hw, C, groups);
}

template <typename T, int V, int GPV>
static void gn_launch_slices(dim3 grid, cudaStream_t st, const T* in, double* slots, float* stats, unsigned* arrivals,
                             long long hw, int C, int ld, int groups, int pps, float eps) {
  if constexpr (GPV <= V)
    groupnorm_slice_kernel<T, V, GPV><<<grid, kGnThreads, 0, st>>>(in, slots, stats, arrivals, hw, C, ld, groups, pps,
                                                                   eps);
}

extern "C" int odt_groupnorm_act(const void* in, void* out, void* workspace, int dtype, int B, long long hw,
                                 int C, int ld, int groups, float eps, const float* gamma, const float* beta,
                                 int act, void* stream) {
  ODT_CHECK_ARG(in && out && workspace && B > 0 && hw > 0 && C > 0 && ld >= C && groups > 0 && C % groups == 0,
                "args");
  ODT_CHECK_ARG(((uintptr_t)workspace & 7) == 0, "workspace must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ODT_ERR_UNSUPPORTED;
  DISPATCH_DTYPE(dtype, {
    constexpr int V = FullVec<T>::V;
    const bool fast = gn_fused_shape(V, B, C, groups) && ld % V == 0 && ((uintptr_t)in % 16) == 0 &&
                      ((uintptr_t)out % 16) == 0 && gn_slices(hw, C, V) <= 0x7fffffff;
    if (fast) {
      const int cpg = C / groups, gpv = cpg >= V ? 1 : V / cpg;
      const long long S = gn_slices(hw, C, V);
      double* slots = (double*)workspace;
      float* stats = (float*)(slots + (long long)B * S * groups * 2);
      unsigned* arrivals = (unsigned*)(stats + (long long)B * groups * 2);
      const dim3 grid((unsigned)S, (unsigned)B);
      const int pps = (int)gn_slice_pixels(C, V);
      const T* x = (const T*)in;
      if (gpv == 1)
        gn_launch_slices<T, V, 1>(grid, st, x, slots, stats, arrivals, hw, C, ld, groups, pps, eps);
      else if (gpv == 2)
        gn_launch_slices<T, V, 2>(grid, st, x, slots, stats, arrivals, hw, C, ld, groups, pps, eps);
      else if (gpv == 4)
        gn_launch_slices<T, V, 4>(grid, st, x, slots, stats, arrivals, hw, C, ld, groups, pps, eps);
      else
        gn_launch_slices<T, V, 8>(grid, st, x, slots, stats, arrivals, hw, C, ld, groups, pps, eps);
      ODT_LAUNCH_OK();
      const long long work = (long long)B * hw * (C / V);
      groupnorm_apply_acc_kernel<T, V><<<grid_for(work, 256), 256, (size_t)B * groups * 2 * sizeof(float), st>>>(
          x, (T*)out, stats, B, hw, C, ld, groups, gamma, beta, act);
      ODT_LAUNCH_OK();
      rc = ODT_OK;
    }
  })
  if (rc == ODT_ERR_UNSUPPORTED) set_error("odt_groupnorm_act: shape outside the two-launch path (use stats + apply)");
  return rc;
}

// ---- PFPNet-R pyramid glue (ref PFPNetR.py:321-362,413-421) -----------------
// One thread per output element: the channel counts are 85 (an odd width, no vector access) or 256, and the three
// kernels move a few MB per image next to the convolutions around them.
namespace odt {

// The four output phases of a 4x4 / stride-2 SAME conv2d_transpose, computed by one stride-1 3x3 convolution with
// 4 * C output channels (phase p = 2 * py + px major, channel minor), placed on the 2x grid:
// out[b, 2i+py, 2j+px, c] = act(in[b, i, j, p*C + c] (+ res[b, 2i+py, 2j+px, c])).
template <typename T>
__global__ void pixel_shuffle2x_kernel(const T* __restrict__ in, T* __restrict__ out, const T* __restrict__ res,
                                       int B, int h, int w, int C, int in_ld, int out_ld, int res_ld, int act) {
  pdl_launch_dependents();
  const int OH = 2 * h, OW = 2 * w;
  const long long total = (long long)B * OH * OW * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const int ox = (int)(pix % OW);
    const long long t = pix / OW;
    const int oy = (int)(t % OH);
    const int b = (int)(t / OH);
    const int ph = 2 * (oy & 1) + (ox & 1);
    float v = Elem<T>::ld(in + (((long long)b * h + (oy >> 1)) * w + (ox >> 1)) * in_ld + ph * C + c);
    if (res) v = __fadd_rn(v, Elem<T>::ld(res + pix * res_ld + c));
    Elem<T>::st(out + pix * out_ld + c, apply_act(v, act));
  }
}

// tf.image.resize_bilinear(align_corners=True), TF 1.13: src = dst * scale, scale = (in - 1) / (out - 1) in float32
// (0 when out == 1: the only sample is 0 either way), lower = floor, upper = min(ceil, in - 1), lerp = src - lower;
// top = tl + (tr - tl) * lx, bottom = bl + (br - bl) * lx, out = top + (bottom - top) * ly, each step rounded.
// out2: an optional second copy (a concat slice) at its own channel stride.
template <typename T>
__global__ void resize_bilinear_ac_kernel(const T* __restrict__ in, T* __restrict__ out, T* __restrict__ out2,
                                          int B, int H, int W, int C, int in_ld, int OH, int OW, int out_ld,
                                          int out2_ld, float hs, float ws) {
  pdl_launch_dependents();
  const long long total = (long long)B * OH * OW * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const int ox = (int)(pix % OW);
    const long long t = pix / OW;
    const int oy = (int)(t % OH);
    const int b = (int)(t / OH);
    const float sy = __fmul_rn((float)oy, hs), sx = __fmul_rn((float)ox, ws);
    const float fy = floorf(sy), fx = floorf(sx);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = min((int)ceilf(sy), H - 1), x1 = min((int)ceilf(sx), W - 1);
    const float ly = __fsub_rn(sy, fy), lx = __fsub_rn(sx, fx);
    const T* base = in + (long long)b * H * W * in_ld + c;
    const float tl = Elem<T>::ld(base + ((long long)y0 * W + x0) * in_ld);
    const float tr = Elem<T>::ld(base + ((long long)y0 * W + x1) * in_ld);
    const float bl = Elem<T>::ld(base + ((long long)y1 * W + x0) * in_ld);
    const float br = Elem<T>::ld(base + ((long long)y1 * W + x1) * in_ld);
    const float top = __fadd_rn(tl, __fmul_rn(__fsub_rn(tr, tl), lx));
    const float bot = __fadd_rn(bl, __fmul_rn(__fsub_rn(br, bl), lx));
    const float v = __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), ly));
    Elem<T>::st(out + pix * out_ld + c, v);
    if (out2) Elem<T>::st(out2 + pix * out2_ld + c, v);
  }
}

// tf.layers.average_pooling2d(2, 2, 'same'): out = ceil(in / 2), padding only after (odd sizes), and the sum of the
// window cells inside the image -- added in row-major order -- divided by their number, not by 4.
template <typename T>
__global__ void avgpool2x2_same_kernel(const T* __restrict__ in, T* __restrict__ out, int B, int H, int W, int C,
                                       int in_ld, int out_ld) {
  pdl_launch_dependents();
  const int OH = (H + 1) / 2, OW = (W + 1) / 2;
  const long long total = (long long)B * OH * OW * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const int ox = (int)(pix % OW);
    const long long t = pix / OW;
    const int oy = (int)(t % OH);
    const int b = (int)(t / OH);
    const T* base = in + (long long)b * H * W * in_ld + c;
    float s = 0.f;
    int n = 0;
    for (int dy = 0; dy < 2; ++dy) {
      const int y = 2 * oy + dy;
      if (y >= H) break;
      for (int dx = 0; dx < 2; ++dx) {
        const int x = 2 * ox + dx;
        if (x >= W) break;
        s = __fadd_rn(s, Elem<T>::ld(base + ((long long)y * W + x) * in_ld));
        ++n;
      }
    }
    Elem<T>::st(out + pix * out_ld + c, __fdiv_rn(s, (float)n));
  }
}

}  // namespace odt

extern "C" int odt_pixel_shuffle2x(const void* in, void* out, const void* res, int dtype, int B, int h, int w, int C,
                                   int in_ld, int out_ld, int res_ld, int act, void* stream) {
  ODT_CHECK_ARG(in && out && B > 0 && h > 0 && w > 0 && C > 0 && in_ld >= 4 * C && out_ld >= C &&
                    (!res || res_ld >= C) && act >= ODT_ACT_NONE && act <= ODT_ACT_LEAKY,
                "args");
  cudaStream_t st = (cudaStream_t)stream;
  DISPATCH_DTYPE(dtype, {
    pixel_shuffle2x_kernel<T><<<grid_for((long long)B * 4 * h * w * C, 256), 256, 0, st>>>(
        (const T*)in, (T*)out, (const T*)res, B, h, w, C, in_ld, out_ld, res_ld, act);
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_resize_bilinear_ac(const void* in, void* out, void* out2, int dtype, int B, int H, int W, int C,
                                      int in_ld, int OH, int OW, int out_ld, int out2_ld, void* stream) {
  ODT_CHECK_ARG(in && out && B > 0 && H > 0 && W > 0 && C > 0 && OH > 0 && OW > 0 && in_ld >= C && out_ld >= C &&
                    (!out2 || out2_ld >= C),
                "args");
  cudaStream_t st = (cudaStream_t)stream;
  const float hs = OH > 1 ? (float)(H - 1) / (float)(OH - 1) : 0.f;
  const float ws = OW > 1 ? (float)(W - 1) / (float)(OW - 1) : 0.f;
  DISPATCH_DTYPE(dtype, {
    resize_bilinear_ac_kernel<T><<<grid_for((long long)B * OH * OW * C, 256), 256, 0, st>>>(
        (const T*)in, (T*)out, (T*)out2, B, H, W, C, in_ld, OH, OW, out_ld, out2_ld, hs, ws);
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_avgpool2x2_same(const void* in, void* out, int dtype, int B, int H, int W, int C, int in_ld,
                                   int out_ld, void* stream) {
  ODT_CHECK_ARG(in && out && B > 0 && H > 0 && W > 0 && C > 0 && in_ld >= C && out_ld >= C, "args");
  cudaStream_t st = (cudaStream_t)stream;
  DISPATCH_DTYPE(dtype, {
    avgpool2x2_same_kernel<T><<<grid_for((long long)B * ((H + 1) / 2) * ((W + 1) / 2) * C, 256), 256, 0, st>>>(
        (const T*)in, (T*)out, B, H, W, C, in_ld, out_ld);
  })
  ODT_LAUNCH_OK();
  return ODT_OK;
}
