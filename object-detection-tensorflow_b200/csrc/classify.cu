// Classification tail of RetinaNet's ImageNet-pretraining mode (ref RetinaNet.py:120-135): global mean pool of the
// last feature tensor -> fp32 logits, first-maximum class and, optionally, the per-image sparse softmax
// cross-entropy.  One CTA per image; every reduction runs in a fixed order, so replays are bit-identical.
#include <math.h>

#include "common.cuh"

namespace odt {

namespace {

constexpr int kClsThreads = 256;
constexpr int kClsMaxC = 4096;  // logits and per-slice partial sums live in shared memory

template <typename T, int V>
struct ClsLoad;
template <>
struct ClsLoad<float, 1> {
  static __device__ __forceinline__ void ld(const float* p, float* v) { v[0] = *p; }
};
template <>
struct ClsLoad<__half, 1> {
  static __device__ __forceinline__ void ld(const __half* p, float* v) { v[0] = __half2float(*p); }
};
template <>
struct ClsLoad<float, 4> {
  static __device__ __forceinline__ void ld(const float* p, float* v) {
    float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
};
template <>
struct ClsLoad<__half, 8> {
  static __device__ __forceinline__ void ld(const __half* p, float* v) {
    uint4 t = __ldg(reinterpret_cast<const uint4*>(p));
    const __half2* h = reinterpret_cast<const __half2*>(&t);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 f = __half22float2(h[i]);
      v[2 * i] = f.x;
      v[2 * i + 1] = f.y;
    }
  }
};

// (value, index) maximum that keeps the lower index on ties: tf.argmax's first maximum
__device__ __forceinline__ void argmax_merge(float& v, int& i, float ov, int oi) {
  if (ov > v || (ov == v && oi < i)) {
    v = ov;
    i = oi;
  }
}

// feat: [B][H+2h][W+2h][ld], real channels [0, C).  Threads split into `slices` pixel slices x `cols` channel vectors;
// thread (s, col) sums the vectors col, col+cols, ... over the pixels s, s+slices, ... in fp64, and the slice partials
// are added in slice order.  Lanes >= C of the last vector are loaded (16-byte sectors) but never summed.
template <typename T, int V>
__global__ void __launch_bounds__(kClsThreads)
pool_classify_kernel(const T* __restrict__ feat, int H, int W, int C, int ld, int halo, int slices, int cols,
                     float* __restrict__ logits, long long* __restrict__ pred, const long long* __restrict__ labels,
                     float* __restrict__ loss) {
  pdl_launch_dependents();
  extern __shared__ double cls_smem[];
  const int nv = (C + V - 1) / V;
  double* part = cls_smem;                                          // [slices][nv * V]
  float* lg = reinterpret_cast<float*>(cls_smem + (size_t)slices * nv * V);  // [C]
  __shared__ float red_v[kClsThreads / 32];
  __shared__ int red_i[kClsThreads / 32];
  __shared__ double red_d[kClsThreads / 32];

  const int b = blockIdx.x, tid = threadIdx.x;
  const int HW = H * W, Wp = W + 2 * halo;
  const T* img = feat + (size_t)b * (H + 2 * halo) * Wp * ld;
  if (tid < slices * cols) {
    const int s = tid / cols, col = tid % cols;
    for (int v = col; v < nv; v += cols) {
      double acc[V];
#pragma unroll
      for (int q = 0; q < V; ++q) acc[q] = 0.0;
      for (int p = s; p < HW; p += slices) {
        const int y = p / W, x = p - y * W;
        float e[V];
        ClsLoad<T, V>::ld(img + ((size_t)(y + halo) * Wp + (x + halo)) * ld + v * V, e);
#pragma unroll
        for (int q = 0; q < V; ++q)
          if (v * V + q < C) acc[q] += (double)e[q];
      }
#pragma unroll
      for (int q = 0; q < V; ++q) part[(size_t)s * nv * V + v * V + q] = acc[q];
    }
  }
  __syncthreads();

  const float hw = (float)HW;
  float bv = -INFINITY;
  int bi = C;
  for (int c = tid; c < C; c += kClsThreads) {
    double sum = 0.0;
    for (int s = 0; s < slices; ++s) sum += part[(size_t)s * nv * V + c];
    const float m = __fdiv_rn((float)sum, hw);
    lg[c] = m;
    logits[(size_t)b * C + c] = m;
    argmax_merge(bv, bi, m, c);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    argmax_merge(bv, bi, __shfl_xor_sync(0xffffffffu, bv, o), __shfl_xor_sync(0xffffffffu, bi, o));
  if ((tid & 31) == 0) {
    red_v[tid >> 5] = bv;
    red_i[tid >> 5] = bi;
  }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kClsThreads / 32; ++w) argmax_merge(bv, bi, red_v[w], red_i[w]);
    // every logit NaN: no strict maximum exists; report index 0 like a scan that starts there
    red_i[0] = bi < C ? bi : 0;
    pred[b] = red_i[0];
  }
  if (labels == nullptr) return;
  __syncthreads();
  const int am = red_i[0];
  const double mx = (double)lg[am];
  // log(sum_c exp(x_c - max)) = log1p(sum over c != argmax), accurate also when the label's probability is ~1
  double t = 0.0;
  for (int c = tid; c < C; c += kClsThreads)
    if (c != am) t += exp((double)lg[c] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((tid & 31) == 0) red_d[tid >> 5] = t;
  __syncthreads();
  if (tid == 0) {
    double tot = 0.0;
    for (int w = 0; w < kClsThreads / 32; ++w) tot += red_d[w];
    const long long lab = labels[b];
    loss[b] = (lab >= 0 && lab < C) ? (float)(log1p(tot) - ((double)lg[lab] - mx)) : __int_as_float(0x7fc00000);
  }
}

template <typename T, int V>
cudaError_t launch_pool_classify(const T* feat, int B, int H, int W, int C, int ld, int halo, float* logits,
                                 long long* pred, const long long* labels, float* loss, cudaStream_t st) {
  const int nv = (C + V - 1) / V;
  const int cols = nv < kClsThreads ? nv : kClsThreads;
  const int slices = (int)min((long long)(kClsThreads / cols), (long long)H * W);
  const size_t smem = (size_t)slices * nv * V * sizeof(double) + (size_t)C * sizeof(float);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(pool_classify_kernel<T, V>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return e;
  }
  pool_classify_kernel<T, V><<<B, kClsThreads, smem, st>>>(feat, H, W, C, ld, halo, slices, cols, logits, pred,
                                                            labels, loss);
  return cudaGetLastError();
}

}  // namespace

}  // namespace odt

using namespace odt;

extern "C" int odt_pool_classify(const void* feat, int dtype, int B, int H, int W, int C, int ld, int halo,
                                 float* logits, long long* pred, const long long* labels, float* loss, void* stream) {
  ODT_CHECK_ARG(feat && logits && pred && B > 0 && H > 0 && W > 0 && C > 0 && ld >= C, "args");
  ODT_CHECK_ARG(halo == 0 || halo == 1, "halo must be 0/1");
  ODT_CHECK_ARG((labels == nullptr) == (loss == nullptr), "labels and loss go together");
  ODT_CHECK_ARG(C <= kClsMaxC, "C exceeds the shared-memory logit buffer (4096)");
  ODT_CHECK_ARG((long long)H * W < (1ll << 24), "H*W must be exact in fp32");
  cudaStream_t st = (cudaStream_t)stream;
  const bool aligned = ((uintptr_t)feat & 15) == 0;
  cudaError_t e;
  if (dtype == ODT_F16) {
    const __half* f = (const __half*)feat;
    e = (aligned && ld % 8 == 0) ? launch_pool_classify<__half, 8>(f, B, H, W, C, ld, halo, logits, pred, labels, loss, st)
                                 : launch_pool_classify<__half, 1>(f, B, H, W, C, ld, halo, logits, pred, labels, loss, st);
  } else if (dtype == ODT_F32) {
    const float* f = (const float*)feat;
    e = (aligned && ld % 4 == 0) ? launch_pool_classify<float, 4>(f, B, H, W, C, ld, halo, logits, pred, labels, loss, st)
                                 : launch_pool_classify<float, 1>(f, B, H, W, C, ld, halo, logits, pred, labels, loss, st);
  } else {
    odt::set_error("%s: bad dtype", __func__);
    return ODT_ERR_INVALID;
  }
  if (e != cudaSuccess) {
    odt::set_error("%s: launch failed: %s", __func__, cudaGetErrorString(e));
    return ODT_ERR_CUDA;
  }
  return ODT_OK;
}
