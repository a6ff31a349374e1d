// CUDA-core convolution for VERY thin layers (RetinaNet's 7*2^i bottlenecks: 16->7, 7->7, 7->28, 14->14 ...).
//
// Such a layer is not tensor-core work: 3x3 7->7 is 441 multiply-adds per pixel, the activations are stored in
// 64-channel (128-byte) pixel rows of which 14 bytes are data, and the tensor-core path moves the whole 128-byte
// rows through TMA and multiplies at least 16 zero-padded input channels per K step whatever Cin / Cout are.  Here one thread owns one output pixel and all its (<= 32) output
// channels: it reads only the 16-byte sectors of the input rows that hold real channels, keeps the filter bank
// in shared memory as fp32 [tap][cin][cout] (warp-broadcast 128-bit reads, 4 FMA per LDS), accumulates in
// fp32 and writes only the 16-byte sectors that hold real output channels (the zero padding of the dedicated
// activation buffers is never touched).  Traffic for 200x200x16 images, 7->7: ~20 MB read + ~10 MB written
// instead of 82 + 41 MB; ~800 instructions per pixel.
//
// The output is epilogue.cuh's fused fp16 step, one 16-byte sector at a time (epi_store_f16<1>).  OPT-IN (ODT_TC_THIN=1: where the per-pixel work is small enough; =2: wherever the layer
// qualifies) -- written after the last GPU minute of round 1: the device launch has not run yet, the body has (below).
// ref call sites: tf.layers.conv2d RetinaNet.py:579,599,609 (bottleneck 1x1 / 3x3 with 7..28 filters).
//
// The per-thread work lives in two __host__ __device__ functions (thin_fill / thin_pixel) so that the very same
// source also runs on the CPU inside a TEST-ONLY harness (tests/native/thin_host.cu, built by
// tests/test_thin_host.py): index arithmetic, rounding chain and epilogue are checked there without a GPU.
// The product library contains no host path.
#include <string.h>

#include "epilogue.cuh"

namespace odt {

struct ThinGeom {
  int B, H, W, OH, OW;
  int Cin, Cout, in_ld, w_ld;
  int stride, pad_t, pad_l;
  int in_halo, out_halo;
  long long M;  // B*OH*OW
};

constexpr int THIN_THREADS = 256;

// KS: filter size (1 or 3); CI8 / CO8: input / output channels in units of 8.
// ws: fp32 filter bank [tap][cin][cout]; par: epi_param's six rows [6][cout].
template <int KS, int CI8, int CO8>
__host__ __device__ __forceinline__ void thin_fill(int tid, float* ws, float* par, const __half* wgt, const ThinGeom& g,
                                                   const Epi& e) {
  constexpr int CI = CI8 * 8, CO = CO8 * 8, TAPS = KS * KS;
  for (int i = tid; i < TAPS * CI * CO; i += THIN_THREADS) {
    const int n = i % CO, c = (i / CO) % CI, tap = i / (CO * CI);
    float v = 0.f;
    if (n < g.Cout && c < g.Cin) v = __half2float(wgt[((long long)n * TAPS + tap) * g.w_ld + c]);
    ws[i] = v;
  }
  for (int i = tid; i < 6 * CO; i += THIN_THREADS) par[i] = epi_param(e, i / CO, i % CO);
}

template <int KS, int CI8, int CO8>
__host__ __device__ __forceinline__ void thin_pixel(long long m, const float* ws, const float* par, const __half* in,
                                                    const ThinGeom& g, const Epi& e) {
  constexpr int CI = CI8 * 8, CO = CO8 * 8;
  const int ohw = g.OH * g.OW;
  const int b = (int)(m / ohw);
  const int pix = (int)(m - (long long)b * ohw);
  const int oy = pix / g.OW, ox = pix - oy * g.OW;
  const int ih = g.in_halo;
  const int IW = g.W + 2 * ih;
  const long long img_base = (long long)b * (g.H + 2 * ih) * IW;

  float acc[CO];
#pragma unroll
  for (int n = 0; n < CO; ++n) acc[n] = 0.f;

#pragma unroll
  for (int r = 0; r < KS; ++r) {
#pragma unroll
    for (int s = 0; s < KS; ++s) {
      const int iy = oy * g.stride - g.pad_t + r;
      const int ix = ox * g.stride - g.pad_l + s;
      // with a halo the first ring outside the image is stored (zeros); anything further out is padding too
      const bool inside = iy >= -ih && iy < g.H + ih && ix >= -ih && ix < g.W + ih;
      const __half* src = in + (img_base + (long long)(iy + ih) * IW + (ix + ih)) * g.in_ld;
#pragma unroll
      for (int c8 = 0; c8 < CI8; ++c8) {
        uint4 raw = make_uint4(0u, 0u, 0u, 0u);
        if (inside) raw = ODT_LDG(reinterpret_cast<const uint4*>(src) + c8);
        const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
        float x[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __half22float2(h2[i]);
          x[2 * i] = f.x;
          x[2 * i + 1] = f.y;
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float4* wrow = reinterpret_cast<const float4*>(ws + ((r * KS + s) * CI + c8 * 8 + c) * CO);
#pragma unroll
          for (int n4 = 0; n4 < CO / 4; ++n4) {
            const float4 w = wrow[n4];
            acc[4 * n4 + 0] = fmaf(x[c], w.x, acc[4 * n4 + 0]);
            acc[4 * n4 + 1] = fmaf(x[c], w.y, acc[4 * n4 + 1]);
            acc[4 * n4 + 2] = fmaf(x[c], w.z, acc[4 * n4 + 2]);
            acc[4 * n4 + 3] = fmaf(x[c], w.w, acc[4 * n4 + 3]);
          }
        }
      }
    }
  }

  // ---- epilogue: 8 channels (one 16-byte sector) at a time ----
  const int oh = g.out_halo;
  const long long o0_row = (long long)b * e.out0_img_stride +
                           (oh ? (long long)((oy + 1) * (g.OW + 2) + ox + 1) : (long long)pix) * e.out0_pix_stride;
  const long long o1_row = aux_row(e.out1_img_stride, e.out1_pix_stride, e.out1_halo, g.OW, b, pix);
  const long long o2_row = aux_row(e.out2_img_stride, e.out2_pix_stride, e.out2_halo, g.OW, b, pix);
  const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(e.residual) + o0_row);
#pragma unroll
  for (int n8 = 0; n8 < CO8; ++n8)
    epi_store_f16<1>(e, acc + 8 * n8, par + 8 * n8, CO, [&](int) { return ODT_LDG(rp + n8); }, o0_row + 8 * n8,
                     o1_row + 8 * n8, o2_row + 8 * n8);
}

template <int KS, int CI8, int CO8>
__global__ void __launch_bounds__(THIN_THREADS)
    conv_thin_kernel(const __half* __restrict__ in, const __half* __restrict__ wgt, const __grid_constant__ ThinGeom g,
                     const __grid_constant__ Epi e) {
  pdl_launch_dependents();
  constexpr int CI = CI8 * 8, CO = CO8 * 8, TAPS = KS * KS;
  __shared__ __align__(16) float ws[TAPS * CI * CO];
  __shared__ __align__(16) float par[6 * CO];
  thin_fill<KS, CI8, CO8>(threadIdx.x, ws, par, wgt, g, e);
  __syncthreads();
  const long long m = (long long)blockIdx.x * THIN_THREADS + threadIdx.x;
  if (m < g.M) thin_pixel<KS, CI8, CO8>(m, ws, par, in, g, e);
}

static int g_thin_launches = 0;  // debug: lets a test assert that the layer really took this path

template <int KS, int CI8, int CO8>
static int launch_thin(const void* in, const void* weights, const ThinGeom& g, const Epi& e, cudaStream_t st,
                       const char* name) {
  const long long blocks = (g.M + THIN_THREADS - 1) / THIN_THREADS;
  conv_thin_kernel<KS, CI8, CO8><<<(unsigned)blocks, THIN_THREADS, 0, st>>>(
      reinterpret_cast<const __half*>(in), reinterpret_cast<const __half*>(weights), g, e);
  ODT_LAUNCH_OK();
  ++g_thin_launches;
  g_last_conv_kernel = name;
  return ODT_OK;
}

// Eligibility + geometry; ODT_ERR_UNSUPPORTED when the layer does not qualify.  `force`: ignore the work-per-pixel gate.
static int thin_plan(const void* in, const odt_conv_params* p, bool force, ThinGeom* gout, int* ks_out, int* ci_out,
                     int* co_out) {
  const int ks = p->R;
  const bool shape_ok = (ks == 1 || ks == 3) && p->S == ks && p->dil == 1 && (p->stride == 1 || p->stride == 2) &&
                        p->out0_pool == 0 && p->out0_group == 0 && (p->in_halo == 0 || p->in_halo == 1) &&
                        (p->out0_halo == 0 || p->out0_halo == 1);
  if (!shape_ok) return ODT_ERR_UNSUPPORTED;
  const int ci8 = (p->Cin + 7) / 8, co8 = (p->Cout + 7) / 8;
  const int ci8r = ci8 <= 1 ? 1 : ci8 <= 2 ? 2 : 4, co8r = co8 <= 1 ? 1 : co8 <= 2 ? 2 : 4;
  if (ci8 > 4 || co8 > 4 || (ks == 3 && (ci8 > 2 || co8 > 2))) return ODT_ERR_UNSUPPORTED;
  const bool io_ok = ((uintptr_t)in & 15) == 0 && p->in_ld % 8 == 0 && p->in_ld >= ci8r * 8 &&
                     f16_sector_outputs_ok(p, co8r * 8);
  if (!io_ok) return ODT_ERR_UNSUPPORTED;
  const long long M = (long long)p->B * p->OH * p->OW;
  if (M >= (1ll << 31) * THIN_THREADS) return ODT_ERR_UNSUPPORTED;
  // default planner (mode 1): only 1x1 layers with few multiply-adds per pixel.  The rule is carried over from the
  // previous target; it has not been re-measured on the H100.
  if (!force && (ks != 1 || ci8r * 8 * co8r * 8 > 1200)) return ODT_ERR_UNSUPPORTED;
  ThinGeom g;
  memset(&g, 0, sizeof(g));
  g.B = p->B;
  g.H = p->H;
  g.W = p->W;
  g.OH = p->OH;
  g.OW = p->OW;
  g.Cin = p->Cin;
  g.Cout = p->Cout;
  g.in_ld = p->in_ld;
  g.w_ld = p->w_ld;
  g.stride = p->stride;
  g.pad_t = p->pad_t;
  g.pad_l = p->pad_l;
  g.in_halo = p->in_halo;
  g.out_halo = p->out0_halo;
  g.M = M;
  *gout = g;
  *ks_out = ks;
  *ci_out = ci8r;
  *co_out = co8r;
  return ODT_OK;
}

// every (filter size, channel width) instantiation, for the device launch and for the test-only host harness
#define ODT_THIN_DISPATCH(CALL)                                                                               \
  CALL(3, 1, 1) CALL(3, 1, 2) CALL(3, 2, 1) CALL(3, 2, 2) CALL(1, 1, 1) CALL(1, 1, 2) CALL(1, 1, 4) CALL(1, 2, 1) \
  CALL(1, 2, 2) CALL(1, 2, 4) CALL(1, 4, 1) CALL(1, 4, 2) CALL(1, 4, 4)

// ODT_ERR_UNSUPPORTED when the layer does not qualify (the caller then takes the tensor-core paths).
int conv_thin_try(const void* in, const void* weights, const odt_conv_params* p, void* stream) {
  ThinGeom g;
  int ks, ci8r, co8r;
  const int rc = thin_plan(in, p, thin_mode() == 2, &g, &ks, &ci8r, &co8r);
  if (rc) return rc;
  const Epi e = make_epi(*p);
  cudaStream_t st = (cudaStream_t)stream;
#define ODT_THIN_CASE(KS_, CI_, CO_)           \
  if (ks == KS_ && ci8r == CI_ && co8r == CO_) \
    return launch_thin<KS_, CI_, CO_>(in, weights, g, e, st, "conv_thin_kernel<" #KS_ "," #CI_ "," #CO_ ">");
  ODT_THIN_DISPATCH(ODT_THIN_CASE)
#undef ODT_THIN_CASE
  return ODT_ERR_UNSUPPORTED;
}

}  // namespace odt

// Debug only: number of convolutions launched through conv_thin_kernel by this process.
extern "C" int odt_debug_thin_launches(void) { return odt::g_thin_launches; }
