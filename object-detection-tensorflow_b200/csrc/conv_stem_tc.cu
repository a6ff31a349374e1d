// wgmma stem convolution (Cin = 3): the first layer of every backbone.
//
// K = KS*KS*3 is far below one TMA/wgmma channel chunk, so instead of im2col TMA
// the A operand is BUILT in shared memory: two groups of 4 producer warps (one thread per
// output pixel of a 128-row tile, the groups take alternate tiles) gather the KS*KS*3 fp32 pixels, subtract the
// RGB mean, convert to fp16 and store 16-byte chunks straight into the
// 128B-swizzled K-major layout the wgmma descriptor expects (chunk c of row m at
// ((c ^ (m & 7)) << 4)); a fence.proxy.async + mbarrier arrive hands the stage to
// the consumer warpgroup.  Weights [COUT x Kpad] sit in shared memory for the
// whole kernel.  The consumer warpgroup multiplies the two 64-row halves of a
// tile (accumulators in registers), hands the stage back, applies bias/BN/
// activation to its fragments and writes fp16 NHWC rows.  The layer is HBM-bound
// (image read + activation write); the tensor pipe is idle most of the time.
//
//
// H4 variant (7x7 / stride 2 only): the image arrives as mean-subtracted fp16 RGBX ([B][H+2P][W+2P][4], zero border,
// written by odt_pack_input_rgbx).  A filter row of an output pixel is then ONE contiguous, aligned span of the image
// (8 pixels = 64 bytes = four 16-byte chunks, the eighth tap has zero weights), so a producer thread issues all of its
// loads back to back (28 LDG.128, adjacent lanes on adjacent addresses) and copies registers straight into the
// swizzled rows: no conversion, no bounds logic, no dependent address arithmetic.  The fp32 gather above is
// latency-bound (7 dependent batches of 11 strided loads per pixel: 0.36 ms for RetinaNet-800 B=16 against ~0.05 ms
// of traffic).
//
// ref: conv1_1 SSD300.py:193-200 (+mean :52-66); YOLOv3.py:388; RetinaNet.py:260-265; FCOS.py:73-78.
#include "epilogue.cuh"
#include "tc_ptx.cuh"

namespace odt {

struct StemGeom {
  int B, H, W, OH, OW, ohw, pad_t, pad_l, w_ld;
  long long M;
  int num_tiles;
  int out_halo;    // output stored as [B][OH+2][OW+2][ld]
  int vec2_ok;     // 7x7/2: filter rows start 8-byte aligned (even W, even left pad, aligned image base)
  float mean[3];
  int in_pad, ipw, iph;  // H4: zero border P of the packed image, padded row length W+2P and height H+2P (pixels)
};

constexpr int ST_MAX_STAGES = 4;
constexpr int ST_PROD_GROUPS = 2;                    // producer groups of 4 warps, round-robin over the CTA's tiles
constexpr int ST_PROD_WARPS = 4 * ST_PROD_GROUPS, ST_EPI_WARPS = 4;
constexpr int ST_THREADS = 32 * (ST_PROD_WARPS + ST_EPI_WARPS);  // producers, one consumer warpgroup
constexpr int ST_PITCH = 144;                  // staging row pitch (bytes)
constexpr int ST_WARP_STAGE = 32 * ST_PITCH;   // staging bytes per epilogue warp

// K extent of one im2col row: fp32 path KS*KS*3; H4 path KS rows of KSP pixels x 4 channels
template <int KS, bool H4>
struct StemK {
  static_assert(!H4 || KS == 7, "the packed-image (H4) stem is 7x7 only");
  static constexpr int KSP = 8;                                // pixels per filter row in the H4 layout
  static constexpr int KREAL = H4 ? KS * KSP * 4 : KS * KS * 3;
  static constexpr int KSTEPS = (KREAL + 15) / 16;
  static constexpr int NBLK = (KSTEPS * 16 + 63) / 64;
  static constexpr int STAGES = NBLK >= 4 ? 3 : ST_MAX_STAGES;  // 64 KiB stages: three fit
};

template <int COUT, int KS, int STRIDE, bool H4>
__global__ void __launch_bounds__(ST_THREADS)
    conv_stem_tc_kernel(const void* __restrict__ img_any, const __half* __restrict__ wgt,
                        const __grid_constant__ StemGeom g, const __grid_constant__ Epi e) {
  const float* img = reinterpret_cast<const float*>(img_any);
  constexpr int ST_STAGES = StemK<KS, H4>::STAGES;
  constexpr int KREAL = StemK<KS, H4>::KREAL;
  constexpr int KSP = StemK<KS, H4>::KSP;
  constexpr int KSTEPS = (KREAL + 15) / 16;        // wgmma k-steps issued
  constexpr int NCHUNK = KSTEPS * 2;               // 16-byte chunks written per row
  constexpr int NBLK = (KSTEPS * 16 + 63) / 64;    // 128-byte-row blocks per stage
  constexpr int A_BYTES = NBLK * 128 * 128;
  constexpr int B_BYTES = NBLK * COUT * 128;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  const uint32_t a_base = base;                               // ST_STAGES x A_BYTES
  const uint32_t b_base = base + ST_STAGES * A_BYTES;         // weights (1024-aligned: A_BYTES % 16384 == 0)
  const uint32_t bar_base = b_base + ((B_BYTES + 1023) & ~1023);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (ST_STAGES + s); };
  float* s_scale = reinterpret_cast<float*>(smem_raw + (bar_base + 128u - raw));
  float* s_shift = s_scale + COUT;
  // per-epilogue-warp store staging: 32 rows x 128 B at a 144 B pitch (ST_PITCH), so
  // the one-row-per-lane 16-byte writes spread over all banks (4 wavefronts per STS.128,
  // the minimum, instead of 32 at a 128 B pitch)
  const uint32_t stage_out = (bar_base + 128u + 2u * COUT * 4u + 127u) & ~127u;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // ---- one-time setup: weights -> swizzled smem, params, barriers ----
  {
    uint8_t* bsm = gbase + (b_base - base);
    // zero the K padding once, then scatter the real weights
    for (int i = threadIdx.x; i < B_BYTES / 16; i += blockDim.x)
      reinterpret_cast<uint4*>(bsm)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    for (int i = threadIdx.x; i < COUT * KS * KS * 3; i += blockDim.x) {
      const int n = i / (KS * KS * 3), kq = i - n * (KS * KS * 3);
      const int tap = kq / 3, ch = kq - tap * 3;
      const __half v = wgt[((long long)n * KS * KS + tap) * g.w_ld + ch];
      // position along K: fp32 path (tap, ch) dense; H4 path (filter row, pixel of the KSP-wide row, 4 channels)
      const int k = H4 ? ((tap / KS) * KSP + tap % KS) * 4 + ch : kq;
      const int blk = k >> 6, kk = k & 63;
      const uint32_t off = blk * COUT * 128 + n * 128 + ((((kk >> 3) ^ (n & 7))) << 4) + (kk & 7) * 2;
      *reinterpret_cast<__half*>(bsm + off) = v;
    }
    for (int c = threadIdx.x; c < COUT; c += blockDim.x) {
      s_scale[c] = e.scale ? e.scale[c] : 1.f;
      s_shift[c] = e.shift ? e.shift[c] : 0.f;
    }
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < ST_STAGES; ++s) {
      mbar_init(full_bar(s), 128);  // one producer group (one thread per tile row)
      mbar_init(empty_bar(s), ST_EPI_WARPS);  // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  fence_proxy_async_smem();  // weight tile written through the generic proxy
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp < ST_PROD_WARPS) {
    // ===================== A-tile producers ====================================
    const int t = threadIdx.x & 127;  // row of the tile
    const int pgroup = threadIdx.x >> 7;
    // group i builds the CTA's tiles i, i + G, i + 2G, ...: G gathers in flight per CTA
    int local = pgroup;
    for (int tile = blockIdx.x + pgroup * gridDim.x; tile < g.num_tiles;
         tile += ST_PROD_GROUPS * gridDim.x, local += ST_PROD_GROUPS) {
      const int stage = local % ST_STAGES;
      const uint32_t phase = (uint32_t)(local / ST_STAGES) & 1u;
      const long long m = (long long)tile * 128 + t;
      const bool ok = m < g.M;
      int b = 0, oy = 0, ox = 0;
      if (ok) {
        b = (int)(m / g.ohw);
        const int pix = (int)(m - (long long)b * g.ohw);
        oy = pix / g.OW;
        ox = pix - oy * g.OW;
      }
      const float* ib = img + (long long)b * g.H * g.W * 3;
      const int iy0 = oy * STRIDE - g.pad_t, ix0 = ox * STRIDE - g.pad_l;
      uint8_t* arow = gbase + (a_base - base) + (uint32_t)stage * A_BYTES + t * 128;
      if (H4) {
        // rows past M read image 0 / pixel 0 (valid memory); the epilogue never stores them
        const __half* src = reinterpret_cast<const __half*>(img_any) +
                            (((long long)b * g.iph + (iy0 + g.in_pad)) * g.ipw + (ix0 + g.in_pad)) * 4;
        const int rs = g.ipw * 4;  // halves per padded image row
        uint4 q[KS][4];
#pragma unroll
        for (int r = 0; r < KS; ++r) {
          const uint4* p4 = reinterpret_cast<const uint4*>(src + (long long)r * rs);
#pragma unroll
          for (int c = 0; c < 4; ++c) q[r][c] = __ldg(p4 + c);
        }
        mbar_wait(empty_bar(stage), phase ^ 1u);
#pragma unroll
        for (int r = 0; r < KS; ++r) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int id = 4 * r + c, blk = id >> 3, cc = id & 7;
            *reinterpret_cast<uint4*>(arow + blk * (128 * 128) + ((cc ^ (t & 7)) << 4)) = q[r][c];
          }
        }
        fence_proxy_async_smem();
        mbar_arrive(full_bar(stage));
        continue;
      }
      mbar_wait(empty_bar(stage), phase ^ 1u);
      // Interior pixels (the whole KSxKS window inside the image) take a branch-free path:
      // one row pointer per filter row, every tap at an immediate offset from it.  (The
      // per-tap predicated form costs ~20 integer/branch instructions per load and made
      // the producers issue-bound.)
      const bool interior = ok && iy0 >= 0 && iy0 + KS <= g.H && ix0 >= 0 && ix0 + KS <= g.W;
      const float* prow[KS];
      {
        const float* p0 = ib + ((long long)iy0 * g.W + ix0) * 3;
        const int rs = g.W * 3;
#pragma unroll
        for (int r = 0; r < KS; ++r) prow[r] = p0 + r * rs;
      }
      const float mean0 = g.mean[0], mean1 = g.mean[1], mean2 = g.mean[2];
      if (KS == 7 && STRIDE == 2 && interior && g.vec2_ok) {
        // 7x7 / stride 2: the 21 floats of one filter row are contiguous and 8-byte aligned
        // (even W, even left pad): 10 LDG.64 + 1 LDG.32 per row instead of 21 scalar loads
        // (the 24-byte lane stride costs ~7 L1 wavefronts per load instruction either way)
        constexpr int RW = KS * 3;
        float v[NCHUNK * 8];
#pragma unroll
        for (int k = KREAL; k < NCHUNK * 8; ++k) v[k] = 0.f;
#pragma unroll
        for (int r = 0; r < KS; ++r) {
          const float2* p2 = reinterpret_cast<const float2*>(prow[r]);
#pragma unroll
          for (int j = 0; j < RW / 2; ++j) {
            const float2 t2 = __ldg(p2 + j);
            const int c0 = (2 * j) % 3, c1 = (2 * j + 1) % 3;
            v[RW * r + 2 * j] = __fsub_rn(t2.x, c0 == 0 ? mean0 : (c0 == 1 ? mean1 : mean2));
            v[RW * r + 2 * j + 1] = __fsub_rn(t2.y, c1 == 0 ? mean0 : (c1 == 1 ? mean1 : mean2));
          }
          if (RW & 1) {
            const int cl = (RW - 1) % 3;
            v[RW * r + RW - 1] = __fsub_rn(__ldg(prow[r] + RW - 1), cl == 0 ? mean0 : (cl == 1 ? mean1 : mean2));
          }
          // store every 16-byte chunk completed by this row (the last row also flushes the zero-padded tail)
#pragma unroll
          for (int c = 0; c < NCHUNK; ++c) {
            const bool ready = (8 * c + 7 < RW * (r + 1)) || (r == KS - 1);
            const bool before = (r > 0) && (8 * c + 7 < RW * r);
            if (ready && !before) {
              uint4 pk;
              __half2* h = reinterpret_cast<__half2*>(&pk);
#pragma unroll
              for (int q = 0; q < 4; ++q) h[q] = __floats2half2_rn(v[8 * c + 2 * q], v[8 * c + 2 * q + 1]);
              const int blk = c >> 3, cc = c & 7;
              *reinterpret_cast<uint4*>(arow + blk * (128 * 128) + ((cc ^ (t & 7)) << 4)) = pk;
            }
          }
        }
      } else if (interior) {
#pragma unroll
        for (int c = 0; c < NCHUNK; ++c) {
          float v[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const int k = c * 8 + q;  // compile-time after unrolling
            if (k < KREAL) {
              const int tap = k / 3, ch = k - tap * 3;
              const int r = tap / KS, sx = tap - r * KS;
              v[q] = __fsub_rn(__ldg(prow[r] + sx * 3 + ch), ch == 0 ? mean0 : (ch == 1 ? mean1 : mean2));
            } else {
              v[q] = 0.f;
            }
          }
          uint4 pk;
          __half2* h = reinterpret_cast<__half2*>(&pk);
#pragma unroll
          for (int q = 0; q < 4; ++q) h[q] = __floats2half2_rn(v[2 * q], v[2 * q + 1]);
          const int blk = c >> 3, cc = c & 7;
          *reinterpret_cast<uint4*>(arow + blk * (128 * 128) + ((cc ^ (t & 7)) << 4)) = pk;
        }
      } else {
#pragma unroll
        for (int c = 0; c < NCHUNK; ++c) {
          float v[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const int k = c * 8 + q;
            if (k < KREAL) {
              const int tap = k / 3, ch = k - tap * 3;
              const int r = tap / KS, sx = tap - r * KS;
              const int iy = iy0 + r, ix = ix0 + sx;
              const bool in = ok && iy >= 0 && iy < g.H && ix >= 0 && ix < g.W;
              v[q] = in ? __fsub_rn(__ldg(prow[r] + sx * 3 + ch), ch == 0 ? mean0 : (ch == 1 ? mean1 : mean2))
                        : 0.f;
            } else {
              v[q] = 0.f;
            }
          }
          uint4 pk;
          __half2* h = reinterpret_cast<__half2*>(&pk);
#pragma unroll
          for (int q = 0; q < 4; ++q) h[q] = __floats2half2_rn(v[2 * q], v[2 * q + 1]);
          const int blk = c >> 3, cc = c & 7;
          *reinterpret_cast<uint4*>(arow + blk * (128 * 128) + ((cc ^ (t & 7)) << 4)) = pk;
        }
      }
      fence_proxy_async_smem();
      mbar_arrive(full_bar(stage));
    }
  } else {
    // ===================== consumer warpgroup: MMA + epilogue ==================
    // Warp w holds rows 16w .. 16w+15 of each 64-row half (wgmma fragment layout, tc_ptx.cuh).
    const int w = warp - ST_PROD_WARPS;
    int stage = 0;
    uint32_t phase = 0;
    // Stage the warp's 32 rows x COUT fp16 in shared memory (144-byte pitch: the fragment writes
    // of one instruction hit 32 distinct banks), then store them with the lanes transposed:
    // CPR consecutive lanes cover one row's COUT*2 bytes, so every STG.128 of the warp
    // writes whole 32-byte sectors of 32/CPR rows -- in the dense and in the halo layout.
    // Staging row h*16 + i holds tile row 64h + 16w + i.
    uint8_t* warp_stage = smem_raw + (stage_out - raw) + (uint32_t)w * ST_WARP_STAGE;
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      float acc[2][COUT / 2];
      mbar_wait(full_bar(stage), phase);
      wg_fence();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int k = 0; k < KSTEPS; ++k) {
          const uint32_t blk = k >> 2, kin = k & 3;
          const uint64_t adesc =
              make_desc_sw128(a_base + (uint32_t)stage * A_BYTES + blk * (128 * 128) + (uint32_t)h * (64 * 128)) +
              (uint64_t)(2 * kin);
          const uint64_t bdesc = make_desc_sw128(b_base + blk * (COUT * 128)) + (uint64_t)(2 * kin);
          wg_mma_f16<COUT>(acc[h], adesc, bdesc, (uint32_t)(k != 0));
        }
      }
      wg_commit();
      wg_wait<0>();
      // the stage has been read: hand it back before the epilogue
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(stage));
      if (++stage == ST_STAGES) {
        stage = 0;
        phase ^= 1u;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint8_t* r0 = warp_stage + (h * 16 + (lane >> 2)) * ST_PITCH;
#pragma unroll
        for (int i = 0; i < COUT / 8; ++i) {
          const int c0 = 8 * i + 2 * (lane & 3);
          const float sc0 = s_scale[c0], sc1 = s_scale[c0 + 1], sh0 = s_shift[c0], sh1 = s_shift[c0 + 1];
          *reinterpret_cast<__half2*>(r0 + c0 * 2) =
              __floats2half2_rn(apply_act(fmaf(acc[h][4 * i], sc0, sh0), e.act),
                                apply_act(fmaf(acc[h][4 * i + 1], sc1, sh1), e.act));
          *reinterpret_cast<__half2*>(r0 + 8 * ST_PITCH + c0 * 2) =
              __floats2half2_rn(apply_act(fmaf(acc[h][4 * i + 2], sc0, sh0), e.act),
                                apply_act(fmaf(acc[h][4 * i + 3], sc1, sh1), e.act));
        }
      }
      __syncwarp();
      const long long m = (long long)tile * 128 + (lane < 16 ? 16 * w + lane : 64 + 16 * w + lane - 16);
      const bool row_ok = m < g.M;
      const int b = row_ok ? (int)(m / g.ohw) : 0;
      const int pix = row_ok ? (int)(m - (long long)b * g.ohw) : 0;
      long long opix = pix;
      if (g.out_halo) {
        const int oy = pix / g.OW, ox = pix - oy * g.OW;
        opix = (long long)(oy + 1) * (g.OW + 2) + ox + 1;
      }
      const long long my_off = row_ok ? (long long)b * e.out0_img_stride + opix * e.out0_pix_stride : -1;
      constexpr int CPR = COUT / 8;    // 16-byte chunks per row (the pad channels stay zero in HBM)
      constexpr int RPI = 32 / CPR;    // rows per store instruction
      const int sub_row = lane / CPR, chunk = lane % CPR;
#pragma unroll
      for (int i = 0; i < CPR; ++i) {
        const int rr = i * RPI + sub_row;
        const uint4 val = *reinterpret_cast<const uint4*>(warp_stage + rr * ST_PITCH + (chunk << 4));
        const long long ro = __shfl_sync(0xffffffffu, my_off, rr);
        if (ro >= 0) *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out0) + ro + chunk * 8) = val;
      }
      __syncwarp();  // staging rows are rewritten by the next tile
    }
  }
}

template <int COUT, int KS, int STRIDE, bool H4>
static int launch_stem_tc(const void* img, const void* w, const StemGeom& g, const Epi& e,
                          cudaStream_t st) {
  constexpr int NBLK = StemK<KS, H4>::NBLK;
  const int smem = StemK<KS, H4>::STAGES * NBLK * 128 * 128 + ((NBLK * COUT * 128 + 1023) & ~1023) + 1024 + 128 +
                   2 * COUT * 4 + 64 + 128 + ST_EPI_WARPS * ST_WARP_STAGE;
  auto kern = conv_stem_tc_kernel<COUT, KS, STRIDE, H4>;
  static bool attr = false;
  if (!attr) {
    ODT_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = true;
  }
  // as many CTAs per SM as registers and shared memory allow (the 384-thread variants take one or two)
  int per_sm = 0;
  ODT_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, ST_THREADS, smem));
  if (per_sm < 1) {
    set_error("launch_stem_tc: the kernel does not fit on an SM (%d bytes of shared memory)", smem);
    return ODT_ERR_CUDA;
  }
  int grid = kNumSMs * per_sm;
  if (grid > g.num_tiles) grid = g.num_tiles;
  kern<<<grid, ST_THREADS, smem, st>>>(img, (const __half*)w, g, e);
  return ODT_OK;
}

}  // namespace odt

using namespace odt;

// Returns ODT_ERR_UNSUPPORTED when the shape has no tensor-core stem variant
// (the caller then uses the CUDA-core stem).
int odt_conv2d_stem_tc_try(const float* images, const float* mean3_host, const void* weights,
                           const odt_conv_params* p, void* stream) {
  const bool ok = p->out0 && !p->out1 && !p->out2 && !p->residual && p->out0_group == 0 && p->R == p->S &&
                  p->dil == 1 && p->in_ld == 3 && p->Cin == 3 && p->out0_dtype == ODT_F16 &&
                  p->out0_pool == 0 && ((uintptr_t)p->out0 % 16) == 0 && p->out0_pix_stride % 8 == 0 &&
                  p->out0_pix_stride >= p->Cout &&
                  p->out0_img_stride % 8 == 0;
  int variant = 0;
  if (ok && p->R == 3 && p->stride == 1 && p->Cout == 64) variant = 1;
  if (ok && p->R == 3 && p->stride == 1 && p->Cout == 32) variant = 2;
  if (ok && p->R == 7 && p->stride == 2 && p->Cout == 16) variant = 3;
  if (!variant) return ODT_ERR_UNSUPPORTED;
  StemGeom g;
  g.B = p->B; g.H = p->H; g.W = p->W; g.OH = p->OH; g.OW = p->OW; g.ohw = p->OH * p->OW;
  g.pad_t = p->pad_t; g.pad_l = p->pad_l; g.w_ld = p->w_ld;
  g.M = (long long)p->B * p->OH * p->OW;
  g.num_tiles = (int)((g.M + 127) / 128);
  g.out_halo = p->out0_halo ? 1 : 0;
  g.vec2_ok = ((p->W & 1) == 0 && (p->pad_l & 1) == 0 && ((uintptr_t)images & 7) == 0) ? 1 : 0;
  g.mean[0] = mean3_host[0]; g.mean[1] = mean3_host[1]; g.mean[2] = mean3_host[2];
  Epi e = make_epi(*p);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ODT_OK;
  g.in_pad = g.ipw = g.iph = 0;
  if (variant == 1) rc = launch_stem_tc<64, 3, 1, false>(images, weights, g, e, st);
  if (variant == 2) rc = launch_stem_tc<32, 3, 1, false>(images, weights, g, e, st);
  if (variant == 3) rc = launch_stem_tc<16, 7, 2, false>(images, weights, g, e, st);
  if (rc) return rc;
  ODT_LAUNCH_OK();
  return ODT_OK;
}

// 7x7 / stride-2 stem on the packed fp16 RGBX image (see the header comment).  `rgbx`: [B][H+2P][W+2P][4] fp16 with a
// zero border, P = p->in_halo = 4 (even W, even left pad).
extern "C" int odt_conv2d_stem_rgbx(const void* rgbx, const void* weights, const odt_conv_params* p, void* stream) {
  int rc0 = check_conv_params(p);
  if (rc0) return rc0;
  ODT_CHECK_ARG(rgbx && weights, "null tensor");
  const bool ok = p->out0 && !p->out1 && !p->out2 && !p->residual && p->out0_group == 0 && p->R == p->S &&
                  p->dil == 1 && p->in_ld == 4 && p->Cin == 3 && p->out0_dtype == ODT_F16 &&
                  p->out0_pool == 0 && ((uintptr_t)p->out0 % 16) == 0 && p->out0_pix_stride % 8 == 0 &&
                  p->out0_pix_stride >= p->Cout && p->out0_img_stride % 8 == 0 && ((uintptr_t)rgbx % 16) == 0;
  // up to 16 real outputs.  The kernel computes and stores 16 channels per pixel, so the filter bank, scale and shift
  // must hold 16 rows (Cout_pad), zero past Cout, and the output row must have room for 16.
  if (!(ok && p->R == 7 && p->stride == 2 && p->Cout <= 16 && p->Cout_pad == 16 && p->out0_pix_stride >= 16 &&
        p->in_halo == 4 && (p->W & 1) == 0 && (p->pad_l & 1) == 0 && p->pad_t <= 4 && p->pad_l <= 4 &&
        // the 8-pixel row window and the 7 filter rows of the last output pixel stay inside the padded image
        (p->OW - 1) * 2 - p->pad_l + 7 <= p->W - 1 + 4 && (p->OH - 1) * 2 - p->pad_t + 6 <= p->H - 1 + 4))
    return ODT_ERR_UNSUPPORTED;
  StemGeom g;
  g.B = p->B; g.H = p->H; g.W = p->W; g.OH = p->OH; g.OW = p->OW; g.ohw = p->OH * p->OW;
  g.pad_t = p->pad_t; g.pad_l = p->pad_l; g.w_ld = p->w_ld;
  g.M = (long long)p->B * p->OH * p->OW;
  g.num_tiles = (int)((g.M + 127) / 128);
  g.out_halo = p->out0_halo ? 1 : 0;
  g.vec2_ok = 0;
  g.mean[0] = g.mean[1] = g.mean[2] = 0.f;
  g.in_pad = p->in_halo;
  g.ipw = p->W + 2 * p->in_halo;
  g.iph = p->H + 2 * p->in_halo;
  Epi e = make_epi(*p);
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = launch_stem_tc<16, 7, 2, true>(rgbx, weights, g, e, st);
  if (rc) return rc;
  ODT_LAUNCH_OK();
  return ODT_OK;
}
