// Transposed wgmma tiles for the narrow 3x3 halo layers (Cout_pad = 64 / 128): D^T[cout, pixel] = W * X^T.
//
// conv_tc_kernel puts the pixels on the M side of the wgmma and the output channels on N, so a layer with 64 or 128
// output channels runs m64n64k16 / m64n128k16, which the tensor pipe cannot issue at its dense rate (DESIGN 3.1: 49 %
// / 64 % with no loads at all; only n256 gets there).  Here the operands trade places:
// * A = one filter tile [64 couts x 64 ch], K-major, 128-byte swizzle -- the tile the weight tensor map loads anyway;
// * B = the activation slab [pixels x 64 ch], K-major, 128-byte swizzle -- the halo-flat / row-block slab of
//   conv_tc.cu, 256 pixels long; the three horizontal taps are row-shifted descriptors of one slab, on the B side;
// * one wgmma.m64n256k16 per (tap, 16-deep K step): 64 couts x 256 pixels, 128 accumulator registers per thread.
// K order (filter row -> channel chunk -> tap -> K step) is conv_tc_kernel's, so every output sums the same products
// in the same sequence.
//
// Work unit = (256-pixel tile, 64-cout half).  The two consumer warpgroups ping-pong over the CTA's units as in
// conv_tc_kernel (the epilogue of one runs under the MMAs of the other); with Cout_pad = 128 the two halves of a pixel
// tile are consecutive units, so warpgroup g always computes couts 64g .. 64g+63 and the second load of the slab hits
// L2.  Cooperative 128-cout tiles would load the slab once but expose every epilogue and leave room for only two
// (slab + 3 x 16 KiB filter) stages; a 64-cout unit's stage is 58 KiB and three fit.
// Tile geometry: halo-flat (no pool) = 256 consecutive padded-linear positions, slab [264 x 64]; row-block (fused
// 2x2/2 max-pool) = RP rows x 256/RP columns, RP in {2, 4, 8} for the fewest tiles, slab box {64, RP, 256/RP + 2, 1}.
// Filter bank resident in shared memory when Cout_pad = 64 and three slab stages fit beside it (Cin = 64: 72 KiB).
// Epilogue (fp16 out0 alone): scale / shift per accumulator ROW (two couts per thread, in registers), activation and
// rounding on the fragments (epi_act_f16x2), halo-flat border positions forced to zero, the 2x2 pool = the in-thread
// maximum of the adjacent pixel pair plus one step across RP (neighbouring register for RP 8, one lane exchange for
// RP 2 / 4); stmatrix.trans turns the [cout][pixel] fragments into [pixel][cout] rows of a 64-pixel x 64-cout staging
// chunk (128-byte swizzle, double-buffered per warpgroup), stored by TMA.
#include <string.h>

#include "epilogue.cuh"
#include "tc_ptx.cuh"

namespace odt {

constexpr int SW_PIX = 256;  // pixels per tile (the wgmma N)
constexpr int SW_CO = 64;    // output channels per unit (the wgmma M)
constexpr int SW_BK = 64;
constexpr int SW_THREADS = 3 * 128;  // producer warpgroup, two consumer warpgroups
constexpr int SW_PRODUCER_REGS = 40, SW_CONSUMER_REGS = 232;
constexpr int SW_FLAT_BOX = 88;                      // the halo-flat slab = 3 boxes of 88 rows (a box dimension is <= 256)
constexpr int SW_SLAB_BYTES = 34 * 1024;             // largest slab: RP 8, (32 + 2) * 8 rows x 128 B
constexpr int SW_W_BYTES = SW_CO * 128;              // one filter tile
constexpr int SW_OUT_BYTES = 64 * 128;               // one staged chunk: 64 pixels x 64 couts
constexpr int SW_MAX_STAGES = 8;
constexpr int SW_SMEM_LIMIT = 232448;                // 227 KiB
constexpr int SW_FIXED_BYTES = 2048 + 4 * SW_OUT_BYTES;  // alignment slack + barriers, two staging chunks per warpgroup
constexpr int SW_BAR_EPI = 1, SW_BAR_ORDER = 3;      // named barriers, as in conv_tc_kernel
// Taken (ODT_TC_SWAP=1) from this many units per SM: below it the CTAs run too few ping-pong rounds to hide the
// epilogues.  Measured with scripts/conv_micro.py on an H100 80GB HBM3 SXM, 700 W power limit (BASELINE 5).
constexpr int SW_MIN_UNITS_PER_SM = 4;

struct SwapGeom {
  int cchunks, klast, halves, num_ptiles, stages, bres, a_tx;
  int RP, XB, xblocks, yblocks;  // RP = 0: halo-flat
  int PW, PH, PHW, H, W;
  long long Q;
};

__global__ void __launch_bounds__(SW_THREADS, 1)
    conv_tc_swap_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                        const __grid_constant__ CUtensorMap tmO, const __grid_constant__ SwapGeom g,
                        const __grid_constant__ Epi e) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int stages = g.stages;
  const uint32_t stage_bytes = SW_SLAB_BYTES + (g.bres ? 0u : 3u * SW_W_BYTES);
  const uint32_t wres_base = base + (uint32_t)stages * stage_bytes;
  const uint32_t wres_bytes = g.bres ? (uint32_t)(9 * g.cchunks) * SW_W_BYTES : 0u;
  const uint32_t bar_base = wres_base + wres_bytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (SW_MAX_STAGES + s); };
  const uint32_t wfull_bar = bar_base + 8u * (2 * SW_MAX_STAGES);
  const uint32_t out_base = bar_base + 1024u;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmO) : "memory");
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4);  // one arrival per warp of the consuming warpgroup
    }
    mbar_init(wfull_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (g.bres && warp == 0) {
    // the filter bank is constant data: fetch it before waiting on the previous kernel
    if (elect_one()) {
      mbar_expect_tx(wfull_bar, wres_bytes);
      for (int t = 0; t < 9 * g.cchunks; ++t)
        tma_load_2d(wres_base + (uint32_t)t * SW_W_BYTES, &tmW, wfull_bar, t * SW_BK, 0);
    }
    __syncwarp();
  }
  pdl_launch_dependents();
  pdl_wait();

  // this CTA's units: pixel tiles blockIdx.x, blockIdx.x + gridDim.x, ..., each with its `halves` cout halves
  const int hs = g.halves - 1;  // halves is 1 or 2: unit i = (tile i >> hs, half i & hs)
  const int units = ((g.num_ptiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x) << hs;
  const int kblocks = 3 * g.cchunks;  // pipeline stages per unit: one per (filter row, channel chunk)
  const int per_img = g.yblocks * g.xblocks;

  if (warp < 4) {
    wg_reg_dealloc<SW_PRODUCER_REGS>();
    if (warp != 0) return;
    // ===================== TMA producer (warp-uniform loop, one elected lane issues) =====================
    int stage = 0;
    uint32_t phase = 0;
    for (int i = 0; i < units; ++i) {
      const int pt = (int)blockIdx.x + (i >> hs) * (int)gridDim.x, half = i & hs;
      int bb = 0, yq = 0, xq = 0;
      if (g.RP) {
        bb = pt / per_img;
        const int rem = pt - bb * per_img;
        yq = rem / g.xblocks;
        xq = rem - yq * g.xblocks;
      }
      for (int r = 0; r < 3; ++r) {
        // halo-flat: padded-linear rows pt*256 + (r-1)*PW - 1 ...; negative / past-the-end rows are TMA zero fill
        const int row0 = pt * SW_PIX + (r - 1) * g.PW - 1;
        for (int cc = 0; cc < g.cchunks; ++cc) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          if (elect_one()) {
            const uint32_t dst = base + (uint32_t)stage * stage_bytes;
            mbar_expect_tx(full_bar(stage), (uint32_t)g.a_tx + (g.bres ? 0u : 3u * SW_W_BYTES));
            if (g.RP) {  // padded rows RP*yq + r .., padded columns XB*xq .. (+2 for the taps)
              tma_load_4d(dst, &tmX, full_bar(stage), cc * SW_BK, g.RP * yq + r, g.XB * xq, bb);
            } else {
#pragma unroll
              for (int b = 0; b < 3; ++b)
                tma_load_2d(dst + (uint32_t)(b * SW_FLAT_BOX * 128), &tmX, full_bar(stage), cc * SW_BK,
                            row0 + b * SW_FLAT_BOX);
            }
            if (!g.bres) {
#pragma unroll
              for (int s = 0; s < 3; ++s)
                tma_load_2d(dst + SW_SLAB_BYTES + (uint32_t)s * SW_W_BYTES, &tmW, full_bar(stage),
                            ((r * 3 + s) * g.cchunks + cc) * SW_BK, half * SW_CO);
            }
          }
          __syncwarp();
          if (++stage == stages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else {
    wg_reg_alloc<SW_CONSUMER_REGS>();
    // ===================== consumer warpgroups (ping-pong over the units) =====================
    const int quarter = warp & 3;
    const int group = (warp - 4) >> 2;
    const int et = threadIdx.x - 128 * (1 + group);
    const int epi_bar = SW_BAR_EPI + group;
    const uint32_t out_buf = out_base + (uint32_t)group * 2u * SW_OUT_BYTES;
    const int q = lane & 3, lr = lane >> 2;
    int sbuf = 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[SW_PIX / 2];
    if (g.bres) mbar_wait(wfull_bar, 0);
    // stmatrix addressing: lane l gives row j = l%8 of matrix l/8 = (cout octet l/8 % 2, pixel octet l/16)
    const int mk = (lane >> 3) & 1, mu = lane >> 4, mj = lane & 7;
    const int piece = 2 * quarter + mk;  // 16-byte piece of the staged row: couts 16*quarter + 8*mk .. +7

    // one staged chunk: hv[k][u] = this lane's fragment pair of matrix (cout octet k, pixel octet u); row(u, j) =
    // the chunk row of that matrix's pixel j.  128-byte swizzle: piece c of row r at r*128 + ((c ^ r%8) * 16).
    auto stage_chunk = [&](const uint32_t (&hv)[2][8], auto row, auto store) {
      const uint32_t buf = out_buf + (uint32_t)sbuf * SW_OUT_BYTES;
#pragma unroll
      for (int u0 = 0; u0 < 8; u0 += 2) {
        const int r = row(u0 + mu, mj);
        stmatrix_x4_trans(buf + (uint32_t)(r * 128 + ((piece ^ (r & 7)) << 4)), hv[0][u0], hv[1][u0], hv[0][u0 + 1],
                          hv[1][u0 + 1]);
      }
      fence_proxy_async_smem();
      if (et == 0) bulk_wait_read<0>();  // the previous chunk's store has read the buffer the next chunk takes
      named_bar_sync(epi_bar, 128);
      if (et == 0) {
        store(buf);
        bulk_commit();
      }
      sbuf ^= 1;
    };

    for (int i = 0; i < units; ++i) {
      if ((i & 1) != group) {  // the other warpgroup's unit: its k-blocks pass through the ring
        const int adv = stage + kblocks;
        stage = adv % stages;
        phase ^= (uint32_t)(adv / stages) & 1u;
        continue;
      }
      const int pt = (int)blockIdx.x + (i >> hs) * (int)gridDim.x, half = i & hs;
      if (i > 0) named_bar_sync(SW_BAR_ORDER + group, 256);
      int prev = -1, cc = 0, r = 0;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t slab = base + (uint32_t)stage * stage_bytes;
        // resident bank: tile ((r*3 + s)*cchunks + cc)
        const uint32_t wt = g.bres ? wres_base + (uint32_t)(r * 3 * g.cchunks + cc) * SW_W_BYTES : slab + SW_SLAB_BYTES;
        const uint64_t wstep = (uint64_t)(((uint32_t)(g.bres ? g.cchunks : 1) * SW_W_BYTES) >> 4);
        const uint64_t xstep = (uint64_t)(g.RP ? 8 * g.RP : 8);  // rows per tap shift x 128 B >> 4
        const int ksteps = __shfl_sync(0xffffffffu, (cc == g.cchunks - 1) ? g.klast : SW_BK / 16, 0);
        if (++cc == g.cchunks) {
          cc = 0;
          ++r;
        }
        const uint64_t wdesc = make_desc_sw128(wt), xdesc = make_desc_sw128(slab);
        wg_fence();
#pragma unroll
        for (int s3 = 0; s3 < 3; ++s3)
          wg_mma_chunk<SW_PIX>(acc, wdesc + wstep * s3, xdesc + xstep * s3, ksteps, (kb | s3) == 0);
        wg_commit();
        wg_wait<1>();  // the previous k-block's MMAs have retired: its stage goes back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == stages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      // every MMA of this unit is issued: the other warpgroup's mainloop may start
      if (i + 1 < units) named_bar_arrive(SW_BAR_ORDER + (group ^ 1), 256);
      wg_wait<0>();
      if (lane == 0) mbar_arrive(empty_bar(prev));

      // ---- epilogue on the fragments: register 4*i + 2*k + {0,1} = cout 16*quarter + lr + 8*k, pixels 8*i + 2*q + {0,1}
      float2 sc[2], sh[2];
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int n = half * SW_CO + 16 * quarter + lr + 8 * k;  // channels past Cout: identity
        const float a = epi_param(e, 0, n), b = epi_param(e, 1, n);
        sc[k] = make_float2(a, a);
        sh[k] = make_float2(b, b);
      }
      if (g.RP == 0) {
        // halo-flat: four chunks of 64 consecutive positions; border positions are stored as zeros.  (yp, xp) = the
        // padded coordinates of this lane's first position of the octet, advanced by 8 per octet (Q < 2^31 - 4096).
        const unsigned m = (unsigned)(pt * SW_PIX + 2 * q);
        const unsigned rem = m % (unsigned)g.PHW;
        int yp = (int)(rem / (unsigned)g.PW), xp = (int)(rem % (unsigned)g.PW);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          if ((long long)pt * SW_PIX + 64 * c >= g.Q) break;  // past the last position (uniform)
          uint32_t hv[2][8];
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int i8 = 8 * c + u;
            int y1 = yp, x1 = xp + 1;
            if (x1 == g.PW) {
              x1 = 0;
              y1 = yp + 1 == g.PH ? 0 : yp + 1;
            }
            const uint32_t mask = ((yp >= 1 && yp <= g.H && xp >= 1 && xp <= g.W) ? 0x0000FFFFu : 0u) |
                                  ((y1 >= 1 && y1 <= g.H && x1 >= 1 && x1 <= g.W) ? 0xFFFF0000u : 0u);
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              __half2 v = epi_act_f16x2(acc[4 * i8 + 2 * k], acc[4 * i8 + 2 * k + 1], sc[k], sh[k], e.act);
              hv[k][u] = *reinterpret_cast<uint32_t*>(&v) & mask;
            }
            xp += 8;
            while (xp >= g.PW) {
              xp -= g.PW;
              if (++yp == g.PH) yp = 0;
            }
          }
          stage_chunk(
              hv, [](int u, int j) { return 8 * u + j; },
              [&](uint32_t buf) { tma_store_2d(&tmO, buf, half * SW_CO, pt * SW_PIX + 64 * c); });
        }
      } else {
        // row-block pooled tile: pixel n = RP*x + y.  The window's y partner is the other pixel of the register pair;
        // its x partner is pixel n ^ RP: octet i ^ 1 (RP 8) or lane ^ RP/2 (RP 2 / 4), where each lane of a pair keeps
        // one octet of two.  The maxima are taken of the rounded values (the fp16 maximum the stand-alone pool takes).
        uint32_t kept[16];  // [v]: half2 (cout k = 0, cout k = 1) of this lane's v-th pooled pixel
        const int X = g.RP >> 1;
        const bool odd = (lane & X) != 0;  // RP 2 / 4: this lane keeps octets 2*v + odd
#pragma unroll
        for (int v = 0; v < 16; ++v) {
          uint32_t m2[2];
#pragma unroll
          for (int o = 0; o < 2; ++o) {
            const int i8 = 2 * v + o;
            const __half2 a = epi_act_f16x2(acc[4 * i8], acc[4 * i8 + 1], sc[0], sh[0], e.act);
            const __half2 b = epi_act_f16x2(acc[4 * i8 + 2], acc[4 * i8 + 3], sc[1], sh[1], e.act);
            const __half2 t = __halves2half2(__hmax(__low2half(a), __high2half(a)), __hmax(__low2half(b), __high2half(b)));
            m2[o] = *reinterpret_cast<const uint32_t*>(&t);
          }
          uint32_t mine = m2[0], other = m2[1];
          if (g.RP != 8) {
            mine = odd ? m2[1] : m2[0];
            other = __shfl_xor_sync(0xffffffffu, odd ? m2[0] : m2[1], X);
          }
          const __half2 t = __hmax2(*reinterpret_cast<__half2*>(&mine), *reinterpret_cast<__half2*>(&other));
          kept[v] = *reinterpret_cast<const uint32_t*>(&t);
        }
        uint32_t hv[2][8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          hv[0][u] = __byte_perm(kept[2 * u], kept[2 * u + 1], 0x5410);
          hv[1][u] = __byte_perm(kept[2 * u], kept[2 * u + 1], 0x7632);
        }
        // pooled pixel (x/2, y/2) is row (y/2)*(XB/2) + x/2 of the staged chunk (the {64, XB/2, RP/2, 1} box); pixel j
        // of matrix u is the (2*u + j%2)-th pooled pixel of the lanes with l%4 = j/2
        const int RP = g.RP;
        const int yq = (pt % per_img) / g.xblocks, xq = (pt % per_img) % g.xblocks;
        stage_chunk(
            hv,
            [RP](int u, int j) {
              const int v = 2 * u + (j & 1), ql = j >> 1;
              return RP == 8 ? ql * 16 + v : RP == 4 ? (ql & 1) * 32 + 2 * v + (ql >> 1) : 4 * v + 2 * (ql & 1) + (ql >> 1);
            },
            [&](uint32_t buf) {
              tma_store_4d(&tmO, buf, half * SW_CO, (g.XB >> 1) * xq, (g.RP >> 1) * yq, pt / per_img);
            });
      }
    }
    // the shared-memory sources of the last output stores stay valid until the stores are done
    if (et == 0) bulk_wait<0>();
  }
}

// ------------------------------------------------------------------ host: plan ----
struct SwapPlan {
  int rp;            // 0: halo-flat, else rows per row-block tile
  long long ptiles;  // 256-pixel tiles
};

// The row-block split of a pooled layer into RP x 256/RP tiles: the RP of {8, 4, 2} with the fewest tiles per image
// (ties keep the larger RP: its pooling stays in registers and its tap shift is a whole swizzle atom)
static int swap_rowblock_rp(int OH, int OW, long long* tiles) {
  int best = 8;
  long long bt = -1;
  for (int rp = 8; rp >= 2; rp >>= 1) {
    const int xb = SW_PIX / rp;
    const long long t = (long long)((OH + rp - 1) / rp) * ((OW + xb - 1) / xb);
    if (bt < 0 || t < bt) {
      bt = t;
      best = rp;
    }
  }
  *tiles = bt;
  return best;
}

// whether the layer is one the transposed tile computes (shape and output layout), and its tile plan
static bool swap_eligible(const odt_conv_params* p, SwapPlan* plan) {
  const long long PHW = (long long)(p->H + 2) * (p->W + 2), Q = (long long)p->B * PHW;
  if (p->in_halo != 1 || p->R != 3 || p->S != 3 || p->stride != 1 || p->dil != 1 || p->pad_t != 1 || p->pad_l != 1 ||
      p->OH != p->H || p->OW != p->W)
    return false;
  if ((p->Cout_pad != 64 && p->Cout_pad != 128) || p->in_ld % 64 != 0 || p->w_ld != p->in_ld) return false;
  if (Q >= (1ll << 31) - 4096) return false;
  // fp16 out0 alone, in a layout one output tensor map covers
  if (!p->out0 || p->out0_dtype != ODT_F16 || p->residual || p->out1 || p->out2 || p->out0_group != 0 ||
      !f16_rows_aligned(p->out0, p->out0_img_stride, p->out0_pix_stride, p->Cout_pad))
    return false;
  if (p->out0_pool == 2) {
    if (p->OH % 2 || p->OW % 2 || (p->out0_halo != 0 && p->out0_halo != 1)) return false;
    long long per_img;
    plan->rp = swap_rowblock_rp(p->OH, p->OW, &per_img);
    plan->ptiles = p->B * per_img;
  } else if (p->out0_pool == 0) {
    if (p->out0_halo != 1 || p->out0_img_stride != PHW * p->out0_pix_stride) return false;
    plan->rp = 0;
    plan->ptiles = (Q + SW_PIX - 1) / SW_PIX;
  } else {
    return false;
  }
  return plan->ptiles < (1ll << 22);  // 256 * tiles stays a 32-bit TMA coordinate
}

static bool swap_taken(const odt_conv_params* p, SwapPlan* plan) {
  const int mode = swap_mode();
  if (mode == 0 || !swap_eligible(p, plan)) return false;
  return mode == 2 || plan->ptiles * (p->Cout_pad / SW_CO) >= (long long)SW_MIN_UNITS_PER_SM * kNumSMs;
}

int conv_swap_try(const void* in, const void* weights, const odt_conv_params* p, void* stream) {
  SwapPlan plan;
  if (!swap_taken(p, &plan)) return ODT_ERR_UNSUPPORTED;
  SwapGeom g;
  memset(&g, 0, sizeof(g));
  g.cchunks = p->in_ld / 64;
  {
    const int rem = p->Cin - (g.cchunks - 1) * SW_BK;  // real channels in the last chunk (see TcGeom::klast)
    g.klast = rem >= SW_BK ? SW_BK / 16 : (rem <= 0 ? 1 : (rem + 15) / 16);
  }
  g.halves = p->Cout_pad / SW_CO;
  g.num_ptiles = (int)plan.ptiles;
  g.H = p->H;
  g.W = p->W;
  g.PW = p->W + 2;
  g.PH = p->H + 2;
  g.PHW = g.PH * g.PW;
  g.Q = (long long)p->B * g.PHW;
  g.RP = plan.rp;
  g.xblocks = g.yblocks = 1;
  g.a_tx = 3 * SW_FLAT_BOX * 128;
  if (g.RP) {
    g.XB = SW_PIX / g.RP;
    g.yblocks = (p->OH + g.RP - 1) / g.RP;
    g.xblocks = (p->OW + g.XB - 1) / g.XB;
    g.a_tx = (g.XB + 2) * g.RP * 128;
  }
  const long long wres = 9ll * g.cchunks * SW_W_BYTES;
  g.bres = g.halves == 1 && wres + 3 * SW_SLAB_BYTES + SW_FIXED_BYTES <= SW_SMEM_LIMIT;
  const int stage_bytes = SW_SLAB_BYTES + (g.bres ? 0 : 3 * SW_W_BYTES);
  int stages = (SW_SMEM_LIMIT - SW_FIXED_BYTES - (g.bres ? (int)wres : 0)) / stage_bytes;
  if (stages > SW_MAX_STAGES) stages = SW_MAX_STAGES;
  g.stages = stages;  // >= 3: a streamed stage is 58 KiB

  CUtensorMap tmX, tmW, tmO;
  int rc;
  if (g.RP) {
    // [ld][H+2][W+2][B] view with the ROW dimension second: a {64, RP, XB+2, 1} box lands in shared memory
    // column-major over the tile (row = column*RP + row), so tap s is the slab shifted by s*RP rows
    const cuuint64_t PH = (cuuint64_t)g.PH, PW = (cuuint64_t)g.PW;
    cuuint64_t dims[4] = {(cuuint64_t)p->in_ld, PH, PW, (cuuint64_t)p->B};
    cuuint64_t strides[3] = {PW * p->in_ld * 2, (cuuint64_t)p->in_ld * 2, PH * PW * p->in_ld * 2};
    cuuint32_t box[4] = {SW_BK, (cuuint32_t)g.RP, (cuuint32_t)(g.XB + 2), 1};
    rc = tc_encode_tiled(&tmX, in, 4, dims, strides, box, false);
  } else {
    cuuint64_t dims[2] = {(cuuint64_t)p->in_ld, (cuuint64_t)g.Q};
    cuuint64_t strides[1] = {(cuuint64_t)p->in_ld * 2};
    cuuint32_t box[2] = {SW_BK, SW_FLAT_BOX};
    rc = tc_encode_tiled(&tmX, in, 2, dims, strides, box, false);
  }
  if (rc) return rc;
  {
    const cuuint64_t ktot = (cuuint64_t)9 * p->w_ld;
    cuuint64_t dims[2] = {ktot, (cuuint64_t)p->Cout_pad};
    cuuint64_t strides[1] = {ktot * 2};
    cuuint32_t box[2] = {SW_BK, SW_CO};
    rc = tc_encode_tiled(&tmW, weights, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  {
    // out0: 64-channel boxes of 64 pixels (128-byte swizzle, like the staging chunks); ragged tiles are clipped
    const cuuint64_t cp = (cuuint64_t)p->Cout_pad, ps = (cuuint64_t)p->out0_pix_stride * 2;
    if (g.RP) {
      const int oh = p->out0_halo;
      const cuuint64_t PW2 = (cuuint64_t)(p->W / 2 + 2 * oh);
      const __half* o = reinterpret_cast<const __half*>(p->out0) + (long long)(oh * PW2 + oh) * p->out0_pix_stride;
      cuuint64_t dims[4] = {cp, (cuuint64_t)(p->W / 2), (cuuint64_t)(p->H / 2), (cuuint64_t)p->B};
      cuuint64_t strides[3] = {ps, PW2 * ps, (cuuint64_t)p->out0_img_stride * 2};
      cuuint32_t box[4] = {SW_CO, (cuuint32_t)(g.XB / 2), (cuuint32_t)(g.RP / 2), 1};
      rc = tc_encode_tiled(&tmO, o, 4, dims, strides, box, false);
    } else {
      cuuint64_t dims[2] = {cp, (cuuint64_t)g.Q};
      cuuint64_t strides[1] = {ps};
      cuuint32_t box[2] = {SW_CO, 64};
      rc = tc_encode_tiled(&tmO, p->out0, 2, dims, strides, box, false);
    }
    if (rc) return rc;
  }
  const int smem = stages * stage_bytes + (g.bres ? (int)wres : 0) + SW_FIXED_BYTES;
  static bool smem_set = false;
  if (!smem_set) {
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_tc_swap_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SW_SMEM_LIMIT));
    smem_set = true;
  }
  ODT_CUDA_OK(launch_pdl(conv_tc_swap_kernel, g.num_ptiles < kNumSMs ? g.num_ptiles : kNumSMs, SW_THREADS, smem,
                         (cudaStream_t)stream, tmX, tmW, tmO, g, make_epi(*p)));
  ODT_LAUNCH_OK();
  return ODT_OK;
}

}  // namespace odt

// The transposed-tile plan of a layer (host only; honours ODT_TC_SWAP): 1 when odt_conv2d_f16_tc runs it on the
// 64-cout x 256-pixel tiles of conv_tc_swap.cu, else 0.  *rp = rows per row-block tile (0: halo-flat), *tiles = the
// layer's 256-pixel tiles, *waste_permille = computed positions that are no output pixel, per thousand.
extern "C" int odt_conv_tc_swap_plan(const odt_conv_params* p, int* rp, long long* tiles, int* waste_permille) {
  odt::SwapPlan plan;
  if (!p || !odt::swap_taken(p, &plan)) return 0;
  if (rp) *rp = plan.rp;
  if (tiles) *tiles = plan.ptiles;
  if (waste_permille) {
    const long long computed = plan.ptiles * odt::SW_PIX, useful = (long long)p->B * p->OH * p->OW;
    *waste_permille = (int)((computed - useful) * 1000 / computed);
  }
  return 1;
}
