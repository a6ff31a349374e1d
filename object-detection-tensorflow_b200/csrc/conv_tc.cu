// wgmma / TMA implicit-GEMM forward convolution for sm_90a.
//
//   D[m, n] = sum_{r,s,c} X[b, p*stride - pad + r*dil, q*stride - pad + s*dil, c] * W[n, r, s, c]
//   m = (b, p, q) linearised over B*OH*OW, fp16 operands, fp32 accumulation in registers.
//
// * A operand (activations, NHWC), three feeding modes:
//   - im2col-mode TMA: one load per (filter tap, 64-channel chunk) brings a [128 pixels x 64
//     channels] slab -- 128 consecutive output pixels in B*OH*OW order, wrapping across rows and
//     images, zero-filled where the tap falls into the SAME padding (any filter geometry);
//   - halo-flat (3x3 / stride 1 / N <= 128, input stored with a zero halo): one [136 x 64] slab of
//     consecutive padded positions per (filter row, chunk) feeds the three horizontal taps
//     through row-shifted wgmma descriptors;
//   - row-block (the same shapes + fused 2x2/2 max-pool): RP rows x 128/RP columns per tile, a 4-D
//     tiled box with the row dimension second, the pooling window in four lanes of one warp.
// * B operand (weights, KRSC = K-major): tiled TMA loads [BN x 64], optionally resident in shared
//   memory for small filter banks.
// * MMA: wgmma m64nBNk16 (BN <= 128), both operands from shared memory; two consumer warpgroups,
//   one per 64-row half of the 128-row tile.  A pipeline stage goes back to the producer as soon
//   as the MMAs that read it have retired (one wgmma group kept in flight).
// * Epilogue: the accumulators pass through an fp32 tile in shared memory so that every epilogue
//   lane owns one pixel row, 32 channels at a time: folded bias/BN scale+shift, activation,
//   residual, up to two extra pre-activated outputs, fused max-pool, fp32 head scatter; 128-bit
//   global stores.
// * Persistent: one CTA per SM, static round-robin tile schedule.  Warp 0 = TMA producer (runs
//   ahead across tiles), warps 4..11 = the two consumer warpgroups (MMA, then the epilogue of the
//   same tile; warps 1..3 only pad the producer warpgroup).
//
// ref call sites: tf.nn.conv2d SSD300.py:519; tf.layers.conv2d SSD300.py:524,
// RetinaNet.py:579,599,609, YOLOv3.py:495, FCOS.py:449,469,479.
#include <stdlib.h>
#include <string.h>

#include "epilogue.cuh"
#include "tc_ptx.cuh"

namespace odt {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;
constexpr int TC_MAX_BN = 128;  // N tile (the wgmma accumulators of one 64-row half live in registers)
constexpr int TC_EPI_WARPS = 8;
constexpr int TC_THREADS = 128 + 32 * TC_EPI_WARPS;  // producer warpgroup, two consumer warpgroups
constexpr int TC_EPI_PAR = 7 * 256;               // floats per parameter block: scale/shift/scale2/shift2/column offset/scale3/shift3
constexpr int TC_EPI_SMEM = 2 * TC_EPI_PAR * 4;   // double-buffered
constexpr int TC_MAX_STAGES = 8;
constexpr int TC_A_BYTES = TC_BM * TC_BK * 2;  // 16 KiB
constexpr int TC_SMEM_LIMIT = 232448;          // 227 KiB
constexpr int tc_acc_bytes(int bn) { return TC_BM * (bn + 4) * 4; }  // staged fp32 accumulator tile

struct TcGeom {
  long long M;  // B*OH*OW
  int OH, OW, ohw;
  int R, S, stride, dil;
  int lower_w, lower_h;
  int cchunks;     // in_ld / 64
  int num_m_tiles, num_n_tiles, BN;
  int stages;
  int fast_store;  // 1: fp16 out0, no regroup, 16-byte aligned rows
  int fast_cols;   // columns that may be written by whole 32-column chunks (min channel stride)
  int a_bytes, b_bytes;  // shared memory per pipeline stage
  // halo-flat mode (3x3, stride 1, input stored with a 1-pixel zero halo): M runs over
  // the padded-linear positions, one [136 x 64] slab per (filter row, channel chunk)
  // feeds the three horizontal taps through row-shifted wgmma descriptors
  int flat;
  int PW, PHW;     // padded row length W+2 and padded image size (H+2)*(W+2)
  int H, W;        // real input (= output) size in flat mode
  long long Q;     // B*(H+2)*(W+2)
  int out_halo;    // out0 / residual are stored with a 1-pixel halo
  int head_mode;   // fp32 scatter into candidate rows: one row per store instruction, lanes on consecutive channels
  // row-block flat mode (flat == 2, fused 2x2/2 max pooling): a tile is RP image rows x XB
  // columns (RP*XB = 128); the slab of one filter row is a [XB+2 columns][RP rows][64 ch]
  // box, column-major over the tile so that tap s is the slab shifted by s*RP rows and the
  // four pixels of a pooling window sit in four lanes of one warp
  int RP, lgRP, XB, xblocks, yblocks;
  int a_tx;        // bytes one activation slab load delivers
  // flat modes with a small filter bank: all 9*cchunks weight tiles [BN x 64] stay resident
  // in shared memory (loaded once per CTA); the pipeline stages then carry activations only
  int bres;
  int klast;        // 16-deep K steps of the LAST 64-channel chunk that hold real input channels (1..4); with
                    // ODT_TC_KSKIP=1 the all-zero steps of a thin layer (Cin = 7..48 padded to 64 on both
                    // operands) are not issued (warpgroup-uniform branch); 4 otherwise
};
constexpr int TC_FLAT_ROWS = 136;                    // 128 + 2 neighbours, padded to 1024 B
constexpr int TC_FLAT_A_BYTES = TC_FLAT_ROWS * 128;  // 17408

// Optional per-role timeline of CTA 0 (compile with -DODT_TC_TIMELINE; off in the product build): lane 0 of
// each role stamps clock64 at its hand-over points so that a tile's latency chain (TMA -> MMA -> epilogue)
// can be read off directly.  Entries: (clock, role << 56 | event << 48 | tile).
#ifdef ODT_TC_TIMELINE
__device__ unsigned long long* g_tl_buf = nullptr;
__device__ unsigned int g_tl_cap = 0, g_tl_len = 0;
__device__ __forceinline__ void tl_stamp(int role, int event, int tile) {
  if (blockIdx.x == 0 && (threadIdx.x & 31) == 0 && g_tl_buf) {
    const unsigned int i = atomicAdd(&g_tl_len, 1u);
    if (i < g_tl_cap) {
      g_tl_buf[2 * i] = (unsigned long long)clock64();
      g_tl_buf[2 * i + 1] = ((unsigned long long)role << 56) | ((unsigned long long)event << 48) | (unsigned)tile;
    }
  }
}
#else
#define tl_stamp(role, event, tile) ((void)0)
#endif

// --------------------------------------------------------------- kernel ----
template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
    conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ TcGeom g, const __grid_constant__ Epi e) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve (base rounded up to 1024 for the 128B swizzle atoms)
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const int stages = g.stages;
  const uint32_t a_bytes = (uint32_t)g.a_bytes, b_bytes = (uint32_t)g.b_bytes;
  const uint32_t a_base = base;
  const uint32_t b_base = base + (uint32_t)stages * a_bytes;
  const uint32_t wres_bytes = g.bres ? (uint32_t)(9 * g.cchunks) * (uint32_t)BN * 128u : 0u;
  const uint32_t bar_base = b_base + (uint32_t)stages * b_bytes + wres_bytes;  // 1024-byte aligned
  // barriers: full[stages], empty[stages], then the resident-weights barrier
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (TC_MAX_STAGES + s); };
  const uint32_t wfull_bar = bar_base + 8u * (2 * TC_MAX_STAGES);  // resident weights landed
  // per-tile epilogue parameters staged in smem: [buf][scale|shift|scale2|shift2|offset|scale3|shift3][256]
  float* epi_par = reinterpret_cast<float*>(smem_raw + (bar_base + 256u - raw));
  // the tile's fp32 accumulators, one 128-row tile at a pitch of BN + 4 floats (row reads of float4 per
  // lane hit distinct banks in every quarter-warp phase)
  constexpr int ACC_PITCH = BN + 4;
  float* acc_tile = reinterpret_cast<float*>(smem_raw + (bar_base + 256u + TC_EPI_SMEM - raw));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), TC_EPI_WARPS);  // one arrival per consumer warp
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
        tma_load_2d(b_base + (uint32_t)t * (uint32_t)BN * 128u, &tmB, wfull_bar, t * TC_BK, 0);
    }
    __syncwarp();
  }
  // Programmatic dependent launch: everything above (barrier init, descriptor prefetch, the
  // resident filter bank) overlapped the tail of the previous kernel in the stream; from here
  // on we touch memory it produced.
  pdl_launch_dependents();
  pdl_wait();

  const int num_tiles = g.num_m_tiles * g.num_n_tiles;
  const int kblocks = g.flat ? 3 * g.cchunks : g.R * g.S * g.cchunks;  // pipeline stages per tile

  if (warp == 0) {
    // ===================== TMA producer ======================================
    // The whole warp runs the loop (warp-uniform control flow, operands stay in
    // uniform registers); one elected lane issues the TMA instructions.
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int n_tile = tile % g.num_n_tiles;
      const int m_tile = tile / g.num_n_tiles;
      const long long m0 = (long long)m_tile * TC_BM;
      const int n0 = n_tile * BN;
      tl_stamp(0, 0, tile);  // producer starts the tile's loads
      if (g.flat) {
        // one slab of 136 consecutive padded-linear rows per (filter row, chunk): rows
        // m0 + (r-1)*PW - 1 ...; negative / past-the-end rows are TMA zero fill
        int bb = 0, yq = 0, xq = 0;
        if (g.flat == 2) {
          const int per_img = g.yblocks * g.xblocks;
          bb = m_tile / per_img;
          const int rem = m_tile - bb * per_img;
          yq = rem / g.xblocks;
          xq = rem - yq * g.xblocks;
        }
        for (int r = 0; r < 3; ++r) {
          const int row0 = (int)m0 + (r - 1) * g.PW - 1;
          for (int cc = 0; cc < g.cchunks; ++cc) {
            mbar_wait(empty_bar(stage), phase ^ 1u);
            if (elect_one()) {
              const uint32_t adst = a_base + (uint32_t)stage * a_bytes, bdst = b_base + (uint32_t)stage * b_bytes;
              mbar_expect_tx(full_bar(stage), (uint32_t)g.a_tx + b_bytes);  // b_bytes == 0 when resident
              if (g.flat == 2)  // padded rows RP*yq + r .., padded columns XB*xq .. (+2 for the taps)
                tma_load_4d(adst, &tmA, full_bar(stage), cc * TC_BK, g.RP * yq + r, g.XB * xq, bb);
              else
                tma_load_2d(adst, &tmA, full_bar(stage), cc * TC_BK, row0);
              if (!g.bres) {
#pragma unroll
                for (int s = 0; s < 3; ++s)
                  tma_load_2d(bdst + (uint32_t)s * (uint32_t)BN * 128u, &tmB, full_bar(stage),
                              ((r * 3 + s) * g.cchunks + cc) * TC_BK, n0);
              }
            }
            __syncwarp();
            if (++stage == stages) {
              stage = 0;
              phase ^= 1u;
            }
          }
        }
        continue;
      }
      const int img = (int)(m0 / g.ohw);
      const int rem = (int)(m0 - (long long)img * g.ohw);
      const int p = rem / g.OW, q = rem - p * g.OW;
      const int cw = q * g.stride + g.lower_w, ch = p * g.stride + g.lower_h;
      int kcol = 0;
      for (int r = 0; r < g.R; ++r) {
        for (int s = 0; s < g.S; ++s) {
          for (int cc = 0; cc < g.cchunks; ++cc) {
            mbar_wait(empty_bar(stage), phase ^ 1u);
            if (elect_one()) {
              mbar_expect_tx(full_bar(stage), a_bytes + b_bytes);
              tma_load_im2col(a_base + (uint32_t)stage * a_bytes, &tmA, full_bar(stage),
                              cc * TC_BK, cw, ch, img, (uint16_t)(s * g.dil),
                              (uint16_t)(r * g.dil));
              tma_load_2d(b_base + (uint32_t)stage * b_bytes, &tmB, full_bar(stage), kcol, n0);
            }
            __syncwarp();
            kcol += TC_BK;
            if (++stage == stages) {
              stage = 0;
              phase ^= 1u;
            }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumer warpgroups ===============================
    // MMA: warpgroup `group` computes rows 64*group .. +63 of the tile over all BN columns.
    // Epilogue: warp (group, quarter) owns pixel rows 32*quarter .. +31 (one per lane) and the
    // 32-column chunks j = group, group + 2, ... of the staged accumulator tile.
    const int quarter = warp & 3;
    const int group = (warp - 4) >> 2;
    const int et = threadIdx.x - 128;  // index among the 256 consumer threads
    int staged_n_tile = -1, pbuf = 0;
    int stage = 0;
    uint32_t phase = 0;
    int cc_mma = 0;  // channel chunk of the current k-block (the k-block order ends with the chunk index)
    float acc[BN / 2];
    if (g.bres) mbar_wait(wfull_bar, 0);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int n_tile = tile % g.num_n_tiles;
      const int m_tile = tile / g.num_n_tiles;
      int prev = -1;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint64_t adesc = make_desc_sw128(a_base + (uint32_t)stage * a_bytes + (uint32_t)group * 64u * 128u);
        // resident bank: tile ((r*3 + s)*cchunks + cc) with kb = r*cchunks + cc
        const uint64_t bdesc = make_desc_sw128(
            g.bres ? b_base + (uint32_t)((kb / g.cchunks) * 3 * g.cchunks + kb % g.cchunks) * (uint32_t)BN * 128u
                   : b_base + (uint32_t)stage * b_bytes);
        // 16-deep K steps of this chunk that hold real channels (see TcGeom::klast)
        // (broadcast from lane 0 so that ptxas sees a warp-uniform count)
        const int ksteps = __shfl_sync(0xffffffffu, (cc_mma == g.cchunks - 1) ? g.klast : TC_BK / 16, 0);
        if (++cc_mma == g.cchunks) cc_mma = 0;
        wg_fence();
        if (g.flat) {
          // three horizontal taps from the same slab: operand rows s .. s+63 of the half, i.e. the
          // descriptor start shifted by s*128 B inside the 1024 B swizzle pattern
          const uint64_t bstep = (uint64_t)(((uint32_t)(g.bres ? g.cchunks : 1) * (uint32_t)BN * 128u) >> 4);
          const uint64_t astep = (uint64_t)(g.flat == 2 ? 8 * g.RP : 8);  // rows per tap shift x 128 B >> 4
#pragma unroll
          for (int s3 = 0; s3 < 3; ++s3)
            wg_mma_chunk<BN>(acc, adesc + astep * s3, bdesc + bstep * s3, ksteps, (kb | s3) == 0);
        } else {
          wg_mma_chunk<BN>(acc, adesc, bdesc, ksteps, kb == 0);
        }
        wg_commit();
        wg_wait<1>();  // the previous k-block's MMAs have retired: its stage goes back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (kb == 0 && quarter == 0) tl_stamp(1 + group, 0, tile);  // first stage of the tile issued
        if (++stage == stages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wg_wait<0>();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      if (quarter == 0) tl_stamp(1 + group, 1, tile);  // accumulators complete
      // accumulators -> shared memory, once every consumer warp has finished reading the previous tile
      asm volatile("bar.sync 1, 256;" ::: "memory");
      wg_acc_to_smem<BN>(acc, acc_tile, ACC_PITCH, 64 * group);
      asm volatile("bar.sync 1, 256;" ::: "memory");

      const long long m = (long long)m_tile * TC_BM + quarter * 32 + lane;
      bool row_ok;
      int img, pix;
      long long pool_row = 0;  // element offset of this lane's pooled pixel (flat == 2)
      int pool_q = 0;          // which 8-channel quarter of a 32-column chunk this lane stores
      if (g.flat == 2) {
        const int per_img = g.yblocks * g.xblocks;
        img = m_tile / per_img;
        const int rem = m_tile - img * per_img;
        const int yq = rem / g.xblocks, xq = rem - yq * g.xblocks;
        const int ml = quarter * 32 + lane;
        const int x = g.XB * xq + (ml >> g.lgRP), y = g.RP * yq + (ml & (g.RP - 1));
        row_ok = x < g.W && y < g.H;  // even sizes: a window is valid or invalid as a whole
        pix = 0;
        const int oh = g.out_halo;
        pool_row = (long long)img * e.out0_img_stride +
                   (long long)(((y >> 1) + oh) * ((g.W >> 1) + 2 * oh) + (x >> 1) + oh) * e.out0_pix_stride;
        pool_q = (ml & 1) | (((ml >> g.lgRP) & 1) << 1);
      } else if (g.flat) {
        // padded-linear position -> (image, padded y, padded x); halo positions are not stored
        img = m < g.Q ? (int)(m / g.PHW) : 0;
        const int rem = (int)(m - (long long)img * g.PHW);
        const int yp = rem / g.PW, xp = rem - yp * g.PW;
        row_ok = m < g.Q && yp >= 1 && yp <= g.H && xp >= 1 && xp <= g.W;
        pix = row_ok ? (yp - 1) * g.W + (xp - 1) : 0;
      } else {
        row_ok = m < g.M;
        img = row_ok ? (int)(m / g.ohw) : 0;
        pix = row_ok ? (int)(m - (long long)img * g.ohw) : 0;
      }
      const int n0 = n_tile * BN;
      // stage the per-channel parameters of this N tile once (broadcast reads later);
      // consecutive tiles of single-N-tile layers reuse them
      if (n_tile != staged_n_tile) {
        staged_n_tile = n_tile;
        pbuf ^= 1;
        float* wpar = epi_par + pbuf * TC_EPI_PAR;
        const int c = et;
        const int n = n0 + c;
        const bool ok = c < BN && n < e.Cout;
        wpar[c] = (ok && e.scale) ? __ldg(e.scale + n) : 1.f;
        wpar[256 + c] = (ok && e.shift) ? __ldg(e.shift + n) : 0.f;
        wpar[512 + c] = (ok && e.scale2) ? __ldg(e.scale2 + n) : 1.f;
        wpar[768 + c] = (ok && e.shift2) ? __ldg(e.shift2 + n) : 0.f;
        reinterpret_cast<int*>(wpar)[1024 + c] = ok ? regroup(e, n) : 0;
        wpar[1280 + c] = (ok && e.scale3) ? __ldg(e.scale3 + n) : 1.f;
        wpar[1536 + c] = (ok && e.shift3) ? __ldg(e.shift3 + n) : 0.f;
        asm volatile("bar.sync 3, 256;" ::: "memory");
      }
      const float* par = epi_par + pbuf * TC_EPI_PAR;
      long long o0_row = (long long)img * e.out0_img_stride;
      if (g.out_halo) {
        const int oy = pix / g.OW, ox = pix - oy * g.OW;
        o0_row += (long long)((oy + 1) * (g.OW + 2) + ox + 1) * e.out0_pix_stride;
      } else {
        o0_row += (long long)pix * e.out0_pix_stride;
      }
      const long long o1_row = aux_row(e.out1_img_stride, e.out1_pix_stride, e.out1_halo, g.OW, img, pix);
      const long long o2_row = aux_row(e.out2_img_stride, e.out2_pix_stride, e.out2_halo, g.OW, img, pix);
      const float* my_acc = acc_tile + (quarter * 32 + lane) * ACC_PITCH;
      for (int j = group; j < BN / 32; j += 2) {
        const int nb = n0 + j * 32;
        if (nb >= e.Cout) break;  // fully padded chunk (uniform)
        uint32_t r[32];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const uint4 t = *reinterpret_cast<const uint4*>(my_acc + j * 32 + 4 * i);
          r[4 * i + 0] = t.x;
          r[4 * i + 1] = t.y;
          r[4 * i + 2] = t.z;
          r[4 * i + 3] = t.w;
        }
        if (g.flat == 2) {
          // fused 2x2/2 max pooling: bias/BN + activation, round to fp16, then the maximum over
          // the window's four lanes (vertical neighbour = lane^1, horizontal = lane^RP); each
          // of the four lanes stores one 8-channel quarter of the pooled pixel
          const float4* ps = reinterpret_cast<const float4*>(par + j * 32);
          const float4* ph4 = reinterpret_cast<const float4*>(par + 256 + j * 32);
          uint4 packed[4];
          __half2* ph = reinterpret_cast<__half2*>(packed);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 sc = ps[i], sh = ph4[i];
            ph[2 * i] = __floats2half2_rn(apply_act(fmaf(__uint_as_float(r[4 * i + 0]), sc.x, sh.x), e.act),
                                          apply_act(fmaf(__uint_as_float(r[4 * i + 1]), sc.y, sh.y), e.act));
            ph[2 * i + 1] = __floats2half2_rn(apply_act(fmaf(__uint_as_float(r[4 * i + 2]), sc.z, sh.z), e.act),
                                              apply_act(fmaf(__uint_as_float(r[4 * i + 3]), sc.w, sh.w), e.act));
          }
          uint32_t* pw = reinterpret_cast<uint32_t*>(packed);
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            uint32_t o = __shfl_xor_sync(0xffffffffu, pw[i], 1);
            __half2 a = __hmax2(*reinterpret_cast<__half2*>(&pw[i]), *reinterpret_cast<__half2*>(&o));
            pw[i] = *reinterpret_cast<uint32_t*>(&a);
            o = __shfl_xor_sync(0xffffffffu, pw[i], g.RP);
            a = __hmax2(a, *reinterpret_cast<__half2*>(&o));
            pw[i] = *reinterpret_cast<uint32_t*>(&a);
          }
          const uint4 sel = pool_q == 0 ? packed[0] : pool_q == 1 ? packed[1] : pool_q == 2 ? packed[2] : packed[3];
          if (row_ok && nb + 8 * pool_q < g.fast_cols)
            *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out0) + pool_row + nb + 8 * pool_q) = sel;
        } else if (g.fast_store && nb + 32 <= g.fast_cols) {
          const float4* ps = reinterpret_cast<const float4*>(par + j * 32);
          const float4* ph4 = reinterpret_cast<const float4*>(par + 256 + j * 32);
          float v[32];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 sc = ps[i], sh = ph4[i];
            v[4 * i + 0] = apply_act(fmaf(__uint_as_float(r[4 * i + 0]), sc.x, sh.x), e.act);
            v[4 * i + 1] = apply_act(fmaf(__uint_as_float(r[4 * i + 1]), sc.y, sh.y), e.act);
            v[4 * i + 2] = apply_act(fmaf(__uint_as_float(r[4 * i + 2]), sc.z, sh.z), e.act);
            v[4 * i + 3] = apply_act(fmaf(__uint_as_float(r[4 * i + 3]), sc.w, sh.w), e.act);
          }
          if (row_ok) {
            const long long o0 = o0_row + nb;
            if (e.residual) {
              const uint4* rp =
                  reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(e.residual) + o0);
#pragma unroll
              for (int qd = 0; qd < 4; ++qd) {
                uint4 t = __ldg(rp + qd);
                const __half2* h = reinterpret_cast<const __half2*>(&t);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  float2 f = __half22float2(h[i]);
                  v[qd * 8 + 2 * i] += f.x;
                  v[qd * 8 + 2 * i + 1] += f.y;
                }
              }
            }
            uint4 packed[4];
            __half2* ph = reinterpret_cast<__half2*>(packed);
#pragma unroll
            for (int i = 0; i < 16; ++i) ph[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
            if (e.out0) {
              uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out0) + o0);
#pragma unroll
              for (int qd = 0; qd < 4; ++qd) op[qd] = packed[qd];
            }
            if (e.out1) {
              const float4* ps2 = reinterpret_cast<const float4*>(par + 512 + j * 32);
              const float4* ph2 = reinterpret_cast<const float4*>(par + 768 + j * 32);
              uint4 packed1[4];
              __half2* p1 = reinterpret_cast<__half2*>(packed1);
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 sc = ps2[i], sh = ph2[i];
                const float2 fa = __half22float2(ph[2 * i]);      // consumer sees the rounded value
                const float2 fb = __half22float2(ph[2 * i + 1]);
                p1[2 * i] = __floats2half2_rn(apply_act(fmaf(fa.x, sc.x, sh.x), e.act2),
                                              apply_act(fmaf(fa.y, sc.y, sh.y), e.act2));
                p1[2 * i + 1] = __floats2half2_rn(apply_act(fmaf(fb.x, sc.z, sh.z), e.act2),
                                                  apply_act(fmaf(fb.y, sc.w, sh.w), e.act2));
              }
              uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out1) + o1_row + nb);
#pragma unroll
              for (int qd = 0; qd < 4; ++qd) op[qd] = packed1[qd];
            }
            if (e.out2) {
              const float4* ps3 = reinterpret_cast<const float4*>(par + 1280 + j * 32);
              const float4* ph3 = reinterpret_cast<const float4*>(par + 1536 + j * 32);
              uint4 packed2[4];
              __half2* p2 = reinterpret_cast<__half2*>(packed2);
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float4 sc = ps3[i], sh = ph3[i];
                const float2 fa = __half22float2(ph[2 * i]);
                const float2 fb = __half22float2(ph[2 * i + 1]);
                p2[2 * i] = __floats2half2_rn(apply_act(fmaf(fa.x, sc.x, sh.x), e.act3),
                                              apply_act(fmaf(fa.y, sc.y, sh.y), e.act3));
                p2[2 * i + 1] = __floats2half2_rn(apply_act(fmaf(fb.x, sc.z, sh.z), e.act3),
                                                  apply_act(fmaf(fb.y, sc.w, sh.w), e.act3));
              }
              uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out2) + o2_row + nb);
#pragma unroll
              for (int qd = 0; qd < 4; ++qd) op[qd] = packed2[qd];
            }
          }
        } else if (row_ok || g.head_mode) {
          // generic path: fp32 head outputs scattered into the candidate rows,
          // channel regrouping, ragged Cout; parameters come from shared memory
          const float* ps = par + j * 32;
          const int* pofs = reinterpret_cast<const int*>(par) + 1024 + j * 32;
          const int nvalid = min(32, e.Cout - nb);
          if (g.head_mode) {
            // head convolutions: fp32 scatter into the candidate rows.  The staged accumulator
            // tile is read column-wise, so the warp writes one row per instruction with the
            // lanes on consecutive channels (4-5 sectors per request instead of 32).
            const float* acol = acc_tile + (quarter * 32) * ACC_PITCH + j * 32 + lane;
            const float sc = ps[lane], sh = ps[256 + lane];
            const int my_ofs = pofs[lane];
            const long long my_row = row_ok ? o0_row : -1;
            float* obase = reinterpret_cast<float*>(e.out0);
#pragma unroll 4
            for (int rr = 0; rr < 32; ++rr) {
              const long long orow_r = __shfl_sync(0xffffffffu, my_row, rr);
              const float val = apply_act(fmaf(acol[rr * ACC_PITCH], sc, sh), e.act);
              if (orow_r >= 0 && lane < nvalid) obase[orow_r + my_ofs] = val;
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              if (i >= nvalid) break;
              const int n = nb + i;
              float v = apply_act(fmaf(__uint_as_float(r[i]), ps[i], ps[256 + i]), e.act);
              const long long o0 = o0_row + pofs[i];
              if (e.residual) v += __half2float(reinterpret_cast<const __half*>(e.residual)[o0]);
              if (e.out0) {
                if (e.out0_dtype == ODT_F32) {
                  reinterpret_cast<float*>(e.out0)[o0] = v;
                } else {
                  const __half hv = __float2half_rn(v);
                  reinterpret_cast<__half*>(e.out0)[o0] = hv;
                  v = __half2float(hv);
                }
              }
              if (e.out1)
                reinterpret_cast<__half*>(e.out1)[o1_row + n] =
                    __float2half_rn(apply_act(fmaf(v, ps[512 + i], ps[768 + i]), e.act2));
              if (e.out2)
                reinterpret_cast<__half*>(e.out2)[o2_row + n] =
                    __float2half_rn(apply_act(fmaf(v, ps[1280 + i], ps[1536 + i]), e.act3));
            }
          }
        }
      }
      if (quarter == 0) tl_stamp(1 + group, 2, tile);  // epilogue done
    }
  }
}

// ----------------------------------------------------- host: tensor maps ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                   const cuuint64_t*, const cuuint64_t*, const int*, const int*,
                                   cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

static EncodeTiledFn g_encode_tiled = nullptr;
static EncodeIm2colFn g_encode_im2col = nullptr;

static int resolve_driver() {
  if (g_encode_tiled && g_encode_im2col) return ODT_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  ODT_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  if (!fn || q != cudaDriverEntryPointSuccess) {
    set_error("cuTensorMapEncodeTiled not available from the driver");
    return ODT_ERR_CUDA;
  }
  g_encode_tiled = (EncodeTiledFn)fn;
  fn = nullptr;
  ODT_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &q));
  if (!fn || q != cudaDriverEntryPointSuccess) {
    set_error("cuTensorMapEncodeIm2col not available from the driver");
    return ODT_ERR_CUDA;
  }
  g_encode_im2col = (EncodeIm2colFn)fn;
  return ODT_OK;
}

int tc_encode_tiled(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                    const cuuint32_t* box, bool l2_promote_256) {
  int rc = resolve_driver();
  if (rc) return rc;
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult cr = g_encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims,
                               strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               l2_promote_256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(rank %d) failed (%d)", rank, (int)cr);
    return ODT_ERR_CUDA;
  }
  return ODT_OK;
}

int conv_tapn_try(const void* in, const void* weights, const odt_conv_params* p, void* stream);  // conv_tapn.cu
int conv_thin_try(const void* in, const void* weights, const odt_conv_params* p, void* stream);  // conv_thin.cu
int conv_pw_try(const void* in, const void* weights, const odt_conv_params* p, void* stream);    // conv_pw.cu

int check_conv_params(const odt_conv_params* p) {
  ODT_CHECK_ARG(p != nullptr, "params null");
  ODT_CHECK_ARG(p->B > 0 && p->H > 0 && p->W > 0 && p->Cin > 0 && p->in_ld >= p->Cin,
                "input geometry");
  ODT_CHECK_ARG(p->OH > 0 && p->OW > 0 && p->Cout > 0, "output geometry");
  ODT_CHECK_ARG(p->R > 0 && p->S > 0 && p->stride > 0 && p->dil > 0, "filter geometry");
  ODT_CHECK_ARG(p->w_ld >= p->Cin && p->Cout_pad >= p->Cout, "weight geometry");
  ODT_CHECK_ARG(p->out0 || p->out1 || p->out2, "no output");
  ODT_CHECK_ARG(p->act >= 0 && p->act <= 2 && p->act2 >= 0 && p->act2 <= 2 && p->act3 >= 0 && p->act3 <= 2,
                "activation code");
  ODT_CHECK_ARG(p->out0_dtype == ODT_F16 || p->out0_dtype == ODT_F32, "out0 dtype");
  ODT_CHECK_ARG((p->out1_halo == 0 || p->out1_halo == 1) && (p->out2_halo == 0 || p->out2_halo == 1),
                "out1_halo / out2_halo must be 0 or 1");
  return ODT_OK;
}

}  // namespace odt

using namespace odt;

// N tile of an im2col-mode layer from a two-term cost model:
//   time ~ rounds * (kblocks * (128 + 4*BN) + 2000 + 8*BN),
//   4*BN    = clocks of the 128 x BN x 64 multiply-adds of one K block at the dense fp16 wgmma rate
//             (2048 FMA/clk/SM), 128 = per-K-block barrier and issue overhead,
//   2000 + 8*BN = the epilogue, which the consumer warpgroups run between two tiles,
//   rounds  = tiles per CTA of the slowest SM.
// Small-M layers (FPN P5-P7 towers, SSD extras) come out with narrow tiles spread over many
// SMs, large ones with 128-wide tiles.
static int pick_bn(int cout_pad, int m_tiles, int kblocks) {
  long long best = -1;
  int best_bn = 32;
  for (int bn = TC_MAX_BN; bn >= 32; bn -= 32) {
    if (cout_pad % bn != 0) continue;
    const long long units = (long long)m_tiles * (cout_pad / bn);
    const long long rounds = (units + kNumSMs - 1) / kNumSMs;
    const long long cost = rounds * ((long long)kblocks * (128 + 4 * bn) + 2000 + 8 * bn);
    if (best < 0 || cost < best) {  // ties keep the wider tile (visited first)
      best = cost;
      best_bn = bn;
    }
  }
  return best_bn;
}

extern "C" int odt_conv2d_f16_tc(const void* in, const void* weights, const odt_conv_params* p,
                                 void* stream) {
  int rc = check_conv_params(p);
  if (rc) return rc;
  ODT_CHECK_ARG(in && weights, "null tensor");
  ODT_CHECK_ARG(p->in_ld % 64 == 0, "in_ld must be a multiple of 64 for the tensor-core path");
  ODT_CHECK_ARG(p->w_ld == p->in_ld, "w_ld must equal in_ld");
  ODT_CHECK_ARG(p->Cout_pad % 32 == 0, "Cout_pad must be a multiple of 32");
  ODT_CHECK_ARG(((uintptr_t)in & 15) == 0 && ((uintptr_t)weights & 15) == 0, "16-byte alignment");
  ODT_CHECK_ARG(p->stride <= 8, "stride > 8 unsupported by TMA traversal stride");
  rc = resolve_driver();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;

  // TF SAME upper pads
  const int pad_b = max((p->OH - 1) * p->stride + (p->R - 1) * p->dil + 1 - p->H, 0) - p->pad_t;
  const int pad_r = max((p->OW - 1) * p->stride + (p->S - 1) * p->dil + 1 - p->W, 0) - p->pad_l;
  ODT_CHECK_ARG(pad_b >= 0 && pad_r >= 0, "pad_t/pad_l exceed the SAME total");

  const int ih = p->in_halo ? 1 : 0;  // input stored as [B][H+2][W+2][ld] with zero borders
  ODT_CHECK_ARG(p->in_halo == 0 || p->in_halo == 1, "in_halo must be 0 or 1");
  ODT_CHECK_ARG(p->out0_halo == 0 || p->out0_halo == 1, "out0_halo must be 0 or 1");
  if (pw_mode()) {  // narrow 1x1 layers: staged, sector-coalesced CUDA-core kernel (conv_pw.cu)
    const int rt = conv_pw_try(in, weights, p, stream);
    if (rt != ODT_ERR_UNSUPPORTED) return rt;
  }
  if (thin_mode()) {  // opt-in: very thin layers on CUDA cores with sector-granular traffic (conv_thin.cu)
    const int rt = conv_thin_try(in, weights, p, stream);
    if (rt != ODT_ERR_UNSUPPORTED) return rt;
  }
  if (tapn_mode()) {  // opt-in: narrow 3x3 layers with the horizontal taps folded into N (conv_tapn.cu)
    const int rt = conv_tapn_try(in, weights, p, stream);
    if (rt != ODT_ERR_UNSUPPORTED) return rt;
  }
  TcGeom g;
  memset(&g, 0, sizeof(g));
  g.M = (long long)p->B * p->OH * p->OW;
  g.OH = p->OH;
  g.OW = p->OW;
  g.ohw = p->OH * p->OW;
  g.R = p->R;
  g.S = p->S;
  g.stride = p->stride;
  g.dil = p->dil;
  g.lower_w = -p->pad_l + ih;
  g.lower_h = -p->pad_t + ih;
  g.cchunks = p->in_ld / 64;
  {
    // ODT_TC_KSKIP (default on, carried over from the previous target, not re-measured on the H100): with the knob
    // off every step is issued
    const int rem = p->Cin - (g.cchunks - 1) * TC_BK;  // real channels in the last chunk
    g.klast = !kskip_enabled() || rem >= TC_BK ? TC_BK / 16 : (rem <= 0 ? 1 : (rem + 15) / 16);
  }
  g.out_halo = p->out0_halo;
  g.H = p->H;
  g.W = p->W;
  g.PW = p->W + 2;
  g.PHW = (p->H + 2) * (p->W + 2);
  g.Q = (long long)p->B * g.PHW;
  // halo-flat path: 3x3 / stride 1 / dilation 1 with a halo input and a narrow N
  const bool flat_shape = ih && p->R == 3 && p->S == 3 && p->stride == 1 && p->dil == 1 &&
                          p->pad_t == 1 && p->pad_l == 1 && p->Cout_pad <= 128 &&
                          g.Q < (1ll << 31) - 4096;
  ODT_CHECK_ARG(p->out0_pool == 0 || p->out0_pool == 2, "out0_pool must be 0 or 2");
  if (p->out0_pool) {
    ODT_CHECK_ARG(flat_shape, "fused pooling needs a halo input and a 3x3/stride-1 filter with Cout_pad <= 128");
    ODT_CHECK_ARG(p->OH % 2 == 0 && p->OW % 2 == 0, "fused pooling needs even OH and OW");
    ODT_CHECK_ARG(p->out0 && p->out0_dtype == ODT_F16 && !p->residual && !p->out1 && !p->out2 && p->out0_group == 0,
                  "fused pooling: fp16 out0 only, no residual / out1 / regrouping");
    ODT_CHECK_ARG(p->out0_pix_stride % 8 == 0 && p->out0_img_stride % 8 == 0 &&
                      ((uintptr_t)p->out0 & 15) == 0 && p->out0_pix_stride >= p->Cout_pad,
                  "fused pooling: out0 alignment / channel stride");
  }
  g.flat = p->out0_pool ? 2 : ((flat_shape && flat_enabled()) ? 1 : 0);
  g.a_tx = TC_A_BYTES;
  int stage_bytes;
  if (g.flat == 2) {
    // tile = RP rows x XB columns; take the split that wastes fewer tile positions
    const long long t2 = (long long)((p->OH + 1) / 2) * ((p->OW + 63) / 64);
    const long long t4 = (long long)((p->OH + 3) / 4) * ((p->OW + 31) / 32);
    g.RP = t4 < t2 ? 4 : 2;
    g.lgRP = g.RP == 4 ? 2 : 1;
    g.XB = TC_BM / g.RP;
    g.yblocks = (p->OH + g.RP - 1) / g.RP;
    g.xblocks = (p->OW + g.XB - 1) / g.XB;
    ODT_CHECK_ARG((long long)p->B * g.yblocks * g.xblocks < (1ll << 31), "too many tiles");
    g.num_m_tiles = p->B * g.yblocks * g.xblocks;
    g.BN = p->Cout_pad;
    g.num_n_tiles = 1;
    g.a_bytes = TC_FLAT_A_BYTES;
    g.a_tx = (g.XB + 2) * g.RP * 128;
    g.b_bytes = 3 * g.BN * 128;
  } else if (g.flat) {
    g.a_tx = TC_FLAT_A_BYTES;
    g.num_m_tiles = (int)((g.Q + TC_BM - 1) / TC_BM);
    g.BN = p->Cout_pad;
    g.num_n_tiles = 1;
    g.a_bytes = TC_FLAT_A_BYTES;
    g.b_bytes = 3 * g.BN * 128;
  } else {
    g.num_m_tiles = (int)((g.M + TC_BM - 1) / TC_BM);
    g.BN = pick_bn(p->Cout_pad, g.num_m_tiles, p->R * p->S * g.cchunks);
    g.num_n_tiles = (p->Cout_pad + g.BN - 1) / g.BN;
    g.a_bytes = TC_A_BYTES;
    g.b_bytes = g.BN * 128;
  }
  stage_bytes = g.a_bytes + g.b_bytes;
  g.head_mode = (p->out0 && p->out0_dtype == ODT_F32 && !p->residual && !p->out1 && !p->out2) ? 1 : 0;
  // barriers + 1024-byte alignment slack, epilogue parameters, staged accumulator tile
  const int fixed_bytes = 2048 + TC_EPI_SMEM + tc_acc_bytes(g.BN);
  // small filter banks of the flat modes stay resident in shared memory if at least three
  // activation stages still fit beside them
  const long long wres = 9ll * g.cchunks * g.BN * 128;
  if (g.flat && wres_enabled() && g.BN >= 128 && wres + 3 * TC_FLAT_A_BYTES + fixed_bytes <= TC_SMEM_LIMIT) {
    g.bres = 1;
    g.b_bytes = 0;
    stage_bytes = g.a_bytes;
  }
  int stages = (TC_SMEM_LIMIT - fixed_bytes - (g.bres ? (int)wres : 0)) / stage_bytes;
  if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
  ODT_CHECK_ARG(stages >= 2, "tile too large for shared memory");
  g.stages = stages;
  g.fast_store = (p->out0_dtype == ODT_F16 || !p->out0) && p->out0_group == 0 &&
                 (p->out0_pix_stride % 8 == 0) && (p->out0_img_stride % 8 == 0) &&
                 (!p->out0 || ((uintptr_t)p->out0 & 15) == 0) &&
                 (!p->residual || ((uintptr_t)p->residual & 15) == 0) &&
                 (!p->out1 || (((uintptr_t)p->out1 & 15) == 0 && p->out1_pix_stride % 8 == 0 &&
                               p->out1_img_stride % 8 == 0)) &&
                 (!p->out2 || (((uintptr_t)p->out2 & 15) == 0 && p->out2_pix_stride % 8 == 0 &&
                               p->out2_img_stride % 8 == 0));
  g.fast_cols = p->out0 ? p->out0_pix_stride : (1 << 30);
  if (p->out1 && p->out1_pix_stride < g.fast_cols) g.fast_cols = p->out1_pix_stride;
  if (p->out2 && p->out2_pix_stride < g.fast_cols) g.fast_cols = p->out2_pix_stride;

  CUtensorMap tmA, tmB;
  if (g.flat == 2) {
    // [ld][H+2][W+2][B] view with the ROW dimension second, so that a {64, RP, XB+2, 1} box
    // lands in shared memory column-major over the tile (smem row = column*RP + row)
    const cuuint64_t PH = (cuuint64_t)p->H + 2, PW = (cuuint64_t)p->W + 2;
    cuuint64_t dims[4] = {(cuuint64_t)p->in_ld, PH, PW, (cuuint64_t)p->B};
    cuuint64_t strides[3] = {PW * p->in_ld * 2, (cuuint64_t)p->in_ld * 2, PH * PW * p->in_ld * 2};
    cuuint32_t box[4] = {TC_BK, (cuuint32_t)g.RP, (cuuint32_t)(g.XB + 2), 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult cr = g_encode_tiled(&tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(in), dims,
                                 strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(row-block activations) failed (%d)", (int)cr);
      return ODT_ERR_CUDA;
    }
  } else if (g.flat) {
    // flat [Q][ld] view of the halo tensor, slabs of 136 consecutive padded-linear pixels
    cuuint64_t dims[2] = {(cuuint64_t)p->in_ld, (cuuint64_t)g.Q};
    cuuint64_t strides[1] = {(cuuint64_t)p->in_ld * 2};
    cuuint32_t box[2] = {TC_BK, TC_FLAT_ROWS};
    cuuint32_t estr[2] = {1, 1};
    CUresult cr = g_encode_tiled(&tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(in), dims,
                                 strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(flat activations) failed (%d)", (int)cr);
      return ODT_ERR_CUDA;
    }
  } else {
    const int IW = p->W + 2 * ih, IH = p->H + 2 * ih;
    cuuint64_t dims[4] = {(cuuint64_t)p->in_ld, (cuuint64_t)IW, (cuuint64_t)IH, (cuuint64_t)p->B};
    cuuint64_t strides[3] = {(cuuint64_t)p->in_ld * 2, (cuuint64_t)IW * p->in_ld * 2,
                             (cuuint64_t)IH * IW * p->in_ld * 2};
    // the halo shifts the image origin by one pixel inside the stored tensor
    int lower[2] = {-p->pad_l + ih, -p->pad_t + ih};
    int upper[2] = {pad_r - (p->S - 1) * p->dil - ih, pad_b - (p->R - 1) * p->dil - ih};
    cuuint32_t estr[4] = {1, (cuuint32_t)p->stride, (cuuint32_t)p->stride, 1};
    CUresult cr = g_encode_im2col(&tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(in),
                                  dims, strides, lower, upper, TC_BK, TC_BM, estr,
                                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeIm2col failed (%d): dims %d %d %d %d lower %d %d upper %d %d stride %d",
                (int)cr, p->in_ld, IW, IH, p->B, lower[0], lower[1], upper[0], upper[1], p->stride);
      return ODT_ERR_CUDA;
    }
  }
  {
    const cuuint64_t ktot = (cuuint64_t)p->R * p->S * p->w_ld;
    cuuint64_t dims[2] = {ktot, (cuuint64_t)p->Cout_pad};
    cuuint64_t strides[1] = {ktot * 2};
    cuuint32_t box[2] = {TC_BK, (cuuint32_t)g.BN};
    cuuint32_t estr[2] = {1, 1};
    CUresult cr = g_encode_tiled(&tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                                 const_cast<void*>(weights), dims, strides, box, estr,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(weights) failed (%d)", (int)cr);
      return ODT_ERR_CUDA;
    }
  }

  const int smem = stages * stage_bytes + (g.bres ? (int)wres : 0) + fixed_bytes;
  void (*kern)(CUtensorMap, CUtensorMap, TcGeom, Epi) =
      g.BN == 32 ? conv_tc_kernel<32> : g.BN == 64 ? conv_tc_kernel<64> : g.BN == 96 ? conv_tc_kernel<96>
                                                                                    : conv_tc_kernel<128>;
  ODT_CHECK_ARG(g.BN % 32 == 0 && g.BN <= TC_MAX_BN, "N tile");
  static bool smem_set = false;
  if (!smem_set) {
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<96>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
    smem_set = true;
  }
  Epi e = make_epi(*p);
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  cfg.attrs = attr;
  const int num_tiles = g.num_m_tiles * g.num_n_tiles;
  cfg.gridDim = dim3(num_tiles < kNumSMs ? num_tiles : kNumSMs);
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  ODT_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, g, e));
  ODT_LAUNCH_OK();
  return ODT_OK;
}

// Debug only (see tl_stamp): hands CTA 0's timeline buffer to the kernels; `entries` pairs of u64.
extern "C" int odt_debug_tc_timeline(void* buf, int entries) {
#ifdef ODT_TC_TIMELINE
  unsigned long long* b = static_cast<unsigned long long*>(buf);
  unsigned int cap = (unsigned int)entries, zero = 0;
  ODT_CUDA_OK(cudaMemcpyToSymbol(g_tl_buf, &b, sizeof(b)));
  ODT_CUDA_OK(cudaMemcpyToSymbol(g_tl_cap, &cap, sizeof(cap)));
  ODT_CUDA_OK(cudaMemcpyToSymbol(g_tl_len, &zero, sizeof(zero)));
  return ODT_OK;
#else
  (void)buf;
  (void)entries;
  set_error("built without -DODT_TC_TIMELINE");
  return ODT_ERR_UNSUPPORTED;
#endif
}
