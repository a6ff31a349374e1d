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
//   (Layers of these two modes with Cout_pad = 64 / 128, fp16 out0 alone and enough tiles go to conv_tc_swap.cu, which
//   puts the pixels on the wgmma N side; this kernel keeps the small maps and every other epilogue.)
// * MMA: wgmma m64nBNk16 (BN <= 128), both operands from shared memory.  Two consumer warpgroups
//   in a ping-pong schedule: each owns whole 128-row tiles (two m64 accumulator sets, one per
//   64-row half) and they take alternate tiles of the CTA's list.  An ordering barrier pair makes
//   their mainloops strictly alternate, so one warpgroup's epilogue runs while the other's MMAs
//   keep the tensor pipe busy.  A pipeline stage goes back to the producer as soon as the MMAs
//   that read it have retired (one wgmma group kept in flight).
//   Wide im2col layers (Cout_pad % 256 == 0, where pick_bn's cost model says so) run 128 x 256
//   tiles instead: both warpgroups on every tile, one m64n256k16 per K step on their own 64-row
//   half, each ring stage consumed by both.  A quarter fewer operand bytes per multiply-add reach
//   shared memory, which lifts the feed-bound mainloop to near the dense wgmma rate; the epilogue
//   is then exposed once per tile, shared by all 256 consumer threads.
// * Epilogue, fp16 out0 alone (tmO): folded bias/BN scale+shift and activation on the accumulator
//   registers, rounded to fp16 there (the fused 2x2/2 max-pool: two lane shuffles), 32-column
//   chunks written with stmatrix into a double-buffered, 64-byte-swizzled staging buffer per
//   warpgroup and stored by TMA (one elected thread; the tensor map clips ragged rows / columns).
//   Every other output (residual, up to two extra pre-activated outputs, channel regrouping, fp32
//   head scatter, strides the maps do not cover): the accumulators pass, one 32-column slice at a
//   time, through a per-warpgroup fp32 buffer so that every epilogue lane owns one pixel row.
// * Persistent: one CTA per SM, static round-robin tile schedule.  Warp 0 = TMA producer (runs
//   ahead across tiles; warps 1..3 only pad the producer warpgroup, which hands most of its
//   registers to the consumers with setmaxnreg), warps 4..11 = the two consumer warpgroups.
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
constexpr int TC_MAX_BN = 128;  // N tile (a consumer warpgroup holds the 128 x BN fp32 accumulators in registers)
constexpr int TC_THREADS = 3 * 128;  // producer warpgroup, two consumer warpgroups
// setmaxnreg split of the 64K-register file: 128 * 40 + 256 * 232 <= 65536
constexpr int TC_PRODUCER_REGS = 40;
constexpr int TC_CONSUMER_REGS = 232;
constexpr int TC_EPI_PAR = 7 * TC_MAX_BN;  // floats per parameter block: epi_param's six rows, then the column offsets
// one 32-column slice of a tile's fp32 accumulators at a pitch of 36 floats (row reads of float4 per lane
// hit distinct banks in every quarter-warp phase)
constexpr int TC_SLICE_PITCH = 36;
constexpr int TC_SLICE_FLOATS = TC_BM * TC_SLICE_PITCH;
constexpr int TC_EPI_SMEM = 2 * (TC_EPI_PAR + TC_SLICE_FLOATS) * 4;  // per consumer warpgroup: parameters + slice
// the fp16 output path stages two 32-column chunks (64-byte rows, 64-byte swizzle) per warpgroup in its slice buffer
constexpr int TC_OUT_COLS = 32;
// Wide tile (BN = 256, im2col mode): both consumer warpgroups work on one 128 x 256 tile, warpgroup g on rows
// 64g .. 64g+63 (one m64n256 accumulator set each).  Epilogue: one parameter block of 256 columns shared by the two
// warpgroups, then per warpgroup a [64 rows x 32 columns] slice in which two lanes share a pixel row (16 columns each).
constexpr int TC_WIDE_BN = 256;
constexpr int TC_WIDE_SLICE_FLOATS = (TC_BM / 2) * TC_SLICE_PITCH;
constexpr int TC_WIDE_EPI_SMEM = (7 * TC_WIDE_BN + 2 * TC_WIDE_SLICE_FLOATS) * 4;
constexpr int TC_MAX_STAGES = 8;
constexpr int TC_A_BYTES = TC_BM * TC_BK * 2;  // 16 KiB
constexpr int TC_SMEM_LIMIT = 232448;          // 227 KiB
// named barriers: 1 + g = the 128 threads of consumer warpgroup g; 3 + g = "warpgroup g may start its mainloop"
// (ping-pong); 5 = all 256 consumer threads (the wide tile's shared parameter block)
constexpr int TC_BAR_EPI = 1;
constexpr int TC_BAR_ORDER = 3;
constexpr int TC_BAR_WIDE = 5;

struct TcGeom {
  long long M;  // B*OH*OW
  int OH, OW, ohw;
  int R, S, stride, dil;
  int lower_w, lower_h;
  int cchunks;     // in_ld / 64
  int num_m_tiles, num_n_tiles, BN;
  int stages;
  int tma_out;     // 1: fp16 out0 alone, through the fragment epilogue and the output tensor map
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
  int RP, XB, xblocks, yblocks;
  int a_tx;        // bytes one activation slab load delivers
  // flat modes with a small filter bank: all 9*cchunks weight tiles [BN x 64] stay resident
  // in shared memory (loaded once per CTA); the pipeline stages then carry activations only
  int bres;
  int klast;        // 16-deep K steps of the LAST 64-channel chunk that hold real input channels (1..4): the
                    // all-zero steps of a thin layer (Cin = 7..48 padded to 64 on both operands) are not issued
                    // (warpgroup-uniform branch)
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
// Bound probes of the timeline build (wrong results by design, never in the product library):
//   -DODT_TC_PROBE_FEED: the consumers wait for each stage and hand it back without issuing MMAs (the feed's rate);
//   -DODT_TC_PROBE_MMA:  the producer loads nothing and the consumers do not wait (the MMAs' rate on stale operands).
#if defined(ODT_TC_PROBE_FEED) || defined(ODT_TC_PROBE_MMA)
#ifndef ODT_TC_TIMELINE
#error "the bound probes belong to the -DODT_TC_TIMELINE build"
#endif
#endif
#ifdef ODT_TC_PROBE_FEED
constexpr bool TC_ISSUE_MMA = false;
#else
constexpr bool TC_ISSUE_MMA = true;
#endif
#ifdef ODT_TC_PROBE_MMA
constexpr bool TC_FEED = false;
#else
constexpr bool TC_FEED = true;
#endif

// --------------------------------------------------------------- kernel ----
template <int BN, bool TMA_OUT>
__global__ void __launch_bounds__(TC_THREADS, 1)
    conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmO, const __grid_constant__ TcGeom g,
                   const __grid_constant__ Epi e) {
  constexpr bool WIDE = BN > TC_MAX_BN;  // the cooperative 128 x 256 tile (im2col mode only)
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
  // epilogue region, 1024 bytes past the barriers (the swizzled staging buffers need the alignment): the two
  // consumer warpgroups' accumulator slices, then the parameter blocks [scale|shift|scale2|shift2|scale3|shift3|offset]
  // (one per warpgroup of TC_MAX_BN columns; the wide tile: one of 256 columns)
  const uint32_t epi_base = bar_base + 1024u;
  float* epi_smem = reinterpret_cast<float*>(smem_raw + (epi_base - raw));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    if (TMA_OUT) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmO) : "memory");
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), WIDE ? 8 : 4);  // one arrival per warp of the consuming warpgroup(s)
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

  if (warp < 4) {
    wg_reg_dealloc<TC_PRODUCER_REGS>();
    if (warp != 0) return;
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
            if (TC_FEED) mbar_wait(empty_bar(stage), phase ^ 1u);
            if (TC_FEED && elect_one()) {
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
  } else {
    wg_reg_alloc<TC_CONSUMER_REGS>();
    // ===================== consumer warpgroups ===============================
    // BN <= 128 (ping-pong): warpgroup `group` owns the tiles i = group, group + 2, ... of the CTA's
    // list, all 128 rows (acc[h] = rows 64*h .. +63).  Its mainloop starts once the other warpgroup
    // has issued every MMA of the previous tile, so the k-blocks reach the ring's stages in the
    // producer's order.  Epilogue: warp `quarter` of the group owns pixel rows 32*quarter .. +31
    // (one per lane), 32 columns per slice.
    // BN = 256 (wide): both warpgroups take every tile and consume every stage together, warpgroup
    // `group` on rows 64*group .. +63 (acc[0]).  Epilogue: warps quarter&1 own rows 32*(quarter&1)
    // .. +31 of the group's half, quarter>>1 picks the 16-column half of each 32-column slice.
    constexpr int EW = WIDE ? 16 : 32;               // columns one epilogue lane handles per slice
    constexpr int P = WIDE ? TC_WIDE_BN : TC_MAX_BN;  // parameter block stride
    const int quarter = warp & 3;
    const int group = (warp - 4) >> 2;
    const int et = threadIdx.x - 128 * (1 + group);  // index among the warpgroup's 128 threads
    const int epi_bar = TC_BAR_EPI + group;
    constexpr int SLICE_FLOATS = WIDE ? TC_WIDE_SLICE_FLOATS : TC_SLICE_FLOATS;
    float* slice = epi_smem + group * SLICE_FLOATS;
    float* par = epi_smem + 2 * SLICE_FLOATS + (WIDE ? 0 : group * TC_EPI_PAR);
    // fp16 output staging: two chunk buffers of 128 (wide tile: 64, pooled tile: 32) rows x 64 bytes at the start
    // of the slice buffer (1024-byte aligned); `sbuf` = the one the next chunk goes to (alternates across chunks and
    // tiles)
    int sbuf = 0;
    const int erow = WIDE ? 32 * (quarter & 1) + lane : 32 * quarter + lane;  // this lane's row of the slice
    const int ecol = WIDE ? 16 * (quarter >> 1) : 0;                          // and its first column
    int staged_n_tile = -1;
    int stage = 0;
    uint32_t phase = 0;
    int cc_mma = 0;  // channel chunk of the current k-block (the k-block order ends with the chunk index)
    float acc[WIDE ? 1 : 2][BN / 2];
    if (g.bres) mbar_wait(wfull_bar, 0);
    int i = 0;  // position of `tile` in the CTA's list
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++i) {
      if (!WIDE && (i & 1) != group) {  // the other warpgroup's tile: its k-blocks pass through the ring
        const int adv = stage + kblocks;
        stage = adv % stages;
        phase ^= (uint32_t)(adv / stages) & 1u;
        continue;
      }
      const int n_tile = tile % g.num_n_tiles;
      const int m_tile = tile / g.num_n_tiles;
      if (!WIDE && i > 0) named_bar_sync(TC_BAR_ORDER + group, 256);
      if (quarter == 0) tl_stamp(1 + group, 0, tile);  // mainloop start
      int prev = -1;
      for (int kb = 0; kb < kblocks; ++kb) {
        if (TC_FEED) mbar_wait(full_bar(stage), phase);
        const uint32_t a_stage = a_base + (uint32_t)stage * a_bytes;
        // 16-deep K steps of this chunk that hold real channels (see TcGeom::klast)
        // (broadcast from lane 0 so that ptxas sees a warp-uniform count)
        const int ksteps = __shfl_sync(0xffffffffu, (cc_mma == g.cchunks - 1) ? g.klast : TC_BK / 16, 0);
        if (++cc_mma == g.cchunks) cc_mma = 0;
        if (TC_ISSUE_MMA) {
          wg_fence();
          if constexpr (WIDE) {
            wg_mma_chunk<BN>(acc[0], make_desc_sw128(a_stage + (uint32_t)group * 64u * 128u),
                             make_desc_sw128(b_base + (uint32_t)stage * b_bytes), ksteps, kb == 0);
          } else {
            const uint64_t adesc0 = make_desc_sw128(a_stage), adesc1 = make_desc_sw128(a_stage + 64u * 128u);
            // resident bank: tile ((r*3 + s)*cchunks + cc) with kb = r*cchunks + cc
            const uint64_t bdesc = make_desc_sw128(
                g.bres ? b_base + (uint32_t)((kb / g.cchunks) * 3 * g.cchunks + kb % g.cchunks) * (uint32_t)BN * 128u
                       : b_base + (uint32_t)stage * b_bytes);
            if (g.flat) {
              // three horizontal taps from the same slab: operand rows s .. s+63 of the half, i.e. the
              // descriptor start shifted by s*128 B inside the 1024 B swizzle pattern
              const uint64_t bstep = (uint64_t)(((uint32_t)(g.bres ? g.cchunks : 1) * (uint32_t)BN * 128u) >> 4);
              const uint64_t astep = (uint64_t)(g.flat == 2 ? 8 * g.RP : 8);  // rows per tap shift x 128 B >> 4
#pragma unroll
              for (int s3 = 0; s3 < 3; ++s3)
                wg_mma_chunk2<BN>(acc[0], acc[1], adesc0 + astep * s3, adesc1 + astep * s3, bdesc + bstep * s3,
                                  ksteps, (kb | s3) == 0);
            } else {
              wg_mma_chunk2<BN>(acc[0], acc[1], adesc0, adesc1, bdesc, ksteps, kb == 0);
            }
          }
        }
        wg_commit();
        wg_wait<1>();  // the previous k-block's MMAs have retired: its stage goes back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == stages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      // every MMA of this tile is issued: the other warpgroup's mainloop may start
      if (!WIDE && tile + (int)gridDim.x < num_tiles) named_bar_arrive(TC_BAR_ORDER + (group ^ 1), 256);
      wg_wait<0>();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      if (quarter == 0) tl_stamp(1 + group, 1, tile);  // accumulators complete

      const int n0 = n_tile * BN;
      // the per-channel parameters of this N tile are staged once (broadcast reads later);
      // consecutive tiles of single-N-tile layers reuse them
      const bool new_par = n_tile != staged_n_tile;
      staged_n_tile = n_tile;
      if (WIDE && new_par) {
        // the shared block: both warpgroups have finished reading the previous one, then stage column t
        const int t = threadIdx.x - 128;
        named_bar_sync(TC_BAR_WIDE, 256);
#pragma unroll
        for (int row = 0; row < 6; ++row) par[row * P + t] = epi_param(e, row, n0 + t);
        reinterpret_cast<int*>(par)[6 * P + t] = n0 + t < e.Cout ? regroup(e, n0 + t) : 0;
        named_bar_sync(TC_BAR_WIDE, 256);
      }
      if constexpr (TMA_OUT) {
        // ---- fp16 out0 alone: epilogue on the accumulator fragments, TMA stores of staged 32-column chunks ----
        // This thread's fragment rows: 64*h + 16*quarter + lane/4 + 8*k of the warpgroup's rows (acc[h], k = register
        // pair), its columns 8*i + 2*(lane%4) + {0,1} of each 32-column chunk.
        constexpr int HALVES = WIDE ? 1 : 2;
        const int m0 = m_tile * TC_BM + (WIDE ? 64 * group : 0);  // TMA coordinates are 32-bit
        const int lr = lane >> 2;
        if (!WIDE && new_par) {
          // this warpgroup's reads of the previous block ended before the barrier of its last chunk
          const int n = et < BN ? n0 + et : e.Cout;  // columns past the tile: identity
          par[et] = epi_param(e, 0, n);
          par[P + et] = epi_param(e, 1, n);
          named_bar_sync(epi_bar, 128);
        }
        // halo-flat: the rows of border positions are stored as zeros (bit 2*h + k set: interior)
        uint32_t keep = 0xFu;
        if (g.flat == 1) {
          keep = 0u;
#pragma unroll
          for (int h = 0; h < HALVES; ++h)
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              // Q < 2^31 - 4096 in this mode: 32-bit arithmetic
              const unsigned m = (unsigned)(m0 + 64 * h + 16 * quarter + lr + 8 * k);
              const unsigned rem = m % (unsigned)g.PHW;
              const int yp = (int)(rem / (unsigned)g.PW), xp = (int)(rem % (unsigned)g.PW);
              if (yp >= 1 && yp <= g.H && xp >= 1 && xp <= g.W) keep |= 1u << (2 * h + k);
            }
        }
        // row-block pooled tile: tile row ml = RP*x + y, its window partners ml^1 and ml^RP sit in lanes ^4 and
        // ^(4*RP); lanes with lr & (1|RP) == 0 keep the window's maximum.  Pooled pixel (x/2, y/2) is row
        // (y/2)*(XB/2) + x/2 of the staged chunk (the {32, XB/2, RP/2, 1} box).
#pragma unroll
        for (int j = 0; j < BN / TC_OUT_COLS; ++j) {
          if (n0 + j * TC_OUT_COLS >= e.Cout) break;  // fully padded chunk (uniform)
          const uint32_t buf = smem_u32(slice) + (uint32_t)(sbuf * (g.flat == 2 ? 32 : (WIDE ? 64 : 128)) * 64);
#pragma unroll
          for (int h = 0; h < HALVES; ++h) {
            uint32_t hv[8];  // [2*i + k]: the half2 of column pair i on row k
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float* f = acc[h] + 4 * (4 * j + i);
              const float* pc = par + 32 * j + 8 * i + 2 * (lane & 3);
              const float2 sc = *reinterpret_cast<const float2*>(pc);
              const float2 sh = *reinterpret_cast<const float2*>(pc + P);
#pragma unroll
              for (int k = 0; k < 2; ++k) {
                __half2 v = epi_act_f16x2(f[2 * k], f[2 * k + 1], sc, sh, e.act);
                hv[2 * i + k] = ((keep >> (2 * h + k)) & 1u) ? *reinterpret_cast<uint32_t*>(&v) : 0u;
              }
            }
            if (!WIDE && g.flat == 2) {
              // the window maximum of the rounded values (the fp16 maximum the stand-alone pool takes)
#pragma unroll
              for (int q = 0; q < 8; ++q) {
                uint32_t o = __shfl_xor_sync(0xffffffffu, hv[q], 4);
                __half2 a = __hmax2(*reinterpret_cast<__half2*>(&hv[q]), *reinterpret_cast<__half2*>(&o));
                uint32_t au = *reinterpret_cast<uint32_t*>(&a);
                o = __shfl_xor_sync(0xffffffffu, au, 4 * g.RP);
                a = __hmax2(a, *reinterpret_cast<__half2*>(&o));
                hv[q] = *reinterpret_cast<uint32_t*>(&a);
              }
              if ((lr & (1 | g.RP)) == 0) {
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                  const int ml = 64 * h + 16 * quarter + 8 * k + lr;
                  const int prow = g.RP == 2 ? ml >> 2 : ((ml >> 1) & 1) * 16 + (ml >> 3);
#pragma unroll
                  for (int i = 0; i < 4; ++i)
                    st_shared_u32(buf + (uint32_t)(prow * 64 + ((i ^ ((prow >> 1) & 3)) << 4) + 4 * (lane & 3)),
                                  hv[2 * i + k]);
                }
              }
            } else {
              // 64-byte swizzle: 16-byte piece c of row r at r*64 + ((c ^ (r/2 % 4)) * 16)
              const int mi = lane >> 3;
              const int row = 64 * h + 16 * quarter + (lane & 7) + 8 * (mi & 1);
#pragma unroll
              for (int s2 = 0; s2 < 2; ++s2) {
                const int c = 2 * s2 + (mi >> 1);
                stmatrix_x4(buf + (uint32_t)(row * 64 + ((c ^ ((row >> 1) & 3)) << 4)), hv[4 * s2], hv[4 * s2 + 1],
                            hv[4 * s2 + 2], hv[4 * s2 + 3]);
              }
            }
          }
          fence_proxy_async_smem();
          if (et == 0) bulk_wait_read<0>();  // the previous chunk's store has read the buffer the next chunk takes
          named_bar_sync(epi_bar, 128);
          if (et == 0) {
            if (!WIDE && g.flat == 2) {
              const int per_img = g.yblocks * g.xblocks;
              const int im = m_tile / per_img, rem = m_tile - im * per_img;
              const int yq = rem / g.xblocks, xq = rem - yq * g.xblocks;
              tma_store_4d(&tmO, buf, j * TC_OUT_COLS, (g.XB >> 1) * xq, (g.RP >> 1) * yq, im);
            } else {
              tma_store_2d(&tmO, buf, n0 + j * TC_OUT_COLS, m0);
            }
            bulk_commit();
          }
          sbuf ^= 1;
        }
      } else {
        // ---- staged path: every output through the per-warpgroup fp32 slice, one pixel row per lane ----
        const long long m = (long long)m_tile * TC_BM + (WIDE ? 64 * group : 0) + erow;
        bool row_ok;
        int img, pix;
        if (g.flat) {
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
        long long o0_row = (long long)img * e.out0_img_stride;
        if (g.out_halo) {
          const int oy = pix / g.OW, ox = pix - oy * g.OW;
          o0_row += (long long)((oy + 1) * (g.OW + 2) + ox + 1) * e.out0_pix_stride;
        } else {
          o0_row += (long long)pix * e.out0_pix_stride;
        }
        const long long o1_row = aux_row(e.out1_img_stride, e.out1_pix_stride, e.out1_halo, g.OW, img, pix);
        const long long o2_row = aux_row(e.out2_img_stride, e.out2_pix_stride, e.out2_halo, g.OW, img, pix);
        const float* my_acc = slice + erow * TC_SLICE_PITCH + ecol;
        for (int j = 0; j < BN / 32; ++j) {
          if (n0 + j * 32 >= e.Cout) break;  // fully padded chunk (uniform)
          const int nb = n0 + j * 32 + ecol;  // this lane's first column
          // every lane of the warpgroup has finished reading the previous slice and, on a new tile, the parameters
          named_bar_sync(epi_bar, 128);
          if (!WIDE && j == 0 && new_par) {
            const int n = et < BN ? n0 + et : e.Cout;  // columns past the tile: identity
#pragma unroll
            for (int row = 0; row < 6; ++row) par[row * P + et] = epi_param(e, row, n);
            reinterpret_cast<int*>(par)[6 * P + et] = n < e.Cout ? regroup(e, n) : 0;
          }
          if constexpr (WIDE) {
            wg_acc_slice_to_smem<BN>(acc[0], j, slice, TC_SLICE_PITCH, 0);
          } else {
            wg_acc_slice_to_smem<BN>(acc[0], j, slice, TC_SLICE_PITCH, 0);
            wg_acc_slice_to_smem<BN>(acc[1], j, slice, TC_SLICE_PITCH, 64);
          }
          named_bar_sync(epi_bar, 128);
          float v[32];
#pragma unroll
          for (int i = 0; i < EW / 4; ++i) {
            const float4 t = *reinterpret_cast<const float4*>(my_acc + 4 * i);
            v[4 * i + 0] = t.x;
            v[4 * i + 1] = t.y;
            v[4 * i + 2] = t.z;
            v[4 * i + 3] = t.w;
          }
          const float* ps = par + j * 32 + ecol;  // this lane's parameter columns
          if (g.fast_store && nb + EW <= g.fast_cols) {
            if (row_ok) {
              const long long o0 = o0_row + nb;
              const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(e.residual) + o0);
              epi_store_f16<EW / 8>(e, v, ps, P, [&](int q) { return __ldg(rp + q); }, o0, o1_row + nb, o2_row + nb);
            }
          } else if (row_ok || g.head_mode) {
            // generic path: fp32 head outputs scattered into the candidate rows,
            // channel regrouping, ragged Cout; parameters come from shared memory
            const int* pofs = reinterpret_cast<const int*>(par) + 6 * P + j * 32 + ecol;
            const int nvalid = min(EW, e.Cout - nb);
            if (g.head_mode) {
              // head convolutions: fp32 scatter into the candidate rows.  The staged accumulator
              // slice is read column-wise, so the warp writes one row per instruction with the
              // lanes on consecutive channels (4-5 sectors per request instead of 32).
              const int cl = lane < EW ? lane : 0;  // this lane's column (lanes past EW store nothing)
              const float* acol = slice + (erow - lane) * TC_SLICE_PITCH + ecol + cl;
              const float sc = ps[cl], sh = ps[P + cl];
              const int my_ofs = pofs[cl];
              const long long my_row = row_ok ? o0_row : -1;
              float* obase = reinterpret_cast<float*>(e.out0);
#pragma unroll 4
              for (int rr = 0; rr < 32; ++rr) {
                const long long orow_r = __shfl_sync(0xffffffffu, my_row, rr);
                const float val = apply_act(fmaf(acol[rr * TC_SLICE_PITCH], sc, sh), e.act);
                if (orow_r >= 0 && lane < nvalid) obase[orow_r + my_ofs] = val;
              }
            } else {
#pragma unroll
              for (int i = 0; i < EW; ++i) {
                if (i >= nvalid) break;
                const int n = nb + i;
                float x = apply_act(fmaf(v[i], ps[i], ps[P + i]), e.act);
                const long long o0 = o0_row + pofs[i];
                if (e.residual) x += __half2float(reinterpret_cast<const __half*>(e.residual)[o0]);
                if (e.out0 && e.out0_dtype == ODT_F32) {
                  reinterpret_cast<float*>(e.out0)[o0] = x;
                } else {
                  // out1 / out2 take the rounded value, as epi_store_f16 does, whether or not out0 is stored
                  const __half hv = __float2half_rn(x);
                  if (e.out0) reinterpret_cast<__half*>(e.out0)[o0] = hv;
                  x = __half2float(hv);
                }
                if (e.out1)
                  reinterpret_cast<__half*>(e.out1)[o1_row + n] =
                      __float2half_rn(apply_act(fmaf(x, ps[2 * P + i], ps[3 * P + i]), e.act2));
                if (e.out2)
                  reinterpret_cast<__half*>(e.out2)[o2_row + n] =
                      __float2half_rn(apply_act(fmaf(x, ps[4 * P + i], ps[5 * P + i]), e.act3));
              }
            }
          }
        }
      }
      if (quarter == 0) tl_stamp(1 + group, 2, tile);  // epilogue done
    }
    // the shared-memory sources of the last output stores stay valid until the stores are done
    if (TMA_OUT && et == 0) bulk_wait<0>();
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
                    const cuuint32_t* box, bool l2_promote_256, CUtensorMapSwizzle swizzle) {
  int rc = resolve_driver();
  if (rc) return rc;
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult cr = g_encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims,
                               strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                               l2_promote_256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(rank %d) failed (%d)", rank, (int)cr);
    return ODT_ERR_CUDA;
  }
  return ODT_OK;
}

int tc_encode_im2col(CUtensorMap* map, const void* base, const cuuint64_t* dims, const cuuint64_t* strides,
                     const int* lower, const int* upper, cuuint32_t channels, cuuint32_t pixels, int stride) {
  int rc = resolve_driver();
  if (rc) return rc;
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult cr = g_encode_im2col(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, lower,
                                upper, channels, pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeIm2col failed (%d): dims %d %d %d %d lower %d %d upper %d %d stride %d", (int)cr,
              (int)dims[0], (int)dims[1], (int)dims[2], (int)dims[3], lower[0], lower[1], upper[0], upper[1], stride);
    return ODT_ERR_CUDA;
  }
  return ODT_OK;
}

int tc_rowblock_rp(int OH, int OW, long long* tiles) {
  const long long t2 = (long long)((OH + 1) / 2) * ((OW + 63) / 64);
  const long long t4 = (long long)((OH + 3) / 4) * ((OW + 31) / 32);
  *tiles = t4 < t2 ? t4 : t2;
  return t4 < t2 ? 4 : 2;
}

int conv_swap_try(const void* in, const void* weights, const odt_conv_params* p, void* stream);  // conv_tc_swap.cu
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
//   time ~ rounds * max(mma, epi) + epi,   mma = kblocks * (128 + 4*BN),   epi = 2000 + 8*BN,
//   4*BN    = clocks of the 128 x BN x 64 multiply-adds of one K block at the dense fp16 wgmma rate
//             (2048 FMA/clk/SM), 128 = per-K-block barrier and issue overhead,
//   epi     = the epilogue of one tile; with the ping-pong consumers it runs under the other
//             warpgroup's mainloop, so a round costs the longer of the two and only the CTA's
//             last epilogue is exposed,
//   rounds  = tiles per CTA of the slowest SM.
// The constants are estimates from the instruction counts, not measured on the H100 (nor refitted to the
// fp16 output path of the fragment epilogue).
// Small-M layers (FPN P5-P7 towers, SSD extras) come out with narrow tiles spread over many
// SMs, large ones with 128-wide tiles.
//
// The 128 x 256 tile (Cout_pad % 256 == 0) is then weighed against the chosen narrow tile in
// clocks measured with scripts/tc_timeline.py (CTA 0, conv4_2 38x38 512->512 and conv7 19x19
// 1024->1024 1x1 at B = 64; H100 SXM, 400 W power limit):
//   narrow = rounds * max(mma, epi) + epi,   wide = rounds * (mma + epi)   (its epilogue is exposed),
//   mma    = kblocks * clk per K block: 1015 for 128 x 128 x 64 (operand-feed bound: the dense
//            rate would be 512; scaled by BN/128 below 128), 1085 for 128 x 256 x 64 (dense: 1024),
//   epi    = 16500 clk for a 128 x 128 tile on 128 threads, 15000 for 128 x 256 on 256 threads.
constexpr long long TC_KB_CLK_128 = 1015, TC_KB_CLK_256 = 1085, TC_EPI_CLK = 16500, TC_EPI_CLK_256 = 15000;
static int pick_bn(int cout_pad, int m_tiles, int kblocks) {
  long long best = -1;
  int best_bn = 32;
  for (int bn = TC_MAX_BN; bn >= 32; bn -= 32) {
    if (cout_pad % bn != 0) continue;
    const long long units = (long long)m_tiles * (cout_pad / bn);
    const long long rounds = (units + kNumSMs - 1) / kNumSMs;
    const long long mma = (long long)kblocks * (128 + 4 * bn), epi = 2000 + 8 * bn;
    const long long cost = rounds * (mma > epi ? mma : epi) + epi;
    if (best < 0 || cost < best) {  // ties keep the wider tile (visited first)
      best = cost;
      best_bn = bn;
    }
  }
  const int wide = wide_mode();
  if (wide == 0 || cout_pad % TC_WIDE_BN != 0) return best_bn;
  if (wide == 2) return TC_WIDE_BN;
  auto rounds = [&](int bn) { return ((long long)m_tiles * (cout_pad / bn) + kNumSMs - 1) / kNumSMs; };
  const long long mma_n = (long long)kblocks * TC_KB_CLK_128 * best_bn / 128, epi_n = TC_EPI_CLK * best_bn / 128;
  const long long narrow = rounds(best_bn) * (mma_n > epi_n ? mma_n : epi_n) + epi_n;
  const long long wide_cost = rounds(TC_WIDE_BN) * ((long long)kblocks * TC_KB_CLK_256 + TC_EPI_CLK_256);
  return wide_cost < narrow ? TC_WIDE_BN : best_bn;
}

// The N tile conv_tc picks for an im2col-mode layer (see pick_bn); lets tests and scripts read the plan.
extern "C" int odt_conv_tc_pick_bn(int cout_pad, long long M, int kblocks) {
  return pick_bn(cout_pad, (int)((M + TC_BM - 1) / TC_BM), kblocks);
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
  if (thin_mode()) {  // very thin layers on CUDA cores with sector-granular traffic (conv_thin.cu)
    const int rt = conv_thin_try(in, weights, p, stream);
    if (rt != ODT_ERR_UNSUPPORTED) return rt;
  }
  if (tapn_mode()) {  // narrow 3x3 layers with the horizontal taps folded into N (conv_tapn.cu)
    const int rt = conv_tapn_try(in, weights, p, stream);
    if (rt != ODT_ERR_UNSUPPORTED) return rt;
  }
  {  // narrow 3x3 halo layers with enough tiles: pixels on the wgmma N side (conv_tc_swap.cu; ODT_TC_SWAP)
    const int rt = conv_swap_try(in, weights, p, stream);
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
    const int rem = p->Cin - (g.cchunks - 1) * TC_BK;  // real channels in the last chunk
    g.klast = rem >= TC_BK ? TC_BK / 16 : (rem <= 0 ? 1 : (rem + 15) / 16);
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
  g.flat = p->out0_pool ? 2 : (flat_shape ? 1 : 0);
  g.a_tx = TC_A_BYTES;
  int stage_bytes;
  if (g.flat == 2) {
    long long tiles_per_img;
    g.RP = tc_rowblock_rp(p->OH, p->OW, &tiles_per_img);
    g.XB = TC_BM / g.RP;
    g.yblocks = (p->OH + g.RP - 1) / g.RP;
    g.xblocks = (p->OW + g.XB - 1) / g.XB;
    ODT_CHECK_ARG(p->B * tiles_per_img < (1ll << 31), "too many tiles");
    g.num_m_tiles = (int)(p->B * tiles_per_img);
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
  // barriers + 1024-byte alignment slack, per consumer warpgroup: epilogue parameters + accumulator slice
  // (the wide tile: one shared parameter block + two 64-row slices)
  // (the staging buffers of the fp16 output path reuse the slices)
  const int fixed_bytes = 2048 + (g.BN > TC_MAX_BN ? TC_WIDE_EPI_SMEM : TC_EPI_SMEM);
  // small filter banks of the flat modes stay resident in shared memory if at least three
  // activation stages still fit beside them
  const long long wres = 9ll * g.cchunks * g.BN * 128;
  if (g.flat && g.BN >= 128 && wres + 3 * TC_FLAT_A_BYTES + fixed_bytes <= TC_SMEM_LIMIT) {
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
  // fp16 out0 alone, in a layout one output tensor map covers: the fragment epilogue with TMA stores.  Rows of the
  // im2col / halo-flat tile are consecutive output rows of the map, so the halo-flat output must keep its halo and
  // the im2col output must not have one; images must be stored back to back.
  const long long pix = p->out0_pix_stride;
  g.tma_out = p->out0 && p->out0_dtype == ODT_F16 && !p->residual && !p->out1 && !p->out2 && p->out0_group == 0 &&
              f16_rows_aligned(p->out0, p->out0_img_stride, p->out0_pix_stride, p->Cout_pad) &&
              (g.flat == 2 ||
               (g.flat == 1 && p->out0_halo == 1 && p->out0_img_stride == (long long)g.PHW * pix) ||
               (g.flat == 0 && p->out0_halo == 0 && p->out0_img_stride == (long long)g.ohw * pix));
  ODT_CHECK_ARG(g.flat != 2 || g.tma_out, "fused pooling: out0 layout");
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
    rc = tc_encode_tiled(&tmA, in, 4, dims, strides, box, false);
  } else if (g.flat) {
    // flat [Q][ld] view of the halo tensor, slabs of 136 consecutive padded-linear pixels
    cuuint64_t dims[2] = {(cuuint64_t)p->in_ld, (cuuint64_t)g.Q};
    cuuint64_t strides[1] = {(cuuint64_t)p->in_ld * 2};
    cuuint32_t box[2] = {TC_BK, TC_FLAT_ROWS};
    rc = tc_encode_tiled(&tmA, in, 2, dims, strides, box, false);
  } else {
    const int IW = p->W + 2 * ih, IH = p->H + 2 * ih;
    cuuint64_t dims[4] = {(cuuint64_t)p->in_ld, (cuuint64_t)IW, (cuuint64_t)IH, (cuuint64_t)p->B};
    cuuint64_t strides[3] = {(cuuint64_t)p->in_ld * 2, (cuuint64_t)IW * p->in_ld * 2,
                             (cuuint64_t)IH * IW * p->in_ld * 2};
    // the halo shifts the image origin by one pixel inside the stored tensor
    int lower[2] = {-p->pad_l + ih, -p->pad_t + ih};
    int upper[2] = {pad_r - (p->S - 1) * p->dil - ih, pad_b - (p->R - 1) * p->dil - ih};
    rc = tc_encode_im2col(&tmA, in, dims, strides, lower, upper, TC_BK, TC_BM, p->stride);
  }
  if (rc) return rc;
  {
    const cuuint64_t ktot = (cuuint64_t)p->R * p->S * p->w_ld;
    cuuint64_t dims[2] = {ktot, (cuuint64_t)p->Cout_pad};
    cuuint64_t strides[1] = {ktot * 2};
    cuuint32_t box[2] = {TC_BK, (cuuint32_t)g.BN};
    rc = tc_encode_tiled(&tmB, weights, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  // out0 of the fp16 output path: 32-column boxes (64-byte swizzle, like the staging buffers), columns up to Cout_pad
  CUtensorMap tmO;
  memset(&tmO, 0, sizeof(tmO));
  if (g.tma_out) {
    const cuuint64_t cp = (cuuint64_t)p->Cout_pad, ps = (cuuint64_t)pix * 2;
    if (g.flat == 2) {
      // [B][H/2][W/2] interior of the pooled tensor (a halo shifts the origin by one row and one column), box = the
      // tile's 32 pooled pixels; ragged column / row blocks are clipped at W/2 / H/2
      const int oh = p->out0_halo;
      const cuuint64_t PW2 = (cuuint64_t)(p->W / 2 + 2 * oh);
      const __half* o = reinterpret_cast<const __half*>(p->out0) + (long long)(oh * PW2 + oh) * pix;
      cuuint64_t dims[4] = {cp, (cuuint64_t)(p->W / 2), (cuuint64_t)(p->H / 2), (cuuint64_t)p->B};
      cuuint64_t strides[3] = {ps, PW2 * ps, (cuuint64_t)p->out0_img_stride * 2};
      cuuint32_t box[4] = {TC_OUT_COLS, (cuuint32_t)(g.XB / 2), (cuuint32_t)(g.RP / 2), 1};
      rc = tc_encode_tiled(&tmO, o, 4, dims, strides, box, false, CU_TENSOR_MAP_SWIZZLE_64B);
    } else {
      // [rows][Cout_pad]: the output positions (im2col) or padded-linear positions (halo-flat); rows past the end
      // are clipped.  The wide tile stores each warpgroup's 64-row half.
      cuuint64_t dims[2] = {cp, (cuuint64_t)(g.flat ? g.Q : g.M)};
      cuuint64_t strides[1] = {ps};
      cuuint32_t box[2] = {TC_OUT_COLS, (cuuint32_t)(g.BN > TC_MAX_BN ? TC_BM / 2 : TC_BM)};
      rc = tc_encode_tiled(&tmO, p->out0, 2, dims, strides, box, false, CU_TENSOR_MAP_SWIZZLE_64B);
    }
    if (rc) return rc;
  }

  const int smem = stages * stage_bytes + (g.bres ? (int)wres : 0) + fixed_bytes;
  ODT_CHECK_ARG(g.BN % 32 == 0 && (g.BN <= TC_MAX_BN || (g.BN == TC_WIDE_BN && !g.flat)), "N tile");
  // the two epilogues are separate instantiations: each gets the register allocation of its own path
  typedef void (*Kern)(CUtensorMap, CUtensorMap, CUtensorMap, TcGeom, Epi);
  static const Kern kerns[2][5] = {
      {conv_tc_kernel<32, false>, conv_tc_kernel<64, false>, conv_tc_kernel<96, false>, conv_tc_kernel<128, false>,
       conv_tc_kernel<TC_WIDE_BN, false>},
      {conv_tc_kernel<32, true>, conv_tc_kernel<64, true>, conv_tc_kernel<96, true>, conv_tc_kernel<128, true>,
       conv_tc_kernel<TC_WIDE_BN, true>}};
  static bool smem_set = false;
  if (!smem_set) {
    for (int t = 0; t < 2; ++t)
      for (int b = 0; b < 5; ++b)
        ODT_CUDA_OK(cudaFuncSetAttribute(kerns[t][b], cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
    smem_set = true;
  }
  static const char* const names[2][5] = {
      {"conv_tc_kernel<32,false>", "conv_tc_kernel<64,false>", "conv_tc_kernel<96,false>", "conv_tc_kernel<128,false>",
       "conv_tc_kernel<256,false>"},
      {"conv_tc_kernel<32,true>", "conv_tc_kernel<64,true>", "conv_tc_kernel<96,true>", "conv_tc_kernel<128,true>",
       "conv_tc_kernel<256,true>"}};
  static_assert(TC_WIDE_BN == 256, "kernel names");
  const Kern kern = kerns[g.tma_out][g.BN > TC_MAX_BN ? 4 : g.BN / 32 - 1];
  const int num_tiles = g.num_m_tiles * g.num_n_tiles;
  ODT_CUDA_OK(launch_pdl(kern, num_tiles < kNumSMs ? num_tiles : kNumSMs, TC_THREADS, smem, st, tmA, tmB, tmO, g,
                         make_epi(*p)));
  ODT_LAUNCH_OK();
  g_last_conv_kernel = names[g.tma_out][g.BN > TC_MAX_BN ? 4 : g.BN / 32 - 1];
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
