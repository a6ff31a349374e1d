// "Taps as N": the 3x3 / stride-1 halo convolution for NARROW outputs (Cout_pad <= 64) with the three
// horizontal filter taps folded into the N dimension of the MMA.  One MMA multiplies the activation tile of
// filter row r by the weights of ALL THREE horizontal taps:
//
//   P[q, s*BN + n] = sum_{r, c} X[q + r*PW, c] * W[n, r, s, c]          (N = 3*BN, K = 3*Cin)
//   out[p, n]      = P[p-1, 0*BN + n] + P[p, 1*BN + n] + P[p+1, 2*BN + n]
//
// so a tile takes 3*cchunks*4 MMAs of N = 3*BN instead of 9*cchunks*4 of N = BN: each activation row that is
// fetched feeds three times as many output columns.  A tile is 4 image rows x 32 columns (shared-memory row
// = 32*row + column); columns 0 and 31 only serve as neighbours, tiles overlap by two columns (30 outputs per
// row and tile).  The shifted sum runs on the fp32 accumulator tile in shared memory; in the epilogue each
// lane owns one column of one row.  The fused 2x2/2 max-pool pairs columns inside the warp and rows through
// a small shared-memory exchange between the warps of an epilogue group.
//
// Roles / pipeline as in conv_tc.cu: w0 TMA producer (one [64 ch][32 x][4 rows] box per filter row and
// channel chunk), w4..11 two consumer warpgroups (wgmma over the two 64-row halves of the tile, then the
// epilogue: group g takes the 32-channel chunks j = g, g + 2, ...); the 9*cchunks weight tiles stay resident
// in shared memory.
//
// On sm_90 a 128 x N x 16 MMA costs about N clocks whatever the operand layout, so folding the taps into N
// saves no MMA time; the planner (ODT_TC_TAPN=1) takes the layer only where its tiles waste fewer positions
// than the regular halo-flat tiles.  ref call sites: tf.nn.conv2d SSD300.py:519 (conv1_2), tf.layers.conv2d
// RetinaNet.py:599-609, YOLOv3.py:495, FCOS.py:469-479.
#include <string.h>

#include "epilogue.cuh"
#include "tc_ptx.cuh"

namespace odt {

constexpr int TN_THREADS = 384;      // producer warpgroup (one active warp), two consumer warpgroups
constexpr int TN_XV = 30;            // output columns per tile row (32 lanes - 2 neighbour lanes)
constexpr int TN_ROWS = 4;           // image rows per tile (one per epilogue warp of a group)
constexpr int TN_A_BYTES = 128 * 128;
constexpr int TN_MAX_STAGES = 8;
constexpr int TN_PAR_FLOATS = 6 * 64;
constexpr int TN_XCH_PITCH = 80;     // bytes per lane in the pooling exchange (64 payload, padded against bank conflicts)
constexpr int TN_XCH_BYTES = 2 * 2 * 2 * 32 * TN_XCH_PITCH;  // [group][buffer][row pair][lane]
constexpr int TN_SMEM_LIMIT = 232448;

struct TnGeom {
  int B, H, W;
  int cchunks, klast;
  int BN;  // Cout_pad: 32 or 64
  int xblocks, yblocks, num_tiles;
  int stages;
  int out_halo;
};

constexpr int tn_sum_bytes(int bn) { return 128 * (bn + 4) * 4; }  // fp32 tile of the shifted sum

template <int BN, int POOL>
__global__ void __launch_bounds__(TN_THREADS, 1)
    conv_tapn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ TnGeom g, const __grid_constant__ Epi e) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const int stages = g.stages;
  const uint32_t a_base = base;
  const uint32_t b_base = base + (uint32_t)stages * TN_A_BYTES;
  const uint32_t wtile = 3u * (uint32_t)BN * 128u;  // weights of one (filter row, chunk): rows s*BN + n
  const uint32_t wbytes = 3u * (uint32_t)g.cchunks * wtile;
  const uint32_t bar_base = b_base + wbytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (TN_MAX_STAGES + s); };
  const uint32_t wfull_bar = bar_base + 8u * (2 * TN_MAX_STAGES);
  float* par = reinterpret_cast<float*>(smem_raw + (bar_base + 256u - raw));  // [scale|shift|scale2|shift2|scale3|shift3][64]
  uint8_t* xch = smem_raw + (bar_base + 256u + TN_PAR_FLOATS * 4u - raw);
  // out[p] = P_centre[p] + P_left[p-1] + P_right[p+1] accumulated in place, BN + 4 floats per row
  constexpr int SUM_PITCH = BN + 4;
  float* sum = reinterpret_cast<float*>(xch + (POOL ? TN_XCH_BYTES : 0));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);  // one arrival per consumer warp
    }
    mbar_init(wfull_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp >= 4) {
    // per-channel epilogue parameters (constant data): one copy per CTA
    for (int i = threadIdx.x - 128; i < TN_PAR_FLOATS; i += 256) {
      const int which = i >> 6, c = i & 63;
      const bool ok = c < e.Cout;
      const float* src = which == 0 ? e.scale : which == 1 ? e.shift : which == 2 ? e.scale2 : which == 3 ? e.shift2
                         : which == 4 ? e.scale3 : e.shift3;
      par[i] = (ok && src) ? __ldg(src + c) : ((which & 1) ? 0.f : 1.f);
    }
  }
  __syncthreads();

  if (warp == 0) {
    // the filter bank is constant data: fetch it before waiting on the previous kernel
    if (elect_one()) {
      mbar_expect_tx(wfull_bar, wbytes);
      for (int r = 0; r < 3; ++r)
        for (int cc = 0; cc < g.cchunks; ++cc)
          for (int s = 0; s < 3; ++s)
            tma_load_2d(b_base + (uint32_t)(r * g.cchunks + cc) * wtile + (uint32_t)s * (uint32_t)BN * 128u, &tmB,
                        wfull_bar, ((r * 3 + s) * g.cchunks + cc) * 64, 0);
    }
    __syncwarp();
  }
  pdl_launch_dependents();
  pdl_wait();

  const int per_img = g.yblocks * g.xblocks;

  if (warp == 0) {
    // ===================== TMA producer ======================================
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      const int img = tile / per_img;
      const int rem = tile - img * per_img;
      const int yq = rem / g.xblocks, xq = rem - yq * g.xblocks;
      for (int r = 0; r < 3; ++r) {
        for (int cc = 0; cc < g.cchunks; ++cc) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          if (elect_one()) {
            mbar_expect_tx(full_bar(stage), TN_A_BYTES);
            // padded coordinates: columns TN_XV*xq .. +31 (real x = TN_XV*xq - 1 ..), rows 4*yq + r .. +3
            // (real y = 4*yq + r - 1 ..); everything past the padded extent is TMA zero fill
            tma_load_4d(a_base + (uint32_t)stage * TN_A_BYTES, &tmA, full_bar(stage), cc * 64, TN_XV * xq,
                        TN_ROWS * yq + r, img);
          }
          __syncwarp();
          if (++stage == stages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumer warpgroups ===============================
    const int quarter = warp & 3;          // epilogue: image row inside the tile
    const int group = (warp - 4) >> 2;     // MMA: rows 64*group .. +63 of the tile; epilogue: chunks group, group + 2
    const int chunks = BN >> 5;            // 32-channel chunks per tile
    int xbuf = 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[3 * BN / 2];
    mbar_wait(wfull_bar, 0);
    for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
      int prev = -1;
      for (int r = 0; r < 3; ++r) {
        for (int cc = 0; cc < g.cchunks; ++cc) {
          mbar_wait(full_bar(stage), phase);
          const uint64_t adesc = make_desc_sw128(a_base + (uint32_t)stage * TN_A_BYTES + (uint32_t)group * 64u * 128u);
          const uint64_t bdesc = make_desc_sw128(b_base + (uint32_t)(r * g.cchunks + cc) * wtile);
          // all-zero K steps of a thin layer are not issued
          const int ksteps = __shfl_sync(0xffffffffu, (cc == g.cchunks - 1) ? g.klast : 4, 0);
          wg_fence();
          wg_mma_chunk<3 * BN>(acc, adesc, bdesc, ksteps, (r | cc) == 0);
          wg_commit();
          wg_wait<1>();  // the previous stage's MMAs have retired
          if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
          prev = stage;
          if (++stage == stages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
      wg_wait<0>();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      // shifted sum in shared memory: out[p] = (P_centre[p] + P_left[p-1]) + P_right[p+1]; row 32*y + 31 feeds
      // row 32*(y+1), column 0, which only serves as a neighbour
      asm volatile("bar.sync 3, 256;" ::: "memory");  // the previous tile's epilogue has read the sum
      {
        const int w = warp & 3;
        const int row0 = 64 * group + 16 * w + (lane >> 2);
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
          const int s3 = pass == 0 ? 1 : (pass == 1 ? 0 : 2);  // centre, left, right
          const int dr = s3 - 1;  // centre writes row p, left adds into p + 1, right into p - 1
          if (pass) asm volatile("bar.sync 3, 256;" ::: "memory");
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) {
            const int c = 8 * i + 2 * (lane & 3);
            const int f = (s3 * BN + 8 * i) / 8 * 4;  // fragment register of column s3*BN + 8i
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int row = row0 + 8 * hh - dr;
              if (row < 0 || row >= 128) continue;
              float2* dst = reinterpret_cast<float2*>(sum + row * SUM_PITCH + c);
              const float2 v = make_float2(acc[f + 2 * hh], acc[f + 2 * hh + 1]);
              if (s3 == 1) {
                *dst = v;
              } else {
                float2 o = *dst;
                o.x += v.x;
                o.y += v.y;
                *dst = o;
              }
            }
          }
        }
      }
      asm volatile("bar.sync 3, 256;" ::: "memory");

      const int img = tile / per_img;
      const int rem = tile - img * per_img;
      const int yq = rem / g.xblocks, xq = rem - yq * g.xblocks;
      const int y = TN_ROWS * yq + quarter;
      const int x = TN_XV * xq - 1 + lane;
      const bool row_ok = lane >= 1 && lane <= TN_XV && x < g.W && y < g.H;
      long long o0_row = (long long)img * e.out0_img_stride;
      long long o1_row = 0, o2_row = 0;
      if (POOL) {
        // pooled pixel of this lane's window (used by the odd lanes of the even rows)
        const int oh = g.out_halo;
        o0_row += (long long)(((y >> 1) + oh) * ((g.W >> 1) + 2 * oh) + (x >> 1) + oh) * e.out0_pix_stride;
      } else {
        const int pix = row_ok ? y * g.W + x : 0;
        o0_row += g.out_halo ? (long long)((y + 1) * (g.W + 2) + x + 1) * e.out0_pix_stride
                             : (long long)pix * e.out0_pix_stride;
        o1_row = aux_row(e.out1_img_stride, e.out1_pix_stride, e.out1_halo, g.W, img, pix);
        o2_row = aux_row(e.out2_img_stride, e.out2_pix_stride, e.out2_halo, g.W, img, pix);
      }
      const float* my_sum = sum + (quarter * 32 + lane) * SUM_PITCH;
      for (int j = group; j < chunks; j += 2) {
        const int nb = j * 32;
        const float4* ps = reinterpret_cast<const float4*>(par + nb);
        const float4* ph4 = reinterpret_cast<const float4*>(par + 64 + nb);
        float v[32];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 t = *reinterpret_cast<const float4*>(my_sum + nb + 4 * i);
          v[4 * i + 0] = t.x;
          v[4 * i + 1] = t.y;
          v[4 * i + 2] = t.z;
          v[4 * i + 3] = t.w;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 sc = ps[i], sh = ph4[i];
          v[4 * i + 0] = apply_act(fmaf(v[4 * i + 0], sc.x, sh.x), e.act);
          v[4 * i + 1] = apply_act(fmaf(v[4 * i + 1], sc.y, sh.y), e.act);
          v[4 * i + 2] = apply_act(fmaf(v[4 * i + 2], sc.z, sh.z), e.act);
          v[4 * i + 3] = apply_act(fmaf(v[4 * i + 3], sc.w, sh.w), e.act);
        }
        if (POOL) {
          // 2x2/2 max-pool of the rounded values: columns (odd lane, next lane), rows (even warp, next warp)
          uint4 packed[4];
          __half2* ph = reinterpret_cast<__half2*>(packed);
          uint32_t* pw = reinterpret_cast<uint32_t*>(packed);
#pragma unroll
          for (int i = 0; i < 16; ++i) ph[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            uint32_t o = __shfl_down_sync(0xffffffffu, pw[i], 1);
            __half2 a = __hmax2(*reinterpret_cast<__half2*>(&pw[i]), *reinterpret_cast<__half2*>(&o));
            pw[i] = *reinterpret_cast<uint32_t*>(&a);
          }
          uint8_t* slot = xch + (size_t)(((group * 2 + xbuf) * 2 + (quarter >> 1)) * 32 + lane) * TN_XCH_PITCH;
          if (quarter & 1) {
            uint4* sp = reinterpret_cast<uint4*>(slot);
#pragma unroll
            for (int qd = 0; qd < 4; ++qd) sp[qd] = packed[qd];
          }
          asm volatile("bar.sync %0, 128;" ::"r"(1 + group) : "memory");
          if (!(quarter & 1)) {
            const uint4* sp = reinterpret_cast<const uint4*>(slot);
#pragma unroll
            for (int qd = 0; qd < 4; ++qd) {
              uint4 t = sp[qd];
              const __half2* th = reinterpret_cast<const __half2*>(&t);
              __half2* mine = reinterpret_cast<__half2*>(&packed[qd]);
#pragma unroll
              for (int i = 0; i < 4; ++i) mine[i] = __hmax2(mine[i], th[i]);
            }
            if (row_ok && (lane & 1)) {  // even x, even y: the window's top-left pixel
              uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(e.out0) + o0_row + nb);
#pragma unroll
              for (int qd = 0; qd < 4; ++qd) op[qd] = packed[qd];
            }
          }
          xbuf ^= 1;  // the next chunk's writers may run ahead of this chunk's readers by one barrier only
        } else if (row_ok) {
          const long long o0 = o0_row + nb;
          if (e.residual) {
            const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(e.residual) + o0);
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
            const float4* ps2 = reinterpret_cast<const float4*>(par + 128 + nb);
            const float4* ph2 = reinterpret_cast<const float4*>(par + 192 + nb);
            uint4 packed1[4];
            __half2* p1 = reinterpret_cast<__half2*>(packed1);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 sc = ps2[i], sh = ph2[i];
              const float2 fa = __half22float2(ph[2 * i]);  // the consumer sees the rounded value
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
            const float4* ps3 = reinterpret_cast<const float4*>(par + 256 + nb);
            const float4* ph3 = reinterpret_cast<const float4*>(par + 320 + nb);
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
      }
    }
  }
}

static int g_tapn_launches = 0;  // debug: lets a test assert that the layer really took this path

// ODT_ERR_UNSUPPORTED when the layer does not qualify (the caller then takes the regular paths).
int conv_tapn_try(const void* in, const void* weights, const odt_conv_params* p, void* stream) {
  const bool shape_ok = p->in_halo == 1 && p->R == 3 && p->S == 3 && p->stride == 1 && p->dil == 1 && p->pad_t == 1 &&
                        p->pad_l == 1 && p->OH == p->H && p->OW == p->W && (p->Cout_pad == 32 || p->Cout_pad == 64) &&
                        p->in_ld % 64 == 0 && p->in_ld / 64 <= 2 && p->w_ld == p->in_ld;
  if (!shape_ok) return ODT_ERR_UNSUPPORTED;
  const bool pool = p->out0_pool == 2;
  auto aligned = [](const void* ptr, long long img, int pix, int need) {
    return ((uintptr_t)ptr & 15) == 0 && img % 8 == 0 && pix % 8 == 0 && pix >= need;
  };
  bool out_ok = p->out0_group == 0 && (!p->out0 || p->out0_dtype == ODT_F16) &&
                (!p->out0 || aligned(p->out0, p->out0_img_stride, p->out0_pix_stride, p->Cout_pad)) &&
                (!p->out1 || aligned(p->out1, p->out1_img_stride, p->out1_pix_stride, p->Cout_pad)) &&
                (!p->out2 || aligned(p->out2, p->out2_img_stride, p->out2_pix_stride, p->Cout_pad)) &&
                (!p->residual || (((uintptr_t)p->residual & 15) == 0 && p->out0_img_stride % 8 == 0 &&
                                  p->out0_pix_stride % 8 == 0 && p->out0_pix_stride >= p->Cout_pad));
  if (pool)
    out_ok = out_ok && p->out0 && !p->residual && !p->out1 && !p->out2 && p->OH % 2 == 0 && p->OW % 2 == 0;
  else
    out_ok = out_ok && p->out0_pool == 0;
  if (!out_ok) return ODT_ERR_UNSUPPORTED;

  TnGeom g;
  memset(&g, 0, sizeof(g));
  g.B = p->B;
  g.H = p->H;
  g.W = p->W;
  g.cchunks = p->in_ld / 64;
  {
    const int rem = p->Cin - (g.cchunks - 1) * 64;
    g.klast = rem >= 64 ? 4 : (rem <= 0 ? 1 : (rem + 15) / 16);
  }
  g.BN = p->Cout_pad;
  g.xblocks = (p->W + TN_XV - 1) / TN_XV;
  g.yblocks = (p->H + TN_ROWS - 1) / TN_ROWS;
  const long long tiles = (long long)p->B * g.xblocks * g.yblocks;
  if (tiles >= (1ll << 31)) return ODT_ERR_UNSUPPORTED;
  g.num_tiles = (int)tiles;
  g.out_halo = p->out0_halo;
  if (tapn_mode() == 1) {
    // rounds of the slowest SM x MMA clocks per tile + a fixed cost per tile; a 128 x N x 16 MMA takes ~N clk
    // (2048 fp16 FMA/clk/SM), so both paths spend 9*cchunks*4*BN clk per tile and only the tile counts differ.
    // Small maps lose here: a 13-wide row still occupies a 32-lane tile row.
    const long long mm = 4ll * g.cchunks;
    const long long c_tapn = (long long)ceil_div(tiles, kNumSMs) * (9 * mm * g.BN + 1200);
    long long t_reg;  // tiles of the regular path
    if (pool) {
      const long long t2 = (long long)((p->H + 1) / 2) * ((p->W + 63) / 64), t4 = (long long)((p->H + 3) / 4) * ((p->W + 31) / 32);
      t_reg = (long long)p->B * (t4 < t2 ? t4 : t2);
    } else {
      t_reg = ((long long)p->B * (p->H + 2) * (p->W + 2) + 127) / 128;
    }
    const long long c_reg = (long long)ceil_div(t_reg, kNumSMs) * (9 * mm * g.BN + 1200);
    if (c_tapn >= c_reg) return ODT_ERR_UNSUPPORTED;
  }
  const int wbytes = 9 * g.cchunks * g.BN * 128;
  const int fixed = wbytes + 256 + TN_PAR_FLOATS * 4 + (pool ? TN_XCH_BYTES : 0) + tn_sum_bytes(g.BN) + 1024;
  int stages = (TN_SMEM_LIMIT - fixed) / TN_A_BYTES;
  if (stages > TN_MAX_STAGES) stages = TN_MAX_STAGES;
  if (stages < 2) return ODT_ERR_UNSUPPORTED;
  g.stages = stages;

  CUtensorMap tmA, tmB;
  {
    // [ld][W+2][H+2][B] view of the halo tensor; one {64, 32, 4, 1} box = the tile's rows of one filter row,
    // column index fastest (shared-memory row = 32*row + column)
    const cuuint64_t PH = (cuuint64_t)p->H + 2, PW = (cuuint64_t)p->W + 2;
    cuuint64_t dims[4] = {(cuuint64_t)p->in_ld, PW, PH, (cuuint64_t)p->B};
    cuuint64_t strides[3] = {(cuuint64_t)p->in_ld * 2, PW * p->in_ld * 2, PH * PW * p->in_ld * 2};
    cuuint32_t box[4] = {64, 32, TN_ROWS, 1};
    int rc = tc_encode_tiled(&tmA, in, 4, dims, strides, box, false);
    if (rc) return rc;
  }
  {
    const cuuint64_t ktot = (cuuint64_t)9 * p->w_ld;
    cuuint64_t dims[2] = {ktot, (cuuint64_t)p->Cout_pad};
    cuuint64_t strides[1] = {ktot * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)g.BN};
    int rc = tc_encode_tiled(&tmB, weights, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_tapn_kernel<32, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, TN_SMEM_LIMIT));
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_tapn_kernel<32, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TN_SMEM_LIMIT));
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_tapn_kernel<64, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, TN_SMEM_LIMIT));
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_tapn_kernel<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TN_SMEM_LIMIT));
    attr_set = true;
  }
  Epi e = make_epi(*p);
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(TN_THREADS);
  cfg.gridDim = dim3(g.num_tiles < kNumSMs ? g.num_tiles : kNumSMs);
  cfg.dynamicSmemBytes = stages * TN_A_BYTES + fixed;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  void (*kern)(CUtensorMap, CUtensorMap, TnGeom, Epi) =
      g.BN == 32 ? (pool ? conv_tapn_kernel<32, 1> : conv_tapn_kernel<32, 0>)
                 : (pool ? conv_tapn_kernel<64, 1> : conv_tapn_kernel<64, 0>);
  ODT_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, g, e));
  ODT_LAUNCH_OK();
  ++g_tapn_launches;
  return ODT_OK;
}

}  // namespace odt

// Debug only: number of convolutions launched through conv_tapn_kernel by this process.
extern "C" int odt_debug_tapn_launches(void) { return odt::g_tapn_launches; }
