// Pointwise (1x1, stride 1) convolution for the narrow layers of RetinaNet's bottlenecks -- the "reduce" convolutions
// (16->7, 28->7, 56->14, 112->28) and the "expand" convolutions that also carry the residual add and the two
// pre-activated copies for the next unit (7->28, 14->56, 28->112).  ref call sites: tf.layers.conv2d
// RetinaNet.py:579,609 (bottleneck 1x1), residual add RetinaNet.py:643, consumer BN + ReLU RetinaNet.py:594-597.
//
// These layers are HBM / LSU work, not tensor-core work: 7->28 is 196 multiply-adds per pixel against 16 + 64
// (residual) + 2 * 64 bytes of traffic.  conv_thin.cu gives one thread one pixel and lets it read and write its own
// 128-byte-strided row 16 bytes at a time (every warp-wide access touches 32 lines; 76 us for the 7->28 layer at
// 200x200x16 against a 24 us traffic floor), and handles at most 32 output channels.  Here every WARP streams groups
// of 32 consecutive pixels on its own (no block-wide barrier after the prologue; 16 warps per SM sit in different
// phases, so loads, arithmetic and stores of different groups overlap):
//   1. load: the real 16-byte sectors of the group's input rows -> the warp's shared-memory slice, consecutive lanes
//      on consecutive sectors (a warp-wide load covers whole rows' worth of contiguous bytes), all loads of a lane
//      issued before the first use;
//   2. compute, COT output channels per pass: lane = pixel, the filter bank as fp32 [cin][cout] in shared memory
//      (filled once per block) read by warp-broadcast 128-bit loads (4 FMA per LDS), fp32 accumulation;
//   3. the accumulators are parked in the warp's slice and epilogue.cuh's fused fp16 output step (epi_store_f16<1>)
//      runs with consecutive lanes on consecutive 16-byte sectors again, so residual loads and all stores are
//      full-sector and row-contiguous.
// The grid is persistent (<= 2 blocks per SM, groups dealt round-robin to the warps).  The filter bank and the affine
// parameters are constants of the network: they are filled BEFORE griddepcontrol.wait, i.e. under the tail of the
// producer kernel (programmatic dependent launch).
//
// The per-lane work of every phase lives in __host__ __device__ functions taking the lane / thread id, so that the
// very same source runs on the CPU, phase by phase, inside the TEST-ONLY harness tests/native/pw_host.cu.  The product
// library contains no host path.
#include <string.h>

#include "epilogue.cuh"

namespace odt {

int pw_mode();  // api.cu: ODT_TC_PW (0 = off, 1 = default planner, 2 = wherever the layer qualifies)

constexpr int PW_THREADS = 256;
constexpr int PW_WARPS = PW_THREADS / 32;
constexpr int PW_BLOCKS_PER_SM = 3;
constexpr int PW_SMEM_LIMIT = 200 * 1024;
constexpr int PW_SMEM_SHARE = 74 * 1024;  // largest block of which PW_BLOCKS_PER_SM fit one SM (228 KB, 1 KB reserved each)

struct PwGeom {
  int B, H, W;  // 1x1 / stride 1: output geometry = input geometry
  int Cin, Cout, in_ld, w_ld;
  int in_halo, out_halo;
  int ci8;     // 16-byte input sectors read per pixel = ceil(Cin / 8)
  int co8;     // 16-byte output sectors stored per pixel = ceil(Cout / 8)
  int passes;  // output-channel groups of COT: ceil(co8 * 8 / COT)
  int cop;     // passes * COT: padded width of the filter bank
  int ci8_inv;  // 65536 / ci8 + 1: i / ci8 = (i * ci8_inv) >> 16 for the item indices of a group
  int xs16;    // staged input row stride in 16-byte units (odd: conflict-free 128-bit reads at one row per lane)
  long long M;
  long long groups;  // ceil(M / 32)
  // shared memory: [filter bank | affine parameters | PW_WARPS warp slices]; a slice = [rows | x | y]
  int off_par, off_warps, slice_bytes, off_x, off_y, smem_bytes;
};

// One warp's private staging area.  Row offsets are kept in units of 16-byte sectors (8 fp16 elements).
struct PwSlice {
  int* rows;  // [4][32]: sector offset of the pixel's row in in / out0 (= residual) / out1 / out2; in < 0: no pixel
  uint4* x;   // [32][xs16]
  float* y;   // [32][COT + 4]
};

__host__ __device__ __forceinline__ PwSlice pw_slice(unsigned char* base, const PwGeom& g, int warp) {
  unsigned char* w = base + g.off_warps + (long long)warp * g.slice_bytes;
  PwSlice s;
  s.rows = reinterpret_cast<int*>(w);
  s.x = reinterpret_cast<uint4*>(w + g.off_x);
  s.y = reinterpret_cast<float*>(w + g.off_y);
  return s;
}

// block prologue (before the grid dependency resolves): filter bank fp32 [cin][cop] and epi_param's six rows [6][cop]
__host__ __device__ __forceinline__ void pw_fill(int tid, unsigned char* base, const __half* wgt, const PwGeom& g,
                                                 const Epi& e) {
  float* ws = reinterpret_cast<float*>(base);
  float* par = reinterpret_cast<float*>(base + g.off_par);
  for (int i = tid; i < g.ci8 * g.cop; i += PW_THREADS) {
    const int n = i % g.cop, c8 = i / g.cop;  // consecutive threads: consecutive filters (conflict-free stores)
    uint4 raw = make_uint4(0u, 0u, 0u, 0u);
    if (n < g.Cout) raw = ODT_LDG(reinterpret_cast<const uint4*>(wgt + (long long)n * g.w_ld) + c8);
    const __half* h = reinterpret_cast<const __half*>(&raw);
#pragma unroll
    for (int j = 0; j < 8; ++j) ws[(c8 * 8 + j) * g.cop + n] = (c8 * 8 + j < g.Cin) ? __half2float(h[j]) : 0.f;
  }
  for (int i = tid; i < 6 * g.cop; i += PW_THREADS) par[i] = epi_param(e, i / g.cop, i % g.cop);
}

// phase 1: where the group's pixels live in the four tensors (lane = pixel); 32-bit arithmetic (pw_plan bounds M)
__host__ __device__ __forceinline__ void pw_rows(int lane, int grp, const PwSlice& s, const PwGeom& g, const Epi& e) {
  const int m = grp * 32 + lane;
  int rin = -1, r0 = 0, r1 = 0, r2 = 0;
  if (m < (int)g.M) {
    const int hw = g.H * g.W;
    const int b = m / hw;
    const int pix = m - b * hw;
    const int y = pix / g.W, x = pix - y * g.W;
    const int hpos = (y + 1) * (g.W + 2) + x + 1;  // position inside a halo image
    rin = (int)((g.in_halo ? ((long long)b * (g.H + 2) * (g.W + 2) + hpos) : (long long)m) * (g.in_ld / 8));
    r0 = (int)((long long)b * (e.out0_img_stride / 8) + (long long)(g.out_halo ? hpos : pix) * (e.out0_pix_stride / 8));
    r1 = (int)((long long)b * (e.out1_img_stride / 8) + (long long)(e.out1_halo ? hpos : pix) * (e.out1_pix_stride / 8));
    r2 = (int)((long long)b * (e.out2_img_stride / 8) + (long long)(e.out2_halo ? hpos : pix) * (e.out2_pix_stride / 8));
  }
  s.rows[lane] = rin;
  s.rows[32 + lane] = r0;
  s.rows[64 + lane] = r1;
  s.rows[96 + lane] = r2;
}

// phase 2: the real input sectors of the group's pixels -> the warp's slice (consecutive lanes: consecutive sectors)
__host__ __device__ __forceinline__ void pw_load(int lane, const PwSlice& s, const __half* in, const PwGeom& g) {
  const uint4* in16 = reinterpret_cast<const uint4*>(in);
  const int items = 32 * g.ci8;
  for (int i0 = 0; i0 < items; i0 += 128) {
    uint4 v[4];
    int dst[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {  // four independent loads in flight per lane
      const int i = i0 + u * 32 + lane;
      v[u] = make_uint4(0u, 0u, 0u, 0u);
      dst[u] = -1;
      if (i < items) {
        const int px = (i * g.ci8_inv) >> 16, ch = i - px * g.ci8;  // exact for i < 512 (pw_plan)
        const int r = s.rows[px];
        dst[u] = px * g.xs16 + ch;
        if (r >= 0) v[u] = ODT_LDG(in16 + r + ch);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (dst[u] >= 0) s.x[dst[u]] = v[u];
  }
}

// phase 3: lane = pixel, output channels [pass * COT, pass * COT + COT); accumulators -> the warp's slice
template <int COT>
__host__ __device__ __forceinline__ void pw_compute(int lane, int pass, const PwSlice& s, const float* ws,
                                                    const PwGeom& g) {
  float acc[COT];
#pragma unroll
  for (int n = 0; n < COT; ++n) acc[n] = 0.f;
  const uint4* xrow = s.x + lane * g.xs16;
  const float* wbase = ws + pass * COT;
  for (int c8 = 0; c8 < g.ci8; ++c8) {
    const uint4 raw = xrow[c8];
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
      const float4* wrow = reinterpret_cast<const float4*>(wbase + (c8 * 8 + c) * g.cop);
#pragma unroll
      for (int n4 = 0; n4 < COT / 4; ++n4) {
        const float4 w = wrow[n4];
        acc[4 * n4 + 0] = fmaf(x[c], w.x, acc[4 * n4 + 0]);
        acc[4 * n4 + 1] = fmaf(x[c], w.y, acc[4 * n4 + 1]);
        acc[4 * n4 + 2] = fmaf(x[c], w.z, acc[4 * n4 + 2]);
        acc[4 * n4 + 3] = fmaf(x[c], w.w, acc[4 * n4 + 3]);
      }
    }
  }
  float4* yrow = reinterpret_cast<float4*>(s.y + lane * (COT + 4));
#pragma unroll
  for (int n4 = 0; n4 < COT / 4; ++n4)
    yrow[n4] = make_float4(acc[4 * n4], acc[4 * n4 + 1], acc[4 * n4 + 2], acc[4 * n4 + 3]);
}

// The lane's epilogue items of one pass: item u = (pixel px[u], sector n8[u]); consecutive lanes sit on consecutive
// sectors of a pixel, then on the next pixel.  px < 0: no item.
template <int COT>
struct PwItems {
  uint4 rs[COT / 8];  // the residual sectors, requested BEFORE the pass is computed (phase 3a) and consumed after it
};

// item u of the lane in a pass with `spp` real sectors per pixel: pixel (or -1) and sector inside the pass
__host__ __device__ __forceinline__ int pw_item(int lane, int u, int spp, const int* rows, int* sector) {
  const int j = u * 32 + lane;
  if (j >= 32 * spp) return -1;
  const int q = (j * (65536 / spp + 1)) >> 16;  // j / spp, exact for j < 128
  *sector = j - q * spp;
  return rows[q] >= 0 ? q : -1;
}

// phase 3a: which (pixel, sector) items the lane owns in this pass + their residual loads put in flight
template <int COT>
__host__ __device__ __forceinline__ void pw_items(int lane, int pass, const PwSlice& s, const PwGeom& g, const Epi& e,
                                                  PwItems<COT>& it) {
  constexpr int SPP = COT / 8;  // sectors per pixel and pass
  const int spp = (g.co8 - pass * SPP) < SPP ? (g.co8 - pass * SPP) : SPP;  // real sectors of this pass (last: fewer)
  const uint4* res16 = reinterpret_cast<const uint4*>(e.residual);
#pragma unroll
  for (int u = 0; u < SPP; ++u) {
    int sec = 0;
    const int px = pw_item(lane, u, spp, s.rows, &sec);
    it.rs[u] = make_uint4(0u, 0u, 0u, 0u);
    if (px >= 0 && res16) it.rs[u] = ODT_LDG(res16 + s.rows[32 + px] + pass * SPP + sec);
  }
}

__host__ __device__ __forceinline__ void pw_ld8(const float* p, float* o) {  // 32-byte aligned [8] floats
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  o[0] = a.x, o[1] = a.y, o[2] = a.z, o[3] = a.w, o[4] = b.x, o[5] = b.y, o[6] = b.z, o[7] = b.w;
}

// phase 4: epilogue of one pass over the lane's items
template <int COT>
__host__ __device__ __forceinline__ void pw_store(int lane, int pass, const PwSlice& s, const float* par,
                                                  const PwGeom& g, const Epi& e, const PwItems<COT>& it) {
  constexpr int SPP = COT / 8;
  const int spp = (g.co8 - pass * SPP) < SPP ? (g.co8 - pass * SPP) : SPP;
#pragma unroll
  for (int u = 0; u < SPP; ++u) {
    int sec = 0;
    const int px = pw_item(lane, u, spp, s.rows, &sec);
    if (px < 0) continue;
    const int n8 = pass * SPP + sec;
    float v[8];
    pw_ld8(s.y + px * (COT + 4) + (n8 * 8 - pass * COT), v);
    epi_store_f16<1>(e, v, par + n8 * 8, g.cop, [&](int) { return it.rs[u]; }, 8ll * (s.rows[32 + px] + n8),
                     8ll * (s.rows[64 + px] + n8), 8ll * (s.rows[96 + px] + n8));
  }
}

#ifdef __CUDA_ARCH__
#define ODT_PW_SYNCWARP() __syncwarp()
#else
#define ODT_PW_SYNCWARP() ((void)0)
#endif

template <int COT>
__global__ void __launch_bounds__(PW_THREADS, PW_BLOCKS_PER_SM)
    conv_pw_kernel(const __half* __restrict__ in, const __half* __restrict__ wgt, const __grid_constant__ PwGeom g,
                   const __grid_constant__ Epi e) {
  extern __shared__ __align__(16) unsigned char pw_smem[];
  pdl_launch_dependents();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pw_fill(tid, pw_smem, wgt, g, e);  // constants of the network: legal before the producer grid has finished
  pdl_wait();
  __syncthreads();
  const float* ws = reinterpret_cast<const float*>(pw_smem);
  const float* par = reinterpret_cast<const float*>(pw_smem + g.off_par);
  const PwSlice s = pw_slice(pw_smem, g, warp);
  const int stride = (int)gridDim.x * PW_WARPS;
  for (int grp = warp * (int)gridDim.x + (int)blockIdx.x; grp < (int)g.groups; grp += stride) {
    pw_rows(lane, grp, s, g, e);
    __syncwarp();
    PwItems<COT> it;
    pw_items<COT>(lane, 0, s, g, e, it);  // the first pass's residual sectors fly together with the inputs
    pw_load(lane, s, in, g);
    __syncwarp();
    for (int pass = 0; pass < g.passes; ++pass) {
      if (pass) pw_items<COT>(lane, pass, s, g, e, it);
      pw_compute<COT>(lane, pass, s, ws, g);
      __syncwarp();
      pw_store<COT>(lane, pass, s, par, g, e, it);
      __syncwarp();
    }
  }
}

static int g_pw_launches = 0;  // debug: lets a test assert that the layer really took this path

// Eligibility + geometry; ODT_ERR_UNSUPPORTED when the layer does not qualify.  `force`: ignore the planner's gate.
static int pw_plan(const void* in, const odt_conv_params* p, bool force, PwGeom* gout, int* cot_out) {
  const bool shape_ok = p->R == 1 && p->S == 1 && p->stride == 1 && p->dil == 1 && p->pad_t == 0 && p->pad_l == 0 &&
                        p->OH == p->H && p->OW == p->W && p->out0_pool == 0 && p->out0_group == 0 &&
                        (p->in_halo == 0 || p->in_halo == 1) && (p->out0_halo == 0 || p->out0_halo == 1);
  if (!shape_ok) return ODT_ERR_UNSUPPORTED;
  const int ci8 = (p->Cin + 7) / 8, co8 = (p->Cout + 7) / 8;
  if (ci8 > 16 || co8 > 32) return ODT_ERR_UNSUPPORTED;
  const int cot = co8 <= 1 ? 8 : co8 <= 2 ? 16 : 32;
  const int passes = (co8 * 8 + cot - 1) / cot;
  const bool io_ok = ((uintptr_t)in & 15) == 0 && p->in_ld % 8 == 0 && p->in_ld >= ci8 * 8 && p->w_ld % 8 == 0 &&
                     p->w_ld >= ci8 * 8 && (p->out0 || p->out1 || p->out2) && f16_sector_outputs_ok(p, co8 * 8);
  if (!io_ok) return ODT_ERR_UNSUPPORTED;
  const long long M = (long long)p->B * p->H * p->W;
  if (M + 64 >= (1ll << 31)) return ODT_ERR_UNSUPPORTED;  // pixel indices are 32-bit
  // row offsets are kept as 32-bit sector indices
  const long long in_elems = (long long)p->B * (p->H + 2) * (p->W + 2) * p->in_ld;
  const long long lim = (1ll << 31) * 8;
  if (in_elems >= lim || (long long)p->B * p->out0_img_stride >= lim ||
      (p->out1 && (long long)p->B * p->out1_img_stride >= lim) || (p->out2 && (long long)p->B * p->out2_img_stride >= lim))
    return ODT_ERR_UNSUPPORTED;
  // The kernel itself takes layers up to 4096 multiply-adds per pixel (beyond that the arithmetic no longer hides
  // under the traffic).  Default planner (mode 1): the 8-channel-input expand layers of large maps only (7->28 of
  // RetinaNet); a rule carried over from the previous target, not re-measured on the H100.
  if ((long long)ci8 * 8 * passes * cot > 4096 && !force) return ODT_ERR_UNSUPPORTED;
  if (!force && !(ci8 == 1 && co8 >= 3 && M >= (1 << 18))) return ODT_ERR_UNSUPPORTED;
  PwGeom g;
  memset(&g, 0, sizeof(g));
  g.B = p->B;
  g.H = p->H;
  g.W = p->W;
  g.Cin = p->Cin;
  g.Cout = p->Cout;
  g.in_ld = p->in_ld;
  g.w_ld = p->w_ld;
  g.in_halo = p->in_halo;
  g.out_halo = p->out0_halo;
  g.ci8 = ci8;
  g.co8 = co8;
  g.passes = passes;
  g.cop = passes * cot;
  g.ci8_inv = 65536 / ci8 + 1;
  g.xs16 = ci8 | 1;
  g.M = M;
  g.groups = (M + 31) / 32;
  int off = ci8 * 8 * g.cop * 4;
  g.off_par = off;
  off += 6 * g.cop * 4;
  off = (off + 15) & ~15;
  g.off_warps = off;
  g.off_x = 4 * 32 * 4;
  g.off_y = g.off_x + 32 * g.xs16 * 16;
  g.slice_bytes = g.off_y + 32 * (cot + 4) * 4;
  g.smem_bytes = g.off_warps + PW_WARPS * g.slice_bytes;
  if (g.smem_bytes > PW_SMEM_LIMIT) return ODT_ERR_UNSUPPORTED;
  *gout = g;
  *cot_out = cot;
  return ODT_OK;
}

// ODT_ERR_UNSUPPORTED when the layer does not qualify (the caller then takes the other paths).
int conv_pw_try(const void* in, const void* weights, const odt_conv_params* p, void* stream) {
  PwGeom g;
  int cot;
  const int rc = pw_plan(in, p, pw_mode() == 2, &g, &cot);
  if (rc) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_pw_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM_LIMIT));
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_pw_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM_LIMIT));
    ODT_CUDA_OK(cudaFuncSetAttribute(conv_pw_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM_LIMIT));
    attr_set = true;
  }
  const Epi e = make_epi(*p);
  const long long want = (g.groups + PW_WARPS - 1) / PW_WARPS;  // blocks that give every warp one group
  const long long cap = (long long)kNumSMs * (g.smem_bytes <= PW_SMEM_SHARE ? PW_BLOCKS_PER_SM : g.smem_bytes <= 113 * 1024 ? 2 : 1);
  const unsigned grid = (unsigned)(want < cap ? want : cap);
  const __half* inh = reinterpret_cast<const __half*>(in);
  const __half* wh = reinterpret_cast<const __half*>(weights);
  cudaStream_t st = (cudaStream_t)stream;
  if (cot == 8)
    ODT_CUDA_OK(launch_pdl(conv_pw_kernel<8>, grid, PW_THREADS, g.smem_bytes, st, inh, wh, g, e));
  else if (cot == 16)
    ODT_CUDA_OK(launch_pdl(conv_pw_kernel<16>, grid, PW_THREADS, g.smem_bytes, st, inh, wh, g, e));
  else
    ODT_CUDA_OK(launch_pdl(conv_pw_kernel<32>, grid, PW_THREADS, g.smem_bytes, st, inh, wh, g, e));
  ODT_LAUNCH_OK();
  ++g_pw_launches;
  g_last_conv_kernel = cot == 8 ? "conv_pw_kernel<8>" : cot == 16 ? "conv_pw_kernel<16>" : "conv_pw_kernel<32>";
  return ODT_OK;
}

}  // namespace odt

// Debug only: number of convolutions launched through conv_pw_kernel by this process.
extern "C" int odt_debug_pw_launches(void) { return odt::g_pw_launches; }
