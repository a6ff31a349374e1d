// Inference tail of the five detectors on sm_90a: score activation, analytic
// anchor/prior generation, box decode, thresholding, candidate compaction and
// exact per-class TF NonMaxSuppressionV3 (iterative arg-max + IoU suppress).
//
// All arithmetic that feeds a discrete decision (class id, keep index) is done
// with explicitly rounded fp32 intrinsics (__fmul_rn/__fadd_rn/__fdiv_rn), in
// the operation order of the reference graphs, so no FMA contraction can change
// a result relative to the TF1.13 CPU kernels.
//
// Reference call sites restated here (never copied): SSD300.py:157-190,323-343;
// RetinaNet.py:224-256,328-355; YOLOv3.py:320-368,419-433; FCOS.py:130-150,197-264.
#include <stdlib.h>

#include "tail_common.cuh"
#include "tc_ptx.cuh"

namespace odt {

// Two families of instantiations.  NFG = 20: the 25-float rows of every model at the VOC class count, 8 warps per
// CTA, row width and class loop fixed at compile time.  NFG = 0 ("wide"): YOLOv3 / FCOS with any num_fg in
// 1..kMaxFg, row width read from the parameters, 4 warps per CTA (32 rows x 133 floats = 17 KB per warp stage at
// num_fg = 128: 8 warps x 2 stages would need 272 KB).  Shared memory: [WARPS][STAGES][32 * row] floats, then the
// [WARPS][STAGES] mbarriers; the dynamic size is sized by the actual row width.
constexpr int kDecodeWarps = 8;
constexpr int kDecodeWarpsWide = 4;
__host__ __device__ constexpr long long decode_smem_bytes(int warps, int stages, int row) {
  return (long long)warps * stages * 32 * row * 4 + (long long)warps * stages * 8;
}

__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// One warp = 32 consecutive candidate rows per iteration.  The group (32 rows, 3200 bytes at num_fg = 20) is fetched
// by ONE bulk copy (TMA, cp.async.bulk) into a per-warp double buffer and signalled on an mbarrier, so no thread holds
// load registers or issues load instructions while it computes (round 1 kept 7 float4 per lane in flight: 80
// registers, 3 CTAs / SM, 826 warp instructions per group; this kernel: KIND at compile time, no 64-bit divisions,
// the row's scores stay in registers only).  Then one lane per row: score activation, background filter, threshold,
// per-class ballots and ONE atomic per (warp, class) to reserve the candidate slots.  Classes come in words of 32:
// pass[w] bit i = class 32 w + i of this row passes, and the ballot / reservation loop runs word by word.
template <int KIND, int WARPS, int OCC, int STAGES, int NFG>
__global__ void __launch_bounds__(WARPS * 32, OCC)
    decode_candidates_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp,
                             long long total_rows, unsigned long long* __restrict__ cand_keys,
                             int* __restrict__ cand_count) {
  static_assert(NFG == 0 ? KIND != ODT_DECODE_SSD : NFG == 20, "instantiations: NFG = 20, or 0 for YOLOv3 / FCOS");
  constexpr int W = NFG ? (NFG + 31) / 32 : kMaskWords;  // pass-mask words per row
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int nfg = NFG ? NFG : p.num_fg;
  const int row = row_floats(nfg);
  const int group_floats = 32 * row;
  const uint32_t group_bytes = (uint32_t)group_floats * 4u;
  extern __shared__ __align__(128) unsigned char dsm_raw[];
  float* rows_sm = reinterpret_cast<float*>(dsm_raw);
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(dsm_raw + (size_t)WARPS * STAGES * group_bytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar0 = smem_u32(&bars[warp * STAGES]);
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; ++s) mbar_init(bar0 + 8u * s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  const long long groups = (total_rows + 31) / 32;
  const long long full_groups = total_rows / 32;  // groups below this index are whole (bulk-copy eligible)
  const int step = (int)gridDim.x * WARPS;        // groups between two iterations of one warp
  long long g = (long long)blockIdx.x * WARPS + warp;
  // (image, row) of the group's first row, advanced incrementally: no 64-bit division in the loop
  const int N = p.N;
  int b = (int)((g * 32) / N), n = (int)((g * 32) % N);
  const int adv_b = (int)(((long long)step * 32) / N), adv_n = (int)(((long long)step * 32) % N);
  auto issue = [&](long long gg, int slot) {  // lane 0 only
    if (gg < full_groups) {
      mbar_expect_tx(bar0 + 8u * slot, group_bytes);
      bulk_load_1d(smem_u32(rows_sm + (size_t)(warp * STAGES + slot) * group_floats), head + gg * group_floats,
                   group_bytes, bar0 + 8u * slot);
    }
  };
  // STAGES - 1 groups in flight ahead of the one being decoded
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s)
      if (g + (long long)s * step < groups) issue(g + (long long)s * step, s);
  }
  uint32_t phase = 0u;  // bit s = parity of stage s
  int slot = 0;
  for (; g < groups; g += step) {
    const int nrows = (int)min((long long)32, total_rows - g * 32);
    float* my = rows_sm + (size_t)(warp * STAGES + slot) * group_floats;
    {
      // refill the stage that was drained in the previous iteration (its readers passed the __syncwarp below)
      const long long gn = g + (long long)(STAGES - 1) * step;
      const int sn = slot == 0 ? STAGES - 1 : slot - 1;
      if (lane == 0 && gn < groups) issue(gn, sn);
    }
    if (g < full_groups) {
      mbar_wait(bar0 + 8u * slot, (phase >> slot) & 1u);
      phase ^= 1u << slot;
    } else {  // ragged last group: plain loads
      const float* src = head + g * group_floats;
      for (int i = lane; i < nrows * row; i += 32) my[i] = __ldg(src + i);
      __syncwarp();
    }
    const bool active = lane < nrows;
    int lb = b, ln = n + lane;
    while (ln >= N) {
      ln -= N;
      ++lb;
    }
    const bool one_image = (n + nrows <= N);  // warp-uniform
    const float* r = my + lane * row;
    // pass bits: the scores themselves are NOT kept in registers across the ballot section: score(c) recomputes the
    // (few) passing ones from the staged row and two saved scalars, bit-identically.
    unsigned pass[W];
#pragma unroll
    for (int w = 0; w < W; ++w) pass[w] = 0u;
    float k0 = 0.f, k1 = 0.f;  // SSD: (max logit, 1/sum); YOLO / FCOS: (sigmoid(obj | ctr), unused)
    if (KIND == ODT_DECODE_SSD) {
      // softmax over 21 logits, TF form exp(x-max) * (1/sum); rows whose arg-max (first maximum) is the
      // background (last index) are dropped: background wins only if strictly greater than every foreground
      // probability.  ref SSD300.py:159-164
      float e[21];
#pragma unroll
      for (int i = 0; i < 21; ++i) e[i] = r[i];
      float m = e[0];
#pragma unroll
      for (int i = 1; i < 21; ++i) m = fmaxf(m, e[i]);
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 21; ++i) {
        e[i] = exp_score(__fsub_rn(e[i], m));
        s = __fadd_rn(s, e[i]);
      }
      const float inv = __frcp_rn(s);
      float best_fg = -1.f;
      unsigned bits = 0u;
#pragma unroll
      for (int i = 0; i < 20; ++i) {
        const float pi = __fmul_rn(e[i], inv);
        best_fg = fmaxf(best_fg, pi);
        bits |= (pi >= p.score_thr) ? (1u << i) : 0u;
      }
      if (!active || __fmul_rn(e[20], inv) > best_fg) bits = 0u;
      pass[0] = bits;
      k0 = m;
      k1 = inv;
    } else {
      // ref YOLOv3.py:338-339,349; FCOS.py:197-201: objectness / centre-ness behind the class scores
      k0 = sigmoid_score(r[KIND == ODT_DECODE_YOLO3 ? nfg + 4 : nfg]);
      // sigmoid_score <= 1 and rounding is monotone, so __fmul_rn(sigmoid_score(x), k0) <= k0: when k0 is below the
      // threshold no class of the row can pass (exact).  Most YOLO rows have a low objectness.
      if (active && (NFG || !(k0 < p.score_thr))) {
#pragma unroll
        for (int w = 0; w < W; ++w) {
          const int cend = NFG ? (NFG - 32 * w < 32 ? NFG - 32 * w : 32) : min(32, nfg - 32 * w);
          unsigned bits = 0u;
#pragma unroll(NFG ? 32 : 4)
          for (int i = 0; i < cend; ++i)
            bits |= (__fmul_rn(sigmoid_score(r[32 * w + i]), k0) >= p.score_thr) ? (1u << i) : 0u;
          pass[w] = bits;
        }
      }
    }
    auto score = [&](int c) -> float {
      if (KIND == ODT_DECODE_SSD) return __fmul_rn(exp_score(__fsub_rn(r[c], k0)), k1);
      return __fmul_rn(sigmoid_score(r[c]), k0);
    };
#pragma unroll
    for (int w = 0; w < W; ++w) {
      if (32 * w >= nfg) break;  // warp-uniform
      const unsigned pass_bits = pass[w];
      const int cbase = 32 * w;
      // classes with at least one candidate in this warp: the work below is proportional to their number
      const unsigned any = __reduce_or_sync(0xffffffffu, pass_bits);
      if (any == 0u) continue;
      if (one_image) {
        // lane i collects the ballot of class cbase + i, then reserves the slots of its class with ONE atomic: up to
        // 32 independent atomics in flight instead of dependent round trips
        unsigned my_mask = 0u;
        for (unsigned rem = any; rem; rem &= rem - 1u) {
          const int c = __ffs(rem) - 1;  // warp-uniform
          const unsigned mk = __ballot_sync(0xffffffffu, (pass_bits >> c) & 1u);
          if (lane == c) my_mask = mk;
        }
        // image index b (warp-uniform), NOT the lane's own lb: lane c only carries class c's ballot and may be an
        // inactive lane of a ragged last group, whose row index lies past the image
        int my_base = 0;
        if (my_mask) my_base = atomicAdd(&cand_count[b * p.num_fg + cbase + lane], __popc(my_mask));
        for (unsigned rem = any; rem; rem &= rem - 1u) {
          const int c = __ffs(rem) - 1;
          const unsigned mk = __shfl_sync(0xffffffffu, my_mask, c);
          const int base = __shfl_sync(0xffffffffu, my_base, c);
          if ((pass_bits >> c) & 1u) {
            const int slot_i = base + __popc(mk & ((1u << lane) - 1));
            if (slot_i < p.cap)
              cand_keys[((long long)b * p.num_fg + cbase + c) * p.cap + slot_i] =
                  ((unsigned long long)__float_as_uint(score(cbase + c)) << 32) | (0xFFFFFFFFu - (unsigned)ln);
          }
        }
      } else {
        for (unsigned rem_c = any; rem_c; rem_c &= rem_c - 1u) {
          const int c = __ffs(rem_c) - 1;
          const bool ok = (pass_bits >> c) & 1u;
          const unsigned mask = __ballot_sync(0xffffffffu, ok);
          // rows of this warp straddle images: aggregate the counter update per image
          unsigned rem = mask;
          int slot_i = -1;
          while (rem) {
            const int leader = __ffs(rem) - 1;
            const int bl = __shfl_sync(0xffffffffu, lb, leader);
            const unsigned grp = __ballot_sync(0xffffffffu, ok && lb == bl);
            int base = 0;
            if (lane == leader) base = atomicAdd(&cand_count[bl * p.num_fg + cbase + c], __popc(grp));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (ok && lb == bl) slot_i = base + __popc(grp & ((1u << lane) - 1));
            rem &= ~grp;
          }
          if (ok && slot_i < p.cap)
            cand_keys[((long long)lb * p.num_fg + cbase + c) * p.cap + slot_i] =
                ((unsigned long long)__float_as_uint(score(cbase + c)) << 32) | (0xFFFFFFFFu - (unsigned)ln);
        }
      }
    }
    __syncwarp();  // every lane is done with this stage before lane 0 refills it (next iteration's issue)
    if (++slot == STAGES) slot = 0;
    n += adv_n;
    b += adv_b;
    if (n >= N) {
      n -= N;
      ++b;
    }
  }
}

// ----------------------------------------------------------------- NMS ----
constexpr int kNmsThreads = 256;
constexpr int kNmsSmemKeys = 1024;  // candidates (keys + boxes, 24 KB) a CTA works on in shared memory: 8 CTAs / SM

constexpr int kNselOverflowBit = 1 << 30;  // per-(image, class) "list was truncated at cap" flag in nsel_all

// Class-major compaction of one image's per-class results into its packed record, run by whoever finishes the
// image's LAST list: `nt` cooperating threads with ranks `t` (nt = 32 -> one warp, barriers are __syncwarp; nt = block
// size -> __syncthreads), `s_off`: C + 1 ints of shared memory (C <= kMaxFg).  The first warp of the group computes the
// prefix sum, 32 classes per pass with a running carry (one load per lane and pass: one L2 round trip for C <= 32).
__device__ __forceinline__ void compact_image(int b, int C, int MB, int t, int nt, int* s_off, const int* nsel_all,
                                              const float* st_det, const int* st_anchor, float* dets,
                                              long long det_img_stride, int* det_anchor, int* det_count, int* work) {
  const long long D = (long long)C * MB;
  float* img_dets = dets + (long long)b * det_img_stride;
  if (t < 32) {
    const int lane = t;
    int acc = 0, ovf = 0;
    for (int c0 = 0; c0 < C; c0 += 32) {
      const int v = c0 + lane < C ? __ldcg(nsel_all + (long long)b * C + c0 + lane) : 0;
      const int n_l = v & ~kNselOverflowBit;
      int incl = n_l;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int up = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += up;
      }
      if (c0 + lane < C) s_off[c0 + lane] = acc + incl - n_l;
      acc += __shfl_sync(0xffffffffu, incl, 31);
      ovf |= __any_sync(0xffffffffu, (v & kNselOverflowBit) != 0);
    }
    if (lane == 0) {
      s_off[C] = acc;
      det_count[b] = acc;
      work[b] = 0;
      // packed record (the unit the multi-GPU all-gather and the host read-back ship): the two floats
      // behind an image's D rows carry its detection count and its overflow flag
      if (det_img_stride >= D * 6 + 2) {
        img_dets[D * 6] = (float)acc;
        img_dets[D * 6 + 1] = ovf ? 1.f : 0.f;
      }
    }
  }
  if (nt == 32) __syncwarp(); else __syncthreads();
  for (int i = t; i < C * MB; i += nt) {
    const int ci = i / MB, k = i % MB;
    const int ns = s_off[ci + 1] - s_off[ci];
    if (k < ns) {
      const long long dst = s_off[ci] + k;
      const float* sp = st_det + (((long long)b * C + ci) * MB + k) * 6;
#pragma unroll
      for (int q = 0; q < 6; ++q) img_dets[dst * 6 + q] = __ldcg(sp + q);
      det_anchor[(long long)b * D + dst] = __ldcg(st_anchor + ((long long)b * C + ci) * MB + k);
    }
  }
}

// Optional timeline of block (0, 0)'s greedy rounds (compile with -DODT_NMS_TIMELINE; off in the product build):
// thread 0 stamps clock64 at the top of a round, after the arg-max barrier and after the suppression barrier
// (scripts/nms_timeline.py).  Entries: (clock, event << 32 | round).
#ifdef ODT_NMS_TIMELINE
__device__ unsigned long long* g_nms_tl_buf = nullptr;
__device__ unsigned int g_nms_tl_cap = 0, g_nms_tl_len = 0;
__device__ __forceinline__ void nms_stamp(int event, int round) {
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && g_nms_tl_buf) {
    const unsigned int i = atomicAdd(&g_nms_tl_len, 1u);
    if (i < g_nms_tl_cap) {
      g_nms_tl_buf[2 * i] = (unsigned long long)clock64();
      g_nms_tl_buf[2 * i + 1] = ((unsigned long long)event << 32) | (unsigned)round;
    }
  }
}
#else
#define nms_stamp(event, round) ((void)0)
#endif

// barrier over the first `nthr` threads of the block (a multiple of 32); id 1 (0 is __syncthreads)
__device__ __forceinline__ void nms_round_barrier(int nthr) {
  asm volatile("bar.sync 1, %0;" ::"r"(nthr) : "memory");
}

struct NmsSmem {
  unsigned long long keys[kNmsSmemKeys];
  float4 box[kNmsSmemKeys];
};

// Exact TF NonMaxSuppressionV3 without a sort: greedy NMS always picks the
// highest-scoring candidate that no kept box suppresses, so each round is
//   (1) block-wide arg-max over the still-alive keys   (key = score bits << 32 | ~row:
//       unique, so "highest score, lowest row on ties" is a plain u64 max),
//   (2) keep it, (3) kill every alive candidate whose IoU with it exceeds the
//   threshold (strict >).
// Rounds = number of kept boxes <= nms_max_boxes (10-20), work per round =
// alive candidates / 256 threads -- no O(n log^2 n) sort, no capacity cliff: lists
// longer than the shared-memory window are processed in place in global memory
// with boxes decoded on the fly.
//
// Long lists (> kNmsPrefilter) first try an exact prefilter: a radix select on the score
// bits finds a threshold T with kNmsSelectMin..kNmsSmemKeys candidates at or above it, and
// the rounds run on that subset S in shared memory.  Greedy NMS visits candidates in
// descending score order, so if nms_max_boxes boxes are kept inside S the result is the
// exact global one (every kept box and every candidate that could have suppressed or
// preceded it has score >= T and therefore is in S).  Only if S runs dry first is the full
// list processed (correct, slower).
constexpr int kNmsPrefilter = kNmsSmemKeys;  // longer lists: prefilter first
constexpr int kNmsSelectMin = 384;

__global__ void __launch_bounds__(kNmsThreads)
    nms_per_class_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp, int B,
                         unsigned long long* __restrict__ cand_keys,
                         const int* __restrict__ cand_count, float* __restrict__ dets,
                         int* __restrict__ det_anchor, int* __restrict__ det_count,
                         int* __restrict__ scratch, int* __restrict__ work,
                         int* __restrict__ status, float4* __restrict__ box_pool,
                         long long box_pool_entries, long long det_img_stride) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NmsSmem& sm = *reinterpret_cast<NmsSmem*>(smem_raw);
  __shared__ long long s_pool_start;
  __shared__ unsigned long long s_wkey[kNmsThreads / 32];
  __shared__ int s_wpos[kNmsThreads / 32];
  __shared__ int s_last;
  __shared__ int s_nsel;
  __shared__ int s_hist[256];
  __shared__ unsigned s_ctl[4];  // radix select: [0] done flag, [1] prefix / threshold, [2] count above the bin, [3] subset fill
  const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int C = p.nms_classes, MB = p.max_boxes;
  // staging: per (b,c): nsel + MB * (6 floats + anchor)
  int* nsel_all = scratch;                                       // [B*C]
  float* st_det = reinterpret_cast<float*>(scratch + B * C);     // [B*C*MB*6]
  int* st_anchor = scratch + B * C + (long long)B * C * MB * 6;  // [B*C*MB]
  const long long bc = (long long)b * C + c;

  int cnt = cand_count[b * p.num_fg + c];
  const bool overflow = cnt > p.cap;
  if (overflow) {
    if (tid == 0) atomicExch(status, ODT_ERR_OVERFLOW);
    cnt = p.cap;
  }
  unsigned long long* gkeys = cand_keys + ((long long)b * p.num_fg + c) * p.cap;
  const int row = row_floats(p.num_fg);
  const float* hb = head + (long long)b * p.N * row;
  const int cnt_all = cnt;
  int nsel = 0;
  {
  for (int attempt = 0; attempt < 2; ++attempt) {
  // ---- attempt 0 on a long list: exact prefilter (see the kernel comment) ----
  bool subset = false;
  cnt = cnt_all;
  if (attempt == 0 && cnt_all > kNmsPrefilter) {
    unsigned prefix = 0u, prefix_mask = 0u;
    bool done = false;
    for (int shift = 24; shift >= 0 && !done; shift -= 8) {
      s_hist[tid] = 0;  // kNmsThreads == 256 bins
      if (tid == 0 && shift == 24) s_ctl[2] = 0u;
      __syncthreads();
      // four independent loads in flight per thread (a 15 000-entry list is 15 dependent L2 round trips per pass
      // instead of 60); only the score half of the key is read
      const unsigned* gscore = reinterpret_cast<const unsigned*>(gkeys) + 1;
      for (int i = tid; i < cnt_all; i += kNmsThreads * 4) {
        unsigned sc4[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int ii = i + u * kNmsThreads;
          sc4[u] = ii < cnt_all ? gscore[2 * ii] : 0u;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int ii = i + u * kNmsThreads;
          if (ii < cnt_all && (sc4[u] & prefix_mask) == prefix) atomicAdd(&s_hist[(sc4[u] >> shift) & 255u], 1);
        }
      }
      __syncthreads();
      if (tid == 0) {
        unsigned cum = s_ctl[2];
        s_ctl[0] = 0u;
        for (int bin = 255; bin >= 0; --bin) {
          const unsigned h = (unsigned)s_hist[bin];
          if (cum + h >= (unsigned)kNmsSelectMin) {
            s_ctl[1] = prefix | ((unsigned)bin << shift);
            if (cum + h <= (unsigned)kNmsSmemKeys) s_ctl[0] = 1u;  // threshold = low end of this bin
            else s_ctl[2] = cum;                                    // refine inside this bin
            break;
          }
          cum += h;
        }
      }
      __syncthreads();
      done = s_ctl[0] != 0u;
      prefix = s_ctl[1];
      prefix_mask |= 0xFFu << shift;
    }
    if (done) {  // (more than kNmsSmemKeys identical scores otherwise: full path)
      const unsigned thr_bits = prefix;
      if (tid == 0) s_ctl[3] = 0u;
      __syncthreads();
      for (int i = tid; i < cnt_all; i += kNmsThreads * 4) {
        unsigned long long k4[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int ii = i + u * kNmsThreads;
          k4[u] = ii < cnt_all ? gkeys[ii] : 0ull;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const unsigned long long k = k4[u];
          if (i + u * kNmsThreads < cnt_all && (unsigned)(k >> 32) >= thr_bits) {
            const unsigned slot = atomicAdd(&s_ctl[3], 1u);
            sm.keys[slot] = k;
            const int n = (int)(0xFFFFFFFFu - (unsigned)(k & 0xFFFFFFFFull));
            Cell cell = locate(p, n);
            sm.box[slot] = decode_box(p, cell, hb + (long long)n * row);
          }
        }
      }
      __syncthreads();
      cnt = (int)s_ctl[3];
      subset = true;
    }
  }
  const bool in_smem = subset || cnt <= kNmsSmemKeys;
  unsigned long long* keys = in_smem ? sm.keys : gkeys;
  // boxes of a list longer than the shared-memory window are decoded ONCE into a
  // slice of the global box pool (bump-allocated per launch); only if the pool is
  // exhausted are they re-decoded on the fly every round (correct, slower)
  const float4* pbox = nullptr;
  if (subset) {
    // already staged
  } else if (in_smem) {
    for (int i = tid; i < cnt; i += blockDim.x) {
      const unsigned long long k = gkeys[i];
      sm.keys[i] = k;
      const int n = (int)(0xFFFFFFFFu - (unsigned)(k & 0xFFFFFFFFull));
      Cell cell = locate(p, n);
      sm.box[i] = decode_box(p, cell, hb + (long long)n * row);
    }
  } else {
    if (tid == 0) {
      long long start = -1;
      if (box_pool) {
        start = (long long)atomicAdd(reinterpret_cast<unsigned long long*>(work + ((B + 1) & ~1)),
                                     (unsigned long long)cnt);
        if (start + cnt > box_pool_entries) start = -1;
      }
      s_pool_start = start;
    }
    __syncthreads();
    if (s_pool_start >= 0) {
      float4* wb = box_pool + s_pool_start;
      for (int i = tid; i < cnt; i += blockDim.x) {
        const int n = (int)(0xFFFFFFFFu - (unsigned)(gkeys[i] & 0xFFFFFFFFull));
        Cell cell = locate(p, n);
        wb[i] = decode_box(p, cell, hb + (long long)n * row);
      }
      pbox = wb;
    }
  }
  __syncthreads();

  // Greedy rounds.  A round costs every participating warp ~150 instructions whatever the list length, and with all
  // lists of a batch resident (SSD300 B=64: 1 280 blocks, 8 per SM) the kernel is bound by that instruction count:
  // only as many warps as the list can feed (64 candidates each, at least 2) take part; the others wait at the
  // block barrier after the loop.
  const int nw = min(kNmsThreads / 32, max(2, (cnt + 63) / 64));
  const int nthr = nw * 32;
  nsel = 0;
  if (tid < nthr) {
  while (nsel < MB && cnt > 0) {
    nms_stamp(0, nsel);
    // (1) arg-max over alive keys: per-thread scan, 3 redux.sync per warp, then every
    //     thread folds the warp partials itself (one barrier, no second shuffle tree)
    unsigned long long bk = 0ull;
    int bp = 0x7fffffff;
    for (int i = tid; i < cnt; i += nthr) {
      const unsigned long long k = keys[i];
      if (k > bk) {
        bk = k;
        bp = i;
      }
    }
    {
      const unsigned hi = (unsigned)(bk >> 32), lo = (unsigned)bk;
      const unsigned whi = __reduce_max_sync(0xffffffffu, hi);
      const unsigned wlo = __reduce_max_sync(0xffffffffu, hi == whi ? lo : 0u);
      const int wpos = __reduce_min_sync(0xffffffffu, (hi == whi && lo == wlo) ? bp : 0x7fffffff);
      if (lane == 0) {
        s_wkey[warp] = ((unsigned long long)whi << 32) | wlo;
        s_wpos[warp] = wpos;
      }
    }
    nms_round_barrier(nthr);
    nms_stamp(1, nsel);
    unsigned long long s_best_key = 0ull;
    int s_best_pos = -1;
#pragma unroll
    for (int w = 0; w < kNmsThreads / 32; ++w) {
      const unsigned long long k = w < nw ? s_wkey[w] : 0ull;
      if (k > s_best_key) {
        s_best_key = k;
        s_best_pos = s_wpos[w];
      }
    }
    const unsigned long long hk = s_best_key;
    const int hp = s_best_pos;
    if (hk == 0ull) break;  // nothing alive
    // (2) keep it
    const int hn = (int)(0xFFFFFFFFu - (unsigned)(hk & 0xFFFFFFFFull));
    float4 cur;
    if (in_smem) {
      cur = sm.box[hp];
    } else if (pbox) {
      cur = pbox[hp];
    } else {
      Cell cell = locate(p, hn);
      cur = decode_box(p, cell, hb + (long long)hn * row);
    }
    if (tid == 0) {
      float* d = st_det + (bc * MB + nsel) * 6;
      d[0] = __uint_as_float((unsigned)(hk >> 32));
      d[1] = cur.x;
      d[2] = cur.y;
      d[3] = cur.z;
      d[4] = cur.w;
      d[5] = (float)c;
      st_anchor[bc * MB + nsel] = hn;
    }
    ++nsel;
    if (nsel >= MB) break;
    // (3) suppress (strict >, TF IoU); the thread that owns slot hp retires the kept key itself (one writer per
    // slot between two barriers: compute-sanitizer racecheck flagged the former "thread 0 clears it" as a RAW hazard,
    // benign but avoidable)
    for (int j = tid; j < cnt; j += nthr) {
      if (j == hp) {
        keys[j] = 0ull;
        continue;
      }
      const unsigned long long kj = keys[j];
      if (kj == 0ull) continue;
      float4 bj;
      if (in_smem) {
        bj = sm.box[j];
      } else if (pbox) {
        bj = pbox[j];
      } else {
        const int n = (int)(0xFFFFFFFFu - (unsigned)(kj & 0xFFFFFFFFull));
        Cell cell = locate(p, n);
        bj = decode_box(p, cell, hb + (long long)n * row);
      }
      if (iou_tf(bj, cur) > p.iou_thr) keys[j] = 0ull;
    }
    nms_round_barrier(nthr);
    nms_stamp(2, nsel);
  }
  if (tid == 0) s_nsel = nsel;
  }
  __syncthreads();
  nsel = s_nsel;  // the warps that sat the rounds out learn the outcome here
  // the subset ran dry before nms_max_boxes boxes were kept: redo on the full list
  if (!(subset && nsel < MB && cnt < cnt_all)) break;
  }  // attempt
  }  // long list
  // class-major compaction by whoever finishes the image's last list
  if (tid == 0) {
    nsel_all[bc] = nsel | (overflow ? kNselOverflowBit : 0);
    __threadfence();  // this thread wrote the kept boxes and the count: release them before the counter moves
    const int done = atomicAdd(&work[b], 1);
    s_last = (done == C - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  __shared__ int s_off[kMaxFg + 1];
  compact_image(b, C, MB, tid, kNmsThreads, s_off, nsel_all, st_det, st_anchor, dets, det_img_stride, det_anchor,
                det_count, work);
}

}  // namespace odt

using namespace odt;

static int check_tail(const odt_tail_params* p) {
  ODT_CHECK_ARG(p != nullptr, "params null");
  ODT_CHECK_ARG(p->kind >= 0 && p->kind <= 2, "kind");
  ODT_CHECK_ARG(p->num_levels >= 1 && p->num_levels <= ODT_MAX_LEVELS, "num_levels");
  // the softmax family (SSD / RetinaNet) decodes 21 logits; YOLOv3 / FCOS rows carry 1..kMaxFg class scores
  if (p->kind == ODT_DECODE_SSD) ODT_CHECK_ARG(p->num_fg == 20, "num_fg must be 20 for the softmax family");
  else ODT_CHECK_ARG(p->num_fg >= 1 && p->num_fg <= kMaxFg, "num_fg must be 1..128");
  // 0 NMS classes: FCOS with one class visits range(num_classes - 1) = no class (ref FCOS.py:252)
  ODT_CHECK_ARG(p->nms_classes >= 0 && p->nms_classes <= p->num_fg, "nms_classes");
  ODT_CHECK_ARG(p->N > 0 && p->cap > 0 && p->max_boxes > 0, "N/cap/max_boxes");
  for (int i = 0; i < p->num_levels; ++i)
    ODT_CHECK_ARG(p->level[i].A >= 1 && p->level[i].A <= ODT_MAX_PRIORS, "level.A");
  return ODT_OK;
}

// Records of a tail without NMS classes: every image's count and overflow flag are 0 (D = 0).
__global__ void empty_records_kernel(int B, float* __restrict__ dets, long long det_img_stride,
                                     int* __restrict__ det_count, int* __restrict__ work) {
  pdl_launch_dependents();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  det_count[b] = 0;
  work[b] = 0;
  if (det_img_stride >= 2) {
    dets[(long long)b * det_img_stride] = 0.f;
    dets[(long long)b * det_img_stride + 1] = 0.f;
  }
}

extern "C" int odt_decode_candidates(const float* head, const odt_tail_params* p, int B,
                                     unsigned long long* cand_keys, int* cand_count,
                                     void* stream) {
  int rc = check_tail(p);
  if (rc) return rc;
  ODT_CHECK_ARG(head && cand_keys && cand_count && B > 0, "null pointer / B");
  ODT_CHECK_ARG(((uintptr_t)head & 15) == 0, "head must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  ODT_CUDA_OK(cudaMemsetAsync(cand_count, 0, sizeof(int) * (size_t)B * p->num_fg, st));
  TailP tp;
  tp.p = *p;
  long long rows = (long long)B * p->N;
  long long groups = (rows + 31) / 32;
  // 25-float rows (num_fg = 20, every family): 8 warps per CTA, 3 CTAs / SM with 2 stages per warp (24 warps x 1
  // group in flight ahead).  Other class counts (YOLOv3 / FCOS): 4 warps x 2 stages, as many CTAs per SM as their
  // staging allows.
  const bool wide = p->num_fg != 20;
  const int warps = wide ? kDecodeWarpsWide : kDecodeWarps;
  int blocks = (int)((groups + warps - 1) / warps);
  int per_sm = 6;  // 2-3 CTAs resident per SM: two to three waves
  if (wide) {
    const long long smem = decode_smem_bytes(kDecodeWarpsWide, 2, row_floats(p->num_fg));
    per_sm = (int)(2 * ((228 * 1024) / (smem + 1024)));  // two waves of the CTAs that fit (1 KB reserved per CTA)
  }
  // a smaller grid makes every warp iterate several times at sizes a test can afford
  if (const char* e = getenv("ODT_DECODE_BLOCKS_PER_SM")) per_sm = atoi(e) > 0 ? atoi(e) : per_sm;
  int maxb = kNumSMs * per_sm;
  if (blocks > maxb) blocks = maxb;
#define ODT_DECODE_LAUNCH(KIND_, WARPS_, OCC_, ST_, NFG_, SMEM_MAX_)                                               \
  do {                                                                                                           \
    static bool attr_done = false;                                                                               \
    if (!attr_done) {                                                                                            \
      ODT_CUDA_OK(cudaFuncSetAttribute(decode_candidates_kernel<KIND_, WARPS_, OCC_, ST_, NFG_>,                 \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(SMEM_MAX_)));           \
      attr_done = true;                                                                                          \
    }                                                                                                            \
    decode_candidates_kernel<KIND_, WARPS_, OCC_, ST_, NFG_>                                                     \
        <<<blocks, (WARPS_) * 32, decode_smem_bytes(WARPS_, ST_, row_floats(p->num_fg)), st>>>(                  \
            head, tp, rows, cand_keys, cand_count);                                                              \
  } while (0)
#define ODT_DECODE_LAUNCH20(KIND_) \
  ODT_DECODE_LAUNCH(KIND_, kDecodeWarps, 3, 2, 20, decode_smem_bytes(kDecodeWarps, 2, row_floats(20)))
#define ODT_DECODE_LAUNCH_WIDE(KIND_) \
  ODT_DECODE_LAUNCH(KIND_, kDecodeWarpsWide, 1, 2, 0, decode_smem_bytes(kDecodeWarpsWide, 2, row_floats(kMaxFg)))
  if (p->kind == ODT_DECODE_SSD) {
    ODT_DECODE_LAUNCH20(ODT_DECODE_SSD);
  } else if (p->kind == ODT_DECODE_YOLO3) {
    if (wide) ODT_DECODE_LAUNCH_WIDE(ODT_DECODE_YOLO3); else ODT_DECODE_LAUNCH20(ODT_DECODE_YOLO3);
  } else {
    if (wide) ODT_DECODE_LAUNCH_WIDE(ODT_DECODE_FCOS); else ODT_DECODE_LAUNCH20(ODT_DECODE_FCOS);
  }
#undef ODT_DECODE_LAUNCH_WIDE
#undef ODT_DECODE_LAUNCH20
#undef ODT_DECODE_LAUNCH
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" long long odt_nms_scratch_bytes(const odt_tail_params* p, int B) {
  if (!p || B <= 0) return -1;
  long long bc = (long long)B * p->nms_classes;
  return bc * 4 + bc * p->max_boxes * 6 * 4 + bc * p->max_boxes * 4;
}

extern "C" int odt_nms_per_class(const float* head, const odt_tail_params* p, int B,
                                 unsigned long long* cand_keys, const int* cand_count, float* dets,
                                 int* det_anchor, int* det_count, int* sel_scratch, int* work,
                                 int* status, float* box_pool, long long box_pool_entries,
                                 long long dets_img_stride, void* stream) {
  int rc = check_tail(p);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (p->nms_classes == 0) {  // no list to visit (D = 0): the records still get their count and overflow flag
    ODT_CHECK_ARG(dets && det_count && work && status && B > 0, "null pointer / B");
    ODT_CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int), st));
    empty_records_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, dets, dets_img_stride, det_count, work);
    ODT_LAUNCH_OK();
    return ODT_OK;
  }
  ODT_CHECK_ARG(head && cand_keys && cand_count && dets && det_anchor && det_count &&
                    sel_scratch && work && status && B > 0,
                "null pointer / B");
  static bool attr_set = false;
  if (!attr_set) {
    ODT_CUDA_OK(cudaFuncSetAttribute(nms_per_class_kernel,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)sizeof(NmsSmem)));
    attr_set = true;
  }
  TailP tp;
  tp.p = *p;
  dim3 grid(p->nms_classes, B);
  int* pool_ctr = work + ((B + 1) & ~1);  // 64-bit bump pointer behind the per-image counters
  ODT_CHECK_ARG(((uintptr_t)pool_ctr & 7) == 0 || !box_pool, "work must be 8-byte aligned");
  ODT_CHECK_ARG(((uintptr_t)box_pool & 15) == 0, "box_pool must be 16-byte aligned");
  if (box_pool) ODT_CUDA_OK(cudaMemsetAsync(pool_ctr, 0, 8, st));  // pool bump pointer
  ODT_CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int), st));        // the status word describes THIS launch
  const long long dense = (long long)p->nms_classes * p->max_boxes * 6;
  if (dets_img_stride == 0) dets_img_stride = dense;
  ODT_CHECK_ARG(dets_img_stride >= dense, "dets_img_stride smaller than nms_classes*max_boxes*6");
  nms_per_class_kernel<<<grid, kNmsThreads, sizeof(NmsSmem), st>>>(
      head, tp, B, cand_keys, cand_count, dets, det_anchor, det_count, sel_scratch, work, status,
      reinterpret_cast<float4*>(box_pool), box_pool ? box_pool_entries : 0, dets_img_stride);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

#ifdef ODT_NMS_TIMELINE
// Debug build only (scripts/nms_timeline.py): device buffer of `cap` (clock, tag) pairs for block (0, 0)'s rounds.
extern "C" int odt_debug_nms_timeline(void* buf, int cap) {
  unsigned long long* b = reinterpret_cast<unsigned long long*>(buf);
  unsigned int c = (unsigned int)cap, z = 0;
  ODT_CUDA_OK(cudaMemcpyToSymbol(odt::g_nms_tl_buf, &b, sizeof(b)));
  ODT_CUDA_OK(cudaMemcpyToSymbol(odt::g_nms_tl_cap, &c, sizeof(c)));
  ODT_CUDA_OK(cudaMemcpyToSymbol(odt::g_nms_tl_len, &z, sizeof(z)));
  return ODT_OK;
}
#endif
