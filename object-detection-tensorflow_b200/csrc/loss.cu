// Training-loss forwards of the five families (RetinaNet, SSD, FCOS, YOLOv3, YOLOv2), forward only.
// RetinaNet (BASELINE config 3 "focal-loss + decode + NMS"): anchor/GT matching, softmax focal loss and
// smooth-L1 box loss.  Restates RetinaNet.py:357-474 (never copied):
//   * GT rows (y,x,h,w,id) padded with -1; valid count = index of first -1 in col 0
//   * IoU[G,A]; for every GT its arg-max anchor is a positive ("best", duplicates kept);
//     the remaining anchors: max IoU > 0.5 -> positive with the arg-max GT,
//     max IoU < 0.4 -> negative (label = background = last class), else ignored
//   * focal: p = clip(softmax(logits)[label], 1e-8, 1); -alpha (1-p)^gamma log p,
//     the same alpha for positives and negatives; sum / #positives
//   * box: smooth-L1 of (t_yx - (g_yx-a_yx)/a_hw) and (t_hw - log(g_hw/a_hw)), mean over positives
// Sums are reduced in a fixed order (per-block partials, then a serial final
// pass) so the result is run-to-run deterministic.
#include "tail_common.cuh"

namespace odt {

constexpr int kLossBlocks = 64;   // anchor blocks per image
constexpr int kLossThreads = 256;
constexpr int kMaxGT = 128;

__device__ __forceinline__ float iou_match(const Anchor& a, float gy1, float gx1, float gy2,
                                           float gx2, float garea) {
  // ref RetinaNet.py:383-388
  float iy1 = fmaxf(a.y1, gy1), ix1 = fmaxf(a.x1, gx1);
  float iy2 = fminf(a.y2, gy2), ix2 = fminf(a.x2, gx2);
  float inter = __fmul_rn(fmaxf(__fsub_rn(iy2, iy1), 0.f), fmaxf(__fsub_rn(ix2, ix1), 0.f));
  float aarea = __fmul_rn(a.h, a.w);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(aarea, garea), inter));
}

__device__ __forceinline__ int gt_count(const float* gt, int G) {
  // tf.argmin(gt, axis=0)[0]: first index of the column minimum (ref :359)
  int arg = 0;
  float best = gt[0];
  for (int i = 1; i < G; ++i) {
    float v = gt[i * 5];
    if (v < best) {
      best = v;
      arg = i;
    }
  }
  return arg;
}

// gt_count of the block's image, computed by thread 0 and handed to every thread
__device__ __forceinline__ int block_gt_count(const float* gb, int G) {
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = gt_count(gb, G);
  __syncthreads();
  return s_cnt;
}

// GT row g, centre form (y, x, h, w) -> corners and area, in the op order iou_match expects
struct GtBox {
  float y1, x1, y2, x2, area;
};
__device__ __forceinline__ GtBox gt_box(const float* gb, int g) {
  const float gy = gb[g * 5], gx = gb[g * 5 + 1], gh = gb[g * 5 + 2], gw = gb[g * 5 + 3];
  const float hh = __fmul_rn(gh, 0.5f), hw = __fmul_rn(gw, 0.5f);
  return {__fsub_rn(gy, hh), __fsub_rn(gx, hw), __fadd_rn(gy, hh), __fadd_rn(gx, hw), __fmul_rn(gh, gw)};
}

// Fixed-order block sum of Q values over the T threads of the block: thread t contributes v[q], the halving
// tree leaves the sums in s[q][0].  The tree's order is what keeps every loss bit-identical from run to run
// and from one batch size to another.  (threadIdx.x is read where it is used: holding it in a variable across the
// tree costs fcos_loss_kernel three registers.)
template <int Q, int T>
__device__ __forceinline__ void block_sum(float (&s)[Q][T], const float (&v)[Q]) {
#pragma unroll
  for (int q = 0; q < Q; ++q) s[q][threadIdx.x] = v[q];
  __syncthreads();
  for (int o = T / 2; o; o >>= 1) {
    if (threadIdx.x < o) {
#pragma unroll
      for (int q = 0; q < Q; ++q) s[q][threadIdx.x] += s[q][threadIdx.x + o];
    }
    __syncthreads();
  }
}

// K1: per (gt, image) arg-max anchor (first maximum)
__global__ void __launch_bounds__(kLossThreads)
    loss_best_anchor_kernel(const __grid_constant__ TailP tp, const float* __restrict__ gt, int G,
                            int* __restrict__ best) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int g = blockIdx.x, b = blockIdx.y;
  const float* gb = gt + (long long)b * G * 5;
  __shared__ float s_v[kLossThreads];
  __shared__ int s_i[kLossThreads];
  if (g >= block_gt_count(gb, G)) {
    if (threadIdx.x == 0) best[b * G + g] = -1;
    return;
  }
  const GtBox box = gt_box(gb, g);
  float bv = -1.f;
  int bi = 0x7fffffff;
  for (int n = threadIdx.x; n < p.N; n += blockDim.x) {
    Cell c = locate(p, n);
    Anchor a = anchor_ssd(p, c);
    float v = iou_match(a, box.y1, box.x1, box.y2, box.x2, box.area);
    if (v > bv) {
      bv = v;
      bi = n;
    }
  }
  s_v[threadIdx.x] = bv;
  s_i[threadIdx.x] = bi;
  __syncthreads();
  for (int o = kLossThreads / 2; o; o >>= 1) {
    if (threadIdx.x < o) {
      float v2 = s_v[threadIdx.x + o];
      int i2 = s_i[threadIdx.x + o];
      if (v2 > s_v[threadIdx.x] || (v2 == s_v[threadIdx.x] && i2 < s_i[threadIdx.x])) {
        s_v[threadIdx.x] = v2;
        s_i[threadIdx.x] = i2;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) best[b * G + g] = s_i[0];
}

__device__ __forceinline__ float smooth_l1(float x) {
  float ax = fabsf(x);
  return ax < 1.f ? __fmul_rn(__fmul_rn(0.5f, x), x) : __fsub_rn(ax, 0.5f);
}

__device__ __forceinline__ void softmax21(const float* r, float* prob) {
  float m = r[0];
#pragma unroll
  for (int i = 1; i < 21; ++i) m = fmaxf(m, r[i]);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 21; ++i) {
    prob[i] = expf(__fsub_rn(r[i], m));
    s = __fadd_rn(s, prob[i]);
  }
  float inv = __fdiv_rn(1.f, s);
#pragma unroll
  for (int i = 0; i < 21; ++i) prob[i] = __fmul_rn(prob[i], inv);
}

__device__ __forceinline__ float focal(float pr, float alpha, float gamma) {
  float q = fminf(fmaxf(pr, 1e-8f), 1.f);
  return -alpha * powf(1.f - q, gamma) * logf(q);
}

__device__ __forceinline__ float coord_loss(const float* r, const Anchor& a, float gy, float gx,
                                            float gh, float gw) {
  float ty = __fdiv_rn(__fsub_rn(gy, a.cy), a.h), tx = __fdiv_rn(__fsub_rn(gx, a.cx), a.w);
  float th = logf(__fdiv_rn(gh, a.h)), tw = logf(__fdiv_rn(gw, a.w));
  float lyx = __fadd_rn(smooth_l1(__fsub_rn(r[21], ty)), smooth_l1(__fsub_rn(r[22], tx)));
  float lhw = __fadd_rn(smooth_l1(__fsub_rn(r[23], th)), smooth_l1(__fsub_rn(r[24], tw)));
  return __fadd_rn(lyx, lhw);
}

// ============================ SSD loss forward ==============================
// Restates SSD300.py:345-453 / SSD512.py (never copied):
//   * matching as above but with ONE threshold: other anchors with best IoU > 0.5 are
//     positives, all the rest are negatives;
//   * cross-entropy (sparse_softmax_cross_entropy = logsumexp(x) - x[label]), positives
//     averaged; smooth-L1 box term averaged over the positives;
//   * hard-negative mining: tf.image.non_max_suppression over the negative ANCHOR boxes
//     (yx -+ hw/2 of the anchor's centre form) scored by their background cross-entropy,
//     max_output = min(#neg, 3 * #pos), IoU 0.7; the loss is the mean of the selected ones.
__device__ __forceinline__ float xent21(const float* r, int label) {
  float m = r[0];
#pragma unroll
  for (int i = 1; i < 21; ++i) m = fmaxf(m, r[i]);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 21; ++i) s = __fadd_rn(s, expf(__fsub_rn(r[i], m)));
  return __fsub_rn(logf(s), __fsub_rn(r[label], m));
}

// classification term of row r for class `label`: SSD cross-entropy, RetinaNet softmax focal loss
template <bool kSsd>
__device__ __forceinline__ float class_loss(const float* r, int label, float alpha, float gamma) {
  if constexpr (kSsd) {
    return xent21(r, label);
  } else {
    float prob[21];
    softmax21(r, prob);
    return focal(prob[label], alpha, gamma);
  }
}

// What the matching kernel records per anchor for the gradient kernels, assign[b][n]: a value >= 0 is a positive
// matched to that GT by IoU > 0.5; the per-GT arg-max anchors are kAsBest (their GTs are found in `best`); the
// mining kernel turns the SSD negatives it selects into kAsMined.
constexpr int kAsBest = -4, kAsMined = -3, kAsIgnored = -2, kAsNegative = -1;

// K2: per-anchor assignment + loss partial sums, partial[b][blk] = (conf, coord, npos).  The families differ in
// three places: RetinaNet ignores best IoUs in [0.4, 0.5] and scores with the focal term (alpha, gamma); SSD
// scores with the cross-entropy and hands every negative to the mining kernel as a (loss, row) key in
// neg_keys / neg_count.  A matched anchor's classification term is computed once, for its GT's class or for the
// background (20).  The anchor loop is warp-uniform for the SSD ballot; each thread still visits
// n_begin + tid, + blockDim.x, ... in that order.
template <bool kSsd>
__global__ void __launch_bounds__(kLossThreads)
    loss_anchor_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp,
                       const float* __restrict__ gt, int G, const int* __restrict__ best, float alpha,
                       float gamma, float* __restrict__ partial, unsigned long long* __restrict__ neg_keys,
                       int* __restrict__ neg_count, int* __restrict__ assign) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int b = blockIdx.y, blk = blockIdx.x;
  const float* gb = gt + (long long)b * G * 5;
  __shared__ float s_gt[kMaxGT][6];  // y1,x1,y2,x2,area,(unused)
  __shared__ int s_best[kMaxGT];
  __shared__ float s_red[3][kLossThreads];
  const int cnt = block_gt_count(gb, G);
  for (int g = threadIdx.x; g < cnt; g += blockDim.x) {
    const GtBox box = gt_box(gb, g);
    s_gt[g][0] = box.y1;
    s_gt[g][1] = box.x1;
    s_gt[g][2] = box.y2;
    s_gt[g][3] = box.x2;
    s_gt[g][4] = box.area;
    s_best[g] = best[b * G + g];
  }
  __syncthreads();
  const int row = row_floats(p.num_fg);
  const float* hb = head + (long long)b * p.N * row;
  float conf = 0.f, coord = 0.f, npos = 0.f;
  auto positive = [&](const float* r, const Anchor& a, int g, float cls) {  // row r, anchor a matched to GT g
    conf += cls;
    coord += coord_loss(r, a, gb[g * 5], gb[g * 5 + 1], gb[g * 5 + 2], gb[g * 5 + 3]);
    npos += 1.f;
  };
  const int per = (p.N + kLossBlocks - 1) / kLossBlocks;
  const int n_begin = blk * per, n_end = min(p.N, n_begin + per);
  for (int n0 = n_begin; n0 < n_end; n0 += blockDim.x) {
    const int n = n0 + threadIdx.x;
    bool is_neg = false;
    float nloss = 0.f;
    if (n < n_end) {
      bool is_best = false;
      for (int g = 0; g < cnt; ++g) is_best |= (s_best[g] == n);
      int as = kAsBest;
      if (!is_best) {  // the best anchors are handled by the per-GT pass below (ref :397-411)
        Cell c = locate(p, n);
        Anchor a = anchor_ssd(p, c);
        float bv = -1.f;
        int bg = 0;
        for (int g = 0; g < cnt; ++g) {
          float v = iou_match(a, s_gt[g][0], s_gt[g][1], s_gt[g][2], s_gt[g][3], s_gt[g][4]);
          if (v > bv) {
            bv = v;
            bg = g;
          }
        }
        const bool pos = bv > 0.5f, neg = kSsd || bv < 0.4f;  // RetinaNet ignores best IoUs in [0.4, 0.5]
        as = pos ? bg : (neg ? kAsNegative : kAsIgnored);
        if (pos || neg) {
          const float* r = hb + (long long)n * row;
          const float cls = class_loss<kSsd>(r, pos ? (int)gb[bg * 5 + 4] : 20, alpha, gamma);
          if (pos) {
            positive(r, a, bg, cls);
          } else if constexpr (kSsd) {
            is_neg = true;
            nloss = cls;
          } else {
            conf += cls;
          }
        }
      }
      assign[(long long)b * p.N + n] = as;
    }
    if constexpr (kSsd) {
      // warp-aggregated append of the negatives (order is irrelevant: keys are unique)
      unsigned long long* nk = neg_keys + (long long)b * p.N;
      const unsigned mask = __ballot_sync(0xffffffffu, is_neg);
      if (mask) {
        const int lane = threadIdx.x & 31, leader = __ffs(mask) - 1;
        int base = 0;
        if (lane == leader) base = atomicAdd(&neg_count[b], __popc(mask));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (is_neg)
          nk[base + __popc(mask & ((1u << lane) - 1))] =
              ((unsigned long long)__float_as_uint(nloss) << 32) | (0xFFFFFFFFu - (unsigned)n);
      }
    }
  }
  if (blk == 0) {  // the G "best anchor" positives (duplicates kept), once per image
    for (int g = threadIdx.x; g < cnt; g += blockDim.x) {
      int n = s_best[g];
      Cell c = locate(p, n);
      const float* r = hb + (long long)n * row;
      positive(r, anchor_ssd(p, c), g, class_loss<kSsd>(r, (int)gb[g * 5 + 4], alpha, gamma));
    }
  }
  block_sum(s_red, {conf, coord, npos});
  if (threadIdx.x < 3) partial[((long long)b * kLossBlocks + blk) * 4 + threadIdx.x] = s_red[threadIdx.x][0];
}

// (conf, coord, npos) of image b: its kLossBlocks partials summed in block order
struct LossSums {
  float conf, coord, npos;
};
__device__ __forceinline__ LossSums image_sums(const float* __restrict__ partial, int b) {
  LossSums s = {0.f, 0.f, 0.f};
  for (int i = 0; i < kLossBlocks; ++i) {
    const float* q = partial + ((long long)b * kLossBlocks + i) * 4;
    s.conf += q[0];
    s.coord += q[1];
    s.npos += q[2];
  }
  return s;
}

// K3 (RetinaNet)
__global__ void loss_final_kernel(const float* __restrict__ partial, int B, float* __restrict__ out) {
  pdl_launch_dependents();
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const LossSums s = image_sums(partial, b);
  out[b] = s.conf / s.npos + s.coord / s.npos;
}

// negative anchor box in the reference's op order: yx -+ hw/2 of the centre form (:419)
__device__ __forceinline__ float4 neg_anchor_box(const odt_tail_params& p, int n) {
  Cell c = locate(p, n);
  Anchor a = anchor_ssd(p, c);
  const float hh = __fdiv_rn(a.h, 2.f), hw = __fdiv_rn(a.w, 2.f);
  return make_float4(__fsub_rn(a.cy, hh), __fsub_rn(a.cx, hw), __fadd_rn(a.cy, hh), __fadd_rn(a.cx, hw));
}

// K3 (SSD): one CTA per image: hard-negative mining (exact greedy NMS by repeated arg-max, as in
// tail.cu) + the final combination.  loss_out[b] = mean(selected neg) + conf/npos + coord/npos.  The selected rows
// become kAsMined in `assign` and their count goes to nsel_out[b], for the gradient.
__global__ void __launch_bounds__(kLossThreads)
    ssd_loss_mine_kernel(const __grid_constant__ TailP tp, const float* __restrict__ partial,
                         unsigned long long* __restrict__ neg_keys, const int* __restrict__ neg_count,
                         float* __restrict__ loss_out, int* __restrict__ info_out, int* __restrict__ assign,
                         int* __restrict__ nsel_out) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ unsigned long long s_wkey[kLossThreads / 32];
  __shared__ int s_wpos[kLossThreads / 32];
  const LossSums sums = image_sums(partial, b);
  const int npos = (int)sums.npos, cnt = neg_count[b];
  const int chosen = cnt > 3 * npos ? 3 * npos : cnt;
  unsigned long long* keys = neg_keys + (long long)b * p.N;
  double neg_sum = 0.0;  // thread 0 only
  int nsel = 0;
  while (nsel < chosen) {
    unsigned long long bk = 0ull;
    int bp = 0x7fffffff;
    for (int i = tid; i < cnt; i += blockDim.x) {
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
    __syncthreads();
    unsigned long long hk = 0ull;
    int hp = -1;
#pragma unroll
    for (int w = 0; w < kLossThreads / 32; ++w) {
      if (s_wkey[w] > hk) {
        hk = s_wkey[w];
        hp = s_wpos[w];
      }
    }
    if (hk == 0ull) break;  // every negative is selected or suppressed
    const int hn = (int)(0xFFFFFFFFu - (unsigned)(hk & 0xFFFFFFFFull));
    const float4 cur = neg_anchor_box(p, hn);
    if (tid == 0) {
      neg_sum += (double)__uint_as_float((unsigned)(hk >> 32));
      keys[hp] = 0ull;
      assign[(long long)b * p.N + hn] = kAsMined;
    }
    ++nsel;
    if (nsel >= chosen) break;
    for (int j = tid; j < cnt; j += blockDim.x) {
      const unsigned long long kj = keys[j];
      if (kj == 0ull || j == hp) continue;
      const int n = (int)(0xFFFFFFFFu - (unsigned)(kj & 0xFFFFFFFFull));
      if (iou_tf(neg_anchor_box(p, n), cur) > 0.7f) keys[j] = 0ull;
    }
    __syncthreads();
  }
  if (tid == 0) {
    loss_out[b] = (float)(neg_sum / (double)nsel) + sums.conf / sums.npos + sums.coord / sums.npos;
    nsel_out[b] = nsel;
    if (info_out) {
      info_out[b * 3 + 0] = npos;
      info_out[b * 3 + 1] = cnt;
      info_out[b * 3 + 2] = nsel;
    }
  }
}

// ============================ FCOS loss forward =============================
// Restates FCOS.py:153-187 (level assignment) and :266-348 (per-level loss), never copied:
//   * GT rows go to pyramid levels by sqrt(h*w) with inclusive, overlapping bounds
//     (<=64 | 64..128 | 128..256 | 256..512 | >=512); a level without GT contributes 0;
//   * per location (grid without +0.5, stride units): inside-box mask per GT; the regression
//     target is the inside GT of minimal area (ties: element-wise max of l,r,t,b);
//   * IoU loss -log(iou + 1e-12) over inside locations, centre-ness BCE-with-logits over ALL
//     locations of the level, sigmoid focal loss (alpha .25, gamma 2) on the per-class inside mask;
//   * level loss = (iou + focal + centre) / #(positive class cells); image loss = sum of levels.
constexpr int kFcosLevels = 5;

__device__ __forceinline__ float softplus_f(float x) {  // log(1 + exp(x)), stable
  return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));
}

// The image's GT rows staged in shared memory for the FCOS kernels: boxes in stride units of every level, class,
// level membership bits.  The caller synchronises.
struct FcosGt {
  float box[kMaxGT][kFcosLevels][4];  // y1,x1,y2,x2 in stride units of each level
  int cls[kMaxGT];
  int lv[kMaxGT];                     // level membership bits
};
__device__ __forceinline__ void fcos_stage_gt(const odt_tail_params& p, const float* gb, int cnt, FcosGt& s) {
  for (int g = threadIdx.x; g < cnt; g += blockDim.x) {
    const float gy = gb[g * 5], gx = gb[g * 5 + 1], gh = gb[g * 5 + 2], gw = gb[g * 5 + 3];
    const float size = __fsqrt_rn(__fmul_rn(gh, gw));
    int bits = 0;
    if (size <= 64.f) bits |= 1;
    if (size >= 64.f && size <= 128.f) bits |= 2;
    if (size >= 128.f && size <= 256.f) bits |= 4;
    if (size >= 256.f && size <= 512.f) bits |= 8;
    if (size >= 512.f) bits |= 16;
    s.lv[g] = bits;
    s.cls[g] = (int)gb[g * 5 + 4];
    for (int l = 0; l < kFcosLevels; ++l) {
      const float st = p.level[l].out_mul;
      const float y = __fdiv_rn(gy, st), x = __fdiv_rn(gx, st), h = __fdiv_rn(gh, st), w = __fdiv_rn(gw, st);
      const float hh = __fdiv_rn(h, 2.f), hw = __fdiv_rn(w, 2.f);
      s.box[g][l][0] = __fsub_rn(y, hh);
      s.box[g][l][1] = __fsub_rn(x, hw);
      s.box[g][l][2] = __fadd_rn(y, hh);
      s.box[g][l][3] = __fadd_rn(x, hw);
    }
  }
}

// Targets of location c: inside any GT of its level (loc), the regression distances of the inside GT of minimal
// area (ties: element-wise max of l,r,t,b), the centre-ness target, and the classes of the inside GTs as a bit mask
// of W words.
struct FcosCell {
  bool loc;
  float dl, dr, dt, db, cgt;
};
template <int W>
__device__ __forceinline__ FcosCell fcos_cell(const Cell& c, int cnt, const FcosGt& s, unsigned (&cmask)[W]) {
  const int l = c.lvl;
  const float yy = (float)c.y, xx = (float)c.x;
  bool loc = false;
  float amin = 3.0e38f, dl = 0.f, dr = 0.f, dt = 0.f, db = 0.f;
#pragma unroll
  for (int w = 0; w < W; ++w) cmask[w] = 0u;
  for (int g = 0; g < cnt; ++g) {
    if (!((s.lv[g] >> l) & 1)) continue;
    const float l_ = __fsub_rn(xx, s.box[g][l][1]), r_ = __fsub_rn(s.box[g][l][3], xx);
    const float t_ = __fsub_rn(yy, s.box[g][l][0]), b_ = __fsub_rn(s.box[g][l][2], yy);
    if (!(l_ > 0.f && r_ > 0.f && t_ > 0.f && b_ > 0.f)) continue;
    loc = true;
    if (W == 1) {
      cmask[0] |= 1u << s.cls[g];
    } else {
#pragma unroll
      for (int w = 0; w < W; ++w)
        if (s.cls[g] >> 5 == w) cmask[w] |= 1u << (s.cls[g] & 31);
    }
    const float area = __fmul_rn(__fadd_rn(l_, r_), __fadd_rn(t_, b_));
    if (area < amin) {
      amin = area;
      dl = l_; dr = r_; dt = t_; db = b_;
    } else if (area == amin) {  // tied minimal areas: element-wise maximum (:300-307)
      dl = fmaxf(dl, l_); dr = fmaxf(dr, r_); dt = fmaxf(dt, t_); db = fmaxf(db, b_);
    }
  }
  // centre-ness target (:331-334), 0 where no GT covers the cell
  const float lrmin = fminf(dl, dr), tbmin = fminf(dt, db), lrmax = fmaxf(dl, dr), tbmax = fmaxf(dt, db);
  const float cgt = __fsqrt_rn(__fdiv_rn(__fmul_rn(lrmin, tbmin), __fadd_rn(__fmul_rn(lrmax, tbmax), 1e-12f)));
  return {loc, dl, dr, dt, db, cgt};
}

// NFG = 20: the 25-float rows, class loop fixed at compile time; NFG = 0: num_fg (1..kMaxFg) from the parameters,
// the per-location class mask in kMaskWords words.
template <int NFG>
__global__ void __launch_bounds__(kLossThreads)
    fcos_loss_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp,
                     const float* __restrict__ gt, int G, float* __restrict__ partial,
                     int* __restrict__ level_cnt) {
  constexpr int W = NFG ? (NFG + 31) / 32 : kMaskWords;  // class-mask words
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int nfg = NFG ? NFG : p.num_fg, row = row_floats(nfg);
  const int b = blockIdx.y, blk = blockIdx.x;
  const float* gb = gt + (long long)b * G * 5;
  __shared__ FcosGt s_gt;
  __shared__ float s_red[1][kLossThreads];
  const int cnt = block_gt_count(gb, G);
  fcos_stage_gt(p, gb, cnt, s_gt);
  __syncthreads();
  if (blk == 0 && threadIdx.x < kFcosLevels) {  // GT count per level (a level without GT contributes nothing)
    int c = 0;
    for (int g = 0; g < cnt; ++g) c += (s_gt.lv[g] >> threadIdx.x) & 1;
    level_cnt[b * kFcosLevels + threadIdx.x] = c;
  }
  const float* hb = head + (long long)b * p.N * row;
  float acc[kFcosLevels][4];  // iou, focal, centre, #positive class cells
#pragma unroll
  for (int l = 0; l < kFcosLevels; ++l)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[l][q] = 0.f;
  const int per = (p.N + kLossBlocks - 1) / kLossBlocks;
  const int n_begin = blk * per, n_end = min(p.N, n_begin + per);
  for (int n = n_begin + threadIdx.x; n < n_end; n += blockDim.x) {
    const Cell c = locate(p, n);
    const int l = c.lvl;
    unsigned cmask[W];
    const FcosCell t = fcos_cell(c, cnt, s_gt, cmask);
    const bool loc = t.loc;
    const float dl = t.dl, dr = t.dr, dt = t.dt, db = t.db, cgt = t.cgt;
    const float* r = hb + (long long)n * row;
    // centre-ness BCE with logits, every location (:331-334)
    const float cx = r[nfg];
    float centre = fmaxf(cx, 0.f) - cx * cgt + log1pf(expf(-fabsf(cx)));
    float iou_l = 0.f;
    if (loc) {
      const float pl = expf(r[nfg + 1]), pr = expf(r[nfg + 2]), pt = expf(r[nfg + 3]), pb = expf(r[nfg + 4]);
      const float iw = __fadd_rn(fminf(dl, pl), fminf(dr, pr)), ih = __fadd_rn(fminf(dt, pt), fminf(db, pb));
      const float inter = __fmul_rn(iw, ih);
      const float uni = __fsub_rn(__fadd_rn(__fmul_rn(__fadd_rn(dl, dr), __fadd_rn(dt, db)),
                                            __fmul_rn(__fadd_rn(pl, pr), __fadd_rn(pt, pb))), inter);
      const float iou = __fdiv_rn(inter, __fadd_rn(uni, 1e-12f));
      iou_l = -logf(__fadd_rn(iou, 1e-12f));
    }
    float focal_l = 0.f, npos = 0.f;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const int kend = NFG ? (NFG - 32 * w < 32 ? NFG - 32 * w : 32) : min(32, nfg - 32 * w);
#pragma unroll 4
      for (int k = 0; k < kend; ++k) {
        const float x = r[32 * w + k];
        const float ls = -softplus_f(-x);                 // log sigmoid(x)
        const float sg = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
        if ((cmask[w] >> k) & 1u) {
          const float om = 1.f - sg;
          focal_l += -0.25f * om * om * ls;
          npos += 1.f;
        } else {
          focal_l += -0.25f * sg * sg * (-x + ls);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < kFcosLevels; ++q) {
      if (q == l) {
        acc[q][0] += iou_l;
        acc[q][1] += focal_l;
        acc[q][2] += centre;
        acc[q][3] += npos;
      }
    }
  }
  // the 5 x 4 sums one at a time
  for (int l = 0; l < kFcosLevels; ++l) {
    for (int q = 0; q < 4; ++q) {
      block_sum(s_red, {acc[l][q]});
      if (threadIdx.x == 0) partial[(((long long)b * kLossBlocks + blk) * kFcosLevels + l) * 4 + q] = s_red[0][0];
    }
  }
}

__global__ void fcos_loss_final_kernel(const float* __restrict__ partial, const int* __restrict__ level_cnt,
                                       int B, float* __restrict__ out) {
  pdl_launch_dependents();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float total = 0.f;
  for (int l = 0; l < kFcosLevels; ++l) {
    if (level_cnt[b * kFcosLevels + l] == 0) continue;
    double s3[4] = {0, 0, 0, 0};
    for (int i = 0; i < kLossBlocks; ++i)
      for (int q = 0; q < 4; ++q) s3[q] += (double)partial[(((long long)b * kLossBlocks + i) * kFcosLevels + l) * 4 + q];
    total += (float)((s3[0] + s3[1] + s3[2]) / s3[3]);
  }
  out[b] = total;
}

// ======================== YOLOv3 / YOLOv2 loss forward ======================
// Restates YOLOv3.py:115-318 (+ :37-41 priors, :419-433 anchors, :435-442 GT normalisation), never copied.
// Quirks kept: level k divides the GT by 32 / 16 / 8 while its priors are priors[k] / (8, 16, 32)[k];
// the GT x anchor intersections are products of UNCLAMPED differences; the no-object anchors are built
// from (yx - hw/2, yx + hw/2) re-used as (centre, size).
__device__ __forceinline__ float sig_xent(float z, float x) {  // sigmoid_cross_entropy_with_logits(labels=z, logits=x)
  return fmaxf(x, 0.f) - x * z + log1pf(expf(-fabsf(x)));
}
__device__ __forceinline__ float iou_unclamped(float gy1, float gx1, float gy2, float gx2, float ay1, float ax1,
                                               float ay2, float ax2, float aarea) {
  const float ih = __fsub_rn(fminf(gy2, ay2), fmaxf(gy1, ay1)), iw = __fsub_rn(fminf(gx2, ax2), fmaxf(gx1, ax1));
  const float inter = __fmul_rn(ih, iw);
  const float garea = __fmul_rn(__fsub_rn(gy2, gy1), __fsub_rn(gx2, gx1));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(aarea, garea), inter));
}
// The two YOLO losses share these kernels; a variant fixes what differs between them at compile time:
//   YOLOv3 (YOLOv3.py:115-318): three levels, no-object where the best IoU <= 0.5, the image loss divided by its GT
//     count;
//   YOLOv2 (YOLOv2.py:105-173): the YOLOv3 loss of level 0 alone (GT divided by 32), no-object where the best
//     IoU <= 0.6, the image loss NOT divided by its GT count -- an image without boxes is all no-object terms.
// Every other operation, and its order, is the same in both.
struct Yolo3Loss {
  static constexpr int kLevels = 3;
  static constexpr float kNoobjIou = 0.5f;
  static constexpr bool kPerGt = true;
  static constexpr const char* kHead = "YOLOv3 head with 3 levels and 1..128 classes expected";
};
struct Yolo2Loss {
  static constexpr int kLevels = 1;
  static constexpr float kNoobjIou = 0.6f;
  static constexpr bool kPerGt = false;
  static constexpr const char* kHead = "YOLOv2 head with 1 level and 1..128 classes expected";
};

// GT row g normalised for level k (divided by 32 / 16 / 8): centre, size and corners
struct YoloGt {
  float y, x, h, w, y1, x1, y2, x2;
};
__device__ __forceinline__ YoloGt yolo_gt(const float* gb, int g, int k) {
  const float norm = k == 0 ? 32.f : (k == 1 ? 16.f : 8.f);
  YoloGt n;
  n.y = __fdiv_rn(gb[g * 5], norm);
  n.x = __fdiv_rn(gb[g * 5 + 1], norm);
  n.h = __fdiv_rn(gb[g * 5 + 2], norm);
  n.w = __fdiv_rn(gb[g * 5 + 3], norm);
  n.y1 = __fsub_rn(n.y, __fdiv_rn(n.h, 2.f));
  n.x1 = __fsub_rn(n.x, __fdiv_rn(n.w, 2.f));
  n.y2 = __fadd_rn(n.y, __fdiv_rn(n.h, 2.f));
  n.x2 = __fadd_rn(n.x, __fdiv_rn(n.w, 2.f));
  return n;
}

// Cells (H * W) of the levels before `lvl`: where that level starts in the per-image occupancy array.  Every level
// holds the same number of priors A (yolo_forward checks it), and a cell's A rows are consecutive.
__device__ __forceinline__ int yolo_cell_base(const odt_tail_params& p, int lvl) {
  int c = 0;
  for (int i = 0; i < lvl; ++i) c += p.level[i].H * p.level[i].W;
  return c;
}

// Level / prior assignment of GT row g (YOLOv3.py:160-200): on every level its cell (clamped to the grid) and the
// first maximum of its IoU with the level's priors centred there; the level of the largest of the three (ties go to
// level 2).  YOLOv2 has level 0 only (YOLOv2.py:106-128).  occ_img (or nullptr): the image's cell occupancy, where
// every GT marks its cell on every level.
struct YoloAssign {
  int k, row;  // level, row of (cell, prior) in the image
};
template <class V>
__device__ __forceinline__ YoloAssign yolo_assign(const odt_tail_params& p, const float* gb, int g,
                                                  unsigned char* occ_img) {
  float mx[V::kLevels];
  int arg[V::kLevels], cy[V::kLevels], cx[V::kLevels];
#pragma unroll
  for (int k = 0; k < V::kLevels; ++k) {
    const odt_level& L = p.level[k];
    const YoloGt n = yolo_gt(gb, g, k);
    cy[k] = min(max((int)floorf(n.y), 0), L.H - 1);
    cx[k] = min(max((int)floorf(n.x), 0), L.W - 1);
    if (occ_img) occ_img[yolo_cell_base(p, k) + cy[k] * L.W + cx[k]] = 1;
    const float ay = (float)cy[k] + 0.5f, ax = (float)cx[k] + 0.5f;
    float bv = 0.f;
    int bi = 0;
    for (int a = 0; a < L.A; ++a) {  // the level's priors; the first maximum wins
      const float hh = __fdiv_rn(L.prior_h[a], 2.f), hw = __fdiv_rn(L.prior_w[a], 2.f);
      const float v = iou_unclamped(n.y1, n.x1, n.y2, n.x2, __fsub_rn(ay, hh), __fsub_rn(ax, hw), __fadd_rn(ay, hh),
                                    __fadd_rn(ax, hw), __fmul_rn(L.prior_h[a], L.prior_w[a]));
      if (a == 0 || v > bv) {
        bv = v;
        bi = a;
      }
    }
    mx[k] = bv;
    arg[k] = bi;
  }
  if constexpr (V::kLevels == 1) {
    return {0, p.level[0].offset + (cy[0] * p.level[0].W + cx[0]) * p.level[0].A + arg[0]};
  }
  int k = 2;
  if (mx[0] > mx[1] && mx[0] > mx[2]) k = 0;
  else if (mx[1] > mx[0] && mx[1] > mx[2]) k = 1;
  const odt_level& L = p.level[k];
  // selects, not cy[k]: a register-resident choice instead of a local-memory array
  const int y = k == 0 ? cy[0] : k == 1 ? cy[1] : cy[2], x = k == 0 ? cx[0] : k == 1 ? cx[1] : cx[2];
  const int a = k == 0 ? arg[0] : k == 1 ? arg[1] : arg[2];
  return {k, L.offset + (y * L.W + x) * L.A + a};
}

// (ty, tx, th, tw) targets of GT g at its assignment
__device__ __forceinline__ float4 yolo_targets(const odt_tail_params& p, const float* gb, int g, const YoloAssign& as) {
  const odt_level& L = p.level[as.k];
  const YoloGt n = yolo_gt(gb, g, as.k);
  const int a = (as.row - L.offset) % L.A;
  return make_float4(__fsub_rn(n.y, floorf(n.y)), __fsub_rn(n.x, floorf(n.x)), logf(__fdiv_rn(n.h, L.prior_h[a])),
                     logf(__fdiv_rn(n.w, L.prior_w[a])));
}

// K1: one block per image, one thread per GT: level / prior assignment, positive terms, cell occupancy.
// NFG = 20: the 25-float rows, class loop fixed at compile time; NFG = 0: num_fg from the parameters.
template <class V, int NFG>
__global__ void __launch_bounds__(kMaxGT)
    yolo_loss_pos_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp,
                         const float* __restrict__ gt, int G, unsigned char* __restrict__ occ,
                         float* __restrict__ pos_out) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int nfg = NFG ? NFG : p.num_fg, row = row_floats(nfg);
  const int b = blockIdx.x, g = threadIdx.x;
  const float* gb = gt + (long long)b * G * 5;
  __shared__ float s_red[3][kMaxGT];
  const int cnt = block_gt_count(gb, G);
  const long long cells = yolo_cell_base(p, V::kLevels);
  float coord = 0.f, cls = 0.f, obj = 0.f;
  if (g < cnt) {
    const YoloAssign as = yolo_assign<V>(p, gb, g, occ + (long long)b * cells);
    const float* r = head + ((long long)b * p.N + as.row) * row;
    const float4 tg = yolo_targets(p, gb, g, as);
    const float ty = tg.x, tx = tg.y, th = tg.z, tw = tg.w;
    const float* t = r + nfg;  // y, x, h, w, obj behind the class scores
    coord = sig_xent(ty, t[0]) + sig_xent(tx, t[1]);
    const float dh = __fsub_rn(t[2], th), dw = __fsub_rn(t[3], tw);
    coord += 0.5f * (dh * dh + dw * dw);
    const int label = (int)gb[g * 5 + 4];
    for (int c = 0; c < nfg; ++c) cls += sig_xent(c == label ? 1.f : 0.f, r[c]);
    obj = sig_xent(1.f, t[4]);
  }
  block_sum(s_red, {coord, cls, obj});
  if (threadIdx.x < 3) pos_out[b * 4 + threadIdx.x] = s_red[threadIdx.x][0];
  if (threadIdx.x == 3) pos_out[b * 4 + 3] = (float)cnt;
}

// GT corners of every level for the no-object test, staged in shared memory by the block's threads (the caller
// synchronises)
template <int NL>
__device__ __forceinline__ void yolo_stage_gt(const float* gb, int cnt, float (*s_g)[NL][4]) {
  for (int g = threadIdx.x; g < cnt; g += blockDim.x) {
#pragma unroll
    for (int k = 0; k < NL; ++k) {
      const YoloGt n = yolo_gt(gb, g, k);
      s_g[g][k][0] = n.y1;
      s_g[g][k][1] = n.x1;
      s_g[g][k][2] = n.y2;
      s_g[g][k][3] = n.x2;
    }
  }
}

// The reference's no-object box of (cell, prior) c (:249-262): (yx - hw/2, yx + hw/2) re-used as (centre, size);
// its IoU with GT g of the level
struct YoloNoobjBox {
  float y1, x1, y2, x2, area;
};
__device__ __forceinline__ YoloNoobjBox yolo_noobj_box(const odt_tail_params& p, const Cell& c) {
  const odt_level& L = p.level[c.lvl];
  const float ay = (float)c.y + 0.5f, ax = (float)c.x + 0.5f;
  const float ph = L.prior_h[c.a], pw = L.prior_w[c.a];
  const float cyy = __fsub_rn(ay, __fdiv_rn(ph, 2.f)), cxx = __fsub_rn(ax, __fdiv_rn(pw, 2.f));  // "centre" = y1x1
  const float sh = __fadd_rn(ay, __fdiv_rn(ph, 2.f)), sw = __fadd_rn(ax, __fdiv_rn(pw, 2.f));   // "size"   = y2x2
  YoloNoobjBox o;
  o.y1 = __fsub_rn(cyy, __fdiv_rn(sh, 2.f));
  o.x1 = __fsub_rn(cxx, __fdiv_rn(sw, 2.f));
  o.y2 = __fadd_rn(cyy, __fdiv_rn(sh, 2.f));
  o.x2 = __fadd_rn(cxx, __fdiv_rn(sw, 2.f));
  o.area = __fmul_rn(__fsub_rn(o.y2, o.y1), __fsub_rn(o.x2, o.x1));
  return o;
}
template <int NL>
__device__ __forceinline__ float yolo_noobj_iou(const float (*s_g)[NL][4], int g, int lvl,
                                                const YoloNoobjBox& o) {
  return iou_unclamped(s_g[g][lvl][0], s_g[g][lvl][1], s_g[g][lvl][2], s_g[g][lvl][3], o.y1, o.x1, o.y2, o.x2, o.area);
}

// K2: no-object term over every (cell, prior) whose cell holds no GT centre
template <class V>
__global__ void __launch_bounds__(kLossThreads)
    yolo_loss_noobj_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp,
                           const float* __restrict__ gt, int G, const unsigned char* __restrict__ occ,
                           float* __restrict__ partial) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int b = blockIdx.y, blk = blockIdx.x;
  const float* gb = gt + (long long)b * G * 5;
  __shared__ float s_g[kMaxGT][V::kLevels][4];
  __shared__ float s_red[1][kLossThreads];
  const int cnt = block_gt_count(gb, G);
  yolo_stage_gt(gb, cnt, s_g);
  __syncthreads();
  const long long cells = yolo_cell_base(p, V::kLevels);
  const int row = row_floats(p.num_fg);
  const float* hb = head + (long long)b * p.N * row;
  float acc = 0.f;
  const int per = (p.N + kLossBlocks - 1) / kLossBlocks;
  const int n_begin = blk * per, n_end = min(p.N, n_begin + per);
  for (int n = n_begin + threadIdx.x; n < n_end; n += blockDim.x) {
    const Cell c = locate(p, n);
    const odt_level& L = p.level[c.lvl];
    if (occ[(long long)b * cells + yolo_cell_base(p, c.lvl) + c.y * L.W + c.x]) continue;
    const YoloNoobjBox o = yolo_noobj_box(p, c);
    float best = -3.0e38f;
    for (int g = 0; g < cnt; ++g) best = fmaxf(best, yolo_noobj_iou(s_g, g, c.lvl, o));
    if (best <= V::kNoobjIou) acc += sig_xent(0.f, hb[(long long)n * row + p.num_fg + 4]);  // objectness
  }
  block_sum(s_red, {acc});
  if (threadIdx.x == 0) partial[(long long)b * kLossBlocks + blk] = s_red[0][0];
}

template <class V>
__global__ void yolo_loss_final_kernel(const float* __restrict__ pos, const float* __restrict__ partial, int B,
                                       float cs, float ns, float os, float ks, float* __restrict__ out) {
  pdl_launch_dependents();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double noobj = 0.0;
  for (int i = 0; i < kLossBlocks; ++i) noobj += (double)partial[(long long)b * kLossBlocks + i];
  if constexpr (V::kPerGt) {
    const float ng = pos[b * 4 + 3];
    out[b] = (cs * pos[b * 4 + 0] + ks * pos[b * 4 + 1] + os * pos[b * 4 + 2]) / ng + ns * (float)noobj / ng;
  } else {
    out[b] = cs * pos[b * 4 + 0] + ks * pos[b * 4 + 1] + os * pos[b * 4 + 2] + ns * (float)noobj;
  }
}

// ============================ loss gradients ================================
// d loss_out[b] / d head[b] of the four families, written to every element of grad [B, N, row].  They restate the
// gradient of the training step's autograd loss (odt_b200/train.py, `image_loss`) and read the matching the forward
// kernels left in scratch.  One warp per candidate row, the lanes over its columns in chunks of 32: the writes of a
// row are contiguous, and a row with no gradient is written as exact zeros.  Contributions of several GTs to one
// row (shared best anchor, shared YOLO cell and prior) are summed in GT order by the row's own lanes: no atomics, so
// the gradient is bit-identical from run to run and does not depend on the batch.
constexpr int kGradWarps = kLossThreads / 32;
constexpr int kGradBlocks = 128;  // row blocks per image (grid-stride beyond)

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// butterfly sum: every lane ends with the same bits (each step adds the same two partials in either order)
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float smooth_l1_grad(float d) { return fabsf(d) < 1.f ? d : copysignf(1.f, d); }

// RetinaNet / SSD: lane c < 21 holds logit c, lanes 21..24 the box deltas.  Per row: positives (a best anchor once
// per GT that chose it, or the GT of an IoU > 0.5 match) get the classification gradient for their GT's class and
// the smooth-L1 gradient toward its box, both / #positives; RetinaNet negatives get the focal gradient for the
// background / #positives; SSD's mined negatives get the cross-entropy gradient for the background / #mined;
// ignored anchors and SSD's unmined negatives get zeros.  RetinaNet's focal term differentiates
// -alpha (1 - q)^gamma log q at q = clamp(softmax[label], 1e-8, 1), zero outside the closed interval.
template <bool kSsd>
__global__ void __launch_bounds__(kLossThreads)
    loss_anchor_grad_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp,
                            const float* __restrict__ gt, int G, const int* __restrict__ best,
                            const int* __restrict__ assign, const float* __restrict__ partial,
                            const int* __restrict__ nsel, float alpha, float gamma, float* __restrict__ grad) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const float* gb = gt + (long long)b * G * 5;
  __shared__ int s_best[kMaxGT];
  __shared__ float s_inv[2];  // 1 / #positives, 1 / #mined negatives
  const int cnt = block_gt_count(gb, G);
  for (int g = threadIdx.x; g < cnt; g += blockDim.x) s_best[g] = best[b * G + g];
  if (threadIdx.x == 0) {
    s_inv[0] = __fdiv_rn(1.f, image_sums(partial, b).npos);
    s_inv[1] = kSsd ? __fdiv_rn(1.f, (float)nsel[b]) : s_inv[0];
  }
  __syncthreads();
  const float inv_pos = s_inv[0], inv_neg = s_inv[1];
  const int neg_kind = kSsd ? kAsMined : kAsNegative;  // the negatives that carry a gradient
  for (int n = blockIdx.x * kGradWarps + (threadIdx.x >> 5); n < p.N; n += gridDim.x * kGradWarps) {
    const long long at = ((long long)b * p.N + n) * 25;
    const int as = assign[(long long)b * p.N + n];
    float gv = 0.f;
    if (as >= 0 || as == kAsBest || as == neg_kind) {  // warp-uniform
      const float x = lane < 25 ? head[at + lane] : 0.f;
      const float m = warp_max(lane < 21 ? x : -INFINITY);
      const float e = lane < 21 ? expf(__fsub_rn(x, m)) : 0.f;
      const float pr = __fdiv_rn(e, warp_sum(e));
      auto cls = [&](int label, float scale) {
        const float hot = lane == label ? 1.f : 0.f;
        if constexpr (kSsd) {
          if (lane < 21) gv += (pr - hot) * scale;
        } else {
          const float pl = __shfl_sync(0xffffffffu, pr, label);
          if (pl >= 1e-8f && pl <= 1.f) {
            const float om = 1.f - pl;
            const float dpow = gamma == 0.f ? 0.f : gamma * powf(om, gamma - 1.f);
            const float dq = -alpha * (__fdiv_rn(powf(om, gamma), pl) - dpow * logf(pl));
            if (lane < 21) gv += dq * pl * (hot - pr) * scale;
          }
        }
      };
      auto box = [&](int g) {
        if (lane >= 21 && lane < 25) {
          const Anchor a = anchor_ssd(p, locate(p, n));
          const float* q = gb + g * 5;
          float t;
          if (lane == 21) t = __fdiv_rn(__fsub_rn(q[0], a.cy), a.h);
          else if (lane == 22) t = __fdiv_rn(__fsub_rn(q[1], a.cx), a.w);
          else if (lane == 23) t = logf(__fdiv_rn(q[2], a.h));
          else t = logf(__fdiv_rn(q[3], a.w));
          gv += smooth_l1_grad(__fsub_rn(x, t)) * inv_pos;
        }
      };
      if (as == kAsBest) {
        for (int g = 0; g < cnt; ++g) {
          if (s_best[g] != n) continue;
          cls((int)gb[g * 5 + 4], inv_pos);
          box(g);
        }
      } else if (as >= 0) {
        cls((int)gb[as * 5 + 4], inv_pos);
        box(as);
      } else {
        cls(20, inv_neg);
      }
    }
    if (lane < 25) grad[at + lane] = gv;
  }
}

// FCOS, per location of a level with GT (others: zeros), everything / the level's #positive class cells: the sigmoid
// focal gradient on every class column, the centre-ness BCE gradient sigmoid(x) - target, and at locations inside a
// GT the gradient of -log(IoU + 1e-12) through exp() of the four distances.
__device__ __forceinline__ float fcos_focal_grad(float x, bool positive) {
  const float s = sigmoid_rn(x), om = 1.f - s;
  const float ls = -softplus_f(-x);  // log sigmoid(x)
  if (positive) return -0.25f * om * om * (om - 2.f * s * ls);
  return -0.25f * s * s * (2.f * om * (ls - x) - s);
}

template <int NFG>
__global__ void __launch_bounds__(kLossThreads)
    fcos_loss_grad_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp,
                          const float* __restrict__ gt, int G, const float* __restrict__ partial,
                          const int* __restrict__ level_cnt, float* __restrict__ grad) {
  constexpr int W = NFG ? (NFG + 31) / 32 : kMaskWords;
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int nfg = NFG ? NFG : p.num_fg, row = row_floats(nfg);
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const float* gb = gt + (long long)b * G * 5;
  __shared__ FcosGt s_gt;
  __shared__ float s_inv[kFcosLevels];  // 1 / #positive class cells; 0 for a level without GT
  const int cnt = block_gt_count(gb, G);
  fcos_stage_gt(p, gb, cnt, s_gt);
  if (threadIdx.x < kFcosLevels) {
    const int l = threadIdx.x;
    double npos = 0.0;  // the final kernel's sum
    for (int i = 0; i < kLossBlocks; ++i) npos += (double)partial[(((long long)b * kLossBlocks + i) * kFcosLevels + l) * 4 + 3];
    s_inv[l] = level_cnt[b * kFcosLevels + l] ? __fdiv_rn(1.f, (float)npos) : 0.f;
  }
  __syncthreads();
  for (int n = blockIdx.x * kGradWarps + (threadIdx.x >> 5); n < p.N; n += gridDim.x * kGradWarps) {
    const Cell c = locate(p, n);
    float* go = grad + ((long long)b * p.N + n) * row;
    const float* r = head + ((long long)b * p.N + n) * row;
    if (!level_cnt[b * kFcosLevels + c.lvl]) {  // warp-uniform
      for (int k = lane; k < row; k += 32) go[k] = 0.f;
      continue;
    }
    const float inv = s_inv[c.lvl];
    unsigned cmask[W];
    const FcosCell t = fcos_cell(c, cnt, s_gt, cmask);
    // lanes 0..3: the gradient of distance column nfg + 1 + lane.  The IoU term is -log(IoU + 1e-12) * loc on every
    // location (FCOS.py:319-320): outside every GT it is 0 * the same product, +0 for a finite product and NaN where
    // an exp() overflowed, as in the reference graph.
    float gbox;
    {
      const float pl = expf(r[nfg + 1]), pr = expf(r[nfg + 2]), pt = expf(r[nfg + 3]), pb = expf(r[nfg + 4]);
      const float iw = __fadd_rn(fminf(t.dl, pl), fminf(t.dr, pr)), ih = __fadd_rn(fminf(t.dt, pt), fminf(t.db, pb));
      const float inter = __fmul_rn(iw, ih);
      const float u = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(__fadd_rn(t.dl, t.dr), __fadd_rn(t.dt, t.db)),
                                                    __fmul_rn(__fadd_rn(pl, pr), __fadd_rn(pt, pb))), inter), 1e-12f);
      const float iou = __fdiv_rn(inter, u);
      const float dl_diou = __fdiv_rn(-1.f, __fadd_rn(iou, 1e-12f));
      // lane k: distance k of (l, r, t, b); d inter / d p_k is the other side's extent where p_k is the minimum
      const float pk = lane == 0 ? pl : lane == 1 ? pr : lane == 2 ? pt : pb;
      const float dk = lane == 0 ? t.dl : lane == 1 ? t.dr : lane == 2 ? t.dt : t.db;
      const float other = lane < 2 ? ih : iw;                                   // extent across
      const float psum = lane < 2 ? __fadd_rn(pt, pb) : __fadd_rn(pl, pr);      // d (pl+pr)(pt+pb) / d p_k
      const float dinter = pk < dk ? other : 0.f;
      const float diou = __fdiv_rn(dinter - iou * (psum - dinter), u);
      const float g = dl_diou * diou * pk * inv;
      gbox = t.loc ? g : __fadd_rn(__fmul_rn(g, 0.f), 0.f);
    }
    for (int k0 = 0; k0 < row; k0 += 32) {
      const int k = k0 + lane;
      const float gb4 = __shfl_sync(0xffffffffu, gbox, (k - nfg - 1) & 31);
      if (k >= row) continue;
      const float x = r[k];
      float gv;
      if (k < nfg) {
        unsigned word = 0u;
#pragma unroll
        for (int w = 0; w < W; ++w)
          if (w == (k >> 5)) word = cmask[w];
        gv = fcos_focal_grad(x, (word >> (k & 31)) & 1u) * inv;
      } else if (k == nfg) {
        gv = (sigmoid_rn(x) - t.cgt) * inv;
      } else {
        gv = gb4;
      }
      go[k] = gv;
    }
  }
}

// YOLOv3, all / #GT (YOLOv2: not divided): the objectness column of a no-object row (a cell without GT, best IoU
// <= the variant's threshold, as the forward decides it) gets noobj_scale * sigmoid(x); an assigned row gets, once
// per GT assigned to it, class_scale * (sigmoid - one-hot) on the classes, coord_scale * (sigmoid - target) on y, x,
// coord_scale * (x - target) on h, w (the 0.5 of the squared term cancels), obj_scale * (sigmoid - 1) on the
// objectness; every other element is zero.  The block re-derives its image's assignments with the forward's
// yolo_assign and reads the forward's occupancy.
template <class V, int NFG>
__global__ void __launch_bounds__(kLossThreads, 4)
    yolo_loss_grad_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp,
                          const float* __restrict__ gt, int G, const unsigned char* __restrict__ occ, float cs,
                          float ns, float os, float ks, float* __restrict__ grad) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int nfg = NFG ? NFG : p.num_fg, row = row_floats(nfg);
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const float* gb = gt + (long long)b * G * 5;
  __shared__ float s_g[kMaxGT][V::kLevels][4];
  __shared__ int s_row[kMaxGT], s_lab[kMaxGT];
  __shared__ float4 s_t[kMaxGT];
  const int cnt = block_gt_count(gb, G);
  yolo_stage_gt(gb, cnt, s_g);
  for (int g = threadIdx.x; g < cnt; g += blockDim.x) {
    const YoloAssign as = yolo_assign<V>(p, gb, g, nullptr);
    s_row[g] = as.row;
    s_t[g] = yolo_targets(p, gb, g, as);
    s_lab[g] = (int)gb[g * 5 + 4];
  }
  __syncthreads();
  const long long cells = yolo_cell_base(p, V::kLevels);
  const float inv = V::kPerGt ? __fdiv_rn(1.f, (float)cnt) : 1.f;
  for (int n = blockIdx.x * kGradWarps + (threadIdx.x >> 5); n < p.N; n += gridDim.x * kGradWarps) {
    const Cell c = locate(p, n);
    const odt_level& L = p.level[c.lvl];
    const bool occupied = occ[(long long)b * cells + yolo_cell_base(p, c.lvl) + c.y * L.W + c.x];
    bool noobj = false;
    if (!occupied) {  // the forward's best IoU, the GTs split over the lanes (a maximum: any order, same value)
      const YoloNoobjBox o = yolo_noobj_box(p, c);
      float best = -3.0e38f;
      for (int g = lane; g < cnt; g += 32) best = fmaxf(best, yolo_noobj_iou(s_g, g, c.lvl, o));
      noobj = warp_max(best) <= V::kNoobjIou;
    }
    float* go = grad + ((long long)b * p.N + n) * row;
    const float* r = head + ((long long)b * p.N + n) * row;
    for (int k = lane; k < row; k += 32) {
      float gv = 0.f;
      if (noobj) {
        if (k == nfg + 4) gv = ns * sigmoid_rn(r[k]) * inv;
      } else if (occupied) {
        const float x = r[k], s = sigmoid_rn(x);
        for (int g = 0; g < cnt; ++g) {
          if (s_row[g] != n) continue;
          const float4 t = s_t[g];
          if (k < nfg) gv += ks * (s - (k == s_lab[g] ? 1.f : 0.f)) * inv;
          else if (k == nfg) gv += cs * (s - t.x) * inv;
          else if (k == nfg + 1) gv += cs * (s - t.y) * inv;
          else if (k == nfg + 2) gv += cs * (x - t.z) * inv;
          else if (k == nfg + 3) gv += cs * (x - t.w) * inv;
          else gv += os * (s - 1.f) * inv;
        }
      }
      go[k] = gv;
    }
  }
}

// ============================ scratch layouts ===============================
// Every loss call gets one caller-allocated scratch buffer, 8-byte aligned, carved into arrays that each start
// on an 8-byte boundary.  A family's layout function is the only place its arrays are placed: the size query
// carves from address 0 and returns the total, the launcher carves the caller's buffer.  (The layouts take()
// inside braced lists, which C++ evaluates left to right.)
struct Carve {
  uintptr_t base;
  long long bytes;
  template <class T>
  T* take(long long n) {
    T* at = reinterpret_cast<T*>(base + bytes);
    bytes += (n * (long long)sizeof(T) + 7) & ~7ll;
    return at;
  }
};

struct RetinaScratch {
  float* partial;  // (conf, coord, npos, -) per (image, anchor block)
  int* best;       // arg-max anchor per (image, GT)
  int* assign;     // per (image, anchor): kAs* or the matched GT
  long long bytes;
};
static RetinaScratch retina_scratch(const odt_tail_params& p, int B, void* base) {
  Carve c{(uintptr_t)base, 0};
  return {c.take<float>((long long)B * kLossBlocks * 4), c.take<int>((long long)B * kMaxGT),
          c.take<int>((long long)B * p.N), c.bytes};
}

struct SsdScratch {
  float* partial;                // as RetinaScratch
  int* best;
  int* neg_count;                // negatives per image
  unsigned long long* neg_keys;  // (background loss, row) per negative, [B][N]
  int* assign;                   // as RetinaScratch, the mined negatives kAsMined
  int* nsel;                     // mined negatives per image
  long long bytes;
};
static SsdScratch ssd_scratch(const odt_tail_params& p, int B, void* base) {
  Carve c{(uintptr_t)base, 0};
  return {c.take<float>((long long)B * kLossBlocks * 4), c.take<int>((long long)B * kMaxGT), c.take<int>(B),
          c.take<unsigned long long>((long long)B * p.N), c.take<int>((long long)B * p.N), c.take<int>(B), c.bytes};
}

struct FcosScratch {
  float* partial;  // (iou, focal, centre, #positive class cells) per (image, anchor block, level)
  int* level_cnt;  // GT per (image, level)
  long long bytes;
};
static FcosScratch fcos_scratch(const odt_tail_params&, int B, void* base) {
  Carve c{(uintptr_t)base, 0};
  return {c.take<float>((long long)B * kLossBlocks * kFcosLevels * 4), c.take<int>((long long)B * kFcosLevels),
          c.bytes};
}

struct YoloScratch {
  float* pos;          // (coord, class, obj, #GT) per image
  float* partial;      // no-object sum per (image, anchor block)
  unsigned char* occ;  // 1 for a cell that holds a GT, [B][sum of H * W over the levels]
  long long bytes;
};
template <class V>
static long long yolo_cells(const odt_tail_params& p) {
  long long c = 0;
  for (int i = 0; i < V::kLevels; ++i) c += (long long)p.level[i].H * p.level[i].W;
  return c;
}
template <class V>
static YoloScratch yolo_scratch(const odt_tail_params& p, int B, void* base) {
  Carve c{(uintptr_t)base, 0};
  return {c.take<float>((long long)B * 4), c.take<float>((long long)B * kLossBlocks),
          c.take<unsigned char>((long long)B * yolo_cells<V>(p)), c.bytes};
}

template <class Layout>
static long long scratch_bytes(const odt_tail_params* p, int B, Layout layout) {
  return p && B > 0 && p->N > 0 ? layout(*p, B, nullptr).bytes : -1;
}

// ============================ launchers =====================================
// One launcher per family runs the forward kernels for both entry points, `_fwd` and `_grad`: the checks (all before
// any CUDA call), the scratch carve and the launches; the gradient entry points then launch their kernel on the
// matching the forward left in scratch.
static dim3 grad_grid(int B) { return dim3(kGradBlocks, B); }

static int retina_forward(const float* head, const odt_tail_params* p, int B, const float* gt, int G, float alpha,
                          float gamma, void* scratch, float* loss_out, cudaStream_t st, RetinaScratch& s) {
  ODT_CHECK_ARG(head && p && gt && scratch && loss_out, "null pointer");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_SSD && p->num_fg == 20, "softmax-family head with 20 classes expected");
  ODT_CHECK_ARG(B > 0 && G > 0 && G <= kMaxGT, "B/G (G <= 128)");
  ODT_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  s = retina_scratch(*p, B, scratch);
  TailP tp;
  tp.p = *p;
  loss_best_anchor_kernel<<<dim3(G, B), kLossThreads, 0, st>>>(tp, gt, G, s.best);
  ODT_LAUNCH_OK();
  loss_anchor_kernel<false><<<dim3(kLossBlocks, B), kLossThreads, 0, st>>>(head, tp, gt, G, s.best, alpha, gamma,
                                                                          s.partial, nullptr, nullptr, s.assign);
  ODT_LAUNCH_OK();
  loss_final_kernel<<<(B + 63) / 64, 64, 0, st>>>(s.partial, B, loss_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

static int ssd_forward(const float* head, const odt_tail_params* p, int B, const float* gt, int G, void* scratch,
                       float* loss_out, int* info_out, cudaStream_t st, SsdScratch& s) {
  ODT_CHECK_ARG(head && p && gt && scratch && loss_out, "null pointer");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_SSD && p->num_fg == 20, "softmax-family head with 20 classes expected");
  ODT_CHECK_ARG(B > 0 && G > 0 && G <= kMaxGT, "B/G (G <= 128)");
  ODT_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  s = ssd_scratch(*p, B, scratch);
  ODT_CUDA_OK(cudaMemsetAsync(s.neg_count, 0, sizeof(int) * (size_t)B, st));
  TailP tp;
  tp.p = *p;
  loss_best_anchor_kernel<<<dim3(G, B), kLossThreads, 0, st>>>(tp, gt, G, s.best);
  ODT_LAUNCH_OK();
  loss_anchor_kernel<true><<<dim3(kLossBlocks, B), kLossThreads, 0, st>>>(head, tp, gt, G, s.best, 0.f, 0.f,
                                                                         s.partial, s.neg_keys, s.neg_count, s.assign);
  ODT_LAUNCH_OK();
  ssd_loss_mine_kernel<<<B, kLossThreads, 0, st>>>(tp, s.partial, s.neg_keys, s.neg_count, loss_out, info_out,
                                                   s.assign, s.nsel);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

static int fcos_forward(const float* head, const odt_tail_params* p, int B, const float* gt, int G, void* scratch,
                        float* loss_out, cudaStream_t st, FcosScratch& s) {
  ODT_CHECK_ARG(head && p && gt && scratch && loss_out, "null pointer");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_FCOS && p->num_levels == kFcosLevels && p->num_fg >= 1 && p->num_fg <= kMaxFg,
                "FCOS head with 5 levels and 1..128 classes expected");
  ODT_CHECK_ARG(B > 0 && G > 0 && G <= kMaxGT, "B/G (G <= 128)");
  ODT_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  s = fcos_scratch(*p, B, scratch);
  TailP tp;
  tp.p = *p;
  if (p->num_fg == 20)
    fcos_loss_kernel<20><<<dim3(kLossBlocks, B), kLossThreads, 0, st>>>(head, tp, gt, G, s.partial, s.level_cnt);
  else
    fcos_loss_kernel<0><<<dim3(kLossBlocks, B), kLossThreads, 0, st>>>(head, tp, gt, G, s.partial, s.level_cnt);
  ODT_LAUNCH_OK();
  fcos_loss_final_kernel<<<(B + 63) / 64, 64, 0, st>>>(s.partial, s.level_cnt, B, loss_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

template <class V>
static int yolo_forward(const float* head, const odt_tail_params* p, int B, const float* gt, int G, float coord_scale,
                        float noobj_scale, float obj_scale, float class_scale, void* scratch, float* loss_out,
                        cudaStream_t st, YoloScratch& s) {
  ODT_CHECK_ARG(head && p && gt && scratch && loss_out, "null pointer");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_YOLO3 && p->num_levels == V::kLevels && p->num_fg >= 1 && p->num_fg <= kMaxFg,
                V::kHead);
  // One prior count on every level (the config's num_priors), and rows laid out level after level, cell after cell:
  // the kernels find a level's rows at its offset and its cells in the occupancy array by these sums.
  const int A = p->level[0].A;
  ODT_CHECK_ARG(A >= 1 && A <= ODT_MAX_PRIORS, "1..9 priors per level expected");
  long long rows = 0;
  for (int i = 0; i < V::kLevels; ++i) {
    const odt_level& L = p->level[i];
    ODT_CHECK_ARG(L.A == A, "the same number of priors on every level expected");
    ODT_CHECK_ARG(L.H >= 1 && L.W >= 1 && L.offset == rows, "level geometry: H, W >= 1, offset = rows before it");
    rows += (long long)L.H * L.W * A;
  }
  ODT_CHECK_ARG(rows == p->N, "N must be the sum of H * W * A over the levels");
  ODT_CHECK_ARG(B > 0 && G > 0 && G <= kMaxGT, "B/G (G <= 128)");
  ODT_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  s = yolo_scratch<V>(*p, B, scratch);
  ODT_CUDA_OK(cudaMemsetAsync(s.occ, 0, (size_t)B * yolo_cells<V>(*p), st));
  TailP tp;
  tp.p = *p;
  if (p->num_fg == 20)
    yolo_loss_pos_kernel<V, 20><<<B, kMaxGT, 0, st>>>(head, tp, gt, G, s.occ, s.pos);
  else
    yolo_loss_pos_kernel<V, 0><<<B, kMaxGT, 0, st>>>(head, tp, gt, G, s.occ, s.pos);
  ODT_LAUNCH_OK();
  yolo_loss_noobj_kernel<V><<<dim3(kLossBlocks, B), kLossThreads, 0, st>>>(head, tp, gt, G, s.occ, s.partial);
  ODT_LAUNCH_OK();
  yolo_loss_final_kernel<V><<<(B + 63) / 64, 64, 0, st>>>(s.pos, s.partial, B, coord_scale, noobj_scale, obj_scale,
                                                          class_scale, loss_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

// forward, then the gradient kernel on the matching the forward left in scratch
template <class V>
static int yolo_forward_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G, float cs,
                             float ns, float os, float ks, void* scratch, float* loss_out, float* grad_out,
                             cudaStream_t st) {
  ODT_CHECK_ARG(grad_out, "null pointer");
  YoloScratch s;
  const int rc = yolo_forward<V>(head, p, B, gt, G, cs, ns, os, ks, scratch, loss_out, st, s);
  if (rc != ODT_OK) return rc;
  TailP tp;
  tp.p = *p;
  if (p->num_fg == 20)
    yolo_loss_grad_kernel<V, 20><<<grad_grid(B), kLossThreads, 0, st>>>(head, tp, gt, G, s.occ, cs, ns, os, ks,
                                                                        grad_out);
  else
    yolo_loss_grad_kernel<V, 0><<<grad_grid(B), kLossThreads, 0, st>>>(head, tp, gt, G, s.occ, cs, ns, os, ks,
                                                                       grad_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

}  // namespace odt

using namespace odt;

extern "C" long long odt_retina_loss_scratch_bytes(const odt_tail_params* p, int B) {
  return scratch_bytes(p, B, retina_scratch);
}
extern "C" long long odt_ssd_loss_scratch_bytes(const odt_tail_params* p, int B) {
  return scratch_bytes(p, B, ssd_scratch);
}
extern "C" long long odt_fcos_loss_scratch_bytes(const odt_tail_params* p, int B) {
  return scratch_bytes(p, B, fcos_scratch);
}
extern "C" long long odt_yolo_loss_scratch_bytes(const odt_tail_params* p, int B) {
  return scratch_bytes(p, B, yolo_scratch<Yolo3Loss>);
}
extern "C" long long odt_yolo2_loss_scratch_bytes(const odt_tail_params* p, int B) {
  return scratch_bytes(p, B, yolo_scratch<Yolo2Loss>);
}

extern "C" int odt_retina_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                   float alpha, float gamma, void* scratch, float* loss_out, void* stream) {
  RetinaScratch s;
  return retina_forward(head, p, B, gt, G, alpha, gamma, scratch, loss_out, (cudaStream_t)stream, s);
}

extern "C" int odt_ssd_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                void* scratch, float* loss_out, int* info_out, void* stream) {
  SsdScratch s;
  return ssd_forward(head, p, B, gt, G, scratch, loss_out, info_out, (cudaStream_t)stream, s);
}

extern "C" int odt_fcos_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                 void* scratch, float* loss_out, void* stream) {
  FcosScratch s;
  return fcos_forward(head, p, B, gt, G, scratch, loss_out, (cudaStream_t)stream, s);
}

extern "C" int odt_yolo_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                 float coord_scale, float noobj_scale, float obj_scale, float class_scale,
                                 void* scratch, float* loss_out, void* stream) {
  YoloScratch s;
  return yolo_forward<Yolo3Loss>(head, p, B, gt, G, coord_scale, noobj_scale, obj_scale, class_scale, scratch,
                                 loss_out, (cudaStream_t)stream, s);
}

extern "C" int odt_yolo2_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                  float coord_scale, float noobj_scale, float obj_scale, float class_scale,
                                  void* scratch, float* loss_out, void* stream) {
  YoloScratch s;
  return yolo_forward<Yolo2Loss>(head, p, B, gt, G, coord_scale, noobj_scale, obj_scale, class_scale, scratch,
                                 loss_out, (cudaStream_t)stream, s);
}

extern "C" int odt_retina_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                    float alpha, float gamma, void* scratch, float* loss_out, float* grad_out,
                                    void* stream) {
  ODT_CHECK_ARG(grad_out, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  RetinaScratch s;
  const int rc = retina_forward(head, p, B, gt, G, alpha, gamma, scratch, loss_out, st, s);
  if (rc != ODT_OK) return rc;
  TailP tp;
  tp.p = *p;
  loss_anchor_grad_kernel<false><<<grad_grid(B), kLossThreads, 0, st>>>(head, tp, gt, G, s.best, s.assign, s.partial,
                                                                        nullptr, alpha, gamma, grad_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_ssd_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                 void* scratch, float* loss_out, int* info_out, float* grad_out, void* stream) {
  ODT_CHECK_ARG(grad_out, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  SsdScratch s;
  const int rc = ssd_forward(head, p, B, gt, G, scratch, loss_out, info_out, st, s);
  if (rc != ODT_OK) return rc;
  TailP tp;
  tp.p = *p;
  loss_anchor_grad_kernel<true><<<grad_grid(B), kLossThreads, 0, st>>>(head, tp, gt, G, s.best, s.assign, s.partial,
                                                                       s.nsel, 0.f, 0.f, grad_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_fcos_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                  void* scratch, float* loss_out, float* grad_out, void* stream) {
  ODT_CHECK_ARG(grad_out, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  FcosScratch s;
  const int rc = fcos_forward(head, p, B, gt, G, scratch, loss_out, st, s);
  if (rc != ODT_OK) return rc;
  TailP tp;
  tp.p = *p;
  if (p->num_fg == 20)
    fcos_loss_grad_kernel<20><<<grad_grid(B), kLossThreads, 0, st>>>(head, tp, gt, G, s.partial, s.level_cnt,
                                                                     grad_out);
  else
    fcos_loss_grad_kernel<0><<<grad_grid(B), kLossThreads, 0, st>>>(head, tp, gt, G, s.partial, s.level_cnt,
                                                                    grad_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_yolo_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                  float coord_scale, float noobj_scale, float obj_scale, float class_scale,
                                  void* scratch, float* loss_out, float* grad_out, void* stream) {
  return yolo_forward_grad<Yolo3Loss>(head, p, B, gt, G, coord_scale, noobj_scale, obj_scale, class_scale, scratch,
                                      loss_out, grad_out, (cudaStream_t)stream);
}

extern "C" int odt_yolo2_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                   float coord_scale, float noobj_scale, float obj_scale, float class_scale,
                                   void* scratch, float* loss_out, float* grad_out, void* stream) {
  return yolo_forward_grad<Yolo2Loss>(head, p, B, gt, G, coord_scale, noobj_scale, obj_scale, class_scale, scratch,
                                      loss_out, grad_out, (cudaStream_t)stream);
}

// ============================ PFPNet-R loss =================================
// Restates _compute_one_image_loss of PFPNetR.py:469-610 (never copied) on the two-step rows
// [ODM logits(21), ODM t(4), ARM logits(2), ARM t(4)]:
//   * matching: each GT's arg-max anchor (loss_best_anchor_kernel, first maximum, duplicates kept); among the other
//     anchors best IoU > 0.5 is a positive of its arg-max GT, < 0.4 a negative (RetinaNet's band);
//   * ARM: positives cross-entropy to label 0 and smooth-L1 against the anchor targets; hard negatives: exact greedy
//     NMS over the negative anchor boxes scored by their ARM cross-entropy to label 1, min(#neg, 3 #pos) of them at
//     IoU 0.7 (the SSD mining), their mean;
//   * ODM: the mined negatives whose RAW ARM logit of class 1 is < 0.99 (:584), cross-entropy to label 20; positives
//     cross-entropy to their GT class and smooth-L1 against targets built from the decoded ARM box (:598-605), so
//     the ODM box term also depends on the ARM deltas, and its gradient reaches them.
//   * every mean over zero elements is 0: tf.losses' Reduction.MEAN divides with div_no_nan (_safe_mean, TF 1.13)
//     [TF-sem], and the kernel applies the same rule where the reference's tf.reduce_mean would give NaN (no mined
//     negative, no positive): an image without boxes has loss 0 and gradient 0.
// One CTA per image; sums in a fixed order (per-thread anchor order, then block_sum), so the loss is run-to-run
// deterministic.  The gradient kernel writes d(image loss)/d(row) for every column of every row.
namespace odt {

constexpr int kPfpOdmT = 21, kPfpArmC = 25, kPfpArmT = 27;

__device__ __forceinline__ float xent2(float a0, float a1, int label) {
  const float m = fmaxf(a0, a1);
  const float s = __fadd_rn(expf(__fsub_rn(a0, m)), expf(__fsub_rn(a1, m)));
  return __fsub_rn(logf(s), __fsub_rn(label ? a1 : a0, m));
}

template <bool kGrad>
__global__ void __launch_bounds__(kLossThreads)
    pfpnet_loss_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp, const float* __restrict__ gt,
                       int G, const int* __restrict__ best, unsigned long long* __restrict__ neg_keys,
                       int* __restrict__ assign_all, float* __restrict__ loss_out, float* __restrict__ grad) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  constexpr int row = kind_row_floats(ODT_DECODE_TWO_STEP, 20);
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = p.N;
  const float* hb = head + (long long)b * N * row;
  const float* gb = gt + (long long)b * G * 5;
  unsigned long long* keys = neg_keys + (long long)b * N;
  int* assign = assign_all + (long long)b * N;
  __shared__ int s_best[kMaxGT];
  __shared__ int s_npos, s_nneg, s_nsel, s_nodm;
  __shared__ unsigned long long s_wkey[kLossThreads / 32];
  __shared__ int s_wpos[kLossThreads / 32];
  __shared__ float s_sum[6][kLossThreads];
  const int cnt = block_gt_count(gb, G);
  for (int g = tid; g < cnt; g += blockDim.x) s_best[g] = best[b * G + g];
  if (tid == 0) {
    s_npos = 0;
    s_nneg = 0;
  }
  __syncthreads();
  // (1) assignment of every anchor; negatives become (ARM cross-entropy, row) mining keys
  for (int n = tid; n < N; n += blockDim.x) {
    bool is_best = false;
    for (int g = 0; g < cnt; ++g) is_best |= s_best[g] == n;
    int as = kAsBest;
    if (!is_best) {
      const Anchor a = anchor_ssd(p, locate(p, n));
      float bv = -INFINITY;  // reduce_max over no GT: every anchor is a negative
      int bg = 0;
      for (int g = 0; g < cnt; ++g) {
        const GtBox gx = gt_box(gb, g);
        const float v = iou_match(a, gx.y1, gx.x1, gx.y2, gx.x2, gx.area);
        if (v > bv) {
          bv = v;
          bg = g;
        }
      }
      if (bv > 0.5f) {
        as = bg;
        atomicAdd(&s_npos, 1);
      } else if (bv < 0.4f) {
        as = kAsNegative;
        const float* r = hb + (long long)n * row;
        const float ce = xent2(r[kPfpArmC], r[kPfpArmC + 1], 1);
        keys[atomicAdd(&s_nneg, 1)] = ((unsigned long long)__float_as_uint(ce) << 32) | (0xFFFFFFFFu - (unsigned)n);
      } else {
        as = kAsIgnored;
      }
    }
    assign[n] = as;
  }
  __syncthreads();
  // (2) hard-negative mining, as ssd_loss_mine_kernel: greedy NMS by repeated arg-max of the keys
  const int P = cnt + s_npos, nneg = s_nneg;
  const int chosen = nneg > 3 * P ? 3 * P : nneg;
  int nsel = 0, nodm = 0;  // thread 0's count of mined rows that pass the ODM test
  while (nsel < chosen) {
    unsigned long long bk = 0ull;
    int bp = 0x7fffffff;
    for (int i = tid; i < nneg; i += blockDim.x) {
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
    __syncthreads();
    unsigned long long hk = 0ull;
    int hp = -1;
#pragma unroll
    for (int w = 0; w < kLossThreads / 32; ++w) {
      if (s_wkey[w] > hk) {
        hk = s_wkey[w];
        hp = s_wpos[w];
      }
    }
    if (hk == 0ull) break;
    const int hn = (int)(0xFFFFFFFFu - (unsigned)(hk & 0xFFFFFFFFull));
    const float4 cur = neg_anchor_box(p, hn);
    ++nsel;
    if (tid == 0) {
      assign[hn] = kAsMined;
      nodm += hb[(long long)hn * row + kPfpArmC + 1] < 0.99f;  // the raw logit, as the reference (:584)
    }
    for (int j = tid; j < nneg; j += blockDim.x) {
      const unsigned long long kj = keys[j];
      if (kj == 0ull) continue;
      if (j == hp) {
        keys[j] = 0ull;
        continue;
      }
      const int n = (int)(0xFFFFFFFFu - (unsigned)(kj & 0xFFFFFFFFull));
      if (iou_tf(neg_anchor_box(p, n), cur) > 0.7f) keys[j] = 0ull;
    }
    __syncthreads();
  }
  if (tid == 0) {
    s_nsel = nsel;
    s_nodm = nodm;
  }
  __syncthreads();
  const int S = s_nsel, M = s_nodm;
  const float invP = P ? __fdiv_rn(1.f, (float)P) : 0.f;
  const float invS = S ? __fdiv_rn(1.f, (float)S) : 0.f;
  const float invM = M ? __fdiv_rn(1.f, (float)M) : 0.f;
  // (3) the terms: v = (ARM pos CE, ARM coord, ODM pos CE, ODM coord, ARM mined CE, ODM mined CE), and the gradient
  float v[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int n = tid; n < N; n += blockDim.x) {
    const int as = assign[n];
    const float* r = hb + (long long)n * row;
    float gr[row];
#pragma unroll
    for (int k = 0; k < row; ++k) gr[k] = 0.f;
    const bool pos = as >= 0 || as == kAsBest;
    if (pos) {
      const Anchor a = anchor_ssd(p, locate(p, n));
      for (int e = 0; e < (as == kAsBest ? cnt : 1); ++e) {  // a best anchor: once per GT it is the best of
        const int g = as == kAsBest ? e : as;
        if (as == kAsBest && s_best[g] != n) continue;
        const float gy = gb[g * 5], gx = gb[g * 5 + 1], gh = gb[g * 5 + 2], gw = gb[g * 5 + 3];
        const int label = (int)gb[g * 5 + 4];
        v[0] += xent2(r[kPfpArmC], r[kPfpArmC + 1], 0);
        v[1] += coord_loss(r + (kPfpArmT - kPfpOdmT), a, gy, gx, gh, gw);
        v[2] += xent21(r, label);
        // the ARM box (:598-599), then the ODM targets relative to it (:602-603)
        const float ay = __fadd_rn(__fmul_rn(r[kPfpArmT], a.h), a.cy);
        const float ax = __fadd_rn(__fmul_rn(r[kPfpArmT + 1], a.w), a.cx);
        const float ah = __fmul_rn(expf(r[kPfpArmT + 2]), a.h);
        const float aw = __fmul_rn(expf(r[kPfpArmT + 3]), a.w);
        const float oy = __fdiv_rn(__fsub_rn(gy, ay), ah), ox = __fdiv_rn(__fsub_rn(gx, ax), aw);
        const float oh = logf(__fdiv_rn(gh, ah)), ow = logf(__fdiv_rn(gw, aw));
        const float e0 = __fsub_rn(r[kPfpOdmT], oy), e1 = __fsub_rn(r[kPfpOdmT + 1], ox);
        const float e2 = __fsub_rn(r[kPfpOdmT + 2], oh), e3 = __fsub_rn(r[kPfpOdmT + 3], ow);
        v[3] += __fadd_rn(__fadd_rn(smooth_l1(e0), smooth_l1(e1)), __fadd_rn(smooth_l1(e2), smooth_l1(e3)));
        if constexpr (kGrad) {
          const float m = fmaxf(r[kPfpArmC], r[kPfpArmC + 1]);
          const float x0 = expf(r[kPfpArmC] - m), x1 = expf(r[kPfpArmC + 1] - m), inv = 1.f / (x0 + x1);
          gr[kPfpArmC] += (x0 * inv - 1.f) * invP;
          gr[kPfpArmC + 1] += x1 * inv * invP;
          float prob[21];
          softmax21(r, prob);
#pragma unroll
          for (int k = 0; k < 21; ++k) gr[k] += (prob[k] - (k == label ? 1.f : 0.f)) * invP;
          const float ty = (gy - a.cy) / a.h, tx = (gx - a.cx) / a.w;
          const float th = logf(gh / a.h), tw = logf(gw / a.w);
          gr[kPfpArmT] += smooth_l1_grad(r[kPfpArmT] - ty) * invP;
          gr[kPfpArmT + 1] += smooth_l1_grad(r[kPfpArmT + 1] - tx) * invP;
          gr[kPfpArmT + 2] += smooth_l1_grad(r[kPfpArmT + 2] - th) * invP;
          gr[kPfpArmT + 3] += smooth_l1_grad(r[kPfpArmT + 3] - tw) * invP;
          const float d0 = smooth_l1_grad(e0), d1 = smooth_l1_grad(e1);
          const float d2 = smooth_l1_grad(e2), d3 = smooth_l1_grad(e3);
          gr[kPfpOdmT] += d0 * invP;
          gr[kPfpOdmT + 1] += d1 * invP;
          gr[kPfpOdmT + 2] += d2 * invP;
          gr[kPfpOdmT + 3] += d3 * invP;
          // through the ODM targets: d oy / d t_y = -a.h / ah, d oy / d t_h = -oy, d oh / d t_h = -1
          gr[kPfpArmT] += d0 * (a.h / ah) * invP;
          gr[kPfpArmT + 1] += d1 * (a.w / aw) * invP;
          gr[kPfpArmT + 2] += (d0 * oy + d2) * invP;
          gr[kPfpArmT + 3] += (d1 * ox + d3) * invP;
        }
      }
    } else if (as == kAsMined) {
      v[4] += xent2(r[kPfpArmC], r[kPfpArmC + 1], 1);
      const bool odm = r[kPfpArmC + 1] < 0.99f;
      if (odm) v[5] += xent21(r, 20);
      if constexpr (kGrad) {
        const float m = fmaxf(r[kPfpArmC], r[kPfpArmC + 1]);
        const float x0 = expf(r[kPfpArmC] - m), x1 = expf(r[kPfpArmC + 1] - m), inv = 1.f / (x0 + x1);
        gr[kPfpArmC] = x0 * inv * invS;
        gr[kPfpArmC + 1] = (x1 * inv - 1.f) * invS;
        if (odm) {
          float prob[21];
          softmax21(r, prob);
#pragma unroll
          for (int k = 0; k < 21; ++k) gr[k] = (prob[k] - (k == 20 ? 1.f : 0.f)) * invM;
        }
      }
    }
    if constexpr (kGrad) {
      float* go = grad + ((long long)b * N + n) * row;
#pragma unroll
      for (int k = 0; k < row; ++k) go[k] = gr[k];
    }
  }
  block_sum<6, kLossThreads>(s_sum, v);
  if (tid == 0) {
    const float arm = __fadd_rn(__fadd_rn(__fmul_rn(s_sum[4][0], invS), __fmul_rn(s_sum[0][0], invP)),
                                __fmul_rn(s_sum[1][0], invP));
    const float odm = __fadd_rn(__fadd_rn(__fmul_rn(s_sum[5][0], invM), __fmul_rn(s_sum[2][0], invP)),
                                __fmul_rn(s_sum[3][0], invP));
    loss_out[b] = __fadd_rn(arm, odm);
  }
}

}  // namespace odt

// scratch: mining keys u64 [B, N], assignment i32 [B, N], per-GT best anchors i32 [B, 128]
extern "C" long long odt_pfpnet_loss_scratch_bytes(const odt_tail_params* p, int B) {
  if (!p || B <= 0 || p->N <= 0) return -1;
  return (long long)B * p->N * 8 + (long long)B * p->N * 4 + (long long)B * kMaxGT * 4;
}

static int pfpnet_loss(const float* head, const odt_tail_params* p, int B, const float* gt, int G, void* scratch,
                       float* loss_out, float* grad_out, bool with_grad, cudaStream_t st) {
  ODT_CHECK_ARG(head && p && gt && scratch && loss_out, "null pointer");
  ODT_CHECK_ARG(!with_grad || grad_out, "null pointer (gradient)");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_TWO_STEP && p->num_fg == 20, "two-step head with 20 classes expected");
  ODT_CHECK_ARG(p->num_levels >= 1 && p->num_levels <= ODT_MAX_LEVELS, "two-step head with 20 classes expected");
  long long rows = 0;
  for (int i = 0; i < p->num_levels; ++i) {
    const odt_level& L = p->level[i];
    ODT_CHECK_ARG(L.A >= 1 && L.A <= ODT_MAX_PRIORS && L.H > 0 && L.W > 0 && L.offset == rows, "level geometry");
    rows += (long long)L.H * L.W * L.A;
  }
  ODT_CHECK_ARG(rows == p->N, "level geometry");
  ODT_CHECK_ARG(B > 0 && G > 0 && G <= kMaxGT, "B/G (G <= 128)");
  ODT_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(scratch);
  int* assign = reinterpret_cast<int*>(keys + (long long)B * p->N);
  int* best = assign + (long long)B * p->N;
  TailP tp;
  tp.p = *p;
  loss_best_anchor_kernel<<<dim3(G, B), kLossThreads, 0, st>>>(tp, gt, G, best);
  ODT_LAUNCH_OK();
  if (with_grad)
    pfpnet_loss_kernel<true><<<B, kLossThreads, 0, st>>>(head, tp, gt, G, best, keys, assign, loss_out, grad_out);
  else
    pfpnet_loss_kernel<false><<<B, kLossThreads, 0, st>>>(head, tp, gt, G, best, keys, assign, loss_out, nullptr);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_pfpnet_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                   void* scratch, float* loss_out, void* stream) {
  return pfpnet_loss(head, p, B, gt, G, scratch, loss_out, nullptr, false, (cudaStream_t)stream);
}

extern "C" int odt_pfpnet_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                    void* scratch, float* loss_out, float* grad_out, void* stream) {
  return pfpnet_loss(head, p, B, gt, G, scratch, loss_out, grad_out, true, (cudaStream_t)stream);
}
