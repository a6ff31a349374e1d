// Training-loss forwards of the four families (RetinaNet, SSD, FCOS, YOLOv3), forward only.
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
                       int* __restrict__ neg_count) {
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
// tail.cu) + the final combination.  loss_out[b] = mean(selected neg) + conf/npos + coord/npos
__global__ void __launch_bounds__(kLossThreads)
    ssd_loss_mine_kernel(const __grid_constant__ TailP tp, const float* __restrict__ partial,
                         unsigned long long* __restrict__ neg_keys, const int* __restrict__ neg_count,
                         float* __restrict__ loss_out, int* __restrict__ info_out) {
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
  __shared__ float s_box[kMaxGT][kFcosLevels][4];  // y1,x1,y2,x2 in stride units of each level
  __shared__ int s_cls[kMaxGT];
  __shared__ int s_lv[kMaxGT];                      // level membership bits
  __shared__ float s_red[1][kLossThreads];
  const int cnt = block_gt_count(gb, G);
  for (int g = threadIdx.x; g < cnt; g += blockDim.x) {
    const float gy = gb[g * 5], gx = gb[g * 5 + 1], gh = gb[g * 5 + 2], gw = gb[g * 5 + 3];
    const float size = __fsqrt_rn(__fmul_rn(gh, gw));
    int bits = 0;
    if (size <= 64.f) bits |= 1;
    if (size >= 64.f && size <= 128.f) bits |= 2;
    if (size >= 128.f && size <= 256.f) bits |= 4;
    if (size >= 256.f && size <= 512.f) bits |= 8;
    if (size >= 512.f) bits |= 16;
    s_lv[g] = bits;
    s_cls[g] = (int)gb[g * 5 + 4];
    for (int l = 0; l < kFcosLevels; ++l) {
      const float st = p.level[l].out_mul;
      const float y = __fdiv_rn(gy, st), x = __fdiv_rn(gx, st), h = __fdiv_rn(gh, st), w = __fdiv_rn(gw, st);
      const float hh = __fdiv_rn(h, 2.f), hw = __fdiv_rn(w, 2.f);
      s_box[g][l][0] = __fsub_rn(y, hh);
      s_box[g][l][1] = __fsub_rn(x, hw);
      s_box[g][l][2] = __fadd_rn(y, hh);
      s_box[g][l][3] = __fadd_rn(x, hw);
    }
  }
  __syncthreads();
  if (blk == 0 && threadIdx.x < kFcosLevels) {  // GT count per level (a level without GT contributes nothing)
    int c = 0;
    for (int g = 0; g < cnt; ++g) c += (s_lv[g] >> threadIdx.x) & 1;
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
    const float yy = (float)c.y, xx = (float)c.x;
    bool loc = false;
    float amin = 3.0e38f, dl = 0.f, dr = 0.f, dt = 0.f, db = 0.f;
    unsigned cmask[W];
#pragma unroll
    for (int w = 0; w < W; ++w) cmask[w] = 0u;
    for (int g = 0; g < cnt; ++g) {
      if (!((s_lv[g] >> l) & 1)) continue;
      const float l_ = __fsub_rn(xx, s_box[g][l][1]), r_ = __fsub_rn(s_box[g][l][3], xx);
      const float t_ = __fsub_rn(yy, s_box[g][l][0]), b_ = __fsub_rn(s_box[g][l][2], yy);
      if (!(l_ > 0.f && r_ > 0.f && t_ > 0.f && b_ > 0.f)) continue;
      loc = true;
      if (W == 1) {
        cmask[0] |= 1u << s_cls[g];
      } else {
#pragma unroll
        for (int w = 0; w < W; ++w)
          if (s_cls[g] >> 5 == w) cmask[w] |= 1u << (s_cls[g] & 31);
      }
      const float area = __fmul_rn(__fadd_rn(l_, r_), __fadd_rn(t_, b_));
      if (area < amin) {
        amin = area;
        dl = l_; dr = r_; dt = t_; db = b_;
      } else if (area == amin) {  // tied minimal areas: element-wise maximum (:300-307)
        dl = fmaxf(dl, l_); dr = fmaxf(dr, r_); dt = fmaxf(dt, t_); db = fmaxf(db, b_);
      }
    }
    const float* r = hb + (long long)n * row;
    // centre-ness BCE with logits, every location (:331-334); target 0 where no GT covers the cell
    const float lrmin = fminf(dl, dr), tbmin = fminf(dt, db), lrmax = fmaxf(dl, dr), tbmax = fmaxf(dt, db);
    const float cgt = __fsqrt_rn(__fdiv_rn(__fmul_rn(lrmin, tbmin), __fadd_rn(__fmul_rn(lrmax, tbmax), 1e-12f)));
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

// ============================ YOLOv3 loss forward ===========================
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
constexpr int kYoloLevels = 3;

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
// holds the same number of priors A (odt_yolo_loss_fwd checks it), and a cell's A rows are consecutive.
__device__ __forceinline__ int yolo_cell_base(const odt_tail_params& p, int lvl) {
  int c = 0;
  for (int i = 0; i < lvl; ++i) c += p.level[i].H * p.level[i].W;
  return c;
}

// K1: one block per image, one thread per GT: level / prior assignment, positive terms, cell occupancy.
// NFG = 20: the 25-float rows, class loop fixed at compile time; NFG = 0: num_fg from the parameters.
template <int NFG>
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
  const long long cells = yolo_cell_base(p, kYoloLevels);
  float coord = 0.f, cls = 0.f, obj = 0.f;
  if (g < cnt) {
    float mx[kYoloLevels];
    int arg[kYoloLevels], cy[kYoloLevels], cx[kYoloLevels];
#pragma unroll
    for (int k = 0; k < kYoloLevels; ++k) {
      const odt_level& L = p.level[k];
      const YoloGt n = yolo_gt(gb, g, k);
      cy[k] = min(max((int)floorf(n.y), 0), L.H - 1);
      cx[k] = min(max((int)floorf(n.x), 0), L.W - 1);
      // every GT marks its cell on every level
      occ[(long long)b * cells + yolo_cell_base(p, k) + cy[k] * L.W + cx[k]] = 1;
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
    int k = 2;
    if (mx[0] > mx[1] && mx[0] > mx[2]) k = 0;
    else if (mx[1] > mx[0] && mx[1] > mx[2]) k = 1;
    const odt_level& L = p.level[k];
    const YoloGt n = yolo_gt(gb, g, k);
    const float* r = head + ((long long)b * p.N + L.offset + (long long)(cy[k] * L.W + cx[k]) * L.A + arg[k]) * row;
    const float ty = __fsub_rn(n.y, floorf(n.y)), tx = __fsub_rn(n.x, floorf(n.x));
    const float th = logf(__fdiv_rn(n.h, L.prior_h[arg[k]])), tw = logf(__fdiv_rn(n.w, L.prior_w[arg[k]]));
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

// K2: no-object term over every (cell, prior) whose cell holds no GT centre
__global__ void __launch_bounds__(kLossThreads)
    yolo_loss_noobj_kernel(const float* __restrict__ head, const __grid_constant__ TailP tp,
                           const float* __restrict__ gt, int G, const unsigned char* __restrict__ occ,
                           float* __restrict__ partial) {
  pdl_launch_dependents();
  const odt_tail_params& p = tp.p;
  const int b = blockIdx.y, blk = blockIdx.x;
  const float* gb = gt + (long long)b * G * 5;
  __shared__ float s_g[kMaxGT][kYoloLevels][4];
  __shared__ float s_red[1][kLossThreads];
  const int cnt = block_gt_count(gb, G);
  for (int g = threadIdx.x; g < cnt; g += blockDim.x) {
#pragma unroll
    for (int k = 0; k < kYoloLevels; ++k) {
      const YoloGt n = yolo_gt(gb, g, k);
      s_g[g][k][0] = n.y1;
      s_g[g][k][1] = n.x1;
      s_g[g][k][2] = n.y2;
      s_g[g][k][3] = n.x2;
    }
  }
  __syncthreads();
  const long long cells = yolo_cell_base(p, kYoloLevels);
  const int row = row_floats(p.num_fg);
  const float* hb = head + (long long)b * p.N * row;
  float acc = 0.f;
  const int per = (p.N + kLossBlocks - 1) / kLossBlocks;
  const int n_begin = blk * per, n_end = min(p.N, n_begin + per);
  for (int n = n_begin + threadIdx.x; n < n_end; n += blockDim.x) {
    const Cell c = locate(p, n);
    const odt_level& L = p.level[c.lvl];
    if (occ[(long long)b * cells + yolo_cell_base(p, c.lvl) + c.y * L.W + c.x]) continue;
    const float ay = (float)c.y + 0.5f, ax = (float)c.x + 0.5f;
    const float ph = L.prior_h[c.a], pw = L.prior_w[c.a];
    const float cyy = __fsub_rn(ay, __fdiv_rn(ph, 2.f)), cxx = __fsub_rn(ax, __fdiv_rn(pw, 2.f));  // "centre" = y1x1
    const float sh = __fadd_rn(ay, __fdiv_rn(ph, 2.f)), sw = __fadd_rn(ax, __fdiv_rn(pw, 2.f));   // "size"   = y2x2
    const float by1 = __fsub_rn(cyy, __fdiv_rn(sh, 2.f)), bx1 = __fsub_rn(cxx, __fdiv_rn(sw, 2.f));
    const float by2 = __fadd_rn(cyy, __fdiv_rn(sh, 2.f)), bx2 = __fadd_rn(cxx, __fdiv_rn(sw, 2.f));
    const float aarea = __fmul_rn(__fsub_rn(by2, by1), __fsub_rn(bx2, bx1));
    float best = -3.0e38f;
    for (int g = 0; g < cnt; ++g)
      best = fmaxf(best, iou_unclamped(s_g[g][c.lvl][0], s_g[g][c.lvl][1], s_g[g][c.lvl][2], s_g[g][c.lvl][3], by1,
                                       bx1, by2, bx2, aarea));
    if (best <= 0.5f) acc += sig_xent(0.f, hb[(long long)n * row + p.num_fg + 4]);  // objectness
  }
  block_sum(s_red, {acc});
  if (threadIdx.x == 0) partial[(long long)b * kLossBlocks + blk] = s_red[0][0];
}

__global__ void yolo_loss_final_kernel(const float* __restrict__ pos, const float* __restrict__ partial, int B,
                                       float cs, float ns, float os, float ks, float* __restrict__ out) {
  pdl_launch_dependents();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double noobj = 0.0;
  for (int i = 0; i < kLossBlocks; ++i) noobj += (double)partial[(long long)b * kLossBlocks + i];
  const float ng = pos[b * 4 + 3];
  out[b] = (cs * pos[b * 4 + 0] + ks * pos[b * 4 + 1] + os * pos[b * 4 + 2]) / ng + ns * (float)noobj / ng;
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
  long long bytes;
};
static RetinaScratch retina_scratch(const odt_tail_params&, int B, void* base) {
  Carve c{(uintptr_t)base, 0};
  return {c.take<float>((long long)B * kLossBlocks * 4), c.take<int>((long long)B * kMaxGT), c.bytes};
}

struct SsdScratch {
  float* partial;                // as RetinaScratch
  int* best;
  int* neg_count;                // negatives per image
  unsigned long long* neg_keys;  // (background loss, row) per negative, [B][N]
  long long bytes;
};
static SsdScratch ssd_scratch(const odt_tail_params& p, int B, void* base) {
  Carve c{(uintptr_t)base, 0};
  return {c.take<float>((long long)B * kLossBlocks * 4), c.take<int>((long long)B * kMaxGT), c.take<int>(B),
          c.take<unsigned long long>((long long)B * p.N), c.bytes};
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
static long long yolo_cells(const odt_tail_params& p) {
  long long c = 0;
  for (int i = 0; i < kYoloLevels; ++i) c += (long long)p.level[i].H * p.level[i].W;
  return c;
}
static YoloScratch yolo_scratch(const odt_tail_params& p, int B, void* base) {
  Carve c{(uintptr_t)base, 0};
  return {c.take<float>((long long)B * 4), c.take<float>((long long)B * kLossBlocks),
          c.take<unsigned char>((long long)B * yolo_cells(p)), c.bytes};
}

template <class Layout>
static long long scratch_bytes(const odt_tail_params* p, int B, Layout layout) {
  return p && B > 0 && p->N > 0 ? layout(*p, B, nullptr).bytes : -1;
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
  return scratch_bytes(p, B, yolo_scratch);
}

extern "C" int odt_retina_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                   float alpha, float gamma, void* scratch, float* loss_out, void* stream) {
  ODT_CHECK_ARG(head && p && gt && scratch && loss_out, "null pointer");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_SSD && p->num_fg == 20, "softmax-family head with 20 classes expected");
  ODT_CHECK_ARG(B > 0 && G > 0 && G <= kMaxGT, "B/G (G <= 128)");
  ODT_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const RetinaScratch s = retina_scratch(*p, B, scratch);
  TailP tp;
  tp.p = *p;
  loss_best_anchor_kernel<<<dim3(G, B), kLossThreads, 0, st>>>(tp, gt, G, s.best);
  ODT_LAUNCH_OK();
  loss_anchor_kernel<false><<<dim3(kLossBlocks, B), kLossThreads, 0, st>>>(head, tp, gt, G, s.best, alpha, gamma,
                                                                          s.partial, nullptr, nullptr);
  ODT_LAUNCH_OK();
  loss_final_kernel<<<(B + 63) / 64, 64, 0, st>>>(s.partial, B, loss_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_ssd_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                void* scratch, float* loss_out, int* info_out, void* stream) {
  ODT_CHECK_ARG(head && p && gt && scratch && loss_out, "null pointer");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_SSD && p->num_fg == 20, "softmax-family head with 20 classes expected");
  ODT_CHECK_ARG(B > 0 && G > 0 && G <= kMaxGT, "B/G (G <= 128)");
  ODT_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const SsdScratch s = ssd_scratch(*p, B, scratch);
  ODT_CUDA_OK(cudaMemsetAsync(s.neg_count, 0, sizeof(int) * (size_t)B, st));
  TailP tp;
  tp.p = *p;
  loss_best_anchor_kernel<<<dim3(G, B), kLossThreads, 0, st>>>(tp, gt, G, s.best);
  ODT_LAUNCH_OK();
  loss_anchor_kernel<true><<<dim3(kLossBlocks, B), kLossThreads, 0, st>>>(head, tp, gt, G, s.best, 0.f, 0.f,
                                                                         s.partial, s.neg_keys, s.neg_count);
  ODT_LAUNCH_OK();
  ssd_loss_mine_kernel<<<B, kLossThreads, 0, st>>>(tp, s.partial, s.neg_keys, s.neg_count, loss_out, info_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_fcos_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                 void* scratch, float* loss_out, void* stream) {
  ODT_CHECK_ARG(head && p && gt && scratch && loss_out, "null pointer");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_FCOS && p->num_levels == kFcosLevels && p->num_fg >= 1 && p->num_fg <= kMaxFg,
                "FCOS head with 5 levels and 1..128 classes expected");
  ODT_CHECK_ARG(B > 0 && G > 0 && G <= kMaxGT, "B/G (G <= 128)");
  ODT_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const FcosScratch s = fcos_scratch(*p, B, scratch);
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

extern "C" int odt_yolo_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                 float coord_scale, float noobj_scale, float obj_scale, float class_scale,
                                 void* scratch, float* loss_out, void* stream) {
  ODT_CHECK_ARG(head && p && gt && scratch && loss_out, "null pointer");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_YOLO3 && p->num_levels == kYoloLevels && p->num_fg >= 1 && p->num_fg <= kMaxFg,
                "YOLOv3 head with 3 levels and 1..128 classes expected");
  // One prior count on every level (the config's num_priors), and rows laid out level after level, cell after cell:
  // the kernels find a level's rows at its offset and its cells in the occupancy array by these sums.
  const int A = p->level[0].A;
  ODT_CHECK_ARG(A >= 1 && A <= ODT_MAX_PRIORS, "1..9 priors per level expected");
  long long rows = 0;
  for (int i = 0; i < kYoloLevels; ++i) {
    const odt_level& L = p->level[i];
    ODT_CHECK_ARG(L.A == A, "the same number of priors on every level expected");
    ODT_CHECK_ARG(L.H >= 1 && L.W >= 1 && L.offset == rows, "level geometry: H, W >= 1, offset = rows before it");
    rows += (long long)L.H * L.W * A;
  }
  ODT_CHECK_ARG(rows == p->N, "N must be the sum of H * W * A over the levels");
  ODT_CHECK_ARG(B > 0 && G > 0 && G <= kMaxGT, "B/G (G <= 128)");
  ODT_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "scratch must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const YoloScratch s = yolo_scratch(*p, B, scratch);
  ODT_CUDA_OK(cudaMemsetAsync(s.occ, 0, (size_t)B * yolo_cells(*p), st));
  TailP tp;
  tp.p = *p;
  if (p->num_fg == 20)
    yolo_loss_pos_kernel<20><<<B, kMaxGT, 0, st>>>(head, tp, gt, G, s.occ, s.pos);
  else
    yolo_loss_pos_kernel<0><<<B, kMaxGT, 0, st>>>(head, tp, gt, G, s.occ, s.pos);
  ODT_LAUNCH_OK();
  yolo_loss_noobj_kernel<<<dim3(kLossBlocks, B), kLossThreads, 0, st>>>(head, tp, gt, G, s.occ, s.partial);
  ODT_LAUNCH_OK();
  yolo_loss_final_kernel<<<(B + 63) / 64, 64, 0, st>>>(s.pos, s.partial, B, coord_scale, noobj_scale, obj_scale,
                                                       class_scale, loss_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}
