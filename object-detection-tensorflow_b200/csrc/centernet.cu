// CenterNet (ref CenterNet.py): the DLA pooled join, the peak + top-k detection tail, and the Gaussian-heatmap focal
// loss with its gradient.  Candidate rows are fp32 [B, H*W, C + 4]: C keypoint logits, (dy, dx), (h, w) per cell of
// the stride-4 grid, raster order.  Every selection and reduction runs in a fixed order: no float atomics.
#include <math.h>

#include "common.cuh"

namespace odt {
namespace {

constexpr int kPeakThreads = 1024;  // one CTA per image selects; also the largest top_k_results_output
constexpr int kLossThreads = 256;   // one pixel per thread
constexpr int kCnMaxGT = 128;
constexpr int kCnMaxFg = 128;  // classes per row, as YOLOv3 and FCOS allow
constexpr float kCenterStride = 4.f;  // ref CenterNet.py:129

inline int cn_grid(long long work, int threads) {
  long long b = (work + threads - 1) / threads;
  long long cap = (long long)kNumSMs * 16;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

__host__ __device__ __forceinline__ int cn_row(int num_fg) { return num_fg + 4; }

// ---- the DLA joins --------------------------------------------------------------------------------------------
// pooled = 0: out = a + b (a _dla_generator's block1 + block2, ref CenterNet.py:394,399).
// pooled = 1: out = max_pool(a, 2, 2, SAME) + average_pool(b, 2, 2, SAME) (the stage joins, ref :93-110): a and b are
// [B, H, W, C], out [B, ceil(H/2), ceil(W/2), C]; each window's cells inside the image, the average summed in
// row-major order and divided by their number.  fp32 math, one rounding per TF op.
template <typename T>
__global__ void dla_join_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out, int B, int H,
                                int W, int C, int a_ld, int b_ld, int out_ld, int pooled) {
  pdl_launch_dependents();
  const int OH = pooled ? (H + 1) / 2 : H, OW = pooled ? (W + 1) / 2 : W;
  const long long total = (long long)B * OH * OW * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    float v;
    if (!pooled) {
      v = __fadd_rn(Elem<T>::ld(a + pix * a_ld + c), Elem<T>::ld(b + pix * b_ld + c));
    } else {
      const int ox = (int)(pix % OW);
      const long long t = pix / OW;
      const int oy = (int)(t % OH);
      const int bi = (int)(t / OH);
      const long long img = (long long)bi * H * W;
      float m = -INFINITY, s = 0.f;
      int n = 0;
      for (int dy = 0; dy < 2; ++dy) {
        const int y = 2 * oy + dy;
        if (y >= H) break;
        for (int dx = 0; dx < 2; ++dx) {
          const int x = 2 * ox + dx;
          if (x >= W) break;
          const long long q = img + (long long)y * W + x;
          m = fmaxf(m, Elem<T>::ld(a + q * a_ld + c));
          s = __fadd_rn(s, Elem<T>::ld(b + q * b_ld + c));
          ++n;
        }
      }
      v = __fadd_rn(m, __fdiv_rn(s, (float)n));
    }
    Elem<T>::st(out + pix * out_ld + c, v);
  }
}

// ---- the detection tail (ref CenterNet.py:159-185) ------------------------------------------------------------
// sigmoid rounded once from float64: the float32 value nearest 1 / (1 + exp(-x)), which the numpy oracle computes the
// same way, so scores, plateaus and ties compare bit for bit
__device__ __forceinline__ float sigmoid_f64(float x) { return (float)(1.0 / (1.0 + exp(-(double)x))); }

// per cell: the largest class sigmoid and its class (first maximum, tf.argmax)
__global__ void peak_score_kernel(const float* __restrict__ head, int HW, int nfg, float* __restrict__ score,
                                  int* __restrict__ cls) {
  pdl_launch_dependents();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= HW) return;
  const long long q = (long long)blockIdx.y * HW + pix;
  const float* r = head + q * cn_row(nfg);
  float best = sigmoid_f64(r[0]);
  int bc = 0;
  for (int c = 1; c < nfg; ++c) {
    const float s = sigmoid_f64(r[c]);
    if (s > best) {
      best = s;
      bc = c;
    }
  }
  score[q] = best;
  cls[q] = bc;
}

// One CTA per image: peak test, threshold, exact top-k, records.  A cell's candidate score is s where s equals the
// 3x3 SAME max-pool of the score map and 0 elsewhere (keypoints * mask, :168-171); it is kept when > score_thr.  Keys
// (score bits << 32) | ~index order by descending score, then ascending index (tf.nn.top_k); the K-th largest key is
// found by an 8-bit radix select over the candidate list, the keys at or above it are sorted bitonically.
__global__ void __launch_bounds__(kPeakThreads)
    peak_select_kernel(const float* __restrict__ head, const __grid_constant__ odt_tail_params p,
                       const float* __restrict__ score, const int* __restrict__ cls,
                       unsigned long long* __restrict__ cand, float* __restrict__ rec, int rec_ld,
                       int* __restrict__ det_anchor) {
  pdl_launch_dependents();
  __shared__ unsigned long long s_sel[kPeakThreads];
  __shared__ int s_hist[256];
  __shared__ int s_n, s_m;
  __shared__ unsigned long long s_prefix, s_mask;
  __shared__ int s_k;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int H = p.level[0].H, W = p.level[0].W, HW = H * W, nfg = p.num_fg, K = p.max_boxes;
  const float* sc = score + (long long)b * HW;
  unsigned long long* ck = cand + (long long)b * HW;
  if (tid == 0) s_n = 0;
  __syncthreads();
  for (int i = tid; i < HW; i += kPeakThreads) {
    const float s = sc[i];
    const int y = i / W, x = i - y * W;
    float m = s;
    for (int dy = -1; dy <= 1; ++dy) {
      const int yy = y + dy;
      if (yy < 0 || yy >= H) continue;
      for (int dx = -1; dx <= 1; ++dx) {
        const int xx = x + dx;
        if (xx < 0 || xx >= W) continue;
        m = fmaxf(m, sc[yy * W + xx]);
      }
    }
    const float v = (s == m) ? s : 0.f;
    if (v > p.score_thr) {
      const int slot = atomicAdd(&s_n, 1);
      ck[slot] = ((unsigned long long)__float_as_uint(v) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i);
    }
  }
  __syncthreads();  // the block's global stores of ck are visible to the block from here
  const int n = s_n;
  if (tid == 0) {
    s_prefix = 0ull;
    s_mask = 0ull;
    s_k = K;
    s_m = 0;
  }
  __syncthreads();
  if (n > K) {
    for (int shift = 56; shift >= 0; shift -= 8) {
      if (tid < 256) s_hist[tid] = 0;
      __syncthreads();
      const unsigned long long pre = s_prefix, msk = s_mask;
      for (int i = tid; i < n; i += kPeakThreads) {
        const unsigned long long key = ck[i];
        if ((key & msk) == pre) atomicAdd(&s_hist[(int)((key >> shift) & 255ull)], 1);
      }
      __syncthreads();
      if (tid == 0) {
        int k = s_k, d = 255;
        for (; d > 0; --d) {
          if (s_hist[d] >= k) break;
          k -= s_hist[d];
        }
        s_k = k;
        s_prefix = pre | ((unsigned long long)d << shift);
        s_mask = msk | (255ull << shift);
      }
      __syncthreads();
    }
  }
  const unsigned long long thr = (n > K) ? s_prefix : 0ull;  // keys are unique: exactly min(n, K) pass
  for (int i = tid; i < n; i += kPeakThreads) {
    const unsigned long long key = ck[i];
    if (key >= thr) s_sel[atomicAdd(&s_m, 1)] = key;
  }
  __syncthreads();
  const int m = s_m;
  int P = 1;
  while (P < m) P <<= 1;
  if (tid >= m && tid < P) s_sel[tid] = 0ull;
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1) {  // bitonic sort, descending
    for (int j = k >> 1; j > 0; j >>= 1) {
      const int ixj = tid ^ j;
      if (tid < P && ixj > tid) {
        const unsigned long long a = s_sel[tid], c = s_sel[ixj];
        const bool desc = (tid & k) == 0;
        if (desc ? (a < c) : (a > c)) {
          s_sel[tid] = c;
          s_sel[ixj] = a;
        }
      }
      __syncthreads();
    }
  }
  float* rb = rec + (long long)b * rec_ld;
  const int row = cn_row(nfg);
  for (int i = tid; i < K; i += kPeakThreads) {
    float o[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int idx = 0;
    if (i < m) {
      const unsigned long long key = s_sel[i];
      idx = (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull));
      const float* r = head + ((long long)b * HW + idx) * row + nfg;
      const int y = idx / W, x = idx - y * W;
      // ((i, j) + (dy, dx) -/+ (h, w) / 2) * 4: the centre is the integer cell (:141-143,173-180)
      const float cy = __fadd_rn((float)y, r[0]), cx = __fadd_rn((float)x, r[1]);
      const float h2 = __fmul_rn(r[2], 0.5f), w2 = __fmul_rn(r[3], 0.5f);
      o[0] = __uint_as_float((unsigned)(key >> 32));
      o[1] = __fmul_rn(__fsub_rn(cy, h2), kCenterStride);
      o[2] = __fmul_rn(__fsub_rn(cx, w2), kCenterStride);
      o[3] = __fmul_rn(__fadd_rn(cy, h2), kCenterStride);
      o[4] = __fmul_rn(__fadd_rn(cx, w2), kCenterStride);
      o[5] = (float)cls[(long long)b * HW + idx];
    }
#pragma unroll
    for (int e = 0; e < 6; ++e) rb[(long long)i * 6 + e] = o[e];
    if (det_anchor) det_anchor[(long long)b * K + i] = i < m ? idx : 0;
  }
  if (tid == 0) {
    rb[(long long)K * 6] = (float)m;
    rb[(long long)K * 6 + 1] = 0.f;
  }
}

// ---- the training loss (ref CenterNet.py:187-270) --------------------------------------------------------------
// Per image, in float64: GT count by the argmin rule; centres, sizes in grid units (/ 4), floored centre cells (clamped
// into the grid); one sigma, the least of the three CornerNet radii over every GT (:254-270); per class the maximum of
// exp(-d^2 / 2 sigma^2) around the unfloored centres of that class's GTs; focal terms over every (cell, class).
// The image's GT summary, written once per image by cn_gt_kernel and copied to shared memory by the loss kernels.
struct CnGT {
  double gy[kCnMaxGT], gx[kCnMaxGT], gh[kCnMaxGT], gw[kCnMaxGT];  // centre and size in grid units (GT / 4)
  double inv2s2, inv_n, w_off;  // 1 / (2 sigma^2), 1 / G, 1 / (2 G); 0 for G = 0
  int cells[kCnMaxGT], clss[kCnMaxGT];
  int order[kCnMaxGT];          // GT indices sorted by class, GT order within a class
  int first[kCnMaxFg + 1];      // class c owns order[first[c] .. first[c + 1])
  int count;
};

// log(1 + t) for t in (0, 1] without log1p's division (a slow-path call): below 1e-8 the series t - t^2 / 2
__device__ __forceinline__ double log1p_small(double t) { return t < 1e-8 ? t - 0.5 * t * t : log(1.0 + t); }

__device__ __forceinline__ double log_sigmoid(double k) {
  return k >= 0 ? -log1p_small(exp(-k)) : k - log1p_small(exp(k));
}

// One CTA of kCnMaxGT threads per image.  A class id outside [0, num_fg) matches no heatmap channel (tf.equal over
// range(num_classes)) but counts everywhere else.
__global__ void __launch_bounds__(kCnMaxGT)
    cn_gt_kernel(const float* __restrict__ gt_all, int G, const __grid_constant__ odt_tail_params p,
                 CnGT* __restrict__ out) {
  pdl_launch_dependents();
  __shared__ CnGT s;
  __shared__ double s_r[kCnMaxGT];
  __shared__ int s_fill[kCnMaxFg];
  const int tid = threadIdx.x, b = blockIdx.x;
  const int H = p.level[0].H, W = p.level[0].W, nfg = p.num_fg;
  const float* gt = gt_all + (long long)b * G * 5;
  if (tid == 0) {
    int cnt = 0;
    float mn = gt[0];
    for (int g = 1; g < G; ++g)  // first minimum of column 0 (tf.argmin, ref :189-190)
      if (gt[g * 5] < mn) {
        mn = gt[g * 5];
        cnt = g;
      }
    s.count = cnt;
  }
  __syncthreads();
  const int cnt = s.count;
  if (tid < cnt) {
    const float* r = gt + tid * 5;
    const float y = __fmul_rn(r[0], 0.25f), x = __fmul_rn(r[1], 0.25f);  // / stride (:191-199)
    const float h = __fmul_rn(r[2], 0.25f), w = __fmul_rn(r[3], 0.25f);
    const int iy = min(max((int)floorf(y), 0), H - 1), ix = min(max((int)floorf(x), 0), W - 1);
    s.cells[tid] = iy * W + ix;
    s.clss[tid] = (int)r[4];
    s.gy[tid] = y;
    s.gx[tid] = x;
    s.gh[tid] = h;
    s.gw[tid] = w;
    // CornerNet's three radii as the reference writes them, (b + sqrt(b^2 - 4ac)) / 2 each (:254-270)
    const double hd = h, wd = w, o = 0.7;
    const double b1 = hd + wd, c1 = wd * hd * (1. - o) / (1. + o);
    const double r1 = (b1 + sqrt(b1 * b1 - 4. * c1)) / 2.;
    const double b2 = 2. * (hd + wd), c2 = (1. - o) * wd * hd;
    const double r2 = (b2 + sqrt(b2 * b2 - 16. * c2)) / 2.;
    const double a3 = 4. * o, b3 = -2. * o * (hd + wd), c3 = (o - 1.) * wd * hd;
    const double r3 = (b3 + sqrt(b3 * b3 - 4. * a3 * c3)) / 2.;
    s_r[tid] = fmin(r1, fmin(r2, r3));
  }
  __syncthreads();
  if (tid == 0) {
    double rmin = INFINITY;  // one sigma per image: tf.reduce_min over every GT's three radii
    for (int g = 0; g < cnt; ++g) rmin = fmin(rmin, s_r[g]);
    s.inv2s2 = cnt ? 1.0 / (2.0 * rmin * rmin) : 0.0;
    s.inv_n = cnt ? 1.0 / cnt : 0.0;
    s.w_off = cnt ? 1.0 / (2.0 * cnt) : 0.0;
    for (int c = 0; c <= nfg; ++c) s.first[c] = 0;
    for (int g = 0; g < cnt; ++g)
      if (s.clss[g] >= 0 && s.clss[g] < nfg) ++s.first[s.clss[g] + 1];
    for (int c = 0; c < nfg; ++c) {
      s.first[c + 1] += s.first[c];
      s_fill[c] = s.first[c];
    }
    for (int g = 0; g < cnt; ++g)
      if (s.clss[g] >= 0 && s.clss[g] < nfg) s.order[s_fill[s.clss[g]]++] = g;
  }
  __syncthreads();
  const int* src = (const int*)&s;
  int* dst = (int*)(out + b);
  for (int i = tid; i < (int)(sizeof(CnGT) / 4); i += blockDim.x) dst[i] = src[i];
}

__device__ __forceinline__ void cn_copy_gt(const CnGT* __restrict__ g, CnGT& s) {
  const int* src = (const int*)g;
  int* dst = (int*)&s;
  for (int i = threadIdx.x; i < (int)(sizeof(CnGT) / 4); i += blockDim.x) dst[i] = src[i];
  __syncthreads();
}

// Focal terms of this CTA's cells, summed in a fixed order into partial[b][block] = (positive sum, negative sum);
// GRAD: also every element of d loss / d row for those cells.
template <bool GRAD>
__global__ void __launch_bounds__(kLossThreads)
    cn_loss_cells_kernel(const float* __restrict__ head, const __grid_constant__ odt_tail_params p,
                         const CnGT* __restrict__ gts, double* __restrict__ partial, float* __restrict__ grad) {
  pdl_launch_dependents();
  __shared__ CnGT sh;
  __shared__ double s_red[2][kLossThreads];
  const int b = blockIdx.y, tid = threadIdx.x;
  const int H = p.level[0].H, W = p.level[0].W, HW = H * W, nfg = p.num_fg, row = cn_row(nfg);
  cn_copy_gt(gts + b, sh);
  const int pix = blockIdx.x * kLossThreads + tid;
  double pos = 0.0, neg = 0.0;
  if (pix < HW) {
    const long long q = (long long)b * HW + pix;
    const float* r = head + q * row;
    float* gr = GRAD ? grad + q * row : nullptr;
    const double yy = pix / W, xx = pix % W;
    const double inv_n = sh.inv_n;
    // an image without boxes: no class has a GT and inv_n = 0, so every term and gradient below is 0
    for (int c = 0; c < nfg; ++c) {
      double red = 0.0;
      bool hit = false;
      for (int t = sh.first[c]; t < sh.first[c + 1]; ++t) {
        const int g = sh.order[t];
        const double dy = sh.gy[g] - yy, dx = sh.gx[g] - xx;
        red = fmax(red, exp(-(dy * dy + dx * dx) * sh.inv2s2));
        hit |= sh.cells[g] == pix;
      }
      const double k = r[c];
      const double ls = log_sigmoid(k), lsn = log_sigmoid(-k);  // log p, log(1 - p)
      const double pr = exp(ls), qr = exp(lsn);                  // p, 1 - p
      double d;
      if (hit) {  // -(1 - p)^2 log p
        pos += -qr * qr * ls;
        d = 2.0 * pr * qr * qr * ls - qr * qr * qr;
      } else {    // -(1 - r)^4 p^2 log(1 - p)
        const double w2 = (1.0 - red) * (1.0 - red), w4 = w2 * w2;
        neg += -w4 * pr * pr * lsn;
        d = -w4 * (2.0 * pr * pr * qr * lsn - pr * pr * pr);
      }
      if (GRAD) gr[c] = (float)(d * inv_n);
    }
    if (GRAD) {  // L1 terms at the GTs' cells, GTs that share a cell added in GT order; sign(0) = 0
      double g4[4] = {0.0, 0.0, 0.0, 0.0};
      const double w_off = sh.w_off, w_size = 0.1 * w_off;
      for (int g = 0; g < sh.count; ++g) {
        if (sh.cells[g] != pix) continue;
        const double t[4] = {sh.gy[g] - floor(sh.gy[g]), sh.gx[g] - floor(sh.gx[g]), sh.gh[g], sh.gw[g]};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const double dlt = t[e] - (double)r[nfg + e];
          const double sg = dlt > 0 ? 1.0 : (dlt < 0 ? -1.0 : 0.0);
          g4[e] += -sg * (e < 2 ? w_off : w_size);
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) gr[nfg + e] = (float)g4[e];
    }
  }
  s_red[0][tid] = pos;
  s_red[1][tid] = neg;
  __syncthreads();
  for (int st = kLossThreads / 2; st > 0; st >>= 1) {
    if (tid < st) {
      s_red[0][tid] += s_red[0][tid + st];
      s_red[1][tid] += s_red[1][tid + st];
    }
    __syncthreads();
  }
  if (tid == 0) {
    double* pp = partial + ((long long)b * gridDim.x + blockIdx.x) * 2;
    pp[0] = s_red[0][0];
    pp[1] = s_red[1][0];
  }
}

// loss[b] = (sum pos + sum neg) / G + 0.1 * mean|size t - size| + mean|offset t - offset| (G x 2 means); 0 for G = 0
__global__ void cn_loss_final_kernel(const float* __restrict__ head, const __grid_constant__ odt_tail_params p,
                                     const CnGT* __restrict__ gts, const double* __restrict__ partial, int nblk,
                                     float* __restrict__ loss_out) {
  pdl_launch_dependents();
  const int b = blockIdx.x;
  const int HW = p.level[0].H * p.level[0].W, nfg = p.num_fg, row = cn_row(nfg);
  const CnGT& sh = gts[b];
  const int cnt = sh.count;
  if (!cnt) {
    loss_out[b] = 0.f;
    return;
  }
  double ps = 0.0, ns = 0.0;
  for (int i = 0; i < nblk; ++i) {
    ps += partial[((long long)b * nblk + i) * 2];
    ns += partial[((long long)b * nblk + i) * 2 + 1];
  }
  double off = 0.0, size = 0.0;
  for (int g = 0; g < cnt; ++g) {
    const float* r = head + ((long long)b * HW + sh.cells[g]) * row + nfg;
    off += fabs(sh.gy[g] - floor(sh.gy[g]) - (double)r[0]) + fabs(sh.gx[g] - floor(sh.gx[g]) - (double)r[1]);
    size += fabs(sh.gh[g] - (double)r[2]) + fabs(sh.gw[g] - (double)r[3]);
  }
  loss_out[b] = (float)(ps / cnt + ns / cnt + 0.1 * size / (2.0 * cnt) + off / (2.0 * cnt));
}

int check_peak_params(const odt_tail_params* p, int B) {
  ODT_CHECK_ARG(p != nullptr, "params null");
  ODT_CHECK_ARG(p->kind == ODT_DECODE_PEAK, "kind must be ODT_DECODE_PEAK");
  ODT_CHECK_ARG(p->num_levels == 1 && p->level[0].A == 1, "one level, one prior");
  ODT_CHECK_ARG(p->level[0].H >= 1 && p->level[0].W >= 1 && (long long)p->level[0].H * p->level[0].W == p->N,
                "N must be H * W");
  ODT_CHECK_ARG(p->num_fg >= 1 && p->num_fg <= kCnMaxFg, "num_fg must be 1..128");
  ODT_CHECK_ARG(B >= 1 && (long long)B * p->N * cn_row(p->num_fg) < (1ll << 40), "B");
  return ODT_OK;
}

long long nblk_of(const odt_tail_params* p) { return (p->N + kLossThreads - 1) / kLossThreads; }

}  // namespace
}  // namespace odt

using namespace odt;

extern "C" int odt_dla_join(const void* a, const void* b, void* out, int dtype, int B, int H, int W, int C, int a_ld,
                            int b_ld, int out_ld, int pooled, void* stream) {
  ODT_CHECK_ARG(a && b && out && B > 0 && H > 0 && W > 0 && C > 0 && a_ld >= C && b_ld >= C && out_ld >= C &&
                    (pooled == 0 || pooled == 1),
                "args");
  cudaStream_t st = (cudaStream_t)stream;
  const long long work = (long long)B * (pooled ? ((H + 1) / 2) * ((W + 1) / 2) : H * W) * C;
  if (dtype == ODT_F16) {
    dla_join_kernel<__half><<<cn_grid(work, 256), 256, 0, st>>>((const __half*)a, (const __half*)b, (__half*)out, B,
                                                                 H, W, C, a_ld, b_ld, out_ld, pooled);
  } else {
    ODT_CHECK_ARG(dtype == ODT_F32, "dtype");
    dla_join_kernel<float><<<cn_grid(work, 256), 256, 0, st>>>((const float*)a, (const float*)b, (float*)out, B, H,
                                                                W, C, a_ld, b_ld, out_ld, pooled);
  }
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" long long odt_peak_topk_scratch_bytes(const odt_tail_params* p, int B) {
  if (check_peak_params(p, B)) return -1;
  return (long long)B * p->N * (4 + 4 + 8);
}

extern "C" int odt_peak_topk(const float* head, const odt_tail_params* p, int B, void* scratch, float* rec, int rec_ld,
                             int* det_anchor, void* stream) {
  int rc = check_peak_params(p, B);
  if (rc) return rc;
  ODT_CHECK_ARG(head && scratch && rec, "null tensor");
  ODT_CHECK_ARG(p->max_boxes >= 1 && p->max_boxes <= kPeakThreads, "max_boxes must be 1..1024");
  ODT_CHECK_ARG(rec_ld >= p->max_boxes * 6 + 2, "rec_ld");
  ODT_CHECK_ARG(((uintptr_t)scratch % 8) == 0, "scratch must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)B * p->N;
  unsigned long long* cand = (unsigned long long*)scratch;
  float* score = (float*)(cand + n);
  int* cls = (int*)(score + n);
  peak_score_kernel<<<dim3((p->N + 255) / 256, B), 256, 0, st>>>(head, p->N, p->num_fg, score, cls);
  ODT_LAUNCH_OK();
  peak_select_kernel<<<B, kPeakThreads, 0, st>>>(head, *p, score, cls, cand, rec, rec_ld, det_anchor);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" long long odt_centernet_loss_scratch_bytes(const odt_tail_params* p, int B) {
  if (check_peak_params(p, B)) return -1;
  return (long long)B * (nblk_of(p) * 2 * 8 + (long long)sizeof(CnGT));
}

static int centernet_loss(const float* head, const odt_tail_params* p, int B, const float* gt, int G, void* scratch,
                          float* loss_out, float* grad_out, void* stream) {
  int rc = check_peak_params(p, B);
  if (rc) return rc;
  ODT_CHECK_ARG(head && gt && scratch && loss_out, "null tensor");
  ODT_CHECK_ARG(G >= 1 && G <= kCnMaxGT, "G must be 1..128");
  ODT_CHECK_ARG(((uintptr_t)scratch % 8) == 0, "scratch must be 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int nblk = (int)nblk_of(p);
  double* partial = (double*)scratch;
  CnGT* gts = (CnGT*)(partial + (long long)B * nblk * 2);
  cn_gt_kernel<<<B, kCnMaxGT, 0, st>>>(gt, G, *p, gts);
  ODT_LAUNCH_OK();
  if (grad_out)
    cn_loss_cells_kernel<true><<<dim3(nblk, B), kLossThreads, 0, st>>>(head, *p, gts, partial, grad_out);
  else
    cn_loss_cells_kernel<false><<<dim3(nblk, B), kLossThreads, 0, st>>>(head, *p, gts, partial, nullptr);
  ODT_LAUNCH_OK();
  cn_loss_final_kernel<<<B, 1, 0, st>>>(head, *p, gts, partial, nblk, loss_out);
  ODT_LAUNCH_OK();
  return ODT_OK;
}

extern "C" int odt_centernet_loss_fwd(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                      void* scratch, float* loss_out, void* stream) {
  return centernet_loss(head, p, B, gt, G, scratch, loss_out, nullptr, stream);
}

extern "C" int odt_centernet_loss_grad(const float* head, const odt_tail_params* p, int B, const float* gt, int G,
                                       void* scratch, float* loss_out, float* grad_out, void* stream) {
  ODT_CHECK_ARG(grad_out != nullptr, "grad_out null");
  return centernet_loss(head, p, B, gt, G, scratch, loss_out, grad_out, stream);
}
