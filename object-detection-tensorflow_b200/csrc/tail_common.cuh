// Device helpers shared by the inference tail (tail.cu) and the training-loss
// forwards (loss.cu): level lookup, analytic anchors / priors, box decode.
#pragma once
#include "common.cuh"

namespace odt {

constexpr int kRow = 25;  // floats per candidate row in the head buffer

struct TailP {
  odt_tail_params p;
};

struct Cell {
  int lvl, y, x, a;
};

__device__ __forceinline__ Cell locate(const odt_tail_params& p, int n) {
  int l = 0;
#pragma unroll 1
  for (int i = 1; i < p.num_levels; ++i)
    if (n >= p.level[i].offset) l = i;
  const odt_level& L = p.level[l];
  int local = n - L.offset;
  Cell c;
  c.lvl = l;
  c.a = local % L.A;
  int cell = local / L.A;
  c.x = cell % L.W;
  c.y = cell / L.W;
  return c;
}

// exp(x) for the score activations of the decode kernel: 2^(x*log2 e) through MUFU.EX2 with the rounding error of the
// product folded back in (hi = fl(x*L2E); r = fma(x, L2E, -hi) is its exact residual, x*L2E_LO the part of log2 e
// beyond fp32; e^x = 2^hi * (1 + ln2*(r + x*L2E_LO))): 6 instructions and ~2 ulp over the whole range, against ~20
// instructions (range checks, exponent re-assembly) for libdevice's expf -- 21 of them per candidate row made up more
// than a third of the decode kernel's instruction stream.  Results below 2^-126 flush to zero (they can never reach a
// threshold).  TF's own CPU exp (Eigen pexp) is a different polynomial again, so no choice of exp is bit-identical
// to it; parity tests compare scores to 1e-6 relative.
__device__ __forceinline__ float exp_score(float x) {
  const float L2E = 1.4426950216293335f;      // fl(log2 e)
  const float L2E_LO = 1.9259629911e-08f;     // log2 e - fl(log2 e)
  const float hi = __fmul_rn(x, L2E);
  const float res = __fmaf_rn(x, L2E, -hi);
  const float corr = __fmul_rn(__fmaf_rn(x, L2E_LO, res), 0.6931471805599453f);
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(hi));
  return __fmaf_rn(r, corr, r);
}

// score sigmoid of the decode kernel: 1/(1+exp(-x)) with exp_score and the correctly rounded reciprocal
// (__frcp_rn(y) == __fdiv_rn(1, y) bit for bit, without the division's slow-path call)
__device__ __forceinline__ float sigmoid_score(float x) { return __frcp_rn(__fadd_rn(1.f, exp_score(-x))); }

__device__ __forceinline__ float sigmoid_rn(float x) {
  // tf.sigmoid = 1/(1+exp(-x))  (SURVEY App. A.9)
  return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
}


// SSD / RetinaNet anchor in the reference's op order (SSD300.py:339-342,
// RetinaNet.py:351-354): corners first, then yx = y1x1/2 + y2x2/2, hw = y2x2 - y1x1.
struct Anchor {
  float y1, x1, y2, x2, cy, cx, h, w;
};
__device__ __forceinline__ Anchor anchor_ssd(const odt_tail_params& p, const Cell& c) {
  const odt_level& L = p.level[c.lvl];
  float cy = __fdiv_rn(__fmul_rn((float)c.y + 0.5f, L.cmul_y), L.cdiv_y);
  float cx = __fdiv_rn(__fmul_rn((float)c.x + 0.5f, L.cmul_x), L.cdiv_x);
  float hh = __fmul_rn(L.prior_h[c.a], 0.5f), hw = __fmul_rn(L.prior_w[c.a], 0.5f);
  Anchor a;
  a.y1 = __fsub_rn(cy, hh);
  a.x1 = __fsub_rn(cx, hw);
  a.y2 = __fadd_rn(cy, hh);
  a.x2 = __fadd_rn(cx, hw);
  a.cy = __fadd_rn(__fmul_rn(a.y1, 0.5f), __fmul_rn(a.y2, 0.5f));
  a.cx = __fadd_rn(__fmul_rn(a.x1, 0.5f), __fmul_rn(a.x2, 0.5f));
  a.h = __fsub_rn(a.y2, a.y1);
  a.w = __fsub_rn(a.x2, a.x1);
  return a;
}

// Box (y1,x1,y2,x2) of candidate row `r` (25 floats) at cell c.
__device__ __forceinline__ float4 decode_box(const odt_tail_params& p, const Cell& c,
                                             const float* __restrict__ r) {
  const odt_level& L = p.level[c.lvl];
  float4 o;
  if (p.kind == ODT_DECODE_SSD) {
    // ref SSD300.py:323-343 (anchors), :167-171 (decode); RetinaNet.py:328-355,:234-238
    const Anchor an = anchor_ssd(p, c);
    const float ay = an.cy, ax = an.cx, ah = an.h, aw = an.w;
    float ty = r[21], tx = r[22], th = r[23], tw = r[24];
    float dy = __fadd_rn(__fmul_rn(ty, ah), ay);
    float dx = __fadd_rn(__fmul_rn(tx, aw), ax);
    float dh = __fmul_rn(ah, expf(th));
    float dw = __fmul_rn(aw, expf(tw));
    float h2 = __fmul_rn(dh, 0.5f), w2 = __fmul_rn(dw, 0.5f);
    o.x = __fsub_rn(dy, h2);
    o.y = __fsub_rn(dx, w2);
    o.z = __fadd_rn(dy, h2);
    o.w = __fadd_rn(dx, w2);
  } else if (p.kind == ODT_DECODE_YOLO3) {
    // ref YOLOv3.py:419-433 (priors), :340-348 (additive exp, x stride multiplier)
    float ay = (float)c.y + 0.5f, ax = (float)c.x + 0.5f;
    float by = __fadd_rn(ay, sigmoid_rn(r[20]));
    float bx = __fadd_rn(ax, sigmoid_rn(r[21]));
    float bh = __fadd_rn(L.prior_h[c.a], expf(r[22]));
    float bw = __fadd_rn(L.prior_w[c.a], expf(r[23]));
    float h2 = __fmul_rn(bh, 0.5f), w2 = __fmul_rn(bw, 0.5f);
    o.x = __fmul_rn(__fsub_rn(by, h2), L.out_mul);
    o.y = __fmul_rn(__fsub_rn(bx, w2), L.out_mul);
    o.z = __fmul_rn(__fadd_rn(by, h2), L.out_mul);
    o.w = __fmul_rn(__fadd_rn(bx, w2), L.out_mul);
  } else {
    // FCOS: ref FCOS.py:130-150 (grid, no +0.5), :363 (exp), :216-240
    float gy = (float)c.y, gx = (float)c.x;
    float l = expf(r[21]), rr = expf(r[22]), t = expf(r[23]), bb = expf(r[24]);
    o.x = __fmul_rn(__fsub_rn(gy, t), L.out_mul);
    o.y = __fmul_rn(__fsub_rn(gx, l), L.out_mul);
    o.z = __fmul_rn(__fadd_rn(gy, bb), L.out_mul);
    o.w = __fmul_rn(__fadd_rn(gx, rr), L.out_mul);
  }
  return o;
}

// TF NonMaxSuppressionV3 IoU, float32, no contraction (SURVEY App. A.8).
__device__ __forceinline__ float iou_tf(const float4& a, const float4& b) {
  float ymin_i = fminf(a.x, a.z), xmin_i = fminf(a.y, a.w);
  float ymax_i = fmaxf(a.x, a.z), xmax_i = fmaxf(a.y, a.w);
  float ymin_j = fminf(b.x, b.z), xmin_j = fminf(b.y, b.w);
  float ymax_j = fmaxf(b.x, b.z), xmax_j = fmaxf(b.y, b.w);
  float area_i = __fmul_rn(__fsub_rn(ymax_i, ymin_i), __fsub_rn(xmax_i, xmin_i));
  float area_j = __fmul_rn(__fsub_rn(ymax_j, ymin_j), __fsub_rn(xmax_j, xmin_j));
  if (area_i <= 0.f || area_j <= 0.f) return 0.f;
  float iy1 = fmaxf(ymin_i, ymin_j), ix1 = fmaxf(xmin_i, xmin_j);
  float iy2 = fminf(ymax_i, ymax_j), ix2 = fminf(xmax_i, xmax_j);
  float inter = __fmul_rn(fmaxf(__fsub_rn(iy2, iy1), 0.f), fmaxf(__fsub_rn(ix2, ix1), 0.f));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_i, area_j), inter));
}

}  // namespace odt
