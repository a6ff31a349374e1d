// Training-image augmentation: image_augmentor's pixel work as restated by odt_b200/tfrecord.py (augment_pixels),
// for a batch of uint8 RGB sources of any sizes, on the GPU.
//
//   A  augment_geometry_kernel: one thread per output pixel, all three channels.  Through the flips and the crop to a
//      canvas pixel, then the resize mode's sample of the source (or the canvas value), then brightness.  An image
//      whose contrast and rotation steps did not fire gets hue as well and is written to `out` directly; the others
//      go to a float32 HWC stage in the scratch.
//   B  augment_mean_kernel + augment_mean_merge_kernel: for the images whose contrast step fired, the per-channel
//      mean of the stage: each slice of kAugSlicePixels pixels sums in fp64 in a fixed order, the slices are merged
//      in slice order, and the mean is rounded once to fp32.  Deterministic, independent of the batch.
//   C  augment_finish_kernel: contrast, hue and the rotation's four-tap bilinear gather (each tap coloured before
//      it is interpolated, which is numpy's "whole image, then rotate" tap for tap; taps outside read 0), into the
//      output layout.
//
// Every value is the numpy expression's, bit for bit: explicitly rounded fp32 operations (no FMA contraction) and
// fp64 where numpy promotes (adjust_hue's int64 + float32 sums).  The sampling and colour functions are
// __host__ __device__ so that tests/native/augment_host.cu runs them on the CPU against numpy.
#include <math.h>

#include <vector>

#include "common.cuh"

namespace odt {

constexpr int kAugThreads = 256;
constexpr int kAugSlicePixels = 4096;  // pixels per fp64 partial sum of the contrast means

// odt_augment_params plus where its stage and mean partials live in the scratch (-1: none)
struct AugImage {
  odt_augment_params p;
  long long stage;    // float offset of the [oh, ow, 3] stage
  long long partial;  // double offset of the [slices, 3] partial sums
};

// Explicitly rounded arithmetic that also compiles for the host (where the harness build turns contraction off)
#ifdef __CUDA_ARCH__
#define ODT_AUG_OP(name, T, dev, op) \
  __host__ __device__ inline T name(T a, T b) { return dev(a, b); }
#else
#define ODT_AUG_OP(name, T, dev, op) \
  __host__ __device__ inline T name(T a, T b) { return a op b; }
#endif
ODT_AUG_OP(f_add, float, __fadd_rn, +)
ODT_AUG_OP(f_sub, float, __fsub_rn, -)
ODT_AUG_OP(f_mul, float, __fmul_rn, *)
ODT_AUG_OP(f_div, float, __fdiv_rn, /)
ODT_AUG_OP(d_add, double, __dadd_rn, +)
ODT_AUG_OP(d_sub, double, __dsub_rn, -)
ODT_AUG_OP(d_mul, double, __dmul_rn, *)
ODT_AUG_OP(d_div, double, __ddiv_rn, /)
#undef ODT_AUG_OP

__host__ __device__ inline float aug_px(const uint8_t* s, int w, int y, int x, int c) {
  return (float)s[((long long)y * w + x) * 3 + c];
}

// float32(a / b) of two ints through a double division, as np.float32(a / b) rounds Python's quotient
__host__ __device__ inline float aug_ratio(int a, int b) { return (float)((double)a / (double)b); }

// align_corners scale of a resize from n_in to n_out: np.float32((in - 1) / (out - 1)), 0 for out == 1
__host__ __device__ inline float aug_aligned_scale(int n_in, int n_out) {
  return n_out > 1 ? aug_ratio(n_in - 1, n_out - 1) : 0.f;
}

// _resize_bilinear_aligned at (y, x) of an rh x rw resize
__host__ __device__ inline void aug_bilinear(const uint8_t* s, int h, int w, int rh, int rw, int y, int x, float* v) {
  const float ys = f_mul((float)y, aug_aligned_scale(h, rh)), xs = f_mul((float)x, aug_aligned_scale(w, rw));
  const float fy = floorf(ys), fx = floorf(xs);
  const float wy = f_sub(ys, fy), wx = f_sub(xs, fx);
  const int y0 = min((int)fy, h - 1), x0 = min((int)fx, w - 1);
  const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  const float ux = f_sub(1.f, wx), uy = f_sub(1.f, wy);
  for (int c = 0; c < 3; ++c) {
    const float top = f_add(f_mul(aug_px(s, w, y0, x0, c), ux), f_mul(aug_px(s, w, y0, x1, c), wx));
    const float bot = f_add(f_mul(aug_px(s, w, y1, x0, c), ux), f_mul(aug_px(s, w, y1, x1, c), wx));
    v[c] = f_add(f_mul(top, uy), f_mul(bot, wy));
  }
}

// _resize_nearest_aligned: min(floor(dst * scale + 0.5), in - 1)
__host__ __device__ inline void aug_nearest(const uint8_t* s, int h, int w, int rh, int rw, int y, int x, float* v) {
  const int sy = min((int)floorf(f_add(f_mul((float)y, aug_aligned_scale(h, rh)), 0.5f)), h - 1);
  const int sx = min((int)floorf(f_add(f_mul((float)x, aug_aligned_scale(w, rw)), 0.5f)), w - 1);
  for (int c = 0; c < 3; ++c) v[c] = aug_px(s, w, sy, sx, c);
}

// _resize_bilinear_legacy (TF1 resize, no align_corners, no half-pixel centres): src = dst * in / out
__host__ __device__ inline void aug_legacy(const uint8_t* s, int h, int w, int oh, int ow, int y, int x, float* v) {
  const float ys = f_mul((float)y, aug_ratio(h, oh)), xs = f_mul((float)x, aug_ratio(w, ow));
  const int y0 = min((int)floorf(ys), h - 1), x0 = min((int)floorf(xs), w - 1);
  const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  const float wy = f_sub(ys, (float)y0), wx = f_sub(xs, (float)x0);
  const float ux = f_sub(1.f, wx), uy = f_sub(1.f, wy);
  for (int c = 0; c < 3; ++c) {
    const float top = f_add(f_mul(aug_px(s, w, y0, x0, c), ux), f_mul(aug_px(s, w, y0, x1, c), wx));
    const float bot = f_add(f_mul(aug_px(s, w, y1, x0, c), ux), f_mul(aug_px(s, w, y1, x1, c), wx));
    v[c] = f_add(f_mul(top, uy), f_mul(bot, wy));
  }
}

// TF's ResizeBicubic table (_bicubic_table): entry [i*2] (even) and [i*2+1] (odd) for x = i / 1024, A = -0.75
__host__ __device__ inline float aug_cubic_near(int i) {
  const float x = f_mul((float)i, 1.f / 1024.f);
  return f_add(f_mul(f_mul(f_sub(f_mul(1.25f, x), 2.25f), x), x), 1.f);
}
__host__ __device__ inline float aug_cubic_far(int i) {
  const float x1 = f_add(f_mul((float)i, 1.f / 1024.f), 1.f);
  const float t = f_add(f_mul(f_sub(f_mul(-0.75f, x1), -3.75f), x1), -6.f);
  return f_sub(f_mul(t, x1), -3.f);
}

// _bicubic_axis at output coordinate d: four clamped source indices and their table weights
__host__ __device__ inline void aug_cubic_axis(int n_in, int n_out, int d, int* idx, float* wt) {
  const float loc = f_mul((float)d, aug_aligned_scale(n_in, n_out));
  const float fl = floorf(loc);
  const int off = (int)rintf(f_mul(f_sub(loc, fl), 1024.f));
  const int base = (int)fl;
  wt[0] = aug_cubic_far(off);
  wt[1] = aug_cubic_near(off);
  wt[2] = aug_cubic_near(1024 - off);
  wt[3] = aug_cubic_far(1024 - off);
  for (int k = 0; k < 4; ++k) idx[k] = min(max(base - 1 + k, 0), n_in - 1);
}

// _resize_bicubic_aligned: along x first, then y; the four taps summed left to right from 0 like Python's sum
__host__ __device__ inline void aug_bicubic(const uint8_t* s, int h, int w, int rh, int rw, int y, int x, float* v) {
  int yi[4], xi[4];
  float yw[4], xw[4];
  aug_cubic_axis(h, rh, y, yi, yw);
  aug_cubic_axis(w, rw, x, xi, xw);
  for (int c = 0; c < 3; ++c) {
    float acc = 0.f;
    for (int j = 0; j < 4; ++j) {
      float row = 0.f;
      for (int k = 0; k < 4; ++k) row = f_add(row, f_mul(aug_px(s, w, yi[j], xi[k], c), xw[k]));
      acc = f_add(acc, f_mul(row, yw[j]));
    }
    v[c] = acc;
  }
}

// The pre-colour value of output pixel (y, x) of the oh x ow image (before rotation): flips, crop, canvas, resize
// mode.  `s` points at the image's source.
__host__ __device__ inline void aug_geometry(const odt_augment_params& p, const uint8_t* s, int y, int x, float* v) {
  if (p.mode == ODT_AUG_LEGACY) {
    aug_legacy(s, p.h, p.w, p.oh, p.ow, y, x, v);
    return;
  }
  const int zy = (p.flip_y ? p.oh - 1 - y : y) + p.crop_y, zx = (p.flip_x ? p.ow - 1 - x : x) + p.crop_x;
  if (zy >= p.rh || zx >= p.rw) {
    v[0] = v[1] = v[2] = p.cval;
  } else if (p.mode == ODT_AUG_PAD) {
    for (int c = 0; c < 3; ++c) v[c] = aug_px(s, p.w, zy, zx, c);
  } else if (p.mode == ODT_AUG_NEAREST) {
    aug_nearest(s, p.h, p.w, p.rh, p.rw, zy, zx, v);
  } else if (p.mode == ODT_AUG_BICUBIC) {
    aug_bicubic(s, p.h, p.w, p.rh, p.rw, zy, zx, v);
  } else {
    aug_bilinear(s, p.h, p.w, p.rh, p.rw, zy, zx, v);
  }
  if (p.brightness_on)
    for (int c = 0; c < 3; ++c) v[c] = f_add(v[c], p.brightness);
}

// adjust_hue on one pixel; hue6 = float32(delta) * 6.  The hexagon sector `cat` and its ties follow numpy's select;
// h = cat + ratio, frac = h - cat2 and mid = vmin + frac * range are float64 in numpy (int64 + float32) and here.
__host__ __device__ inline void aug_hue(float* v, float hue6) {
  const float r = v[0], g = v[1], b = v[2];
  const float vmax = fmaxf(fmaxf(r, g), b), vmin = fminf(fminf(r, g), b);
  const float range = f_sub(vmax, vmin);
  const float safe = range > 0.f ? range : 1.f;
  const int cat = (r < g && b < r) ? 1 : (r < g && b > g) ? 3 : (r < g) ? 2 : (b < g) ? 0 : (b > r) ? 4 : 5;
  const float vmid = f_sub(f_sub(f_add(f_add(r, g), b), vmax), vmin);
  const float ratio = f_div(f_sub(vmid, vmin), safe);
  float h = 0.f;
  if (range > 0.f) h = (float)d_add((double)cat, (double)(cat % 2 == 0 ? ratio : f_sub(1.f, ratio)));
  // np.mod(h + hue6, 6): fmod, then the divisor's sign (a zero remainder is +0)
  float m = fmodf(f_add(h, hue6), 6.f);
  if (m != 0.f) {
    if (m < 0.f) m = f_add(m, 6.f);
  } else {
    m = 0.f;
  }
  const int cat2 = min((int)m, 5);
  double frac = d_sub((double)m, (double)cat2);
  if (cat2 % 2) frac = d_sub(1.0, frac);
  const float mid = (float)d_add((double)vmin, d_mul(frac, (double)range));
  switch (cat2) {
    case 0: v[0] = vmax; v[1] = mid; v[2] = vmin; break;
    case 1: v[0] = mid; v[1] = vmax; v[2] = vmin; break;
    case 2: v[0] = vmin; v[1] = vmax; v[2] = mid; break;
    case 3: v[0] = vmin; v[1] = mid; v[2] = vmax; break;
    case 4: v[0] = mid; v[1] = vmin; v[2] = vmax; break;
    default: v[0] = vmax; v[1] = vmin; v[2] = mid; break;
  }
}

// adjust_contrast (with the given means) and adjust_hue, each where it fired
__host__ __device__ inline void aug_colour(const odt_augment_params& p, const float* mean, float* v) {
  if (p.contrast_on)
    for (int c = 0; c < 3; ++c) v[c] = f_add(f_mul(f_sub(v[c], mean[c]), p.contrast), mean[c]);
  if (p.hue_on) aug_hue(v, p.hue6);
}

// rotate_bilinear at output pixel (y, x); tap(yy, xx, v) yields the coloured value of an in-image pixel
template <typename Tap>
__host__ __device__ inline void aug_rotate(const odt_augment_params& p, int y, int x, Tap tap, float* v) {
  const float sx = f_add(f_sub(f_mul(p.rot_c, (float)x), f_mul(p.rot_s, (float)y)), p.rot_x_off);
  const float sy = f_add(f_add(f_mul(p.rot_s, (float)x), f_mul(p.rot_c, (float)y)), p.rot_y_off);
  const float fx = floorf(sx), fy = floorf(sy);
  const float wx = f_sub(sx, fx), wy = f_sub(sy, fy);
  const float ux = f_sub(1.f, wx), uy = f_sub(1.f, wy);
  const int x0 = (int)fx, y0 = (int)fy;
  float t[4][3];
  for (int k = 0; k < 4; ++k) {
    const int yy = y0 + (k >> 1), xx = x0 + (k & 1);
    if (yy >= 0 && yy < p.oh && xx >= 0 && xx < p.ow) {
      tap(yy, xx, t[k]);
    } else {
      t[k][0] = t[k][1] = t[k][2] = 0.f;
    }
  }
  for (int c = 0; c < 3; ++c) {
    const float top = f_add(f_mul(t[0][c], ux), f_mul(t[1][c], wx));
    const float bot = f_add(f_mul(t[2][c], ux), f_mul(t[3][c], wx));
    v[c] = f_add(f_mul(top, uy), f_mul(bot, wy));
  }
}

__host__ __device__ inline bool aug_staged(const odt_augment_params& p) { return p.contrast_on || p.rotate_on; }

__host__ __device__ inline void aug_store(const odt_augment_params& p, float* out, int b, int y, int x,
                                          const float* v) {
  const long long hw = (long long)p.oh * p.ow, pix = (long long)y * p.ow + x;
  float* o = out + (long long)b * hw * 3;
  if (p.layout == ODT_AUG_NCHW) {
    for (int c = 0; c < 3; ++c) o[c * hw + pix] = v[c];
  } else {
    for (int c = 0; c < 3; ++c) o[pix * 3 + c] = v[c];
  }
}

__global__ void __launch_bounds__(kAugThreads)
    augment_geometry_kernel(const uint8_t* __restrict__ src, const AugImage* __restrict__ imgs, float* out,
                            float* stage) {
  pdl_launch_dependents();
  const AugImage& im = imgs[blockIdx.y];
  const odt_augment_params& p = im.p;
  const long long pix = (long long)blockIdx.x * kAugThreads + threadIdx.x;
  if (pix >= (long long)p.oh * p.ow) return;
  const int y = (int)(pix / p.ow), x = (int)(pix % p.ow);
  float v[3];
  aug_geometry(p, src + p.src_offset, y, x, v);
  if (aug_staged(p)) {
    float* s = stage + im.stage + pix * 3;
    s[0] = v[0];
    s[1] = v[1];
    s[2] = v[2];
    return;
  }
  if (p.hue_on) aug_hue(v, p.hue6);
  aug_store(p, out, blockIdx.y, y, x, v);
}

// one CTA per (slice, image): the slice's per-channel fp64 sum, thread order fixed, then a fixed tree
__global__ void __launch_bounds__(kAugThreads)
    augment_mean_kernel(const AugImage* __restrict__ imgs, const float* __restrict__ stage, double* partial) {
  pdl_launch_dependents();
  __shared__ double s_sum[3][kAugThreads];
  const AugImage& im = imgs[blockIdx.y];
  const long long hw = (long long)im.p.oh * im.p.ow;
  const long long p0 = (long long)blockIdx.x * kAugSlicePixels;
  if (!im.p.contrast_on || p0 >= hw) return;
  const long long p1 = min(hw, p0 + kAugSlicePixels);
  double acc[3] = {0.0, 0.0, 0.0};
  const float* s = stage + im.stage;
  for (long long q = p0 + threadIdx.x; q < p1; q += kAugThreads)
    for (int c = 0; c < 3; ++c) acc[c] = d_add(acc[c], (double)s[q * 3 + c]);
  for (int c = 0; c < 3; ++c) s_sum[c][threadIdx.x] = acc[c];
  __syncthreads();
  for (int n = kAugThreads / 2; n > 0; n >>= 1) {
    if (threadIdx.x < n)
      for (int c = 0; c < 3; ++c) s_sum[c][threadIdx.x] = d_add(s_sum[c][threadIdx.x], s_sum[c][threadIdx.x + n]);
    __syncthreads();
  }
  if (threadIdx.x < 3) partial[im.partial + blockIdx.x * 3 + threadIdx.x] = s_sum[threadIdx.x][0];
}

// one thread per (image, channel): the slices merged in slice order, / (oh * ow) in fp64, rounded once.
// means_out rows of images without contrast are NaN.
__global__ void __launch_bounds__(kAugThreads)
    augment_mean_merge_kernel(const AugImage* __restrict__ imgs, int B, const double* __restrict__ partial,
                              float* means, float* means_out) {
  pdl_launch_dependents();
  const int i = blockIdx.x * kAugThreads + threadIdx.x;
  if (i >= B * 3) return;
  const AugImage& im = imgs[i / 3];
  float m = nanf("");
  if (im.p.contrast_on) {
    const long long hw = (long long)im.p.oh * im.p.ow;
    const int slices = (int)((hw + kAugSlicePixels - 1) / kAugSlicePixels);
    double sum = 0.0;
    for (int k = 0; k < slices; ++k) sum = d_add(sum, partial[im.partial + k * 3 + i % 3]);
    m = (float)d_div(sum, (double)hw);
  }
  means[i] = m;
  if (means_out) means_out[i] = m;
}

__global__ void __launch_bounds__(kAugThreads)
    augment_finish_kernel(const AugImage* __restrict__ imgs, const float* __restrict__ stage,
                          const float* __restrict__ means, float* out) {
  pdl_launch_dependents();
  const AugImage& im = imgs[blockIdx.y];
  const odt_augment_params& p = im.p;
  const long long pix = (long long)blockIdx.x * kAugThreads + threadIdx.x;
  if (!aug_staged(p) || pix >= (long long)p.oh * p.ow) return;
  const int y = (int)(pix / p.ow), x = (int)(pix % p.ow);
  const float* s = stage + im.stage;
  float mean[3] = {0.f, 0.f, 0.f};
  if (p.contrast_on)
    for (int c = 0; c < 3; ++c) mean[c] = means[blockIdx.y * 3 + c];
  float v[3];
  if (p.rotate_on) {
    aug_rotate(p, y, x,
               [&](int yy, int xx, float* t) {
                 const float* q = s + ((long long)yy * p.ow + xx) * 3;
                 t[0] = q[0];
                 t[1] = q[1];
                 t[2] = q[2];
                 aug_colour(p, mean, t);
               },
               v);
  } else {
    v[0] = s[pix * 3];
    v[1] = s[pix * 3 + 1];
    v[2] = s[pix * 3 + 2];
    aug_colour(p, mean, v);
  }
  aug_store(p, out, blockIdx.y, y, x, v);
}

// scratch layout: [AugImage x B] | stages (float) | partial sums (double) | means (float [B, 3]), each 256-aligned
struct AugLayout {
  long long imgs, stage, partial, means, total;
  long long stage_floats, partial_doubles;
};

static long long aug_align(long long n) { return (n + 255) / 256 * 256; }

static AugLayout aug_layout(const odt_augment_params* p, int B, AugImage* fill) {
  AugLayout L = {};
  for (int b = 0; b < B; ++b) {
    const long long hw = (long long)p[b].oh * p[b].ow;
    if (fill) {
      fill[b].p = p[b];
      fill[b].stage = aug_staged(p[b]) ? L.stage_floats : -1;
      fill[b].partial = p[b].contrast_on ? L.partial_doubles : -1;
    }
    if (aug_staged(p[b])) L.stage_floats += hw * 3;
    if (p[b].contrast_on) L.partial_doubles += (hw + kAugSlicePixels - 1) / kAugSlicePixels * 3;
  }
  L.imgs = 0;
  L.stage = aug_align((long long)B * sizeof(AugImage));
  L.partial = L.stage + aug_align(L.stage_floats * 4);
  L.means = L.partial + aug_align(L.partial_doubles * 8);
  L.total = L.means + aug_align((long long)B * 3 * 4);
  return L;
}

static bool aug_flag(int f) { return f == 0 || f == 1; }

// every check of odt_augment_batch on the host-side parameters; the message names the image and the field
static int aug_check(const odt_augment_params* params, int B) {
  ODT_CHECK_ARG(params, "null params_host");
  ODT_CHECK_ARG(B >= 1 && B <= 65535, "B must be in [1, 65535]");
  for (int b = 0; b < B; ++b) {
    const odt_augment_params& p = params[b];
    const bool ok_size = p.h >= 1 && p.w >= 1 && p.oh >= 1 && p.ow >= 1 && p.zh >= 1 && p.zw >= 1 &&
                         (long long)p.oh * p.ow <= (1LL << 28) && (long long)p.h * p.w <= (1LL << 28);
    if (!ok_size) {
      set_error("odt_augment_batch: invalid argument: image %d: sizes must be >= 1 (and below 2^28 pixels)", b);
      return ODT_ERR_INVALID;
    }
    if (p.oh != params[0].oh || p.ow != params[0].ow || p.layout != params[0].layout) {
      set_error("odt_augment_batch: invalid argument: image %d: output size and layout differ from image 0's", b);
      return ODT_ERR_INVALID;
    }
    const bool ok_mode = p.mode >= ODT_AUG_BILINEAR && p.mode <= ODT_AUG_LEGACY &&
                         (p.layout == ODT_AUG_NHWC || p.layout == ODT_AUG_NCHW) && p.src_offset >= 0;
    const bool ok_flags = aug_flag(p.flip_y) && aug_flag(p.flip_x) && aug_flag(p.brightness_on) &&
                          aug_flag(p.contrast_on) && aug_flag(p.hue_on) && aug_flag(p.rotate_on);
    const bool ok_rect = p.rh >= 0 && p.rh <= p.zh && p.rw >= 0 && p.rw <= p.zw &&
                         (p.mode != ODT_AUG_PAD || (p.rh == min(p.h, p.zh) && p.rw == min(p.w, p.zw)));
    const bool ok_crop = p.crop_y >= 0 && p.crop_x >= 0 && p.crop_y + p.oh <= p.zh && p.crop_x + p.ow <= p.zw;
    const bool ok_legacy = p.mode != ODT_AUG_LEGACY ||
                           (p.zh == p.oh && p.zw == p.ow && p.crop_y == 0 && p.crop_x == 0 && !p.flip_y && !p.flip_x &&
                            !p.brightness_on && !p.contrast_on && !p.hue_on && !p.rotate_on);
    if (!(ok_mode && ok_flags && ok_rect && ok_crop && ok_legacy)) {
      set_error("odt_augment_batch: invalid argument: image %d: %s", b,
                !ok_mode    ? "mode, layout or src_offset out of range"
                : !ok_flags ? "a flag is not 0 or 1"
                : !ok_rect  ? "the inner rectangle does not fit the canvas (or the pad mode's is not min(src, canvas))"
                : !ok_crop  ? "the crop window leaves the canvas"
                            : "the legacy mode takes no canvas, crop, flip, jitter or rotation");
      return ODT_ERR_INVALID;
    }
  }
  return ODT_OK;
}

}  // namespace odt

using namespace odt;

extern "C" long long odt_augment_scratch_bytes(const odt_augment_params* params_host, int B) {
  if (aug_check(params_host, B) != ODT_OK) return -1;
  return aug_layout(params_host, B, nullptr).total;
}

extern "C" int odt_augment_batch(const uint8_t* src, const odt_augment_params* params_host, int B, float* out,
                                 float* means_out, void* scratch, void* stream) {
  ODT_CHECK_ARG(src && out && scratch, "null pointer");
  const int rc = aug_check(params_host, B);
  if (rc != ODT_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<AugImage> host(B);
  const AugLayout L = aug_layout(params_host, B, host.data());
  char* base = static_cast<char*>(scratch);
  AugImage* imgs = reinterpret_cast<AugImage*>(base + L.imgs);
  float* stage = reinterpret_cast<float*>(base + L.stage);
  double* partial = reinterpret_cast<double*>(base + L.partial);
  float* means = reinterpret_cast<float*>(base + L.means);
  // pageable source: the copy has taken the bytes when it returns
  ODT_CUDA_OK(cudaMemcpyAsync(imgs, host.data(), sizeof(AugImage) * B, cudaMemcpyHostToDevice, st));
  const odt_augment_params& p0 = params_host[0];
  const long long hw = (long long)p0.oh * p0.ow;
  bool any_contrast = false, any_staged = false;
  for (int b = 0; b < B; ++b) {
    any_contrast |= params_host[b].contrast_on != 0;
    any_staged |= aug_staged(params_host[b]);
  }
  const dim3 grid((unsigned)((hw + kAugThreads - 1) / kAugThreads), (unsigned)B);
  augment_geometry_kernel<<<grid, kAugThreads, 0, st>>>(src, imgs, out, stage);
  ODT_LAUNCH_OK();
  if (any_contrast) {
    const dim3 sgrid((unsigned)((hw + kAugSlicePixels - 1) / kAugSlicePixels), (unsigned)B);
    augment_mean_kernel<<<sgrid, kAugThreads, 0, st>>>(imgs, stage, partial);
    ODT_LAUNCH_OK();
  }
  if (any_contrast || means_out) {
    augment_mean_merge_kernel<<<ceil_div(B * 3, kAugThreads), kAugThreads, 0, st>>>(imgs, B, partial, means,
                                                                                     means_out);
    ODT_LAUNCH_OK();
  }
  if (any_staged) {
    augment_finish_kernel<<<grid, kAugThreads, 0, st>>>(imgs, stage, means, out);
    ODT_LAUNCH_OK();
  }
  return ODT_OK;
}
