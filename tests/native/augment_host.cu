// TEST-ONLY: runs the per-pixel functions of csrc/augment.cu (aug_geometry, aug_hue, aug_colour, aug_rotate,
// aug_store: __host__ __device__) on the CPU, so that tests/test_augment.py can compare the kernels' sampling and
// colour arithmetic with numpy's augment_pixels bit for bit without a GPU.  Built by that test into
// tests/native/_build/; never linked into libodt_b200.so (the product has no host path).
#include <stdarg.h>

#include <vector>

#include "../../object-detection-tensorflow_b200/csrc/augment.cu"

namespace odt {
void set_error(const char*, ...) {}
}  // namespace odt

// One image, host pointers: stage A for every pixel, then (where contrast or rotation fired) stage C with the given
// contrast means, as the kernels chain them.  out: the output layout of p.
extern "C" int odt_test_augment_host(const uint8_t* src, const odt_augment_params* p, const float* mean, float* out) {
  using namespace odt;
  const int oh = p->oh, ow = p->ow;
  std::vector<float> stage((size_t)oh * ow * 3);
  for (int y = 0; y < oh; ++y)
    for (int x = 0; x < ow; ++x) {
      float v[3];
      aug_geometry(*p, src + p->src_offset, y, x, v);
      if (aug_staged(*p)) {
        for (int c = 0; c < 3; ++c) stage[((size_t)y * ow + x) * 3 + c] = v[c];
      } else {
        if (p->hue_on) aug_hue(v, p->hue6);
        aug_store(*p, out, 0, y, x, v);
      }
    }
  if (!aug_staged(*p)) return 0;
  for (int y = 0; y < oh; ++y)
    for (int x = 0; x < ow; ++x) {
      float v[3];
      if (p->rotate_on) {
        aug_rotate(*p, y, x,
                   [&](int yy, int xx, float* t) {
                     for (int c = 0; c < 3; ++c) t[c] = stage[((size_t)yy * ow + xx) * 3 + c];
                     aug_colour(*p, mean, t);
                   },
                   v);
      } else {
        for (int c = 0; c < 3; ++c) v[c] = stage[((size_t)y * ow + x) * 3 + c];
        aug_colour(*p, mean, v);
      }
      aug_store(*p, out, 0, y, x, v);
    }
  return 0;
}

// adjust_hue of n RGB float pixels (in place)
extern "C" void odt_test_augment_hue(float* rgb, long long n, float hue6) {
  for (long long i = 0; i < n; ++i) odt::aug_hue(rgb + i * 3, hue6);
}
