// TEST-ONLY: runs the fp16 vector step of csrc/epilogue.cuh (epi_store_f16, the fused output of conv_tc, conv_tapn,
// conv_thin and conv_pw) and its scalar form (epi_store_one, conv_direct) on the CPU over the same inputs, so that
// tests/test_epilogue_host.py can compare them bit for bit.  Built by that test into tests/native/_build/; never
// linked into libodt_b200.so.
#include <vector>

#include "../../object-detection-tensorflow_b200/csrc/epilogue.cuh"

// acc: [B][OH*OW][cpad] fp32, cpad a multiple of 8*nv.  For every pixel and every run of 8*nv channels below cpad:
//   vec != 0: epi_store_f16<nv> with the parameters staged by epi_param (rows of cpad floats) and the residual
//             sectors read at out0's offset, as the kernels do;
//   vec == 0: epi_store_one<__half> channel by channel, with the identity parameters (no pointers) at channels at or
//             past Cout, which is what epi_param stages there.
extern "C" int odt_test_epilogue_host(const odt_conv_params* p, const float* acc, int cpad, int nv, int vec) {
  using namespace odt;
  if ((nv != 1 && nv != 4) || cpad % (8 * nv) != 0) return ODT_ERR_INVALID;
  const Epi e = make_epi(*p);
  std::vector<float> raw((size_t)6 * cpad + 4);
  float* par = reinterpret_cast<float*>(((uintptr_t)raw.data() + 15) & ~(uintptr_t)15);  // 16-byte aligned rows
  for (int i = 0; i < 6 * cpad; ++i) par[i] = epi_param(e, i / cpad, i % cpad);
  const int hw = p->OH * p->OW;
  for (int b = 0; b < p->B; ++b) {
    for (int pix = 0; pix < hw; ++pix) {
      const float* a = acc + ((long long)b * hw + pix) * cpad;
      const long long o0 = (long long)b * e.out0_img_stride + (long long)pix * e.out0_pix_stride;
      const long long o1 = aux_row(e.out1_img_stride, e.out1_pix_stride, e.out1_halo, e.OW, b, pix);
      const long long o2 = aux_row(e.out2_img_stride, e.out2_pix_stride, e.out2_halo, e.OW, b, pix);
      for (int nb = 0; nb < cpad; nb += 8 * nv) {
        if (vec) {
          float v[32];
          for (int i = 0; i < 8 * nv; ++i) v[i] = a[nb + i];
          const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(e.residual) + o0 + nb);
          auto res = [&](int q) { return rp[q]; };
          if (nv == 1)
            epi_store_f16<1>(e, v, par + nb, cpad, res, o0 + nb, o1 + nb, o2 + nb);
          else
            epi_store_f16<4>(e, v, par + nb, cpad, res, o0 + nb, o1 + nb, o2 + nb);
        } else {
          for (int n = nb; n < nb + 8 * nv; ++n) {
            Epi es = e;
            if (n >= e.Cout) es.scale = es.shift = es.scale2 = es.shift2 = es.scale3 = es.shift3 = nullptr;
            epi_store_one<__half>(es, b, pix, n, a[n]);
          }
        }
      }
    }
  }
  return ODT_OK;
}
