// TEST-ONLY: runs the per-lane phases of csrc/conv_pw.cu (pw_fill / pw_rows / pw_load / pw_compute / pw_store,
// all __host__ __device__) on the CPU -- block by block, warp by warp, group by group, each phase for all 32 lanes
// before the next one starts (= the kernel's __syncwarp), on a heap buffer carved exactly like the kernel's shared
// memory -- so that tests/test_pw_host.py can check staging indices, the group round-robin, the rounding chain and
// the epilogue against the oracle without a GPU.  Built by that test into tests/native/_build/; never linked into
// libodt_b200.so (the product has no host path).
#include <vector>

#include "../../object-detection-tensorflow_b200/csrc/conv_pw.cu"

namespace odt {
int pw_mode() { return 2; }
void set_error(const char*, ...) {}

template <int COT>
static void run_pw_host(const void* in, const void* weights, const PwGeom& g, const Epi& e) {
  std::vector<unsigned char> raw((size_t)g.smem_bytes + 64, 0xCD);  // poison: reads of unwritten smem show up
  unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)raw.data() + 15) & ~(uintptr_t)15);
  const long long want = (g.groups + PW_WARPS - 1) / PW_WARPS;
  const int grid = (int)(want < 3 ? want : 3);  // a small persistent grid: every warp streams several groups
  const __half* inh = reinterpret_cast<const __half*>(in);
  const float* ws = reinterpret_cast<const float*>(base);
  const float* par = reinterpret_cast<const float*>(base + g.off_par);
  for (int blk = 0; blk < grid; ++blk) {
    for (int tid = 0; tid < PW_THREADS; ++tid) pw_fill(tid, base, reinterpret_cast<const __half*>(weights), g, e);
    for (int warp = 0; warp < PW_WARPS; ++warp) {
      const PwSlice s = pw_slice(base, g, warp);
      for (long long grp = (long long)warp * grid + blk; grp < g.groups; grp += (long long)grid * PW_WARPS) {
        for (int lane = 0; lane < 32; ++lane) pw_rows(lane, (int)grp, s, g, e);
        PwItems<COT> it[32];  // per-lane registers of the kernel
        for (int lane = 0; lane < 32; ++lane) pw_items<COT>(lane, 0, s, g, e, it[lane]);
        for (int lane = 0; lane < 32; ++lane) pw_load(lane, s, inh, g);
        for (int pass = 0; pass < g.passes; ++pass) {
          if (pass)
            for (int lane = 0; lane < 32; ++lane) pw_items<COT>(lane, pass, s, g, e, it[lane]);
          for (int lane = 0; lane < 32; ++lane) pw_compute<COT>(lane, pass, s, ws, g);
          for (int lane = 0; lane < 32; ++lane) pw_store<COT>(lane, pass, s, par, g, e, it[lane]);
        }
      }
    }
  }
}
}  // namespace odt

// host pointers everywhere; returns ODT_OK, or ODT_ERR_UNSUPPORTED exactly where conv_pw_try would decline
extern "C" int odt_test_pw_host(const void* in, const void* weights, const odt_conv_params* p, int force) {
  using namespace odt;
  PwGeom g;
  int cot;
  const int rc = pw_plan(in, p, force != 0, &g, &cot);
  if (rc) return rc;
  const Epi e = make_epi(*p);
  if (cot == 8) run_pw_host<8>(in, weights, g, e);
  else if (cot == 16) run_pw_host<16>(in, weights, g, e);
  else run_pw_host<32>(in, weights, g, e);
  return ODT_OK;
}

// the planner's shape for a layer (pixels per group, output-channel passes, shared-memory bytes per block)
extern "C" int odt_test_pw_plan(const void* in, const odt_conv_params* p, int force, int* pix, int* nsplit, int* smem) {
  using namespace odt;
  PwGeom g;
  int cot;
  const int rc = pw_plan(in, p, force != 0, &g, &cot);
  if (rc) return rc;
  *pix = 32;
  *nsplit = g.passes;
  *smem = g.smem_bytes;
  return ODT_OK;
}
