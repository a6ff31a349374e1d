// Error reporting and small host-side helpers of the C ABI.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace odt {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
static int conv_mode(const char* var) {
  const char* e = getenv(var);  // read every call: lets one process compare both paths
  return (e && e[0] >= '0' && e[0] <= '2') ? e[0] - '0' : 1;
}
int pw_mode() { return conv_mode("ODT_TC_PW"); }
int thin_mode() { return conv_mode("ODT_TC_THIN"); }
int tapn_mode() { return conv_mode("ODT_TC_TAPN"); }
int swap_mode() { return conv_mode("ODT_TC_SWAP"); }
int wide_mode() { return conv_mode("ODT_TC_WIDE"); }
}  // namespace odt

extern "C" int odt_abi_version(void) { return 5; }

// CRC-32C (Castagnoli, reflected 0x82F63B78) of a host buffer, continuing from `crc`
// (0 for a fresh sum): the checksum of TensorBundle index blocks and tensor payloads
// (tf.train.Saver V2 files read / written by odt_b200/tf_checkpoint.py).  Host-only utility.
extern "C" unsigned int odt_crc32c(unsigned int crc, const void* data, unsigned long long n) {
  static unsigned int table[8][256];
  static bool init = false;
  if (!init) {
    for (unsigned int i = 0; i < 256; ++i) {
      unsigned int c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ 0x82F63B78u : (c >> 1);
      table[0][i] = c;
    }
    for (unsigned int i = 0; i < 256; ++i)
      for (int t = 1; t < 8; ++t) table[t][i] = (table[t - 1][i] >> 8) ^ table[0][table[t - 1][i] & 0xFFu];
    init = true;
  }
  const unsigned char* p = static_cast<const unsigned char*>(data);
  unsigned int c = ~crc;
  while (n >= 8) {
    unsigned int lo, hi;
    memcpy(&lo, p, 4);
    memcpy(&hi, p + 4, 4);
    lo ^= c;
    c = table[7][lo & 0xFFu] ^ table[6][(lo >> 8) & 0xFFu] ^ table[5][(lo >> 16) & 0xFFu] ^ table[4][lo >> 24] ^
        table[3][hi & 0xFFu] ^ table[2][(hi >> 8) & 0xFFu] ^ table[1][(hi >> 16) & 0xFFu] ^ table[0][hi >> 24];
    p += 8;
    n -= 8;
  }
  while (n--) c = table[0][(c ^ *p++) & 0xFFu] ^ (c >> 8);
  return ~c;
}
extern "C" const char* odt_last_error(void) { return odt::g_err; }

// Debug only: name of the convolution kernel the last odt_conv2d_* call of this process launched.
extern "C" const char* odt_debug_last_conv_kernel(void) { return odt::g_last_conv_kernel; }

// TF SAME padding (SURVEY App. A.1): out = ceil(in/stride),
// pad_total = max((out-1)*stride + (k-1)*dil + 1 - in, 0), before = total/2.
extern "C" int odt_same_pad(int in, int k, int stride, int dil, int* out, int* pad_before,
                            int* pad_after) {
  ODT_CHECK_ARG(in > 0 && k > 0 && stride > 0 && dil > 0, "non-positive geometry");
  int o = (in + stride - 1) / stride;
  int total = (o - 1) * stride + (k - 1) * dil + 1 - in;
  if (total < 0) total = 0;
  if (out) *out = o;
  if (pad_before) *pad_before = total / 2;
  if (pad_after) *pad_after = total - total / 2;
  return ODT_OK;
}
