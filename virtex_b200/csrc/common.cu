// Error handling + device queries shared by all translation units of libvirtex_b200.so
#include <stdarg.h>
#include <stdio.h>
#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {
static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(VTX_ECUDA, "%s: %s", what, cudaGetErrorString(e));
  return VTX_OK;
}
}  // namespace vtx

extern "C" const char* vtx_last_error(void) { return vtx::g_err; }
extern "C" int vtx_version(void) { return 200; }
/* sizeof(VtxGemm) as this library was compiled: bindings check their own struct against it */
extern "C" int vtx_sizeof_gemm(void) { return (int)sizeof(VtxGemm); }
extern "C" int vtx_num_sms(void) {
  static int sms[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (sms[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    sms[dev] = v;
  }
  return sms[dev];
}
