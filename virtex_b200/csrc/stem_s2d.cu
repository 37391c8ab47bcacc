// The 7x7 / stride-2 / pad-3 stem convolution as a 4-tap implicit GEMM over a space-to-depth (s2d) view of the image
// (the im2col route of backbone.cu remains only for image sizes whose stem output is not
// tiled exactly by the 16 x 8 TMA boxes).
//
//   S[n, i, j, (r*2+q)*3 + c] = x[n, c, 2i + r - 3, 2j + q - 3]      (zero outside the image, channels 12..15 zero)
//   y[n, oh, ow, o] = sum_{a<4} sum_{b<4} sum_{ch<16} S[n, oh + a, ow + b, ch] * Wp[o, a*64 + b*16 + ch]
//   Wp[o, a*64 + b*16 + (r*2+q)*3 + c] = w[o, c, 2a + r, 2b + q]      (zero where 2a + r = 7 or 2b + q = 7)
//
// The four pixels (ow .. ow+3) x 16 channels of a tap row are 64 CONTIGUOUS bf16 in S, so the A operand of k-block `a`
// is one 4-D TMA box of a tensor map whose W stride is a single pixel (overlapping rows): vtx_gemm conv_mode 5 / 6.
// HBM traffic: 154 MB (fp32 image) + 2 x 108 MB (S write, read) instead of 1 GB written + 1 GB read for the im2col
// matrix (and once more in the wgrad).  Replaces torchvision resnet.py:197 `self.conv1` fwd / wgrad on this path.
#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {

// one CTA per (n, i): the two image rows 2i-3, 2i-2 of the three channels are staged in shared memory
__global__ void __launch_bounds__(256) stem_s2d_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ S, int N,
                                                      int H, int W, int Hs, int Ws) {
  VTX_PDL_TRIGGER();
  extern __shared__ float tile[];  // [3][2][Wp], Wp = W + 8: image column x lives at tile column x + 4
  const int Wp = W + 8;
  const int n = blockIdx.x / Hs, i = blockIdx.x % Hs;
  const int quads = Wp / 4;
  for (int e = threadIdx.x; e < 6 * quads; e += blockDim.x) {
    const int cr = e / quads, qd = e % quads;
    const int c = cr >> 1, r = cr & 1;
    const int h = 2 * i + r - 3;
    const int w0 = qd * 4 - 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (h >= 0 && h < H && w0 >= 0 && w0 + 3 < W)
      v = *reinterpret_cast<const float4*>(img + (((long long)n * 3 + c) * H + h) * W + w0);
    *reinterpret_cast<float4*>(tile + cr * Wp + qd * 4) = v;
  }
  __syncthreads();
  __nv_bfloat16* row = S + ((long long)n * Hs + i) * Ws * 16;
  for (int e = threadIdx.x; e < Ws * 2; e += blockDim.x) {
    const int j = e >> 1, half = e & 1;
    float v[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int ch = half * 8 + t;
      float f = 0.f;
      if (ch < 12) {
        const int rq = ch / 3, c = ch - rq * 3;
        const int r = rq >> 1, q = rq & 1;
        f = tile[(c * 2 + r) * Wp + 2 * j + q + 1];  // image column 2j + q - 3  ->  tile column 2j + q + 1
      }
      v[t] = f;
    }
    *reinterpret_cast<bf16x8*>(row + j * 16 + half * 8) = pack8(v);
  }
}

__global__ void stem_w_pack_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ wp, int O) {
  VTX_PDL_TRIGGER();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= O * 256) return;
  const int o = t >> 8, k = t & 255;
  const int a = k >> 6, b = (k >> 4) & 3, ch = k & 15;
  float f = 0.f;
  if (ch < 12) {
    const int rq = ch / 3, c = ch - rq * 3;
    const int kh = 2 * a + (rq >> 1), kw = 2 * b + (rq & 1);
    if (kh < 7 && kw < 7) f = w[((o * 3 + c) * 7 + kh) * 7 + kw];
  }
  wp[t] = __float2bfloat16(f);
}

__global__ void stem_w_unpack_add_kernel(const float* __restrict__ dwp, float* __restrict__ grad, int O) {
  VTX_PDL_TRIGGER();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= O * 147) return;
  const int kw = t % 7, kh = (t / 7) % 7, c = (t / 49) % 3, o = t / 147;
  const int k = (kh >> 1) * 64 + (kw >> 1) * 16 + ((kh & 1) * 2 + (kw & 1)) * 3 + c;
  grad[t] += dwp[o * 256 + k];
}

}  // namespace vtx

using namespace vtx;

#define STREAM reinterpret_cast<cudaStream_t>(stream)

extern "C" int vtx_stem_s2d(const float* img, void* S, int N, int H, int W, void* stream) {
  if (!img || !S || N <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 3))
    return set_error(VTX_EINVAL, "vtx_stem_s2d: bad arguments (H must be even, W a multiple of 4)");
  const size_t smem = (size_t)6 * (W + 8) * sizeof(float);
  if (smem > 48 * 1024) return set_error(VTX_EINVAL, "vtx_stem_s2d: image too wide");
  const int Hs = H / 2 + 3, Ws = W / 2 + 3;
  stem_s2d_kernel<<<N * Hs, 256, smem, STREAM>>>(img, (__nv_bfloat16*)S, N, H, W, Hs, Ws);
  return check_launch("stem_s2d");
}
extern "C" int vtx_stem_s2d_w_pack(const float* w, void* wp, int O, void* stream) {
  if (!w || !wp || O <= 0) return set_error(VTX_EINVAL, "vtx_stem_s2d_w_pack: bad arguments");
  stem_w_pack_kernel<<<(O * 256 + 255) / 256, 256, 0, STREAM>>>(w, (__nv_bfloat16*)wp, O);
  return check_launch("stem_w_pack");
}
extern "C" int vtx_stem_s2d_w_unpack_add(const float* dwp, float* grad, int O, void* stream) {
  if (!dwp || !grad || O <= 0) return set_error(VTX_EINVAL, "vtx_stem_s2d_w_unpack_add: bad arguments");
  stem_w_unpack_add_kernel<<<(O * 147 + 255) / 256, 256, 0, STREAM>>>(dwp, grad, O);
  return check_launch("stem_w_unpack_add");
}
