// Memory-bound kernels of the ResNet backbone (NHWC bf16 activations, fp32 statistics).
// They surround the wgmma GEMM (gemm_tc.cu): train-mode BatchNorm finalize/apply/backward, ReLU, residual add,
// stem im2col + fused BN/ReLU/max-pool, strided-conv gathers, and conv-weight layout transforms.
// Reference semantics: torchvision/models/resnet.py:143-163 (Bottleneck), :268-276 (stem), nn.BatchNorm2d train mode
// (SURVEY.md Appendix C.2): biased variance for normalisation, unbiased for running_var, momentum 0.1, eps 1e-5.
// All kernels are HBM-bound: 16-byte vector accesses along the contiguous channel dimension, grid-stride loops
// sized to a multiple of the SM count.
#include <algorithm>

#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {

static inline int grid_for(long long work_items, int threads, int per_sm = 16) {
  long long blocks = (work_items + threads - 1) / threads;
  long long cap = (long long)vtx_num_sms() * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// threads = (C/8) x the largest divisor of `extent` that keeps the block <= 256 threads: a row of `extent` positions is
// then walked in whole passes (56 pooled columns x 8 channel groups -> 224 threads, 2 passes, no idle tail)
static inline int row_threads(int cg, int extent) {
  int best = 1;
  for (int d = 1; d * cg <= 256 && d <= extent; ++d)
    if (extent % d == 0) best = d;
  return best * cg;
}

// ---------------------------------------------------------------------------------------------- stem im2col
// image fp32 NCHW [N,3,H,W] -> cols bf16 [N*Ho*Wo, ldc], k = (kh*7 + kw)*3 + c for the 7x7/stride 2/pad 3 stem,
// columns [147, ldc) zero.  One CTA per output row (n, ho): the 7 x 3 input rows it needs are staged in shared memory
// with coalesced float4 loads (scalar loads when W % 4 != 0, where image rows are not 16-byte aligned), then the
// ldc-wide column rows are written as coalesced 16-byte vectors.
__global__ void __launch_bounds__(256) stem_im2col_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ cols,
                                                         int N, int H, int W, int Ho, int Wo, int ldc) {
  VTX_PDL_TRIGGER();
  extern __shared__ float tile[];  // [3][7][Wp], Wp = W + 8 rounded up to 4: at least 4 zero columns on each side
  __shared__ int lut[160];         // k -> (c*7 + kh)*Wp + kw  or -1   (left pad 3 -> x offset 4)
  const int Wp = (W + 8 + 3) / 4 * 4;
  const int n = blockIdx.x / Ho, ho = blockIdx.x % Ho;
  for (int k = threadIdx.x; k < 160; k += blockDim.x) {
    int v = -1;
    if (k < 147) {
      const int c = k % 3, t = k / 3, kw = t % 7, kh = t / 7;
      v = (c * 7 + kh) * Wp + kw;
    }
    lut[k] = v;
  }
  // stage rows: tile[c][r][4 + w] = img[n][c][2*ho - 3 + r][w]
  if (W % 4 == 0) {
    const int quads = Wp / 4;
    for (int e = threadIdx.x; e < 21 * quads; e += blockDim.x) {
      const int cr = e / quads, qd = e % quads;
      const int c = cr / 7, r = cr % 7;
      const int h = 2 * ho - 3 + r;
      const int w0 = qd * 4 - 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (h >= 0 && h < H && w0 >= 0 && w0 + 3 < W)
        v = *reinterpret_cast<const float4*>(img + (((long long)n * 3 + c) * H + h) * W + w0);
      *reinterpret_cast<float4*>(tile + cr * Wp + qd * 4) = v;
    }
  } else {
    for (int e = threadIdx.x; e < 21 * Wp; e += blockDim.x) {
      const int cr = e / Wp, x = e % Wp;
      const int c = cr / 7, r = cr % 7;
      const int h = 2 * ho - 3 + r, w = x - 4;
      tile[e] = (h >= 0 && h < H && w >= 0 && w < W) ? img[(((long long)n * 3 + c) * H + h) * W + w] : 0.f;
    }
  }
  __syncthreads();
  const int groups = ldc / 8;
  const long long row0 = ((long long)n * Ho + ho) * Wo;
  for (int e = threadIdx.x; e < Wo * groups; e += blockDim.x) {
    const int wo = e / groups, g = e % groups;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = g * 8 + j;
      const int o = k < 160 ? lut[k] : -1;
      v[j] = o >= 0 ? tile[o + 2 * wo + 1] : 0.f;  // x = 2*wo - 3 + kw  ->  tile column 4 + x = 2*wo + 1 + kw
    }
    *reinterpret_cast<bf16x8*>(cols + (row0 + wo) * ldc + g * 8) = pack8(v);
  }
}

// ---------------------------------------------------------------------------------------------- generic 3x3 im2col
// x bf16 NHWC [N,H,W,C] -> cols [N*Ho*Wo, 9*C], k = (kh*3+kw)*C + c, pad 1, given stride.
__global__ void im2col3x3_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ cols, int N, int H,
                                 int W, int C, int Ho, int Wo, int stride) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const long long total = (long long)N * Ho * Wo * 9 * cg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    long long r = i / cg;
    const int tap = (int)(r % 9);
    const long long pos = r / 9;
    const int wo = (int)(pos % Wo);
    const int ho = (int)((pos / Wo) % Ho);
    const int n = (int)(pos / ((long long)Wo * Ho));
    const int kh = tap / 3, kw = tap % 3;
    const int h = ho * stride - 1 + kh, w = wo * stride - 1 + kw;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (h >= 0 && h < H && w >= 0 && w < W)
      v = *reinterpret_cast<const uint4*>(x + (((long long)n * H + h) * W + w) * C + g * 8);
    *reinterpret_cast<uint4*>(cols + pos * (9LL * C) + (long long)tap * C + g * 8) = v;
  }
}

// dcols [N*Ho*Wo, 9*C] -> dx [N,H,W,C]  (gather form: every input pixel sums the taps that touched it)
__global__ void col2im3x3_kernel(const __nv_bfloat16* __restrict__ dcols, __nv_bfloat16* __restrict__ dx, int N, int H,
                                 int W, int C, int Ho, int Wo, int stride) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const long long total = (long long)N * H * W * cg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    const long long pix = i / cg;
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const int n = (int)(pix / ((long long)W * H));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hn = h + 1 - kh;
      if (hn < 0 || hn % stride != 0) continue;
      const int ho = hn / stride;
      if (ho >= Ho) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wn = w + 1 - kw;
        if (wn < 0 || wn % stride != 0) continue;
        const int wo = wn / stride;
        if (wo >= Wo) continue;
        const long long pos = ((long long)n * Ho + ho) * Wo + wo;
        const bf16x8 u = *reinterpret_cast<const bf16x8*>(dcols + pos * (9LL * C) + (long long)(kh * 3 + kw) * C + g * 8);
        float f[8];
        unpack8(u, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
      }
    }
    *reinterpret_cast<bf16x8*>(dx + pix * C + g * 8) = pack8(acc);
  }
}

// the two gather kernels above spend most of their time in 64-bit integer division
// (seven div/mod by run-time values per 16-byte copy); when the item count fits 31 bits the same index arithmetic in
// 32 bits is 4-5x fewer instructions.  Identical results.
__global__ void im2col3x3_i32_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ cols, int N, int H,
                                     int W, int C, int Ho, int Wo, int stride) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const int total = N * Ho * Wo * 9 * cg;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int g = i % cg;
    const int r = i / cg;
    const int tap = r % 9;
    const int pos = r / 9;
    const int wo = pos % Wo;
    const int t2 = pos / Wo;
    const int ho = t2 % Ho;
    const int n = t2 / Ho;
    const int kh = tap / 3, kw = tap % 3;
    const int h = ho * stride - 1 + kh, w = wo * stride - 1 + kw;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (h >= 0 && h < H && w >= 0 && w < W)
      v = *reinterpret_cast<const uint4*>(x + (((long long)n * H + h) * W + w) * C + g * 8);
    *reinterpret_cast<uint4*>(cols + (long long)pos * (9LL * C) + (long long)tap * C + g * 8) = v;
  }
}
__global__ void col2im3x3_i32_kernel(const __nv_bfloat16* __restrict__ dcols, __nv_bfloat16* __restrict__ dx, int N, int H,
                                     int W, int C, int Ho, int Wo, int stride) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const int total = N * H * W * cg;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int g = i % cg;
    const int pix = i / cg;
    const int w = pix % W;
    const int t2 = pix / W;
    const int h = t2 % H;
    const int n = t2 / H;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hn = h + 1 - kh;
      if (hn < 0 || hn % stride != 0) continue;
      const int ho = hn / stride;
      if (ho >= Ho) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wn = w + 1 - kw;
        if (wn < 0 || wn % stride != 0) continue;
        const int wo = wn / stride;
        if (wo >= Wo) continue;
        const long long pos = ((long long)n * Ho + ho) * Wo + wo;
        const bf16x8 u = *reinterpret_cast<const bf16x8*>(dcols + pos * (9LL * C) + (long long)(kh * 3 + kw) * C + g * 8);
        float f[8];
        unpack8(u, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
      }
    }
    *reinterpret_cast<bf16x8*>(dx + (long long)pix * C + g * 8) = pack8(acc);
  }
}

// xs[n,ho,wo,:] = x[n,ho*s,wo*s,:]
__global__ void subsample_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ xs, int N, int H,
                                 int W, int C, int Ho, int Wo, int stride) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const long long total = (long long)N * Ho * Wo * cg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    const long long pos = i / cg;
    const int wo = (int)(pos % Wo);
    const int ho = (int)((pos / Wo) % Ho);
    const int n = (int)(pos / ((long long)Wo * Ho));
    *reinterpret_cast<uint4*>(xs + pos * C + g * 8) =
        *reinterpret_cast<const uint4*>(x + (((long long)n * H + ho * stride) * W + wo * stride) * C + g * 8);
  }
}

// dx[n,ho*s,wo*s,:] += dxs[n,ho,wo,:]
__global__ void upsample_add_kernel(const __nv_bfloat16* __restrict__ dxs, __nv_bfloat16* __restrict__ dx, int N, int H,
                                    int W, int C, int Ho, int Wo, int stride) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const long long total = (long long)N * Ho * Wo * cg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    const long long pos = i / cg;
    const int wo = (int)(pos % Wo);
    const int ho = (int)((pos / Wo) % Ho);
    const int n = (int)(pos / ((long long)Wo * Ho));
    __nv_bfloat16* p = dx + (((long long)n * H + ho * stride) * W + wo * stride) * C + g * 8;
    float a[8], b[8];
    unpack8(*reinterpret_cast<const bf16x8*>(p), a);
    unpack8(*reinterpret_cast<const bf16x8*>(dxs + pos * C + g * 8), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    *reinterpret_cast<bf16x8*>(p) = pack8(a);
  }
}

// 32-bit index arithmetic, see im2col3x3_i32_kernel
__global__ void subsample_i32_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ xs, int N, int H,
                                     int W, int C, int Ho, int Wo, int stride) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const int total = N * Ho * Wo * cg;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int g = i % cg;
    const int pos = i / cg;
    const int wo = pos % Wo;
    const int t2 = pos / Wo;
    const int ho = t2 % Ho;
    const int n = t2 / Ho;
    *reinterpret_cast<uint4*>(xs + (long long)pos * C + g * 8) =
        *reinterpret_cast<const uint4*>(x + (((long long)n * H + ho * stride) * W + wo * stride) * C + g * 8);
  }
}
__global__ void upsample_add_i32_kernel(const __nv_bfloat16* __restrict__ dxs, __nv_bfloat16* __restrict__ dx, int N, int H,
                                        int W, int C, int Ho, int Wo, int stride) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const int total = N * Ho * Wo * cg;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int g = i % cg;
    const int pos = i / cg;
    const int wo = pos % Wo;
    const int t2 = pos / Wo;
    const int ho = t2 % Ho;
    const int n = t2 / Ho;
    __nv_bfloat16* p = dx + (((long long)n * H + ho * stride) * W + wo * stride) * C + g * 8;
    float a[8], b[8];
    unpack8(*reinterpret_cast<const bf16x8*>(p), a);
    unpack8(*reinterpret_cast<const bf16x8*>(dxs + (long long)pos * C + g * 8), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    *reinterpret_cast<bf16x8*>(p) = pack8(a);
  }
}

// ---------------------------------------------------------------------------------------------- BatchNorm forward
// stats [2,C] (sum, sumsq over `count` samples)  ->  bnp [4,C] = mean, invstd, scale = gamma*invstd, shift
// training: also running_mean/var (momentum, unbiased var) and num_batches_tracked.  eval: statistics come from
// the running buffers instead (stats may be null).
__global__ void bn_finalize_kernel(const float* __restrict__ stats, float count, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float* __restrict__ rmean, float* __restrict__ rvar,
                                   long long* __restrict__ nbt, float momentum, float eps, int training,
                                   float* __restrict__ bnp, int C) {
  VTX_PDL_TRIGGER();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0 && training && nbt != nullptr) *nbt += 1;
  if (c >= C) return;
  float mean, var;
  if (training) {
    mean = stats[c] / count;
    var = fmaxf(stats[C + c] / count - mean * mean, 0.f);
    rmean[c] = (1.f - momentum) * rmean[c] + momentum * mean;
    rvar[c] = (1.f - momentum) * rvar[c] + momentum * var * (count / fmaxf(count - 1.f, 1.f));
  } else {
    mean = rmean[c];
    var = rvar[c];
  }
  const float invstd = rsqrtf(var + eps);
  const float sc = gamma[c] * invstd;
  bnp[c] = mean;
  bnp[C + c] = invstd;
  bnp[2 * C + c] = sc;
  bnp[3 * C + c] = beta[c] - mean * sc;
}

// a = act( y*scale + shift  [+ res  |  + res*scale2 + shift2] );  relu_mask (optional): bit j of byte (m*C/8 + c/8) =
// [pre-activation of channel 8*(c/8)+j of row m > 0]
constexpr int kU = 4;  // independent 16-byte loads per tensor in flight per thread (memory-level parallelism)
constexpr int kUbwd = 6;  // single-BN backward apply (two input streams): 96 KB in flight per SM
constexpr int kUred = 5;  // single-BN backward reduce (one more load would spill at 128 registers)

// Optional fold of bn_finalize into the apply kernel: every thread derives scale/shift of its 8 channels from the raw
// batch sums (or the running statistics in eval mode); block 0 also publishes bnp and updates the running buffers.
struct BnFwdFold {
  const float* stats;  // [2,C] sum, sumsq (training) -- may be null in eval mode
  const float* gamma;
  const float* beta;
  float* rmean;
  float* rvar;
  long long* nbt;
  float count, momentum, eps;
  int training;
};

// kUa = independent 16-byte loads per tensor in flight per thread: HBM bandwidth needs many bytes in flight per SM, so
// the single-input variants (no residual operand) run 8 loads deep.
template <bool kFold, int kUa>
__global__ void __launch_bounds__(256, 2) bn_act_kernel(const __nv_bfloat16* __restrict__ y, float* __restrict__ bnp,
                              const __nv_bfloat16* __restrict__ res, const float* __restrict__ bnp_res,
                              __nv_bfloat16* __restrict__ out, uint8_t* __restrict__ relu_mask, long long M, int C,
                              int relu, const BnFwdFold f) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const long long total = M * cg;
  // blockDim.x (256) is a multiple of cg, so a thread's 8-channel group never changes across the grid-stride loop:
  // per-channel parameters live in registers.
  const long long i0 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int c0 = (int)(i0 % cg) * 8;
  float sc[8], sh[8], sc2[8], sh2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j;
    if (kFold) {
      float mean, var;
      if (f.training) {
        mean = f.stats[c] / f.count;
        var = fmaxf(f.stats[C + c] / f.count - mean * mean, 0.f);
      } else {
        mean = f.rmean[c];
        var = f.rvar[c];
      }
      const float invstd = rsqrtf(var + f.eps);
      sc[j] = f.gamma[c] * invstd;
      sh[j] = f.beta[c] - mean * sc[j];
      if (blockIdx.x == 0 && threadIdx.x < cg) {  // thread t < cg of block 0 owns channels [8t, 8t+8)
        bnp[c] = mean;
        bnp[C + c] = invstd;
        bnp[2 * C + c] = sc[j];
        bnp[3 * C + c] = sh[j];
        if (f.training) {
          f.rmean[c] = (1.f - f.momentum) * f.rmean[c] + f.momentum * mean;
          f.rvar[c] = (1.f - f.momentum) * f.rvar[c] + f.momentum * var * (f.count / fmaxf(f.count - 1.f, 1.f));
        }
      }
    } else {
      sc[j] = bnp[2 * C + c];
      sh[j] = bnp[3 * C + c];
    }
    sc2[j] = bnp_res ? bnp_res[2 * C + c] : 1.f;
    sh2[j] = bnp_res ? bnp_res[3 * C + c] : 0.f;
  }
  if (kFold && blockIdx.x == 0 && threadIdx.x == 0 && f.training && f.nbt != nullptr) *f.nbt += 1;
  for (long long i = i0; i < total; i += stride * kUa) {
    bf16x8 vy[kUa], vr[kUa];
#pragma unroll
    for (int u = 0; u < kUa; ++u) {
      const long long idx = i + u * stride;
      if (idx < total) {
        vy[u] = *reinterpret_cast<const bf16x8*>(y + idx * 8);
        if (res != nullptr) vr[u] = *reinterpret_cast<const bf16x8*>(res + idx * 8);
      }
    }
#pragma unroll
    for (int u = 0; u < kUa; ++u) {
      const long long idx = i + u * stride;
      if (idx >= total) break;
      float v[8];
      unpack8(vy[u], v);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = v[j] * sc[j] + sh[j];
      if (res != nullptr) {
        float r[8];
        unpack8(vr[u], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += r[j] * sc2[j] + sh2[j];
      }
      if (relu) {
        // one bit per channel: what backward needs of this activation (its sign), 1/16 of the bytes of `out`
        if (relu_mask != nullptr) {
          uint32_t bits = 0;
#pragma unroll
          for (int j = 0; j < 8; ++j) bits |= (v[j] > 0.f ? 1u : 0u) << j;
          relu_mask[idx] = (uint8_t)bits;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.f);
      }
      *reinterpret_cast<bf16x8*>(out + idx * 8) = pack8(v);
    }
  }
}

// stem: pooled[n,ph,pw,:] = max over the 3x3/stride 2/pad 1 window of relu(y*scale+shift); idx = window slot of the max
// Row-per-block form of the kernel below for C/8 dividing 256 (every ResNet stem): one CTA walks pooled rows (n, ph);
// a thread keeps its channel group and BN coefficients for the whole launch and steps pw by blockDim / (C/8), so the loop has
// no division at all (the flat-index form spent ~400 of its ~900 instructions per item on five 64-bit div / mod).
__global__ void __launch_bounds__(256) bn_relu_maxpool_rows_kernel(const __nv_bfloat16* __restrict__ y,
                                                                   const float* __restrict__ bnp,
                                                                   __nv_bfloat16* __restrict__ out,
                                                                   uint8_t* __restrict__ idx, int N, int H, int W, int C,
                                                                   int Ho, int Wo) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const int g = threadIdx.x % cg, pw0 = threadIdx.x / cg, pstep = blockDim.x / cg;
  const int c0 = g * 8;
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    sc[j] = __ldg(bnp + 2 * C + c0 + j);
    sh[j] = __ldg(bnp + 3 * C + c0 + j);
  }
  for (int row = blockIdx.x; row < N * Ho; row += gridDim.x) {
    const int n = row / Ho, ph = row - n * Ho;
    const __nv_bfloat16* yn = y + (long long)n * H * W * C + c0;
    for (int pw = pw0; pw < Wo; pw += pstep) {
      float best[8];
      int bi[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        best[j] = -INFINITY;
        bi[j] = 0;
      }
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int h = ph * 2 - 1 + kh;
        if (h < 0 || h >= H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int w = pw * 2 - 1 + kw;
          if (w < 0 || w >= W) continue;
          float v[8];
          unpack8(*reinterpret_cast<const bf16x8*>(yn + (h * W + w) * C), v);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            // the reference rounds the BN output and the ReLU output to bf16 before pooling
            const float a = bf2f(f2bf(fmaxf(v[j] * sc[j] + sh[j], 0.f)));
            if (a > best[j]) { best[j] = a; bi[j] = kh * 3 + kw; }
          }
        }
      }
      const long long o = ((long long)row * Wo + pw) * C + c0;
      *reinterpret_cast<bf16x8*>(out + o) = pack8(best);
      uint8_t b[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = (uint8_t)bi[j];
      *reinterpret_cast<uint2*>(idx + o) = *reinterpret_cast<uint2*>(b);
    }
  }
}

__global__ void bn_relu_maxpool_kernel(const __nv_bfloat16* __restrict__ y, const float* __restrict__ bnp,
                                       __nv_bfloat16* __restrict__ out, uint8_t* __restrict__ idx, int N, int H, int W,
                                       int C, int Ho, int Wo) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const long long total = (long long)N * Ho * Wo * cg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    const int c0 = g * 8;
    const long long pos = i / cg;
    const int pw = (int)(pos % Wo);
    const int ph = (int)((pos / Wo) % Ho);
    const int n = (int)(pos / ((long long)Wo * Ho));
    float sc[8], sh[8], best[8];
    int bi[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      sc[j] = __ldg(bnp + 2 * C + c0 + j);
      sh[j] = __ldg(bnp + 3 * C + c0 + j);
      best[j] = -INFINITY;
      bi[j] = 0;
    }
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int h = ph * 2 - 1 + kh;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int w = pw * 2 - 1 + kw;
        if (w < 0 || w >= W) continue;
        float v[8];
        unpack8(*reinterpret_cast<const bf16x8*>(y + (((long long)n * H + h) * W + w) * C + c0), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          // the reference rounds the BN output and the ReLU output to bf16 before pooling
          const float a = bf2f(f2bf(fmaxf(v[j] * sc[j] + sh[j], 0.f)));
          if (a > best[j]) { best[j] = a; bi[j] = kh * 3 + kw; }
        }
      }
    }
    *reinterpret_cast<bf16x8*>(out + pos * C + c0) = pack8(best);
    uint8_t b[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) b[j] = (uint8_t)bi[j];
    *reinterpret_cast<uint2*>(idx + pos * C + c0) = *reinterpret_cast<uint2*>(b);
  }
}

// da[n,h,w,:] = sum over pooled windows (ph,pw) whose argmax slot points at (h,w) of dpool[n,ph,pw,:]
__global__ void maxpool_bwd_kernel(const __nv_bfloat16* __restrict__ dpool, const uint8_t* __restrict__ idx,
                                   __nv_bfloat16* __restrict__ da, int N, int H, int W, int C, int Ho, int Wo) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const long long total = (long long)N * H * W * cg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % cg);
    const int c0 = g * 8;
    const long long pix = i / cg;
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const int n = (int)(pix / ((long long)W * H));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hn = h + 1 - kh;
      if (hn < 0 || (hn & 1)) continue;
      const int ph = hn >> 1;
      if (ph >= Ho) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wn = w + 1 - kw;
        if (wn < 0 || (wn & 1)) continue;
        const int pw = wn >> 1;
        if (pw >= Wo) continue;
        const long long pos = ((long long)n * Ho + ph) * Wo + pw;
        const uint2 raw = *reinterpret_cast<const uint2*>(idx + pos * C + c0);
        const uint8_t* b = reinterpret_cast<const uint8_t*>(&raw);
        float d[8];
        unpack8(*reinterpret_cast<const bf16x8*>(dpool + pos * C + c0), d);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (b[j] == kh * 3 + kw) acc[j] += d[j];
      }
    }
    *reinterpret_cast<bf16x8*>(da + pix * C + c0) = pack8(acc);
  }
}

// (A shared-memory tiled variant of the FORWARD pool was slower than the direct kernel above and deleted: the ~2.25x
// re-normalisation it saved is cheaper than its staging pass.)
// same arithmetic as maxpool_bwd_kernel, but a CTA first stages the kTP + 1 pooled rows
// (gradients + argmax slots) it needs in shared memory with linear coalesced copies and then produces 2 * kTP input
// rows from them.  The validated kernel gathers every pooled element from L2 up to nine times (1.4 GB of L2 -> SM
// traffic for 565 MB of algorithmic bytes at batch 256).
constexpr int kTP = 4;
__global__ void __launch_bounds__(256) maxpool_bwd_tiled_kernel(const __nv_bfloat16* __restrict__ dpool,
                                                               const uint8_t* __restrict__ idx,
                                                               __nv_bfloat16* __restrict__ da, int N, int H, int W, int C,
                                                               int Ho, int Wo) {
  VTX_PDL_TRIGGER();
  extern __shared__ __align__(16) uint8_t pool_smem[];
  const int row_elems = Wo * C;                                   // elements of one pooled row
  __nv_bfloat16* sd = reinterpret_cast<__nv_bfloat16*>(pool_smem);            // [kTP + 1][Wo][C] gradients
  uint8_t* si = pool_smem + (size_t)(kTP + 1) * row_elems * 2;               // [kTP + 1][Wo][C] argmax slots
  const int tiles = (Ho + kTP - 1) / kTP;
  const int n = blockIdx.x / tiles, ph0 = (blockIdx.x % tiles) * kTP;
  const int prow = min(kTP + 1, Ho - ph0);                        // pooled rows that exist
  {
    const uint4* gd = reinterpret_cast<const uint4*>(dpool + ((long long)n * Ho + ph0) * row_elems);
    uint4* d4 = reinterpret_cast<uint4*>(sd);
    for (int i = threadIdx.x; i < prow * row_elems / 8; i += blockDim.x) d4[i] = gd[i];
    const uint4* gi = reinterpret_cast<const uint4*>(idx + ((long long)n * Ho + ph0) * row_elems);
    uint4* i4 = reinterpret_cast<uint4*>(si);
    for (int i = threadIdx.x; i < prow * row_elems / 16; i += blockDim.x) i4[i] = gi[i];
  }
  __syncthreads();
  const int cg = C / 8;
  const int h0 = 2 * ph0, h1 = min(H, 2 * (ph0 + kTP));
  // thread-fixed channel group, w stepping by blockDim / cg (the launcher guarantees cg | blockDim): no division in the loops, and
  // the 1 or 2 pooled columns / rows that can point at (h, w) depend only on the parity of w / h
  const int c0 = (threadIdx.x % cg) * 8;
  for (int w = threadIdx.x / cg; w < W; w += blockDim.x / cg) {
    int kws[2], pws[2], nw = 0;
    if (w & 1) {
      if (((w + 1) >> 1) < Wo) { kws[nw] = 0; pws[nw++] = (w + 1) >> 1; }
      kws[nw] = 2; pws[nw++] = (w - 1) >> 1;
    } else {
      kws[0] = 1; pws[0] = w >> 1; nw = 1;
    }
    for (int h = h0; h < h1; ++h) {
      int khs[2], phs[2], nh = 0;
      if (h & 1) {
        if (((h + 1) >> 1) < Ho) { khs[nh] = 0; phs[nh++] = (h + 1) >> 1; }
        khs[nh] = 2; phs[nh++] = (h - 1) >> 1;
      } else {
        khs[0] = 1; phs[0] = h >> 1; nh = 1;
      }
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        if (a >= nh) continue;
#pragma unroll
        for (int b2 = 0; b2 < 2; ++b2) {
          if (b2 >= nw) continue;
          const int off = ((phs[a] - ph0) * Wo + pws[b2]) * C + c0;
          const int slot = khs[a] * 3 + kws[b2];
          const uint2 raw = *reinterpret_cast<const uint2*>(si + off);
          const uint8_t* b = reinterpret_cast<const uint8_t*>(&raw);
          float d[8];
          unpack8(*reinterpret_cast<const bf16x8*>(sd + off), d);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (b[j] == slot) acc[j] += d[j];
        }
      }
      *reinterpret_cast<bf16x8*>(da + (((long long)n * H + h) * W + w) * C + c0) = pack8(acc);
    }
  }
}

// ---------------------------------------------------------------------------------------------- BatchNorm backward
// sums[0,c] = sum_m dz, sums[1,c] = sum_m dz * xhat, with dz = dA * [relu_mask bit] (relu_mask == null: no ReLU, or the
// mask recomputed from y when mask_from_y) and
// xhat = (y - mean) * invstd.  Optionally the same for a second BN (y2, bnp2) sharing dz (downsample branch).
template <int kTwo, int kUb>
__global__ void __launch_bounds__(256, kTwo ? 1 : 2) bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ dA, const uint8_t* __restrict__ a,
                                     const __nv_bfloat16* __restrict__ y, const float* __restrict__ bnp,
                                     const __nv_bfloat16* __restrict__ y2, const float* __restrict__ bnp2,
                                     float* __restrict__ sums, float* __restrict__ sums2, long long M, int C,
                                     int mask_from_y) {
  VTX_PDL_TRIGGER();
  extern __shared__ float red[];  // [rows_par][C][2 or 4]
  const int cg = C / 8;
  const int rows_par = blockDim.x / cg;  // rows handled in parallel by one CTA
  const int g = threadIdx.x % cg;
  const int rr = threadIdx.x / cg;
  const int c0 = g * 8;
  float s1[8], s2[8], t1[8], t2[8];
  float mean[8], istd[8], mean2[8], istd2[8], msc[8], msh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s1[j] = s2[j] = t1[j] = t2[j] = 0.f;
    mean[j] = __ldg(bnp + c0 + j);
    istd[j] = __ldg(bnp + C + c0 + j);
    msc[j] = __ldg(bnp + 2 * C + c0 + j);
    msh[j] = __ldg(bnp + 3 * C + c0 + j);
    if (kTwo) {
      mean2[j] = __ldg(bnp2 + c0 + j);
      istd2[j] = __ldg(bnp2 + C + c0 + j);
    }
  }
  if (rr < rows_par) {
    const long long mstride = (long long)gridDim.x * rows_par;
    for (long long m0 = (long long)blockIdx.x * rows_par + rr; m0 < M; m0 += mstride * kUb) {
      bf16x8 vd[kUb], vy[kUb], vy2[kUb];
      uint32_t va[kUb];
#pragma unroll
      for (int u = 0; u < kUb; ++u) {
        const long long m = m0 + u * mstride;
        if (m < M) {
          const long long off = m * C + c0;
          vd[u] = *reinterpret_cast<const bf16x8*>(dA + off);
          vy[u] = *reinterpret_cast<const bf16x8*>(y + off);
          if (a != nullptr) va[u] = a[m * cg + g];
          if (kTwo) vy2[u] = *reinterpret_cast<const bf16x8*>(y2 + off);
        }
      }
#pragma unroll
      for (int u = 0; u < kUb; ++u) {
        const long long m = m0 + u * mstride;
        if (m >= M) break;
        float d[8], yy[8];
        unpack8(vd[u], d);
        unpack8(vy[u], yy);
        if (a != nullptr) {
#pragma unroll
          for (int j = 0; j < 8; ++j) d[j] = ((va[u] >> j) & 1u) ? d[j] : 0.f;
        } else if (mask_from_y) {  // ReLU mask recomputed from the BN output sign: a = relu(y*scale + shift)
#pragma unroll
          for (int j = 0; j < 8; ++j) d[j] = (yy[j] * msc[j] + msh[j] > 0.f) ? d[j] : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s1[j] += d[j];
          s2[j] += d[j] * (yy[j] - mean[j]) * istd[j];
        }
        if (kTwo) {
          unpack8(vy2[u], yy);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            t1[j] += d[j];
            t2[j] += d[j] * (yy[j] - mean2[j]) * istd2[j];
          }
        }
      }
    }
  }
  // cross-row reduction through shared memory, then one atomic per channel per CTA
  const int per = kTwo ? 4 : 2;
  if (rr < rows_par) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float* p = red + ((long long)rr * C + c0 + j) * per;
      p[0] = s1[j];
      p[1] = s2[j];
      if (kTwo) { p[2] = t1[j]; p[3] = t2[j]; }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r = 0; r < rows_par; ++r) {
      const float* p = red + ((long long)r * C + c) * per;
      acc[0] += p[0];
      acc[1] += p[1];
      if (kTwo) { acc[2] += p[2]; acc[3] += p[3]; }
    }
    atomicAdd(sums + c, acc[0]);
    atomicAdd(sums + C + c, acc[1]);
    if (kTwo) {
      atomicAdd(sums2 + c, acc[2]);
      atomicAdd(sums2 + C + c, acc[3]);
    }
  }
}

// sums [2,C] -> coef [3,C] = (scale, sum_dz/count, sum_dz_xhat/count);  dgamma += sum_dz_xhat, dbeta += sum_dz
__global__ void bn_bwd_finalize_kernel(const float* __restrict__ sums, const float* __restrict__ bnp, float count,
                                       float* __restrict__ coef, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                       int C) {
  VTX_PDL_TRIGGER();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float s1 = sums[c], s2 = sums[C + c];
  coef[c] = bnp[2 * C + c];
  coef[C + c] = s1 / count;
  coef[2 * C + c] = s2 / count;
  if (dgamma != nullptr) dgamma[c] += s2;
  if (dbeta != nullptr) dbeta[c] += s1;
}

// dy = scale * (dz - m1 - xhat * m2);  optional second BN sharing dz;  optional dz output (identity shortcut grad)
// Optional fold of bn_bwd_finalize: coefficients derived from the raw sums in the prologue; block 0 accumulates dgamma/dbeta
struct BnBwdFold {
  const float* sums;
  const float* sums2;
  float* dgamma;
  float* dbeta;
  float* dgamma2;
  float* dbeta2;
  float count;
};

template <int kTwo, bool kFold, int kUb>
__global__ void __launch_bounds__(256, kTwo ? 1 : 2) bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ dA, const uint8_t* __restrict__ a,
                                    const __nv_bfloat16* __restrict__ y, const float* __restrict__ bnp,
                                    const float* __restrict__ coef, __nv_bfloat16* __restrict__ dy,
                                    const __nv_bfloat16* __restrict__ y2, const float* __restrict__ bnp2,
                                    const float* __restrict__ coef2, __nv_bfloat16* __restrict__ dy2,
                                    __nv_bfloat16* __restrict__ dz_out, long long M, int C, int mask_from_y,
                                    const BnBwdFold f) {
  VTX_PDL_TRIGGER();
  const int cg = C / 8;
  const long long total = M * cg;
  const long long i0 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int c0 = (int)(i0 % cg) * 8;  // loop invariant (blockDim.x % cg == 0)
  float msc[8], msh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    msc[j] = bnp[2 * C + c0 + j];
    msh[j] = bnp[3 * C + c0 + j];
  }
  // dy = k0*dz + k1*y + k2 with k0 = scale, k1 = -scale*m2*invstd, k2 = scale*(m2*invstd*mean - m1)
  float k0[8], k1[8], k2[8], q0[8], q1[8], q2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + j;
    const float mean = bnp[c], istd = bnp[C + c];
    float scl, m1, m2;
    if (kFold) {
      const float s1 = f.sums[c], s2 = f.sums[C + c];
      scl = bnp[2 * C + c];
      m1 = s1 / f.count;
      m2 = s2 / f.count;
      if (blockIdx.x == 0 && threadIdx.x < cg) {
        if (f.dgamma) f.dgamma[c] += s2;
        if (f.dbeta) f.dbeta[c] += s1;
      }
    } else {
      scl = coef[c]; m1 = coef[C + c]; m2 = coef[2 * C + c];
    }
    k0[j] = scl;
    k1[j] = -scl * m2 * istd;
    k2[j] = scl * (m2 * istd * mean - m1);
    if (kTwo) {
      const float mean_b = bnp2[c], istd_b = bnp2[C + c];
      float scl_b, m1b, m2b;
      if (kFold) {
        const float s1 = f.sums2[c], s2 = f.sums2[C + c];
        scl_b = bnp2[2 * C + c];
        m1b = s1 / f.count;
        m2b = s2 / f.count;
        if (blockIdx.x == 0 && threadIdx.x < cg) {
          if (f.dgamma2) f.dgamma2[c] += s2;
          if (f.dbeta2) f.dbeta2[c] += s1;
        }
      } else {
        scl_b = coef2[c]; m1b = coef2[C + c]; m2b = coef2[2 * C + c];
      }
      q0[j] = scl_b;
      q1[j] = -scl_b * m2b * istd_b;
      q2[j] = scl_b * (m2b * istd_b * mean_b - m1b);
    }
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = i0; i < total; i += stride * kUb) {
    bf16x8 vd[kUb], vy[kUb], vy2[kUb];
    uint32_t va[kUb];
#pragma unroll
    for (int u = 0; u < kUb; ++u) {
      const long long idx = i + u * stride;
      if (idx < total) {
        vd[u] = *reinterpret_cast<const bf16x8*>(dA + idx * 8);
        vy[u] = *reinterpret_cast<const bf16x8*>(y + idx * 8);
        if (a != nullptr) va[u] = a[idx];
        if (kTwo) vy2[u] = *reinterpret_cast<const bf16x8*>(y2 + idx * 8);
      }
    }
#pragma unroll
    for (int u = 0; u < kUb; ++u) {
      const long long idx = i + u * stride;
      if (idx >= total) break;
      float d[8], yy[8], o[8];
      unpack8(vd[u], d);
      unpack8(vy[u], yy);
      if (a != nullptr) {
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = ((va[u] >> j) & 1u) ? d[j] : 0.f;
      } else if (mask_from_y) {
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = (yy[j] * msc[j] + msh[j] > 0.f) ? d[j] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = k0[j] * d[j] + k1[j] * yy[j] + k2[j];
      *reinterpret_cast<bf16x8*>(dy + idx * 8) = pack8(o);
      if (kTwo) {
        unpack8(vy2[u], yy);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = q0[j] * d[j] + q1[j] * yy[j] + q2[j];
        *reinterpret_cast<bf16x8*>(dy2 + idx * 8) = pack8(o);
      }
      if (dz_out != nullptr) *reinterpret_cast<bf16x8*>(dz_out + idx * 8) = pack8(d);
    }
  }
}

// ---------------------------------------------------------------------------------------------- weight layouts
// fp32 OIHW [O,I,KH,KW] -> bf16 [O, ldk] with k = (kh*KW + kw)*I + i   (columns >= KH*KW*I zero)
__global__ void conv_w_pack_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int O, int I, int KH,
                                   int KW, int ldk) {
  VTX_PDL_TRIGGER();
  const long long total = (long long)O * ldk;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(t % ldk);
    const int o = (int)(t / ldk);
    float v = 0.f;
    if (k < KH * KW * I) {
      const int i = k % I;
      const int tap = k / I;
      v = w[((long long)o * I + i) * KH * KW + tap];
    }
    out[t] = f2bf(v);
  }
}
// fp32 OIHW [O,I,3,3] -> bf16 [I, 9*O] with k = ((2-kh)*3 + (2-kw))*O + o   (flipped + transposed: dgrad weights)
__global__ void conv_w_pack_dgrad_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int O, int I) {
  VTX_PDL_TRIGGER();
  const long long total = (long long)I * 9 * O;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int o = (int)(t % O);
    const int tapf = (int)((t / O) % 9);
    const int i = (int)(t / (9LL * O));
    const int tap = 8 - tapf;  // (2-kh)*3 + (2-kw)
    out[t] = f2bf(w[((long long)o * I + i) * 9 + tap]);
  }
}
// grad OIHW += dwp [O, ldk] (k = tap*I + i)
__global__ void conv_w_unpack_add_kernel(const float* __restrict__ dwp, float* __restrict__ grad, int O, int I, int KH,
                                         int KW, int ldk) {
  VTX_PDL_TRIGGER();
  const long long total = (long long)O * I * KH * KW;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int tap = (int)(t % (KH * KW));
    const int i = (int)((t / (KH * KW)) % I);
    const int o = (int)(t / ((long long)KH * KW * I));
    grad[t] += dwp[(long long)o * ldk + (long long)tap * I + i];
  }
}
// grad OIHW += dwt [(tap, i), O]   (transposed layout produced by the halo-reuse wgrad, conv_mode 4)
__global__ void conv_w_unpack_add_t_kernel(const float* __restrict__ dwt, float* __restrict__ grad, int O, int I, int KH,
                                           int KW) {
  VTX_PDL_TRIGGER();
  const long long total = (long long)O * I * KH * KW;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int tap = (int)(t % (KH * KW));
    const int i = (int)((t / (KH * KW)) % I);
    const int o = (int)(t / ((long long)KH * KW * I));
    grad[t] += dwt[((long long)tap * I + i) * O + o];
  }
}
// Batched weight-layout jobs: ONE launch runs every pack (after an optimiser step) or every unpack-accumulate (per
// gradient bucket) of the k > 1 convolution weights instead of one ~3 us launch per tensor (R50: 31 + 17 per step).
// The job table lives in device memory and is built once (pointers into the arenas and workspaces never move).
//   kind 0: pack           fp32 OIHW -> bf16 [O, ldk], k = (kh*KW + kw)*I + i  (columns >= KH*KW*I zero)
//   kind 1: pack (dgrad)   fp32 OIHW [O,I,3,3] -> bf16 [I, 9*O], k = ((2-kh)*3 + (2-kw))*O + o
//   kind 2: unpack-add     grad OIHW += dwp [O, ldk]
//   kind 3: unpack-add (T) grad OIHW += dwt [(tap, i), O]          (halo-reuse wgrad layout, conv_mode 4)
//   kind 4: stem s2d pack  fp32 [O,3,7,7] -> bf16 [O, 256]         (index map of csrc/stem_s2d.cu)
//   kind 5: stem s2d unpack-add  grad [O,3,7,7] += dwp [O, 256]
//   kind 6: pack (stride-2 dgrad, parity class (ph, pw) = (KH, KW) of the input gradient):
//           fp32 OIHW [O,I,3,3] -> bf16 [I, ntaps*O], k = (a*tw + b)*O + o with (th, tw) = (1+ph, 1+pw) taps and
//           (kh, kw) = (ph + 1 - 2a, pw + 1 - 2b): input row 2i+ph receives dy row i+a through kernel row kh
//   kind 7: transpose      fp32 [O, I] (1x1 weight) -> bf16 [I, O]   (K-major B operand of the strided downsample's dgrad)
constexpr int kJobElemsPerBlock = 2048;
__global__ void __launch_bounds__(256) conv_w_jobs_kernel(const VtxWeightJob* __restrict__ jobs, int njobs) {
  VTX_PDL_TRIGGER();
  int j = 0;
  while (j + 1 < njobs && (int)blockIdx.x >= jobs[j + 1].block0) ++j;
  const VtxWeightJob jb = jobs[j];
  const long long e0 = (long long)((int)blockIdx.x - jb.block0) * kJobElemsPerBlock;
  const int O = jb.O, I = jb.I, KH = jb.KH, KW = jb.KW, ldk = jb.ldk;
  const float* fs = reinterpret_cast<const float*>(jb.src);
  for (long long t = e0 + threadIdx.x; t < e0 + kJobElemsPerBlock && t < jb.total; t += blockDim.x) {
    switch (jb.kind) {
      case 0: {
        const int k = (int)(t % ldk), o = (int)(t / ldk);
        float v = 0.f;
        if (k < KH * KW * I) v = fs[((long long)o * I + k % I) * KH * KW + k / I];
        reinterpret_cast<__nv_bfloat16*>(jb.dst)[t] = f2bf(v);
        break;
      }
      case 1: {
        const int o = (int)(t % O), tapf = (int)((t / O) % 9), i = (int)(t / (9LL * O));
        reinterpret_cast<__nv_bfloat16*>(jb.dst)[t] = f2bf(fs[((long long)o * I + i) * 9 + (8 - tapf)]);
        break;
      }
      case 2: {
        const int tap = (int)(t % (KH * KW)), i = (int)((t / (KH * KW)) % I), o = (int)(t / ((long long)KH * KW * I));
        reinterpret_cast<float*>(jb.dst)[t] += fs[(long long)o * ldk + (long long)tap * I + i];
        break;
      }
      case 3: {
        const int tap = (int)(t % (KH * KW)), i = (int)((t / (KH * KW)) % I), o = (int)(t / ((long long)KH * KW * I));
        reinterpret_cast<float*>(jb.dst)[t] += fs[((long long)tap * I + i) * O + o];
        break;
      }
      case 4: {
        const int o = (int)(t >> 8), k = (int)(t & 255);
        const int a = k >> 6, b = (k >> 4) & 3, ch = k & 15;
        float f = 0.f;
        if (ch < 12) {
          const int rq = ch / 3, c = ch - rq * 3;
          const int kh = 2 * a + (rq >> 1), kw = 2 * b + (rq & 1);
          if (kh < 7 && kw < 7) f = fs[((o * 3 + c) * 7 + kh) * 7 + kw];
        }
        reinterpret_cast<__nv_bfloat16*>(jb.dst)[t] = f2bf(f);
        break;
      }
      case 6: {
        const int ph = KH, pw = KW, tw = 1 + pw, nt = (1 + ph) * tw;
        const int o = (int)(t % O), tap = (int)((t / O) % nt), i = (int)(t / ((long long)nt * O));
        const int a = tap / tw, b = tap - a * tw;
        const int kh = ph + 1 - 2 * a, kw = pw + 1 - 2 * b;
        reinterpret_cast<__nv_bfloat16*>(jb.dst)[t] = f2bf(fs[((long long)o * I + i) * 9 + kh * 3 + kw]);
        break;
      }
      case 7: {  // transpose of a 1x1 weight: fp32 [O, I] -> bf16 [I, O]
        const int o = (int)(t % O), i = (int)(t / O);
        reinterpret_cast<__nv_bfloat16*>(jb.dst)[t] = f2bf(fs[(long long)o * I + i]);
        break;
      }
      default: {
        const int kw = (int)(t % 7), kh = (int)((t / 7) % 7), c = (int)((t / 49) % 3), o = (int)(t / 147);
        const int k = (kh >> 1) * 64 + (kw >> 1) * 16 + ((kh & 1) * 2 + (kw & 1)) * 3 + c;
        reinterpret_cast<float*>(jb.dst)[t] += fs[o * 256 + k];
        break;
      }
    }
  }
}

__global__ void cast_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, long long n) {
  VTX_PDL_TRIGGER();
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(in)[i];
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&a);
    u.y = *reinterpret_cast<uint32_t*>(&b);
    reinterpret_cast<uint2*>(out)[i] = u;
  }
  for (long long i = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = f2bf(in[i]);
}
// NHWC bf16 [N,H,W,C] -> NCHW fp32 (the reference-shaped `visual_features` handed back to callers)
__global__ void nhwc_to_nchw_f32_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, int N, int HW,
                                        int C) {
  VTX_PDL_TRIGGER();
  const long long total = (long long)N * HW * C;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(t % HW);
    const int c = (int)((t / HW) % C);
    const int n = (int)(t / ((long long)HW * C));
    out[t] = bf2f(in[((long long)n * HW + p) * C + c]);
  }
}

}  // namespace vtx

using namespace vtx;
#define STREAM reinterpret_cast<cudaStream_t>(stream)
#define REQ(cond, msg) \
  if (!(cond)) return set_error(VTX_EINVAL, "%s: %s", __func__, msg)
// bn_act_kernel and bn_bwd_apply_kernel keep a thread's 8 channels of BN parameters in registers for the whole
// grid-stride loop.  That is only right when the channel group of element i, i % (C/8), does not change when i steps by
// the grid stride (a multiple of 256): C/8 must divide 256.
static const char kBnGroupMsg[] = "needs 256 % (C / 8) == 0, i.e. C in {8, 16, 32, ..., 2048}";

extern "C" int vtx_stem_im2col(const float* img, void* cols, int N, int H, int W, int ldc, void* stream) {
  REQ(img && cols && ldc >= 152 && ldc % 8 == 0, "bad arguments");
  REQ(ldc <= 160 + 96, "bad arguments");
  const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
  const size_t smem = (size_t)21 * ((W + 8 + 3) / 4 * 4) * sizeof(float);
  REQ(smem <= 48 * 1024, "image too wide for the stem im2col tile");
  stem_im2col_kernel<<<N * Ho, 256, smem, STREAM>>>(img, (__nv_bfloat16*)cols, N, H, W, Ho, Wo, ldc);
  return check_launch("stem_im2col");
}
extern "C" int vtx_im2col3x3(const void* x, void* cols, int N, int H, int W, int C, int stride, void* stream) {
  REQ(x && cols && C % 8 == 0 && stride >= 1, "bad arguments");
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long total = (long long)N * Ho * Wo * 9 * (C / 8);
  if (total < (1LL << 31) - (1LL << 24)) {  // headroom: the grid-stride increment must not overflow either
    im2col3x3_i32_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)cols, N, H, W,
                                                                   C, Ho, Wo, stride);
    return check_launch("im2col3x3_i32");
  }
  im2col3x3_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)cols, N, H, W, C,
                                                             Ho, Wo, stride);
  return check_launch("im2col3x3");
}
extern "C" int vtx_col2im3x3(const void* dcols, void* dx, int N, int H, int W, int C, int stride, void* stream) {
  REQ(dcols && dx && C % 8 == 0 && stride >= 1, "bad arguments");
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long total = (long long)N * H * W * (C / 8);
  if (total < (1LL << 31) - (1LL << 24)) {
    col2im3x3_i32_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)dcols, (__nv_bfloat16*)dx, N, H, W,
                                                                   C, Ho, Wo, stride);
    return check_launch("col2im3x3_i32");
  }
  col2im3x3_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)dcols, (__nv_bfloat16*)dx, N, H, W,
                                                             C, Ho, Wo, stride);
  return check_launch("col2im3x3");
}
extern "C" int vtx_subsample(const void* x, void* xs, int N, int H, int W, int C, int stride, void* stream) {
  REQ(x && xs && C % 8 == 0, "bad arguments");
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long total = (long long)N * Ho * Wo * (C / 8);
  if (total < (1LL << 31) - (1LL << 24)) {
    subsample_i32_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)xs, N, H, W, C,
                                                                   Ho, Wo, stride);
    return check_launch("subsample_i32");
  }
  subsample_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)xs, N, H, W, C,
                                                             Ho, Wo, stride);
  return check_launch("subsample");
}
extern "C" int vtx_upsample_add(const void* dxs, void* dx, int N, int H, int W, int C, int stride, void* stream) {
  REQ(dxs && dx && C % 8 == 0, "bad arguments");
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long total = (long long)N * Ho * Wo * (C / 8);
  if (total < (1LL << 31) - (1LL << 24)) {
    upsample_add_i32_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)dxs, (__nv_bfloat16*)dx, N, H,
                                                                      W, C, Ho, Wo, stride);
    return check_launch("upsample_add_i32");
  }
  upsample_add_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)dxs, (__nv_bfloat16*)dx, N, H, W,
                                                                C, Ho, Wo, stride);
  return check_launch("upsample_add");
}
extern "C" int vtx_bn_finalize(const float* stats, float count, const float* gamma, const float* beta, float* rmean,
                               float* rvar, int64_t* nbt, float momentum, float eps, int training, float* bnp, int C,
                               void* stream) {
  REQ(gamma && beta && rmean && rvar && bnp && (stats || !training), "bad arguments");
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, STREAM>>>(stats, count, gamma, beta, rmean, rvar, (long long*)nbt,
                                                          momentum, eps, training, bnp, C);
  return check_launch("bn_finalize");
}
extern "C" int vtx_bn_act(const void* y, const float* bnp, const void* res, const float* bnp_res, void* out,
                          uint8_t* relu_mask, int64_t M, int C, int relu, void* stream) {
  REQ(y && bnp && out && C % 8 == 0, "bad arguments");
  REQ(C >= 8 && 256 % (C / 8) == 0, kBnGroupMsg);
  BnFwdFold f;
  memset(&f, 0, sizeof(f));
  if (res == nullptr)
    bn_act_kernel<false, 8><<<grid_for((M * (C / 8) + 7) / 8, 256, 2), 256, 0, STREAM>>>(
        (const __nv_bfloat16*)y, const_cast<float*>(bnp), nullptr, bnp_res, (__nv_bfloat16*)out, relu_mask, M, C, relu, f);
  else
    bn_act_kernel<false, kU><<<grid_for((M * (C / 8) + kU - 1) / kU, 256, 2), 256, 0, STREAM>>>(
        (const __nv_bfloat16*)y, const_cast<float*>(bnp), (const __nv_bfloat16*)res, bnp_res, (__nv_bfloat16*)out,
        relu_mask, M, C, relu, f);
  return check_launch("bn_act");
}
// bn_finalize + bn_act in one launch (the statistics -> scale/shift step runs in every thread's prologue)
extern "C" int vtx_bn_finalize_act(const float* stats, float count, const float* gamma, const float* beta, float* rmean,
                                   float* rvar, int64_t* nbt, float momentum, float eps, int training, float* bnp,
                                   const void* y, const void* res, const float* bnp_res, void* out, uint8_t* relu_mask,
                                   int64_t M, int C, int relu, void* stream) {
  REQ(y && bnp && out && gamma && beta && rmean && rvar && C % 8 == 0 && (stats || !training), "bad arguments");
  REQ(C >= 8 && 256 % (C / 8) == 0, kBnGroupMsg);
  BnFwdFold f;
  f.stats = stats; f.gamma = gamma; f.beta = beta; f.rmean = rmean; f.rvar = rvar; f.nbt = (long long*)nbt;
  f.count = count; f.momentum = momentum; f.eps = eps; f.training = training;
  if (res == nullptr)
    bn_act_kernel<true, 8><<<grid_for((M * (C / 8) + 7) / 8, 256, 2), 256, 0, STREAM>>>(
        (const __nv_bfloat16*)y, bnp, nullptr, bnp_res, (__nv_bfloat16*)out, relu_mask, M, C, relu, f);
  else
    bn_act_kernel<true, kU><<<grid_for((M * (C / 8) + kU - 1) / kU, 256, 2), 256, 0, STREAM>>>(
        (const __nv_bfloat16*)y, bnp, (const __nv_bfloat16*)res, bnp_res, (__nv_bfloat16*)out, relu_mask, M, C, relu, f);
  return check_launch("bn_finalize_act");
}
extern "C" int vtx_bn_relu_maxpool(const void* y, const float* bnp, void* out, uint8_t* idx, int N, int H, int W, int C,
                                   void* stream) {
  REQ(y && bnp && out && idx && C % 8 == 0, "bad arguments");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long long total = (long long)N * Ho * Wo * (C / 8);
  if (C / 8 <= 256 && (long long)H * W * C < (1LL << 31)) {
    bn_relu_maxpool_rows_kernel<<<(int)std::min<long long>((long long)N * Ho, (long long)vtx_num_sms() * 16),
                                  row_threads(C / 8, Wo), 0, STREAM>>>(
        (const __nv_bfloat16*)y, bnp, (__nv_bfloat16*)out, idx, N, H, W, C, Ho, Wo);
    return check_launch("bn_relu_maxpool_rows");
  }
  bn_relu_maxpool_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)y, bnp, (__nv_bfloat16*)out,
                                                                   idx, N, H, W, C, Ho, Wo);
  return check_launch("bn_relu_maxpool");
}
extern "C" int vtx_maxpool_bwd(const void* dpool, const uint8_t* idx, void* da, int N, int H, int W, int C,
                               void* stream) {
  REQ(dpool && idx && da && C % 8 == 0, "bad arguments");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  {
    const size_t smem = (size_t)(kTP + 1) * Wo * C * 3;  // bf16 gradients + u8 slots
    if (C % 16 == 0 && C / 8 <= 256 && smem <= 200 * 1024) {
      static size_t attr = 0;
      if (smem > 48 * 1024 && smem > attr) {
        cudaFuncSetAttribute(maxpool_bwd_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        attr = smem;
      }
      const int tiles = (Ho + kTP - 1) / kTP;
      maxpool_bwd_tiled_kernel<<<N * tiles, row_threads(C / 8, W), smem, STREAM>>>((const __nv_bfloat16*)dpool, idx, (__nv_bfloat16*)da, N,
                                                                 H, W, C, Ho, Wo);
      return check_launch("maxpool_bwd_tiled");
    }
  }
  const long long total = (long long)N * H * W * (C / 8);
  maxpool_bwd_kernel<<<grid_for(total, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)dpool, idx, (__nv_bfloat16*)da, N,
                                                               H, W, C, Ho, Wo);
  return check_launch("maxpool_bwd");
}
extern "C" int vtx_bn_bwd_reduce(const void* dA, const uint8_t* a, const void* y, const float* bnp, const void* y2,
                                 const float* bnp2, float* sums, float* sums2, int64_t M, int C, int mask_from_y,
                                 void* stream) {
  REQ(dA && y && bnp && sums && C % 8 == 0 && C / 8 <= 256, "bad arguments");
  const int threads = 256;
  const int rows_par = threads / (C / 8);
  const bool two = (y2 != nullptr);
  const size_t smem = (size_t)rows_par * C * (two ? 4 : 2) * sizeof(float);
  const int ku = y2 != nullptr ? kU : kUred;
  long long blocks = (M + (long long)rows_par * ku - 1) / ((long long)rows_par * ku);
  const long long cap = (long long)vtx_num_sms() * (two ? 1 : 2);
  if (blocks > cap) blocks = cap;
  if (two) {
    REQ(bnp2 && sums2, "second BN needs bnp2/sums2");
    bn_bwd_reduce_kernel<1, kU><<<(int)blocks, threads, smem, STREAM>>>((const __nv_bfloat16*)dA, (const uint8_t*)a,
                                                                    (const __nv_bfloat16*)y, bnp,
                                                                    (const __nv_bfloat16*)y2, bnp2, sums, sums2, M, C,
                                                                    mask_from_y);
  } else {
    bn_bwd_reduce_kernel<0, kUred><<<(int)blocks, threads, smem, STREAM>>>((const __nv_bfloat16*)dA, (const uint8_t*)a,
                                                                    (const __nv_bfloat16*)y, bnp, nullptr, nullptr,
                                                                    sums, nullptr, M, C, mask_from_y);
  }
  return check_launch("bn_bwd_reduce");
}
extern "C" int vtx_bn_bwd_finalize(const float* sums, const float* bnp, float count, float* coef, float* dgamma,
                                   float* dbeta, int C, void* stream) {
  REQ(sums && bnp && coef, "bad arguments");
  bn_bwd_finalize_kernel<<<(C + 127) / 128, 128, 0, STREAM>>>(sums, bnp, count, coef, dgamma, dbeta, C);
  return check_launch("bn_bwd_finalize");
}
static int launch_bn_bwd_apply(bool fold, const BnBwdFold& f, const void* dA, const uint8_t* a, const void* y,
                               const float* bnp, const float* coef, void* dy, const void* y2, const float* bnp2,
                               const float* coef2, void* dy2, void* dz_out, int64_t M, int C, int mask_from_y,
                               cudaStream_t st) {
  const int ku = y2 != nullptr ? kU : kUbwd;
  const int grid = grid_for((M * (C / 8) + ku - 1) / ku, 256, y2 != nullptr ? 1 : 2);
#define VTX_APPLY_ARGS (const __nv_bfloat16*)dA, (const uint8_t*)a, (const __nv_bfloat16*)y, bnp, coef,                \
                       (__nv_bfloat16*)dy, (const __nv_bfloat16*)y2, bnp2, coef2, (__nv_bfloat16*)dy2,                  \
                       (__nv_bfloat16*)dz_out, M, C, mask_from_y, f
  if (y2 != nullptr) {
    if (fold) bn_bwd_apply_kernel<1, true, kU><<<grid, 256, 0, st>>>(VTX_APPLY_ARGS);
    else bn_bwd_apply_kernel<1, false, kU><<<grid, 256, 0, st>>>(VTX_APPLY_ARGS);
  } else {
    if (fold) bn_bwd_apply_kernel<0, true, kUbwd><<<grid, 256, 0, st>>>(VTX_APPLY_ARGS);
    else bn_bwd_apply_kernel<0, false, kU><<<grid, 256, 0, st>>>(VTX_APPLY_ARGS);
  }
#undef VTX_APPLY_ARGS
  return check_launch("bn_bwd_apply");
}
extern "C" int vtx_bn_bwd_apply(const void* dA, const uint8_t* a, const void* y, const float* bnp, const float* coef,
                                void* dy, const void* y2, const float* bnp2, const float* coef2, void* dy2,
                                void* dz_out, int64_t M, int C, int mask_from_y, void* stream) {
  REQ(dA && y && bnp && coef && dy && C % 8 == 0, "bad arguments");
  REQ(C >= 8 && 256 % (C / 8) == 0, kBnGroupMsg);
  if (y2 != nullptr) REQ(bnp2 && coef2 && dy2, "second BN needs bnp2/coef2/dy2");
  BnBwdFold f;
  memset(&f, 0, sizeof(f));
  return launch_bn_bwd_apply(false, f, dA, a, y, bnp, coef, dy, y2, bnp2, coef2, dy2, dz_out, M, C, mask_from_y, STREAM);
}
// bn_bwd_finalize + bn_bwd_apply in one launch: sums [2,C] (and sums2) straight from vtx_bn_bwd_reduce
extern "C" int vtx_bn_bwd_finalize_apply(const float* sums, const float* sums2, float count, float* dgamma, float* dbeta,
                                         float* dgamma2, float* dbeta2, const void* dA, const uint8_t* a, const void* y,
                                         const float* bnp, void* dy, const void* y2, const float* bnp2, void* dy2,
                                         void* dz_out, int64_t M, int C, int mask_from_y, void* stream) {
  REQ(sums && dA && y && bnp && dy && C % 8 == 0, "bad arguments");
  REQ(C >= 8 && 256 % (C / 8) == 0, kBnGroupMsg);
  if (y2 != nullptr) REQ(bnp2 && sums2 && dy2, "second BN needs bnp2/sums2/dy2");
  BnBwdFold f;
  f.sums = sums; f.sums2 = sums2; f.dgamma = dgamma; f.dbeta = dbeta; f.dgamma2 = dgamma2; f.dbeta2 = dbeta2;
  f.count = count;
  return launch_bn_bwd_apply(true, f, dA, a, y, bnp, nullptr, dy, y2, bnp2, nullptr, dy2, dz_out, M, C, mask_from_y,
                             STREAM);
}
extern "C" int vtx_conv_w_pack(const float* w, void* out, int O, int I, int KH, int KW, int ldk, void* stream) {
  REQ(w && out && ldk >= KH * KW * I, "bad arguments");
  conv_w_pack_kernel<<<grid_for((long long)O * ldk, 256), 256, 0, STREAM>>>(w, (__nv_bfloat16*)out, O, I, KH, KW, ldk);
  return check_launch("conv_w_pack");
}
extern "C" int vtx_conv_w_pack_dgrad(const float* w, void* out, int O, int I, void* stream) {
  REQ(w && out, "bad arguments");
  conv_w_pack_dgrad_kernel<<<grid_for((long long)O * I * 9, 256), 256, 0, STREAM>>>(w, (__nv_bfloat16*)out, O, I);
  return check_launch("conv_w_pack_dgrad");
}
extern "C" int vtx_conv_w_unpack_add(const float* dwp, float* grad, int O, int I, int KH, int KW, int ldk,
                                     void* stream) {
  REQ(dwp && grad && ldk >= KH * KW * I, "bad arguments");
  conv_w_unpack_add_kernel<<<grid_for((long long)O * I * KH * KW, 256), 256, 0, STREAM>>>(dwp, grad, O, I, KH, KW, ldk);
  return check_launch("conv_w_unpack_add");
}
extern "C" int vtx_conv_w_unpack_add_t(const float* dwt, float* grad, int O, int I, int KH, int KW, void* stream) {
  REQ(dwt && grad, "bad arguments");
  conv_w_unpack_add_t_kernel<<<grid_for((long long)O * I * KH * KW, 256), 256, 0, STREAM>>>(dwt, grad, O, I, KH, KW);
  return check_launch("conv_w_unpack_add_t");
}
extern "C" int vtx_conv_w_jobs(const VtxWeightJob* jobs, int njobs, int total_blocks, void* stream) {
  REQ(jobs && njobs > 0 && total_blocks > 0, "bad arguments");
  conv_w_jobs_kernel<<<total_blocks, 256, 0, STREAM>>>(jobs, njobs);
  return check_launch("conv_w_jobs");
}
extern "C" int vtx_weight_job_block_elems(void) { return kJobElemsPerBlock; }
extern "C" int vtx_cast_bf16(const float* in, void* out, int64_t n, void* stream) {
  REQ(in && out && n >= 0, "bad arguments");
  if (n == 0) return VTX_OK;
  cast_bf16_kernel<<<grid_for(n / 4 + 1, 256), 256, 0, STREAM>>>(in, (__nv_bfloat16*)out, n);
  return check_launch("cast_bf16");
}
extern "C" int vtx_nhwc_to_nchw_f32(const void* in, float* out, int N, int HW, int C, void* stream) {
  REQ(in && out, "bad arguments");
  nhwc_to_nchw_f32_kernel<<<grid_for((long long)N * HW * C, 256), 256, 0, STREAM>>>((const __nv_bfloat16*)in, out, N,
                                                                                   HW, C);
  return check_launch("nhwc_to_nchw_f32");
}
