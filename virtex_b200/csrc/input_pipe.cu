// GPU input pipeline (SURVEY section 8 row f-3): decoded uint8 HWC images -> fp32 NCHW network input, and ragged
// caption token lists -> padded caption / reversed-caption matrices.  Replaces, for the training loop, the per-sample
// albumentations/cv2 CPU transforms and the collate of virtex/data/datasets/captioning.py:51-100 with the transform
// lists of virtex/factories.py:131-155:
//   train: random_resized_crop(224) -> horizontal_flip -> color_jitter(0.4, 0.4, 0.4, 0.1) -> normalize -> HWC->CHW
//   val  : smallest_resize(256) -> center_crop(224) -> normalize -> HWC->CHW
// Random parameters (crop box, flip coin, jitter factors and op order) are SAMPLED ON THE HOST and passed in; the
// kernels are deterministic functions of (image, parameters).  Integer arithmetic follows OpenCV's uint8 code paths
// bit for bit (11-bit fixed-point bilinear resize, 15-bit RGB2GRAY, 12-bit-table RGB2HSV, float32-fma addWeighted);
// every float op that must match the CPU oracle (oracle/input_pipeline.py) uses explicit _rn intrinsics so that the
// compiler cannot contract it into an fma the oracle does not perform.  HBM-bound byte work: one read of the crop,
// 3 B + 3 B per output pixel of intermediate traffic, 12 B per pixel of fp32 output.
#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {

// 11-bit coefficient pair and clamped source index of destination index d (cv::resize, INTER_LINEAR, 8U).
//   f = (float)((d + off + 0.5) * scale - 0.5);  s = floor(f);  f -= s
//   x direction (clamp_f): borders zero the fraction;  y direction: only the row index is clamped.
__device__ __forceinline__ void lin_coef(int d, int off, double scale, int n, bool clamp_f, int* i0, int* i1, int* a0,
                                         int* a1) {
  float f = (float)__dsub_rn(__dmul_rn((double)(d + off) + 0.5, scale), 0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (clamp_f) {
    if (s < 0) { s = 0; f = 0.f; }
    if (s >= n - 1) { s = n - 1; f = 0.f; }
  }
  *a0 = (int)rintf(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  *a1 = (int)rintf(__fmul_rn(f, 2048.f));
  *i0 = min(max(s, 0), n - 1);
  *i1 = min(max(s + 1, 0), n - 1);
}

// geom_i [B, 8] = {H, W, ry0, rx0, rh, rw, oy, ox}: source image size, source region (crop box), offset of the output
// window inside the resized region;  geom_d [B, 2] = {scale_y, scale_x} = region size / resized size (doubles).
__global__ void __launch_bounds__(256) image_resample_kernel(const uint8_t* __restrict__ src, const long long* __restrict__ src_off,
                                                            const int* __restrict__ geom_i, const double* __restrict__ geom_d,
                                                            const int* __restrict__ jit_i, uint8_t* __restrict__ out, int S) {
  VTX_PDL_TRIGGER();
  const int n = blockIdx.y;
  const int* gi = geom_i + n * 8;
  const int W = gi[1], ry0 = gi[2], rx0 = gi[3], rh = gi[4], rw = gi[5], oy = gi[6], ox = gi[7];
  const double sy = geom_d[2 * n], sx = geom_d[2 * n + 1];
  const bool flip = jit_i[n * 6] != 0;
  const uint8_t* img = src + src_off[n];
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < S * S; p += gridDim.x * blockDim.x) {
    const int y = p / S, x = p - y * S;
    int x0, x1, ax0, ax1, y0, y1, by0, by1;
    lin_coef(x, ox, sx, rw, true, &x0, &x1, &ax0, &ax1);
    lin_coef(y, oy, sy, rh, false, &y0, &y1, &by0, &by1);
    const uint8_t* r0 = img + ((long long)(ry0 + y0) * W + rx0) * 3;
    const uint8_t* r1 = img + ((long long)(ry0 + y1) * W + rx0) * 3;
    uint8_t* o = out + ((long long)n * S * S + (long long)y * S + (flip ? S - 1 - x : x)) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int h0 = (int)r0[x0 * 3 + c] * ax0 + (int)r0[x1 * 3 + c] * ax1;
      const int h1 = (int)r1[x0 * 3 + c] * ax0 + (int)r1[x1 * 3 + c] * ax1;
      const int v = (((by0 * (h0 >> 4)) >> 16) + ((by1 * (h1 >> 4)) >> 16) + 2) >> 2;
      o[c] = (uint8_t)min(max(v, 0), 255);
    }
  }
}

// ------------------------------------------------------------------------------------------------ colour ops (uint8)
__device__ __forceinline__ int gray15(int r, int g, int b) { return (r * 9798 + g * 19235 + b * 3735 + (1 << 14)) >> 15; }

// uint8 LUT entry clip(v * scale + bias, 0, 255) truncated, evaluated in float64 like numpy builds the table
__device__ __forceinline__ int lut_affine(int v, double scale, double bias) {
  double t = __dadd_rn(__dmul_rn((double)v, scale), bias);
  t = fmin(fmax(t, 0.0), 255.0);
  return (int)t;
}

__device__ __forceinline__ void op_saturation(int* px, double s) {
  const float al = (float)s, be = (float)(1.0 - s);
  const float g = (float)gray15(px[0], px[1], px[2]);
  const float t = __fmul_rn(g, be);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = rintf(__fmaf_rn((float)px[c], al, t));
    px[c] = (int)fminf(fmaxf(v, 0.f), 255.f);
  }
}

__device__ __forceinline__ void op_hue(int* px, double hf) {
  const int r = px[0], g = px[1], b = px[2];
  const int v = max(max(r, g), b), diff = v - min(min(r, g), b);
  const long long sdiv = v > 0 ? (long long)rint(1044480.0 / (double)v) : 0;             // (255 << 12) / v
  const long long hdiv = diff > 0 ? (long long)rint(737280.0 / (6.0 * (double)diff)) : 0;  // (180 << 12) / (6 diff)
  const int s8 = (int)(((long long)diff * sdiv + 2048) >> 12);
  long long h = (v == r) ? (g - b) : (v == g) ? (b - r + 2 * diff) : (r - g + 4 * diff);
  h = (h * hdiv + 2048) >> 12;
  if (h < 0) h += 180;
  // hue LUT: mod(h + 180 * factor, 180) in float64 (numpy's sign-of-divisor modulo), truncated to uint8
  double m = fmod(__dadd_rn((double)h, __dmul_rn(180.0, hf)), 180.0);
  if (m != 0.0 && m < 0.0) m += 180.0;
  const int h8 = (int)m;
  // HSV -> RGB (float32, truncating store)
  const float hh = __fmul_rn((float)h8, (float)(6.0 / 180.0));
  const float ss = __fmul_rn((float)s8, (float)(1.0 / 255.0));
  const float vv = __fmul_rn((float)v, (float)(1.0 / 255.0));
  int sector = (int)floorf(hh);
  const float f = __fsub_rn(hh, (float)sector);
  sector %= 6;
  float tab[4];
  tab[0] = vv;
  tab[1] = __fmul_rn(vv, __fsub_rn(1.f, ss));
  tab[2] = __fmul_rn(vv, __fsub_rn(1.f, __fmul_rn(ss, f)));
  tab[3] = __fmul_rn(vv, __fsub_rn(1.f, __fmul_rn(ss, __fsub_rn(1.f, f))));
  // sector table of OpenCV (b, g, r): {1,3,0} {1,0,2} {3,0,1} {0,2,1} {0,1,3} {2,1,0}
  int ib, ig, ir;
  switch (sector) {
    case 0: ib = 1; ig = 3; ir = 0; break;
    case 1: ib = 1; ig = 0; ir = 2; break;
    case 2: ib = 3; ig = 0; ir = 1; break;
    case 3: ib = 0; ig = 2; ir = 1; break;
    case 4: ib = 0; ig = 1; ir = 3; break;
    default: ib = 2; ig = 1; ir = 0; break;
  }
  const float o[3] = {tab[ir], tab[ig], tab[ib]};
#pragma unroll
  for (int c = 0; c < 3; ++c) px[c] = (int)fminf(fmaxf(floorf(__fmul_rn(o[c], 255.f)), 0.f), 255.f);
}

// Applies the jitter ops of `order` to one pixel, stopping BEFORE op `stop_at` (4 = apply all).  jf = {brightness,
// contrast, saturation, hue} factors (doubles), mean = grey mean of the image at the contrast stage.
__device__ __forceinline__ void apply_jitter(int* px, const double* jf, const int* order, int stop_at, double mean) {
#pragma unroll 1
  for (int k = 0; k < 4; ++k) {
    const int op = order[k];
    if (op == stop_at) return;
    if (op == 0) {
      if (jf[0] != 1.0)
        for (int c = 0; c < 3; ++c) px[c] = lut_affine(px[c], jf[0], 0.0);
    } else if (op == 1) {
      if (jf[1] == 0.0) {
        const int m = (int)(mean + 0.5);
        px[0] = px[1] = px[2] = m;
      } else if (jf[1] != 1.0) {
        const double bias = __dmul_rn(mean, __dsub_rn(1.0, jf[1]));
        for (int c = 0; c < 3; ++c) px[c] = lut_affine(px[c], jf[1], bias);
      }
    } else if (op == 2) {
      if (jf[2] == 0.0) {
        const int g = gray15(px[0], px[1], px[2]);
        px[0] = px[1] = px[2] = g;
      } else if (jf[2] != 1.0) {
        op_saturation(px, jf[2]);
      }
    } else {
      if (jf[3] != 0.0) op_hue(px, jf[3]);
    }
  }
}

// jit_i [B, 6] = {flip, apply, order[4]};  jit_d [B, 4].  gray_sum[n] += sum of the grey values of image n at the stage
// where contrast is applied (exact integer sum; the mean is sum / (S*S) in float64 like cv2's mean()).
__global__ void __launch_bounds__(256) image_gray_sum_kernel(const uint8_t* __restrict__ img, const int* __restrict__ jit_i,
                                                            const double* __restrict__ jit_d,
                                                            unsigned long long* __restrict__ gray_sum, int S) {
  VTX_PDL_TRIGGER();
  const int n = blockIdx.y;
  const int* ji = jit_i + n * 6;
  if (!ji[1] || jit_d[n * 4 + 1] == 1.0) return;  // no jitter, or contrast is the identity
  double jf[4];
  int order[4];
  for (int k = 0; k < 4; ++k) { jf[k] = jit_d[n * 4 + k]; order[k] = ji[2 + k]; }
  unsigned long long acc = 0;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < S * S; p += gridDim.x * blockDim.x) {
    const uint8_t* q = img + ((long long)n * S * S + p) * 3;
    int px[3] = {q[0], q[1], q[2]};
    apply_jitter(px, jf, order, 1, 0.0);
    acc += (unsigned long long)gray15(px[0], px[1], px[2]);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(gray_sum + n, acc);
}

// norm = {m[3], inv[3]}: out = (v - m) * inv, written as fp32 NCHW [B, 3, S, S]
__global__ void __launch_bounds__(256) image_jitter_normalize_kernel(const uint8_t* __restrict__ img, const int* __restrict__ jit_i,
                                                                    const double* __restrict__ jit_d,
                                                                    const unsigned long long* __restrict__ gray_sum,
                                                                    const float* __restrict__ norm, float* __restrict__ out,
                                                                    int S) {
  VTX_PDL_TRIGGER();
  const int n = blockIdx.y;
  const int* ji = jit_i + n * 6;
  const bool apply = ji[1] != 0;
  double jf[4];
  int order[4];
  for (int k = 0; k < 4; ++k) { jf[k] = jit_d[n * 4 + k]; order[k] = ji[2 + k]; }
  const double mean = (double)gray_sum[n] / (double)((long long)S * S);
  const float m0 = norm[0], m1 = norm[1], m2 = norm[2], i0 = norm[3], i1 = norm[4], i2 = norm[5];
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < S * S; p += gridDim.x * blockDim.x) {
    const uint8_t* q = img + ((long long)n * S * S + p) * 3;
    int px[3] = {q[0], q[1], q[2]};
    if (apply) apply_jitter(px, jf, order, 4, mean);
    float* o = out + (long long)n * 3 * S * S + p;
    o[0] = __fmul_rn(__fsub_rn((float)px[0], m0), i0);
    o[(long long)S * S] = __fmul_rn(__fsub_rn((float)px[1], m1), i1);
    o[2LL * S * S] = __fmul_rn(__fsub_rn((float)px[2], m2), i2);
  }
}

// flat tokens + offsets [B+1] -> caption_tokens / noitpac_tokens [B, T] right-padded with `pad`, lengths [B]
// (captioning.py:68-100; captions longer than max_len are trimmed from the right before being reversed)
__global__ void collate_tokens_kernel(const long long* __restrict__ flat, const long long* __restrict__ offs,
                                      long long* __restrict__ cap, long long* __restrict__ rev,
                                      long long* __restrict__ lengths, int B, int T, int max_len, long long pad) {
  VTX_PDL_TRIGGER();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * T) return;
  const int b = i / T, t = i - b * T;
  const long long o = offs[b];
  const int len = (int)min((long long)max_len, offs[b + 1] - o);
  cap[i] = t < len ? flat[o + t] : pad;
  rev[i] = t < len ? flat[o + len - 1 - t] : pad;
  if (t == 0) lengths[b] = len;
}

// The masked-LM collate: vtx_collate_tokens' trim + right-pad, then virtex/data/datasets/masked_lm.py:64-91's masking
// of every caption.  One CTA per caption, one thread per position; a caption of trimmed length n picks
// k = ceil((n - 2) * proportion) of its positions 1 .. n-2: the k smallest (key, position) pairs, each key an
// independent 64-bit hash, so every k-subset is equally likely (random.sample's distribution).  A picked position
// becomes [MASK] (label = the original id) when k == 1 or its uniform u <= mask_prob, a uniform id of [0, vocab) (no
// label) when u <= mask_prob + replace_prob, and stays as it is (no label) otherwise.  All draws are hash_u64 of
// (seed, site, caption << 32 | position): the host replays them bit for bit (tests/masked_lm_oracle.py).
constexpr uint32_t kMlmKeySite = 5000u, kMlmFlagSite = 5001u, kMlmTokenSite = 5002u;  // dropout < 2000, nucleus 4000

__global__ void __launch_bounds__(VTX_MLM_MAX_T) collate_masked_lm_kernel(
    const long long* __restrict__ flat, const long long* __restrict__ offs, long long* __restrict__ cap,
    long long* __restrict__ labels, long long* __restrict__ lengths, int T, int max_len, long long pad, long long mask_id,
    long long vocab, double proportion, double mask_prob, double replace_prob, const uint64_t* __restrict__ seed_ptr) {
  VTX_PDL_TRIGGER();
  __shared__ uint64_t keys[VTX_MLM_MAX_T];
  const int b = blockIdx.x, t = threadIdx.x;
  const long long o = offs[b];
  const int n = (int)min((long long)max_len, offs[b + 1] - o);
  const uint64_t seed = *seed_ptr;
  const uint64_t ctr = ((uint64_t)b << 32) | (uint32_t)t;
  const bool cand = t >= 1 && t < n - 1;
  if (t < T) keys[t] = cand ? hash_u64(seed, kMlmKeySite, ctr) : 0ull;
  __syncthreads();
  if (t >= T) return;
  long long tok = t < n ? flat[o + t] : pad, lab = pad;
  if (cand) {
    const int k = (int)ceil(__dmul_rn((double)(n - 2), proportion));  // Python's math.ceil((n - 2) * p), p <= 1
    const uint64_t mine = keys[t];
    int rank = 0;
    for (int q = 1; q < n - 1; ++q) {
      const uint64_t kq = keys[q];
      rank += (kq < mine) || (kq == mine && q < t);
    }
    if (rank < k) {
      bool mask = k == 1;
      if (!mask) {
        const double u = (double)(hash_u64(seed, kMlmFlagSite, ctr) >> 11) * 0x1p-53;
        if (u <= mask_prob)
          mask = true;
        else if (u <= __dadd_rn(mask_prob, replace_prob))
          tok = (long long)__umul64hi(hash_u64(seed, kMlmTokenSite, ctr), (uint64_t)vocab);
      }
      if (mask) {
        lab = tok;
        tok = mask_id;
      }
    }
  }
  cap[(long long)b * T + t] = tok;
  labels[(long long)b * T + t] = lab;
  if (t == 0) lengths[b] = n;
}

}  // namespace vtx

using namespace vtx;
#define STREAM reinterpret_cast<cudaStream_t>(stream)

extern "C" int vtx_image_resample(const uint8_t* src, const int64_t* src_off, const int32_t* geom_i, const double* geom_d,
                                  const int32_t* jit_i, uint8_t* out, int B, int S, void* stream) {
  if (!src || !src_off || !geom_i || !geom_d || !jit_i || !out || B <= 0 || S <= 0)
    return set_error(VTX_EINVAL, "vtx_image_resample: bad arguments");
  const int bx = (S * S + 255) / 256;
  image_resample_kernel<<<dim3(bx, B), 256, 0, STREAM>>>(src, (const long long*)src_off, geom_i, geom_d, jit_i, out, S);
  return check_launch("image_resample");
}
extern "C" int vtx_image_gray_sum(const uint8_t* img, const int32_t* jit_i, const double* jit_d, uint64_t* gray_sum, int B,
                                  int S, void* stream) {
  if (!img || !jit_i || !jit_d || !gray_sum || B <= 0 || S <= 0) return set_error(VTX_EINVAL, "vtx_image_gray_sum: bad arguments");
  image_gray_sum_kernel<<<dim3(8, B), 256, 0, STREAM>>>(img, jit_i, jit_d, (unsigned long long*)gray_sum, S);
  return check_launch("image_gray_sum");
}
extern "C" int vtx_image_jitter_normalize(const uint8_t* img, const int32_t* jit_i, const double* jit_d,
                                          const uint64_t* gray_sum, const float* norm, float* out, int B, int S,
                                          void* stream) {
  if (!img || !jit_i || !jit_d || !gray_sum || !norm || !out || B <= 0 || S <= 0)
    return set_error(VTX_EINVAL, "vtx_image_jitter_normalize: bad arguments");
  const int bx = (S * S + 255) / 256;
  image_jitter_normalize_kernel<<<dim3(bx, B), 256, 0, STREAM>>>(img, jit_i, jit_d, (const unsigned long long*)gray_sum,
                                                                 norm, out, S);
  return check_launch("image_jitter_normalize");
}
extern "C" int vtx_collate_tokens(const int64_t* flat, const int64_t* offs, int64_t* cap, int64_t* rev, int64_t* lengths,
                                  int B, int T, int max_len, int64_t pad, void* stream) {
  if (!flat || !offs || !cap || !rev || !lengths || B <= 0 || T <= 0) return set_error(VTX_EINVAL, "vtx_collate_tokens: bad arguments");
  collate_tokens_kernel<<<(B * T + 255) / 256, 256, 0, STREAM>>>((const long long*)flat, (const long long*)offs,
                                                                 (long long*)cap, (long long*)rev, (long long*)lengths, B,
                                                                 T, max_len, (long long)pad);
  return check_launch("collate_tokens");
}
extern "C" int vtx_collate_masked_lm(const int64_t* flat, const int64_t* offs, int64_t* cap, int64_t* labels,
                                     int64_t* lengths, int B, int T, int max_len, int64_t pad, int64_t mask_id,
                                     int64_t vocab, double proportion, double mask_prob, double replace_prob,
                                     const uint64_t* seed, void* stream) {
  const auto prob = [](double p) { return p >= 0.0 && p <= 1.0; };  // false for NaN
  if (!flat || !offs || !cap || !labels || !lengths || !seed || B <= 0 || T <= 0 || T > VTX_MLM_MAX_T || vocab <= 0 ||
      !prob(proportion) || !prob(mask_prob) || !prob(replace_prob))
    return set_error(VTX_EINVAL, "vtx_collate_masked_lm: bad arguments (T <= %d, probabilities in [0, 1], vocab > 0)",
                     VTX_MLM_MAX_T);
  const int threads = (T + 31) / 32 * 32;
  collate_masked_lm_kernel<<<B, threads, 0, STREAM>>>((const long long*)flat, (const long long*)offs, (long long*)cap,
                                                      (long long*)labels, (long long*)lengths, T, max_len,
                                                      (long long)pad, (long long)mask_id, (long long)vocab, proportion,
                                                      mask_prob, replace_prob, seed);
  return check_launch("collate_masked_lm");
}
