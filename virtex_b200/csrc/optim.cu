// Fused optimiser tail over the flat fp32 parameter / gradient arenas (SURVEY.md section 8f-1):
//   global L2 norm -> clip coefficient (x 1/world_size for the DDP mean) -> SGD(momentum) or AdamW, both with
//   per-tensor lr / weight decay -> optional Lookahead interpolation -> refreshed bf16 copy of the parameters for the
//   next step's GEMMs.
// Reference semantics: scripts/pretrain_virtex.py:157-162, virtex/factories.py:503-545 (one param group per tensor),
// torch.optim.SGD (first step: buf = g), torch.optim.AdamW (default betas / eps), virtex/optim/lookahead.py:82-102.
#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {

__global__ void sumsq_kernel(const float* __restrict__ x, long long n, float* __restrict__ out) {
  VTX_PDL_TRIGGER();
  float acc = 0.f;
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  for (long long i = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc += x[i] * x[i];
  __shared__ float red[32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) atomicAdd(out, v);
  }
}

// ctl[0] = grad scale applied in the update = (1/world) * min(1, max_norm / (norm + 1e-6)),  ctl[1] = norm of the mean grad
// The clamp keeps a NaN coefficient, as torch.clamp(coef, max=1) in clip_grad_norm_ does (fminf would return 1 and
// let a NaN-norm step run unclipped); an inf norm gives 0.  max_norm <= 0 means no clipping.
__global__ void clip_coef_kernel(const float* __restrict__ sumsq, float inv_world, float max_norm, float* __restrict__ ctl) {
  VTX_PDL_TRIGGER();
  const float norm = sqrtf(*sumsq) * inv_world;
  float c = max_norm > 0.f ? max_norm / (norm + 1e-6f) : 1.f;
  c = c > 1.f ? 1.f : c;
  ctl[0] = c * inv_world;
  ctl[1] = norm;
}

struct Seg {  // one parameter tensor inside the flat arena
  long long begin, end;
  float lr, wd;
};

// hyper[0] = lr multiplier of this step, hyper[1] = 1 on the very first optimiser step (momentum buffer := grad),
// hyper[2] = 1 when this step ends a Lookahead cycle.
__global__ void sgd_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ mom,
                                float* __restrict__ slow, __nv_bfloat16* __restrict__ p_bf, const Seg* __restrict__ segs,
                                int nseg, const float* __restrict__ ctl, const float* __restrict__ hyper, float momentum,
                                float la_alpha) {
  VTX_PDL_TRIGGER();
  const float gscale = ctl[0];
  const float mult = hyper[0];
  const bool first = hyper[1] != 0.f;
  const bool do_la = hyper[2] != 0.f;
  for (int s = blockIdx.y; s < nseg; s += gridDim.y) {
    const Seg sg = segs[s];
    const float lr = sg.lr * mult;
    for (long long i = sg.begin + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < sg.end;
         i += (long long)gridDim.x * blockDim.x) {
      float w = p[i];
      const float gg = g[i] * gscale + sg.wd * w;
      const float m = first ? gg : momentum * mom[i] + gg;
      mom[i] = m;
      w -= lr * m;
      if (do_la && slow != nullptr) {
        w = la_alpha * w + (1.f - la_alpha) * slow[i];
        slow[i] = w;
      }
      p[i] = w;
      if (p_bf != nullptr) p_bf[i] = f2bf(w);
    }
  }
}

// torch.optim.AdamW (amsgrad off, single step count for every tensor) with the same segment table and launch shape.
// hyper[0] = lr multiplier of this step, hyper[1] = 1 / (1 - beta1^t), hyper[2] = 1 / sqrt(1 - beta2^t) (both from the
// host's double-precision step count), hyper[3] = 1 when this step ends a Lookahead cycle.  c1 = 1 - beta1 and
// c2 = 1 - beta2 come from double precision (in fp32, 1 - 0.999f is 1.3e-5 off 0.001), as torch's scalars do.
__global__ void adamw_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ exp_avg,
                                  float* __restrict__ exp_avg_sq, float* __restrict__ slow,
                                  __nv_bfloat16* __restrict__ p_bf, const Seg* __restrict__ segs, int nseg,
                                  const float* __restrict__ ctl, const float* __restrict__ hyper, float c1,
                                  float beta2, float c2, float eps, float la_alpha) {
  VTX_PDL_TRIGGER();
  const float gscale = ctl[0];
  const float mult = hyper[0];
  const float inv_bc1 = hyper[1];
  const float inv_sqrt_bc2 = hyper[2];
  const bool do_la = hyper[3] != 0.f;
  for (int s = blockIdx.y; s < nseg; s += gridDim.y) {
    const Seg sg = segs[s];
    const float lr = sg.lr * mult;
    const float decay = 1.f - lr * sg.wd;  // decoupled weight decay, applied before the moments as torch does
    const float step_size = lr * inv_bc1;
    for (long long i = sg.begin + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < sg.end;
         i += (long long)gridDim.x * blockDim.x) {
      const float gg = g[i] * gscale;
      float m = exp_avg[i];
      m += c1 * (gg - m);  // torch: exp_avg.lerp_(grad, 1 - beta1)
      const float v = beta2 * exp_avg_sq[i] + c2 * gg * gg;
      exp_avg[i] = m;
      exp_avg_sq[i] = v;
      float w = p[i] * decay;
      w -= step_size * m / (sqrtf(v) * inv_sqrt_bc2 + eps);
      if (do_la && slow != nullptr) {
        w = la_alpha * w + (1.f - la_alpha) * slow[i];
        slow[i] = w;
      }
      p[i] = w;
      if (p_bf != nullptr) p_bf[i] = f2bf(w);
    }
  }
}

}  // namespace vtx

using namespace vtx;
#define STREAM reinterpret_cast<cudaStream_t>(stream)
#define REQ(cond, msg) \
  if (!(cond)) return set_error(VTX_EINVAL, "%s: %s", __func__, msg)

extern "C" int vtx_sumsq(const float* x, int64_t n, float* out, void* stream) {
  REQ(x && out && n >= 0, "bad arguments");
  if (n == 0) return VTX_OK;
  long long blocks = (n / 4 + 255) / 256;
  const long long cap = (long long)vtx_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  sumsq_kernel<<<(int)blocks, 256, 0, STREAM>>>(x, n, out);
  return check_launch("sumsq");
}
extern "C" int vtx_clip_coef(const float* sumsq, int world_size, float max_norm, float* ctl, void* stream) {
  REQ(sumsq && ctl && world_size >= 1, "bad arguments");
  clip_coef_kernel<<<1, 1, 0, STREAM>>>(sumsq, 1.0f / (float)world_size, max_norm, ctl);
  return check_launch("clip_coef");
}
extern "C" int vtx_sgd_step(float* p, const float* g, float* mom, float* slow, void* p_bf, const void* segs, int nseg,
                            const float* ctl, const float* hyper, float momentum, float la_alpha, void* stream) {
  REQ(p && g && mom && segs && nseg > 0 && ctl && hyper, "bad arguments");
  dim3 grid(4, nseg < 65535 ? nseg : 65535);  // callers pass chunks of <= 64 Ki elements
  sgd_step_kernel<<<grid, 256, 0, STREAM>>>(p, g, mom, slow, (__nv_bfloat16*)p_bf, (const Seg*)segs, nseg, ctl, hyper,
                                            momentum, la_alpha);
  return check_launch("sgd_step");
}
extern "C" int vtx_adamw_step(float* p, const float* g, float* exp_avg, float* exp_avg_sq, float* slow, void* p_bf,
                              const void* segs, int nseg, const float* ctl, const float* hyper, double beta1,
                              double beta2, float eps, float la_alpha, void* stream) {
  REQ(p && g && exp_avg && exp_avg_sq && segs && nseg > 0 && ctl && hyper, "bad arguments");
  dim3 grid(4, nseg < 65535 ? nseg : 65535);  // callers pass chunks of <= 64 Ki elements
  adamw_step_kernel<<<grid, 256, 0, STREAM>>>(p, g, exp_avg, exp_avg_sq, slow, (__nv_bfloat16*)p_bf, (const Seg*)segs,
                                              nseg, ctl, hyper, (float)(1.0 - beta1), (float)beta2,
                                              (float)(1.0 - beta2), eps, la_alpha);
  return check_launch("adamw_step");
}
