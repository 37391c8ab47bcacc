// Kernels of the classification pretext models (token / multilabel classification): global average pooling of the
// backbone's NHWC feature rows and its adjoint, the K-hot cross entropy (forward + dlogits in place) and a per-row top-k.
// Reference semantics: virtex/modules/textual_heads.py:46-95 (LinearTextualHead: mean over h*w, then nn.Linear) and
// virtex/models/classification.py:43-108 (mean over the UNIQUE non-ignored labels of a row of -log_softmax, mean over
// the batch; eval predictions = logprobs.topk(10)).  The linear layer itself is the wgmma GEMM (gemm_tc.cu).
#include <math.h>

#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {

constexpr int kKhotThreads = 256;
constexpr int kTopkThreads = 256;

// ------------------------------------------------------------------------------------------------ global average pool
// pooled[b, c] = bf16( (1 / hw) * sum_i feat[b*hw + i, c] ), fp32 accumulation; one thread per 8 channels of one image
__global__ void group_mean_fwd_kernel(const __nv_bfloat16* __restrict__ feat, __nv_bfloat16* __restrict__ pooled, int HW,
                                      int C) {
  VTX_PDL_TRIGGER();
  const int b = blockIdx.x;
  const int c8 = blockIdx.y * blockDim.x + threadIdx.x;
  if (c8 * 8 >= C) return;
  const __nv_bfloat16* src = feat + (long long)b * HW * C + c8 * 8;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll 7
  for (int i = 0; i < HW; ++i) {
    float f[8];
    unpack8(*reinterpret_cast<const bf16x8*>(src + (long long)i * C), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += f[j];
  }
  const float inv = 1.f / (float)HW;
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] *= inv;
  *reinterpret_cast<bf16x8*>(pooled + (long long)b * C + c8 * 8) = pack8(acc);
}

// dfeat[b*hw + i, c] = bf16( dpooled[b, c] / hw ); grid-stride over 8-channel groups of the output
__global__ void group_mean_bwd_kernel(const __nv_bfloat16* __restrict__ dpooled, __nv_bfloat16* __restrict__ dfeat,
                                      long long n8, int HW, int C8, float inv) {
  VTX_PDL_TRIGGER();
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n8; v += (long long)gridDim.x * blockDim.x) {
    const long long r = v / C8;
    const int c8 = (int)(v - r * C8);
    const long long b = r / HW;
    float f[8];
    unpack8(*reinterpret_cast<const bf16x8*>(dpooled + (b * C8 + c8) * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= inv;
    *reinterpret_cast<bf16x8*>(dfeat + v * 8) = pack8(f);
  }
}

// ------------------------------------------------------------------------------------------------ K-hot cross entropy
// block-wide sums of two values (all threads receive both); `red` holds 2 x 32 floats
__device__ __forceinline__ void block_sum2(float& a, float& b, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  a = warp_sum(a);
  b = warp_sum(b);
  __syncthreads();  // `red` may still be read by a previous reduction
  if (lane == 0) { red[warp] = a; red[32 + warp] = b; }
  __syncthreads();
  a = lane < nwarps ? red[lane] : 0.f;
  b = lane < nwarps ? red[32 + lane] : 0.f;
  a = warp_sum(a);
  b = warp_sum(b);
}
__device__ __forceinline__ float block_max(float a, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  a = warp_max(a);
  __syncthreads();
  if (lane == 0) red[warp] = a;
  __syncthreads();
  a = lane < nwarps ? red[lane] : -INFINITY;
  return warp_max(a);
}

// One CTA per row b of bf16 logits [B, ldl] (V valid columns).  U_b = the distinct ids of labels[b, 0:L] that lie in
// [0, V) and are not in `ignore`; K = |U_b|.  A bitmap over V in shared memory deduplicates: the ignored ids are set
// first, so a label equal to one of them never wins the atomicOr that admits a new id, and they are cleared again
// before the gradient pass, leaving exactly U_b.  Labels outside [0, V) are skipped: they are never read as a column.
//   loss += inv_b * (lse_b - (1/K) sum_{u in U_b} z[b, u])          (NaN when K = 0, as the mean over an empty set)
//   write_grad: z[b, v] := inv_b * (softmax_v - [v in U_b] / K)      (all zeros when K = 0)
__global__ void __launch_bounds__(kKhotThreads) khot_xent_kernel(
    __nv_bfloat16* __restrict__ logits, long long ldl, const long long* __restrict__ labels, long long ldlab, int L, int V,
    const long long* __restrict__ ignore, int n_ignore, float inv_b, float* __restrict__ loss, int write_grad) {
  VTX_PDL_TRIGGER();
  __shared__ uint32_t bits[VTX_KHOT_MAX_V / 32];
  __shared__ float red[64];
  const int row = blockIdx.x;
  __nv_bfloat16* z = logits + (long long)row * ldl;
  const long long* lab = labels + (long long)row * ldlab;
  const int nwords = (V + 31) >> 5;
  for (int i = threadIdx.x; i < nwords; i += blockDim.x) bits[i] = 0u;
  __syncthreads();
  for (int i = threadIdx.x; i < n_ignore; i += blockDim.x) {
    const long long id = ignore[i];
    if (id >= 0 && id < V) atomicOr(&bits[id >> 5], 1u << (id & 31));
  }
  __syncthreads();
  float k = 0.f, zsum = 0.f;
  for (int j = threadIdx.x; j < L; j += blockDim.x) {
    const long long id = lab[j];
    if (id < 0 || id >= V) continue;
    const uint32_t bit = 1u << (id & 31);
    if (!(atomicOr(&bits[id >> 5], bit) & bit)) {  // first occurrence of a non-ignored id
      k += 1.f;
      zsum += bf2f(z[id]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_ignore; i += blockDim.x) {
    const long long id = ignore[i];
    if (id >= 0 && id < V) atomicAnd(&bits[id >> 5], ~(1u << (id & 31)));
  }
  // (the barriers of the reductions below order these clears before the gradient pass)
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, bf2f(z[v]));
  mx = block_max(mx, red);
  float s = 0.f, unused = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) s += expf(bf2f(z[v]) - mx);
  block_sum2(s, unused, red);
  block_sum2(k, zsum, red);
  if (threadIdx.x == 0) atomicAdd(loss, k > 0.f ? (mx + logf(s) - zsum / k) * inv_b : NAN);
  if (!write_grad) return;
  const float inv_s = 1.f / s, inv_k = k > 0.f ? 1.f / k : 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    float g = 0.f;
    if (k > 0.f) {
      const float on = (bits[v >> 5] >> (v & 31)) & 1u ? inv_k : 0.f;
      g = (expf(bf2f(z[v]) - mx) * inv_s - on) * inv_b;
    }
    z[v] = f2bf(g);
  }
}

// ------------------------------------------------------------------------------------------------ top-k
// (v, i) precedes (w, j) in the output order iff v > w, or v == w and i < j
__device__ __forceinline__ bool topk_before(float v, int i, float w, int j) { return v > w || (v == w && i < j); }

// One CTA per row of fp32 X [M, ld]: the k largest of N values, descending, ties broken by the lower index; NaN ranks
// as -inf.  Round r picks the first element (in that order) that comes after the pick of round r - 1, so no list of
// earlier picks is kept.
__global__ void __launch_bounds__(kTopkThreads) topk_rows_kernel(const float* __restrict__ X, long long ld, int N, int k,
                                                                  long long* __restrict__ out) {
  VTX_PDL_TRIGGER();
  __shared__ float sv[32];
  __shared__ int si[32];
  const float* x = X + (long long)blockIdx.x * ld;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  float pv = INFINITY;
  int pi = -1;
  for (int r = 0; r < k; ++r) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      float v = x[i];
      if (isnan(v)) v = -INFINITY;
      if (topk_before(pv, pi, v, i) && topk_before(v, i, bv, bi)) { bv = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (topk_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    __syncthreads();  // the previous round's readers of sv / si are done
    if (lane == 0) { sv[warp] = bv; si[warp] = bi; }
    __syncthreads();
    bv = lane < nwarps ? sv[lane] : -INFINITY;
    bi = lane < nwarps ? si[lane] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (topk_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (threadIdx.x == 0) out[(long long)blockIdx.x * k + r] = bi;
    pv = bv;
    pi = bi;
  }
}

}  // namespace vtx

using namespace vtx;
#define STREAM reinterpret_cast<cudaStream_t>(stream)
#define REQ(cond, msg) \
  if (!(cond)) return set_error(VTX_EINVAL, "%s: %s", __func__, msg)

extern "C" int vtx_group_mean_fwd(const void* feat, void* pooled, int B, int HW, int C, void* stream) {
  REQ(feat && pooled && B > 0 && HW > 0 && C > 0 && C % 8 == 0, "needs C % 8 == 0 and a non-empty input");
  REQ(((reinterpret_cast<uintptr_t>(feat) | reinterpret_cast<uintptr_t>(pooled)) & 15) == 0, "pointers must be 16B aligned");
  const int threads = 128;
  group_mean_fwd_kernel<<<dim3(B, (C / 8 + threads - 1) / threads), threads, 0, STREAM>>>(
      (const __nv_bfloat16*)feat, (__nv_bfloat16*)pooled, HW, C);
  return check_launch("group_mean_fwd");
}

extern "C" int vtx_group_mean_bwd(const void* dpooled, void* dfeat, int B, int HW, int C, void* stream) {
  REQ(dpooled && dfeat && B > 0 && HW > 0 && C > 0 && C % 8 == 0, "needs C % 8 == 0 and a non-empty input");
  REQ(((reinterpret_cast<uintptr_t>(dpooled) | reinterpret_cast<uintptr_t>(dfeat)) & 15) == 0,
      "pointers must be 16B aligned");
  const long long n8 = (long long)B * HW * (C / 8);
  long long blocks = (n8 + 255) / 256;
  const long long cap = (long long)vtx_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  group_mean_bwd_kernel<<<(int)blocks, 256, 0, STREAM>>>((const __nv_bfloat16*)dpooled, (__nv_bfloat16*)dfeat, n8, HW,
                                                         C / 8, 1.f / (float)HW);
  return check_launch("group_mean_bwd");
}

extern "C" int vtx_khot_xent(void* logits, int64_t ldl, const int64_t* labels, int64_t ldlab, int B, int L, int V,
                             const int64_t* ignore, int n_ignore, float* loss, int write_grad, void* stream) {
  if (V > VTX_KHOT_MAX_V)
    return set_error(VTX_EUNSUPPORTED, "vtx_khot_xent: V = %d exceeds the label bitmap's bound of %d classes", V,
                     VTX_KHOT_MAX_V);
  REQ(logits && loss && B > 0 && V > 0 && ldl >= V && L >= 0 && (labels || L == 0) && ldlab >= L, "bad arguments");
  REQ(n_ignore >= 0 && (ignore || n_ignore == 0), "bad ignore list");
  khot_xent_kernel<<<B, kKhotThreads, 0, STREAM>>>((__nv_bfloat16*)logits, ldl, (const long long*)labels, ldlab, L, V,
                                                   (const long long*)ignore, n_ignore, 1.f / (float)B, loss, write_grad);
  return check_launch("khot_xent");
}

extern "C" int vtx_topk_rows(const float* X, int64_t ld, int M, int N, int k, int64_t* out, void* stream) {
  REQ(X && out && M > 0 && k > 0 && N >= k && ld >= N, "needs 0 < k <= N");
  topk_rows_kernel<<<M, kTopkThreads, 0, STREAM>>>(X, ld, N, k, (long long*)out);
  return check_launch("topk_rows");
}
