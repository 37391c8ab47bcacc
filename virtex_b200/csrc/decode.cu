// Kernels of the incremental beam-search decoder (virtex/utils/beam_search.py, virtex/models/captioning.py:144-213):
// single-query attention over a key block per row (self-attention over the growing cache, cross-attention over the
// image's projected features), and the two halves of one beam step -- per-row log-softmax with the reference's
// repetition penalty and EOS continuation + per-row top-k, then the per-image selection that also gathers the
// predictions and the cache index table of the surviving beams -- and one step of nucleus sampling
// (virtex/utils/nucleus_sampling.py).  Everything else of a decoding step is a GEMM or an existing head kernel run with
// dropout p = 0.
#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {

constexpr int kDecWarps = 4;
constexpr int kBeamRowThreads = 256;
constexpr int kSelectWarps = 4;

// ------------------------------------------------------------------------------------------------ attention
// One warp per (key block, head).  Block b serves the `group` query rows b*group .. b*group + group-1.  Lane j holds
// keys j and j + 32 (all 64 head dimensions, bf16 in registers) and computes their scores; the softmax is a warp
// reduction; for the output each lane owns two head dimensions and walks the keys.  Key j of block b lives at
// k + blk * ldb + j * ldkv with blk = b, or blk = kv_index[j * ld_index + b] when the index table is given.
__global__ void __launch_bounds__(32 * kDecWarps) attn_decode_kernel(
    const __nv_bfloat16* __restrict__ q, long long ldq, const __nv_bfloat16* __restrict__ k,
    const __nv_bfloat16* __restrict__ v, long long ldkv, long long ldb, const int* __restrict__ kv_index,
    long long ld_index, __nv_bfloat16* __restrict__ out, long long ldo, int blocks, int heads, int group, int Tk) {
  VTX_PDL_TRIGGER();
  __shared__ float qs[kDecWarps][64];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long unit = (long long)blockIdx.x * kDecWarps + warp;
  if (unit >= (long long)blocks * heads) return;
  const int b = (int)(unit / heads), h = (int)(unit % heads);
  uint4 kr[2][8];
  int blk[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int j = lane + 32 * r;
    blk[r] = b;
    if (j < Tk) {
      if (kv_index) blk[r] = kv_index[(long long)j * ld_index + b];
      const uint4* src = reinterpret_cast<const uint4*>(k + blk[r] * ldb + (long long)j * ldkv + h * 64);
#pragma unroll
      for (int i = 0; i < 8; ++i) kr[r][i] = src[i];
    }
  }
  for (int g = 0; g < group; ++g) {
    const long long m = (long long)b * group + g;
    __syncwarp();
    const __nv_bfloat162 q2 = *reinterpret_cast<const __nv_bfloat162*>(q + m * ldq + h * 64 + 2 * lane);
    qs[warp][2 * lane] = __low2float(q2) * 0.125f;  // 1/sqrt(head_dim)
    qs[warp][2 * lane + 1] = __high2float(q2) * 0.125f;
    __syncwarp();
    float p[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      p[r] = -INFINITY;
      if (lane + 32 * r < Tk) {
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          bf16x8 u;
          *reinterpret_cast<uint4*>(&u) = kr[r][i];
          float f[8];
          unpack8(u, f);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc = fmaf(f[e], qs[warp][8 * i + e], acc);
        }
        p[r] = acc;
      }
    }
    const float mx = warp_max(fmaxf(p[0], p[1]));
#pragma unroll
    for (int r = 0; r < 2; ++r) p[r] = (lane + 32 * r < Tk) ? expf(p[r] - mx) : 0.f;
    const float inv = 1.f / warp_sum(p[0] + p[1]);
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j < Tk; ++j) {
      const float pj = __shfl_sync(0xffffffffu, j < 32 ? p[0] : p[1], j & 31);
      const int bj = __shfl_sync(0xffffffffu, j < 32 ? blk[0] : blk[1], j & 31);
      const __nv_bfloat162 v2 =
          *reinterpret_cast<const __nv_bfloat162*>(v + bj * ldb + (long long)j * ldkv + h * 64 + 2 * lane);
      o0 = fmaf(pj, __low2float(v2), o0);
      o1 = fmaf(pj, __high2float(v2), o1);
    }
    *reinterpret_cast<__nv_bfloat162*>(out + m * ldo + h * 64 + 2 * lane) = __floats2bfloat162_rn(o0 * inv, o1 * inv);
  }
}

// ------------------------------------------------------------------------------------------------ beam step
// (v, i) precedes (w, j) iff v > w, or v == w and i < j: descending value, ties in ascending index (vtx_topk_rows)
__device__ __forceinline__ bool beam_before(float v, int i, float w, int j) { return v > w || (v == w && i < j); }

__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  const float mm = fmaxf(m, m2);
  if (mm == -INFINITY) return;
  s = s * expf(m - mm) + s2 * expf(m2 - mm);
  m = mm;
}

// One CTA per row of fp32 logits.  The row's scores are log_softmax(x) (fp32), then -10000 at the row's own last token,
// then -- for a row whose last token is EOS -- 0 at EOS and -inf everywhere else (beam_search.py:152-172).  Writes the
// k best (value, index) pairs in descending order.  last == NULL: plain log_softmax (the first step).
__global__ void __launch_bounds__(kBeamRowThreads) beam_rows_kernel(const float* __restrict__ X, long long ld, int V,
                                                                   const long long* __restrict__ last, int eos, int k,
                                                                   float* __restrict__ cand_val,
                                                                   int* __restrict__ cand_idx) {
  VTX_PDL_TRIGGER();
  __shared__ float sm[32], ss[32];
  __shared__ int si[32];
  const int row = blockIdx.x;
  const float* x = X + (long long)row * ld;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  // log-sum-exp in one pass (running maximum, rescaled sum)
  float m = -INFINITY, s = 0.f;
  for (int i = threadIdx.x; i < V; i += blockDim.x) lse_merge(m, s, x[i], 1.f);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    lse_merge(m, s, m2, s2);
  }
  if (lane == 0) { sm[warp] = m; ss[warp] = s; }
  __syncthreads();
  m = -INFINITY;
  s = 0.f;
  for (int w = 0; w < nwarps; ++w) lse_merge(m, s, sm[w], ss[w]);
  const float lse = m + logf(s);
  const long long lt = last ? last[row] : -1;
  const bool ended = lt == eos;
  float pv = INFINITY;
  int pi = -1;
  for (int r = 0; r < k; ++r) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
      float val = ended ? (i == eos ? 0.f : -INFINITY) : (i == lt ? -10000.f : x[i] - lse);
      if (isnan(val)) val = -INFINITY;
      if (beam_before(pv, pi, val, i) && beam_before(val, i, bv, bi)) { bv = val; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (beam_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    __syncthreads();  // the previous round's readers of sm / si are done
    if (lane == 0) { sm[warp] = bv; si[warp] = bi; }
    __syncthreads();
    bv = lane < nwarps ? sm[lane] : -INFINITY;
    bi = lane < nwarps ? si[lane] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (beam_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (threadIdx.x == 0) {
      cand_val[(long long)row * k + r] = bv;
      cand_idx[(long long)row * k + r] = bi;
    }
    pv = bv;
    pi = bi;
  }
}

// One warp per image.  Candidate c (< parents * k) of image b is (parent p = c / k, its (c % k)-th row candidate); its
// score is the row candidate's value plus the parent's score.  The `beam` best candidates, in descending order (ties in
// ascending candidate index), become the new beams r = 0 .. beam-1 of the image; their rows of the step-major tables
// pred [steps, R] and index [steps, R] (R = B * beam) are the parent's rows up to step s-1, then the new token at step
// s (pred) and the beam's own row (index: slot s of the key/value cache is where this row writes its next key/value).
// alive[s] = 1 when any new token of the image is not EOS (alive[] is zeroed by the caller once per search).
__global__ void __launch_bounds__(32 * kSelectWarps) beam_select_kernel(
    const float* __restrict__ cand_val, const int* __restrict__ cand_idx, int parents, int k, int beam,
    const float* scores_in, float* scores_out, int* __restrict__ parent_out, const long long* __restrict__ pred_in,
    long long* __restrict__ pred_out, const int* __restrict__ index_in, int* __restrict__ index_out, int B, int s,
    int eos, int* __restrict__ alive) {
  VTX_PDL_TRIGGER();
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * kSelectWarps + (threadIdx.x >> 5);
  if (b >= B) return;
  const int R = B * beam;
  const int nc = parents * k;
  float val = -INFINITY;
  int tok = 0;
  if (lane < nc) {
    const int p = b * parents + lane / k;
    val = cand_val[(long long)p * k + lane % k] + (scores_in ? scores_in[p] : 0.f);
    tok = cand_idx[(long long)p * k + lane % k];
  }
  bool picked = lane >= nc;
  float my_val = 0.f;
  int my_tok = 0, my_parent = 0;
  for (int r = 0; r < beam; ++r) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    if (!picked) { bv = val; bi = lane; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (beam_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == bi) picked = true;
    const int t = __shfl_sync(0xffffffffu, tok, bi & 31);
    if (lane == r) { my_val = bv; my_tok = t; my_parent = b * parents + bi / k; }
  }
  __syncwarp();  // every read of scores_in (which may alias scores_out) is done
  const int i = b * beam + lane;
  if (lane < beam) {
    scores_out[i] = my_val;
    if (parent_out) parent_out[i] = my_parent;
    pred_out[(long long)s * R + i] = my_tok;
    index_out[(long long)s * R + i] = i;
  }
  for (int r = 0; r < beam; ++r) {
    const int p = __shfl_sync(0xffffffffu, my_parent, r);
    for (int j = lane; j < s; j += 32) {
      pred_out[(long long)j * R + b * beam + r] = pred_in[(long long)j * R + p];
      index_out[(long long)j * R + b * beam + r] = index_in[(long long)j * R + p];
    }
  }
  if (__any_sync(0xffffffffu, lane < beam && my_tok != eos) && lane == 0) alive[s] = 1;
}

// ------------------------------------------------------------------------------------------------ nucleus sampling
// One CTA per row of fp32 logits (AutoRegressiveNucleusSampling.search, nucleus_sampling.py:77-113).  The row is staged
// once in shared memory; every later pass reads it from there.
//   1. p_i = exp(x_i - lse) in fp32 (one-pass log-sum-exp), as fixed-point mass q_i = rint(p_i * 2^40): integer sums
//      are exact, so every cumulative mass below is independent of summation order.
//   2. The crossing token -- the first token, in (descending value, ascending id) order, whose inclusive cumulative
//      mass exceeds thr = floor(p * 2^40) -- by a radix select over order-preserving 32-bit value keys, 11 + 11 + 10
//      bits, with a mass histogram per digit.  Exact ties share one mass, so the crossing tie's rank is arithmetic,
//      and a scan in id order finds its id.  The nucleus is every token up to and including it (all tokens when the
//      whole mass is <= thr).
//   3. The row's last token is banned after the nucleus is chosen.  The sample is the inverse CDF, in ascending id,
//      of the weights rint(exp(x_i - m) * 2^40) of the kept unbanned tokens (m: their largest logit), at the uniform
//      u = (hash_u64(seed, kNucleusSite, s * R + row) >> 40) / 2^24; when the nucleus is the last token alone, the
//      reference's softmax over all -1e12 logits is uniform: token floor(u * V).
// Tokens of mass below 2^-41 (nucleus) or weight below 2^-41 of the largest (sampling) round to zero and are never
// drawn; the reference draws them with probability below 1e-12.
constexpr int kNucThreads = 256;
constexpr int kNucBins = 2048;
constexpr uint32_t kNucleusSite = 4000u;  // hash site of the sampler's uniforms; dropout sites are below 2000

// ascending key = descending value (the logits are NaN-free and -0 is +0 by now)
__device__ __forceinline__ uint32_t nuc_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? u : ~(u | 0x80000000u);
}
__device__ __forceinline__ float nuc_value(uint32_t key) {
  return __uint_as_float((key & 0x80000000u) ? key : (~key & 0x7fffffffu));
}
__device__ __forceinline__ unsigned long long nuc_fixed(float x, float ref) {
  return __float2ull_rn(expf(x - ref) * 0x1p40f);
}

__device__ __forceinline__ unsigned long long bin_mass(const uint32_t* lo, const uint32_t* hi, int b) {
  return ((unsigned long long)hi[b] << 32) + lo[b];
}

// exclusive prefix sum of v over the CTA in thread order; `total` receives the CTA's sum.  scratch: 32 entries.
__device__ __forceinline__ unsigned long long block_scan_u64(unsigned long long v, unsigned long long* scratch,
                                                            unsigned long long& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  unsigned long long inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  __syncthreads();  // the previous scan's readers of scratch are done
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  unsigned long long base = 0;
  total = 0;
  for (int w = 0; w < nwarps; ++w) {
    if (w < warp) base += scratch[w];
    total += scratch[w];
  }
  return base + inc - v;
}

__global__ void __launch_bounds__(kNucThreads) nucleus_sample_kernel(const float* __restrict__ X, long long ld, int V,
                                                                     const long long* __restrict__ last, int eos,
                                                                     float p, const unsigned long long* __restrict__ seed,
                                                                     int s, int R, long long* __restrict__ pred,
                                                                     int* __restrict__ alive) {
  VTX_PDL_TRIGGER();
  extern __shared__ float xs[];
  __shared__ uint32_t hist_lo[kNucBins], hist_hi[kNucBins];  // a 64-bit mass histogram as two native-atomic halves
  __shared__ unsigned long long scratch[32];
  __shared__ float sm[32], ss[32];
  __shared__ unsigned long long sel_before;
  __shared__ int sel_bin, sel_id;
  const int row = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
  const long long lt = last[row];
  long long* dst = pred + (long long)s * R + row;
  if (lt == eos) {  // rule 6: an ended caption continues with EOS
    if (tid == 0) *dst = eos;
    return;
  }
  const float* x = X + (long long)row * ld;
  float m = -INFINITY, sum = 0.f;
  for (int i = tid; i < V; i += nt) {
    float v = x[i];
    if (isnan(v)) v = -INFINITY;
    if (v == 0.f) v = 0.f;  // -0 ties with +0, as in a sort by value
    xs[i] = v;
    lse_merge(m, sum, v, 1.f);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, sum, o);
    lse_merge(m, sum, m2, s2);
  }
  if (lane == 0) { sm[warp] = m; ss[warp] = sum; }
  __syncthreads();
  m = -INFINITY;
  sum = 0.f;
  for (int w = 0; w < nwarps; ++w) lse_merge(m, sum, sm[w], ss[w]);
  const float lse = m + logf(sum);

  // ---- the crossing token's value key: three radix digits, most significant first
  const unsigned long long thr = (unsigned long long)((double)p * 0x1p40);
  uint32_t prefix = 0, pmask = 0;
  unsigned long long before = 0;  // mass of every token whose key is below the current prefix
  bool all_kept = false;
  for (int pass = 0; pass < 3; ++pass) {
    const int shift = pass == 0 ? 21 : pass == 1 ? 10 : 0;
    const int nb = pass == 2 ? 1024 : 2048;
    for (int b = tid; b < nb; b += nt) hist_lo[b] = hist_hi[b] = 0;
    __syncthreads();
    for (int i = tid; i < V; i += nt) {
      const float v = xs[i];
      const uint32_t k = nuc_key(v);
      if ((k & pmask) == prefix) {
        const unsigned long long q = nuc_fixed(v, lse);
        if (q) {  // 64-bit add from two 32-bit atomics (a shared 64-bit atomic add is a compare-and-swap loop)
          const int b = (k >> shift) & (nb - 1);
          const uint32_t ql = (uint32_t)q, old = atomicAdd(&hist_lo[b], ql);
          const uint32_t qh = (uint32_t)(q >> 32) + (old + ql < old ? 1u : 0u);
          if (qh) atomicAdd(&hist_hi[b], qh);
        }
      }
    }
    __syncthreads();
    const int per = nb / nt;
    unsigned long long local = 0;
    for (int j = 0; j < per; ++j) local += bin_mass(hist_lo, hist_hi, tid * per + j);
    unsigned long long total;
    unsigned long long run = before + block_scan_u64(local, scratch, total);
    if (pass == 0 && total <= thr) {  // no token crosses p: the nucleus is the whole vocabulary
      all_kept = true;
      break;
    }
    for (int j = 0; j < per; ++j) {
      const unsigned long long h = bin_mass(hist_lo, hist_hi, tid * per + j);
      if (run <= thr && run + h > thr) { sel_bin = tid * per + j; sel_before = run; }
      run += h;
    }
    __syncthreads();
    prefix |= (uint32_t)sel_bin << shift;
    pmask |= (uint32_t)(nb - 1) << shift;
    before = sel_before;
  }

  // ---- the crossing token's id: tie rank j = floor((thr - before) / q*) among the tokens of key `prefix`, in id order.
  // The same pass takes the largest logit among the kept unbanned tokens of smaller key.
  const uint32_t vkey = all_kept ? 0xffffffffu : prefix;  // no token has key 0xffffffff (a NaN)
  const float vstar = nuc_value(vkey);
  const unsigned long long rank = all_kept ? 0 : (thr - before) / nuc_fixed(vstar, lse);
  const int chunk = (V + nt - 1) / nt;
  const int lo = min(V, tid * chunk), hi = min(V, lo + chunk);
  unsigned long long ties = 0;
  float mk = -INFINITY;
  for (int i = lo; i < hi; ++i) {
    const uint32_t k = nuc_key(xs[i]);
    if (k == vkey) ++ties;
    else if (k < vkey && i != lt) mk = fmaxf(mk, xs[i]);
  }
  unsigned long long nties;
  const unsigned long long tie0 = block_scan_u64(ties, scratch, nties);
  if (!all_kept && tie0 <= rank && rank < tie0 + ties) {
    unsigned long long r = tie0;
    for (int i = lo; i < hi; ++i)
      if (nuc_key(xs[i]) == vkey && r++ == rank) { sel_id = i; break; }
  }
  mk = warp_max(mk);
  if (lane == 0) sm[warp] = mk;
  __syncthreads();
  const int cid = all_kept ? 0x7fffffff : sel_id;
  mk = -INFINITY;
  for (int w = 0; w < nwarps; ++w) mk = fmaxf(mk, sm[w]);
  if (!all_kept) {  // the kept ties are the rank + 1 first ones; the last token may be one of them
    const bool last_is_kept_tie = lt >= 0 && lt < V && nuc_key(xs[lt]) == vkey && lt <= cid;
    if (rank + 1 > (last_is_kept_tie ? 1ull : 0ull)) mk = fmaxf(mk, vstar);
  }

  // ---- inverse CDF over the kept unbanned tokens in ascending id
  const uint32_t u24 = (uint32_t)(hash_u64(*seed, kNucleusSite, (unsigned long long)s * R + row) >> 40);
  long long tok;
  if (mk == -INFINITY) {  // the nucleus is the banned token alone: uniform over the vocabulary
    tok = (long long)(((unsigned long long)u24 * (unsigned long long)V) >> 24);
    if (tid == 0) *dst = tok;
  } else {
    unsigned long long wsum = 0;
    for (int i = lo; i < hi; ++i) {
      const uint32_t k = nuc_key(xs[i]);
      if (i != lt && (k < vkey || (k == vkey && i <= cid))) wsum += nuc_fixed(xs[i], mk);
    }
    unsigned long long W;
    const unsigned long long w0 = block_scan_u64(wsum, scratch, W);
    // target = floor(W * u24 / 2^24) < W (W < 2^56, so the product needs 128 bits)
    const unsigned long long target = (__umul64hi(W, u24) << 40) | ((W * u24) >> 24);
    tok = -1;
    if (w0 <= target && target < w0 + wsum) {
      unsigned long long run = w0;
      for (int i = lo; i < hi; ++i) {
        const uint32_t k = nuc_key(xs[i]);
        if (i != lt && (k < vkey || (k == vkey && i <= cid))) {
          run += nuc_fixed(xs[i], mk);
          if (run > target) { tok = i; break; }
        }
      }
      *dst = tok;
    }
  }
  if (tok >= 0 && tok != eos) alive[s] = 1;
}

}  // namespace vtx

using namespace vtx;
#define STREAM reinterpret_cast<cudaStream_t>(stream)
#define REQ(cond, msg) \
  if (!(cond)) return set_error(VTX_EINVAL, "%s: %s", __func__, msg)

extern "C" int vtx_attn_decode(const void* q, int64_t ldq, const void* k, const void* v, int64_t ldkv, int64_t ldb,
                               const int32_t* kv_index, int64_t ld_index, void* out, int64_t ldo, int blocks, int heads,
                               int group, int Tk, void* stream) {
  REQ(q && k && v && out && blocks > 0 && heads > 0 && group > 0, "bad arguments");
  REQ(Tk >= 1 && Tk <= VTX_DECODE_MAX_KEYS, "needs 1 <= Tk <= 64");
  REQ(!kv_index || group == 1, "an index table needs group == 1");
  REQ(ldq % 2 == 0 && ldo % 2 == 0 && ldkv % 8 == 0 && ldb % 8 == 0, "leading dimensions: q / out even, k / v % 8");
  REQ(((reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v)) & 15) == 0, "k and v must be 16B aligned");
  const long long units = (long long)blocks * heads;
  attn_decode_kernel<<<(unsigned)((units + kDecWarps - 1) / kDecWarps), 32 * kDecWarps, 0, STREAM>>>(
      (const __nv_bfloat16*)q, ldq, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, ldkv, ldb, kv_index, ld_index,
      (__nv_bfloat16*)out, ldo, blocks, heads, group, Tk);
  return check_launch("attn_decode");
}

extern "C" int vtx_beam_rows(const float* logits, int64_t ldl, int R, int V, const int64_t* last, int eos, int k,
                             float* cand_val, int32_t* cand_idx, void* stream) {
  REQ(logits && cand_val && cand_idx && R > 0 && V > 0 && ldl >= V, "bad arguments");
  REQ(k >= 1 && k <= V && k <= 32, "needs 1 <= k <= min(V, 32)");
  beam_rows_kernel<<<R, kBeamRowThreads, 0, STREAM>>>(logits, ldl, V, (const long long*)last, eos, k, cand_val,
                                                      cand_idx);
  return check_launch("beam_rows");
}

extern "C" int vtx_beam_select(const float* cand_val, const int32_t* cand_idx, int parents, int k, int beam,
                               const float* scores_in, float* scores_out, int32_t* parent_out, const int64_t* pred_in,
                               int64_t* pred_out, const int32_t* index_in, int32_t* index_out, int B, int s, int eos,
                               int32_t* alive, void* stream) {
  REQ(cand_val && cand_idx && scores_out && pred_out && index_out && alive && B > 0 && s >= 0, "bad arguments");
  REQ(parents >= 1 && k >= 1 && beam >= 1 && parents * k <= 32 && beam <= parents * k, "needs beam <= parents * k <= 32");
  REQ(s == 0 || (pred_in && index_in && pred_in != pred_out && index_in != index_out),
      "steps after the first gather from separate input tables");
  beam_select_kernel<<<(B + kSelectWarps - 1) / kSelectWarps, 32 * kSelectWarps, 0, STREAM>>>(
      cand_val, cand_idx, parents, k, beam, scores_in, scores_out, parent_out, (const long long*)pred_in,
      (long long*)pred_out, index_in, index_out, B, s, eos, alive);
  return check_launch("beam_select");
}

extern "C" int vtx_nucleus_sample(const float* logits, int64_t ldl, int R, int V, const int64_t* last, int eos,
                                  float p, const uint64_t* seed, int s, int64_t* pred, int32_t* alive, void* stream) {
  REQ(logits && last && seed && pred && alive && R > 0 && V > 0 && ldl >= V && s >= 0, "bad arguments");
  REQ(V <= VTX_NUCLEUS_MAX_V, "needs V <= VTX_NUCLEUS_MAX_V (32768)");
  REQ(p >= 0.f && p <= 1.f, "needs 0 <= p <= 1");
  const int smem = V * (int)sizeof(float);
  cudaFuncSetAttribute(nucleus_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  nucleus_sample_kernel<<<R, kNucThreads, smem, STREAM>>>(logits, ldl, V, (const long long*)last, eos, p,
                                                          (const unsigned long long*)seed, s, R, (long long*)pred,
                                                          alive);
  return check_launch("nucleus_sample");
}
