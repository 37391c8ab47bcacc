// Kernels of the CIDEr caption metric (the reference's CocoCaptionsEvaluator, virtex/utils/metrics.py:177-264): exact
// n-gram identity through a device hash table with full 64-bit keys, document frequencies by integer atomics, tf-idf
// vectors, norms and the per-image Gaussian-penalised cosine scores in double.  Every float reduction runs in a fixed
// order on one thread, so two calls return bit-identical results; the only atomics are the table's key CAS and the
// integer df counters.  Per-occurrence arrays are [words, 4]: entry (w, k - 1) belongs to the k-gram starting at word w.
#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {

constexpr int kCiderOrders = 4;
constexpr int kDfThreads = 256;
constexpr int kScoreWarps = 4;

// Key of the n-gram (prefix, word): the prefix is the table slot of the (k-1)-gram, or -1 for a unigram.  prev + 2 >= 1
// keeps every key non-zero (0 marks an empty slot), and since a slot holds one key, equal keys mean equal n-grams.
__device__ __forceinline__ unsigned long long cider_key(int prev, int word) {
  return ((unsigned long long)(unsigned)(prev + 2) << 32) | (unsigned)word;
}
__device__ __forceinline__ unsigned long long cider_mix(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}

// Linear probing over a power-of-two table.  The host sizes it to at least twice the n-grams it can hold, so a probe
// always meets its key or an empty slot.
__device__ int cider_insert(unsigned long long* keys, long long mask, unsigned long long key) {
  long long s = (long long)(cider_mix(key) & (unsigned long long)mask);
  while (true) {
    const unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(keys + s);
    if (cur == key) return (int)s;
    if (cur == 0ull) {
      const unsigned long long old = atomicCAS(keys + s, 0ull, key);
      if (old == 0ull || old == key) return (int)s;
    }
    s = (s + 1) & mask;
  }
}
__device__ int cider_lookup(const unsigned long long* keys, long long mask, unsigned long long key) {
  long long s = (long long)(cider_mix(key) & (unsigned long long)mask);
  while (true) {
    const unsigned long long cur = keys[s];
    if (cur == key) return (int)s;
    if (cur == 0ull) return -1;
    s = (s + 1) & mask;
  }
}

// One warp per sentence, one lane per start position: the lane walks k = 1..4, each k-gram's key built from the slot
// of its (k-1)-gram, so no lane waits on another.
__global__ void cider_intern_kernel(const int32_t* __restrict__ words, const int32_t* __restrict__ sent_off,
                                    int n_sent, unsigned long long* keys, long long mask, int insert,
                                    int32_t* __restrict__ gid) {
  VTX_PDL_TRIGGER();
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < n_sent; s += warps) {
    const int b = sent_off[s], L = sent_off[s + 1] - b;
    for (int p = lane; p < L; p += 32) {
      int prev = -1;
      for (int k = 1; k <= kCiderOrders; ++k) {
        int g = -1;
        if (p + k <= L && (k == 1 || prev >= 0)) {
          const unsigned long long key = cider_key(prev, words[b + p + k - 1]);
          g = insert ? cider_insert(keys, mask, key) : cider_lookup(keys, mask, key);
        }
        gid[(long long)(b + p) * kCiderOrders + k - 1] = g;
        prev = g;
      }
    }
  }
}

// One CTA per image: every distinct n-gram of the image's references (first occurrence in the image) adds 1 to its df.
__global__ void __launch_bounds__(kDfThreads) cider_df_kernel(const int32_t* __restrict__ gid,
                                                              const int32_t* __restrict__ sent_off,
                                                              const int32_t* __restrict__ img_off,
                                                              int32_t* __restrict__ df) {
  VTX_PDL_TRIGGER();
  __shared__ int32_t sg[VTX_CIDER_MAX_IMAGE_WORDS * kCiderOrders];
  const int w0 = sent_off[img_off[blockIdx.x]], w1 = sent_off[img_off[blockIdx.x + 1]];
  const int n = (w1 - w0) * kCiderOrders;
  for (int o = threadIdx.x; o < n; o += kDfThreads) sg[o] = gid[(long long)w0 * kCiderOrders + o];
  __syncthreads();
  for (int o = threadIdx.x; o < n; o += kDfThreads) {
    const int g = sg[o];
    if (g < 0) continue;
    bool first = true;
    for (int j = 0; j < o && first; ++j) first = sg[j] != g;
    if (first) atomicAdd(df + g, 1);
  }
}

// One warp per sentence.  A lane takes start positions; for each order it compares words with every other start
// position, so repeated n-grams are found exactly whether or not the table holds them.  The first occurrence gets
// tf and the entry tf * (log N - log max(1, df)), later ones tf 0 and entry -1.  Lanes 0..3 then add the squares of
// order lane + 1 in position order, the reference's order.
__global__ void cider_vectors_kernel(const int32_t* __restrict__ words, const int32_t* __restrict__ gid,
                                     const int32_t* __restrict__ sent_off, int n_sent, const int32_t* __restrict__ df,
                                     int n_img, int32_t* __restrict__ tf, double* __restrict__ ent,
                                     double* __restrict__ norm) {
  VTX_PDL_TRIGGER();
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  const double log_n = log((double)n_img);
  for (int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < n_sent; s += warps) {
    const int b = sent_off[s], L = sent_off[s + 1] - b;
    const int32_t* w = words + b;
    for (int p = lane; p < L; p += 32) {
      for (int k = 1; k <= kCiderOrders; ++k) {
        const long long e = (long long)(b + p) * kCiderOrders + k - 1;
        int count = 0;
        bool first = p + k <= L;
        for (int q = 0; first && q + k <= L; ++q) {
          bool eq = true;
          for (int j = 0; j < k && eq; ++j) eq = w[q + j] == w[p + j];
          if (eq && q < p) first = false;
          count += eq;
        }
        if (first) {
          const int g = gid[e];
          const int d = g >= 0 ? df[g] : 0;
          tf[e] = count;
          ent[e] = (double)count * (log_n - log((double)(d > 1 ? d : 1)));
        } else {
          tf[e] = 0;
          ent[e] = -1.0;
        }
      }
    }
    __syncwarp();
    if (lane < kCiderOrders) {
      double acc = 0.0;
      for (int p = 0; p + lane < L; ++p) {
        const double v = ent[(long long)(b + p) * kCiderOrders + lane];
        if (v >= 0.0) acc += v * v;
      }
      norm[(long long)s * kCiderOrders + lane] = sqrt(acc);
    }
    __syncwarp();
  }
}

// One warp per image; lane t of a pass takes (reference r, order k).  sim = sum over the hypothesis's distinct k-grams,
// in position order, of min(vh, vr) * vr (vr = 0 when the reference lacks the n-gram), divided by (|h| |r|) or 1 and
// scaled by e^(-(len_h - len_r)^2 / (2 sigma^2)); lane 0 adds the references in order, then the mean over the orders.
__global__ void __launch_bounds__(kScoreWarps * 32) cider_score_kernel(
    const int32_t* __restrict__ hyp_gid, const double* __restrict__ hyp_ent, const double* __restrict__ hyp_norm,
    const int32_t* __restrict__ hyp_off, const int32_t* __restrict__ ref_gid, const double* __restrict__ ref_ent,
    const double* __restrict__ ref_norm, const int32_t* __restrict__ ref_off, const int32_t* __restrict__ img_off,
    int n_img, double sigma, double* __restrict__ img_score) {
  VTX_PDL_TRIGGER();
  __shared__ double vals[kScoreWarps][VTX_CIDER_MAX_REFS * kCiderOrders];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int img = blockIdx.x * kScoreWarps + wp;
  if (img >= n_img) return;
  const int hb = hyp_off[img], Lh = hyp_off[img + 1] - hb;
  const int r0 = img_off[img], R = img_off[img + 1] - r0;
  const double two_s2 = 2.0 * (sigma * sigma);
  for (int t = lane; t < R * kCiderOrders; t += 32) {
    const int r = t / kCiderOrders, k = t % kCiderOrders + 1;
    const int rb = ref_off[r0 + r], Lr = ref_off[r0 + r + 1] - rb;
    double val = 0.0;
    for (int p = 0; p + k <= Lh; ++p) {
      const long long eh = (long long)(hb + p) * kCiderOrders + k - 1;
      const double vh = hyp_ent[eh];
      if (vh < 0.0) continue;
      const int g = hyp_gid[eh];
      double vr = 0.0;
      if (g >= 0) {
        for (int q = 0; q + k <= Lr; ++q) {
          const long long er = (long long)(rb + q) * kCiderOrders + k - 1;
          if (ref_gid[er] == g && ref_ent[er] >= 0.0) { vr = ref_ent[er]; break; }
        }
      }
      val += (vr < vh ? vr : vh) * vr;
    }
    const double den = hyp_norm[(long long)img * kCiderOrders + k - 1] * ref_norm[(long long)(r0 + r) * kCiderOrders + k - 1];
    val /= den != 0.0 ? den : 1.0;
    const double delta = (double)((Lh > 1 ? Lh - 1 : 0) - (Lr > 1 ? Lr - 1 : 0));
    val *= pow(2.718281828459045, -(delta * delta) / two_s2);
    vals[wp][t] = val;
  }
  __syncwarp();
  if (lane == 0) {
    double sum = 0.0;
    for (int k = 0; k < kCiderOrders; ++k) {
      double acc = 0.0;
      for (int r = 0; r < R; ++r) acc += vals[wp][r * kCiderOrders + k];
      sum += acc;
    }
    img_score[img] = sum / kCiderOrders / (double)R * 10.0;
  }
}

// One CTA: strided per-thread sums, then a fixed shared-memory tree.
constexpr int kMeanThreads = 1024;
__global__ void __launch_bounds__(kMeanThreads) cider_mean_kernel(const double* __restrict__ x, int n,
                                                                   double* __restrict__ out) {
  VTX_PDL_TRIGGER();
  __shared__ double sh[kMeanThreads];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += kMeanThreads) acc += x[i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int h = kMeanThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) sh[threadIdx.x] += sh[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = sh[0] / (double)n;
}

}  // namespace vtx

using namespace vtx;
#define STREAM reinterpret_cast<cudaStream_t>(stream)
#define REQ(cond, msg) \
  if (!(cond)) return set_error(VTX_EINVAL, "%s: %s", __func__, msg)

static int warp_grid(int n_sent) {
  const int blocks = (n_sent + 7) / 8;  // 8 warps per CTA
  return blocks < 8192 ? (blocks > 0 ? blocks : 1) : 8192;
}

extern "C" int vtx_cider_intern(const int32_t* words, const int32_t* sent_off, int n_sent, unsigned long long* keys,
                                int64_t capacity, int insert, int32_t* gid, void* stream) {
  REQ(words && sent_off && keys && gid && n_sent > 0, "bad arguments");
  REQ(capacity >= 2 && (capacity & (capacity - 1)) == 0 && capacity <= (1ll << 30), "capacity must be a power of two <= 2^30");
  cider_intern_kernel<<<warp_grid(n_sent), 256, 0, STREAM>>>(words, sent_off, n_sent, keys, capacity - 1, insert, gid);
  return check_launch("cider_intern");
}

extern "C" int vtx_cider_df(const int32_t* gid, const int32_t* sent_off, const int32_t* img_off, int n_img, int32_t* df,
                            void* stream) {
  REQ(gid && sent_off && img_off && df && n_img > 0, "bad arguments");
  cider_df_kernel<<<n_img, kDfThreads, 0, STREAM>>>(gid, sent_off, img_off, df);
  return check_launch("cider_df");
}

extern "C" int vtx_cider_vectors(const int32_t* words, const int32_t* gid, const int32_t* sent_off, int n_sent,
                                 const int32_t* df, int n_img, int32_t* tf, double* ent, double* norm, void* stream) {
  REQ(words && gid && sent_off && df && tf && ent && norm && n_sent > 0 && n_img > 0, "bad arguments");
  cider_vectors_kernel<<<warp_grid(n_sent), 256, 0, STREAM>>>(words, gid, sent_off, n_sent, df, n_img, tf, ent, norm);
  return check_launch("cider_vectors");
}

extern "C" int vtx_cider_score(const int32_t* hyp_gid, const double* hyp_ent, const double* hyp_norm,
                               const int32_t* hyp_off, const int32_t* ref_gid, const double* ref_ent,
                               const double* ref_norm, const int32_t* ref_off, const int32_t* img_off, int n_img,
                               double sigma, double* img_score, void* stream) {
  REQ(hyp_gid && hyp_ent && hyp_norm && hyp_off && ref_gid && ref_ent && ref_norm && ref_off && img_off && img_score &&
      n_img > 0, "bad arguments");
  REQ(sigma != 0.0, "sigma must be non-zero");
  cider_score_kernel<<<(n_img + kScoreWarps - 1) / kScoreWarps, kScoreWarps * 32, 0, STREAM>>>(
      hyp_gid, hyp_ent, hyp_norm, hyp_off, ref_gid, ref_ent, ref_norm, ref_off, img_off, n_img, sigma, img_score);
  return check_launch("cider_score");
}

extern "C" int vtx_cider_mean(const double* x, int n, double* out, void* stream) {
  REQ(x && out && n > 0, "bad arguments");
  cider_mean_kernel<<<1, kMeanThreads, 0, STREAM>>>(x, n, out);
  return check_launch("cider_mean");
}
