// Kernels of the VOC07 linear-SVM evaluation (scripts/clf_voc07.py:56-105): every (class, cost, fold-or-full) problem
// of the reference's per-class LinearSVC sweep is one column of a batched truncated-Newton solve of liblinear's
// L2R_L2LOSS_SVC objective, and sklearn's average_precision_score scores the results.  The products with the feature
// matrix are vtx_gemm calls over the bf16 hi/lo operands written here; everything between them is one of the column
// kernels below.  Per-problem vectors are [rows, P] fp32 (problem p = column p); column reductions write per-slice
// partial sums [VTX_SVM_SLICES, P] in double that their consumers add in a fixed order, so a solve is bitwise
// deterministic.
#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {

constexpr int kSl = VTX_SVM_SLICES;
constexpr int kTy = 8;             // rows of a column block per pass (block = 32 columns x kTy rows)
constexpr int kLsThreads = 512;    // line search: one CTA per problem
constexpr int kApThreads = 1024;   // average precision: one CTA per scored column

// x = hi + lo, hi = bf16(x), lo = bf16(x - hi)
__device__ __forceinline__ void split2(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = f2bf(v);
  lo = f2bf(v - bf2f(hi));
}
// operand [hi; lo; hi] of a [rows, P] fp32 matrix: bf16 [3 * rows, P]
__device__ __forceinline__ void store_split(__nv_bfloat16* op, long long rows, int P, long long i, int p, float v) {
  __nv_bfloat16 hi, lo;
  split2(v, hi, lo);
  op[i * P + p] = hi;
  op[(rows + i) * P + p] = lo;
  op[(2 * rows + i) * P + p] = hi;
}

// Sum of NV per-thread values over the kTy rows of the block, written as slice blockIdx.y of part[NV][kSl][P].
template <int NV>
__device__ __forceinline__ void col_store(const double (&v)[NV], double* part, int P) {
  __shared__ double sh[NV][kTy][32];
  const int tx = threadIdx.x, ty = threadIdx.y, p = blockIdx.x * 32 + tx;
#pragma unroll
  for (int j = 0; j < NV; ++j) sh[j][ty][tx] = v[j];
  __syncthreads();
  if (ty == 0) {
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      double s = 0.0;
#pragma unroll
      for (int r = 0; r < kTy; ++r) s += sh[j][r][tx];
      part[((long long)j * kSl + blockIdx.y) * P + p] = s;
    }
  }
}
__device__ __forceinline__ double col_sum(const double* part, int P, int p) {
  double s = 0.0;
  for (int k = 0; k < kSl; ++k) s += part[(long long)k * P + p];
  return s;
}

__global__ void split_x_kernel(const float* __restrict__ x, long long ldx, int n, int d, int n_pad, int dp,
                               __nv_bfloat16* __restrict__ xcat, __nv_bfloat16* __restrict__ xstk) {
  VTX_PDL_TRIGGER();
  const long long total = (long long)n_pad * dp;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / dp;
    const int j = (int)(e % dp);
    const float v = i >= n ? 0.f : j < d ? x[i * ldx + j] : j == d ? 1.f : 0.f;
    __nv_bfloat16 hi, lo;
    split2(v, hi, lo);
    if (xcat) {  // [n_pad, 3 dp] = [hi | hi | lo]
      __nv_bfloat16* row = xcat + i * 3 * dp;
      row[j] = hi; row[dp + j] = hi; row[2 * dp + j] = lo;
    }
    if (xstk) {  // [3 n_pad, dp] = [hi; hi; lo]
      xstk[i * dp + j] = hi;
      xstk[((long long)n_pad + i) * dp + j] = hi;
      xstk[(2LL * n_pad + i) * dp + j] = lo;
    }
  }
}

// Column-kernel geometry: block (32, kTy), grid (P / 32, kSl); thread (tx, ty) of block (bx, by) visits column
// bx * 32 + tx at rows by * kTy + ty + k * kSl * kTy.
#define VTX_COL_LOOP(rows) \
  const int p = blockIdx.x * 32 + threadIdx.x; \
  for (long long i = (long long)blockIdx.y * kTy + threadIdx.y; i < (rows); i += (long long)kSl * kTy)

__global__ void split_cols_kernel(const float* __restrict__ v, int rows, int P, __nv_bfloat16* __restrict__ op) {
  VTX_PDL_TRIGGER();
  VTX_COL_LOOP(rows) store_split(op, rows, P, i, p, v[i * P + p]);
}

// u = 2 c (z - y) on the active set {c > 0, y z < 1}, else 0 (the loss derivative); dact = c on the active set;
// part[0] = sum of c (1 - y z)^2 over the active set.  cy = y * c.
__global__ void margin_kernel(const float* __restrict__ z, const float* __restrict__ cy, int n, int P,
                              __nv_bfloat16* __restrict__ uop, float* __restrict__ dact, double* __restrict__ part) {
  VTX_PDL_TRIGGER();
  double loss[1] = {0.0};
  VTX_COL_LOOP(n) {
    const float zc = z[i * P + p], s = cy[i * P + p];
    const float c = fabsf(s), y = s < 0.f ? -1.f : 1.f;
    const float m = 1.f - y * zc;
    const bool act = c > 0.f && m > 0.f;
    if (act) loss[0] += (double)c * (double)m * (double)m;
    store_split(uop, n, P, i, p, act ? 2.f * c * (zc - y) : 0.f);
    dact[i * P + p] = act ? c : 0.f;
  }
  col_store<1>(loss, part, P);
}

// y += x when add; part[0] = sum y^2, part[1] = sum x y, part[2] = sum x^2 (after the add)
__global__ void axpy_dot_kernel(float* __restrict__ y, const float* __restrict__ x, int rows, int P, int add,
                                double* __restrict__ part) {
  VTX_PDL_TRIGGER();
  double acc[3] = {0.0, 0.0, 0.0};
  VTX_COL_LOOP(rows) {
    const float xv = x[i * P + p];
    float yv = y[i * P + p];
    if (add) { yv += xv; y[i * P + p] = yv; }
    acc[0] += (double)yv * yv;
    acc[1] += (double)xv * yv;
    acc[2] += (double)xv * xv;
  }
  col_store<3>(acc, part, P);
}

// v = 2 dact t: the generalised Hessian's middle factor applied to t = X d
__global__ void hess_mid_kernel(const float* __restrict__ t, const float* __restrict__ dact, int n, int P,
                                __nv_bfloat16* __restrict__ vop) {
  VTX_PDL_TRIGGER();
  VTX_COL_LOOP(n) store_split(vop, n, P, i, p, 2.f * dact[i * P + p] * t[i * P + p]);
}

// Start of a Newton step, one thread per problem: objective, gradient norm and the convergence test; CG set-up.
__global__ void newton_begin_kernel(const double* __restrict__ part_loss, const double* __restrict__ part_g, int P,
                                   double* __restrict__ scal, int* __restrict__ flags, double eps, int max_newton,
                                   int* __restrict__ n_running) {
  VTX_PDL_TRIGGER();
  __shared__ int cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  int mine = 0;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    double* sc = scal + p;
    int* fl = flags + p;
    const double g2 = col_sum(part_g, P, p), ww = col_sum(part_g + 2LL * kSl * P, P, p);
    sc[VTX_SVM_F * P] = 0.5 * ww + col_sum(part_loss, P, p);
    sc[VTX_SVM_GNORM * P] = sqrt(g2);
    if (fl[VTX_SVM_NEWTON * P] == 0) sc[VTX_SVM_GNORM0 * P] = sqrt(g2);
    if (fl[VTX_SVM_STATUS * P] == 0) {
      if (g2 <= eps * eps * sc[VTX_SVM_GNORM0 * P] * sc[VTX_SVM_GNORM0 * P]) fl[VTX_SVM_STATUS * P] = 1;
      else if (fl[VTX_SVM_NEWTON * P] >= max_newton) fl[VTX_SVM_STATUS * P] = 2;
    }
    const bool run = fl[VTX_SVM_STATUS * P] == 0;
    fl[VTX_SVM_CG_DONE * P] = run ? 0 : 1;
    fl[VTX_SVM_CG_ITERS * P] = 0;
    sc[VTX_SVM_RR * P] = g2;
    sc[VTX_SVM_CG_TOL2 * P] = 0.01 * g2;  // forcing term 0.1: ||H s + g|| <= 0.1 ||g||
    mine += run;
  }
  atomicAdd(&cnt, mine);
  __syncthreads();
  if (threadIdx.x == 0) *n_running = cnt;
}

// r = -g, d = r, s = 0 (zero for problems that do not run), dop = split(d)
__global__ void cg_start_kernel(const float* __restrict__ g, float* __restrict__ r, float* __restrict__ d,
                                float* __restrict__ s, const int* __restrict__ flags, int rows, int P,
                                __nv_bfloat16* __restrict__ dop) {
  VTX_PDL_TRIGGER();
  VTX_COL_LOOP(rows) {
    const float v = flags[VTX_SVM_CG_DONE * P + p] ? 0.f : -g[i * P + p];
    r[i * P + p] = v; d[i * P + p] = v; s[i * P + p] = 0.f;
    store_split(dop, rows, P, i, p, v);
  }
}

// alpha = rr / d.Hd;  s += alpha d;  r -= alpha Hd;  part[0] = sum r^2 (the new residual norm)
__global__ void cg_update_kernel(float* __restrict__ s, float* __restrict__ r, const float* __restrict__ d,
                                 const float* __restrict__ hd, const double* __restrict__ part_dhd,
                                 const double* __restrict__ scal, const int* __restrict__ flags, int rows, int P,
                                 double* __restrict__ part_rr) {
  VTX_PDL_TRIGGER();
  double acc[1] = {0.0};
  {
    const int pc = blockIdx.x * 32 + threadIdx.x;
    const bool run = flags[VTX_SVM_CG_DONE * P + pc] == 0;
    const float alpha = run ? (float)(scal[VTX_SVM_RR * P + pc] / col_sum(part_dhd, P, pc)) : 0.f;
    VTX_COL_LOOP(rows) {
      float rv = r[i * P + p];
      if (run) {
        s[i * P + p] += alpha * d[i * P + p];
        rv -= alpha * hd[i * P + p];
        r[i * P + p] = rv;
      }
      acc[0] += (double)rv * rv;
    }
  }
  col_store<1>(acc, part_rr, P);
}

// End of a CG iteration, one thread per problem: beta, the residual test and the iteration cap.
__global__ void cg_scalars_kernel(const double* __restrict__ part_rr, int P, double* __restrict__ scal,
                                  int* __restrict__ flags, int max_cg, int* __restrict__ n_running) {
  VTX_PDL_TRIGGER();
  __shared__ int cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  int mine = 0;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    double* sc = scal + p;
    int* fl = flags + p;
    sc[VTX_SVM_BETA * P] = 0.0;
    if (fl[VTX_SVM_CG_DONE * P]) continue;
    const double rr = col_sum(part_rr, P, p);
    const int it = ++fl[VTX_SVM_CG_ITERS * P];
    ++fl[VTX_SVM_CG_TOTAL * P];
    sc[VTX_SVM_BETA * P] = rr / sc[VTX_SVM_RR * P];
    sc[VTX_SVM_RR * P] = rr;
    if (rr <= sc[VTX_SVM_CG_TOL2 * P]) {
      fl[VTX_SVM_CG_DONE * P] = 1;
    } else if (it >= max_cg) {
      fl[VTX_SVM_CG_DONE * P] = 1;
      fl[VTX_SVM_CG_CAPPED * P] = 1;
    } else {
      ++mine;
    }
  }
  atomicAdd(&cnt, mine);
  __syncthreads();
  if (threadIdx.x == 0) *n_running = cnt;
}

// d = r + beta d for problems still in CG; dop = split(d)
__global__ void cg_direction_kernel(const float* __restrict__ r, float* __restrict__ d, const double* __restrict__ scal,
                                    const int* __restrict__ flags, int rows, int P, __nv_bfloat16* __restrict__ dop) {
  VTX_PDL_TRIGGER();
  VTX_COL_LOOP(rows) {
    float dv = d[i * P + p];
    if (!flags[VTX_SVM_CG_DONE * P + p]) {
      dv = r[i * P + p] + (float)scal[VTX_SVM_BETA * P + p] * dv;
      d[i * P + p] = dv;
    }
    store_split(dop, rows, P, i, p, dv);
  }
}

// block-wide sums in a fixed order (deterministic); every thread gets the result
template <int NV>
__device__ __forceinline__ void block_sum(double (&v)[NV], double* sh /* [NV][kLsThreads / 32] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    double x = v[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == 0) sh[j * 32 + warp] = x;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    double s = 0.0;
    for (int w = 0; w < nw; ++w) s += sh[j * 32 + w];
    v[j] = s;
  }
  __syncthreads();
}

// Exact line search on phi(a) = f(w + a s), one CTA per problem.  phi is a convex piecewise quadratic:
//   phi'(a) = w.s + a s.s + sum_{active at a} 2 c (z + a t - y) t,   t = X s,
// whose root is found by Newton's method on the current piece inside a bracket [lo, hi] (bisection when a Newton
// point leaves it); the point is exact once a Newton point has the active set it was computed from.  step = the root;
// the problem converges when the decrease phi(0) - phi(step) is at most decrease_tol * phi(0).
__global__ void __launch_bounds__(kLsThreads) line_search_kernel(
    const float* __restrict__ z, const float* __restrict__ t, const float* __restrict__ cy, int n, int P,
    const double* __restrict__ part_dots, double* __restrict__ scal, int* __restrict__ flags, double decrease_tol) {
  VTX_PDL_TRIGGER();
  extern __shared__ float ls_smem[];
  __shared__ double red[3 * 32];
  const int p = blockIdx.x;
  if (flags[VTX_SVM_STATUS * P + p] != 0) {
    if (threadIdx.x == 0) scal[VTX_SVM_STEP * P + p] = 0.0;
    return;
  }
  float* zs = ls_smem;
  float* ts = zs + n;
  float* cs = ts + n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    zs[i] = z[(long long)i * P + p]; ts[i] = t[(long long)i * P + p]; cs[i] = cy[(long long)i * P + p];
  }
  __syncthreads();
  // part_dots: [0] = s.s, [1] = w.s, [2] = w.w (axpy_dot with y = s, x = w)
  const double ss = col_sum(part_dots, P, p), ws = col_sum(part_dots + (long long)kSl * P, P, p);
  double lo = 0.0, hi = INFINITY, a = 1.0, a_prev = 0.0;
  bool from_newton = false;
  for (int it = 0; it < 100; ++it) {
    double v[3] = {0.0, 0.0, 0.0};  // phi' - (w.s + a s.s), phi'' - s.s, active-set changes since a_prev
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const double c = fabs((double)cs[i]), y = cs[i] < 0.f ? -1.0 : 1.0, zi = zs[i], ti = ts[i];
      const bool act = c > 0.0 && 1.0 - y * (zi + a * ti) > 0.0;
      const bool act_prev = c > 0.0 && 1.0 - y * (zi + a_prev * ti) > 0.0;
      if (act) { v[0] += 2.0 * c * (zi + a * ti - y) * ti; v[1] += 2.0 * c * ti * ti; }
      v[2] += act != act_prev;
    }
    block_sum<3>(v, red);
    const double d1 = ws + a * ss + v[0], d2 = ss + v[1];
    if (from_newton && v[2] == 0.0) break;  // a came from a Newton step on this very piece: the root
    if (d1 == 0.0) break;
    if (d1 < 0.0) lo = a; else hi = a;
    double an = a - d1 / d2;
    from_newton = an > lo && an < hi;
    if (!from_newton) an = isinf(hi) ? 2.0 * a : 0.5 * (lo + hi);
    if (an == a) break;
    a_prev = a;
    a = an;
  }
  // decrease = phi(0) - phi(a)
  double v[1] = {0.0};
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double c = fabs((double)cs[i]), y = cs[i] < 0.f ? -1.0 : 1.0, zi = zs[i], ti = ts[i];
    const double m0 = fmax(0.0, 1.0 - y * zi), m1 = fmax(0.0, 1.0 - y * (zi + a * ti));
    v[0] += c * (m0 * m0 - m1 * m1);
  }
  block_sum<1>(v, red);
  if (threadIdx.x == 0) {
    const double dec = v[0] - a * ws - 0.5 * a * a * ss;
    scal[VTX_SVM_STEP * P + p] = a;
    ++flags[VTX_SVM_NEWTON * P + p];
    if (dec <= decrease_tol * scal[VTX_SVM_F * P + p]) flags[VTX_SVM_STATUS * P + p] = 1;
  }
}

// w += step s; wop = split(w)
__global__ void newton_step_kernel(float* __restrict__ w, const float* __restrict__ s, const double* __restrict__ scal,
                                   int rows, int P, __nv_bfloat16* __restrict__ wop) {
  VTX_PDL_TRIGGER();
  VTX_COL_LOOP(rows) {
    float wv = w[i * P + p];
    const double a = scal[VTX_SVM_STEP * P + p];
    if (a != 0.0) { wv += (float)a * s[i * P + p]; w[i * P + p] = wv; }
    store_split(wop, rows, P, i, p, wv);
  }
}

// ------------------------------------------------------------------------------------------------ average precision
// Order-preserving key of a float (larger float -> larger key); -0 and +0 are one threshold, as they compare equal
__device__ __forceinline__ uint32_t float_key(float f) {
  const uint32_t u = __float_as_uint(f == 0.f ? 0.f : f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Inclusive block scan over one value per thread (kApThreads threads); op 0 = sum, 1 = max
template <int OP>
__device__ __forceinline__ int block_scan(int v, int* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = OP == 0 ? v + u : max(v, u);
  }
  if (lane == 31) sh[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int x = sh[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x = OP == 0 ? x + u : max(x, u);
    }
    sh[lane] = x;
  }
  __syncthreads();
  if (warp > 0) v = OP == 0 ? v + sh[warp - 1] : max(v, sh[warp - 1]);
  __syncthreads();
  return v;
}

// One CTA per scored column j: (score column, label column, fold) = cols[3j .. 3j+2].  Sample i takes part when its
// label labels[i, label column] is 0 or 1 and (fold < 0 or folds[i, label column] == fold).  Keys (score, label) are
// bitonic-sorted in descending order in shared memory; AP = sum over distinct thresholds of
// (recall_k - recall_{k-1}) precision_k, ties forming one threshold (sklearn's average_precision_score); 0 when the
// column has no positive sample.
__global__ void __launch_bounds__(kApThreads) average_precision_kernel(
    const float* __restrict__ scores, long long lds, int n, const int8_t* __restrict__ labels, long long ldl,
    const int8_t* __restrict__ folds, long long ldf, const int* __restrict__ cols, int npow2, double* __restrict__ ap) {
  VTX_PDL_TRIGGER();
  extern __shared__ unsigned long long ap_keys[];
  __shared__ int scan_sh[32];
  __shared__ double red[32];
  const int sc = cols[3 * blockIdx.x], lc = cols[3 * blockIdx.x + 1], fold = cols[3 * blockIdx.x + 2];
  for (int i = threadIdx.x; i < npow2; i += blockDim.x) {
    unsigned long long key = 0ull;  // excluded samples sort last
    if (i < n) {
      const int lab = labels[(long long)i * ldl + lc];
      if ((lab == 0 || lab == 1) && (fold < 0 || folds[(long long)i * ldf + lc] == fold))
        key = ((unsigned long long)float_key(scores[(long long)i * lds + sc]) << 32) | (unsigned)(2 * lab + 1);
    }
    ap_keys[i] = key;
  }
  __syncthreads();
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < npow2; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = ap_keys[i], b = ap_keys[l];
          const bool desc = (i & k) == 0;
          if (desc ? a < b : a > b) { ap_keys[i] = b; ap_keys[l] = a; }
        }
      }
      __syncthreads();
    }
  }
  // Thread t owns the contiguous items [t * per, (t + 1) * per).  A boundary closes a tie group (the last item of a
  // run of equal scores among the included samples).  AP * #positives = sum over boundaries b of
  // (tps_b - tps_{previous boundary}) * tps_b / (b + 1) = sum over positives i of tps_{b(i)} / (b(i) + 1), where b(i)
  // is the boundary closing i's group and tps_b the number of positives up to b.
  const int per = npow2 / kApThreads, base = threadIdx.x * per;
  int* tps_at = reinterpret_cast<int*>(ap_keys + npow2);
  __shared__ int first_b[kApThreads];
  __shared__ int total_pos;
  auto boundary = [&](int i, unsigned long long key) {
    return key != 0ull && (i + 1 == npow2 || ap_keys[i + 1] == 0ull || (ap_keys[i + 1] >> 32) != (key >> 32));
  };
  int pos = 0, firstb = INT_MAX;
  for (int q = 0; q < per; ++q) {
    const unsigned long long key = ap_keys[base + q];
    pos += (int)((key >> 1) & 1ull);
    if (firstb == INT_MAX && boundary(base + q, key)) firstb = base + q;
  }
  const int pos_incl = block_scan<0>(pos, scan_sh);
  first_b[threadIdx.x] = firstb;
  if (threadIdx.x == kApThreads - 1) total_pos = pos_incl;
  int run = pos_incl - pos;
  for (int q = 0; q < per; ++q) {
    run += (int)((ap_keys[base + q] >> 1) & 1ull);
    tps_at[base + q] = run;
  }
  __syncthreads();
  // the boundary closing a group that runs past this chunk is the first boundary of a later chunk
  int b = INT_MAX;
  if (ap_keys[base] != 0ull)
    for (int t2 = threadIdx.x + 1; t2 < kApThreads && b == INT_MAX; ++t2) b = first_b[t2];
  double acc = 0.0;
  for (int q = per - 1; q >= 0; --q) {
    const int i = base + q;
    const unsigned long long key = ap_keys[i];
    if (key == 0ull) continue;
    if (boundary(i, key)) b = i;
    if ((key >> 1) & 1ull) acc += (double)tps_at[b] / (double)(b + 1);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kApThreads / 32; ++w) s += red[w];
    ap[blockIdx.x] = total_pos > 0 ? s / (double)total_pos : 0.0;
  }
}

}  // namespace vtx

using namespace vtx;
#define STREAM reinterpret_cast<cudaStream_t>(stream)
#define REQ(cond, msg) \
  if (!(cond)) return set_error(VTX_EINVAL, "%s: %s", __func__, msg)

static dim3 col_grid(int P) { return dim3((unsigned)(P / 32), kSl); }
static const dim3 kColBlock(32, kTy);

extern "C" int vtx_svm_split_x(const float* x, int64_t ldx, int n, int d, int n_pad, int dp, void* xcat, void* xstk,
                               void* stream) {
  REQ(x && (xcat || xstk) && n > 0 && d > 0 && ldx >= d, "bad arguments");
  REQ(n_pad >= n && n_pad % 64 == 0 && dp > d && dp % 64 == 0, "needs n_pad >= n, dp > d, both multiples of 64");
  const long long total = (long long)n_pad * dp;
  const int blocks = (int)((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096);
  split_x_kernel<<<blocks, 256, 0, STREAM>>>(x, ldx, n, d, n_pad, dp, (__nv_bfloat16*)xcat, (__nv_bfloat16*)xstk);
  return check_launch("svm_split_x");
}

#define REQ_COLS(rows, P) REQ((rows) > 0 && (P) > 0 && (P) % 64 == 0, "needs rows > 0 and P % 64 == 0")

extern "C" int vtx_svm_split_cols(const float* v, int rows, int P, void* op, void* stream) {
  REQ(v && op, "bad arguments");
  REQ_COLS(rows, P);
  split_cols_kernel<<<col_grid(P), kColBlock, 0, STREAM>>>(v, rows, P, (__nv_bfloat16*)op);
  return check_launch("svm_split_cols");
}

extern "C" int vtx_svm_margin(const float* z, const float* cy, int n, int P, void* uop, float* dact, double* part,
                              void* stream) {
  REQ(z && cy && uop && dact && part, "bad arguments");
  REQ_COLS(n, P);
  margin_kernel<<<col_grid(P), kColBlock, 0, STREAM>>>(z, cy, n, P, (__nv_bfloat16*)uop, dact, part);
  return check_launch("svm_margin");
}

extern "C" int vtx_svm_axpy_dot(float* y, const float* x, int rows, int P, int add, double* part, void* stream) {
  REQ(y && x && part, "bad arguments");
  REQ_COLS(rows, P);
  axpy_dot_kernel<<<col_grid(P), kColBlock, 0, STREAM>>>(y, x, rows, P, add, part);
  return check_launch("svm_axpy_dot");
}

extern "C" int vtx_svm_hess_mid(const float* t, const float* dact, int n, int P, void* vop, void* stream) {
  REQ(t && dact && vop, "bad arguments");
  REQ_COLS(n, P);
  hess_mid_kernel<<<col_grid(P), kColBlock, 0, STREAM>>>(t, dact, n, P, (__nv_bfloat16*)vop);
  return check_launch("svm_hess_mid");
}

extern "C" int vtx_svm_newton_begin(const double* part_loss, const double* part_g, int P, double* scal, int32_t* flags,
                                    double eps, int max_newton, int32_t* n_running, void* stream) {
  REQ(part_loss && part_g && scal && flags && n_running && P > 0 && eps >= 0.0 && max_newton > 0, "bad arguments");
  newton_begin_kernel<<<1, 1024, 0, STREAM>>>(part_loss, part_g, P, scal, flags, eps, max_newton, n_running);
  return check_launch("svm_newton_begin");
}

extern "C" int vtx_svm_cg_start(const float* g, float* r, float* d, float* s, const int32_t* flags, int rows, int P,
                                void* dop, void* stream) {
  REQ(g && r && d && s && flags && dop, "bad arguments");
  REQ_COLS(rows, P);
  cg_start_kernel<<<col_grid(P), kColBlock, 0, STREAM>>>(g, r, d, s, flags, rows, P, (__nv_bfloat16*)dop);
  return check_launch("svm_cg_start");
}

extern "C" int vtx_svm_cg_update(float* s, float* r, const float* d, const float* hd, const double* part_dhd,
                                 const double* scal, const int32_t* flags, int rows, int P, double* part_rr,
                                 void* stream) {
  REQ(s && r && d && hd && part_dhd && scal && flags && part_rr, "bad arguments");
  REQ_COLS(rows, P);
  cg_update_kernel<<<col_grid(P), kColBlock, 0, STREAM>>>(s, r, d, hd, part_dhd, scal, flags, rows, P, part_rr);
  return check_launch("svm_cg_update");
}

extern "C" int vtx_svm_cg_scalars(const double* part_rr, int P, double* scal, int32_t* flags, int max_cg,
                                  int32_t* n_running, void* stream) {
  REQ(part_rr && scal && flags && n_running && P > 0 && max_cg > 0, "bad arguments");
  cg_scalars_kernel<<<1, 1024, 0, STREAM>>>(part_rr, P, scal, flags, max_cg, n_running);
  return check_launch("svm_cg_scalars");
}

extern "C" int vtx_svm_cg_direction(const float* r, float* d, const double* scal, const int32_t* flags, int rows, int P,
                                    void* dop, void* stream) {
  REQ(r && d && scal && flags && dop, "bad arguments");
  REQ_COLS(rows, P);
  cg_direction_kernel<<<col_grid(P), kColBlock, 0, STREAM>>>(r, d, scal, flags, rows, P, (__nv_bfloat16*)dop);
  return check_launch("svm_cg_direction");
}

extern "C" int vtx_svm_line_search(const float* z, const float* t, const float* cy, int n, int P,
                                   const double* part_dots, double* scal, int32_t* flags, double decrease_tol,
                                   void* stream) {
  REQ(z && t && cy && part_dots && scal && flags && P > 0 && decrease_tol >= 0.0, "bad arguments");
  REQ(n > 0 && n <= VTX_SVM_MAX_N, "needs 0 < n <= VTX_SVM_MAX_N (16384)");
  const int smem = 3 * n * (int)sizeof(float);
  cudaFuncSetAttribute(line_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  line_search_kernel<<<P, kLsThreads, smem, STREAM>>>(z, t, cy, n, P, part_dots, scal, flags, decrease_tol);
  return check_launch("svm_line_search");
}

extern "C" int vtx_svm_newton_step(float* w, const float* s, const double* scal, int rows, int P, void* wop,
                                   void* stream) {
  REQ(w && s && scal && wop, "bad arguments");
  REQ_COLS(rows, P);
  newton_step_kernel<<<col_grid(P), kColBlock, 0, STREAM>>>(w, s, scal, rows, P, (__nv_bfloat16*)wop);
  return check_launch("svm_newton_step");
}

extern "C" int vtx_svm_average_precision(const float* scores, int64_t lds, int n, const int8_t* labels, int64_t ldl,
                                         const int8_t* folds, int64_t ldf, const int32_t* cols, int ncols, double* ap,
                                         void* stream) {
  REQ(scores && labels && cols && ap && ncols > 0 && n > 0, "bad arguments");
  if (n > VTX_SVM_MAX_N) return set_error(VTX_EUNSUPPORTED, "%s: needs n <= VTX_SVM_MAX_N (16384)", __func__);
  int npow2 = 2 * kApThreads;
  while (npow2 < n) npow2 <<= 1;
  const int smem = npow2 * (int)(sizeof(unsigned long long) + sizeof(int));
  cudaFuncSetAttribute(average_precision_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  average_precision_kernel<<<ncols, kApThreads, smem, STREAM>>>(scores, lds, n, labels, ldl, folds, ldf, cols, npow2,
                                                                ap);
  return check_launch("svm_average_precision");
}
