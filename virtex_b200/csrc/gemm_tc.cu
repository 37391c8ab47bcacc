// wgmma / TMA GEMM for sm_90a -- the one tensor-core kernel behind every GEMM-shaped op of the VirTex bicaptioning
// step (1x1 convs, implicit 3x3 convs, im2col'd strided convs, all nn.Linear fwd/dgrad/wgrad, vocabulary projection).
// See include/virtex_b200.h (VtxGemm) for the contract.
//
// Structure (persistent, warp specialised, one CTA per SM, 384 threads = three warpgroups):
//   warpgroup 0 : TMA producer (one thread)  global -> 128B-swizzled smem ring of (A 16 KB, B = tile_n*128 B) stages;
//                 the ring depth is whatever fits next to the output staging tile (2..8 stages); it also owns the tile
//                 schedule: every tile index (static round robin, or fetched from a per-launch atomic counter) is
//                 published to the consumers through a small index ring in shared memory.  It hands most of its
//                 registers to the consumers (setmaxnreg).
//   warpgroups 1, 2 : MMA + epilogue: wgmma.mma_async m64nNk16 (N = tile_n in {64, 128, 192, 256}) with fp32
//                 accumulators in registers, then bias / residual / activation -> bf16 tile in 128B-swizzled smem ->
//                 one thread issues TMA stores (cp.async.bulk.tensor, out-of-bounds rows/columns clipped by the
//                 hardware); a statistics pass over the staged tile accumulates, in registers across the CTA's tiles,
//                 either the BN batch statistics of a conv output or (p.bnr) the BN-BACKWARD sums of a gradient.
//                 (fp32 / split-K outputs skip staging: stores or fp32 atomics straight from registers.)
//                 Two schedules (template parameter PP, chosen per launch on the host): lockstep -- both warpgroups
//                 on every tile, rows [0, 64) and [64, 128) -- or ping-pong -- each warpgroup computes every other
//                 tile whole, and its epilogue overlaps the other warpgroup's MMAs (tiles up to 128 wide).
// Mbarrier pipelines: smem full/empty (TMA <-> MMA), residual landed, the tile-index ring, and (ping-pong) the order in
// which the two warpgroups issue their K loops.
//
// Operand "major-ness" is a runtime property (wgmma transpose bits + smem descriptor strides), so the same kernel serves
// fprop (A,B K-major), dgrad (B MN-major) and wgrad (A,B MN-major) without transposing activations.
// conv_mode 1/2 replace the 2D TMA loads by 4D NHWC box loads whose out-of-bounds elements are zero-filled by the TMA
// unit: that *is* the im2col of a 3x3/stride-1/pad-1 convolution, with no extra HBM traffic.  conv_mode 4 (the
// [(tap, cin), cout] weight gradient of a 64 -> 64 3x3 conv) runs as conv_mode 2 with a transposed fp32 store.
#include <stdlib.h>
#include "ptx.cuh"
#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

// The tap geometry of the implicit-conv modes 1 / 2 is a runtime parameter (taps per kernel row, zero padding, tap
// count): 3 x 3 / pad 1 for the bottleneck convs, and 4 x 1 / pad 0 for conv_mode 5 / 6 -- the 7x7/2 stem conv as a
// 4-tap implicit GEMM over the space-to-depth view of the image (csrc/stem_s2d.cu).
#define KP_TAPS_W p.taps_w
#define KP_PAD p.pad
#define KP_NTAPS p.ntaps

namespace vtx {

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kMaxStages = 8;
constexpr int kABytes = kBM * kBK * 2;        // 16384
constexpr int kSmemTotal = 232448;            // 227 KB: the per-block maximum on sm_90
constexpr int kCtrlBytes = 1024;              // barriers + tile-index ring, placed right after the 1024-aligned base
constexpr int kThreads = 384;                 // producer warpgroup + two MMA / epilogue warpgroups
constexpr int kEpiThreads = 256;

// x / d for 0 <= x < 2^31 and the launch-invariant divisor d: (umulhi(x, mul) >> shr), d == 1 handled apart
struct FastDiv {
  uint32_t mul, shr;  // mul == 0 encodes d == 1
};
__device__ __forceinline__ int fdiv(int x, const FastDiv& f) {
  return f.mul == 0u ? x : (int)(__umulhi((uint32_t)x, f.mul) >> f.shr);
}
static FastDiv make_fastdiv(int d) {
  FastDiv f;
  f.mul = 0;
  f.shr = 0;
  if (d > 1) {
    int l = 0;
    while ((1u << l) < (uint32_t)d) ++l;  // ceil(log2 d)
    const int pw = 31 + l;
    const unsigned long long m = ((1ull << pw) + (uint32_t)d - 1) / (uint32_t)d;  // 2^31 <= m < 2^32: never 0
    f.mul = (uint32_t)m;
    f.shr = (uint32_t)(pw - 32);
  }
  return f;
}

struct GemmKParams {
  int M, N, K;
  int bn;
  int a_mn, b_mn;
  int m_tiles, n_tiles, k_splits;
  int kb_total, kb_per_split;
  int mode;
  int cH, cW, cN, cpb;
  int lbw, lbh, lbn;
  int tiles_w, tiles_h;
  int out_f32, atomic, act;
  int stages, stage_bytes;   // smem ring depth / bytes per stage
  int cbytes, nbuf;          // bytes of one bf16 staging buffer (0: no staging) / number of staging buffers
  int res_tma;               // residual tile is TMA-loaded into the staging buffer and added there
  float alpha;
  void* D;
  long long ldd;
  const float* bias;
  int bias_pairs;            // the bias can be read as float2 pairs: 8-byte aligned and N even
  const __nv_bfloat16* residual;
  long long ldr;
  const uint8_t* res_mask;   // optional bit mask [M, N/8]: the residual of (row, col) is added only where its bit is set
  float* stats;
  int taps_w, pad, ntaps;    // taps per kernel row / zero padding / number of taps of the implicit conv (3, 1, 9 for 3x3)
  int cstride;               // spatial stride of the implicit conv (1 or 2): output position w reads input cstride*w + kw - pad
  // division by the launch-invariant tile-schedule extents as multiply-high + shift (a runtime integer division costs
  // ~25 dependent instructions; the schedule decode was ~13 % of the epilogue's instructions on the short-K convs)
  FastDiv d_mn, d_nt, d_mt, d_tw, d_twh, d_cpb, d_taps;
  // Dynamic tile scheduler: *sched is a counter that only ever grows; this launch owns the values [sched_base,
  // sched_base + chunks + gridDim.x) of it (the host knows how many fetches a launch performs: one per chunk of
  // sched_chunk consecutive tiles plus exactly one end marker per CTA), so nothing is reset and no CTA has to wait for an
  // atomic on its way out.  With a static round-robin schedule an SM that is held by somebody else's CTA (NCCL's
  // all-reduce kernels during the overlapped gradient exchange) delays ITS fixed share of tiles to the end of every GEMM
  // issued meanwhile; here the CTAs that do run drain the counter and a late CTA finds nothing left.
  // nullptr: static schedule (single-GPU default -- see vtx_gemm_set_dynamic_schedule).
  unsigned int* sched;
  unsigned int sched_base;
  int sched_chunk;
  int nt_major;
  // BN-backward reduction fused into the epilogue (bnr != 0; `stats` then holds the [2, N] sums of dz and dz * xhat):
  // y has the geometry of D -- row stride bnr_ldy for plain GEMMs, (w, h, n) strides for implicit-conv outputs and views
  const __nv_bfloat16* bnr_y;
  const float* bnr_bnp;      // [4, N]: mean, invstd, scale, shift of the BN whose output gradient D is
  const uint8_t* bnr_mask;   // optional ReLU bit mask [M, N/8] (plain GEMMs); nullptr: mask recomputed from y
  long long bnr_ldy, bnr_sw, bnr_sh, bnr_sn;
  int vW, vH;                // extent of the output (view) grid of the implicit-conv modes
  int bnr_prefetch;          // pull the y tile into L2 with a TMA prefetch when the tile starts
  int bnr;                   // 0: plain statistics (or none), 1: BN-backward sums, ReLU mask from y, 2: from a bit mask
  int trans_d;               // fp32 output stored transposed: D[col * ldd + row] (conv_mode 4)
  // folded eval-mode BatchNorm (kernel variant SS): per-column affine map of the accumulators, [N] each
  const float* col_scale;
  const float* col_shift;
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

__device__ __forceinline__ void epi_bar(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// schedule index -> (split, row tile, column tile)
__device__ __forceinline__ void decode_tile(const GemmKParams& p, int t, int& ks, int& mt, int& nt) {
  ks = fdiv(t, p.d_mn);
  const int rem = t - ks * (p.m_tiles * p.n_tiles);
  if (p.nt_major) {
    nt = fdiv(rem, p.d_mt);
    mt = rem - nt * p.m_tiles;
  } else {
    mt = fdiv(rem, p.d_nt);
    nt = rem - mt * p.n_tiles;
  }
}
__device__ __forceinline__ void tma_prefetch_l2_2d(const void* tmap, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(tmap)),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_prefetch_l2_4d(const void* tmap, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ uint4 ldg128_nc(const void* ptr) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.b32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(ptr));
  return v;
}
constexpr int kSched = 8;  // depth of the tile-index ring between the producer (who fetches) and the MMA / epilogue roles

// acc pair -> bf16x2, + (optionally masked) bf16x2 residual word in ONE packed add (the rounding torch's own bf16 graph
// applies: conv output rounded to bf16, then the bf16 sum rounded again)
__device__ __forceinline__ uint32_t add_res_bf16x2(float lo, float hi, uint32_t res) {
  const __nv_bfloat162 a = __floats2bfloat162_rn(lo, hi);
  const __nv_bfloat162 r = *reinterpret_cast<const __nv_bfloat162*>(&res);
  const __nv_bfloat162 o = __hadd2(a, r);
  return *reinterpret_cast<const uint32_t*>(&o);
}
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ uint32_t lds32(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(saddr));
  return v;
}
__device__ __forceinline__ void sts32(uint32_t saddr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_bn(float* d, uint64_t ad, uint64_t bd, uint32_t accumulate) {
  if constexpr (BN == 64) wgmma_n64<TA, TB>(d, ad, bd, accumulate);
  else if constexpr (BN == 128) wgmma_n128<TA, TB>(d, ad, bd, accumulate);
  else if constexpr (BN == 192) wgmma_n192<TA, TB>(d, ad, bd, accumulate);
  else wgmma_n256<TA, TB>(d, ad, bd, accumulate);
}

// K loop of one tile for one consumer warpgroup: NH wgmma m64nBNk16 per 16-deep K step (NH = 1: the 64 rows starting at
// byte a_off of the A stage; NH = 2: all 128 rows, two MMAs sharing the B descriptor), one commit group per stage.  A
// stage is handed back to the producer (one arrive per warpgroup) as soon as the MMAs of the NEXT stage are issued and
// the ones reading it have completed, so one stage's MMAs are always in flight while the warpgroup waits for the
// following stage.  `order_next` (ping-pong schedule): arrived on by every thread once the tile's last MMAs are issued,
// which lets the other consumer warpgroup start its K loop while these complete.
template <int BN, int NH, int TA, int TB>
__device__ __forceinline__ void mma_tile(float* acc, uint8_t* smem, const GemmKParams& p, int kb0, int kb1,
                                         uint32_t a_off, uint64_t* full_bar, uint64_t* empty_bar, int stage,
                                         uint32_t phase, bool signal, uint64_t* order_next) {
  constexpr uint32_t a_step = TA ? 2048u : 32u;  // 16 k: two 8-row groups (MN-major) / 32 bytes along a row (K-major)
  constexpr uint32_t b_step = TB ? 2048u : 32u;
  constexpr uint32_t a_lbo = TA ? 8192u : 16u;
  constexpr uint32_t b_lbo = TB ? 8192u : 16u;
  int prev = -1;
#pragma unroll
  for (int i = 0; i < NH * BN / 2; ++i) fence_operand(acc[i]);
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t s0 = smem_u32(smem + stage * p.stage_bytes);
    const uint32_t sA = s0 + a_off;  // 64 rows (K-major) or a 64-row atom (MN-major) per 8 KB
    const uint32_t sB = s0 + (uint32_t)kABytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) {
      const uint64_t bd = make_wgmma_desc(sB + k * b_step, b_lbo, 1024);
#pragma unroll
      for (int h = 0; h < NH; ++h)
        wgmma_bn<BN, TA, TB>(acc + h * (BN / 2), make_wgmma_desc(sA + h * 8192u + k * a_step, a_lbo, 1024), bd,
                             (kb > kb0 || k > 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && signal) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == p.stages) { stage = 0; phase ^= 1; }
  }
  if (order_next != nullptr) mbar_arrive(order_next);
  wgmma_wait<0>();
  if (prev >= 0 && signal) mbar_arrive(&empty_bar[prev]);
#pragma unroll
  for (int i = 0; i < NH * BN / 2; ++i) fence_operand(acc[i]);
}

// p.bnr (1: ReLU mask recomputed from y, 2: ReLU bit mask): the statistics pass over the staged output tile computes the
// BATCH-NORM BACKWARD sums instead of sum / sum of squares: this GEMM's output is the gradient dA w.r.t. a BN(+ReLU)
// output, and  sum_m dz,  sum_m dz * xhat  with dz = dA * [ReLU mask], xhat = (y - mean) * invstd  used to be a separate
// pass over dA and y (vtx_bn_bwd_reduce).  The y tile is pulled into L2 by a TMA prefetch when the tile starts and read
// with 16-byte loads in the pass.
//
// PP selects the consumer schedule:
//   false (lockstep): both consumer warpgroups work on every tile, rows [0, 64) and [64, 128), and run its epilogue
//         together while the tensor cores idle (BN up to 256);
//   true (ping-pong): each consumer warpgroup computes whole 128-row tiles on its own (BN <= 128: 2 x BN / 2
//         accumulators per thread), taking every other slot of the tile-index ring.  A pair of barriers makes the two
//         K loops alternate whole tiles, so one warpgroup's epilogue runs while the other one's MMAs do.  Each
//         warpgroup has its own staging buffer, residual barrier, named barrier and BN-statistics partials.
// SS selects the epilogue: false runs the loops below for every option; true runs only the scale / shift loop of a
// folded eval-mode BatchNorm (p.col_scale / p.col_shift, optional TMA-staged residual, optional ReLU).  A variant of
// its own keeps that loop out of the training instantiations, whose register allocation it would otherwise perturb.
template <int BN, bool PP, bool SS>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmR,
                  const __grid_constant__ CUtensorMap tmY, const GemmKParams p) {
  static_assert(!PP || BN <= 128, "ping-pong tiles keep 2 x BN / 2 accumulators per thread");
  VTX_PDL_TRIGGER();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(base);
  uint64_t* full_bar = bars;                     // [kMaxStages]
  uint64_t* empty_bar = bars + kMaxStages;       // [kMaxStages]
  uint64_t* res_bar = bars + 2 * kMaxStages;     // [2] residual tile landed in staging buffer b
  uint64_t* sch_full = res_bar + 2;              // [kSched] tile index published
  uint64_t* sch_empty = sch_full + kSched;       // [kSched] tile index read by every consumer thread that uses it
  uint64_t* order_bar = sch_empty + kSched;      // [2] (ping-pong) the other warpgroup has issued its tile's MMAs
  // [kSched] tile index | (k-blocks the producer queued before the tile << 32): the latter gives the tile's first stage
  // and phase in the operand ring (one 64-bit word: both halves are written and read together)
  volatile unsigned long long* sch_tile = reinterpret_cast<volatile unsigned long long*>(order_bar + 2);
  uint8_t* smem = base + kCtrlBytes;                       // stage ring (1024-aligned)
  uint8_t* cstage0 = smem + p.stages * p.stage_bytes;      // bf16 staging: nbuf x [bn/64 slabs][128 rows][128 B], SW128

  // broadcast from lane 0 so that the compiler sees the warp index (and every role branch on it) as warp-uniform
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int total_tiles = p.m_tiles * p.n_tiles * p.k_splits;
  const int nstages = p.stages;

  // the producer thread's first tile: requested before anything else (the counter belongs to this launch alone, so it
  // need not wait for the previous kernel) and consumed after the prologue
  int t_first = blockIdx.x;
  if (warp == 0 && lane == 0) {
    if (p.sched != nullptr) t_first = (int)(atomicAdd(p.sched, 1u) - p.sched_base) * p.sched_chunk;
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.cbytes) tma_prefetch_desc(&tmD);
    if (p.res_tma) tma_prefetch_desc(&tmR);
    if (p.bnr) tma_prefetch_desc(&tmY);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < nstages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], PP ? 1 : 2);  // one arrive per consumer warpgroup that reads the stage
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&res_bar[i], 1);
      mbar_init(&order_bar[i], 128);
    }
    for (int i = 0; i < kSched; ++i) {
      mbar_init(&sch_full[i], 1);
      mbar_init(&sch_empty[i], PP ? 128 : kEpiThreads);
    }
    fence_mbar_init();
  }
  __syncthreads();
  VTX_PDL_WAIT();  // everything above overlapped the previous kernel's tail; its results are visible from here

  if (warp < 4) {
    // ===================================================== TMA producer (warpgroup 0, one thread)
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      const uint32_t b_bytes = (uint32_t)p.bn * kBK * 2;
      int stage = 0;
      uint32_t phase = 0;
      // every tile index goes through the ring, whether it came from the counter or from the static schedule; an end
      // marker (>= total_tiles) closes it, published into two slots under the ping-pong schedule so that both consumer
      // warpgroups see one
      int t = t_first, sit = 0, kpos = 0;
      // tile after `t_`: the next one of the current chunk, else the first one of a freshly fetched chunk (dynamic), or
      // the CTA's next round-robin tile (static)
      auto next_after = [&](int t_) -> int {
        if (p.sched == nullptr) return t_ + (int)gridDim.x;
        if ((t_ + 1) % p.sched_chunk != 0 && t_ + 1 < total_tiles) return t_ + 1;
        return (int)(atomicAdd(p.sched, 1u) - p.sched_base) * p.sched_chunk;
      };
      auto publish = [&](int t_) {
        const int slot = sit & (kSched - 1);
        mbar_wait(&sch_empty[slot], ((sit / kSched) & 1) ^ 1);
        sch_tile[slot] = (unsigned long long)(uint32_t)t_ | ((unsigned long long)(uint32_t)kpos << 32);
        mbar_arrive(&sch_full[slot]);
        ++sit;
      };
      for (;;) {
        publish(t);
        if (t >= total_tiles) {
          if (PP) publish(t);
          break;
        }
        // the next index is requested now and needed only after this tile's loads are queued
        const int t_next = next_after(t);
        int ks, mt, nt;
        decode_tile(p, t, ks, mt, nt);
        const int kb0 = ks * p.kb_per_split;
        const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
        kpos += kb1 - kb0;
        int w0 = 0, h0 = 0, n0 = 0;
        if (p.mode == 1) {
          const int tn = fdiv(mt, p.d_twh);
          const int r_wh = mt - tn * (p.tiles_w * p.tiles_h);
          const int th = fdiv(r_wh, p.d_tw);
          const int tw = r_wh - th * p.tiles_w;
          w0 = tw << p.lbw; h0 = th << p.lbh; n0 = tn << p.lbn;
        }
        const int nb0 = nt * p.bn;  // first B row (column of the output)
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sA = smem + stage * p.stage_bytes;
          uint8_t* sB = sA + kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], kABytes + b_bytes);
          if (p.mode == 0) {
            if (!p.a_mn) {
              tma_load_2d(sA, &tmA, &full_bar[stage], kb * kBK, mt * kBM);
            } else {
              tma_load_2d(sA, &tmA, &full_bar[stage], mt * kBM, kb * kBK);
              tma_load_2d(sA + 8192, &tmA, &full_bar[stage], mt * kBM + 64, kb * kBK);
            }
            if (!p.b_mn) {
              tma_load_2d(sB, &tmB, &full_bar[stage], kb * kBK, nb0);
            } else {
              for (int j = 0; j < (p.bn >> 6); ++j)
                tma_load_2d(sB + j * 8192, &tmB, &full_bar[stage], nb0 + 64 * j, kb * kBK);
            }
          } else if (p.mode == 1) {
            const int tap = fdiv(kb, p.d_cpb);
            const int cb = kb - tap * p.cpb;
            const int kh = fdiv(tap, p.d_taps), kw = tap - kh * KP_TAPS_W;
            tma_load_4d(sA, &tmA, &full_bar[stage], cb * 64, p.cstride * w0 + kw - KP_PAD, p.cstride * h0 + kh - KP_PAD,
                        n0);
            tma_load_2d(sB, &tmB, &full_bar[stage], kb * kBK, nb0);
          } else {
            // wgrad: reduction block kb is a spatial box of 64 output positions
            const int tn = fdiv(kb, p.d_twh);
            const int r_wh = kb - tn * (p.tiles_w * p.tiles_h);
            const int th = fdiv(r_wh, p.d_tw);
            const int tw = r_wh - th * p.tiles_w;
            const int bw0 = tw << p.lbw, bh0 = th << p.lbh, bn0 = tn << p.lbn;
            tma_load_4d(sA, &tmA, &full_bar[stage], mt * kBM, bw0, bh0, bn0);
            tma_load_4d(sA + 8192, &tmA, &full_bar[stage], mt * kBM + 64, bw0, bh0, bn0);
            for (int j = 0; j < (p.bn >> 6); ++j) {
              const int atom = (nb0 >> 6) + j;
              const int tap = fdiv(atom, p.d_cpb);
              const int cb = atom - tap * p.cpb;
              const int kh = fdiv(tap, p.d_taps), kw = tap - kh * KP_TAPS_W;
              // atoms past the last tap are loaded fully out of bounds (zero fill) to keep the tx count fixed
              const int nn = tap < KP_NTAPS ? bn0 : p.cN + 1;
              tma_load_4d(sB + j * 8192, &tmB, &full_bar[stage], cb * 64, p.cstride * bw0 + kw - KP_PAD,
                          p.cstride * bh0 + kh - KP_PAD, nn);
            }
          }
          if (++stage == nstages) { stage = 0; phase ^= 1; }
        }
        t = t_next;
      }
    }
    return;
  }

  // ===================================================== MMA + epilogue (warpgroups 1 and 2)
  setmaxnreg_inc<232>();
  const int ct = threadIdx.x - 128;  // 0..255
  const int wg = ct >> 7;            // lockstep: this warpgroup owns rows [64 wg, 64 wg + 64) of every tile
  const int wl = (ct >> 5) & 3;      // warp within the warpgroup: rows 16 wl .. 16 wl + 15 of each 64-row block
  const bool signal = (ct & 127) == 0;
  // the threads that share an epilogue: both warpgroups (lockstep) or one (ping-pong, named barrier 1 + wg)
  constexpr int NH = PP ? 2 : 1;     // 64-row accumulator blocks per thread
  constexpr int epi_threads = PP ? 128 : kEpiThreads;
  const int bar_id = PP ? 1 + wg : 1;
  const int et = PP ? (ct & 127) : ct;
  const bool staged = p.cbytes != 0;
  // BN statistics: thread (scg, srg) owns 8 columns x st_rpt rows of every staged tile and keeps running partial sums
  // in registers across all tiles of this CTA that share the same column block; they are reduced through shared memory
  // and flushed with one atomic per column only when the column block changes (or at the end).  64 / 128 / 256-wide
  // tiles = 8 / 16 / 32 column groups x 32 / 16 / 8 row groups of 4 / 8 / 16 rows.
  const int st_lg = (p.bn == 64) ? 3 : (p.bn == 128) ? 4 : 5;  // log2(column groups)
  const int st_rgs = min(epi_threads >> st_lg, 32), st_rpt = 128 / st_rgs;  // <= 32 row groups: the flush scratch is one staging buffer
  const int scg = et & ((1 << st_lg) - 1), srg = et >> st_lg;
  const bool st_on = (scg * 8 < p.bn) && (srg < st_rgs);
  float st_s[8], st_q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) st_s[i] = st_q[i] = 0.f;
  int st_nt = -1;
  auto flush_stats = [&](uint8_t* scratch) {
    // `scratch` is a staging buffer no TMA store is reading and nobody is writing (callers guarantee it)
    float* scr = reinterpret_cast<float*>(scratch);
    if (st_on) {
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        *reinterpret_cast<float4*>(scr + (srg * p.bn + scg * 8 + i) * 2) =
            make_float4(st_s[i], st_q[i], st_s[i + 1], st_q[i + 1]);
        st_s[i] = st_q[i] = st_s[i + 1] = st_q[i + 1] = 0.f;
      }
    }
    epi_bar(bar_id, epi_threads);
    if (et < p.bn && st_nt * p.bn + et < p.N) {
      float a = 0.f, b = 0.f;
      for (int g = 0; g < st_rgs; ++g) {
        const float2 v = *reinterpret_cast<const float2*>(scr + (g * p.bn + et) * 2);
        a += v.x;
        b += v.y;
      }
      if (p.bnr) b *= __ldg(p.bnr_bnp + p.N + st_nt * p.bn + et);  // sum dz * (y - mean)  ->  sum dz * xhat
      atomicAdd(p.stats + st_nt * p.bn + et, a);
      atomicAdd(p.stats + p.N + st_nt * p.bn + et, b);
    }
    epi_bar(bar_id, epi_threads);
  };
  // asynchronous, coalesced TMA load of the residual tile of schedule slot `t_` into staging buffer `bi_`
  // (called by ONE thread, only once the TMA store that last read that buffer has finished reading it)
  auto issue_residual = [&](int t_, int bi_) {
    int ks_, mt_, nt_;
    decode_tile(p, t_, ks_, mt_, nt_);
    const int nb_ = nt_ * p.bn;
    uint8_t* buf_ = cstage0 + (size_t)bi_ * p.cbytes;
    const int slabs = (min(p.bn, p.N - nb_) + 63) >> 6;
    mbar_arrive_expect_tx(&res_bar[bi_], (uint32_t)slabs * 16384u);
    for (int sl = 0; sl < slabs; ++sl) {
      if (p.mode & 1) {
        const int tn_ = fdiv(mt_, p.d_twh);
        const int rwh_ = mt_ - tn_ * (p.tiles_w * p.tiles_h);
        const int th_ = fdiv(rwh_, p.d_tw), tw_ = rwh_ - th_ * p.tiles_w;
        tma_load_4d(buf_ + sl * 16384, &tmR, &res_bar[bi_], nb_ + sl * 64, tw_ << p.lbw, th_ << p.lbh, tn_ << p.lbn);
      } else {
        tma_load_2d(buf_ + sl * 16384, &tmR, &res_bar[bi_], nb_ + sl * 64, mt_ * kBM);
      }
    }
  };
  float acc[NH * BN / 2];
  // it: this warpgroup's tiles so far; sit: their ring slot (ping-pong: warpgroup wg takes slots wg, wg + 2, ...)
  for (int it = 0;; ++it) {
    const int sit = PP ? 2 * it + wg : it;
    const int slot = sit & (kSched - 1);
    mbar_wait(&sch_full[slot], (sit / kSched) & 1);
    const unsigned long long tk = sch_tile[slot];
    const int t = (int)(uint32_t)tk;
    const int kpos = (int)(tk >> 32);
    mbar_arrive(&sch_empty[slot]);
    if (t >= total_tiles) break;
    int ks, mt, nt;
    decode_tile(p, t, ks, mt, nt);
    const int n_base = nt * p.bn;
    int tw = 0, th = 0, tn = 0;
    if (p.mode & 1) {
      tn = fdiv(mt, p.d_twh);
      const int r_wh = mt - tn * (p.tiles_w * p.tiles_h);
      th = fdiv(r_wh, p.d_tw);
      tw = r_wh - th * p.tiles_w;
    }
    const int cbi = PP ? wg : p.nbuf > 1 ? (it & 1) : 0;
    uint8_t* cbuf = cstage0 + (size_t)cbi * p.cbytes;
    if (staged) {
      // (fused BN reduction over a TMA-loaded residual: every thread must be done READING the previous tile in its
      // statistics pass before the next residual tile lands in the same buffer)
      if (p.bnr && p.res_tma) epi_bar(bar_id, epi_threads);
      // the TMA store that last read this staging buffer must have finished reading it (with two buffers every tile
      // commits one bulk group, so the one before the latest is this buffer's)
      if (et == 0) {
        if (!PP && p.nbuf > 1) tma_store_wait_read<1>();
        else tma_store_wait_read<0>();
      }
      // the column block changed: the sums kept in registers go out through the (now idle) staging buffer -- with a
      // TMA-loaded residual that has to happen BEFORE the residual tile is requested into the same buffer
      const bool new_block = p.stats != nullptr && st_nt != nt;
      if (new_block && st_nt >= 0 && p.res_tma) {
        epi_bar(bar_id, epi_threads);
        flush_stats(cbuf);
      }
      if (et == 0) {
        if (p.res_tma) issue_residual(t, cbi);  // requested now that this buffer is free: it lands during the K loop
        if (p.bnr && p.bnr_prefetch) {
          const int slabs = (min(p.bn, p.N - n_base) + 63) >> 6;
          for (int sl = 0; sl < slabs; ++sl) {
            if (p.mode & 1) tma_prefetch_l2_4d(&tmY, n_base + sl * 64, tw << p.lbw, th << p.lbh, tn << p.lbn);
            else tma_prefetch_l2_2d(&tmY, n_base + sl * 64, mt * kBM);
          }
        }
      }
      epi_bar(bar_id, epi_threads);
      if (new_block) {
        if (st_nt >= 0 && !p.res_tma) flush_stats(cbuf);
        st_nt = nt;
      }
    }

    // ---------------- K loop: fp32 accumulators of this warpgroup's (NH x 64) x BN block in registers
    {
      const int kb0 = ks * p.kb_per_split;
      const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);
      // the tile's first k-block: the producer queued kpos k-blocks before it (ping-pong: the other warpgroup's too)
      const int stage = kpos % p.stages;
      const uint32_t phase = (uint32_t)(kpos / p.stages) & 1u;
      const uint32_t a_off = PP ? 0u : (uint32_t)wg * 8192u;
      uint64_t* order_next = nullptr;
      if (PP) {
        // the K loops alternate whole tiles: wait until the other warpgroup has issued the MMAs of the tile before
        // this one in the ring (warpgroup 1's tile `it` follows warpgroup 0's tile `it`, warpgroup 0's tile `it`
        // follows warpgroup 1's tile `it - 1`)
        if (wg == 1) mbar_wait(&order_bar[1], (uint32_t)it & 1u);
        else if (it > 0) mbar_wait(&order_bar[0], (uint32_t)(it - 1) & 1u);
        order_next = &order_bar[wg ^ 1];
      }
      if (!p.a_mn && !p.b_mn)
        mma_tile<BN, NH, 0, 0>(acc, smem, p, kb0, kb1, a_off, full_bar, empty_bar, stage, phase, signal, order_next);
      else if (!p.a_mn)
        mma_tile<BN, NH, 0, 1>(acc, smem, p, kb0, kb1, a_off, full_bar, empty_bar, stage, phase, signal, order_next);
      else if (!p.b_mn)
        mma_tile<BN, NH, 1, 0>(acc, smem, p, kb0, kb1, a_off, full_bar, empty_bar, stage, phase, signal, order_next);
      else
        mma_tile<BN, NH, 1, 1>(acc, smem, p, kb0, kb1, a_off, full_bar, empty_bar, stage, phase, signal, order_next);
    }
    if (p.res_tma) {
      const int uses = PP ? it : p.nbuf > 1 ? (it >> 1) : it;
      mbar_wait(&res_bar[cbi], uses & 1);
    }

    // ---------------- registers -> fp32 epilogue math -> swizzled bf16 staging (or fp32 global)
    // wgmma accumulator layout: element 4 j + 2 h + e of thread (wl, lane) is row 16 wl + lane / 4 + 8 h of the
    // 64-row block, column 8 j + 2 (lane % 4) + e
    const int q = lane & 3;
    // The epilogue kinds run as separate loops.  One fully unrolled loop that tests every option for every element
    // pair spans tens of KB of code per tile; with 128 accumulators per thread it ran the 1x1 convs of layer1 at a
    // tenth of the HBM bandwidth, whichever options were set (DESIGN.md section 1).  The plain bf16 output (every conv
    // that feeds a BatchNorm), the bf16 output with a bias (the linear layers), the TMA-staged residual and the
    // unstaged fp32 output get compact loops of their own; activation, alpha != 1, a residual read from global memory
    // and fp32 outputs with a bias take the general loop.
    const bool plain = staged && !p.res_tma && p.bias == nullptr && p.residual == nullptr && p.act == 0 &&
                       p.alpha == 1.0f;
    const bool bias_only = staged && p.bias_pairs && p.residual == nullptr && p.act == 0 && p.alpha == 1.0f;
    const bool f32_only = !staged && p.bias == nullptr && p.residual == nullptr && p.act == 0;
    // output row of row r of the tile (-1: outside the output)
    auto tile_row = [&](int r) -> long long {
      if (p.mode & 1) {
        const int dw = r & ((1 << p.lbw) - 1);
        const int dh = (r >> p.lbw) & ((1 << p.lbh) - 1);
        const int dn = r >> (p.lbw + p.lbh);
        const int w = (tw << p.lbw) + dw, h = (th << p.lbh) + dh, n = (tn << p.lbn) + dn;
        return (w < p.cW && h < p.cH && n < p.cN) ? ((long long)(n * p.cH + h) * p.cW + w) : -1;
      }
      const int r_ = mt * kBM + r;
      return r_ < p.M ? (long long)r_ : -1;
    };
    if constexpr (SS) {
      // folded eval-mode BatchNorm: bf16_rn(act(fmaf(acc, scale, shift) + residual)), laid out like the bias loop:
      // one float2 of scale and one of shift and one swizzled address per column pair j serve every row the thread
      // holds; pairs at or past N (N is even) read zeros and are clipped by the TMA store.  The residual is the tile
      // the TMA staged in this buffer (rows outside the output are zero filled).
      const uint32_t srow = smem_u32(cbuf) + ((PP ? 0 : wg) * 64 + wl * 16 + (lane >> 2)) * 128 + q * 4;
      const int sw = lane >> 2;
      const int col0 = n_base + 2 * q;
      const bool res = p.res_tma != 0, relu = p.act == 1;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = col0 + 8 * j;
        const bool in = col < p.N;
        const float2 sc = in ? __ldg(reinterpret_cast<const float2*>(p.col_scale + col)) : make_float2(0.f, 0.f);
        const float2 sh = in ? __ldg(reinterpret_cast<const float2*>(p.col_shift + col)) : make_float2(0.f, 0.f);
        const uint32_t sa = srow + (j >> 3) * 16384 + (((j & 7) ^ sw) << 4);
#pragma unroll
        for (int hh = 0; hh < 2 * NH; ++hh) {
          const float* accb = acc + (hh >> 1) * (BN / 2) + 4 * j + 2 * (hh & 1);
          const uint32_t a = sa + ((hh >> 1) * 64 + 8 * (hh & 1)) * 128;
          float v0 = fmaf(accb[0], sc.x, sh.x), v1 = fmaf(accb[1], sc.y, sh.y);
          if (res) {
            const uint32_t r = lds32(a);  // bf16 pair: low half is column col, high half col + 1
            v0 += __uint_as_float(r << 16);
            v1 += __uint_as_float(r & 0xffff0000u);
          }
          if (relu) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
          sts32(a, pack_bf16x2(v0, v1));
        }
      }
    } else if (bias_only) {
      // bf16 output + bias: fp32(acc + bias) rounded once to bf16, as the general loop computes it (alpha == 1 makes
      // its multiplication exact, fused or not).  A thread's columns 8 j + 2 q are the same in every row it holds, so
      // one bias pair per j serves all of them; pairs at or past N (N is even) read zeros and are clipped by the TMA
      // store.  The swizzle (row & 7 == lane / 4) is the same for every row, which leaves one address per j.
      // (Tested before the plain / residual branch: in that order the 256-wide instantiation spills less.)
      const uint32_t srow = smem_u32(cbuf) + ((PP ? 0 : wg) * 64 + wl * 16 + (lane >> 2)) * 128 + q * 4;
      const int sw = lane >> 2;
      const int col0 = n_base + 2 * q;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = col0 + 8 * j;
        const float2 b = col < p.N ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);
        const uint32_t sa = srow + (j >> 3) * 16384 + (((j & 7) ^ sw) << 4);
#pragma unroll
        for (int hh = 0; hh < 2 * NH; ++hh) {
          const float* accb = acc + (hh >> 1) * (BN / 2) + 4 * j + 2 * (hh & 1);
          sts32(sa + ((hh >> 1) * 64 + 8 * (hh & 1)) * 128, pack_bf16x2(accb[0] + b.x, accb[1] + b.y));
        }
      }
    } else if (plain || p.res_tma) {
#pragma unroll
      for (int hh = 0; hh < 2 * NH; ++hh) {
        const int hr = hh & 1;
        const float* accb = acc + (hh >> 1) * (BN / 2);
        const int r_in_tile = (PP ? (hh >> 1) : wg) * 64 + wl * 16 + (lane >> 2) + 8 * hr;
        const uint32_t srow = smem_u32(cbuf) + r_in_tile * 128 + q * 4;
        const int sw = r_in_tile & 7;
        // (columns >= N of the staged tile are clipped by the TMA store)
        if (plain) {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j)
            sts32(srow + (j >> 3) * 16384 + (((j & 7) ^ sw) << 4), pack_bf16x2(accb[4 * j + 2 * hr], accb[4 * j + 2 * hr + 1]));
        } else if (p.res_mask == nullptr) {
          // residual tile staged by TMA, added in packed bf16 after the accumulators are rounded (host guarantees
          // alpha == 1, no bias, no activation)
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const uint32_t sa = srow + (j >> 3) * 16384 + (((j & 7) ^ sw) << 4);
            sts32(sa, add_res_bf16x2(accb[4 * j + 2 * hr], accb[4 * j + 2 * hr + 1], lds32(sa)));
          }
        } else {
          // the same with the residual's ReLU bit mask: bit (col % 32) of the 32-bit word (row * N + col) / 32 (N % 32
          // == 0, checked on the host), one load per row and 32-column chunk, zeroes residual elements
          const long long grow = tile_row(r_in_tile);
          uint32_t mword = 0u;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = n_base + 8 * j + 2 * q;
            if ((j & 3) == 0)
              mword = (grow >= 0 && col < p.N)
                          ? __ldg(reinterpret_cast<const uint32_t*>(p.res_mask) + ((grow * p.N + col) >> 5)) : 0u;
            const uint32_t sa = srow + (j >> 3) * 16384 + (((j & 7) ^ sw) << 4);
            const uint32_t r = lds32(sa) & ((((mword >> (col & 31)) & 1u) ? 0x0000ffffu : 0u) |
                                            (((mword >> ((col & 31) + 1)) & 1u) ? 0xffff0000u : 0u));
            sts32(sa, add_res_bf16x2(accb[4 * j + 2 * hr], accb[4 * j + 2 * hr + 1], r));
          }
        }
      }
    } else if (f32_only) {
      float* const D = reinterpret_cast<float*>(p.D);
#pragma unroll
      for (int hh = 0; hh < 2 * NH; ++hh) {
        const int hr = hh & 1;
        const float* accb = acc + (hh >> 1) * (BN / 2);
        const int r_in_tile = (PP ? (hh >> 1) : wg) * 64 + wl * 16 + (lane >> 2) + 8 * hr;
        const long long grow = tile_row(r_in_tile);
        if (grow < 0) continue;
        if (p.trans_d) {
          // conv_mode 4: D[col, row]
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = n_base + 8 * j + 2 * q;
            if (col >= p.N) continue;
            float* op = D + (long long)col * p.ldd + grow;
            atomicAdd(op, accb[4 * j + 2 * hr] * p.alpha);
            if (col + 1 < p.N) atomicAdd(op + p.ldd, accb[4 * j + 2 * hr + 1] * p.alpha);
          }
        } else if (p.atomic) {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = n_base + 8 * j + 2 * q;
            if (col >= p.N) continue;
            float* op = D + grow * p.ldd + col;
            const float v0 = accb[4 * j + 2 * hr] * p.alpha, v1 = accb[4 * j + 2 * hr + 1] * p.alpha;
            if (col + 1 < p.N) red_add_v2(op, v0, v1);
            else atomicAdd(op, v0);
          }
        } else {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = n_base + 8 * j + 2 * q;
            if (col >= p.N) continue;
            float* op = D + grow * p.ldd + col;
            const float v0 = accb[4 * j + 2 * hr] * p.alpha, v1 = accb[4 * j + 2 * hr + 1] * p.alpha;
            if (col + 1 < p.N) *reinterpret_cast<float2*>(op) = make_float2(v0, v1);
            else op[0] = v0;
          }
        }
      }
    } else {
#pragma unroll
      for (int hh = 0; hh < 2 * NH; ++hh) {
        const int hr = hh & 1;
        float* const accb = acc + (hh >> 1) * (BN / 2);
        const int r_in_tile = (PP ? (hh >> 1) : wg) * 64 + wl * 16 + (lane >> 2) + 8 * hr;
        long long grow = -1;
        if (!staged || p.residual != nullptr) grow = tile_row(r_in_tile);
        const uint32_t srow = smem_u32(cbuf) + r_in_tile * 128;
        const int sw = r_in_tile & 7;
        uint32_t mword = 0u;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n_base + 8 * j + 2 * q;
          if (col >= p.N) continue;
          const bool two = col + 1 < p.N;
          float v0 = accb[4 * j + 2 * hr], v1 = accb[4 * j + 2 * hr + 1];
          const uint32_t sa = srow + (j >> 3) * 16384 + ((((j & 7) ^ sw)) << 4) + q * 4;
          // ReLU bit mask of the residual: bit (col % 32) of the 32-bit word (row * N + col) / 32 (N % 32 == 0, checked on
          // the host), one load per row and 32-column chunk
          uint32_t mb0 = 1u, mb1 = 1u;
          if (p.res_mask != nullptr) {
            if ((j & 3) == 0)
              mword = grow >= 0 ? __ldg(reinterpret_cast<const uint32_t*>(p.res_mask) + ((grow * p.N + col) >> 5)) : 0u;
            mb0 = (mword >> (col & 31)) & 1u;
            mb1 = (mword >> ((col & 31) + 1)) & 1u;
          }
          v0 *= p.alpha;
          v1 *= p.alpha;
          if (p.bias != nullptr) {
            v0 += __ldg(p.bias + col);
            if (two) v1 += __ldg(p.bias + col + 1);
          }
          if (p.residual != nullptr && grow >= 0) {
            const __nv_bfloat16* rp = p.residual + grow * p.ldr + col;
            if (mb0) v0 += __bfloat162float(rp[0]);
            if (two && mb1) v1 += __bfloat162float(rp[1]);
          }
          if (p.act == 1) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          } else if (p.act == 2) {
            v0 = gelu_erf(v0);
            v1 = gelu_erf(v1);
          }
          if (staged) {
            sts32(sa, pack_bf16x2(v0, v1));  // columns >= N are clipped by the TMA store
          } else if (grow >= 0) {
            float* D = reinterpret_cast<float*>(p.D);
            if (p.trans_d) {
              // conv_mode 4: D[col, row]
              float* op = D + (long long)col * p.ldd + grow;
              atomicAdd(op, v0);
              if (two) atomicAdd(op + p.ldd, v1);
            } else {
              float* op = D + grow * p.ldd + col;
              if (p.atomic) {
                if (two) red_add_v2(op, v0, v1);
                else atomicAdd(op, v0);
              } else if (two) {
                *reinterpret_cast<float2*>(op) = make_float2(v0, v1);
              } else {
                op[0] = v0;
              }
            }
          }
        }
      }
    }

    // fused BN reduction: this thread's rows / columns of the staged tile, and the loader of one batch of four rows of
    // y (16 bytes each) and of the ReLU mask words; rows outside the output contribute nothing -- their mask word is 0
    const int bnr_r0 = srg * st_rpt;           // first row of this thread (a multiple of 4)
    const int bnr_col = n_base + scg * 8;
    const bool bnr_on = p.bnr && st_on && bnr_col < p.N;
    // (element offsets fit 32 bits: the host checks M * ldy < 2^31; the four mask bytes of a batch share one register)
    auto bnr_load = [&](int rb, uint4* yv, uint32_t& mbits) {
      mbits = 0u;
#pragma unroll
      for (int r4 = 0; r4 < 4; ++r4) {
        const int r = bnr_r0 + rb + r4;  // row of the tile
        uint32_t off, lin = 0;
        bool ok;
        if (p.mode & 1) {
          const int dw = r & ((1 << p.lbw) - 1);
          const int dh = (r >> p.lbw) & ((1 << p.lbh) - 1);
          const int dn = r >> (p.lbw + p.lbh);
          const int w = (tw << p.lbw) + dw, h = (th << p.lbh) + dh, n = (tn << p.lbn) + dn;
          ok = (w < p.vW) && (h < p.vH) && (n < p.cN);
          off = (uint32_t)n * (uint32_t)p.bnr_sn + (uint32_t)h * (uint32_t)p.bnr_sh + (uint32_t)w * (uint32_t)p.bnr_sw;
          // the bit mask's row: the NHWC output pixel (the host allows the mask only without an output view)
          lin = ((uint32_t)n * (uint32_t)p.cH + (uint32_t)h) * (uint32_t)p.cW + (uint32_t)w;
        } else {
          lin = (uint32_t)(mt * kBM + r);
          ok = lin < (uint32_t)p.M;
          off = lin * (uint32_t)p.bnr_ldy;
        }
        yv[r4] = ok ? ldg128_nc(p.bnr_y + off + bnr_col) : make_uint4(0u, 0u, 0u, 0u);
        const uint32_t mw = ok ? (p.bnr == 2 ? (uint32_t)__ldg(p.bnr_mask + ((lin * (uint32_t)p.N + bnr_col) >> 3)) : 0xffu) : 0u;
        mbits |= mw << (8 * r4);
      }
    };

    if (staged) {
      fence_proxy_async();  // make this thread's staging writes visible to the TMA (async proxy)
      epi_bar(bar_id, epi_threads);
      // ---------------- TMA store of the staged tile: one 64-column slab per instruction
      if (et == 0) {
        const int slabs = (min(p.bn, p.N - n_base) + 63) >> 6;
        for (int sl = 0; sl < slabs; ++sl) {
          if (p.mode & 1)
            tma_store_4d(&tmD, cbuf + sl * 16384, n_base + sl * 64, tw << p.lbw, th << p.lbh, tn << p.lbn);
          else
            tma_store_2d(&tmD, cbuf + sl * 16384, n_base + sl * 64, mt * kBM);
        }
        tma_store_commit();
      }
      // ---------------- BN statistics of the staged (bf16-rounded) tile, accumulated in registers.
      // Rows outside the problem are exact zeros (TMA zero fill; stats forbids bias/residual): no masking needed.
      if (bnr_on) {
        const uint32_t cp = smem_u32(cbuf) + (scg >> 3) * 16384 + bnr_r0 * 128;
        const int c8 = scg & 7;
        // (y - mean per element, like the stand-alone pass: taking the mean out of the loop -- sum dz * y - mean * sum dz
        // -- cancels catastrophically when |mean| >> std, which post-ReLU inputs with a common mode do produce)
        float mean[8], sc[8], sh[8];
        {
          const float4 m0 = __ldg(reinterpret_cast<const float4*>(p.bnr_bnp + bnr_col));
          const float4 m1 = __ldg(reinterpret_cast<const float4*>(p.bnr_bnp + bnr_col + 4));
          mean[0] = m0.x; mean[1] = m0.y; mean[2] = m0.z; mean[3] = m0.w;
          mean[4] = m1.x; mean[5] = m1.y; mean[6] = m1.z; mean[7] = m1.w;
          const float4 a0 = __ldg(reinterpret_cast<const float4*>(p.bnr_bnp + 2 * p.N + bnr_col));
          const float4 a1 = __ldg(reinterpret_cast<const float4*>(p.bnr_bnp + 2 * p.N + bnr_col + 4));
          const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bnr_bnp + 3 * p.N + bnr_col));
          const float4 b1 = __ldg(reinterpret_cast<const float4*>(p.bnr_bnp + 3 * p.N + bnr_col + 4));
          sc[0] = a0.x; sc[1] = a0.y; sc[2] = a0.z; sc[3] = a0.w; sc[4] = a1.x; sc[5] = a1.y; sc[6] = a1.z; sc[7] = a1.w;
          sh[0] = b0.x; sh[1] = b0.y; sh[2] = b0.z; sh[3] = b0.w; sh[4] = b1.x; sh[5] = b1.y; sh[6] = b1.z; sh[7] = b1.w;
        }
        for (int rb = 0; rb < st_rpt; rb += 4) {
          uint4 yv[4];
          uint32_t mbits;
          bnr_load(rb, yv, mbits);
#pragma unroll
          for (int r4 = 0; r4 < 4; ++r4) {
            const int r = rb + r4;
            const uint4 raw = lds128(cp + r * 128 + ((c8 ^ ((bnr_r0 + r) & 7)) << 4));
            float f[8], yy[8];
            unpack8(*reinterpret_cast<const bf16x8*>(&raw), f);
            unpack8(*reinterpret_cast<const bf16x8*>(&yv[r4]), yy);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const bool on = p.bnr == 1 ? ((yy[i] * sc[i] + sh[i] > 0.f) && ((mbits >> (8 * r4)) & 0xffu) != 0u)
                                         : (((mbits >> (8 * r4 + i)) & 1u) != 0u);
              const float dz = on ? f[i] : 0.f;
              st_s[i] += dz;
              st_q[i] += dz * (yy[i] - mean[i]);
            }
          }
        }
      }
      if (!p.bnr && p.stats != nullptr && st_on) {
        const int r0 = srg * st_rpt;  // first row of this thread (a multiple of 4)
        const uint32_t cp = smem_u32(cbuf) + (scg >> 3) * 16384 + r0 * 128;
        const int c8 = scg & 7;
        for (int rb = 0; rb < st_rpt; rb += 4) {
#pragma unroll
          for (int r4 = 0; r4 < 4; ++r4) {
            const int r = rb + r4;
            const uint4 raw = lds128(cp + r * 128 + ((c8 ^ ((r0 + r) & 7)) << 4));
            float f[8];
            unpack8(*reinterpret_cast<const bf16x8*>(&raw), f);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              st_s[i] += f[i];
              st_q[i] += f[i] * f[i];
            }
          }
        }
      }
    }
  }
  if (staged) {
    if (et == 0) tma_store_wait_read<0>();
    epi_bar(bar_id, epi_threads);
    if (p.stats != nullptr && st_nt >= 0) flush_stats(cstage0 + (PP ? (size_t)wg * p.cbytes : 0));
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// bf16 tensor map of rank 2 or 4; dims[0] is the contiguous dimension; strides in elements for dims 1..rank-1.
// estr (optional): TMA traversal strides per dimension (1..8): the box then covers box[i] elements of the tensor and
// delivers every estr[i]-th of them, i.e. ceil(box[i] / estr[i]) elements land in shared memory (strided convolutions).
static int make_tmap(CUtensorMap* tm, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                     const uint32_t* box, const uint32_t* estr = nullptr) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(VTX_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = estr ? estr[i] : 1;
  }
  for (int i = 0; i < rank - 1; ++i) gstr[i] = strides_elems[i] * 2;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) return set_error(VTX_EINVAL, "TMA base pointer not 16B aligned");
  for (int i = 0; i < rank - 1; ++i)
    if (gstr[i] % 16 != 0) return set_error(VTX_EINVAL, "TMA stride not a multiple of 16 bytes");
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(VTX_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return VTX_OK;
}

// Tile counters of the dynamic scheduler.  Launch i of a device uses counter i mod kSchedSlots (adjacent launches overlap
// under programmatic dependent launch, launches thousands apart do not) and the host keeps the value every counter will
// have reached when its users so far are done: a launch performs exactly `fetches` atomic increments (one per chunk of
// tiles + one end marker per CTA), so its window starts at the running total.  Counters wrap modulo 2^32 with the
// window arithmetic.  (A captured CUDA graph would replay stale windows: capture with the static schedule.)
constexpr int kSchedSlots = 4096;
static int g_sched_dynamic = 0;  // 0: static round-robin schedule (default), 1: dynamic
static struct SchedRing {
  unsigned int* ctr;
  unsigned int base[kSchedSlots];
  unsigned int next;
} g_sched[64];
static bool sched_is_dynamic() {
  static const char* env = getenv("VTX_GEMM_SCHEDULE");  // measurement knob: "static" / "dynamic" overrides the setter
  return env != nullptr ? (env[0] == 'd') : (g_sched_dynamic != 0);
}
static unsigned int* sched_slot(unsigned int fetches, unsigned int* base_out) {
  if (!sched_is_dynamic()) return nullptr;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return nullptr;
  SchedRing& r = g_sched[dev];
  if (r.ctr == nullptr) {
    unsigned int* ptr = nullptr;
    if (cudaMalloc(&ptr, sizeof(unsigned int) * kSchedSlots) != cudaSuccess) return nullptr;
    cudaMemset(ptr, 0, sizeof(unsigned int) * kSchedSlots);
    cudaDeviceSynchronize();
    memset(r.base, 0, sizeof(r.base));
    r.next = 0;
    r.ctr = ptr;
  }
  const unsigned int slot = r.next++ % kSchedSlots;
  *base_out = r.base[slot];
  r.base[slot] += fetches;
  return r.ctr + slot;
}

static int ilog2(int x) {
  int l = 0;
  while ((1 << l) < x) ++l;
  return l;
}

// choose a power-of-two (w,h,n) box with w*h*n == positions that tiles an H x W image with the least waste
static void choose_box(int H, int W, int positions, int* bw, int* bh, int* bn) {
  int best_w = 1, best_h = 1;
  double best_eff = -1;
  for (int w = 1; w <= positions; w <<= 1)
    for (int h = 1; w * h <= positions; h <<= 1) {
      if (w > 2 * W || h > 2 * H) continue;
      const int tw = (W + w - 1) / w, th = (H + h - 1) / h;
      const double eff = (double)(W * H) / ((double)tw * w * th * h);
      // prefer higher efficiency, then larger contiguous w, then larger h
      const double score = eff * 1000.0 + w * 0.01 + h * 0.0001;
      if (score > best_eff) { best_eff = score; best_w = w; best_h = h; }
    }
  *bw = best_w; *bh = best_h; *bn = positions / (best_w * best_h);
}

// the instantiation of a launch: tile width, schedule and epilogue variant
template <bool SS>
static cudaError_t launch_gemm(const cudaLaunchConfig_t& cfg, bool pingpong, int bn, const CUtensorMap& tmA,
                               const CUtensorMap& tmB, const CUtensorMap& tmD, const CUtensorMap& tmR,
                               const CUtensorMap& tmY, const GemmKParams& p) {
  if (pingpong && bn == 64) return cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<64, true, SS>, tmA, tmB, tmD, tmR, tmY, p);
  if (pingpong) return cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<128, true, SS>, tmA, tmB, tmD, tmR, tmY, p);
  if (bn == 64) return cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<64, false, SS>, tmA, tmB, tmD, tmR, tmY, p);
  if (bn == 128) return cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<128, false, SS>, tmA, tmB, tmD, tmR, tmY, p);
  if (bn == 192) return cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<192, false, SS>, tmA, tmB, tmD, tmR, tmY, p);
  return cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<256, false, SS>, tmA, tmB, tmD, tmR, tmY, p);
}

// the streaming kernel of the masked-residual 1x1 dgrads (gemm_resid.cu)
bool resid_dgrad_serves(const VtxGemm* g);
int resid_dgrad(const VtxGemm* g, cudaStream_t stream);

}  // namespace vtx

using namespace vtx;

extern "C" int vtx_gemm_set_dynamic_schedule(int on) {
  g_sched_dynamic = on ? 1 : 0;
  return VTX_OK;
}

extern "C" int vtx_gemm(const VtxGemm* g, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!g || !g->A || !g->B || !g->D) return set_error(VTX_EINVAL, "vtx_gemm: null pointer");
  if (g->M <= 0 || g->N <= 0 || g->K <= 0) return set_error(VTX_EINVAL, "vtx_gemm: empty problem");
  if (g->atomic && !g->out_f32) return set_error(VTX_EINVAL, "vtx_gemm: atomic accumulate needs fp32 output");
  if (g->split_k > 1 && !g->atomic) return set_error(VTX_EINVAL, "vtx_gemm: split_k > 1 needs atomic = 1");
  if (g->stats && (g->out_f32 || g->bias || g->residual || g->act || (g->alpha != 0.f && g->alpha != 1.f)))
    return set_error(VTX_EINVAL, "vtx_gemm: stats needs a plain bf16 output (no bias/residual/activation/alpha)");
  if (g->ldd % (g->out_f32 ? 4 : 8) != 0) return set_error(VTX_EINVAL, "vtx_gemm: ldd must keep rows 16B aligned");
  // conv_mode 4 (D[(tap, cin), cout] of a 64 -> 64 3x3 conv) is the transpose of conv_mode 2's D[cout, (tap, cin)]: it
  // runs as conv_mode 2 with a transposed store, split over the positions so that the three output tiles fill the GPU
  if (g->conv_mode < 0 || g->conv_mode > 6 || g->conv_mode == 3)
    return set_error(VTX_EINVAL, "vtx_gemm: conv_mode must be 0, 1, 2, 4, 5 or 6");
  VtxGemm g4;
  const bool trans_d = g->conv_mode == 4;
  if (trans_d) {
    if (g->conv_c != 64 || g->N != 64 || g->M != 9 * 64 || !g->out_f32 || !g->atomic)
      return set_error(VTX_EINVAL, "vtx_gemm: conv_mode 4 needs C = Cout = 64, M = 576, fp32 atomic output");
    g4 = *g;
    g4.conv_mode = 2;
    g4.M = g->N;
    g4.N = g->M;
    g4.split_k = vtx_num_sms() / 3;
    g4.conv_stride = 1;
    g4.conv_taps = 0;
    g = &g4;
  }
  const int split_k = g->split_k > 1 ? g->split_k : 1;

  GemmKParams p;
  memset(&p, 0, sizeof(p));
  p.M = g->M; p.N = g->N; p.K = g->K;
  p.a_mn = g->a_mn; p.b_mn = g->b_mn;
  p.mode = g->conv_mode;
  // conv_mode 5 / 6: stem conv over the space-to-depth view = modes 1 / 2 with 4 x 1 taps, no padding
  const bool stem = g->conv_mode == 5 || g->conv_mode == 6;
  p.taps_w = 3; p.pad = 1; p.ntaps = 9;
  if (stem) { p.mode = g->conv_mode == 5 ? 1 : 2; p.taps_w = 1; p.pad = 0; p.ntaps = 4; }
  // conv_taps = 1: a 1x1 convolution through the gather path (only useful with conv_stride = 2: the strided downsample)
  const bool one_tap = !stem && g->conv_taps == 1;
  if (one_tap) { p.taps_w = 1; p.pad = 0; p.ntaps = 1; }
  // explicit tap grid (conv_mode 1): conv_taps_h x conv_taps_w taps, tap (a, b) reads position (h + a - pad, w + b - pad).
  // Used by the four parity classes of a stride-2 dgrad (1x1, 1x2, 2x1, 2x2 taps, pad 0).
  const bool tap_grid = !stem && !one_tap && g->conv_taps_h > 0;
  if (tap_grid) {
    if (p.mode != 1 || g->conv_taps_w <= 0 || g->conv_taps_h > 3 || g->conv_taps_w > 3 || g->conv_pad < 0 || g->conv_pad > 1)
      return set_error(VTX_EINVAL, "vtx_gemm: bad explicit tap grid");
    p.taps_w = g->conv_taps_w; p.pad = g->conv_pad; p.ntaps = g->conv_taps_h * g->conv_taps_w;
  }
  const int cstride = (g->conv_stride == 2 && (p.mode == 1 || p.mode == 2) && !stem) ? 2 : 1;
  if (g->conv_stride != 0 && g->conv_stride != 1 && cstride != 2)
    return set_error(VTX_EINVAL, "vtx_gemm: conv_stride 2 is supported for conv_mode 1 / 2 only");
  if (g->conv_taps != 0 && g->conv_taps != 1 && g->conv_taps != 9) return set_error(VTX_EINVAL, "vtx_gemm: conv_taps must be 0, 1 or 9");
  p.cstride = cstride;
  const int ntaps = stem ? 4 : one_tap ? 1 : tap_grid ? p.ntaps : 9;
  if (p.mode == 1) { p.a_mn = 0; p.b_mn = 0; }
  if (p.mode == 2) { p.a_mn = 1; p.b_mn = 1; }
  // ---- tile_n
  int bn = g->tile_n;
  if (bn == 0) {
    const int gran = p.b_mn ? 64 : 16;
    if (g->N >= 256) bn = 256;
    else bn = ((g->N + gran - 1) / gran) * gran;
    // Width heuristics:
    //  * N = 1152 weight gradients (3x3, 128 channels) run 256-wide tiles even though the fifth tile is half empty:
    //    every N-tile re-reads the dy operand;
    //  * problems with few tiles pick the width that minimises  rounds x (width + per-tile overhead) over the SMs;
    //  * tiny problems (under ~100 tiles of 256) use 128-wide tiles to fill the machine.
    if (bn == 256 && split_k == 1) {
      const long mt = (g->M + kBM - 1) / kBM;
      const long t256 = mt * ((g->N + 255) / 256);
      const int sms = vtx_num_sms();
      if (t256 < 100 || (t256 < sms && g->N % 256 != 0 && g->N <= 2048)) {
        bn = 128;
      } else if (t256 < 3L * sms && p.mode <= 1) {
        long best_cost = 0;
        int best_bn = 256;
        for (int cand = 256; cand >= 128; cand -= 64) {
          const long tiles = mt * ((g->N + cand - 1) / cand);
          const long cost = ((tiles + sms - 1) / sms) * (cand + 64);
          if (best_cost == 0 || cost < best_cost) { best_cost = cost; best_bn = cand; }
        }
        bn = best_bn;
      }
    }
  }
  if (bn < 16 || bn > 256 || bn % 16 != 0 || (p.b_mn && bn % 64 != 0))
    return set_error(VTX_EINVAL, "vtx_gemm: bad tile_n %d", bn);
  // the kernel is instantiated for four wgmma widths; a narrower request runs the next one up (the extra B rows are
  // zero-filled by the TMA unit, the extra output columns clipped by the store)
  bn = bn <= 64 ? 64 : bn <= 128 ? 128 : bn <= 192 ? 192 : 256;
  // Ping-pong where it keeps the tile geometry: bf16 outputs whose tiles are at most 128 wide (N <= 128, or the width
  // heuristics above chose 128).  Wider tiles would have to be split into 128-wide ones there, and the extra tiles and
  // operand re-reads cost more than the overlap gains; fp32 / split-K outputs ran faster in lockstep as well (per-class
  // A/B in DESIGN.md section 1).
  const bool pingpong = bn <= 128 && !g->out_f32;
  p.bn = bn;
  p.n_tiles = (g->N + bn - 1) / bn;
  p.trans_d = trans_d ? 1 : 0;
  p.out_f32 = g->out_f32; p.atomic = g->atomic; p.act = g->act;
  p.alpha = g->alpha == 0.f ? 1.0f : g->alpha;
  p.D = g->D; p.ldd = g->ldd;
  p.bias = g->bias;
  p.bias_pairs = (g->bias != nullptr && g->N % 2 == 0 && (reinterpret_cast<uintptr_t>(g->bias) & 7) == 0) ? 1 : 0;
  p.residual = reinterpret_cast<const __nv_bfloat16*>(g->residual);
  p.ldr = g->ldr;
  // the bit masks (residual_mask, bnr_mask) address row m of D: a plain GEMM's row, or a conv_mode 1 output's NHWC pixel
  const bool mask_rows = g->conv_mode == 0 || (g->conv_mode == 1 && g->conv_out_w <= 0);
  p.res_mask = reinterpret_cast<const uint8_t*>(g->residual_mask);
  if (p.res_mask != nullptr && (g->residual == nullptr || g->N % 32 != 0 || !mask_rows || g->out_f32 ||
                                (reinterpret_cast<uintptr_t>(g->residual_mask) & 3) != 0))
    return set_error(VTX_EINVAL, "vtx_gemm: residual_mask needs a residual, a bf16 output of a plain GEMM or of conv_mode "
                                 "1 without an output view, and N %% 32 == 0");
  p.stats = g->stats;
  const bool bnr = g->bnr_y != nullptr;
  if (bnr) {
    if (!g->bnr_bnp || !g->bnr_sums || g->stats || g->out_f32 || g->bias || g->act || (g->alpha != 0.f && g->alpha != 1.f) ||
        g->N % 8 != 0 || g->bnr_ldy % 8 != 0 || (reinterpret_cast<uintptr_t>(g->bnr_y) & 15) != 0 ||
        (reinterpret_cast<uintptr_t>(g->bnr_bnp) & 15) != 0 || (g->bnr_mask != nullptr && !mask_rows) ||
        g->conv_mode == 2 || g->conv_mode >= 4 || split_k > 1)
      return set_error(VTX_EINVAL, "vtx_gemm: bnr needs a plain bf16 output (no stats/bias/activation/alpha/split-K), "
                                   "N %% 8 == 0, 16-byte aligned y / bnp; the bit-mask form needs conv_mode 0, or 1 without an output view");
    if ((long long)g->M * (g->bnr_ldy > g->N ? g->bnr_ldy : g->N) >= (1ll << 31))
      return set_error(VTX_EUNSUPPORTED, "vtx_gemm: bnr needs M * ld(y) < 2^31");
    p.stats = g->bnr_sums;
    p.bnr_y = reinterpret_cast<const __nv_bfloat16*>(g->bnr_y);
    p.bnr_bnp = g->bnr_bnp;
    p.bnr_mask = g->bnr_mask;
    p.bnr_ldy = g->bnr_ldy;
    const char* pf = getenv("VTX_BNR_PREFETCH");  // measurement knob, read per call
    p.bnr_prefetch = (pf != nullptr && pf[0] == '0') ? 0 : 1;
    p.bnr = g->bnr_mask == nullptr ? 1 : 2;
  }
  // The identity bottlenecks' masked-residual 1x1 dgrads (K <= 128) are memory-bound: they stream through a kernel of
  // their own, which computes the same D.  An explicit tile width keeps them on this kernel (the reference route).
  if (g->tile_n == 0 && resid_dgrad_serves(g)) return resid_dgrad(g, stream);
  // folded eval-mode BatchNorm: the scale / shift variant, whose only epilogue is act(acc * scale + shift + residual)
  const bool ss = g->col_scale != nullptr || g->col_shift != nullptr;
  if (ss) {
    if (!g->col_scale || !g->col_shift || g->out_f32 || (g->alpha != 0.f && g->alpha != 1.f) || g->bias || g->stats ||
        bnr || g->act < 0 || g->act > 1 || g->N % 2 != 0 || (reinterpret_cast<uintptr_t>(g->col_scale) & 7) != 0 ||
        (reinterpret_cast<uintptr_t>(g->col_shift) & 7) != 0 || g->residual_mask || g->conv_out_w > 0 ||
        (g->conv_mode != 0 && g->conv_mode != 1) ||
        (g->residual && (g->ldr % 8 != 0 || (reinterpret_cast<uintptr_t>(g->residual) & 15) != 0)))
      return set_error(VTX_EINVAL, "vtx_gemm: col_scale / col_shift need both vectors 8-byte aligned, a bf16 output, "
                                   "alpha 1, act 0 or 1, N %% 2 == 0, conv_mode 0 or 1 without an output view, no bias / "
                                   "stats / bnr / residual mask, and a 16-byte aligned residual with ldr %% 8 == 0");
    p.col_scale = g->col_scale;
    p.col_shift = g->col_shift;
  }

  CUtensorMap tmA, tmB;
  int rc;
  if (p.mode == 0) {
    p.m_tiles = (g->M + kBM - 1) / kBM;
    p.kb_total = (g->K + kBK - 1) / kBK;
    {
      uint64_t dims[2], str[1];
      uint32_t box[2];
      if (!p.a_mn) { dims[0] = g->K; dims[1] = g->M; box[0] = 64; box[1] = 128; }
      else { dims[0] = g->M; dims[1] = g->K; box[0] = 64; box[1] = 64; }
      str[0] = g->lda;
      if ((rc = make_tmap(&tmA, g->A, 2, dims, str, box)) != VTX_OK) return rc;
    }
    {
      uint64_t dims[2], str[1];
      uint32_t box[2];
      if (!p.b_mn) { dims[0] = g->K; dims[1] = g->N; box[0] = 64; box[1] = (uint32_t)bn; }
      else { dims[0] = g->N; dims[1] = g->K; box[0] = 64; box[1] = 64; }
      str[0] = g->ldb;
      if ((rc = make_tmap(&tmB, g->B, 2, dims, str, box)) != VTX_OK) return rc;
    }
  } else {
    // conv_h / conv_w are the INPUT extent of the activation operand; with stride 2 the tile schedule, the output tensor
    // map and the row masks run over the OUTPUT extent (H - 1) / 2 + 1 (3x3 / pad 1 and 1x1 / pad 0 alike)
    const int C = g->conv_c, Hin = g->conv_h, Win = g->conv_w, NI = g->conv_n;
    const int H = (Hin - 1) / cstride + 1, W = (Win - 1) / cstride + 1;
    if (C <= 0 || C % 64 != 0) return set_error(VTX_EINVAL, "vtx_gemm: implicit conv needs channels %% 64 == 0");
    p.cH = H; p.cW = W; p.cN = NI; p.cpb = C / 64;
    // the activation operand of the implicit convs: [NI, H, W, C] NHWC; for the stem view [NI, H + 3, W + 3, 16] whose
    // "channel" extent is 4 pixels x 16 channels and whose W stride is ONE pixel (overlapping rows, legal for TMA)
    const uint64_t xdims[4] = {(uint64_t)C, (uint64_t)Win, (uint64_t)(stem ? Hin + 3 : Hin), (uint64_t)NI};
    const uint64_t xstr[3] = {(uint64_t)(stem ? 16 : C), stem ? (uint64_t)(Win + 3) * 16 : (uint64_t)Win * C,
                              stem ? (uint64_t)(Hin + 3) * (Win + 3) * 16 : (uint64_t)Hin * Win * C};
    int bw, bh, bnn;
    choose_box(H, W, p.mode == 1 ? 128 : 64, &bw, &bh, &bnn);
    p.lbw = ilog2(bw); p.lbh = ilog2(bh); p.lbn = ilog2(bnn);
    p.tiles_w = (W + bw - 1) / bw;
    p.tiles_h = (H + bh - 1) / bh;
    const int tiles_n = (NI + bnn - 1) / bnn;
    if (p.mode == 1) {
      // A: activation [NI,H,W,C]; M = NI*H*W (tiled as boxes); K = 9*C; B: weights [N, 9*C] K-major
      if (g->M != NI * H * W || g->K != ntaps * C) return set_error(VTX_EINVAL, "vtx_gemm: conv fprop shape mismatch");
      // rows of a partial box below the image are real rows of the padded view: they would reach the BN statistics
      if (stem && g->stats && (W % bw != 0 || H % bh != 0))
        return set_error(VTX_EUNSUPPORTED, "vtx_gemm: conv_mode 5 with stats needs an output size tiled exactly by %dx%d", bw, bh);
      p.m_tiles = p.tiles_w * p.tiles_h * tiles_n;
      p.kb_total = ntaps * p.cpb;
      uint32_t box[4] = {64, (uint32_t)(bw * cstride), (uint32_t)(bh * cstride), (uint32_t)bnn};
      const uint32_t es[4] = {1, (uint32_t)cstride, (uint32_t)cstride, 1};
      if ((rc = make_tmap(&tmA, g->A, 4, xdims, xstr, box, cstride > 1 ? es : nullptr)) != VTX_OK) return rc;
      uint64_t bd[2] = {(uint64_t)g->K, (uint64_t)g->N};
      uint64_t bs[1] = {(uint64_t)g->ldb};
      uint32_t bb[2] = {64, (uint32_t)bn};
      if ((rc = make_tmap(&tmB, g->B, 2, bd, bs, bb)) != VTX_OK) return rc;
    } else {
      // wgrad: D[M = Cout, N = 9*C] += sum over positions dy[pos, Cout] * x_shift[pos, C]
      //   A = dy [NI,H,W,Cout] (lda = Cout), B = x [NI,H,W,C]
      if (g->N != ntaps * C) return set_error(VTX_EINVAL, "vtx_gemm: conv wgrad shape mismatch");
      const int Cout = g->M;
      if (Cout % 64 != 0) return set_error(VTX_EINVAL, "vtx_gemm: conv wgrad needs Cout %% 64 == 0");
      p.m_tiles = (Cout + kBM - 1) / kBM;
      p.kb_total = p.tiles_w * p.tiles_h * tiles_n;
      uint64_t ad[4] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)NI};
      uint64_t as[3] = {(uint64_t)Cout, (uint64_t)W * Cout, (uint64_t)H * W * Cout};
      uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bnn};
      if ((rc = make_tmap(&tmA, g->A, 4, ad, as, box)) != VTX_OK) return rc;
      uint32_t xbox[4] = {64, (uint32_t)(bw * cstride), (uint32_t)(bh * cstride), (uint32_t)bnn};
      const uint32_t es[4] = {1, (uint32_t)cstride, (uint32_t)cstride, 1};
      if ((rc = make_tmap(&tmB, g->B, 4, xdims, xstr, xbox, cstride > 1 ? es : nullptr)) != VTX_OK) return rc;
    }
  }
  p.k_splits = split_k;
  if (p.k_splits > p.kb_total) p.k_splits = p.kb_total;
  p.kb_per_split = (p.kb_total + p.k_splits - 1) / p.k_splits;
  p.k_splits = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;

  // ---- shared-memory carve-up: [1 KB control][stages x (A 16 KB + B bn*128 B)][nbuf x bf16 staging tile 128 x bn]
  p.stage_bytes = kABytes + bn * kBK * 2;
  p.cbytes = p.out_f32 ? 0 : ((bn + 63) / 64) * 16384;
  {
    // two staging buffers (the TMA store of tile i overlaps the epilogue of tile i+1) whenever the operand ring still
    // gets >= 4 stages, or holds a whole tile's K loop
    const int kb_tile = p.kb_per_split;
    const int budget = kSmemTotal - 1024 /*alignment slack*/ - kCtrlBytes;
    int st = 0;
    p.nbuf = 1;
    if (pingpong) {
      p.nbuf = 2;  // one staging buffer per consumer warpgroup
    } else if (p.cbytes) {
      const int st2 = (budget - 2 * p.cbytes) / p.stage_bytes;
      if (st2 >= 4 || (st2 >= 2 && st2 >= kb_tile)) { p.nbuf = 2; st = st2; }
    }
    if (st == 0) st = (budget - p.nbuf * p.cbytes) / p.stage_bytes;
    if (st > kMaxStages) st = kMaxStages;
    if (st < 2) return set_error(VTX_EUNSUPPORTED, "vtx_gemm: not enough shared memory for a 2-stage pipeline");
    p.stages = st;
  }
  CUtensorMap tmD, tmR, tmY;
  memset(&tmY, 0, sizeof(tmY));
  memset(&tmD, 0, sizeof(tmD));
  memset(&tmR, 0, sizeof(tmR));
  // the TMA-staged residual is added in packed bf16 AFTER the accumulator is rounded, which is only the documented
  // order (alpha * acc + bias + residual, then the activation) when there is nothing else in the epilogue; the scale /
  // shift variant adds it in fp32 before its ReLU
  p.res_tma = (p.cbytes && g->residual != nullptr && g->ldr % 8 == 0 &&
               (reinterpret_cast<uintptr_t>(g->residual) & 15) == 0 && p.alpha == 1.0f && g->bias == nullptr &&
               (g->act == 0 || ss)) ? 1 : 0;
  if (p.cbytes) {
    if (p.mode & 1) {
      uint64_t dd[4] = {(uint64_t)g->N, (uint64_t)p.cW, (uint64_t)p.cH, (uint64_t)g->conv_n};
      uint64_t ds[3] = {(uint64_t)g->ldd, (uint64_t)p.cW * g->ldd, (uint64_t)p.cH * p.cW * g->ldd};
      if (g->conv_out_w > 0) {
        // output VIEW override: D is a strided sub-grid [conv_n, conv_out_h, conv_out_w, N] of a larger NHWC tensor
        // (element strides ldd_n / ldd_h / ldd_w); tiles still run over the conv_h x conv_w grid of the A operand and
        // rows beyond the view are clipped by the TMA store.  (stride-2 dgrad: one parity class of the input gradient)
        if (g->conv_out_h <= 0 || g->ldd_w % 8 || g->ldd_h % 8 || g->ldd_n % 8 || (g->residual != nullptr && !p.res_tma))
          return set_error(VTX_EINVAL, "vtx_gemm: bad output view");
        dd[1] = (uint64_t)g->conv_out_w; dd[2] = (uint64_t)g->conv_out_h;
        ds[0] = (uint64_t)g->ldd_w; ds[1] = (uint64_t)g->ldd_h; ds[2] = (uint64_t)g->ldd_n;
      }
      uint32_t db[4] = {64, 1u << p.lbw, 1u << p.lbh, 1u << p.lbn};
      if ((rc = make_tmap(&tmD, g->D, 4, dd, ds, db)) != VTX_OK) return rc;
      p.vW = (int)dd[1]; p.vH = (int)dd[2];
      if (bnr) {
        // y has D's geometry: the same strides for a view (y of the strided sub-grid), its own row stride otherwise
        uint64_t ys[3] = {(uint64_t)g->bnr_ldy, (uint64_t)p.cW * g->bnr_ldy, (uint64_t)p.cH * p.cW * g->bnr_ldy};
        if (g->conv_out_w > 0) { ys[0] = ds[0]; ys[1] = ds[1]; ys[2] = ds[2]; }
        p.bnr_sw = (long long)ys[0]; p.bnr_sh = (long long)ys[1]; p.bnr_sn = (long long)ys[2];
        if ((rc = make_tmap(&tmY, g->bnr_y, 4, dd, ys, db)) != VTX_OK) return rc;
      }
      if (p.res_tma) {
        // a residual of a view GEMM is a view with the SAME strides (in-place accumulation into the strided sub-grid)
        uint64_t rs[3] = {(uint64_t)g->ldr, (uint64_t)p.cW * g->ldr, (uint64_t)p.cH * p.cW * g->ldr};
        if (g->conv_out_w > 0) { rs[0] = ds[0]; rs[1] = ds[1]; rs[2] = ds[2]; }
        if ((rc = make_tmap(&tmR, g->residual, 4, dd, rs, db)) != VTX_OK) return rc;
      }
    } else {
      uint64_t dd[2] = {(uint64_t)g->N, (uint64_t)g->M};
      uint64_t ds[1] = {(uint64_t)g->ldd};
      uint32_t db[2] = {64, 128};
      if ((rc = make_tmap(&tmD, g->D, 2, dd, ds, db)) != VTX_OK) return rc;
      if (bnr) {
        uint64_t ys[1] = {(uint64_t)g->bnr_ldy};
        if ((rc = make_tmap(&tmY, g->bnr_y, 2, dd, ys, db)) != VTX_OK) return rc;
      }
      if (p.res_tma) {
        uint64_t rs[1] = {(uint64_t)g->ldr};
        if ((rc = make_tmap(&tmR, g->residual, 2, dd, rs, db)) != VTX_OK) return rc;
      }
    }
  }
  {
    // the attribute is per device: remember which devices of this process already have it
    static bool attr_set[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !attr_set[dev]) {
      cudaError_t e = cudaSuccess;
      const void* kernels[12] = {
          (const void*)gemm_wgmma_kernel<64, false, false>,  (const void*)gemm_wgmma_kernel<128, false, false>,
          (const void*)gemm_wgmma_kernel<192, false, false>, (const void*)gemm_wgmma_kernel<256, false, false>,
          (const void*)gemm_wgmma_kernel<64, true, false>,   (const void*)gemm_wgmma_kernel<128, true, false>,
          (const void*)gemm_wgmma_kernel<64, false, true>,   (const void*)gemm_wgmma_kernel<128, false, true>,
          (const void*)gemm_wgmma_kernel<192, false, true>,  (const void*)gemm_wgmma_kernel<256, false, true>,
          (const void*)gemm_wgmma_kernel<64, true, true>,    (const void*)gemm_wgmma_kernel<128, true, true>};
      for (int i = 0; i < 12 && e == cudaSuccess; ++i)
        e = cudaFuncSetAttribute(kernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal);
      if (e != cudaSuccess) return set_error(VTX_ECUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      if (dev >= 0 && dev < 64) attr_set[dev] = true;
    }
  }
  p.d_mn = make_fastdiv(p.m_tiles * p.n_tiles);
  p.d_nt = make_fastdiv(p.n_tiles);
  p.d_mt = make_fastdiv(p.m_tiles);
  // BN statistics are kept in registers per column block: run over the row tiles first, so that a CTA's column block
  // changes at most n_tiles - 1 times whatever order the tiles are handed out in
  p.nt_major = (p.stats != nullptr && p.n_tiles > 1) ? 1 : 0;
  const long total = (long)p.m_tiles * p.n_tiles * p.k_splits;
  const int sms = vtx_num_sms();
  const int grid = (int)(total < sms ? total : sms);
  // many short tiles per CTA (64-wide layer1 / stem convs): one fetch hands out a few consecutive tiles
  p.sched_chunk = total >= 32L * grid ? 4 : total >= 12L * grid ? 2 : 1;
  const unsigned int fetches = (unsigned int)((total + p.sched_chunk - 1) / p.sched_chunk) + (unsigned int)grid;
  p.sched = sched_slot(fetches, &p.sched_base);
  p.d_tw = make_fastdiv(p.tiles_w);
  p.d_twh = make_fastdiv(p.tiles_w * p.tiles_h);
  p.d_cpb = make_fastdiv(p.cpb);
  p.d_taps = make_fastdiv(p.taps_w);
  {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = kSmemTotal;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const cudaError_t le = ss ? launch_gemm<true>(cfg, pingpong, bn, tmA, tmB, tmD, tmR, tmY, p)
                              : launch_gemm<false>(cfg, pingpong, bn, tmA, tmB, tmD, tmR, tmY, p);
    if (le != cudaSuccess) return set_error(VTX_ECUDA, "gemm_wgmma_kernel PDL launch: %s", cudaGetErrorString(le));
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(VTX_ECUDA, "gemm_wgmma_kernel launch: %s", cudaGetErrorString(e));
  return VTX_OK;
}
