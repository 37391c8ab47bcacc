// Streaming kernel for the masked-residual 1x1 dgrads of the identity bottlenecks (Engine.backbone_backward):
//
//   dx[M, N] = bf16( bf16_rn(dy1[M, K] . W1[K, N]) + m3 (.) dOut )       (packed bf16 add, as add_res_bf16x2)
//   [+ the BN-backward sums of the previous block over dx: sum dz, sum dz * (y - mean) * invstd, dz = dx * bnr_mask]
//
// K is 64 to 256, so the MMAs are a small part of the launch: its time is the bytes of dOut, y, the two bit masks and
// dx.  The persistent GEMM (gemm_tc.cu) runs these calls on 256-wide tiles whose epilogue phases (residual wait, mask
// loads, y loads, store) follow one another on one CTA per SM, and reached 40-55 % of the HBM bandwidth.  Here:
//   * one CTA per SM owns one column block (BN = 128 columns, 64 for K = 256) for its whole life: the W1 slice [K, BN]
//     is loaded once and stays in shared memory; the CTA walks 64-row tiles mt = w, w + walkers, ...  All CTAs with the same walker index w run
//     the same row tile at about the same time, so dy1 is read from HBM once and re-read from L2 by the others;
//   * a producer warp streams, per row tile, dy1 [64, K], dOut [64, BN], y [64, BN] and both masks' bytes into a
//     ring of 3-4 stages (150-170 KB in flight per SM) with the TMA;
//   * two consumer warpgroups take alternate row tiles: m64nBNk16 wgmma in the persistent kernel's K order (D is bit
//     for bit that route's), then the epilogue entirely out of shared memory into a bf16 tile of their own that one
//     thread stores with the TMA while the warpgroup moves on;
//   * the BN-backward sums stay in registers, per thread over its BN / 4 columns and all its rows of the CTA's tiles, and
//     are reduced once at the end: lanes (shuffles), then the eight warps in order, then one atomic per column per CTA.
// Selected by vtx_gemm (gemm_tc.cu) for the calls resid_dgrad_serves() accepts.
#include "ptx.cuh"
#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {

namespace {

constexpr int kRBM = 64;                 // rows of a tile: one wgmma m64 block per consumer warpgroup
constexpr int kRMaxStages = 8;
constexpr int kRThreads = 288;           // consumer warpgroups 0 and 1 (warps 0-7), producer warp 8
constexpr int kRSmem = 232448;           // 227 KB: the per-block maximum on sm_90
constexpr int kRCtrl = 1024;             // barriers, then the column block's BN means at byte 512
constexpr int kRMaskBytes = kRBM * 16;   // the mask bytes of 128 columns of a tile: [64 rows][16 B]

struct ResidParams {
  int m_tiles, walkers, nblk;
  int stages, stage_bytes, a_bytes;
  int N;
  const float* bnp;  // [4, N] of the BN whose output gradient dx is (bnr)
  float* sums;       // [2, N]
};

// acc pair -> bf16x2 + (masked) bf16x2 residual word in one packed add: the rounding of the persistent kernel's
// TMA-staged residual (and of torch's own bf16 graph)
__device__ __forceinline__ uint32_t res_add(float lo, float hi, uint32_t res) {
  const __nv_bfloat162 o = __hadd2(__floats2bfloat162_rn(lo, hi), *reinterpret_cast<const __nv_bfloat162*>(&res));
  return *reinterpret_cast<const uint32_t*>(&o);
}
__device__ __forceinline__ uint32_t lds32r(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts32r(uint32_t a, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void named_bar(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// zero the bf16 halves of a word whose mask bits (bit 0: low half, bit 1: high half) are clear
__device__ __forceinline__ uint32_t keep_halves(uint32_t w, uint32_t bits) {
  return w & (((bits & 1u) ? 0x0000ffffu : 0u) | ((bits & 2u) ? 0xffff0000u : 0u));
}

// Stage layout (every part 1024-aligned): dy1 rows [K / 64 slabs of 64 rows x 128 B] | dOut [BN / 64 slabs] | y
// [BN / 64 slabs, BNR] | m3 bytes [64 rows x 16 B] | bnr mask bytes [64 x 16 B, BNR].  The mask boxes cover the 128
// columns around the block (16-byte aligned); a 64-wide block uses the half it owns.
// KB = K / 64 (1, 2 or 4): a compile-time K loop keeps the accumulators out of the compiler's way around the wgmma.
// BN = 128 (K <= 128) or 64 (K = 256: the W1 slice and a 3-stage ring fit in shared memory only that way).
template <bool BNR, int KB, int BN>
__global__ void __launch_bounds__(kRThreads, 1)
resid_dgrad_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                   const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmM,
                   const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmMB,
                   const __grid_constant__ CUtensorMap tmD, const ResidParams p) {
  VTX_PDL_TRIGGER();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(base);  // [kRMaxStages]
  uint64_t* empty_bar = full_bar + kRMaxStages;            // [kRMaxStages]
  uint64_t* w_bar = empty_bar + kRMaxStages;               // the W slice landed
  float* s_mean = reinterpret_cast<float*>(base + 512);    // [BN]
  constexpr int NS = BN / 64;                              // 64-column slabs of a tile
  constexpr int kOutBytes = kRBM * BN * 2;                 // one bf16 output tile: NS slabs of [64 rows][128 B], SW128
  uint8_t* sW = base + kRCtrl;                             // [K / 64][NS slabs][64 k rows][128 B]
  uint8_t* sOut = sW + KB * NS * 8192;                     // [2 warpgroups][kOutBytes]
  uint8_t* sStage = sOut + 2 * kOutBytes;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int nb = blockIdx.x % p.nblk;  // column block
  const int wk = blockIdx.x / p.nblk;  // walker: row tiles wk, wk + walkers, ...
  const int mask_off = p.a_bytes + NS * 8192 + (BNR ? NS * 8192 : 0);

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmR);
    tma_prefetch_desc(&tmM);
    tma_prefetch_desc(&tmD);
    if (BNR) {
      tma_prefetch_desc(&tmY);
      tma_prefetch_desc(&tmMB);
    }
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 1);  // a tile is consumed by one warpgroup; one thread of it hands the stage back
    }
    mbar_init(w_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  VTX_PDL_WAIT();

  if (warp == 8) {
    // ===================================================== TMA producer (one thread)
    if (lane == 0) {
      mbar_arrive_expect_tx(w_bar, (uint32_t)(KB * NS * 8192));
      for (int kb = 0; kb < KB; ++kb)
        for (int j = 0; j < NS; ++j) tma_load_2d(sW + (kb * NS + j) * 8192, &tmW, w_bar, nb * BN + 64 * j, kb * 64);
      const uint32_t tx = (uint32_t)(p.a_bytes + NS * 8192 + kRMaskBytes + (BNR ? NS * 8192 + kRMaskBytes : 0));
      int s = 0;
      for (int mt = wk; mt < p.m_tiles; mt += p.walkers, ++s) {
        const int stage = s % p.stages;
        mbar_wait(&empty_bar[stage], ((uint32_t)(s / p.stages) & 1u) ^ 1u);
        uint8_t* st = sStage + stage * p.stage_bytes;
        uint64_t* fb = &full_bar[stage];
        mbar_arrive_expect_tx(fb, tx);
        const int r0 = mt * kRBM, c0 = nb * BN, mc0 = (c0 / 128) * 16;
        for (int kb = 0; kb < KB; ++kb) tma_load_2d(st + kb * 8192, &tmA, fb, kb * 64, r0);
        for (int j = 0; j < NS; ++j) tma_load_2d(st + p.a_bytes + j * 8192, &tmR, fb, c0 + 64 * j, r0);
        tma_load_2d(st + mask_off, &tmM, fb, mc0, r0);
        if (BNR) {
          for (int j = 0; j < NS; ++j) tma_load_2d(st + p.a_bytes + (NS + j) * 8192, &tmY, fb, c0 + 64 * j, r0);
          tma_load_2d(st + mask_off + kRMaskBytes, &tmMB, fb, mc0, r0);
        }
      }
    }
    return;
  }

  // ===================================================== consumers: warpgroup wg takes the CTA's tiles wg, wg + 2, ...
  const int ct = threadIdx.x;  // 0..255
  const int wg = ct >> 7;
  const int wl = (ct >> 5) & 3;
  const int t = ct & 127;
  const int q = lane & 3;
  const int sw = lane >> 2;  // row & 7 of both rows this thread holds (rows 16 wl + lane / 4 + 8 hh)
  if (BNR) {
    if (ct < BN) s_mean[ct] = __ldg(p.bnp + nb * BN + ct);
    named_bar(3, 256);
  }
  constexpr int NP = BNR ? BN / 4 : 1;
  float ps[NP], pq[NP];  // partial sums of columns 8 j + 2 q + e, index 2 j + e
#pragma unroll
  for (int i = 0; i < NP; ++i) ps[i] = pq[i] = 0.f;

  uint8_t* out = sOut + wg * kOutBytes;
  const uint32_t sW0 = smem_u32(sW);
  mbar_wait(w_bar, 0);
  for (int s = wg;; s += 2) {
    const int mt = wk + s * p.walkers;
    if (mt >= p.m_tiles) break;
    const int stage = s % p.stages;
    const int round = s / p.stages;
    // With an odd ring depth the stage's previous round (tile s - stages) belonged to the other warpgroup, and a parity
    // wait on full_bar alone would pass on that round's phase if it had not landed yet.  Waiting first until that tile
    // was handed back (empty_bar's phase round - 1: this warpgroup handed back round - 2 itself, and round cannot
    // complete before it) leaves full_bar's parity only one meaning.
    if (round > 0) mbar_wait(&empty_bar[stage], (uint32_t)(round - 1) & 1u);
    mbar_wait(&full_bar[stage], (uint32_t)round & 1u);
    const uint32_t st = smem_u32(sStage + stage * p.stage_bytes);

    // ---- K loop: the persistent kernel's order (k-block, then four k16 steps)
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) fence_operand(acc[i]);
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t ad = make_wgmma_desc(st + kb * 8192 + k * 32, 16, 1024);
        const uint64_t bd = make_wgmma_desc(sW0 + kb * NS * 8192 + k * 2048, 8192, 1024);
        if constexpr (BN == 128) wgmma_n128<0, 1>(acc, ad, bd, (kb > 0 || k > 0) ? 1u : 0u);
        else wgmma_n64<0, 1>(acc, ad, bd, (kb > 0 || k > 0) ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) fence_operand(acc[i]);

    // ---- the output tile's previous TMA store must have read it
    if (t == 0) tma_store_wait_read<0>();
    named_bar(1 + wg, 128);

    // ---- epilogue: accumulator element 4 j + 2 hh + e is row 16 wl + lane / 4 + 8 hh, column 8 j + 2 q + e
    // (mask word w of a row: columns 32 w .. 32 w + 31 of the block; a 64-wide block in the upper half of its
    // 128-column mask box starts at word 2)
    uint32_t m3[2][BN / 32], mb[2][BN / 32];
    const bool upper = BN == 64 && (nb & 1);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = wl * 16 + sw + 8 * hh;
      const uint4 v = lds128(st + mask_off + r * 16);
      m3[hh][0] = upper ? v.z : v.x; m3[hh][1] = upper ? v.w : v.y;
      if (BN == 128) { m3[hh][BN / 64] = v.z; m3[hh][BN / 32 - 1] = v.w; }
      if (BNR) {
        const uint4 b = lds128(st + mask_off + kRMaskBytes + r * 16);
        mb[hh][0] = upper ? b.z : b.x; mb[hh][1] = upper ? b.w : b.y;
        if (BN == 128) { mb[hh][BN / 64] = b.z; mb[hh][BN / 32 - 1] = b.w; }
      }
    }
    const uint32_t row0 = (uint32_t)(wl * 16 + sw) * 128 + q * 4;
    const uint32_t so = smem_u32(out);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const uint32_t off = row0 + (j >> 3) * 8192 + (((j & 7) ^ sw) << 4);
      const int bit = 8 * (j & 3) + 2 * q;
      float2 mean = make_float2(0.f, 0.f);
      if (BNR) mean = *reinterpret_cast<const float2*>(s_mean + 8 * j + 2 * q);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const uint32_t a = off + hh * 8 * 128;
        const uint32_t res = keep_halves(lds32r(st + p.a_bytes + a), m3[hh][j >> 2] >> bit);
        const uint32_t o = res_add(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1], res);
        sts32r(so + a, o);
        if (BNR) {
          const uint32_t dz = keep_halves(o, mb[hh][j >> 2] >> bit);
          const uint32_t y = lds32r(st + p.a_bytes + NS * 8192 + a);
          const float dz0 = __uint_as_float(dz << 16), dz1 = __uint_as_float(dz & 0xffff0000u);
          ps[2 * j] += dz0;
          ps[2 * j + 1] += dz1;
          pq[2 * j] += dz0 * (__uint_as_float(y << 16) - mean.x);
          pq[2 * j + 1] += dz1 * (__uint_as_float(y & 0xffff0000u) - mean.y);
        }
      }
    }
    fence_proxy_async();  // the staging writes become visible to the TMA store
    named_bar(1 + wg, 128);
    if (t == 0) {
      mbar_arrive(&empty_bar[stage]);
      for (int j = 0; j < NS; ++j) tma_store_2d(&tmD, out + j * 8192, nb * BN + 64 * j, mt * kRBM);
      tma_store_commit();
    }
  }
  if (t == 0) tma_store_wait_read<0>();
  if (BNR) {
    // lanes with the same q hold the same columns: add them (xor 4, 8, 16), then the eight warps in order through
    // the (now idle) output tiles, then one atomic per column and sum
#pragma unroll
    for (int i = 0; i < NP; ++i) {
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        ps[i] += __shfl_xor_sync(0xffffffffu, ps[i], o);
        pq[i] += __shfl_xor_sync(0xffffffffu, pq[i], o);
      }
    }
    named_bar(3, 256);
    float2* scr = reinterpret_cast<float2*>(sOut);  // [8 warps][BN]
    if (sw == 0) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        scr[warp * BN + 8 * j + 2 * q] = make_float2(ps[2 * j], pq[2 * j]);
        scr[warp * BN + 8 * j + 2 * q + 1] = make_float2(ps[2 * j + 1], pq[2 * j + 1]);
      }
    }
    named_bar(3, 256);
    if (ct < BN) {
      float a = 0.f, b = 0.f;
      for (int w = 0; w < 8; ++w) {
        const float2 v = scr[w * BN + ct];
        a += v.x;
        b += v.y;
      }
      const int col = nb * BN + ct;
      atomicAdd(p.sums + col, a);
      atomicAdd(p.sums + p.N + col, b * __ldg(p.bnp + p.N + col));  // sum dz * (y - mean)  ->  sum dz * xhat
    }
  }
}

typedef CUresult (*PFN_encode)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                               const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                               CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 2-D tensor map: rows x cols elements of `esize` bytes, row stride ld elements, box of box_c x box_r elements
// (bf16 operands 128B-swizzled, mask bytes unswizzled); rows and columns past the extent read as zeros / are clipped
int tmap2d(CUtensorMap* tm, const void* ptr, bool bytes, uint64_t cols, uint64_t rows, uint64_t ld, uint32_t box_c,
           uint32_t box_r) {
  static PFN_encode enc = nullptr;
  if (enc == nullptr) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &qr) != cudaSuccess ||
        qr != cudaDriverEntryPointSuccess)
      return set_error(VTX_ECUDA, "cuTensorMapEncodeTiled entry point not available");
    enc = reinterpret_cast<PFN_encode>(fp);
  }
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t str[1] = {ld * (bytes ? 1 : 2)};
  const cuuint32_t box[2] = {box_c, box_r};
  const cuuint32_t es[2] = {1, 1};
  const CUresult r = enc(tm, bytes ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                         const_cast<void*>(ptr), dims, str, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         bytes ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(VTX_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return VTX_OK;
}

bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// column-block width of a call: 128, or 64 for K = 256 (a 128-wide W1 slice would leave room for one stage)
int resid_bn(const VtxGemm* g) { return g->K > 128 ? 64 : 128; }
// stage bytes / ring depth of a call (0 stages: the W slice and three stages do not fit)
int resid_stage_bytes(const VtxGemm* g) {
  const bool bnr = g->bnr_y != nullptr;
  const int slabs = resid_bn(g) / 64;
  return (g->K / 64) * 8192 + slabs * 8192 + kRMaskBytes + (bnr ? slabs * 8192 + kRMaskBytes : 0);
}
int resid_stages(const VtxGemm* g) {
  const int bn = resid_bn(g);
  const int fixed = 1024 /*alignment slack*/ + kRCtrl + (g->K / 64) * (bn / 64) * 8192 + 2 * kRBM * bn * 2;
  const int st = (kRSmem - fixed) / resid_stage_bytes(g);
  return st < 3 ? 0 : st > kRMaxStages ? kRMaxStages : st;
}

template <bool BNR, int KB, int BN>
cudaError_t launch_resid(const cudaLaunchConfig_t& cfg, const CUtensorMap& tmA, const CUtensorMap& tmW,
                         const CUtensorMap& tmR, const CUtensorMap& tmM, const CUtensorMap& tmY,
                         const CUtensorMap& tmMB, const CUtensorMap& tmD, const ResidParams& p) {
  cudaError_t e = cudaFuncSetAttribute(resid_dgrad_kernel<BNR, KB, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       kRSmem);
  if (e != cudaSuccess) return e;
  return cudaLaunchKernelEx(&cfg, resid_dgrad_kernel<BNR, KB, BN>, tmA, tmW, tmR, tmM, tmY, tmMB, tmD, p);
}

}  // namespace

// The calls this kernel serves: conv_mode 0, A [M, K] K-major, B [K, N] N-major, bf16 D, alpha 1, nothing in the
// epilogue but a TMA-stageable residual under its bit mask, optionally the BN-backward sums with a bit mask; N a
// multiple of 128, K 64, 128 or 256 (the W slice and a ring of at least three stages fit); every operand fit for the
// TMA (16-byte aligned, row strides multiples of 16 bytes).  Everything else runs the persistent kernel.
bool resid_dgrad_serves(const VtxGemm* g) {
  const bool bnr = g->bnr_y != nullptr;
  if (g->conv_mode != 0 || g->a_mn || !g->b_mn || g->out_f32 || g->atomic || g->split_k > 1 || g->act || g->bias ||
      g->stats || (g->alpha != 0.f && g->alpha != 1.f) || g->col_scale || g->col_shift)
    return false;
  if (!g->residual || !g->residual_mask || g->N % 128 != 0 || (g->K != 64 && g->K != 128 && g->K != 256) ||
      resid_stages(g) == 0)
    return false;
  if (g->lda % 8 || g->ldb % 8 || g->ldd % 8 || g->ldr % 8 || !al16(g->A) || !al16(g->B) || !al16(g->D) ||
      !al16(g->residual) || !al16(g->residual_mask))
    return false;
  if (bnr && (!g->bnr_mask || !g->bnr_bnp || !g->bnr_sums || g->bnr_ldy % 8 || !al16(g->bnr_y) || !al16(g->bnr_mask)))
    return false;
  return true;
}

int resid_dgrad(const VtxGemm* g, cudaStream_t stream) {
  const bool bnr = g->bnr_y != nullptr;
  const int bn = resid_bn(g);
  const uint64_t M = (uint64_t)g->M, N = (uint64_t)g->N, K = (uint64_t)g->K;
  CUtensorMap tmA, tmW, tmR, tmM, tmY, tmMB, tmD;
  memset(&tmY, 0, sizeof(tmY));
  memset(&tmMB, 0, sizeof(tmMB));
  int rc;
  if ((rc = tmap2d(&tmA, g->A, false, K, M, (uint64_t)g->lda, 64, kRBM)) != VTX_OK) return rc;
  if ((rc = tmap2d(&tmW, g->B, false, N, K, (uint64_t)g->ldb, 64, 64)) != VTX_OK) return rc;
  if ((rc = tmap2d(&tmR, g->residual, false, N, M, (uint64_t)g->ldr, 64, kRBM)) != VTX_OK) return rc;
  if ((rc = tmap2d(&tmM, g->residual_mask, true, N / 8, M, N / 8, 16, kRBM)) != VTX_OK) return rc;
  if ((rc = tmap2d(&tmD, g->D, false, N, M, (uint64_t)g->ldd, 64, kRBM)) != VTX_OK) return rc;
  if (bnr) {
    if ((rc = tmap2d(&tmY, g->bnr_y, false, N, M, (uint64_t)g->bnr_ldy, 64, kRBM)) != VTX_OK) return rc;
    if ((rc = tmap2d(&tmMB, g->bnr_mask, true, N / 8, M, N / 8, 16, kRBM)) != VTX_OK) return rc;
  }
  ResidParams p;
  memset(&p, 0, sizeof(p));
  p.m_tiles = (g->M + kRBM - 1) / kRBM;
  p.nblk = g->N / bn;
  const int kb = g->K / 64;
  p.a_bytes = kb * 8192;
  p.stage_bytes = resid_stage_bytes(g);
  p.stages = resid_stages(g);
  p.N = g->N;
  p.bnp = g->bnr_bnp;
  p.sums = g->bnr_sums;
  // one CTA per SM: every column block gets the same number of walkers, and none without a row tile
  const int sms = vtx_num_sms();
  int walkers = sms / p.nblk;
  if (walkers < 1) walkers = 1;
  if (walkers > p.m_tiles) walkers = p.m_tiles;
  p.walkers = walkers;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(walkers * p.nblk));
  cfg.blockDim = dim3(kRThreads);
  cfg.dynamicSmemBytes = kRSmem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t le;
  if (kb == 1) le = bnr ? launch_resid<true, 1, 128>(cfg, tmA, tmW, tmR, tmM, tmY, tmMB, tmD, p)
                        : launch_resid<false, 1, 128>(cfg, tmA, tmW, tmR, tmM, tmY, tmMB, tmD, p);
  else if (kb == 2) le = bnr ? launch_resid<true, 2, 128>(cfg, tmA, tmW, tmR, tmM, tmY, tmMB, tmD, p)
                             : launch_resid<false, 2, 128>(cfg, tmA, tmW, tmR, tmM, tmY, tmMB, tmD, p);
  else le = bnr ? launch_resid<true, 4, 64>(cfg, tmA, tmW, tmR, tmM, tmY, tmMB, tmD, p)
                : launch_resid<false, 4, 64>(cfg, tmA, tmW, tmR, tmM, tmY, tmMB, tmD, p);
  if (le != cudaSuccess) return set_error(VTX_ECUDA, "resid_dgrad_kernel launch: %s", cudaGetErrorString(le));
  return VTX_OK;
}

}  // namespace vtx
