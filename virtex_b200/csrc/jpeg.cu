// Baseline JPEG decoding on the device: compressed bytes -> uint8 HWC RGB, bit-exact with libjpeg-turbo's default
// decompression as OpenCV's cv2.imdecode(IMREAD_COLOR) + cvtColor(BGR2RGB) runs it (the reference's image reads,
// virtex/data/datasets/*.py): islow integer IDCT with its 10-bit wrap-around range limit, fancy (triangle) chroma
// upsampling, table-driven YCbCr -> RGB, grey replicated to three channels, EXIF orientation.  The arithmetic is
// written from ITU T.81 and libjpeg's documented fixed-point constants.
//
// One batch of heterogeneous images per call; the host parses headers (virtex_b200/jpeg.py) into the per-image tables
// described in include/virtex_b200.h.  Stages, each one kernel:
//   unstuff      one CTA per image: drop FF00 stuffing and fill bytes, split the entropy data at RSTn markers
//   sync         Huffman decoding over fixed-size bit chunks that self-synchronise (Weissenberger & Schmidt, ICPP
//                2018): round 0 decodes every chunk from its first bit as if an MCU started there; round r re-decodes
//                chunk j from the exit state of chunk j-1 whenever that changed in round r-1.  A state is (bit
//                position, block in the MCU, zig-zag index).
//   count_scan   exclusive scan of the blocks each chunk completes
//   coefs        decodes every chunk once more from its predecessor's exit and writes the coefficients.  It also
//                re-checks the exit state and block count each chunk recorded: a mismatch marks the image UNSYNCED,
//                and the host runs more rounds.  Exactness never depends on how fast the chunks synchronise.
//   dc_scan      DC differences -> absolute values, per component, restarting at every restart interval
//   idct         dequantise + islow IDCT into per-component sample planes
//   color        upsampling + colour conversion + orientation into the caller's RGB buffer
// Every read of entropy data is bounds-checked against its segment; a code missing from the table, a run past
// coefficient 63, running out of bits or an unexpected marker set the image's status word instead.
#include <cub/block/block_scan.cuh>

#include "vtx_common.cuh"
#include "../../include/virtex_b200.h"

namespace vtx {
namespace jpg {

struct HuffTab {            // VTX_JPEG_HUFF_BYTES, built by virtex_b200/jpeg.py
  uint16_t look[512];       // 9-bit prefix -> (code length << 8) | symbol, 0 when the code is longer than 9 bits
  int32_t maxcode[18];      // largest code of each length, -1 when none
  int32_t valoff[17];       // index into vals of the first code of each length, minus that code
  uint8_t vals[256];
  uint8_t pad[VTX_JPEG_HUFF_BYTES - 1024 - 72 - 68 - 256];
};
static_assert(sizeof(HuffTab) == VTX_JPEG_HUFF_BYTES, "HuffTab layout");

__constant__ uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// MSB-first reader over one unstuffed segment; bytes past its end read as zero (the caller checks the bit count).
struct Bits {
  const uint8_t* p;
  int pos, end, nb;
  uint64_t buf;
  __device__ __forceinline__ void init(const uint8_t* base, int len, int bit) {
    p = base; end = len; pos = bit >> 3; buf = 0; nb = 0;
    fill();
    buf <<= (bit & 7);
    nb -= (bit & 7);
  }
  __device__ __forceinline__ void fill() {
    while (nb <= 56) {
      const uint64_t b = pos < end ? p[pos] : 0u;
      ++pos;
      buf |= b << (56 - nb);
      nb += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t)(buf >> (64 - n)); }
  __device__ __forceinline__ void skip(int n) { buf <<= n; nb -= n; }
};

__device__ __forceinline__ int extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

struct Run {
  int bit, u, count, err;
};

// Decodes symbols from state (bit, u = block-in-MCU * 64 + zig-zag index) while bit < stop.  count = blocks completed.
// FINAL: blocks with index first_blk + count < expected are written to coef (block `first_blk + count` at
// coef + (blk_base + first_blk + count) * 64) and errors in them are reported; `last` stops once expected is reached.
template <bool FINAL>
__device__ Run decode_run(const uint8_t* seg, int seglen, int bit, int u, int stop, const int* inf, const HuffTab* huff,
                          int first_blk, int expected, bool last, int16_t* coef) {
  Run r{bit, u, 0, 0};
  const int segbits = seglen * 8;
  const int bpm = inf[VTX_JPEG_I_BPM];
  const int n0 = inf[VTX_JPEG_I_COMP] * inf[VTX_JPEG_I_COMP + 1];
  int b = u >> 6, k = u & 63;
  Bits br;
  br.init(seg, seglen, bit);
  int16_t* blk = nullptr;
  bool active = FINAL && first_blk < expected;
  if (FINAL && active) blk = coef + (long long)first_blk * 64;
  while (r.bit < stop) {
    if (FINAL && last && !active) break;
    const int c = b < n0 ? 0 : b - n0 + 1;
    const HuffTab* t = huff + inf[VTX_JPEG_I_COMP + 8 * c + (k == 0 ? 3 : 4)];
    br.fill();
    const uint32_t w = br.peek(16);
    int len, sym;
    const uint32_t e = t->look[w >> 7];
    if (e) {
      len = (int)(e >> 8);
      sym = (int)(e & 255u);
    } else {
      len = 10;
      while (len <= 16 && (int)(w >> (16 - len)) > t->maxcode[len]) ++len;
      if (len > 16) {  // not a code of this table: consume one bit so that speculative decoding keeps moving
        len = 1;
        sym = 0;
        if (FINAL && active) r.err |= VTX_JPEG_ST_BADCODE;
      } else {
        sym = t->vals[min(max(t->valoff[len] + (int)(w >> (16 - len)), 0), 255)];
      }
    }
    br.skip(len);
    r.bit += len;
    if (k == 0) {
      const int s = sym & 15;
      int v = 0;
      if (s) { v = extend((int)br.peek(s), s); br.skip(s); r.bit += s; }
      if (FINAL && active) blk[0] = (int16_t)v;  // DC difference; dc_scan makes it absolute
      k = 1;
    } else {
      const int rr = sym >> 4, s = sym & 15;
      if (s) {
        k += rr;
        const int v = extend((int)br.peek(s), s);
        br.skip(s);
        r.bit += s;
        if (k > 63) {
          if (FINAL && active) r.err |= VTX_JPEG_ST_RUN;
          k = 64;
        } else {
          if (FINAL && active) blk[kNatural[k]] = (int16_t)v;
          ++k;
        }
      } else if (rr == 15) {
        k += 16;
        if (k > 64) {
          if (FINAL && active) r.err |= VTX_JPEG_ST_RUN;
          k = 64;
        }
      } else {
        k = 64;
      }
    }
    if (FINAL && active && r.bit > segbits) r.err |= VTX_JPEG_ST_OUT;
    if (k >= 64) {
      k = 0;
      ++r.count;
      if (++b == bpm) b = 0;
      if (FINAL) {
        active = first_blk + r.count < expected;
        if (active) blk += 64;
      }
    }
    if (FINAL && r.err) break;
  }
  if (FINAL && last && active && !r.err) r.err |= VTX_JPEG_ST_OUT;  // the segment ended before its last block
  r.u = b * 64 + k;
  return r;
}

// Image of a flat slot index: the last n with base(n) <= slot, base read from info (int32 column) or info64.
__device__ __forceinline__ int image_of(const int* info, int B, int slot) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (info[mid * VTX_JPEG_NI + VTX_JPEG_I_CHUNK_BASE] <= slot) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ int segment_of(const int* chunk0, int nseg, int j) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (chunk0[mid] <= j) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ int segment_blocks(const int* inf, int s) {
  const int nmcu = inf[VTX_JPEG_I_MCUX] * inf[VTX_JPEG_I_MCUY], ri = inf[VTX_JPEG_I_RI];
  const int mcus = ri > 0 ? min(ri, nmcu - s * ri) : nmcu;
  return mcus * inf[VTX_JPEG_I_BPM];
}

// ------------------------------------------------------------------------------------------------------- unstuff
__global__ void __launch_bounds__(256) jpeg_unstuff_kernel(const uint8_t* __restrict__ src, const int* __restrict__ info,
                                                          const long long* __restrict__ info64, uint8_t* __restrict__ ent,
                                                          int* __restrict__ seg_start, int* __restrict__ seg_len,
                                                          int* __restrict__ seg_chunk0, int* __restrict__ nchunks,
                                                          int* __restrict__ status, int chunk_bits) {
  VTX_PDL_TRIGGER();
  typedef cub::BlockScan<int, 256> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int carry_keep, carry_rst, bad;
  const int n = blockIdx.x, tid = threadIdx.x;
  const int* inf = info + n * VTX_JPEG_NI;
  const long long* q = info64 + n * VTX_JPEG_N64;
  const uint8_t* in = src + q[VTX_JPEG_Q_ENT_SRC];
  const int L = (int)q[VTX_JPEG_Q_ENT_LEN];  // in[L], in[L + 1] are the EOI marker (checked by the host)
  uint8_t* out = ent + q[VTX_JPEG_Q_ENT_DST];
  const int nseg = inf[VTX_JPEG_I_NSEG];
  int* sst = seg_start + inf[VTX_JPEG_I_SEG_BASE];
  int* sln = seg_len + inf[VTX_JPEG_I_SEG_BASE];
  int* sc0 = seg_chunk0 + inf[VTX_JPEG_I_SEG_BASE];
  if (tid == 0) { carry_keep = 0; carry_rst = 0; bad = 0; sst[0] = 0; }
  __syncthreads();
  for (int base = 0; base < L; base += 256 * 16) {
    // per byte: keep (entropy data), drop (stuffed 00, fill FF, marker code), or an RST boundary at its FF
    uint32_t keep = 0, rst = 0;
    const int i0 = base + tid * 16;
    for (int t = 0; t < 16; ++t) {
      const int i = i0 + t;
      if (i >= L) break;
      const int b = in[i], prev = i > 0 ? in[i - 1] : 0, next = in[i + 1];
      if (b == 0xFF) {
        if (next == 0x00) keep |= 1u << t;
        else if (next >= 0xD0 && next <= 0xD7) rst |= 1u << t;
        else if (next != 0xFF) bad = 1;  // any other marker inside the scan
      } else if (prev != 0xFF) {
        keep |= 1u << t;
      }  // else: stuffed 00 or the code byte of a marker
    }
    const int packed = __popc(keep) | (__popc(rst) << 16);
    int excl, total;
    Scan(tmp).ExclusiveSum(packed, excl, total);
    int o = carry_keep + (excl & 0xffff), kr = carry_rst + (excl >> 16);
    for (int t = 0; t < 16; ++t) {
      const int i = i0 + t;
      if (i >= L) break;
      if (keep >> t & 1u) {
        out[o++] = in[i];
      } else if (rst >> t & 1u) {
        if (in[i + 1] != 0xD0 + (kr & 7) || kr + 1 >= nseg) bad = 1;
        else sst[kr + 1] = o;
        ++kr;
      }
    }
    __syncthreads();
    if (tid == 0) { carry_keep += total & 0xffff; carry_rst += total >> 16; }
    __syncthreads();
  }
  if (tid == 0 && carry_rst != nseg - 1) bad = 1;
  __syncthreads();
  if (bad) {
    if (tid == 0) { atomicOr(status + n, VTX_JPEG_ST_MARKER); nchunks[n] = 0; }
    return;
  }
  // segment lengths and their chunk counts (an empty segment still gets one chunk, which reports it)
  int carry = 0;
  for (int s0 = 0; s0 < nseg; s0 += 256) {
    const int s = s0 + tid;
    int nc = 0;
    if (s < nseg) {
      const int end = s + 1 < nseg ? sst[s + 1] : carry_keep;
      sln[s] = end - sst[s];
      nc = max(1, (int)(((long long)sln[s] * 8 + chunk_bits - 1) / chunk_bits));
    }
    int excl, total;
    Scan(tmp).ExclusiveSum(nc, excl, total);
    if (s < nseg) sc0[s] = carry + excl;
    carry += total;
    __syncthreads();
  }
  if (tid == 0) {
    if (carry > inf[VTX_JPEG_I_CHUNK_CAP]) { atomicOr(status + n, VTX_JPEG_ST_MARKER); carry = 0; }
    nchunks[n] = carry;
  }
}

// ---------------------------------------------------------------------------------------------- chunk decoding
struct ChunkCtx {
  int n, j, s, i, nc_seg;
  const int* inf;
  const uint8_t* seg;
  int seglen;
};

__device__ __forceinline__ bool chunk_ctx(int slot, const uint8_t* ent, const int* info, const long long* info64,
                                          const int* seg_start, const int* seg_len, const int* seg_chunk0,
                                          const int* nchunks, int B, ChunkCtx* c) {
  c->n = image_of(info, B, slot);
  c->inf = info + c->n * VTX_JPEG_NI;
  c->j = slot - c->inf[VTX_JPEG_I_CHUNK_BASE];
  const int total = nchunks[c->n];
  if (c->j >= total) return false;
  const int sb = c->inf[VTX_JPEG_I_SEG_BASE], nseg = c->inf[VTX_JPEG_I_NSEG];
  c->s = segment_of(seg_chunk0 + sb, nseg, c->j);
  const int first = seg_chunk0[sb + c->s];
  c->i = c->j - first;
  c->nc_seg = (c->s + 1 < nseg ? seg_chunk0[sb + c->s + 1] : total) - first;
  c->seg = ent + info64[c->n * VTX_JPEG_N64 + VTX_JPEG_Q_ENT_DST] + seg_start[sb + c->s];
  c->seglen = seg_len[sb + c->s];
  return true;
}

// state int4 {exit bit, exit u, blocks completed, exit changed in this round}, two buffers [2][slots]
__global__ void __launch_bounds__(128) jpeg_sync_kernel(const uint8_t* __restrict__ ent, const int* __restrict__ info,
                                                       const long long* __restrict__ info64, const void* __restrict__ huff,
                                                       const int* __restrict__ seg_start, const int* __restrict__ seg_len,
                                                       const int* __restrict__ seg_chunk0, const int* __restrict__ nchunks,
                                                       int B, int slots, const int4* __restrict__ st_in,
                                                       int4* __restrict__ st_out, int round, int* __restrict__ rounds,
                                                       int chunk_bits) {
  VTX_PDL_TRIGGER();
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= slots) return;
  ChunkCtx c;
  if (!chunk_ctx(slot, ent, info, info64, seg_start, seg_len, seg_chunk0, nchunks, B, &c)) return;
  const HuffTab* tabs = (const HuffTab*)huff;
  const int stop = min((c.i + 1) * chunk_bits, c.seglen * 8);
  if (c.i == c.nc_seg - 1) {  // a segment's last chunk has no successor: nothing reads its exit or count
    st_out[slot] = make_int4(0, 0, 0, 0);
    return;
  }
  if (round == 0) {
    const Run r = decode_run<false>(c.seg, c.seglen, c.i * chunk_bits, 0, stop, c.inf, tabs, 0, 0, false, nullptr);
    st_out[slot] = make_int4(r.bit, r.u, r.count, 1);
    return;
  }
  const int4 old = st_in[slot];
  if (c.i == 0 || st_in[slot - 1].w == 0) {  // entry unchanged since the last round (a segment's first is exact)
    st_out[slot] = make_int4(old.x, old.y, old.z, 0);
    return;
  }
  const int4 e = st_in[slot - 1];
  const Run r = decode_run<false>(c.seg, c.seglen, e.x, e.y, stop, c.inf, tabs, 0, 0, false, nullptr);
  const int changed = r.bit != old.x || r.u != old.y;
  st_out[slot] = make_int4(r.bit, r.u, r.count, changed);
  if (changed) atomicMax(rounds + c.n, round);
}

__global__ void __launch_bounds__(256) jpeg_count_scan_kernel(const int* __restrict__ info, const int* __restrict__ nchunks,
                                                             const int4* __restrict__ st, int* __restrict__ excl) {
  VTX_PDL_TRIGGER();
  typedef cub::BlockScan<int, 256> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const int n = blockIdx.x;
  const int base = info[n * VTX_JPEG_NI + VTX_JPEG_I_CHUNK_BASE], total = nchunks[n];
  int carry = 0;
  for (int j0 = 0; j0 < total; j0 += 256) {
    const int j = j0 + threadIdx.x;
    const int v = j < total ? st[base + j].z : 0;
    int e, agg;
    Scan(tmp).ExclusiveSum(v, e, agg);
    if (j < total) excl[base + j] = carry + e;
    carry += agg;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(128) jpeg_coefs_kernel(const uint8_t* __restrict__ ent, const int* __restrict__ info,
                                                        const long long* __restrict__ info64, const void* __restrict__ huff,
                                                        const int* __restrict__ seg_start, const int* __restrict__ seg_len,
                                                        const int* __restrict__ seg_chunk0, const int* __restrict__ nchunks,
                                                        int B, int slots, const int4* __restrict__ st,
                                                        const int* __restrict__ excl, int16_t* __restrict__ coef,
                                                        int* __restrict__ status, int chunk_bits) {
  VTX_PDL_TRIGGER();
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= slots) return;
  ChunkCtx c;
  if (!chunk_ctx(slot, ent, info, info64, seg_start, seg_len, seg_chunk0, nchunks, B, &c)) return;
  const int base = c.inf[VTX_JPEG_I_CHUNK_BASE];
  const int first = base + c.j - c.i;
  const int start = excl[slot] - excl[first];  // blocks of the segment before this chunk's entry
  const int expected = segment_blocks(c.inf, c.s);
  if (start >= expected) return;
  const int ri = c.inf[VTX_JPEG_I_RI];
  const long long blk0 = info64[c.n * VTX_JPEG_N64 + VTX_JPEG_Q_COEF] +
                         (ri > 0 ? (long long)c.s * ri * c.inf[VTX_JPEG_I_BPM] : 0);
  const int4 e = c.i == 0 ? make_int4(0, 0, 0, 0) : st[slot - 1];
  const bool last = c.i == c.nc_seg - 1;
  const int stop = min((c.i + 1) * chunk_bits, c.seglen * 8);
  const Run r = decode_run<true>(c.seg, c.seglen, e.x, e.y, stop, c.inf, (const HuffTab*)huff, start, expected, last,
                                 coef + blk0 * 64);
  int flags = r.err;
  if (!last && !r.err) {
    const int4 mine = st[slot];
    if (mine.x != r.bit || mine.y != r.u || mine.z != r.count) flags |= VTX_JPEG_ST_UNSYNCED;
  }
  if (flags) atomicOr(status + c.n, flags);
}

// ------------------------------------------------------------------------------------------------------- DC scan
struct SegSum {
  int f, v;
};
struct SegSumOp {
  __device__ __forceinline__ SegSum operator()(const SegSum& a, const SegSum& b) const {
    return SegSum{a.f | b.f, b.f ? b.v : a.v + b.v};
  }
};

// One CTA per image; per component, the DC differences in decode order are summed, restarting at each restart interval
// (libjpeg keeps the predictor as int and stores the sum as a 16-bit coefficient).
__global__ void __launch_bounds__(512) jpeg_dc_scan_kernel(const int* __restrict__ info, const long long* __restrict__ info64,
                                                          int16_t* __restrict__ coef) {
  VTX_PDL_TRIGGER();
  constexpr int T = 512, ITEMS = 8;
  typedef cub::BlockScan<SegSum, T> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const int n = blockIdx.x, tid = threadIdx.x;
  const int* inf = info + n * VTX_JPEG_NI;
  int16_t* cf = coef + info64[n * VTX_JPEG_N64 + VTX_JPEG_Q_COEF] * 64;
  const int bpm = inf[VTX_JPEG_I_BPM], ri = inf[VTX_JPEG_I_RI];
  const int nmcu = inf[VTX_JPEG_I_MCUX] * inf[VTX_JPEG_I_MCUY];
  for (int comp = 0; comp < inf[VTX_JPEG_I_NCOMP]; ++comp) {
    const int* ci = inf + VTX_JPEG_I_COMP + 8 * comp;
    const int nb = ci[0] * ci[1], b0 = ci[7];
    const int items = nmcu * nb;
    SegSum carry{0, 0};
    for (int t0 = 0; t0 < items; t0 += T * ITEMS) {
      int g[ITEMS];
      SegSum loc{0, 0};
      SegSum x[ITEMS];
#pragma unroll
      for (int k = 0; k < ITEMS; ++k) {
        const int it = t0 + tid * ITEMS + k;
        g[k] = -1;
        x[k] = SegSum{0, 0};
        if (it < items) {
          const int mcu = it / nb, r = it - mcu * nb;
          g[k] = mcu * bpm + b0 + r;
          x[k] = SegSum{(r == 0 && ri > 0 && mcu % ri == 0) ? 1 : 0, (int)cf[(long long)g[k] * 64]};
        }
        loc = k == 0 ? x[k] : SegSumOp()(loc, x[k]);
      }
      SegSum pre, agg;
      Scan(tmp).ExclusiveScan(loc, pre, SegSum{0, 0}, SegSumOp(), agg);
      SegSum run = SegSumOp()(carry, pre);
#pragma unroll
      for (int k = 0; k < ITEMS; ++k) {
        run = SegSumOp()(run, x[k]);
        if (g[k] >= 0) cf[(long long)g[k] * 64] = (int16_t)run.v;
      }
      carry = SegSumOp()(carry, agg);
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- IDCT
constexpr int CONST_BITS = 13, PASS1_BITS = 2;
constexpr long long F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                    F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

__device__ __forceinline__ long long descale(long long x, int n) { return (x + (1LL << (n - 1))) >> n; }

// 8-point islow butterfly on in[0..7] (stride-free); out[i] = descale(result, shift)
__device__ __forceinline__ void idct8(const long long* in, long long* out, int shift) {
  long long z2 = in[2], z3 = in[6];
  long long z1 = (z2 + z3) * F0541;
  long long tmp2 = z1 + z3 * -F1847;
  long long tmp3 = z1 + z2 * F0765;
  long long tmp0 = (in[0] + in[4]) * (1LL << CONST_BITS);
  long long tmp1 = (in[0] - in[4]) * (1LL << CONST_BITS);
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in[7]; tmp1 = in[5]; tmp2 = in[3]; tmp3 = in[1];
  z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * F1175;
  tmp0 *= F0298; tmp1 *= F2053; tmp2 *= F3072; tmp3 *= F1501;
  z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
  z3 += z5; z4 += z5;
  tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
  out[0] = descale(tmp10 + tmp3, shift); out[7] = descale(tmp10 - tmp3, shift);
  out[1] = descale(tmp11 + tmp2, shift); out[6] = descale(tmp11 - tmp2, shift);
  out[2] = descale(tmp12 + tmp1, shift); out[5] = descale(tmp12 - tmp1, shift);
  out[3] = descale(tmp13 + tmp0, shift); out[4] = descale(tmp13 - tmp0, shift);
}

// libjpeg's post-IDCT range limit: the value wraps modulo 1024 around the centre, then clamps to 0..255
__device__ __forceinline__ uint32_t range_limit(long long x) {
  const int y = (int)((x + 512) & 1023) - 512 + 128;
  return (uint32_t)min(max(y, 0), 255);
}

// one thread per 8x8 block of the batch (block index over every image's coefficient range)
__global__ void __launch_bounds__(128) jpeg_idct_kernel(const int* __restrict__ info, const long long* __restrict__ info64,
                                                       const int16_t* __restrict__ coef, const uint16_t* __restrict__ quant,
                                                       uint8_t* __restrict__ planes, int B, long long nblocks) {
  VTX_PDL_TRIGGER();
  const long long G = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (G >= nblocks) return;
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (info64[mid * VTX_JPEG_N64 + VTX_JPEG_Q_COEF] <= G) lo = mid; else hi = mid - 1;
  }
  const int n = lo;
  const int* inf = info + n * VTX_JPEG_NI;
  const long long* q64 = info64 + n * VTX_JPEG_N64;
  const long long g = G - q64[VTX_JPEG_Q_COEF];
  const int bpm = inf[VTX_JPEG_I_BPM];
  if (g >= (long long)inf[VTX_JPEG_I_MCUX] * inf[VTX_JPEG_I_MCUY] * bpm) return;  // padding between images
  const int mcu = (int)(g / bpm), bb = (int)(g - (long long)mcu * bpm);
  const int n0 = inf[VTX_JPEG_I_COMP] * inf[VTX_JPEG_I_COMP + 1];
  const int comp = bb < n0 ? 0 : bb - n0 + 1;
  const int* ci = inf + VTX_JPEG_I_COMP + 8 * comp;
  const int h = ci[0], v = ci[1], t = bb - ci[7];
  const int mx = mcu % inf[VTX_JPEG_I_MCUX], my = mcu / inf[VTX_JPEG_I_MCUX];
  const int bx = mx * h + t % h, by = my * v + t / h;
  const int pw = ci[5] * 8;
  const uint16_t* qt = quant + ci[2] * 64;
  const int16_t* c = coef + G * 64;
  long long ws[64];
  for (int col = 0; col < 8; ++col) {
    long long in[8], out[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) in[r] = (long long)c[r * 8 + col] * qt[r * 8 + col];
    idct8(in, out, CONST_BITS - PASS1_BITS);
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[r * 8 + col] = (int)out[r];  // libjpeg's workspace is int
  }
  uint8_t* dst = planes + q64[VTX_JPEG_Q_PLANE + comp] + (long long)by * 8 * pw + bx * 8;
  for (int r = 0; r < 8; ++r) {
    long long out[8];
    idct8(ws + r * 8, out, CONST_BITS + PASS1_BITS + 3);
    uint32_t lo4 = 0, hi4 = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      lo4 |= range_limit(out[k]) << (8 * k);
      hi4 |= range_limit(out[k + 4]) << (8 * k);
    }
    *reinterpret_cast<uint2*>(dst + (long long)r * pw) = make_uint2(lo4, hi4);
  }
}

// --------------------------------------------------------------------------------------------------------- colour
__device__ __forceinline__ int px(const uint8_t* p, int pw, int y, int x) { return p[(long long)y * pw + x]; }

// chroma sample at full-resolution (y, x): libjpeg-turbo's h2v1 / h1v2 / h2v2 triangle filters (box replication when
// the chroma plane is at most 2 samples wide), edges replicated from the component's real width / height
__device__ __forceinline__ int chroma(const uint8_t* p, int pw, int h0, int v0, int cw, int ch, int y, int x) {
  if (h0 == 1 && v0 == 1) return px(p, pw, y, x);
  if (h0 == 2 && v0 == 1) {
    const int c = x >> 1;
    if (cw <= 2) return px(p, pw, y, c);
    if (x & 1) return (3 * px(p, pw, y, c) + px(p, pw, y, min(c + 1, cw - 1)) + 2) >> 2;
    return (3 * px(p, pw, y, c) + px(p, pw, y, max(c - 1, 0)) + 1) >> 2;
  }
  if (h0 == 1) {  // h1v2
    const int r = y >> 1;
    if (y & 1) return (3 * px(p, pw, r, x) + px(p, pw, min(r + 1, ch - 1), x) + 2) >> 2;
    return (3 * px(p, pw, r, x) + px(p, pw, max(r - 1, 0), x) + 1) >> 2;
  }
  const int r = y >> 1, c = x >> 1;
  if (cw <= 2) return px(p, pw, r, c);
  const int r2 = (y & 1) ? min(r + 1, ch - 1) : max(r - 1, 0);
  const int c2 = (x & 1) ? min(c + 1, cw - 1) : max(c - 1, 0);
  const int s1 = 3 * px(p, pw, r, c) + px(p, pw, r2, c);
  const int s2 = 3 * px(p, pw, r, c2) + px(p, pw, r2, c2);
  return (x & 1) ? (3 * s1 + s2 + 7) >> 4 : (3 * s1 + s2 + 8) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_color_kernel(const int* __restrict__ info, const long long* __restrict__ info64,
                                                        const uint8_t* __restrict__ planes, uint8_t* __restrict__ out) {
  VTX_PDL_TRIGGER();
  const int n = blockIdx.y;
  const int* inf = info + n * VTX_JPEG_NI;
  const long long* q64 = info64 + n * VTX_JPEG_N64;
  const int H = inf[VTX_JPEG_I_H], W = inf[VTX_JPEG_I_W], OH = inf[VTX_JPEG_I_OH], OW = inf[VTX_JPEG_I_OW];
  const int orient = inf[VTX_JPEG_I_ORIENT], ncomp = inf[VTX_JPEG_I_NCOMP];
  const int h0 = inf[VTX_JPEG_I_COMP], v0 = inf[VTX_JPEG_I_COMP + 1];
  const int pw0 = inf[VTX_JPEG_I_COMP + 5] * 8, pwc = inf[VTX_JPEG_I_COMP + 8 + 5] * 8;
  const int cw = (W + h0 - 1) / h0, ch = (H + v0 - 1) / v0;
  const uint8_t* p0 = planes + q64[VTX_JPEG_Q_PLANE];
  const uint8_t* p1 = planes + q64[VTX_JPEG_Q_PLANE + 1];
  const uint8_t* p2 = planes + q64[VTX_JPEG_Q_PLANE + 2];
  uint8_t* o = out + q64[VTX_JPEG_Q_OUT];
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < (long long)OH * OW;
       p += (long long)gridDim.x * blockDim.x) {
    const int oy = (int)(p / OW), ox = (int)(p - (long long)oy * OW);
    int y, x;  // EXIF orientation as OpenCV applies it (flip / transpose of the decoded image)
    switch (orient) {
      case 2: y = oy; x = W - 1 - ox; break;
      case 3: y = H - 1 - oy; x = W - 1 - ox; break;
      case 4: y = H - 1 - oy; x = ox; break;
      case 5: y = ox; x = oy; break;
      case 6: y = H - 1 - ox; x = oy; break;
      case 7: y = H - 1 - ox; x = W - 1 - oy; break;
      case 8: y = ox; x = W - 1 - oy; break;
      default: y = oy; x = ox; break;
    }
    const int Y = px(p0, pw0, y, x);
    int R = Y, G = Y, Bc = Y;
    if (ncomp == 3) {
      const int cb = chroma(p1, pwc, h0, v0, cw, ch, y, x) - 128;
      const int cr = chroma(p2, pwc, h0, v0, cw, ch, y, x) - 128;
      R = Y + ((91881 * cr + 32768) >> 16);
      G = Y + ((-46802 * cr + (-22554 * cb + 32768)) >> 16);
      Bc = Y + ((116130 * cb + 32768) >> 16);
      R = min(max(R, 0), 255); G = min(max(G, 0), 255); Bc = min(max(Bc, 0), 255);
    }
    uint8_t* d = o + p * 3;
    d[0] = (uint8_t)R; d[1] = (uint8_t)G; d[2] = (uint8_t)Bc;
  }
}

}  // namespace jpg
}  // namespace vtx

using namespace vtx;
using namespace vtx::jpg;
#define STREAM reinterpret_cast<cudaStream_t>(stream)

static bool chunk_bits_ok(int cb) { return cb >= 64 && cb % 8 == 0 && cb <= (1 << 20); }

extern "C" int vtx_jpeg_unstuff(const uint8_t* src, const int32_t* info, const int64_t* info64, int B, uint8_t* ent,
                                int32_t* seg_start, int32_t* seg_len, int32_t* seg_chunk0, int32_t* nchunks,
                                int32_t* status, int chunk_bits, void* stream) {
  if (!src || !info || !info64 || !ent || !seg_start || !seg_len || !seg_chunk0 || !nchunks || !status || B <= 0 ||
      !chunk_bits_ok(chunk_bits))
    return set_error(VTX_EINVAL, "vtx_jpeg_unstuff: bad arguments");
  jpeg_unstuff_kernel<<<B, 256, 0, STREAM>>>(src, info, (const long long*)info64, ent, seg_start, seg_len, seg_chunk0,
                                             nchunks, status, chunk_bits);
  return check_launch("jpeg_unstuff");
}

extern "C" int vtx_jpeg_sync(const uint8_t* ent, const int32_t* info, const int64_t* info64, const void* huff,
                             const int32_t* seg_start, const int32_t* seg_len, const int32_t* seg_chunk0,
                             const int32_t* nchunks, int B, int slots, const void* st_in, void* st_out, int round,
                             int32_t* rounds, int chunk_bits, void* stream) {
  if (!ent || !info || !info64 || !huff || !seg_start || !seg_len || !seg_chunk0 || !nchunks || !st_out || !rounds ||
      B <= 0 || slots <= 0 || round < 0 || (round > 0 && !st_in) || !chunk_bits_ok(chunk_bits))
    return set_error(VTX_EINVAL, "vtx_jpeg_sync: bad arguments");
  jpeg_sync_kernel<<<(slots + 127) / 128, 128, 0, STREAM>>>(ent, info, (const long long*)info64, huff, seg_start, seg_len,
                                                            seg_chunk0, nchunks, B, slots, (const int4*)st_in,
                                                            (int4*)st_out, round, rounds, chunk_bits);
  return check_launch("jpeg_sync");
}

extern "C" int vtx_jpeg_count_scan(const int32_t* info, const int32_t* nchunks, const void* st, int32_t* excl, int B,
                                   void* stream) {
  if (!info || !nchunks || !st || !excl || B <= 0) return set_error(VTX_EINVAL, "vtx_jpeg_count_scan: bad arguments");
  jpeg_count_scan_kernel<<<B, 256, 0, STREAM>>>(info, nchunks, (const int4*)st, excl);
  return check_launch("jpeg_count_scan");
}

extern "C" int vtx_jpeg_coefs(const uint8_t* ent, const int32_t* info, const int64_t* info64, const void* huff,
                              const int32_t* seg_start, const int32_t* seg_len, const int32_t* seg_chunk0,
                              const int32_t* nchunks, int B, int slots, const void* st, const int32_t* excl,
                              int16_t* coef, int32_t* status, int chunk_bits, void* stream) {
  if (!ent || !info || !info64 || !huff || !seg_start || !seg_len || !seg_chunk0 || !nchunks || !st || !excl || !coef ||
      !status || B <= 0 || slots <= 0 || !chunk_bits_ok(chunk_bits))
    return set_error(VTX_EINVAL, "vtx_jpeg_coefs: bad arguments");
  jpeg_coefs_kernel<<<(slots + 127) / 128, 128, 0, STREAM>>>(ent, info, (const long long*)info64, huff, seg_start, seg_len,
                                                             seg_chunk0, nchunks, B, slots, (const int4*)st, excl, coef,
                                                             status, chunk_bits);
  return check_launch("jpeg_coefs");
}

extern "C" int vtx_jpeg_dc_scan(const int32_t* info, const int64_t* info64, int16_t* coef, int B, void* stream) {
  if (!info || !info64 || !coef || B <= 0) return set_error(VTX_EINVAL, "vtx_jpeg_dc_scan: bad arguments");
  jpeg_dc_scan_kernel<<<B, 512, 0, STREAM>>>(info, (const long long*)info64, coef);
  return check_launch("jpeg_dc_scan");
}

extern "C" int vtx_jpeg_idct(const int32_t* info, const int64_t* info64, const int16_t* coef, const uint16_t* quant,
                             uint8_t* planes, int B, int64_t nblocks, void* stream) {
  if (!info || !info64 || !coef || !quant || !planes || B <= 0 || nblocks <= 0)
    return set_error(VTX_EINVAL, "vtx_jpeg_idct: bad arguments");
  jpeg_idct_kernel<<<(unsigned)((nblocks + 127) / 128), 128, 0, STREAM>>>(info, (const long long*)info64, coef, quant,
                                                                          planes, B, (long long)nblocks);
  return check_launch("jpeg_idct");
}

extern "C" int vtx_jpeg_color(const int32_t* info, const int64_t* info64, const uint8_t* planes, uint8_t* out, int B,
                              int64_t max_pixels, void* stream) {
  if (!info || !info64 || !planes || !out || B <= 0 || max_pixels <= 0)
    return set_error(VTX_EINVAL, "vtx_jpeg_color: bad arguments");
  const int bx = (int)min((max_pixels + 255) / 256, (int64_t)1024);
  jpeg_color_kernel<<<dim3(bx, B), 256, 0, STREAM>>>(info, (const long long*)info64, planes, out);
  return check_launch("jpeg_color");
}
