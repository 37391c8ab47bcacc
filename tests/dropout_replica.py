"""Host replica of the dropout RNG of the head kernels (hash_u64 / drop4 in virtex_b200/csrc/vtx_common.cuh).

The kernels never store a dropout mask: every kernel that applies one (forward and backward) recomputes it from
(step seed, dropout site, element index).  This module restates that function in numpy so that tests can compare a
kernel at p > 0 with a float64 reference fed the very same mask.

  * one 64-bit hash of (seed, site, element index // 4) serves 4 consecutive elements, 16 bits each (element e uses
    bits [16 * (e % 4), 16 * (e % 4) + 16));
  * an element is dropped iff its 16-bit slice < thr, thr = (uint32)(p_f32 * 65536.f + 0.5f), computed from the
    float32 value of p; kept elements are scaled by the float32 1 / (1 - p);
  * p <= 0 keeps everything with scale 1 (the kernels do not hash at all then).

Element-index layout of each site (what the kernels hash, see head.cu):
  * vtx_embed_fwd / _bwd, vtx_add_ln_fwd, vtx_ln_bwd: row * H + col of the [M, H] tensor;
  * vtx_gelu_dropout_fwd / _bwd: the flat index into the [M, F] tensor;
  * vtx_attn_fwd / _bwd: ((b * heads + h) * 32 + i) * 64 + j for query i and key j, whatever Tq and Tk are.
"""
import numpy as np

MASK64 = (1 << 64) - 1
_K1 = 0x9E3779B97F4A7C15
_K2 = 0xD6E8FEB86659FD93


def as_u64(seed):
    """Python int (negative: an int64's two's complement) -> the uint64 the device reads."""
    return int(seed) & MASK64


def as_i64(seed):
    """The int64 value whose bytes are the uint64 `seed` (how an int64 seed tensor carries seeds >= 2^63)."""
    s = as_u64(seed)
    return s - (1 << 64) if s >= 1 << 63 else s


def threshold(p):
    """Drop threshold on the 16-bit slices: (uint32)(p * 65536.f + 0.5f) in float32 arithmetic."""
    pf = np.float32(p)
    if not pf > 0:
        return 0
    return int(np.float32(pf * np.float32(65536.0)) + np.float32(0.5))


def inv_keep(p):
    """Scale of a kept element, 1.f / (1.f - p) in float32 (1 when p <= 0)."""
    pf = np.float32(p)
    if not pf > 0:
        return np.float32(1.0)
    return np.float32(np.float32(1.0) / (np.float32(1.0) - pf))


def hash_u64(seed, site, ctr):
    """Vectorised hash_u64 over an array of group counters `ctr` (element index // 4); uint64 array out."""
    base = as_u64(seed) ^ ((_K1 * ((int(site) + 1) & 0xFFFFFFFF)) & MASK64)   # Python ints: no overflow warnings
    with np.errstate(over="ignore"):
        x = np.uint64(base) ^ (np.asarray(ctr, dtype=np.uint64) * np.uint64(_K2))
        x ^= x >> np.uint64(32)
        x *= np.uint64(_K2)
        x ^= x >> np.uint64(32)
        x *= np.uint64(_K2)
        x ^= x >> np.uint64(32)
    return x


def keep_scale(seed, site, idx, p):
    """float32 array of the dropout scale (0 or 1/(1-p)) of every element index in `idx` (any integer array)."""
    idx = np.asarray(idx, dtype=np.uint64)
    thr = threshold(p)
    if thr == 0:
        return np.ones(idx.shape, dtype=np.float32)
    h = hash_u64(seed, site, idx >> np.uint64(2))
    bits = (h >> ((idx & np.uint64(3)) * np.uint64(16))) & np.uint64(0xFFFF)
    return np.where(bits < np.uint64(thr), np.float32(0.0), inv_keep(p)).astype(np.float32)


def flat_scale(seed, site, shape, p):
    """Scale of every element of a row-major tensor of `shape` whose element index is its flat index (embedding,
    residual and GELU sites)."""
    n = int(np.prod(shape))
    return keep_scale(seed, site, np.arange(n, dtype=np.uint64), p).reshape(shape)


def attn_index(B, heads, Tq, Tk):
    """[B, heads, Tq, Tk] element indices of the attention-probability site."""
    b = np.arange(B, dtype=np.uint64)[:, None, None, None]
    h = np.arange(heads, dtype=np.uint64)[None, :, None, None]
    i = np.arange(Tq, dtype=np.uint64)[None, None, :, None]
    j = np.arange(Tk, dtype=np.uint64)[None, None, None, :]
    return ((b * np.uint64(heads) + h) * np.uint64(32) + i) * np.uint64(64) + j


def attn_scale(seed, site, B, heads, Tq, Tk, p):
    """[B, heads, Tq, Tk] scale of the attention probabilities (query i, key j)."""
    return keep_scale(seed, site, attn_index(B, heads, Tq, Tk), p)


def keep_scale_scalar(seed, site, idx, p):
    """The same function for one element, in plain Python integers (the unvectorised statement of the kernel code)."""
    thr = threshold(p)
    if thr == 0:
        return 1.0
    x = as_u64(seed) ^ ((_K1 * ((site + 1) & 0xFFFFFFFF)) & MASK64) ^ (((idx >> 2) * _K2) & MASK64)
    for _ in range(2):
        x ^= x >> 32
        x = (x * _K2) & MASK64
    x ^= x >> 32
    return 0.0 if ((x >> (16 * (idx & 3))) & 0xFFFF) < thr else float(inv_keep(p))
