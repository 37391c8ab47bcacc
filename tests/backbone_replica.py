"""Float64 replicas of the rounding points of the backbone's memory-bound kernels (virtex_b200/csrc/backbone.cu).

Every function takes and returns torch float64 tensors (on any device) whose values are fp32 or bf16 numbers, and
rounds where the kernel rounds, so that a kernel's output can be compared with its replica bit for bit.

What the sm_90a build does (default -fmad=true, no fast math; read from `cuobjdump -sass` of the built object):
  * bn_act_kernel (all four instantiations), bn_relu_maxpool_rows_kernel, bn_relu_maxpool_kernel and the
    mask-from-y test of bn_bwd_apply_kernel / bn_bwd_reduce_kernel evaluate y*scale + shift as ONE FFMA, e.g.
        FFMA R62, R79, R62, R78           (bn_act_kernel<false, 8>, then FSETP.GT / FMNMX RZ for the ReLU)
        FFMA R33, R6, R33, R15 ; FMNMX R44, RZ, R33, !PT ; F2F.BF16.F32 R49, R49   (bn_relu_maxpool_rows_kernel)
        FFMA R60, R14, R56, R23 ; FSETP.GT.AND P2, PT, R60, RZ, PT                  (bn_bwd_apply_kernel<0, false, 4>)
    and the residual operand of bn_act_kernel as a second FFMA (res * scale_r + shift_r) followed by one FADD;
  * bn_finalize_kernel and the fold prologue of bn_act_kernel<true, *> compute
        mean = s / count, q = sumsq / count       (IEEE divisions)
        var = max(fma(-mean, mean, q), 0)          (FFMA R3, -R8, R8, R3 ; FMNMX R12, RZ, R3)
        invstd = rsqrtf(var + eps)                 (MUFU.RSQ: not correctly rounded, 2 ulp)
        scale = gamma * invstd ; shift = fma(scale, -mean, beta)
        running_mean = fma(mean, momentum, running_mean * (1 - momentum))
        running_var = fma(1 - momentum, running_var, (var * momentum) * (count / max(count - 1, 1)))

A bf16 value has 8 significant bits and an fp32 value 24, so a bf16 x fp32 product (32 bits) and an fp32 x fp32
product (48 bits) are exact in float64.  The sum that completes the FFMA is rounded to float64 first; rounding that
again to fp32 is wrong only where the float64 sum lands exactly on the midpoint of two fp32 values while the exact sum
does not.  fma_f32 detects that case with the error term of the float64 addition (TwoSum) and rounds it the way the
exact sum rounds, so its result is the correctly rounded fma for every input.  Sums and quotients of two fp32 values
need no such care: double rounding through float64 (53 >= 2 * 24 + 2 bits) is innocuous for them.

Comparisons treat +0 and -0 as equal: the kernels' fmaxf(v, 0) may keep either sign of a zero.
"""
import torch

F32, F64 = torch.float32, torch.float64
U = 2.0 ** -24  # unit roundoff of fp32


def ulp_bf16(x):
    """Spacing of bf16 numbers at |x| (the smallest normal spacing below 2^-126)."""
    e = torch.floor(torch.log2(x.abs())).clamp_min(-126)
    return torch.exp2(e - 7)


def f32(x):
    """Round float64 values to the nearest fp32 value (ties to even); float64 out."""
    return x.to(F32).to(F64)


def bf16(x):
    """fp32 values (in a float64 tensor) -> the nearest bf16 value, ties to even; float64 out.  Finite inputs only."""
    b = x.to(F32).view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    r = torch.where(r >= 1 << 31, r - (1 << 32), r)
    return r.to(torch.int32).view(F32).to(F64)


def fma_f32(a, b, c):
    """fp32 fma(a, b, c) rounded once, for a * b exact in float64 (bf16 x fp32 or fp32 x fp32 operands)."""
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)  # exact (p + c) - s
    r = f32(s)
    other = 2 * s - r  # when s is an fp32 midpoint: the fp32 neighbour on the other side of it
    tie = (e != 0) & (s != r) & (f32(other) == other)
    if bool(tie.any()):
        toward = torch.where(e > 0, torch.full_like(s, float("inf")), torch.full_like(s, float("-inf")))
        r = torch.where(tie, f32(torch.nextafter(s, toward)), r)
    return r


def bn_act(y, scale, shift, res=None, scale_r=None, shift_r=None, relu=True):
    """vtx_bn_act on [M, C] bf16 values with the fp32 [C] rows of bnp: returns (pre-activation fp32, bf16 output).
    The ReLU bit mask is pack_mask(pre > 0)."""
    pre = fma_f32(y, scale, shift)
    if res is not None:
        t = res if scale_r is None else fma_f32(res, scale_r, shift_r)
        pre = f32(pre + t)
    out = bf16(pre.clamp_min(0.0) if relu else pre)
    return pre, out


def pack_mask(keep):
    """[M, C] bool -> uint8 [M, C/8]: bit j of byte (m, g) = keep[m, 8g + j] (the layout vtx_bn_act writes)."""
    M, C = keep.shape
    w = (1 << torch.arange(8, device=keep.device, dtype=torch.int32))
    return (keep.reshape(M, C // 8, 8).to(torch.int32) * w).sum(-1).to(torch.uint8)


def unpack_mask(bits, C):
    """uint8 [M, C/8] -> [M, C] bool, the inverse of pack_mask."""
    M = bits.shape[0]
    sh = torch.arange(8, device=bits.device, dtype=torch.int32)
    return ((bits.to(torch.int32).unsqueeze(-1) >> sh) & 1).reshape(M, C).bool()


def pool_extent(H, W):
    """Output extent of the 3x3 / stride 2 / pad 1 max pool."""
    return (H - 1) // 2 + 1, (W - 1) // 2 + 1


def maxpool_fwd(act):
    """3x3 / stride 2 / pad 1 max pool of NHWC act [N, H, W, C] (the bf16-rounded post-ReLU values): (out, idx) with
    idx = kh * 3 + kw of the FIRST maximum in (kh, kw) order under strict `>` (ATen's rule); taps outside the image
    are skipped."""
    N, H, W, C = act.shape
    Ho, Wo = pool_extent(H, W)
    x = act.new_full((N, H + 2, W + 2, C), float("-inf"))
    x[:, 1:H + 1, 1:W + 1] = act
    best = act.new_full((N, Ho, Wo, C), float("-inf"))
    idx = torch.zeros(N, Ho, Wo, C, dtype=torch.uint8, device=act.device)
    for kh in range(3):
        for kw in range(3):
            v = x[:, kh:kh + 2 * Ho - 1:2, kw:kw + 2 * Wo - 1:2]
            upd = v > best
            best = torch.where(upd, v, best)
            idx = torch.where(upd, torch.full_like(idx, kh * 3 + kw), idx)
    return best, idx


def maxpool_bwd(dpool, idx, H, W):
    """da [N, H, W, C] = sum of dpool over the pooled windows whose slot `idx` points at (h, w), in float64 (exact when
    the terms are multiples of 2^-6 bounded by 1: the caller rounds it as the kernel does, bf16(f32(.)))."""
    N, Ho, Wo, C = dpool.shape
    da = dpool.new_zeros(N, H + 2, W + 2, C)
    for kh in range(3):
        for kw in range(3):
            da[:, kh:kh + 2 * Ho - 1:2, kw:kw + 2 * Wo - 1:2] += torch.where(idx == kh * 3 + kw, dpool, 0.0)
    return da[:, 1:H + 1, 1:W + 1]


def bn_finalize(stats, count, gamma, beta, rmean, rvar, momentum, eps, training):
    """vtx_bn_finalize up to rsqrtf: returns mean, var (fp32 values, exact replicas), invstd_ref = float64 1/sqrt of the
    fp32 var + eps, and the updated running buffers (the inputs unchanged in eval mode).  stats is [2, C] in training."""
    m = f32(torch.tensor(momentum, dtype=F64))
    e = f32(torch.tensor(eps, dtype=F64))
    if training:
        n = f32(torch.tensor(float(count), dtype=F64))
        mean = f32(stats[0] / n)
        q = f32(stats[1] / n)
        var = fma_f32(-mean, mean, q).clamp_min(0.0)
        one_m = f32(1.0 - m)
        rmean = fma_f32(mean, m, f32(rmean * one_m))
        unbiased = f32(n / f32(n - 1.0).clamp_min(1.0))
        rvar = fma_f32(one_m, rvar, f32(f32(var * m) * unbiased))
    else:
        mean, var = rmean, rvar
    invstd_ref = 1.0 / torch.sqrt(f32(var + e))
    return mean, var, invstd_ref, rmean, rvar


def bn_scale_shift(gamma, beta, mean, invstd):
    """Rows 2 and 3 of bnp from the device's own invstd: scale = gamma * invstd, shift = fma(scale, -mean, beta)."""
    sc = f32(gamma * invstd)
    return sc, fma_f32(sc, -mean, beta)


def reduce_depth(sms, M, C, two):
    """Sequential depth of vtx_bn_bwd_reduce's fp32 accumulation (mirrors its launch geometry): terms per thread + rows
    reduced per CTA + atomics per channel."""
    rows_par = 256 // (C // 8)
    ku = 4 if two else 5
    blocks = min(-(-M // (rows_par * ku)), sms * (1 if two else 2))
    return -(-M // (rows_par * blocks)) + rows_par + blocks


def bn_bwd_sums(dz, y, bnp, depth):
    """BN-backward sums [sum_m dz, sum_m dz * (y - mean) * invstd] of [M, C] dz (float64) and bf16 y with the device's
    fp32 bnp, in float64, and their bound (depth + 3) * 2^-24 * sum |term| for an fp32 accumulation of sequential depth
    `depth` (the 3 for the rounding of each term).  dgamma += sums[1], dbeta += sums[0]."""
    t = dz * (y.to(F64) - bnp[0].to(F64)) * bnp[1].to(F64)
    ref = torch.stack([dz.sum(0), t.sum(0)])
    tol = (depth + 3) * U * torch.stack([dz.abs().sum(0), t.abs().sum(0)]) + 1e-30
    return ref, tol


def bn_bwd_dy(dz, y, bnp, sums, M):
    """Train-mode BN backward dy = k0 * dz + k1 * y + k2 of [M, C] dz (float64) and y with the device's bnp and sums
    (k0 = scale, k1 = -scale * m2 * invstd, k2 = scale * (m2 * invstd * mean - m1), m1 / m2 = sums / M), and its
    bound: 1 bf16 ulp plus 2^-21 * (|k0 dz| + |k1 y| + |scale| * (|m2 invstd mean| + |m1|)) for the fp32 coefficients
    (k2 cancels when |mean| is large) and their evaluation."""
    yd = y.to(F64)
    scl, mean, istd = bnp[2].to(F64), bnp[0].to(F64), bnp[1].to(F64)
    m1, m2 = sums[0].to(F64) / M, sums[1].to(F64) / M
    k0, k1, k2 = scl, -scl * m2 * istd, scl * (m2 * istd * mean - m1)
    ref = k0 * dz + k1 * yd + k2
    floor = 2.0 ** -21 * ((k0 * dz).abs() + (k1 * yd).abs() + scl.abs() * ((m2 * istd * mean).abs() + m1.abs()))
    return ref, ulp_bf16(ref) + floor
