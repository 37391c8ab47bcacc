"""Float64 references of the backbone's stages, one function per stage, each a function of tensors the engine produced
(tests/test_backbone_stages_gpu.py) or of exact float64 values (tests/test_backbone_stages_cpu.py, against autograd).

Activations are NHWC float64 tensors [N, H, W, C]; weights OIHW float64 [O, C, kh, kw] (on the GPU: the modules'
parameters rounded to bf16 by torch, never the engine's mirror or packed layouts).  A GEMM-like stage returns the
reference and sum_k |a_k b_k| of each element (`mag`); a bound is built from them by the rules of tests/gemm_reference.py:

  * bf16 output of a K-long reduction: E + ulp_bf16(|ref| + E), E = (L + 2) * 2^-22 * mag, L = ceil(K / 16) wgmma
    steps + 1 (one split), plus one ulp_bf16 of every intermediate the kernel rounds to bf16 on the way (the
    pre-residual tile of a TMA-staged residual, a GEMM output accumulated onto in place);
  * fp32 weight gradient: (L + 2) * 2^-22 * mag, L the sequential depth of the launch (gemm_reference.seq_depth);
  * BN backward: tests/backbone_replica.bn_bwd_dy and bn_bwd_sums (the bounds of test_backbone_kernels_gpu.py);
  * BN apply, ReLU bit mask, max pool: bit-exact through the replicas of tests/backbone_replica.py.

`exact=True` replaces each replica by plain float64 arithmetic: chained that way, the stages reproduce float64 autograd
of torchvision's Bottleneck, of its BasicBlock and of the stem.
"""
import math

import torch
import torch.nn.functional as F

from tests import backbone_replica as R

F64 = torch.float64
STEP = 2.0 ** -22   # per sequential fp32 step of a tensor-core accumulation (tests/gemm_reference.py)
EPS, MOM = 1e-5, 0.1
_CHUNK = 1 << 25    # float64 elements per image chunk of a weight-gradient reference


# ------------------------------------------------------------------------------------------------ convolutions
def out_extent(H, W, k, stride, pad):
    return (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1


def _tap(xp, a, b, s, Ho, Wo):
    return xp[:, a:a + s * (Ho - 1) + 1:s, b:b + s * (Wo - 1) + 1:s]


def conv(x, w, stride, pad):
    """Forward conv of NHWC x: (y [N, Ho, Wo, O], mag), a sum over taps of float64 matmuls."""
    N, H, W, C = x.shape
    O, _, kh, kw = w.shape
    Ho, Wo = out_extent(H, W, kh, stride, pad)
    xp = F.pad(x, (0, 0, pad, pad, pad, pad))
    y = x.new_zeros(N * Ho * Wo, O)
    mag = x.new_zeros(N * Ho * Wo, O)
    for a in range(kh):
        for b in range(kw):
            v = _tap(xp, a, b, stride, Ho, Wo).reshape(-1, C)
            wt = w[:, :, a, b].t()
            y += v @ wt
            mag += v.abs() @ wt.abs()
    return y.view(N, Ho, Wo, O), mag.view(N, Ho, Wo, O)


def conv_dgrad(dy, w, stride, pad, H, W):
    """Input gradient [N, H, W, C] of a conv with output gradient dy [N, Ho, Wo, O], at the real input extent H x W
    (odd extents included), and its mag."""
    N, Ho, Wo, O = dy.shape
    _, C, kh, kw = w.shape
    Hp, Wp = max(H + 2 * pad, kh + stride * (Ho - 1)), max(W + 2 * pad, kw + stride * (Wo - 1))
    dx = dy.new_zeros(N, Hp, Wp, C)
    mag = dy.new_zeros(N, Hp, Wp, C)
    d, da = dy.reshape(-1, O), dy.reshape(-1, O).abs()
    for a in range(kh):
        for b in range(kw):
            wt = w[:, :, a, b]
            _tap(dx, a, b, stride, Ho, Wo).add_((d @ wt).view(N, Ho, Wo, C))
            _tap(mag, a, b, stride, Ho, Wo).add_((da @ wt.abs()).view(N, Ho, Wo, C))
    return dx[:, pad:pad + H, pad:pad + W], mag[:, pad:pad + H, pad:pad + W]


def conv_wgrad(dy, x, kh, kw, stride, pad):
    """Weight gradient [O, C, kh, kw] of a conv of NHWC x with output gradient dy, and its mag, over all images."""
    N, H, W, C = x.shape
    O = dy.shape[-1]
    Ho, Wo = dy.shape[1], dy.shape[2]
    g = x.new_zeros(O, C, kh, kw)
    mag = x.new_zeros(O, C, kh, kw)
    step = max(1, _CHUNK // ((H + 2 * pad) * (W + 2 * pad) * C + Ho * Wo * O))
    for n0 in range(0, N, step):
        xp = F.pad(x[n0:n0 + step], (0, 0, pad, pad, pad, pad))
        d = dy[n0:n0 + step].reshape(-1, O).t()
        da = d.abs()
        for a in range(kh):
            for b in range(kw):
                v = _tap(xp, a, b, stride, Ho, Wo).reshape(-1, C)
                g[:, :, a, b] += d @ v
                mag[:, :, a, b] += da @ v.abs()
    return g, mag


# ------------------------------------------------------------------------------------------------ bounds
def gemm_err(mag, K, scale=None, shift=None):
    """E of a bf16-output GEMM of reduction length K (one split), with a folded per-column scale / shift."""
    if scale is not None:
        mag = mag * scale.abs() + shift.abs()
    return (4 * math.ceil(K / 64) + 1 + 2) * STEP * mag


def bf16_bound(ref, E, *rounded):
    """E + ulp_bf16(|ref| + E), plus one ulp_bf16 of each intermediate the kernel rounds to bf16."""
    b = E + R.ulp_bf16(ref.abs() + E)
    for t in rounded:
        b = b + R.ulp_bf16(t.abs() + E)
    return b


def wgrad_bound(mag, depth):
    return (depth + 2) * STEP * mag


# ------------------------------------------------------------------------------------------------ BatchNorm forward
def bn_params(y, gamma, beta):
    """Exact float64 train-mode bnp [4, C] = (mean, invstd, scale, shift) of [M, C] y (biased variance)."""
    mean = y.mean(0)
    invstd = 1.0 / torch.sqrt(((y - mean) ** 2).mean(0) + EPS)
    scale = gamma * invstd
    return torch.stack([mean, invstd, scale, beta - scale * mean])


def bn_train(stats, M, gamma, beta, rmean, rvar):
    """The device's train-mode bnp and running buffers from its own [2, C] statistics: (mean, invstd_ref, rmean,
    rvar), mean and the buffers bit-exact, invstd_ref the float64 1 / sqrt of the fp32 var + eps (rsqrtf: 2 ulp)."""
    mean, _, inv, rm, rv = R.bn_finalize(stats, M, gamma, beta, rmean, rvar, MOM, EPS, True)
    return mean, inv, rm, rv


def bn_eval(gamma, beta, rmean, rvar):
    """The eval-mode bnp from the running buffers: (mean, invstd_ref)."""
    _, _, inv, _, _ = R.bn_finalize(None, 0, gamma, beta, rmean, rvar, MOM, EPS, False)
    return rmean, inv


def bn_apply(y, bnp, res=None, bnp_res=None, relu=True, exact=False):
    """BN + (shortcut, itself through its BN when bnp_res) + ReLU of [M, C] y: (pre-activation, output).  The block's
    ReLU bit mask is pack_mask(pre > 0)."""
    if exact:
        pre = y * bnp[2] + bnp[3]
        if res is not None:
            pre = pre + (res if bnp_res is None else res * bnp_res[2] + bnp_res[3])
        return pre, (pre.clamp_min(0.0) if relu else pre)
    kw = {}
    if bnp_res is not None:
        kw = dict(scale_r=bnp_res[2], shift_r=bnp_res[3])
    return R.bn_act(y, bnp[2], bnp[3], res=res, relu=relu, **kw)


def relu_keep(y, bnp, exact=False):
    """Open ReLUs of BN(y) recomputed from y (the mask_from_y test: one fp32 fma)."""
    return (y * bnp[2] + bnp[3] if exact else R.fma_f32(y, bnp[2], bnp[3])) > 0


def maxpool(act):
    """Max pool of the post-ReLU stem activation [N, H, W, 64]: (values, slots)."""
    return R.maxpool_fwd(act)


# ------------------------------------------------------------------------------------------------ backward
def bn_backward(dA, keep, y, bnp, sums, M):
    """ReLU (keep: [M, C] bool, or None) + train-mode BN backward of [M, C] dA with the given [2, C] sums:
    (dz, dy reference, its bound)."""
    dz = dA if keep is None else dA * keep
    dy, tol = R.bn_bwd_dy(dz, y, bnp, sums, M)
    return dz, dy, tol


def bn_sums(dz, y, bnp, depth=0):
    """(sum dz, sum dz * xhat) = (dbeta, dgamma) of one BN, and its bound for an fp32 accumulation of `depth`."""
    return R.bn_bwd_sums(dz, y, bnp, depth)


def block_dx(dy1, w1, H, W, dOut=None, keep3=None, dyd=None, wd=None, stride=1):
    """Outgoing gradient [N, H, W, Cin] of a bottleneck and its bound: dy1 . W1 plus the shortcut term, dOut * keep3
    for an identity block (added to the bf16-rounded conv1 dgrad tile), dyd . Wd at the stride positions for a
    transition block (accumulated in place onto the stored conv1 dgrad, itself rounded to bf16)."""
    t1, m1 = conv_dgrad(dy1, w1, 1, 0, H, W)
    E1 = gemm_err(m1, dy1.shape[-1])
    if wd is None:
        sc = dOut * keep3
        ref = t1 + sc
        return ref, bf16_bound(ref, E1, t1)
    t2, m2 = conv_dgrad(dyd, wd, stride, 0, H, W)
    E2 = gemm_err(m2, dyd.shape[-1])
    ref = t1 + t2
    return ref, bf16_bound(ref, E1 + E2, t1, t2)


def _dgrad_err(mag, C, stride):
    """E of a 3x3 / pad 1 conv dgrad of C output channels: one 9-tap launch at stride 1; at stride 2 one launch per
    parity class (ph, pw) of the input position, (1 + ph) * (1 + pw) taps long."""
    if stride == 1:
        return gemm_err(mag, 9 * C)
    E = mag.new_empty(mag.shape)
    for ph in (0, 1):
        for pw in (0, 1):
            E[:, ph::2, pw::2] = gemm_err(mag[:, ph::2, pw::2], (1 + ph) * (1 + pw) * C)
    return E


def basic_block_dx(dy1, w1, stride, H, W, dOut=None, keep2=None, dyd=None, wd=None):
    """Outgoing gradient [N, H, W, Cin] of a basic block and its bound: the 3x3 conv1 dgrad dy1 . W1 (stride) plus the
    shortcut term.

    Identity block: dOut * keep2, added by the dgrad's own epilogue (residual under the bit mask) to its
    bf16-rounded tile, so E carries |dOut * keep2| and the bound one more ulp of the dgrad.  Transition block: dyd . Wd
    at the stride positions, a second launch that reads the stored conv1 dgrad (bf16) as its residual and adds it to
    its own bf16-rounded tile: three roundings and both accumulations where it lands, the conv1 dgrad's alone
    elsewhere (the odd positions of a stride-2 block)."""
    t1, m1 = conv_dgrad(dy1, w1, stride, 1, H, W)
    E1 = _dgrad_err(m1, dy1.shape[-1], stride)
    if wd is None:
        sc = dOut * keep2
        ref = t1 + sc
        return ref, bf16_bound(ref, E1 + gemm_err(sc.abs(), 9 * dy1.shape[-1]), t1)
    t2, m2 = conv_dgrad(dyd, wd, stride, 0, H, W)
    stored = t1.abs() + E1 + R.ulp_bf16(t1.abs() + E1)  # |the bf16 conv1 dgrad| the second launch reads
    on = torch.zeros_like(t1[..., :1])
    on[:, ::stride, ::stride] = 1.0
    E = E1 + on * gemm_err(m2 + stored, dyd.shape[-1])
    ref = t1 + t2
    b = E + R.ulp_bf16(ref.abs() + E)
    return ref, b + on * (R.ulp_bf16(t1.abs() + E1) + R.ulp_bf16(t2.abs() + E))


def maxpool_backward(dpool, idx, H, W):
    """Stem max-pool gradient [N, H, W, C] of dpool [N, Ho, Wo, C] through the slots idx, and its bound: at most four
    windows overlap, summed in fp32 and rounded to bf16."""
    ref = R.maxpool_bwd(dpool, idx, H, W)
    mag = R.maxpool_bwd(dpool.abs(), idx, H, W)
    return ref, R.ulp_bf16(ref) + 4 * R.U * mag


# ------------------------------------------------------------------------------------------------ eval forward
def eval_conv_bn(x, w, stride, pad, bnp, res=None, relu=True):
    """A conv with its eval-mode BN (scale / shift rows of bnp) folded into the GEMM epilogue, (+ shortcut) (+ ReLU):
    (reference, bound)."""
    acc, mag = conv(x, w, stride, pad)
    sc, sh = bnp[2], bnp[3]
    pre = acc * sc + sh
    E = gemm_err(mag, w.shape[1] * w.shape[2] * w.shape[3], sc, sh)
    v = pre if res is None else pre + res
    ref = v.clamp_min(0.0) if relu else v
    return ref, (bf16_bound(ref, E) if res is None else bf16_bound(ref, E, pre))
