"""Stand-alone tests of the backbone's memory-bound kernels (virtex_b200/csrc/backbone.cu) against float64 references:
BatchNorm finalize / apply / backward, the stem's fused BN + ReLU + max pool and its backward, the batched weight-layout
jobs and the layout kernels.  Every kernel is called through the C ABI (virtex_b200.ops.call).

Shapes: the batch-256 extents of a ResNet-50 at 224 px, (C, M) = (64, 3 211 264) for the stem BN up to
(2048, 12 544), where the grid-stride loops wrap many times and vtx_bn_bwd_reduce runs at its grid cap; and at every
ResNet width M = 1, 7, 33, 1001 (grids of one block, partial unroll groups).  Outputs start as a sentinel with rows
beyond M that must stay untouched; accumulated outputs (dgamma, dbeta, unpack-add gradients) start non-zero.

What is compared (tests/backbone_replica.py states the rounding points, read from the sm_90a SASS):
  * bit for bit: BN mean, scale and shift (from the device's invstd), running buffers, the BN + ReLU (+ residual)
    output and its bit mask, fused against unfused forward launches, max-pool values and slots, the max-pool
    gradient (dpool = k / 64 with |k| <= 64, so that every fp32 sum of at most 4 of them is exact), dz_out = dA * mask,
    dgamma / dbeta, weight layouts and layout kernels;
  * invstd: rsqrtf is a 2-ulp function: within 4 fp32 ulp of float64 1 / sqrt(var + eps) of the replica's fp32 var.
    Against float64 evaluated from the same fp32 stats it is also within 4 ulp plus a relative 2 * 2^-24 * (sumsq /
    count) / (var + eps): fp32 E[y^2] - mean^2 cancels when |mean| >> std (channels here go up to |mean| / std = 8).
    That loss is a known property of the sum / sum-of-squares statistics, not a bug;
  * BN backward sums: sum_m dz and sum_m dz * (y - mean) * invstd against float64 sums of the same terms, within
    (L + 3) * 2^-24 * sum |term|, L = terms per thread + rows reduced per CTA + atomics per channel (the sequential
    depth of the kernel's fp32 accumulation), the 3 for the rounding of each term;
  * fused against unfused BN backward: NOT bit-identical.  On an H100 a few outputs in 10^5 - 10^8 differ, mostly by
    1 bf16 ulp and up to the fp32 floor below where k0 dz + k1 y + k2 cancels; the fused kernel derives its fp32
    coefficients in its own prologue.  Each path is held to the float64 bound below, and fused to unfused within that
    bound plus 1 ulp; the two unfused launches (with and without dz_out) are bit-identical;
  * BN backward dy = k0 * dz + k1 * y + k2 (k0 = scale, k1 = -scale * m2 * invstd, k2 = scale * (m2 * invstd * mean -
    m1), m1 / m2 = device sums / count): within 1 bf16 ulp of float64, plus 2^-21 * (|k0 dz| + |k1 y| + |scale| *
    (|m2 invstd mean| + |m1|)) for the fp32 coefficients (k2 cancels when |mean| is large) and evaluation.
"""
import struct

import pytest
import torch
import torch.nn.functional as F

from tests import backbone_replica as R

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
U = R.U
MOM, EPS = 0.1, 1e-5
EXTRA = 3  # rows beyond M that must stay untouched
WIDTHS = (64, 128, 256, 512, 1024, 2048)
STAGE = [(64, 3211264), (64, 802816), (256, 802816), (128, 200704), (512, 200704), (256, 50176), (1024, 50176),
         (512, 12544), (2048, 12544)]
SHAPES = STAGE + [(C, M) for C in WIDTHS for M in (1, 7, 33, 1001)]
SHAPE_IDS = [f"C{C}-M{M}" for C, M in SHAPES]


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _ops():
    from virtex_b200 import ops
    return ops


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return 0 if t is None else t.data_ptr()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _d(t):
    return t.to(F64)


def ulp_f32(x):
    e = torch.floor(torch.log2(x.abs())).clamp_min(-126)
    return torch.exp2(e - 23)


def assert_equal(got, want, what):
    """Value equality (+0 == -0); NaN is never expected here."""
    bad = _d(got) != want
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} elements differ"


def assert_within(got, want, tol, what):
    err = (_d(got) - want).abs()
    bad = ~(err <= tol)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} beyond tolerance; worst err/tol "
                                 f"{(err / tol).max().item():.3g}")


def _bf16_rows(M, C, g, mean=None, std=None):
    """[M + EXTRA, C] bf16 ~ N(mean_c, std_c), so that views [:M] are the operand and the tail is readable junk."""
    x = torch.randn(M + EXTRA, C, device=DEV, generator=g)
    if std is not None:
        x.mul_(std)
    if mean is not None:
        x.add_(mean)
    return x.to(BF16)


def _channel_moments(C, g):
    """Per-channel mean and std with |mean| / std up to 8."""
    std = torch.rand(C, device=DEV, generator=g) * 1.5 + 0.25
    ratio = (torch.rand(C, device=DEV, generator=g) * 2 - 1) * 8
    return ratio * std, std


def _stats(y):
    yd = _d(y)
    return torch.stack([yd.sum(0), (yd * yd).sum(0)]).to(F32).contiguous()


class _Bn:
    """BN parameters and running buffers of one layer."""

    def __init__(self, C, g):
        self.gamma = torch.rand(C, device=DEV, generator=g) + 0.5
        self.beta = torch.randn(C, device=DEV, generator=g) * 0.3
        self.rm = torch.randn(C, device=DEV, generator=g)
        self.rv = torch.rand(C, device=DEV, generator=g) + 0.5
        self.nbt = torch.tensor([41], dtype=torch.int64, device=DEV)

    def clone(self):
        b = object.__new__(_Bn)
        b.gamma, b.beta, b.rm, b.rv, b.nbt = self.gamma, self.beta, self.rm.clone(), self.rv.clone(), self.nbt.clone()
        return b


def _finalize(ops, bn, stats, count, training, C):
    bnp = torch.full((4, C), 7.0, device=DEV)
    ops.call("vtx_bn_finalize", _p(stats), float(count), bn.gamma.data_ptr(), bn.beta.data_ptr(), bn.rm.data_ptr(),
             bn.rv.data_ptr(), bn.nbt.data_ptr(), MOM, EPS, int(training), bnp.data_ptr(), C, _s())
    return bnp


# ------------------------------------------------------------------------------------------------ BN finalize
@pytest.mark.parametrize("count", [1, 2, 7, 1001, 3211264])
@pytest.mark.parametrize("C", [8, 64, 200, 2048, 4096])
def test_bn_finalize_training_and_eval(C, count):
    _need_cuda()
    ops = _ops()
    g = _gen(C * 7 + count)
    mean, std = _channel_moments(C, g)
    var = std * std
    var[::5] = 0.0                          # constant channels
    s1 = _d(mean) * count
    s2 = (_d(var) + _d(mean) ** 2) * count
    s2[1::7] = s1[1::7] ** 2 / count * 0.999  # sumsq / count < mean^2 in fp32: var clamps at 0
    stats = torch.stack([s1, s2]).to(F32).contiguous()
    bn = _Bn(C, g)
    start = bn.clone()
    bnp = _finalize(ops, bn, stats, count, True, C)
    mean_r, var_r, inv_ref, rm_r, rv_r = R.bn_finalize(_d(stats), count, _d(bn.gamma), _d(bn.beta), _d(start.rm),
                                                       _d(start.rv), MOM, EPS, True)
    assert_equal(bnp[0], mean_r, "mean")
    inv = _d(bnp[1])
    assert_within(bnp[1], inv_ref, 4 * ulp_f32(inv_ref), "invstd vs the fp32 variance")
    # against float64 from the fp32 stats: the cancellation of E[y^2] - mean^2 in fp32
    q = _d(stats[1]) / count
    m64 = _d(stats[0]) / count
    v64 = (q - m64 * m64).clamp_min(0)
    inv64 = 1 / torch.sqrt(v64 + EPS)
    assert_within(bnp[1], inv64, 4 * ulp_f32(inv64) + inv64 * 2 * U * q / (v64 + EPS), "invstd vs float64 stats")
    sc, sh = R.bn_scale_shift(_d(bn.gamma), _d(bn.beta), mean_r, inv)
    assert_equal(bnp[2], sc, "scale")
    assert_equal(bnp[3], sh, "shift")
    assert_equal(bn.rm, rm_r, "running_mean")
    assert_equal(bn.rv, rv_r, "running_var (unbiased)")
    assert int(bn.nbt) == 42
    # eval: statistics from the running buffers, stats = NULL, buffers and the counter untouched
    ev = start.clone()
    bnp_e = _finalize(ops, ev, None, 0.0, False, C)
    assert torch.equal(ev.rm, start.rm) and torch.equal(ev.rv, start.rv) and int(ev.nbt) == 41
    assert_equal(bnp_e[0], _d(start.rm), "eval mean")
    inv_e = R.bn_finalize(None, 0, None, None, _d(start.rm), _d(start.rv), MOM, EPS, False)[2]
    assert_within(bnp_e[1], inv_e, 4 * ulp_f32(inv_e), "eval invstd")
    sc, sh = R.bn_scale_shift(_d(bn.gamma), _d(bn.beta), _d(start.rm), _d(bnp_e[1]))
    assert_equal(bnp_e[2], sc, "eval scale")
    assert_equal(bnp_e[3], sh, "eval shift")


# ------------------------------------------------------------------------------------------------ BN apply
ACT_VARIANTS = [  # (operand: none / residual / residual with its own BN, relu, mask pointer)
    ("plain", 1, True), ("plain", 1, False), ("plain", 0, True),
    ("res", 1, True), ("res_bn", 1, True), ("res_bn", 0, False)]


@pytest.mark.parametrize("C,M", SHAPES, ids=SHAPE_IDS)
def test_bn_act_and_fused_finalize_act(C, M):
    _need_cuda()
    ops = _ops()
    g = _gen(C + 3 * M)
    mu, sd = _channel_moments(C, g)
    y = _bf16_rows(M, C, g, mu, sd)
    res = _bf16_rows(M, C, g, mu.flip(0), sd.flip(0))
    stats, stats_r = _stats(y[:M]), _stats(res[:M])
    bn, bn_r = _Bn(C, g), _Bn(C, g)
    bnp_r = _finalize(ops, bn_r.clone(), stats_r, M, True, C)
    yd = _d(y[:M])
    for mode, relu, with_mask in ACT_VARIANTS:
        r = res if mode != "plain" else None
        br = bnp_r if mode == "res_bn" else None
        what = f"{mode} relu={relu} mask={with_mask}"
        outs = {}
        for path in ("unfused", "fused", "unfused_eval", "fused_eval"):
            b = bn.clone()
            training = not path.endswith("eval")
            out = torch.full((M + EXTRA, C), -3.0, dtype=BF16, device=DEV)
            mask = torch.full((M + EXTRA, C // 8), 0xA5, dtype=torch.uint8, device=DEV) if with_mask else None
            if path.startswith("unfused"):
                bnp = _finalize(ops, b, stats if training else None, M, training, C)
                ops.call("vtx_bn_act", y.data_ptr(), bnp.data_ptr(), _p(r), _p(br), out.data_ptr(), _p(mask), M, C,
                         relu, _s())
            else:
                bnp = torch.full((4, C), 7.0, device=DEV)
                ops.call("vtx_bn_finalize_act", _p(stats if training else None), float(M), b.gamma.data_ptr(),
                         b.beta.data_ptr(), b.rm.data_ptr(), b.rv.data_ptr(), b.nbt.data_ptr(), MOM, EPS,
                         int(training), bnp.data_ptr(), y.data_ptr(), _p(r), _p(br), out.data_ptr(), _p(mask), M, C,
                         relu, _s())
            outs[path] = (bnp, out, mask, b)
        bnp, out, mask, b = outs["unfused"]
        kw = {}
        if r is not None:
            kw["res"] = _d(r[:M])
        if br is not None:
            kw["scale_r"], kw["shift_r"] = _d(br[2]), _d(br[3])
        pre, ref = R.bn_act(yd, _d(bnp[2]), _d(bnp[3]), relu=bool(relu), **kw)
        assert_equal(out[:M], ref, what)
        assert bool((out[M:] == -3.0).all()), f"{what}: rows beyond M written"
        if mask is not None:
            if relu:
                assert torch.equal(mask[:M], R.pack_mask(pre > 0)), f"{what}: ReLU bit mask"
                assert bool((mask[M:] == 0xA5).all()), f"{what}: mask rows beyond M written"
            else:
                assert bool((mask == 0xA5).all()), f"{what}: mask written without ReLU"
        del pre, ref, kw
        # fused == finalize-then-act, bit for bit: bnp, output, mask, running buffers, counter
        for a, f in (("unfused", "fused"), ("unfused_eval", "fused_eval")):
            (bnp_a, out_a, mask_a, b_a), (bnp_f, out_f, mask_f, b_f) = outs[a], outs[f]
            assert torch.equal(bnp_a, bnp_f), f"{what} {f}: bnp"
            assert torch.equal(out_a.view(torch.int16), out_f.view(torch.int16)), f"{what} {f}: output"
            assert mask_a is None or torch.equal(mask_a, mask_f), f"{what} {f}: mask"
            assert torch.equal(b_a.rm, b_f.rm) and torch.equal(b_a.rv, b_f.rv), f"{what} {f}: running buffers"
            assert int(b_a.nbt) == int(b_f.nbt) == (42 if a == "unfused" else 41), f"{what} {f}: num_batches_tracked"
        del outs


# ------------------------------------------------------------------------------------------------ BN backward
def _reduce_depth(ops, M, C, two):
    return R.reduce_depth(ops.num_sms(), M, C, two)


def _check_sums(sums, dz, y, bnp, depth, what):
    ref, tol = R.bn_bwd_sums(dz, y, bnp, depth)
    for row in range(2):
        assert_within(sums[row], ref[row], tol[row], f"{what}: sums[{row}]")


def _bwd_setup(ops, C, M, g):
    ys, bnps = [], []
    for k in range(2):
        mu, sd = _channel_moments(C, g)
        y = _bf16_rows(M, C, g, mu, sd)
        ys.append(y)
        bnps.append(_finalize(ops, _Bn(C, g), _stats(y[:M]), M, True, C))
    dA = _bf16_rows(M, C, g, std=0.1)
    bits = torch.randint(0, 256, (M + EXTRA, C // 8), dtype=torch.uint8, device=DEV, generator=g)
    return ys, bnps, dA, bits


def _keep(mode, bits, y, bnp, M, C):
    if mode == "bits":
        return R.unpack_mask(bits[:M], C)
    if mode == "from_y":
        return R.fma_f32(_d(y[:M]), _d(bnp[2]), _d(bnp[3])) > 0
    return None


BWD_VARIANTS = [("one", "bits"), ("one", "from_y"), ("one", "none"), ("two", "bits"), ("two", "from_y")]


@pytest.mark.parametrize("C,M", SHAPES, ids=SHAPE_IDS)
def test_bn_backward_reduce_finalize_apply(C, M):
    _need_cuda()
    ops = _ops()
    g = _gen(5 * C + M)
    (y, y2), (bnp, bnp2), dA, bits = _bwd_setup(ops, C, M, g)
    dAd = _d(dA[:M])
    for branches, mode in BWD_VARIANTS:
        two = branches == "two"
        what = f"{branches} mask={mode}"
        a = bits if mode == "bits" else None
        from_y = int(mode == "from_y")
        keep = _keep(mode, bits, y, bnp, M, C)
        dz = dAd if keep is None else dAd * keep
        sums = torch.zeros(2, C, device=DEV)
        sums2 = torch.zeros(2, C, device=DEV) if two else None
        ops.call("vtx_bn_bwd_reduce", dA.data_ptr(), _p(a), y.data_ptr(), bnp.data_ptr(), _p(y2 if two else None),
                 _p(bnp2 if two else None), sums.data_ptr(), _p(sums2), M, C, from_y, _s())
        depth = _reduce_depth(ops, M, C, two)
        _check_sums(sums, dz, y[:M], bnp, depth, what)
        if two:
            _check_sums(sums2, dz, y2[:M], bnp2, depth, what + " branch 2")
        # unfused (finalize + apply) and fused, with and without dz_out
        start = [torch.randn(C, device=DEV, generator=g) for _ in range(4)]
        acc = {k: [s.clone() for s in start] for k in ("unfused", "fused")}
        res = {}
        for path, with_dz in (("unfused", True), ("fused", True), ("unfused", False), ("fused", False)):
            dy = torch.full((M + EXTRA, C), -3.0, dtype=BF16, device=DEV)
            dy2 = torch.full((M + EXTRA, C), -3.0, dtype=BF16, device=DEV) if two else None
            dzo = torch.full((M + EXTRA, C), -3.0, dtype=BF16, device=DEV) if with_dz else None
            dg = acc[path] if with_dz else [None] * 4  # accumulate dgamma / dbeta once per path
            if path == "unfused":
                coef = torch.full((3, C), 7.0, device=DEV)
                coef2 = torch.full((3, C), 7.0, device=DEV) if two else None
                ops.call("vtx_bn_bwd_finalize", sums.data_ptr(), bnp.data_ptr(), float(M), coef.data_ptr(),
                         _p(dg[0]), _p(dg[1]), C, _s())
                if two:
                    ops.call("vtx_bn_bwd_finalize", sums2.data_ptr(), bnp2.data_ptr(), float(M), coef2.data_ptr(),
                             _p(dg[2]), _p(dg[3]), C, _s())
                ops.call("vtx_bn_bwd_apply", dA.data_ptr(), _p(a), y.data_ptr(), bnp.data_ptr(), coef.data_ptr(),
                         dy.data_ptr(), _p(y2 if two else None), _p(bnp2 if two else None), _p(coef2), _p(dy2),
                         _p(dzo), M, C, from_y, _s())
            else:
                ops.call("vtx_bn_bwd_finalize_apply", sums.data_ptr(), _p(sums2), float(M), _p(dg[0]), _p(dg[1]),
                         _p(dg[2]), _p(dg[3]), dA.data_ptr(), _p(a), y.data_ptr(), bnp.data_ptr(), dy.data_ptr(),
                         _p(y2 if two else None), _p(bnp2 if two else None), _p(dy2), _p(dzo), M, C, from_y, _s())
            res[path, with_dz] = (dy, dy2, dzo)
        dy, dy2, dzo = res["unfused", True]
        assert_equal(dzo[:M], dz, what + ": dz_out")
        refs = [R.bn_bwd_dy(dz, y[:M], bnp, sums, M)] + ([R.bn_bwd_dy(dz, y2[:M], bnp2, sums2, M)] if two else [])
        for key, (d1, d2, dz_o) in res.items():
            for k, (got, base) in enumerate(((d1, dy), (d2, dy2))[:len(refs)]):
                ref, tol = refs[k]
                assert_within(got[:M], ref, tol, f"{what} {key}: dy{k + 1}")
                # same launcher: bit for bit; fused against unfused: not bit-identical (see the module docstring)
                if key[0] == "unfused":
                    assert torch.equal(got.view(torch.int16), base.view(torch.int16)), f"{what} {key}: dy{k + 1}"
                else:
                    assert_within(got[:M], _d(base[:M]), tol + R.ulp_bf16(_d(base[:M])),
                                  f"{what} {key}: dy{k + 1} vs unfused")
                assert bool((got[M:] == -3.0).all()), f"{what} {key}: dy{k + 1} rows beyond M written"
            if dz_o is not None:
                assert torch.equal(dz_o, dzo) and bool((dz_o[M:] == -3.0).all()), f"{what} {key}: dz_out"
        del refs
        for path in ("unfused", "fused"):
            dgam, dbet = acc[path][0], acc[path][1]
            assert_equal(dgam, R.f32(_d(start[0]) + _d(sums[1])), f"{what} {path}: dgamma")
            assert_equal(dbet, R.f32(_d(start[1]) + _d(sums[0])), f"{what} {path}: dbeta")
            if two:
                assert_equal(acc[path][2], R.f32(_d(start[2]) + _d(sums2[1])), f"{what} {path}: dgamma2")
                assert_equal(acc[path][3], R.f32(_d(start[3]) + _d(sums2[0])), f"{what} {path}: dbeta2")
            else:
                assert torch.equal(acc[path][2], start[2]) and torch.equal(acc[path][3], start[3])
        del res, dz, keep


# ------------------------------------------------------------------------------------------------ channel widths
ODD_WIDTHS = (24, 40, 96, 160, 320, 4096)
ODD_M = {1: (1, 1, 1), 100: (1, 10, 10), 1001: (1, 7, 143), 200704: (16, 112, 112)}  # M -> an (N, H, W) image


@pytest.mark.parametrize("M", sorted(ODD_M))
@pytest.mark.parametrize("C", ODD_WIDTHS)
def test_channel_widths_outside_the_register_layout(C, M):
    """C / 8 not dividing 256: the four BN-apply launchers reject it; the reduce and both pool kernels, which idle the
    threads beyond a whole number of channel groups, match float64 at every such C <= 2048."""
    _need_cuda()
    ops = _ops()
    from virtex_b200.lib import VtxError
    g = _gen(C * 11 + M)
    y = _bf16_rows(M, C, g)
    bnp = R.f32(torch.stack([torch.randn(C, device=DEV, generator=g, dtype=F64) * 0.1,
                             torch.rand(C, device=DEV, generator=g, dtype=F64) + 0.5,
                             torch.rand(C, device=DEV, generator=g, dtype=F64) + 0.5,
                             torch.randn(C, device=DEV, generator=g, dtype=F64) * 0.2])).to(F32).contiguous()
    out = torch.full((M + EXTRA, C), -3.0, dtype=BF16, device=DEV)
    mask = torch.full((M + EXTRA, C // 8), 0xA5, dtype=torch.uint8, device=DEV)
    st = torch.ones(2, C, device=DEV)
    bn = _Bn(C, g)
    bnp_w = bnp.clone()
    calls = [
        ("vtx_bn_act", (y.data_ptr(), bnp.data_ptr(), 0, 0, out.data_ptr(), mask.data_ptr(), M, C, 1, _s())),
        ("vtx_bn_finalize_act", (st.data_ptr(), float(M), bn.gamma.data_ptr(), bn.beta.data_ptr(), bn.rm.data_ptr(),
                                 bn.rv.data_ptr(), bn.nbt.data_ptr(), MOM, EPS, 1, bnp_w.data_ptr(), y.data_ptr(),
                                 0, 0, out.data_ptr(), mask.data_ptr(), M, C, 1, _s())),
        ("vtx_bn_bwd_apply", (y.data_ptr(), mask.data_ptr(), y.data_ptr(), bnp.data_ptr(), bnp.data_ptr(),
                              out.data_ptr(), 0, 0, 0, 0, 0, M, C, 0, _s())),
        ("vtx_bn_bwd_finalize_apply", (st.data_ptr(), 0, float(M), 0, 0, 0, 0, y.data_ptr(), mask.data_ptr(),
                                       y.data_ptr(), bnp.data_ptr(), out.data_ptr(), 0, 0, 0, 0, M, C, 0, _s()))]
    for name, args in calls:
        with pytest.raises(VtxError, match=r"256 % \(C / 8\) == 0"):
            ops.call(name, *args)
    torch.cuda.synchronize()
    assert bool((out == -3.0).all()) and bool((mask == 0xA5).all())
    if C > 2048:
        return
    # backward reduce, single and two-branch, mask from bits
    dA = _bf16_rows(M, C, g, std=0.1)
    y2 = _bf16_rows(M, C, g)
    bits = torch.randint(0, 256, (M, C // 8), dtype=torch.uint8, device=DEV, generator=g)
    dz = _d(dA[:M]) * R.unpack_mask(bits, C)
    for two in (False, True):
        sums, sums2 = torch.zeros(2, C, device=DEV), torch.zeros(2, C, device=DEV)
        ops.call("vtx_bn_bwd_reduce", dA.data_ptr(), bits.data_ptr(), y.data_ptr(), bnp.data_ptr(),
                 _p(y2 if two else None), _p(bnp if two else None), sums.data_ptr(), sums2.data_ptr(), M, C, 0, _s())
        depth = _reduce_depth(ops, M, C, two)
        _check_sums(sums, dz, y[:M], bnp, depth, f"reduce two={two}")
        if two:
            _check_sums(sums2, dz, y2[:M], bnp, depth, "reduce branch 2")
    _check_pool(ops, *ODD_M[M], C, g, f"C={C}")


# ------------------------------------------------------------------------------------------------ max pool
def _check_pool(ops, N, H, W, C, g, what):
    """vtx_bn_relu_maxpool and vtx_maxpool_bwd against the replica, bit for bit."""
    Ho, Wo = R.pool_extent(H, W)
    P = N * Ho * Wo
    y = _bf16_rows(N * H * W, C, g)
    # scale ~ 1, shift ~ 0: about half of the BN outputs are negative, so zeros (ties) fill many windows
    sc = R.f32(torch.rand(C, device=DEV, generator=g, dtype=F64) + 0.5)
    sh = R.f32(torch.randn(C, device=DEV, generator=g, dtype=F64) * 0.05)
    bnp = torch.stack([torch.zeros_like(sc), torch.ones_like(sc), sc, sh]).to(F32).contiguous()
    out = torch.full((P + EXTRA, C), -3.0, dtype=BF16, device=DEV)
    idx = torch.full((P + EXTRA, C), 0xEE, dtype=torch.uint8, device=DEV)
    ops.call("vtx_bn_relu_maxpool", y.data_ptr(), bnp.data_ptr(), out.data_ptr(), idx.data_ptr(), N, H, W, C, _s())
    act = R.bf16(R.fma_f32(_d(y[:N * H * W]), sc, sh).clamp_min(0.0)).view(N, H, W, C)
    ref, ref_idx = R.maxpool_fwd(act)
    assert_equal(out[:P], ref.reshape(P, C), what + ": pooled values")
    assert torch.equal(idx[:P], ref_idx.reshape(P, C)), (f"{what}: {int((idx[:P] != ref_idx.reshape(P, C)).sum())} "
                                                         f"argmax slots differ")
    assert bool((out[P:] == -3.0).all()) and bool((idx[P:] == 0xEE).all()), what + ": rows beyond the pool written"
    k = torch.randint(-64, 65, (P + EXTRA, C), device=DEV, generator=g)
    dpool = (k.to(F32) / 64).to(BF16)
    da = torch.full((N * H * W + EXTRA, C), -3.0, dtype=BF16, device=DEV)
    ops.call("vtx_maxpool_bwd", dpool.data_ptr(), idx.data_ptr(), da.data_ptr(), N, H, W, C, _s())
    ref_da = R.maxpool_bwd(_d(dpool[:P]).view(N, Ho, Wo, C), ref_idx, H, W).reshape(N * H * W, C)
    assert_equal(da[:N * H * W], R.bf16(ref_da), what + ": max-pool gradient")
    assert bool((da[N * H * W:] == -3.0).all()), what + ": gradient rows beyond the image written"


POOL_IMAGES = [(2, 112, 112), (2, 100, 100), (3, 7, 9), (2, 1, 1), (2, 2, 3)]


@pytest.mark.parametrize("C", [64, 8, 24, 128])
@pytest.mark.parametrize("N,H,W", POOL_IMAGES, ids=[f"{n}x{h}x{w}" for n, h, w in POOL_IMAGES])
def test_bn_relu_maxpool_and_backward(N, H, W, C):
    """Row kernel for C / 8 <= 256; backward: tiled under 48 KB (100 x 100, C 64: Wo = 50), tiled above 48 KB
    (112 x 112, C 64 or 128), generic for C % 16 != 0 (8, 24)."""
    _need_cuda()
    _check_pool(_ops(), N, H, W, C, _gen(N * H * W + C), f"{N}x{H}x{W}x{C}")


@pytest.mark.parametrize("N,H,W,C", [(2, 15, 16, 4096), (1, 224, 224, 128)], ids=["flat-fwd-C4096", "generic-bwd-smem"])
def test_maxpool_other_launch_paths(N, H, W, C):
    """The flat forward kernel (C / 8 > 256), and the generic backward kernel reached by shared memory: 5 pooled rows
    of 112 x 128 gradients and slots take 215 040 B, more than the tiled kernel's 200 KB."""
    _need_cuda()
    _check_pool(_ops(), N, H, W, C, _gen(C + W), f"{N}x{H}x{W}x{C}")


# ------------------------------------------------------------------------------------------------ weight jobs
def test_weight_jobs_all_kinds_at_resnet50_shapes():
    _need_cuda()
    ops = _ops()
    g = _gen(17)
    blk = ops.L.load().vtx_weight_job_block_elems()
    jobs = []  # (src, dst, total, O, I, KH, KW, ldk, kind, reference of dst[:total])

    def add(src, total, O, I, KH, KW, ldk, kind, ref, dst_dtype):
        start = 3.0 if dst_dtype == F32 else -3.0
        dst = torch.full((total + 40,), start, dtype=dst_dtype, device=DEV)
        if dst_dtype == F32:
            dst[:total] = torch.randn(total, device=DEV, generator=g)
            ref = dst[:total].clone() + ref.reshape(-1)  # fp32 add: what the kernel does
        jobs.append((src, dst, total, O, I, KH, KW, ldk, kind, ref.reshape(-1), start))

    for planes in (128, 256, 512):  # kind 6: the stride-2 3x3 conv2 of layers 2-4, all four parity classes
        w = torch.randn(planes, planes, 3, 3, device=DEV, generator=g)
        for ph in (0, 1):
            for pw in (0, 1):
                th, tw = 1 + ph, 1 + pw
                ref = torch.empty(planes, th, tw, planes, device=DEV)
                for a in range(th):
                    for b in range(tw):
                        ref[:, a, b, :] = w[:, :, ph + 1 - 2 * a, pw + 1 - 2 * b].t()
                add(w, planes * th * tw * planes, planes, planes, ph, pw, 0, 6, ref.bfloat16(), BF16)
    for c4, cin in ((512, 256), (1024, 512), (2048, 1024)):  # kind 7: the strided downsample's 1x1 weight
        w = torch.randn(c4, cin, device=DEV, generator=g)
        add(w, cin * c4, c4, cin, 1, 1, 0, 7, w.t().bfloat16(), BF16)
    w7 = torch.randn(64, 3, 7, 7, device=DEV, generator=g)
    for ldk in (152, 160):  # kind 0 with ldk > KH * KW * I: zero columns; 64 x 152 is not a multiple of the block
        ref = torch.zeros(64, ldk, device=DEV)
        ref[:, :147] = w7.permute(0, 2, 3, 1).reshape(64, 147)
        add(w7, 64 * ldk, 64, 3, 7, 7, ldk, 0, ref.bfloat16(), BF16)
    w3 = torch.randn(64, 64, 3, 3, device=DEV, generator=g)
    add(w3, 64 * 576, 64, 64, 3, 3, 576, 0, w3.permute(0, 2, 3, 1).reshape(64, 576).bfloat16(), BF16)
    add(w3, 64 * 576, 64, 64, 3, 3, 0, 1, w3.flip(2, 3).permute(1, 2, 3, 0).reshape(64, 576).bfloat16(), BF16)
    dwp = torch.randn(64, 584, device=DEV, generator=g)  # kind 2 with ldk > 9 * I
    add(dwp, 64 * 576, 64, 64, 3, 3, 584, 2, dwp[:, :576].reshape(64, 3, 3, 64).permute(0, 3, 1, 2), F32)
    dwt = torch.randn(576, 64, device=DEV, generator=g)
    add(dwt, 64 * 576, 64, 64, 3, 3, 0, 3, dwt.view(3, 3, 64, 64).permute(3, 2, 0, 1), F32)
    s2d = torch.zeros(64, 4, 4, 16, device=DEV)  # kind 4: k = a*64 + b*16 + (r*2+q)*3 + c, (kh, kw) = (2a+r, 2b+q)
    for a in range(4):
        for b in range(4):
            for r in range(2):
                for q in range(2):
                    if 2 * a + r < 7 and 2 * b + q < 7:
                        s2d[:, a, b, (r * 2 + q) * 3:(r * 2 + q) * 3 + 3] = w7[:, :, 2 * a + r, 2 * b + q]
    add(w7, 64 * 256, 64, 3, 7, 7, 256, 4, s2d.bfloat16(), BF16)
    dw7 = torch.randn(64, 4, 4, 16, device=DEV, generator=g)
    ref5 = torch.empty(64, 3, 7, 7, device=DEV)
    for kh in range(7):
        for kw in range(7):
            k0 = ((kh % 2) * 2 + kw % 2) * 3
            ref5[:, :, kh, kw] = dw7[:, kh // 2, kw // 2, k0:k0 + 3]
    add(dw7, 64 * 147, 64, 3, 7, 7, 256, 5, ref5, F32)
    assert len(jobs) >= 12 and {j[8] for j in jobs} == set(range(8))
    assert any(j[2] % blk for j in jobs)
    blob, b0 = b"", 0
    for src, dst, total, O, I, KH, KW, ldk, kind, _, _ in jobs:
        blob += struct.pack("<QQq8i", src.data_ptr(), dst.data_ptr(), total, O, I, KH, KW, ldk, kind, b0, 0)
        b0 += -(-total // blk)
    table = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(DEV)
    ops.call("vtx_conv_w_jobs", table.data_ptr(), len(jobs), b0, _s())
    for src, dst, total, O, I, KH, KW, ldk, kind, ref, start in jobs:
        what = f"kind {kind} O={O} I={I} KH={KH} KW={KW} ldk={ldk}"
        if dst.dtype == BF16:
            assert torch.equal(dst[:total].view(torch.int16), ref.contiguous().view(torch.int16)), what
        else:
            assert torch.equal(dst[:total], ref), what
        assert bool((dst[total:] == start).all()), what + ": tail written"


# ------------------------------------------------------------------------------------------------ layout kernels
@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, (1 << 22) + 3])
def test_cast_bf16(n):
    _need_cuda()
    ops = _ops()
    g = _gen(n)
    x = torch.randn(n, device=DEV, generator=g) * torch.exp2(torch.randint(-140, 120, (n,), device=DEV, generator=g)
                                                              .float())
    fmax = torch.finfo(F32).max
    tiny = torch.finfo(F32).tiny
    special = torch.tensor([0.0, -0.0, tiny / 3, -tiny / 7, float("inf"), float("-inf"), float("nan"), fmax, -fmax,
                            1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8), 2.0 ** -133 * 3], device=DEV)
    k = min(n, special.numel())
    pos = torch.randperm(n, device=DEV, generator=g)[:k]
    x[pos] = special[:k]
    out = torch.full((n + EXTRA,), -3.0, dtype=BF16, device=DEV)
    ops.call("vtx_cast_bf16", x.data_ptr(), out.data_ptr(), n, _s())
    ref = x.bfloat16()
    nan = torch.isnan(x)
    assert torch.equal(torch.isnan(out[:n]), nan)
    assert torch.equal(out[:n][~nan].view(torch.int16), ref[~nan].view(torch.int16))
    assert bool((out[n:] == -3.0).all())


@pytest.mark.parametrize("N,HW,C", [(2, 49, 2048), (3, 91, 24)])
def test_nhwc_to_nchw_f32(N, HW, C):
    _need_cuda()
    ops = _ops()
    x = torch.randn(N, HW, C, device=DEV, generator=_gen(C)).bfloat16()
    out = torch.full((N * C * HW + EXTRA,), -3.0, device=DEV)
    ops.call("vtx_nhwc_to_nchw_f32", x.data_ptr(), out.data_ptr(), N, HW, C, _s())
    assert torch.equal(out[:N * C * HW].view(N, C, HW), x.float().permute(0, 2, 1))
    assert bool((out[N * C * HW:] == -3.0).all())


@pytest.mark.parametrize("H,W", [(224, 224), (200, 200), (199, 200), (199, 230), (7, 9)])
def test_stem_im2col_matches_unfold(H, W):
    _need_cuda()
    ops = _ops()
    N, ldc = 2, 160
    img = torch.randn(N, 3, H, W, device=DEV, generator=_gen(H * W))
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    rows = N * Ho * Wo
    cols = torch.full((rows + EXTRA, ldc), -3.0, dtype=BF16, device=DEV)
    ops.call("vtx_stem_im2col", img.data_ptr(), cols.data_ptr(), N, H, W, ldc, _s())
    unf = F.unfold(img, 7, padding=3, stride=2)  # [N, c*49 + kh*7 + kw, L]
    ref = torch.zeros(rows, ldc, device=DEV)
    ref[:, :147] = unf.view(N, 3, 49, Ho * Wo).permute(0, 3, 2, 1).reshape(rows, 147)
    assert torch.equal(cols[:rows].view(torch.int16), ref.bfloat16().view(torch.int16))
    assert bool((cols[rows:] == -3.0).all())
