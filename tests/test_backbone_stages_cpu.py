"""The stage references of tests/backbone_stages.py, fed exact float64 values and chained with no rounding in between,
against float64 autograd of torchvision's Bottleneck, of its BasicBlock and of the ResNet stem (7x7 / stride 2 conv,
train-mode BN, ReLU, 3x3 / stride 2 max pool): every forward value, every intermediate gradient, every weight and BN
parameter gradient (biases included) and the outgoing input gradient, to 1e-12 relative to the largest value of each."""
import pytest
import torch
from torch import nn
from torchvision.models.resnet import BasicBlock, Bottleneck

from tests import backbone_replica as R
from tests import backbone_stages as S

F64 = torch.float64
TOL = 1e-12


def _close(got, want, what):
    want = want.detach()
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    assert scale > 0, f"{what}: reference is all zero"
    assert err <= TOL * scale, f"{what}: max err {err:.3g} vs max |ref| {scale:.3g}"


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _live_bn(bn, g):
    with torch.no_grad():
        bn.weight.copy_(torch.rand(bn.weight.shape, generator=g, dtype=F64) + 0.5)
        bn.bias.copy_(torch.randn(bn.bias.shape, generator=g, dtype=F64) * 0.3)


def _capture(mods):
    """Forward hooks keeping each module's input and output in the graph with their gradients retained."""
    seen = {}

    def hook(name):
        def f(m, inp, out):
            inp[0].retain_grad()
            out.retain_grad()
            seen[name] = (inp[0], out)
        return f
    for name, m in mods.items():
        m.register_forward_hook(hook(name))
    return seen


BLOCKS = [  # (Cin, planes, stride, H, W): identity, stride-1 transition, stride-2 transition on an odd extent
    pytest.param(64, 16, 1, 9, 11, id="identity"),
    pytest.param(32, 16, 1, 8, 6, id="transition-s1"),
    pytest.param(32, 8, 2, 13, 15, id="transition-s2-13x15"),
]


@pytest.mark.parametrize("Cin,planes,stride,H,W", BLOCKS)
def test_bottleneck_stages_match_autograd(Cin, planes, stride, H, W):
    g = torch.Generator().manual_seed(Cin + planes + H * W)
    torch.manual_seed(Cin * stride + H)
    C4 = 4 * planes
    down = None
    if stride != 1 or Cin != C4:
        down = nn.Sequential(nn.Conv2d(Cin, C4, 1, stride=stride, bias=False), nn.BatchNorm2d(C4))
    blk = Bottleneck(Cin, planes, stride=stride, downsample=down).to(F64).train()
    blk.relu = nn.ReLU()  # the shared in-place ReLU would overwrite the BN outputs the hooks keep
    for bn in [blk.bn1, blk.bn2, blk.bn3] + ([down[1]] if down is not None else []):
        _live_bn(bn, g)
    N = 3
    x = torch.randn(N, Cin, H, W, generator=g, dtype=F64).requires_grad_(True)
    mods = {"conv1": blk.conv1, "conv2": blk.conv2, "conv3": blk.conv3}
    if down is not None:
        mods["ds"] = down[0]
    seen = _capture(mods)
    out = blk(x)
    dOut = torch.randn(out.shape, generator=g, dtype=F64)
    out.backward(dOut)

    w = {k: m.weight.detach() for k, m in mods.items()}
    xh = _nhwc(x.detach())
    Ho, Wo = S.out_extent(H, W, 3, stride, 1)
    Min, Mout = N * H * W, N * Ho * Wo
    # ---- forward
    y1 = S.conv(xh, w["conv1"], 1, 0)[0]
    _close(y1, _nhwc(seen["conv1"][1]), "y1")
    bnp1 = S.bn_params(y1.reshape(Min, -1), blk.bn1.weight.detach(), blk.bn1.bias.detach())
    pre1, a1 = S.bn_apply(y1.reshape(Min, -1), bnp1, exact=True)
    a1 = a1.view(N, H, W, -1)
    _close(a1, _nhwc(seen["conv2"][0]), "a1")
    y2 = S.conv(a1, w["conv2"], stride, 1)[0]
    _close(y2, _nhwc(seen["conv2"][1]), "y2")
    bnp2 = S.bn_params(y2.reshape(Mout, -1), blk.bn2.weight.detach(), blk.bn2.bias.detach())
    a2 = S.bn_apply(y2.reshape(Mout, -1), bnp2, exact=True)[1].view(N, Ho, Wo, -1)
    _close(a2, _nhwc(seen["conv3"][0]), "a2")
    y3 = S.conv(a2, w["conv3"], 1, 0)[0]
    _close(y3, _nhwc(seen["conv3"][1]), "y3")
    bnp3 = S.bn_params(y3.reshape(Mout, -1), blk.bn3.weight.detach(), blk.bn3.bias.detach())
    if down is not None:
        yd = S.conv(xh, w["ds"], stride, 0)[0]
        _close(yd, _nhwc(seen["ds"][1]), "yd")
        bnpd = S.bn_params(yd.reshape(Mout, -1), down[1].weight.detach(), down[1].bias.detach())
        pre3, o = S.bn_apply(y3.reshape(Mout, -1), bnp3, res=yd.reshape(Mout, -1), bnp_res=bnpd, exact=True)
    else:
        pre3, o = S.bn_apply(y3.reshape(Mout, -1), bnp3, res=xh.reshape(Mout, -1), exact=True)
    _close(o.view(N, Ho, Wo, -1), _nhwc(out), "block output")
    assert torch.equal(R.unpack_mask(R.pack_mask(pre3 > 0), C4), pre3 > 0)
    # ---- backward
    dO = _nhwc(dOut).reshape(Mout, C4)
    dz3 = dO * (pre3 > 0)
    sums3 = S.bn_sums(dz3, y3.reshape(Mout, -1), bnp3)[0]
    _, dy3, _ = S.bn_backward(dO, pre3 > 0, y3.reshape(Mout, -1), bnp3, sums3, Mout)
    _close(dy3.view(N, Ho, Wo, -1), _nhwc(seen["conv3"][1].grad), "dy3")
    _close(sums3[1], blk.bn3.weight.grad, "bn3 dgamma")
    _close(sums3[0], blk.bn3.bias.grad, "bn3 dbeta")
    dyd = None
    if down is not None:
        sumsd = S.bn_sums(dz3, yd.reshape(Mout, -1), bnpd)[0]
        dyd = S.bn_backward(dO, pre3 > 0, yd.reshape(Mout, -1), bnpd, sumsd, Mout)[1].view(N, Ho, Wo, -1)
        _close(dyd, _nhwc(seen["ds"][1].grad), "dyd")
        _close(sumsd[1], down[1].weight.grad, "downsample.1 dgamma")
        _close(sumsd[0], down[1].bias.grad, "downsample.1 dbeta")
    dy3 = dy3.view(N, Ho, Wo, -1)
    da2 = S.conv_dgrad(dy3, w["conv3"], 1, 0, Ho, Wo)[0]
    _close(da2, _nhwc(seen["conv3"][0].grad), "da2")
    keep2 = S.relu_keep(y2.reshape(Mout, -1), bnp2, exact=True)
    dz2 = da2.reshape(Mout, -1) * keep2
    sums2 = S.bn_sums(dz2, y2.reshape(Mout, -1), bnp2)[0]
    dy2 = S.bn_backward(da2.reshape(Mout, -1), keep2, y2.reshape(Mout, -1), bnp2, sums2, Mout)[1]
    dy2 = dy2.view(N, Ho, Wo, -1)
    _close(dy2, _nhwc(seen["conv2"][1].grad), "dy2")
    _close(sums2[1], blk.bn2.weight.grad, "bn2 dgamma")
    _close(sums2[0], blk.bn2.bias.grad, "bn2 dbeta")
    da1 = S.conv_dgrad(dy2, w["conv2"], stride, 1, H, W)[0]
    _close(da1, _nhwc(seen["conv2"][0].grad), "da1")
    keep1 = S.relu_keep(y1.reshape(Min, -1), bnp1, exact=True)
    sums1 = S.bn_sums(da1.reshape(Min, -1) * keep1, y1.reshape(Min, -1), bnp1)[0]
    dy1 = S.bn_backward(da1.reshape(Min, -1), keep1, y1.reshape(Min, -1), bnp1, sums1, Min)[1].view(N, H, W, -1)
    _close(dy1, _nhwc(seen["conv1"][1].grad), "dy1")
    _close(sums1[1], blk.bn1.weight.grad, "bn1 dgamma")
    _close(sums1[0], blk.bn1.bias.grad, "bn1 dbeta")
    if down is None:
        dx = S.block_dx(dy1, w["conv1"], H, W, dOut=_nhwc(dOut), keep3=(pre3 > 0).view(N, Ho, Wo, -1))[0]
    else:
        dx = S.block_dx(dy1, w["conv1"], H, W, dyd=dyd, wd=w["ds"], stride=stride)[0]
    _close(dx, _nhwc(x.grad), "dx")
    # ---- weight gradients
    _close(S.conv_wgrad(dy3, a2, 1, 1, 1, 0)[0], blk.conv3.weight.grad, "conv3 dW")
    _close(S.conv_wgrad(dy2, a1, 3, 3, stride, 1)[0], blk.conv2.weight.grad, "conv2 dW")
    _close(S.conv_wgrad(dy1, xh, 1, 1, 1, 0)[0], blk.conv1.weight.grad, "conv1 dW")
    if down is not None:
        _close(S.conv_wgrad(dyd, xh, 1, 1, stride, 0)[0], down[0].weight.grad, "downsample.0 dW")


BASIC_BLOCKS = [  # (Cin, planes, stride, H, W): identity, stride-2 transition on an odd extent, stride-1 Cin != C
    pytest.param(16, 16, 1, 9, 11, id="identity"),
    pytest.param(8, 16, 2, 13, 15, id="transition-s2-13x15"),
    pytest.param(8, 16, 1, 8, 6, id="transition-s1"),
]


@pytest.mark.parametrize("Cin,planes,stride,H,W", BASIC_BLOCKS)
def test_basic_block_stages_match_autograd(Cin, planes, stride, H, W):
    g = torch.Generator().manual_seed(7 * Cin + planes + H * W)
    torch.manual_seed(Cin * stride + W)
    C = planes
    down = None
    if stride != 1 or Cin != C:
        down = nn.Sequential(nn.Conv2d(Cin, C, 1, stride=stride, bias=False), nn.BatchNorm2d(C))
    blk = BasicBlock(Cin, planes, stride=stride, downsample=down).to(F64).train()
    blk.relu = nn.ReLU()  # the shared in-place ReLU would overwrite the BN outputs the hooks keep
    for bn in [blk.bn1, blk.bn2] + ([down[1]] if down is not None else []):
        _live_bn(bn, g)
    N = 3
    x = torch.randn(N, Cin, H, W, generator=g, dtype=F64).requires_grad_(True)
    mods = {"conv1": blk.conv1, "conv2": blk.conv2}
    if down is not None:
        mods["ds"] = down[0]
    seen = _capture(mods)
    out = blk(x)
    dOut = torch.randn(out.shape, generator=g, dtype=F64)
    out.backward(dOut)

    w = {k: m.weight.detach() for k, m in mods.items()}
    xh = _nhwc(x.detach())
    Ho, Wo = S.out_extent(H, W, 3, stride, 1)
    Mout = N * Ho * Wo
    # ---- forward
    y1 = S.conv(xh, w["conv1"], stride, 1)[0]
    _close(y1, _nhwc(seen["conv1"][1]), "y1")
    bnp1 = S.bn_params(y1.reshape(Mout, -1), blk.bn1.weight.detach(), blk.bn1.bias.detach())
    a1 = S.bn_apply(y1.reshape(Mout, -1), bnp1, exact=True)[1].view(N, Ho, Wo, -1)
    _close(a1, _nhwc(seen["conv2"][0]), "a1")
    y2 = S.conv(a1, w["conv2"], 1, 1)[0]
    _close(y2, _nhwc(seen["conv2"][1]), "y2")
    bnp2 = S.bn_params(y2.reshape(Mout, -1), blk.bn2.weight.detach(), blk.bn2.bias.detach())
    if down is not None:
        yd = S.conv(xh, w["ds"], stride, 0)[0]
        _close(yd, _nhwc(seen["ds"][1]), "yd")
        bnpd = S.bn_params(yd.reshape(Mout, -1), down[1].weight.detach(), down[1].bias.detach())
        pre2, o = S.bn_apply(y2.reshape(Mout, -1), bnp2, res=yd.reshape(Mout, -1), bnp_res=bnpd, exact=True)
    else:
        pre2, o = S.bn_apply(y2.reshape(Mout, -1), bnp2, res=xh.reshape(Mout, -1), exact=True)
    _close(o.view(N, Ho, Wo, -1), _nhwc(out), "block output")
    assert torch.equal(R.unpack_mask(R.pack_mask(pre2 > 0), C), pre2 > 0)
    # ---- backward
    dO = _nhwc(dOut).reshape(Mout, C)
    dz2 = dO * (pre2 > 0)
    sums2 = S.bn_sums(dz2, y2.reshape(Mout, -1), bnp2)[0]
    dy2 = S.bn_backward(dO, pre2 > 0, y2.reshape(Mout, -1), bnp2, sums2, Mout)[1].view(N, Ho, Wo, -1)
    _close(dy2, _nhwc(seen["conv2"][1].grad), "dy2")
    _close(sums2[1], blk.bn2.weight.grad, "bn2 dgamma")
    _close(sums2[0], blk.bn2.bias.grad, "bn2 dbeta")
    dyd = None
    if down is not None:
        sumsd = S.bn_sums(dz2, yd.reshape(Mout, -1), bnpd)[0]
        dyd = S.bn_backward(dO, pre2 > 0, yd.reshape(Mout, -1), bnpd, sumsd, Mout)[1].view(N, Ho, Wo, -1)
        _close(dyd, _nhwc(seen["ds"][1].grad), "dyd")
        _close(sumsd[1], down[1].weight.grad, "downsample.1 dgamma")
        _close(sumsd[0], down[1].bias.grad, "downsample.1 dbeta")
    da1 = S.conv_dgrad(dy2, w["conv2"], 1, 1, Ho, Wo)[0]
    _close(da1, _nhwc(seen["conv2"][0].grad), "da1")
    keep1 = S.relu_keep(y1.reshape(Mout, -1), bnp1, exact=True)
    sums1 = S.bn_sums(da1.reshape(Mout, -1) * keep1, y1.reshape(Mout, -1), bnp1)[0]
    dy1 = S.bn_backward(da1.reshape(Mout, -1), keep1, y1.reshape(Mout, -1), bnp1, sums1, Mout)[1]
    dy1 = dy1.view(N, Ho, Wo, -1)
    _close(dy1, _nhwc(seen["conv1"][1].grad), "dy1")
    _close(sums1[1], blk.bn1.weight.grad, "bn1 dgamma")
    _close(sums1[0], blk.bn1.bias.grad, "bn1 dbeta")
    if down is None:
        dx = S.basic_block_dx(dy1, w["conv1"], stride, H, W, dOut=_nhwc(dOut),
                              keep2=(pre2 > 0).view(N, Ho, Wo, -1))[0]
    else:
        dx = S.basic_block_dx(dy1, w["conv1"], stride, H, W, dyd=dyd, wd=w["ds"])[0]
    _close(dx, _nhwc(x.grad), "dx")
    # ---- weight gradients
    _close(S.conv_wgrad(dy2, a1, 3, 3, 1, 1)[0], blk.conv2.weight.grad, "conv2 dW")
    _close(S.conv_wgrad(dy1, xh, 3, 3, stride, 1)[0], blk.conv1.weight.grad, "conv1 dW")
    if down is not None:
        _close(S.conv_wgrad(dyd, xh, 1, 1, stride, 0)[0], down[0].weight.grad, "downsample.0 dW")


@pytest.mark.parametrize("H,W", [(224, 224), (199, 230)])
def test_stem_stages_match_autograd(H, W):
    g = torch.Generator().manual_seed(H + W)
    torch.manual_seed(H * W)
    conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False).to(F64)
    bn1 = nn.BatchNorm2d(64).to(F64).train()
    _live_bn(bn1, g)
    N = 2
    img = torch.randn(N, 3, H, W, generator=g, dtype=F64)
    y0_t = conv1(img)
    y0_t.retain_grad()
    act_t = torch.relu(bn1(y0_t))
    act_t.retain_grad()
    pool_t = nn.functional.max_pool2d(act_t, 3, 2, 1)
    dpool = torch.randn(pool_t.shape, generator=g, dtype=F64)
    pool_t.backward(dpool)

    Ho, Wo = S.out_extent(H, W, 7, 2, 3)
    M0 = N * Ho * Wo
    w0 = conv1.weight.detach()
    y0 = S.conv(_nhwc(img), w0, 2, 3)[0]
    _close(y0, _nhwc(y0_t), "y0")
    bnp0 = S.bn_params(y0.reshape(M0, 64), bn1.weight.detach(), bn1.bias.detach())
    act = S.bn_apply(y0.reshape(M0, 64), bnp0, exact=True)[1].view(N, Ho, Wo, 64)
    _close(act, _nhwc(act_t), "stem activation")
    pool, idx = S.maxpool(act)
    _close(pool, _nhwc(pool_t), "max pool")
    da0 = S.maxpool_backward(_nhwc(dpool), idx, Ho, Wo)[0]
    _close(da0, _nhwc(act_t.grad), "max-pool gradient")
    keep0 = S.relu_keep(y0.reshape(M0, 64), bnp0, exact=True)
    sums0 = S.bn_sums(da0.reshape(M0, 64) * keep0, y0.reshape(M0, 64), bnp0)[0]
    dy0 = S.bn_backward(da0.reshape(M0, 64), keep0, y0.reshape(M0, 64), bnp0, sums0, M0)[1]
    _close(dy0.view(N, Ho, Wo, 64), _nhwc(y0_t.grad), "dy0")
    _close(sums0[1], bn1.weight.grad, "bn1 dgamma")
    _close(sums0[0], bn1.bias.grad, "bn1 dbeta")
    _close(S.conv_wgrad(dy0.view(N, Ho, Wo, 64), _nhwc(img), 7, 7, 2, 3)[0], conv1.weight.grad, "conv1 dW")
