"""Stand-alone GPU tests of every backbone elementwise / gather kernel and of the dropout sites, each against a plain
torch fp32 formula of the same op (the library ops the reference calls: torchvision/models/resnet.py:143-163 BatchNorm +
ReLU + residual, F.max_pool2d, F.unfold/fold for the strided-conv gathers; nn.Dropout for the head).  All calls go
through the C ABI (virtex_b200.ops.call).  Tolerances: bf16 outputs -> 1 bf16 ulp of the fp32 result (rel 8e-3 on the
tensor norm, and max-abs 2^-7 relative to the largest magnitude); fp32 reductions -> 1e-4 relative.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _ops():
    from virtex_b200 import ops
    return ops


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _s():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(params=["static", "dynamic"])
def schedule(request):
    """Both tile schedules of the persistent GEMM (round robin / per-launch atomic tile counter)."""
    _need_cuda()
    ops = _ops()
    ops.set_dynamic_gemm_schedule(request.param == "dynamic")
    yield request.param
    ops.set_dynamic_gemm_schedule(False)


def _pack_mask(keep):
    """[M, C] bool -> uint8 [M, C/8], bit j of byte g = channel 8g + j (the layout vtx_bn_act writes)."""
    M, C = keep.shape
    w = (1 << torch.arange(8, device=keep.device)).to(torch.int32)
    return (keep.view(M, C // 8, 8).to(torch.int32) * w).sum(-1).to(torch.uint8).contiguous()


def _bnp(C, g, dev="cuda"):
    """[4, C]: mean, invstd, scale = gamma * invstd, shift = beta - mean * scale."""
    mean = torch.randn(C, generator=g) * 0.5
    invstd = torch.rand(C, generator=g) + 0.5
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g) * 0.3
    sc = gamma * invstd
    return torch.stack([mean, invstd, sc, beta - mean * sc]).contiguous().to(dev)


# ------------------------------------------------------------------------------------------------ BN forward family
@pytest.mark.parametrize("M,C,mode", [(1000, 64, "plain"), (777, 256, "res"), (513, 512, "res_bn"), (64, 2048, "plain")])
def test_bn_act_matches_formula(M, C, mode):
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(M + C)
    y = torch.randn(M, C, generator=g).bfloat16().cuda()
    bnp = _bnp(C, g)
    res = torch.randn(M, C, generator=g).bfloat16().cuda() if mode != "plain" else None
    bnp_r = _bnp(C, g) if mode == "res_bn" else None
    out = torch.empty(M, C, dtype=BF16, device="cuda")
    mask = torch.full((M, C // 8), 0xAA, dtype=torch.uint8, device="cuda")
    ops.call("vtx_bn_act", y.data_ptr(), bnp.data_ptr(), ops._p(res), ops._p(bnp_r), out.data_ptr(), mask.data_ptr(), M,
             C, 1, _s())
    ref = y.float() * bnp[2] + bnp[3]
    if mode == "res":
        ref = ref + res.float()
    if mode == "res_bn":
        ref = ref + res.float() * bnp_r[2] + bnp_r[3]
    pre = ref
    ref = ref.clamp_min(0)
    assert rel(out, ref) < 4e-3
    assert (out.float() - ref).abs().max().item() <= 2 ** -7 * ref.abs().max().item()
    # the ReLU bit mask is exactly the sign of the stored activation (what backward used to read), up to fp32 contraction
    # of values within 1e-6 of zero
    got = mask.view(M, C // 8, 1).bitwise_right_shift(torch.arange(8, device="cuda").to(torch.uint8)).bitwise_and(1)
    got = got.view(M, C).bool()
    sure = pre.abs() > 1e-5
    assert torch.equal(got[sure], (pre > 0)[sure])
    assert torch.equal(got, out.float() > 0) or (got != (out.float() > 0)).sum().item() <= 2


def test_bn_finalize_act_fold_matches_batchnorm():
    """sum / sumsq -> (mean, invstd, scale, shift), running-statistics update and apply in one launch == F.batch_norm."""
    _need_cuda()
    ops = _ops()
    M, C = 1536, 128
    g = torch.Generator().manual_seed(1)
    y = (torch.randn(M, C, generator=g) * 2 + 0.5).bfloat16().cuda()
    yf = y.float()
    stats = torch.stack([yf.sum(0), (yf * yf).sum(0)]).contiguous()
    gamma, beta = (torch.rand(C, generator=g) + 0.5).cuda(), torch.randn(C, generator=g).cuda()
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    nbt = torch.zeros(1, dtype=torch.int64, device="cuda")
    bnp = torch.empty(4, C, device="cuda")
    out = torch.empty(M, C, dtype=BF16, device="cuda")
    ops.call("vtx_bn_finalize_act", stats.data_ptr(), float(M), gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(),
             rv.data_ptr(), nbt.data_ptr(), 0.1, 1e-5, 1, bnp.data_ptr(), y.data_ptr(), 0, 0, out.data_ptr(), 0, M, C, 1,
             _s())
    rm_ref, rv_ref = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    ref = F.relu(F.batch_norm(yf, rm_ref, rv_ref, gamma, beta, True, 0.1, 1e-5))
    assert rel(out, ref) < 4e-3
    assert rel(rm, rm_ref) < 1e-4 and rel(rv, rv_ref) < 1e-4
    assert int(nbt) == 1
    assert rel(bnp[0], yf.mean(0)) < 1e-4 and rel(bnp[1], (yf.var(0, unbiased=False) + 1e-5).rsqrt()) < 1e-3


# ------------------------------------------------------------------------------------------------ BN backward family
@pytest.mark.parametrize("M,C,mask", [(2000, 64, "from_a"), (1111, 256, "from_y"), (640, 1024, "none")])
def test_bn_backward_reduce_and_apply_match_autograd(M, C, mask):
    """dz = dA * relu'(.) ; dy = BN-backward(dz) with batch statistics; dgamma / dbeta accumulate."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(M)
    y = (torch.randn(M, C, generator=g) * 1.5).bfloat16().cuda()
    yf = y.float()
    gamma, beta = (torch.rand(C, generator=g) + 0.5).cuda(), (torch.randn(C, generator=g) * 0.3).cuda()
    mean, var = yf.mean(0), yf.var(0, unbiased=False)
    invstd = (var + 1e-5).rsqrt()
    bnp = torch.stack([mean, invstd, gamma * invstd, beta - mean * gamma * invstd]).contiguous()
    dA = (torch.randn(M, C, generator=g) * 0.1).bfloat16().cuda()
    pre = yf * bnp[2] + bnp[3]
    a = _pack_mask(pre > 0) if mask == "from_a" else None  # the bit mask vtx_bn_act writes next to the activation
    if mask == "from_a":
        keep = (pre > 0).float()
    elif mask == "from_y":
        keep = (pre > 0).float()
    else:
        keep = torch.ones_like(pre)
    dz = dA.float() * keep
    sums = torch.zeros(2, C, device="cuda")
    ops.call("vtx_bn_bwd_reduce", dA.data_ptr(), ops._p(a), y.data_ptr(), bnp.data_ptr(), 0, 0, sums.data_ptr(), 0, M,
             C, int(mask == "from_y"), _s())
    xhat = (yf - mean) * invstd
    assert rel(sums[0], dz.sum(0)) < 1e-4
    assert rel(sums[1], (dz * xhat).sum(0)) < 1e-4
    dgamma, dbeta = torch.full((C,), 0.5, device="cuda"), torch.full((C,), -0.25, device="cuda")
    dy = torch.empty(M, C, dtype=BF16, device="cuda")
    dz_out = torch.empty(M, C, dtype=BF16, device="cuda")
    ops.call("vtx_bn_bwd_finalize_apply", sums.data_ptr(), 0, float(M), dgamma.data_ptr(), dbeta.data_ptr(), 0, 0,
             dA.data_ptr(), ops._p(a), y.data_ptr(), bnp.data_ptr(), dy.data_ptr(), 0, 0, 0, dz_out.data_ptr(), M, C,
             int(mask == "from_y"), _s())
    # autograd reference of y -> batch_norm(train) with upstream gradient dz
    yr = yf.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    F.batch_norm(yr, None, None, gr, br, True, 0.0, 1e-5).backward(dz)
    assert rel(dy, yr.grad) < 6e-3
    assert rel(dgamma - 0.5, gr.grad) < 1e-3 and rel(dbeta + 0.25, br.grad) < 1e-3
    assert rel(dz_out, dz) < 1e-6 or mask == "none"  # dz is dA with zeros: exact in bf16


def test_bn_backward_two_branch_variant_shares_dz():
    """bn3 + downsample BN of a transition block: one masked dz feeds both BN backward formulas."""
    _need_cuda()
    ops = _ops()
    M, C = 900, 512
    g = torch.Generator().manual_seed(9)
    ys = [(torch.randn(M, C, generator=g) * s).bfloat16().cuda() for s in (1.0, 2.0)]
    bnps, gammas = [], []
    for y in ys:
        yf = y.float()
        gamma, beta = (torch.rand(C, generator=g) + 0.5).cuda(), (torch.randn(C, generator=g) * 0.3).cuda()
        mean, invstd = yf.mean(0), (yf.var(0, unbiased=False) + 1e-5).rsqrt()
        bnps.append(torch.stack([mean, invstd, gamma * invstd, beta - mean * gamma * invstd]).contiguous())
        gammas.append(gamma)
    pre = ys[0].float() * bnps[0][2] + bnps[0][3] + ys[1].float() * bnps[1][2] + bnps[1][3]
    a = _pack_mask(pre > 0)
    dA = (torch.randn(M, C, generator=g) * 0.1).bfloat16().cuda()
    dz = dA.float() * (pre > 0).float()
    s1, s2 = torch.zeros(2, C, device="cuda"), torch.zeros(2, C, device="cuda")
    ops.call("vtx_bn_bwd_reduce", dA.data_ptr(), a.data_ptr(), ys[0].data_ptr(), bnps[0].data_ptr(), ys[1].data_ptr(),
             bnps[1].data_ptr(), s1.data_ptr(), s2.data_ptr(), M, C, 0, _s())
    dg = [torch.zeros(C, device="cuda") for _ in range(4)]
    dy1, dy2 = torch.empty(M, C, dtype=BF16, device="cuda"), torch.empty(M, C, dtype=BF16, device="cuda")
    ops.call("vtx_bn_bwd_finalize_apply", s1.data_ptr(), s2.data_ptr(), float(M), dg[0].data_ptr(), dg[1].data_ptr(),
             dg[2].data_ptr(), dg[3].data_ptr(), dA.data_ptr(), a.data_ptr(), ys[0].data_ptr(), bnps[0].data_ptr(),
             dy1.data_ptr(), ys[1].data_ptr(), bnps[1].data_ptr(), dy2.data_ptr(), 0, M, C, 0, _s())
    for y, gamma, dy, dgam, dbet in ((ys[0], gammas[0], dy1, dg[0], dg[1]), (ys[1], gammas[1], dy2, dg[2], dg[3])):
        yr = y.float().clone().requires_grad_(True)
        gr = gamma.clone().requires_grad_(True)
        br = torch.zeros(C, device="cuda", requires_grad=True)
        F.batch_norm(yr, None, None, gr, br, True, 0.0, 1e-5).backward(dz)
        assert rel(dy, yr.grad) < 6e-3
        assert rel(dgam, gr.grad) < 1e-3 and rel(dbet, br.grad) < 1e-3


# ------------------------------------------------------------------------------------------------ stem pooling pair
@pytest.mark.parametrize("N,H,W,C", [(3, 112, 112, 64), (2, 30, 22, 64), (2, 7, 9, 64)])
def test_bn_relu_maxpool_and_backward_match_torch(N, H, W, C):
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(H * W)
    y = torch.randn(N * H * W, C, generator=g).bfloat16().cuda()
    bnp = _bnp(C, g)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = torch.empty(N * Ho * Wo, C, dtype=BF16, device="cuda")
    idx = torch.empty(N * Ho * Wo, C, dtype=torch.uint8, device="cuda")
    ops.call("vtx_bn_relu_maxpool", y.data_ptr(), bnp.data_ptr(), out.data_ptr(), idx.data_ptr(), N, H, W, C, _s())
    # the kernel pools the bf16-ROUNDED activation (what a separate bn_act pass would have stored)
    act = (y.float() * bnp[2] + bnp[3]).clamp_min(0).bfloat16().float()
    act_nchw = act.view(N, H, W, C).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    ref = F.max_pool2d(act_nchw, 3, 2, 1)
    ref_nhwc = ref.permute(0, 2, 3, 1).reshape(N * Ho * Wo, C)
    # the kernel evaluates y*scale + shift as one fma, eager torch as mul + add: the fp32 values differ in the last bit
    # and a handful of the 2.4 M elements round to the neighbouring bf16 value
    d = (out.float() - ref_nhwc.detach()).abs()
    assert (d > 0).float().mean().item() < 1e-3 and (d <= 2 ** -7 * ref_nhwc.detach().abs().clamp_min(1e-3)).all()
    dpool = torch.randn(N * Ho * Wo, C, generator=g).bfloat16().cuda()
    da = torch.empty(N * H * W, C, dtype=BF16, device="cuda")
    ops.call("vtx_maxpool_bwd", dpool.data_ptr(), idx.data_ptr(), da.data_ptr(), N, H, W, C, _s())
    # window scan order and the strict `>` comparison are those of ATen's max_pool2d: ties (several zeros after the
    # ReLU in one window) go to the first element in (kh, kw) order in both, so the gradients agree element-wise
    ref.backward(dpool.float().view(N, Ho, Wo, C).permute(0, 3, 1, 2))
    ref_da = act_nchw.grad.permute(0, 2, 3, 1).reshape(N * H * W, C)
    assert rel(da, ref_da) < 3e-2  # the few last-bit flips above move a window's gradient to a neighbouring position
    assert rel(da.float().view(N, H * W, C).sum(1), dpool.float().view(N, Ho * Wo, C).sum(1)) < 2e-2  # mass conserved


# ------------------------------------------------------------------------------------------------ strided-conv gathers
@pytest.mark.parametrize("N,H,W,C,stride", [(2, 14, 14, 128, 2), (3, 9, 11, 64, 2), (2, 8, 8, 64, 1)])
def test_im2col3x3_col2im3x3_match_unfold_fold(N, H, W, C, stride):
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(H + W)
    x = torch.randn(N, H, W, C, generator=g).bfloat16().cuda()
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    cols = torch.empty(N * Ho * Wo, 9 * C, dtype=BF16, device="cuda")
    ops.call("vtx_im2col3x3", x.data_ptr(), cols.data_ptr(), N, H, W, C, stride, _s())
    unf = F.unfold(x.float().permute(0, 3, 1, 2), 3, padding=1, stride=stride)          # [N, C*9, L], k = c*9 + tap
    ref = unf.view(N, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(N * Ho * Wo, 9 * C)     # k = tap*C + c
    assert torch.equal(cols.float(), ref)
    dcols = torch.randn(N * Ho * Wo, 9 * C, generator=g).bfloat16().cuda()
    dx = torch.empty(N, H, W, C, dtype=BF16, device="cuda")
    ops.call("vtx_col2im3x3", dcols.data_ptr(), dx.data_ptr(), N, H, W, C, stride, _s())
    d = dcols.float().view(N, Ho * Wo, 9, C).permute(0, 3, 2, 1).reshape(N, C * 9, Ho * Wo)
    ref_dx = F.fold(d, (H, W), 3, padding=1, stride=stride).permute(0, 2, 3, 1)
    assert rel(dx, ref_dx) < 4e-3


@pytest.mark.parametrize("N,H,W,C", [(2, 14, 14, 256), (3, 7, 9, 64)])
def test_subsample_upsample_add_match_slicing(N, H, W, C):
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(C)
    x = torch.randn(N, H, W, C, generator=g).bfloat16().cuda()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xs = torch.empty(N, Ho, Wo, C, dtype=BF16, device="cuda")
    ops.call("vtx_subsample", x.data_ptr(), xs.data_ptr(), N, H, W, C, 2, _s())
    assert torch.equal(xs, x[:, ::2, ::2])
    dxs = torch.randn(N, Ho, Wo, C, generator=g).bfloat16().cuda()
    dx = torch.randn(N, H, W, C, generator=g).bfloat16().cuda()
    ref = dx.float().clone()
    ref[:, ::2, ::2] += dxs.float()
    ops.call("vtx_upsample_add", dxs.data_ptr(), dx.data_ptr(), N, H, W, C, 2, _s())
    assert rel(dx, ref) < 4e-3


# ------------------------------------------------------------------------------------------------ dropout sites
def _seed(v):
    return torch.tensor([v], dtype=torch.int64, device="cuda")


def test_gelu_dropout_keep_rate_scaling_and_mask_agreement():
    """nn.Dropout semantics (embedding.py:46, transformer.py:1173-1199): keep rate 1-p within 3 sigma, kept values
    scaled by 1/(1-p) (so E[out] = gelu(u)), and backward applies the SAME mask as forward."""
    _need_cuda()
    ops = _ops()
    n, p = 1 << 20, 0.1
    g = torch.Generator().manual_seed(0)
    u = (torch.randn(n, generator=g) + 1.5).bfloat16().cuda()
    h = torch.empty(n, dtype=BF16, device="cuda")
    seed = _seed(77)
    ops.call("vtx_gelu_dropout_fwd", u.data_ptr(), h.data_ptr(), n, p, seed.data_ptr(), 14, _s())
    gl = F.gelu(u.float())
    nz = gl.abs() > 1e-3
    kept = (h.float() != 0) & nz
    rate = kept.sum().item() / nz.sum().item()
    sigma = math.sqrt(p * (1 - p) / nz.sum().item())
    assert abs(rate - (1 - p)) < 3 * sigma + 1e-4, (rate, sigma)
    assert rel(h.float()[kept], gl[kept] / (1 - p)) < 4e-3
    assert abs(h.float().mean().item() - gl.mean().item()) < 4 * gl.std().item() * math.sqrt(p / (1 - p) / n) + 2e-3
    # same seed, same site -> identical mask; different seed -> different mask
    h2 = torch.empty_like(h)
    ops.call("vtx_gelu_dropout_fwd", u.data_ptr(), h2.data_ptr(), n, p, seed.data_ptr(), 14, _s())
    assert torch.equal(h, h2)
    seed2 = _seed(78)
    ops.call("vtx_gelu_dropout_fwd", u.data_ptr(), h2.data_ptr(), n, p, seed2.data_ptr(), 14, _s())
    assert not torch.equal(h, h2)
    # backward of ones: du = mask/(1-p) * gelu'(u): zero exactly where forward dropped
    dh = torch.ones(n, dtype=BF16, device="cuda")
    du = torch.empty(n, dtype=BF16, device="cuda")
    ops.call("vtx_gelu_dropout_bwd", dh.data_ptr(), u.data_ptr(), du.data_ptr(), n, p, seed.data_ptr(), 14, _s())
    uf = u.float().requires_grad_(True)
    F.gelu(uf).sum().backward()
    mask = (h.float() != 0).float()
    chk = nz & (uf.grad.abs() > 1e-2)
    assert torch.equal((du.float() != 0)[chk], mask.bool()[chk])
    assert rel(du.float()[chk], (uf.grad * mask / (1 - p))[chk]) < 6e-3


def test_residual_dropout_layernorm_site_is_unbiased_and_replayed_in_backward():
    """z = res + dropout(branch) (transformer.py:1131-1143): statistics of the mask, and ln_bwd's d_branch uses it."""
    _need_cuda()
    ops = _ops()
    M, H, p = 2048, 256, 0.1
    g = torch.Generator().manual_seed(3)
    res = torch.zeros(M, H, device="cuda")
    branch = torch.ones(M, H, dtype=BF16, device="cuda")
    z = torch.empty(M, H, device="cuda")
    seed = _seed(5)
    ops.call("vtx_add_ln_fwd", res.data_ptr(), branch.data_ptr(), 0, 0, z.data_ptr(), 0, 0, 0, M, H, 0.0, p,
             seed.data_ptr(), 21, 0, _s())
    n = M * H
    rate = (z != 0).float().mean().item()
    assert abs(rate - (1 - p)) < 3 * math.sqrt(p * (1 - p) / n) + 1e-4
    vals = z[z != 0]
    assert (vals - 1 / (1 - p)).abs().max().item() < 1e-5
    assert abs(z.mean().item() - 1.0) < 4 * math.sqrt(p / (1 - p) / n) + 1e-4
    # backward through the same site: d_branch = dy * mask / (1-p)
    dy = torch.ones(M, H, device="cuda")
    d_branch = torch.empty(M, H, dtype=BF16, device="cuda")
    ops.call("vtx_ln_bwd", dy.data_ptr(), 0, 0, 0, 0, 0, 0, d_branch.data_ptr(), 0, 0, M, H, p, seed.data_ptr(), 21, 0,
             _s())
    assert rel(d_branch.float(), z) < 4e-3
    assert torch.equal(d_branch.float() != 0, z != 0)


def test_attention_dropout_keeps_rows_normalised_in_expectation():
    """Attention-probability dropout (functional.py:6608-6682): E[out] equals the p = 0 output."""
    _need_cuda()
    ops = _ops()
    B, A, T = 64, 4, 30
    H = A * 64
    g = torch.Generator().manual_seed(2)
    qkv = (torch.randn(B * T, 3 * H, generator=g) * 0.5).bfloat16().cuda()
    lengths = torch.full((B,), T, dtype=torch.int64, device="cuda")
    lse = torch.empty(B * A * 32, device="cuda")
    outs = []
    for p, sd in ((0.0, 1), (0.1, 1), (0.1, 2), (0.1, 3), (0.1, 4)):
        o = torch.empty(B * T, H, dtype=BF16, device="cuda")
        seed = _seed(sd)
        ops.call("vtx_attn_fwd", qkv.data_ptr(), 3 * H, qkv.data_ptr() + 2 * H, 3 * H, qkv.data_ptr() + 4 * H, 3 * H,
                 o.data_ptr(), H, lse.data_ptr(), B, A, T, T, lengths.data_ptr(), 1, p, seed.data_ptr(), 7, _s())
        outs.append(o.float())
    base = outs[0]
    mean_drop = sum(outs[1:]) / 4
    assert not torch.equal(outs[1], outs[2])
    # the average over 4 independent masks is closer to the p = 0 output than any single draw, and unbiased overall
    assert rel(mean_drop, base) < rel(outs[1], base)
    assert abs((mean_drop - base).mean().item()) < 5e-3


# ------------------------------------------------------------------------------------------------ weight-layout jobs
def test_batched_weight_jobs_match_the_per_tensor_kernels():
    """vtx_conv_w_jobs (one launch, device job table) == vtx_conv_w_pack / _pack_dgrad / _unpack_add / _unpack_add_t /
    vtx_stem_s2d_w_pack / _unpack_add, bit for bit, including the OIHW <-> [O, (kh,kw,I)] index maps vs torch.permute."""
    _need_cuda()
    import struct
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    dev = "cuda"
    w3 = torch.randn(128, 128, 3, 3, generator=g).to(dev)
    w7 = torch.randn(64, 3, 7, 7, generator=g).to(dev)
    dwp3 = torch.randn(128, 1152, generator=g).to(dev)
    dwt3 = torch.randn(1152, 128, generator=g).to(dev)
    dw7 = torch.randn(64, 256, generator=g).to(dev)
    dw7c = torch.randn(64, 160, generator=g).to(dev)
    outs = {k: torch.full(shape, 3.0, dtype=dt, device=dev) for k, (shape, dt) in {
        "p3": ((128, 1152), BF16), "pd3": ((128, 1152), BF16), "p7": ((64, 160), BF16), "ps2d": ((64, 256), BF16),
        "g3": ((128, 128, 3, 3), F32), "g3t": ((128, 128, 3, 3), F32), "g7": ((64, 3, 7, 7), F32),
        "g7c": ((64, 3, 7, 7), F32)}.items()}
    rows = [(w3, outs["p3"], 128 * 1152, 128, 128, 3, 3, 1152, 0), (w3, outs["pd3"], 128 * 1152, 128, 128, 3, 3, 1152, 1),
            (w7, outs["p7"], 64 * 160, 64, 3, 7, 7, 160, 0), (w7, outs["ps2d"], 64 * 256, 64, 3, 7, 7, 256, 4),
            (dwp3, outs["g3"], 128 * 1152, 128, 128, 3, 3, 1152, 2), (dwt3, outs["g3t"], 128 * 1152, 128, 128, 3, 3, 1152, 3),
            (dw7, outs["g7"], 64 * 147, 64, 3, 7, 7, 256, 5), (dw7c, outs["g7c"], 64 * 147, 64, 3, 7, 7, 160, 2)]
    blk = ops.L.load().vtx_weight_job_block_elems()
    blob, b0 = b"", 0
    for src, dst, total, O, I, KH, KW, ldk, kind in rows:
        blob += struct.pack("<QQq8i", src.data_ptr(), dst.data_ptr(), total, O, I, KH, KW, ldk, kind, b0, 0)
        b0 += (total + blk - 1) // blk
    table = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(dev)
    ops.call("vtx_conv_w_jobs", table.data_ptr(), len(rows), b0, _s())
    # references: torch index maps
    assert torch.equal(outs["p3"], w3.permute(0, 2, 3, 1).reshape(128, 1152).bfloat16())
    assert torch.equal(outs["pd3"], w3.flip(2, 3).permute(1, 2, 3, 0).reshape(128, 1152).bfloat16())
    ref7 = torch.zeros(64, 160, device=dev)
    ref7[:, :147] = w7.permute(0, 2, 3, 1).reshape(64, 147)
    assert torch.equal(outs["p7"], ref7.bfloat16())
    assert torch.equal(outs["g3"], 3.0 + dwp3.view(128, 3, 3, 128).permute(0, 3, 1, 2))
    assert torch.equal(outs["g3t"], 3.0 + dwt3.view(3, 3, 128, 128).permute(3, 2, 0, 1))
    assert torch.equal(outs["g7c"], 3.0 + dw7c[:, :147].reshape(64, 7, 7, 3).permute(0, 3, 1, 2))
    # stem s2d maps: against the per-tensor kernels of csrc/stem_s2d.cu
    ps = torch.empty(64, 256, dtype=BF16, device=dev)
    ops.call("vtx_stem_s2d_w_pack", w7.data_ptr(), ps.data_ptr(), 64, _s())
    assert torch.equal(outs["ps2d"], ps)
    g7 = torch.full((64, 3, 7, 7), 3.0, device=dev)
    ops.call("vtx_stem_s2d_w_unpack_add", dw7.data_ptr(), g7.data_ptr(), 64, _s())
    assert torch.equal(outs["g7"], g7)


def test_gemm_masked_residual_epilogue():
    """D = A.B^T + residual * [mask bit]: the shortcut gradient of a bottleneck (dz = dOut * [out > 0]) added by the
    conv1-dgrad epilogue without dz ever being materialised; TMA-staged and direct residual paths."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(11)
    for M, N, K, b_mn in ((1000, 256, 64, 1), (777, 64, 256, 1), (300, 1024, 256, 0)):
        A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
        B = (torch.randn(K, N, generator=g) * 0.5).bfloat16().cuda() if b_mn else \
            (torch.randn(N, K, generator=g) * 0.5).bfloat16().cuda()
        R = torch.randn(M, N, generator=g).bfloat16().cuda()
        keep = (torch.rand(M, N, generator=g) > 0.4).cuda()
        mask = _pack_mask(keep)
        D = torch.empty(M, N, dtype=BF16, device="cuda")
        ops.gemm(A, B, D, M, N, K, b_mn=b_mn, residual=R, residual_mask=mask)
        ref = A.float() @ (B.float() if b_mn else B.float().t()) + R.float() * keep.float()
        assert rel(D, ref) < 4e-3, (M, N, K)
        D2 = torch.empty(M, N, dtype=BF16, device="cuda")
        ops.gemm(A, B, D2, M, N, K, b_mn=b_mn, residual=R)  # no mask: plain residual add, unchanged
        assert rel(D2, A.float() @ (B.float() if b_mn else B.float().t()) + R.float()) < 4e-3


@pytest.mark.parametrize("M,N,K,tile_n", [
    (60000, 64, 64, 0),      # 64-wide tiles, two staging buffers, 3+ tiles per CTA
    (19077, 64, 192, 0),     # same, ragged last M tile, odd tile count per CTA
    (150, 64, 64, 0),        # two tiles in the whole launch: most CTAs idle
    (60000, 128, 64, 0),     # 128-wide tiles
    (40000, 256, 128, 0),    # 256-wide tiles
    (30011, 96, 64, 0),      # width that is not a multiple of 64
    (20000, 200, 64, 0),     # partial last column tile
    (30000, 256, 64, 128),   # forced 128-wide tiles over two column blocks (statistics flushed on block changes)
    (20000, 1024, 128, 0),   # four column blocks with statistics: the schedule runs over the row tiles first (nt_major)
    (9000, 2048, 64, 0),     # eight column blocks, 568 tiles: the tile counter hands most CTAs three or four tiles
])
def test_gemm_epilogue_configurations_many_tiles(M, N, K, tile_n, schedule):
    """Every epilogue configuration of the GEMM kernel (wgmma width and staging buffers depend on the tile width)
    on launches with several tiles per CTA: output, BN statistics of the bf16-rounded output, and the packed residual path."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(M + N)
    A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
    B = (torch.randn(N, K, generator=g) * 0.5).bfloat16().cuda()
    ref = A.float() @ B.float().t()
    D = torch.full((M + 8, N), 7.0, dtype=BF16, device="cuda")
    st = torch.zeros(2, N, device="cuda")
    ops.gemm(A, B, D, M, N, K, stats=st, tile_n=tile_n)
    out = D[:M]
    assert rel(out, ref) < 4e-3
    assert torch.all(D[M:] == 7.0)
    assert rel(st[0], out.double().sum(0)) < 1e-4 and rel(st[1], (out.double() ** 2).sum(0)) < 1e-4
    ops.gemm(A, B, D, M, N, K, bias=torch.ones(N, device="cuda"), act=1, tile_n=tile_n)   # fp32 epilogue math path
    assert rel(D[:M], torch.relu(ref + 1.0)) < 4e-3
    R = torch.randn(M, N, generator=g).bfloat16().cuda()
    ops.gemm(A, B, D, M, N, K, residual=R, tile_n=tile_n)
    assert rel(D[:M], ref + R.float()) < 4e-3
    if N % 32 == 0:
        keep = (torch.rand(M, N, generator=g) > 0.5).cuda()
        ops.gemm(A, B, D, M, N, K, residual=R, residual_mask=_pack_mask(keep), tile_n=tile_n)
        assert rel(D[:M], ref + R.float() * keep.float()) < 4e-3
    Df = torch.zeros(M, N, device="cuda")
    ops.gemm(A, B, Df, M, N, K, out_f32=True, tile_n=tile_n)                                # unstaged fp32 output
    assert rel(Df, ref) < 1e-5


def _bn_reduce_ref(ops, D, y, bnp, mask_bits):
    """The stand-alone reduction (vtx_bn_bwd_reduce) and the torch formula over the SAME bf16 gradient D."""
    M, C = D.shape
    sums = torch.zeros(2, C, device="cuda")
    ops.call("vtx_bn_bwd_reduce", D.data_ptr(), ops._p(mask_bits), y.data_ptr(), bnp.data_ptr(), 0, 0, sums.data_ptr(), 0,
             M, C, int(mask_bits is None), _s())
    return sums


def _check_bnr(ops, D, y, bnp, sums, mask_bits, keep):
    ref = _bn_reduce_ref(ops, D, y, bnp, mask_bits)
    dz = D.double() * keep.double()
    xhat = (y.double() - bnp[0].double()) * bnp[1].double()
    assert rel(sums[0], dz.sum(0)) < 1e-4 and rel(sums[1], (dz * xhat).sum(0)) < 1e-4
    assert rel(sums, ref) < 1e-4


@pytest.mark.parametrize("M,N,K", [(5000, 64, 256), (5001, 128, 512), (20000, 256, 64), (3000, 512, 128), (700, 2048, 64)])
def test_gemm_fused_bn_backward_reduce_plain(M, N, K, schedule):
    """VtxGemm.bnr_*: the dgrad epilogue accumulates sum dz / sum dz * xhat of its own output (conv3 dgrad -> bn2: ReLU
    mask recomputed from y; conv1 dgrad + shortcut gradient -> previous block's bn3: ReLU bit mask), D itself unchanged;
    against vtx_bn_bwd_reduce over the same D and the torch formula."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(M + N + K)
    A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
    B = (torch.randn(K, N, generator=g) * 0.2).bfloat16().cuda()
    y = (torch.randn(M, N, generator=g) * 1.5).bfloat16().cuda()
    bnp = _bnp(N, g)
    # --- mask recomputed from y
    D0 = torch.empty(M, N, dtype=BF16, device="cuda")
    ops.gemm(A, B, D0, M, N, K, b_mn=1)
    D = torch.empty(M, N, dtype=BF16, device="cuda")
    sums = torch.zeros(2, N, device="cuda")
    ops.gemm(A, B, D, M, N, K, b_mn=1, bnr=(y, bnp, sums, None))
    assert torch.equal(D, D0)
    keep = (y.float() * bnp[2] + bnp[3]) > 0
    _check_bnr(ops, D, y, bnp, sums, None, keep)
    # --- bit mask, on top of the masked-residual epilogue (the shape of the conv1 dgrad of an identity block)
    if N % 32 == 0:
        R = torch.randn(M, N, generator=g).bfloat16().cuda()
        rkeep = (torch.rand(M, N, generator=g) > 0.5).cuda()
        bkeep = (torch.rand(M, N, generator=g) > 0.45).cuda()
        rbits, bbits = _pack_mask(rkeep), _pack_mask(bkeep)
        ops.gemm(A, B, D0, M, N, K, b_mn=1, residual=R, residual_mask=rbits)
        sums.zero_()
        ops.gemm(A, B, D, M, N, K, b_mn=1, residual=R, residual_mask=rbits, bnr=(y, bnp, sums, bbits))
        assert torch.equal(D, D0)
        _check_bnr(ops, D, y, bnp, sums, bbits, bkeep)


@pytest.mark.parametrize("NI,H,W,C", [(4, 14, 14, 128), (3, 56, 56, 64), (2, 30, 22, 64), (6, 7, 7, 256)])
def test_gemm_fused_bn_backward_reduce_conv_dgrad(NI, H, W, C, schedule):
    """The same through the implicit 3x3 dgrad (conv2 dgrad -> bn1), including 64-channel layers whose partial
    spatial tiles have rows outside the image."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(H * W + C)
    M = NI * H * W
    dy = (torch.randn(NI, H, W, C, generator=g) * 0.5).bfloat16().cuda()
    wq = (torch.randn(C, 9 * C, generator=g) * 0.05).bfloat16().cuda()
    y = (torch.randn(M, C, generator=g) * 1.5).bfloat16().cuda()
    bnp = _bnp(C, g)
    D0 = torch.empty(M, C, dtype=BF16, device="cuda")
    ops.gemm(dy, wq, D0, M, C, 9 * C, lda=C, conv=(NI, H, W, C), conv_mode=1)
    D = torch.empty(M, C, dtype=BF16, device="cuda")
    sums = torch.zeros(2, C, device="cuda")
    ops.gemm(dy, wq, D, M, C, 9 * C, lda=C, conv=(NI, H, W, C), conv_mode=1, bnr=(y, bnp, sums, None))
    assert torch.equal(D, D0)
    _check_bnr(ops, D, y, bnp, sums, None, (y.float() * bnp[2] + bnp[3]) > 0)


@pytest.mark.parametrize("NI,H,W,C,Cout", [(8, 28, 28, 128, 128), (3, 13, 15, 64, 128)])
def test_gemm_fused_bn_backward_reduce_strided_parity_classes(NI, H, W, C, Cout):
    """Stride-2 dgrad as four parity-class GEMMs writing strided sub-grids of dx: each accumulates the sums of ITS
    sub-grid (y addressed through the same view), together the reduction over all of dx."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(H + W + C + 1)
    w = (torch.randn(Cout, C, 3, 3, generator=g) * 0.05).bfloat16().cuda()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dy = (torch.randn(NI, Ho, Wo, Cout, generator=g) * 0.5).bfloat16().cuda()
    y = (torch.randn(NI * H * W, C, generator=g) * 1.5).bfloat16().cuda()
    bnp = _bnp(C, g)
    outs = []
    for fused in (False, True):
        dx = torch.full((NI, H, W, C), 9.0, dtype=BF16, device="cuda")
        sums = torch.zeros(2, C, device="cuda")
        for ph in (0, 1):
            for pw in (0, 1):
                th, tw = 1 + ph, 1 + pw
                taps = [w.float()[:, :, ph + 1 - 2 * a, pw + 1 - 2 * b].t() for a in range(th) for b in range(tw)]
                wc = torch.cat(taps, dim=1).bfloat16().contiguous()
                Hs, Ws = (H - ph + 1) // 2, (W - pw + 1) // 2
                voff = (ph * W + pw) * C * 2
                ops.gemm(dy, wc, dx, NI * Ho * Wo, C, th * tw * Cout, lda=Cout, conv=(NI, Ho, Wo, Cout), conv_mode=1,
                         tap_grid=(th, tw, 0), d_ptr=dx.data_ptr() + voff, out_view=(Hs, Ws, 2 * C, 2 * W * C, H * W * C),
                         bnr=(y, bnp, sums, None, y.data_ptr() + voff) if fused else None)
        outs.append((dx, sums))
    assert torch.equal(outs[0][0], outs[1][0])
    D = outs[1][0].view(-1, C)
    _check_bnr(ops, D, y, bnp, outs[1][1], None, (y.float() * bnp[2] + bnp[3]) > 0)


@pytest.mark.parametrize("N", [256, 512, 1024])
def test_gemm_fused_bn_backward_reduce_over_residual_is_exact_for_every_tile_count(N):
    """The fused reduction over the TMA-staged residual tile (conv1 dgrad + shortcut gradient -> the previous block's bn3)
    across launches with 1, 1-2, 2-3 ... tiles per CTA and one to four column blocks: the bf16 output must equal the
    plain epilogue's bit for bit (the statistics pass only READS the staged tile; the register sums leave through the
    staging buffer BEFORE the next residual tile is requested into it), and the sums must match the stand-alone pass."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(N)
    K = 64
    sms = ops.num_sms()
    for tiles in (sms - 9, sms + 1, sms + 9, 2 * sms - 3, 2 * sms + 20, 3 * sms + 5):
        M = tiles * 128 - 37
        A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
        B = (torch.randn(K, N, generator=g) * 0.2).bfloat16().cuda()
        y = (torch.randn(M, N, generator=g) * 1.5).bfloat16().cuda()
        bnp = _bnp(N, g)
        R = torch.randn(M, N, generator=g).bfloat16().cuda()
        rbits = _pack_mask((torch.rand(M, N, generator=g) > 0.5).cuda())
        bkeep = (torch.rand(M, N, generator=g) > 0.45).cuda()
        bbits = _pack_mask(bkeep)
        for kw in (dict(residual=R, residual_mask=rbits), dict(residual=R)):
            D0 = torch.full((M, N), 7.0, dtype=BF16, device="cuda")
            ops.gemm(A, B, D0, M, N, K, b_mn=1, **kw)
            for mask in (bbits, None):
                D = torch.full((M, N), 7.0, dtype=BF16, device="cuda")
                sums = torch.zeros(2, N, device="cuda")
                ops.gemm(A, B, D, M, N, K, b_mn=1, bnr=(y, bnp, sums, mask), **kw)
                assert torch.equal(D, D0), (tiles, N, mask is None)
                _check_bnr(ops, D, y, bnp, sums, mask, bkeep if mask is not None else (y.float() * bnp[2] + bnp[3]) > 0)


def _both_schedules(ops, run):
    """run() under the static round-robin and the dynamic tile-counter schedule: {False: static, True: dynamic}."""
    outs = {}
    try:
        for dynamic in (False, True):
            ops.set_dynamic_gemm_schedule(dynamic)
            outs[dynamic] = run()
    finally:
        ops.set_dynamic_gemm_schedule(False)
    return outs


@pytest.mark.parametrize("M,N,K", [(7680, 1024, 1024), (1000, 256, 512), (896, 10000, 256), (50176, 256, 1024), (641, 384, 320)])
def test_gemm_cta_pairs_match_single_cta_and_torch(M, N, K):
    """Long-K and wide shapes that split into many tiles per CTA (the shapes the Blackwell build ran as 2-CTA pairs; every
    tile is one CTA here): every operand layout (K-major / MN-major A and B, split-K fp32 atomics), a partial last row
    tile, bias / activation / residual / statistics / fused BN-backward sums -- against torch, and the static tile
    schedule against the dynamic tile counter, which hands the same tiles to CTAs in another order."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(M + N)
    A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
    B = (torch.randn(N, K, generator=g) * 0.1).bfloat16().cuda()
    Bt = B.t().contiguous()                      # [K, N]: MN-major B
    At = A.t().contiguous()                      # [K, M]: MN-major A
    ref = A.float() @ B.float().t()
    bias = torch.randn(N, generator=g).cuda()
    R = torch.randn(M, N, generator=g).bfloat16().cuda()
    y = (torch.randn(M, N, generator=g) * 1.5).bfloat16().cuda()
    bnp = _bnp(N, g)

    def run():
        D1 = torch.empty(M, N, dtype=BF16, device="cuda")
        st = torch.zeros(2, N, device="cuda")
        ops.gemm(A, B, D1, M, N, K, stats=st)
        D2 = torch.empty(M, N, dtype=BF16, device="cuda")
        ops.gemm(A, Bt, D2, M, N, K, b_mn=1, bias=bias, act=1)
        D3 = torch.zeros(M, N, dtype=BF16, device="cuda")
        sums = torch.zeros(2, N, device="cuda")
        if N % 32 == 0:
            ops.gemm(A, Bt, D3, M, N, K, b_mn=1, residual=R, bnr=(y, bnp, sums, None))
        D4 = torch.zeros(M, N, device="cuda")
        if M % 8 == 0:
            ops.gemm(At, Bt, D4, M, N, K, a_mn=1, b_mn=1, atomic=True, split_k=2, out_f32=True)
        return D1, st, D2, D3, sums, D4

    outs = _both_schedules(ops, run)
    D1, st, D2, D3, sums, D4 = outs[False]
    assert rel(D1, ref) < 4e-3 and rel(D2, torch.relu(ref + bias)) < 4e-3
    assert rel(st[0], D1.double().sum(0)) < 1e-4 and rel(st[1], (D1.double() ** 2).sum(0)) < 1e-4
    if N % 32 == 0:
        assert rel(D3, ref + R.float()) < 4e-3
        _check_bnr(ops, D3, y, bnp, sums, None, (y.float() * bnp[2] + bnp[3]) > 0)
    if M % 8 == 0:
        assert rel(D4, ref) < 1e-4
    for a, b in zip(outs[False], outs[True]):
        assert rel(a, b) < (2e-3 if a.dtype == BF16 else 1e-4)   # (bf16: at most a few last-bit flips)


@pytest.mark.parametrize("NI,H,W,C,Cout", [(16, 14, 14, 256, 256), (9, 7, 7, 512, 512), (5, 28, 28, 128, 128)])
def test_gemm_cta_pairs_implicit_conv(NI, H, W, C, Cout):
    """The implicit 3x3 convolution modes on 128- to 512-channel layers (the shapes the Blackwell build ran as 2-CTA
    pairs): fprop (4-D activation boxes, K-major weight tiles, BN statistics) and split-K wgrad (every 64-column atom of
    the (tap, cin) columns gathered by its own box) -- against torch, under both tile schedules."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(H + C)
    M = NI * H * W
    x = (torch.randn(NI, H, W, C, generator=g) * 0.5).bfloat16().cuda()
    w = (torch.randn(Cout, 3, 3, C, generator=g) * 0.03).bfloat16().cuda()
    dy = (torch.randn(NI, H, W, Cout, generator=g) * 0.5).bfloat16().cuda()

    def run():
        yo = torch.empty(M, Cout, dtype=BF16, device="cuda")
        st = torch.zeros(2, Cout, device="cuda")
        ops.gemm(x, w.view(Cout, 9 * C), yo, M, Cout, 9 * C, lda=C, stats=st, conv=(NI, H, W, C), conv_mode=1)
        dw = torch.zeros(Cout, 9 * C, device="cuda")
        ops.gemm(dy, x, dw, Cout, 9 * C, M, atomic=True, split_k=2, lda=Cout, ldb=C, conv=(NI, H, W, C), conv_mode=2,
                 out_f32=True)
        return yo, st, dw

    outs = _both_schedules(ops, run)
    yo, st, dw = outs[False]
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1).reshape(M, Cout)
    assert rel(yo, ref) < 4e-3
    assert rel(st[0], yo.double().sum(0)) < 1e-4
    dwr = torch.nn.grad.conv2d_weight(x.float().permute(0, 3, 1, 2), (Cout, C, 3, 3), dy.float().permute(0, 3, 1, 2), padding=1)
    assert rel(dw.view(Cout, 3, 3, C), dwr.permute(0, 2, 3, 1)) < 2e-3
    assert rel(outs[True][0], outs[False][0]) < 2e-3 and rel(outs[True][2], outs[False][2]) < 1e-4


def test_gemm_tile_counter_windows_stay_in_step():
    """The dynamic tile scheduler takes its tiles from a ring of 4096 ever-growing counters whose per-launch windows the
    host keeps track of: more launches than counters (of alternating sizes and chunk widths, so that a window that is
    off by one fetch would skip or repeat tiles) stay exact."""
    _need_cuda()
    ops = _ops()
    ops.set_dynamic_gemm_schedule(True)
    try:
        _tile_counter_windows(ops)
    finally:
        ops.set_dynamic_gemm_schedule(False)


def _tile_counter_windows(ops):
    g = torch.Generator().manual_seed(3)
    shapes = [(700, 64, 64), (40000, 64, 64), (3000, 256, 128), (700000, 64, 64), (250000, 64, 64)]  # chunks of 1, 4, 2 tiles
    data = []
    for M, N, K in shapes:
        A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
        B = (torch.randn(N, K, generator=g) * 0.5).bfloat16().cuda()
        data.append((A, B, torch.empty(M, N, dtype=BF16, device="cuda"), A.float() @ B.float().t()))
    for i in range(4400):
        A, B, D, _ = data[i % 3] if i % 40 else data[3 + (i // 40) % 2]
        ops.gemm(A, B, D, A.shape[0], B.shape[0], A.shape[1])
        if i % 1100 == 1099:
            for A, B, D, ref in data:
                assert rel(D, ref) < 4e-3, i
            for _, _, D, _ in data:
                D.zero_()
    for j, (A, B, D, ref) in enumerate(data):
        ops.gemm(A, B, D, A.shape[0], B.shape[0], A.shape[1])
        assert rel(D, ref) < 4e-3, j


# ------------------------------------------------------------------------------------------------ strided implicit convs
@pytest.mark.parametrize("NI,H,W,C,Cout", [(8, 28, 28, 128, 128), (4, 14, 14, 256, 256), (6, 13, 15, 64, 128)])
def test_strided_implicit_conv3x3_fprop_and_wgrad(NI, H, W, C, Cout):
    """3x3 / stride 2 / pad 1 (torchvision resnet.py:133-138, first block of layers 2-4) as implicit GEMMs whose gather
    uses TMA traversal strides: fprop (+ BN statistics) vs F.conv2d, weight gradient vs conv2d_weight."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(H * W + C)
    x = (torch.randn(NI, H, W, C, generator=g) * 0.5).bfloat16().cuda()
    w = (torch.randn(Cout, C, 3, 3, generator=g) * 0.05).bfloat16().cuda()
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * C).contiguous()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    M = NI * Ho * Wo
    y = torch.full((M + 16, Cout), 7.0, dtype=BF16, device="cuda")
    st = torch.zeros(2, Cout, device="cuda")
    ops.gemm(x, wp, y, M, Cout, 9 * C, lda=C, stats=st, conv=(NI, H, W, C), conv_mode=1, conv_stride=2)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), stride=2, padding=1).permute(0, 2, 3, 1).reshape(M, Cout)
    assert rel(y[:M], ref) < 4e-3
    assert torch.all(y[M:] == 7.0)
    assert rel(st[0], y[:M].float().sum(0)) < 2e-3 and rel(st[1], (y[:M].float() ** 2).sum(0)) < 2e-3
    dy = (torch.randn(NI, Ho, Wo, Cout, generator=g) * 0.5).bfloat16().cuda()
    dw = torch.zeros(Cout, 9 * C, device="cuda")
    ops.gemm(dy, x, dw, Cout, 9 * C, M, lda=Cout, ldb=C, atomic=True, out_f32=True, split_k=4, conv=(NI, H, W, C),
             conv_mode=2, conv_stride=2)
    gref = torch.nn.grad.conv2d_weight(x.float().permute(0, 3, 1, 2), (Cout, C, 3, 3), dy.float().permute(0, 3, 1, 2),
                                       stride=2, padding=1)
    assert rel(dw.view(Cout, 3, 3, C).permute(0, 3, 1, 2), gref) < 2e-3


@pytest.mark.parametrize("NI,H,W,C,Cout", [(8, 28, 28, 256, 512), (5, 7, 9, 64, 128)])
def test_strided_downsample_one_tap_fprop_and_wgrad(NI, H, W, C, Cout):
    """1x1 / stride 2 downsample (resnet.py:239-243) as a one-tap implicit GEMM over the strided view of x."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(C + H)
    x = (torch.randn(NI, H, W, C, generator=g) * 0.5).bfloat16().cuda()
    w = (torch.randn(Cout, C, generator=g) * 0.05).bfloat16().cuda()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    M = NI * Ho * Wo
    y = torch.empty(M, Cout, dtype=BF16, device="cuda")
    st = torch.zeros(2, Cout, device="cuda")
    ops.gemm(x, w, y, M, Cout, C, lda=C, stats=st, conv=(NI, H, W, C), conv_mode=1, conv_stride=2, conv_taps=1)
    xs = x[:, ::2, ::2].reshape(M, C).float()
    assert rel(y, xs @ w.float().t()) < 4e-3
    assert rel(st[0], y.float().sum(0)) < 2e-3
    dy = (torch.randn(M, Cout, generator=g) * 0.5).bfloat16().cuda()
    dw = torch.zeros(Cout, C, device="cuda")
    ops.gemm(dy, x, dw, Cout, C, M, lda=Cout, ldb=C, atomic=True, out_f32=True, split_k=2, conv=(NI, H, W, C),
             conv_mode=2, conv_stride=2, conv_taps=1)
    assert rel(dw, dy.float().t() @ xs) < 2e-3


@pytest.mark.parametrize("NI,H,W,C,Cout", [(8, 28, 28, 128, 128), (4, 14, 14, 256, 256), (3, 13, 15, 64, 128)])
def test_strided_dgrad_by_parity_classes(NI, H, W, C, Cout):
    """Input gradient of a 3x3 / stride 2 / pad 1 convolution as four implicit GEMMs (one per parity class of the input
    position, explicit tap grids 1x1 / 1x2 / 2x1 / 2x2 over dy, each writing its own strided sub-grid of dx) against
    autograd of F.conv2d."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(H + W + C)
    w = (torch.randn(Cout, C, 3, 3, generator=g) * 0.05).bfloat16().cuda()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dy = (torch.randn(NI, Ho, Wo, Cout, generator=g) * 0.5).bfloat16().cuda()
    dx = torch.full((NI, H, W, C), 9.0, dtype=BF16, device="cuda")
    for ph in (0, 1):
        for pw in (0, 1):
            th, tw = 1 + ph, 1 + pw
            taps = []
            for a in range(th):
                for b in range(tw):
                    taps.append(w.float()[:, :, ph + 1 - 2 * a, pw + 1 - 2 * b].t())   # [C(in), Cout]
            wc = torch.cat(taps, dim=1).bfloat16().contiguous()                          # [C, taps*Cout], k = tap*Cout + co
            Hs, Ws = (H - ph + 1) // 2, (W - pw + 1) // 2
            ops.gemm(dy, wc, dx, NI * Ho * Wo, C, th * tw * Cout, lda=Cout, conv=(NI, Ho, Wo, Cout), conv_mode=1,
                     tap_grid=(th, tw, 0), d_ptr=dx.data_ptr() + (ph * W + pw) * C * 2,
                     out_view=(Hs, Ws, 2 * C, 2 * W * C, H * W * C))
    x = torch.zeros(NI, C, H, W, device="cuda", requires_grad=True)
    F.conv2d(x, w.float(), stride=2, padding=1).backward(dy.float().permute(0, 3, 1, 2))
    assert rel(dx, x.grad.permute(0, 2, 3, 1)) < 4e-3   # every element written exactly once (no 9.0 left), values match


@pytest.mark.parametrize("NI,H,W,Cin,C4", [(8, 28, 28, 256, 512), (3, 13, 15, 64, 128)])
def test_strided_downsample_dgrad_accumulates_in_place(NI, H, W, Cin, C4):
    """dx[:, ::2, ::2] += dyd . Wd (input gradient of the 1x1 / stride-2 downsample added to the conv1 dgrad already in
    dx): one-tap implicit GEMM whose output AND residual are the even-position sub-grid of dx."""
    _need_cuda()
    ops = _ops()
    g = torch.Generator().manual_seed(Cin + H)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dyd = (torch.randn(NI, Ho, Wo, C4, generator=g) * 0.5).bfloat16().cuda()
    wd = (torch.randn(C4, Cin, generator=g) * 0.05).bfloat16().cuda()
    wt = wd.t().contiguous()                                   # [Cin, C4]: K-major B operand
    dx0 = torch.randn(NI, H, W, Cin, generator=g).bfloat16().cuda()
    dx = dx0.clone()
    ops.gemm(dyd, wt, dx, NI * Ho * Wo, Cin, C4, lda=C4, conv=(NI, Ho, Wo, C4), conv_mode=1, conv_taps=1, residual=dx,
             d_ptr=dx.data_ptr(), out_view=((H + 1) // 2, (W + 1) // 2, 2 * Cin, 2 * W * Cin, H * W * Cin))
    ref = dx0.float().clone()
    ref[:, ::2, ::2] += (dyd.float().reshape(-1, C4) @ wd.float()).view(NI, Ho, Wo, Cin)
    assert rel(dx, ref) < 4e-3
    odd = torch.ones(H, W, dtype=torch.bool)
    odd[::2, ::2] = False
    assert torch.equal(dx[:, odd], dx0[:, odd])   # positions outside the sub-grid are untouched
