"""The downstream classification path on the GPU: the scale / shift GEMM epilogue (VtxGemm.col_scale / col_shift) against
its float64 formula, Engine.backbone_infer and ResNetParams.forward against the float64 oracle (tests/downstream_oracle.py,
pinned to the reference's torchvision ResNet-50), the frozen linear probe of scripts/clf_linear.py against an autograd
loop on fc, and fine-tuning in train mode."""
import os

import pytest
import torch
import torch.nn.functional as F
from torch import nn

from tests import downstream_oracle as DO

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32


def _ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from virtex_b200 import ops
    return ops


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def cos(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm() + 1e-30)).item()


def _within_one_bf16_ulp(out, ref, mag):
    """out (bf16) is ref (float64) rounded to bf16, or one of its bf16 neighbours.  `mag` (the sum of the magnitudes
    of the terms) bounds the fp32 accumulation and fma error, which decides the rounding where terms cancel."""
    r = ref.double().cpu()
    o = out.double().cpu()
    ulp = 2.0 ** (torch.floor(torch.log2(r.abs().clamp_min(1e-30))) - 7)
    bad = (o - r).abs() > ulp + 2.0 ** -20 * mag.double().cpu()
    assert not bad.any(), (int(bad.sum()), o[bad][:4], r[bad][:4])


def _ss_case(g, N):
    """Per-column scale and shift vectors, as the eval-mode BN fold produces them."""
    return (torch.rand(N, generator=g) + 0.5).cuda(), (torch.randn(N, generator=g) * 0.5).cuda()


# ------------------------------------------------------------------------------------------------------ the epilogue
@pytest.mark.parametrize("M,N,K", [
    (1000, 64, 128),     # 64-wide tiles
    (4099, 128, 256),    # ragged last row tile
    (3001, 192, 64),     # 192-wide tiles
    (9000, 512, 256),    # 256-wide tiles (auto width)
    (2050, 100, 128),    # partial column tile (N even, not a multiple of 8)
    (777, 1000, 64),     # several column tiles, ragged in both directions
])
@pytest.mark.parametrize("residual,act", [(False, 0), (False, 1), (True, 0), (True, 1)])
def test_scale_shift_epilogue_matches_formula(M, N, K, residual, act):
    ops = _ops()
    g = torch.Generator().manual_seed(M + N + K + 7 * residual + act)
    A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
    B = (torch.randn(N, K, generator=g) * 0.5).bfloat16().cuda()
    scale, shift = _ss_case(g, N)
    ld = (N + 7) // 8 * 8  # bf16 rows of D and R stay 16-byte aligned
    R = torch.randn(M, ld, generator=g).bfloat16().cuda()[:, :N] if residual else None
    acc = A.double() @ B.double().t()
    ref = acc * scale.double() + shift.double() + (R.double() if residual else 0)
    mag = (A.double().abs() @ B.double().abs().t()) * scale.double() + shift.double().abs() + \
        (R.double().abs() if residual else 0)
    if act:
        ref = ref.clamp_min(0)
    outs = []
    widths = [0, 64, 128, 192, 256] if N <= 256 else [0, 256]
    for tile_n in widths:
        D = torch.full((M, ld), float("nan"), dtype=BF16, device="cuda")[:, :N]
        ops.gemm(A, B, D, M, N, K, residual=R, act=act, col_scale=scale, col_shift=shift, tile_n=tile_n)
        outs.append(D)
    torch.cuda.synchronize()
    _within_one_bf16_ulp(outs[0], ref, mag)
    for o in outs[1:]:  # every width and both schedules (<= 128 wide: ping-pong; wider: lockstep) give the same bits
        assert torch.equal(o, outs[0])


@pytest.mark.parametrize("H,C,N,stride,taps", [
    (56, 64, 64, 1, 9),      # layer1 3x3
    (28, 128, 128, 1, 9),
    (56, 128, 128, 2, 9),    # layer2's strided 3x3
    (15, 64, 192, 2, 9),     # odd extent, ragged boxes
    (56, 256, 512, 2, 1),    # one-tap strided downsample
    (13, 128, 256, 2, 1),
])
@pytest.mark.parametrize("act", [0, 1])
def test_scale_shift_epilogue_on_implicit_convs(H, C, N, stride, taps, act):
    ops = _ops()
    g = torch.Generator().manual_seed(H * C + N + stride + taps + act)
    NI = 3
    x = (torch.randn(NI, H, H, C, generator=g) * 0.5).bfloat16().cuda()
    k = 3 if taps == 9 else 1
    w = (torch.randn(N, C, k, k, generator=g) * 0.1).bfloat16().cuda()
    wp = w.permute(0, 2, 3, 1).reshape(N, k * k * C).contiguous()  # [N, (kh, kw, c)]
    scale, shift = _ss_case(g, N)
    Ho = (H - 1) // stride + 1
    M = NI * Ho * Ho
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), stride=stride, padding=(k - 1) // 2)
    mag = F.conv2d(x.permute(0, 3, 1, 2).double().abs(), w.double().abs(), stride=stride, padding=(k - 1) // 2)
    mag = mag.permute(0, 2, 3, 1).reshape(M, N) * scale.double() + shift.double().abs()
    ref = ref.permute(0, 2, 3, 1).reshape(M, N) * scale.double() + shift.double()
    if act:
        ref = ref.clamp_min(0)
    outs = []
    for tile_n in ([0, 256] if N <= 128 else [0]):
        D = torch.full((M, N), float("nan"), dtype=BF16, device="cuda")
        ops.gemm(x, wp, D, M, N, k * k * C, lda=C, conv=(NI, H, H, C), conv_mode=1, conv_stride=stride,
                 conv_taps=1 if taps == 1 else 0, act=act, col_scale=scale, col_shift=shift, tile_n=tile_n)
        outs.append(D)
    torch.cuda.synchronize()
    _within_one_bf16_ulp(outs[0], ref, mag)
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


# ------------------------------------------------------------------------------------------------------ the module
def _cnn(state, device="cuda"):
    from virtex_b200.modules import ResNetParams
    cnn = ResNetParams("resnet50")
    cnn.fc = nn.Linear(2048, DO.NUM_CLASSES)
    cnn.load_state_dict(state, strict=True)
    return cnn.to(device)


def _golden():
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", DO.GOLDEN), weights_only=False)


@pytest.mark.parametrize("case", list(DO.CASES))
def test_eval_forward_matches_oracle_and_training_schedule(case):
    _ops()
    g = _golden()[case]["eval"]
    state, batch = DO.case_inputs(case)
    cnn = _cnn(state).eval()
    image = batch["image"].cuda()
    with torch.no_grad():
        logits = cnn(image)
        fc = cnn.fc
        cnn.fc = nn.Identity()
        pooled = cnn(image)
        cnn.fc = fc
    assert logits.dtype == F32 and pooled.dtype == F32 and tuple(pooled.shape) == (image.shape[0], 2048)
    r_p, r_l = rel(pooled, g["pooled"]), rel(logits, g["logits"])
    assert r_p < 2e-2 and r_l < 2e-2, (r_p, r_l)
    loss = F.cross_entropy(logits, batch["label"].cuda())
    assert abs(loss.item() - g["loss"].item()) < 2e-3 * g["loss"].item()
    # against the unfused eval forward of the same engine (raw conv outputs, then BN passes)
    from virtex_b200 import ops
    eng = cnn._vtx_engine
    feat, h, w = eng.backbone_forward(image, training=False)
    ref = torch.empty(image.shape[0], 2048, dtype=BF16, device="cuda")
    ops.call("vtx_group_mean_fwd", feat.data_ptr(), ref.data_ptr(), image.shape[0], h * w, 2048, ops._stream())
    torch.cuda.synchronize()
    assert rel(pooled, ref.float()) < 1e-2, rel(pooled, ref.float())


def test_linear_probe_three_iterations_match_autograd_on_fc():
    """clf_linear.py with the frozen ImageNet config: CE, torch SGD (momentum 0.9, lr 0.3) on fc only.  Every
    iteration's loss and fc gradients are compared with float64 autograd on the oracle's features and the fc the GPU
    model holds at its start (lr 0.3 on these random-network features diverges, which would amplify any difference
    along the trajectory); the backbone parameters and every BN buffer stay bit for bit."""
    _ops()
    state, _ = DO.case_inputs("b2_224")
    batches = [DO.synth_batch(4, 90 + i, 224) for i in range(3)]
    P = {k: (v.double() if v.is_floating_point() else v) for k, v in state.items()}
    with torch.no_grad():
        feats = [DO.cnn_forward(P, b["image"].double(), training=False)[0] for b in batches]
    cnn = _cnn(state)
    cnn.fc = nn.Linear(2048, DO.NUM_CLASSES).cuda()  # assigned after construction, then re-initialised in place
    torch.nn.init.normal_(cnn.fc.weight.data, mean=0.0, std=0.01)
    torch.nn.init.constant_(cnn.fc.bias.data, 0.0)
    cnn.eval()
    for name, p in cnn.named_parameters():
        if "fc" not in name:
            p.requires_grad = False
    before = {k: v.detach().clone() for k, v in cnn.state_dict().items() if not k.startswith("fc.")}
    opt = torch.optim.SGD([p for p in cnn.parameters() if p.requires_grad], lr=0.3, momentum=0.9)
    for it, (f, b) in enumerate(zip(feats, batches)):
        loss_r, gw, gb = DO.probe_step(f, b["label"], cnn.fc.weight, cnn.fc.bias)
        opt.zero_grad()
        loss = F.cross_entropy(cnn(b["image"].cuda()), b["label"].cuda())
        loss.backward()
        assert abs(loss.item() - loss_r.item()) < 2e-3 * loss_r.item(), (it, loss.item(), loss_r.item())
        for got, want in ((cnn.fc.weight.grad, gw), (cnn.fc.bias.grad, gb)):
            assert cos(got, want) > 0.998 and rel(got, want) < 5e-2, (it, cos(got, want), rel(got, want))
        opt.step()
    for k, v in cnn.state_dict().items():
        if not k.startswith("fc."):
            assert torch.equal(v, before[k]), k


def test_fine_tuning_two_iterations_match_oracle():
    """inaturalist_clf: the whole ResNet in train mode with a new fc, two iterations of torch SGD.  Each iteration is
    compared with the oracle run from the parameters and running statistics the GPU model holds at its start; the
    first one also with the reference's own loss (fixture)."""
    _ops()
    case = "b2_224"
    g = _golden()[case]["train"]
    state, batch = DO.case_inputs(case)
    cnn = _cnn(state).train()
    opt = torch.optim.SGD(cnn.parameters(), lr=0.025, momentum=0.9, weight_decay=1e-4)
    for it in range(2):
        start = {k: v.detach().cpu().clone() for k, v in cnn.state_dict().items()}
        _, _, loss_r, grads_r, nb_r = DO.run(start, batch, training=True)
        opt.zero_grad()
        loss = F.cross_entropy(cnn(batch["image"].cuda()), batch["label"].cuda())
        loss.backward()
        if it == 0:
            assert abs(loss_r.item() - g["loss"].item()) < 1e-9 * g["loss"].item()
        named = dict(cnn.named_parameters())
        buffers = dict(cnn.named_buffers())
        print("fine-tune", it, loss.item(), loss_r.item(),
              {k: round(cos(named[k].grad, grads_r[k]), 5) for k in ("fc.weight", "fc.bias") + DO.CONV_PROBES})
        # (the second loss is small, so it is compared in absolute terms too: nats, not a fraction of itself)
        assert abs(loss.item() - loss_r.item()) < 5e-3 * max(loss_r.item(), 1.0), (it, loss.item(), loss_r.item())
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in cnn.parameters())
        for k in ("fc.weight", "fc.bias"):
            assert cos(named[k].grad, grads_r[k]) > 0.998 and rel(named[k].grad, grads_r[k]) < 5e-2, k
        # backbone gradients of two images through batch statistics are ill-conditioned in bf16 at this init (the same
        # holds for the pretraining models, tests/test_gpu_parity.py): loosely aligned with the float64 oracle
        for k in DO.CONV_PROBES:
            assert cos(named[k].grad, grads_r[k]) > 0.8, (k, cos(named[k].grad, grads_r[k]))
        for k in DO.BN_PROBES:
            for leaf in ("running_mean", "running_var"):
                r = rel(buffers[f"{k}.{leaf}"], nb_r[f"{k}.{leaf}"])
                assert r < 5e-3, (it, k, leaf, r)
            assert int(buffers[f"{k}.num_batches_tracked"]) == it + 1
        opt.step()
