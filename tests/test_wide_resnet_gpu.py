"""Wide ResNet-50-2 (the reference's R_50W2X backbone ablation) on the sm_90a kernels.

A wide bottleneck of `planes` is 2 * planes wide inside (conv1 / conv2 / bn1 / bn2) and 4 * planes at its output, so
its 3x3 convs run at C = 128 ... 1024 where ResNet-50's run at 64 ... 512, and conv3 reduces over K = width.  The
kernel tests below run every GEMM shape class the wide stages add, at batch 2, against float64 references computed
from the same bf16 operands:
  * implicit 3x3 fprop with BN statistics, stride 1 and stride 2 (C = 256 over 56 x 56, C = 1024 over 14 x 14);
  * implicit 3x3 dgrad with the fused BN-backward sums, stride 1, and the four parity-class GEMMs of the stride-2
    dgrad at the same widths;
  * split-K implicit 3x3 wgrad (conv_mode 2) into fp32 [C, 9 C], up to [1024, 9216];
  * the 1x1 conv3 with K = width (fprop with statistics, dgrad with the BN-backward sums at N = width up to 1024, and
    its wgrad).
The BN finalize / apply / backward kernels at C = 1024 are covered at these extents by tests/test_backbone_kernels_gpu.py.
Tolerances: bf16 outputs are compared by relative L2 error (4e-3, the bf16 rounding of the output), fp32 outputs
(wgrad, statistics, BN-backward sums) to their fp32 summation order.  The BN statistics are sums over the bf16 output
as stored, so they are checked against float64 sums of that output.

Then the whole backbone and model against the CPU oracle with the bounds of tests/test_gpu_parity.py, the downstream
forward against torchvision's wide_resnet50_2 in float64, six Trainer steps, and the R_50W2X config at batch 256."""
import math

import pytest
import torch
import torch.nn.functional as F
from torch import nn

from oracle import virtex_oracle as O
from tests.helpers import build_model, to_cuda

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
WIDE = "wide_resnet50_2"
# (input extent, width, stride) of the 3x3 convs of the wide stages
CONV_SHAPES = [(56, 128, 1), (56, 256, 2), (28, 256, 1), (28, 512, 2), (14, 512, 1), (14, 1024, 2), (7, 1024, 1)]
CONV_IDS = [f"H{h}-C{c}-s{s}" for h, c, s in CONV_SHAPES]
# (output extent, conv3 output width 4 * planes, inner width) of the 1x1 conv3 of each stage
CONV3_SHAPES = [(56, 256, 128), (28, 512, 256), (14, 1024, 512), (7, 2048, 1024)]
NI = 2


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


def _nchw(t, H):
    return t.double().view(NI, H, H, -1).permute(0, 3, 1, 2)


def _nhwc_rows(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _bnp(C, g):
    """[4, C] = mean, invstd, scale, shift of a train-mode BN (what vtx_bn_finalize writes)."""
    mean = torch.randn(C, device=DEV, generator=g) * 0.3
    invstd = torch.rand(C, device=DEV, generator=g) + 0.5
    gamma = torch.rand(C, device=DEV, generator=g) + 0.5
    beta = torch.randn(C, device=DEV, generator=g) * 0.3
    scale = gamma * invstd
    return torch.stack([mean, invstd, scale, beta - mean * scale]).contiguous()


def _bnr_sums_ref(dA, y, bnp):
    """float64 [2, C] = sum dz, sum dz * (y - mean) * invstd with dz = dA * [y * scale + shift > 0]."""
    mask = (y.float() * bnp[2] + bnp[3]) > 0
    dz = dA.double() * mask.double()
    return torch.stack([dz.sum(0), (dz * (y.double() - bnp[0].double()) * bnp[1].double()).sum(0)])


def _check_sums(sums, ref, what):
    C = ref.shape[1]
    r = max(rel(sums[:C], ref[0]), rel(sums[C:2 * C], ref[1]))
    assert r < 1e-3, (what, r)


def _check_stats(st, y):
    """BN statistics of the epilogue: sum and sum of squares of the bf16 output as stored, per column."""
    yd = y.double()
    assert rel(st[0], yd.sum(0)) < 1e-4 and rel(st[1], (yd * yd).sum(0)) < 1e-4, (rel(st[0], yd.sum(0)),
                                                                                 rel(st[1], (yd * yd).sum(0)))


# ------------------------------------------------------------------------------------------------------ 3x3 convs
@pytest.mark.parametrize("H,C,stride", CONV_SHAPES, ids=CONV_IDS)
def test_conv3x3_fprop_with_statistics(H, C, stride):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(H * C + stride)
    x = (torch.randn(NI, H, H, C, device=DEV, generator=g) * 0.5).bfloat16()
    w = (torch.randn(C, C, 3, 3, device=DEV, generator=g) * math.sqrt(2.0 / (9 * C))).bfloat16()
    Ho = (H - 1) // stride + 1
    M = NI * Ho * Ho
    y = torch.full((M + 64, C), 7.0, dtype=BF16, device=DEV)  # guard rows behind the output
    st = torch.zeros(2, C, device=DEV)
    ops.gemm(x, w.permute(0, 2, 3, 1).reshape(C, 9 * C).contiguous(), y, M, C, 9 * C, lda=C, stats=st,
             conv=(NI, H, H, C), conv_mode=1, conv_stride=stride)
    ref = _nhwc_rows(F.conv2d(_nchw(x, H), w.double(), stride=stride, padding=1))
    torch.cuda.synchronize()
    assert rel(y[:M], ref) < 4e-3, rel(y[:M], ref)
    assert torch.all(y[M:] == 7.0)
    _check_stats(st, y[:M])


@pytest.mark.parametrize("H,C,stride", CONV_SHAPES, ids=CONV_IDS)
def test_conv3x3_dgrad_with_fused_bn_sums(H, C, stride):
    """The engine's conv2 dgrad: stride 1 one implicit GEMM over the flipped weights, stride 2 four parity-class GEMMs
    that each write a strided sub-grid of the input gradient; both accumulate bn1's backward sums in the epilogue."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(7 * H * C + stride)
    w = (torch.randn(C, C, 3, 3, device=DEV, generator=g) * math.sqrt(2.0 / (9 * C))).bfloat16()
    Ho = (H - 1) // stride + 1
    Min, Mout = NI * H * H, NI * Ho * Ho
    dy = (torch.randn(Mout, C, device=DEV, generator=g) * 0.5).bfloat16()
    y1 = torch.randn(Min, C, device=DEV, generator=g).bfloat16()
    bnp = _bnp(C, g)
    da = torch.full((Min, C), float("nan"), dtype=BF16, device=DEV)
    sums = torch.zeros(2 * C, device=DEV)
    if stride == 1:
        wd = w.flip(2, 3).permute(1, 2, 3, 0).reshape(C, 9 * C).contiguous()
        ops.gemm(dy, wd, da, Min, C, 9 * C, lda=C, conv=(NI, H, H, C), conv_mode=1, bnr=(y1, bnp, sums, None))
    else:
        for ph in (0, 1):
            for pw in (0, 1):
                th, tw = 1 + ph, 1 + pw
                wp = torch.empty(C, th, tw, C, dtype=BF16, device=DEV)
                for a in range(th):
                    for b in range(tw):
                        wp[:, a, b, :] = w[:, :, ph + 1 - 2 * a, pw + 1 - 2 * b].t()
                Hs, Ws = (H - ph + 1) // 2, (H - pw + 1) // 2
                voff = (ph * H + pw) * C * 2
                ops.gemm(dy, wp.view(C, th * tw * C), da, Mout, C, th * tw * C, lda=C, conv=(NI, Ho, Ho, C),
                         conv_mode=1, tap_grid=(th, tw, 0), d_ptr=da.data_ptr() + voff,
                         out_view=(Hs, Ws, 2 * C, 2 * H * C, H * H * C),
                         bnr=(y1, bnp, sums, None, y1.data_ptr() + voff))
    ref = _nhwc_rows(torch.nn.grad.conv2d_input((NI, C, H, H), w.double(), _nchw(dy, Ho), stride=stride, padding=1))
    torch.cuda.synchronize()
    assert not torch.isnan(da).any()  # every element written exactly by one launch
    assert rel(da, ref) < 4e-3, rel(da, ref)
    _check_sums(sums, _bnr_sums_ref(da, y1, bnp), "bn1 sums")


@pytest.mark.parametrize("H,C,stride", CONV_SHAPES, ids=CONV_IDS)
def test_conv3x3_splitk_wgrad(H, C, stride):
    """conv_mode 2 wgrad with the engine's split-K choice, accumulating (+=) into a non-zero fp32 [C, 9 C] buffer."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(11 * H * C + stride)
    Ho = (H - 1) // stride + 1
    Mout = NI * Ho * Ho
    a1 = (torch.randn(NI * H * H, C, device=DEV, generator=g) * 0.5).bfloat16()
    dy = (torch.randn(Mout, C, device=DEV, generator=g) * 0.5).bfloat16()
    dw0 = torch.randn(C, 9 * C, device=DEV, generator=g)
    dw = dw0.clone()
    tiles = ((C + 127) // 128) * ((9 * C + 255) // 256)
    sk = ops.split_k_for(tiles, (Mout + 63) // 64)
    ops.gemm(dy, a1, dw, C, 9 * C, Mout, atomic=True, split_k=sk, lda=C, ldb=C, conv=(NI, H, H, C), conv_mode=2,
             out_f32=True, conv_stride=stride)
    ref = torch.nn.grad.conv2d_weight(_nchw(a1, H), (C, C, 3, 3), _nchw(dy, Ho), stride=stride, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(C, 9 * C)
    torch.cuda.synchronize()
    assert rel(dw - dw0, ref) < 1e-4, (sk, rel(dw - dw0, ref))


# ------------------------------------------------------------------------------------------------------ 1x1 conv3
@pytest.mark.parametrize("H,C4,width", CONV3_SHAPES, ids=[f"H{h}-N{c}-K{w}" for h, c, w in CONV3_SHAPES])
def test_conv3_fprop_dgrad_wgrad(H, C4, width):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(H + C4 + width)
    M = NI * H * H
    a2 = (torch.randn(M, width, device=DEV, generator=g) * 0.5).bfloat16()
    w3 = (torch.randn(C4, width, device=DEV, generator=g) * math.sqrt(2.0 / C4)).bfloat16()
    y3 = torch.empty(M, C4, dtype=BF16, device=DEV)
    st = torch.zeros(2, C4, device=DEV)
    ops.gemm(a2, w3, y3, M, C4, width, stats=st)
    ref = a2.double() @ w3.double().t()
    # dgrad into da2 [M, width] with bn2's backward sums (N = width), and the [C4, width] wgrad
    dy3 = (torch.randn(M, C4, device=DEV, generator=g) * 0.5).bfloat16()
    y2 = torch.randn(M, width, device=DEV, generator=g).bfloat16()
    bnp = _bnp(width, g)
    da2 = torch.empty(M, width, dtype=BF16, device=DEV)
    sums = torch.zeros(2 * width, device=DEV)
    ops.gemm(dy3, w3, da2, M, width, C4, b_mn=1, bnr=(y2, bnp, sums, None))
    dw = torch.zeros(C4, width, device=DEV)
    tiles = ((C4 + 127) // 128) * ((width + 255) // 256)
    ops.gemm(dy3, a2, dw, C4, width, M, a_mn=1, b_mn=1, atomic=True, split_k=ops.split_k_for(tiles, (M + 63) // 64),
             ldd=width, out_f32=True)
    torch.cuda.synchronize()
    assert rel(y3, ref) < 4e-3
    _check_stats(st, y3)
    assert rel(da2, dy3.double() @ w3.double()) < 4e-3
    _check_sums(sums, _bnr_sums_ref(da2, y2, bnp), "bn2 sums")
    assert rel(dw, dy3.double().t() @ a2.double()) < 1e-4


# ------------------------------------------------------------------------------------------------------- backbone
SMALL = O.Spec(backbone=WIDE, hidden=128, layers=1, heads=2, ffn=256)  # the spec of tests/golden/r50w2x_*.pt


def test_backbone_forward_backward_vs_oracle():
    """tests/test_gpu_parity.py::test_backbone_forward_backward_vs_oracle on the wide backbone, same bounds."""
    _ops()
    state = O.synth_state(SMALL, 5, bn3_gain=0.25)
    model = build_model(SMALL, state)
    B = 4
    batch = O.synth_batch(B, seed=3)
    eng = model.engine
    model.train()
    feat, h, w = eng.backbone_forward(batch["image"].cuda(), training=True)
    P = {k: (v.clone().requires_grad_(True) if not O.is_buffer(k) else v.clone()) for k, v in state.items()}
    nb = {}
    ref = O.backbone_forward(P, batch["image"], SMALL, training=True, new_buffers=nb, emulate_bf16=True)
    ref_nhwc = ref.permute(0, 2, 3, 1).reshape(B * h * w, -1)
    with torch.no_grad():
        ref32 = O.backbone_forward(state, batch["image"], SMALL, training=True)
    f_emul, f_32 = rel(feat, ref_nhwc), rel(feat, ref32.permute(0, 2, 3, 1).reshape(B * h * w, -1))
    dfeat = (torch.randn(ref_nhwc.shape, generator=torch.Generator().manual_seed(0)) * 0.01).bfloat16().float()
    ref_nhwc.backward(dfeat)
    eng.arena.grads.zero_()
    eng.backbone_backward(dfeat.cuda().bfloat16().contiguous())
    torch.cuda.synchronize()
    worst = sorted((cos(eng.G(n), P[n].grad), rel(eng.G(n), P[n].grad), n) for n in eng.arena.names
                   if n.startswith("visual."))
    med = sorted(r for _, r, _ in worst)[len(worst) // 2]
    print(f"wide: feat rel vs bf16-placement oracle {f_emul:.5f} vs fp32 oracle {f_32:.5f}; median grad rel {med:.4f}; "
          f"worst cos {worst[0][0]:.5f} ({worst[0][2]})")
    assert f_emul < 5e-2, f_emul
    assert f_32 < 8e-2, f_32
    assert worst[0][0] > 0.85, worst[:5]
    assert med < 0.5, (med, worst[:5])
    for k in ("visual.cnn.bn1.running_var", "visual.cnn.layer4.2.bn3.running_mean",
              "visual.cnn.layer2.0.downsample.1.running_var", "visual.cnn.layer4.0.bn2.running_mean"):
        assert rel(eng.buffers[k], nb[k]) < 2e-2, k


# ---------------------------------------------------------------------------------------------------------- model
def test_model_loss_grads_and_folded_eval_vs_oracle():
    _ops()
    spec = SMALL
    state = O.synth_state(spec, 11, bn3_gain=0.25)
    model = build_model(spec, state)
    model.train()
    batch = O.synth_batch(4, seed=6, ragged=True)
    out = model(to_cuda(batch))
    ref, grads, _ = O.loss_and_grads(state, batch, spec)
    assert abs(out["loss"].item() - ref["loss"].item()) < 1e-3 * ref["loss"].item(), (out["loss"].item(), ref["loss"].item())
    out["loss"].backward()
    named = dict(model.named_parameters())
    bad = [(n, rel(named[n].grad, g), cos(named[n].grad, g)) for n, g in grads.items() if not n.startswith("visual.")
           and not (cos(named[n].grad, g) > 0.998 and rel(named[n].grad, g) < 5e-2)]
    assert not bad, bad
    assert all(torch.isfinite(named[n].grad).all() for n in grads if n.startswith("visual."))
    # eval mode through backbone_infer (every BN folded into its GEMM's epilogue), the path of beam search and of the
    # downstream forward: features, logits and loss against the eval-mode oracle
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    model.eval()
    eng = model.engine
    image = batch["image"].cuda()
    with torch.no_grad():
        ref_e = O.model_forward(state, batch, spec, training=False, return_logits=True)
        feat, h, w = eng.backbone_infer(image)
        B = image.shape[0]
        mem = eng.visual_projection_forward(feat, B * h * w)
        rec = eng.head_forward("textual", mem, batch["caption_tokens"].cuda(), batch["caption_lengths"].cuda(), False,
                               want_logits_f32=True)
        logits = rec["logits_f32"].view(B, spec.max_len, -1)[..., :spec.vocab].double().cpu()
        unfused, _, _ = eng.backbone_forward(image, training=False)
    vf = ref_e["visual_features"].permute(0, 2, 3, 1).reshape(B * h * w, -1)
    torch.cuda.synchronize()
    assert rel(feat, vf) < 5e-2, rel(feat, vf)
    assert rel(feat, unfused) < 1e-2, rel(feat, unfused)
    loss_f = O.caption_loss(logits, batch["caption_tokens"])
    ref_f = ref_e["loss_components"]["captioning_forward"]
    assert abs(loss_f.item() - ref_f.item()) < 2e-3 * ref_f.item(), (loss_f.item(), ref_f.item())
    valid = torch.arange(spec.max_len)[None, :] < batch["caption_lengths"][:, None]
    err = (logits - ref_e["logits"].double()).abs().amax(-1)[valid].max().item()
    assert err < 0.15, err
    top2 = ref_e["logits"].topk(2, dim=-1).values
    sure = ((top2[..., 0] - top2[..., 1]) > 0.25) & valid
    assert torch.equal(logits.argmax(-1)[sure], ref_e["predictions"][sure])


# ----------------------------------------------------------------------------------------------------- downstream
def test_downstream_forward_vs_torchvision_float64():
    """ResNetParams("wide_resnet50_2") with an fc, in eval mode, against torchvision's wide_resnet50_2 in float64 on the
    same weights (randomised BN statistics and affine parameters, residual gain 0.25)."""
    _ops()
    import torchvision
    from virtex_b200.modules import ResNetParams
    full = O.synth_state(SMALL, 41, bn3_gain=0.25)
    state = {k[len("visual.cnn."):]: v for k, v in full.items() if k.startswith("visual.cnn.")}
    g = torch.Generator().manual_seed(42)
    state["fc.weight"] = torch.randn(10, 2048, generator=g) * 0.01
    state["fc.bias"] = torch.randn(10, generator=g) * 0.1
    cnn = ResNetParams(WIDE)
    cnn.fc = nn.Linear(2048, 10)
    cnn.load_state_dict(state, strict=True)
    cnn = cnn.cuda().eval()
    tv = torchvision.models.wide_resnet50_2(num_classes=10)
    tv.load_state_dict(state, strict=True)
    tv = tv.double().eval()
    image = torch.randn(3, 3, 224, 224, generator=g)
    with torch.no_grad():
        logits = cnn(image.cuda())
        cnn.fc = nn.Identity()
        pooled = cnn(image.cuda())
        ref = tv(image.double())
        tv.fc = nn.Identity()
        ref_pooled = tv(image.double())
    r_p, r_l = rel(pooled, ref_pooled), rel(logits, ref)
    print(f"wide downstream: pooled rel {r_p:.5f}, logits rel {r_l:.5f}")
    assert logits.dtype == F32 and tuple(pooled.shape) == (3, 2048)
    assert r_p < 2e-2 and r_l < 2e-2, (r_p, r_l)


# -------------------------------------------------------------------------------------------------------- trainer
def test_trainer_trajectory_vs_oracle():
    """tests/test_gpu_parity.py::test_trainer_trajectory_vs_oracle on the wide spec."""
    _ops()
    from virtex_b200.config import Config
    from virtex_b200.trainer import Trainer
    spec = SMALL
    state = O.synth_state(spec, 3, bn3_gain=0.25)
    model = build_model(spec, state)
    model.train()
    cfg = Config(None, ["MODEL.VISUAL.NAME", "torchvision::" + WIDE, "MODEL.TEXTUAL.NAME",
                        "transdec_postnorm::L1_H128_A2_F256", "MODEL.TEXTUAL.DROPOUT", 0.0, "OPTIM.WARMUP_STEPS", 3,
                        "OPTIM.NUM_ITERATIONS", 20, "OPTIM.BATCH_SIZE", 4, "OPTIM.CNN_LR", 0.005])
    tr = Trainer(model, cfg)
    ora = O.OracleTrainer(state, spec, O.OptimCfg(warmup_steps=3, num_iterations=20, cnn_lr=0.005))
    for it in range(6):
        batch = O.synth_batch(4, seed=30 + it, ragged=True)
        loss = tr.step(to_cuda(batch)).sum().item()
        ref = ora.step(batch)
        print(f"wide trainer step {it}: loss {loss:.6f} vs {ref['loss'].item():.6f}, grad norm "
              f"{tr.grad_norm.item():.4f} vs {ref['grad_norm'].item():.4f}")
        assert abs(loss - ref["loss"].item()) < 3e-3 * ref["loss"].item(), (it, loss, ref["loss"].item())
        assert abs(tr.grad_norm.item() - ref["grad_norm"].item()) < 0.1 * ref["grad_norm"].item(), it
    k = "textual.transformer.layers.0.linear1.weight"
    d_ours = dict(model.named_parameters())[k].detach().cpu() - state[k]
    assert cos(d_ours, ora.state[k] - state[k]) > 0.99


# ------------------------------------------------------------------------------------------------------ full size
def _fp32_oracle(state, batch, spec, training):
    """O.model_forward in fp32 with the backbone evaluated on the GPU (TF32 off) and the head on the CPU: the CPU
    would take minutes over a batch of 256 wide-ResNet images."""
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        P = {k: v.cuda() for k, v in state.items()}
        with torch.no_grad():
            vf = O.backbone_forward(P, batch["image"].cuda(), spec, training=training).cpu()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    with torch.no_grad():
        logits = O.head_forward(state, vf, batch["caption_tokens"], batch["caption_lengths"], spec, "textual")
        back = O.head_forward(state, vf, batch["noitpac_tokens"], batch["caption_lengths"], spec, "backward_textual")
    loss = O.caption_loss(logits, batch["caption_tokens"]) + O.caption_loss(back, batch["noitpac_tokens"])
    return loss, logits


def test_full_size_r50w2x_batch_256():
    """The R_50W2X config (wide_resnet50_2, L1_H1024) at batch 256: train-mode loss within 1e-3 of the fp32 oracle,
    the eval argmax rule of test_full_size_forward_vs_oracle_batch_256, and a training step with finite gradients."""
    _ops()
    torch.set_num_threads(max(1, min(32, (torch.get_num_threads() or 1))))
    spec = O.Spec(backbone=WIDE)
    state = O.synth_state(spec, 23, bn3_gain=0.25)
    model = build_model(spec, state)
    B = 256
    batch = O.synth_batch(B, seed=31, ragged=True)
    cb = to_cuda(batch)
    torch.cuda.reset_peak_memory_stats()
    model.train()
    with torch.no_grad():
        out_t = model(cb)
    ref_t, _ = _fp32_oracle(state, batch, spec, training=True)
    rel_t = abs(out_t["loss"].item() - ref_t.item()) / ref_t.item()
    assert rel_t < 1e-3, (out_t["loss"].item(), ref_t.item())
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    model.eval()
    with torch.no_grad():
        out_e = model(cb)
    ref_e, logits_ref = _fp32_oracle(state, batch, spec, training=False)
    assert abs(out_e["loss"].item() - ref_e.item()) < 1e-3 * ref_e.item()
    lg = model.engine._recs[0]["logits_f32"].view(B, 30, -1).cpu()
    valid = torch.arange(30)[None, :] < batch["caption_lengths"][:, None]
    err = (lg - logits_ref).abs().amax(-1)[valid].max().item()
    assert err < 0.15, err
    pred, pref = out_e["predictions"].cpu(), logits_ref.argmax(-1)
    top2 = logits_ref.topk(2, dim=-1).values
    sure = ((top2[..., 0] - top2[..., 1]) > 0.25) & valid
    assert sure.float().mean().item() > 0.3
    assert torch.equal(pred[sure], pref[sure])
    diff = (pred != pref) & valid
    if diff.any():
        ours = logits_ref.gather(-1, pred.unsqueeze(-1)).squeeze(-1)
        assert ((top2[..., 0] - ours)[diff] <= 0.25).all()
    # one training step: every gradient finite
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    model.train()
    out = model(cb)
    out["loss"].backward()
    for n, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    torch.cuda.synchronize()
    print(f"B=256 R50W2X-L1-H1024: train loss rel {rel_t:.2e}; eval logits max abs err {err:.4f}; confident positions "
          f"{int(sure.sum())}/{int(valid.sum())}, {int(diff.sum())} differing; "
          f"max_memory_allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
