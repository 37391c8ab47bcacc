"""Token / multilabel classification on the H100: the new kernels against float64 torch formulas, both models against
the CPU oracle (tests/classification_oracle.py, pinned to the reference by tests/test_classification_cpu.py), the frozen
backbone, and Trainer.step against the autograd loop body."""
import pytest
import torch

from tests import classification_oracle as CO
from tests.helpers import to_cuda

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def cos(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm() + 1e-30)).item()


def _call(name, *args):
    from virtex_b200 import ops
    ops.call(name, *args, ops._stream())
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------ kernels
def test_group_mean_forward_and_backward():
    _need_cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    B, HW, C = 5, 49, 2048
    feat = torch.randn(B * HW, C, device="cuda", generator=g).to(BF16)
    pooled = torch.empty(B, C, device="cuda", dtype=BF16)
    _call("vtx_group_mean_fwd", feat.data_ptr(), pooled.data_ptr(), B, HW, C)
    ref = feat.double().view(B, HW, C).mean(1)
    assert torch.allclose(pooled.double(), ref, rtol=8e-3, atol=1e-6)
    dpooled = torch.randn(B, C, device="cuda", generator=g).to(BF16)
    dfeat = torch.empty(B * HW, C, device="cuda", dtype=BF16)
    _call("vtx_group_mean_bwd", dpooled.data_ptr(), dfeat.data_ptr(), B, HW, C)
    ref = (dpooled.double() / HW)[:, None, :].expand(B, HW, C).reshape(B * HW, C)
    assert torch.allclose(dfeat.double(), ref, rtol=8e-3, atol=1e-9)


def _khot_inputs(B, V, ignore, empty_row=None, seed=0):
    g = torch.Generator().manual_seed(seed)
    ld = (V + 7) // 8 * 8
    logits = torch.full((B, ld), 1024.0).to(BF16)  # the padded columns must stay untouched
    logits[:, :V] = (torch.randn(B, V, generator=g) * 3).to(BF16)
    L = 9
    labels = torch.randint(0, V, (B, L), generator=g)
    labels[:, 1] = labels[:, 0]                        # duplicates
    labels[:, 2] = ignore[-1]                          # ignored ids
    for b in range(B):
        labels[b, 3 + b % 5:] = 0                      # ragged padding
    labels[B - 1, 3] = V + 5                           # out-of-range labels are skipped
    labels[B - 1, 4] = -1
    if empty_row is not None:
        labels[empty_row] = torch.tensor(ignore)[torch.arange(L) % len(ignore)]
    return logits, labels, ld


def _khot_reference(logits, labels, V, ignore):
    """float64 loss per row and dlogits = (softmax - K-hot / K) / B (zero rows for an empty label set)."""
    z = logits[:, :V].double()
    B = z.shape[0]
    p = torch.softmax(z, dim=1)
    grad = torch.zeros_like(z)
    rows = []
    for b in range(B):
        U = sorted({int(u) for u in labels[b] if 0 <= int(u) < V} - set(ignore))
        rows.append(torch.logsumexp(z[b], 0) - z[b, U].mean() if U else torch.tensor(float("nan"), dtype=z.dtype))
        if U:
            grad[b] = p[b]
            grad[b, U] -= 1.0 / len(U)
            grad[b] /= B
    return torch.stack(rows), grad


@pytest.mark.parametrize("V,ignore", [(81, [0]), (10000, [0, 1, 2, 3])])
@pytest.mark.parametrize("empty_row", [None, 2])
def test_khot_xent_against_float64(V, ignore, empty_row):
    _need_cuda()
    B = 7  # not a multiple of 8
    logits, labels, ld = _khot_inputs(B, V, ignore, empty_row, seed=V)
    rows, grad = _khot_reference(logits, labels, V, ignore)
    dl, dlab = logits.cuda(), labels.cuda()
    ign = torch.tensor(ignore, dtype=torch.int64, device="cuda")
    loss = torch.zeros(2, device="cuda")
    _call("vtx_khot_xent", dl.data_ptr(), ld, dlab.data_ptr(), dlab.stride(0), B, dlab.shape[1], V, ign.data_ptr(),
          ign.numel(), loss.data_ptr(), 1)
    want = rows.mean()
    if empty_row is None:
        assert abs(loss[0].item() - want.item()) < 1e-5 * abs(want.item())
    else:
        assert torch.isnan(loss[0]) and torch.isnan(want)
        assert torch.equal(dl[empty_row, :V].float().cpu(), torch.zeros(V))
    assert loss[1].item() == 0.0
    assert torch.allclose(dl[:, :V].double().cpu(), grad, rtol=1e-2, atol=2e-7)
    assert torch.equal(dl[:, V:].cpu(), logits[:, V:])
    # forward only: the logits stay as they were
    dl2, loss2 = logits.cuda(), torch.zeros(2, device="cuda")
    _call("vtx_khot_xent", dl2.data_ptr(), ld, dlab.data_ptr(), dlab.stride(0), B, dlab.shape[1], V, ign.data_ptr(),
          ign.numel(), loss2.data_ptr(), 0)
    assert torch.equal(dl2.cpu(), logits)
    if empty_row is None:
        assert abs(loss2[0].item() - loss[0].item()) <= 1e-6 * abs(loss[0].item())
    else:
        assert torch.isnan(loss2[0])


def test_khot_xent_rejects_a_vocabulary_beyond_the_bitmap():
    _need_cuda()
    from virtex_b200 import lib as L
    V = 65536 + 8
    logits = torch.zeros(1, V, device="cuda", dtype=BF16)
    labels = torch.zeros(1, 1, device="cuda", dtype=torch.int64)
    loss = torch.zeros(1, device="cuda")
    with pytest.raises(L.VtxError, match="bitmap"):
        _call("vtx_khot_xent", logits.data_ptr(), V, labels.data_ptr(), 1, 1, 1, V, 0, 0, loss.data_ptr(), 1)


@pytest.mark.parametrize("M,N,ld", [(3, 81, 88), (6, 10000, 10000), (2, 10, 16)])
def test_topk_rows_against_torch(M, N, ld):
    _need_cuda()
    g = torch.Generator().manual_seed(N)
    x = torch.full((M, ld), float("inf"))  # padding columns beyond N are never read
    x[:, :N] = torch.stack([torch.randperm(N, generator=g).float() * 0.37 - 100 for _ in range(M)])
    xd = x.cuda()
    out = torch.empty(M, 10, dtype=torch.int64, device="cuda")
    _call("vtx_topk_rows", xd.data_ptr(), ld, M, N, 10, out.data_ptr())
    assert torch.equal(out.cpu(), x[:, :N].topk(10, dim=1).indices)


# ------------------------------------------------------------------------------------------------------------- models
def _model(name, frozen=False):
    from virtex_b200.models import MultiLabelClassificationModel, TokenClassificationModel
    from virtex_b200.modules import LinearTextualHead, TorchvisionVisualBackbone
    _, vocab, ignore, seed, batch_seed = CO.CASES[name]
    cls = TokenClassificationModel if name == "token_classification" else MultiLabelClassificationModel
    model = cls(TorchvisionVisualBackbone("resnet50", 2048, frozen=frozen), LinearTextualHead(2048, vocab), ignore)
    state = CO.synth_classification_state(vocab, seed)
    model.load_state_dict(state, strict=True)
    return model.cuda().train(), state, vocab, ignore, batch_seed


@pytest.mark.parametrize("name", list(CO.CASES))
@pytest.mark.parametrize("frozen", [False, True])
def test_classification_model_vs_oracle(name, frozen):
    """Loss 1e-3 relative; textual.output.* gradients cos > 0.998, rel < 5e-2; backbone gradients finite (absent when
    frozen); eval loss, and the top-10 wherever the oracle's margins exceed the measured logit error."""
    _need_cuda()
    model, state, vocab, ignore, batch_seed = _model(name, frozen)
    batch = CO.synth_label_batch(6, seed=batch_seed, vocab=vocab, ignore=ignore, image_size=224)
    out = model(to_cuda(batch))
    ref, grads = CO.loss_and_grads(state, batch, ignore, torch.float64)
    assert set(out["loss_components"]) == {"classification"}
    assert abs(out["loss"].item() - ref["loss"].item()) < 1e-3 * ref["loss"].item(), (out["loss"].item(), ref["loss"].item())
    out["loss"].backward()
    for pname, p in model.named_parameters():
        if pname.startswith("textual."):
            r, c = rel(p.grad, grads[pname]), cos(p.grad, grads[pname])
            assert c > 0.998 and r < 5e-2, (pname, r, c)
        elif frozen:
            assert p.grad is None
        else:
            assert p.grad is not None and torch.isfinite(p.grad).all(), pname
    if not frozen:
        assert model.visual.cnn.conv1.weight.grad.abs().sum() > 0
    model.load_state_dict(state, strict=True)  # the BN running statistics the oracle's eval pass uses
    model.eval()
    with torch.no_grad():
        ev = model(to_cuda(batch))
    ref_ev = CO.eval_forward(state, batch, ignore, torch.float64)
    assert abs(ev["loss"].item() - ref_ev["loss"].item()) < 2e-3 * ref_ev["loss"].item()
    pred = ev["predictions"].cpu()
    assert pred.dtype == torch.int64 and pred.shape == (6, 10)
    mine = model.engine._cls["logits_f32"][:, :vocab].double().cpu()
    tol = 4 * (mine - ref_ev["logits"]).abs().max().item()
    top = ref_ev["logits"].topk(11, dim=1).values
    checked = 0
    for b in range(6):
        if top[b, 9] - top[b, 10] > tol:  # the top-10 SET is certain
            assert set(pred[b].tolist()) == set(ref_ev["predictions"][b].tolist()), b
            checked += 1
        gaps = top[b, :-1] - top[b, 1:]
        for i in range(10):  # positions whose neighbours are separated beyond the error
            if (i == 0 or gaps[i - 1] > tol) and gaps[i] > tol:
                assert pred[b, i] == ref_ev["predictions"][b, i], (b, i)
    assert checked >= 1, tol


def test_empty_label_set_on_the_engine():
    """An image with only ignored labels: NaN loss like the reference, finite gradients equal to the oracle's."""
    _need_cuda()
    model, state, vocab, ignore, batch_seed = _model("multilabel_classification")
    batch = CO.synth_label_batch(3, seed=batch_seed, vocab=vocab, ignore=ignore, image_size=224,
                                 empty_rows=(CO.EMPTY_ROW,))
    out = model(to_cuda(batch))
    assert torch.isnan(out["loss"])
    out["loss"].backward()
    _, grads = CO.loss_and_grads(state, batch, ignore, torch.float64)
    g = model.textual.output.weight.grad
    assert torch.isfinite(g).all() and cos(g, grads["textual.output.weight"]) > 0.998
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


def test_trainer_steps_match_the_autograd_loop():
    """Three Trainer.step calls against model -> loss.backward() -> clip -> torch SGD -> LR schedule on a twin."""
    _need_cuda()
    from virtex_b200.config import Config
    from virtex_b200.factories import LRSchedulerFactory, OptimizerFactory, PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = Config("_base_bicaptioning_R_50_L1_H1024.yaml",
                 ["MODEL.NAME", "token_classification", "MODEL.TEXTUAL.NAME", "none", "OPTIM.NO_DECAY", "none",
                  "OPTIM.WARMUP_STEPS", 0, "OPTIM.NUM_ITERATIONS", 100, "OPTIM.LR", 0.05, "OPTIM.CNN_LR", 0.002])
    state = CO.synth_classification_state(10000, 7)
    models = []
    for _ in range(2):
        m = PretrainingModelFactory.from_config(cfg)
        m.load_state_dict(state, strict=True)
        models.append(m.cuda().train())
    trainer = Trainer(models[0], cfg)
    ref = models[1]
    opt = OptimizerFactory.from_config(cfg, ref.named_parameters())
    sched = LRSchedulerFactory.from_config(cfg, opt)
    for it in range(3):
        batch = to_cuda(CO.synth_label_batch(4, seed=60 + it, vocab=10000, ignore=CO.TOKEN_IGNORE,
                                             image_size=224))
        loss = trainer.step(batch)
        opt.zero_grad()
        out = ref(batch)
        out["loss"].backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), cfg.OPTIM.CLIP_GRAD_NORM)
        opt.step()
        sched.step()
        assert loss[1].item() == 0.0
        assert abs(loss[0].item() - out["loss"].item()) < 1e-3 * out["loss"].item(), (it, loss[0].item(), out["loss"].item())
    torch.cuda.synchronize()
    a, b = dict(models[0].named_parameters()), dict(ref.named_parameters())
    for name in ("textual.output.weight", "textual.output.bias"):
        d_a, d_b = a[name].detach().cpu() - state[name], b[name].detach().cpu() - state[name]
        assert d_b.norm() > 0 and rel(d_a, d_b) < 5e-2, (name, rel(d_a, d_b))
    # backbone updates: both moved, finite (bf16 backbone gradients are too ill-conditioned for a tight comparison)
    for name in ("visual.cnn.conv1.weight", "visual.cnn.layer4.2.conv3.weight"):
        d_a = a[name].detach().cpu() - state[name]
        assert torch.isfinite(d_a).all() and d_a.norm() > 0, name
