"""AdamW in the fused optimiser tail on the H100: `vtx_adamw_step` against float64 AdamW, a 6-step Trainer run against
the AdamW oracle (tests/adamw_oracle.py, pinned to the reference by tests/test_adamw_cpu.py), checkpoint resume, and
frozen parameters.

Per-element parameter updates are checked on identical gradients only: AdamW's first steps are close to sign(g), so
elements with tiny gradients flip with bf16 gradient noise and a trainer-vs-oracle comparison of parameter deltas says
little.  The trajectory against the oracle is checked on losses and gradient norms."""
import struct

import pytest
import torch

from oracle import virtex_oracle as O
from tests import adamw_oracle as AO

pytestmark = pytest.mark.gpu


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _seg_blob(segs, dev="cuda"):
    return torch.frombuffer(bytearray(b"".join(struct.pack("<qqff", *s) for s in segs)), dtype=torch.uint8).to(dev)


def _adamw_ref(p, g, m, v, slow, lr, wd, t, do_la, alpha):
    """float64 AdamW (+ the Lookahead interpolation when do_la); lr / wd scalars or per-element vectors.  Returns the
    new (p, m, v) and the tolerances of fp32 p and m.  m = m0 + (1 - beta1) (g - m0) can cancel to far below its
    terms, so fp32 rounds it relative to |m0| and |g|: the same step on |m0| and |g| gives the scale of m and of the
    update whose error the fp32 step may carry; p adds its own rounding."""
    fast, m1, v1 = AO.adamw_update(p, g, m, v, lr, wd, t)
    big, m_scale, _ = AO.adamw_update(p, g.abs(), m.abs(), v, lr, 0.0, t)
    tol = 1e-5 * (big - p.double()).abs() + 1e-6 * fast.abs()
    if do_la:
        fast = alpha * fast + (1.0 - alpha) * slow.double()
        tol = alpha * tol + 1e-6 * (fast.abs() + slow.double().abs())
    return fast, m1, v1, tol, 1e-6 * m_scale


@pytest.mark.parametrize("t", [1, 1000])
@pytest.mark.parametrize("max_norm", [1.0, 1e6])  # clip coefficient < 1, = 1
@pytest.mark.parametrize("do_la", [False, True])
def test_adamw_step_kernel_against_float64(t, max_norm, do_la):
    """Ragged segments (tails of 64 Ki chunks, a wd = 0 group, gaps standing for frozen tensors): parameters, moments
    and slow weights within fp32 rounding of float64 AdamW, the gaps bit-identical, the bf16 mirror == bf16(p)."""
    _need_cuda()
    from virtex_b200.ops import _stream, call
    torch.manual_seed(11)
    dev = "cuda"
    n = 300_017
    # (begin, end, lr, wd): a 3-chunk tensor with a 13-element tail, a wd = 0 tensor, a gap, a short odd tensor, a gap
    tensors = [(0, 2 * 65536 + 13, 0.2, 1e-4), (2 * 65536 + 13, 200_000, 1e-3, 0.0), (210_000, 210_777, 5e-3, 1e-2),
               (211_000, 300_000, 1e-3, 1e-4)]
    segs = [(c, min(e, c + 65536), lr, wd) for b, e, lr, wd in tensors for c in range(b, e, 65536)]
    blob = _seg_blob(segs)
    p = torch.randn(n, device=dev)
    g = torch.randn(n, device=dev) * torch.logspace(-9, 0, n, device=dev)[torch.randperm(n, device=dev)]
    # moments of a run in progress: |m| <= sqrt(v), as AdamW's own moments are (up to the bias corrections)
    m = torch.randn(n, device=dev) * 1e-2 if t > 1 else torch.zeros(n, device=dev)
    v = m * m * (1.0 + 9.0 * torch.rand(n, device=dev)) if t > 1 else torch.zeros(n, device=dev)
    slow = torch.randn(n, device=dev)
    bf = torch.zeros(n, device=dev, dtype=torch.bfloat16)
    p0, m0, v0, s0 = p.clone(), m.clone(), v.clone(), slow.clone()
    ssq = (g.double() ** 2).sum().float().reshape(1)
    ctl = torch.zeros(2, device=dev)
    call("vtx_clip_coef", ssq.data_ptr(), 1, max_norm, ctl.data_ptr(), _stream())
    mult = 0.37
    hyper = torch.tensor([mult, 1.0 / (1.0 - 0.9 ** t), 1.0 / (1.0 - 0.999 ** t) ** 0.5, float(do_la)], device=dev)
    call("vtx_adamw_step", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), slow.data_ptr(), bf.data_ptr(),
         blob.data_ptr(), len(segs), ctl.data_ptr(), hyper.data_ptr(), 0.9, 0.999, 1e-8, 0.5, _stream())
    torch.cuda.synchronize()
    scale = ctl[0].item()
    assert (scale < 1.0) == (max_norm == 1.0)
    inside = torch.zeros(n, dtype=torch.bool, device=dev)
    for b, e, lr, wd in tensors:
        inside[b:e] = True
        rp, rm, rv, tol, mtol = _adamw_ref(p0[b:e], g[b:e].double() * scale, m0[b:e], v0[b:e], s0[b:e], lr * mult,
                                           wd, t, do_la, 0.5)
        assert ((p[b:e].double() - rp).abs() <= tol).all(), (b, e)
        assert ((m[b:e].double() - rm).abs() <= mtol).all(), (b, e)
        assert torch.allclose(v[b:e].double(), rv, rtol=1e-5, atol=1e-20), (b, e)
        if do_la:
            assert torch.equal(slow[b:e], p[b:e])
        assert torch.equal(bf[b:e], p[b:e].bfloat16())
    out = ~inside
    assert torch.equal(p[out], p0[out]) and torch.equal(m[out], m0[out]) and torch.equal(v[out], v0[out])
    assert torch.equal(slow[out], s0[out]) and (bf[out] == 0).all()
    if not do_la:
        assert torch.equal(slow, s0)


def _arena_hparams(tr):
    """Per-element float64 (lr, wd) vectors of a Trainer's arena (0 outside every trainable tensor)."""
    from virtex_b200.factories import param_group_hparams
    a = tr.arena
    lr = torch.zeros(a.total, dtype=torch.float64, device=a.params.device)
    wd = torch.zeros_like(lr)
    for n in a.names:
        if a._param_objs[n].requires_grad:
            o, k = a.offsets[n], a.numels[n]
            lr[o:o + k], wd[o:o + k] = param_group_hparams(tr.config, n)
    return lr, wd


def _trainer_config(*extra):
    from virtex_b200.config import Config
    return Config(None, AO.CONFIG_OVERRIDES + ["OPTIM.BATCH_SIZE", 4] + list(extra))


def test_adamw_trainer_trajectory_vs_oracle():
    """6 fused AdamW steps (crossing the Lookahead boundary) track the float64 AdamW oracle on losses and gradient
    norms, and every step's update equals float64 AdamW applied to the trainer's own clipped gradient arena."""
    _need_cuda()
    from tests.helpers import build_model, to_cuda
    from virtex_b200.trainer import Trainer
    spec = O.Spec(hidden=128, layers=1, heads=2, ffn=256)
    state = O.synth_state(spec, 3, bn3_gain=0.25)
    model = build_model(spec, state).train()
    cfg = _trainer_config()
    tr = Trainer(model, cfg)
    ora = AO.AdamWOracleTrainer(state, spec, O.OptimCfg(**AO.OPTIM))
    a = tr.arena
    lr_vec, wd_vec = _arena_hparams(tr)
    trainable = lr_vec != 0
    for it in range(6):
        p0, m0, v0, s0 = a.params.clone(), tr.exp_avg.clone(), tr.exp_avg_sq.clone(), tr.slow.clone()
        batch = O.synth_batch(4, seed=30 + it, ragged=True)
        loss = tr.step(to_cuda(batch)).sum().item()
        ref = ora.step(batch)
        assert abs(loss - ref["loss"].item()) < 3e-3 * ref["loss"].item(), (it, loss, ref["loss"].item())
        assert abs(tr.grad_norm.item() - ref["grad_norm"].item()) < 0.1 * ref["grad_norm"].item(), it
        # the optimiser step itself, on the gradients this step produced
        mult = tr.lr_fn(it)
        do_la = it == 4  # k = 5
        rp, rm, rv, tol, mtol = _adamw_ref(p0, a.grads.double() * tr.ctl[0].item(), m0, v0, s0, lr_vec * mult,
                                           wd_vec, it + 1, do_la, tr.la_alpha)
        err = (a.params.double() - rp)[trainable].abs()
        assert (err <= tol[trainable]).all(), (it, err.max().item())
        assert ((tr.exp_avg.double() - rm)[trainable].abs() <= mtol[trainable]).all(), it
        assert torch.allclose(tr.exp_avg_sq.double()[trainable], rv[trainable], rtol=1e-5, atol=1e-20), it
        assert torch.equal(a.mirror[trainable], a.params[trainable].bfloat16()), it
    assert tr.adam_step == 6 and tr._k_counter == 1


def _resume_config():
    return _trainer_config("OPTIM.BATCH_SIZE", 2, "OPTIM.WARMUP_STEPS", 2, "OPTIM.LOOKAHEAD.USE", False)


def test_adamw_trainer_checkpoint_resume_matches_uninterrupted_run(tmp_path):
    """3 steps -> CheckpointManager.step -> fresh model + Trainer -> load -> 3 more steps == 6 uninterrupted steps."""
    _need_cuda()
    from tests.helpers import to_cuda
    from virtex_b200.checkpointing import CheckpointManager
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = _resume_config()
    batch = to_cuda(O.synth_batch(2, seed=9, ragged=True))

    def fresh():
        torch.manual_seed(3)
        m = PretrainingModelFactory.from_config(cfg).cuda().train()
        return m, Trainer(m, cfg)

    m_a, tr_a = fresh()
    losses_a = [tr_a.step(batch).sum().item() for _ in range(6)]
    m_b, tr_b = fresh()
    losses_b = [tr_b.step(batch).sum().item() for _ in range(3)]
    CheckpointManager(str(tmp_path), model=m_b, optimizer=tr_b.optimizer, scheduler=tr_b.scheduler).step(3)
    ck = torch.load(tmp_path / "checkpoint_3.pth", weights_only=False)
    assert all(float(st["step"]) == 3.0 for st in ck["optimizer"]["state"].values())
    m_c, tr_c = fresh()
    mgr = CheckpointManager(str(tmp_path), model=m_c, optimizer=tr_c.optimizer, scheduler=tr_c.scheduler)
    assert mgr.load(str(tmp_path / "checkpoint_3.pth")) == 3 and tr_c.iteration == 3 and tr_c.adam_step == 3
    assert torch.equal(tr_c.exp_avg, tr_b.exp_avg) and torch.equal(tr_c.exp_avg_sq, tr_b.exp_avg_sq)
    tr_c.engine.mark_weights_dirty()
    losses_b += [tr_c.step(batch).sum().item() for _ in range(3)]
    for a, b in zip(losses_a, losses_b):
        assert abs(a - b) < 2e-3 * abs(a), (losses_a, losses_b)


def test_adamw_trainer_continues_a_checkpoint_of_the_eager_torch_loop(tmp_path):
    """The eager loop (autograd on the engine, clip_grad_norm_, torch.optim.AdamW on CUDA, LambdaLR) writes a checkpoint
    after 3 steps; a fresh Trainer loads it and its next 3 losses follow the eager loop's next 3."""
    _need_cuda()
    from tests.helpers import to_cuda
    from virtex_b200.checkpointing import CheckpointManager
    from virtex_b200.factories import LRSchedulerFactory, OptimizerFactory, PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = _resume_config()
    torch.manual_seed(3)
    model = PretrainingModelFactory.from_config(cfg).cuda().train()
    opt = OptimizerFactory.from_config(cfg, model.named_parameters())
    assert isinstance(opt, torch.optim.AdamW)
    sch = LRSchedulerFactory.from_config(cfg, opt)
    batches = [to_cuda(O.synth_batch(2, seed=40 + i, ragged=True)) for i in range(6)]
    eager = []
    for i in range(6):
        if i == 3:
            CheckpointManager(str(tmp_path), model=model, optimizer=opt, scheduler=sch).step(3)
        opt.zero_grad()
        out = model(batches[i])
        out["loss"].backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), cfg.OPTIM.CLIP_GRAD_NORM)
        opt.step()
        sch.step()
        eager.append(out["loss"].item())
    torch.manual_seed(4)  # different initial weights: everything must come from the file
    m2 = PretrainingModelFactory.from_config(cfg).cuda().train()
    tr = Trainer(m2, cfg)
    mgr = CheckpointManager(str(tmp_path), model=m2, optimizer=tr.optimizer, scheduler=tr.scheduler)
    assert mgr.load(str(tmp_path / "checkpoint_3.pth")) == 3 and tr.adam_step == 3 and not mgr.not_loaded
    tr.engine.mark_weights_dirty()
    fused = [tr.step(batches[i]).sum().item() for i in range(3, 6)]
    for a, b in zip(eager[3:], fused):
        assert abs(a - b) < 2e-3 * abs(a), (eager, fused)


def test_adamw_trainer_leaves_a_frozen_backbone_and_its_moments_bit_identical():
    """Token classification with MODEL.VISUAL.FROZEN: two AdamW Trainer steps leave every backbone parameter, its
    moments (set to non-zero values, as after a checkpoint load) and its bf16 mirror bit-identical, and move the head."""
    _need_cuda()
    from tests import classification_oracle as CO
    from virtex_b200.config import Config
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = Config("_base_bicaptioning_R_50_L1_H1024.yaml",
                 ["MODEL.NAME", "token_classification", "MODEL.TEXTUAL.NAME", "none", "MODEL.VISUAL.FROZEN", True,
                  "OPTIM.OPTIMIZER_NAME", "adamw", "OPTIM.WARMUP_STEPS", 0, "OPTIM.NUM_ITERATIONS", 100,
                  "OPTIM.LR", 1e-3, "OPTIM.CNN_LR", 1e-3, "OPTIM.LOOKAHEAD.STEPS", 2])
    model = PretrainingModelFactory.from_config(cfg)
    model.load_state_dict(CO.synth_classification_state(10000, 7), strict=True)
    model = model.cuda().train()
    tr = Trainer(model, cfg)
    a = tr.arena
    frozen = [n for n in a.names if not a._param_objs[n].requires_grad]
    assert frozen and all(n.startswith("visual.") for n in frozen)
    torch.manual_seed(1)
    tr.exp_avg.copy_(torch.randn_like(tr.exp_avg))
    tr.exp_avg_sq.copy_(torch.rand_like(tr.exp_avg_sq))
    before = {n: [a.view(x, n).clone() for x in (a.params, tr.exp_avg, tr.exp_avg_sq, a.mirror)] for n in a.names}
    for it in range(2):  # the second step ends a Lookahead cycle
        tr.step({k: v.cuda() for k, v in CO.synth_label_batch(4, seed=60 + it, vocab=10000, ignore=CO.TOKEN_IGNORE,
                                                                image_size=224).items()})
    torch.cuda.synchronize()
    for n in frozen:
        for x, b in zip((a.params, tr.exp_avg, tr.exp_avg_sq, a.mirror), before[n]):
            assert torch.equal(a.view(x, n), b), n
    assert not torch.equal(a.p("textual.output.weight"), before["textual.output.weight"][0])
    sd = tr.optimizer.state_dict()
    assert set(sd["state"]) == {i for i, n in enumerate(a.names) if n not in frozen}
