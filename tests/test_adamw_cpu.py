"""AdamW in the fused optimiser tail, host side: the float64 AdamW oracle against the reference's own AdamW run, and
the `torch.optim.AdamW`-layout checkpoint view of the Trainer against real torch optimisers."""
import os

import pytest
import torch

from oracle import virtex_oracle as O
from tests import adamw_oracle as AO
from tests.test_host_cpu import _fake_trainer


def test_adamw_oracle_trajectory_matches_reference_fixture(golden_dir):
    """6 reference steps of Lookahead(AdamW) (per-parameter groups, clip 10, k = 5, warm-up LR): losses, gradient norms,
    final parameter norms and the accumulated update of the head probes."""
    g = torch.load(os.path.join(golden_dir, "trainer_adamw_r50_l1_h128_6steps.pt"), weights_only=False)
    spec = O.Spec(**g["spec"])
    init = O.synth_state(spec, g["seed"])
    tr = AO.AdamWOracleTrainer(init, spec, O.OptimCfg(**g["optim"]))
    for it in range(6):
        out = tr.step(O.synth_batch(2, seed=10 + it))
        assert abs(out["loss"].item() - g["losses"][it].item()) < 5e-4 * g["losses"][it].item(), it
        assert abs(out["grad_norm"].item() - g["grad_norms"][it].item()) < 5e-2 * g["grad_norms"][it].item(), it
    assert tr.adam_step == 6 and tr.k_counter == 1
    lr = g["optim"]["lr"]
    assert g["optim"]["cnn_lr"] == lr
    for k, ref_norm in g["final_param_norms"].items():
        err = abs(tr.state[k].double().norm().item() - ref_norm)
        if k.startswith("visual."):
            # float32 backbone gradients carry ~2% noise (see the SGD trajectory test), and AdamW moves every element
            # by ~lr per step whatever its gradient's size, so an element whose gradient sign is noise lands up to a
            # few lr away: bound the norm by that displacement (measured: at most 0.18 sqrt(n) lr)
            assert err <= 0.5 * tr.state[k].numel() ** 0.5 * lr, k
        else:
            assert err <= 1e-3 * ref_norm, k  # measured: at most 4.9e-4 relative
    for k, probe in g["final_probe"].items():
        if k.startswith("visual."):  # see above
            continue
        d_ref = probe.double() - init[k].flatten()[:64].double()
        d_ora = tr.state[k].flatten()[:64].double() - init[k].flatten()[:64].double()
        assert (d_ora - d_ref).norm() <= 0.02 * d_ref.norm(), k  # measured: 2.7e-3


def test_adamw_update_matches_torch_adamw():
    """The float64 restatement == torch.optim.AdamW in float64 over steps 1..3 with lr, weight decay and a large t."""
    torch.manual_seed(0)
    p = torch.randn(50, dtype=torch.float64)
    for lr, wd in ((1e-3, 1e-4), (0.2, 0.0)):
        q = torch.nn.Parameter(p.clone())
        opt = torch.optim.AdamW([q], lr=lr, weight_decay=wd)
        x, m, v = p.clone(), torch.zeros_like(p), torch.zeros_like(p)
        for t in range(1, 4):
            g = torch.randn_like(p)
            q.grad = g.clone()
            opt.step()
            x, m, v = AO.adamw_update(x, g, m, v, lr, wd, t)
            assert torch.allclose(q.detach(), x, rtol=1e-12, atol=1e-14)
            assert torch.allclose(opt.state[q]["exp_avg_sq"], v, rtol=1e-12, atol=1e-16)


# ------------------------------------------------------------------------------------------ checkpoint interchange
def _adamw_config(lookahead=True):
    from virtex_b200.config import Config
    return Config(None, ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256", "OPTIM.OPTIMIZER_NAME", "adamw",
                         "OPTIM.CNN_LR", 0.1, "OPTIM.LR", 0.001, "OPTIM.WARMUP_STEPS", 4, "OPTIM.NUM_ITERATIONS", 20,
                         "OPTIM.LOOKAHEAD.USE", lookahead])


def _fake_adamw_trainer(model, config):
    """`_fake_trainer` plus the AdamW fields of `Trainer`."""
    t = _fake_trainer(model, config)
    t.exp_avg = torch.zeros_like(t.arena.params)
    t.exp_avg_sq = torch.zeros_like(t.arena.params)
    t.adam_step = 0
    return t


def _torch_adamw(cfg, seed=0, steps=3):
    """The reference recipe: Lookahead(AdamW) + LambdaLR from the factories, `steps` steps on random gradients."""
    from virtex_b200.factories import LRSchedulerFactory, OptimizerFactory, PretrainingModelFactory
    torch.manual_seed(seed)
    model = PretrainingModelFactory.from_config(cfg)
    opt = OptimizerFactory.from_config(cfg, model.named_parameters())
    sch = LRSchedulerFactory.from_config(cfg, opt)
    for _ in range(steps):
        for p in model.parameters():
            if p.requires_grad:
                p.grad = torch.randn_like(p) * 0.01
        opt.step()
        sch.step()
    return model, opt, sch


def test_adamw_view_has_the_layout_of_torch_adamw():
    from virtex_b200.checkpointing import FusedOptimizerState
    from virtex_b200.factories import PretrainingModelFactory
    cfg = _adamw_config()
    _, opt, _ = _torch_adamw(cfg, steps=2)
    ref = opt.state_dict()
    tr = _fake_adamw_trainer(PretrainingModelFactory.from_config(cfg), cfg)
    tr.adam_step, tr.iteration = 2, 2
    sd = FusedOptimizerState(tr).state_dict()
    assert len(sd["param_groups"]) == len(ref["param_groups"]) == len(tr.arena.names)
    for g, gr in zip(sd["param_groups"], ref["param_groups"]):
        assert set(g) == set(gr)
        for k, v in gr.items():
            assert g[k] == pytest.approx(v, rel=1e-12, abs=0) if isinstance(v, float) else g[k] == v, k
    assert set(sd["state"]) == set(ref["state"])
    for i, st in ref["state"].items():
        assert set(sd["state"][i]) == set(st)
        for k, v in st.items():
            assert sd["state"][i][k].dtype == v.dtype and sd["state"][i][k].shape == v.shape, (i, k)
        assert sd["state"][i]["step"].item() == st["step"].item() == 2.0


def test_adamw_checkpoint_interchange_both_ways(tmp_path):
    """Reference layout -> fused view -> file -> fresh torch AdamW + scheduler, which then steps exactly like the
    optimiser that wrote the first file."""
    from virtex_b200.checkpointing import CheckpointManager, FusedOptimizerState, FusedSchedulerState
    from virtex_b200.factories import LRSchedulerFactory, OptimizerFactory, PretrainingModelFactory
    cfg = _adamw_config()
    model, opt, sch = _torch_adamw(cfg, steps=3)
    CheckpointManager(str(tmp_path / "ref"), model=model, optimizer=opt, scheduler=sch).step(3)

    model2 = PretrainingModelFactory.from_config(cfg)
    tr = _fake_adamw_trainer(model2, cfg)
    mgr = CheckpointManager(str(tmp_path / "ours"), model=model2, optimizer=FusedOptimizerState(tr),
                            scheduler=FusedSchedulerState(tr))
    assert mgr.load(str(tmp_path / "ref" / "checkpoint_3.pth")) == 3
    assert mgr.not_loaded == [] and mgr.not_found == []
    assert tr.iteration == 3 and tr.adam_step == 3 and tr._k_counter == 0 and not tr.momentum_ready
    sd = opt.state_dict()
    for i, n in enumerate(tr.arena.names):
        assert torch.equal(tr.arena.view(tr.exp_avg, n), sd["state"][i]["exp_avg"]), n
        assert torch.equal(tr.arena.view(tr.exp_avg_sq, n), sd["state"][i]["exp_avg_sq"]), n
    assert torch.equal(tr.slow, tr.arena.params)  # Lookahead restarts from the loaded weights

    mgr.step(3)
    model3 = PretrainingModelFactory.from_config(cfg)
    opt3 = OptimizerFactory.from_config(cfg, model3.named_parameters())
    sch3 = LRSchedulerFactory.from_config(cfg, opt3)
    assert CheckpointManager(str(tmp_path / "x"), model=model3, optimizer=opt3, scheduler=sch3).load(
        str(tmp_path / "ours" / "checkpoint_3.pth")) == 3
    sd3 = opt3.state_dict()
    for g, g3 in zip(sd["param_groups"], sd3["param_groups"]):
        assert g == pytest.approx(g3, rel=1e-12, abs=0)
    for i in sd["state"]:
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(sd["state"][i][k], sd3["state"][i][k]), (i, k)
    assert sch3.last_epoch == 3 and sch3.get_last_lr() == pytest.approx(sch.get_last_lr())
    # opt3 starts a Lookahead cycle at the loaded weights: put the writer on the same footing (slow weights, counter)
    opt.load_state_dict(opt.state_dict())
    opt._k_counter = 0
    gen = torch.Generator().manual_seed(5)
    for _ in range(3):
        for p, p3 in zip(model.parameters(), model3.parameters()):
            p.grad = torch.randn(p.shape, generator=gen) * 0.01
            p3.grad = p.grad.clone()
        opt.step(); sch.step(); opt3.step(); sch3.step()
    for (n, p), p3 in zip(model.named_parameters(), model3.parameters()):
        assert torch.equal(p, p3), n


def test_adamw_view_is_empty_before_the_first_step_and_skips_frozen_parameters():
    from virtex_b200.checkpointing import FusedOptimizerState
    from virtex_b200.factories import PretrainingModelFactory
    cfg = _adamw_config()
    model = PretrainingModelFactory.from_config(cfg)
    for p in model.visual.parameters():
        p.requires_grad = False
    tr = _fake_adamw_trainer(model, cfg)
    view = FusedOptimizerState(tr)
    sd = view.state_dict()
    assert sd["state"] == {} and len(sd["param_groups"]) == len(tr.arena.names)
    assert all(g["lr"] == 0.0 and g["betas"] == (0.9, 0.999) for g in sd["param_groups"])
    tr.adam_step, tr.iteration = 1, 1
    sd = view.state_dict()
    frozen = [i for i, n in enumerate(tr.arena.names) if n.startswith("visual.")]
    assert frozen and all(i not in sd["state"] for i in frozen)
    assert len(sd["state"]) == len(tr.arena.names) - len(frozen)
    # and a file written with frozen parameters loads back (no state for them, one step count for the others)
    tr.exp_avg.fill_(1.0)
    view.load_state_dict(sd)
    assert tr.adam_step == 1 and all(tr.arena.view(tr.exp_avg, tr.arena.names[i]).eq(0).all() for i in frozen)


def test_adamw_view_rejects_foreign_states():
    from virtex_b200.checkpointing import FusedOptimizerState
    from virtex_b200.factories import PretrainingModelFactory
    cfg = _adamw_config(lookahead=False)
    tr = _fake_adamw_trainer(PretrainingModelFactory.from_config(cfg), cfg)
    view = FusedOptimizerState(tr)
    # an SGD-layout state (the reference recipe with OPTIMIZER_NAME sgd)
    from tests.test_host_cpu import _tiny_config
    from virtex_b200.factories import OptimizerFactory
    model = PretrainingModelFactory.from_config(_tiny_config())
    sgd = OptimizerFactory.from_config(_tiny_config(), model.named_parameters())
    for p in model.parameters():
        p.grad = torch.ones_like(p)
    sgd.step()
    with pytest.raises(ValueError, match="SGD"):
        view.load_state_dict(sgd.state_dict())
    # a group count mismatch
    _, opt, _ = _torch_adamw(cfg, steps=1)
    sd = opt.state_dict()
    with pytest.raises(ValueError, match="one parameter group per parameter"):
        view.load_state_dict({"state": sd["state"], "param_groups": sd["param_groups"][:-1]})
    # trainable parameters at different step counts
    sd["state"][4]["step"] = torch.tensor(2.0)
    with pytest.raises(ValueError, match="step count"):
        view.load_state_dict(sd)
    assert tr.adam_step == 0


def test_trainer_rejects_an_unknown_optimizer():
    from virtex_b200.config import Config
    from virtex_b200.trainer import Trainer
    with pytest.raises(NotImplementedError, match="adamw"):
        Trainer(None, Config(None, ["OPTIM.OPTIMIZER_NAME", "adagrad"]))
