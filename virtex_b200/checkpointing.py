"""Checkpoint interchange with the reference (SURVEY.md section 8f-4).

`CheckpointManager` keeps the reference's interface and on-disk format (virtex/utils/checkpointing.py:12-174):
`checkpoint_{iteration}.pth` / `checkpoint_best.pth` holding `{name: state_dict, ..., "iteration": int}`, so a file
written by either implementation loads into the other:

  * the model's `state_dict` has the reference's 370 keys (tests/test_host_cpu.py);
  * `FusedOptimizerState` / `FusedSchedulerState` present the fused device-side optimiser tail of
    `virtex_b200.trainer.Trainer` (flat moment arenas, per-name lr / weight decay, step counter) in the state-dict
    layouts the reference's `Lookahead(SGD)` or `Lookahead(AdamW)` + `LinearWarmup*LR` serialise, chosen by
    OPTIM.OPTIMIZER_NAME: one param group per parameter in `named_parameters()` order, `last_epoch`, and per trainable
    parameter index either `momentum_buffer` (torch.optim.SGD) or `step` / `exp_avg` / `exp_avg_sq`
    (torch.optim.AdamW; `step` a 0-dim float32 tensor, the same for every parameter since the fused tail keeps one
    step count -- a file whose parameters disagree on it is refused).  The state is empty before the first step.
    As in the reference, Lookahead's slow weights and k-counter are not part of the state (lookahead.py:61-66): after
    a load the slow weights restart from the loaded parameters.
"""
import copy
import pathlib
from typing import Any, Dict, List, Optional

import torch
from torch import nn

from . import distributed as vdist
from .factories import param_group_hparams
from .trainer import ADAMW_BETAS, ADAMW_EPS


def _unwrap(obj):
    return obj.module if isinstance(obj, nn.parallel.DistributedDataParallel) else obj


class CheckpointManager:
    """Periodically serialise checkpointables (anything with `state_dict` / `load_state_dict`), keep the `keep_recent`
    newest files and, when a metric is given, the best one ("higher is better")."""

    def __init__(self, serialization_dir: str = "/tmp", keep_recent: int = 200, **checkpointables: Any):
        self.serialization_dir = pathlib.Path(serialization_dir)
        self.keep_recent = keep_recent
        self.checkpointables = copy.copy(checkpointables)
        self._best_metric: float = -1e-12
        self._best_ckpt: Dict[str, Any] = {}
        self._recent_iterations: List[int] = []

    def _state_dict(self) -> Dict[str, Any]:
        return {key: _unwrap(obj).state_dict() for key, obj in self.checkpointables.items()}

    def step(self, iteration: int, metric: Optional[float] = None):
        state = self._state_dict()
        state["iteration"] = iteration
        if metric is not None and metric > self._best_metric:
            self._best_metric = metric
            self._best_ckpt = copy.copy(state)
        self.serialization_dir.mkdir(parents=True, exist_ok=True)
        torch.save(state, self.serialization_dir / f"checkpoint_{iteration}.pth")
        if self._best_metric != -1e-12:
            torch.save(self._best_ckpt, self.serialization_dir / "checkpoint_best.pth")
        self._recent_iterations.append(iteration)
        if len(self._recent_iterations) > self.keep_recent:
            self.remove_earliest_checkpoint()

    def remove_earliest_checkpoint(self):
        earliest = self._recent_iterations.pop(0)
        (self.serialization_dir / f"checkpoint_{earliest}.pth").unlink()

    def load(self, checkpoint_path: str) -> int:
        """Load every checkpointable found in the file; returns its iteration (-1 for a best / foreign checkpoint)."""
        checkpoint = torch.load(checkpoint_path, map_location="cpu", weights_only=False)
        iteration = checkpoint.pop("iteration", -1)
        loaded = {key: False for key in self.checkpointables}
        for key, state in checkpoint.items():
            if key in self.checkpointables:
                _unwrap(self.checkpointables[key]).load_state_dict(state)
                loaded[key] = True
        self.not_loaded = [key for key, ok in loaded.items() if not ok]
        self.not_found = [key for key in checkpoint if key not in self.checkpointables]
        return iteration


# ------------------------------------------------------------------------------------- fused optimiser tail <-> torch
_SGD_DEFAULTS = {"dampening": 0, "nesterov": False, "maximize": False, "foreach": None, "differentiable": False,
                 "fused": None}
_ADAMW_DEFAULTS = {"betas": ADAMW_BETAS, "eps": ADAMW_EPS, "amsgrad": False, "maximize": False, "foreach": None,
                   "capturable": False, "differentiable": False, "fused": None, "decoupled_weight_decay": True}


class FusedOptimizerState:
    """`torch.optim.SGD`- or `torch.optim.AdamW`-layout view of a Trainer's moment arenas (one param group per
    parameter, by name), after OPTIM.OPTIMIZER_NAME."""

    def __init__(self, trainer):
        self._t = trainer
        self._adamw = trainer.config.OPTIM.OPTIMIZER_NAME == "adamw"

    def _hparams(self):
        t = self._t
        return [param_group_hparams(t.config, n) for n in t.arena.names]

    @property
    def param_groups(self) -> List[Dict[str, Any]]:
        t = self._t
        mult = t.lr_fn(t.iteration)
        groups = []
        for i, (lr, wd) in enumerate(self._hparams()):
            if self._adamw:
                g = {"lr": lr * mult, "weight_decay": wd}
                g.update(_ADAMW_DEFAULTS)
            else:
                g = {"lr": lr * mult, "weight_decay": wd, "momentum": t.momentum}
                g.update(_SGD_DEFAULTS)
            g["initial_lr"] = lr
            g["params"] = [i]
            groups.append(g)
        return groups

    def state_dict(self) -> Dict[str, Any]:
        if self._adamw:
            return self._adamw_state_dict()
        t = self._t
        a = t.arena
        state = {}
        if t.momentum_ready:
            for i, n in enumerate(a.names):
                if a._param_objs[n].requires_grad:  # torch creates the buffer when a parameter first sees a gradient
                    state[i] = {"momentum_buffer": a.view(t.mom, n).detach().clone()}
        return {"state": state, "param_groups": self.param_groups}

    def _check_groups(self, groups):
        n = len(self._t.arena.names)
        if len(groups) != n or any(len(g["params"]) != 1 for g in groups):
            raise ValueError(f"expected one parameter group per parameter ({n} groups, as built by "
                             f"OptimizerFactory.from_config); the checkpoint has {len(groups)}")

    def load_state_dict(self, state_dict: Dict[str, Any]):
        if self._adamw:
            return self._adamw_load_state_dict(state_dict)
        t = self._t
        a = t.arena
        groups = state_dict["param_groups"]
        self._check_groups(groups)
        state = state_dict.get("state", {})
        t.mom.zero_()
        ready = False
        with torch.no_grad():
            for i, (n, g) in enumerate(zip(a.names, groups)):
                st = state.get(g["params"][0], state.get(str(g["params"][0])))
                buf = None if st is None else st.get("momentum_buffer")
                if buf is None:
                    continue
                if tuple(buf.shape) != tuple(a.shapes[n]):
                    raise ValueError(f"momentum buffer of {n}: shape {tuple(buf.shape)} != {tuple(a.shapes[n])}")
                a.view(t.mom, n).copy_(buf.to(device=t.mom.device, dtype=t.mom.dtype))
                ready = True
        t.momentum_ready = ready
        t.reset_lookahead()

    # ---------------------------------------------------------------------------------------------------- AdamW
    def _adamw_state_dict(self) -> Dict[str, Any]:
        t = self._t
        a = t.arena
        state = {}
        if t.adam_step >= 1:
            for i, n in enumerate(a.names):
                if a._param_objs[n].requires_grad:
                    state[i] = {"step": torch.tensor(float(t.adam_step), dtype=torch.float32),
                                "exp_avg": a.view(t.exp_avg, n).detach().clone(),
                                "exp_avg_sq": a.view(t.exp_avg_sq, n).detach().clone()}
        return {"state": state, "param_groups": self.param_groups}

    def _adamw_load_state_dict(self, state_dict: Dict[str, Any]):
        t = self._t
        a = t.arena
        groups = state_dict["param_groups"]
        state = state_dict.get("state", {})
        if any("momentum_buffer" in st for st in state.values()) or any("betas" not in g for g in groups):
            raise ValueError("the checkpoint holds a torch.optim.SGD state; this Trainer runs AdamW "
                             "(OPTIM.OPTIMIZER_NAME adamw)")
        self._check_groups(groups)
        for g in groups:
            if (tuple(g["betas"]) != ADAMW_BETAS or g["eps"] != ADAMW_EPS or g.get("amsgrad", False)
                    or g.get("maximize", False)):
                raise ValueError(f"the fused AdamW runs betas {ADAMW_BETAS}, eps {ADAMW_EPS}, no amsgrad / maximize; "
                                 f"the checkpoint has betas {g['betas']}, eps {g['eps']}, amsgrad {g.get('amsgrad')}, "
                                 f"maximize {g.get('maximize')}")
        entries, steps = [], set()
        for n, g in zip(a.names, groups):
            if not a._param_objs[n].requires_grad:
                continue
            st = state.get(g["params"][0], state.get(str(g["params"][0])))
            steps.add(0 if st is None else int(round(float(st["step"]))))
            if st is not None:
                for k in ("exp_avg", "exp_avg_sq"):
                    if tuple(st[k].shape) != tuple(a.shapes[n]):
                        raise ValueError(f"{k} of {n}: shape {tuple(st[k].shape)} != {tuple(a.shapes[n])}")
                entries.append((n, st))
        if len(steps) > 1:
            raise ValueError(f"the trainable parameters of the checkpoint have different AdamW step counts "
                             f"{sorted(steps)}; the fused optimiser tail keeps one step count for all of them")
        t.exp_avg.zero_()
        t.exp_avg_sq.zero_()
        with torch.no_grad():
            for n, st in entries:
                a.view(t.exp_avg, n).copy_(st["exp_avg"].to(device=t.exp_avg.device, dtype=t.exp_avg.dtype))
                a.view(t.exp_avg_sq, n).copy_(st["exp_avg_sq"].to(device=t.exp_avg_sq.device, dtype=t.exp_avg_sq.dtype))
        t.adam_step = steps.pop() if steps else 0
        t.reset_lookahead()


class FusedSchedulerState:
    """`LambdaLR`-layout view of a Trainer's step counter (virtex/optim/lr_scheduler.py:9-183 attribute names)."""

    def __init__(self, trainer):
        self._t = trainer

    def state_dict(self) -> Dict[str, Any]:
        t = self._t
        O = t.config.OPTIM
        base = [lr for lr, _ in (param_group_hparams(t.config, n) for n in t.arena.names)]
        mult = t.lr_fn(t.iteration)
        sd: Dict[str, Any] = {"wsteps": O.WARMUP_STEPS}
        if O.LR_DECAY_NAME == "multistep":
            sd.update(milestones=list(O.LR_STEPS), gamma=O.LR_GAMMA)
        else:
            sd["tsteps"] = O.NUM_ITERATIONS
        sd.update(base_lrs=base, last_epoch=t.iteration, _step_count=t.iteration + 1, _is_initial=False,
                  _get_lr_called_within_step=False, _last_lr=[b * mult for b in base], lr_lambdas=[None] * len(base))
        return sd

    def load_state_dict(self, state_dict: Dict[str, Any]):
        self._t.iteration = int(state_dict["last_epoch"])
        sync = getattr(self._t, "sync_dropout_seed", None)
        if sync is not None:
            sync()  # dropout stream position follows the iteration

    def get_last_lr(self) -> List[float]:
        return self.state_dict()["_last_lr"]
