"""Float64 AdamW oracle of the fused optimiser tail -- TEST INFRASTRUCTURE, NOT PRODUCT.

`adamw_update` restates one torch.optim.AdamW step (decoupled weight decay, default betas / eps, no amsgrad) in float64;
`AdamWOracleTrainer` is `oracle.virtex_oracle.OracleTrainer` with that update in place of SGD: the same fp32 CPU
forward / backward, global-norm clip, per-name (lr, weight decay), LR schedule and Lookahead, with the moments, the
Lookahead slow weights and the update arithmetic in float64.  Pinned by tests/golden/trainer_adamw_r50_l1_h128_6steps.pt
(written from the reference's own factories and loop body by scripts/make_adamw_golden.py).
"""
import math
from typing import Dict

import torch

from oracle import virtex_oracle as O

BETAS, EPS = (0.9, 0.999), 1e-8
# OPTIM overrides of the trainer fixture (besides OPTIMIZER_NAME adamw) and the matching oracle configuration
CONFIG_OVERRIDES = ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256", "MODEL.TEXTUAL.DROPOUT", 0.0,
                    "OPTIM.OPTIMIZER_NAME", "adamw", "OPTIM.WARMUP_STEPS", 3, "OPTIM.NUM_ITERATIONS", 20,
                    "OPTIM.BATCH_SIZE", 2, "OPTIM.LR", 1e-3, "OPTIM.CNN_LR", 1e-3]
OPTIM = dict(warmup_steps=3, num_iterations=20, lr=1e-3, cnn_lr=1e-3)


def adamw_update(p, g, m, v, lr, wd, t, betas=BETAS, eps=EPS):
    """One AdamW step at step count t >= 1 on float64 copies; returns (p, m, v).  `g` is the already clipped and scaled
    gradient, `lr` the scheduled learning rate of the tensor."""
    b1, b2 = betas
    p, g, m, v = p.double(), g.double(), m.double(), v.double()
    p = p * (1.0 - lr * wd)
    m = m + (1.0 - b1) * (g - m)
    v = b2 * v + (1.0 - b2) * g * g
    p = p - (lr / (1.0 - b1 ** t)) * m / (v.sqrt() / math.sqrt(1.0 - b2 ** t) + eps)
    return p, m, v


class AdamWOracleTrainer(O.OracleTrainer):
    """The reference step sequence (scripts/pretrain_virtex.py:145-163) with `Lookahead(AdamW)`; the parameters are
    kept as float64 master copies, of which `state` holds the float32 values the forward pass reads."""

    def __init__(self, state, spec: O.Spec, cfg: O.OptimCfg = None):
        super().__init__(state, spec, cfg)
        self.master = {k: v.double() for k, v in self.state.items() if not O.is_buffer(k)}
        self.slow = {k: v.clone() for k, v in self.master.items()}
        self.exp_avg = {k: torch.zeros_like(v) for k, v in self.master.items()}
        self.exp_avg_sq = {k: torch.zeros_like(v) for k, v in self.master.items()}
        self.adam_step = 0

    def step(self, batch) -> Dict[str, torch.Tensor]:
        cfg = self.cfg
        out, grads, new_buffers = O.loss_and_grads(self.state, batch, self.spec)
        self.state.update(new_buffers)
        total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).float()
        clip = min(1.0, cfg.clip_grad_norm / (float(total) + 1e-6))
        mult = O.lr_multiplier(self.iteration, cfg)  # step i uses lambda(i-1)
        self.adam_step += 1
        for name, g in grads.items():
            lr, wd = O.param_hparams(name, cfg)
            self.master[name], self.exp_avg[name], self.exp_avg_sq[name] = adamw_update(
                self.master[name], g.double() * clip, self.exp_avg[name], self.exp_avg_sq[name], lr * mult, wd,
                self.adam_step)
        if cfg.lookahead:
            self.k_counter += 1
            if self.k_counter >= cfg.lookahead_steps:
                self.k_counter = 0
                for name, slow in self.slow.items():
                    slow.add_(self.master[name] - slow, alpha=cfg.lookahead_alpha)
                    self.master[name] = slow.clone()
        for name, p in self.master.items():
            self.state[name] = p.float()
        self.iteration += 1
        out["grad_norm"] = total
        return out
