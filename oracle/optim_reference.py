"""Float64 restatement of the reference's optimizer step (src/trainer.py:373-377): `torch.nn.utils.clip_grad_norm_` with the
default 2-norm, then torch 2.11's `AdamW` (decoupled weight decay, amsgrad / maximize off), over parameter groups split the way
`utils.configure_opt` (src/utils.py:129-166) splits them.  Plain Python / torch float64 arithmetic, no torch optimizer: the
checker for diamond_b200.optim (tests/test_optim_host.py pins it to torch itself on CPU)."""
from typing import Dict, List, Sequence

import torch
import torch.nn as nn

# utils.py:134-135: weights of these modules decay, everything else (biases, norm / embedding weights) does not
DECAY_MODULES = (nn.Linear, nn.Conv1d, nn.Conv2d, nn.LSTMCell, nn.LSTM)


def configure_opt_groups(model: nn.Module, weight_decay: float) -> List[Dict]:
    """The two parameter groups of utils.configure_opt: decayed weights and the rest, each sorted by parameter name."""
    mods = dict(model.named_modules())
    decay, no_decay = [], []
    for name, _ in model.named_parameters():
        owner, _, leaf = name.rpartition(".")
        is_weight = leaf.endswith("weight") or leaf.startswith("weight_")
        if "bias" not in leaf and is_weight and isinstance(mods[owner], DECAY_MODULES):
            decay.append(name)
        else:
            no_decay.append(name)
    params = dict(model.named_parameters())
    return [{"params": [params[n] for n in sorted(decay)], "weight_decay": weight_decay},
            {"params": [params[n] for n in sorted(no_decay)], "weight_decay": 0.0}]


def clip_grad_norm(grads: Sequence[torch.Tensor], max_norm: float):
    """(clipped grads, total_norm, coefficient) in float64: total = ||all grads||_2, coef = min(1, max_norm / (total + 1e-6))."""
    g64 = [g.double() for g in grads]
    total = torch.sqrt(sum((g * g).sum() for g in g64)) if g64 else torch.zeros((), dtype=torch.float64)
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    return [g * coef for g in g64], total, coef


def adamw_step(params: Sequence[torch.Tensor], grads: Sequence[torch.Tensor], exp_avgs: Sequence[torch.Tensor],
               exp_avg_sqs: Sequence[torch.Tensor], weight_decays: Sequence[float], step: int, lr: float, betas=(0.9, 0.999),
               eps: float = 1e-8):
    """One AdamW step at step count `step` (after the increment), float64.  Returns new (params, exp_avgs, exp_avg_sqs)."""
    b1, b2 = betas
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    out_p, out_m, out_v = [], [], []
    for p, g, m, v, wd in zip(params, grads, exp_avgs, exp_avg_sqs, weight_decays):
        p, g, m, v = p.double(), g.double(), m.double(), v.double()
        p = p * (1 - lr * wd)
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        p = p - (lr / bc1) * m / (v.sqrt() / bc2 ** 0.5 + eps)
        out_p.append(p)
        out_m.append(m)
        out_v.append(v)
    return out_p, out_m, out_v


def train_steps(params: Sequence[torch.Tensor], grads_per_step: Sequence[Sequence[torch.Tensor]], weight_decays: Sequence[float],
                max_norm, lr: float, betas=(0.9, 0.999), eps: float = 1e-8):
    """`len(grads_per_step)` steps of clip (skipped when max_norm is None) + AdamW from zero moments; float64 params out."""
    p = [t.double() for t in params]
    m = [torch.zeros_like(t) for t in p]
    v = [torch.zeros_like(t) for t in p]
    for k, grads in enumerate(grads_per_step):
        g = [t.double() for t in grads]
        if max_norm is not None:
            g = clip_grad_norm(g, max_norm)[0]
        p, m, v = adamw_step(p, g, m, v, weight_decays, k + 1, lr, betas, eps)
    return p, m, v
