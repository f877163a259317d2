"""Test-infrastructure tool (CPU): error budget of the BACKWARD pass when conv operands are rounded the way the wgmma
kernels round them (fp16 operands, fp32 accumulate), measured on the oracle against exact fp32 autograd.

    python oracle/grad_error_budget.py [small|default]

It answers, before any backward kernel is written: which backward GEMMs (dgrad, wgrad) can take single-fp16 operands with
a per-tensor power-of-two scale on the gradient, and which need the split-fp16 treatment the forward uses on the
residual-stream layers.  Results are quoted in DESIGN.md section 7.
"""
import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import torch_oracle as O  # noqa: E402
from oracle.make_golden import CASES, TRAIN_CASES  # noqa: E402

_real_conv2d = F.conv2d


def _h(t):
    return t.half().float()


def _scaled_h(g):
    """fp16 rounding of a gradient tensor with a per-tensor power-of-two scale that puts its max near 2^12."""
    m = float(g.abs().max())
    if m == 0.0:
        return g
    s = 2.0 ** (12 - math.ceil(math.log2(m)))
    return _h(g * s) / s


class QConv(torch.autograd.Function):
    """conv2d whose forward / dgrad / wgrad operands are rounded per `mode` = (fwd, dgrad, wgrad), each in {0: exact, 1: fp16}."""

    @staticmethod
    def forward(ctx, x, w, b, stride, padding, mode):
        ctx.save_for_backward(x, w)
        ctx.cfg = (stride, padding, mode, b is not None)
        xq, wq = (_h(x), _h(w)) if mode[0] else (x, w)
        return _real_conv2d(xq, wq, b, stride=stride, padding=padding)

    @staticmethod
    def backward(ctx, gy):
        x, w = ctx.saved_tensors
        stride, padding, mode, has_b = ctx.cfg
        gd = _scaled_h(gy) if mode[1] else gy
        gx = torch.nn.grad.conv2d_input(x.shape, _h(w) if mode[1] else w, gd, stride=stride, padding=padding)
        gwy = _scaled_h(gy) if mode[2] else gy
        gw = torch.nn.grad.conv2d_weight(_h(x) if mode[2] else x, w.shape, gwy, stride=stride, padding=padding)
        gb = gy.sum(dim=(0, 2, 3)) if has_b else None
        return gx, gw, gb, None, None, None


def run(case_name, mode_main, mode_stream):
    """mode_main: 3x3 ResBlock / up / down convs; mode_stream: 1x1 projections, conv_in (read the raw residual stream)."""
    tc = TRAIN_CASES[case_name]
    c = CASES[tc["case"]]
    g = np.load(os.path.join(ROOT, "tests", "golden", case_name + ".npz"))
    inner = c["inner"]

    def grads(patched):
        sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
        for k, v in sd.items():
            if k != "noise_emb.weight":
                v.requires_grad_(True)
        draws = [tuple(torch.from_numpy(g[k][i]) for k in ("raw_sigma", "raw_offset", "raw_noise")) for i in range(tc["seq"])]

        def conv2d(x, w, b=None, stride=1, padding=0):
            stream = w.shape[-1] == 1 or w.shape[1] == (inner.num_steps_conditioning + 1) * inner.img_channels
            return QConv.apply(x, w, b, stride, padding, mode_stream if stream else mode_main)

        F.conv2d = conv2d if patched else _real_conv2d
        try:
            loss = O.denoiser_loss(torch.from_numpy(g["obs"]), torch.from_numpy(g["act"]), torch.from_numpy(g["mask_padding"]),
                                   draws, sd, O.DenoiserCfg(inner=inner), O.SigmaDistCfg())
            loss.backward()
        finally:
            F.conv2d = _real_conv2d
        return loss.item(), {k: v.grad for k, v in sd.items() if v.grad is not None}

    l0, g0 = grads(False)
    l1, g1 = grads(True)
    num = math.sqrt(sum(float((g1[k] - g0[k]).double().pow(2).sum()) for k in g0))
    den = math.sqrt(sum(float(g0[k].double().pow(2).sum()) for k in g0))
    per = sorted(((float((g1[k] - g0[k]).norm() / g0[k].norm().clamp_min(1e-30)), k) for k in g0), reverse=True)
    return abs(l1 - l0) / abs(l0), num / den, per[:3]


if __name__ == "__main__":
    torch.set_num_threads(8)
    which = sys.argv[1] if len(sys.argv) > 1 else "small"
    name = {"small": "denoiser_small_training", "default": "denoiser_default_training"}[which]
    E, H = (0, 0, 0), (1, 1, 1)
    rows = [
        ("forward fp16 (stream layers exact), backward exact", (1, 0, 0), E),
        ("+ dgrad fp16", (1, 1, 0), E),
        ("+ wgrad fp16", (1, 1, 1), E),
        ("everything fp16 incl. stream layers", H, H),
        ("backward only fp16 (forward exact)", (0, 1, 1), E),
    ]
    print(f"case {name}: relative error of the loss / of the whole gradient (L2) / worst tensors")
    for label, mm, ms in rows:
        dl, dg, worst = run(name, mm, ms)
        print(f"{label:55s} loss {dl:.2e}  grad {dg:.2e}  worst {[(round(e, 5), k) for e, k in worst]}")
