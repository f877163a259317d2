"""Test-infrastructure tool (CPU): error budget of the BACKWARD pass when conv operands are rounded the way the wgmma
kernels round them (fp16 operands, fp32 accumulate), measured on the oracle against exact fp32 autograd.

    python oracle/grad_error_budget.py [small|default]                 operand-rounding rows, per-tensor gradient scale
    python oracle/grad_error_budget.py [small|default] --exp 12 8 ...  the kernels' scheme: ONE scale per backward call

It answers, before any backward kernel is written: which backward GEMMs (dgrad, wgrad) can take single-fp16 operands with
a per-tensor power-of-two scale on the gradient, and which need the split-fp16 treatment the forward uses on the
residual-stream layers.  Results are quoted in DESIGN.md section 7.

The kernels do not scale per tensor: dmd_denoiser_backward picks one power-of-two S per call from max|dL/d(model output)| so
that it lands in [2^(E-1), 2^E), E = DMD_LOSS_SCALE_EXP (include/diamond_b200.h), and every conv gradient operand of that call
is fp16(S * dL/dy).  `--exp` emulates exactly that (conv_out, the first conv the backward meets, fixes S), which shows the cost
of a smaller E: gradients far below max|dL/d(output)| fall into the fp16 subnormals (2^-24 .. 2^-14) and lose precision.
`--gain k` multiplies conv_out.weight by k, which makes inner gradients ~0.29 k times the output gradient (default net): the
headroom a trained network may need; an overflowing operand shows up as a non-finite error.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import torch_oracle as O  # noqa: E402
from oracle.fp16_emulation import denoiser_stream, grad_errors  # noqa: E402
from oracle.make_golden import CASES, TRAIN_CASES  # noqa: E402


def run(case_name, mode_main, mode_stream, exp=None, gain=1.0):
    """mode_main: 3x3 ResBlock / up / down convs; mode_stream: 1x1 projections, conv_in (read the raw residual stream).
    exp: None = per-tensor gradient scale, else one scale per backward call with max|S dL/d(output)| in [2^(exp-1), 2^exp).
    gain: multiplies conv_out.weight."""
    tc = TRAIN_CASES[case_name]
    c = CASES[tc["case"]]
    g = np.load(os.path.join(ROOT, "tests", "golden", case_name + ".npz"))
    inner = c["inner"]
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
    sd["conv_out.weight"] *= gain
    for k, v in sd.items():
        if k != "noise_emb.weight":
            v.requires_grad_(True)
    draws = [tuple(torch.from_numpy(g[k][i]) for k in ("raw_sigma", "raw_offset", "raw_noise")) for i in range(tc["seq"])]

    def loss_fn(p):
        return O.denoiser_loss(torch.from_numpy(g["obs"]), torch.from_numpy(g["act"]), torch.from_numpy(g["mask_padding"]),
                               draws, p, O.DenoiserCfg(inner=inner), O.SigmaDistCfg())

    l0, l1, whole, per, _ = grad_errors(loss_fn, sd, denoiser_stream(sd), "conv_out.weight", exp, mode_main, mode_stream)
    worst = sorted(((e, k) for k, e in per.items()), reverse=True)
    return abs(l1 - l0) / abs(l0), whole, worst[:3]


def per_call_rows(name, exps, gain=1.0):
    """The kernels' operand rounding (forward fp16 with exact stream layers, backward fp16 everywhere) under a per-tensor scale
    and under one scale per call for each E in exps: [(label, loss error, whole-gradient error, worst tensors)]."""
    rows = [("per-tensor scale", *run(name, (1, 1, 1), (0, 1, 1), None, gain))]
    for e in exps:
        rows.append((f"one scale per call, E = {e}", *run(name, (1, 1, 1), (0, 1, 1), e, gain)))
    return rows


if __name__ == "__main__":
    torch.set_num_threads(8)
    args = sys.argv[1:]
    which = args[0] if args and not args[0].startswith("--") else "small"
    name = {"small": "denoiser_small_training", "default": "denoiser_default_training"}[which]
    if "--exp" in args:
        i = args.index("--exp") + 1
        exps = []
        while i < len(args) and not args[i].startswith("--"):
            exps.append(int(args[i])); i += 1
        gain = float(args[args.index("--gain") + 1]) if "--gain" in args else 1.0
        print(f"case {name}, conv_out.weight x {gain}: relative error of the loss / of the whole gradient (L2) / worst tensors")
        for label, dl, dg, worst in per_call_rows(name, exps, gain):
            print(f"{label:30s} loss {dl:.2e}  grad {dg:.2e}  worst {[(round(e, 5), k) for e, k in worst]}")
        sys.exit(0)
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
