"""The native kernels' operand rounding, emulated on the oracle (CPU): conv operands rounded to fp16 with exact accumulation,
the residual-stream layers (conv_in, 1x1 projections) exact as the split-fp16 kernels make them.

- QConv: conv2d whose forward / dgrad / wgrad operands are rounded per layer (oracle/grad_error_budget.py's backward budget).
- grad_errors(): the whole-gradient and per-tensor errors of that rounding against exact autograd, for any loss over a state
  dict (the denoiser, reward / termination and actor-critic training tests bound the native gradients by it).
- fp16_forward(): a context that patches F.conv2d (and optionally F.group_norm) for a forward pass of the oracle, which calls
  both through the module attribute.  Its GroupNorm can move each (image, group) (sum, sumsq) by +-1 fp32 ulp under a seed:
  the spread that a valid regrouping of the conv epilogue's fp32 partial sums produces.
- rew_end_logits(): the reward / termination logits of the golden training batch under that emulation (float64), and
  rew_end_ensemble(), the emulation repeated under several statistics perturbations.
"""
import contextlib
import functools
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

_real_conv2d = F.conv2d
_real_group_norm = F.group_norm


def _h(t):
    """fp16 rounding of t, in t's dtype."""
    return t.half().to(t.dtype)


# the loss-scale scheme: None = a per-tensor scale (max near 2^12); an int E = one scale per backward call, set by conv_out
_SCALE = {"exp": None, "S": None}


def _pow2_scale(m, e):
    """2^(e - k) for m = f 2^k, f in [0.5, 1): loss_scale_kernel's choice, max |S g| in [2^(e-1), 2^e)."""
    return 1.0 if m == 0.0 else 2.0 ** (e - math.frexp(m)[1])


def _scaled_h(g):
    """fp16 rounding of a gradient tensor under the loss scale of _SCALE."""
    s = _SCALE["S"] if _SCALE["exp"] is not None else _pow2_scale(float(g.abs().max()), 12)
    return _h(g * s) / s


class QConv(torch.autograd.Function):
    """conv2d whose forward / dgrad / wgrad operands are rounded per `mode` = (fwd, dgrad, wgrad), each in {0: exact, 1: fp16}."""

    @staticmethod
    def forward(ctx, x, w, b, stride, padding, mode, is_out=False):
        ctx.save_for_backward(x, w)
        ctx.cfg = (stride, padding, mode, b is not None)
        ctx.is_out = is_out
        xq, wq = (_h(x), _h(w)) if mode[0] else (x, w)
        return _real_conv2d(xq, wq, b, stride=stride, padding=padding)

    @staticmethod
    def backward(ctx, gy):
        x, w = ctx.saved_tensors
        stride, padding, mode, has_b = ctx.cfg
        if ctx.is_out and _SCALE["exp"] is not None:   # conv_out: its dL/dy is the gradient of the model output
            _SCALE["S"] = _pow2_scale(float(gy.abs().max()), _SCALE["exp"])
        gd = _scaled_h(gy) if mode[1] else gy
        gx = torch.nn.grad.conv2d_input(x.shape, _h(w) if mode[1] else w, gd, stride=stride, padding=padding)
        gwy = _scaled_h(gy) if mode[2] else gy
        gw = torch.nn.grad.conv2d_weight(_h(x) if mode[2] else x, w.shape, gwy, stride=stride, padding=padding)
        gb = gy.sum(dim=(0, 2, 3)) if has_b else None
        return gx, gw, gb, None, None, None, None


MODE_MAIN, MODE_STREAM = (1, 1, 1), (0, 1, 1)   # the kernels' rounding: fp16 everywhere, but split-fp16 stream layers forward


def grad_errors(loss_fn, sd, stream, out_key=None, exp=None, mode_main=MODE_MAIN, mode_stream=MODE_STREAM):
    """The backward error budget of the kernels' operand rounding at one model's own inputs.

    loss_fn(sd) -> scalar loss, computing every conv through F.conv2d with weights taken from sd; sd: the state dict, its
    leaves with requires_grad set.  stream(name): True for the layers the kernels run split-fp16 in the forward (conv_in /
    conv0, the 1x1 projections and skips).  out_key: the model's single output conv, whose dL/dy fixes one loss scale per
    backward call with max|S dL/dy| in [2^(exp-1), 2^exp) when exp is given (the denoiser, exp = DMD_LOSS_SCALE_EXP); without
    it every gradient operand gets a per-tensor scale.  Gradients are exact autograd at sd's dtype, once as is and once with
    every conv replaced by QConv.  Returns (loss, emulated loss, whole-gradient relative L2 error, {name: relative L2 error},
    {name: exact gradient})."""

    def grads(emulate):
        params = {k: v.detach().clone().requires_grad_(v.requires_grad) for k, v in sd.items()}
        names = {id(v): k for k, v in params.items()}

        def conv2d(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
            assert dilation == 1 and groups == 1
            k = names.get(id(w))
            mode = mode_stream if k is not None and stream(k) else mode_main
            return QConv.apply(x, w, b, stride, padding, mode, k is not None and k == out_key)

        F.conv2d = conv2d if emulate else _real_conv2d
        _SCALE["exp"], _SCALE["S"] = exp, None
        try:
            loss = loss_fn(params)
            loss.backward()
        finally:
            F.conv2d = _real_conv2d
            _SCALE["exp"], _SCALE["S"] = None, None
        return float(loss.detach()), {k: v.grad for k, v in params.items() if v.grad is not None}

    l0, g0 = grads(False)
    l1, g1 = grads(True)
    assert set(g0) == set(g1)
    num = math.sqrt(sum(float((g1[k] - g0[k]).double().pow(2).sum()) for k in g0))
    den = math.sqrt(sum(float(g0[k].double().pow(2).sum()) for k in g0))
    per = {k: float((g1[k] - g0[k]).double().norm() / g0[k].double().norm().clamp_min(1e-30)) for k in g0}
    return l0, l1, num / den, per, g0


def denoiser_stream(sd):
    """grad_errors' stream predicate for InnerModel: conv_in and every 1x1 conv (projections, attention)."""
    return lambda k: k == "conv_in.weight" or (sd[k].dim() == 4 and sd[k].shape[-1] == 1)


def rew_end_stream(sd):
    """The same for RewEndModel: its encoder's conv_in and every 1x1 conv."""
    return lambda k: k == "encoder.conv_in.weight" or (sd[k].dim() == 4 and sd[k].shape[-1] == 1)


def actor_critic_stream(sd):
    """The same for ActorCritic, whose encoder runs every conv split-fp16 in the forward (conv0, the 3x3s, the skips)."""
    return lambda k: sd[k].dim() == 4


def _ulp_step(s, gen):
    """s rounded to fp32, then moved by one fp32 ulp up or down (a random sign per element), back in s's dtype."""
    f = s.float()
    up = torch.randint(0, 2, f.shape, generator=gen).bool()
    return torch.nextafter(f, torch.where(up, torch.full_like(f, math.inf), torch.full_like(f, -math.inf))).to(s.dtype)


@contextlib.contextmanager
def fp16_forward(stream, gn_seed=None, gn_swap_call=None):
    """Patches F.conv2d so that every conv whose weight `stream(w)` rejects takes fp16-rounded operands, and F.group_norm so that
    it normalises from (sum, sumsq) per (image, group), as the prep kernels do.  gn_seed: move every such sum by +-1 fp32 ulp
    (torch.Generator seed).  gn_swap_call: the GroupNorm call (0-based, in order) that reads group 0's statistics of the NEXT
    image (a negative control)."""
    gen = torch.Generator().manual_seed(gn_seed) if gn_seed is not None else None
    calls = [0]

    def conv2d(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
        if not stream(w):
            x, w = _h(x), _h(w)
        return _real_conv2d(x, w, b, stride, padding, dilation, groups)

    def group_norm(x, num_groups, weight=None, bias=None, eps=1e-5):
        n = x.shape[0]
        v = x.reshape(n, num_groups, -1)
        s, ss = v.sum(-1), (v * v).sum(-1)
        if gen is not None:
            s, ss = _ulp_step(s, gen), _ulp_step(ss, gen)
        if calls[0] == gn_swap_call:
            s, ss = s.clone(), ss.clone()
            s[:, 0], ss[:, 0] = s[:, 0].roll(-1, 0), ss[:, 0].roll(-1, 0)
        calls[0] += 1
        cnt = v.shape[-1]
        mean = s / cnt
        var = (ss / cnt - mean * mean).clamp_min(0)
        y = ((v - mean[..., None]) / (var[..., None] + eps).sqrt()).reshape(x.shape)
        shape = (1, -1) + (1,) * (x.dim() - 2)
        if weight is not None:
            y = y * weight.view(shape)
        if bias is not None:
            y = y + bias.view(shape)
        return y

    F.conv2d, F.group_norm = conv2d, group_norm
    try:
        yield
    finally:
        F.conv2d, F.group_norm = _real_conv2d, _real_group_norm


def rew_end_logits(sd=None, gn_seed=None, gn_swap_call=None):
    """Logits (rew [b, T-1, 3], end [b, T-1, 2]) of the golden training batch (tests/golden/rew_end_training.npz) at its
    seeded weights, in float64 under fp16_forward: conv_in and the 1x1 projections exact, the other convs on fp16 operands."""
    from oracle import rew_end_training as RT
    from oracle import torch_oracle as O

    cfg = O.RewEndCfg()
    (obs, act, rew, end, mask, final_obs), _ = RT.load_golden()
    if sd is None:
        sd = O.seeded_state_dict(O.rew_end_shapes(cfg), 778)
    sd = {k: v.double() for k, v in sd.items()}
    stream = lambda w: w.shape[-1] == 1 or w.shape[1] == 2 * cfg.img_channels  # noqa: E731
    with torch.no_grad(), fp16_forward(stream, gn_seed, gn_swap_call):
        out = RT.rew_end_loss(obs.double(), act, rew.double(), end, mask, {k: v.double() for k, v in final_obs.items()}, sd, cfg)
    return out[3], out[4]


ENSEMBLE_SEEDS = tuple(range(1, 9))
LOGITS_MARGIN = 1.5    # bound = margin * the ensemble's worst distance to the reference


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@functools.lru_cache(maxsize=1)
def rew_end_ensemble():
    """(emulation without perturbation, [emulation under each of ENSEMBLE_SEEDS])."""
    return rew_end_logits(), [rew_end_logits(gn_seed=s) for s in ENSEMBLE_SEEDS]


def rew_end_logits_bounds():
    """Per head (rew, end): the relative L2 bound of logits against the reference's fp32 logits, LOGITS_MARGIN times the
    ensemble's worst distance to them, and the ensemble's spread, its worst distance to the unperturbed emulation.  Returns
    ({head: bound}, {head: spread}, the unperturbed emulation's logits (rew, end))."""
    from oracle import rew_end_training as RT

    _, g = RT.load_golden()
    ref = (torch.from_numpy(g["logits_rew"]), torch.from_numpy(g["logits_end"]))
    emu, members = rew_end_ensemble()
    bound, spread = {}, {}
    for k, head in enumerate(("rew", "end")):
        bound[head] = LOGITS_MARGIN * max(_rel(m[k], ref[k]) for m in [emu] + members)
        spread[head] = max(_rel(m[k], emu[k]) for m in members)
    return bound, spread, emu
