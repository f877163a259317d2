"""Native optimizer step: `clip_grad_norm_` and `AdamW` on the sm_90a kernels of csrc/optim_kernels.cuh (C ABI
`dmd_grad_norm_clip` / `dmd_adamw_step`), drop-in for the reference's `torch.nn.utils.clip_grad_norm_` (src/trainer.py:374)
and the `torch.optim.AdamW` that `utils.configure_opt` builds (src/utils.py:164).  Each is a fixed number of launches for the
whole parameter list (norm + reduction + scale, then one AdamW launch) instead of torch's per-tensor-list kernels.

The arithmetic is torch 2.11's: `AdamW` follows `_single_tensor_adam` operation for operation (fp32, the same roundings), and
`state_dict()` / `load_state_dict()` use torch's format, so a checkpoint moves either way between this class and
`torch.optim.AdamW`.  The norm is accumulated in fp64 (torch: fp32 norms of per-tensor norms), so the clip coefficient can
differ from torch's in its last bits."""
import ctypes as C
from typing import Dict, Iterable, Tuple, Union

import torch
from torch import Tensor
from torch.optim import Optimizer

from . import _lib

_UNSUPPORTED = ("amsgrad", "maximize", "capturable", "differentiable")


def _check_tensor(t: Tensor, what: str) -> None:
    if not isinstance(t, Tensor):
        raise TypeError(f"diamond_b200.optim: {what} must be a torch.Tensor, got {type(t).__name__}")
    if t.device.type != "cuda":
        raise ValueError(f"diamond_b200.optim: {what} is on {t.device}; the native optimizer runs on CUDA only")
    if t.dtype != torch.float32:
        raise ValueError(f"diamond_b200.optim: {what} is {t.dtype}; the native optimizer takes fp32 only")
    if t.layout != torch.strided or not t.is_contiguous():
        raise ValueError(f"diamond_b200.optim: {what} must be a contiguous dense tensor")


def _table(entries) -> "C.Array":
    """A dmd_optim_tensor array from (param, grad, exp_avg, exp_avg_sq, numel, weight_decay) tuples of pointers / numbers."""
    arr = (_lib.OptimTensor * len(entries))()
    for e, (p, g, m, v, n, wd) in zip(arr, entries):
        e.param, e.grad, e.exp_avg, e.exp_avg_sq, e.numel, e.weight_decay = p, g, m, v, n, wd
    return arr


_clip_cache: Dict[tuple, tuple] = {}


def clip_grad_norm_(parameters: Union[Tensor, Iterable[Tensor]], max_norm: float, norm_type: float = 2.0,
                    error_if_nonfinite: bool = False, foreach=None) -> Tensor:
    """torch.nn.utils.clip_grad_norm_ for the 2-norm: returns the total norm of all gradients (a 0-d fp32 tensor on their
    device, no host synchronisation) and multiplies every gradient by min(1, max_norm / (total_norm + 1e-6)) in place."""
    if float(norm_type) != 2.0:
        raise ValueError(f"diamond_b200.optim.clip_grad_norm_: norm_type {norm_type} is not supported (only the 2-norm)")
    if foreach is not None:
        raise ValueError("diamond_b200.optim.clip_grad_norm_: foreach selects torch's implementation; leave it None")
    if isinstance(parameters, Tensor):
        parameters = [parameters]
    grads = [p.grad for p in parameters]
    grads = [g for g in grads if g is not None]
    if not grads:
        return torch.tensor(0.0)
    # The launch table of a gradient list is kept by (pointer, numel): a list seen before was checked then.  (Norm and scale
    # are order-free, so a later view of the same block in another layout would be clipped correctly too.)
    key = tuple((g.data_ptr(), g.numel()) for g in grads)
    hit = _clip_cache.get(key)
    lib = _lib.lib()
    dev = grads[0].device
    if hit is None:
        for g in grads:
            _check_tensor(g, "a gradient")
            if g.device != dev:
                raise ValueError(f"diamond_b200.optim.clip_grad_norm_: gradients on {dev} and {g.device}; one device per call")
        arr = _table([(None, g.data_ptr(), None, None, g.numel(), 0.0) for g in grads])
        nbytes = lib.dmd_grad_norm_partial_bytes(arr, len(grads))
        if nbytes == 0:
            raise RuntimeError("diamond_b200: " + lib.dmd_last_error().decode())
        if len(_clip_cache) >= 8:
            _clip_cache.clear()
        hit = _clip_cache[key] = (arr, nbytes)
    arr, nbytes = hit
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        buf = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device=dev)   # [total_norm, coefficient] (fp32) + partials
        out, partial = buf[:1].view(torch.float32), buf[1:]
        if error_if_nonfinite:
            _lib.check(lib.dmd_grad_norm_clip(arr, len(grads), float(max_norm), 0, out.data_ptr(), partial.data_ptr(), nbytes, stream))
            if not bool(torch.isfinite(out[0])):
                raise RuntimeError("The total norm of order 2.0 for gradients from `parameters` is non-finite, so it cannot be "
                                   "clipped. To disable this error and scale the gradients by the non-finite norm anyway, set "
                                   "`error_if_nonfinite=False`")
        _lib.check(lib.dmd_grad_norm_clip(arr, len(grads), float(max_norm), 1, out.data_ptr(), partial.data_ptr(), nbytes, stream))
    torch.autograd.graph.increment_version(grads)
    return out[0]


class AdamW(Optimizer):
    """torch.optim.AdamW (torch 2.11 arithmetic, decoupled weight decay) as one kernel launch per step for all parameters.

    Takes the parameter groups `utils.configure_opt` builds (and any other list of CUDA fp32 contiguous parameters on one
    device).  `exp_avg` / `exp_avg_sq` of all parameters live in one flat buffer each; `self.state[p]` holds views of them
    and a CPU float32 `step`, torch's format.  Parameters whose `.grad` is None are skipped.  After a step the parameters'
    autograd version counters are bumped, so modules that cache derived weights (the native models' packed fp16 copies,
    `utils.NativeStateMixin`) re-pack them before their next forward."""

    def __init__(self, params, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 1e-2, amsgrad: bool = False, *, maximize: bool = False, foreach=None,
                 capturable: bool = False, differentiable: bool = False, fused=None) -> None:
        for name, val in (("amsgrad", amsgrad), ("maximize", maximize), ("capturable", capturable), ("differentiable", differentiable)):
            if val:
                raise ValueError(f"diamond_b200.optim.AdamW does not support {name}=True")
        for name, val in (("foreach", foreach), ("fused", fused)):
            if val is not None:
                raise ValueError(f"diamond_b200.optim.AdamW: {name} selects torch's implementation; leave it None")
        self._check_hyper(lr, betas, eps, weight_decay)
        self._flat = None            # (exp_avg flat, exp_avg_sq flat, {param: offset}) once the first step (or a load) needs it
        self._plan = None            # (key, params, step tensors, table entries) of the last step
        self._calls = None           # [(ctypes table, n, lr, beta1, beta2, eps, parameter indices)]
        self._device = None
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False, foreach=None,
                        capturable=False, differentiable=False, fused=None, decoupled_weight_decay=True)
        super().__init__(params, defaults)

    @staticmethod
    def _check_hyper(lr, betas, eps, weight_decay) -> None:
        for name, val in (("lr", lr), ("beta1", betas[0]), ("beta2", betas[1]), ("eps", eps), ("weight_decay", weight_decay)):
            if isinstance(val, Tensor):
                raise ValueError(f"diamond_b200.optim.AdamW: {name} must be a Python number, not a Tensor")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")

    def add_param_group(self, param_group: dict) -> None:
        super().add_param_group(param_group)
        group = self.param_groups[-1]
        self._check_hyper(group["lr"], group["betas"], group["eps"], group["weight_decay"])
        for p in group["params"]:
            _check_tensor(p, "a parameter")
            if self._device is None:
                self._device = p.device
            elif p.device != self._device:
                raise ValueError(f"diamond_b200.optim.AdamW: parameters on {self._device} and {p.device}; one device per optimizer")
        self._flat = None
        self._plan = None

    def load_state_dict(self, state_dict) -> None:
        super().load_state_dict(state_dict)
        self._flat = None      # the loaded moments are separate tensors: move them into the flat buffers
        self._flatten()

    def _flatten(self) -> None:
        """One exp_avg and one exp_avg_sq buffer for all parameters (each slot 16-byte aligned); existing state is moved in."""
        params = [p for g in self.param_groups for p in g["params"]]
        if not params:
            return
        offs, off = {}, 0
        for p in params:
            offs[p] = off
            off += (p.numel() + 3) & ~3
        m = torch.zeros(max(off, 4), dtype=torch.float32, device=self._device)
        v = torch.zeros_like(m)
        for p in params:
            st = self.state.get(p)
            if st and "exp_avg" in st:
                o, n = offs[p], p.numel()
                m[o:o + n].copy_(st["exp_avg"].reshape(-1))
                v[o:o + n].copy_(st["exp_avg_sq"].reshape(-1))
                st["exp_avg"], st["exp_avg_sq"] = m[o:o + n].view_as(p), v[o:o + n].view_as(p)
        self._flat = (m, v, offs)
        self._plan = None

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if self._flat is None:
            self._flatten()
            if self._flat is None:
                return loss
        flat_m, flat_v, _ = self._flat
        # What the launch tables depend on, read every step: gradient pointers (-1: not contiguous), parameter pointers and
        # the groups' settings.  Anything else -- a new gradient buffer after zero_grad(set_to_none=True) or gradient
        # accumulation, a moved parameter, a changed group -- rebuilds them.
        allp = [p for g in self.param_groups for p in g["params"]]
        grads = [p.grad for p in allp]
        key = (tuple(None if g is None else (g.data_ptr() if g.is_contiguous() else -1) for g in grads),
               tuple(p.data_ptr() for p in allp),
               tuple((g["lr"], tuple(g["betas"]), g["eps"], g["weight_decay"]) + tuple(bool(g.get(f)) for f in _UNSUPPORTED)
                     for g in self.param_groups))
        plan = self._plan
        if plan is None or plan[0] != key:
            plan = self._plan = (key,) + self._collect()
            self._calls = None
        _, params, steps, entries = plan
        if not params:
            return loss
        torch._foreach_add_(steps, 1.0)
        vals = torch.stack(steps).tolist()
        calls = self._calls
        if calls is None or any(len({vals[i] for i in idx}) != 1 for *_, idx in calls):
            calls = self._calls = self._build_calls(entries, vals)
        lib = _lib.lib()
        with torch.cuda.device(self._device):
            stream = torch.cuda.current_stream(self._device).cuda_stream
            for arr, n, lr, b1, b2, eps, idx in calls:
                _lib.check(lib.dmd_adamw_step(arr, n, lr, b1, b2, eps, vals[idx[0]], stream))
        torch.autograd.graph.increment_version(params)
        torch.autograd.graph.increment_version([flat_m, flat_v])
        return loss

    def _collect(self):
        """(params, step tensors, table entries) of the parameters that have a gradient, their state created on first use."""
        flat_m, flat_v, offs = self._flat
        params, steps, entries = [], [], []
        for group in self.param_groups:
            for flag in _UNSUPPORTED:
                if group.get(flag):
                    raise ValueError(f"diamond_b200.optim.AdamW does not support {flag}=True")
            hyper = (float(group["lr"]), float(group["betas"][0]), float(group["betas"][1]), float(group["eps"]))
            wd = float(group["weight_decay"])
            for p in group["params"]:
                g = p.grad
                if g is None:
                    continue
                if g.is_sparse or not g.is_contiguous():
                    raise ValueError("diamond_b200.optim.AdamW: gradients must be contiguous dense tensors")
                st = self.state[p]
                if len(st) == 0:
                    o, n = offs[p], p.numel()
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = flat_m[o:o + n].view_as(p)
                    st["exp_avg_sq"] = flat_v[o:o + n].view_as(p)
                params.append(p)
                steps.append(st["step"])
                entries.append((hyper, (p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(),
                                        p.numel(), wd)))
        return params, steps, entries

    @staticmethod
    def _build_calls(entries, vals):
        """One dmd_adamw_step call per distinct (lr, betas, eps, step count): normally one for the whole model.  Each call
        keeps the indices of its parameters, whose step counts then advance together."""
        calls: Dict[tuple, Tuple[list, list]] = {}
        for i, ((hyper, e), s) in enumerate(zip(entries, vals)):
            es, idx = calls.setdefault(hyper + (s,), ([], []))
            es.append(e)
            idx.append(i)
        return [(_table(es), len(es)) + k[:4] + (idx,) for k, (es, idx) in calls.items()]
