"""The two helpers of the reference's src/utils.py that the mirrored models need (init_lstm utils.py:184-196)."""
import ctypes as C
import weakref
from typing import Any, Dict, Tuple

import torch
import torch.nn as nn
from torch import Tensor
from torch.nn.parallel import DistributedDataParallel

from . import _lib

LossAndLogs = Tuple[Tensor, Dict[str, Any]]


def init_lstm(model: nn.Module) -> None:
    for name, p in model.named_parameters():
        if "weight_ih" in name:
            nn.init.xavier_uniform_(p.data)
        elif "weight_hh" in name:
            nn.init.orthogonal_(p.data)
        elif "bias_ih" in name:
            p.data.fill_(0)
            n = p.size(0)
            p.data[(n // 4):(n // 2)].fill_(1)  # forget-gate bias
        elif "bias_hh" in name:
            p.data.fill_(0)


class NativeStateMixin:
    """Modules with a native executor check on every call whether a parameter changed (data_ptr, _version) before reusing the
    packed fp16 copies.  Walking state_dict() for that costs ~0.4 ms per call on the 235 tensors of the denoiser; the tensor
    list is therefore cached and dropped whenever `_apply` (to / cuda / float ...) may have replaced tensors.  In-place updates
    (optimizer steps, load_state_dict, p.data.copy_) keep the objects and bump `_version`, which the key sees; code that REPLACES
    a Parameter object or writes through `.data.fill_` must call `refresh_weights()`.

    A subclass names its C entry points by `_NATIVE_PREFIX` (`dmd_denoiser_`, ...) and provides `_native_config(*params)`
    (the create-time config struct) and the `device` its parameters live on."""

    _NATIVE_PREFIX = ""
    _h = _h_key = _wkey = _packed = _ws = None

    def __del__(self):
        try:
            if self._h is not None:
                getattr(_lib.lib(), self._NATIVE_PREFIX + "destroy")(self._h)
        except Exception:
            pass

    def _native_handle(self, *params):
        """The native handle with up-to-date weights: (re)created when the device or the create-time `params` change,
        re-packed when any parameter changed."""
        lib, pre = _lib.lib(), self._NATIVE_PREFIX
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("diamond_b200 runs on CUDA (sm_90a) only; move the model to a cuda device")
        self.require_current_device(dev)
        key = (dev.index,) + params
        if self._h is None or self._h_key != key:
            if self._h is not None:
                getattr(lib, pre + "destroy")(self._h)
                self._h = None
            h = getattr(lib, pre + "create")(C.byref(self._native_config(*params)))
            if not h:
                raise RuntimeError("diamond_b200: " + lib.dmd_last_error().decode())
            self._h, self._h_key, self._wkey, self._packed = h, key, None, None
        tensors = self._state_tensors()
        wkey = tuple((t.data_ptr(), t._version) for t in tensors)
        if wkey != self._wkey:
            n = getattr(lib, pre + "num_tensors")(self._h)
            if n != len(tensors):
                raise RuntimeError(f"native {type(self).__name__} expects {n} tensors, module has {len(tensors)}")
            for t in tensors:
                if t.dtype != torch.float32 or not t.is_contiguous():
                    raise RuntimeError("parameters must be contiguous fp32")
            if self._packed is None:
                self._packed = torch.empty(getattr(lib, pre + "packed_bytes")(self._h), dtype=torch.uint8, device=dev)
            arr = (C.c_void_p * n)(*[t.data_ptr() for t in tensors])
            _lib.check(getattr(lib, pre + "set_weights")(self._h, arr, n, self._packed.data_ptr(), _lib.current_stream()))
            self._wkey = wkey
        # torch.use_deterministic_algorithms selects the native fixed-order reductions; the handle keys its plans on it
        _lib.check(getattr(lib, pre + "set_deterministic")(self._h, int(torch.are_deterministic_algorithms_enabled())))
        return self._h

    def _native(self):
        return self._native_handle()

    def grad_layout(self):
        """(offsets, numels, total) of the flat fp32 gradient buffer the native backward fills (state_dict order)."""
        lib = _lib.lib()
        h = self._native()
        n = getattr(lib, self._NATIVE_PREFIX + "num_tensors")(h)
        offs, nums = (C.c_longlong * n)(), (C.c_longlong * n)()
        total = getattr(lib, self._NATIVE_PREFIX + "grad_layout")(h, offs, nums, n)
        if total < 0:
            raise RuntimeError("diamond_b200: " + lib.dmd_last_error().decode())
        return list(offs), list(nums), int(total)

    def _grad_views_layout(self):
        """(offsets, numels) of every PARAMETER (in `parameters()` order) inside the flat gradient buffer, and its length.
        Static for a module, so it is computed once (walking state_dict() costs ~0.2 ms, and a backward pass may run many nodes)."""
        cached = self.__dict__.get("_gv_layout")
        if cached is None:
            offs, nums, total = self.grad_layout()
            index = {k: i for i, k in enumerate(self.state_dict().keys())}
            names = [k for k, _ in self.named_parameters()]
            cached = self.__dict__["_gv_layout"] = ([offs[index[k]] for k in names], [nums[index[k]] for k in names], total)
        return cached

    def _acquire_ws(self, nbytes: int):
        """A workspace that lives from a native forward to its backward (one per live autograd node), from a pool that is
        reused across optimizer steps."""
        dev = self.device
        pool = self.__dict__.setdefault("_ws_pool", [])
        for i, ws in enumerate(pool):
            if ws.numel() >= nbytes and ws.device == dev:
                return pool.pop(i)
        return torch.empty(nbytes, dtype=torch.uint8, device=dev)

    def _release_ws(self, ws, cap: int) -> None:
        pool = self.__dict__.setdefault("_ws_pool", [])
        if len(pool) < cap:
            pool.append(ws)

    def _state_tensors(self):
        ts = self.__dict__.get("_state_tensor_cache")
        if ts is None:
            ts = list(self.state_dict(keep_vars=True).values())
            self.__dict__["_state_tensor_cache"] = ts
        return ts

    # ------------------------------------------------------------------ gradients of native backward nodes
    # A native backward writes every parameter gradient into one flat fp32 buffer (layout: grad_layout()).  When a backward pass
    # stores gradients into `.grad`, its nodes ADD into one buffer natively and `.grad` becomes views of it when the pass ends,
    # so that a data-parallel step all-reduces the whole model in one collective (allreduce_native_gradients).  `_grad_acc` is
    # the buffer of the running pass, `last_flat_grad` the one of the last pass.
    #
    # Under DistributedDataParallel that callback would come too late: DDP averages what the parameters' AccumulateGrad nodes
    # receive, and its own end-of-pass callback, which runs after ours, overwrites `.grad` with that average.  A node made
    # inside a DDP forward therefore hands autograd views of the pass's buffer instead (once per pass; every other node of
    # the pass still adds natively and returns None).  Each AccumulateGrad node depends on every native node of the pass, so it
    # runs after the last native add and passes the complete sum to DDP's hook once.

    def _under_ddp(self) -> bool:
        """True while a DistributedDataParallel wrapper whose module is this one or contains it runs its forward.  torch sets
        `_active_ddp_module` for the duration of that forward only, so a native autograd Function asks here in its forward
        and keeps the answer on its ctx for the backward.  The containment walk is cached per wrapper."""
        ddp = DistributedDataParallel._active_ddp_module
        if ddp is None:
            return False
        seen = self.__dict__.get("_ddp_wrappers")
        if seen is None:
            seen = self.__dict__["_ddp_wrappers"] = weakref.WeakKeyDictionary()
        inside = seen.get(ddp)
        if inside is None:
            inside = seen[ddp] = any(m is self for m in ddp.module.modules())
        return inside

    def _pass_param_grads(self, node, flat):
        """What a node that wrote or added its parameter gradients into the pass's buffer `flat` returns to autograd: views of
        `flat` for the first node of the pass made inside a DDP forward (`node.under_ddp`), None for every other one."""
        offs, nums, _ = self._grad_views_layout()
        if getattr(node, "under_ddp", False) and self.__dict__.get("_grad_views") is not flat:
            self.__dict__["_grad_views"] = flat
            return [flat[o:o + n].view_as(p) for o, n, p in zip(offs, nums, self.parameters())]
        return [None] * len(offs)

    def _adopt_accumulated_grads(self) -> None:
        """End of a backward pass (autograd engine callback): the flat buffer the nodes accumulated into becomes `.grad` (added to
        an existing `.grad`, like AccumulateGrad) and is remembered as `last_flat_grad` for a one-collective all-reduce.  When a
        node already handed autograd views of it (DDP), AccumulateGrad has stored them and only `last_flat_grad` is set."""
        flat = self.__dict__.pop("_grad_acc", None)
        if flat is None:
            return
        if self.__dict__.pop("_grad_views", None) is not flat:
            offs, nums, _ = self._grad_views_layout()
            for p, o, n in zip(self.parameters(), offs, nums):
                if not p.requires_grad:
                    continue
                g = flat[o:o + n].view_as(p)
                if p.grad is None:
                    p.grad = g
                else:
                    p.grad.add_(g)
        self.last_flat_grad = flat

    def _engine_stores_grads(self, node) -> bool:
        """True when the running backward pass stores the gradient of every trainable parameter into `.grad`
        (`loss.backward()`), False when it hands gradients back to its caller (`torch.autograd.grad(loss, params)`) or skips
        some parameters (`backward(inputs=...)`).  `node` is the native call's autograd node (its `ctx`); its last edges lead to
        the parameters' AccumulateGrad nodes.  Asked once per pass (graph task); a new pass also drops the buffer of a pass that
        died before its end."""
        task = torch._C._current_graph_task_id()
        cached = self.__dict__.get("_grad_task")
        if cached is not None and cached[0] == task:
            return cached[1]
        self.__dict__.pop("_grad_acc", None)
        self.__dict__.pop("_grad_views", None)
        n = len(self._grad_views_layout()[0])
        accs = [f for f, _ in node.next_functions[-n:] if f is not None]
        try:
            stores = all(torch._C._will_engine_execute_node(f) for f in accs)
        except RuntimeError:
            # torch refuses the query for a leaf that torch.autograd.grad captures: that pass returns the gradients instead
            stores = False
        self.__dict__["_grad_task"] = (task, stores)
        return stores

    def _native_param_grads(self, node, run):
        """The parameter gradients a native backward node returns to autograd.  `run(flat, accumulate)` makes the native call
        that writes (accumulate False) or adds (True) every parameter gradient into the flat buffer `flat`.

        Under `loss.backward()` the first node of the pass writes a new buffer and every later node of the pass (the autoregressive
        steps of Denoiser.forward) adds to it; a callback at the end of the pass makes it `.grad`, so no per-tensor
        AccumulateGrad runs inside a pass (under DDP one node returns views of it instead, see `_pass_param_grads`).  Otherwise
        (torch.autograd.grad, backward(inputs=...)) each node returns views of its own buffer, as autograd expects."""
        offs, nums, total = self._grad_views_layout()
        dev = self.device
        if not self._engine_stores_grads(node):
            flat = torch.empty(total, dtype=torch.float32, device=dev)
            run(flat, False)
            self.last_flat_grad = flat
            return [flat[o:o + n].view_as(p) for o, n, p in zip(offs, nums, self.parameters())]
        flat = self.__dict__.get("_grad_acc")
        if flat is not None:
            run(flat, True)
        else:
            # first node of the pass.  The previous pass's buffer is released first: when the `.grad`s were set to None it is
            # free, and the allocator can hand its memory back
            self.__dict__.pop("last_flat_grad", None)
            flat = self.__dict__["_grad_acc"] = torch.empty(total, dtype=torch.float32, device=dev)
            run(flat, False)
            torch.autograd.Variable._execution_engine.queue_callback(self._adopt_accumulated_grads)
        return self._pass_param_grads(node, flat)

    def refresh_weights(self) -> None:
        self.__dict__["_state_tensor_cache"] = None
        self.__dict__["_wkey"] = None

    def _apply(self, fn, recurse=True):
        self.__dict__["_state_tensor_cache"] = None
        return super()._apply(fn, recurse)

    # The native handle (`_h`, a raw pointer owned by __del__), the packed fp16 weights, workspaces and cached layouts belong
    # to ONE module object.  copy.deepcopy (EMA copies) and pickle (multiprocessing) go through __getstate__: the copy starts
    # without native state and builds its own on first use, so two objects never own -- and free -- the same handle.
    _NATIVE_RESET = ("_h", "_h_key", "_wkey", "_packed", "_ws")
    _NATIVE_DROP = ("_state_tensor_cache", "_ws_pool", "_bwd_scratch", "_grad_acc", "_grad_task", "_gv_layout", "last_flat_grad",
                    "_ws_bytes", "_op_key", "_grad_views", "_ddp_wrappers")

    def __getstate__(self):
        state = self.__dict__.copy()
        for k in self._NATIVE_RESET:
            if k in state:
                state[k] = None
        for k in self._NATIVE_DROP:
            state.pop(k, None)
        return state

    @staticmethod
    def require_current_device(dev) -> None:
        """The native layer launches on the CURRENT CUDA device and on its current stream; a model that lives on another device
        would silently run on the wrong GPU.  Fail loudly instead (the reference trainer calls torch.cuda.set_device, trainer.py:52)."""
        import torch

        if dev.index is not None and dev.index != torch.cuda.current_device():
            raise RuntimeError(f"diamond_b200: the module is on {dev} but the current CUDA device is cuda:{torch.cuda.current_device()}; "
                               f"call torch.cuda.set_device({dev.index}) (or wrap the call in torch.cuda.device) first")


# ----------------------------------------------------------------------------------------------- data-parallel plumbing
# SURVEY.md 8 a26.  The reference wraps each agent module in torch DDP (utils.py:105-106, trainer.py:110) and relies on
# autograd hooks to average gradients.  A native executor produces all gradients of a module in one C-ABI call, outside
# autograd, so the averaging is explicit: flat fp32 buckets, one all_reduce per bucket (NCCL over NVLink on GPUs, gloo in
# the CPU tests), same result as DDP (sum over ranks / world size).


def broadcast_if_needed(*args):
    """utils.py:97-102: every rank ends up with rank 0's objects; a no-op without a process group."""
    import torch.distributed as dist

    objects = list(args)
    if dist.is_available() and dist.is_initialized():
        dist.broadcast_object_list(objects, src=0)
    return objects


def allreduce_gradients(params, bucket_bytes: int = 32 << 20, group=None) -> int:
    """Average `.grad` of `params` over the process group in flat buckets of <= bucket_bytes (one collective each; with
    NVSwitch the cost is launch latency, not link count, so buckets are large).  Parameters without a gradient are treated
    as zero on this rank (DDP's find_unused_parameters semantics) so that every rank issues identical collectives.
    Returns the number of all_reduce calls issued (0 without a process group)."""
    import torch
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return 0
    world = dist.get_world_size(group)
    params = [p for p in params if p.requires_grad]
    calls, i = 0, 0
    while i < len(params):
        j, nbytes = i, 0
        while j < len(params) and (j == i or nbytes + params[j].numel() * 4 <= bucket_bytes):
            nbytes += params[j].numel() * 4
            j += 1
        chunk = params[i:j]
        flat = torch.zeros(sum(p.numel() for p in chunk), dtype=torch.float32, device=chunk[0].device)
        off = 0
        for p in chunk:
            if p.grad is not None:
                flat[off:off + p.numel()].copy_(p.grad.reshape(-1))
            off += p.numel()
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat.div_(world)
        off = 0
        for p in chunk:
            g = flat[off:off + p.numel()].view_as(p)
            if p.grad is None:
                p.grad = g.clone()
            else:
                p.grad.copy_(g)
            off += p.numel()
        calls += 1
        i = j
    return calls


def allreduce_native_gradients(inner_module, group=None) -> int:
    """Data-parallel gradient averaging for a model whose backward ran natively (diamond_b200 InnerModel): the native
    backward wrote EVERY parameter gradient into one flat fp32 buffer and autograd adopted views of it as `.grad`, so the whole
    model is averaged by ONE all_reduce on that buffer (NCCL over NVLink / NVSwitch; the reference wraps each model in DDP,
    utils.py:105-106, which buckets the same bytes into several collectives).  Falls back to `allreduce_gradients` (flatten,
    reduce, scatter) when the gradients do not alias the flat buffer (e.g. after gradient accumulation).  Returns the number of
    collectives issued."""
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return 0
    flat = getattr(inner_module, "last_flat_grad", None)
    params = [p for p in inner_module.parameters() if p.requires_grad]
    aliased = flat is not None and all(
        p.grad is not None and flat.data_ptr() <= p.grad.data_ptr() < flat.data_ptr() + flat.numel() * 4 for p in params)
    if not aliased:
        return allreduce_gradients(params, group=group)
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    flat.div_(dist.get_world_size(group))
    return 1
