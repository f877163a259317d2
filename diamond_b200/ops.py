"""Per-op Python wrappers over the C ABI (NHWC fp32 tensors on a CUDA device).  Thin: they only marshal pointers."""
import ctypes as C
from typing import Optional, Tuple

import torch
from torch import Tensor

from . import _lib


def _cuda(*ts):
    for t in ts:
        if t is not None and not (t.is_cuda and t.is_contiguous()):
            raise RuntimeError("diamond_b200 ops need contiguous CUDA tensors (no CPU fallback)")


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def nchw_to_nhwc(x: Tensor, cpad: Optional[int] = None) -> Tensor:
    _cuda(x)
    b, c, h, w = x.shape
    cp = cpad or c
    out = torch.empty(b, h, w, cp, device=x.device, dtype=torch.float32)
    _lib.check(_lib.lib().dmd_nchw_to_nhwc(x.data_ptr(), out.data_ptr(), b, c, cp, h * w, _lib.current_stream()))
    return out


def nhwc_to_nchw(x: Tensor, c: Optional[int] = None) -> Tensor:
    _cuda(x)
    b, h, w, cp = x.shape
    c = c or cp
    out = torch.empty(b, c, h, w, device=x.device, dtype=torch.float32)
    _lib.check(_lib.lib().dmd_nhwc_to_nchw(x.data_ptr(), out.data_ptr(), b, c, cp, h * w, _lib.current_stream()))
    return out


def pack_conv_weight(w: Tensor, cin_pad: int, c0_real: Optional[int] = None, c0_store: Optional[int] = None,
                     precise: bool = False, trs: bool = False) -> Tuple[Tensor, int]:
    """torch weight [Cout][Cin][k][k] -> fp16 operand [taps][cin_pad/8][CoutPad][8]; returns (packed, CoutPad).
    trs: see _reject_removed."""
    _reject_removed(trs=trs)
    _cuda(w)
    cout, cin, kh, kw = w.shape
    taps = kh * kw
    cout_pad = round_up(cout, 16)
    c0_real = cin if c0_real is None else c0_real
    c0_store = c0_real if c0_store is None else c0_store
    out = torch.empty(taps * cin_pad * cout_pad * (3 if precise else 1), device=w.device, dtype=torch.float16)
    _lib.check(_lib.lib().dmd_pack_conv_weight(w.data_ptr(), out.data_ptr(), cout, cout_pad, cin, cin_pad, taps,
                                              c0_real, c0_store, int(precise), _lib.current_stream()))
    return out, cout_pad


def _reject_removed(trs: bool = False, debug: int = 0) -> None:
    """`trs` (the tap-row-stacked weight layout) and `debug` (kernel debug switches) name options the kernels no longer
    have.  Callers such as bench.py still pass their defaults, which are accepted; anything else raises."""
    if trs:
        raise ValueError("trs=True: only the tap-major weight layout is supported")
    if debug:
        raise ValueError(f"debug={debug}: the kernels have no debug switches")


def gn_stats(x: Tensor, gs: int, *, out: Optional[Tensor] = None, det: bool = False) -> Tensor:
    """(sum, sumsq) per (image, group) of an NHWC tensor, fp64 [B][C/gs][2], added to `out` (default: zeros); det: the
    fixed-order sums of deterministic mode."""
    _cuda(x, out)
    b, h, w, c = x.shape
    st = torch.zeros(b, c // gs, 2, device=x.device, dtype=torch.float64) if out is None else out
    fn = _lib.lib().dmd_gn_stats_det if det else _lib.lib().dmd_gn_stats
    _lib.check(fn(x.data_ptr(), st.data_ptr(), b, h * w, c, gs, _lib.current_stream()))
    return st


def prep_act(src0: Tensor, *, src1: Optional[Tensor] = None, upsample: bool = False, mode: int = 0, silu: bool = False,
             stats0: Optional[Tensor] = None, stats1: Optional[Tensor] = None, gs0: int = 0, gs1: int = 0,
             film: Optional[Tensor] = None, film_off: int = 0, gamma: Optional[Tensor] = None, beta: Optional[Tensor] = None,
             eps: float = 1e-5, also_raw: bool = False, split: bool = False, raw_split: bool = False):
    """NHWC fp32 -> PLC16 fp16 operand(s) with the conv-input transform fused.  Returns (n0, n1, r0, r1, H, W); with
    split=True the low fp16 parts of the main operands are returned as extra elements (l0, l1).  raw_split=True (needs
    also_raw) also writes the low parts of the raw operands, the split-fp16 operand of a fused skip projection, and returns
    (n0, n1, r0, r1, H, W, l0, l1, rl0, rl1) with l0 = l1 = None unless split."""
    _cuda(src0, src1, stats0, stats1, film, gamma, beta)
    if raw_split and not also_raw:
        raise ValueError("raw_split needs also_raw")
    lib = _lib.lib()
    b, hs, ws, c0 = src0.shape
    h, w = (2 * hs, 2 * ws) if upsample else (hs, ws)
    c1 = src1.shape[3] if src1 is not None else 0

    def buf(c):
        return torch.empty(lib.dmd_plc16_bytes(b, h, w, c), dtype=torch.uint8, device=src0.device)

    n0, n1 = buf(c0), (buf(c1) if c1 else None)
    r0, r1 = (buf(c0) if also_raw else None), (buf(c1) if (also_raw and c1) else None)
    d = _lib.PrepDesc()
    d.src0, d.src1, d.C0, d.C1 = src0.data_ptr(), _lib.ptr(src1), c0, c1
    d.B, d.Hs, d.Ws, d.upsample, d.mode, d.silu = b, hs, ws, int(upsample), mode, int(silu)
    d.stats0, d.stats1, d.gs0, d.gs1 = _lib.ptr(stats0), _lib.ptr(stats1), gs0, gs1
    d.film, d.film_stride, d.film_off = _lib.ptr(film), (film.shape[1] if film is not None else 0), film_off
    d.gamma, d.beta, d.eps = _lib.ptr(gamma), _lib.ptr(beta), eps
    d.dst0, d.dst1, d.dst_raw0, d.dst_raw1 = n0.data_ptr(), _lib.ptr(n1), _lib.ptr(r0), _lib.ptr(r1)
    l0, l1 = (buf(c0) if split else None), (buf(c1) if (split and c1) else None)
    d.dst_lo0, d.dst_lo1 = _lib.ptr(l0), _lib.ptr(l1)
    rl0, rl1 = (buf(c0) if raw_split else None), (buf(c1) if (raw_split and c1) else None)
    d.dst_raw_lo0, d.dst_raw_lo1 = _lib.ptr(rl0), _lib.ptr(rl1)
    _lib.check(lib.dmd_prep_act(C.byref(d), _lib.current_stream()))
    if raw_split:
        return n0, n1, r0, r1, h, w, l0, l1, rl0, rl1
    if split:
        return n0, n1, r0, r1, h, w, l0, l1
    return n0, n1, r0, r1, h, w


def conv2d_operand(n0: Tensor, n1: Optional[Tensor], c0: int, c1: int, b: int, h: int, w: int, wpk: Tensor, cout: int,
                   cout_pad: int, taps: int = 9, *, bias: Optional[Tensor] = None, stride: int = 1,
                   residual: Optional[Tensor] = None, out_gs: int = 0, out: Optional[Tensor] = None,
                   ostats: Optional[Tensor] = None, lo0: Optional[Tensor] = None, lo1: Optional[Tensor] = None,
                   xproj=None, trs: bool = False):
    """wgmma conv on already prepared PLC16 operand(s) (one kernel launch).  trs: see _reject_removed."""
    _reject_removed(trs=trs)
    _cuda(n0, n1, wpk, bias, residual)
    ho, wo = h // stride, w // stride
    if out is None:
        out = torch.empty(b, ho, wo, cout, device=n0.device, dtype=torch.float32)
    if ostats is None and out_gs:
        ostats = torch.zeros(b, cout // out_gs, 2, device=n0.device, dtype=torch.float64)
    d = _lib.ConvDesc()
    d.src0, d.src1, d.C0, d.C1 = n0.data_ptr(), _lib.ptr(n1), c0, c1
    d.B, d.H, d.W, d.taps, d.stride = b, h, w, taps, stride
    d.wpk, d.bias, d.Cout, d.CoutPad = wpk.data_ptr(), _lib.ptr(bias), cout, cout_pad
    d.residual, d.out, d.out_stats, d.out_gs = _lib.ptr(residual), out.data_ptr(), _lib.ptr(ostats), out_gs
    d.precise, d.src0_lo, d.src1_lo = int(lo0 is not None), _lib.ptr(lo0), _lib.ptr(lo1)
    if xproj is not None:  # fused split-fp16 1x1 projection: (hi0, hi1, lo0, lo1, C0, C1, wpk_x, bias_x)
        xh0, xh1, xl0, xl1, xc0, xc1, wpk_x, bias_x = xproj
        d.xsrc0, d.xsrc1, d.xsrc0_lo, d.xsrc1_lo = xh0.data_ptr(), _lib.ptr(xh1), xl0.data_ptr(), _lib.ptr(xl1)
        d.xC0, d.xC1, d.wpk_x, d.bias_x = xc0, xc1, wpk_x.data_ptr(), _lib.ptr(bias_x)
    _lib.check(_lib.lib().dmd_conv2d_fprop(C.byref(d), _lib.current_stream()))
    return out, ostats


def conv2d_fprop(src0: Tensor, wpk: Tensor, cout: int, cout_pad: int, cin_pad: int, taps: int = 9, *,
                 src1: Optional[Tensor] = None, bias: Optional[Tensor] = None, upsample: bool = False, stride: int = 1,
                 prologue: int = 0, silu: bool = False, stats0: Optional[Tensor] = None, stats1: Optional[Tensor] = None,
                 gs0: int = 0, gs1: int = 0, film: Optional[Tensor] = None, film_off: int = 0,
                 gamma: Optional[Tensor] = None, beta: Optional[Tensor] = None, eps: float = 1e-5,
                 residual: Optional[Tensor] = None, out_gs: int = 0, debug: int = 0,
                 precise: bool = False, trs: bool = False) -> Tuple[Tensor, Optional[Tensor]]:
    """The reference's `conv(act(norm(cat(x, skip))))` on NHWC fp32 tensors: one prep launch + one wgmma conv launch.
    precise=True: split-fp16 operands (weights must be packed with precise=True).  debug, trs: see _reject_removed."""
    _reject_removed(trs=trs, debug=debug)
    res = prep_act(src0, src1=src1, upsample=upsample, mode=prologue, silu=silu, stats0=stats0, stats1=stats1,
                   gs0=gs0, gs1=gs1, film=film, film_off=film_off, gamma=gamma, beta=beta, eps=eps, split=precise)
    n0, n1, _, _, h, w = res[:6]
    lo0, lo1 = (res[6], res[7]) if precise else (None, None)
    c0, c1 = round_up(src0.shape[3], 16), (round_up(src1.shape[3], 16) if src1 is not None else 0)
    if c0 + c1 != cin_pad:
        raise ValueError(f"operand channels {c0}+{c1} do not match the packed weights ({cin_pad})")
    return conv2d_operand(n0, n1, c0, c1, src0.shape[0], h, w, wpk, cout, cout_pad, taps, bias=bias, stride=stride,
                          residual=residual, out_gs=out_gs, lo0=lo0, lo1=lo1)


def attn_fwd(x: Tensor, stats_in: Tensor, gamma: Tensor, beta: Tensor, wqkv: Tensor, bqkv: Tensor, wout: Tensor,
             bout: Tensor, gs: int, eps: float = 1e-5, want_stats: bool = True) -> Tuple[Tensor, Optional[Tensor]]:
    _cuda(x, stats_in, gamma, beta, wqkv, bqkv, wout, bout)
    b, h, w, c = x.shape
    out = torch.empty_like(x)
    ostats = torch.zeros(b, c // gs, 2, device=x.device, dtype=torch.float64) if want_stats else None
    _lib.check(_lib.lib().dmd_attn_fwd(x.data_ptr(), stats_in.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                       wqkv.data_ptr(), bqkv.data_ptr(), wout.data_ptr(), bout.data_ptr(), out.data_ptr(),
                                       _lib.ptr(ostats), b, h * w, c, gs, eps, _lib.current_stream()))
    return out, ostats


# ------------------------------------------------------------------------------------------------ forward CUDA-core kernels
# One wrapper per C entry point; the launch geometry is the library's (the launchers the executors use).

def linear(x: Tensor, w: Tensor, bias: Optional[Tensor] = None, *, out: Optional[Tensor] = None, silu: bool = False,
           accumulate: bool = False, hw_perm: int = 0) -> Tensor:
    """out [B][F] (+)= silu?(x W^T + bias) for x [B][K] (or NHWC [B][H][W][C] read in NCHW-flatten order with hw_perm = H*W),
    W [F][K]; accumulate adds to `out` before the SiLU."""
    _cuda(x, w, bias, out)
    b, k, f = x.shape[0], x[0].numel(), w.shape[0]
    if out is None:
        if accumulate:
            raise ValueError("accumulate needs out")
        out = torch.empty(b, f, device=x.device, dtype=torch.float32)
    _lib.check(_lib.lib().dmd_linear(x.data_ptr(), w.data_ptr(), _lib.ptr(bias), out.data_ptr(), b, k, f, int(silu), int(accumulate),
                                     hw_perm, _lib.current_stream()))
    return out


def maxpool2_stats(x: Tensor, y: Tensor, stats: Optional[Tensor] = None, gs: int = 0) -> Tensor:
    """MaxPool2d(2) of NHWC x [B][H][W][C] into y [B][H/2][W/2][C]; with stats [B][C/gs][2] (float64), adds y's GroupNorm
    (sum, sumsq) to it."""
    _cuda(x, y, stats)
    b, h, w, c = x.shape
    _lib.check(_lib.lib().dmd_maxpool2_stats(x.data_ptr(), y.data_ptr(), _lib.ptr(stats), b, h, w, c, gs, _lib.current_stream()))
    return y


def lstm_gates(gates: Tensor, c_in: Tensor, h_out: Tensor, c_out: Tensor) -> Tuple[Tensor, Tensor]:
    """LSTMCell pointwise part from the gate pre-activations [B][4H] (order i, f, g, o) into h_out, c_out [B][H] (c_out may be
    c_in)."""
    _cuda(gates, c_in, h_out, c_out)
    b, hd = c_in.shape
    _lib.check(_lib.lib().dmd_lstm_gates(gates.data_ptr(), c_in.data_ptr(), h_out.data_ptr(), c_out.data_ptr(), b, hd, _lib.current_stream()))
    return h_out, c_out


def resize_nhwc(x: Tensor, out: Tensor, stats: Optional[Tensor] = None, gs: int = 0) -> Tensor:
    """Zero-pad / crop NHWC x [B][H][W][C] at the bottom / right into out [B][Hd][Wd][C]; with stats [B][C/gs][2] (float64),
    adds out's GroupNorm (sum, sumsq) to it."""
    _cuda(x, out, stats)
    b, h, w, c = x.shape
    _lib.check(_lib.lib().dmd_resize_nhwc(x.data_ptr(), out.data_ptr(), b, h, w, out.shape[1], out.shape[2], c, _lib.ptr(stats), gs,
                                          _lib.current_stream()))
    return out


def pack_conv_weight_T(w: Tensor, ci_off: int = 0, cin_k: Optional[int] = None) -> Tuple[Tensor, int, int]:
    """Weights of the dgrad conv (= fprop on dL/dy with transposed, tap-flipped weights) for the input channels
    [ci_off, ci_off + cin_k) of a torch weight [Cout][Cin][k][k]; returns (packed, CinP = round16(Cout), CoutP = round16(cin_k))."""
    _cuda(w)
    cout, cin, kh, kw = w.shape
    cin_k = cin - ci_off if cin_k is None else cin_k
    cin_p, cout_p = round_up(cout, 16), round_up(cin_k, 16)
    out = torch.empty(kh * kw * cin_p * cout_p, device=w.device, dtype=torch.float16)
    _lib.check(_lib.lib().dmd_pack_conv_weight_dgrad(w.data_ptr(), out.data_ptr(), cout, cin, ci_off, cin_k, kh * kw, _lib.current_stream()))
    return out, cin_p, cout_p


_partial = {}


def conv2d_wgrad(grad_op: Tensor, cg: int, act_op: Tensor, ca: int, b: int, h: int, w: int, cout: int, cin: int, taps: int = 9, *,
                 dw: Optional[Tensor] = None, cin_tot: Optional[int] = None, ci_off: int = 0, inv_scale: Optional[Tensor] = None,
                 accumulate: bool = False, debug: int = 0) -> Tensor:
    """wgmma weight gradient from two PLC16 operands (dL/dy with `cg` stored channels, conv input with `ca`).  debug: see
    _reject_removed."""
    _reject_removed(debug=debug)
    _cuda(grad_op, act_op)
    lib = _lib.lib()
    cin_tot = cin if cin_tot is None else cin_tot
    if dw is None:
        dw = torch.zeros(cout, cin_tot, taps, device=grad_op.device, dtype=torch.float32)
    key = grad_op.device.index
    if key not in _partial:
        _partial[key] = torch.empty(lib.dmd_wgrad_partial_bytes(), dtype=torch.uint8, device=grad_op.device)
    part = _partial[key]
    d = _lib.WgradDesc()
    d.grad, d.act, d.Cg, d.Ca, d.B, d.H, d.W, d.taps = grad_op.data_ptr(), act_op.data_ptr(), cg, ca, b, h, w, taps
    d.dW, d.Cout, d.Cin, d.CinTot, d.ci_off = dw.data_ptr(), cout, cin, cin_tot, ci_off
    d.inv_scale, d.accumulate, d.partial, d.partial_bytes = _lib.ptr(inv_scale), int(accumulate), part.data_ptr(), part.numel()
    _lib.check(lib.dmd_conv2d_wgrad(C.byref(d), _lib.current_stream()))
    return dw


class ConvLayer:
    """One nn.Conv2d as the executors build it (dmd_conv_layer_create): its K-split chunks, split-fp16 passes, backward-data
    chunks and weight-gradient blocks are the executors' own.  The *_plan methods record those launches without a device."""

    _PLAN_CAP = 16

    def __init__(self, cout: int, cin_real: int, taps: int, c0_real: int, c0_store: int, c1: int = 0, split: bool = False,
                 dgrad: bool = True):
        lib = _lib.lib()
        self.h = lib.dmd_conv_layer_create(cout, cin_real, taps, c0_real, c0_store, c1, int(split), int(dgrad))
        if not self.h:
            raise RuntimeError("diamond_b200: " + lib.dmd_last_error().decode("utf-8", "replace"))
        self._destroy = lib.dmd_conv_layer_destroy
        self.cout, self.cin_real, self.taps, self.c0_real, self.c0_store, self.c1 = cout, cin_real, taps, c0_real, c0_store, c1
        s = _lib.ConvLayerShape()
        _lib.check(lib.dmd_conv_layer_info(self.h, C.byref(s)))
        self.info = {f: (list(getattr(s, f)) if f.endswith("_launches") and f != "fprop_launches" else getattr(s, f))
                     for f, _ in s._fields_}

    def __del__(self):
        if getattr(self, "h", None):
            self._destroy(self.h)
            self.h = None

    def pack(self, w: Tensor) -> Tensor:
        """The layer's packs of the torch weight w [cout][cin_real][k][k] in a new buffer."""
        _cuda(w)
        packed = torch.empty(self.info["packed_bytes"], dtype=torch.uint8, device=w.device)
        _lib.check(_lib.lib().dmd_conv_layer_pack(self.h, w.data_ptr(), packed.data_ptr(), _lib.current_stream()))
        return packed

    def _desc(self, n0, n1, lo0, lo1, b, h, w, stride, bias, residual, out, ostats, out_gs):
        d = _lib.ConvDesc()
        d.src0, d.src1, d.C0, d.C1 = n0, n1, self.c0_store, self.c1
        d.src0_lo, d.src1_lo = lo0, lo1
        d.B, d.H, d.W, d.stride = b, h, w, stride
        d.bias, d.residual, d.out, d.out_stats, d.out_gs = bias, residual, out, ostats, out_gs
        return d

    def fprop(self, packed: Tensor, n0: Tensor, n1: Optional[Tensor], b: int, h: int, w: int, out: Tensor, *,
              lo0: Optional[Tensor] = None, lo1: Optional[Tensor] = None, stride: int = 1, bias: Optional[Tensor] = None,
              residual: Optional[Tensor] = None, ostats: Optional[Tensor] = None, out_gs: int = 0) -> Tensor:
        """out (NHWC [b][h/stride][w/stride][cout]) = conv of the PLC16 operands (+ bias, + residual); ostats += its GroupNorm
        (sum, sumsq) in groups of out_gs channels."""
        _cuda(packed, n0, n1, lo0, lo1, bias, residual, out, ostats)
        d = self._desc(n0.data_ptr(), _lib.ptr(n1), _lib.ptr(lo0), _lib.ptr(lo1), b, h, w, stride, _lib.ptr(bias), _lib.ptr(residual),
                       out.data_ptr(), _lib.ptr(ostats), out_gs)
        _lib.check(_lib.lib().dmd_conv_layer_fprop(self.h, packed.data_ptr(), C.byref(d), _lib.current_stream()))
        return out

    def dgrad(self, packed: Tensor, k: int, gy_op: Tensor, b: int, h: int, w: int, out: Tensor, accumulate: bool = False) -> Tensor:
        """out (NHWC [b][h][w][channels of source k]) (+)= the input gradient of source k from the PLC16 gradient operand at the
        conv input size."""
        _cuda(packed, gy_op, out)
        _lib.check(_lib.lib().dmd_conv_layer_dgrad(self.h, packed.data_ptr(), k, gy_op.data_ptr(), b, h, w, out.data_ptr(),
                                                   int(accumulate), _lib.current_stream()))
        return out

    def wgrad(self, gy_op: Tensor, act_op: Tensor, ca: int, cin: int, ci_off: int, b: int, h: int, w: int, dw: Tensor,
              inv_scale: Optional[Tensor] = None, partial: Optional[Tensor] = None) -> Tensor:
        """dw [cout][cin_real][taps] += inv_scale * the weight gradient of input channels [ci_off, ci_off + cin) (act_op: ca
        stored channels)."""
        _cuda(gy_op, act_op, dw, inv_scale, partial)
        lib = _lib.lib()
        if partial is None:
            partial = torch.empty(lib.dmd_wgrad_partial_bytes(), dtype=torch.uint8, device=dw.device)
        _lib.check(lib.dmd_conv_layer_wgrad(self.h, gy_op.data_ptr(), act_op.data_ptr(), ca, cin, ci_off, b, h, w, partial.data_ptr(),
                                            partial.numel() * partial.element_size(), _lib.ptr(inv_scale), dw.data_ptr(),
                                            _lib.current_stream()))
        return dw

    @staticmethod
    def _launches(buf, n):
        return [{f: (list(getattr(buf[i], f)) if f in ("src", "plane") else getattr(buf[i], f)) for f, _ in _lib.ConvLayerLaunch._fields_}
                for i in range(n.value)]

    def fprop_plan(self, b: int, h: int, w: int, *, stride: int = 1, bias: bool = True, residual: bool = False, stats: bool = False,
                   out_gs: int = 0, lo: Optional[bool] = None) -> list:
        """The forward's launches (dicts of dmd_conv_layer_launch), recorded without a device; lo: pass low operand parts
        (default: when the layer is split-fp16)."""
        lo = bool(self.info["precise"] or self.info["three_pass"]) if lo is None else lo
        d = self._desc(1, 1 if self.c1 else None, 1 if lo else None, 1 if (lo and self.c1) else None, b, h, w, stride,
                       1 if bias else None, 1 if residual else None, 1, 1 if stats else None, out_gs)
        buf, n = (_lib.ConvLayerLaunch * self._PLAN_CAP)(), C.c_int(0)
        _lib.check(_lib.lib().dmd_conv_layer_fprop_plan(self.h, C.byref(d), buf, self._PLAN_CAP, C.byref(n)))
        return self._launches(buf, n)

    def dgrad_plan(self, k: int, b: int, h: int, w: int, accumulate: bool = False) -> list:
        buf, n = (_lib.ConvLayerLaunch * self._PLAN_CAP)(), C.c_int(0)
        _lib.check(_lib.lib().dmd_conv_layer_dgrad_plan(self.h, k, b, h, w, int(accumulate), buf, self._PLAN_CAP, C.byref(n)))
        return self._launches(buf, n)

    def wgrad_plan(self, ca: int, cin: int, ci_off: int, b: int, h: int, w: int) -> list:
        buf, n = (_lib.ConvLayerLaunch * self._PLAN_CAP)(), C.c_int(0)
        _lib.check(_lib.lib().dmd_conv_layer_wgrad_plan(self.h, ca, cin, ci_off, b, h, w, buf, self._PLAN_CAP, C.byref(n)))
        return self._launches(buf, n)


# ------------------------------------------------------------------------------------------------ backward kernels
# One wrapper per C entry point of the CUDA-core backward kernels.  Outputs that the kernels accumulate into are passed in
# by the caller; the launch geometry is the library's (the same launchers the training executors use).

def _inv(inv_scale):
    return _lib.ptr(inv_scale)


def norm_bwd(x: Tensor, gy: Tensor, stats: Tensor, gs: int, gx: Tensor, sum_a: Tensor, sum_b: Tensor, sum_stride: int, *, mode: int,
             act: bool = True, film: Optional[Tensor] = None, film_off: int = 0, film_ctot: int = 0, c_off: int = 0,
             gamma: Optional[Tensor] = None, beta: Optional[Tensor] = None, eps: float = 1e-5, addend: Optional[Tensor] = None,
             accumulate: bool = False, dgamma: Optional[Tensor] = None, dbeta: Optional[Tensor] = None,
             inv_scale: Optional[Tensor] = None, det: bool = False) -> None:
    """(Ada)GroupNorm [+ SiLU] backward of NHWC x [B][H][W][C] as the executors run it: pass 1 adds the per-channel sums to
    sum_a / sum_b (rows of sum_stride floats; they may be views into a larger buffer such as the FiLM gradient), then the
    affine parameter gradients when dgamma / dbeta are given, then pass 2 writes (or adds to) gx.  det: pass 1 as
    deterministic mode runs it."""
    _cuda(x, gy, stats, gx, film, gamma, beta, addend)
    lib = _lib.lib()
    b, c = x.shape[0], x.shape[-1]
    d = _lib.NormBwdDesc()
    d.x, d.gy, d.stats, d.B, d.HW, d.C, d.gs = x.data_ptr(), gy.data_ptr(), stats.data_ptr(), b, x.numel() // (b * c), c, gs
    d.mode, d.act = mode, int(act)
    d.film, d.film_stride, d.film_off, d.film_ctot, d.c_off = _lib.ptr(film), (film.shape[1] if film is not None else 0), film_off, film_ctot, c_off
    d.gamma, d.beta, d.eps = _lib.ptr(gamma), _lib.ptr(beta), eps
    d.sumA, d.sumB, d.sum_stride = sum_a.data_ptr(), sum_b.data_ptr(), sum_stride
    d.gx, d.addend, d.accumulate = gx.data_ptr(), _lib.ptr(addend), int(accumulate)
    st = _lib.current_stream()
    _lib.check((lib.dmd_norm_bwd_det if det else lib.dmd_norm_bwd)(C.byref(d), 1, st))
    if dgamma is not None:
        _lib.check(lib.dmd_norm_affine_grad(C.byref(d), dgamma.data_ptr(), dbeta.data_ptr(), _inv(inv_scale), st))
    _lib.check(lib.dmd_norm_bwd(C.byref(d), 2, st))


def attn_bwd(x: Tensor, stats_in: Tensor, gamma: Tensor, beta: Tensor, wqkv: Tensor, bqkv: Tensor, wout: Tensor, gout: Tensor, gs: int,
             pgrads: Tuple[Tensor, ...], inv_scale: Optional[Tensor] = None, eps: float = 1e-5) -> Tensor:
    """SelfAttention2d backward of NHWC x [B][8][8][C]: returns g_x; ADDS the parameter gradients to
    pgrads = (dgamma, dbeta, dwqkv, dbqkv, dwout, dbout)."""
    _cuda(x, stats_in, gamma, beta, wqkv, bqkv, wout, gout, *pgrads)
    b, h, w, c = x.shape
    gx = torch.empty_like(x)
    _lib.check(_lib.lib().dmd_attn_bwd(x.data_ptr(), stats_in.data_ptr(), gamma.data_ptr(), beta.data_ptr(), wqkv.data_ptr(),
                                       bqkv.data_ptr(), wout.data_ptr(), gout.data_ptr(), gx.data_ptr(), *[t.data_ptr() for t in pgrads],
                                       _inv(inv_scale), b, h * w, c, gs, eps, _lib.current_stream()))
    return gx


def attn_split_bwd(x: Tensor, stats_in: Tensor, gamma: Tensor, beta: Tensor, wqkv: Tensor, bqkv: Tensor, wout: Tensor, gout: Tensor,
                   gs: int, grads: Tensor, goffs, inv_scale: Optional[Tensor] = None, det: bool = False) -> Tensor:
    """The training plans' split SelfAttention2d backward of NHWC x [B][H][W][C] (H*W <= 64, C in {32, 64, 128}): returns g_x;
    ADDS the parameter gradients (gamma, beta, Wqkv, bqkv, Wout, bout) to the flat buffer `grads` at the six float offsets
    `goffs`."""
    _cuda(x, stats_in, gamma, beta, wqkv, bqkv, wout, gout, grads, inv_scale)
    lib = _lib.lib()
    b, h, w, c = x.shape
    gx = torch.empty_like(x)
    ws = torch.empty(lib.dmd_attn_split_bwd_workspace_bytes(b, h * w, c), dtype=torch.uint8, device=x.device)
    offs = (C.c_longlong * 6)(*[int(o) for o in goffs])
    _lib.check(lib.dmd_attn_split_bwd(x.data_ptr(), stats_in.data_ptr(), gamma.data_ptr(), beta.data_ptr(), wqkv.data_ptr(),
                                      bqkv.data_ptr(), wout.data_ptr(), gout.data_ptr(), gx.data_ptr(), grads.data_ptr(), offs,
                                      _inv(inv_scale), b, h * w, c, gs, int(det), ws.data_ptr(), ws.numel(), _lib.current_stream()))
    return gx


def sgemm(a: Tensor, sam: int, sak: int, bm: Tensor, sbk: int, sbn: int, c: Tensor, ldc: int, m: int, n: int, k: int, *,
          alpha: Optional[Tensor] = None, accumulate: bool = False, chunks: int = 0) -> Tensor:
    """c[i*ldc + j] (+)= alpha * sum_k a[i*sam + k*sak] * bm[k*sbk + j*sbn]; chunks > 1: split-K through a partial buffer."""
    _cuda(a, bm, c, alpha)
    lib = _lib.lib()
    nf = lib.dmd_sgemm_partial_floats(m, n, k, chunks)
    part = torch.empty(max(nf, 1), device=c.device, dtype=torch.float32) if nf else None
    _lib.check(lib.dmd_sgemm(a.data_ptr(), sam, sak, bm.data_ptr(), sbk, sbn, c.data_ptr(), ldc, m, n, k, _lib.ptr(alpha),
                             int(accumulate), chunks, _lib.ptr(part), _lib.current_stream()))
    return c


def film_wgrad(dfilm: Tensor, cond: Tensor, grads: Tensor, woff: Tensor, boff: Tensor, inv_scale: Optional[Tensor] = None) -> Tensor:
    """grads[woff[f] + k] += sum_n dfilm[n][f] cond[n][k], grads[boff[f]] += sum_n dfilm[n][f] (times inv_scale)."""
    _cuda(dfilm, cond, grads, woff, boff)
    b, rows = dfilm.shape
    _lib.check(_lib.lib().dmd_film_wgrad(dfilm.data_ptr(), cond.data_ptr(), grads.data_ptr(), woff.data_ptr(), boff.data_ptr(), b, rows,
                                         cond.shape[1], _inv(inv_scale), _lib.current_stream()))
    return grads


def embedding_bwd(de: Tensor, act: Tensor, de_table: Tensor, inv_scale: Optional[Tensor] = None, det: bool = False) -> Tensor:
    """de [B][T*E], act [B][T] int64 -> de_table [num_actions][E] += scattered rows; det: gathered in a fixed order."""
    _cuda(de, act, de_table)
    b, t = act.shape
    fn = _lib.lib().dmd_embedding_bwd_det if det else _lib.lib().dmd_embedding_bwd
    _lib.check(fn(de.data_ptr(), act.data_ptr(), de_table.data_ptr(), b, de.shape[1], t, de_table.shape[0],
               _inv(inv_scale), _lib.current_stream()))
    return de_table


def colsum(x: Tensor, out: Tensor, out2: Optional[Tensor] = None, inv_scale: Optional[Tensor] = None, creal: Optional[int] = None,
           det: bool = False, partial: Optional[Tensor] = None) -> Tensor:
    """out[c] (and out2[c]) += sum over the rows of x [rows][C] for c < creal (default C).  det: the block sums go through
    `partial` (default: a buffer of dmd_colsum_partial_bytes) and are added in block order."""
    _cuda(x, out, out2, partial)
    lib = _lib.lib()
    rows, c = x.shape
    creal = c if creal is None else creal
    if not det:
        _lib.check(lib.dmd_colsum(x.data_ptr(), out.data_ptr(), _lib.ptr(out2), _inv(inv_scale), rows, c, creal, _lib.current_stream()))
        return out
    if partial is None:
        partial = torch.empty(lib.dmd_colsum_partial_bytes(rows, c), dtype=torch.uint8, device=x.device)
    _lib.check(lib.dmd_colsum_det(x.data_ptr(), out.data_ptr(), _lib.ptr(out2), _inv(inv_scale), rows, c, creal, partial.data_ptr(),
                                  partial.numel() * partial.element_size(), _lib.current_stream()))
    return out


def sumpool2(inp: Tensor, out: Tensor, accumulate: bool = False) -> Tensor:
    """out [B][H][W][C] (+)= sum of the 2x2 blocks of inp [B][2H][2W][C]."""
    _cuda(inp, out)
    b, h, w, c = out.shape
    _lib.check(_lib.lib().dmd_sumpool2(inp.data_ptr(), out.data_ptr(), b, h, w, c, int(accumulate), _lib.current_stream()))
    return out


def dsilu_mul(pre: Tensor, dh: Tensor) -> Tensor:
    _cuda(pre, dh)
    out = torch.empty_like(pre)
    _lib.check(_lib.lib().dmd_dsilu_mul(pre.data_ptr(), dh.data_ptr(), out.data_ptr(), pre.numel(), _lib.current_stream()))
    return out


def maxpool2_bwd(y: Tensor, gp: Tensor) -> Tensor:
    """MaxPool2d(2) backward: y NHWC [B][H][W][C] (pre-pool), gp [B][H/2][W/2][C] -> gradient wrt y."""
    _cuda(y, gp)
    b, h, w, c = y.shape
    gy = torch.empty_like(y)
    _lib.check(_lib.lib().dmd_maxpool2_bwd(y.data_ptr(), gp.data_ptr(), gy.data_ptr(), b, h, w, c, _lib.current_stream()))
    return gy


def lstm_cell_bwd(gates: Tensor, c_in: Tensor, g_h: Optional[Tensor], g_c: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    """LSTMCell backward from the gate pre-activations [B][4H]: returns (dgates, gradient wrt c_in)."""
    _cuda(gates, c_in, g_h, g_c)
    b, hd = c_in.shape
    dgates, gc = torch.empty_like(gates), torch.empty_like(c_in)
    _lib.check(_lib.lib().dmd_lstm_cell_bwd(gates.data_ptr(), c_in.data_ptr(), _lib.ptr(g_h), _lib.ptr(g_c), dgates.data_ptr(),
                                            gc.data_ptr(), b, hd, _lib.current_stream()))
    return dgates, gc


def heads_bwd(g_hx: Optional[Tensor], g_logits: Optional[Tensor], g_val: Optional[Tensor], hx_out: Tensor, wa: Tensor, wc: Tensor,
              dba: Tensor, dwc: Tensor, dbc: Tensor) -> Tensor:
    """Actor / critic heads backward: returns g_h; adds the actor bias and critic weight / bias gradients of the given heads."""
    _cuda(g_hx, g_logits, g_val, hx_out, wa, wc, dba, dwc, dbc)
    b, hd = hx_out.shape
    g_h = torch.empty_like(hx_out)
    _lib.check(_lib.lib().dmd_heads_bwd(_lib.ptr(g_hx), _lib.ptr(g_logits), _lib.ptr(g_val), hx_out.data_ptr(), wa.data_ptr(),
                                        wc.data_ptr(), g_h.data_ptr(), dba.data_ptr(), dwc.data_ptr(), dbc.data_ptr(), b, hd,
                                        wa.shape[0], _lib.current_stream()))
    return g_h


def loss_scale(g: Tensor) -> Tensor:
    """The backward loss scale of a gradient tensor: [S, 1/S]."""
    _cuda(g)
    amax = torch.zeros(1, device=g.device, dtype=torch.int32)
    scale = torch.empty(2, device=g.device, dtype=torch.float32)
    _lib.check(_lib.lib().dmd_loss_scale(g.data_ptr(), g.numel(), amax.data_ptr(), scale.data_ptr(), _lib.current_stream()))
    return scale
