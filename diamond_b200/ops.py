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
    trs=True: the tap-row-stacked layout of 3x3 kernels (pass trs=True to the conv call as well)."""
    _cuda(w)
    cout, cin, kh, kw = w.shape
    taps = kh * kw
    cout_pad = round_up(cout, 16)
    c0_real = cin if c0_real is None else c0_real
    c0_store = c0_real if c0_store is None else c0_store
    out = torch.empty(taps * cin_pad * cout_pad * (3 if precise else 1), device=w.device, dtype=torch.float16)
    _lib.check(_lib.lib().dmd_pack_conv_weight(w.data_ptr(), out.data_ptr(), cout, cout_pad, cin, cin_pad, taps,
                                              c0_real, c0_store, 3 if trs else int(precise), _lib.current_stream()))
    return out, cout_pad


def gn_stats(x: Tensor, gs: int) -> Tensor:
    """(sum, sumsq) per (image, group) of an NHWC tensor, fp64 [B][C/gs][2]."""
    _cuda(x)
    b, h, w, c = x.shape
    st = torch.zeros(b, c // gs, 2, device=x.device, dtype=torch.float64)
    _lib.check(_lib.lib().dmd_gn_stats(x.data_ptr(), st.data_ptr(), b, h * w, c, gs, _lib.current_stream()))
    return st


def prep_act(src0: Tensor, *, src1: Optional[Tensor] = None, upsample: bool = False, mode: int = 0, silu: bool = False,
             stats0: Optional[Tensor] = None, stats1: Optional[Tensor] = None, gs0: int = 0, gs1: int = 0,
             film: Optional[Tensor] = None, film_off: int = 0, gamma: Optional[Tensor] = None, beta: Optional[Tensor] = None,
             eps: float = 1e-5, also_raw: bool = False, split: bool = False):
    """NHWC fp32 -> PLC16 fp16 operand(s) with the conv-input transform fused.  Returns (n0, n1, r0, r1, H, W); with
    split=True the low fp16 parts of the main operands are returned as extra elements (l0, l1)."""
    _cuda(src0, src1, stats0, stats1, film, gamma, beta)
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
    _lib.check(lib.dmd_prep_act(C.byref(d), _lib.current_stream()))
    if split:
        return n0, n1, r0, r1, h, w, l0, l1
    return n0, n1, r0, r1, h, w


def conv2d_operand(n0: Tensor, n1: Optional[Tensor], c0: int, c1: int, b: int, h: int, w: int, wpk: Tensor, cout: int,
                   cout_pad: int, taps: int = 9, *, bias: Optional[Tensor] = None, stride: int = 1,
                   residual: Optional[Tensor] = None, out_gs: int = 0, out: Optional[Tensor] = None,
                   ostats: Optional[Tensor] = None, debug: int = 0, debug_buf: Optional[Tensor] = None,
                   lo0: Optional[Tensor] = None, lo1: Optional[Tensor] = None, xproj=None, trs: bool = False):
    """wgmma conv on already prepared PLC16 operand(s) (one kernel launch)."""
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
    d.residual, d.out, d.out_stats, d.out_gs, d.debug = _lib.ptr(residual), out.data_ptr(), _lib.ptr(ostats), out_gs, debug
    d.debug_buf = _lib.ptr(debug_buf)
    d.precise, d.src0_lo, d.src1_lo = int(lo0 is not None), _lib.ptr(lo0), _lib.ptr(lo1)
    d.wpk_layout = int(trs)
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
                 residual: Optional[Tensor] = None, out_gs: int = 0, debug: int = 0, debug_buf: Optional[Tensor] = None,
                 precise: bool = False, trs: bool = False) -> Tuple[Tensor, Optional[Tensor]]:
    """The reference's `conv(act(norm(cat(x, skip))))` on NHWC fp32 tensors: one prep launch + one wgmma conv launch.
    precise=True: split-fp16 operands (weights must be packed with precise=True)."""
    res = prep_act(src0, src1=src1, upsample=upsample, mode=prologue, silu=silu, stats0=stats0, stats1=stats1,
                   gs0=gs0, gs1=gs1, film=film, film_off=film_off, gamma=gamma, beta=beta, eps=eps, split=precise)
    n0, n1, _, _, h, w = res[:6]
    lo0, lo1 = (res[6], res[7]) if precise else (None, None)
    c0, c1 = round_up(src0.shape[3], 16), (round_up(src1.shape[3], 16) if src1 is not None else 0)
    if c0 + c1 != cin_pad:
        raise ValueError(f"operand channels {c0}+{c1} do not match the packed weights ({cin_pad})")
    return conv2d_operand(n0, n1, c0, c1, src0.shape[0], h, w, wpk, cout, cout_pad, taps, bias=bias, stride=stride,
                          residual=residual, out_gs=out_gs, debug=debug, debug_buf=debug_buf, lo0=lo0, lo1=lo1, trs=trs)


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
    """wgmma weight gradient from two PLC16 operands (dL/dy with `cg` stored channels, conv input with `ca`)."""
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
    d.inv_scale, d.accumulate, d.partial, d.partial_bytes, d.debug = _lib.ptr(inv_scale), int(accumulate), part.data_ptr(), part.numel(), debug
    _lib.check(lib.dmd_conv2d_wgrad(C.byref(d), _lib.current_stream()))
    return dw
