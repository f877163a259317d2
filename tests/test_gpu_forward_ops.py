"""The forward CUDA-core kernels (diamond_b200/csrc/aux_kernels.cuh) and the conv-operand prep (conv_tc.cuh), one entry point at a
time, against float64 references of the same op (written as in oracle/torch_oracle.py).

The entry points launch through the same launchers as the executors, so the shapes below run the executors' launch geometry:
every prep kernel arm (generic, fast <4|8, raw|no-raw>, zero insertion) on both sides of the positions-per-block heuristic,
both attention kernels, all three linear arms (J = 1, 2, 4) at the call sites' shapes.  Errors are relative L2 and bounded at
TOL = 1e-5 unless a test says why not.  Output buffers are pre-filled (NaN, or 0xFF bytes = fp16 NaN) so that an element
the kernel fails to write shows, and buffers the kernels accumulate into hold random values of which only the added part is
compared.

The references are device-agnostic; the tests without the gpu marker show on the CPU that a plausible kernel mistake (an image
slot swapped, a pad column left unwritten, the wrong group size, a lost K tail, permuted gates, ...) moves the result far past
its bound, and they pin the argument checks of the new entry points (which run before any CUDA call)."""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

TOL = 1e-5
STATS_TOL = 1e-6
SPLIT_TOL = 1e-6
GN_EPS = 1e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.double(), b.double().to(a.device)
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _acc_rel(got, prefill, ref):
    """Error of what a kernel ADDED to a pre-filled buffer."""
    return _rel(got.double() - prefill.double(), ref)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _round_up(x, m):
    return (x + m - 1) // m * m


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _gn_stats(x, gs):
    """(sum, sumsq) per (image, group) of NHWC x, float64 [B][C/gs][2]."""
    b, c = x.shape[0], x.shape[-1]
    v = x.double().reshape(b, -1, c // gs, gs)
    return torch.stack([v.sum(dim=(1, 3)), v.pow(2).sum(dim=(1, 3))], dim=-1).contiguous()


def _images(g, b, h, w, c):
    """NHWC inputs whose images differ clearly in mean (in [-1, 1]) and spread (in [0.6, 1.6)), with per-channel offsets: a
    coefficient applied to the wrong image is far off.  |mean| / spread stays small, so the fp32 affine map of the norm is
    accurate to ~1e-7 of its result."""
    n = torch.arange(b, dtype=torch.float64)
    mean = torch.sin(1.7 * n + 0.3).float().view(b, 1, 1, 1)
    std = (0.6 + torch.remainder(0.37 * n + 0.1, 1.0)).float().view(b, 1, 1, 1)
    return torch.randn(b, h, w, c, generator=g) * std * (1 + 0.2 * torch.rand(c, generator=g)) + mean + 0.2 * torch.randn(c, generator=g)


# ------------------------------------------------------------------------------------------------ PLC16 operand
def plc_geometry(b, h, w):
    """conv_tc.cuh plc_geometry: position q = (n * PH + y) * PW + x with PW = W + 1, PH = H + 1; G = PW + 1 zero guard positions
    in front; a plane of 8 channels spans Qalloc positions of 16 bytes."""
    pw, ph = w + 1, h + 1
    q = b * ph * pw
    g = pw + 1
    return pw, ph, q, g, g + -(-q // 128) * 128 + 128 + pw + 1


def plc_decode(buf, b, h, w, c):
    """PLC16 bytes -> (data fp16 NHWC [B][H][W][C], number of non-zero fp16 words anywhere else: guard, pad rows and columns,
    pad channels, the tail behind the last image)."""
    pw, ph, q, g, qa = plc_geometry(b, h, w)
    nch = _round_up(c, 16) // 8
    assert buf.numel() == nch * qa * 16
    planes = buf.view(torch.float16).view(nch, qa, 8)
    data = planes[:, g:g + q].reshape(nch, b, ph, pw, 8)[:, :, :h, :w].permute(1, 2, 3, 0, 4).reshape(b, h, w, 8 * nch)[..., :c]
    inside = torch.zeros(b, ph, pw, dtype=torch.bool, device=buf.device)
    inside[:, :h, :w] = True
    other = torch.ones(nch, qa, 8, dtype=torch.bool, device=buf.device)
    other[:c // 8, g:g + q] = ~inside.reshape(1, q, 1)
    return data, int((planes.view(torch.int16)[other] != 0).sum())


def plc_encode(x16, c):
    """Inverse of plc_decode for a float16 NHWC tensor (zero guard and padding), as a uint8 buffer."""
    b, h, w, _ = x16.shape
    pw, ph, q, g, qa = plc_geometry(b, h, w)
    nch = _round_up(c, 16) // 8
    planes = torch.zeros(nch, qa, 8, dtype=torch.float16, device=x16.device)
    img = torch.zeros(b, ph, pw, 8 * nch, dtype=torch.float16, device=x16.device)
    img[:, :h, :w, :c] = x16
    planes[:, g:g + q] = img.reshape(q, nch, 8).permute(1, 0, 2)
    return planes.view(torch.uint8).reshape(-1)


def prep_excess(got, ref, mag):
    """Largest |got - ref| over its bound: one fp16 ulp (at the larger magnitude; the kernel rounds an fp32 value, so a tie can
    flip) plus 2^-21 of `mag`, the sum of the magnitudes of the terms the kernel's fp32 affine map adds (a cancellation error
    of a few fp32 ulps of those terms, which exceeds an fp16 ulp where the result is within ~1e-4 of zero).  <= 1 passes."""
    g, r = got.double(), ref.double()
    big = torch.maximum(g.abs(), r.abs()).clamp_min(2.0 ** -14)
    bound = torch.exp2(torch.floor(torch.log2(big)) - 10) + 2.0 ** -21 * mag.double()
    e = (g - r).abs() / bound
    return float(torch.where(torch.isfinite(g), e, torch.full_like(e, math.inf)).max())


def ref_prep(x, mode, silu, gs=32, film=None, film_off=0, gamma=None, beta=None, upsample=0):
    """The conv-input transform of NHWC x in float64 (blocks.py:28 GroupNorm, :41-45 AdaGroupNorm, :143-144 SiLU, :109
    nearest-2x upsample; upsample = 2 is the zero insertion of the stride-2 adjoint).  x may be a channel concat: FiLM scale at
    film[:, film_off + c], shift at film[:, film_off + C + c] over all C channels, groups of gs.  Returns (value, mag) with mag
    as prep_excess wants it."""
    xd = _nchw(x.double())
    b, c = xd.shape[:2]
    if mode:
        v = xd.reshape(b, c // gs, -1)
        mean = v.mean(-1, keepdim=True)
        rstd = 1.0 / (v.var(-1, unbiased=False, keepdim=True) + GN_EPS).sqrt()
        mean, rstd = (t.expand(b, c // gs, gs).reshape(b, c, 1, 1) for t in (mean, rstd))
        y = F.group_norm(xd, c // gs, eps=GN_EPS)
        if mode == 1:
            k = 1 + film.double()[:, film_off:film_off + c, None, None]
            sh = film.double()[:, film_off + c:film_off + 2 * c, None, None]
        else:
            k, sh = gamma.double()[None, :, None, None], beta.double()[None, :, None, None]
        y = y * k + sh
        mag = (xd * rstd * k).abs() + (mean * rstd * k).abs() + sh.abs()
    else:
        y, mag = xd, torch.zeros_like(xd)
    if silu:
        y = F.silu(y)
    if upsample == 1:
        y, mag = (F.interpolate(t, scale_factor=2.0, mode="nearest") for t in (y, mag))
    elif upsample == 2:
        z = torch.zeros(b, c, 2 * xd.shape[2], 2 * xd.shape[3], dtype=torch.float64, device=x.device)
        z[:, :, ::2, ::2] = y
        y, mag = z, torch.zeros_like(z)
    return _nhwc(y), _nhwc(mag)


def _prep_call(src0, src1=None, *, mode=0, silu=False, gs=0, film=None, film_off=0, gamma=None, beta=None, upsample=0, raw=False,
               lo=False, raw_lo=False):
    """dmd_prep_act with every requested output pre-filled with 0xFF bytes (fp16 NaN).  Returns ({name: buffer}, H, W); names
    n0 / n1 (operand), r* (raw operand), l* (low parts), rl* (low parts of the raw operand)."""
    from diamond_b200 import _lib

    lib = _lib.lib()
    b, hs, ws, c0 = src0.shape
    c1 = src1.shape[3] if src1 is not None else 0
    h, w = (2 * hs, 2 * ws) if upsample else (hs, ws)
    outs = {}
    for key, on in (("n", True), ("r", raw), ("l", lo), ("rl", raw_lo)):
        for k, c in ((0, c0), (1, c1)):
            if on and c:
                outs[f"{key}{k}"] = torch.full((lib.dmd_plc16_bytes(b, h, w, c),), 0xFF, dtype=torch.uint8, device=src0.device)
    stats = [_gn_stats(s, gs).to(src0.device) if (mode and s is not None) else None for s in (src0, src1)]
    d = _lib.PrepDesc()
    d.src0, d.src1, d.C0, d.C1, d.B, d.Hs, d.Ws = src0.data_ptr(), _lib.ptr(src1), c0, c1, b, hs, ws
    d.upsample, d.mode, d.silu = upsample, mode, int(silu)
    d.stats0, d.stats1, d.gs0, d.gs1 = _lib.ptr(stats[0]), _lib.ptr(stats[1]), gs if mode else 0, (gs if (mode and c1) else 0)
    d.film, d.film_stride, d.film_off = _lib.ptr(film), (film.shape[1] if film is not None else 0), film_off
    d.gamma, d.beta, d.eps = _lib.ptr(gamma), _lib.ptr(beta), GN_EPS
    d.dst0, d.dst1, d.dst_raw0, d.dst_raw1 = (_lib.ptr(outs.get(k)) for k in ("n0", "n1", "r0", "r1"))
    d.dst_lo0, d.dst_lo1, d.dst_raw_lo0, d.dst_raw_lo1 = (_lib.ptr(outs.get(k)) for k in ("l0", "l1", "rl0", "rl1"))
    _lib.check(lib.dmd_prep_act(C.byref(d), _lib.current_stream()))
    return outs, h, w


def _prep_inputs(g, b, hs, ws, c0, c1, mode):
    x0 = _images(g, b, hs, ws, c0)
    x1 = _images(g, b, hs, ws, c1) * 1.3 + 0.2 if c1 else None
    ctot = c0 + c1
    film = 0.3 * torch.randn(b, 2 * ctot + 11, generator=g) if mode == 1 else None   # film_off = 5, 6 floats of slack
    gb = (1 + 0.2 * torch.randn(ctot, generator=g), 0.2 * torch.randn(ctot, generator=g)) if mode == 2 else (None, None)
    return x0, x1, film, gb


def _check_prep(b, hs, ws, c0, c1=0, mode=0, silu=False, gs=32, upsample=0, raw=False, lo=False, raw_lo=False, seed=0):
    """Runs one prep launch and returns its errors: 'junk' (non-zero guard / pad words, must be 0), 'ulp' (prep_excess of the
    operand, <= 1), 'split' / 'raw_split' (relative L2 of hi + lo against the float64 value, <= SPLIT_TOL), 'raw' (exact)."""
    dev = _dev()
    g = _gen(seed)
    x0, x1, film, (gamma, beta) = _prep_inputs(g, b, hs, ws, c0, c1, mode)
    to = lambda t: None if t is None else t.to(dev)  # noqa: E731
    outs, h, w = _prep_call(to(x0), to(x1), mode=mode, silu=silu, gs=gs, film=to(film), film_off=5, gamma=to(gamma), beta=to(beta),
                            upsample=upsample, raw=raw, lo=lo, raw_lo=raw_lo)
    xcat = torch.cat([x0, x1], dim=-1) if c1 else x0
    ref, mag = ref_prep(xcat.to(dev), mode, silu, gs, film=to(film), film_off=5, gamma=to(gamma), beta=to(beta), upsample=upsample)
    raw_ref = ref_prep(xcat.to(dev), 0, False, upsample=upsample)[0]
    errs = {"junk": 0, "ulp": 0.0}
    for k, (lo_c, hi_c) in enumerate(((0, c0), (c0, c0 + c1))):
        if hi_c == lo_c:
            continue
        c = hi_c - lo_c
        dec = {name[:-1]: plc_decode(buf, b, h, w, c) for name, buf in outs.items() if name.endswith(str(k))}
        errs["junk"] += sum(j for _, j in dec.values())
        errs["ulp"] = max(errs["ulp"], prep_excess(dec["n"][0], ref[..., lo_c:hi_c], mag[..., lo_c:hi_c]))
        if "l" in dec:
            errs[f"split{k}"] = _rel(dec["n"][0].double() + dec["l"][0].double(), ref[..., lo_c:hi_c])
        if "r" in dec:   # the raw operand is fp16(x): exact
            errs[f"raw{k}"] = int((dec["r"][0] != raw_ref[..., lo_c:hi_c].half()).sum())
        if "rl" in dec:
            errs[f"raw_split{k}"] = _rel(dec["r"][0].double() + dec["rl"][0].double(), raw_ref[..., lo_c:hi_c])
    return errs, outs


def _assert_prep(errs):
    assert errs["junk"] == 0, errs
    assert errs["ulp"] <= 1.0, errs
    for k, v in errs.items():
        if k.startswith("raw") and not k.startswith("raw_split"):
            assert v == 0, errs
        if "split" in k:
            assert v <= SPLIT_TOL, errs


# which kernel prep_launch (api.cu) runs: prep_fast_kernel<Cpad / 8, raw> for norm + SiLU without upsample or normalised low
# part, every source of the same padded width and raw + raw-low on all sources or none; zero_insert_prep_kernel for upsample 2;
# prep_act_kernel otherwise
PREP_ARMS = [
    dict(c0=64, mode=0),                                             # generic: raw
    dict(c0=64, mode=0, silu=True, raw=True),                        # generic: raw + SiLU (raw operand alongside)
    dict(c0=64, mode=0, upsample=1),                                 # generic: nearest 2x
    dict(c0=32, mode=0, silu=True, upsample=1, lo=True),             # generic: SiLU + nearest 2x, low parts
    dict(c0=64, mode=0, lo=True, raw=True, raw_lo=True),             # generic: the fused-projection operand of the executors
    dict(c0=64, mode=1),                                             # generic: AdaGroupNorm without SiLU
    dict(c0=64, mode=1, silu=True, lo=True),                         # generic: low parts force it
    dict(c0=64, mode=2),                                             # generic: GroupNorm without SiLU
    dict(c0=64, mode=2, silu=True, lo=True, raw=True, raw_lo=True),  # generic: every output
    dict(c0=32, c1=64, mode=1, silu=True),                           # generic: two sources of unequal padding
    dict(c0=32, c1=64, mode=1, silu=True, lo=True, raw=True, raw_lo=True),
    dict(c0=16, mode=1, silu=True, gs=16),                           # generic: 2 chunks
    dict(c0=128, mode=1, silu=True),                                 # generic: 16 chunks, 4 groups
    dict(c0=128, mode=2, silu=True, raw=True, raw_lo=True),
    dict(c0=8, mode=0),                                              # C = 8 stored as 16: a zero pad chunk
    dict(c0=8, mode=2, silu=True, gs=8),
    dict(c0=24, mode=0, silu=True),                                  # C = 24 stored as 32
    dict(c0=32, mode=1, silu=True),                                  # fast <4, false>
    dict(c0=24, mode=1, silu=True, gs=8),                            # fast <4, false>, 3 groups, C = 24 stored as 32
    dict(c0=32, c1=32, mode=2, silu=True, raw=True, raw_lo=True),    # fast <4, true>, two sources
    dict(c0=64, mode=1, silu=True),                                  # fast <8, false>
    dict(c0=64, c1=64, mode=1, silu=True, raw=True, raw_lo=True),    # fast <8, true>: the up path's conv1 + fused projection
    dict(c0=64, mode=0, upsample=2),                                 # zero insertion
    dict(c0=8, mode=0, upsample=2),                                  # zero insertion, C = 8 stored as 16
]


@gpu
@pytest.mark.parametrize("arm", PREP_ARMS, ids=lambda a: "-".join(f"{k}{int(v)}" for k, v in a.items()))
def test_prep_arms(arm):
    """Every kernel arm at 3 images of 12 x 20 (PH x PW = 13 x 21 = 273 positions, 256-position blocks straddle images)."""
    errs, _ = _check_prep(3, 12, 20, seed=len(PREP_ARMS) + sum(map(int, arm.values())), **arm)
    print("prep", arm, errs)
    _assert_prep(errs)


@gpu
@pytest.mark.parametrize("b,hs,ws", [(1, 8, 8), (2, 8, 8), (3, 8, 8), (4, 8, 8), (5, 8, 8), (1, 16, 16), (1, 32, 32), (1, 64, 64),
                                     (256, 64, 64), (3, 24, 40), (2, 60, 62), (7, 5, 9)])
@pytest.mark.parametrize("fast", [True, False], ids=["fast8-raw", "generic-lo"])
def test_prep_block_heuristic(b, hs, ws, fast):
    """Both sides of the positions-per-block heuristic of prep_fill (64 .. 256 positions per block; an 8 x 8 image is 81 positions,
    so blocks straddle images at B >= 2), the benchmarked batch, non-square and odd sizes."""
    kw = dict(raw=True, raw_lo=True) if fast else dict(lo=True)
    errs, _ = _check_prep(b, hs, ws, 64, 0, mode=1, silu=True, seed=b * 1000 + hs * 10 + ws, **kw)
    print(f"prep B={b} {hs}x{ws} fast={fast}:", errs)
    _assert_prep(errs)


@gpu
@pytest.mark.parametrize("c,c1,mode,raw", [(32, 0, 1, False), (32, 32, 2, True), (64, 0, 2, False), (64, 64, 1, True), (24, 0, 1, False)])
@pytest.mark.parametrize("b,hs", [(5, 8), (3, 64)])
def test_prep_fast_path_is_bit_identical_to_generic(c, c1, mode, raw, b, hs):
    """prep_fast_kernel promises bit-identical results to prep_act_kernel.  A normalised low part forces the generic kernel, so
    the same call with and without it must give the same bytes of every other output."""
    dev = _dev()
    g = _gen(b + c + c1 + mode)
    x0, x1, film, (gamma, beta) = _prep_inputs(g, b, hs, hs, c, c1, mode)
    to = lambda t: None if t is None else t.to(dev)  # noqa: E731
    gs = 8 if c == 24 else 32
    kw = dict(mode=mode, silu=True, gs=gs, film=to(film), film_off=5, gamma=to(gamma), beta=to(beta), raw=raw, raw_lo=raw)
    fast, _, _ = _prep_call(to(x0), to(x1), **kw)
    generic, _, _ = _prep_call(to(x0), to(x1), lo=True, **kw)
    for name, buf in fast.items():
        assert torch.equal(buf, generic[name]), name


@gpu
def test_prep_act_wrapper_writes_the_raw_low_parts():
    """ops.prep_act(raw_split=True) reaches prep_fast_kernel<8, true> and returns what the entry point writes."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(4)
    x = _images(g, 2, 16, 16, 64).to(dev)
    film = (0.3 * torch.randn(2, 2 * 64 + 11, generator=g)).to(dev)
    res = ops.prep_act(x, mode=1, silu=True, stats0=_gn_stats(x, 32), gs0=32, film=film, film_off=5, also_raw=True, raw_split=True)
    outs, _, _ = _prep_call(x, mode=1, silu=True, gs=32, film=film, film_off=5, raw=True, raw_lo=True)
    assert res[6] is None and res[9] is None and res[1] is None
    for got, name in ((res[0], "n0"), (res[2], "r0"), (res[8], "rl0")):
        assert torch.equal(got, outs[name]), name


# ------------------------------------------------------------------------------------------------ GroupNorm statistics
@gpu
@pytest.mark.parametrize("b,h,w,c,gs", [(3, 16, 16, 64, 8), (3, 16, 16, 64, 16), (3, 16, 16, 64, 32), (3, 16, 16, 64, 64),
                                        (5, 8, 8, 128, 32), (256, 64, 64, 64, 32), (2, 144, 144, 64, 32)])
def test_gn_stats(b, h, w, c, gs):
    """(sum, sumsq) per (image, group) added to a pre-filled buffer; 144 x 144 x 64 (1.3 M elements per image) reaches the cap of
    64 chunks per image."""
    dev = _dev()
    from diamond_b200 import _lib

    g = torch.Generator(device=dev).manual_seed(b + h + c + gs)
    n = torch.arange(b, device=dev, dtype=torch.float32).view(b, 1, 1, 1)
    x = torch.randn(b, h, w, c, generator=g, device=dev) * (0.6 + torch.remainder(0.37 * n, 1.0)) + torch.sin(1.7 * n + 0.3)
    ref = _gn_stats(x, gs)
    pre = torch.randn(ref.shape, generator=g, device=dev, dtype=torch.float64) * ref.abs().mean()
    st = pre.clone()
    _lib.check(_lib.lib().dmd_gn_stats(x.data_ptr(), st.data_ptr(), b, h * w, c, gs, _lib.current_stream()))
    e = _acc_rel(st, pre, ref)
    print(f"gn_stats B={b} {h}x{w}x{c} gs={gs}: {e:.2e}")
    assert e < STATS_TOL, e


# ------------------------------------------------------------------------------------------------ attention forward
def ref_attn_fwd(x, gs, gamma, beta, wqkv, bqkv, wout, bout):
    """oracle.torch_oracle.self_attention (blocks.py:62-72) with groups of gs channels, float64; x NHWC [B][8][8][C]."""
    xd = _nchw(x.double())
    n, c, h, w = xd.shape
    n_head = max(1, c // 8)
    y = F.group_norm(xd, c // gs, gamma.double(), beta.double(), eps=GN_EPS)
    qkv = F.conv2d(y, wqkv.double().view(3 * c, c, 1, 1), bqkv.double())
    qkv = qkv.view(n, n_head * 3, c // n_head, h * w).transpose(2, 3).contiguous()
    q, k, v = qkv.chunk(3, dim=1)
    att = F.softmax((q @ k.transpose(-2, -1)) / math.sqrt(k.size(-1)), dim=-1)
    a = (att @ v).transpose(2, 3).reshape(n, c, h, w)
    return _nhwc(y + F.conv2d(a, wout.double().view(c, c, 1, 1), bout.double()))


def _attn_inputs(g, b, c):
    n = torch.arange(b, dtype=torch.float32).view(b, 1, 1, 1)
    x = torch.randn(b, 8, 8, c, generator=g) * (0.8 + torch.remainder(0.37 * n, 1.0)) + torch.sin(1.7 * n)
    w = lambda *s: torch.randn(*s, generator=g) / math.sqrt(s[-1])  # noqa: E731
    return (x, 1 + 0.2 * torch.randn(c, generator=g), 0.2 * torch.randn(c, generator=g), w(3 * c, c), 0.1 * torch.randn(3 * c, generator=g),
            w(c, c), 0.1 * torch.randn(c, generator=g))


def attn_errors(b, c, gs, seed=0):
    """One dmd_attn_fwd call: output (pre-filled with NaN) against ref_attn_fwd, and the output statistics it adds to a
    pre-filled buffer against float64 sums of the output it wrote."""
    from diamond_b200 import _lib

    dev = torch.device("cuda:0")
    g = _gen(seed + 1000 * b + c + gs)
    params = [t.to(dev) for t in _attn_inputs(g, b, c)]
    x = params[0]
    ref = ref_attn_fwd(x, gs, *params[1:])
    out = torch.full_like(x, math.nan)
    pre = torch.randn(b, c // gs, 2, generator=g, dtype=torch.float64).to(dev) * 100
    st = pre.clone()
    _lib.check(_lib.lib().dmd_attn_fwd(*[t.data_ptr() for t in (x, _gn_stats(x, gs))], *[t.data_ptr() for t in params[1:]], out.data_ptr(),
                                       st.data_ptr(), b, 64, c, gs, GN_EPS, _lib.current_stream()))
    return {"out": _rel(out, ref), "stats": _acc_rel(st, pre, _gn_stats(out, gs))}


@gpu
@pytest.mark.parametrize("b", [1, 3, 133, 256])
@pytest.mark.parametrize("c,gs", [(32, 32), (64, 32), (64, 64), (32, 8), (64, 8)],
                         ids=["cluster32", "cluster64", "cluster64-gs64", "cluster32-gs8", "single64-gs8"])
def test_attn_fwd(b, c, gs):
    """attn_cluster_kernel (gs a multiple of C / 4) and the one-CTA attn_kernel<64> (gs = 8 at C = 64: eight groups)."""
    _dev()
    errs = attn_errors(b, c, gs)
    print(f"attn_fwd B={b} C={c} gs={gs}:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert errs["out"] < TOL and errs["stats"] < STATS_TOL, errs


@gpu
def test_attn_fwd_single_cta_kernels_without_clusters():
    """DMD_ATTN_CLUSTER=0 (read once per process) runs attn_kernel<32> and attn_kernel<64> for every shape; a child process
    with a timeout runs them."""
    _dev()
    cases = [(1, 32, 32), (133, 32, 32), (3, 32, 8), (3, 64, 32), (256, 64, 64)]
    code = ("import json, sys; sys.path[:0] = [{root!r}, {tests!r}]; import test_gpu_forward_ops as T; "
            "print(json.dumps([T.attn_errors(*c) for c in {cases!r}]))").format(root=ROOT, tests=os.path.join(ROOT, "tests"), cases=cases)
    env = dict(os.environ, DMD_ATTN_CLUSTER="0")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-3000:]
    results = json.loads(res.stdout.strip().splitlines()[-1])
    for case, errs in zip(cases, results):
        print(f"attn_fwd single-CTA B, C, gs = {case}:", {k: f"{v:.2e}" for k, v in errs.items()})
        assert errs["out"] < TOL and errs["stats"] < STATS_TOL, (case, errs)


# ------------------------------------------------------------------------------------------------ linear
def ref_linear(x, w, bias, silu=False, hw_perm=0):
    """F.linear in float64; hw_perm > 0: x is NHWC [B][hw][C] flattened in NCHW order (actor_critic.py:71)."""
    xd = x.double()
    if hw_perm:
        xd = xd.reshape(x.shape[0], hw_perm, -1).transpose(1, 2)
    y = F.linear(xd.reshape(x.shape[0], -1), w.double(), None if bias is None else bias.double())
    return F.silu(y) if silu else y


def linear_arm(b, f):
    """J of linear_launch (api.cu): 32 output features per block if that gives 2 blocks per SM of the H100's 132, else 16 if
    that gives one, else 8."""
    by = -(-b // 32)
    return 4 if -(-f // 32) * by >= 2 * 132 else (2 if -(-f // 16) * by >= 132 else 1)


def _film_rows():
    from oracle import torch_oracle as O

    return sum(s[0] for k, s in O.inner_model_shapes(O.InnerCfg()) if k.endswith(".linear.weight"))


# (name, B, K, F, silu, accumulate, hw_perm, bias, arm J)
LINEAR_CASES = [
    ("cond-mlp", 1, 256, 256, True, False, 0, True, 1),
    ("cond-mlp-b256", 256, 256, 256, True, False, 0, True, 1),
    ("cond-mlp-b288", 288, 256, 256, False, False, 0, True, 2),
    ("film-b1", 1, 256, 7168, False, False, 0, True, 2),
    ("film-b32", 32, 256, 7168, False, False, 0, True, 2),
    ("film-b96", 96, 256, 7168, False, False, 0, True, 4),         # 3 sampler evaluations x 32 environments
    ("lstm-in-b1", 1, 1024, 2048, False, False, 16, True, 1),     # 64 channels of 4 x 4 pixels
    ("lstm-in-b37", 37, 1024, 2048, False, False, 16, True, 2),
    ("lstm-in-b256", 256, 1024, 2048, False, False, 16, True, 4),
    ("lstm-rec-b5", 5, 512, 2048, False, True, 0, True, 1),
    ("lstm-rec-b256", 256, 512, 2048, False, True, 0, True, 4),
    ("actor", 37, 512, 6, False, False, 0, True, 1),
    ("critic", 37, 512, 1, False, False, 0, True, 1),
    ("rew-end-hidden", 37, 512, 512, True, False, 0, True, 1),
    ("rew-end-head", 37, 512, 5, False, False, 0, False, 1),     # Linear(D, 5, bias=False)
    ("k-tail", 37, 1000, 40, False, False, 0, True, 1),           # K = 3 * 256 + 232
    ("k-tail4", 70, 260, 100, True, True, 0, True, 1),            # K = 256 + 4, accumulate before the SiLU
    ("k-tail-perm", 33, 1000, 300, False, False, 250, True, 1),
]


def test_linear_cases_cover_every_arm():
    assert _film_rows() == 7168
    assert {c[-1] for c in LINEAR_CASES} == {1, 2, 4}
    for name, b, _, f, *_, arm in LINEAR_CASES:
        assert linear_arm(b, f) == arm, name


@gpu
@pytest.mark.parametrize("case", LINEAR_CASES, ids=[c[0] for c in LINEAR_CASES])
def test_linear(case):
    """Outputs pre-filled with NaN (every element must be written) or, when accumulating, with random values of which only the
    added part is compared."""
    dev = _dev()
    from diamond_b200 import ops

    name, b, k, f, silu, acc, hw_perm, has_bias, _ = case
    g = _gen(b * 7 + k + f)
    x = torch.randn((b, hw_perm, k // hw_perm) if hw_perm else (b, k), generator=g)
    w = torch.randn(f, k, generator=g) / math.sqrt(k)
    bias = 0.1 * torch.randn(f, generator=g) if has_bias else None
    pre = torch.randn(b, f, generator=g)
    out = pre.to(dev) if acc else torch.full((b, f), math.nan, device=dev)
    ops.linear(x.to(dev), w.to(dev), None if bias is None else bias.to(dev), out=out, silu=silu, accumulate=acc, hw_perm=hw_perm)
    if acc and not silu:   # the recurrent GEMM: only what was added
        e = _acc_rel(out, pre.to(dev), ref_linear(x, w, bias, hw_perm=hw_perm).to(dev))
    elif acc:              # the sum goes through the SiLU
        e = _rel(out, F.silu(ref_linear(x, w, bias, hw_perm=hw_perm) + pre.double()).to(dev))
    else:
        e = _rel(out, ref_linear(x, w, bias, silu, hw_perm).to(dev))
    print(f"linear {name}: {e:.2e}")
    assert e < TOL, e


# ------------------------------------------------------------------------------------------------ max-pool + statistics
def ref_maxpool2(x):
    return _nhwc(F.max_pool2d(_nchw(x.double()), 2))


@gpu
@pytest.mark.parametrize("b,h,c", [(256, 64, 32), (256, 32, 32), (256, 16, 64), (256, 8, 64), (3, 64, 64), (1, 8, 32), (2, 10, 64)])
@pytest.mark.parametrize("stats", [True, False])
def test_maxpool2_stats(b, h, c, stats):
    """The actor-critic encoder's pools (64 -> 32 -> 16 -> 8 -> 4, C = 32, 32, 64, 64, gs = 32): the pooled tensor is exact, its
    statistics are added to a pre-filled buffer; the last pool has none."""
    dev = _dev()
    from diamond_b200 import ops

    g = torch.Generator(device=dev).manual_seed(b + h + c)
    n = torch.arange(b, device=dev, dtype=torch.float32).view(b, 1, 1, 1)
    x = torch.randn(b, h, h + 2, c, generator=g, device=dev) * (0.6 + torch.remainder(0.37 * n, 1.0)) + torch.sin(1.7 * n)
    y = torch.full((b, h // 2, h // 2 + 1, c), math.nan, device=dev)
    ref = ref_maxpool2(x)
    pre = torch.randn(b, c // 32, 2, generator=g, device=dev, dtype=torch.float64) * 100 if stats else None
    st = pre.clone() if stats else None
    ops.maxpool2_stats(x, y, st, 32)
    assert torch.equal(y.double(), ref)
    if stats:
        e = _acc_rel(st, pre, _gn_stats(ref, 32))
        print(f"maxpool2_stats B={b} {h}x{h + 2} C={c}: stats {e:.2e}")
        assert e < STATS_TOL, e


# ------------------------------------------------------------------------------------------------ LSTM gates
def ref_lstm_gates(gates, c_in):
    """float64 nn.LSTMCell whose input weights are the identity and recurrent weights and biases zero: it sees `gates` as its
    pre-activations.  Returns (h, c)."""
    b, hd = c_in.shape
    cell = torch.nn.LSTMCell(4 * hd, hd, dtype=torch.float64, device=gates.device)
    with torch.no_grad():
        cell.weight_ih.copy_(torch.eye(4 * hd, dtype=torch.float64))
        cell.weight_hh.zero_(); cell.bias_ih.zero_(); cell.bias_hh.zero_()
        return cell(gates.double(), (torch.zeros_like(c_in, dtype=torch.float64), c_in.double()))


@gpu
@pytest.mark.parametrize("b,hd,in_place", [(5, 512, False), (256, 512, False), (37, 512, True), (3, 100, False)])
def test_lstm_gates(b, hd, in_place):
    """Gates of +-30 saturate every nonlinearity; in_place: c_out aliases c_in (the reward/termination LSTM over time)."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(b + hd + in_place)
    gates = 2 * torch.randn(b, 4 * hd, generator=g)
    sat = torch.rand(b, 4 * hd, generator=g) < 0.2
    gates[sat] = 30.0 * torch.sign(torch.randn(int(sat.sum()), generator=g))
    c_in = torch.randn(b, hd, generator=g)
    h_ref, c_ref = ref_lstm_gates(gates, c_in)
    gd, cd = gates.to(dev), c_in.to(dev)
    h_out = torch.full((b, hd), math.nan, device=dev)
    c_out = cd if in_place else torch.full((b, hd), math.nan, device=dev)
    ops.lstm_gates(gd, cd, h_out, c_out)
    errs = {"h": _rel(h_out, h_ref), "c": _rel(c_out, c_ref)}
    print(f"lstm_gates B={b} Hd={hd} in_place={in_place}:", errs)
    assert max(errs.values()) < TOL, errs


# ------------------------------------------------------------------------------------------------ resize
@gpu
@pytest.mark.parametrize("b,hs,ws,hd,wd,c,gs", [(3, 5, 7, 8, 8, 16, 16), (3, 8, 8, 5, 7, 64, 32), (2, 30, 36, 32, 32, 64, 32),
                                                (256, 60, 60, 64, 64, 64, 32), (1, 9, 9, 9, 9, 12, 0)])
def test_resize_nhwc(b, hs, ws, hd, wd, c, gs):
    """Zero pad and crop at the bottom / right (UNet.forward) are exact; the statistics of the result are added to a pre-filled
    buffer."""
    dev = _dev()
    from diamond_b200 import ops

    g = torch.Generator(device=dev).manual_seed(b + hs + wd + c)
    x = torch.randn(b, hs, ws, c, generator=g, device=dev) + 0.5
    ref = torch.zeros(b, hd, wd, c, device=dev)
    ref[:, :min(hs, hd), :min(ws, wd)] = x[:, :hd, :wd]
    out = torch.full((b, hd, wd, c), math.nan, device=dev)
    pre = torch.randn(b, c // gs, 2, generator=g, device=dev, dtype=torch.float64) * 100 if gs else None
    st = pre.clone() if gs else None
    ops.resize_nhwc(x, out, st, gs)
    assert torch.equal(out, ref)
    if gs:
        e = _acc_rel(st, pre, _gn_stats(ref, gs))
        print(f"resize {hs}x{ws} -> {hd}x{wd} B={b} C={c}: stats {e:.2e}")
        assert e < STATS_TOL, e


# ------------------------------------------------------------------------------------------------ CPU: argument checks
def test_forward_entry_points_reject_bad_arguments():
    """The checks run before any CUDA call (pointers are dummies), so they are pinned without a GPU."""
    from diamond_b200 import _lib

    lib, p = _lib.lib(), 0x1000

    def err(rc):
        assert rc != 0
        return lib.dmd_last_error().decode()

    assert "bad arguments" in err(lib.dmd_linear(p, p, None, None, 4, 64, 8, 0, 0, 0, None))
    assert "bad arguments" in err(lib.dmd_linear(p, p, None, p, 4, 64, 8, 0, 0, -16, None))
    assert "multiple of 4" in err(lib.dmd_linear(p, p, None, p, 4, 62, 8, 0, 0, 0, None))
    assert "bad hw_perm" in err(lib.dmd_linear(p, p, None, p, 4, 64, 8, 0, 0, 12, None))
    assert "must be even" in err(lib.dmd_maxpool2_stats(p, p, p, 2, 8, 7, 32, 32, None))
    assert "must be even" in err(lib.dmd_maxpool2_stats(p, p, None, 2, 9, 8, 32, 32, None))
    for c, gs in ((48, 24), (64, 48), (48, 16), (24, 8), (64, 0), (32, 64)):   # outside the warp-segment rule of the kernel
        assert "statistics need" in err(lib.dmd_maxpool2_stats(p, p, p, 2, 8, 8, c, gs, None)), (c, gs)
    assert "bad arguments" in err(lib.dmd_maxpool2_stats(None, p, p, 2, 8, 8, 32, 32, None))
    assert "bad arguments" in err(lib.dmd_lstm_gates(p, p, p, None, 2, 16, None))
    assert "bad arguments" in err(lib.dmd_lstm_gates(p, p, p, p, 0, 16, None))
    assert "32-bit" in err(lib.dmd_lstm_gates(p, p, p, p, 1 << 16, 1 << 15, None))
    assert "multiple of 4" in err(lib.dmd_resize_nhwc(p, p, 2, 8, 8, 8, 8, 6, None, 0, None))
    assert "C % gs" in err(lib.dmd_resize_nhwc(p, p, 2, 8, 8, 8, 8, 64, p, 24, None))
    assert "bad arguments" in err(lib.dmd_gn_stats(p, p, 2, 64, 64, 24, None))


# ------------------------------------------------------------------------------------------------ CPU: the tolerances have teeth
def test_plc_codec_round_trip_and_unwritten_pad():
    """The PLC16 decoder inverts the encoder; one pad column left holding 0xFF bytes (an unwritten position) is counted."""
    g = _gen(1)
    x = torch.randn(3, 5, 7, 24, generator=g).half()
    buf = plc_encode(x, 24)
    data, junk = plc_decode(buf, 3, 5, 7, 24)
    assert torch.equal(data, x) and junk == 0
    pw, ph, q, gd, qa = plc_geometry(3, 5, 7)
    planes = buf.view(4, qa, 16)
    planes[:, gd + (1 * ph + 2) * pw + 7] = 0xFF    # image 1, row 2, the pad column x = W
    data, junk = plc_decode(buf, 3, 5, 7, 24)
    assert torch.equal(data, x) and junk == 4 * 8
    buf2 = plc_encode(x, 24)
    buf2.view(4, qa, 16)[3, gd + 5] = 0xFF          # a pad-channel word
    assert plc_decode(buf2, 3, 5, 7, 24)[1] == 8


def test_reference_mistakes_exceed_tolerance():
    """Each GPU test above would fail on a kernel that made one of these mistakes: the mistaken result misses its bound by far
    (computed here on the CPU with the same reference functions, small shapes)."""
    g = _gen(0)
    far = 100
    # prep: image slot swapped in a two-image block (image 1's coefficients on image 0's pixels), the group size wrong
    x = _images(g, 2, 8, 8, 64)
    film = 0.3 * torch.randn(2, 2 * 64 + 11, generator=g)
    ref, mag = ref_prep(x, 1, True, 32, film=film, film_off=5)
    v = x.double().reshape(2, 64, 2, 32)
    mean, rstd = v.mean(dim=(1, 3)), 1 / (v.var(dim=(1, 3), unbiased=False) + GN_EPS).sqrt()
    mean, rstd = (t[[1, 0]].repeat_interleave(32, dim=1).view(2, 1, 1, 64) for t in (mean, rstd))
    k, sh = 1 + film.double()[[1, 0], 5:69].view(2, 1, 1, 64), film.double()[[1, 0], 69:133].view(2, 1, 1, 64)
    swapped = F.silu((x.double() - mean) * rstd * k + sh)
    assert prep_excess(swapped.half(), ref, mag) > far
    assert prep_excess(ref_prep(x, 1, True, 16, film=film, film_off=5)[0].half(), ref, mag) > far
    assert prep_excess(ref.half(), ref, mag) <= 1.0
    # linear: hw_perm read in NHWC order, and the K tail past the last 256-chunk lost
    xl, w = torch.randn(5, 16, 64, generator=g), torch.randn(40, 1024, generator=g)
    assert _rel(ref_linear(xl, w, None), ref_linear(xl, w, None, hw_perm=16)) > far * TOL
    xk, wk = torch.randn(5, 1000, generator=g), torch.randn(40, 1000, generator=g)
    assert _rel(ref_linear(xk[:, :768], wk[:, :768], None), ref_linear(xk, wk, None)) > far * TOL
    # LSTM: gate order i, f, g, o read as f, i, g, o
    gates, c_in = 2 * torch.randn(3, 64, generator=g), torch.randn(3, 16, generator=g)
    ref_h, ref_c = ref_lstm_gates(gates, c_in)
    bad_h, bad_c = ref_lstm_gates(torch.cat([gates[:, 16:32], gates[:, :16], gates[:, 32:]], dim=1), c_in)
    assert min(_rel(bad_h, ref_h), _rel(bad_c, ref_c)) > far * TOL
    # maxpool statistics credited to the neighbouring group
    y = ref_maxpool2(_images(g, 3, 8, 8, 64))
    st = _gn_stats(y, 32)
    assert _rel(st.roll(1, dims=1), st) > far * STATS_TOL
    # attention: two images swapped
    params = _attn_inputs(g, 3, 32)
    ref = ref_attn_fwd(params[0], 32, *params[1:])
    assert _rel(ref[[1, 0, 2]], ref) > far * TOL
    # the attention reference is oracle.torch_oracle.self_attention at its group size of 32
    from oracle import torch_oracle as O

    xa, gam, bet, wq, bq, wo, bo = params
    sd = {"norm.norm.weight": gam.double(), "norm.norm.bias": bet.double(), "qkv_proj.weight": wq.double().view(96, 32, 1, 1),
          "qkv_proj.bias": bq.double(), "out_proj.weight": wo.double().view(32, 32, 1, 1), "out_proj.bias": bo.double()}
    assert _rel(ref, _nhwc(O.self_attention(_nchw(xa.double()), sd, ""))) < 1e-14
