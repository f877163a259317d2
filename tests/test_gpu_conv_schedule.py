"""GPU: the conv kernel's persistent schedule (conv_tc_kernel, diamond_b200/csrc/conv_tc.cuh) against float64.

The kernel runs min(num_tiles, SMs) CTAs and each walks a contiguous range of 128-row tiles, so the shapes here are chosen to
give every CTA several tiles: the shared-memory slab ring wraps (its full / empty parities flip), GroupNorm statistics run in
registers across a CTA's single-image tiles and flush when the image changes, straddling tiles mix with single-image ones in
one CTA, and the tile count does not divide evenly over the CTAs.  Each case states the regime it is meant to reach, and the
test derives that regime from the host plan (dmd_conv_plan) and the device's SM count and asserts it, so a change to the
grid, the ring depth or the tile size fails here instead of silently testing less.

Every case checks:
- every output element against a float64 conv of the operands the kernel actually read (the prepared fp16 operand is decoded
  back, so the reference isolates the conv from the prep), within C_OUT * 2^-23 * (K * sum|x16 w16| + |bias| + |resid|):
  the fp32 accumulation error of K products, with 2^-23 rather than 2^-24 because the tensor cores' fp32 adds need not round
  to nearest; the relative RMS error stays below 2e-5 as in test_gpu_conv.py;
- that `out` and `ostats` are written inside their views and nowhere else: the views sit in larger buffers whose guards
  keep their bit patterns, and no NaN of the fill survives inside the view;
- the statistics against float64 sums of the kernel's own fp32 output within gamma_m * (sum|o|, sum o^2), m the longest fp32
  addition chain of the epilogue (_stats_chain), plus the fp64 atomics' reordering;
- that a second launch gives bit-identical outputs, and statistics that differ only by the order of the fp64 atomics.

The bounds are derived, not fitted.  Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit): the worst output error is
1.4e-2 of its bound (1x1-cout128), the worst statistics error 6.5e-2 of its bound (min-image-7x7), the worst relative RMS
error 1.0e-6; the negative controls miss their bounds by factors of 4e3 to 6e4."""
import ctypes as C
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # fp32 unit roundoff
U64 = 2.0 ** -53          # fp64 unit roundoff
C_OUT = 2.0               # constant of the per-element output bound (see the module docstring)
TILE_M = 128              # kTileM


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _case(id_, b, h, w, c0, cout, **kw):
    d = dict(id=id_, b=b, h=h, w=w, c0=c0, c1=0, cout=cout, taps=9, stride=1, upsample=False, prologue=False, residual=False,
             gs=0, trs=False, precise=False, xproj=False, regime=())
    d.update(kw)
    return d


# regime names: "wrap" the slab ring wraps inside some CTA; "multi" every CTA runs >= 2 tiles; "uneven" CTAs run different tile
# counts; "mixed" some CTA runs both single-image and straddling tiles; "3img" some tile touches three images (kStatSlots);
# "allstraddle" every tile touches two or more images; "all2img" every tile touches exactly two; "aligned" some CTA runs two
# single-image tiles of different images back to back (an image boundary on a tile boundary: the statistics flush on an image
# change without a straddling tile in between).  "uneven" is not claimed where it rests on the all-padding tail tile alone.
CASES = [
    _case("d0-64x64-tapmajor", 32, 64, 64, 64, 64, gs=32, regime=("wrap", "multi")),
    _case("d0-64x64-rowstacked", 32, 64, 64, 64, 64, gs=32, trs=True, regime=("wrap", "multi")),
    _case("resblock-64x64-adagn-silu-residual", 32, 64, 64, 64, 64, gs=32, prologue=True, residual=True, regime=("wrap", "multi")),
    _case("concat-64x64", 16, 64, 64, 64, 64, c1=64, gs=32, regime=("wrap", "multi")),
    _case("concat-16x16", 64, 16, 16, 64, 64, c1=64, gs=32, regime=("wrap", "mixed")),
    _case("split-fp16-conv_in-32x32", 64, 32, 32, 16, 64, precise=True, regime=("wrap", "multi")),
    _case("fused-projection-32x32", 16, 32, 32, 64, 64, xproj=True, gs=32, regime=("wrap", "uneven")),
    _case("1x1-cout64", 64, 32, 32, 64, 64, taps=1, regime=("wrap", "multi")),
    _case("1x1-cout128", 64, 32, 32, 64, 128, taps=1, regime=("wrap", "multi")),
    _case("n16-cout16-gs16", 64, 32, 32, 64, 16, gs=16, regime=("wrap", "multi")),
    _case("n32-cout32-gs16", 64, 32, 32, 64, 32, gs=16, regime=("wrap", "multi")),
    _case("n32-cout32-gs32", 64, 32, 32, 64, 32, gs=32, regime=("wrap", "multi")),
    _case("n128-cout128-gs32", 64, 32, 32, 64, 128, gs=32, regime=("wrap", "multi")),
    _case("n128-cout128-gs64", 64, 32, 32, 64, 128, gs=64, regime=("wrap", "multi")),
    _case("n128-cout128-gs128", 64, 32, 32, 64, 128, gs=128, regime=("wrap", "multi")),
    _case("n128-cout96", 64, 32, 32, 64, 96, regime=("wrap", "multi")),
    _case("stride2-64x64", 32, 64, 64, 64, 64, stride=2, gs=32, regime=("wrap", "multi")),
    _case("stride2-152x280", 8, 152, 280, 64, 64, stride=2, gs=32, regime=("wrap", "multi")),
    # 8x8 images (81 positions) put every tile across an image boundary, up to three images; single-image and straddling
    # tiles meet in one CTA at 16x16 and above (the "mixed" cases)
    _case("straddle-512x8x8", 512, 8, 8, 64, 64, gs=32, regime=("multi", "uneven", "allstraddle", "3img")),
    _case("straddle-1024x8x8", 1024, 8, 8, 64, 64, gs=32, regime=("wrap", "multi", "uneven", "allstraddle", "3img")),
    # PH * PW = 64, the smallest image the statistics epilogue accepts: tiles align with image pairs, so every tile touches
    # exactly two images; 7x8 (PH * PW = 72) is the smallest shape whose tiles touch three
    _case("min-image-7x7", 1024, 7, 7, 64, 64, gs=32, regime=("multi", "all2img")),
    _case("min-image-7x8", 1024, 7, 8, 64, 64, gs=32, regime=("wrap", "multi", "uneven", "allstraddle", "3img")),
    _case("wide-152x280", 8, 152, 280, 64, 64, gs=32, regime=("wrap", "multi", "uneven")),
    # PH * PW = 720 = 45 * 16: every eighth image boundary is a tile boundary
    _case("wide-19x35", 128, 19, 35, 64, 64, gs=32, regime=("wrap", "multi", "uneven", "mixed", "aligned")),
    _case("upsample-16x16-to-32x32", 64, 16, 16, 64, 64, upsample=True, gs=32, regime=("wrap", "multi")),
    _case("conv_out-cout3", 32, 64, 64, 64, 3, regime=("wrap", "multi")),
]


# ------------------------------------------------------------------------------------------------ plan and regime (host side)

def _geometry(b, h, w):
    pw, ph = w + 1, h + 1
    q = b * ph * pw
    g = pw + 1
    return pw, ph, q, g, g + -(-q // TILE_M) * TILE_M + TILE_M + pw + 1


def _conv_size(c):
    h, w = (2 * c["h"], 2 * c["w"]) if c["upsample"] else (c["h"], c["w"])
    return h, w


def _plan(c):
    """dmd_conv_plan of the case: the same validation and planning as the launch (pointers are only tested for NULL)."""
    from diamond_b200 import _lib

    p = 0x1000
    h, w = _conv_size(c)
    d = _lib.ConvDesc()
    d.src0, d.out, d.wpk, d.C0, d.C1 = p, p, p, c["c0"], c["c1"]
    d.src1 = p if c["c1"] else None
    d.B, d.H, d.W, d.taps, d.stride = c["b"], h, w, c["taps"], c["stride"]
    d.Cout, d.CoutPad = c["cout"], -(-c["cout"] // 16) * 16
    if c["gs"]:
        d.out_stats, d.out_gs = p, c["gs"]
    if c["precise"]:
        d.precise, d.src0_lo, d.src1_lo = 1, p, (p if c["c1"] else None)
    d.wpk_layout = int(c["trs"])
    if c["xproj"]:
        d.xsrc0, d.xsrc1, d.xsrc0_lo, d.xsrc1_lo, d.xC0, d.xC1, d.wpk_x = p, p, p, p, 64, 64, p
    info = _lib.ConvPlanInfo()
    rc = _lib.lib().dmd_conv_plan(C.byref(d), C.byref(info))
    assert rc == 0, _lib.lib().dmd_last_error().decode()
    return info


def _regime(c, sms):
    """What the persistent schedule does with the case on `sms` SMs (conv_tc_kernel's tile ranges, api.cu conv_launch_t)."""
    info = _plan(c)
    h, w = _conv_size(c)
    pw, ph, q, _, _ = _geometry(c["b"], h, w)
    tiles = info.tiles
    grid = min(tiles, sms)
    lo, rem = divmod(tiles, grid)
    t = torch.arange(tiles, dtype=torch.int64)
    n_lo = (t * TILE_M) // (ph * pw)
    n_hi = (torch.clamp(t * TILE_M + TILE_M, max=q) - 1) // (ph * pw)
    straddle = n_hi != n_lo
    cta = torch.arange(grid, dtype=torch.int64)
    begin = cta * lo + torch.clamp(cta, max=rem)
    count = lo + (cta < rem).long()
    mixed = any(bool(straddle[b0:b0 + n].any()) and not bool(straddle[b0:b0 + n].all())
                for b0, n in zip(begin.tolist(), count.tolist()))
    owner = torch.repeat_interleave(cta, count)
    change = (owner[1:] == owner[:-1]) & ~straddle[1:] & ~straddle[:-1] & (n_lo[1:] != n_lo[:-1])
    # the last tile holds no output position (only the last image's pad row / column): the all-padding tail tile
    tail = torch.arange((tiles - 1) * TILE_M, q)
    tail_pad = not bool((((tail // pw) % ph < h) & (tail % pw < w)).any())
    return dict(tiles=tiles, grid=grid, tmin=lo, tmax=lo + (rem > 0), kslabs=info.kslabs, stages=info.stages,
                wraps=(lo + (rem > 0)) * info.kslabs > info.stages, mixed=mixed, aligned=bool(change.any()), max_images=int((n_hi - n_lo).max()) + 1,
                min_images=int((n_hi - n_lo).min()) + 1, tail_pad=bool(tail_pad))


def _assert_regime(c, r):
    want = set(c["regime"])
    got = {"wrap": r["wraps"], "multi": r["tmin"] >= 2, "uneven": r["tmin"] != r["tmax"], "mixed": r["mixed"],
           "3img": r["max_images"] == 3, "allstraddle": r["min_images"] >= 2, "all2img": r["min_images"] == r["max_images"] == 2,
           "aligned": r["aligned"]}
    missing = [k for k in want if not got[k]]
    assert not missing, (c["id"], "regime not reached", missing, r)


def _stats_chain(gs, tmax):
    """Longest fp32 addition chain of one statistics value (RegEpilogue::tile / flush_stats): o.x + o.y (sumsq: o.y * o.y and
    an fma) = 2, the gs / 8 column blocks of a row's group sum, one addition per row of the thread (2 per tile) over the CTA's
    tiles, then the 5 butterfly rounds of the warp reduction.  (The sums are converted to fp64 exactly.)"""
    return 2 + gs // 8 + 2 * tmax + 5


def _gamma(m):
    return m * U32 / (1 - m * U32)


def _atomics_per_sum(h, w):
    """fp64 atomics into one (image, group) sum: at most one per warp (8) and tile touching the image."""
    pw, ph = w + 1, h + 1
    return 8 * (-(-(ph * pw) // TILE_M) + 1)


# ------------------------------------------------------------------------------------------------ device side

def _decode(buf, b, h, w, c):
    """PLC16 operand -> NCHW float64 of the C stored channels; also asserts that the pad positions hold zeros (the conv reads
    them as the 3x3 window's zero padding)."""
    pw, ph, q, g, qa = _geometry(b, h, w)
    nch = -(-c // 16) * 2
    planes = buf.view(torch.float16).view(nch, qa, 8)[:, g:g + q].reshape(nch, b, ph, pw, 8)
    assert not planes[:, :, h].any() and not planes[:, :, :, w].any(), "non-zero pad positions in the operand"
    return planes[:, :, :h, :w].permute(1, 0, 4, 2, 3).reshape(b, nch * 8, h, w)[:, :c].double()


def _guarded(shape, dtype, fill, dev, pad=256):
    """A zero-offset-free view of `shape` inside a buffer with `pad` guard elements on each side, every element set to the
    bit pattern `fill` (an int of the dtype's width).  Returns (view, buffer)."""
    n = math.prod(shape)
    ity = {torch.float32: torch.int32, torch.float64: torch.int64}[dtype]
    buf = torch.full((n + 2 * pad,), fill, dtype=ity, device=dev).view(dtype)
    return buf[pad:pad + n].view(shape), buf


NAN32 = 0x7FC0DEAD                    # a quiet NaN with a payload: the fill of `out`
SENT64 = -0x0123456789ABCDEF          # the guard pattern of `ostats` (a finite negative double)


def _check_guards(buf, view, fill):
    ity = {torch.float32: torch.int32, torch.float64: torch.int64}[buf.dtype]
    bits = buf.view(ity)
    off = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
    n = view.numel()
    front, back = bits[:off], bits[off + n:]
    assert bool((front == fill).all()) and bool((back == fill).all()), "a write outside the view"


class Run:
    """One case's operands, weights and float64 reference; launch() runs the conv into fresh guarded buffers."""

    def __init__(self, c, dev, x0=None, wt=None, bias=None):
        from diamond_b200 import ops

        self.c = c
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(c["id"].encode()))
        b, hs, ws, c0, c1, cout = c["b"], c["h"], c["w"], c["c0"], c["c1"], c["cout"]
        self.h, self.w = _conv_size(c)
        self.ho, self.wo = self.h // c["stride"], self.w // c["stride"]
        k = 3 if c["taps"] == 9 else 1
        cin = c0 + c1
        self.x0 = x0 if x0 is not None else torch.randn(b, hs, ws, c0, device=dev, generator=g)
        self.x1 = torch.randn(b, hs, ws, c1, device=dev, generator=g) * 1.5 + 0.3 if c1 else None
        self.wt = wt if wt is not None else torch.randn(cout, cin, k, k, device=dev, generator=g) / math.sqrt(cin * k * k)
        # a per-channel offset makes the groups' sums clearly different, so a sum credited to the wrong group shows
        self.bias = bias if bias is not None else torch.randn(cout, device=dev, generator=g) * 0.1 + torch.arange(cout, device=dev) * 0.02
        self.resid = torch.randn(b, self.ho, self.wo, cout, device=dev, generator=g) if c["residual"] else None
        kw = {}
        if c["prologue"]:   # AdaGroupNorm + SiLU of the ResBlock convs
            film = torch.randn(b, 2 * cin + 5, device=dev, generator=g) * 0.3
            kw = dict(mode=1, silu=True, stats0=ops.gn_stats(self.x0, 32), gs0=32, film=film, film_off=5)
        res = ops.prep_act(self.x0, src1=self.x1, upsample=c["upsample"], split=c["precise"], **kw)
        self.n0, self.n1 = res[0], res[1]
        self.lo0, self.lo1 = (res[6], res[7]) if c["precise"] else (None, None)
        self.wpk, self.cout_pad = ops.pack_conv_weight(self.wt, cin, precise=c["precise"], trs=c["trs"])
        self.xproj = None
        if c["xproj"]:   # ResBlock tail: + proj(cat(x, skip)), split-fp16 operands, centre tap
            xs, sk = torch.randn(b, hs, ws, 64, device=dev, generator=g) * 2, torch.randn(b, hs, ws, 64, device=dev, generator=g) + 0.5
            r = ops.prep_act(xs, src1=sk, also_raw=False, split=True)
            self.wp = torch.randn(cout, 128, 1, 1, device=dev, generator=g) / 11
            self.bp = torch.randn(cout, device=dev, generator=g) * 0.1
            wpkx, _ = ops.pack_conv_weight(self.wp, 128, precise=True)
            self.xproj = (r[0], r[1], r[6], r[7], 64, 64, wpkx, self.bp)
        self._reference()

    def _reference(self):
        """float64 conv of the decoded operands; mag = the same conv of |x16| and |w16| (sum of |products| per output)."""
        c = self.c
        b, h, w = c["b"], self.h, self.w
        pad = 1 if c["taps"] == 9 else 0
        xs = [_decode(self.n0, b, h, w, c["c0"])] + ([_decode(self.n1, b, h, w, c["c1"])] if c["c1"] else [])
        xh = torch.cat(xs, 1)
        wd = self.wt.double()
        wh = self.wt.half().double()
        terms = [(xh, wh)]
        if c["precise"]:    # [A_hi | A_lo | A_hi] against [W_hi | W_hi | W_lo]
            xl = torch.cat([_decode(self.lo0, b, h, w, c["c0"])] + ([_decode(self.lo1, b, h, w, c["c1"])] if c["c1"] else []), 1)
            terms += [(xl, wh), (xh, (wd - wh).half().double())]
        ref = sum(F.conv2d(x, wt, stride=c["stride"], padding=pad) for x, wt in terms)
        mag = sum(F.conv2d(x.abs(), wt.abs(), stride=c["stride"], padding=pad) for x, wt in terms)
        self.K = (c["c0"] + c["c1"]) * c["taps"] * len(terms)
        addend = self.bias.double().view(1, -1, 1, 1).expand_as(ref).clone()
        if self.xproj is not None:
            xh0, xh1, xl0, xl1 = (_decode(t, b, h, w, 64) for t in self.xproj[:4])
            ph_, pl_ = torch.cat([xh0, xh1], 1), torch.cat([xl0, xl1], 1)
            wph = self.wp.half().double()
            wpl = (self.wp.double() - wph).half().double()
            for x, wt in ((ph_, wph), (pl_, wph), (ph_, wpl)):
                ref = ref + F.conv2d(x, wt)
                mag = mag + F.conv2d(x.abs(), wt.abs())
            self.K += 3 * 128
            addend = addend + self.bp.double().view(1, -1, 1, 1)
        if self.resid is not None:
            addend = addend + self.resid.permute(0, 3, 1, 2).double()
        self.ref = ref + addend
        self.bound = C_OUT * 2.0 ** -23 * (self.K * mag + addend.abs()) + 1e-300

    def launch(self):
        from diamond_b200 import ops

        c = self.c
        dev = self.n0.device
        b, cout = c["b"], c["cout"]
        out, obuf = _guarded((b, self.ho, self.wo, cout), torch.float32, NAN32, dev)
        ost = sbuf = None
        if c["gs"]:
            ost, sbuf = _guarded((b, cout // c["gs"], 2), torch.float64, SENT64, dev, pad=16)
            ost.zero_()
        ops.conv2d_operand(self.n0, self.n1, c["c0"], c["c1"], b, self.h, self.w, self.wpk, cout, self.cout_pad, c["taps"],
                           bias=self.bias, stride=c["stride"], residual=self.resid, out_gs=c["gs"], out=out, ostats=ost,
                           lo0=self.lo0, lo1=self.lo1, xproj=self.xproj, trs=c["trs"])
        torch.cuda.synchronize()
        _check_guards(obuf, out, NAN32)
        assert not bool(out.isnan().any()), "output elements left unwritten"
        if sbuf is not None:
            _check_guards(sbuf, ost, SENT64)
        return out, ost


def output_excess(run, out):
    """max over elements of |got - ref| / bound (<= 1 passes)."""
    got = out.permute(0, 3, 1, 2).double()
    return float(((got - run.ref).abs() / run.bound).max())


def _rel_rms(run, out):
    got = out.permute(0, 3, 1, 2).double()
    return float((got - run.ref).pow(2).mean().sqrt() / run.ref.pow(2).mean().sqrt())


def _sums(out, gs):
    b, ho, wo, cout = out.shape
    o = out.double().view(b, ho * wo, cout // gs, gs).permute(0, 2, 1, 3).reshape(b, cout // gs, -1)
    return torch.stack([o.sum(-1), o.pow(2).sum(-1)], -1), torch.stack([o.abs().sum(-1), o.pow(2).sum(-1)], -1)


def stats_excess(st, out, gs, tmax, h, w):
    """max over (image, group, sum|sumsq) of |st - float64 sums of out| / (gamma_m * scale + fp64 reordering)."""
    want, scale = _sums(out, gs)
    n64 = _atomics_per_sum(h, w) + 64       # + the reference sum's own fp64 error (generous)
    bound = (_gamma(_stats_chain(gs, tmax)) + n64 * U64) * scale + 1e-300
    return float(((st - want).abs() / bound).max())


def _regime_line(c, r):
    return (f"{c['id']:36s} tiles {r['tiles']:5d} grid {r['grid']:3d} tiles/CTA {r['tmin']}-{r['tmax']} kslabs {r['kslabs']:2d} "
            f"stages {r['stages']:2d} ring wraps {str(r['wraps']):5s} mixed {str(r['mixed']):5s} aligned {str(r['aligned']):5s} images/tile <= {r['max_images']} "
            f"tail all-pad {r['tail_pad']}")


@pytest.mark.parametrize("c", CASES, ids=[c["id"] for c in CASES])
def test_conv_schedule_against_float64(c):
    dev = _dev()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    r = _regime(c, sms)
    print(_regime_line(c, r))
    _assert_regime(c, r)
    run = Run(c, dev)
    out, st = run.launch()
    ex, rms = output_excess(run, out), _rel_rms(run, out)
    msg = f"{c['id']}: output error / bound {ex:.3e}, rel RMS {rms:.2e}"
    if c["gs"]:
        sx = stats_excess(st, out, c["gs"], r["tmax"], run.h, run.w)
        msg += f", statistics error / bound {sx:.3e}"
    print(msg)
    assert ex <= 1.0, msg
    assert rms < 2e-5, msg
    if c["gs"]:
        assert sx <= 1.0, msg
    # a second launch: the same bits; statistics up to the order of the fp64 atomics
    out2, st2 = run.launch()
    assert torch.equal(out.view(torch.int32), out2.view(torch.int32)), "two launches differ"
    if c["gs"]:
        _, scale = _sums(out, c["gs"])
        n64 = _atomics_per_sum(run.h, run.w)
        assert bool(((st - st2).abs() <= 2 * n64 * U64 * scale).all()), float((st - st2).abs().max())


def test_every_operand_configuration_wraps_the_ring():
    """Coverage of the table above on this device: for each operand configuration and each accumulator width some case runs
    more slabs per CTA than the ring holds."""
    dev = _dev()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    wraps = {}
    for c in CASES:
        r = _regime(c, sms)
        print(_regime_line(c, r))
        kind = ("projection" if c["xproj"] else "split" if c["precise"] else "1x1" if c["taps"] == 1 else
                "concat" if c["c1"] else "single")
        n = 16 if c["cout"] <= 16 else 32 if c["cout"] <= 32 else 64 if c["cout"] <= 64 else 128
        for key in (kind, f"N{n}"):
            wraps[key] = wraps.get(key, False) or r["wraps"]
    print("ring wraps per configuration:", wraps)
    for key in ("single", "concat", "split", "projection", "1x1", "N16", "N32", "N64", "N128"):
        assert wraps.get(key), (key, wraps)


INVARIANCE = [
    (_case("inv-64x64", 32, 64, 64, 64, 64), (0, 13, 31)),
    (_case("inv-8x8-stats", 512, 8, 8, 64, 64, gs=32), (1, 257, 511)),
    (_case("inv-stride2-64x64", 32, 64, 64, 64, 64, stride=2, gs=32), (0, 17, 31)),
]


@pytest.mark.parametrize("c,images", INVARIANCE, ids=[c["id"] for c, _ in INVARIANCE])
def test_conv_output_independent_of_batch_position(c, images):
    """An image's output does not depend on the batch around it: each output element is one fixed-order K reduction of the
    same operands, and the schedule only decides which CTA, tile and accumulator row computes it.  The batch run is compared
    bit for bit with the image alone (B = 1) and with three other images in front of it (a different tile alignment): the
    three before it, or for the first images the three after it.  The statistics of an image agree within the two runs'
    gamma_m bounds."""
    dev = _dev()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    full = Run(c, dev)
    out, st = full.launch()
    t_full = _regime(c, sms)["tmax"]
    for i in images:
        front = list(range(i - 3, i)) if i >= 3 else list(range(i + 1, i + 4))
        for order in ([i], front + [i]):
            sub = dict(c, id=f"{c['id']}-{order[0]}-{i}", b=len(order))
            part = Run(sub, dev, x0=full.x0[order].contiguous(), wt=full.wt, bias=full.bias)
            o2, s2 = part.launch()
            k = len(order) - 1
            assert torch.equal(out[i].view(torch.int32), o2[k].view(torch.int32)), (i, order)
            if c["gs"]:
                t_sub = _regime(sub, sms)["tmax"]
                _, scale = _sums(out[i:i + 1], c["gs"])
                n64 = 2 * _atomics_per_sum(full.h, full.w)
                bound = (_gamma(_stats_chain(c["gs"], t_full)) + _gamma(_stats_chain(c["gs"], t_sub)) + n64 * U64) * scale
                assert bool(((st[i:i + 1] - s2[k:k + 1]).abs() <= bound).all()), (i, order)


def test_schedule_mistakes_exceed_bounds():
    """Negative controls: the checks above fail on the mistakes a schedule change can make, each by far."""
    dev = _dev()
    c = next(c for c in CASES if c["id"] == "straddle-512x8x8")
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tmax = _regime(c, sms)["tmax"]
    run = Run(c, dev)
    out, st = run.launch()
    gs, h, w = c["gs"], run.h, run.w
    assert output_excess(run, out) <= 1.0 and stats_excess(st, out, gs, tmax, h, w) <= 1.0
    pw, ph = w + 1, h + 1
    # the pixels (flat NHWC row index) of tile 101 in padded-linear order; it straddles images 159 and 160
    t = 101
    q = torch.arange(t * TILE_M, (t + 1) * TILE_M, device=dev)
    n, y, x = q // (ph * pw), (q // pw) % ph, q % pw
    keep = (y < h) & (x < w)
    pix = (n * h * w + y * w + x)[keep]
    imgs = n[keep].unique().tolist()
    assert len(imgs) >= 2, imgs
    flat = out.view(-1, c["cout"])
    # 1. one image's statistics swapped with its neighbour's for one group
    bad = st.clone()
    bad[imgs[0], 1], bad[imgs[0] + 1, 1] = st[imgs[0] + 1, 1], st[imgs[0], 1]
    e1 = stats_excess(bad, out, gs, tmax, h, w)
    # 2. the output rows of one tile shifted by one position
    shifted = out.clone()
    shifted.view(-1, c["cout"])[pix] = flat[pix.roll(1)]
    e2 = output_excess(run, shifted)
    # 3. one 8-column block (group 1's first) missing from one tile's statistics of its first image
    bad = st.clone()
    rows = flat[pix[n[keep] == imgs[0]]][:, 32:40].double()
    bad[imgs[0], 1, 0] -= rows.sum()
    bad[imgs[0], 1, 1] -= rows.pow(2).sum()
    e3 = stats_excess(bad, out, gs, tmax, h, w)
    print(f"mistakes / bound: swapped statistics {e1:.3g}, shifted tile rows {e2:.3g}, missing column block {e3:.3g}")
    assert min(e1, e2, e3) > 100, (e1, e2, e3)
