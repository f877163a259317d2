"""The CUDA-core backward kernels (diamond_b200/csrc/bwd_kernels.cuh), one entry point at a time, against float64 torch
autograd of the reference op (forwards written as in oracle/torch_oracle.py).

The entry points launch through the same launchers as the training executors, so the shapes below run the executors'
launch geometry: both sides of the norm-backward pixels-per-block heuristic, the capped column-sum grid at 256 x 64 x 64 rows,
FiLM weight gradients past one 64-sample chunk, the split-K SGEMM plan.  The kernels are fp32; errors are relative L2 and
bounded at TOL = 1e-5 unless a test says why not.  Buffers the kernels accumulate into are pre-filled, and only the added
part is compared.

The references are device-agnostic; the tests without the gpu marker show on the CPU that a plausible kernel mistake (a
dropped pixel lane, two images swapped, a wrong group size, a lost K tail, ...) moves the result far past TOL."""
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

TOL = 1e-5
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


def _loss_scale_exp():
    text = open(os.path.join(ROOT, "include", "diamond_b200.h")).read()
    return int(re.search(r"#define\s+DMD_LOSS_SCALE_EXP\s+(\d+)", text).group(1))


# ------------------------------------------------------------------------------------------------ references (float64)
def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _gn_stats(x, gs):
    """(sum, sumsq) per (image, group) of NHWC x, float64 [B][C/gs][2]: what the forward's statistics epilogue stores."""
    b, c = x.shape[0], x.shape[-1]
    v = x.double().reshape(b, -1, c // gs, gs)
    return torch.stack([v.sum(dim=(1, 3)), v.pow(2).sum(dim=(1, 3))], dim=-1).contiguous()


def ref_norm(x, gy, gs, mode, act, film=None, film_off=0, ctot=None, c_off=0, gamma=None, beta=None):
    """silu(GroupNorm(x) * k + sh) backward (blocks.py:28,41-45); x, gy NHWC.  Returns (gx NHWC, d film | (d gamma, d beta))."""
    x = _nchw(x.double()).detach().requires_grad_()
    c = x.shape[1]
    z = F.group_norm(x, c // gs, eps=GN_EPS)
    if mode == 1:
        film = film.double().detach().requires_grad_()
        sc = film[:, film_off + c_off:film_off + c_off + c, None, None]
        sh = film[:, film_off + ctot + c_off:film_off + ctot + c_off + c, None, None]
        z = z * (1 + sc) + sh
        leaves = [x, film]
    else:
        gamma, beta = gamma.double().detach().requires_grad_(), beta.double().detach().requires_grad_()
        z = z * gamma[c_off:c_off + c, None, None] + beta[c_off:c_off + c, None, None]
        leaves = [x, gamma, beta]
    y = F.silu(z) if act else z
    g = torch.autograd.grad(y, leaves, _nchw(gy.double()))
    return (_nhwc(g[0]),) + tuple(g[1:])


def ref_attn(x, gout, gamma, beta, wqkv, bqkv, wout, bout):
    """autograd of oracle.torch_oracle.self_attention (blocks.py:62-72); x, gout NHWC [B][8][8][C].  Returns
    (gx NHWC, dgamma, dbeta, dwqkv, dbqkv, dwout, dbout)."""
    from oracle import torch_oracle as O

    c = x.shape[-1]
    leaves = [t.double().detach().requires_grad_() for t in (x, gamma, beta, wqkv, bqkv, wout, bout)]
    xx, g_, b_, wq, bq, wo, bo = leaves
    sd = {"norm.norm.weight": g_, "norm.norm.bias": b_, "qkv_proj.weight": wq.view(3 * c, c, 1, 1), "qkv_proj.bias": bq,
          "out_proj.weight": wo.view(c, c, 1, 1), "out_proj.bias": bo}
    y = O.self_attention(_nchw(xx), sd, "")
    g = torch.autograd.grad(y, leaves, _nchw(gout.double()))
    return tuple(g)


def ref_sgemm(a_mat, b_mat):
    return a_mat.double() @ b_mat.double()


def ref_film_wgrad(dfilm, cond):
    """FiLM linear (blocks.py:39) weight / bias gradients of the batched [rows][CC] matrix."""
    d = dfilm.double()
    return d.t() @ cond.double(), d.sum(0)


def ref_colsum(x):
    return x.double().sum(0)


def ref_embedding(de, act, num_actions, e_dim):
    """act_emb (inner_model.py:27-30): gradient of F.embedding(act, E).flatten(1) given de [B][T*E]."""
    table = torch.zeros(num_actions, e_dim, dtype=torch.float64, device=de.device, requires_grad=True)
    (g,) = torch.autograd.grad(F.embedding(act, table).flatten(1), table, de.double())
    return g


def ref_sumpool2(gin):
    """adjoint of nearest-2x upsampling (blocks.py:109); gin NHWC [B][2H][2W][C] -> [B][H][W][C]."""
    b, h2, w2, c = gin.shape
    u = torch.zeros(b, c, h2 // 2, w2 // 2, dtype=torch.float64, device=gin.device, requires_grad=True)
    (g,) = torch.autograd.grad(F.interpolate(u, scale_factor=2.0, mode="nearest"), u, _nchw(gin.double()))
    return _nhwc(g)


def ref_maxpool2(y, gp):
    """torch's own MaxPool2d(2) backward (actor_critic.py:109), float64; y NHWC pre-pool, gp NHWC pooled."""
    yy = _nchw(y.double()).detach().requires_grad_()
    (g,) = torch.autograd.grad(F.max_pool2d(yy, 2), yy, _nchw(gp.double()))
    return _nhwc(g)


def ref_lstm(gates, c_in, g_h, g_c):
    """nn.LSTMCell autograd wrt its gate pre-activations and the incoming cell state: a cell whose input weights are the
    identity and whose recurrent weights and biases are zero sees `gates` as its pre-activations."""
    b, hd = c_in.shape
    cell = torch.nn.LSTMCell(4 * hd, hd, dtype=torch.float64, device=gates.device)
    with torch.no_grad():
        cell.weight_ih.copy_(torch.eye(4 * hd, dtype=torch.float64))
        cell.weight_hh.zero_(); cell.bias_ih.zero_(); cell.bias_hh.zero_()
    x = gates.double().detach().requires_grad_()
    c0 = c_in.double().detach().requires_grad_()
    h1, c1 = cell(x, (torch.zeros_like(c0), c0))
    zero = torch.zeros_like(c0)
    return torch.autograd.grad((h1, c1), (x, c0), (zero if g_h is None else g_h.double(), zero if g_c is None else g_c.double()))


def ref_heads(hx_out, wa, ba, wc, bc, g_hx, g_logits, g_val):
    """actor / critic heads (actor_critic.py:73): gradients wrt hx_out, actor bias, critic weight and bias."""
    hx, ba_, wc_, bc_ = [t.double().detach().requires_grad_() for t in (hx_out, ba, wc, bc)]
    total = hx.sum() * 0
    if g_hx is not None:
        total = total + (hx * g_hx.double()).sum()
    if g_logits is not None:
        total = total + ((hx @ wa.double().t() + ba_) * g_logits.double()).sum()
    if g_val is not None:
        total = total + ((hx @ wc_.view(-1, 1) + bc_).squeeze(1) * g_val.double()).sum()
    return torch.autograd.grad(total, (hx, ba_, wc_, bc_), allow_unused=True, materialize_grads=True)


def ref_dsilu(pre, dh):
    p = pre.double().detach().requires_grad_()
    (g,) = torch.autograd.grad(F.silu(p), p, dh.double())
    return g


def loss_scale_ok(scale, amax, e):
    """S a power of two with max|S g| in [2^(e-1), 2^e), or S = 1 for a zero gradient."""
    s, inv = float(scale[0]), float(scale[1])
    if amax == 0.0:
        return s == 1.0 and inv == 1.0
    m, _ = math.frexp(s)
    return m == 0.5 and inv == 1.0 / s and 2.0 ** (e - 1) <= amax * s < 2.0 ** e


# ------------------------------------------------------------------------------------------------ norm + SiLU backward
def _norm_inputs(g, b, hw, c, mode, film_stride=None):
    x = torch.randn(b, hw, 1, c, generator=g) * (0.5 + torch.rand(c, generator=g)) + 0.3 * torch.randn(c, generator=g)
    gy = torch.randn(b, hw, 1, c, generator=g)
    if mode == 1:
        return x, gy, 0.2 * torch.randn(b, film_stride, generator=g)
    return x, gy, (1 + 0.2 * torch.randn(c, generator=g), 0.2 * torch.randn(c, generator=g))


@gpu
@pytest.mark.parametrize("mode,act,b,hw,c,gs,acc", [
    (1, True, 1, 64, 32, 32, False),
    (1, True, 2, 4096, 64, 32, False),      # level 0 of the default net at the fixtures' batch: 32-pixel blocks
    (1, False, 5, 1024, 96, 32, True),
    (1, True, 256, 4096, 64, 32, True),     # the benchmarked batch: 2048-pixel blocks, 128 pixels per thread lane
    (1, True, 256, 256, 128, 32, False),
    (1, True, 2, 64, 16, 16, False),        # one group of C < 32 channels (gs = C)
    (2, True, 2, 256, 128, 32, False),
    (2, True, 256, 1024, 64, 32, True),
    (2, False, 5, 64, 16, 16, True),
    (2, True, 1, 4096, 32, 32, False),
])
def test_norm_bwd(mode, act, b, hw, c, gs, acc):
    """Both passes (and the affine parameter gradients in mode 2).  Mode 1 writes d scale / d shift into a FiLM-layout buffer
    at a row offset; acc: gx accumulates and an addend rides along; mode 2 carries a loss scale of 4 (inv_scale 1/4)."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(100 + 7 * b + c + hw + mode)
    film_off, stride = 24, 2 * c + 40
    x, gy, par = _norm_inputs(g, b, hw, c, mode, stride)
    s = 4.0 if mode == 2 else 1.0
    if mode == 1:
        gx_ref, dfilm_ref = ref_norm(x.to(dev), gy.to(dev), gs, 1, act, film=par.to(dev), film_off=film_off, ctot=c)
    else:
        gx_ref, dgam_ref, dbet_ref = ref_norm(x.to(dev), gy.to(dev), gs, 2, act, gamma=par[0].to(dev), beta=par[1].to(dev))
    xd, gyd = x.to(dev), (gy * s).to(dev)
    pre = torch.randn(x.shape, generator=g).to(dev) if acc else torch.zeros(x.shape, device=dev)
    addend = torch.randn(x.shape, generator=g).to(dev) if acc else None
    gx = pre.clone()
    kw = dict(mode=mode, act=act, addend=addend, accumulate=acc)
    if mode == 1:
        dfilm = torch.zeros(b, stride, device=dev)
        ops.norm_bwd(xd, gyd, _gn_stats(x, gs).to(dev), gs, gx, dfilm[:, film_off + c:], dfilm[:, film_off:], stride,
                     film=par.to(dev), film_off=film_off, film_ctot=c, **kw)
        errs = {"gx": _acc_rel(gx, pre + (addend if acc else 0), gx_ref), "dfilm": _rel(dfilm, dfilm_ref)}
    else:
        sums = torch.zeros(2, b, 128, device=dev)
        pg, pb = torch.randn(c, generator=g).to(dev), torch.randn(c, generator=g).to(dev)
        dgam, dbet = pg.clone(), pb.clone()
        inv = torch.tensor([1 / s], device=dev)
        ops.norm_bwd(xd, gyd, _gn_stats(x, gs).to(dev), gs, gx, sums[0], sums[1], 128, gamma=par[0].to(dev), beta=par[1].to(dev),
                     dgamma=dgam, dbeta=dbet, inv_scale=inv, **kw)
        errs = {"gx": _acc_rel(gx, pre + (addend if acc else 0), gx_ref * s), "dgamma": _acc_rel(dgam, pg, dgam_ref),
                "dbeta": _acc_rel(dbet, pb, dbet_ref)}
    print(f"norm_bwd mode={mode} act={act} B={b} HW={hw} C={c} gs={gs} acc={acc}:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs


@gpu
def test_norm_bwd_concat_pair():
    """A norm over cat(x0, x1) (the up path's channel concat, blocks.py:174) runs as two launches, source 1 at channel offset
    64 of 128, sharing one FiLM row block; each writes its own columns of d scale / d shift."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(77)
    b, hw, c, gs, stride = 3, 1024, 128, 32, 2 * 128 + 8
    x, gy, film = _norm_inputs(g, b, hw, c, 1, stride)
    gx_ref, dfilm_ref = ref_norm(x.to(dev), gy.to(dev), gs, 1, True, film=film.to(dev), film_off=8, ctot=c)
    dfilm = torch.zeros(b, stride, device=dev)
    gxs = []
    for k in range(2):
        xs, gys = x[..., 64 * k:64 * (k + 1)].contiguous(), gy[..., 64 * k:64 * (k + 1)].contiguous()
        gx = torch.zeros(xs.shape, device=dev)
        ops.norm_bwd(xs.to(dev), gys.to(dev), _gn_stats(xs, gs).to(dev), gs, gx, dfilm[:, 8 + c + 64 * k:], dfilm[:, 8 + 64 * k:], stride,
                     mode=1, film=film.to(dev), film_off=8, film_ctot=c, c_off=64 * k)
        gxs.append(gx)
    errs = {"gx": _rel(torch.cat(gxs, dim=-1), gx_ref), "dfilm": _rel(dfilm, dfilm_ref)}
    print("norm_bwd concat pair:", errs)
    assert max(errs.values()) < TOL, errs


# ------------------------------------------------------------------------------------------------ attention backward
def _attn_inputs(g, b, c):
    x = torch.randn(b, 8, 8, c, generator=g) * 1.5 + 0.2
    w = lambda *s: torch.randn(*s, generator=g) / math.sqrt(s[-1])  # noqa: E731
    return (x, torch.randn(b, 8, 8, c, generator=g), 1 + 0.2 * torch.randn(c, generator=g), 0.2 * torch.randn(c, generator=g),
            w(3 * c, c), 0.1 * torch.randn(3 * c, generator=g), w(c, c), 0.1 * torch.randn(c, generator=g))


@gpu
@pytest.mark.parametrize("c", [32, 64])
@pytest.mark.parametrize("b", [1, 3, 133])
def test_attn_bwd(b, c):
    """g_x and all six parameter gradients; the parameter gradients are added (times inv_scale = 1/2, g_out scaled by 2) to
    pre-filled buffers."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(300 + b + c)
    x, gout, gamma, beta, wqkv, bqkv, wout, bout = _attn_inputs(g, b, c)
    ref = ref_attn(*(t.to(dev) for t in (x, gout, gamma, beta, wqkv, bqkv, wout, bout)))
    pre = [(torch.randn(r.shape, generator=g) * float(r.std())).float().to(dev) for r in ref[1:]]
    pgrads = tuple(p.clone() for p in pre)
    gs = 32
    gx = ops.attn_bwd(x.to(dev), _gn_stats(x, gs).to(dev), gamma.to(dev), beta.to(dev), wqkv.to(dev), bqkv.to(dev), wout.to(dev),
                      (2 * gout).to(dev), gs, pgrads, inv_scale=torch.tensor([0.5], device=dev))
    names = ["gx", "dgamma", "dbeta", "dwqkv", "dbqkv", "dwout", "dbout"]
    errs = {"gx": _rel(gx, 2 * ref[0])}
    errs.update({n: _acc_rel(p, q, r) for n, p, q, r in zip(names[1:], pgrads, pre, ref[1:])})
    print(f"attn_bwd B={b} C={c}:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs


# ------------------------------------------------------------------------------------------------ SGEMM
def _sgemm_operands(g, m, n, k, sak1, sbk1):
    """A(m,k), B(k,n) as the call sites store them: sak == 1 -> A row-major [M][K], else [K][M]; sbk == 1 -> B stored [N][K],
    else [K][N]."""
    a_mat, b_mat = torch.randn(m, k, generator=g), torch.randn(k, n, generator=g)
    a = a_mat.contiguous() if sak1 else a_mat.t().contiguous()
    bm = b_mat.t().contiguous() if sbk1 else b_mat.contiguous()
    strides = ((k, 1) if sak1 else (1, m)) + ((1, k) if sbk1 else (n, 1))
    return a_mat, b_mat, a, bm, strides


@gpu
@pytest.mark.parametrize("sak1", [True, False])
@pytest.mark.parametrize("sbk1", [True, False])
@pytest.mark.parametrize("m,n,k,chunks", [(3, 257, 7168, 0), (65, 130, 33, 0), (256, 256, 256, 0), (256, 256, 7001, 28), (3, 257, 100, 8)])
def test_sgemm(m, n, k, chunks, sak1, sbk1):
    """Off-tile M, N, K, a device alpha, accumulation onto a pre-filled C, and the planned split-K (K not divisible by the
    chunk count; K = 100 over 8 chunks plans 7 splits of 16).  Two runs are bit-identical."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(m + n + k + chunks + 2 * sak1 + sbk1)
    a_mat, b_mat, a, bm, (sam, sak, sbk, sbn) = _sgemm_operands(g, m, n, k, sak1, sbk1)
    ref = ref_sgemm(a_mat, b_mat) * 0.375
    pre = torch.randn(m, n, generator=g) * float(ref.std())
    alpha = torch.tensor([0.375], device=dev)
    outs = []
    for _ in range(2):
        c = pre.to(dev).clone()
        ops.sgemm(a.to(dev), sam, sak, bm.to(dev), sbk, sbn, c, n, m, n, k, alpha=alpha, accumulate=True, chunks=chunks)
        outs.append(c)
    e = _acc_rel(outs[0], pre.to(dev), ref.to(dev))
    print(f"sgemm M={m} N={n} K={k} chunks={chunks} sak1={sak1} sbk1={sbk1}: {e:.2e}")
    assert e < TOL, e
    assert torch.equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ FiLM wgrad
@gpu
@pytest.mark.parametrize("cc", [64, 256])
@pytest.mark.parametrize("b", [1, 63, 64, 65, 256])
def test_film_wgrad(b, cc):
    """203 FiLM rows (not a multiple of 8) scattered over a flat gradient buffer by shuffled offset tables; batches on both
    sides of the kernel's 64-sample chunk; inv_scale; accumulation onto non-zero gradients."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(b * 7 + cc)
    rows = 203
    dfilm, cond = torch.randn(b, rows, generator=g), torch.randn(b, cc, generator=g)
    dw, db = ref_film_wgrad(dfilm, cond)
    inv = 0.125
    woff = torch.randperm(rows, generator=g) * cc
    boff = rows * cc + torch.randperm(rows, generator=g)
    n = rows * cc + rows + 5
    inc = torch.zeros(n, dtype=torch.float64)
    inc[(woff[:, None] + torch.arange(cc)).reshape(-1)] = (dw * inv).reshape(-1)
    inc[boff] = db * inv
    pre = torch.randn(n, generator=g) * float(inc.std())
    grads = pre.to(dev).clone()
    ops.film_wgrad(dfilm.to(dev), cond.to(dev), grads, woff.to(dev), boff.to(dev), torch.tensor([inv], device=dev))
    e = _acc_rel(grads, pre.to(dev), inc.to(dev))
    print(f"film_wgrad B={b} CC={cc}: {e:.2e}")
    assert e < TOL, e


# ------------------------------------------------------------------------------------------------ column sums
@gpu
@pytest.mark.parametrize("c,creal,rows", [
    (8, 3, 1), (8, 3, 3), (8, 3, 256 * 64 * 64),       # conv_out bias: 3 real channels of 8
    (16, 16, 1), (16, 16, 256 * 64 * 64),
    (64, 64, 3), (64, 64, 256 * 64 * 64),              # a 64-channel conv bias at the benchmarked batch: the 592-block cap
    (256, 256, 256 * 64 * 64),
    (2048, 2048, 1), (2048, 2048, 3), (2048, 2048, 4096),   # LSTM biases (4 x 512): 8 column blocks
])
def test_colsum(c, creal, rows):
    """out and out2 receive the same inv_scale-weighted sums for c < Creal and are untouched above."""
    dev = _dev()
    from diamond_b200 import ops

    g = torch.Generator(device=dev).manual_seed(c + rows)
    x = torch.randn(rows, c, generator=g, device=dev)
    ref = ref_colsum(x) * 0.5
    pre1, pre2 = torch.randn(c, generator=g, device=dev), torch.randn(c, generator=g, device=dev)
    out, out2 = pre1.clone(), pre2.clone()
    ops.colsum(x, out, out2, torch.tensor([0.5], device=dev), creal)
    e = max(_acc_rel(out[:creal], pre1[:creal], ref[:creal]), _acc_rel(out2[:creal], pre2[:creal], ref[:creal]))
    print(f"colsum C={c} Creal={creal} rows={rows}: {e:.2e}")
    assert e < TOL, e
    assert torch.equal(out[creal:], pre1[creal:]) and torch.equal(out2[creal:], pre2[creal:])


# ------------------------------------------------------------------------------------------------ embedding backward
@gpu
@pytest.mark.parametrize("b,same", [(256, False), (3, True)])
def test_embedding_bwd(b, same):
    """T = 4 actions per sample from 4 possible actions: rows of the table receive many colliding atomic adds (all of them
    when every action is the same)."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(b + 1)
    t, e_dim, na = 4, 64, 4
    act = torch.full((b, t), 2, dtype=torch.int64) if same else torch.randint(0, na, (b, t), generator=g)
    de = torch.randn(b, t * e_dim, generator=g)
    ref = ref_embedding(de, act, na, e_dim) * 0.25
    pre = torch.randn(na, e_dim, generator=g) * float(ref.std())
    table = pre.to(dev).clone()
    ops.embedding_bwd(de.to(dev), act.to(dev), table, torch.tensor([0.25], device=dev))
    e = _acc_rel(table, pre.to(dev), ref.to(dev))
    print(f"embedding_bwd B={b} same={same}: {e:.2e}")
    assert e < TOL, e


# ------------------------------------------------------------------------------------------------ elementwise adjoints
@gpu
@pytest.mark.parametrize("b,h,w,c", [(3, 5, 7, 16), (2, 4, 4, 64), (1, 32, 16, 32)])
@pytest.mark.parametrize("acc", [False, True])
def test_sumpool2(b, h, w, c, acc):
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(b * h * w + c + acc)
    gin = torch.randn(b, 2 * h, 2 * w, c, generator=g)
    ref = ref_sumpool2(gin)
    pre = torch.randn(b, h, w, c, generator=g) if acc else torch.zeros(b, h, w, c)
    out = pre.to(dev).clone()
    ops.sumpool2(gin.to(dev), out, accumulate=acc)
    e = _acc_rel(out, pre.to(dev), ref.to(dev))
    print(f"sumpool2 B={b} {h}x{w} C={c} acc={acc}: {e:.2e}")
    assert e < TOL, e


@gpu
def test_dsilu_mul():
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(5)
    pre, dh = 3 * torch.randn(1000, generator=g), torch.randn(1000, generator=g)
    e = _rel(ops.dsilu_mul(pre.to(dev), dh.to(dev)), ref_dsilu(pre, dh).to(dev))
    print(f"dsilu_mul: {e:.2e}")
    assert e < TOL, e


# ------------------------------------------------------------------------------------------------ actor-critic pieces
def _tied_pool_input(g, b, h, w, c):
    """Values on a 3-level grid: most 2x2 windows hold an exact tie for the maximum."""
    return torch.randint(0, 3, (b, h, w, c), generator=g).float() - 1.0


@gpu
@pytest.mark.parametrize("b,h,w,c", [(2, 8, 6, 64), (3, 16, 16, 64), (1, 64, 64, 32)])
def test_maxpool2_bwd_ties(b, h, w, c):
    """Exact ties resolved as torch's float64 max_pool2d backward resolves them; the result is exact."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(b * h + w + c)
    y = _tied_pool_input(g, b, h, w, c)
    gp = torch.randn(b, h // 2, w // 2, c, generator=g)
    got = ops.maxpool2_bwd(y.to(dev), gp.to(dev)).cpu()
    ref = ref_maxpool2(y, gp)
    print(f"maxpool2_bwd B={b} {h}x{w} C={c}: mismatches {int((got.double() != ref).sum())}")
    assert torch.equal(got.double(), ref)


@gpu
@pytest.mark.parametrize("has_gh,has_gc", [(True, False), (True, True), (False, True)])
def test_lstm_cell_bwd(has_gh, has_gc):
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(11 + has_gh + 2 * has_gc)
    b, hd = 5, 512
    gates, c_in = 2 * torch.randn(b, 4 * hd, generator=g), torch.randn(b, hd, generator=g)
    g_h = torch.randn(b, hd, generator=g) if has_gh else None
    g_c = torch.randn(b, hd, generator=g) if has_gc else None
    dg_ref, gc_ref = ref_lstm(gates, c_in, g_h, g_c)
    dg, gc = ops.lstm_cell_bwd(gates.to(dev), c_in.to(dev), None if g_h is None else g_h.to(dev), None if g_c is None else g_c.to(dev))
    errs = {"dgates": _rel(dg.cpu(), dg_ref), "g_c_in": _rel(gc.cpu(), gc_ref)}
    print(f"lstm_cell_bwd g_h={has_gh} g_c={has_gc}:", errs)
    assert max(errs.values()) < TOL, errs


@gpu
@pytest.mark.parametrize("a", [6, 3])
@pytest.mark.parametrize("heads", ["both", "actor", "critic"])
def test_heads_bwd(a, heads):
    """A not a multiple of 4; either head's gradient may be absent (its parameter gradients are then left untouched)."""
    dev = _dev()
    from diamond_b200 import ops

    g = _gen(a + len(heads))
    b, hd = 5, 512
    hx_out, g_hx = torch.randn(b, hd, generator=g), torch.randn(b, hd, generator=g)
    wa, ba = torch.randn(a, hd, generator=g) / 20, torch.randn(a, generator=g)
    wc, bc = torch.randn(1, hd, generator=g) / 20, torch.randn(1, generator=g)
    g_logits = torch.randn(b, a, generator=g) if heads != "critic" else None
    g_val = torch.randn(b, generator=g) if heads != "actor" else None
    r_gh, r_dba, r_dwc, r_dbc = ref_heads(hx_out, wa, ba, wc, bc, g_hx, g_logits, g_val)
    pre = [torch.randn(a, generator=g), torch.randn(1, hd, generator=g), torch.randn(1, generator=g)]
    dba, dwc, dbc = [p.to(dev).clone() for p in pre]
    to = lambda t: None if t is None else t.to(dev)  # noqa: E731
    gh = ops.heads_bwd(g_hx.to(dev), to(g_logits), to(g_val), hx_out.to(dev), wa.to(dev), wc.to(dev), dba, dwc, dbc)
    errs = {"g_h": _rel(gh.cpu(), r_gh)}
    if g_logits is not None:
        errs["dba"] = _acc_rel(dba.cpu(), pre[0], r_dba)
    else:
        assert torch.equal(dba.cpu(), pre[0])
    if g_val is not None:
        errs["dWc"], errs["dbc"] = _acc_rel(dwc.cpu(), pre[1], r_dwc), _acc_rel(dbc.cpu(), pre[2], r_dbc)
    else:
        assert torch.equal(dwc.cpu(), pre[1]) and torch.equal(dbc.cpu(), pre[2])
    print(f"heads_bwd A={a} {heads}:", errs)
    assert max(errs.values()) < TOL, errs


# ------------------------------------------------------------------------------------------------ loss scale
@gpu
def test_loss_scale():
    """S = 1 for a zero gradient; an exact power of two lands at the bottom of [2^(E-1), 2^E), the float below 1.0 just
    under its top; a large gradient (grid-stride loop, negative maximum at the very end) lands inside."""
    dev = _dev()
    from diamond_b200 import ops

    e = _loss_scale_exp()
    assert torch.equal(ops.loss_scale(torch.zeros(1000, device=dev)).cpu(), torch.tensor([1.0, 1.0]))
    for m in (2.0 ** -7, 2.0 ** 3, 1.0):
        g = torch.full((300,), m / 4, device=dev)
        g[17] = -m
        s = ops.loss_scale(g).cpu()
        assert loss_scale_ok(s, m, e) and m * float(s[0]) == 2.0 ** (e - 1), (m, s)
    below = float(torch.nextafter(torch.tensor(1.0), torch.tensor(0.0)))
    s = ops.loss_scale(torch.tensor([0.25, below, -0.5], device=dev)).cpu()
    assert float(s[0]) == 2.0 ** e and loss_scale_ok(s, below, e), s
    big = torch.randn(3 << 20, generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    big[-1] = -2 * float(big.abs().max())
    amax = float(big.abs().max())
    s = ops.loss_scale(big).cpu()
    print(f"loss scale E={e}: max|g| {amax:.4g} -> S {float(s[0])}, max|S g| {amax * float(s[0]):.1f}")
    assert loss_scale_ok(s, amax, e), (amax, s)


# ------------------------------------------------------------------------------------------------ CPU: the tolerance has teeth
def test_reference_mistakes_exceed_tolerance():
    """Each GPU test above would fail on a kernel that made one of these mistakes: the mistaken result differs from the
    reference by far more than TOL (computed here on the CPU with the same reference functions, small shapes)."""
    g = _gen(0)
    far = 100 * TOL
    # norm: a pixel lane dropped (every 16th pixel: 16 lanes at C = 64), two images swapped, the wrong group size
    x, gy, film = _norm_inputs(g, 2, 64, 64, 1, 128)
    ref = ref_norm(x, gy, 32, 1, True, film=film, ctot=64)
    lane = gy.clone(); lane[:, ::16] = 0
    swap = gy[[1, 0]]
    for bad in (ref_norm(x, lane, 32, 1, True, film=film, ctot=64), ref_norm(x, swap, 32, 1, True, film=film, ctot=64),
                ref_norm(x, gy, 16, 1, True, film=film, ctot=64)):
        assert max(_rel(bad[0], ref[0]), _rel(bad[1], ref[1])) > far
    # attention: g_out of two images swapped
    x, gout, *p = _attn_inputs(g, 3, 32)
    ref = ref_attn(x, gout, *p)
    bad = ref_attn(x, gout[[1, 0, 2]], *p)
    assert max(_rel(b_, r_) for b_, r_ in zip(bad, ref)) > far
    # sgemm: the K tail past the last full 16-slice lost
    a_mat, b_mat = torch.randn(3, 7001, generator=g), torch.randn(7001, 257, generator=g)
    assert _rel(ref_sgemm(a_mat[:, :6992], b_mat[:6992]), ref_sgemm(a_mat, b_mat)) > far
    # FiLM wgrad: only the first 64-sample chunk of a batch of 65
    dfilm, cond = torch.randn(65, 203, generator=g), torch.randn(65, 64, generator=g)
    assert _rel(ref_film_wgrad(dfilm[:64], cond[:64])[0], ref_film_wgrad(dfilm, cond)[0]) > far
    # column sums: the last row lost
    x = torch.randn(4097, 64, generator=g)
    assert _rel(ref_colsum(x[:-1]), ref_colsum(x)) > far
    # embedding: colliding rows overwritten instead of added
    act = torch.randint(0, 4, (256, 4), generator=g)
    de = torch.randn(256, 256, generator=g)
    ref = ref_embedding(de, act, 4, 64)
    last = torch.zeros(4, 64, dtype=torch.float64)
    for n in range(256):
        for t in range(4):
            last[act[n, t]] = de[n, t * 64:(t + 1) * 64].double()
    assert _rel(last, ref) > far
    # sumpool2: only the top-left pixel of each 2x2 block
    gin = torch.randn(2, 10, 14, 16, generator=g)
    assert _rel(_nhwc(_nchw(gin.double())[:, :, ::2, ::2]), ref_sumpool2(gin)) > far
    # maxpool2: the LAST maximum of a tied window instead of the first
    y = _tied_pool_input(g, 2, 8, 6, 64)
    gp = torch.randn(2, 4, 3, 64, generator=g)
    last = ref_maxpool2(y.flip(1, 2), gp.flip(1, 2)).flip(1, 2)
    assert _rel(last, ref_maxpool2(y, gp)) > far
    # LSTM cell: the incoming cell-state gradient ignored
    gates, c_in, g_h, g_c = 2 * torch.randn(3, 64, generator=g), torch.randn(3, 16, generator=g), torch.randn(3, 16, generator=g), torch.randn(3, 16, generator=g)
    assert _rel(ref_lstm(gates, c_in, g_h, None)[0], ref_lstm(gates, c_in, g_h, g_c)[0]) > far
    # heads: the actions past the last multiple of 4 dropped
    hx, g_hx, wa, ba = torch.randn(5, 32, generator=g), torch.randn(5, 32, generator=g), torch.randn(6, 32, generator=g), torch.randn(6, generator=g)
    g_l, wc, bc = torch.randn(5, 6, generator=g), torch.randn(1, 32, generator=g), torch.randn(1, generator=g)
    ref = ref_heads(hx, wa, ba, wc, bc, g_hx, g_l, None)[0]
    assert _rel(ref_heads(hx, wa[:4], ba[:4], wc, bc, g_hx, g_l[:, :4], None)[0], ref) > far
    # dsilu: silu instead of its derivative
    pre, dh = torch.randn(100, generator=g), torch.randn(100, generator=g)
    assert _rel(F.silu(pre.double()) * dh.double(), ref_dsilu(pre, dh)) > far
    # loss scale: the interval (2^(E-1), 2^E] puts an exact power of two at 2^E, which the check rejects
    e = _loss_scale_exp()
    assert not loss_scale_ok(torch.tensor([2.0 ** (e - 3), 2.0 ** -(e - 3)]), 8.0, e)
    assert loss_scale_ok(torch.tensor([2.0 ** (e - 4), 2.0 ** -(e - 4)]), 8.0, e)
