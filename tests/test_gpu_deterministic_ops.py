"""The deterministic arms of the CUDA-core kernels (what torch.use_deterministic_algorithms selects in place of the atomics) and
the training plans' split attention backward, one entry point at a time, against float64 references.

- The split attention backward (dmd_attn_split_bwd) is BwdBuilder::attn_split's own op list run through the executors' op
  dispatch: the recomputed q | k | v and normed input, attn_core_bwd_kernel, four sgemms (two of them split-K over every token
  of the batch), two column sums and the two-pass norm backward without SiLU.  It runs at C = 128 in every mode and at every C
  in deterministic mode.
- GroupNorm sums (gn_stats_det_kernel: one 8-CTA cluster per (image, group)), column sums through per-block partials
  (colsum_part_kernel + colsum_reduce_kernel), norm backward pass 1 with one block per image, and the gathered embedding
  gradient (embedding_bwd_det_kernel).

Every kernel here is fp32 (the GroupNorm sums fp64 across threads): errors are relative L2 against float64, bounded at
TOL = 1e-5 (STATS_TOL = 1e-6 for the sums), and where the atomic arm exists it is held to the same reference.  Buffers the
kernels add to are pre-filled and only the added part is compared.  Every deterministic arm runs twice and must give the same
bytes; the second run gets workspaces, partials and assigned outputs poisoned with 0xFF and runs beside a bounded load on
another stream, so its blocks are scheduled in another order.

The tests without the gpu marker show on the CPU that a plausible mistake of these kernels (a lost token, two heads swapped,
dWqkv taken from g_qkv untransposed, a lost last partial, a skipped cluster rank) moves the result far past its bound."""
import ctypes as C
import functools
import importlib.util
import math
import os

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
gpu = pytest.mark.gpu


def _load(name):
    """A sibling test module by file (its helpers; the module is not a package)."""
    spec = importlib.util.spec_from_file_location(f"_deterministic_ops_{name}", os.path.join(HERE, name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


BO = _load("test_gpu_backward_ops")
FO = _load("test_gpu_forward_ops")
TOL, STATS_TOL = BO.TOL, FO.STATS_TOL
_rel, _acc_rel, _gen, _nchw, _nhwc = BO._rel, BO._acc_rel, BO._gen, BO._nchw, BO._nhwc


def gn_group_size(c):
    """blocks.py:12,27: num_groups = max(1, C // 32)."""
    return c // max(1, c // 32)


@functools.lru_cache(maxsize=None)
def _det():
    """test_gpu_deterministic: poisoned() (0xFF in every buffer the package allocates, beside one bounded side-stream load)
    and assert_bit_equal()."""
    return _load("test_gpu_deterministic")


def _twice(dev, run):
    """run() on a clean start, then again under test_gpu_deterministic.poisoned; the bytes must match.  Returns the first
    run's results as CPU tensors."""
    TD = _det()
    first = [t.detach().cpu().clone() for t in run()]
    with TD.poisoned(dev):
        second = [t.detach().cpu().clone() for t in run()]
    TD.assert_bit_equal("second run", first, second)
    return first


# ------------------------------------------------------------------------------------------------ references (float64)
def ref_colsum_blocks(x, blocks, lanes):
    """The fixed-order column sum as colsum_part / colsum_reduce compute it, in float64: block b's rows are
    r = (b + k * blocks) * lanes + lane; the partials are added in block order."""
    r = torch.arange(x.shape[0])
    owner = (r // lanes) % blocks
    return torch.stack([x[owner == b].double().sum(0) for b in range(blocks)])


def ref_gn_stats_ranks(x, gs, split=8):
    """GroupNorm sums of NHWC x [B][HW][C] as gn_stats_det_kernel splits them: rank r of the cluster owns pixels
    [r * ceil(HW / 8), ...); float64 [split][B][C/gs][2]."""
    hw = x.shape[1]
    per = -(-hw // split)
    return torch.stack([BO._gn_stats(x[:, min(hw, r * per):min(hw, r * per + per)], gs) for r in range(split)])


def attn_parts(x, gout, gamma, beta, wqkv, bqkv, wout):
    """The split backward's intermediates in float64: xn = GroupNorm(x) [rows][C] and g_qkv [rows][3C] (NHWC rows), from
    the same forward as oracle.torch_oracle.self_attention."""
    from oracle import torch_oracle as O

    n, h, w, c = x.shape
    xn = O.group_norm(_nchw(x.double()), gamma.double(), beta.double())
    qkv = F.conv2d(xn, wqkv.double().view(3 * c, c, 1, 1), bqkv.double()).detach().requires_grad_()
    q, k, v = qkv.view(n, c // 8 * 3, 8, h * w).transpose(2, 3).chunk(3, dim=1)
    y = (F.softmax(q @ k.transpose(-2, -1) / math.sqrt(8), dim=-1) @ v).transpose(2, 3).reshape(n, c, h, w)
    (g_qkv,) = torch.autograd.grad(F.conv2d(y, wout.double().view(c, c, 1, 1)), qkv, _nchw(gout.double()))
    return _nhwc(xn).reshape(-1, c), _nhwc(g_qkv).reshape(-1, 3 * c)


# ------------------------------------------------------------------------------------------------ split attention backward
ATTN_NAMES = ["dgamma", "dbeta", "dwqkv", "dbqkv", "dwout", "dbout"]


def _attn_inputs(g, b, L, c):
    """x, g_out NHWC [B][1][L][C] and the six parameters."""
    x = torch.randn(b, 1, L, c, generator=g) * 1.5 + 0.2
    w = lambda *s: torch.randn(*s, generator=g) / math.sqrt(s[-1])  # noqa: E731
    return (x, torch.randn(b, 1, L, c, generator=g), 1 + 0.2 * torch.randn(c, generator=g), 0.2 * torch.randn(c, generator=g),
            w(3 * c, c), 0.1 * torch.randn(3 * c, generator=g), w(c, c), 0.1 * torch.randn(c, generator=g))


def _grad_layout(shapes, g):
    """Offsets of the six gradients in a flat buffer: 16-byte aligned slices in a shuffled order, eight guard floats around
    each.  Returns (offsets, total floats, mask of the guard floats)."""
    offs, off = [0] * len(shapes), 8
    for i in torch.randperm(len(shapes), generator=g).tolist():
        offs[i] = off
        off += (math.prod(shapes[i]) + 3) // 4 * 4 + 8
    guard = torch.ones(off, dtype=torch.bool)
    for o, s in zip(offs, shapes):
        guard[o:o + math.prod(s)] = False
    return offs, off, guard


@gpu
@pytest.mark.parametrize("b", [1, 3, 133])
@pytest.mark.parametrize("L", [1, 4, 16, 25, 36, 49, 64])
@pytest.mark.parametrize("c", [32, 64, 128])
def test_attn_split_bwd(c, L, b):
    """g_x and the six parameter gradients of both arms against float64 autograd; g_out scaled by 2, inv_scale = 1/2.  The
    gradients are added to slices of a pre-filled flat buffer whose guard floats stay untouched.  B = 133 at L = 64 contracts
    dWo and dWqkv over K = 8512 tokens in 32 split-K chunks.  At C <= 64 dmd_attn_bwd is held to the same reference; at L = 1
    the softmax is constant, so the q and k rows of dWqkv and dbqkv get exactly nothing."""
    dev = BO._dev()
    from diamond_b200 import ops

    g = _gen(900 + 3 * b + L + c)
    x, gout, gamma, beta, wqkv, bqkv, wout, bout = (t.to(dev) for t in _attn_inputs(g, b, L, c))
    gs = gn_group_size(c)
    stats = BO._gn_stats(x, gs)
    ref = BO.ref_attn(x, gout, gamma, beta, wqkv, bqkv, wout, bout)
    shapes = [tuple(r.shape) for r in ref[1:]]
    offs, total, guard = _grad_layout(shapes, g)
    pre = torch.randn(total, generator=g)
    for o, r in zip(offs, ref[1:]):
        pre[o:o + r.numel()] *= float(r.std())
    pre = pre.to(dev)
    inv = torch.tensor([0.5], device=dev)

    def run(det):
        grads = pre.clone()
        gx = ops.attn_split_bwd(x, stats, gamma, beta, wqkv, bqkv, wout, 2 * gout, gs, grads, offs, inv_scale=inv, det=det)
        return gx, grads

    def errors(gx, grads):
        assert torch.equal(grads[guard.to(dev)], pre[guard.to(dev)]), "a guard float of the gradient buffer was written"
        got = [grads[o:o + math.prod(s)].view(s) for o, s in zip(offs, shapes)]
        errs = {"gx": _rel(gx, 2 * ref[0])}
        errs.update({n: _acc_rel(t, pre[o:o + t.numel()].view(t.shape), r) for n, t, o, r in zip(ATTN_NAMES, got, offs, ref[1:])})
        if L == 1:
            for t, o in zip(got[2:4], offs[2:4]):
                assert torch.equal(t[:2 * c], pre[o:o + t.numel()].view(t.shape)[:2 * c]), "q / k rows got a gradient at L = 1"
        return errs

    arms = {"det": errors(*[t.to(dev) for t in _twice(dev, lambda: run(True))]), "atomic": errors(*run(False))}
    if c <= 64:
        pg = [pre[o:o + math.prod(s)].view(s).clone() for o, s in zip(offs, shapes)]
        gx = ops.attn_bwd(x, stats, gamma, beta, wqkv, bqkv, wout, 2 * gout, gs, tuple(pg), inv_scale=inv)
        errs = {"gx": _rel(gx, 2 * ref[0])}
        errs.update({n: _acc_rel(t, pre[o:o + t.numel()].view(t.shape), r) for n, t, o, r in zip(ATTN_NAMES, pg, offs, ref[1:])})
        arms["attn_bwd"] = errs
    for arm, errs in arms.items():
        print(f"attn_split_bwd {arm} B={b} L={L} C={c}:", {k: f"{v:.2e}" for k, v in errs.items()})
        assert max(errs.values()) < TOL, (arm, errs)


# ------------------------------------------------------------------------------------------------ GroupNorm sums
GN_CASES = [(3, hw, c, gs) for hw in (1, 4, 7, 16, 49, 121, 665, 4096) for c in (16, 32, 64, 128)
            for gs in sorted({8, 16, 32, 64, c}) if gs <= c and c % gs == 0] + [(256, 4096, 64, 32)]


@gpu
@pytest.mark.parametrize("b,hw,c,gs", GN_CASES)
def test_gn_stats_det(b, hw, c, gs):
    """Both arms added onto pre-filled statistics.  Below 8 pixels some CTAs of a cluster get none; 121 and 665 pixels do not
    split evenly over 8 ranks; 256 x 4096 x 64 is the benchmarked level 0."""
    dev = BO._dev()
    from diamond_b200 import ops

    g = torch.Generator(device=dev).manual_seed(b + hw + c + gs)
    n = torch.arange(b, device=dev, dtype=torch.float32).view(b, 1, 1, 1)
    x = torch.randn(b, hw, 1, c, generator=g, device=dev) * (0.6 + torch.remainder(0.37 * n, 1.0)) + torch.sin(1.7 * n + 0.3)
    ref = BO._gn_stats(x, gs)
    pre = torch.randn(ref.shape, generator=g, device=dev, dtype=torch.float64) * ref.abs().mean()
    (det,) = _twice(dev, lambda: [ops.gn_stats(x, gs, out=pre.clone(), det=True)])
    errs = {"det": _acc_rel(det.to(dev), pre, ref), "atomic": _acc_rel(ops.gn_stats(x, gs, out=pre.clone()), pre, ref)}
    print(f"gn_stats B={b} HW={hw} C={c} gs={gs}:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) < STATS_TOL, errs


# ------------------------------------------------------------------------------------------------ column sums
COLSUM_CASES = [
    (8, 3, 1), (8, 3, 3), (8, 3, 256 * 64 * 64),
    (16, 16, 1), (16, 16, 256 * 64 * 64),
    (64, 64, 3), (64, 64, 256 * 64 * 64),
    (256, 256, 256 * 64 * 64),
    (2048, 2048, 1), (2048, 2048, 3), (2048, 2048, 4096),
    # the split attention's qkv bias: 96 / 192 / 384 columns; 256 is no multiple of C / 4 at 96 and 192 (idle lanes)
    (96, 96, 1), (96, 96, 133 * 64), (96, 93, 1 << 16),
    (192, 192, 3), (192, 192, 133 * 64), (192, 192, 1 << 17),
    (384, 384, 1), (384, 384, 133 * 64), (384, 381, 1 << 16),
]


@gpu
@pytest.mark.parametrize("c,creal,rows", COLSUM_CASES)
def test_colsum_det(c, creal, rows):
    """test_colsum's table in both arms, plus the 3C-column bias sums of the split attention; the largest row counts hit the
    592-block cap.  Columns at or above Creal stay untouched."""
    dev = BO._dev()
    from diamond_b200 import ops

    g = torch.Generator(device=dev).manual_seed(c + rows + creal)
    x = torch.randn(rows, c, generator=g, device=dev)
    ref = BO.ref_colsum(x) * 0.5
    pre1, pre2 = torch.randn(c, generator=g, device=dev), torch.randn(c, generator=g, device=dev)
    inv = torch.tensor([0.5], device=dev)

    def run(det):
        out, out2 = pre1.clone(), pre2.clone()
        ops.colsum(x, out, out2, inv, creal, det=det)
        return out, out2

    errs = {}
    for arm, (out, out2) in (("det", [t.to(dev) for t in _twice(dev, lambda: run(True))]), ("atomic", run(False))):
        errs[arm] = max(_acc_rel(out[:creal], pre1[:creal], ref[:creal]), _acc_rel(out2[:creal], pre2[:creal], ref[:creal]))
        assert torch.equal(out[creal:], pre1[creal:]) and torch.equal(out2[creal:], pre2[creal:]), arm
    print(f"colsum C={c} Creal={creal} rows={rows}:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs


@gpu
def test_colsum_det_refuses_a_short_partial_buffer():
    """One float short of dmd_colsum_partial_bytes: the library's error, and nothing is written."""
    dev = BO._dev()
    from diamond_b200 import _lib, ops

    x = torch.randn(1 << 16, 384, device=dev)
    need = _lib.lib().dmd_colsum_partial_bytes(x.shape[0], 384)
    assert need == 592 * 384 * 4
    out = torch.zeros(384, device=dev)
    with pytest.raises(RuntimeError, match="exceed the partial buffer"):
        ops.colsum(x, out, det=True, partial=torch.zeros(need - 4, dtype=torch.uint8, device=dev))
    torch.cuda.synchronize()
    assert not out.any()


# ------------------------------------------------------------------------------------------------ norm backward
NORM_CASES = [
    (1, True, 1, 64, 32, 32, False),
    (1, True, 2, 4096, 64, 32, False),
    (1, False, 5, 1024, 96, 32, True),
    (1, True, 256, 4096, 64, 32, True),
    (1, True, 256, 256, 128, 32, False),
    (1, True, 2, 64, 16, 16, False),
    (2, True, 2, 256, 128, 32, False),
    (2, True, 256, 1024, 64, 32, True),
    (2, False, 5, 64, 16, 16, True),
    (2, True, 1, 4096, 32, 32, False),
    # the small frames' deepest levels: 4 x 4, 6 x 6, 7 x 7
    (1, True, 3, 16, 64, 32, False),
    (1, True, 3, 36, 32, 32, True),
    (1, True, 133, 49, 128, 32, False),
    # the attention's own norm: mode 2 without SiLU, g_x assigned
    (2, False, 3, 64, 128, 32, False),
    (2, False, 133, 16, 128, 32, False),
    (2, False, 3, 49, 64, 32, False),
]


def _norm_run(dev, x, gy, stats, gs, mode, act, par, pre, addend, acc, det, stride, film_off, s):
    from diamond_b200 import ops

    gx = pre.clone()
    kw = dict(mode=mode, act=act, addend=addend, accumulate=acc, det=det)
    if mode == 1:
        dfilm = torch.zeros(x.shape[0], stride, device=dev)
        ops.norm_bwd(x, gy, stats, gs, gx, dfilm[:, film_off + x.shape[-1]:], dfilm[:, film_off:], stride, film=par,
                     film_off=film_off, film_ctot=x.shape[-1], **kw)
        return gx, dfilm
    sums = torch.zeros(2, x.shape[0], 128, device=dev)
    dgam, dbet = par[2].clone(), par[3].clone()
    ops.norm_bwd(x, gy, stats, gs, gx, sums[0], sums[1], 128, gamma=par[0], beta=par[1], dgamma=dgam, dbeta=dbet,
                 inv_scale=torch.tensor([1 / s], device=dev), **kw)
    return gx, dgam, dbet


@gpu
@pytest.mark.parametrize("mode,act,b,hw,c,gs,acc", NORM_CASES)
def test_norm_bwd_det(mode, act, b, hw, c, gs, acc):
    """test_norm_bwd's table and the small frames' level sizes, pass 1 in both arms; without accumulation the second run's
    g_x starts poisoned (pass 2 assigns it)."""
    dev = BO._dev()
    g = _gen(500 + 7 * b + c + hw + mode)
    film_off, stride = 24, 2 * c + 40
    x, gy, par = BO._norm_inputs(g, b, hw, c, mode, stride)
    s = 4.0 if mode == 2 else 1.0
    if mode == 1:
        ref = BO.ref_norm(x.to(dev), gy.to(dev), gs, 1, act, film=par.to(dev), film_off=film_off, ctot=c)
        par = par.to(dev)
    else:
        ref = BO.ref_norm(x.to(dev), gy.to(dev), gs, 2, act, gamma=par[0].to(dev), beta=par[1].to(dev))
        par = [t.to(dev) for t in par] + [torch.randn(c, generator=g).to(dev), torch.randn(c, generator=g).to(dev)]
    xd, gyd, stats = x.to(dev), (gy * s).to(dev), BO._gn_stats(x, gs).to(dev)
    pre = torch.randn(x.shape, generator=g).to(dev) if acc else torch.zeros(x.shape, device=dev)
    addend = torch.randn(x.shape, generator=g).to(dev) if acc else None
    run = lambda det, p=pre: _norm_run(dev, xd, gyd, stats, gs, mode, act, par, p, addend, acc, det, stride, film_off, s)  # noqa: E731
    first = [t.to(dev) for t in run(True)]
    TD = _det()
    with TD.poisoned(dev):
        second = [t.to(dev) for t in run(True, pre if acc else TD.TP.poison_(torch.empty_like(pre), 0xFF))]
    TD.assert_bit_equal("norm_bwd det second run", [t.cpu() for t in first], [t.cpu() for t in second])
    errs = {}
    for arm, out in (("det", first), ("atomic", run(False))):
        gx_ref = ref[0] * s if mode == 2 else ref[0]
        errs[arm + " gx"] = _acc_rel(out[0], pre + (addend if acc else 0), gx_ref)
        if mode == 1:
            errs[arm + " dfilm"] = _rel(out[1], ref[1])
        else:
            errs[arm + " dgamma"] = _acc_rel(out[1], par[2], ref[1])
            errs[arm + " dbeta"] = _acc_rel(out[2], par[3], ref[2])
    print(f"norm_bwd mode={mode} act={act} B={b} HW={hw} C={c} gs={gs} acc={acc}:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs


@gpu
def test_norm_bwd_det_concat_pair():
    """test_norm_bwd_concat_pair with pass 1 one block per image: two launches at channel offsets 0 and 64 of 128 share one
    FiLM row block, each writing its own columns of d scale / d shift."""
    dev = BO._dev()
    from diamond_b200 import ops

    g = _gen(78)
    b, hw, c, gs, stride = 3, 1024, 128, 32, 2 * 128 + 8
    x, gy, film = BO._norm_inputs(g, b, hw, c, 1, stride)
    gx_ref, dfilm_ref = BO.ref_norm(x.to(dev), gy.to(dev), gs, 1, True, film=film.to(dev), film_off=8, ctot=c)

    def run():
        dfilm = torch.zeros(b, stride, device=dev)
        gxs = []
        for k in range(2):
            xs, gys = x[..., 64 * k:64 * (k + 1)].contiguous(), gy[..., 64 * k:64 * (k + 1)].contiguous()
            gx = torch.empty(xs.shape, device=dev)
            ops.norm_bwd(xs.to(dev), gys.to(dev), BO._gn_stats(xs, gs).to(dev), gs, gx, dfilm[:, 8 + c + 64 * k:], dfilm[:, 8 + 64 * k:],
                         stride, mode=1, film=film.to(dev), film_off=8, film_ctot=c, c_off=64 * k, det=True)
            gxs.append(gx)
        return torch.cat(gxs, dim=-1), dfilm

    gx, dfilm = _twice(dev, run)
    errs = {"gx": _rel(gx.to(dev), gx_ref), "dfilm": _rel(dfilm.to(dev), dfilm_ref)}
    print("norm_bwd det concat pair:", errs)
    assert max(errs.values()) < TOL, errs


# ------------------------------------------------------------------------------------------------ embedding gradient
@gpu
@pytest.mark.parametrize("t", [1, 4])
@pytest.mark.parametrize("b", [3, 256])
def test_embedding_bwd_det(b, t):
    """Three table rows, so rows collide; actions below 0 and at or above num_actions are clamped by the kernels, and the
    reference clamps them the same way.  inv_scale = 1/4, added onto a pre-filled table."""
    dev = BO._dev()
    from diamond_b200 import ops

    g = _gen(40 + b + t)
    e_dim, na = 64, 3
    act = torch.randint(-3, na + 3, (b, t), generator=g)
    act.view(-1)[:4] = torch.tensor([-1, na, na + 7, -9])[:act.numel()]
    de = torch.randn(b, t * e_dim, generator=g)
    ref = BO.ref_embedding(de, act.clamp(0, na - 1), na, e_dim) * 0.25
    pre = (torch.randn(na, e_dim, generator=g) * float(ref.std())).to(dev)
    inv = torch.tensor([0.25], device=dev)
    run = lambda det: [ops.embedding_bwd(de.to(dev), act.to(dev), pre.clone(), inv, det=det)]  # noqa: E731
    (det,) = _twice(dev, lambda: run(True))
    errs = {"det": _acc_rel(det.to(dev), pre, ref.to(dev)), "atomic": _acc_rel(run(False)[0], pre, ref.to(dev))}
    print(f"embedding_bwd B={b} T={t}:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs


# ------------------------------------------------------------------------------------------------ CPU
def test_entry_points_refuse_bad_arguments():
    """The argument checks run before any CUDA call: the split attention backward's shapes and workspace, and the
    deterministic GroupNorm sums' four channels per load (C or gs not a multiple of 4 is refused, not summed wrongly).  The
    partial-size query is the column-sum launcher's block count (at most 592) times C."""
    from diamond_b200 import _lib

    lib = _lib.lib()
    assert lib.dmd_colsum_partial_bytes(1, 96) == 96 * 4
    assert lib.dmd_colsum_partial_bytes(133 * 64, 384) == 266 * 384 * 4      # 4 row lanes of 8 rows per block
    assert lib.dmd_colsum_partial_bytes(1 << 20, 64) == 592 * 64 * 4
    assert lib.dmd_attn_split_bwd_workspace_bytes(133, 64, 128) >= 3 * 6 * 133 * 64 * 128 * 4
    p = 256
    offs = (C.c_longlong * 6)(*range(6))
    for L, c, gs, msg in [(65, 128, 32, "unsupported shape"), (64, 96, 32, "unsupported shape"), (0, 64, 32, "unsupported shape"),
                          (16, 128, 12, "bad group size"), (16, 128, 8, "bad group size")]:
        rc = lib.dmd_attn_split_bwd(*[p] * 10, offs, None, 3, L, c, gs, 1, p, 1 << 30, None)
        assert rc == 1 and msg in lib.dmd_last_error().decode(), (L, c, gs, lib.dmd_last_error())
    rc = lib.dmd_attn_split_bwd(*[p] * 10, offs, None, 3, 16, 64, 32, 0, p, 4096, None)
    assert rc == 1 and "workspace too small" in lib.dmd_last_error().decode()
    for c, gs in [(12, 6), (6, 6)]:
        assert lib.dmd_gn_stats_det(p, p, 2, 16, c, gs, None) == 1 and "multiples of 4" in lib.dmd_last_error().decode()


def test_reference_mistakes_exceed_tolerance():
    """Each GPU test above would fail on a kernel that made one of these mistakes: the mistaken result differs from the
    reference by far more than its bound (computed here on the CPU with the same references, small shapes)."""
    g = _gen(1)
    far = 100 * TOL
    # split attention: the float64 intermediates reproduce autograd's dWqkv = g_qkv^T xn
    b, L, c = 3, 64, 32
    x, gout, gamma, beta, wqkv, bqkv, wout, bout = _attn_inputs(g, b, L, c)
    ref = BO.ref_attn(x, gout, gamma, beta, wqkv, bqkv, wout, bout)
    xn, g_qkv = attn_parts(x, gout, gamma, beta, wqkv, bqkv, wout)
    assert _rel(g_qkv.t() @ xn, ref[3]) < 1e-12
    # a lost token: the last token left out of every sum
    lost = BO.ref_attn(x[:, :, :-1].contiguous(), gout[:, :, :-1].contiguous(), gamma, beta, wqkv, bqkv, wout, bout)
    assert min(_rel(a, r) for a, r in zip(lost[1:], ref[1:])) > far
    # two heads swapped: head 0's q gradient rows written as head 1's and back
    swap = ref[3].clone()
    swap[0:8], swap[8:16] = ref[3][8:16], ref[3][0:8]
    assert _rel(swap, ref[3]) > far
    # dWqkv from g_qkv read untransposed (the dWqkv sgemm's sam and sak swapped): A(i, k) = g_qkv.flat[i * 3C + k]
    rows = b * L
    untransposed = g_qkv.reshape(-1).as_strided((3 * c, rows), (3 * c, 1)) @ xn
    assert _rel(untransposed, ref[3]) > far
    # column sums: the fixed-order reduction losing its last partial (592 blocks of 4 row lanes at 384 columns)
    xs = torch.randn(1 << 16, 384, generator=g)
    parts = ref_colsum_blocks(xs, 592, 4)
    assert _rel(parts.sum(0), BO.ref_colsum(xs)) < 1e-12
    assert _rel(parts[:-1].sum(0), BO.ref_colsum(xs)) > far
    # GroupNorm sums: rank 0 skipping the last cluster rank, at 16 and 665 pixels (ranks of 2 and 84 pixels)
    for hw in (16, 665):
        xg = torch.randn(3, hw, 64, generator=g) + 0.5
        ranks = ref_gn_stats_ranks(xg, 32)
        assert _rel(ranks.sum(0), BO._gn_stats(xg, 32)) < 1e-12
        assert _rel(ranks[:-1].sum(0), BO._gn_stats(xg, 32)) > 100 * STATS_TOL
