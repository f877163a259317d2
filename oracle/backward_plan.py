"""Test infrastructure (CPU): the ALGORITHMS the round-2 backward kernels will implement, restated on the data layouts the
forward kernels already use and checked against torch autograd (tests/test_backward_plan.py).  Nothing here is product
code; it pins the formulations (indexing, boundary handling, reduction structure) before they are written in CUDA.

Layouts (diamond_b200/csrc/conv_tc.cuh): the padded-linear position q = (n*(H+1) + y)*(W+1) + x with a shared zero column
x == W and zero row y == H, so that tap (dy, dx) of a 3x3 window is position q + dy*(W+1) + dx.
"""
import torch
import torch.nn.functional as F
from torch import Tensor


def to_padded_linear(x: Tensor) -> Tensor:
    """NCHW [B, C, H, W] -> [G + Q + G, C] on the padded line (zeros at pad / guard positions), G = W + 2 guard rows."""
    b, c, h, w = x.shape
    pw, ph = w + 1, h + 1
    line = torch.zeros(b, ph, pw, c, dtype=x.dtype)
    line[:, :h, :w] = x.permute(0, 2, 3, 1)
    g = pw + 1
    out = torch.zeros(g + b * ph * pw + g, c, dtype=x.dtype)
    out[g:g + b * ph * pw] = line.reshape(-1, c)
    return out


def wgrad_over_positions(x: Tensor, gy: Tensor) -> Tensor:
    """Weight gradient of a 3x3 / stride-1 / pad-1 conv as nine GEMMs with K = positions (blocks.py:18 backward):
        gw[co, ci, dy+1, dx+1] = sum_q  GY[q, co] * X[q + dy*(W+1) + dx, ci]
    over ALL positions q of the padded line.  No boundary tests: out-of-image taps read the shared zero pads, and GY is zero
    at pad positions because its operand is written by the same prep kernel.  This is the wgmma formulation: both operands
    are the PLC16 planes the forward already uses, read as MN-major (K = position) tiles."""
    b, c, h, w = x.shape
    pw = w + 1
    g = pw + 1
    X, GY = to_padded_linear(x), to_padded_linear(gy)
    q = b * (h + 1) * pw
    gw = torch.zeros(gy.shape[1], c, 3, 3, dtype=x.dtype)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            s = dy * pw + dx
            gw[:, :, dy + 1, dx + 1] = GY[g:g + q].t() @ X[g + s:g + s + q]
    return gw


def dgrad_as_forward_conv(gy: Tensor, w: Tensor) -> Tensor:
    """Backward-data of the same conv = the forward implicit GEMM on gy with weights transposed and taps flipped
    (verified on the wgmma kernel itself in tests/test_gpu_conv.py)."""
    return F.conv2d(gy, w.transpose(0, 1).flip(2, 3), padding=1)


def adagn_silu_backward_two_pass(x: Tensor, scale: Tensor, shift: Tensor, gz: Tensor, group_size: int = 32, eps: float = 1e-5):
    """Backward of z = silu((1 + scale[n,c]) * groupnorm(x) + shift[n,c])  (blocks.py:41-45, :143-144) as the two passes a
    fused kernel pair makes over the data, NHWC-friendly (all reductions are per (n, c) over pixels first):

      pass 1 (one read of x and gz):  gyv = gz * silu'(y);   A[n,c] = sum_hw gyv;   Bm[n,c] = sum_hw gyv * xhat
              -> g_shift = A,  g_scale = Bm          (FiLM gradients, blocks.py:39)
              -> per group:  m1 = sum_c (1+scale) A / cnt,   m2 = sum_c (1+scale) Bm / cnt
      pass 2 (second read):  gx = rstd * ((1+scale) * gyv - m1 - xhat * m2)

    The forward statistics (mean, rstd per (n, group)) are the ones the forward epilogue already produced.
    Returns (gx, g_scale, g_shift)."""
    b, c, h, w = x.shape
    ng = max(1, c // group_size)
    xg = x.reshape(b, ng, -1)
    mean = xg.mean(dim=2, keepdim=True)
    var = xg.var(dim=2, unbiased=False, keepdim=True)
    rstd = (var + eps).rsqrt()
    xhat = ((xg - mean) * rstd).reshape(b, c, h, w)
    k = (1 + scale)[:, :, None, None]
    y = k * xhat + shift[:, :, None, None]
    sig = torch.sigmoid(y)
    gyv = gz * (sig * (1 + y * (1 - sig)))                       # silu'(y)
    A = gyv.sum(dim=(2, 3))                                       # pass 1
    Bm = (gyv * xhat).sum(dim=(2, 3))
    cnt = (c // ng) * h * w
    kk = 1 + scale
    m1 = (kk * A).reshape(b, ng, -1).sum(dim=2) / cnt
    m2 = (kk * Bm).reshape(b, ng, -1).sum(dim=2) / cnt
    m1c = m1.repeat_interleave(c // ng, dim=1)[:, :, None, None]
    m2c = m2.repeat_interleave(c // ng, dim=1)[:, :, None, None]
    rstd_c = rstd.reshape(b, ng).repeat_interleave(c // ng, dim=1)[:, :, None, None]
    gx = rstd_c * (k * gyv - m1c - xhat * m2c)                    # pass 2
    return gx, Bm, A
