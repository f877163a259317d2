"""Parameter containers that mirror the reference's NN blocks (src/models/blocks.py).

These classes own the parameters under exactly the reference's attribute names (so `state_dict()` keys, `Agent.load`
and `utils.configure_opt`'s isinstance-based weight-decay split keep working: every weight lives in an nn.Conv2d /
nn.Linear / nn.GroupNorm).  They do NOT compute anything in PyTorch: the arithmetic of a whole network runs in the
native executor (diamond_b200/csrc), which reads these tensors through their device pointers.  Calling a container
directly raises, so an accidental eager path cannot hide behind the CUDA one.
"""
from typing import List

import torch
from torch import nn

GN_GROUP_SIZE = 32  # blocks.py:12
GN_EPS = 1e-5  # blocks.py:13
ATTN_HEAD_DIM = 8  # blocks.py:14


def conv3x3(cin: int, cout: int) -> nn.Conv2d:  # blocks.py:19
    return nn.Conv2d(cin, cout, kernel_size=3, stride=1, padding=1)


def conv1x1(cin: int, cout: int) -> nn.Conv2d:  # blocks.py:18
    return nn.Conv2d(cin, cout, kernel_size=1, stride=1, padding=0)


class _NativeOnly(nn.Module):
    def forward(self, *args, **kwargs):
        raise RuntimeError(
            f"{type(self).__name__} is a parameter container; it is executed by the native sm_90a executor of the "
            "enclosing model (InnerModel / ActorCritic), not called directly"
        )


class GroupNorm(_NativeOnly):  # blocks.py:24-31
    """Affine GroupNorm (groups of 32 channels).  Executed as: (sum, sumsq) per (image, group) from the PRODUCER's conv epilogue
    (fp64 atomics), apply + SiLU inside the consumer's operand pass (`prep_fast_kernel` mode 2); backward = `norm_bwd_pass1/2`."""

    def __init__(self, in_channels: int) -> None:
        super().__init__()
        self.norm = nn.GroupNorm(max(1, in_channels // GN_GROUP_SIZE), in_channels, eps=GN_EPS)


class AdaGroupNorm(_NativeOnly):  # blocks.py:34-45
    """GroupNorm without affine + FiLM (1 + scale, shift) from the conditioning vector.  All AdaGroupNorm.linear layers of a network are
    packed into ONE [sum 2C, cond] matrix and evaluated by a single GEMM per forward (`linear_kernel`), for every denoising step up
    front in the sampler; the apply runs in the operand pass (mode 1).  Backward: `film_wgrad_kernel` scatters the batched gradient
    back to the individual `linear.weight` / `linear.bias` slices of the flat gradient buffer."""

    def __init__(self, in_channels: int, cond_channels: int) -> None:
        super().__init__()
        self.in_channels = in_channels
        self.num_groups = max(1, in_channels // GN_GROUP_SIZE)
        self.linear = nn.Linear(cond_channels, in_channels * 2)


class SelfAttention2d(_NativeOnly):  # blocks.py:51-72
    """Multi-head self-attention over the H*W positions (head_dim 8) with a residual connection.  Executed by `attn_cluster_kernel`
    (a 4-CTA cluster per image exchanging K / V through distributed shared memory; 64 positions) and `attn_bwd_kernel`."""

    def __init__(self, in_channels: int, head_dim: int = ATTN_HEAD_DIM) -> None:
        super().__init__()
        self.n_head = max(1, in_channels // head_dim)
        assert in_channels % self.n_head == 0
        self.norm = GroupNorm(in_channels)
        self.qkv_proj = conv1x1(in_channels, in_channels * 3)
        self.out_proj = conv1x1(in_channels, in_channels)
        nn.init.zeros_(self.out_proj.weight)
        nn.init.zeros_(self.out_proj.bias)


class FourierFeatures(_NativeOnly):  # blocks.py:78-87
    """Random Fourier features of the noise level; a BUFFER (no gradient), consumed by `cond_embed_kernel`."""

    def __init__(self, cond_channels: int) -> None:
        super().__init__()
        assert cond_channels % 2 == 0
        self.register_buffer("weight", torch.randn(1, cond_channels // 2))


class Downsample(_NativeOnly):  # blocks.py:93-100
    """3x3 stride-2 conv, orthogonal init.  Executed as the stride-1 wgmma conv stored at even (y, x) (exact for k = 3, p = 1);
    backward-data through `zero_insert_prep_kernel` (the adjoint of the subsampling) + the transposed conv."""

    def __init__(self, in_channels: int) -> None:
        super().__init__()
        self.conv = nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=1)
        nn.init.orthogonal_(self.conv.weight)


class Upsample(_NativeOnly):  # blocks.py:103-110
    """Nearest-2x upsample + 3x3 conv.  The upsample is addressing inside the operand pass (no upsampled tensor exists); its adjoint
    in the backward pass is `sumpool2_kernel`."""

    def __init__(self, in_channels: int) -> None:
        super().__init__()
        self.conv = conv3x3(in_channels, in_channels)


class SmallResBlock(_NativeOnly):  # blocks.py:116-123
    """Actor-critic encoder block: skip(x) + conv3x3(silu(GroupNorm(x))); the 1x1 skip projection (when widths differ) runs split-fp16
    so that the max-pool arg-max that follows matches the reference."""

    def __init__(self, in_channels: int, out_channels: int) -> None:
        super().__init__()
        self.f = nn.Sequential(GroupNorm(in_channels), nn.SiLU(inplace=True), conv3x3(in_channels, out_channels))
        self.skip_projection = nn.Identity() if in_channels == out_channels else conv1x1(in_channels, out_channels)


class ResBlock(_NativeOnly):  # blocks.py:129-147
    """U-Net residual block.  Executed as: operand pass (AdaGN1 + SiLU [+ raw split-fp16 copy for proj]) -> conv1 -> operand pass
    (AdaGN2 + SiLU) -> conv2 whose accumulator also receives the 1x1 skip projection as extra centre-tap K slabs (or the residual in
    the epilogue when there is no projection) -> optional attention.  conv2 starts at zero like the reference (blocks.py:139)."""

    def __init__(self, in_channels: int, out_channels: int, cond_channels: int, attn: bool) -> None:
        super().__init__()
        self.proj = conv1x1(in_channels, out_channels) if in_channels != out_channels else nn.Identity()
        self.norm1 = AdaGroupNorm(in_channels, cond_channels)
        self.conv1 = conv3x3(in_channels, out_channels)
        self.norm2 = AdaGroupNorm(out_channels, cond_channels)
        self.conv2 = conv3x3(out_channels, out_channels)
        self.attn = SelfAttention2d(out_channels) if attn else nn.Identity()
        nn.init.zeros_(self.conv2.weight)


class ResBlocks(_NativeOnly):  # blocks.py:153-177
    """A level of the U-Net; in the up path every block reads cat(x, skip), which the conv consumes as TWO operand sources along K
    (no concatenated tensor is materialised)."""

    def __init__(self, list_in_channels: List[int], list_out_channels: List[int], cond_channels: int, attn: bool) -> None:
        super().__init__()
        assert len(list_in_channels) == len(list_out_channels)
        self.in_channels = list_in_channels[0]
        self.resblocks = nn.ModuleList(
            ResBlock(i, o, cond_channels, attn) for i, o in zip(list_in_channels, list_out_channels)
        )


class UNet(_NativeOnly):  # blocks.py:183-220 (constructor); forward lives in csrc/api.cu PlanBuilder::build
    """Registration order (d_blocks, u_blocks reversed, mid_blocks, downsamples, upsamples) fixes the `state_dict` key order the native
    executor indexes by (`Walker` in csrc/api.cu), so it must stay the reference's.  Pad / crop of `forward` (blocks.py:225-229,245) =
    `resize_nhwc_kernel` around the level loop."""

    def __init__(self, cond_channels: int, depths: List[int], channels: List[int], attn_depths: List[int]) -> None:
        super().__init__()
        assert len(depths) == len(channels) == len(attn_depths)
        self._num_down = len(channels) - 1
        d_blocks, u_blocks = [], []
        for i, n in enumerate(depths):
            c1, c2 = channels[max(0, i - 1)], channels[i]
            d_blocks.append(ResBlocks([c1] + [c2] * (n - 1), [c2] * n, cond_channels, attn_depths[i]))
            u_blocks.append(ResBlocks([2 * c2] * n + [c1 + c2], [c2] * n + [c1], cond_channels, attn_depths[i]))
        self.d_blocks = nn.ModuleList(d_blocks)
        self.u_blocks = nn.ModuleList(reversed(u_blocks))
        self.mid_blocks = ResBlocks([channels[-1]] * 2, [channels[-1]] * 2, cond_channels, True)
        self.downsamples = nn.ModuleList([nn.Identity()] + [Downsample(c) for c in channels[:-1]])
        self.upsamples = nn.ModuleList([nn.Identity()] + [Upsample(c) for c in reversed(channels[:-1])])
