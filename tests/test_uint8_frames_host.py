"""CPU: the uint8 frame format (diamond_b200/frames.py) and the argument checks of the `_u8` C entry points."""
import ctypes

import numpy as np
import pytest
import torch

from diamond_b200 import _lib
from diamond_b200 import frames as F

U = torch.arange(256, dtype=torch.uint8)


def test_cpu_row_is_episode_load():
    t = F.decode_table("cpu")
    # Episode.load (src/data/episode.py:39) on the CPU, written out
    assert torch.equal(t[F.KIND_CPU], U.div(255).mul(2).sub(1))
    assert torch.equal(t[F.KIND_PADDING], torch.zeros(256))


def test_round_to_nearest_inverts_every_row_and_truncation_does_not():
    t = F.decode_table("cpu")
    for k in (F.KIND_CPU, F.KIND_GPU):
        levels, kinds = F.encode(t[k].view(1, 1, 256))
        assert torch.equal(levels.view(-1), U)
        assert torch.equal(F.decode(levels, kinds, t), t[k].view(1, 1, 256))
    # the reference's Episode.save: add(1).div(2).mul(255).byte() truncates
    trunc = t[F.KIND_CPU].add(1).div(2).mul(255).byte()
    assert int((trunc != U).sum()) == 63
    # fp32 arithmetic of the GPU-row form u * fl(1/255), checked in numpy: differs from u / 255 on 111 levels
    u = np.arange(256, dtype=np.float32)
    gpu_like = (u * np.float32(1 / 255)) * np.float32(2) - np.float32(1)
    assert int((gpu_like != (u / np.float32(255)) * np.float32(2) - np.float32(1)).sum()) == 111


def test_off_grid_frames_raise():
    t = F.decode_table("cpu")
    f = t[F.KIND_CPU][U.long()].view(1, 1, 256).clone()
    f[0, 0, 7] += 1e-3
    with pytest.raises(ValueError, match="not decoded levels"):
        F.encode(f)
    with pytest.raises(ValueError):
        F.encode(torch.zeros(1, 2, 2))   # 0.0 (padding) is not a level


def test_decode_reads_out_of_range_kinds_as_padding():
    levels = torch.full((2, 1, 2, 2), 200, dtype=torch.uint8)
    kinds = torch.tensor([1, 9], dtype=torch.uint8)
    out = F.decode(levels, kinds)
    assert torch.equal(out[1], torch.zeros(1, 2, 2)) and bool((out[0] != 0).all())


def test_reference_make_segment_pads_exactly_where_mask_is_false(golden_dir):
    g = np.load(f"{golden_dir}/uint8_segments.npz")
    obs, mask, ep = g["obs"], g["mask_padding"], g["episode"]
    assert obs.dtype == np.uint8
    assert (obs[~mask] == 0).all()                       # F.pad pads the bytes with 0 ...
    assert (obs[mask] != 0).all()                        # ... and the fixture's real frames hold no zero byte
    for i, (a, b) in enumerate(zip(g["starts"], g["stops"])):
        real = obs[i][mask[i]]
        assert np.array_equal(real, ep[max(0, a):min(len(ep), b)])
    kinds = F.kinds_from_mask(torch.from_numpy(mask), mask.shape, "cpu")
    dec = F.decode(torch.from_numpy(obs), kinds)
    assert bool((dec[torch.from_numpy(~mask)] == 0).all())


def _frames(**over):
    s = _lib.U8Frames()
    s.levels, s.batch_stride, s.frame_stride = 4096, 0, 0
    s.kinds, s.kind_batch_stride, s.kind_frame_stride = 4096, 0, 0
    s.table = 4096
    for k, v in over.items():
        setattr(s, k, v)
    return s


# every check runs before the handle is used or anything is launched: dummy non-NULL pointers suffice
BAD_FRAMES = [({"levels": None}, "obs->levels is NULL"), ({"kinds": None}, "obs->kinds is NULL"),
              ({"table": None}, "obs->table is NULL"), ({"table": 4098}, "obs->table is not 4-byte aligned"),
              ({"frame_stride": -1}, "batch_stride / frame_stride must be >= 0"),
              ({"kind_batch_stride": -1}, "kind_batch_stride / kind_frame_stride must be >= 0")]


@pytest.mark.parametrize("name", ["dmd_inner_model_forward_u8", "dmd_inner_model_forward_train_u8"])
def test_inner_model_u8_rejects_bad_arguments(name):
    lib = _lib.lib()
    fn = getattr(lib, name)
    p = 4096

    def call(h=p, noisy=p, cn=p, obs=None, act=p, out=p, frames=True):
        f = ctypes.byref(_frames(**(obs or {}))) if frames else None
        return fn(h, 2, 64, 64, noisy, cn, 0, f, act, out, p, 1 << 20, None)
    for kw, msg in [({"h": None}, "handle is NULL"), ({"noisy": None}, "noisy_rescaled is NULL"), ({"cn": None}, "c_noise is NULL"),
                    ({"act": None}, "act is NULL"), ({"out": None}, "out is NULL"), ({"frames": False}, "obs is NULL")]:
        assert call(**kw) == 1 and msg in lib.dmd_last_error().decode(), msg
    for over, msg in BAD_FRAMES:
        assert call(obs=over) == 1 and msg in lib.dmd_last_error().decode(), msg


@pytest.mark.parametrize("name", ["dmd_rew_end_predict_u8", "dmd_rew_end_forward_train_u8"])
def test_rew_end_u8_rejects_bad_arguments(name):
    lib = _lib.lib()
    fn = getattr(lib, name)
    p = 4096

    def call(h=p, b=2, t=3, obs=None, nxt=None, act=p, lr=p, hxo=p, ws=p, frames=True):
        o = ctypes.byref(_frames(**(obs or {}))) if frames else None
        n = ctypes.byref(_frames(**(nxt or {})))
        return fn(h, b, t, o, n, act, None, None, lr, p, hxo, p, ws, 1 << 20, None)
    for kw, msg in [({"h": None}, "handle is NULL"), ({"b": 0}, "bad shape"), ({"act": None}, "act is NULL"),
                    ({"lr": None}, "logits_rew / logits_end is NULL"), ({"hxo": None}, "hx_out / cx_out is NULL"),
                    ({"ws": None}, "workspace is NULL"), ({"frames": False}, "obs is NULL"),
                    ({"nxt": {"table": 8192}}, "obs->table and next_obs->table differ")]:
        assert call(**kw) == 1 and msg in lib.dmd_last_error().decode(), msg
    for over, msg in BAD_FRAMES:
        assert call(obs=over) == 1 and msg in lib.dmd_last_error().decode(), msg
        assert call(nxt=over) == 1 and msg.replace("obs", "next_obs") in lib.dmd_last_error().decode(), msg


def test_u8_frames_struct_matches_header_layout():
    assert ctypes.sizeof(_lib.U8Frames) == 7 * 8
