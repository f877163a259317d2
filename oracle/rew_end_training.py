"""Reward / termination model training (RewEndModel.forward, rew_end_model.py:57-90): the loss restated over
torch_oracle.predict_rew_end, a chunked variant for the trainer's batch, and the generator of tests/golden/rew_end_training.npz,
which runs the UNMODIFIED reference where its source tree is available:

    DIAMOND_REFERENCE_SRC=<reference checkout>/src python oracle/rew_end_training.py
"""
import os
import sys
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import torch_oracle as O  # noqa: E402

SD = Dict[str, Tensor]
GOLDEN = os.path.join(ROOT, "tests", "golden", "rew_end_training.npz")


def rew_end_loss(obs: Tensor, act: Tensor, rew: Tensor, end: Tensor, mask_padding: Tensor, final_obs: Dict[int, Tensor], sd: SD,
                 cfg: O.RewEndCfg):
    """RewEndModel.forward (rew_end_model.py:57-90) over predict_rew_end.  obs [b, T, c, h, w], act / rew / end / mask_padding
    [b, T]; final_obs[i]: the `final_observation` of segment i, which must be given for every segment whose `end` is set.  The
    frame after a segment's termination is replaced by its final observation in a copy of obs (the reference writes through
    the view into batch.obs).  Returns (loss, loss_rew, loss_end, logits_rew [b, T-1, 3], logits_end [b, T-1, 2], that copy)."""
    obs = obs.clone()
    o, a, nxt = obs[:, :-1], act[:, :-1], obs[:, 1:]
    r, e, m = rew[:, :-1], end[:, :-1], mask_padding[:, :-1]
    dead = e.bool().any(dim=1)
    if dead.any():
        fo = torch.stack([final_obs[i] for i in range(dead.numel()) if dead[i]]).to(obs.dtype)
        nxt[dead, e[dead].argmax(dim=1)] = fo
    lr, le, _ = O.predict_rew_end(o, a, nxt, sd, cfg)
    loss_rew = F.cross_entropy(lr[m], r[m].sign().long().add(1))
    loss_end = F.cross_entropy(le[m], e[m])
    return loss_rew + loss_end, loss_rew, loss_end, lr, le, obs


def rew_end_loss_grads_chunked(obs: Tensor, act: Tensor, rew: Tensor, end: Tensor, mask_padding: Tensor, final_obs: Dict[int, Tensor],
                               sd: SD, cfg: O.RewEndCfg, chunk: int):
    """rew_end_loss and its gradient wrt the parameters that require grad, accumulated over groups of `chunk` segments so that
    one group's autograd graph is alive at a time.  The LSTM couples only the rows of one segment and both cross-entropies are
    means over the masked rows of the WHOLE batch, so a group's loss enters weighted by its share of those rows: exact up to
    summation order.  Returns (loss, {name: grad})."""
    m = mask_padding[:, :-1]
    total = int(m.sum())
    leaves = {k: v for k, v in sd.items() if v.requires_grad}
    grads = {k: torch.zeros_like(v) for k, v in leaves.items()}
    loss = 0.0
    for s in range(0, obs.size(0), chunk):
        sl = slice(s, s + chunk)
        share = int(m[sl].sum()) / total
        if share == 0:
            continue
        fo = {i - s: f for i, f in final_obs.items() if s <= i < s + chunk}
        part = rew_end_loss(obs[sl], act[sl], rew[sl], end[sl], mask_padding[sl], fo, sd, cfg)[0] * share
        for k, g in zip(leaves, torch.autograd.grad(part, list(leaves.values()), allow_unused=True)):
            if g is not None:
                grads[k] += g
        loss += part.item()
    return loss, grads



def frames(u8) -> Tensor:
    """uint8 frames -> the float32 values on the 1/255 grid in [-1, 1] that the reference sees (episode.py:36-43)."""
    return torch.from_numpy(np.asarray(u8).astype(np.float32)).div(255).mul(2).sub(1)


def to_u8(x: Tensor) -> np.ndarray:
    """The inverse of frames() for values on its grid (exact)."""
    u = x.add(1).div(2).mul(255).round()
    assert torch.equal(frames(u.numpy().astype(np.uint8)), x), "frames are not on the 1/255 grid"
    return u.numpy().astype(np.uint8)


def golden_inputs():
    """The fixture's batch: 4 segments of seq_length 7 (6 transitions) at the default config.  Segment 1 dies at step 3 and
    carries info["final_observation"]; its later frames are padding (mask off).  Segment 2 runs past the
    end of its episode without dying (padding from step 5 on, can_sample_beyond_end).  Rewards of every sign, some above 1."""
    cfg = O.RewEndCfg()
    rng = np.random.default_rng(96)
    b, T = 4, 7
    obs_u8 = rng.integers(0, 256, size=(b, T, cfg.img_channels, cfg.img_size, cfg.img_size), dtype=np.uint8)
    act = torch.from_numpy(rng.integers(0, cfg.num_actions, size=(b, T)).astype(np.int64))
    rew = torch.from_numpy(rng.choice([-3.0, -1.0, 0.0, 0.0, 0.5, 1.0, 2.5], size=(b, T)).astype(np.float32))
    end = torch.zeros(b, T, dtype=torch.long)
    mask = torch.ones(b, T, dtype=torch.bool)
    end[1, 3] = 1
    for i, t0 in ((1, 4), (2, 5)):   # padding: a uniform frame (uint8 127, next to the gray 0.0, stays on the 1/255 grid)
        mask[i, t0:] = False
        obs_u8[i, t0:] = 127
        rew[i, t0:] = 0
        act[i, t0:] = 0
    obs = frames(obs_u8)
    final_obs = {1: frames(rng.integers(0, 256, size=(cfg.img_channels, cfg.img_size, cfg.img_size), dtype=np.uint8))}
    return obs, act, rew, end, mask, final_obs


def make_rew_end_training():
    """Reference RewEndModel.forward (loss, rew_end_model.py:57-90) + backward on seeded weights and golden_inputs()."""
    from oracle import ref_import

    ns = ref_import.load()
    R = ns.rew_end_model
    cfg = O.RewEndCfg()
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), 778)
    m = R.RewEndModel(R.RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths),
                                          list(cfg.channels), list(cfg.attn_depths), cfg.num_actions))
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == O.rew_end_shapes(cfg)
    m.load_state_dict(sd)
    obs, act, rew, end, mask, final_obs = golden_inputs()
    b = obs.size(0)
    info = [{"final_observation": final_obs[i]} if i in final_obs else {} for i in range(b)]
    batch = ns.data.Batch(obs=obs.clone(), act=act, rew=rew, end=end, trunc=torch.zeros_like(end), mask_padding=mask, info=info,
                          segment_ids=[None] * b)
    loss, metrics = m(batch)
    loss.backward()
    with torch.no_grad():   # the logits forward() computed, from the substituted frames
        lr, le, _ = m.predict_rew_end(batch.obs[:, :-1], act[:, :-1], batch.obs[:, 1:])
    grads = [(k, p.grad) for k, p in m.named_parameters()]
    assert all(g is not None for _, g in grads)
    keys, norms, samples = O.grad_summary(grads)
    np.savez_compressed(GOLDEN, weights_checksum=np.float64(O.state_checksum(sd)), obs_u8=to_u8(obs), act=act.numpy(), rew=rew.numpy(),
                        end=end.numpy(), mask_padding=mask.numpy(), final_obs_u8=to_u8(final_obs[1]), final_obs_segment=np.int64(1),
                        obs_substituted_u8=to_u8(batch.obs), logits_rew=lr.numpy(), logits_end=le.numpy(),
                        loss_rew=np.float64(metrics["loss_rew"].item()), loss_end=np.float64(metrics["loss_end"].item()),
                        loss=np.float64(loss.item()), grad_keys=np.array(keys), grad_norms=norms, grad_samples=samples)
    print("rew_end_training loss", loss.item(), "grad norm", float(np.sqrt((norms ** 2).sum())), "size", os.path.getsize(GOLDEN))


def load_golden():
    """The fixture's inputs as tensors (obs before substitution, act, rew, end, mask_padding, final_obs {segment: frame}) and
    the raw npz."""
    g = np.load(GOLDEN)
    final_obs = {int(g["final_obs_segment"]): frames(g["final_obs_u8"])}
    return (frames(g["obs_u8"]), torch.from_numpy(g["act"]), torch.from_numpy(g["rew"]), torch.from_numpy(g["end"]),
            torch.from_numpy(g["mask_padding"]), final_obs), g


if __name__ == "__main__":
    make_rew_end_training()
