"""CPU: the oracle restatement and the mirror's host-side pieces against what the unmodified reference computed on the same
seeded inputs (tests/golden/reference_records.npz, recorded by oracle/make_reference_records.py)."""
import os

import numpy as np
import torch

from oracle import make_reference_records as R
from oracle import torch_oracle as O


def _records(golden_dir):
    return np.load(os.path.join(golden_dir, "reference_records.npz"))


def test_blocks_and_denoise_match_reference(golden_dir):
    torch.set_num_threads(8)
    rec = _records(golden_dir)
    inner = O.InnerCfg(**R.DENOISE_INNER)
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), 31337)
    obs, act, x = O.synthetic_inputs(3, inner, 32, 32, 9)
    sig = torch.tensor([0.01, 0.5, 7.0])
    cfg = O.DenoiserCfg(inner=inner)
    with torch.no_grad():
        want = torch.from_numpy(rec["denoise"])
        got = O.denoise(x, sig, obs.reshape(3, 12, 32, 32), act, sd, cfg)
        want_mo = torch.from_numpy(rec["model_output"])
        got_mo = O.model_output(x, sig, obs.reshape(3, 12, 32, 32), act, sd, cfg)
    assert torch.allclose(got_mo, want_mo, rtol=1e-5, atol=1e-5)
    assert float((got != want).float().mean()) < 1e-3


def test_denoiser_host_side_edm_pieces_match_the_reference(golden_dir):
    """The torch-level pieces of diamond_b200's Denoiser that the TRAINING forward uses on the host side (noise-level draw,
    apply_noise, conditioners, wrap + truncating quantiser) against the unmodified reference on the same RNG stream: bit-equal."""
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig

    rec = _records(golden_dir)
    mine = Denoiser(DenoiserConfig(InnerModelConfig(*R.EDM_INNER), 0.5, 0.3))
    got = R.edm_pieces(mine, SigmaDistributionConfig, R.edm_x())
    assert sorted("edm_" + k for k in got) == sorted(k for k in rec.files if k.startswith("edm_"))
    for k, v in got.items():
        want = torch.from_numpy(rec["edm_" + k])
        assert v.shape == want.shape and v.dtype == want.dtype and torch.equal(v, want), k
