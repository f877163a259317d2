"""Records tests/golden/uint8_segments.npz: uint8 segments built by the reference's own make_segment /
collate_segments_to_batch (src/data/utils.py:12-41) from a uint8 episode, left- and right-padded.  Needs the reference
tree (DIAMOND_REFERENCE_SRC=<reference>/src); tests/test_uint8_frames_host.py reads only the fixture.

    DIAMOND_REFERENCE_SRC=... python scripts/make_uint8_segment_fixture.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402


def main():
    ref = ref_import.load()
    from data.episode import Episode
    from data.segment import SegmentId
    from data.utils import collate_segments_to_batch, make_segment

    rng = np.random.default_rng(0)
    n = 7
    obs = torch.from_numpy(rng.integers(1, 256, size=(n, 3, 8, 8), dtype=np.uint8))   # no zero byte in the real frames
    ep = Episode(obs, torch.arange(n), torch.zeros(n), torch.zeros(n, dtype=torch.uint8), torch.zeros(n, dtype=torch.uint8), {})
    ids = [(-3, 2), (0, 5), (4, 9), (-1, 4)]   # five frames each: left-padded, inside, right-padded
    batch = collate_segments_to_batch([make_segment(ep, SegmentId(0, a, b)) for a, b in ids])
    assert batch.obs.dtype == torch.uint8
    out = os.path.join(ROOT, "tests", "golden", "uint8_segments.npz")
    np.savez_compressed(out, episode=obs.numpy(), starts=np.array([a for a, _ in ids]), stops=np.array([b for _, b in ids]),
                        obs=batch.obs.numpy(), mask_padding=batch.mask_padding.numpy())
    del ref
    print("wrote", out)


if __name__ == "__main__":
    main()
