"""Mutual nearest-neighbour matching of keypoints for engine outputs (demo_guided_matching.py:48-62), on the device.

The demo takes the predictions of the zoom-in engines in both directions, finds for every prediction the nearest
keypoint of the other image (scipy.spatial.distance_matrix + np.argmin, fp64) and keeps the pairs that choose each other
with a Python double loop.  `mutual_nearest` gives the same result from one cotr_mutual_nearest call, without the
K_a x K_b distance matrices.  COTR.match_keypoints does the whole step, decode included, for an image set.
"""
import numpy as np
import torch

from .. import capi


def mutual_nearest(corrs_a_b, kp_b, corrs_b_a, kp_a, device="cuda"):
    """corrs_a_b: (K_a,2) predicted pixels in b of a's keypoints (an engine's corrs[:, 2:]), kp_b: (K_b,2) b's keypoints,
    corrs_b_a / kp_a the other direction -> the demo's final_matches as an (M,2) int64 array of (index into kp_a, index
    into kp_b), in ascending first index.  Ties and NaNs are decided as np.argmin decides them; an image without
    keypoints gives no matches (the demo raises there)."""
    corrs_a_b, kp_b, corrs_b_a, kp_a = (np.asarray(x, dtype=np.float64).reshape(-1, 2) for x in (corrs_a_b, kp_b, corrs_b_a, kp_a))
    assert corrs_a_b.shape[0] == kp_a.shape[0] and corrs_b_a.shape[0] == kp_b.shape[0], \
        "one prediction per keypoint: corrs_a_b must have len(kp_a) rows and corrs_b_a len(kp_b) rows"
    dev = torch.device(device)
    kpts = torch.from_numpy(np.concatenate([kp_a, kp_b])).to(dev)
    corr = torch.from_numpy(np.concatenate([corrs_a_b, corrs_b_a])).to(dev)
    _, match, count = capi.mutual_nearest(kpts, [0, kp_a.shape[0], kp_a.shape[0] + kp_b.shape[0]], [(0, 1)], corr)
    return match[:int(count.cpu()[0])].cpu().numpy().astype(np.int64)
