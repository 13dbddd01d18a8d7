"""CPU: the keypoint-matching oracle (oracle/match_oracle.py) against what demo_guided_matching.py runs - scipy's
distance_matrix + np.argmin and the demo's double loop - and its pixel / query formulas against RefinementTask with a
whole-image patch."""
import os
import types
import warnings

import numpy as np
import pytest
from scipy.spatial import distance_matrix

from oracle import match_oracle as mo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DISK_A = "disk_kpts_21526113_4379776807.npy"      # image 1033 x 771
DISK_B = "disk_kpts_21126421_4537535153.npy"      # image 694 x 1061


def scipy_nearest(corr, kp):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # deprecation warnings of distance_matrix on some scipy versions
        return np.argmin(distance_matrix(corr, kp), axis=1)


def demo_loop(inds_a_b, inds_b_a):
    """demo_guided_matching.py:49-61, literally."""
    matched_a_b = np.stack([np.arange(len(inds_a_b)), inds_a_b]).T
    matched_b_a = np.stack([np.arange(len(inds_b_a)), inds_b_a]).T
    final_matches = []
    for m_ab in matched_a_b:
        for m_ba in matched_b_a:
            if (m_ab == m_ba[::-1]).all():
                final_matches.append(m_ab)
                break
    return np.array(final_matches).reshape(-1, 2)


def disk(name):
    return np.load(os.path.join(GOLDEN, name))


def cases():
    rs = np.random.RandomState(0)
    out = {}
    out["random"] = (rs.uniform(0, 800, (300, 2)), rs.uniform(0, 800, (257, 2)))
    out["large_coords"] = (rs.uniform(-1e5, 1e5, (200, 2)), rs.uniform(-1e5, 1e5, (150, 2)))
    out["tie_grid"] = mo.tie_grid(12, seed=1)
    kp = rs.randint(0, 20, (100, 2)).astype(np.float64)
    out["duplicates"] = (rs.randint(0, 20, (120, 2)).astype(np.float64), np.concatenate([kp, kp[::-1], kp[:7]]))
    out["sqrt_collisions"] = mo.sqrt_collisions(64, seed=2)
    c, k = rs.uniform(0, 100, (50, 2)), rs.uniform(0, 100, (60, 2))
    c[7, 1] = np.nan
    out["nan_point"] = (c, k)
    k = k.copy()
    k[33, 0] = np.nan
    out["nan_keypoint"] = (c[:, ::-1].copy(), k)
    a, b = disk(DISK_A).astype(np.float64), disk(DISK_B).astype(np.float64)
    out["disk"] = (a * [694 / 1033, 1061 / 771] + rs.normal(0, 2.0, a.shape), b)
    return out


@pytest.mark.parametrize("name", list(cases()))
def test_nearest_is_scipy_argmin(name):
    corr, kp = cases()[name]
    got = mo.nearest(corr, kp, rows_per_block=37)
    ref = scipy_nearest(corr, kp)
    assert np.array_equal(got, ref)
    if name == "sqrt_collisions":
        n = corr.shape[0]
        assert np.array_equal(got, np.arange(n))                   # the larger squared distance at the lower index
        assert not np.array_equal(np.argmin(((kp[None] - corr[:, None]) ** 2).sum(-1), axis=1), got)
    if name == "nan_keypoint":
        assert got[7] == 0 and (np.delete(got, 7) == 33).all()     # row 7 is a NaN point as well
    if name == "nan_point":
        assert got[7] == 0


def test_sqrt_collisions_in_lanes_layout():
    """The same-lane collision data of the device test: far and near keypoint of a pair in one lane (index mod 4), in
    one staged chunk of 1024 or in consecutive ones, and np.argmin picks the far (lower-index, larger d^2) one."""
    corr, kp, far, near = mo.sqrt_collisions_in_lanes(100, 100, seed=9)
    assert ((near - far) % 4 == 0).all() and (near > far).all()
    assert ((far[:100] // 1024) == (near[:100] // 1024)).all() and ((near[100:] // 1024) == far[100:] // 1024 + 1).all()
    got = mo.nearest(corr, kp)
    assert np.array_equal(got, far) and np.array_equal(got, scipy_nearest(corr, kp))


def test_nearest_without_keypoints():
    assert np.array_equal(mo.nearest(np.zeros((3, 2)), np.zeros((0, 2))), [-1, -1, -1])
    assert mo.mutual(np.array([-1, -1]), np.zeros(0, np.int64)).shape == (0, 2)


@pytest.mark.parametrize("name", ["random", "tie_grid", "duplicates", "disk"])
def test_mutual_is_the_demo_loop(name):
    """Both directions of a pair; the literal loop runs on at most 300 keypoints per image."""
    corr_ab, kp_b = cases()[name]
    rs = np.random.RandomState(3)
    kp_a = corr_ab + rs.normal(0, 0.5, corr_ab.shape)
    corr_ba = kp_b + rs.normal(0, 0.5, kp_b.shape)
    if name == "disk":
        kp_a, corr_ab, kp_b, corr_ba = kp_a[:300], corr_ab[:300], kp_b[:300], corr_ba[:300]
    n_ab, n_ba, got = mo.match_pair(corr_ab, kp_b, corr_ba, kp_a)
    assert np.array_equal(n_ab, scipy_nearest(corr_ab, kp_b)) and np.array_equal(n_ba, scipy_nearest(corr_ba, kp_a))
    ref = demo_loop(n_ab, n_ba)
    assert got.dtype == np.int64 and np.array_equal(got, ref)
    assert len(got) > 0


def test_mutual_on_full_disk_fixtures():
    a, b = disk(DISK_A).astype(np.float64), disk(DISK_B).astype(np.float64)
    rs = np.random.RandomState(4)
    corr_ab = a * [694 / 1033, 1061 / 771] + rs.normal(0, 1.0, a.shape)
    corr_ba = b * [1033 / 694, 771 / 1061] + rs.normal(0, 1.0, b.shape)
    n_ab, n_ba, got = mo.match_pair(corr_ab, b, corr_ba, a)
    ref_ab, ref_ba = scipy_nearest(corr_ab, b), scipy_nearest(corr_ba, a)
    assert np.array_equal(n_ab, ref_ab) and np.array_equal(n_ba, ref_ba)
    # the demo loop's output, computed without its O(K_a K_b) scan: for each i the first j' with (j', ba[j']) == (ab[i], i)
    ref = [(i, ref_ab[i]) for i in range(len(a)) if ref_ba[ref_ab[i]] == i]
    assert np.array_equal(got, np.array(ref).reshape(-1, 2))


def _task(W, H):
    """A RefinementTask at its first level with the whole image as both patches."""
    from cotr_b200.inference.refinement_task import RefinementTask
    from cotr_b200.utils.utils import ImagePatch
    t = types.SimpleNamespace(cur_job={"patch_to": ImagePatch(None, 0, 0, W, H, W, H)})
    return RefinementTask, t, ImagePatch(None, 0, 0, W, H, W, H)


@pytest.mark.parametrize("W,H", [(1033, 771), (694, 1061), (1, 1), (65536, 65536), (683, 1050)])
def test_pixels_are_scale_to_loc(W, H):
    RefinementTask, task, _ = _task(W, H)
    rs = np.random.RandomState(W)
    pred = np.concatenate([rs.uniform(-0.2, 1.2, (500, 2)), [[0.5, 0.0], [1.0, 1.0], [0.75, 0.3], [0.5000001, 1e-7]]]).astype(np.float32)
    got = mo.pixels(pred, (W, H))
    ref = np.stack([RefinementTask.scale_to_loc(task, p) for p in pred])
    assert ref.dtype == np.float64 and np.array_equal(got, ref)


@pytest.mark.parametrize("W,H", [(1033, 771), (694, 1061), (1, 1), (65536, 65536), (683, 1050)])
def test_queries_are_query_in(W, H):
    RefinementTask, _, patch = _task(W, H)
    rs = np.random.RandomState(H)
    kp = np.concatenate([rs.uniform(0, [W, H], (300, 2)), [[0, 0], [W, H], [W / 3, H / 7]]]).astype(np.float32)
    got = mo.queries(kp, (W, H))
    ref = np.concatenate([RefinementTask._query_in(types.SimpleNamespace(loc_from=k.astype(np.float64)), patch).numpy() for k in kp])
    assert got.dtype == np.float32 and np.array_equal(got, ref)
