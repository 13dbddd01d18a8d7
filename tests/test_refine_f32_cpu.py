"""CPU: float32 points on the device zoom-in walk (cotr_refine).

The walk computes in fp64.  For float32 points the host loop computes `pos - size // 2` and `loc - patch.x` in float32
and divides in float32; these tests feed float32 points to that Python (get_patch_centered_at, RefinementTask._query_in)
and the same values widened to fp64 to the C++ of the walk (cotr_test_refine_math), and require equal bits."""
import os

import numpy as np
import pytest

from cotr_b200.inference.inference_helper import get_patch_centered_at
from cotr_b200.inference.refinement_task import RefinementTask
from cotr_b200.inference.sparse_engine import _exact_point
from cotr_b200.utils.utils import ImagePatch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ZOOMS = np.linspace(0.5, 0.0625, 4)
F32 = np.float32


@pytest.fixture(scope="module")
def capi(built_lib):
    from cotr_b200 import capi
    return capi


def _disk():
    return np.concatenate([np.load(os.path.join(GOLDEN, f)) for f in ("disk_kpts_21526113_4379776807.npy",
                                                                      "disk_kpts_21126421_4537535153.npy")])


def _check_crops(capi, pts, scales, shapes):
    """pts (n,2) float32, scales (n,), shapes (n,2) (h, w): the walk's crop of the widened point == Python's on float32."""
    pts = np.asarray(pts, dtype=F32)
    rows = np.concatenate([pts.astype(np.float64), np.asarray(scales, np.float64)[:, None]], axis=1)
    out = capi.test_refine_math(0, rows, shapes)
    for p, s, (h, w), (left, top, size, flag) in zip(pts, scales, shapes, out):
        ref = get_patch_centered_at(None, p, scale=float(s), return_content=False, img_shape=(int(h), int(w), 3))
        assert (left, top, size, flag) == (ref.x, ref.y, ref.w, 0), (p, s, h, w)
    return out


def _check_queries(capi, pts, crops):
    """the walk's fp32 canvas query of the widened point == RefinementTask._query_in on the float32 point (crops of at
    least 2 pixels, points the engine hands to the walk: below 2**24 in magnitude, where `loc - patch.x` is exact)"""
    pts = np.asarray(pts, dtype=F32)
    keep = (np.asarray(crops)[:, 2] >= 2) & np.array([_exact_point(p) for p in pts], dtype=bool)
    pts, crops = pts[keep], np.asarray(crops)[keep]
    got = capi.test_refine_math(1, pts.astype(np.float64), np.asarray(crops, np.int64)[:, :3])
    for p, (px, py, size), g in zip(pts, np.asarray(crops)[:, :3], got):
        t = RefinementTask(None, None, p, np.zeros(2), 1.0, 1.0, 1, [1.0])
        ref = t._query_in(ImagePatch(None, int(px), int(py), int(size), int(size), 0, 0)).numpy()[0]
        assert np.array_equal(g.astype(F32), ref) and np.array_equal(g, ref.astype(np.float64)), (p, px, py, size)


def _adversarial(rs, h, w, size):
    """float32 positions where pos - size // 2 sits just below / at / above 0 and integers, signed zeros, subnormals,
    negatives, values >= 2**24 and points outside the image."""
    half = size // 2
    base = [F32(half), F32(half + rs.randint(0, max(h, w))), F32(half + 1)]
    vals = []
    for b in base:
        vals += [b, np.nextafter(b, F32(-np.inf)), np.nextafter(b, F32(np.inf)), b + F32(0.5), b - F32(0.5)]
    vals += [F32(0.0), F32(-0.0), F32(1e-45), F32(-1e-45), F32(1.1754942e-38), F32(-3.5), F32(-1e6), F32(2 ** 24),
             F32(2 ** 24 + 2), F32(3e38), F32(-3e38), F32(max(h, w) + 0.75), F32(max(h, w) * 3.3), F32(0.49999997)]
    return np.array(vals, dtype=F32)


def test_exact_point_takes_finite_float32():
    assert _exact_point(np.array([1.5, 2.0], dtype=F32))
    assert not _exact_point(np.array([np.nan, 2.0], dtype=F32))
    assert not _exact_point(np.array([np.inf, 2.0], dtype=F32))
    assert not _exact_point(np.array([1.5, 2.0], dtype=np.float16))
    # from 2**24 on, `loc - patch.x` rounds in float32 (2**24 + 2 - 1): such points keep the host loop
    assert _exact_point(np.array([2 ** 24 - 1, -(2 ** 24 - 1)], dtype=F32))
    assert not _exact_point(np.array([2 ** 24, 0], dtype=F32))
    assert float(np.float32(2 ** 24 + 2) - 1) != 2 ** 24 + 1


def test_random_float32_points(capi):
    rs = np.random.RandomState(0)
    pts, scales, shapes = [], [], []
    for _ in range(4000):
        h, w = int(rs.randint(2, 5000)), int(rs.randint(2, 5000))
        pts.append(rs.uniform(-100, max(h, w) + 100, 2))
        scales.append(float(rs.choice([rs.uniform(0, 1.2), 1.0, 0.5, 0.0625, 2.0 / min(h, w)])))
        shapes.append((h, w))
    crops = _check_crops(capi, pts, scales, shapes)
    _check_queries(capi, pts, crops)


def test_adversarial_float32_points(capi):
    rs = np.random.RandomState(1)
    pts, scales, shapes = [], [], []
    for _ in range(300):
        h, w = int(rs.choice([2, 3, 256, 771, 1500, 65536, int(rs.randint(2, 3000))])), int(rs.choice([2, 5, 300, 1000, int(rs.randint(2, 3000))]))
        scale = float(rs.choice([1.0, 0.5, 0.0625, 0.3, 2.0 / min(h, w)]))
        size = int((min(h, w) * scale // 2) * 2)
        vals = _adversarial(rs, h, w, size)
        for x in vals:
            for y in (vals[rs.randint(len(vals))], F32(rs.uniform(0, h))):
                pts.append((x, y))
                scales.append(scale)
                shapes.append((h, w))
    crops = _check_crops(capi, pts, scales, shapes)
    _check_queries(capi, pts, crops)


@pytest.mark.parametrize("shape", [(1000, 1500), (4000, 3000)])
@pytest.mark.parametrize("s", [1.0, 1.7])
def test_disk_keypoints_at_every_level(capi, shape, s):
    """The DISK fixture (float32, as DISK writes it), scaled into the image, at every level of the demo's schedule."""
    kp = _disk()
    assert kp.dtype == F32
    h, w = shape
    kp = (kp * F32(min(h / 1100.0, w / 1100.0))).astype(F32)
    for z in ZOOMS:
        scales = np.full(len(kp), s * z)
        crops = _check_crops(capi, kp, scales, [shape] * len(kp))
        _check_queries(capi, kp, crops)
