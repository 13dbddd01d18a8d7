"""CPU: the per-task arithmetic of the device zoom-in walk (cotr_refine), run on the host through cotr_test_refine_math,
against the Python it restates - get_patch_centered_at, RefinementTask._query_in / scale_to_loc / conclude - bit for
bit on random and adversarial inputs."""
import numpy as np
import pytest

from cotr_b200.inference import refinement_task
from cotr_b200.inference.inference_helper import get_patch_centered_at
from cotr_b200.inference.refinement_task import RefinementTask
from cotr_b200.utils.utils import ImagePatch


@pytest.fixture(scope="module")
def capi(built_lib):
    from cotr_b200 import capi
    return capi


class _Shape:
    def __init__(self, h, w):
        self.shape = (h, w, 3)


def _task(loc_from=(0.0, 0.0)):
    return RefinementTask(None, None, np.asarray(loc_from, dtype=np.float64), np.zeros(2), 1.0, 1.0, 1, [1.0])


def _crop_cases():
    rs = np.random.RandomState(0)
    rows = []
    for _ in range(4000):
        h, w = int(rs.randint(2, 1200)), int(rs.randint(2, 1200))
        scale = float(rs.choice([rs.uniform(0, 1.2), 1.0, 0.5, 0.0625, 2.0 / min(h, w), rs.uniform(-0.5, 0)]))
        size = int((min(h, w) * min(max(scale, 0.0), 1.0) // 2) * 2)
        kind = rs.randint(5)
        if kind == 0:
            pos = rs.uniform(-50, max(h, w) + 50, 2)
        elif kind == 1:      # pos - size // 2 exactly on .5 and on integers, both signs
            pos = rs.randint(-3, max(h, w) + 3, 2) + size // 2 + rs.choice([0.5, -0.5, 0.0, 0.4999999999999999], 2)
        elif kind == 2:
            pos = rs.choice([1e300, -1e300, 1e17, -1e17, -0.0, 0.0, -0.9999999999999999], 2)
        elif kind == 3:      # crops of the image side and of 2 pixels
            scale = float(rs.choice([1.0, 2.0 / min(h, w), 3.0 / min(h, w)]))
            pos = rs.uniform(0, max(h, w), 2)
        else:
            pos = rs.uniform(0, max(h, w), 2).round()
        rows.append((float(pos[0]), float(pos[1]), scale, h, w))
    return rows


def test_crop_matches_get_patch_centered_at(capi):
    rows = _crop_cases()
    out = capi.test_refine_math(0, [r[:3] for r in rows], [r[3:] for r in rows])
    for (x, y, scale, h, w), (left, top, size, flag) in zip(rows, out):
        p = get_patch_centered_at(None, np.array([x, y]), scale=scale, return_content=False, img_shape=(h, w, 3))
        assert (left, top, size, flag) == (p.x, p.y, p.w, 0), (x, y, scale, h, w)


def test_non_finite_positions_are_clamped_and_flagged(capi):
    rows = []
    for a in (np.nan, np.inf, -np.inf):
        for b in (np.nan, np.inf, -np.inf, 10.0):
            rows += [(a, b, 0.5), (b, a, 0.5)]
    out = capi.test_refine_math(0, rows, [(300, 400)] * len(rows))
    size = 150
    assert (out[:, 2] == size).all() and (out[:, 3] == 1).all()
    assert (out[:, 0] >= 0).all() and (out[:, 0] + size <= 400).all() and (out[:, 1] >= 0).all() and (out[:, 1] + size <= 300).all()
    with pytest.raises((ValueError, OverflowError)):
        get_patch_centered_at(None, np.array([np.nan, 10.0]), scale=0.5, return_content=False, img_shape=(300, 400, 3))
    nan_scale = capi.test_refine_math(0, [(10.0, 10.0, np.nan)], [(300, 400)])
    assert nan_scale[0, 2] == -1


def test_query_matches_refinement_task(capi):
    rs = np.random.RandomState(1)
    pts, ints = [], []
    for _ in range(4000):
        size = int(rs.choice([2, 4, 256, 512, int(rs.randint(1, 700)) * 2]))
        px, py = int(rs.randint(0, 2000)), int(rs.randint(0, 2000))
        kind = rs.randint(3)
        if kind == 0:
            p = rs.uniform(-100, 2500, 2)
        elif kind == 1:
            p = np.array([px, py]) + rs.choice([0.5, 0.25, size / 2, size - 0.5, 1e-300], 2)
        else:
            p = rs.choice([1e300, -1e300, 1e-17, 3e38, 4e38], 2)
        pts.append(p)
        ints.append((px, py, size))
    got = capi.test_refine_math(1, pts, ints)
    for p, (px, py, size), g in zip(pts, ints, got):
        ref = _task(p)._query_in(ImagePatch(None, px, py, size, size, 0, 0)).numpy()[0]
        assert np.array_equal(g.astype(np.float32), ref, equal_nan=True) and np.array_equal(g, ref.astype(np.float64), equal_nan=True), (p, px, py, size)


def test_scale_to_loc_matches_refinement_task(capi):
    rs = np.random.RandomState(2)
    raws, ints = [], []
    for _ in range(4000):
        raw = rs.choice([rs.uniform(-0.5, 1.5), 0.5, 0.75, 1.0, 0.0, np.float32(0.5000001), 1e-30, 3.4e38, -3.4e38, np.nan], 2)
        raws.append(np.asarray(raw, dtype=np.float32))
        ints.append((int(rs.randint(0, 5000)), int(rs.randint(0, 5000)), int(rs.choice([2, 256, int(rs.randint(1, 900)) * 2]))))
    got = capi.test_refine_math(2, np.array(raws, dtype=np.float64), ints)
    for raw, (px, py, size), g in zip(raws, ints, got):
        t = _task()
        t.cur_job = {'patch_to': ImagePatch(None, px, py, size, size, 0, 0)}
        ref = t.scale_to_loc(raw)
        assert ref.dtype == np.float64 and np.array_equal(g, ref, equal_nan=True), (raw, px, py, size)


@pytest.mark.parametrize("levels", [1, 2, 4, 7])
def test_conclude_matches_refinement_task(capi, monkeypatch, levels):
    rs = np.random.RandomState(3 + levels)
    hist, ints = [], []
    for k in range(3000):
        kind = k % 5
        base = rs.uniform(0, 1000, 2)
        if kind == 0:
            h = base + rs.normal(0, rs.choice([0.1, 1, 5, 20, 100]), (levels + 1, 2))
        elif kind == 1:      # identical rows and exact multiples: zero and representable spreads
            h = np.tile(base.round(), (levels + 1, 1)) + rs.randint(-2, 3, (levels + 1, 2)) * 0.5
        elif kind == 2:
            h = rs.choice([np.nan, np.inf, -np.inf, 1e300, -1e300, 0.0, -0.0, 5.0], (levels + 1, 2))
        elif kind == 3:
            h = base + rs.uniform(-1, 1, (levels + 1, 2)) * 1e-9
        else:
            h = rs.uniform(-1e6, 1e6, (levels + 1, 2))
        hist.append(h)
        ints.append((int(rs.randint(1, 3000)), int(rs.randint(1, 3000))) if k % 7 else (2, 1))
    for rel in (refinement_task.THRESHOLD_PIXELS_RELATIVE, 0.0, 0.001, 0.3, np.inf, np.nan):
        monkeypatch.setattr(refinement_task, "THRESHOLD_PIXELS_RELATIVE", rel)
        got = capi.test_refine_math(3, np.array(hist), ints, levels=levels, rel_threshold=rel)
        for h, (ht, wt), g in zip(hist, ints, got):
            t = _task()
            t.image_to = _Shape(ht, wt)
            t.loc_history = list(h)
            t.best_loc_to = h[-1]
            with np.errstate(invalid="ignore", over="ignore"):
                ref = t.conclude() is not None
            assert bool(g) == ref, (rel, h, ht, wt)


def test_rejects_unknown_op(capi):
    with pytest.raises(RuntimeError):
        capi.test_refine_math(9, [(0.0, 0.0)], [(1, 1)])
