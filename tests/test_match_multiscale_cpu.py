"""CPU: the host planning of match_keypoints_multiscale against what the per-pair engine does - the group table and task
order, the crop scales from the area counts (gen_tasks' force branch, sparse_engine.py:224-258, and
RefinementTask.__init__), the errors of the first crop, the row layout of cotr_mutual_nearest, and the refused inputs."""
import numpy as np
import pytest
import torch

from cotr_b200.inference import matching
from cotr_b200.inference.inference_helper import THRESHOLD_AREA
from cotr_b200.inference.refinement_task import RefinementTask
from oracle.fake_model import synthetic_image

ZOOMS = np.linspace(0.5, 0.0625, 4)
F32_002 = np.float32(0.02)


def test_group_table_and_task_order():
    counts = np.array([3, 0, 2, 5])
    pairs = np.array([[0, 1], [2, 0], [1, 1], [3, 2], [0, 3]])
    got = matching.plan_groups(counts, pairs)
    want, first = [], 0
    for p, (a, b) in enumerate(pairs):
        for f, t in ((a, b), (b, a)):          # group 2p = a -> b, 2p+1 = b -> a; an image without keypoints walks nothing
            if counts[f]:
                want.append((p, f, t, first, counts[f]))
                first += counts[f]
    assert got == want
    assert [g[:3] for g in got] == [(0, 0, 1), (1, 2, 0), (1, 0, 2), (3, 3, 2), (3, 2, 3), (4, 0, 3), (4, 3, 0)]
    assert all(type(v) is int for g in got for v in g[1:])


def test_match_layout_is_the_task_order():
    """The walk's rows, in task order, are the rows cotr_mutual_nearest expects: context 2p = a's keypoints into b, 2p+1
    = b's into a, each image's keypoints in their order."""
    counts = np.array([4, 0, 7, 1])
    pairs = np.array([[0, 2], [1, 2], [3, 0], [2, 2]])
    groups = matching.plan_groups(counts, pairs)
    rows = counts[pairs].reshape(-1)
    ctx_off = np.concatenate([[0], np.cumsum(rows)])
    by_ctx = {}
    for p, f, t, first, count in groups:
        c = 2 * p + (1 if 2 * p in by_ctx or counts[pairs[p][0]] == 0 else 0)      # a -> b first, even for a == b
        assert (f, t) == (pairs[p][c % 2], pairs[p][1 - c % 2])
        by_ctx[c] = (first, count, f)
    for c in range(2 * len(pairs)):
        left = pairs[c // 2][c % 2]
        if counts[left] == 0:
            assert c not in by_ctx
        else:
            assert by_ctx[c] == (ctx_off[c], counts[left], left)
    assert sum(g[4] for g in groups) == ctx_off[-1]


def _numpy_force_branch(conf_from, conf_to, img_from, img_to):
    """gen_tasks' areas (float64 maps, as the engine holds them) and the scales of the task it builds."""
    con_a, con_b = conf_from.astype(np.float64), conf_to.astype(np.float64)
    area_a = (con_a < THRESHOLD_AREA).sum() / con_a.size
    area_b = (con_b < THRESHOLD_AREA).sum() / con_b.size
    t = RefinementTask(img_from, img_to, np.zeros(2), np.zeros(2), area_a, area_b, 1, ZOOMS)
    return (int((con_a < THRESHOLD_AREA).sum()), int((con_b < THRESHOLD_AREA).sum())), t


def _conf(rs, h, w, frac):
    c = rs.uniform(0.0, 0.2, (h, w)).astype(np.float32)
    spots = rs.uniform(size=(h, w)) < frac
    c[spots] = rs.choice(np.array([F32_002, np.nextafter(F32_002, np.float32(0)), np.nextafter(F32_002, np.float32(1)),
                                   np.float32(np.nan), np.float32(np.inf), np.float32(0.0)], dtype=np.float32), spots.sum())
    return c


@pytest.mark.parametrize("frac_from, frac_to", [(0.3, 0.6), (0.7, 0.1), (0.5, 0.5)])
def test_scales_from_counts(frac_from, frac_to):
    rs = np.random.RandomState(int(frac_from * 10 + frac_to * 100))
    shapes = [(61, 90), (77, 52)]
    conf_from, conf_to = _conf(rs, *shapes[0], frac_from), _conf(rs, *shapes[1], frac_to)
    counts, task = _numpy_force_branch(conf_from, conf_to, np.zeros(shapes[0] + (3,), np.uint8), np.zeros(shapes[1] + (3,), np.uint8))
    (s_from, s_to), = matching.group_scales([counts], shapes, [(0, 0, 1, 0, 1)])
    assert type(s_from) is type(task.s_from) and type(s_to) is type(task.s_to)
    assert np.array_equal(np.float64(s_from), np.float64(task.s_from)) and np.array_equal(np.float64(s_to), np.float64(task.s_to))
    assert (s_from == 1.0) != (s_to == 1.0) or s_from == s_to == 1.0
    matching.check_crops([(0, 0, 1, 0, 1)], [(s_from, s_to)], shapes, [float(z) for z in ZOOMS])


def test_float32_threshold_is_compared_in_fp64():
    """float32(0.02) lies below 0.02: the engine (float64 maps) counts it."""
    assert np.float64(F32_002) < THRESHOLD_AREA
    conf = np.full((4, 5), F32_002, dtype=np.float32)
    conf[0, :] = np.nextafter(F32_002, np.float32(1))
    conf[1, 0] = np.nan
    counts, _ = _numpy_force_branch(conf, conf, np.zeros((4, 5, 3), np.uint8), np.zeros((4, 5, 3), np.uint8))
    assert counts == (14, 14)


def test_zero_area_on_one_side():
    """area_from = 0 < area_to: s_to = sqrt(area_to / 0) = inf, which crops the whole short side at every level."""
    shapes = [(100, 140), (120, 90)]
    img_from, img_to = np.zeros(shapes[0] + (3,), np.uint8), np.zeros(shapes[1] + (3,), np.uint8)
    for below in ((0, 500), (500, 0)):
        (s_from, s_to), = matching.group_scales([below], shapes, [(0, 0, 1, 0, 1)])
        with np.errstate(divide='ignore'):
            task = RefinementTask(img_from, img_to, np.zeros(2), np.zeros(2), np.int64(below[0]) / 14000, np.int64(below[1]) / 10800, 1, ZOOMS)
        assert np.array_equal([s_from, s_to], [task.s_from, task.s_to]) and np.isinf(max(s_from, s_to))
        matching.check_crops([(0, 0, 1, 0, 1)], [(s_from, s_to)], shapes, [float(z) for z in ZOOMS])
        task.get_task_fast()                   # the engine crops fine too


def test_zero_area_on_both_sides_raises_like_the_engine():
    shapes = [(100, 140), (120, 90)]
    (s_from, s_to), = matching.group_scales([(0, 0)], shapes, [(0, 0, 1, 0, 1)])
    assert np.isnan(s_from) and s_to == 1.0
    with np.errstate(invalid='ignore'):
        task = RefinementTask(np.zeros(shapes[0] + (3,), np.uint8), np.zeros(shapes[1] + (3,), np.uint8), np.zeros(2), np.zeros(2),
                              np.float64(0.0), np.float64(0.0), 1, ZOOMS)
    with pytest.raises(ValueError) as engine:
        task.get_task_fast()
    with pytest.raises(ValueError) as ours:
        matching.check_crops([(0, 0, 1, 0, 1)], [(s_from, s_to)], shapes, [float(z) for z in ZOOMS])
    assert str(ours.value) == str(engine.value) == 'cannot convert float NaN to integer'


def test_crop_below_two_pixels_raises():
    shapes = [(20, 30), (24, 24)]
    matching.check_crops([(0, 0, 1, 0, 1)], [(1.0, 1.0)], shapes, [0.1])          # 2-pixel crops
    with pytest.raises(RuntimeError, match="at least 2 pixels"):
        matching.check_crops([(0, 0, 1, 0, 1)], [(1.0, 1.0)], shapes, [0.5, 0.05])


# ---- refused inputs ------------------------------------------------------------------------------------------------------

def _cpu_model():
    from cotr_b200.models import build_model
    return build_model(None)


def _inputs():
    imgs = [synthetic_image(1, 64, 80), synthetic_image(2, 70, 70)]
    kps = [np.array([[3.0, 4.0], [10.5, 20.25]]), np.array([[5.0, 6.0]], dtype=np.float32)]
    return imgs, kps, np.array([[0, 1]])


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_refuses_non_finite_keypoints(bad):
    imgs, kps, pairs = _inputs()
    kps[0][1, 0] = bad
    with pytest.raises(ValueError, match="cannot be walked exactly"):
        matching.match_keypoints_multiscale(_cpu_model(), imgs, kps, pairs)


def test_refuses_large_float32_keypoints():
    imgs, kps, pairs = _inputs()
    kps[1] = np.array([[2.0 ** 24, 3.0]], dtype=np.float32)
    with pytest.raises(ValueError, match="cannot be walked exactly"):
        matching.match_keypoints_multiscale(_cpu_model(), imgs, kps, pairs)
    kps[1] = np.array([[2.0 ** 24 - 1, 3.0]], dtype=np.float32)       # accepted: fails later, at the CPU model
    with pytest.raises(RuntimeError, match="CUDA device"):
        matching.match_keypoints_multiscale(_cpu_model(), imgs, kps, pairs)


def test_refuses_other_keypoint_types_and_shapes():
    imgs, kps, pairs = _inputs()
    for bad in (np.array([[1, 2]]), np.zeros((3, 3)), np.zeros(4)):
        with pytest.raises(ValueError, match="float32 or float64"):
            matching.match_keypoints_multiscale(_cpu_model(), imgs, [bad, kps[1]], pairs)
    with pytest.raises(ValueError, match="sets for 2 images"):
        matching.match_keypoints_multiscale(_cpu_model(), imgs, kps[:1], pairs)


def test_refuses_attention_hooks():
    imgs, kps, pairs = _inputs()
    model = _cpu_model()
    _, dec = model._attention_modules()
    h = dec[2].register_forward_hook(lambda *a: None)
    with pytest.raises(RuntimeError, match="attention hooks"):
        matching.match_keypoints_multiscale(model, imgs, kps, pairs)
    h.remove()
    with pytest.raises(RuntimeError, match="CUDA device"):
        matching.match_keypoints_multiscale(model, imgs, kps, pairs)


def test_refuses_models_without_the_native_extensions():
    imgs, kps, pairs = _inputs()
    with pytest.raises(RuntimeError, match="native cotr_b200 COTR model"):
        matching.match_keypoints_multiscale(torch.nn.Linear(2, 2), imgs, kps, pairs)


def test_refuses_too_wide_images():
    imgs, kps, pairs = _inputs()
    imgs[1] = synthetic_image(3, 40, 81)
    with pytest.raises(NotImplementedError):
        matching.match_keypoints_multiscale(_cpu_model(), imgs, kps, pairs)
    imgs[1] = synthetic_image(3, 40, 80)                                 # exactly twice: two tiles
    with pytest.raises(RuntimeError, match="CUDA device"):
        matching.match_keypoints_multiscale(_cpu_model(), imgs, kps, pairs)


def test_refuses_bad_schedules_pairs_and_images():
    imgs, kps, pairs = _inputs()
    model = _cpu_model()
    for zooms in ([], np.linspace(0.5, 0.05, 8)):
        with pytest.raises(ValueError, match="zoom_ins"):
            matching.match_keypoints_multiscale(model, imgs, kps, pairs, zoom_ins=zooms)
    for bad in (np.array([[0, 2]]), np.array([[-1, 0]]), np.zeros((0, 2), np.int64), np.array([[0.0, 1.0]])):
        with pytest.raises(ValueError, match="pairs"):
            matching.match_keypoints_multiscale(model, imgs, kps, bad)
    with pytest.raises(ValueError, match="batch_size"):
        matching.match_keypoints_multiscale(model, imgs, kps, pairs, batch_size=0)
    with pytest.raises(ValueError, match="uint8"):
        matching.match_keypoints_multiscale(model, [imgs[0].astype(np.float32), imgs[1]], kps, pairs)
