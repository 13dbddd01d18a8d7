"""GPU: FasterSparseEngine(device_walk=True), whose grouped zoom-in levels run one cotr_refine_grouped call per batch,
against the host loop (device_walk=False) driven by the same native model with device pixels, under fix_randomness(0):
every task attribute, the engine returns, the printed lines and np.random's state afterwards must be identical, and the
device path must actually run."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import fixtures
from oracle.fake_model import synthetic_image

pytestmark = pytest.mark.gpu

ZOOMS = np.linspace(0.5, 0.0625, 4)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SOLVED = re.compile(r"solved (\d+) sub-tasks in one invocation with (\d+) image pairs")


def _model(sd):
    from cotr_b200.models import build_model
    m = build_model(None)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m.cuda().eval()


def centred_state_dict():
    """Fixture weights whose last layer answers near the centre of the crop (0.75, 0.5) with a small spread: members
    converge on their pilot's centre, so later levels form squads with many members."""
    sd = {k: v.copy() for k, v in fixtures.make_state_dict(0).items()}
    sd["corr_embed.layers.2.weight"] *= 0.01
    sd["corr_embed.layers.2.bias"][:] = (0.75, 0.5)
    return sd


@pytest.fixture(scope="module")
def centred(built_lib):
    return _model(centred_state_dict())


@pytest.fixture(scope="module")
def images():
    return synthetic_image(61, 300, 400), synthetic_image(62, 520, 360)


# ---- task comparison, as tests/test_refine_gpu.py compares -------------------------------------------------------------

def _same_patch(a, b):
    return (a.patch is None and b.patch is None and (a.x, a.y, a.w, a.h, a.ow, a.oh) == (b.x, b.y, b.w, b.h, b.ow, b.oh)
            and all(type(u) is type(v) for u, v in zip((a.x, a.y, a.w, a.h), (b.x, b.y, b.w, b.h))))


def _same_array(a, b):
    return type(a) is type(b) and np.asarray(a).dtype == np.asarray(b).dtype and np.array_equal(a, b)


def assert_same_task(a, b, what=""):
    for name in ("status", "result", "cur_zoom_idx", "cur_iter", "total_iter", "submitted", "job_history"):
        assert getattr(a, name) == getattr(b, name), (what, name, getattr(a, name), getattr(b, name))
    for name in ("best_loc_to", "cur_loc_to"):
        assert _same_array(getattr(a, name), getattr(b, name)), (what, name)
    for name in ("loc_to_at_zoom", "loc_history"):
        la, lb = getattr(a, name), getattr(b, name)
        assert len(la) == len(lb) and all(_same_array(u, v) for u, v in zip(la, lb)), (what, name, la, lb)
    assert list(a.all_loc_to_dict) == list(b.all_loc_to_dict), what
    assert all(_same_array(a.all_loc_to_dict[k], b.all_loc_to_dict[k]) for k in a.all_loc_to_dict), what
    assert sorted(a.cur_job) == sorted(b.cur_job), what
    for k in a.cur_job:
        u, v = a.cur_job[k], b.cur_job[k]
        if k.startswith("patch"):
            assert _same_patch(u, v), (what, k)
        elif k == "img":
            assert u is None and v is None
        else:
            assert _same_array(u, v), (what, k)


def _equal_returns(a, b):
    if isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for u, v in zip(a, b):
            _equal_returns(u, v)
    else:
        assert _same_array(a, b), (a, b)


def _same_rng(a, b):
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def _both(model, call, batch, capsys, monkeypatch, expect_device=True, **kw):
    """call(engine) with device_walk False, then True -> (host result, device result, stdout); stdout and the RNG state
    afterwards must match, and with expect_device the grouped device walk must have run."""
    from cotr_b200.inference.sparse_engine import FasterSparseEngine
    from cotr_b200.utils.utils import fix_randomness
    calls = []
    real = model.refine_grouped_batch
    monkeypatch.setattr(model, "refine_grouped_batch", lambda *a, **k: calls.append(1) or real(*a, **k), raising=False)
    got = []
    for walk in (False, True):
        fix_randomness(0)
        capsys.readouterr()
        eng = FasterSparseEngine(model, batch, device_walk=walk, **kw)
        r = call(eng)
        got.append((r, capsys.readouterr().out, np.random.get_state()))
        if not walk:
            assert not calls
    (host, host_out, host_rng), (dev, dev_out, dev_rng) = got
    assert dev_out == host_out
    _same_rng(host_rng, dev_rng)
    assert bool(calls) == expect_device
    return host, dev, host_out


def _spread(rs, n, h, w):
    return np.stack([rs.uniform(1, w - 1, n), rs.uniform(1, h - 1, n)], axis=1)


@pytest.mark.parametrize("max_load", [6, 256])
@pytest.mark.parametrize("batch", [8, 32])
def test_squads_fill_and_strand(centred, images, batch, max_load, capsys, monkeypatch):
    """Forced queries over the image: squads that reach max_load (6) and squads that never fill (256); some batch steps
    more members than it has pilots, and some level ends on num_steps <= batch_size with tasks left behind."""
    img_a, img_b = images
    q = _spread(np.random.RandomState(batch + max_load), 400, 300, 400)
    host, dev, out = _both(centred, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=400, queries_a=q.copy(),
                                                                    force=True, return_tasks_only=True),
                           batch, capsys, monkeypatch, mode='tile', max_load=max_load)
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)
    solved = [(int(s), int(p)) for s, p in SOLVED.findall(out)]
    assert any(s > p for s, p in solved)
    assert any(s <= batch for s, _ in solved)
    assert any(t.status == 'unfinished' and t.cur_zoom_idx < len(ZOOMS) - 1 for t in host)      # stranded
    assert all(s <= p * (max_load + 1) for s, p in solved)


def test_max_corrs_stop_at_the_last_level(centred, images, capsys, monkeypatch):
    """Every task is good: max_corrs = 37 stops inside the last level, leaving squads submitted but never stepped;
    the single-query fallback then submits its own batch."""
    from cotr_b200.inference import refinement_task
    monkeypatch.setattr(refinement_task, "THRESHOLD_PIXELS_RELATIVE", 1e6)
    img_a, img_b = images
    q = _spread(np.random.RandomState(31), 300, 300, 400)
    host, dev, out = _both(centred, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=37, queries_a=q.copy(),
                                                                    force=True, return_tasks_only=True),
                           8, capsys, monkeypatch, mode='tile', max_load=12)
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)
    assert any(t.submitted and t.cur_zoom_idx == len(ZOOMS) - 1 for t in host)
    assert sum(t.result == 'good' for t in host) >= 37
    host, dev, _ = _both(centred, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=37, queries_a=q.copy(),
                                                                  force=True, return_idx=True),
                         8, capsys, monkeypatch, mode='tile', max_load=12)
    _equal_returns(host, dev)


def test_max_corrs_zero(centred, images, capsys, monkeypatch):
    """max_corrs = 0: the first batch of every level is formed (submitted) and the loop stops at once."""
    img_a, img_b = images
    q = _spread(np.random.RandomState(33), 120, 300, 400)
    host, dev, out = _both(centred, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=0, queries_a=q.copy(), force=True,
                                                                    return_tasks_only=True), 8, capsys, monkeypatch, mode='tile')
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)
    assert "solved" not in out and any(t.submitted for t in host)


@pytest.mark.parametrize("rescue", [False, True])
@pytest.mark.parametrize("mode", ["tile", "stretching"])
def test_modes_and_rescue(centred, images, mode, rescue, capsys, monkeypatch):
    """Unforced calls on the sampling path (integer source points) and with queries, rescue_stranded on and off."""
    img_a, img_b = images
    q = _spread(np.random.RandomState(41), 150, 300, 400)
    for kw in ({}, {"queries_a": q}):
        kw = {k: v.copy() for k, v in kw.items()}
        host, dev, _ = _both(centred, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=60, return_tasks_only=True, **kw),
                             16, capsys, monkeypatch, mode=mode, max_load=32, rescue_stranded=rescue)
        for i, (a, b) in enumerate(zip(host, dev)):
            assert_same_task(a, b, i)
        host, dev, _ = _both(centred, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=60, return_idx=True, **kw),
                             16, capsys, monkeypatch, mode=mode, max_load=32, rescue_stranded=rescue)
        _equal_returns(host, dev)


def test_known_scales(centred, images, capsys, monkeypatch):
    """areas= with s_from != s_to (tile mode, forced)."""
    img_a, img_b = images
    q = _spread(np.random.RandomState(43), 200, 300, 400)
    host, dev, _ = _both(centred, lambda e: e.cotr_corr_multiscale(img_a, img_b, np.linspace(0.6, 0.1, 3), 1, max_corrs=200,
                                                                  queries_a=q.copy(), force=True, return_tasks_only=True, areas=(0.4, 0.9)),
                         32, capsys, monkeypatch, mode='tile', max_load=64)
    assert host[0].s_from != host[0].s_to
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)


def test_cycle_consistency(centred, capsys, monkeypatch):
    """A small configs[4]: a 512 x 512 pair, tile mode, cycle consistency, zooms linspace(0.5, 0.0625, 4)."""
    from cotr_b200.inference import refinement_task
    monkeypatch.setattr(refinement_task, "THRESHOLD_PIXELS_RELATIVE", 0.5)
    img_a, img_b = synthetic_image(63, 512, 512), synthetic_image(64, 512, 512)
    q = _spread(np.random.RandomState(45), 300, 512, 512)
    host, dev, _ = _both(centred, lambda e: e.cotr_corr_multiscale_with_cycle_consistency(
        img_a, img_b, ZOOMS, 1, max_corrs=40, queries_a=q.copy(), return_idx=True, return_cycle_error=True),
        32, capsys, monkeypatch, mode='tile')
    _equal_returns(host, dev)
    assert len(host[0]) > 0


def test_disk_float32_points(centred, capsys, monkeypatch):
    """The float32 DISK fixture on a synthetic image that holds all its keypoints (768 x 1032), forced, 4 levels."""
    kp = np.load(os.path.join(GOLDEN, "disk_kpts_21526113_4379776807.npy"))[:700]
    assert kp.dtype == np.float32
    img_a, img_b = synthetic_image(65, 768, 1032), synthetic_image(66, 768, 1032)
    host, dev, _ = _both(centred, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=len(kp), queries_a=kp.copy(),
                                                                  force=True, return_tasks_only=True), 32, capsys, monkeypatch, mode='tile')
    assert host[0].loc_from.dtype == np.float32
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)


def test_nan_bias_raises_the_same_exception(built_lib, images, capsys, monkeypatch):
    """A NaN output bias: every prediction is NaN, so the first pilot at level 1 raises at its crop (ValueError) on both
    paths, after the same printed lines.  The tasks start from finite first guesses (the dense first guess of this
    model is NaN too, which would keep the host loop)."""
    from cotr_b200.inference.refinement_task import RefinementTask
    from cotr_b200.inference.sparse_engine import FasterSparseEngine
    from cotr_b200.utils.utils import fix_randomness
    sd = centred_state_dict()
    sd["corr_embed.layers.2.bias"][0] = np.nan
    model = _model(sd)
    img_a, img_b = images
    rs = np.random.RandomState(47)
    lf, lt = _spread(rs, 100, 300, 400), _spread(rs, 100, 520, 360)
    calls = []
    real = model.refine_grouped_batch
    monkeypatch.setattr(model, "refine_grouped_batch", lambda *a, **k: calls.append(1) or real(*a, **k), raising=False)
    out = []
    for walk in (False, True):
        fix_randomness(0)
        capsys.readouterr()
        eng = FasterSparseEngine(model, 8, mode='tile', device_walk=walk)
        eng.gen_tasks = lambda img_a, img_b, zoom_ins, *a, **k: [RefinementTask(img_a, img_b, f.copy(), t.copy(), 1.0, 1.0, 1, zoom_ins)
                                                                 for f, t in zip(lf, lt)]
        with pytest.raises(ValueError):
            eng.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=100)
        out.append((capsys.readouterr().out, np.random.get_state()))
    assert calls and out[0][0] == out[1][0] and "solved" in out[0][0]
    _same_rng(out[0][1], out[1][1])


def _python_failure(pos, scale, shape):
    from cotr_b200.inference.inference_helper import get_patch_centered_at
    try:
        get_patch_centered_at(None, pos, scale=scale, return_content=False, img_shape=shape)
    except ValueError:
        return 1
    except OverflowError:
        return 2
    return 0


def test_pilot_boxes_match_host_bit_for_bit(built_lib):
    """The candidate kernel's pilot boxes equal FasterSparseEngine._pilot_boxes bit for bit, and its failure codes are
    the exceptions get_patch_centered_at raises, on border-clamped and adversarial end points."""
    import warnings
    from cotr_b200 import capi
    from cotr_b200.inference.refinement_task import RefinementTask
    from cotr_b200.inference.sparse_engine import FasterSparseEngine
    rs = np.random.RandomState(7)
    img_a, img_b = np.zeros((300, 400, 3), np.uint8), np.zeros((520, 360, 3), np.uint8)
    special = [0.0, -0.0, 1e-300, -3.5, 31.999999999999996, 32.0, 32.00000000000001, 44.5, 399.9999999999999, 400.0, 1e6,
               -1e6, 1e300, -1e300, 2.0 ** 63, -2.0 ** 63, 2.0 ** 63 - 1024, np.inf, -np.inf, np.nan]
    for zoom in (0.5, 0.0625):
        pts = np.concatenate([_spread(rs, 300, 300, 400), rs.uniform(-60, 460, (300, 2))], axis=0)
        to = np.concatenate([_spread(rs, 300, 520, 360), rs.uniform(-60, 580, (300, 2))], axis=0)
        for k, v in enumerate(special):
            pts[k] = (v, pts[k, 1]) if k % 2 else (pts[k, 0], v)
            to[300 + k] = (v, to[300 + k, 1]) if k % 3 else (to[300 + k, 0], v)
            to[400 + k] = (v, special[-1 - k])
        finite_from = np.isfinite(pts).all(axis=1)
        pts, to = pts[finite_from], to[finite_from]
        tasks = [RefinementTask(img_a, img_b, f, t, 5.8467, 1.0, 1, [zoom]) for f, t in zip(pts, to)]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = FasterSparseEngine._pilot_boxes(tasks)
        t0 = tasks[0]
        sizes = [int((min(s[:2]) * min(max(sc * zoom, 0.0), 1.0) // 2) * 2) for s, sc in ((img_a.shape, t0.s_from), (img_b.shape, t0.s_to))]
        box, fail = capi.test_pilot_boxes(np.concatenate([pts, to], axis=1), [300, 400, 520, 360] + sizes)
        assert np.array_equal(box.view(np.int64), ref.view(np.int64))
        want = [_python_failure(t, t0.s_to * zoom, img_b.shape) for t in to]
        assert fail.tolist() == want and 1 in want and 2 in want
