"""GPU: the device zoom-in walk (cotr_refine / COTR.refine_walk / SparseEngine(device_walk=True)) against the host loop
of SparseEngine driven by the same native model with device pixels: every task attribute, the engine returns and the
printed progress lines must be identical."""
import numpy as np
import pytest
import torch

from oracle import fixtures
from oracle.fake_model import synthetic_image

pytestmark = pytest.mark.gpu

ZOOMS = np.linspace(0.5, 0.0625, 4)
# area_from / area_to = 5.8467 gives s_from = 2.418: "from" crops of 300 (the image side, above 256), 256, 150 and 44
# pixels in the 300 x 400 image; the "to" crops in the 520 x 360 image are 180, 126, 74 and 22 pixels
AREAS = (5.8467, 1.0)


def _model(sd):
    from cotr_b200.models import build_model
    m = build_model(None)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m.cuda().eval()


@pytest.fixture(scope="module")
def native(built_lib):
    return _model(fixtures.make_state_dict(0))


@pytest.fixture(scope="module")
def images():
    return synthetic_image(51, 300, 400), synthetic_image(52, 520, 360)


def _engine(model, batch, walk, cls=None, **kw):
    from cotr_b200.inference.sparse_engine import SparseEngine
    return (cls or SparseEngine)(model, batch, device_walk=walk, **kw)


def _border_points(rs, n, h, w, spill):
    """Points spread over the image with a third of them within 3 pixels of a border (and beyond it by `spill`)."""
    pts = np.stack([rs.uniform(0, w, n), rs.uniform(0, h, n)], axis=1)
    edge = rs.rand(n) < 0.35
    side = rs.randint(4, size=n)
    off = rs.uniform(-spill, 3, n)
    pts[edge & (side == 0), 0] = off[edge & (side == 0)]
    pts[edge & (side == 1), 0] = w - off[edge & (side == 1)]
    pts[edge & (side == 2), 1] = off[edge & (side == 2)]
    pts[edge & (side == 3), 1] = h - off[edge & (side == 3)]
    return pts


def _tasks(img_a, img_b, loc_from, loc_to, areas, zooms, converge_iters=1):
    from cotr_b200.inference.refinement_task import RefinementTask
    return [RefinementTask(img_a, img_b, f.copy(), t.copy(), areas[0], areas[1], converge_iters, zooms) for f, t in zip(loc_from, loc_to)]


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


def _walk_both(native, make_tasks, batch, max_corrs, capsys, cls=None, **kw):
    out = []
    for walk in (False, True):
        tasks = make_tasks()
        eng = _engine(native, batch, walk, cls=cls, **kw)
        capsys.readouterr()
        eng._single_query_loop(tasks, max_corrs)
        out.append((tasks, capsys.readouterr().out, eng.total_tasks))
    return out


def test_full_task_state(native, images, capsys):
    """70 tasks = two full chunks and a partial one at batch 32; crops clamp at the borders; crop sides above, equal to
    and below 256."""
    img_a, img_b = images
    rs = np.random.RandomState(5)
    loc_from = _border_points(rs, 70, 300, 400, 0)
    loc_to = _border_points(rs, 70, 520, 360, 40)
    (host, host_out, host_n), (dev, dev_out, dev_n) = _walk_both(
        native, lambda: _tasks(img_a, img_b, loc_from, loc_to, AREAS, ZOOMS), 32, 70, capsys)
    sizes = {s for t in host for j in t.job_history for s in j}
    assert {300, 256}.issubset(sizes) and min(sizes) < 256
    assert any(j.x == 0 or j.x + j.w == 400 for t in host for j in [t.cur_job['patch_from']])
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)
    assert {t.status for t in dev} == {'finished'}
    assert dev_out == host_out and dev_out.count("\n") == 3 * 4 + 1
    assert dev_n == host_n == 70 * 4


@pytest.mark.parametrize("batch", [1, 8, 32])
def test_batch_sizes_and_known_scales(native, images, batch, capsys):
    """The known-scale path (areas=) with unequal s_from / s_to through the engine, task states compared."""
    img_a, img_b = images
    rs = np.random.RandomState(7 + batch)
    queries = _border_points(rs, 21, 300, 400, 0)
    got = []
    for walk in (False, True):
        eng = _engine(native, batch, walk, mode='tile')
        capsys.readouterr()
        tasks = eng.cotr_corr_multiscale(img_a, img_b, np.linspace(0.6, 0.1, 3), 1, max_corrs=21, queries_a=queries.copy(),
                                         force=True, return_tasks_only=True, areas=(0.4, 0.9))
        got.append((tasks, capsys.readouterr().out))
    (host, host_out), (dev, dev_out) = got
    assert host[0].s_from != host[0].s_to
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)
    assert dev_out == host_out


def _returns_both(native, call, batch, capsys, cls=None):
    from cotr_b200.utils.utils import fix_randomness
    got = []
    for walk in (False, True):
        fix_randomness(0)
        capsys.readouterr()
        r = call(_engine(native, batch, walk, cls=cls))
        got.append((r, capsys.readouterr().out))
    (host, host_out), (dev, dev_out) = got
    assert dev_out == host_out
    return host, dev


def _equal_returns(a, b):
    if isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for u, v in zip(a, b):
            _equal_returns(u, v)
    else:
        assert _same_array(a, b), (a, b)


def test_engine_returns_forced(native, images, capsys):
    img_a, img_b = images
    q = _border_points(np.random.RandomState(9), 50, 300, 400, 0)
    host, dev = _returns_both(native, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=50, queries_a=q.copy(),
                                                                        force=True, return_idx=True), 16, capsys)
    _equal_returns(host, dev)
    assert host[0].shape == (50, 4)


def test_engine_returns_max_corrs_stop_in_a_later_wave(native, images, capsys, monkeypatch):
    """Every task is good, so max_corrs = 85 stops the loop after chunk 10 (tasks 80 .. 87) at batch 8, in the second
    wave of 8 chunks: the tasks the device walked after it must come back untouched."""
    from cotr_b200.inference import refinement_task
    monkeypatch.setattr(refinement_task, "THRESHOLD_PIXELS_RELATIVE", 1e6)
    img_a, img_b = images
    q = _border_points(np.random.RandomState(11), 150, 300, 400, 0)
    host, dev = _returns_both(native, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=85, queries_a=q.copy(),
                                                                        force=True, return_tasks_only=True), 8, capsys)
    assert len(host) == 150
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)
    walked = [t.status == 'finished' for t in host]
    assert sum(walked) == 88 and all(walked[:88])
    host, dev = _returns_both(native, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=85, queries_a=q.copy(),
                                                                        force=True), 8, capsys)
    _equal_returns(host, dev)


def centred_state_dict():
    """Fixture weights whose last layer answers near the centre of the crop (0.75, 0.5) with a small spread, so that
    the engines' border and cycle filters keep correspondences."""
    sd = {k: v.copy() for k, v in fixtures.make_state_dict(0).items()}
    sd["corr_embed.layers.2.weight"] *= 0.01
    sd["corr_embed.layers.2.bias"][:] = (0.75, 0.5)
    return sd


def test_engine_returns_cycle_consistency(built_lib, images, capsys, monkeypatch):
    from cotr_b200.inference import refinement_task
    monkeypatch.setattr(refinement_task, "THRESHOLD_PIXELS_RELATIVE", 0.5)
    native = _model(centred_state_dict())
    img_a, img_b = images
    q = np.stack([np.random.RandomState(15).uniform(20, 380, 60), np.random.RandomState(16).uniform(20, 280, 60)], axis=1)
    host, dev = _returns_both(native, lambda e: e.cotr_corr_multiscale_with_cycle_consistency(
        img_a, img_b, ZOOMS, 1, max_corrs=12, queries_a=q.copy(), return_idx=True, return_cycle_error=True), 16, capsys)
    _equal_returns(host, dev)
    assert len(host[0]) == 12


def test_engine_returns_faster_engine_and_stretching(native, images, capsys):
    """mode='stretching' (the default), unforced, on the sampling path (integer source points) and with queries;
    FasterSparseEngine keeps its own loop either way."""
    from cotr_b200.inference.sparse_engine import FasterSparseEngine
    img_a, img_b = images
    q = _border_points(np.random.RandomState(21), 40, 300, 400, 0)
    host, dev = _returns_both(native, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=30, return_idx=True), 32, capsys)
    _equal_returns(host, dev)
    host, dev = _returns_both(native, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=30, queries_a=q.copy(),
                                                                        return_idx=True), 32, capsys)
    _equal_returns(host, dev)
    host, dev = _returns_both(native, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=30, queries_a=q.copy(),
                                                                        return_idx=True), 8, capsys, cls=FasterSparseEngine)
    _equal_returns(host, dev)


def test_multi_group_call(native, images, capsys):
    """a -> b (45 tasks) and b -> a (20 tasks) in one call equal two host loops."""
    from cotr_b200.inference import refinement_task
    img_a, img_b = images
    rs = np.random.RandomState(13)
    groups = [(img_a, img_b, _border_points(rs, 45, 300, 400, 0), _border_points(rs, 45, 520, 360, 10), (1.0, 2.5)),
              (img_b, img_a, _border_points(rs, 20, 520, 360, 0), _border_points(rs, 20, 300, 400, 10), (1.7, 1.0))]
    host = []
    for a, b, lf, lt, areas in groups:
        tasks = _tasks(a, b, lf, lt, areas, ZOOMS)
        _engine(native, 16, False)._single_query_loop(tasks, len(tasks))
        host += tasks
    t_ab, t_ba = host[0], host[45]
    dev_a, dev_b = (torch.from_numpy(np.ascontiguousarray(i)).cuda() for i in (img_a, img_b))
    history, rects, good, walked, status = native.refine_walk(
        [dev_a, dev_b], [(0, 1, 0, 45, t_ab.s_from, t_ab.s_to), (1, 0, 45, 20, t_ba.s_from, t_ba.s_to)], list(ZOOMS), 16, 65,
        refinement_task.THRESHOLD_PIXELS_RELATIVE, np.concatenate([g[2] for g in groups]), np.concatenate([g[3] for g in groups]))
    assert walked == 65 and status == (0, 0, 0)
    for i, t in enumerate(host):
        assert np.array_equal(history[i], np.array(t.loc_history)), i
        assert [tuple(r[[2, 2, 5, 5]]) for r in rects[i]] == t.job_history, i
        last = t.cur_job
        assert tuple(rects[i, -1]) == (last['patch_from'].x, last['patch_from'].y, last['patch_from'].w,
                                       last['patch_to'].x, last['patch_to'].y, last['patch_to'].w), i
        assert bool(good[i]) == (t.result == 'good'), i


def test_falls_back_for_converge_iters_2(native, images, capsys, monkeypatch):
    img_a, img_b = images
    calls = []
    real = native.refine_walk
    monkeypatch.setattr(native, "refine_walk", lambda *a, **k: calls.append(1) or real(*a, **k), raising=False)
    rs = np.random.RandomState(17)
    lf, lt = _border_points(rs, 20, 300, 400, 0), _border_points(rs, 20, 520, 360, 0)
    (host, host_out, _), (dev, dev_out, _) = _walk_both(
        native, lambda: _tasks(img_a, img_b, lf, lt, AREAS, ZOOMS, converge_iters=2), 8, 20, capsys)
    assert not calls
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)
    assert dev_out == host_out
    _walk_both(native, lambda: _tasks(img_a, img_b, lf, lt, AREAS, ZOOMS), 8, 20, capsys)
    assert calls == [1]


def test_nan_prediction_raises_on_both_paths(built_lib, images, capsys):
    sd = fixtures.make_state_dict(0)
    sd = {k: v.copy() for k, v in sd.items()}
    sd["corr_embed.layers.2.bias"][0] = np.nan
    model = _model(sd)
    img_a, img_b = images
    rs = np.random.RandomState(19)
    lf, lt = _border_points(rs, 40, 300, 400, 0), _border_points(rs, 40, 520, 360, 0)
    out = []
    for walk in (False, True):
        capsys.readouterr()
        with pytest.raises(ValueError, match="NaN in prediction"):
            _engine(model, 16, walk)._single_query_loop(_tasks(img_a, img_b, lf, lt, AREAS, ZOOMS), 40)
        out.append(capsys.readouterr().out)
    assert out[0] == out[1]


def test_level_launch_sequence(native, images):
    """Both walks run each level as refine_geometry, resize_h, resize_v, the forward's launches at (squads, longest) and
    refine_step: cotr_refine with squads of one task, cotr_refine_grouped with the squads of its batch."""
    nat = native.native()
    dev_a, dev_b = (torch.from_numpy(np.ascontiguousarray(i)).cuda() for i in images)
    rs = np.random.RandomState(29)
    n, zooms = 12, [0.5, 0.25]
    # clustered points: every task lies inside its pilot's boxes, so the grouped batch forms squads of several members
    lf = torch.from_numpy(150 + rs.uniform(-5, 5, (n, 2))).cuda()
    lt = torch.from_numpy(200 + rs.uniform(-5, 5, (n, 2))).cuda()

    def forward(B, Q):
        nat.profile_begin()
        nat.forward(torch.zeros((B, 3, 256, 512), device="cuda"), torch.full((B, Q, 2), 0.5, device="cuda"))
        return [r[:4] for r in nat.profile_end()]

    def level(entries, l, n_squads, longest):
        return ([("refine_geometry", entries, l, 0), ("resize_h", 2 * n_squads, 0, 0), ("resize_v", 2 * n_squads, 0, 0)] +
                forward(n_squads, longest) + [("refine_step", entries, l, 0)])

    expect = [rec for count in (8, 4) for l in range(len(zooms)) for rec in level(count, l, count, 1)]
    nat.profile_begin()
    _, _, _, walked, status = nat.refine([dev_a, dev_b], [(0, 1, 0, n, 1.0, 1.0)], zooms, 8, 4, n, 0.02, lf, lt)
    rec = [r[:4] for r in nat.profile_end()]
    assert walked == n and status == (0, 0, 0)
    assert rec == expect and nat.last_launch_count() == len(rec)

    history = torch.zeros((n, len(zooms) + 1, 2), dtype=torch.float64, device="cuda")
    history[:, 0] = lt
    rects = torch.zeros((n, len(zooms), 6), dtype=torch.int32, device="cuda")
    good = torch.zeros((n + 1,), dtype=torch.int32, device="cuda")
    nat.profile_begin()
    squad, (n_squads, longest, steps, stepped, fail) = nat.refine_grouped(dev_a, dev_b, 1.0, 1.0, zooms, 0, rs.permutation(n), 4, 3,
                                                                          10 ** 6, 0.02, lf, history, rects, good)
    rec = [r[:4] for r in nat.profile_end()]
    assert stepped == 1 and fail == 0 and steps == n and longest > 1
    assert nat.last_launch_count() == len(rec)
    assert rec == [("grouped_candidates", n, 0, 0), ("group_tasks", n, 0, 0)] + level(n, 0, n_squads, longest)
