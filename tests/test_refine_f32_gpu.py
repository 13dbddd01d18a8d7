"""GPU: float32 points (what DISK writes, and what demo_homography.py passes) on the device zoom-in walk of
SparseEngine(device_walk=True) against the host loop: every task attribute, the engine returns and the printed progress
lines must be identical, and the walk must actually run."""
import os

import numpy as np
import pytest
import torch

from oracle import fixtures
from oracle.fake_model import synthetic_image

pytestmark = pytest.mark.gpu

ZOOMS = np.linspace(0.5, 0.0625, 4)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _model(sd):
    from cotr_b200.models import build_model
    m = build_model(None)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m.cuda().eval()


@pytest.fixture(scope="module")
def native(built_lib):
    return _model(fixtures.make_state_dict(0))


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


def _both(native, call, batch, capsys, monkeypatch, **kw):
    from cotr_b200.inference.sparse_engine import SparseEngine
    calls = []
    real = native.refine_walk
    monkeypatch.setattr(native, "refine_walk", lambda *a, **k: calls.append(1) or real(*a, **k), raising=False)
    got = []
    for walk in (False, True):
        capsys.readouterr()
        eng = SparseEngine(native, batch, device_walk=walk, **kw)
        got.append((call(eng), capsys.readouterr().out, eng.total_tasks))
    assert calls, "the device walk did not run"
    return got


def test_device_walk_disk_float32(native, capsys, monkeypatch):
    """The float32 DISK fixture, scaled into a 300 x 400 image, forced through 4 levels: every task attribute, the
    returns and the printed lines equal the host loop's."""
    kp = np.load(os.path.join(GOLDEN, "disk_kpts_21526113_4379776807.npy"))[:60]
    assert kp.dtype == np.float32
    kp = (kp * np.float32(0.38)).astype(np.float32)
    img_a, img_b = synthetic_image(71, 300, 400), synthetic_image(72, 280, 330)
    (host, host_out, host_n), (dev, dev_out, dev_n) = _both(
        native, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=len(kp), queries_a=kp, force=True,
                                                 return_tasks_only=True), 16, capsys, monkeypatch, mode='tile')
    assert host[0].loc_from.dtype == np.float32
    for i, (a, b) in enumerate(zip(host, dev)):
        assert_same_task(a, b, i)
    assert dev_out == host_out and dev_n == host_n
    (host, host_out, _), (dev, dev_out, _) = _both(
        native, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=len(kp), queries_a=kp, force=True,
                                                 return_idx=True), 16, capsys, monkeypatch, mode='tile')
    assert dev_out == host_out
    assert all(_same_array(u, v) for u, v in zip(host, dev))


def test_device_walk_homography_style_float32(native, capsys, monkeypatch):
    """demo_homography.py's call: four float32 corner points, stretching mode (the default), forced."""
    img_a, img_b = synthetic_image(73, 240, 320), synthetic_image(74, 256, 256)
    q = np.array([[10.5, 12.25], [300.0, 15.75], [305.5, 220.0], [8.0, 230.5]], dtype=np.float32)
    (host, host_out, host_n), (dev, dev_out, dev_n) = _both(
        native, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, queries_a=q, force=True), 32, capsys, monkeypatch)
    assert dev_out == host_out and dev_n == host_n
    assert _same_array(host, dev) and host.shape == (4, 4)
