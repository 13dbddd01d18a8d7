"""CPU: FasterSparseEngine's device walk of the grouped levels (cotr_refine_grouped).

- A squad member's canvas query is its own loc_from in its pilot's "from" patch.  The walk computes it in fp64 on the
  widened value; for a float32 point the host loop computes `loc - patch.x` in float32.  The member lies strictly inside
  the pilot's central-half box, so 0 <= patch.x < loc and patch.x is a multiple of ulp(loc) below 2**24: the difference
  is exact in float32 and both give the same bits (cotr_test_refine_math op 1 against RefinementTask._query_in).
- Which calls take the device walk and which keep the host loop."""
import numpy as np
import pytest

from cotr_b200.inference.inference_helper import get_patch_centered_at
from cotr_b200.inference.refinement_task import RefinementTask
from cotr_b200.inference.sparse_engine import FasterSparseEngine
from cotr_b200.utils.utils import ImagePatch

F32 = np.float32
ZOOMS = np.linspace(0.5, 0.0625, 4)


@pytest.fixture(scope="module")
def capi(built_lib):
    from cotr_b200 import capi
    return capi


def _safe_box(p):
    """form_squad's central half of a patch: (l, r, u, d)"""
    cx, cy = p.x + p.w / 2, p.y + p.h / 2
    return cx - p.w / 2 * 0.5, cx + p.w / 2 * 0.5, cy - p.h / 2 * 0.5, cy + p.h / 2 * 0.5


def _inside(lo, hi, v):
    """float32 values strictly inside (lo, hi) in fp64 terms: the box test the member passed"""
    v = np.asarray(v, dtype=F32)
    return v[(v.astype(np.float64) > lo) & (v.astype(np.float64) < hi)]


def _member_points(rs, box):
    """float32 member positions inside a pilot box: random, the first and last float32 inside each edge"""
    l, r, u, d = box
    xs = [rs.uniform(l, r, 6).astype(F32), np.nextafter(F32(l), F32(np.inf)), np.nextafter(F32(r), F32(-np.inf)),
          np.nextafter(np.nextafter(F32(l), F32(np.inf)), F32(np.inf)), F32(np.ceil(l)), F32(np.floor(r))]
    ys = [rs.uniform(u, d, 6).astype(F32), np.nextafter(F32(u), F32(np.inf)), np.nextafter(F32(d), F32(-np.inf)), F32(np.ceil(u))]
    xs = _inside(l, r, np.hstack(xs))
    ys = _inside(u, d, np.hstack(ys))
    return [(x, ys[rs.randint(len(ys))]) for x in xs] + [(xs[rs.randint(len(xs))], y) for y in ys]


def _check_members(capi, members, patches):
    """the walk's query of each widened member point in its pilot's patch == _query_in on the float32 point"""
    pts = np.array(members, dtype=F32)
    crops = np.array([(p.x, p.y, p.w) for p in patches], dtype=np.int64)
    got = capi.test_refine_math(1, pts.astype(np.float64), crops)
    for pt, p, g in zip(pts, patches, got):
        t = RefinementTask(None, None, pt, np.zeros(2), 1.0, 1.0, 1, [1.0])
        ref = t._query_in(ImagePatch(None, p.x, p.y, p.w, p.h, 0, 0)).numpy()[0]
        assert np.array_equal(g.astype(F32), ref) and np.array_equal(g, ref.astype(np.float64)), (pt, p.x, p.y, p.w)
        assert 0 <= p.x < float(pt[0]) and 0 <= p.y < float(pt[1])


def test_member_queries_in_pilot_frames(capi):
    """Pilots anywhere in images of 2 .. 5000 pixels (clamped at the borders too), members strictly inside their boxes."""
    rs = np.random.RandomState(3)
    members, patches = [], []
    for _ in range(1500):
        h, w = int(rs.randint(2, 5000)), int(rs.randint(2, 5000))
        scale = float(rs.choice([rs.uniform(0, 1.2), 1.0, 0.5, 0.0625, 4.0 / min(h, w)]))
        pilot = np.array([rs.uniform(-50, w + 50), rs.uniform(-50, h + 50)], dtype=F32)
        p = get_patch_centered_at(None, pilot, scale=scale, return_content=False, img_shape=(h, w, 3))
        if p.w < 2:
            continue
        for m in _member_points(rs, _safe_box(p)):
            members.append(m)
            patches.append(p)
    assert len(members) > 10000
    _check_members(capi, members, patches)


def test_member_queries_at_the_float32_bound(capi):
    """Members at and just below 2**24 - 1 (the largest float32 points the walk takes), in pilots whose box reaches them."""
    rs = np.random.RandomState(4)
    top = F32(2 ** 24 - 1)
    members, patches = [], []
    for size in (4, 6, 44, 256, 1024, 4096):
        for pilot_x in (top, top - F32(size // 4), top - F32(1.5)):
            w = 2 ** 24 + 8192
            p = get_patch_centered_at(None, np.array([pilot_x, F32(size)], dtype=F32), scale=1.0,
                                      return_content=False, img_shape=(size, w, 3))
            l, r, u, d = _safe_box(p)
            for x in _inside(l, r, [top, np.nextafter(top, F32(0)), F32(r) - F32(1), np.nextafter(F32(l), F32(np.inf))]):
                for y in _inside(u, d, [F32(size / 2), np.nextafter(F32(u), F32(np.inf))]):
                    members.append((x, y))
                    patches.append(p)
    assert any(m[0] == top for m in members)
    _check_members(capi, members, patches)


# ---- eligibility ------------------------------------------------------------------------------------------------------
class _Stub:
    """A model that offers the device walks; pixels count as on the device (see the fixture)."""
    supports_device_preprocess = True

    def __init__(self):
        self.hooked = False

    def attention_hooked(self):
        return self.hooked

    def refine_walk(self, *a, **k):
        raise AssertionError("not called by the eligibility check")

    def refine_grouped_batch(self, *a, **k):
        raise AssertionError("not called by the eligibility check")


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(FasterSparseEngine, "_use_device_pixels", lambda self, tasks: True)
    return _Stub()


def _tasks(n=12, zooms=ZOOMS, dtype_from=np.float64, dtype_to=np.float64, converge_iters=1):
    rs = np.random.RandomState(0)
    img_a, img_b = np.zeros((300, 400, 3), np.uint8), np.zeros((520, 360, 3), np.uint8)
    return [RefinementTask(img_a, img_b, rs.uniform(10, 290, 2).astype(dtype_from), rs.uniform(10, 350, 2).astype(dtype_to),
                           1.0, 1.0, converge_iters, zooms) for _ in range(n)]


def _fits(model, tasks, zooms=ZOOMS, **kw):
    kw.setdefault("device_walk", True)
    return FasterSparseEngine(model, 8, mode='tile', **kw)._grouped_walk_fits(tasks, zooms)


def test_eligible_call(stub):
    assert _fits(stub, _tasks())
    # float32 source points with float64 first guesses: get_tasks_map is float64
    assert _fits(stub, _tasks(dtype_from=F32))
    assert _fits(stub, _tasks(dtype_to=F32))


def test_host_loop_by_default_and_without_device_grouping(stub):
    assert not _fits(stub, _tasks(), device_walk=False)
    assert not _fits(stub, _tasks(), device_grouping=False)


def test_repeated_zoom_values_keep_the_host_loop(stub):
    zooms = [0.5, 0.25, 0.5, 0.125]
    assert not _fits(stub, _tasks(zooms=zooms), zooms=zooms)
    zooms = [0.5, 0.25, 0.25]
    assert not _fits(stub, _tasks(zooms=zooms), zooms=zooms)


def test_float32_task_map_keeps_the_host_loop(stub):
    assert not _fits(stub, _tasks(dtype_from=F32, dtype_to=F32))


def test_attention_hooks_keep_the_host_loop(stub):
    stub.hooked = True
    assert not _fits(stub, _tasks())


def test_converge_iters_2_keeps_the_host_loop(stub):
    assert not _fits(stub, _tasks(converge_iters=2))


def test_other_conditions_keep_the_host_loop(stub):
    assert not _fits(stub, _tasks(zooms=list(np.linspace(0.5, 0.05, 8))), zooms=list(np.linspace(0.5, 0.05, 8)))
    tasks = _tasks()
    tasks[3].submitted = True                       # not fresh
    assert not _fits(stub, tasks)
    tasks = _tasks()
    tasks[5].cur_loc_to = np.array([np.nan, 1.0])   # not an exact point
    assert not _fits(stub, tasks)
    assert not _fits(stub, _tasks(zooms=[0.5, 0.001]), zooms=[0.5, 0.001])    # a crop side below 2
    assert not _fits(object(), _tasks())            # a model without the device walk
