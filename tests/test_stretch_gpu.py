"""GPU: 'stretching' mode's dense first guess on the device.

* cotr_resize_image bit for bit against PIL and cotr_resize_maps bit for bit against utils.float_image_resize, over
  stretches, up- and downscales, an unchanged axis, odd and prime sizes and 1-pixel sides.
* The engines with inference_helper.DEVICE_STRETCH on against off: returns, task attributes, printed lines and the
  np.random state afterwards, with the device walk off and on; tile mode against cotr_flow-based first guesses.
* cotr_dense_first_guess_f32 against a numpy restatement of the engine's float32 arithmetic.
* match_keypoints_multiscale(mode='stretching') against the per-pair engine sequence.

NaN payloads are not compared: numpy, Pillow and the engines never look at them (every float compare treats any NaN alike),
and the device's double arithmetic returns the canonical NaN where x86 propagates an input's payload.  Every other bit is."""
import numpy as np
import PIL.Image
import pytest
import torch

from oracle import fixtures
from oracle.fake_model import synthetic_image

pytestmark = pytest.mark.gpu

ZOOMS = np.linspace(0.5, 0.0625, 4)

# (h, w) -> (h', w')
SHAPES = [
    ((300, 400), (400, 400)), ((520, 360), (520, 520)), ((3024, 4032), (4032, 4032)),     # stretches
    ((37, 53), (101, 77)), ((300, 400), (61, 123)), ((64, 300), (200, 50)),                # up / down / mixed
    ((131, 97), (131, 256)), ((131, 97), (17, 97)),                                        # one axis unchanged
    ((997, 13), (7, 1009)), ((23, 29), (23, 29)),                                          # primes, identity
    ((1, 1), (5, 3)), ((1, 40), (1, 7)), ((9, 1), (2, 1)), ((5, 6), (1, 1)),               # 1-pixel sides
]


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


def _same_bits(got, want):
    """Equal dtype and shape, NaN at the same places and every other bit equal (-0.0 included)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    if got.dtype.kind != 'f':
        return np.array_equal(got, want)
    gn, wn = np.isnan(got), np.isnan(want)
    ints = {4: np.uint32, 8: np.uint64}[got.dtype.itemsize]
    return np.array_equal(gn, wn) and np.array_equal(got[~gn].view(ints), want[~wn].view(ints))


# ---- the resize kernels ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("src, dst", SHAPES)
def test_resize_image_is_pil(native, src, dst):
    rs = np.random.RandomState(src[0] * 31 + dst[1])
    img = rs.randint(0, 256, src + (3,)).astype(np.uint8)
    img[: max(1, src[0] // 3)] = rs.choice([0, 255], img[: max(1, src[0] // 3)].shape)         # saturated rows clip
    want = np.array(PIL.Image.fromarray(img).resize(dst[::-1], resample=PIL.Image.BILINEAR))
    got = native.resize_image(torch.from_numpy(img).cuda(), dst).cpu().numpy()
    assert got.dtype == np.uint8 and np.array_equal(got, want)


def _maps(rs, shape, c):
    h, w = shape
    m = (rs.standard_normal((h, w, c)) * rs.choice([1e-3, 1.0, 1e6, 1e30], (h, w, c))).astype(np.float32)
    specials = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 3.4e38, -3.4e38, 1e-45], dtype=np.float32)
    spots = rs.uniform(size=(h, w, c)) < 0.03
    m[spots] = rs.choice(specials, int(spots.sum()))
    return m


@pytest.mark.parametrize("src, dst", SHAPES)
def test_resize_maps_is_float_image_resize(native, src, dst):
    from cotr_b200.utils import utils
    rs = np.random.RandomState(src[1] * 17 + dst[0])
    for c in ((1,) if src[0] * src[1] > 10 ** 6 else (1, 2, 3)):
        m = _maps(rs, src, c)
        if src == (131, 97):
            m[60, 40, 0] = np.nan            # an unchanged axis next to a NaN: Pillow does not run that pass
        arg = m[..., 0] if c == 1 else m     # (H, W) for one channel, as the engine passes confidence maps
        want = utils.float_image_resize(arg, dst)
        got = native.resize_maps(torch.from_numpy(np.ascontiguousarray(arg)).cuda(), dst).cpu().numpy()
        assert want.dtype == np.float32 and _same_bits(got, want), c


def test_resize_rejects_bad_arguments(native):
    from cotr_b200 import capi
    lib, p, nat = capi.lib(), capi._ptr, native.native()
    stream = torch.cuda.current_stream().cuda_stream
    img = torch.zeros((4, 5, 3), dtype=torch.uint8, device="cuda")
    out = torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda")
    maps = torch.zeros((4, 5, 3), dtype=torch.float32, device="cuda")
    mout = torch.zeros((8, 8, 3), dtype=torch.float32, device="cuda")
    assert lib.cotr_resize_image(nat.handle, p(img), 4, 5, p(out), 8, 8, stream) == 0
    assert lib.cotr_resize_maps(nat.handle, p(maps), 4, 5, 3, p(mout), 8, 8, stream) == 0
    for args in ((None, p(img), 4, 5, p(out), 8, 8), (nat.handle, None, 4, 5, p(out), 8, 8), (nat.handle, p(img), 0, 5, p(out), 8, 8),
                 (nat.handle, p(img), 4, 5, p(out), 8, 70000), (nat.handle, p(img), 4, 5, p(img), 4, 5)):
        assert lib.cotr_resize_image(*args, stream) != 0
        assert "cotr_resize_image" in capi.last_error()
    for args in ((nat.handle, p(maps), 4, 5, 4, p(mout), 8, 8), (nat.handle, p(maps), 4, 5, 0, p(mout), 8, 8),
                 (nat.handle, p(maps), 4, 5, 3, None, 8, 8), (nat.handle, p(maps), 4, 5, 3, capi.ctypes.c_void_p(mout.data_ptr() + 2), 8, 8),
                 (nat.handle, p(maps), 4, 5, 3, capi.ctypes.c_void_p(maps.data_ptr() + 16), 4, 5)):
        assert lib.cotr_resize_maps(*args, stream) != 0
        assert "cotr_resize_maps" in capi.last_error()
    torch.cuda.synchronize()


def test_resize_profiler_records(native):
    """One record per pass: 22 / 23, M = output rows of the pass, N = output columns, K = 0 horizontal / 1 vertical;
    an unchanged axis launches nothing."""
    nat = native.native()
    img = torch.zeros((30, 40, 3), dtype=torch.uint8, device="cuda")
    maps = torch.zeros((30, 40, 2), dtype=torch.float32, device="cuda")
    native.resize_image(img, (50, 60))
    native.resize_maps(maps, (30, 70))
    torch.cuda.synchronize()
    nat.profile_begin()
    native.resize_image(img, (50, 60))
    native.resize_maps(maps, (30, 70))
    native.resize_maps(maps, (30, 40))
    rec = [r[:4] for r in nat.profile_end()]
    assert rec == [("resize_image", 30, 60, 0), ("resize_image", 50, 60, 1), ("resize_maps", 30, 70, 0)], rec


# ---- the engines ----------------------------------------------------------------------------------------------------

def _same_array(a, b):
    return type(a) is type(b) and np.asarray(a).dtype == np.asarray(b).dtype and _same_bits(a, b)


def _same_patch(a, b):
    return (a.patch is None and b.patch is None and (a.x, a.y, a.w, a.h, a.ow, a.oh) == (b.x, b.y, b.w, b.h, b.ow, b.oh)
            and all(type(u) is type(v) for u, v in zip((a.x, a.y, a.w, a.h), (b.x, b.y, b.w, b.h))))


def assert_same_task(a, b, what=""):
    """Every attribute of two RefinementTasks, as tests/test_refine_gpu.py compares them, plus the first-guess inputs."""
    for name in ("status", "result", "cur_zoom_idx", "cur_iter", "total_iter", "submitted", "job_history", "identifier"):
        assert getattr(a, name) == getattr(b, name), (what, name, getattr(a, name), getattr(b, name))
    for name in ("area_from", "area_to", "s_from", "s_to"):
        assert _same_array(np.asarray(getattr(a, name)), np.asarray(getattr(b, name))), (what, name)
    for name in ("loc_from", "best_loc_to", "cur_loc_to"):
        assert _same_array(getattr(a, name), getattr(b, name)), (what, name)
    for name in ("loc_to_at_zoom", "loc_history"):
        la, lb = getattr(a, name), getattr(b, name)
        assert len(la) == len(lb) and all(_same_array(u, v) for u, v in zip(la, lb)), (what, name)
    assert list(a.all_loc_to_dict) == list(b.all_loc_to_dict), what
    assert all(_same_array(a.all_loc_to_dict[k], b.all_loc_to_dict[k]) for k in a.all_loc_to_dict), what
    assert sorted(a.cur_job) == sorted(b.cur_job), what
    for k in a.cur_job:
        u, v = a.cur_job[k], b.cur_job[k]
        if k.startswith("patch"):
            assert _same_patch(u, v), (what, k)
        elif k == "img":
            assert (u is None) == (v is None), (what, k)
        else:
            assert _same_array(u, v), (what, k)


def _run(engine, call, capsys, seed=3):
    """call(engine) under np.random.seed(seed) -> (return, [task lists gen_tasks made], printed text, RNG state after)."""
    made = []
    real = engine.gen_tasks
    engine.gen_tasks = lambda *a, **k: made.append(real(*a, **k)) or made[-1]
    np.random.seed(seed)
    capsys.readouterr()
    ret = call(engine)
    return ret, made, capsys.readouterr().out, np.random.get_state()


def _assert_same_run(x, y):
    (ra, ta, pa, sa), (rb, tb, pb, sb) = x, y
    ra, rb = (list(r) if isinstance(r, (list, tuple)) else [r] for r in (ra, rb))
    assert len(ra) == len(rb) and all(_same_array(u, v) for u, v in zip(ra, rb))
    assert len(ta) == len(tb)
    for i, (la, lb) in enumerate(zip(ta, tb)):
        assert len(la) == len(lb), i
        for j, (u, v) in enumerate(zip(la, lb)):
            assert_same_task(u, v, (i, j))
    assert pa == pb
    assert sa[0] == sb[0] and np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


def _both_flags(native, make_engine, call, capsys, monkeypatch):
    """The same call with DEVICE_STRETCH on and off; the device path must have resized maps and the host path not."""
    from cotr_b200 import capi
    from cotr_b200.inference import inference_helper as ih
    counts = []
    real = capi.NativeModel.resize_maps
    monkeypatch.setattr(capi.NativeModel, "resize_maps", lambda *a, **k: counts.append(1) or real(*a, **k))
    out = {}
    for flag in (True, False):
        monkeypatch.setattr(ih, "DEVICE_STRETCH", flag)
        counts.clear()
        out[flag] = _run(make_engine(), call, capsys)
        assert (len(counts) > 0) == flag, (flag, len(counts))
    _assert_same_run(out[True], out[False])
    return out[True]


def _corners(h, w):
    return np.array([[0, 0], [w, 0], [w, h], [0, h]], dtype=np.float32)


@pytest.mark.parametrize("walk", [False, True])
def test_sparse_engine_forced_float32_corners(native, images, walk, capsys, monkeypatch):
    """demo_homography.py's call: four float32 image corners, forced."""
    from cotr_b200.inference.sparse_engine import SparseEngine
    img_a, img_b = images
    q = _corners(*img_a.shape[:2])
    ret, made, _, _ = _both_flags(native, lambda: SparseEngine(native, 32, mode='stretching', device_walk=walk),
                                  lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, queries_a=q, force=True), capsys, monkeypatch)
    assert ret.shape == (4, 4) and made[0][0].cur_loc_to.dtype == np.float64


@pytest.mark.parametrize("walk", [False, True])
def test_sparse_engine_unforced_queries(native, images, walk, capsys, monkeypatch):
    """demo_face.py's call: 68 landmarks, unforced (confident ones first, then the top-up)."""
    from cotr_b200.inference.sparse_engine import SparseEngine
    img_a, img_b = images
    rs = np.random.RandomState(68)
    q = np.stack([rs.uniform(-5, 405, 68), rs.uniform(-5, 305, 68)], axis=1)
    ret, made, _, _ = _both_flags(native, lambda: SparseEngine(native, 32, mode='stretching', device_walk=walk),
                                  lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=68, queries_a=q, return_idx=True),
                                  capsys, monkeypatch)
    assert len(made[0]) > 0


@pytest.fixture(scope="module")
def centred(built_lib):
    """Fixture weights whose last layer answers near the centre of the crop (0.75, 0.5) with a small spread, so that the
    engines' border and cycle filters keep correspondences (as in tests/test_refine_gpu.py)."""
    sd = {k: v.copy() for k, v in fixtures.make_state_dict(0).items()}
    sd["corr_embed.layers.2.weight"] *= 0.01
    sd["corr_embed.layers.2.bias"][:] = (0.75, 0.5)
    return _model(sd)


@pytest.mark.parametrize("walk", [False, True])
def test_sparse_engine_sampling(native, images, walk, capsys, monkeypatch):
    """queries_a=None: np.random.choice over both confident masks, a -> b samples and b -> a samples."""
    from cotr_b200.inference.sparse_engine import SparseEngine
    img_a, img_b = images
    ret, made, _, _ = _both_flags(native, lambda: SparseEngine(native, 32, mode='stretching', device_walk=walk),
                                  lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=30, return_idx=True),
                                  capsys, monkeypatch)
    assert len(made[0]) > 0


@pytest.mark.parametrize("walk", [False, True])
def test_sparse_engine_cycle_consistency(centred, images, walk, capsys, monkeypatch):
    """a -> b, then b -> a on the answers, with the weights and threshold of tests/test_refine_gpu.py's cycle test."""
    from cotr_b200.inference import refinement_task
    from cotr_b200.inference.sparse_engine import SparseEngine
    monkeypatch.setattr(refinement_task, "THRESHOLD_PIXELS_RELATIVE", 0.5)
    img_a, img_b = images
    rs = np.random.RandomState(15)
    q = np.stack([rs.uniform(20, 380, 60), rs.uniform(20, 280, 60)], axis=1)
    ret, made, _, _ = _both_flags(centred, lambda: SparseEngine(centred, 16, mode='stretching', device_walk=walk),
                                  lambda e: e.cotr_corr_multiscale_with_cycle_consistency(img_a, img_b, ZOOMS, 1, max_corrs=12, queries_a=q,
                                                                                          return_idx=True, return_cycle_error=True),
                                  capsys, monkeypatch)
    assert len(made) == 2 and len(ret[0]) > 0


@pytest.mark.parametrize("walk", [False, True])
def test_faster_sparse_engine(native, images, walk, capsys, monkeypatch):
    from cotr_b200.inference.sparse_engine import FasterSparseEngine
    img_a, img_b = images
    rs = np.random.RandomState(30)
    q = np.stack([rs.uniform(0, 400, 40), rs.uniform(0, 300, 40)], axis=1)
    _both_flags(native, lambda: FasterSparseEngine(native, 8, mode='stretching', device_walk=walk),
                lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=30, queries_a=q, return_idx=True), capsys, monkeypatch)


def _flow_based(model, mode):
    """The engine's first guess as it was computed before: the full cotr_flow, warped images included, and in
    'stretching' mode all six of its outputs resized back."""
    from cotr_b200.inference.inference_helper import cotr_flow
    from cotr_b200.inference.sparse_engine import stretch_to_square_np
    from cotr_b200.utils import utils

    def first_guess(img_a, img_b):
        if mode == 'tile':
            return cotr_flow(model, img_a, img_b)
        maps = cotr_flow(model, stretch_to_square_np(img_a.copy()), stretch_to_square_np(img_b.copy()))
        return tuple(utils.float_image_resize(m, s) for m, s in zip(maps, (img_a.shape[:2],) * 3 + (img_b.shape[:2],) * 3))
    return first_guess


@pytest.mark.parametrize("mode", ["tile", "stretching"])
def test_returns_equal_the_cotr_flow_first_guess(native, images, mode, capsys):
    """Skipping the two warped images changes nothing the engines return, in either mode."""
    from cotr_b200.inference.sparse_engine import SparseEngine
    img_a, img_b = images
    rs = np.random.RandomState(9)
    q = np.stack([rs.uniform(0, 400, 30), rs.uniform(0, 300, 30)], axis=1)
    runs = []
    for old in (False, True):
        eng = SparseEngine(native, 32, mode=mode, device_walk=True)
        if old:
            eng._dense_first_guess = _flow_based(native, mode)
        runs.append(_run(eng, lambda e: e.cotr_corr_multiscale(img_a, img_b, ZOOMS, 1, max_corrs=30, queries_a=q, return_idx=True), capsys))
    _assert_same_run(*runs)


# ---- cotr_dense_first_guess_f32 -------------------------------------------------------------------------------------

F32_002 = np.float32(0.02)


def _numpy_stretch_branch(flow, conf_from, conf_to, kp, size_to_xy):
    """The force branch of gen_tasks on float32 maps, restated: float32 compares, float32 scale and offset."""
    below = [(conf_from < 0.02).sum(), (conf_to < 0.02).sum()]
    out = []
    for loc in kp:
        pos = loc[::-1]
        pos = np.array([np.clip(pos[0], 0, flow.shape[0] - 1), np.clip(pos[1], 0, flow.shape[1] - 1)], dtype=int)
        out.append((flow[tuple(pos)].copy() * 0.5 + 0.5) * size_to_xy)
    return below, np.array(out)


@pytest.mark.parametrize("size_from, size_to", [((1, 1), (1, 1)), ((3, 2), (2, 3)), ((257, 300), (771, 1033)), ((1061, 694), (512, 512))])
def test_dense_first_guess_f32_is_the_stretching_branch(built_lib, size_from, size_to):
    from cotr_b200 import capi
    from cotr_b200.inference.sparse_engine import SparseEngine
    rs = np.random.RandomState(size_from[1] * 3 + size_to[0])
    (hf, wf), (ht, wt) = size_from, size_to
    flow = rs.uniform(-1.3, 1.3, (hf, wf, 2)).astype(np.float32)
    flow.reshape(-1)[::5] = np.float32(1e-8)                  # f32: 0.5 exactly, f64: 0.500000005
    flow.reshape(-1)[1::7] = np.float32(np.nan)

    def conf(h, w):
        c = rs.uniform(0.0, 0.06, (h, w)).astype(np.float32)
        c.reshape(-1)[::3] = F32_002                          # not counted in float32, counted in float64
        c.reshape(-1)[1::11] = np.float32(np.nan)
        return c
    conf_from, conf_to = conf(hf, wf), conf(ht, wt)
    dev = [torch.from_numpy(a).cuda() for a in (flow, conf_from, conf_to)]
    for dtype in (np.float32, np.float64):
        kp = np.stack([rs.uniform(-3, wf + 3, 200), rs.uniform(-3, hf + 3, 200)], axis=1).astype(dtype)
        kp[:3] = [[-0.5, -1e-30], [wf - 1 + 0.999, hf - 1 + 0.999], [wf, hf]]
        below, want = _numpy_stretch_branch(flow, conf_from, conf_to, kp, (wt, ht))
        # the engine's own force branch on these float32 maps (what stretching mode hands it)
        eng = SparseEngine(None, 1, mode='stretching')
        eng._dense_first_guess = lambda a, b: (flow, conf_from, None, None, conf_to, None)
        with np.errstate(divide='ignore', invalid='ignore'):
            tasks = eng.gen_tasks(np.empty((hf, wf, 3), np.uint8), np.empty((ht, wt, 3), np.uint8), ZOOMS, 1, len(kp), kp.copy(), True)
        assert _same_bits(np.array([t.cur_loc_to for t in tasks]), want)
        loc = torch.full((len(kp), 2), 7.0, dtype=torch.float64, device="cuda")
        counts = torch.full((2,), -1, dtype=torch.int64, device="cuda")
        capi.dense_first_guess(*dev, torch.from_numpy(kp).cuda(), loc, counts, f32_maps=True)
        counts = counts.cpu().numpy()
        assert list(counts) == below
        assert np.int64(counts[0]) / (hf * wf) == tasks[0].area_from and np.int64(counts[1]) / (ht * wt) == tasks[0].area_to
        assert _same_bits(loc.cpu().numpy(), want), dtype
        if hf * wf > 20:
            assert counts[0] != (conf_from.astype(np.float64) < 0.02).sum()                # the float32 compare matters
            wide = (flow.astype(np.float64) * 0.5 + 0.5)[np.isfinite(flow)]
            assert not np.array_equal(wide, (flow * np.float32(0.5) + np.float32(0.5))[np.isfinite(flow)])


def test_dense_first_guess_f32_rejects_bad_arguments(built_lib):
    from cotr_b200 import capi
    flow = torch.zeros((4, 5, 2), dtype=torch.float32, device="cuda")
    conf = torch.zeros((4, 5), dtype=torch.float32, device="cuda")
    kp = torch.zeros((3, 2), dtype=torch.float64, device="cuda")
    loc = torch.zeros((3, 2), dtype=torch.float64, device="cuda")
    counts = torch.zeros((2,), dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    lib, p = capi.lib(), capi._ptr
    assert lib.cotr_dense_first_guess_f32(0, p(flow), p(conf), 4, 5, p(conf), 4, 5, p(kp), 0, 3, p(loc), p(counts), stream) == 0
    for args in ((0, p(flow), p(conf), 0, 5, p(conf), 4, 5, p(kp), 0, 3, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 70000, p(kp), 0, 3, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, p(kp), 2, 3, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, None, 0, 3, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, p(kp), 0, -1, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, p(kp), 0, 3, p(loc), None),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, capi.ctypes.c_void_p(kp.data_ptr() + 4), 0, 3, p(loc), p(counts))):
        assert lib.cotr_dense_first_guess_f32(*args, stream) != 0
        assert "cotr_dense_first_guess_f32" in capi.last_error()
    torch.cuda.synchronize()


# ---- match_keypoints_multiscale(mode='stretching') -------------------------------------------------------------------

def _image_set():
    rs = np.random.RandomState(11)
    shapes = [(200, 520), (300, 300), (340, 260), (240, 180), (256, 256)]     # image 0: long side > 2 x short side
    images = [synthetic_image(90 + i, h, w) for i, (h, w) in enumerate(shapes)]
    kps = []
    for i, (h, w) in enumerate(shapes):
        n = 0 if i == 3 else 40
        k = np.stack([rs.uniform(0, w, n), rs.uniform(0, h, n)], axis=1)
        kps.append(k.astype(np.float32) if i in (0, 2) else k)
    return images, kps


def test_match_multiscale_stretching_equals_the_engine(native):
    """Pairs: non-square with square, square with non-square, two non-square, an image without keypoints, two squares."""
    from cotr_b200.inference.matching import match_keypoints_multiscale, mutual_nearest
    from cotr_b200.inference.sparse_engine import SparseEngine
    images, kps = _image_set()
    pairs = [(0, 1), (1, 2), (2, 0), (3, 1), (1, 4)]
    with pytest.raises(NotImplementedError):
        match_keypoints_multiscale(native, images, kps, pairs)                 # tile mode refuses image 0
    res = match_keypoints_multiscale(native, images, kps, np.array(pairs), ZOOMS, 16, mode='stretching')
    eng = SparseEngine(native, 16, mode='stretching', device_walk=True)
    for p, (a, b) in enumerate(pairs):
        c = []
        for f, t in ((a, b), (b, a)):
            if len(kps[f]) == 0:
                c.append(np.zeros((0, 2)))
                continue
            c.append(eng.cotr_corr_multiscale(images[f], images[t], ZOOMS, 1, max_corrs=len(kps[f]), queries_a=kps[f], force=True)[:, 2:])
        got_ab, got_ba = res.corrs_ab[p].cpu().numpy(), res.corrs_ba[p].cpu().numpy()
        assert _same_bits(got_ab, c[0].astype(np.float64)) and _same_bits(got_ba, c[1].astype(np.float64)), p
        assert np.array_equal(res.matches[p].cpu().numpy(), mutual_nearest(c[0], kps[b], c[1], kps[a])), p
    assert res.matches[3].shape == (0, 2) and len(res.matches[0]) + len(res.matches[2]) > 0
