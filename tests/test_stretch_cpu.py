"""CPU: which path SparseEngine._dense_first_guess takes ('stretching' mode's stretch, dense pass and resize back on the
device, or the host path), the dtypes each hands gen_tasks, and the argument checks of
match_keypoints_multiscale(mode=...).  The dense passes are stand-ins: only the routing is under test here."""
import types

import numpy as np
import pytest
import torch

from cotr_b200.inference import inference_helper as ih
from cotr_b200.inference import sparse_engine as se
from cotr_b200.utils import utils


class _Model:
    """Looks like the native model to the routing checks (parameters on a CUDA device, the device-pixel methods)."""
    supports_device_preprocess = True

    def __init__(self, resize=True):
        if resize:
            self.resize_image = self.resize_maps = lambda *a: None

    def parameters(self):
        yield types.SimpleNamespace(device=torch.device("cuda"))

    def flow_tile_merge(self, *a):
        pass

    def dense_postprocess(self, *a):
        pass

    def preprocess_canvases(self, *a):
        pass


def _img(h, w, seed=0):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)


def _host_maps(img_a, img_b):
    """Stand-in for cotr_flow_maps: float64 maps of the images' shapes, as cotr_flow returns them."""
    rs = np.random.RandomState(img_a.shape[0] + img_b.shape[1])
    (ha, wa), (hb, wb) = img_a.shape[:2], img_b.shape[:2]
    return (rs.uniform(-1, 1, (ha, wa, 2)).astype(np.float32).astype(np.float64), rs.uniform(0, 0.1, (ha, wa)).astype(np.float32).astype(np.float64),
            rs.uniform(-1, 1, (hb, wb, 2)).astype(np.float32).astype(np.float64), rs.uniform(0, 0.1, (hb, wb)).astype(np.float32).astype(np.float64))


@pytest.fixture
def routes(monkeypatch):
    calls = []

    def flow_maps(model, img_a, img_b):
        calls.append(("host", img_a.shape, img_b.shape))
        return _host_maps(img_a, img_b)

    def stretched(model, dev_a, dev_b, shape_a, shape_b):
        calls.append(("device", tuple(shape_a), tuple(shape_b)))
        return tuple((torch.zeros(tuple(s) + (2,)), torch.zeros(tuple(s))) for s in (shape_a, shape_b))

    def no_warp(*a):
        raise AssertionError("the engines do not compute the warped images")

    monkeypatch.setattr(se, "cotr_flow_maps", flow_maps)
    monkeypatch.setattr(se, "stretched_flow_maps", stretched)
    monkeypatch.setattr(ih, "_resample", no_warp)
    monkeypatch.setattr(se.SparseEngine, "_device_image", lambda self, img: img)
    return calls


def test_native_model_stretches_on_the_device(routes):
    img_a, img_b = _img(30, 40), _img(52, 36)
    for cls in (se.SparseEngine, se.FasterSparseEngine):
        routes.clear()
        out = cls(_Model(), 8)._dense_first_guess(img_a, img_b)
        assert routes == [("device", (30, 40), (52, 36))]
        assert out[2] is None and out[5] is None
        assert [m.shape for i, m in enumerate(out) if i not in (2, 5)] == [(30, 40, 2), (30, 40), (52, 36, 2), (52, 36)]
        assert all(m.dtype == np.float32 and isinstance(m, np.ndarray) for i, m in enumerate(out) if i not in (2, 5))


@pytest.mark.parametrize("why", ["no resize methods", "flag off", "no device pixels", "host flow merge"])
def test_host_stretch(routes, monkeypatch, why):
    """The host path: PIL stretch, the dense pass on the squares, float_image_resize of the four maps (float32)."""
    model, engine_kw = _Model(resize=why != "no resize methods"), {}
    img_a, img_b = _img(30, 40), _img(52, 36, 1)
    if why == "flag off":
        monkeypatch.setattr(ih, "DEVICE_STRETCH", False)
    if why == "no device pixels":
        engine_kw["device_preprocess"] = False
    if why == "host flow merge":
        monkeypatch.setattr(ih, "DEVICE_FLOW_MERGE", False)
    out = se.SparseEngine(model, 8, **engine_kw)._dense_first_guess(img_a, img_b)
    assert routes == [("host", (40, 40, 3), (52, 52, 3))]
    want = _host_maps(se.stretch_to_square_np(img_a.copy()), se.stretch_to_square_np(img_b.copy()))
    for got, m, shape in zip([out[i] for i in (0, 1, 3, 4)], want, [(30, 40)] * 2 + [(52, 36)] * 2):
        assert got.dtype == np.float32 and np.array_equal(got, utils.float_image_resize(m, shape), equal_nan=True)
    assert out[2] is None and out[5] is None


@pytest.mark.parametrize("mode", ["stretching", "tile"])
def test_square_pairs_and_tile_mode_keep_float64_maps(routes, mode):
    """Two square images in 'stretching' mode are not stretched, and tile mode never is: cotr_flow's float64 maps, as
    they are, without the warped images."""
    img_a, img_b = (_img(32, 32), _img(48, 48)) if mode == "stretching" else (_img(30, 40), _img(52, 36))
    out = se.SparseEngine(_Model(), 8, mode=mode)._dense_first_guess(img_a, img_b)
    assert routes == [("host", img_a.shape, img_b.shape)]
    want = _host_maps(img_a, img_b)
    assert all(got.dtype == np.float64 and np.array_equal(got, w) for got, w in zip([out[i] for i in (0, 1, 3, 4)], want))
    assert out[2] is None and out[5] is None


def test_stretched_flow_maps_leaves_squares_alone():
    """A square image goes to the dense pass as it is (Pillow would copy it); a non-square one is resized."""
    sizes = []

    class M:
        def resize_image(self, img, size):
            sizes.append(size)
            return torch.zeros(size + (3,), dtype=torch.uint8)

    assert ih.stretch_to_square(M(), torch.zeros((20, 20, 3), dtype=torch.uint8)).shape == (20, 20, 3)
    assert ih.stretch_to_square(M(), torch.zeros((20, 45, 3), dtype=torch.uint8)).shape == (45, 45, 3)
    assert ih.stretch_to_square(M(), torch.zeros((61, 45, 3), dtype=torch.uint8)).shape == (61, 61, 3)
    assert sizes == [(45, 45), (61, 61)]


# ---- match_keypoints_multiscale(mode=...) -----------------------------------------------------------------------------

def _args():
    images = [_img(100, 260), _img(120, 120, 1)]          # image 0: long side more than twice the short side
    kps = [np.array([[10.0, 20.0]]), np.array([[5.0, 6.0]], np.float32)]
    return images, kps, [(0, 1)]


def test_match_multiscale_mode_is_checked():
    from cotr_b200.inference.matching import match_keypoints_multiscale
    images, kps, pairs = _args()
    for bad in ("stretch", "", None, "TILE"):
        with pytest.raises(ValueError, match="mode"):
            match_keypoints_multiscale(object(), images, kps, pairs, mode=bad)


def test_match_multiscale_aspect_limit_only_in_tile_mode():
    """Tile mode refuses image 0 before it looks at the model; 'stretching' takes it and goes on to the model check."""
    from cotr_b200.inference.matching import match_keypoints_multiscale
    images, kps, pairs = _args()
    with pytest.raises(NotImplementedError, match="stretching"):
        match_keypoints_multiscale(object(), images, kps, pairs)
    with pytest.raises(RuntimeError, match="native"):
        match_keypoints_multiscale(object(), images, kps, pairs, mode='stretching')
    with pytest.raises(ValueError, match="uint8"):
        match_keypoints_multiscale(object(), [images[0].astype(np.float32), images[1]], kps, pairs, mode='stretching')
