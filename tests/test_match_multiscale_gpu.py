"""GPU: match_keypoints_multiscale.  The first-guess kernel (cotr_dense_first_guess) bit for bit against the force branch
of SparseEngine.gen_tasks on the same maps, and the whole call against the per-pair sequence it replaces
(SparseEngine(device_walk=True).cotr_corr_multiscale in both directions + mutual_nearest), with fixture weights."""
import os

import numpy as np
import pytest
import torch

from cotr_b200.utils import synthetic
from oracle import match_oracle as mo

pytestmark = pytest.mark.gpu

ZOOMS = np.linspace(0.5, 0.0625, 4)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DISK_A = "disk_kpts_21526113_4379776807.npy"      # image 1033 x 771 (W x H)
DISK_B = "disk_kpts_21126421_4537535153.npy"      # image 694 x 1061


def _model(sd):
    from cotr_b200.models import build_model
    m = build_model(None)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return m.cuda().eval()


@pytest.fixture(scope="module")
def native(built_lib):
    return _model(synthetic.make_state_dict(0))


def _bits(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a.view(np.int64)


# ---- the whole call against the per-pair sequence ---------------------------------------------------------------------

def _disk(name, n, rs, scale=1.0):
    k = np.load(os.path.join(GOLDEN, name))[:n] * np.float32(scale)
    return (k + rs.uniform(-0.5, 0.5, k.shape)).astype(np.float32)


def _image_set(n_kp):
    rs = np.random.RandomState(5)
    images = [synthetic.synthetic_image(81, 771, 1033), synthetic.synthetic_image(82, 1061, 694), synthetic.synthetic_image(83, 512, 512)]
    kps = [_disk(DISK_A, n_kp, rs), _disk(DISK_B, n_kp, rs), _disk(DISK_A, n_kp, rs, 0.49).astype(np.float64)]
    return images, kps


def _per_pair(model, images, kps, pairs, batch, device_walk=True):
    from cotr_b200.inference.matching import mutual_nearest
    from cotr_b200.inference.sparse_engine import SparseEngine
    eng = SparseEngine(model, batch, mode='tile', device_walk=device_walk)
    out = []
    for a, b in pairs:
        c = []
        for f, t in ((a, b), (b, a)):
            if len(kps[f]) == 0:
                c.append(np.zeros((0, 2)))
                continue
            c.append(eng.cotr_corr_multiscale(images[f], images[t], ZOOMS, 1, max_corrs=len(kps[f]), queries_a=kps[f], force=True)[:, 2:])
        out.append((c[0], c[1], mutual_nearest(c[0], kps[b], c[1], kps[a])))
    return out


def _assert_same(res, ref, kps, pairs):
    for p, (a, b) in enumerate(pairs):
        c_ab, c_ba, m = ref[p]
        got_ab, got_ba = res.corrs_ab[p].cpu().numpy(), res.corrs_ba[p].cpu().numpy()
        assert got_ab.dtype == got_ba.dtype == np.float64 and got_ab.shape == c_ab.shape and got_ba.shape == c_ba.shape, p
        assert np.array_equal(_bits(got_ab), _bits(c_ab)) and np.array_equal(_bits(got_ba), _bits(c_ba)), p
        got_m = res.matches[p].cpu().numpy()
        assert got_m.dtype == np.int64 and np.array_equal(got_m, m), p
        n_ab, n_ba, _ = mo.match_pair(c_ab, np.asarray(kps[b], np.float64), c_ba, np.asarray(kps[a], np.float64))
        assert np.array_equal(res.nearest_ab[p].cpu().numpy(), n_ab) and np.array_equal(res.nearest_ba[p].cpu().numpy(), n_ba), p


@pytest.mark.parametrize("batch", [32, 8])
def test_equals_the_per_pair_sequence(native, batch, monkeypatch):
    """Three images (two of them tiled), 200 DISK-fixture keypoints each (one set float64), three pairs: every corr bit for
    bit and every match; cotr_refine runs once, and the only device-to-host copies are the area counts (with the
    first guesses' finiteness flag) and the match counts."""
    from cotr_b200 import capi
    from cotr_b200.inference.matching import match_keypoints_multiscale
    images, kps = _image_set(200)
    pairs = [(0, 1), (1, 2), (2, 0)]
    ref = _per_pair(native, images, kps, pairs, batch)
    refine_calls, to_host = [], []
    real_refine, real_cpu, real_to = capi.NativeModel.refine, torch.Tensor.cpu, torch.Tensor.to

    def cpu(t, *a, **k):
        if t.is_cuda:
            to_host.append((tuple(t.shape), t.dtype))
        return real_cpu(t, *a, **k)

    def to(t, *a, **k):
        out = real_to(t, *a, **k)
        if t.is_cuda and not out.is_cuda:
            to_host.append((tuple(t.shape), t.dtype))
        return out

    monkeypatch.setattr(capi.NativeModel, "refine", lambda *a, **k: refine_calls.append(1) or real_refine(*a, **k))
    monkeypatch.setattr(torch.Tensor, "cpu", cpu)
    monkeypatch.setattr(torch.Tensor, "to", to)
    res = match_keypoints_multiscale(native, images, kps, np.array(pairs), ZOOMS, batch)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert len(refine_calls) == 1
    assert to_host == [((4 * len(pairs) + 1,), torch.int64), ((len(pairs),), torch.int32)], to_host
    _assert_same(res, ref, kps, pairs)
    if batch == 32:
        # and one pair against the host loop of the engine
        host = _per_pair(native, images, kps, pairs[:1], batch, device_walk=False)
        _assert_same(res, host + ref[1:], kps, pairs)


def test_image_without_keypoints_and_cuda_images(native):
    """An image with no keypoints walks no direction from it, and its pairs get no matches; the other direction still
    equals the engine's.  Images may be passed as CUDA tensors."""
    from cotr_b200.inference.matching import match_keypoints_multiscale
    images, kps = _image_set(40)
    kps[2] = np.zeros((0, 2), np.float64)
    pairs = [(0, 2), (2, 1), (0, 1)]
    ref = _per_pair(native, images, kps, pairs, 32)
    res = match_keypoints_multiscale(native, [torch.from_numpy(i).cuda() for i in images], kps, pairs)
    assert res.matches[0].shape == (0, 2) and res.matches[1].shape == (0, 2)
    assert res.corrs_ba[0].shape == (0, 2) and res.corrs_ab[1].shape == (0, 2)
    _assert_same(res, ref, kps, pairs)
    assert len(res.matches[2]) > 0
    empty = match_keypoints_multiscale(native, images, [np.zeros((0, 2))] * 3, pairs)
    assert all(m.shape == (0, 2) for m in empty.matches)


def test_nan_bias_raises_the_engine_error(built_lib):
    """A NaN output bias: the dense predictions are NaN, so the first crop around a first guess raises on both paths
    (the walk would report a NaN prediction instead)."""
    from cotr_b200.inference.matching import match_keypoints_multiscale
    sd = synthetic.make_state_dict(0)
    sd["corr_embed.layers.2.bias"][0] = np.nan
    model = _model(sd)
    images, kps = _image_set(20)
    pairs = [(0, 1)]
    with pytest.raises(ValueError) as engine:
        _per_pair(model, images, kps, pairs, 32)
    with pytest.raises(ValueError) as ours:
        match_keypoints_multiscale(model, images, kps, pairs)
    assert str(ours.value) == str(engine.value)


# ---- cotr_dense_first_guess -------------------------------------------------------------------------------------------

F32_002 = np.float32(0.02)
SPECIALS = np.array([F32_002, np.nextafter(F32_002, np.float32(0)), np.nextafter(F32_002, np.float32(1)), np.float32(0.02 - 1e-9),
                     np.float32(np.nan), np.float32(np.inf), np.float32(-np.inf), np.float32(0.0)], dtype=np.float32)


def _conf(rs, h, w):
    c = rs.uniform(0.0, 0.06, (h, w)).astype(np.float32)
    spots = rs.uniform(size=(h, w)) < 0.2
    c[spots] = rs.choice(SPECIALS, int(spots.sum()))
    return c


def _keypoints(rs, h, w, dtype):
    n = 300
    x = rs.uniform(-0.2 * w - 3, 1.2 * w + 3, n)
    y = rs.uniform(-0.2 * h - 3, 1.2 * h + 3, n)
    k = np.stack([x, y], axis=1)
    k[:60] = np.floor(k[:60])                                         # x.0
    k[60:120] = np.floor(k[60:120]) + 0.999999                        # x.999999
    k[120:140] = -rs.uniform(0, 2, (20, 2))                           # negative, some in (-1, 0)
    k[140] = (-0.0, -1e-30)
    k[141] = (w - 1, h - 1)
    k[142] = (w - 1 + 0.999999, h - 1 + 0.999999)
    k[143] = (w, h)
    k[144] = (1e6, -1e6)
    return k.astype(dtype)


def _engine_force_branch(flow, conf_from, conf_to, kp):
    """gen_tasks(force=True) of the engine itself, on these maps (widened to float64, as cotr_flow returns them)."""
    from cotr_b200.inference.sparse_engine import SparseEngine
    eng = SparseEngine(None, 1, mode='tile')
    maps = (flow.astype(np.float64), conf_from.astype(np.float64), None, None, conf_to.astype(np.float64), None)
    eng._dense_first_guess = lambda img_a, img_b: maps
    img_a = np.empty(conf_from.shape + (3,), np.uint8)
    img_b = np.empty(conf_to.shape + (3,), np.uint8)
    with np.errstate(divide='ignore', invalid='ignore'):
        tasks = eng.gen_tasks(img_a, img_b, ZOOMS, 1, len(kp), kp.copy(), True)
    return tasks


@pytest.mark.parametrize("size_from, size_to", [((1, 1), (1, 1)), ((1, 7), (5, 1)), ((3, 2), (2, 3)), ((257, 300), (771, 1033)),
                                                ((1061, 694), (512, 512)), ((3000, 4000), (4000, 3000))])
def test_dense_first_guess_is_the_force_branch(built_lib, size_from, size_to):
    from cotr_b200 import capi
    rs = np.random.RandomState(size_from[0] * 7 + size_to[1])
    (hf, wf), (ht, wt) = size_from, size_to
    flow = rs.uniform(-1.3, 1.3, (hf, wf, 2)).astype(np.float32)
    conf_from, conf_to = _conf(rs, hf, wf), _conf(rs, ht, wt)
    dev = {k: torch.from_numpy(v).cuda() for k, v in (("flow", flow), ("cf", conf_from), ("ct", conf_to))}
    for dtype in (np.float32, np.float64):
        kp = _keypoints(rs, hf, wf, dtype)
        tasks = _engine_force_branch(flow, conf_from, conf_to, kp)
        loc_to = torch.full((len(kp), 2), np.nan, dtype=torch.float64, device="cuda")
        counts = torch.full((2,), -1, dtype=torch.int64, device="cuda")
        capi.dense_first_guess(dev["flow"], dev["cf"], dev["ct"], torch.from_numpy(kp).cuda(), loc_to, counts)
        counts = counts.cpu().numpy()
        assert counts[0] == (conf_from.astype(np.float64) < 0.02).sum() and counts[1] == (conf_to.astype(np.float64) < 0.02).sum()
        assert counts[0] != (conf_from < np.float32(0.02)).sum() or hf * wf < 20            # the fp64 compare matters
        assert np.int64(counts[0]) / (hf * wf) == tasks[0].area_from and np.int64(counts[1]) / (ht * wt) == tasks[0].area_to
        want = np.array([t.cur_loc_to for t in tasks])
        assert want.dtype == np.float64
        assert np.array_equal(_bits(loc_to.cpu().numpy()), _bits(want)), dtype


def test_dense_first_guess_rejects_bad_arguments(built_lib):
    from cotr_b200 import capi
    flow = torch.zeros((4, 5, 2), dtype=torch.float32, device="cuda")
    conf = torch.zeros((4, 5), dtype=torch.float32, device="cuda")
    kp = torch.zeros((3, 2), dtype=torch.float64, device="cuda")
    loc = torch.zeros((3, 2), dtype=torch.float64, device="cuda")
    counts = torch.zeros((2,), dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    lib = capi.lib()
    p = capi._ptr
    assert lib.cotr_dense_first_guess(0, p(flow), p(conf), 4, 5, p(conf), 4, 5, p(kp), 0, 3, p(loc), p(counts), stream) == 0
    for args in ((0, p(flow), p(conf), 0, 5, p(conf), 4, 5, p(kp), 0, 3, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 70000, p(kp), 0, 3, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, p(kp), 2, 3, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, None, 0, 3, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, p(kp), 0, -1, p(loc), p(counts)),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, p(kp), 0, 3, p(loc), None),
                 (0, p(flow), p(conf), 4, 5, p(conf), 4, 5, capi.ctypes.c_void_p(kp.data_ptr() + 4), 0, 3, p(loc), p(counts))):
        assert lib.cotr_dense_first_guess(*args, stream) != 0
        assert "cotr_dense_first_guess" in capi.last_error()
