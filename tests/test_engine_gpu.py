"""GPU: the zoom-in engines (cotr_b200.inference) driving the native sm_90a model, against the same engines driving
the CPU oracle.  The loop is discontinuous in the network output (integer crop corners, accept / reject thresholds),
so the comparison is reported in pixels on forced queries (SURVEY.md section 7 "what engine-level parity can mean")."""
import numpy as np
import pytest
import torch
from torch import nn

from oracle import cotr_oracle, fixtures
from oracle.fake_model import synthetic_image

pytestmark = pytest.mark.gpu


class OracleCOTR(nn.Module):
    """The CPU oracle behind the model(img, queries)['pred_corrs'] contract (test-side only)."""

    def __init__(self, sd):
        super().__init__()
        self.anchor = nn.Parameter(torch.zeros(1), requires_grad=False)
        self.sd = cotr_oracle.cast_state_dict(sd, torch.float32)

    @torch.no_grad()
    def forward(self, img, queries):
        return {'pred_corrs': cotr_oracle.forward(self.sd, img.cpu(), queries.cpu(), torch.float32)}


@pytest.fixture(scope="module")
def models(built_lib):
    from cotr_b200.models import build_model
    sd = fixtures.make_state_dict(0)
    native = build_model(None)
    native.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return native.cuda().eval(), OracleCOTR(sd)


def test_dense_flow_matches_oracle(models):
    """cotr_flow: one dense pass (131 072 grid queries) per direction on a square pair."""
    from cotr_b200.inference.inference_helper import cotr_flow
    native, oracle = models
    img_a = synthetic_image(31, 256, 256)
    img_b = synthetic_image(32, 256, 256)
    got = cotr_flow(native, img_a, img_b)
    ref = cotr_flow(oracle, img_a, img_b)
    for g, r, name in zip((got[0], got[1], got[3], got[4]), (ref[0], ref[1], ref[3], ref[4]), ("corr_a", "conf_a", "corr_b", "conf_b")):
        assert g.shape == r.shape
        # The north-star tolerance is 1e-3 on the network output (x over the 512-wide canvas, y over 256, both in
        # [0,1]).  Dense maps are in [-1,1] units of ONE image: x is scaled by 4 (canvas -> half -> [-1,1]), y by 2;
        # the cycle confidence is a norm of a bilinear resampling of those (grid_sample), bounded by the x scale.
        if name.startswith("corr"):
            assert np.abs(g[..., 0] - r[..., 0]).max() < 4e-3, name + ".x"
            assert np.abs(g[..., 1] - r[..., 1]).max() < 2e-3, name + ".y"
        else:
            assert np.abs(g - r).max() < 4e-3, name


def test_device_dense_postprocess_matches_host_path(models):
    """cotr_dense_postprocess against the reference's host tail of the dense pass (inference_helper.py:131-145: torch
    grid_sample on the CPU, norm, per-half remap) on the same predictions.  fp32 both sides; the tolerance covers the
    different summation order of the four bilinear taps (2e-6 on values in [-3, 3])."""
    from cotr_b200.inference import inference_helper as ih
    native, _ = models
    img_a = synthetic_image(37, 256, 256)
    img_b = synthetic_image(38, 256, 256)
    out = {}
    for flag in (True, False):
        ih.DEVICE_DENSE_POST = flag
        try:
            out[flag] = ih._dense_pass(native, img_a, img_b)
        finally:
            ih.DEVICE_DENSE_POST = True
    for dev, host in zip(out[True], out[False]):
        assert dev.shape == host.shape == (256, 256, 3) and dev.dtype == host.dtype == np.float32
        assert np.isfinite(dev).all()
        assert np.abs(dev - host).max() < 2e-6, np.abs(dev - host).max(axis=(0, 1))
    # synthetic predictions that leave the canvas exercise the zero padding of grid_sample
    rs = np.random.RandomState(11)
    pred = torch.from_numpy(rs.uniform(-0.3, 1.3, size=(2, 256 * 512, 2)).astype(np.float32)).cuda()
    dev = native.dense_postprocess(pred).cpu()
    for n in range(2):
        og = pred[n].cpu().view(1, 256, 512, 2) * 2 - 1
        cyc = torch.nn.functional.grid_sample(og.permute(0, 3, 1, 2), og, align_corners=False).permute(0, 2, 3, 1)[0]
        grid = torch.from_numpy(ih._dense_grid()).float() * 2 - 1
        conf = torch.norm(cyc - grid, dim=-1)
        ref = og[0].clone()
        ref[:, :256, 0] = ref[:, :256, 0] * 2 - 1
        ref[:, 256:, 0] = ref[:, 256:, 0] * 2 + 1
        ref = torch.cat([ref, conf[..., None]], dim=-1)
        assert (dev[n] - ref).abs().max().item() < 4e-6


def test_sparse_engine_matches_oracle_in_pixels(models, capsys):
    from cotr_b200.inference.sparse_engine import SparseEngine
    from cotr_b200.utils.utils import fix_randomness
    native, oracle = models
    img_a = synthetic_image(33, 320, 320)
    img_b = synthetic_image(34, 288, 288)
    rs = np.random.RandomState(3)
    queries = np.stack([rs.uniform(20, 300, 12), rs.uniform(20, 300, 12)], axis=1)
    zooms = np.linspace(0.5, 0.125, 3)
    out = []
    for model in (native, oracle):
        fix_randomness(0)
        corrs = SparseEngine(model, 8, mode='tile').cotr_corr_multiscale(
            img_a, img_b, zooms, 1, max_corrs=12, queries_a=queries.copy(), force=True)
        out.append(corrs)
    got, ref = out
    assert got.shape == ref.shape == (12, 4)
    assert np.array_equal(got[:, :2], ref[:, :2])                 # the forced source points
    diff = np.linalg.norm(got[:, 2:] - ref[:, 2:], axis=1)
    # a 1e-3 deviation of the network output is 0.3 px at the coarsest level and shrinks with the zoom
    assert np.median(diff) < 0.25 and diff.max() < 1.5, diff


def test_device_preprocess_is_bit_identical_to_pillow(models):
    """cotr_preprocess (crop + Pillow-exact antialiased resize + to_tensor + normalize on the device) against the
    host path of the reference (PIL resize, torchvision to_tensor / normalize) - every pixel, every bit."""
    from cotr_b200.inference.inference_helper import _to_network_canvas
    native, _ = models
    img_a = synthetic_image(41, 783, 1064)
    img_b = synthetic_image(42, 1053, 689)
    rs = np.random.RandomState(7)
    rects = []
    for size_a, size_b in [(782, 688), (390, 344), (276, 256), (256, 162), (162, 48), (48, 2), (600, 100), (254, 258)]:
        xa = rs.randint(0, img_a.shape[1] - size_a + 1); ya = rs.randint(0, img_a.shape[0] - size_a + 1)
        xb = rs.randint(0, img_b.shape[1] - size_b + 1); yb = rs.randint(0, img_b.shape[0] - size_b + 1)
        rects.append((xa, ya, size_a, xb, yb, size_b))
    rects = np.array(rects, dtype=np.int32)
    dev = native.preprocess_canvases(torch.from_numpy(img_a).cuda(), torch.from_numpy(img_b).cuda(), rects).cpu()
    for i, (xa, ya, sa, xb, yb, sb) in enumerate(rects):
        ref = _to_network_canvas(img_a[ya:ya + sa, xa:xa + sa], img_b[yb:yb + sb, xb:xb + sb])
        assert torch.equal(dev[i], ref), (i, (dev[i] - ref).abs().max().item())


def test_preprocess_survives_gemm_path_toggle(models):
    """cotr_set_gemm_path drops the captured graphs; it must not touch the device preprocessor (a stray
    preprocessor_destroy there once left a dangling pointer: use-after-free on the next cotr_preprocess)."""
    native, _ = models
    img_a = synthetic_image(45, 300, 300)
    img_b = synthetic_image(46, 280, 280)
    rects = np.array([(10, 20, 256, 5, 7, 200), (0, 0, 300, 0, 0, 280)], dtype=np.int32)
    a_dev, b_dev = torch.from_numpy(img_a).cuda(), torch.from_numpy(img_b).cuda()
    first = native.preprocess_canvases(a_dev, b_dev, rects).clone()
    nat = native.native()
    for _ in range(3):
        nat.set_gemm_path(1)
        nat.set_gemm_path(0)
        again = native.preprocess_canvases(a_dev, b_dev, rects)
        assert torch.equal(again, first)
    q = torch.rand(2, 5, 2, device="cuda")
    assert torch.isfinite(native(first, q)["pred_corrs"]).all()


def test_engine_device_pixels_equal_host_pixels(models):
    """The engines give identical correspondences whether the crops are resized on the device or by PIL on the host."""
    from cotr_b200.inference.sparse_engine import FasterSparseEngine, SparseEngine
    from cotr_b200.utils.utils import fix_randomness
    native, _ = models
    img_a = synthetic_image(43, 300, 400)
    img_b = synthetic_image(44, 360, 288)
    rs = np.random.RandomState(9)
    queries = np.stack([rs.uniform(5, 395, 24), rs.uniform(5, 295, 24)], axis=1)
    zooms = np.linspace(0.5, 0.0625, 4)
    for engine_cls, kw in ((SparseEngine, {}), (FasterSparseEngine, {"max_load": 8})):
        results = []
        for on_device in (True, False):
            fix_randomness(0)
            eng = engine_cls(native, 8, mode='tile', device_preprocess=on_device, **kw)
            results.append(eng.cotr_corr_multiscale(img_a, img_b, zooms, 2, max_corrs=24, queries_a=queries.copy(), force=True))
        assert results[0].shape == results[1].shape
        assert np.array_equal(results[0], results[1])


def test_context_reuse_in_corr_base(models):
    """cotr_corr_base uses encode_context/decode on the native model (one context, two decodes)."""
    from cotr_b200.inference.inference_helper import cotr_corr_base
    native, oracle = models
    img_a = synthetic_image(35, 256, 256)
    img_b = synthetic_image(36, 256, 256)
    rs = np.random.RandomState(4)
    q = np.stack([rs.uniform(5, 250, 20), rs.uniform(5, 250, 20)], axis=1)
    got = cotr_corr_base(native, img_a, img_b, q.copy())
    ref = cotr_corr_base(oracle, img_a, img_b, q.copy())
    assert np.abs(got - ref).max() < 0.6          # pixels: 1e-3 * 2 * 256 = 0.5 px per axis at full scale


def test_triangulate_corr_cuda_rasteriser_matches_oracle(built_lib):
    """cotr_rasterize_triangles (the GL rendering of inference_helper.py:293-308 as a CUDA kernel) against the CPU
    restatement: same Delaunay triangles (scipy on both sides), barycentric interpolation at every pixel centre.
    Coverage may differ only for pixel centres that lie (numerically) ON a hull edge; values are piecewise linear and
    continuous across interior edges, so they agree wherever both sides are inside."""
    from cotr_b200.inference.inference_helper import triangulate_corr
    from oracle import triangulate_oracle
    rs = np.random.RandomState(12)
    for (h, w, n) in ((240, 320, 40), (783, 1064, 300), (64, 64, 3)):
        src = np.stack([rs.uniform(2, w - 2, n), rs.uniform(2, h - 2, n)], axis=1)
        dst = src * np.array([0.9, 1.1]) + rs.uniform(-20, 20, (n, 2))
        corr = np.concatenate([src, dst], axis=1)
        got = triangulate_corr(corr, (h, w, 3), (h + 10, w + 10, 3))
        ref, inside = triangulate_oracle.triangulate_corr(corr, (h, w, 3), (h + 10, w + 10, 3))
        assert got.shape == ref.shape == (h, w, 2) and got.dtype == np.float32
        got_inside = (got != 0).any(axis=2)
        assert (got_inside != inside).mean() < 2e-4                      # hull-edge pixel centres only
        both = got_inside & inside
        assert both.sum() > 30 and both.sum() > 0.9 * inside.sum()
        # pixels of the target image (coordinates up to ~1e3); sliver triangles amplify the fp32 vertex rounding
        assert np.abs(got[both] - ref[both]).max() < 2e-2 and np.abs(got[both] - ref[both]).mean() < 1e-4
        assert (got[~got_inside] == 0).all()


def test_device_flow_merge_equals_host_path(models):
    """cotr_flow_tile_merge (patch affine + Pillow-exact mode-'F' resize + min-confidence merge on the device) against
    the reference's host sequence (numpy affine, PIL float resize per channel, merge_flow_patches) on the same dense
    answers: non-square images, so each side has two overlapping tiles (4 dense passes) and the merge really chooses."""
    from cotr_b200.inference import inference_helper as ih
    native, _ = models
    img_a = synthetic_image(47, 300, 420)
    img_b = synthetic_image(48, 380, 290)
    out = {}
    for flag in (True, False):
        ih.DEVICE_FLOW_MERGE = flag
        try:
            out[flag] = ih.cotr_flow(native, img_a, img_b)
        finally:
            ih.DEVICE_FLOW_MERGE = True
    for k, name in ((0, "corr_a"), (1, "con_a"), (3, "corr_b"), (4, "con_b")):
        dev, host = out[True][k], out[False][k]
        assert dev.shape == host.shape and dev.dtype == host.dtype == np.float64
        # both sides start from the same fp32 dense answers (same kernels, same inputs) and the resampler is restated
        # exactly (double accumulation, fp32 stores), so the maps agree to the last bit
        assert np.array_equal(dev, host), (name, np.abs(dev - host).max())


def test_device_squad_formation_equals_host_walk(models):
    """cotr_group_tasks (form_squad for a whole batch in one device call) against the host walk of the reference's
    form_grouped_batch: same squads, same member order -> identical correspondences, with and without the
    stranded-task fix, for a load small enough that squads fill up (max_load) and large enough that they do not."""
    from cotr_b200.inference.sparse_engine import FasterSparseEngine
    from cotr_b200.utils.utils import fix_randomness
    native, _ = models
    img_a = synthetic_image(49, 400, 520)
    img_b = synthetic_image(50, 460, 380)
    rs = np.random.RandomState(21)
    queries = np.stack([rs.uniform(5, 515, 90), rs.uniform(5, 395, 90)], axis=1)
    zooms = np.linspace(0.5, 0.0625, 4)
    for max_load, rescue in ((6, False), (64, True)):
        results = []
        for on_device in (True, False):
            fix_randomness(0)
            eng = FasterSparseEngine(native, 8, mode='tile', max_load=max_load, rescue_stranded=rescue, device_grouping=on_device)
            results.append(eng.cotr_corr_multiscale(img_a, img_b, zooms, 1, max_corrs=90, queries_a=queries.copy(), force=True))
        assert results[0].shape == results[1].shape and results[0].shape[0] > 3
        assert np.array_equal(results[0], results[1])
    # the kernel alone, against a direct numpy restatement of the walk
    from cotr_b200 import capi
    n = 3000
    pts = rs.uniform(0, 100, (n, 4))
    centre = rs.uniform(0, 100, (n, 4))
    half = rs.uniform(2, 15, (n, 1))
    boxes = np.stack([centre[:, 0] - half[:, 0], centre[:, 0] + half[:, 0], centre[:, 1] - half[:, 0], centre[:, 1] + half[:, 0],
                      centre[:, 2] - 3 * half[:, 0], centre[:, 2] + 3 * half[:, 0], centre[:, 3] - 3 * half[:, 0], centre[:, 3] + 3 * half[:, 0]], axis=1)
    squad, rank, n_squads = capi.group_tasks(pts, boxes, 32, 20, "cuda")
    free = np.ones(n, dtype=bool)
    ref_squad = -np.ones(n, dtype=np.int32); ref_rank = -np.ones(n, dtype=np.int32)
    made = 0
    for i in range(n):
        if not free[i]:
            continue
        free[i] = False
        ref_squad[i] = made; ref_rank[i] = 0
        b = boxes[i]
        fits = ((pts[:, 0] > b[0]) & (pts[:, 0] < b[1]) & (pts[:, 1] > b[2]) & (pts[:, 1] < b[3]) &
                (pts[:, 2] > b[4]) & (pts[:, 2] < b[5]) & (pts[:, 3] > b[6]) & (pts[:, 3] < b[7]))
        loads = np.where(fits & free)[0][:20]
        ref_squad[loads] = made; ref_rank[loads] = 1 + np.arange(len(loads))
        free[loads] = False
        made += 1
        if made >= 32:
            break
    assert n_squads == made and np.array_equal(squad, ref_squad) and np.array_equal(rank, ref_rank)
