"""Dense first-guess pass and patch geometry of the zoom-in loop (reference: COTR/inference/inference_helper.py).

Observable behaviour follows the reference function by function (cited below); the implementation differs where the
reference burns host time for nothing: the 131 072-query grid is built vectorised instead of by a Python double loop
(:116-122), and when the model exposes `encode_context` / `decode` (cotr_b200.models.COTR) the cycle pass of
`cotr_corr_base` re-uses the encoded image pair instead of re-running backbone + encoder (:197-198).
"""
import warnings

import cv2
import numpy as np
import PIL.Image
import torch
from torchvision.transforms import functional as tvtf

from ..utils import utils
from ..utils.constants import MAX_SIZE
from ..utils.utils import ImagePatch

THRESHOLD_SPARSE = 0.02
THRESHOLD_PIXELS_RELATIVE = 0.02
BASE_ZOOM = 1.0
DEVICE_DENSE_POST = True   # native model: finish the dense pass on the device (cotr_dense_postprocess); False = host path
DEVICE_FLOW_MERGE = True   # native model: patch affine + float_image_resize + tile merge on the device (cotr_flow_tile_merge)
DEVICE_STRETCH = True      # native model: 'stretching' mode stretches, dense-passes and resizes back on the device
THRESHOLD_AREA = 0.02
LARGE_GPU = True

_MEAN = (0.485, 0.456, 0.406)
_STD = (0.229, 0.224, 0.225)


def find_prediction_loop(arr):
    """Rows between the first earlier occurrence of the last row and the end (exclusive) (:22-28)."""
    assert arr.shape[1] == 2, 'requires shape (N, 2)'
    same = np.all(arr[:-1] == arr[-1], axis=1)
    first = int(np.flatnonzero(same)[0])
    return arr[first:-1]


def two_images_side_by_side(img_a, img_b):
    """(h,w,c) + (h,w,c) -> (h,2w,c), left = a (:31-38)."""
    assert img_a.shape == img_b.shape, f'{img_a.shape} vs {img_b.shape}'
    assert img_a.dtype == img_b.dtype
    return np.concatenate([img_a, img_b], axis=1)


def to_square_patches(img):
    """One square for a square image, two overlapping corner squares when long <= 2*short (:41-58)."""
    h, w, _ = img.shape
    size = min(h, w)
    if max(h, w) == size:
        return [ImagePatch(img[:size, :size], 0, 0, size, size, w, h)]
    if max(h, w) <= 2 * size:
        warnings.warn('Spatial smoothness in dense optical flow is lost, but sparse matching and triangulation should be fine')
        return [ImagePatch(img[:size, :size], 0, 0, size, size, w, h),
                ImagePatch(img[-size:, -size:], w - size, h - size, size, size, w, h)]
    raise NotImplementedError


def merge_flow_patches(corrs):
    """Per pixel keep the tile with the smallest cycle confidence; ties go to the later tile (:61-75)."""
    oh, ow = corrs[0].oh, corrs[0].ow
    confidence = np.full((oh, ow), 100.0)
    flow = np.zeros((oh, ow, 2))
    cmap = np.full((oh, ow), -1.0)
    for i, c in enumerate(corrs):
        conf_i = np.full((c.oh, c.ow), 100.0)
        flow_i = np.zeros((c.oh, c.ow, 2))
        rows, cols = slice(c.y, c.y + c.h), slice(c.x, c.x + c.w)
        conf_i[rows, cols] = c.patch[..., 2]
        flow_i[rows, cols] = c.patch[..., :2]
        take = conf_i <= confidence
        confidence[take] = conf_i[take]
        flow[take] = flow_i[take]
        cmap[take] = i
    return flow, confidence, cmap


def get_patch_centered_at(img, pos, scale=1.0, return_content=True, img_shape=None):
    """Even-sized square crop of side short*scale around pos=[x,y]; shifted (not shrunk) to stay inside (:78-102)."""
    if img_shape is None:
        img_shape = img.shape
    h, w, _ = img_shape
    scale = min(max(scale, 0.0), 1.0)          # np.clip on a scalar, without the array machinery (called ~10^5 times per run)
    size = min(h, w) * scale
    size = int((size // 2) * 2)
    top = int(pos[1] - size // 2)        # int() truncates toward zero, like the reference
    left = int(pos[0] - size // 2)
    top = max(top, 0)
    left = max(left, 0)
    if top + size > h:
        top = h - size
    if left + size > w:
        left = w - size
    content = img[top:top + size, left:left + size] if return_content else None
    return ImagePatch(content, left, top, size, size, w, h)


def _to_network_canvas(img_a, img_b):
    """Two square uint8 crops -> normalised (3,256,512) float32 tensor (:108-113, refinement_task.py:117-120)."""
    assert img_a.shape[0] == img_a.shape[1]
    assert img_b.shape[0] == img_b.shape[1]
    a = np.array(PIL.Image.fromarray(img_a).resize((MAX_SIZE, MAX_SIZE), resample=PIL.Image.BILINEAR))
    b = np.array(PIL.Image.fromarray(img_b).resize((MAX_SIZE, MAX_SIZE), resample=PIL.Image.BILINEAR))
    canvas = two_images_side_by_side(a, b)
    return tvtf.normalize(tvtf.to_tensor(canvas), _MEAN, _STD).float()


def _dense_grid():
    """Queries (j/512, i/256) for every canvas pixel corner, row-major, float64 like the reference's list of lists."""
    xs = np.arange(MAX_SIZE * 2) / (MAX_SIZE * 2)
    ys = np.arange(MAX_SIZE) / MAX_SIZE
    grid = np.empty((MAX_SIZE, MAX_SIZE * 2, 2))
    grid[..., 0] = xs[None, :]
    grid[..., 1] = ys[:, None]
    return grid


def _model_device(model):
    return next(model.parameters()).device


def _dense_pass(model, img_a, img_b):
    """One forward with all 131 072 grid queries + cycle-consistency confidence (:106-145)."""
    device = _model_device(model)
    img = _to_network_canvas(img_a, img_b)[None].to(device)
    grid = _dense_grid()
    if LARGE_GPU:
        try:
            queries = torch.from_numpy(grid.reshape(-1, 2))[None].float().to(device)
            pred = model.forward(img, queries)['pred_corrs'].detach()
        except Exception:
            assert 0, 'set LARGE_GPU to False'
        if DEVICE_DENSE_POST and pred.is_cuda and hasattr(model, 'dense_postprocess'):
            # the native model finishes the pass on the device (cycle grid_sample, confidence, per-half x remap)
            corr = model.dense_postprocess(pred).cpu().numpy()[0]
            return corr[:, :MAX_SIZE, :], corr[:, MAX_SIZE:, :]
        out = pred.cpu().numpy()[0].reshape(MAX_SIZE, MAX_SIZE * 2, -1)
    else:
        if hasattr(model, 'encode_context'):
            ctx = model.encode_context(img, reuse=True)
            rows = [model.decode(ctx, torch.from_numpy(r)[None].float().to(device))['pred_corrs'].detach().cpu().numpy()[0] for r in grid]
        else:
            rows = [model.forward(img, torch.from_numpy(r)[None].float().to(device))['pred_corrs'].detach().cpu().numpy()[0] for r in grid]
        out = np.array(rows)
    in_grid = torch.from_numpy(grid).float()[None] * 2 - 1
    out_grid = torch.from_numpy(out).float()[None] * 2 - 1
    cycle_grid = torch.nn.functional.grid_sample(out_grid.permute(0, 3, 1, 2), out_grid).permute(0, 2, 3, 1)
    confidence = torch.norm(cycle_grid[0, ...] - in_grid[0, ...], dim=-1)
    corr = out_grid[0].clone()
    corr[:, :MAX_SIZE, 0] = corr[:, :MAX_SIZE, 0] * 2 - 1      # left half answers in the right image
    corr[:, MAX_SIZE:, 0] = corr[:, MAX_SIZE:, 0] * 2 + 1      # right half answers in the left image
    corr = torch.cat([corr, confidence[..., None]], dim=-1).numpy()
    return corr[:, :MAX_SIZE, :], corr[:, MAX_SIZE:, :]


def _patch_corners_ndc(p):
    """First three corners of the patch rectangle in [-1,1] coordinates of the full image."""
    px = np.array([[p.x, p.y], [p.x + p.w, p.y], [p.x + p.w, p.y + p.h], [p.x, p.y + p.h]])
    return ((px / np.array([p.ow, p.oh])) * 2 + np.array([-1, -1]))[:3].astype(np.float32)


def cotr_patch_flow_exhaustive(model, patches_a, patches_b):
    """Dense pass for every (tile of a, tile of b), predictions re-expressed in full-image coordinates (:105-165)."""
    unit = np.array([[-1, -1], [1, -1], [1, 1]], dtype=np.float32)
    corrs_a, corrs_b = [], []
    for p_i in patches_a:
        for p_j in patches_b:
            c_i, c_j = _dense_pass(model, p_i.patch, p_j.patch)
            to_j = cv2.getAffineTransform(unit, _patch_corners_ndc(p_j))
            to_i = cv2.getAffineTransform(unit, _patch_corners_ndc(p_i))
            c_i[..., :2] = c_i[..., :2] @ to_j[:2, :2] + to_j[:, 2]
            c_j[..., :2] = c_j[..., :2] @ to_i[:2, :2] + to_i[:, 2]
            c_i = utils.float_image_resize(c_i, (p_i.h, p_i.w))
            c_j = utils.float_image_resize(c_j, (p_j.h, p_j.w))
            corrs_a.append(ImagePatch(c_i, p_i.x, p_i.y, p_i.w, p_i.h, p_i.ow, p_i.oh))
            corrs_b.append(ImagePatch(c_j, p_j.x, p_j.y, p_j.w, p_j.h, p_j.ow, p_j.oh))
    return corrs_a, corrs_b


def _resample(img_src, corr):
    src = utils.np_img_to_torch_img(img_src)[None].float()
    return utils.torch_img_to_np_img(torch.nn.functional.grid_sample(src, torch.from_numpy(corr)[None].float())[0])


def _affine_terms(to):
    """cv2 2x3 affine `to` as the reference applies it (`c[..., :2] @ to[:2, :2] + to[:, 2]`, :157-158) ->
    [a0..a5] with x' = a0 x + a1 y + a2, y' = a3 x + a4 y + a5."""
    return [to[0, 0], to[1, 0], to[0, 2], to[0, 1], to[1, 1], to[1, 2]]


def dense_flow_maps(model, img_a_dev, img_b_dev, patches_a, patches_b):
    """cotr_patch_flow_exhaustive + merge_flow_patches with every per-tile array left on the device: the tile canvases
    are cut and resized by cotr_preprocess (bit for bit the PIL canvases of _to_network_canvas), the dense pass'
    (256,512,3) answer is split into its halves by pointer, mapped / resized / merged by cotr_flow_tile_merge.
    img_*_dev: uint8 HWC CUDA images; patches_*: their to_square_patches.  -> ((flow_a (H_a,W_a,2), conf_a (H_a,W_a)),
    (flow_b, conf_b)) fp32 device tensors."""
    device = _model_device(model)
    unit = np.array([[-1, -1], [1, -1], [1, 1]], dtype=np.float32)
    canv = {}
    for key, p in (("a", patches_a[0]), ("b", patches_b[0])):
        canv[key] = (torch.empty((p.oh, p.ow, 2), dtype=torch.float32, device=device), torch.empty((p.oh, p.ow), dtype=torch.float32, device=device))
    first = True
    queries = torch.from_numpy(_dense_grid().reshape(-1, 2))[None].float().to(device)
    for p_i in patches_a:
        for p_j in patches_b:
            rect = np.array([[p_i.x, p_i.y, p_i.w, p_j.x, p_j.y, p_j.w]], dtype=np.int32)
            img = model.preprocess_canvases(img_a_dev, img_b_dev, rect)
            pred = model.forward(img, queries)['pred_corrs'].detach()
            corr = model.dense_postprocess(pred)[0]                           # (256,512,3) on the device
            to_j = cv2.getAffineTransform(unit, _patch_corners_ndc(p_j))
            to_i = cv2.getAffineTransform(unit, _patch_corners_ndc(p_i))
            model.flow_tile_merge(corr[:, :MAX_SIZE, :], _affine_terms(to_j), p_i, canv["a"][0], canv["a"][1], first)
            model.flow_tile_merge(corr[:, MAX_SIZE:, :], _affine_terms(to_i), p_j, canv["b"][0], canv["b"][1], first)
            first = False
    return canv["a"], canv["b"]


def _cotr_flow_device(model, img_a, img_b, patches_a, patches_b):
    device = _model_device(model)
    maps = dense_flow_maps(model, torch.from_numpy(np.ascontiguousarray(img_a)).to(device),
                           torch.from_numpy(np.ascontiguousarray(img_b)).to(device), patches_a, patches_b)
    # the reference's arrays are float64
    return [(flow.cpu().numpy().astype(np.float64), conf.cpu().numpy().astype(np.float64)) for flow, conf in maps]


def _device_pixels(img):
    return isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3


def flow_on_device(model, img_a, img_b):
    """Whether cotr_flow's maps come from the device path (dense_flow_maps) for this model and these images."""
    return (LARGE_GPU and DEVICE_DENSE_POST and DEVICE_FLOW_MERGE and hasattr(model, 'flow_tile_merge') and hasattr(model, 'dense_postprocess')
            and hasattr(model, 'preprocess_canvases') and _device_pixels(img_a) and _device_pixels(img_b)
            and _model_device(model).type == 'cuda')


def cotr_flow_maps(model, img_a, img_b):
    """The maps of cotr_flow without the two warped images: (corr_a, con_a, corr_b, con_b), float64."""
    patches_a, patches_b = to_square_patches(img_a), to_square_patches(img_b)
    if flow_on_device(model, img_a, img_b):
        (corr_a, con_a), (corr_b, con_b) = _cotr_flow_device(model, img_a, img_b, patches_a, patches_b)
    else:
        corrs_a, corrs_b = cotr_patch_flow_exhaustive(model, patches_a, patches_b)
        corr_a, con_a, _ = merge_flow_patches(corrs_a)
        corr_b, con_b, _ = merge_flow_patches(corrs_b)
    return corr_a, con_a, corr_b, con_b


def cotr_flow(model, img_a, img_b):
    """Dense correspondence maps in [-1,1] + cycle confidence + warped images, both directions (:168-182)."""
    corr_a, con_a, corr_b, con_b = cotr_flow_maps(model, img_a, img_b)
    return corr_a, con_a, _resample(img_b, corr_a), corr_b, con_b, _resample(img_a, corr_b)


def stretch_to_square(model, img_dev):
    """A uint8 HWC CUDA image resized to max(h, w) squared on the device, bit for bit sparse_engine.stretch_to_square_np
    (a square image is returned as it is: Pillow would copy it)."""
    h, w = int(img_dev.shape[0]), int(img_dev.shape[1])
    return img_dev if h == w else model.resize_image(img_dev, (max(h, w), max(h, w)))


def stretched_flow_maps(model, img_a_dev, img_b_dev, shape_a, shape_b):
    """'stretching' mode's dense first guess on the device: both uint8 CUDA images stretched to max(h, w) squares
    (COTR.resize_image, bit for bit stretch_to_square_np), one dense pass on the squares (each is a single tile), and the
    flow and confidence maps resized back to the original (H, W) shapes (COTR.resize_maps, bit for bit
    utils.float_image_resize) -> ((flow_a (H_a,W_a,2), conf_a (H_a,W_a)), (flow_b, conf_b)) fp32 CUDA tensors."""
    sq_a, sq_b = stretch_to_square(model, img_a_dev), stretch_to_square(model, img_b_dev)
    maps = dense_flow_maps(model, sq_a, sq_b, to_square_patches(sq_a), to_square_patches(sq_b))
    return tuple((model.resize_maps(flow, shape), model.resize_maps(conf, shape)) for (flow, conf), shape in zip(maps, (shape_a, shape_b)))


def _sparse_pass(model, img_a, img_b, queries):
    """Forward + cycle forward on the predictions (:186-204); the image pair is encoded once when the model allows."""
    device = _model_device(model)
    img = _to_network_canvas(img_a, img_b)[None].to(device)
    q = torch.from_numpy(queries)[None].float().to(device)
    if hasattr(model, 'encode_context'):
        ctx = model.encode_context(img, reuse=True)
        out = model.decode(ctx, q)['pred_corrs'].clone().detach()
        cycle = model.decode(ctx, out)['pred_corrs'].clone().detach()
    else:
        out = model.forward(img, q)['pred_corrs'].clone().detach()
        cycle = model.forward(img, out)['pred_corrs'].clone().detach()
    q_np = q.cpu().numpy()[0]
    conf = np.linalg.norm(q_np - cycle.cpu().numpy()[0], axis=1, keepdims=True)
    return np.concatenate([out.cpu().numpy()[0], conf], axis=1)


def cotr_corr_base(model, img_a, img_b, queries_a):
    """Known-scale sparse pass: per tile pair predict + cycle error, keep the best tile pair per query (:185-232)."""
    per_pair = []
    for p_i in to_square_patches(img_a):
        for p_j in to_square_patches(img_b):
            q = queries_a.copy()
            inside = (q[:, 0] >= p_i.x) & (q[:, 1] >= p_i.y) & (q[:, 0] <= p_i.x + p_i.w) & (q[:, 1] <= p_i.y + p_i.h)
            q[:, 0] -= p_i.x
            q[:, 1] -= p_i.y
            q[:, 0] /= 2 * p_i.w
            q[:, 1] /= p_i.h
            pred = _sparse_pass(model, p_i.patch, p_j.patch, q)
            pred[~inside, 2] = np.inf
            pred[:, 0] -= 0.5
            pred[:, 0] *= 2 * p_j.w
            pred[:, 0] += p_j.x
            pred[:, 1] *= p_j.h
            pred[:, 1] += p_j.y
            per_pair.append(pred)
    per_query = np.stack(per_pair).transpose(1, 0, 2)
    best = np.array([cands[np.argmin(cands[..., 2], axis=0)] for cands in per_query])[..., :2]
    return np.concatenate([queries_a, best], axis=1)


def triangulate_corr(corr, from_shape, to_shape):
    """Densify sparse correspondences (:293-308): Delaunay triangulation of the source points on the host (scipy, as
    in the reference), then barycentric interpolation of the target coordinates over every triangle.  The reference
    renders the triangles with OpenGL through vispy (and is `None` without vispy); here the rendering is a CUDA
    rasteriser behind the C ABI (cotr_rasterize_triangles): pixel (x, y) is sampled at its centre (x + 0.5, y + 0.5)
    like GL does.  Returns (H_from, W_from, 2) float32 target pixel coordinates, zeros outside the triangulated hull."""
    from scipy.spatial import Delaunay
    from .. import capi
    if not torch.cuda.is_available():
        raise RuntimeError("triangulate_corr renders on the GPU (cotr_rasterize_triangles); no CUDA device is visible")
    corr = np.asarray(corr, dtype=np.float64)
    h, w = from_shape[:2]
    tri = Delaunay(corr[:, :2])
    verts = corr[tri.simplices].astype(np.float32)                   # (n_tri, 3, [x_from, y_from, x_to, y_to])
    out = capi.rasterize_triangles(torch.from_numpy(np.ascontiguousarray(verts)).cuda(), h, w)
    return out.cpu().numpy()
