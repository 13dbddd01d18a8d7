"""Mutual nearest-neighbour matching of keypoints for engine outputs (demo_guided_matching.py:48-62), on the device.

The demo takes the predictions of the zoom-in engines in both directions, finds for every prediction the nearest
keypoint of the other image (scipy.spatial.distance_matrix + np.argmin, fp64) and keeps the pairs that choose each other
with a Python double loop.  `mutual_nearest` gives the same result from one cotr_mutual_nearest call, without the
K_a x K_b distance matrices.  COTR.match_keypoints does the whole step, decode included, for an image set, at the first
zoom level; `match_keypoints_multiscale` does it through every zoom level of the demo.
"""
import numpy as np
import torch

from .. import capi
from . import refinement_task
from .inference_helper import dense_flow_maps, get_patch_centered_at, stretch_to_square, to_square_patches
from .refinement_task import crop_scales
from .sparse_engine import _exact_point


def mutual_nearest(corrs_a_b, kp_b, corrs_b_a, kp_a, device="cuda"):
    """corrs_a_b: (K_a,2) predicted pixels in b of a's keypoints (an engine's corrs[:, 2:]), kp_b: (K_b,2) b's keypoints,
    corrs_b_a / kp_a the other direction -> the demo's final_matches as an (M,2) int64 array of (index into kp_a, index
    into kp_b), in ascending first index.  Ties and NaNs are decided as np.argmin decides them; an image without
    keypoints gives no matches (the demo raises there)."""
    corrs_a_b, kp_b, corrs_b_a, kp_a = (np.asarray(x, dtype=np.float64).reshape(-1, 2) for x in (corrs_a_b, kp_b, corrs_b_a, kp_a))
    assert corrs_a_b.shape[0] == kp_a.shape[0] and corrs_b_a.shape[0] == kp_b.shape[0], \
        "one prediction per keypoint: corrs_a_b must have len(kp_a) rows and corrs_b_a len(kp_b) rows"
    dev = torch.device(device)
    kpts = torch.from_numpy(np.concatenate([kp_a, kp_b])).to(dev)
    corr = torch.from_numpy(np.concatenate([corrs_a_b, corrs_b_a])).to(dev)
    _, match, count = capi.mutual_nearest(kpts, [0, kp_a.shape[0], kp_a.shape[0] + kp_b.shape[0]], [(0, 1)], corr)
    return match[:int(count.cpu()[0])].cpu().numpy().astype(np.int64)


# ---- the whole zoom-in for an image set -----------------------------------------------------------------------------

def _check_model(model):
    if not (getattr(model, 'supports_device_preprocess', False) and hasattr(model, 'native') and hasattr(model, 'attention_hooked')):
        raise RuntimeError("match_keypoints_multiscale runs on the native cotr_b200 COTR model (its dense pass, first guesses "
                           "and zoom-in walk are CUDA kernels of the library); got a model without them")
    if model.attention_hooked():
        raise RuntimeError("match_keypoints_multiscale does not fire attention hooks: remove them or use the engines' host loop")
    if next(model.parameters()).device.type != 'cuda':
        raise RuntimeError("match_keypoints_multiscale: the model is not on a CUDA device: call model.cuda() first")


def _check_keypoints(keypoints, n_images):
    """N (K_i,2) float32 / float64 keypoint sets as numpy arrays; a point the device walk cannot take exactly
    (sparse_engine._exact_point: non-finite, or float32 at or above 2^24 in magnitude) raises ValueError."""
    if len(keypoints) != n_images:
        raise ValueError(f"keypoints: {len(keypoints)} sets for {n_images} images")
    out = []
    for i, k in enumerate(keypoints):
        k = k.detach().cpu().numpy() if isinstance(k, torch.Tensor) else np.asarray(k)
        if k.dtype not in (np.float32, np.float64) or k.ndim != 2 or k.shape[1] != 2:
            raise ValueError(f"keypoints: set {i} must be a (K,2) float32 or float64 array, got {k.shape} {k.dtype}")
        bad = [j for j in range(k.shape[0]) if not _exact_point(k[j])]
        if bad:
            raise ValueError(f"keypoints: set {i} point {bad[0]} = {k[bad[0]]} cannot be walked exactly (non-finite, or float32 "
                             "at or above 2^24 in magnitude)")
        out.append(np.ascontiguousarray(k))
    return out


def _check_images(images, tiled=True):
    """-> the (H, W) of every image; uint8 HWC RGB arrays or tensors, and when `tiled` (mode 'tile') long side <= 2 x
    short side (to_square_patches)."""
    shapes = []
    for i, img in enumerate(images):
        ok = img.dtype == torch.uint8 if isinstance(img, torch.Tensor) else isinstance(img, np.ndarray) and img.dtype == np.uint8
        if not (ok and img.ndim == 3 and img.shape[2] == 3):
            raise ValueError(f"images: image {i} must be a uint8 H x W x 3 array or tensor, got {tuple(img.shape)} {img.dtype}")
        h, w = int(img.shape[0]), int(img.shape[1])
        if tiled and max(h, w) > 2 * min(h, w):
            raise NotImplementedError(f"images: image {i} is {h} x {w}; the dense pass tiles images whose long side is at most "
                                      "twice the short side (to_square_patches); mode='stretching' takes any shape")
        shapes.append((h, w))
    return shapes


def _check_pairs(pairs, n_images):
    p = pairs.detach().cpu().numpy() if isinstance(pairs, torch.Tensor) else np.asarray(pairs)
    if not (p.ndim == 2 and p.shape[1] == 2 and p.shape[0] >= 1 and p.dtype.kind in 'iu'):
        raise ValueError(f"pairs must be a non-empty (B,2) integer table, got shape {p.shape} dtype {p.dtype}")
    if not ((p >= 0) & (p < n_images)).all():
        raise ValueError(f"pairs: image index outside [0, {n_images})")
    return p.astype(np.int64)


def plan_groups(counts, pairs):
    """The walk's groups: for pair p = (a, b) the direction a -> b, then b -> a, each with its image's keypoints as
    consecutive tasks; a direction whose source image has no keypoints makes no group.  counts: keypoints per image.
    -> list of (pair, image_from, image_to, first task, count)."""
    groups, first = [], 0
    for p, (a, b) in enumerate(pairs):
        for f, t in ((a, b), (b, a)):
            if counts[f] > 0:
                groups.append((p, int(f), int(t), first, int(counts[f])))
                first += int(counts[f])
    return groups


def group_scales(below, shapes, groups):
    """(s_from, s_to) of every group from its two area counts (below[g] = pixels under THRESHOLD_AREA in the source and
    target confidence maps), as gen_tasks (sparse_engine.py:227-228) and RefinementTask.__init__ compute them."""
    out = []
    with np.errstate(divide='ignore', invalid='ignore'):
        for g, (_, f, t, _, _) in enumerate(groups):
            area_from = np.int64(below[g][0]) / (shapes[f][0] * shapes[f][1])
            area_to = np.int64(below[g][1]) / (shapes[t][0] * shapes[t][1])
            out.append(crop_scales(area_from, area_to))
    return out


def check_crops(groups, scales, shapes, zooms, first_guesses=None):
    """What the crops of the per-pair engine would raise, checked before the walk, group by group: a NaN scale (both
    areas 0) -> ValueError; with `first_guesses` ((n,2) fp64, given when one is not finite: the engine then keeps its host
    loop) the first crop around each of them, which raises ValueError / OverflowError on NaN / inf; a crop side below 2
    pixels -> RuntimeError (cotr_preprocess refuses it)."""
    for (p, f, t, first, count), (s_from, s_to) in zip(groups, scales):
        if any(s * z != s * z for z in zooms for s in (s_from, s_to)):
            raise ValueError('cannot convert float NaN to integer')
        if first_guesses is not None:
            for loc in first_guesses[first:first + count]:
                get_patch_centered_at(None, loc, s_to * zooms[0], False, shapes[t] + (3,))
        for z in zooms:
            for s, img in ((s_from, f), (s_to, t)):
                side = get_patch_centered_at(None, (0, 0), s * z, False, shapes[img] + (3,)).w
                if side < 2:
                    raise RuntimeError(f"match_keypoints_multiscale: pair {p}, {f} -> {t}: zoom {z} crops a {side}-pixel side out "
                                       f"of the {shapes[img][0]} x {shapes[img][1]} image {img}; crops must be at least 2 pixels")


@torch.no_grad()
def match_keypoints_multiscale(model, images, keypoints, pairs, zoom_ins=np.linspace(0.5, 0.0625, 4), batch_size=32, mode='tile'):
    """Mutual nearest-neighbour matches of keypoints across image pairs through the whole zoom-in of
    demo_guided_matching.py, on the device.  For pair p = (a, b) the results equal, bit for bit,

        eng = SparseEngine(model, batch_size, mode=mode, device_walk=True)
        c_ab = eng.cotr_corr_multiscale(img_a, img_b, zoom_ins, 1, max_corrs=len(kp_a), queries_a=kp_a, force=True)
        c_ba = eng.cotr_corr_multiscale(img_b, img_a, zoom_ins, 1, max_corrs=len(kp_b), queries_a=kp_b, force=True)
        mutual_nearest(c_ab[:, 2:], kp_b, c_ba[:, 2:], kp_a)

    mode: the engine's first-guess mode.  'tile' (the default) runs the dense pass on each image's square tiles and takes
    images whose long side is at most twice the short side.  'stretching' runs it once per direction on both images
    stretched to max(h, w) squares on the device, resizes the maps back to the images' shapes, and takes any shape; when
    an image of the pair is not square the first guesses and area counts then follow the engine's float32 arithmetic on
    the resized maps (cotr_dense_first_guess_f32).  The crops of the walk are always cut from the original images.
    images: N uint8 H x W x 3 RGB arrays or CUDA tensors (sizes may differ);
    keypoints: N (K_i,2) float32 or float64 (x, y) pixel arrays; pairs: (B,2) image indices.  -> KeypointMatches
    (cotr_b200.models.cotr_model): matches[p] (M_p,2) int64, corrs_ab[p] (K_a,2) / corrs_ba[p] (K_b,2) fp64 (c_ab[:, 2:],
    c_ba[:, 2:]), nearest_ab[p] / nearest_ba[p] int32, all device tensors.  An image without keypoints walks no
    direction from it, and its pairs get no matches.

    Every direction runs the dense pass of cotr_flow (or of the stretched squares) on the device and cotr_dense_first_guess;
    one small copy brings back the area counts, the crop scales are computed on the host, and one cotr_refine call
    walks every direction of every pair; cotr_mutual_nearest keeps the mutual matches and one last copy reads the B match
    counts.  Raises what the per-pair engine raises (ValueError on a NaN scale or prediction), refuses attention hooks,
    models without the native extensions and keypoints the device walk cannot take exactly."""
    from ..models.cotr_model import KeypointMatches
    if mode not in ('tile', 'stretching'):
        raise ValueError(f"mode must be 'tile' or 'stretching', got {mode!r}")
    zooms = [float(z) for z in zoom_ins]
    if not 1 <= len(zooms) <= 7:
        raise ValueError(f"zoom_ins: {len(zooms)} levels; the device walk takes 1 .. 7")
    if not (isinstance(batch_size, (int, np.integer)) and batch_size >= 1):
        raise ValueError(f"batch_size must be a positive integer, got {batch_size!r}")
    shapes = _check_images(images, tiled=mode == 'tile')
    kps = _check_keypoints(keypoints, len(images))
    pairs = _check_pairs(pairs, len(images))
    _check_model(model)
    counts = np.array([k.shape[0] for k in kps], dtype=np.int64)
    groups = plan_groups(counts, pairs)
    dev = next(model.parameters()).device

    # image i's keypoints in their own dtype (the first guesses clip in it) and widened to fp64 (the walk, the matching)
    kp_dev = [torch.from_numpy(k).to(dev) for k in kps]
    kp64 = torch.cat([k.to(torch.float64) for k in kp_dev]) if kps else torch.zeros((0, 2), dtype=torch.float64, device=dev)
    kp_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    n = sum(g[4] for g in groups)
    L = len(zooms)
    if n:
        img_dev = [img.to(dev).contiguous() if isinstance(img, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(img)).to(dev)
                   for img in images]
        patches, squares = {}, {}                     # per image, made on first use
        loc_to = torch.empty((n, 2), dtype=torch.float64, device=dev)
        below = torch.empty((len(groups), 2), dtype=torch.int64, device=dev)
        for g, (_, f, t, first, count) in enumerate(groups):
            stretch = mode == 'stretching' and any(shapes[i][0] != shapes[i][1] for i in (f, t))
            if stretch:
                for i in (f, t):
                    if i not in squares:
                        squares[i] = stretch_to_square(model, img_dev[i])
                sq_f, sq_t = squares[f], squares[t]
                (flow_f, conf_f), (_, conf_t) = dense_flow_maps(model, sq_f, sq_t, to_square_patches(sq_f), to_square_patches(sq_t))
                flow_f, conf_f, conf_t = (model.resize_maps(m, shapes[i]) for m, i in ((flow_f, f), (conf_f, f), (conf_t, t)))
            else:
                for i in (f, t):
                    if i not in patches:
                        patches[i] = to_square_patches(img_dev[i])
                (flow_f, conf_f), (_, conf_t) = dense_flow_maps(model, img_dev[f], img_dev[t], patches[f], patches[t])
            capi.dense_first_guess(flow_f, conf_f, conf_t, kp_dev[f], loc_to[first:first + count], below[g], f32_maps=stretch)
        # one copy: the area counts and whether a first guess is not finite (a NaN / inf dense prediction)
        host = torch.cat([below.view(-1), (~torch.isfinite(loc_to)).any().view(1).long()]).cpu().numpy()
        scales = group_scales(host[:-1].reshape(-1, 2), shapes, groups)
        check_crops(groups, scales, shapes, zooms, loc_to.cpu().numpy() if host[-1] else None)
        loc_from = torch.cat([kp64[kp_off[f]:kp_off[f + 1]] for _, f, _, _, _ in groups])
        table = [(f, t, first, count, float(s_f), float(s_t)) for (_, f, t, first, count), (s_f, s_t) in zip(groups, scales)]
        # force: max_corrs = K per direction, so the engine's stop can only fall after a group's last chunk
        history, _, _, _, (code, _, _) = model.native().refine(img_dev, table, zooms, batch_size, 8, n,
                                                               refinement_task.THRESHOLD_PIXELS_RELATIVE, loc_from, loc_to)
        if code != 0:
            raise ValueError('NaN in prediction' if code == 1 else 'non-finite position in the zoom-in walk')
        corr = history[:, L].contiguous()             # conclude(force=True) returns best_loc_to
        nearest, match, n_match = capi.mutual_nearest(kp64, kp_off, pairs, corr)
        n_match = n_match.cpu().numpy()
    else:
        corr = torch.zeros((0, 2), dtype=torch.float64, device=dev)
        nearest = torch.zeros((0,), dtype=torch.int32, device=dev)
        match = torch.zeros((0, 2), dtype=torch.int32, device=dev)
        n_match = np.zeros(len(pairs), dtype=np.int64)
    rows = counts[pairs].reshape(-1)                  # rows of contexts 0, 1, ..., 2B-1 (cotr_mutual_nearest's layout)
    ctx_off = np.concatenate([[0], np.cumsum(rows)])
    match = match.long()
    res = KeypointMatches([], [], [], [], [])
    for p in range(len(pairs)):
        ab, ba, end = int(ctx_off[2 * p]), int(ctx_off[2 * p + 1]), int(ctx_off[2 * p + 2])
        res.matches.append(match[ab:ab + int(n_match[p])])
        res.corrs_ab.append(corr[ab:ba]); res.corrs_ba.append(corr[ba:end])
        res.nearest_ab.append(nearest[ab:ba]); res.nearest_ba.append(nearest[ba:end])
    return res
