"""Numpy restatement of keypoint matching (cotr_match_keypoints / cotr_mutual_nearest in include/cotr_b200.h).

Formulas are the reference's first zoom level with the whole image as the patch (x = y = 0, w = W, h = H):
  * query, COTR/inference/refinement_task.py:110: q = fp32(fp64(x) / (2 W_left)), fp32(fp64(y) / H_left);
  * pixel, scale_to_loc, refinement_task.py:145-151: raw[0] = (raw[0] - 0.5) * 2 in the prediction's fp32, then
    raw * [w, h] + [x, y] in fp64: c = fp64(fp32((p_x - 0.5) * 2)) * W_right, fp64(p_y) * H_right;
  * nearest, demo_guided_matching.py:48,50: np.argmin(scipy.spatial.distance_matrix(corrs, kp), axis=1), i.e. the first
    index of the smallest sqrt(dx*dx + dy*dy) in fp64 (dx = kp_x - c_x), a NaN distance winning (np.argmin's rule);
  * mutual, demo_guided_matching.py:53-61: (i, nearest_ab[i]) in ascending i where nearest_ba[nearest_ab[i]] == i.
Rows of a call: pair p = (a, b) uses context 2p = [a | b], which decodes a's keypoints, and 2p+1 = [b | a], which decodes
b's, packed in context order.  An image without keypoints gives nearest = -1 (the reference raises there).
"""
import numpy as np


def queries(kp, size):
    """(K,2) pixels of the left image, size (W, H) -> (K,2) fp32 canvas queries."""
    kp = np.asarray(kp, dtype=np.float64).reshape(-1, 2)
    W, H = (float(v) for v in size)
    return np.stack([kp[:, 0] / (2.0 * W), kp[:, 1] / H], axis=1).astype(np.float32)


def pixels(pred, size):
    """(K,2) fp32 predictions on the canvas, size (W, H) of the right image -> (K,2) fp64 pixels in the right image."""
    pred = np.asarray(pred, dtype=np.float32).reshape(-1, 2)
    x = (pred[:, 0] - np.float32(0.5)) * np.float32(2.0)
    return np.stack([x.astype(np.float64) * float(size[0]), pred[:, 1].astype(np.float64) * float(size[1])], axis=1)


def nearest(corr, kp, rows_per_block=256):
    """(R,2) fp64 points, (K,2) keypoints -> (R,) int64 index of the nearest keypoint (-1 when K == 0), decided exactly as
    np.argmin over the rows of scipy's distance_matrix; computed in row blocks so that no R x K matrix is held."""
    corr = np.asarray(corr, dtype=np.float64).reshape(-1, 2)
    kp = np.asarray(kp, dtype=np.float64).reshape(-1, 2)
    out = np.full(corr.shape[0], -1, dtype=np.int64)
    if kp.shape[0] == 0:
        return out
    for r0 in range(0, corr.shape[0], rows_per_block):
        c = corr[r0:r0 + rows_per_block]
        dx = kp[None, :, 0] - c[:, None, 0]
        dy = kp[None, :, 1] - c[:, None, 1]
        out[r0:r0 + rows_per_block] = np.argmin(np.sqrt(dx * dx + dy * dy), axis=1)
    return out


def mutual(nearest_ab, nearest_ba):
    """The demo's final_matches: (M,2) int64 (i, j) with j = nearest_ab[i] and nearest_ba[j] == i, ascending i."""
    ab = np.asarray(nearest_ab, dtype=np.int64)
    ba = np.asarray(nearest_ba, dtype=np.int64)
    i = np.arange(ab.shape[0])
    ok = ab >= 0
    ok[ok] = ba[ab[ok]] == i[ok]
    return np.stack([i[ok], ab[ok]], axis=1).astype(np.int64)


def match_pair(corr_ab, kp_b, corr_ba, kp_a):
    """One pair: (nearest_ab, nearest_ba, matches)."""
    n_ab, n_ba = nearest(corr_ab, kp_b), nearest(corr_ba, kp_a)
    return n_ab, n_ba, mutual(n_ab, n_ba)


# ---- cases whose decisions a plain comparison of squared distances, or a float32 one, would get wrong -------------------
def tie_grid(n_side, seed=0):
    """Keypoints on an n_side x n_side integer grid (shuffled) and points at integer and half-integer positions: many
    rows have 2 or 4 candidates at exactly the same distance."""
    rs = np.random.RandomState(seed)
    g = np.stack(np.meshgrid(np.arange(n_side), np.arange(n_side)), axis=-1).reshape(-1, 2).astype(np.float64)
    kp = g[rs.permutation(g.shape[0])]
    corr = rs.randint(-1, 2 * n_side + 1, size=(4 * n_side, 2)) * 0.5
    return corr, kp


def sqrt_collisions(n, seed=0, spread=1e3):
    """n points, each with two keypoints at distinct squared distances s_far > s_near whose fp64 sqrt rounds to the same
    value; the s_far keypoint has the lower index, so np.argmin picks it.  Pairs sit in different candidate lanes and,
    for n > 1024 / 2, in different staged chunks of the device kernel."""
    rs = np.random.RandomState(seed)
    corr, near, far = [], [], []
    while len(corr) < n:
        c = np.array([len(corr) * 4 * spread + rs.uniform(-1.0, 1.0), rs.uniform(-spread, spread)])   # own pair nearest
        a = rs.uniform(1.0, spread)
        dy = np.ldexp(rs.uniform(0.5, 1.0), int(np.floor(np.log2(a))) - 25)
        kn = np.array([c[0] + a, c[1]])
        kf = np.array([c[0] + a, c[1] + dy])
        dxn, dyn = kn - c
        dxf, dyf = kf - c
        sn, sf = dxn * dxn + dyn * dyn, dxf * dxf + dyf * dyf
        if sf > sn and np.sqrt(sf) == np.sqrt(sn):
            corr.append(c); near.append(kn); far.append(kf)
    n = len(corr)
    kp = np.empty((2 * n + 3, 2))
    kp[:n] = np.array(far)                # lower indices: the larger squared distances
    kp[n:2 * n] = np.array(near)[::-1]
    kp[2 * n:] = [1e9, 1e9]               # far away filler, so the pairs straddle lanes
    return np.array(corr), kp


def sqrt_collisions_in_lanes(n_chunk, n_cross, seed=0, lanes=4, chunk=1024):
    """Collision pairs (see sqrt_collisions) whose two keypoints the device's nearest kernel scans in the same candidate
    lane (indices congruent mod `lanes`), far before near: n_chunk pairs with near = far + lanes inside one staged chunk
    of `chunk` keypoints, and n_cross pairs with near = far + chunk + lanes in the next chunk.  There the lane itself
    must keep the far keypoint on an equal sqrt; the merge of the lanes never sees the near one.
    -> (corr, kp, far, near): far[i] is the index np.argmin picks for point i, near[i] its collision partner."""
    step = 2 * lanes
    assert step * (n_chunk - 1) + lanes < chunk and step * (n_cross - 1) + 1 + lanes < chunk
    corr, pairs_kp = sqrt_collisions(n_chunk + n_cross, seed)
    n = n_chunk + n_cross
    far_kp, near_kp = pairs_kp[:n], pairs_kp[n:2 * n][::-1]
    base = chunk                                   # the crossing pairs start in the second chunk
    kp = np.full((base + 2 * chunk, 2), 1e9)
    far, near = np.empty(n, dtype=np.int64), np.empty(n, dtype=np.int64)
    for i in range(n):
        f, d = (step * i, lanes) if i < n_chunk else (base + step * (i - n_chunk) + 1, chunk + lanes)
        kp[f], kp[f + d] = far_kp[i], near_kp[i]
        far[i], near[i] = f, f + d
    return corr, kp, far, near
