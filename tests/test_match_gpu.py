"""GPU: keypoint matching - cotr_mutual_nearest against the numpy oracle (oracle/match_oracle.py, itself pinned to scipy
and the demo's loop by test_match_cpu.py), and cotr_match_keypoints / COTR.match_keypoints bitwise against the
composition of existing public calls: encode_context_pairs, a ragged decode of oracle-built queries, the oracle's pixel
formula and rule."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import fixtures
from oracle import match_oracle as mo

pytestmark = pytest.mark.gpu

TC, SIMT = 0, 1
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DISK_A = "disk_kpts_21526113_4379776807.npy"      # image 1033 x 771
DISK_B = "disk_kpts_21126421_4537535153.npy"      # image 694 x 1061


def _disk(name):
    return np.load(os.path.join(GOLDEN, name)).astype(np.float64)


def _layout(kps, pairs):
    """Rows of contexts 0 .. 2B-1: (left image, right image) per context."""
    return [(a, b) if c == 0 else (b, a) for a, b in pairs for c in (0, 1)]


def _check_mutual_nearest(kps, pairs, corrs):
    """kps: N keypoint arrays, pairs: B (a, b), corrs: 2B arrays (one per context, rows = the left image's keypoints)."""
    from cotr_b200 import capi
    ctxs = _layout(kps, pairs)
    assert [len(c) for c in corrs] == [len(kps[l]) for l, _ in ctxs]
    off = np.concatenate([[0], np.cumsum([len(k) for k in kps])]).astype(np.int64)
    kpts = torch.from_numpy(np.concatenate([np.asarray(k, np.float64).reshape(-1, 2) for k in kps])).cuda()
    corr = torch.from_numpy(np.concatenate([np.asarray(c, np.float64).reshape(-1, 2) for c in corrs])).cuda()
    nearest, match, count = capi.mutual_nearest(kpts, off, pairs, corr)
    nearest, match, count = nearest.cpu().numpy(), match.cpu().numpy(), count.cpu().numpy()
    row = 0
    for p in range(len(pairs)):
        (a, b), rows_a, rows_b = pairs[p], len(kps[pairs[p][0]]), len(kps[pairs[p][1]])
        n_ab, n_ba, ref = mo.match_pair(corrs[2 * p], kps[b], corrs[2 * p + 1], kps[a])
        assert np.array_equal(nearest[row:row + rows_a], n_ab), (p, "ab")
        assert np.array_equal(nearest[row + rows_a:row + rows_a + rows_b], n_ba), (p, "ba")
        assert count[p] == len(ref) and np.array_equal(match[row:row + count[p]], ref), p
        row += rows_a + rows_b
    assert row == corr.shape[0]
    return count


def _random_corrs(kps, pairs, rs, lo=0.0, hi=1000.0):
    return [rs.uniform(lo, hi, (len(kps[l]), 2)) for l, _ in _layout(kps, pairs)]


def test_mutual_nearest_sizes(built_lib):
    """0, 1, 255, 256, 257 and 4099 keypoints per side, all 36 ordered pairs (self-pairs included) in one call."""
    rs = np.random.RandomState(0)
    kps = [rs.uniform(0, 1000, (n, 2)) for n in (0, 1, 255, 256, 257, 4099)]
    pairs = [(a, b) for a in range(6) for b in range(6)]
    count = _check_mutual_nearest(kps, pairs, _random_corrs(kps, pairs, rs))
    assert count.sum() > 0


def test_mutual_nearest_repeats_and_self_pair(built_lib):
    rs = np.random.RandomState(1)
    kps = [rs.uniform(0, 500, (n, 2)) for n in (500, 700, 1300)]
    pairs = [(0, 1), (1, 0), (2, 2), (0, 1), (1, 2), (2, 0)]
    corrs = [kps[r][rs.randint(0, len(kps[r]), len(kps[l]))] + rs.normal(0, 3.0, (len(kps[l]), 2)) for l, r in _layout(kps, pairs)]
    assert _check_mutual_nearest(kps, pairs, corrs).sum() > 0


def test_mutual_nearest_exact_ties(built_lib):
    """Integer grids probed at integer and half-integer points (equal distances: the lowest index wins), and duplicate
    keypoints."""
    rs = np.random.RandomState(2)
    c0, g0 = mo.tie_grid(40, seed=3)
    c1, g1 = mo.tie_grid(33, seed=4)
    dup = np.concatenate([g1[:300], g1[:300][::-1], g1[:5]])
    kps = [g0, g1, dup]
    pairs = [(0, 1), (1, 2), (2, 0)]
    corrs = [np.concatenate([c0, c1])[rs.randint(0, len(c0) + len(c1), len(kps[l]))] for l, _ in _layout(kps, pairs)]
    _check_mutual_nearest(kps, pairs, corrs)


def test_mutual_nearest_sqrt_collisions(built_lib):
    """Distinct squared distances whose sqrt rounds equal: the lower index (the larger squared distance) wins, also when
    the two sit in different lanes and staged chunks."""
    corr, kp = mo.sqrt_collisions(700, seed=5)
    rs = np.random.RandomState(6)
    kps = [rs.uniform(0, 1e3, (700, 2)), kp]
    corrs = [corr, rs.uniform(0, 1e3, (len(kp), 2))]
    from cotr_b200 import capi
    _check_mutual_nearest(kps, [(0, 1)], corrs)
    # and the device picks the far keypoint of each collision pair
    off = [0, 700, 700 + len(kp)]
    nearest, _, _ = capi.mutual_nearest(torch.from_numpy(np.concatenate(kps)).cuda(), off, [(0, 1)],
                                        torch.from_numpy(np.concatenate(corrs)).cuda())
    assert np.array_equal(nearest[:700].cpu().numpy(), np.arange(700))


def test_mutual_nearest_sqrt_collisions_in_one_lane(built_lib):
    """The same collisions with both keypoints in one candidate lane of nearest_kernel, in one staged chunk and across
    a chunk boundary: the lane's own scan must keep the far keypoint (replace only on a strictly smaller sqrt), since the
    merge of the lanes never sees the near one."""
    from cotr_b200 import capi
    corr, kp, far, _ = mo.sqrt_collisions_in_lanes(120, 120, seed=10)
    rs = np.random.RandomState(11)
    kps = [rs.uniform(0, 1e3, (len(corr), 2)), kp]
    corrs = [corr, rs.uniform(0, 1e3, (len(kp), 2))]
    _check_mutual_nearest(kps, [(0, 1)], corrs)
    off = [0, len(corr), len(corr) + len(kp)]
    nearest, _, _ = capi.mutual_nearest(torch.from_numpy(np.concatenate(kps)).cuda(), off, [(0, 1)],
                                        torch.from_numpy(np.concatenate(corrs)).cuda())
    assert np.array_equal(nearest[:len(corr)].cpu().numpy(), far)


def test_mutual_nearest_large_coordinates_and_nan(built_lib):
    rs = np.random.RandomState(7)
    kps = [rs.uniform(-1e5, 1e5, (900, 2)), rs.uniform(-1e5, 1e5, (1100, 2)), rs.uniform(0, 100, (300, 2))]
    kps[2][123, 1] = np.nan                      # every distance to keypoint 123 of image 2 is NaN: it wins every row
    pairs = [(0, 1), (0, 2)]
    corrs = _random_corrs(kps, pairs, rs, -1e5, 1e5)
    corrs[0][17, 0] = np.nan                     # a NaN prediction: its first candidate wins
    _check_mutual_nearest(kps, pairs, corrs)


def test_mutual_nearest_disk_fixtures(built_lib):
    a, b = _disk(DISK_A), _disk(DISK_B)
    rs = np.random.RandomState(8)
    corrs = [a * [694 / 1033, 1061 / 771] + rs.normal(0, 1.0, a.shape), b * [1033 / 694, 771 / 1061] + rs.normal(0, 1.0, b.shape)]
    assert _check_mutual_nearest([a, b], [(0, 1)], corrs)[0] > 0


@pytest.mark.parametrize("name", ["engine_corr_base", "engine_faster_cycle", "engine_faster_tile_forced", "engine_sparse_known_scale",
                                  "engine_sparse_square_queries", "engine_sparse_stretch_forced", "engine_sparse_tile_random"])
def test_mutual_nearest_engine_goldens(built_lib, name):
    """Engine outputs [x_a, y_a, x_b, y_b]: keypoints of b jittered around the predictions, and the demo-style wrapper."""
    from cotr_b200.inference.matching import mutual_nearest
    corrs = np.load(os.path.join(GOLDEN, name + ".npz"))["out0"].astype(np.float64)
    rs = np.random.RandomState(len(corrs))
    kp_a = corrs[:, :2]
    kp_b = corrs[rs.permutation(len(corrs)), 2:] + rs.normal(0, 0.5, (len(corrs), 2))
    corr_ba = kp_a[rs.randint(0, len(kp_a), len(kp_b))] + rs.normal(0, 0.5, kp_b.shape)
    _check_mutual_nearest([kp_a, kp_b], [(0, 1)], [corrs[:, 2:], corr_ba])
    got = mutual_nearest(corrs[:, 2:], kp_b, corr_ba, kp_a)
    assert got.dtype == np.int64 and np.array_equal(got, mo.match_pair(corrs[:, 2:], kp_b, corr_ba, kp_a)[2])


# ---- cotr_match_keypoints ---------------------------------------------------------------------------------------------
SIZES = [(1024, 768), (683, 1050), (1033, 771), (640, 480), (1920, 1080)]
PAIRS = [(0, 1), (1, 0), (2, 3), (3, 2), (2, 2), (0, 1), (4, 0), (1, 4), (3, 4), (2, 1), (0, 3), (4, 2)]


def _build():
    from cotr_b200.models import build_model
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in fixtures.make_state_dict(0).items()})
    return model.cuda().eval()


@pytest.fixture(scope="module")
def model(built_lib):
    return _build()


def _images(seed, n):
    img, _ = fixtures.make_inputs(seed, (n + 1) // 2, 1)
    B = img.shape[0]
    halves = img.reshape(B, 3, 256, 2, 256).transpose(0, 3, 1, 2, 4).reshape(2 * B, 3, 256, 256)
    return torch.from_numpy(np.ascontiguousarray(halves[:n])).cuda()


def _keypoints(counts, seed):
    rs = np.random.RandomState(seed)
    kps = []
    for n, (W, H) in zip(counts, SIZES):
        if n == 2048:
            kps.append(np.load(os.path.join(GOLDEN, DISK_A)))            # float32, as DISK writes them; image 1033 x 771
        else:
            kps.append(rs.uniform(0, [W, H], (n, 2)).astype(np.float32))
    return kps


def _composition(model, feats, pairs, kps):
    """The same step from existing public calls and the oracle -> (corrs, nearest, matches per pair, launches)."""
    nat = model.native()
    table = [t for a, b in pairs for t in ((a, b), (b, a))]
    ctx = model.encode_context_pairs(feats, table)
    launches = nat.last_launch_count()
    qs = [torch.from_numpy(mo.queries(kps[l], SIZES[l])).cuda() for l, _ in table]
    preds = model.decode(ctx, qs)["pred_corrs"]
    launches += nat.last_launch_count()
    corrs = [mo.pixels(p.cpu().numpy(), SIZES[r]) for p, (_, r) in zip(preds, table)]
    nearest = [mo.nearest(c, np.asarray(kps[r], np.float64)) for c, (_, r) in zip(corrs, table)]
    matches = [mo.mutual(nearest[2 * p], nearest[2 * p + 1]) for p in range(len(pairs))]
    return corrs, nearest, matches, launches


@pytest.mark.parametrize("path,counts,n_pairs", [
    (TC, (31, 32, 2048, 33, 40000), 12),
    (TC, (0, 1, 31, 32, 33), 12),
    (SIMT, (1, 32, 33, 0, 64), 5),
], ids=["tc-large", "tc-small", "simt-small"])
def test_match_keypoints_is_the_composition(model, path, counts, n_pairs):
    nat = model.native()
    nat.set_gemm_path(path)
    try:
        feats = model.encode_images(_images(300 + n_pairs, 5))
        kps = _keypoints(counts, 301)
        pairs = PAIRS[:n_pairs]
        res = model.match_keypoints(feats, pairs, kps, np.array(SIZES))
        launches = nat.last_launch_count()
        corrs, nearest, matches, ref_launches = _composition(model, feats, pairs, kps)
        assert launches == ref_launches + 4
        for p in range(n_pairs):
            assert np.array_equal(res.corrs_ab[p].cpu().numpy(), corrs[2 * p]), p
            assert np.array_equal(res.corrs_ba[p].cpu().numpy(), corrs[2 * p + 1]), p
            assert np.array_equal(res.nearest_ab[p].cpu().numpy(), nearest[2 * p]), p
            assert np.array_equal(res.nearest_ba[p].cpu().numpy(), nearest[2 * p + 1]), p
            assert res.matches[p].dtype == torch.int64 and np.array_equal(res.matches[p].cpu().numpy(), matches[p]), p
        assert sum(len(m) for m in matches) > 0
    finally:
        nat.set_gemm_path(TC)


def test_match_keypoints_profile_records(model):
    feats = model.encode_images(_images(310, 3))
    kps = _keypoints((100, 70, 0), 311)
    nat = model.native()
    nat.profile_begin()
    model.match_keypoints(feats, [(0, 1), (2, 0)], kps, np.array(SIZES[:3]))
    rec = nat.profile_end()
    assert len(rec) == nat.last_launch_count()
    tail = [r[:3] for r in rec if r[0] in ("match_queries", "match_pixels", "nearest", "mutual")]
    assert tail == [("match_queries", 270, 2), ("match_pixels", 270, 2), ("nearest", 270, 2), ("mutual", 2, 0)]
    names = [r[0] for r in rec]
    q, px = names.index("match_queries"), names.index("match_pixels")
    assert names[q + 1] == "query_encode" and names[-3:] == ["match_pixels", "nearest", "mutual"] and px == len(names) - 3


def test_match_keypoints_rejected_inputs(model):
    from cotr_b200 import capi
    nat, lib = model.native(), capi.lib()
    feats = model.encode_images(_images(320, 3))
    kps = np.random.RandomState(321).uniform(0, 500, (30, 2))
    kpts = torch.from_numpy(kps).cuda()
    ctx = capi.NativeContext(nat, 4)
    R = 40
    corr = torch.full((R, 2), 7.0, dtype=torch.float64, device="cuda")
    nearest = torch.full((R,), -7, dtype=torch.int32, device="cuda")
    match = torch.full((R, 2), -7, dtype=torch.int32, device="cuda")
    count = torch.full((2,), -7, dtype=torch.int32, device="cuda")
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda x: ctypes.c_void_p(x.data_ptr()) if x is not None else None
    h = lambda a: ctypes.c_void_p(a.ctypes.data) if a is not None else None
    good_off = np.array([0, 10, 20, 30], np.int64)
    good_pairs = np.array([[0, 1], [2, 0]], np.int32)
    good_sizes = np.array([[640, 480], [100, 100], [65536, 1]], np.int32)

    def call(off=good_off, pairs=good_pairs, sizes=good_sizes, B=2, c=ctx, n=3, cnt=count):
        rc = lib.cotr_match_keypoints(nat.handle, p(feats.tensor), n, h(sizes), p(kpts), h(off), h(pairs), B, c.handle,
                                      p(corr), p(nearest), p(match), p(cnt), s)
        return rc, capi.last_error(), nat.last_launch_count()

    def mn(off=good_off, pairs=good_pairs, B=2, n=3, cnt=count):
        rc = lib.cotr_mutual_nearest(torch.cuda.current_device(), p(kpts), h(off), n, h(pairs), B, p(corr), p(nearest),
                                     p(match), p(cnt), s)
        return rc, capi.last_error()

    other = _build()               # a context of another model
    bad = [({"off": np.array([1, 10, 20, 30], np.int64)}, "must be 0"),
           ({"off": np.array([0, 10, 5, 30], np.int64)}, "decreases"),
           ({"pairs": np.array([[0, 3], [2, 0]], np.int32)}, "outside [0, 3)"),
           ({"pairs": np.array([[0, 1], [-1, 0]], np.int32)}, "outside [0, 3)"),
           ({"B": 0}, "B must be >= 1"),
           ({"n": 0}, "n_images must be >= 1"),
           ({"cnt": None}, "null count_dev")]
    for kw, msg in bad:
        rc, err, launches = call(**kw)
        assert rc != 0 and msg in err and launches == 0, (kw, err)
        rc, err = mn(**kw)
        assert rc != 0 and msg in err, (kw, err)
    for kw, msg in [({"sizes": np.array([[640, 480], [0, 100], [1, 1]], np.int32)}, "outside [1, 65536]"),
                    ({"sizes": np.array([[640, 65537], [100, 100], [1, 1]], np.int32)}, "outside [1, 65536]"),
                    ({"sizes": None}, "null feat_dev or sizes_host"),
                    ({"B": 3, "pairs": np.array([[0, 1], [2, 0], [1, 1]], np.int32)}, "at most 4"),
                    ({"c": capi.NativeContext(other.native(), 4)}, "does not belong")]:
        rc, err, launches = call(**kw)
        assert rc != 0 and msg in err and launches == 0, (kw, err)
    torch.cuda.synchronize()
    assert (corr == 7.0).all() and (nearest == -7).all() and (match == -7).all() and (count == -7).all()   # nothing enqueued

    # the module: stale features, hooks, malformed inputs
    sizes = np.array(SIZES[:3])
    three = [kps[:10], kps[10:20], kps[20:]]
    hook = getattr(model.transformer.encoder.layers, "1").self_attn.register_forward_hook(lambda m, a, o: None)
    try:
        with pytest.raises(RuntimeError, match="attention hooks"):
            model.match_keypoints(feats, [(0, 1)], three, sizes)
    finally:
        hook.remove()
    hook = getattr(model.transformer.decoder.layers, "4").multihead_attn.register_forward_hook(lambda m, a, o: None)
    try:
        with pytest.raises(RuntimeError, match="attention hooks"):
            model.match_keypoints(feats, [(0, 1)], three, sizes)
    finally:
        hook.remove()
    with pytest.raises(AssertionError):
        model.match_keypoints(feats, [(0, 1)], three[:2], sizes)
    with pytest.raises(AssertionError):
        model.match_keypoints(feats, [(0, 1)], three, sizes[:2])
    with pytest.raises(AssertionError, match="set 1 must be"):
        model.match_keypoints(feats, [(0, 1)], [three[0], [[1.0, 2.0, 3.0]], three[2]], sizes)
    as_list = model.match_keypoints(feats, [(0, 1)], [three[0].tolist(), three[1], three[2]], sizes)   # nested lists work too
    as_array = model.match_keypoints(feats, [(0, 1)], three, sizes)
    assert torch.equal(as_list.matches[0], as_array.matches[0]) and torch.equal(as_list.corrs_ab[0], as_array.corrs_ab[0])
    with pytest.raises(RuntimeError, match="sizes"):
        model.match_keypoints(feats, [(0, 1)], three, sizes + 0.5)
    with pytest.raises(RuntimeError, match="outside"):
        model.match_keypoints(feats, [(0, 1)], three, np.array([[1, 1], [0, 5], [3, 3]]))
    res = model.match_keypoints(feats, [(0, 1), (1, 1)], [kps[:10], kps[:0], kps[20:]], sizes)
    assert [tuple(m.shape) for m in res.matches] == [(0, 2), (0, 2)]
    assert (res.nearest_ab[0] == -1).all() and res.corrs_ba[0].shape == (0, 2)
    model.refresh_native()
    with pytest.raises(RuntimeError, match="other weights"):
        model.match_keypoints(feats, [(0, 1)], three, sizes)
