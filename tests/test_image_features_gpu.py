"""GPU: the image-level feature cache - cotr_encode_images / cotr_encode_context_pairs and COTR.encode_images /
COTR.encode_context_pairs.  A context built from cached halves must be bitwise the canvas context; arbitrary pairs of
cached images must predict what the canvas forward of the assembled canvases predicts."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import cotr_oracle, fixtures

pytestmark = pytest.mark.gpu

TC, SIMT = 0, 1
ENC_MASK = 0b100001          # encoder layers 0 and 5
# batch composition only changes split-K / tile choices in the backbone: the bound of
# test_batch_items_and_queries_are_independent
BATCH_TOL = 2e-4
ORACLE_TOL = 3e-4


def _build():
    from cotr_b200.models import build_model
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in fixtures.make_state_dict(0).items()})
    return model.cuda().eval()


@pytest.fixture(scope="module")
def model(built_lib):
    return _build()


def _halves(canvases):
    """(B,3,256,512) -> (2B,3,256,256) in canvas order: image 2p = left half of canvas p, 2p+1 = its right half."""
    B = canvases.shape[0]
    return canvases.view(B, 3, 256, 2, 256).permute(0, 3, 1, 2, 4).reshape(2 * B, 3, 256, 256).contiguous()


def _enc_hooks(model):
    fired = []
    handles = [getattr(model.transformer.encoder.layers, str(l)).self_attn.register_forward_hook(
        lambda m, a, o, l=l: fired.append((l, o[1].clone()))) for l in range(6) if (ENC_MASK >> l) & 1]
    return fired, handles


@pytest.mark.parametrize("path,B", [(TC, 1), (TC, 3), (TC, 16), (SIMT, 1), (SIMT, 3)],
                         ids=["tc-b1", "tc-b3", "tc-b16", "simt-b1", "simt-b3"])
def test_pairs_of_halves_are_bitwise_the_canvas_context(model, path, B):
    img, queries = fixtures.make_inputs(70 + B, B, 128)
    t, q = torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()
    pairs = [(2 * p, 2 * p + 1) for p in range(B)]
    model.native().set_gemm_path(path)
    try:
        ref = model.decode(model.encode_context(t), q)["pred_corrs"]
        feats = model.encode_images(_halves(t))
        assert feats.n == 2 * B and tuple(feats.tensor.shape) == (2, 2 * B, 256, 1024) and feats.tensor.dtype == torch.float16
        got = model.decode(model.encode_context_pairs(feats, pairs), q)["pred_corrs"]
        assert torch.equal(got, ref)
        # the encoder attention hooks fire the same maps
        fired, handles = _enc_hooks(model)
        try:
            model.encode_context(t)
            ref_maps = list(fired)
            fired.clear()
            ctx = model.encode_context_pairs(feats, torch.tensor(pairs))
            got_maps = list(fired)
        finally:
            for h in handles:
                h.remove()
        assert [l for l, _ in got_maps] == [0, 5] and [l for l, _ in ref_maps] == [0, 5]
        for (_, a), (_, b) in zip(got_maps, ref_maps):
            assert tuple(a.shape) == (B, 512, 512) and torch.equal(a, b)
        assert torch.equal(model.decode(ctx, q)["pred_corrs"], ref)
    finally:
        model.native().set_gemm_path(TC)


def test_reuse_swaps_self_pairs_and_repeats(model):
    img, _ = fixtures.make_inputs(80, 3, 1)
    images = _halves(torch.from_numpy(img))[:5].cuda()
    pairs = np.array([(0, 1), (1, 0), (2, 2), (3, 4), (4, 3), (0, 1), (1, 2), (2, 0), (4, 4), (3, 0), (0, 3), (2, 4)])
    _, queries = fixtures.make_inputs(81, len(pairs), 100)
    q = torch.from_numpy(queries).cuda()
    canvases = torch.stack([torch.cat([images[i], images[j]], dim=-1) for i, j in pairs])
    ref = model(canvases, q)["pred_corrs"]
    feats = model.encode_images(images)
    ctx = model.encode_context_pairs(feats, pairs, reuse=True)
    got = model.decode(ctx, q)["pred_corrs"]
    assert (got - ref).abs().max().item() < BATCH_TOL
    sd = fixtures.make_state_dict(0)
    for k in (1, 2):            # a swap and a self-pair against the fp64 oracle
        ora = cotr_oracle.forward(sd, canvases[k:k + 1].cpu().numpy(), queries[k:k + 1], torch.float64)
        assert (got[k].cpu().double() - ora[0]).abs().max().item() < ORACLE_TOL, k
    # reuse=True hands back the same device buffer for the same batch size
    assert model.encode_context_pairs(feats, pairs.tolist(), reuse=True).native is ctx.native


def test_chunked_encode_and_host_round_trip(model):
    from cotr_b200.models.cotr_model import ImageFeatures
    rs = np.random.RandomState(90)
    images = torch.from_numpy(rs.standard_normal((70, 3, 256, 256)).astype(np.float32)).cuda()
    whole = model.encode_images(images)                   # crosses the 64-image chunk boundary
    singles = [model.encode_images(images[i:i + 1]) for i in range(70)]
    joined = ImageFeatures(torch.cat([f.tensor for f in singles], dim=1), 70, singles[0].generation)
    pairs = [(i, 69 - i) for i in range(35)]               # every image once; pairs 0..5 join the two chunks
    _, queries = fixtures.make_inputs(91, 35, 16)
    q = torch.from_numpy(queries).cuda()
    a = model.decode(model.encode_context_pairs(whole, pairs), q)["pred_corrs"]
    b = model.decode(model.encode_context_pairs(joined, pairs), q)["pred_corrs"]
    assert (a - b).abs().max().item() < BATCH_TOL
    # images 64.. sit in the second chunk; image 63 in the first
    ref = model(torch.cat([images[63], images[64]], dim=-1)[None], q[:1])["pred_corrs"]
    c = model.decode(model.encode_context_pairs(whole, [(63, 64)]), q[:1])["pred_corrs"]
    assert (c - ref).abs().max().item() < BATCH_TOL
    # the bytes survive a trip through host memory
    back = ImageFeatures(whole.tensor.cpu().cuda(), whole.n, whole.generation)
    assert torch.equal(model.decode(model.encode_context_pairs(back, pairs), q)["pred_corrs"], a)


def test_errors(model):
    from cotr_b200 import capi
    img, _ = fixtures.make_inputs(95, 2, 1)
    t = torch.from_numpy(img).cuda()
    feats = model.encode_images(_halves(t))
    for bad in ([(0, 4)], [(-1, 0)], [(0, 1), (3, 7)]):
        with pytest.raises(RuntimeError, match="outside"):
            model.encode_context_pairs(feats, bad)
    with pytest.raises(AssertionError):
        model.encode_images(t)                             # a (N,3,256,512) canvas batch
    with pytest.raises(AssertionError):
        model.encode_context_pairs(feats, [0, 1])          # not (B,2)
    nat, lib = model.native(), capi.lib()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    ctx = capi.NativeContext(nat, 1)
    table = np.array([[0, 1], [1, 0]], dtype=np.int32)
    tp = ctypes.c_void_p(table.ctypes.data)
    assert lib.cotr_encode_context_pairs(nat.handle, p(feats.tensor), 4, tp, 2, ctx.handle, 0, None, s) != 0
    assert "capacity" in capi.last_error()
    assert lib.cotr_encode_context_pairs(nat.handle, p(feats.tensor), 0, tp, 1, ctx.handle, 0, None, s) != 0
    assert "n_images" in capi.last_error()
    assert lib.cotr_encode_context_pairs(nat.handle, p(feats.tensor), 4, tp, 0, ctx.handle, 0, None, s) != 0
    assert "B must be" in capi.last_error()
    assert lib.cotr_encode_context_pairs(nat.handle, p(feats.tensor), 4, tp, 1, ctx.handle, 1 << 6, None, s) != 0
    assert "layer_mask" in capi.last_error()
    assert lib.cotr_encode_context_pairs(nat.handle, p(feats.tensor), 4, tp, 1, ctx.handle, 1, None, s) != 0
    assert "attn_dev" in capi.last_error()
    assert lib.cotr_encode_context_pairs(nat.handle, ctypes.c_void_p(feats.tensor.data_ptr() + 8), 4, tp, 1, ctx.handle, 0, None, s) != 0
    assert "aligned" in capi.last_error()
    assert lib.cotr_encode_images(nat.handle, p(t), 0, p(feats.tensor), s) != 0
    assert "N must be" in capi.last_error()
    torch.cuda.synchronize()
    ctx.close()
    # features of replaced weights
    m2 = _build()
    stale = m2.encode_images(_halves(t))
    m2.load_state_dict({k: torch.from_numpy(v) for k, v in fixtures.make_state_dict(0).items()})
    with pytest.raises(RuntimeError, match="other weights"):
        m2.encode_context_pairs(stale, [(0, 1)])
    with pytest.raises(RuntimeError, match="other weights"):
        model.encode_context_pairs(m2.encode_images(_halves(t)), [(0, 1)])     # another model's features


@pytest.mark.parametrize("B", [1, 3])
def test_launch_counts(model, B):
    from cotr_b200 import capi
    img, queries = fixtures.make_inputs(5, B, 1024)
    t, q = torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()
    nat = model.native()
    ctx = capi.NativeContext(nat, B)
    nat.encode_context(t, ctx)
    n_ctx = nat.last_launch_count()
    feat = nat.encode_images(_halves(t))
    n_img = nat.last_launch_count()
    nat.encode_context_pairs(feat, [(2 * p, 2 * p + 1) for p in range(B)], ctx)
    assert n_img + nat.last_launch_count() == n_ctx
    if B == 1:
        model(t, q)
        assert nat.last_launch_count() == 111
    torch.cuda.synchronize()
    ctx.close()
