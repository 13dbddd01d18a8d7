"""GPU: the halo loader of the 3x3 stride-1 convolutions (gemm_tc.cu LD_HALO) against the implicit im2col it replaces
(cotr_debug_set_variant bit 20), at the kernel level and through the whole forward, eager and graph-replayed."""
import numpy as np
import pytest
import torch

from oracle import fixtures

pytestmark = pytest.mark.gpu

IM2COL = 1 << 20


def _conv(n_img, H, C, N, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n_img, H, H, C, generator=g).abs() * 0.5           # post-ReLU NHWC activations
    w = torch.randn(N, 3, 3, C, generator=g) * (2.0 / (9 * C)) ** 0.5  # K ordered (kh, kw, c)
    b = torch.randn(N, generator=g) * 0.1
    return x, w, b


def _run_conv(x, w, b, variant):
    from cotr_b200 import capi
    n_img, H, W, C = x.shape
    N = w.shape[0]
    conv = dict(H=H, W=W, C=C, OH=H, OW=W, KH=3, KW=3, stride=1, pad=1)
    capi.lib().cotr_debug_set_variant(variant)
    try:
        return capi.test_gemm(0, x.cuda().contiguous(), w.reshape(N, 9 * C).numpy(), bias=b.cuda(), relu=True,
                              a_mode=1, conv=conv, M=n_img * H * W).cpu()
    finally:
        capi.lib().cotr_debug_set_variant(0)


# (images, H = W, C, N): the stride-1 3x3 convolutions of layer1 / layer2 / layer3 at one pair (layer2's grid is too
# small for the halo loader and runs the im2col), a ragged last row tile (20 x 22 padded rows per image), and layer1 /
# layer2 at 8 pairs (64-wide tiles, layer2 with two resident channel chunks)
SHAPES = [(2, 64, 64, 64), (2, 32, 128, 128), (2, 16, 256, 256), (12, 20, 64, 64), (16, 64, 64, 64), (16, 32, 128, 128)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_halo_conv_matches_im2col(built_lib, shape):
    n_img, H, C, N = shape
    x, w, b = _conv(n_img, H, C, N, seed=H + C)
    halo = _run_conv(x, w, b, 0)
    ref = _run_conv(x, w, b, IM2COL)
    expect = torch.relu(torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(),
                                                   b.double(), padding=1)).permute(0, 2, 3, 1).reshape(-1, N)
    scale = expect.abs().max().item()
    assert (halo.double() - expect).abs().max().item() < 1e-5 * scale
    diff = (halo - ref).abs().max().item()
    if C == 64 and n_img in (2, 12):
        # one channel chunk, no split-K, same tile width: the same products in the same order
        assert diff == 0.0, diff
    else:
        # split-K partials (or accumulator slots) summed in another order: rounding of the fp32 sums only
        assert diff <= 2e-6 * scale, (diff, scale)


def _model():
    from cotr_b200.models import build_model
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in fixtures.make_state_dict(0).items()})
    return model.cuda().eval()


def _forward(model, img, queries, variant, graph):
    from cotr_b200 import capi
    nat = model.native()
    capi.lib().cotr_debug_set_variant(variant)
    try:
        nat.set_gemm_path(1)
        nat.set_gemm_path(0)             # drops graphs captured under another variant
        nat.set_graph_mode(graph)
        outs = []
        for _ in range(3 if graph else 1):            # graph mode: eager first call, then captured, then replayed
            pred = model(img, queries)["pred_corrs"].cpu().numpy()
            outs.append((pred, nat.debug_read("feat", 2 * img.shape[0] * 16 * 16 * 1024)))
        return outs
    finally:
        nat.set_graph_mode(True)
        capi.lib().cotr_debug_set_variant(0)


@pytest.mark.parametrize("B,Q", [(1, 1024), (2, 100), (3, 1), (16, 1024)])
def test_forward_with_halo_matches_im2col(built_lib, B, Q):
    model = _model()
    img, queries = fixtures.make_inputs(31 + B, B, Q)
    img = torch.from_numpy(img).cuda()
    queries = torch.from_numpy(queries).cuda()
    ref_pred, ref_feat = _forward(model, img, queries, IM2COL, graph=False)[0]
    (eager_pred, eager_feat), = _forward(model, img, queries, 0, graph=False)
    runs = _forward(model, img, queries, 0, graph=True)
    for pred, feat in runs[1:]:
        # replays are bitwise equal to each other and to the eager forward
        assert np.array_equal(pred, runs[-1][0]) and np.array_equal(feat, runs[-1][1])
        assert np.array_equal(pred, eager_pred) and np.array_equal(feat, eager_feat)
    feat_diff = np.abs(eager_feat - ref_feat).max() / np.abs(ref_feat).max()
    pred_diff = np.abs(eager_pred - ref_pred).max()
    print(f"B={B} Q={Q}: feat max rel diff {feat_diff:.2e}, pred max abs diff {pred_diff:.2e}")
    assert feat_diff < 1e-5, feat_diff
    assert pred_diff < 2e-5, pred_diff
