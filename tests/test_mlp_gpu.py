"""GPU: the fused feed-forward launch (csrc/mlp_tc.cu) against the separate linear1 / linear2 / LayerNorm launches
that cotr_debug_set_variant bit 16 keeps, on shapes with ragged row tiles in both transformer sections."""
import pytest
import torch

from oracle import fixtures

pytestmark = pytest.mark.gpu

SEPARATE = 1 << 16


def _build():
    from cotr_b200.models import build_model
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in fixtures.make_state_dict(0).items()})
    return model.cuda().eval()


@pytest.fixture(scope="module")
def model(built_lib):
    return _build()


def _run_three(model, t, q, variant):
    """eager, captured and replayed predictions under `variant` (the cached graphs are dropped first)."""
    from cotr_b200 import capi
    capi.lib().cotr_debug_set_variant(variant)
    nat = model.native()
    nat.set_gemm_path(1)
    nat.set_gemm_path(0)
    try:
        return [model(t, q)["pred_corrs"].clone() for _ in range(3)], nat.last_launch_count()
    finally:
        capi.lib().cotr_debug_set_variant(0)
        nat.set_gemm_path(1)
        nat.set_gemm_path(0)


@pytest.mark.parametrize("B,Q", [(1, 1024), (2, 100), (3, 1), (1, 2047)])
def test_fused_feed_forward_matches_separate_launches(model, B, Q):
    # B = 3: 1536 encoder rows (24 row tiles); Q = 2047: the largest decoder section of the explicit schedule
    img, queries = fixtures.make_inputs(30 + B, B, Q)
    t, q = torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()
    fused, n_fused = _run_three(model, t, q, 0)
    separate, _ = _run_three(model, t, q, SEPARATE)
    assert torch.isfinite(fused[0]).all()
    assert torch.equal(fused[0], fused[1]) and torch.equal(fused[0], fused[2])
    assert (fused[0] - separate[0]).abs().max().item() < 2e-4
    if (B, Q) == (1, 1024):
        # 136 launches with separate ones, minus 12 linear1 launches, 12 LayerNorms and the final decoder.norm
        assert n_fused == 111
