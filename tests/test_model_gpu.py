"""GPU: the parity tests proper - the CUDA hot path (called through the C ABI) against the oracle and the golden
vectors produced by the real reference.  North-star tolerance: |delta(x,y)| <= 1e-3 on predicted correspondences."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import cotr_oracle, fixtures

pytestmark = pytest.mark.gpu

TOL = 1e-3            # BASELINE.json north_star: "within 1e-3 on predicted (x,y)"
TOL_INTERNAL = 3e-4   # what the kernels are actually expected to deliver on these fixtures (regression guard)
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "model_*.npz")))


def _build(sd):
    from cotr_b200.models import build_model
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return model.cuda().eval()


@pytest.fixture(scope="module")
def default_model(built_lib):
    return _build(fixtures.make_state_dict(0))


def _case(golden_dir, name):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    params = g["params"]
    wseed, qk, hg, iseed, b, q = params[:6]
    stem_gain, q_stride = (float(params[6]), int(params[7])) if len(params) > 6 else (1.0, 1)
    sd = fixtures.make_state_dict(int(wseed), float(qk), float(hg), stem_gain)
    img, queries = fixtures.make_inputs(int(iseed), int(b), int(q))
    return g, sd, img, queries, q_stride


@pytest.mark.parametrize("path", [0, 1], ids=["tcgen05", "simt"])
@pytest.mark.parametrize("name", CASES)
def test_forward_matches_reference_goldens(golden_dir, built_lib, name, path):
    g, sd, img, queries, q_stride = _case(golden_dir, name)
    if path == 1 and img.shape[0] * queries.shape[1] > 20000:
        pytest.skip("the fp32 SIMT cross-check path is not run on the large-batch cases")
    model = _build(sd)
    model.native().set_gemm_path(path)
    pred = model(torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda())["pred_corrs"]
    assert pred.shape == (img.shape[0], queries.shape[1], 2) and pred.dtype == torch.float32 and pred.is_cuda
    pred = pred.cpu().numpy()
    assert np.isfinite(pred).all()
    pred = pred[:, ::q_stride]            # large cases store every q_stride-th query only
    if "feat_absmax" in g.files and float(g["params"][6]) > 1.0:
        # the big-activation fixture must really exercise the upper range of the fp16 hi/lo storage
        feat = model.native().debug_read("feat", 2 * img.shape[0] * 16 * 16 * 1024)
        assert np.abs(feat).max() > 1e4 and float(g["feat_absmax"]) > 1e4
    err32 = np.abs(pred - g["ref_pred_fp32"]).max()
    err64 = np.abs(pred - g["ref_pred_fp64"]).max()
    assert err32 < TOL and err64 < TOL, (err32, err64)
    assert err64 < TOL_INTERNAL, err64


@pytest.mark.parametrize("path", [0, 1], ids=["tcgen05", "simt"])
def test_intermediates_match_oracle(default_model, path):
    """Hand-off tensors of the path (feat -> src -> mem -> hs) against the oracle in fp64: localises a regression."""
    sd = fixtures.make_state_dict(0)
    img, queries = fixtures.make_inputs(1, 1, 1024)
    default_model.native().set_gemm_path(path)
    default_model(torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda())
    nat = default_model.native()
    _, inter = cotr_oracle.forward(sd, img, queries, torch.float64, return_intermediates=True)
    feat = torch.from_numpy(nat.debug_read("feat", 2 * 16 * 16 * 1024)).view(2, 16, 16, 1024)
    feat = torch.cat([feat[0], feat[1]], dim=1).permute(2, 0, 1)[None]
    got = {"pos": torch.from_numpy(nat.debug_read("pos", 512 * 256)).view(512, 256), "feat": feat,
           "src": torch.from_numpy(nat.debug_read("src", 512 * 256)).view(1, 512, 256),
           "mem": torch.from_numpy(nat.debug_read("mem", 512 * 256)).view(1, 512, 256),
           "hs": torch.from_numpy(nat.debug_read("hs", 1024 * 256)).view(1, 1024, 256)}
    bound = {"pos": 1e-6, "feat": 2e-5, "src": 2e-5, "mem": 1e-4, "hs": 1e-4}
    for name, b in bound.items():
        ref = inter[name].double()
        rel = ((got[name].double() - ref).norm() / ref.norm()).item()
        assert rel < b, (name, rel)
    default_model.native().set_gemm_path(0)


def test_batch_items_and_queries_are_independent(default_model):
    """SURVEY.md app. E.4: a pair alone == the same pair inside a batch; a query alone == inside a 1024 batch."""
    img, queries = fixtures.make_inputs(9, 3, 200)
    img = torch.from_numpy(img).cuda(); queries = torch.from_numpy(queries).cuda()
    full = default_model(img, queries)["pred_corrs"]
    one = default_model(img[1:2], queries[1:2])["pred_corrs"]
    # not bitwise: tile width / split-K are chosen from the launch shape, so the summation order depends on B and Q
    assert (full[1:2] - one).abs().max().item() < 2e-4
    single = default_model(img[1:2], queries[1:2, 57:58])["pred_corrs"]
    assert (full[1:2, 57:58] - single).abs().max().item() < 2e-4


def test_context_reuse_equals_forward(default_model):
    """encode_context + decode (context cached on the device) == forward, also for query sets larger than a chunk."""
    img, queries = fixtures.make_inputs(10, 2, 333)
    img = torch.from_numpy(img).cuda(); queries = torch.from_numpy(queries).cuda()
    ref = default_model(img, queries)["pred_corrs"]
    ctx = default_model.encode_context(img)
    a = default_model.decode(ctx, queries)["pred_corrs"]
    b = default_model.decode(ctx, queries[:, :7].contiguous())["pred_corrs"]
    assert (a - ref).abs().max().item() < 2e-4
    assert (b - ref[:, :7]).abs().max().item() < 2e-4


def test_large_query_count_is_chunked_exactly(default_model):
    """Q above the decoder chunk (32768 rows): chunked result == per-slice results."""
    img, queries = fixtures.make_inputs(11, 1, 40000)
    img = torch.from_numpy(img).cuda(); queries = torch.from_numpy(queries).cuda()
    full = default_model(img, queries)["pred_corrs"]
    part = default_model(img, queries[:, 35000:36000].contiguous())["pred_corrs"]
    assert torch.isfinite(full).all()
    assert (full[:, 35000:36000] - part).abs().max().item() < 2e-4


def test_host_buffer_entry_point(default_model):
    """cotr_forward_host (H2D + forward + D2H inside the C call) == device-pointer forward."""
    img, queries = fixtures.make_inputs(12, 2, 64)
    dev = default_model(torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda())["pred_corrs"].cpu().numpy()
    host = default_model.native().forward_host(img, queries)
    assert np.array_equal(dev, host)


def test_accepts_list_and_nested_tensor(default_model):
    from cotr_b200.models.misc import NestedTensor
    img, queries = fixtures.make_inputs(13, 2, 16)
    t = torch.from_numpy(img).cuda(); q = torch.from_numpy(queries).cuda()
    ref = default_model(t, q)["pred_corrs"]
    assert torch.equal(default_model([t[0], t[1]], q)["pred_corrs"], ref)
    assert torch.equal(default_model(NestedTensor(t, None), q)["pred_corrs"], ref)


def test_zero_padded_queries_are_harmless(default_model):
    """FasterSparseEngine pads query sets with zeros (sparse_engine.py:366); real queries must be unaffected."""
    img, queries = fixtures.make_inputs(14, 1, 50)
    t = torch.from_numpy(img).cuda(); q = torch.from_numpy(queries).cuda()
    ref = default_model(t, q)["pred_corrs"]
    padded = torch.cat([q, torch.zeros(1, 207, 2, device="cuda")], dim=1)
    out = default_model(t, padded)["pred_corrs"]
    assert (out[:, :50] - ref).abs().max().item() < 2e-4
    assert torch.isfinite(out).all()


def test_weights_reload_repacks(built_lib):
    """load_state_dict after the first forward must invalidate the packed device copy."""
    img, queries = fixtures.make_inputs(15, 1, 32)
    t = torch.from_numpy(img).cuda(); q = torch.from_numpy(queries).cuda()
    m = _build(fixtures.make_state_dict(0))
    a = m(t, q)["pred_corrs"].clone()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in fixtures.make_state_dict(3).items()})
    b = m(t, q)["pred_corrs"]
    assert (a - b).abs().max().item() > 1e-3
    ref = cotr_oracle.forward(fixtures.make_state_dict(3), img, queries, torch.float32)
    assert (b.cpu() - ref).abs().max().item() < TOL


def test_graph_replay_survives_workspace_growth(built_lib):
    """A shape's captured graph embeds workspace addresses; a later, larger shape reallocates the workspace.  The
    earlier shape must still replay correctly (graphs are dropped and re-captured), bit-identical to its first run."""
    m = _build(fixtures.make_state_dict(0))
    img1, q1 = fixtures.make_inputs(21, 1, 64)
    img4, q4 = fixtures.make_inputs(22, 4, 64)
    imgq, qq = fixtures.make_inputs(23, 1, 5000)
    t1, u1 = torch.from_numpy(img1).cuda(), torch.from_numpy(q1).cuda()
    t4, u4 = torch.from_numpy(img4).cuda(), torch.from_numpy(q4).cuda()
    tq, uq = torch.from_numpy(imgq).cuda(), torch.from_numpy(qq).cuda()
    first = m(t1, u1)["pred_corrs"].clone()                # eager
    assert torch.equal(m(t1, u1)["pred_corrs"], first)     # captured
    assert torch.equal(m(t1, u1)["pred_corrs"], first)     # replayed
    big = [m(t4, u4)["pred_corrs"].clone() for _ in range(3)]      # encoder workspace + staging grow
    assert torch.equal(big[0], big[1]) and torch.equal(big[0], big[2])
    assert torch.equal(m(t1, u1)["pred_corrs"], first)
    many = [m(tq, uq)["pred_corrs"].clone() for _ in range(3)]     # decoder workspace + query staging grow
    assert torch.equal(many[0], many[1]) and torch.equal(many[0], many[2])
    assert torch.equal(m(t1, u1)["pred_corrs"], first)
    assert torch.equal(m(t4, u4)["pred_corrs"], big[0])
    torch.cuda.synchronize()


@pytest.mark.parametrize("variant,name", [(1 << 19, "deferred-layernorm"), (1 << 16, "explicit-layernorm")])
def test_experimental_schedules_match_the_reference(golden_dir, built_lib, variant, name):
    """The schedules cotr_debug_set_variant can force (bit 19: LayerNorms applied on the fly by their consumers from
    partial row statistics, everywhere; bit 16: explicit LayerNorm launches everywhere - by default each section picks
    by its row count) both stay correct: same goldens, same tolerance, eager and
    graph-replayed, also for a batch whose query count is not a tile multiple."""
    from cotr_b200 import capi
    capi.lib().cotr_debug_set_variant(variant)
    try:
        for case in ("model_b1_q1024", "model_b2_q100", "model_b16_q1024"):
            g, sd, img, queries, q_stride = _case(golden_dir, case)
            model = _build(sd)
            t, q = torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()
            for rep in range(3):                                   # eager, capture, replay
                pred = model(t, q)["pred_corrs"].cpu().numpy()[:, ::q_stride]
                assert np.abs(pred - g["ref_pred_fp64"]).max() < TOL_INTERNAL, (case, rep)
            if case == "model_b1_q1024":
                assert model.native().last_launch_count() == (136 if variant == (1 << 16) else 112)
    finally:
        capi.lib().cotr_debug_set_variant(0)
