"""GPU: ragged decode - cotr_decode_ragged, NativeModel.decode_ragged and COTR.decode with a list of query sets, one
count per pair.  With equal counts it must be bitwise the uniform decode with the same launches; with mixed counts every
pair must predict what its own queries predict in a uniform decode, also across chunk boundaries and on both attention
kernels in one call."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import fixtures

pytestmark = pytest.mark.gpu

TC, SIMT = 0, 1
TOL_INTERNAL = 3e-4     # test_model_gpu.py: against the fp64 reference
TOL = 1e-3              # ... and the fp32 reference
BATCH_TOL = 2e-4        # launch shapes differ (tile width, split-K, key split): the bound of test_batch_items_and_queries_are_independent


def _build(sd=None):
    from cotr_b200.models import build_model
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in (sd if sd is not None else fixtures.make_state_dict(0)).items()})
    return model.cuda().eval()


@pytest.fixture(scope="module")
def model(built_lib):
    return _build()


def _halves(canvases):
    B = canvases.shape[0]
    return canvases.view(B, 3, 256, 2, 256).permute(0, 3, 1, 2, 4).reshape(2 * B, 3, 256, 256).contiguous()


def _context(model, t, source):
    if source == "canvas":
        return model.encode_context(t)
    feats = model.encode_images(_halves(t))
    return model.encode_context_pairs(feats, [(2 * p, 2 * p + 1) for p in range(t.shape[0])])


def _offsets(counts):
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)


def _random_queries(seed, counts):
    rs = np.random.RandomState(seed)
    return [torch.from_numpy(rs.uniform(0.0, 1.0, (n, 2)).astype(np.float32)).cuda() for n in counts]


def _padded_reference(model, ctx, qs):
    """The uniform decode of every pair's queries on the same context: zero-padded to the largest count."""
    Q = max(q.shape[0] for q in qs)
    pad = torch.zeros((len(qs), Q, 2), dtype=torch.float32, device="cuda")
    for p, q in enumerate(qs):
        pad[p, :q.shape[0]] = q
    ref = model.decode(ctx, pad)["pred_corrs"]
    return [ref[p, :q.shape[0]] for p, q in enumerate(qs)]


@pytest.mark.parametrize("source", ["canvas", "pairs"])
@pytest.mark.parametrize("path,B,Q", [(TC, 1, 1024), (TC, 2, 100), (TC, 3, 1), (TC, 16, 1024), (SIMT, 1, 1024), (SIMT, 2, 100), (SIMT, 3, 1)],
                         ids=["tc-b1-q1024", "tc-b2-q100", "tc-b3-q1", "tc-b16-q1024", "simt-b1-q1024", "simt-b2-q100", "simt-b3-q1"])
def test_equal_counts_are_the_uniform_decode(model, path, B, Q, source):
    img, queries = fixtures.make_inputs(100 + B, B, Q)
    t, q = torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()
    nat = model.native()
    nat.set_gemm_path(path)
    try:
        ctx = _context(model, t, source)
        ref = nat.decode(ctx.native, q)
        n_ref = nat.last_launch_count()
        got = nat.decode_ragged(ctx.native, q.reshape(B * Q, 2), np.arange(B + 1) * Q)
        assert nat.last_launch_count() == n_ref
        assert torch.equal(got.view(B, Q, 2), ref)
        # the module's list form: views of one packed output
        lst = model.decode(ctx, [q[p] for p in range(B)])["pred_corrs"]
        assert len(lst) == B
        for p in range(B):
            assert lst[p].shape == (Q, 2) and torch.equal(lst[p], ref[p])
            assert lst[p].untyped_storage().data_ptr() == lst[0].untyped_storage().data_ptr()
    finally:
        nat.set_gemm_path(TC)


SUBSET_SIZES = (0, 1, 31, 32, 33, 128, 129, -1)      # -1: every stored query of the pair


@pytest.mark.parametrize("name", ["model_b1_q1024", "model_b2_q100", "model_b3_q1", "model_b16_q1024", "model_b32_q1",
                                  "model_b64_q1024", "model_bigact_b1_q256", "model_peaked_b1_q257"])
def test_ragged_subsets_match_reference_goldens(golden_dir, built_lib, name):
    """Decoder queries are independent (no decoder self-attention, every other step works row by row), so any subset
    of a golden's queries must give the golden's predictions for them.  Contexts repeat the golden's pairs up to 8
    pairs, so that every golden mixes all subset sizes in one call; the strided goldens use stored queries only."""
    import os
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    params = g["params"]
    wseed, qk, hg, iseed, b, nq = params[:6]
    stem_gain, q_stride = (float(params[6]), int(params[7])) if len(params) > 6 else (1.0, 1)
    sd = fixtures.make_state_dict(int(wseed), float(qk), float(hg), stem_gain)
    img, queries = fixtures.make_inputs(int(iseed), int(b), int(nq))
    B = img.shape[0]
    stored = np.arange(0, queries.shape[1], q_stride)
    pairs = [i % B for i in range(max(B, len(SUBSET_SIZES)))]
    rs = np.random.RandomState(7)
    sel = []
    for i, _ in enumerate(pairs):
        size = SUBSET_SIZES[i % len(SUBSET_SIZES)]
        size = len(stored) if size < 0 else min(size, len(stored))
        sel.append(np.sort(rs.choice(len(stored), size, replace=False)))
    model = _build(sd)
    t = torch.from_numpy(img[pairs]).cuda()
    qs = [torch.from_numpy(queries[p, stored[s]]).cuda() for p, s in zip(pairs, sel)]
    for path in (TC, SIMT):
        if path == SIMT and B * queries.shape[1] > 20000:
            continue          # test_model_gpu.py does not run the fp32 SIMT path on the large-batch cases either
        model.native().set_gemm_path(path)
        ctx = model.encode_context(t)
        got = model.decode(ctx, qs)["pred_corrs"]
        for i, (p, s) in enumerate(zip(pairs, sel)):
            pred = got[i].cpu().numpy()
            assert pred.shape == (len(s), 2) and np.isfinite(pred).all()
            if len(s) == 0:
                continue
            err64 = np.abs(pred - g["ref_pred_fp64"][p, s]).max()
            err32 = np.abs(pred - g["ref_pred_fp32"][p, s]).max()
            assert err64 < TOL_INTERNAL and err32 < TOL, (path, i, len(s), err64, err32)
    model.native().set_gemm_path(TC)


@pytest.mark.parametrize("path", [TC, SIMT], ids=["tc", "simt"])
def test_mixed_counts_use_both_attention_kernels(model, path):
    counts = [1, 31, 0, 32, 300, 129]
    img, _ = fixtures.make_inputs(120, len(counts), 1)
    nat = model.native()
    nat.set_gemm_path(path)
    try:
        ctx = model.encode_context(torch.from_numpy(img).cuda())
        qs = _random_queries(121, counts)
        ref = _padded_reference(model, ctx, qs)
        nat.profile_begin()
        got = nat.decode_ragged(ctx.native, torch.cat(qs), _offsets(counts))
        rec = nat.profile_end()
        assert len(rec) == nat.last_launch_count()
        attn = {}
        for kernel, M, _, _, _ in rec:
            if kernel.startswith("attention"):
                attn.setdefault(kernel, []).append(M)
        if path == TC:       # pairs with < 32 rows go to the SIMT kernel, the others to the tensor-core kernel
            assert attn == {"attention_tc": [32 + 300 + 129] * 6, "attention_simt": [1 + 31] * 6}
        else:
            assert attn == {"attention_simt": [sum(counts)] * 6}
        for p, n in enumerate(counts):
            rows = got[sum(counts[:p]):sum(counts[:p + 1])]
            assert rows.shape == (n, 2)
            if n:
                assert (rows - ref[p]).abs().max().item() < BATCH_TOL, p
    finally:
        nat.set_gemm_path(TC)


@pytest.mark.parametrize("counts", [[20000, 20000, 5], [40000, 3]], ids=["straddle", "slices"])
def test_chunk_boundaries(model, counts):
    """[20000, 20000, 5]: the packed rows cross the 32768-row decode chunk; [40000, 3]: a pair is cut into slices."""
    img, _ = fixtures.make_inputs(130, len(counts), 1)
    ctx = model.encode_context(torch.from_numpy(img).cuda())
    qs = _random_queries(131, counts)
    ref = _padded_reference(model, ctx, qs)
    got = model.decode(ctx, qs)["pred_corrs"]
    for p, n in enumerate(counts):
        assert got[p].shape == (n, 2)
        assert (got[p] - ref[p]).abs().max().item() < BATCH_TOL, p


def test_workspace_growth_keeps_graphs_correct(built_lib):
    """A ragged decode that grows the decode workspace drops the captured graphs; the replayed forward stays exact."""
    m = _build()
    img, q = fixtures.make_inputs(140, 2, 64)
    t, u = torch.from_numpy(img).cuda(), torch.from_numpy(q).cuda()
    first = m(t, u)["pred_corrs"].clone()                  # eager
    m(t, u)                                                # captured
    replay = m(t, u)["pred_corrs"].clone()                 # replayed
    assert torch.equal(replay, first)
    ctx = m.encode_context(t)
    counts = [30000, 2500]                                 # one chunk of 32500 rows: far above the 128 rows of the forward
    got = m.decode(ctx, _random_queries(141, counts))["pred_corrs"]
    assert all(torch.isfinite(x).all() for x in got)
    assert torch.equal(m(t, u)["pred_corrs"], replay)
    assert torch.equal(m(t, u)["pred_corrs"], replay)
    torch.cuda.synchronize()


def test_rejected_inputs(model):
    from cotr_b200 import capi
    nat, lib = model.native(), capi.lib()
    img, queries = fixtures.make_inputs(150, 2, 8)
    t = torch.from_numpy(img).cuda()
    ctx = model.encode_context(t)
    q = torch.from_numpy(queries).cuda().reshape(16, 2)
    pred = torch.full((16, 2), float("nan"), device="cuda")
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda x: ctypes.c_void_p(x.data_ptr())

    def call(offsets, B=2, c=ctx.native.handle, qp=None, pp=None, m=nat):
        off = np.ascontiguousarray(offsets, dtype=np.int64) if offsets is not None else None
        rc = lib.cotr_decode_ragged(m.handle, c, qp if qp is not None else p(q), ctypes.c_void_p(off.ctypes.data) if off is not None else None,
                                    B, pp if pp is not None else p(pred), s)
        return rc, capi.last_error(), m.last_launch_count()

    for args, msg in [(([1, 8, 16],), "must be 0"), (([0, 9, 8],), "decreases"), (([0, 8, 16, 16], 3), "context holds"),
                      (([0, 16], 1), "context holds"), ((None,), "null offsets"),
                      (([0, 8, 16], 2, ctx.native.handle, ctypes.c_void_p(0)), "null queries_dev"),
                      (([0, 8, 16], 2, ctx.native.handle, None, ctypes.c_void_p(0)), "null queries_dev or pred_dev")]:
        rc, err, launches = call(*args)
        assert rc != 0 and msg in err and launches == 0, (args, err)
    # another model's context
    other = _build()
    octx = other.encode_context(t)
    rc, err, launches = call([0, 8, 16], 2, octx.native.handle)
    assert rc != 0 and "does not belong" in err and launches == 0
    # a context encoded under the other matrix-multiply path
    nat.set_gemm_path(SIMT)
    try:
        rc, err, launches = call([0, 8, 16])
        assert rc != 0 and "other matrix-multiply path" in err and launches == 0
    finally:
        nat.set_gemm_path(TC)
    torch.cuda.synchronize()
    assert torch.isnan(pred).all()                          # nothing was enqueued
    # R == 0 (NULL buffers allowed): no launch
    rc, _, launches = call([0, 0, 0], 2, ctx.native.handle, ctypes.c_void_p(0), ctypes.c_void_p(0))
    assert rc == 0 and launches == 0
    # the list form
    qs = [q[:8], q[8:]]
    with pytest.raises(AssertionError):
        model.decode(ctx, qs[:1])                           # one query set for two pairs
    with pytest.raises(AssertionError):
        model.decode(ctx, [q[:8], q[8:].reshape(-1)])       # not (Q,2)
    with pytest.raises(AssertionError):
        model.decode(ctx, [q[:8], torch.zeros(3, 3, device="cuda")])
    h = getattr(model.transformer.decoder.layers, "2").multihead_attn.register_forward_hook(lambda mod, a, o: None)
    try:
        with pytest.raises(RuntimeError, match="not produced for ragged decodes"):
            model.decode(ctx, qs)
    finally:
        h.remove()
    empty = model.decode(ctx, [q[:0], q[:0]])["pred_corrs"]
    assert [tuple(x.shape) for x in empty] == [(0, 2), (0, 2)]
