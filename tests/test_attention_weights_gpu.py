"""GPU: head-averaged attention maps (csrc/attention_weights.cu) at model level - through forward hooks on the 12
attention containers against the fp64 oracle - and the C ABI around them.  The kernels themselves are tested against
fp64 in test_attention_maps_gpu.py."""
import ctypes

import pytest
import torch

from oracle import attention_oracle, fixtures

pytestmark = pytest.mark.gpu

TC, SIMT = 0, 1
SEPARATE, DEFERRED = 1 << 16, 1 << 19
# per layer against the fp64 oracle: the maps carry the same upstream drift as the predictions (mem / hs ~1e-4 relative)
MAP_REL, MAP_ABS = 5e-4, 1e-3
# measured on the B = 2, Q = 100 fixture (H100): at most 2.2e-4 relative and 3.1e-4 absolute, both in encoder layer 0
# on the fp32 SIMT path (its logits reach 7.9e3); the tensor-core path is at 1.2e-4 / 1.8e-4 there
FIXTURE_REL, FIXTURE_ABS = 3e-4, 5e-4


def _build(sd=None):
    from cotr_b200.models import build_model
    model = build_model(None)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in (sd if sd is not None else fixtures.make_state_dict(0)).items()})
    return model.cuda().eval()


@pytest.fixture(scope="module")
def model(built_lib):
    return _build()


def _mods(model):
    t = model.transformer
    return ([getattr(t.encoder.layers, str(l)).self_attn for l in range(6)] +
            [getattr(t.decoder.layers, str(l)).multihead_attn for l in range(6)])


def _hook(model, which=range(12)):
    """Forward hooks on the selected containers (odd ones plain, even ones with_kwargs) -> (fired, handles)."""
    mods = _mods(model)
    fired, handles = [], []
    for i in which:
        if i % 2:
            handles.append(mods[i].register_forward_hook(lambda m, a, o, i=i: fired.append((i, a, None, o))))
        else:
            handles.append(mods[i].register_forward_hook(lambda m, a, k, o, i=i: fired.append((i, a, k, o)), with_kwargs=True))
    return fired, handles


def _unhook(handles):
    for h in handles:
        h.remove()


def _maps(fired):
    return {i: o[1].clone() for i, _, _, o in fired}


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.fixture(scope="module")
def b2_q100():
    sd = fixtures.make_state_dict(0, 3.0, 1.35)
    img, queries = fixtures.make_inputs(2, 2, 100)
    _, ref = attention_oracle.forward(sd, img, queries, torch.float64)
    return sd, torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda(), ref


@pytest.mark.parametrize("path,variant", [(TC, 0), (TC, SEPARATE), (TC, DEFERRED), (SIMT, 0)],
                         ids=["tc", "tc-separate", "tc-deferred", "simt"])
def test_hooked_maps_match_oracle(built_lib, b2_q100, path, variant):
    from cotr_b200 import capi
    sd, t, q, ref = b2_q100
    m = _build(sd)
    m.native().set_gemm_path(path)
    capi.lib().cotr_debug_set_variant(variant)
    fired, handles = _hook(m)
    try:
        m(t, q)
    finally:
        capi.lib().cotr_debug_set_variant(0)
        _unhook(handles)
    assert [f[0] for f in fired] == list(range(12))                  # encoder 0..5, then decoder 0..5
    for i, args, kwargs, out in fired:
        assert args == () and (kwargs is None if i % 2 else kwargs == {})
        assert isinstance(out, tuple) and len(out) == 2 and out[0] is None
        w = out[1]
        assert w.dtype == torch.float32 and w.is_cuda and tuple(w.shape) == ((2, 512, 512) if i < 6 else (2, 100, 512))
        assert (w >= 0).all()
        assert (w.double().sum(-1) - 1).abs().max().item() < 1e-5
        err, rel = (w.cpu().double() - ref[i]).abs().max().item(), _rel(w.cpu(), ref[i])
        assert err < FIXTURE_ABS and rel < FIXTURE_REL, (i, err, rel)


def test_hooks_leave_predictions_and_graphs_bitwise(built_lib):
    m = _build()
    img, queries = fixtures.make_inputs(41, 2, 100)
    t, q = torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()
    plain = m(t, q)["pred_corrs"].clone()                            # eager
    fired, handles = _hook(m)
    a = m(t, q)["pred_corrs"].clone()
    maps_a = _maps(fired)
    fired.clear()
    b = m(t, q)["pred_corrs"].clone()
    maps_b = _maps(fired)
    _unhook(handles)
    assert torch.equal(a, plain) and torch.equal(b, plain)
    assert all(torch.equal(maps_a[i], maps_b[i]) for i in range(12))
    assert torch.equal(m(t, q)["pred_corrs"], plain)                 # captured
    assert torch.equal(m(t, q)["pred_corrs"], plain)                 # replayed


def test_engine_shape_and_chunked_decoder(model):
    # Q = 1 at B = 3 (the default engine's step)
    sd = fixtures.make_state_dict(0)
    img, queries = fixtures.make_inputs(3, 3, 1)
    fired, handles = _hook(model)
    try:
        model(torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda())
    finally:
        _unhook(handles)
    _, ref = attention_oracle.forward(sd, img, queries, torch.float64)
    for i, _, _, out in fired:
        w = out[1]
        assert tuple(w.shape) == ((3, 512, 512) if i < 6 else (3, 1, 512))
        assert (w.cpu().double() - ref[i]).abs().max().item() < MAP_ABS and _rel(w.cpu(), ref[i]) < MAP_REL, i
    # Q = 40000 > one decoder chunk of 32768 rows: per-slice chunks write at their query offset
    img, queries = fixtures.make_inputs(11, 1, 40000)
    t, q = torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()
    fired, handles = _hook(model, (6, 11))
    try:
        full = model(t, q)["pred_corrs"]
        big = _maps(fired)
        fired.clear()
        part = model(t, q[:, 35000:36000].contiguous())["pred_corrs"]
        small = _maps(fired)
    finally:
        _unhook(handles)
    assert (full[:, 35000:36000] - part).abs().max().item() < 2e-4
    for i in (6, 11):
        assert tuple(big[i].shape) == (1, 40000, 512)
        assert (big[i][:, 35000:36000] - small[i]).abs().max().item() < 2e-4, i
        assert (big[i].double().sum(-1) - 1).abs().max().item() < 1e-5


def test_c_abi_masks(model):
    from cotr_b200 import capi
    nat = model.native()
    img, queries = fixtures.make_inputs(42, 2, 64)
    t, q = torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()
    ctx = capi.NativeContext(nat, 2)
    nat.encode_context(t, ctx)
    plain = nat.decode(ctx, q)
    assert nat.encode_context_attention(t, ctx, 0).shape == (0, 2, 512, 512)
    pred, maps = nat.decode_attention(ctx, q, 0)
    assert maps.shape == (0, 2, 64, 512) and torch.equal(pred, plain)
    enc = nat.encode_context_attention(t, ctx, 0b100001)
    pred, maps = nat.decode_attention(ctx, q, 0b010010)
    assert enc.shape == (2, 2, 512, 512) and maps.shape == (2, 2, 64, 512) and torch.equal(pred, plain)
    lib, s = capi.lib(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.empty(7 * 2 * 512 * 512, device="cuda")
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    assert lib.cotr_encode_context_attention(nat.handle, p(t), 2, ctx.handle, 1 << 6, p(buf), s) != 0
    assert "layer_mask" in capi.last_error()
    assert lib.cotr_encode_context_attention(nat.handle, p(t), 2, ctx.handle, 1, None, s) != 0
    assert "attn_dev" in capi.last_error()
    out = torch.empty(2, 64, 2, device="cuda")
    assert lib.cotr_decode_attention(nat.handle, ctx.handle, p(q), 2, 64, 0x41, p(buf), p(out), s) != 0
    assert "layer_mask" in capi.last_error()
    assert lib.cotr_decode_attention(nat.handle, ctx.handle, p(q), 2, 64, 2, None, p(out), s) != 0
    assert "attn_dev" in capi.last_error()
    torch.cuda.synchronize()
    ctx.close()


def test_launch_count(model):
    from cotr_b200 import capi
    img, queries = fixtures.make_inputs(1, 1, 1024)
    t, q = torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()
    nat = model.native()
    model(t, q)
    assert nat.last_launch_count() == 111
    ctx = capi.NativeContext(nat, 1)
    nat.encode_context(t, ctx)
    n_enc = nat.last_launch_count()
    nat.decode(ctx, q)
    assert n_enc + nat.last_launch_count() == 111
    nat.encode_context_attention(t, ctx, 0b000101)
    assert nat.last_launch_count() == n_enc + 2
    nat.decode_attention(ctx, q, 0b111000)
    assert nat.last_launch_count() == 111 - n_enc + 3
    nat.encode_context_attention(t, ctx, 0b111111)
    n = nat.last_launch_count()
    nat.decode_attention(ctx, q, 0b111111)
    assert n + nat.last_launch_count() == 111 + 12
    torch.cuda.synchronize()
    ctx.close()
