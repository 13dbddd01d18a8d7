"""GPU: every GEMM the model launches, through the kernel-level hook (cotr_test_gemm) in its own configuration, against
fp64 torch math on both matrix-multiply paths.

The model's GEMMs are written down once (`model_gemms`), and that table is checked against the profiler records of
whole forwards, so a schedule change that adds, drops or reshapes a GEMM makes this file fail rather than go stale.
Each row then runs with the plan the launch rule picks (asserted against a restatement of the rule) and with every
other legal tile width and split-K forced.  As in test_kernels_gpu.py, inputs are split16 fixed points, memory a launch
must not read holds NaN, and memory it must not write holds SENTINEL and has to come back bitwise."""
import collections

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TC, SIMT = 0, 1
SENTINEL = 1000.5
NAN = float("nan")
VARIANT_EXPLICIT, VARIANT_DEFERRED = 1 << 16, 1 << 19
IMG_HEAD = 132096                     # common.cuh kAttnHeadImgBytes: K image 65536 B, V image 64 x 1040 B
# Relative error bounds against fp64, Frobenius norm over the output / worst single row (see _check), about twice the
# largest measured over both paths and every plan on an H100 SXM (80 GB HBM3, 700 W): backbone 1.4e-6 / 1.7e-6,
# transformer 7.0e-7 / 4.2e-6, deferred LayerNorm 5.5e-7 / 1.6e-6, redirected keys and values 4.0e-7 / 1.3e-6.
BOUNDS = {"backbone": (3e-6, 4e-6), "transformer": (1.5e-6, 1e-5), "deferred": (1.2e-6, 4e-6), "redirected": (1e-6, 3e-6)}


def _fix16(x):
    """x rounded to a split16 fixed point (hi = fp16(x), lo = fp16(x - hi), twice: at fp16 ties the split of hi + lo
    is not the split of x)."""
    for _ in range(2):
        hi = x.half().float()
        x = hi + (x - hi).half().float()
    return x


def _check(out, ref, group):
    """Relative error of the whole output and of its worst row against the group's bounds; returns both.  A row is
    measured against at least a tenth of the RMS row norm: the 2-wide head has rows near zero whose relative error is
    that of a cancelling dot product."""
    out, ref = out.double(), ref.double()
    assert torch.isfinite(out).all(), "non-finite output: the launch read memory it must not read"
    err = ((out - ref).norm() / ref.norm()).item()
    norms = ref.norm(dim=-1)
    row = ((out - ref).norm(dim=-1) / norms.clamp_min(0.1 * norms.square().mean().sqrt().item())).max().item()
    print(f"ERR {group} {err:.3e} {row:.3e}")
    rel, row_rel = BOUNDS[group]
    assert err < rel and row < row_rel, (group, err, row)
    return err, row


@pytest.fixture(scope="module")
def capi(built_lib):
    from cotr_b200 import capi
    capi.lib()
    return capi


# ---- the model's GEMMs -------------------------------------------------------------------------------------------
# A row: name, (M, N, K) as the profiler records it, and how the launch is made.  conv: (H, W, C, OH, OW, k, stride,
# pad) of a backbone convolution (k = 1 and stride 1: a row-major GEMM over pixels); epi: the epilogue operands
# ("relu", "res", "ln", "a_ln", "res_ln", "part", "add", "kv", "qres", "f32").
Row = collections.namedtuple("Row", "name M N K conv epi")
BLOCKS = [(64, 64, 256, 3, 1), (256, 128, 512, 4, 2), (512, 256, 1024, 6, 2)]     # (in, mid, out, blocks, stride) of layer1-3


def _backbone(n):
    rows = [Row("stem", n * 128 * 128, 64, 224, (256, 256, 3, 128, 128, 7, 2, 3), ("relu",))]
    H = 64
    for li, (cin, mid, cout, nb, stride) in enumerate(BLOCKS):
        for b in range(nb):
            s = stride if b == 0 else 1
            ci = cin if b == 0 else cout
            OH = H // s
            tag = f"layer{li + 1}.{b}"
            rows.append(Row(f"{tag}.c1", n * H * H, mid, ci, (H, H, ci, H, H, 1, 1, 0), ("relu",)))
            rows.append(Row(f"{tag}.c2", n * OH * OH, mid, 9 * mid, (H, H, mid, OH, OH, 3, s, 1), ("relu",)))
            if b == 0:
                rows.append(Row(f"{tag}.ds", n * OH * OH, cout, ci, (H, H, ci, OH, OH, 1, s, 0), ()))
            rows.append(Row(f"{tag}.c3", n * OH * OH, cout, mid, (OH, OH, mid, OH, OH, 1, 1, 0), ("relu", "res")))
            H = OH
    return rows


def _deferred(rows, tc, variant):
    """deferred_ln_enabled: the tensor-core path, from 2048 rows, unless a variant bit pins the schedule."""
    if not tc or variant == VARIANT_EXPLICIT:
        return False
    return variant == VARIANT_DEFERRED or rows >= 2048


def model_gemms(B, R, tc=True, variant=0, encode=True):
    """(kernel, row) of every GEMM launch of a forward of B pairs decoding R rows in one chunk (encode=False: the
    decode alone).  kernel is the profiler's name."""
    T = B * 512
    kern = "gemm_tc" if tc else "gemm_simt"
    fused = tc and variant != VARIANT_EXPLICIT            # fused_mlp_enabled (explicit schedule only)
    rows = []
    if encode:
        rows += _backbone(2 * B)
        rows.append(Row("input_proj", T, 256, 1024, None, ("pairs",)))
        d = _deferred(T, tc, variant)
        for l in range(6):
            a_ln = ("a_ln",) if d and l > 0 else ()
            rows.append(Row(f"enc{l}.qkv", T, 768, 256, None, ("add", "kv") + a_ln))
            if d:
                rows.append(Row(f"enc{l}.o", T, 256, 256, None, ("res", "part") + (("res_ln",) if l > 0 else ())))
                rows.append(Row(f"enc{l}.l1", T, 1024, 256, None, ("relu", "a_ln")))
                rows.append(Row(f"enc{l}.l2", T, 256, 1024, None, ("res", "res_ln", "part")))
            else:
                rows.append(Row(f"enc{l}.o", T, 256, 256, None, ("res", "ln")))
                if not fused:
                    rows.append(Row(f"enc{l}.l1", T, 1024, 256, None, ("relu",)))
                    rows.append(Row(f"enc{l}.l2", T, 256, 1024, None, ("res", "ln")))
        rows.append(Row("kv_all", T, 3072, 256, None, ("add", "kv") + (("a_ln",) if d else ())))
    d = _deferred(R, tc, variant)
    rows.append(Row("qpos_all", R, 1536, 256, None, ()))
    for l in range(6):
        if l > 0:
            rows.append(Row(f"dec{l}.q", R, 256, 256, None, ("qres",) + (("a_ln",) if d else ())))
        if d:
            rows.append(Row(f"dec{l}.o", R, 256, 256, None, ("part",) + (("res", "res_ln") if l > 0 else ())))
            rows.append(Row(f"dec{l}.l1", R, 1024, 256, None, ("relu", "a_ln")))
            rows.append(Row(f"dec{l}.l2", R, 256, 1024, None, ("res", "res_ln", "part")))
        else:
            rows.append(Row(f"dec{l}.o", R, 256, 256, None, ("ln",) + (("res",) if l > 0 else ())))
            if not fused:
                rows.append(Row(f"dec{l}.l1", R, 1024, 256, None, ("relu",)))
                rows.append(Row(f"dec{l}.l2", R, 256, 1024, None, ("res", "ln")))
    rows += [Row("head0", R, 256, 256, None, ("relu",)), Row("head1", R, 256, 256, None, ("relu",)),
             Row("head2", R, 2, 256, None, ("f32",))]
    return [(kern, r) for r in rows]


FORWARDS = [(1, 1024), (2, 100), (4, 1024), (16, 1024)]
SETTINGS = {"default": (TC, 0), "explicit": (TC, VARIANT_EXPLICIT), "deferred": (TC, VARIANT_DEFERRED), "simt": (SIMT, 0)}


@pytest.fixture(scope="module")
def native_model(built_lib):
    from cotr_b200 import capi
    from cotr_b200.utils import synthetic
    model = capi.NativeModel(synthetic.make_state_dict(0), 0)
    yield model
    model.close()


def _gemm_records(model):
    return collections.Counter((r[0], r[1], r[2], r[3]) for r in model.profile_end() if r[0] in ("gemm_tc", "gemm_simt"))


@pytest.mark.parametrize("setting", list(SETTINGS))
def test_table_is_the_models(capi, native_model, setting):
    """The table's (kernel, M, N, K) multiset equals the profiler's GEMM records of whole forwards and of one ragged
    decode, under each schedule and on both paths."""
    from cotr_b200.utils import synthetic
    path, variant = SETTINGS[setting]
    capi.lib().cotr_debug_set_variant(variant)
    try:
        native_model.set_gemm_path(1 - path)          # a path switch drops graphs captured under another variant
        native_model.set_gemm_path(path)
        for B, Q in FORWARDS:
            img, q = (torch.from_numpy(t).cuda() for t in synthetic.make_inputs(B * 7 + Q, B, Q))
            native_model.profile_begin(8192)
            native_model.forward(img, q)
            got = _gemm_records(native_model)
            want = collections.Counter((k, r.M, r.N, r.K) for k, r in model_gemms(B, B * Q, path == TC, variant))
            assert got == want, (B, Q, got - want, want - got)
        counts = [3, 0, 100, 1500]
        ctx = capi.NativeContext(native_model, len(counts))
        img, _ = synthetic.make_inputs(5, len(counts), 1)
        native_model.encode_context(torch.from_numpy(img).cuda(), ctx)
        offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        q = torch.rand((int(offsets[-1]), 2), generator=torch.Generator().manual_seed(3)).cuda()
        native_model.profile_begin(8192)
        native_model.decode_ragged(ctx, q, offsets)
        got = _gemm_records(native_model)
        want = collections.Counter((k, r.M, r.N, r.K) for k, r in model_gemms(len(counts), sum(counts), path == TC, variant, encode=False))
        assert got == want, (got - want, want - got)
        ctx.close()
    finally:
        capi.lib().cotr_debug_set_variant(0)
        native_model.set_gemm_path(1)
        native_model.set_gemm_path(0)


# ---- the launch rule (gemm_tc.cu rule_tile / plan_split), restated ---------------------------------------------------
def _halo_candidate(conv):
    H, W, C, OH, OW, k, s, pd = conv
    return k == 3 and s == 1 and pd == 1 and OH == H and OW == W and C % 64 == 0


def _halo_tiles(conv, M):
    H, W, C, OH, OW = conv[:5]
    return M // (OH * OW) * -(-(OH * (W + 2)) // 128)


def _loader(row):
    if row.conv is None or (row.conv[5] == 1 and row.conv[6] == 1):
        return "gather"
    if row.name == "stem":
        return "stem"
    return "halo" if _halo_candidate(row.conv) else "im2col"


def _grid(row, bn, loader):
    bm = 64 if bn == 256 else 128
    gx = _halo_tiles(row.conv, row.M) if loader == "halo" else -(-row.M // bm)
    return gx, -(-row.N // bn)


def _split_rule(row, bn, loader):
    if bn == 256 or loader == "stem":
        return 1
    kc = -(-row.K // 64)
    cc = row.conv[2] // 64 if loader == "halo" else kc
    gx, gy = _grid(row, bn, loader)
    wave = 132 if loader == "halo" else 144
    if kc >= 16:
        for ks in (4, 2):
            if kc % ks == 0 and cc % ks == 0 and gx * gy * ks <= wave:
                return ks
    return 1


def _halo_fits(row, ks, grid):
    H, W, C = row.conv[:3]
    ccp = C // 64 // ks
    plane = (128 + 2 * (W + 2) + 2 + 7) // 8 * 8 * 128
    return ccp <= 4 and ccp * 2 * plane <= 100 * 1024 and grid[0] * grid[1] * ks >= 86


def _plan(row, bn=None, ks=None):
    """The plan the launch makes for this row, with the tile width / split forced where given (the test hook's rule)."""
    loader = _loader(row)
    if bn is None:
        if row.N < 64:
            bn = 16
        else:
            mt = _halo_tiles(row.conv, row.M) if loader == "halo" else -(-row.M // 128)
            bn = 64 if mt * -(-row.N // 64) >= 86 or loader == "stem" or row.N % 32 else 32
    split = ks or _split_rule(row, bn, loader)
    if loader == "halo" and not _halo_fits(row, split, _grid(row, bn, loader)):
        loader = "im2col"
        split = ks or _split_rule(row, bn, loader)
    dln = bn < 256 and any(e in row.epi for e in ("a_ln", "res_ln", "part"))
    return dict(bn=bn, loader=loader, dln=int(dln), ksplit=split, grid=_grid(row, bn, loader))


def _legal(row, bn, ks, loader):
    kc = -(-row.K // 64)
    cc = row.conv[2] // 64 if loader == "halo" else kc
    return ks <= (4 if bn in (32, 64) else 1) and (ks == 1 or loader != "stem") and kc % ks == 0 and cc % ks == 0


# ---- one row through the hook --------------------------------------------------------------------------------------
def _inputs(row, g, B):
    """Operands at the layer's magnitudes: post-ReLU activations behind the stem, rows with a mean of several sigma
    where a deferred LayerNorm applies; weights scaled like a trained layer's."""
    t = {}
    W = torch.randn(row.N, row.K if row.name != "stem" else 147, generator=g) * (2.0 / row.K) ** 0.5
    t["W"] = W
    t["bias"] = (torch.randn(row.N, generator=g) * 0.1).cuda()
    if row.conv is not None:
        H, Wd, C, OH, OW, k, s, pd = row.conv
        n = row.M // (OH * OW)
        if row.name == "stem":
            t["A"] = torch.randn(n // 2, 3, 256, 512, generator=g).cuda()
        else:
            t["A"] = _fix16(torch.randn(n, H, Wd, C, generator=g).abs() * 0.5).cuda()
    elif "pairs" in row.epi:
        t["A"] = _fix16(torch.randn(2 * B + 1, 16, 16, 1024, generator=g).abs() * 0.5).cuda()
        t["A"][-1] = NAN                               # an image no pair reads
    else:
        A = torch.randn(row.M, row.K, generator=g)
        if "a_ln" in row.epi:
            A = A * (0.5 + torch.rand(row.M, 1, generator=g) * 4) + 3.0
        t["A"] = _fix16(A).cuda()
    if "res" in row.epi:
        res = torch.randn(row.M, row.N, generator=g)
        res = res.abs() if row.conv is not None else res * 2 + (0.7 if "res_ln" in row.epi else 0)
        t["res"] = _fix16(res).cuda()
    if "qres" in row.epi:
        t["res"] = _fix16(torch.randn(row.M, 1536, generator=g)).cuda()
    if any(e in row.epi for e in ("ln", "a_ln", "res_ln")):
        n = row.K if "a_ln" in row.epi else row.N
        t["ln"] = ((1 + 0.2 * torch.randn(n, generator=g)).cuda(), (0.2 * torch.randn(n, generator=g)).cuda())
    if "add" in row.epi:
        t["add"] = torch.randn(512, row.N, generator=g).cuda()
    return t


def _ref(row, t, l_res=0, pairs=None):
    Wd = t["W"].cuda().double()
    if row.name == "stem":
        img = t["A"].double()
        halves = torch.stack([img[..., :256], img[..., 256:]], 1).reshape(-1, 3, 256, 256)     # image 2 pair + half
        w = Wd.reshape(row.N, 7, 7, 3).permute(0, 3, 1, 2)
        y = F.conv2d(halves, w, stride=2, padding=3).permute(0, 2, 3, 1).reshape(-1, row.N)
    elif row.conv is not None:
        H, W_, C, OH, OW, k, s, pd = row.conv
        w = Wd.reshape(row.N, k, k, C).permute(0, 3, 1, 2)
        y = F.conv2d(t["A"].double().permute(0, 3, 1, 2), w, stride=s, padding=pd).permute(0, 2, 3, 1).reshape(-1, row.N)
    elif "pairs" in row.epi:
        f = t["A"].double()
        y = torch.cat([torch.cat([f[a], f[b]], 1).reshape(512, 1024) for a, b in pairs]) @ Wd.t()
    else:
        A = t["A"].double()
        if "a_ln" in row.epi:
            A = F.layer_norm(A, (row.K,), t["ln"][0].double(), t["ln"][1].double(), 1e-5)
        y = A @ Wd.t()
    y = y + t["bias"].double()
    if "add" in row.epi:
        y = y + t["add"].double().repeat(row.M // 512, 1)
    if "res" in row.epi:
        r = t["res"].double()
        if "res_ln" in row.epi:
            r = F.layer_norm(r, (row.N,), t["ln"][0].double(), t["ln"][1].double(), 1e-5)
        y = y + r
    if "qres" in row.epi:
        y = y + t["res"].double()[:, l_res:l_res + row.N]
    if "relu" in row.epi:
        y = y.relu()
    if "ln" in row.epi:
        y = F.layer_norm(y, (row.N,), t["ln"][0].double(), t["ln"][1].double(), 1e-5)
    return y


def _kv_blocks(row):
    """the model's redirect_kv of the row (vt layout): [q,] then a (key, value) block pair per slot"""
    if row.N == 768:
        return [0, 256, -1], 1, 512
    return [x for l in range(6) for x in (256 * l, -(l + 1))], 6, 1536


def _run(capi, row, t, path, pairs=None, **kw):
    """The row through the hook -> (row-major output restricted to the row's values, plan)."""
    plan = {}
    args = dict(bias=t["bias"], relu="relu" in row.epi, plan=plan, **kw)
    if "ln" in t:
        args["ln"] = t["ln"]
    if "a_ln" in row.epi:
        args["a_ln"] = True
    if "res_ln" in row.epi:
        args["res_ln"] = True
    if "res" in t:
        args["residual"] = t["res"]
    if "add" in row.epi:
        args.update(addmat=t["add"], add_period=512)
    if "part" in row.epi and path == TC:
        args["part_out"] = torch.zeros(row.M, 16, 2, device="cuda")
    W = t["W"].numpy()
    if row.name == "stem":
        out = capi.test_gemm(path, t["A"], W, a_mode=2, M=row.M, conv=dict(zip("H W C OH OW".split(), row.conv[:5]),
                             KH=7, KW=7, stride=2, pad=3), **args)
        return out, plan
    if row.conv is not None and not (row.conv[5] == 1 and row.conv[6] == 1):
        H, W_, C, OH, OW, k, s, pd = row.conv
        out = capi.test_gemm(path, t["A"], W, a_mode=1, M=row.M, conv=dict(H=H, W=W_, C=C, OH=OH, OW=OW, KH=k, KW=k, stride=s, pad=pd), **args)
        return out, plan
    A = t["A"].reshape(-1, t["A"].shape[-1]) if row.conv is not None else t["A"]
    if "pairs" in row.epi:
        return capi.test_gemm(path, t["A"], W, a_mode=3, M=row.M, pairs=pairs, **args), plan
    if "kv" in row.epi:
        blk, n_vt, ldc = _kv_blocks(row)
        B = row.M // 512
        vt = torch.full((B, n_vt, 256, 512), SENTINEL, device="cuda")
        out = torch.full((row.M, ldc), SENTINEL, device="cuda")
        capi.test_gemm(path, A, W, blk_map=blk, n_vt=n_vt, vt=vt, out=out, **args)
        vals = torch.empty(row.M, row.N, device="cuda")
        for b, m in enumerate(blk):
            if m >= 0:
                vals[:, 256 * b:256 * b + 256] = out[:, m:m + 256]
            else:
                vals[:, 256 * b:256 * b + 256] = vt[:, -m - 1].transpose(1, 2).reshape(row.M, 256)
        assert (vt == SENTINEL).sum() == 0 and (out == SENTINEL).sum() == (row.M * (ldc - 256 * sum(m >= 0 for m in blk)))
        return vals, plan
    return capi.test_gemm(path, A, W, **args), plan


def _group(row):
    if row.conv is not None:
        return "backbone"
    return "deferred" if any(e in row.epi for e in ("a_ln", "res_ln", "part")) else "transformer"


def _check_row(capi, row, path, B, seed):
    g = torch.Generator().manual_seed(seed)
    t = _inputs(row, g, B)
    pairs = None
    if "pairs" in row.epi:         # repeats, self-pairs and swapped pairs; image 2B is NaN and never read
        pairs = [(2 * p, 2 * p + 1) if p % 3 == 0 else ((2 * p + 1, 2 * p) if p % 3 == 1 else (p, p)) for p in range(B)]
        if B > 1:
            pairs[-1] = pairs[0]
    l_res = 256 * int(row.name[3]) if "qres" in row.epi else 0
    kw = dict(res_col0=l_res) if "qres" in row.epi else {}
    ref = _ref(row, t, l_res, pairs)
    out, plan = _run(capi, row, t, path, pairs, **kw)
    _check(out, ref, _group(row))
    if path == SIMT:
        return
    rule = _plan(row)
    if "ln" in row.epi:
        defused = (row.M + 127) // 128 < 64
        assert plan["ln_defused"] == int(defused)
        rule = _plan(row, bn=None if defused else 256)
    assert {k: plan[k] for k in rule} == rule, (row, plan, rule)
    # every other legal tile width and split on the same inputs
    widths = [16] if row.N < 64 else ([64, 32] if row.N % 32 == 0 and row.name != "stem" else [64])
    if "ln" in row.epi:
        widths = [256] + widths
    for bn in widths:
        for ks in (1, 2, 4):
            forced = _plan(row, bn=bn, ks=ks)
            if (bn, ks) == (rule["bn"], rule["ksplit"]) or not _legal(row, bn, ks, _loader(row)):
                continue
            out_f, plan_f = _run(capi, row, t, path, pairs, bn=bn, ksplit=ks, **kw)
            assert {k: plan_f[k] for k in forced} == forced, (row, plan_f, forced)
            _check(out_f, ref, _group(row))


def _unique(rows):
    seen, out = set(), []
    for _, r in rows:
        key = (r.M, r.N, r.K, r.conv, r.epi)
        if key not in seen:
            seen.add(key)
            out.append(r)
    return out


@pytest.mark.parametrize("B", [1, 4, 16])
@pytest.mark.parametrize("path", [TC, SIMT])
def test_backbone_gemms(capi, B, path):
    """Every convolution of the backbone of B pairs: the 86-CTA tile threshold, split-K 4 / 2 / 1 and halo versus
    im2col fall on different rows at 2, 8 and 32 images."""
    for i, row in enumerate(_unique([("", r) for r in _backbone(2 * B)])):
        _check_row(capi, row, path, B, seed=i + 100 * B)


@pytest.mark.parametrize("B,R", [(1, 100), (1, 2047), (4, 2048), (16, 1024), (16, 8192)])
@pytest.mark.parametrize("setting", ["explicit", "deferred", "simt"])
def test_transformer_gemms(capi, B, R, setting):
    """Every transformer GEMM: 512 .. 8192 context rows and 100 .. 8192 decode rows straddle the 2048-row deferred
    threshold and the 64-tile LayerNorm defuse threshold (8192 rows); both schedules on the tensor cores."""
    path, variant = SETTINGS[setting]
    rows = [r for k, r in model_gemms(B, R, path == TC, variant) if r.conv is None]
    for i, row in enumerate(_unique([("", r) for r in rows])):
        _check_row(capi, row, path, B, seed=i + 1000 * B + R)


# ---- redirected stores: the operand images -------------------------------------------------------------------------
def _decode_images(img, pairs, n_vt):
    """(pairs*n_vt*8*132096,) uint8 -> K, V (pairs, n_vt, 512, 256) fp32 (hi + lo) and the 16-byte pads of the V groups.
    K image [plane][4 groups of 8 dims][512 keys][8 halves]; V image [64 groups of 8 keys][hi 32 dims x 8 | lo | pad]."""
    b = img.cpu().numpy().reshape(pairs, n_vt, 8, IMG_HEAD)
    k = b[..., :65536].copy().view(np.float16).reshape(pairs, n_vt, 8, 2, 4, 512, 8).astype(np.float32)
    k = k[:, :, :, 0] + k[:, :, :, 1]                                 # (P, S, head, group, key, e)
    K = k.transpose(0, 1, 4, 2, 3, 5).reshape(pairs, n_vt, 512, 256)
    vg = b[..., 65536:].reshape(pairs, n_vt, 8, 64, 1040)
    pad = vg[..., 1024:]
    v = vg[..., :1024].copy().view(np.float16).reshape(pairs, n_vt, 8, 64, 2, 32, 8).astype(np.float32)
    v = v[:, :, :, :, 0] + v[:, :, :, :, 1]                           # (P, S, head, group, dim, e)
    V = v.transpose(0, 1, 3, 5, 2, 4).reshape(pairs, n_vt, 512, 256)
    return K, V, pad


@pytest.mark.parametrize("which,B,a_ln", [("qkv", 1, False), ("qkv", 3, True), ("kv_all", 1, False), ("kv_all", 2, True),
                                          ("kv_all", 16, True)])
def test_redirected_stores(capi, which, B, a_ln):
    """The qkv / kv_all GEMMs into the operand images, under the rule's plan and every forced one: the decoded planes
    equal bitwise the K and transposed V of the same GEMM with the row-major target; every image byte outside the
    layout (V group pads, the slot and pair no block writes) stays 0xFF; passthrough blocks land at their blk_map
    columns and the other columns keep the sentinel."""
    M, N = B * 512, 768 if which == "qkv" else 3072
    row = Row(which, M, N, 256, None, ("add", "kv") + (("a_ln",) if a_ln else ()))
    g = torch.Generator().manual_seed(B * 13 + N)
    t = _inputs(row, g, B)
    blk_vt, n_vt, ldc = _kv_blocks(row)
    off = 1 if which == "qkv" else 0                    # the key block of slot l is block off + 2 l
    blk_img = [0, -1000, -1] if which == "qkv" else [x for l in range(6) for x in (-1000 - l, -(l + 1))]
    slots, pairs = n_vt + 1, B + 1                       # one slot and one pair the launch never writes
    kw = dict(bias=t["bias"], addmat=t["add"], add_period=512, n_vt=slots)
    if a_ln:
        kw.update(ln=t["ln"], a_ln=True)
    ref = _ref(row, t)
    for bn, ks in [(0, 0), (64, 1), (32, 1), (64, 2), (32, 4)]:
        out = torch.full((M + 3, ldc), SENTINEL, device="cuda")
        vt = torch.full((pairs, slots, 256, 512), SENTINEL, device="cuda")
        plan_v, plan_i = {}, {}
        capi.test_gemm(TC, t["A"], t["W"].numpy(), blk_map=blk_vt, vt=vt, out=out, bn=bn, ksplit=ks, plan=plan_v, **kw)
        out_i = torch.full((M + 3, ldc), SENTINEL, device="cuda")
        img = torch.full((pairs * slots * 8 * IMG_HEAD,), 0xFF, dtype=torch.uint8, device="cuda")
        capi.test_gemm(TC, t["A"], t["W"].numpy(), blk_map=blk_img, img=img, out=out_i, bn=bn, ksplit=ks, plan=plan_i, **kw)
        assert plan_v == plan_i
        K, V, pad = _decode_images(img, pairs, slots)
        for l in range(n_vt):
            kb = off + 2 * l
            kcol = blk_vt[kb]
            k_rm = out[:M, kcol:kcol + 256].cpu().numpy().reshape(B, 512, 256)
            v_rm = vt[:B, l].transpose(1, 2).cpu().numpy()
            assert np.array_equal(K[:B, l].view(np.uint32), k_rm.view(np.uint32))
            assert np.array_equal(V[:B, l].view(np.uint32), v_rm.view(np.uint32))
            _check(torch.from_numpy(K[:B, l].reshape(M, 256)), ref[:, 256 * kb:256 * kb + 256].cpu(), "redirected")
            _check(torch.from_numpy(V[:B, l].reshape(M, 256)), ref[:, 256 * kb + 256:256 * kb + 512].cpu(), "redirected")
        assert (pad == 0xFF).all()
        raw = img.cpu().numpy().reshape(pairs, slots, 8 * IMG_HEAD)
        assert (raw[B:] == 0xFF).all() and (raw[:, n_vt:] == 0xFF).all()
        assert (vt[B:] == SENTINEL).all() and (vt[:, n_vt:] == SENTINEL).all() and (out[M:] == SENTINEL).all()
        if which == "qkv":                     # q passes through to columns 0..255; the key columns stay untouched
            assert torch.equal(out_i[:M, :256], out[:M, :256])
            assert (out_i[:, 256:] == SENTINEL).all() and (out_i[M:] == SENTINEL).all()
            _check(out_i[:M, :256], ref[:, :256], "redirected")
        else:
            assert (out_i == SENTINEL).all()


# ---- token gather through a pair table -----------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 16])
@pytest.mark.parametrize("path", [TC, SIMT])
def test_input_proj_pair_table(capi, B, path):
    """input_proj reading the (n,16,16,1024) features through a pair table with repeats, self-pairs and swapped pairs;
    one image no pair names is NaN."""
    n_img = max(2, B)
    g = torch.Generator().manual_seed(B + 77)
    feat = _fix16(torch.randn(n_img + 1, 16, 16, 1024, generator=g).abs() * 0.5)
    feat[n_img] = NAN
    feat = feat.cuda()
    rnd = np.random.default_rng(B)
    pairs = rnd.integers(0, n_img, size=(B, 2))
    if B >= 3:
        pairs[0] = (0, 0)                   # self-pair
        pairs[1] = pairs[2][::-1]           # swapped
        pairs[-1] = pairs[2]                # repeat
    W = torch.randn(256, 1024, generator=g) * (2 / 1024) ** 0.5
    bias = (torch.randn(256, generator=g) * 0.1).cuda()
    f = feat.double()
    ref = torch.cat([torch.cat([f[a], f[b]], 1).reshape(512, 1024) for a, b in pairs]) @ W.cuda().double().t() + bias.double()
    out = capi.test_gemm(path, feat, W.numpy(), bias=bias, a_mode=3, M=B * 512, pairs=pairs)
    _check(out, ref, "transformer")


# ---- N that is not a multiple of the tile width --------------------------------------------------------------------
@pytest.mark.parametrize("M", [200, 20000])
@pytest.mark.parametrize("N,bn", [(80, 0), (112, 0), (208, 0), (96, 32), (96, 64), (96, 0)])
@pytest.mark.parametrize("ldc_pad", [0, 48])
def test_columns_past_n(capi, M, N, bn, ldc_pad):
    """The 64-wide tile's last column tile covers columns past N: they must not be stored.  Spare sentinel rows and
    columns past ldc = N + ldc_pad must come back bitwise."""
    g = torch.Generator().manual_seed(M + N + bn + ldc_pad)
    K = 256
    A = torch.full((M, K + 64), NAN)
    A[:, :K] = _fix16(torch.randn(M, K, generator=g))
    A = A.cuda()
    W = torch.randn(N, K, generator=g) * 0.06
    bias = (torch.randn(N, generator=g) * 0.1).cuda()
    ref = A[:, :K].double() @ W.cuda().double().t() + bias.double()
    out = torch.full((M + 5, N + ldc_pad), SENTINEL, device="cuda")
    plan = {}
    capi.test_gemm(TC, A, W.numpy(), bias=bias, M=M, out=out, bn=bn, plan=plan)
    _check(out[:M, :N], ref, "transformer")
    assert (out[:M, N:] == SENTINEL).all() and (out[M:] == SENTINEL).all()
    if bn == 0:
        assert plan["bn"] == _plan(Row("", M, N, K, None, ()))["bn"]


# ---- rejections ----------------------------------------------------------------------------------------------------
def test_gemm_rejects_bad_descriptors(capi):
    """Bad descriptors fail with a message before anything is launched: out comes back untouched."""
    A = torch.zeros(512, 256, device="cuda")
    W = np.zeros((256, 256), np.float32)
    A6 = torch.zeros(512, 384, device="cuda")
    feat = torch.zeros(2, 16, 16, 1024, device="cuda")
    x = torch.zeros(2, 64, 64, 64, device="cuda")
    conv = dict(H=64, W=64, C=64, OH=64, OW=64, KH=3, KW=3, stride=1, pad=1)
    img = torch.zeros(8 * IMG_HEAD, dtype=torch.uint8, device="cuda")
    bad = [
        (dict(A=A6, w=np.zeros((256, 384), np.float32), ksplit=4), "split-K 4 does not divide 6 K chunks"),
        (dict(A=A, w=W, ksplit=3), "split-K 3"),
        (dict(A=torch.zeros(512, 1024, device="cuda"), w=np.zeros((2, 1024), np.float32), ksplit=2, out=torch.full((512, 2), SENTINEL, device="cuda")),
         "split-K 2 on the 16-wide tile"),
        (dict(A=A, w=np.zeros((80, 256), np.float32), bn=32), "no 32-wide tile for N = 80"),
        (dict(A=A, w=W, residual=torch.zeros(512, 512, device="cuda"), res_col0=272), "residual columns 272 .. 527 of ldr 512"),
        (dict(A=feat, w=np.zeros((256, 1024), np.float32), a_mode=3, M=512, pairs=[[0, 2]]), "pair 0 reads image 2 of 2"),
        (dict(A=x.reshape(-1, 64), w=np.zeros((256, 576), np.float32), a_mode=1, M=2 * 64 * 64, conv=conv, blk_map=[-1000],
              n_vt=1, img=img.repeat(16)), "the halo loader needs whole images and a plain split16 output"),
        (dict(A=A, w=W, blk_map=[-2], n_vt=1, vt=torch.zeros(1, 1, 256, 512, device="cuda")), "blk_map\\[0\\] = -2"),
    ]
    for kw, msg in bad:
        kw = dict(kw)
        A_, w_ = kw.pop("A"), kw.pop("w")
        M = kw.get("M", A_.shape[0])
        out = kw.pop("out", torch.full((M, 256), SENTINEL, device="cuda"))
        with pytest.raises(RuntimeError, match=msg):
            capi.test_gemm(TC, A_, w_, out=out, **kw)
        assert (out == SENTINEL).all(), msg
