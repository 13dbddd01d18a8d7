"""GPU: kernel-level parity of the hand-written CUDA kernels (through the C ABI test hooks) against fp64 torch math."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TC, SIMT = 0, 1
# relative (Frobenius) error bounds: fp32 SIMT accumulates in fp32; the wgmma path uses the fp16 hi/lo split
# (3 products, fp32 accumulate in registers), which is fp32-class (gemm_tc.cu header)
REL = {SIMT: 2e-6, TC: 2.5e-6}


def _rel(a, b):
    a = a.double(); b = b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.fixture(scope="module")
def capi(built_lib):
    from cotr_b200 import capi
    capi.lib()
    return capi


def _gen(seed=0):
    return torch.Generator(device="cpu").manual_seed(seed)


@pytest.mark.parametrize("path", [TC, SIMT])
@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (512, 256, 256), (1000, 768, 256), (512, 256, 1024), (37, 2, 256),
                                   (8192, 64, 256), (300, 3072, 256), (1, 256, 256), (129, 1024, 256)])
def test_gemm_bias_relu(capi, path, M, N, K):
    g = _gen(M + N + K)
    A = torch.randn(M, K, generator=g).cuda()
    W = torch.randn(N, K, generator=g) * 0.1
    bias = torch.randn(N, generator=g).cuda()
    ref = (A.double() @ W.cuda().double().t() + bias.double()).relu()
    out = capi.test_gemm(path, A, W.numpy(), bias=bias, relu=True)
    assert _rel(out, ref) < REL[path]


@pytest.mark.parametrize("path", [TC, SIMT])
def test_gemm_residual_layernorm_epilogue(capi, path):
    g = _gen(3)
    M, N, K = 700, 256, 1024
    A = torch.randn(M, K, generator=g).cuda()
    W = torch.randn(N, K, generator=g) * 0.05
    bias = torch.randn(N, generator=g).cuda()
    res = torch.randn(M, N, generator=g).cuda()
    gam = (1 + 0.1 * torch.randn(N, generator=g)).cuda()
    bet = (0.1 * torch.randn(N, generator=g)).cuda()
    ref = F.layer_norm(A.double() @ W.cuda().double().t() + bias.double() + res.double(), (N,), gam.double(), bet.double(), 1e-5)
    out = capi.test_gemm(path, A, W.numpy(), bias=bias, residual=res, ln=(gam, bet))
    assert _rel(out, ref) < REL[path]


@pytest.mark.parametrize("M,N,mean", [(512, 768, 0.0), (1024, 1024, 3.0), (300, 256, -1.5), (4100, 3072, 0.5), (9000, 1024, 0.0)])
def test_gemm_deferred_layernorm_on_a(capi, M, N, mean):
    """GemmParams::a_ln_cs: A holds pre-LayerNorm rows, the GEMM consumes LN(A) without materialising it (weights carry
    gamma, two spare warps compute the row statistics from the staged tile, the epilogue finishes the algebra).
    Rows with a mean of several sigma stress the  x W'^T - mean colsum(W')  cancellation."""
    g = _gen(M + N)
    K = 256
    A = (torch.randn(M, K, generator=g) * (0.5 + torch.rand(M, 1, generator=g) * 4) + mean).cuda()
    W = torch.randn(N, K, generator=g) * 0.08
    bias = torch.randn(N, generator=g).cuda()
    gam = (1 + 0.2 * torch.randn(K, generator=g)).cuda()
    bet = (0.2 * torch.randn(K, generator=g)).cuda()
    ref = (F.layer_norm(A.double(), (K,), gam.double(), bet.double(), 1e-5) @ W.cuda().double().t() + bias.double()).relu()
    out = capi.test_gemm(TC, A, W.numpy(), bias=bias, relu=True, ln=(gam, bet), a_ln=True)
    assert _rel(out, ref) < 4e-6


@pytest.mark.parametrize("M,K", [(512, 1024), (1000, 256), (4224, 256)])
def test_gemm_emits_partial_row_statistics(capi, M, K):
    """GemmParams::ln_part_out: a GEMM whose 256-wide output rows will be layer-normalised later leaves, per row and
    16-column chunk, the chunk's (mean, M2) - what the deferred-LayerNorm consumers merge into (mean, rstd)."""
    g = _gen(M + K + 1)
    A = torch.randn(M, K, generator=g).cuda()
    W = torch.randn(256, K, generator=g) * 0.1
    bias = (torch.randn(256, generator=g) * 2).cuda()
    part = torch.zeros(M, 16, 2, device="cuda")
    out = capi.test_gemm(TC, A, W.numpy(), bias=bias, part_out=part)
    chunks = out.double().view(M, 16, 16)
    mean = chunks.mean(-1)
    m2 = ((chunks - mean[..., None]) ** 2).sum(-1)
    assert (part[..., 0].double() - mean).abs().max().item() < 1e-5
    assert ((part[..., 1].double() - m2).abs() / m2.clamp_min(1e-3)).max().item() < 1e-4


@pytest.mark.parametrize("M,K", [(512, 256), (1024, 1024), (512, 1024), (200, 256)])
def test_gemm_deferred_layernorm_residual(capi, M, K):
    """GemmParams::res_ln_part: the residual operand is a deferred LayerNorm of stored pre-norm rows, normalised on the
    fly from the partial row statistics ((512, 1024) is the encoder's FFN2: split-K over a cluster of 4)."""
    g = _gen(M + K)
    N = 256
    A = torch.randn(M, K, generator=g).cuda()
    W = torch.randn(N, K, generator=g) * 0.05
    bias = torch.randn(N, generator=g).cuda()
    res = (torch.randn(M, N, generator=g) * 2 + 0.7).cuda()
    gam = (1 + 0.2 * torch.randn(N, generator=g)).cuda()
    bet = (0.2 * torch.randn(N, generator=g)).cuda()
    ref = A.double() @ W.cuda().double().t() + bias.double() + F.layer_norm(res.double(), (N,), gam.double(), bet.double(), 1e-5)
    out = capi.test_gemm(TC, A, W.numpy(), bias=bias, residual=res, ln=(gam, bet), res_ln=True)
    assert _rel(out, ref) < 2.5e-6


@pytest.mark.parametrize("path", [TC, SIMT])
def test_gemm_periodic_add_matrix(capi, path):
    """The constant (pos W^T + b) matrices are added with a 512-row period (one period per image pair)."""
    g = _gen(4)
    M, N, K = 1024, 768, 256
    A = torch.randn(M, K, generator=g).cuda()
    W = torch.randn(N, K, generator=g) * 0.05
    add = torch.randn(512, N, generator=g).cuda()
    ref = A.double() @ W.cuda().double().t() + add.double().repeat(2, 1)
    out = capi.test_gemm(path, A, W.numpy(), addmat=add, add_period=512)
    assert _rel(out, ref) < REL[path]


@pytest.mark.parametrize("path", [TC, SIMT])
def test_gemm_wide_dynamic_range(capi, path):
    """Operands spanning 1e-4 .. 3e2 (post-ReLU features are like that): the fp16 split must not lose the small ones."""
    g = _gen(5)
    M, N, K = 256, 128, 512
    A = (torch.randn(M, K, generator=g) * torch.exp(torch.randn(M, K, generator=g) * 3)).clamp(-3e2, 3e2).cuda() * 0.5
    W = torch.randn(N, K, generator=g) * torch.exp(torch.randn(N, K, generator=g) * 2) * 1e-2
    ref = A.double() @ W.cuda().double().t()
    assert ref.abs().max() < 6.5e4        # full-precision range of split16 (hi alone saturates at 65504)
    out = capi.test_gemm(path, A, W.numpy())
    assert _rel(out, ref) < REL[path]


@pytest.mark.parametrize("path", [TC, SIMT])
def test_split16_storage_saturates_instead_of_overflowing(capi, path):
    """Activations are stored as fp16 hi + fp16 lo: values beyond +-131008 clamp, they never become inf / NaN."""
    A = torch.full((128, 64), 4000.0).cuda()
    W = torch.full((64, 64), 1.0)
    W[1] = -1.0
    out = capi.test_gemm(path, A, W.numpy())           # exact result 256000
    assert torch.isfinite(out).all()
    assert (out[:, 0] == 131008.0).all() and (out[:, 1] == -131008.0).all()


@pytest.mark.parametrize("path", [TC, SIMT])
@pytest.mark.parametrize("n,H,C,Co,k,s,pd", [(2, 16, 64, 64, 3, 1, 1), (2, 32, 128, 128, 3, 2, 1), (2, 16, 256, 256, 3, 2, 1),
                                            (2, 32, 256, 512, 1, 2, 0), (4, 64, 64, 256, 1, 1, 0)])
def test_implicit_gemm_convolution(capi, path, n, H, C, Co, k, s, pd):
    g = _gen(C + Co + k)
    x = torch.randn(n, C, H, H, generator=g)
    w = torch.randn(Co, C, k, k, generator=g) * 0.05
    bias = torch.randn(Co, generator=g).cuda()
    ref = F.conv2d(x.cuda().double(), w.cuda().double(), bias.double(), stride=s, padding=pd).permute(0, 2, 3, 1).reshape(-1, Co)
    OH = (H + 2 * pd - k) // s + 1
    xn = x.permute(0, 2, 3, 1).contiguous().cuda()                       # NHWC activations
    wk = w.permute(0, 2, 3, 1).reshape(Co, -1).contiguous()              # [Cout][kh][kw][Cin]
    out = capi.test_gemm(path, xn, wk.numpy(), bias=bias, a_mode=1, M=n * OH * OH,
                         conv=dict(H=H, W=H, C=C, OH=OH, OW=OH, KH=k, KW=k, stride=s, pad=pd))
    assert _rel(out, ref) < REL[path]


@pytest.mark.parametrize("path", [TC, SIMT])
def test_stem_convolution_on_side_by_side_canvas(capi, path):
    """7x7/2 conv reading the (B,3,256,512) NCHW canvas; the halves must not bleed into each other (backbone.py:81-82)."""
    g = _gen(6)
    img = torch.randn(1, 3, 256, 512, generator=g)
    w = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    bias = torch.randn(64, generator=g).cuda()
    halves = torch.cat([img[..., :256], img[..., 256:]], 0)
    ref = F.conv2d(halves.cuda().double(), w.cuda().double(), bias.double(), stride=2, padding=3).relu().permute(0, 2, 3, 1).reshape(-1, 64)
    wk = w.permute(0, 2, 3, 1).reshape(64, -1).contiguous()
    out = capi.test_gemm(path, img.cuda(), wk.numpy(), bias=bias, relu=True, a_mode=2, M=2 * 128 * 128,
                         conv=dict(H=256, W=256, C=3, OH=128, OW=128, KH=7, KW=7, stride=2, pad=3))
    assert _rel(out, ref) < REL[path]


# ---- attention, the fused feed-forward block and the row kernels, in the configurations the model launches ---------
# Inputs are split16 fixed points (_fix16), so every path stages the same hi / lo planes and the fp64 reference sees the
# values the kernels see.  Memory a launch must not read holds NaN (fp32 NaN stays NaN through the split, and the
# attention hook leaves the other slots' operand images 0xFF): a read of the wrong pair, slot, row or column makes the
# output non-finite.  Output rows a launch does not own hold SENTINEL (exact in split16) and must come back bitwise.
SENTINEL = 1000.5
NAN = float("nan")
# Relative error bounds, Frobenius norm over the output / worst single row.  Largest measured on an H100 SXM (80 GB
# HBM3, 700 W): attention 1.4e-6 / 3.3e-6, fused feed-forward 3.0e-7 / 4.3e-7, LayerNorms 1.6e-6 / 4.9e-6 (rows with
# a mean of 50 sigma: the fp32 row sum of 256 such values rounds at ~2^-24 of 12800 sigma, and the mean's error shifts
# the whole normalised row).  query_encode: 1.4e-7 absolute.
ATTN_REL, ATTN_ROW = 5e-6, 1e-5
MLP_REL, MLP_ROW = 1e-6, 2e-6
LN_REL, LN_ROW = 3e-6, 1e-5
QENC_ABS = 3e-7


def _fix16(x):
    """x rounded to a split16 fixed point: hi = fp16(x), lo = fp16(x - hi), x = hi + lo, twice (at fp16 ties the
    split of hi + lo is not the split of x)."""
    for _ in range(2):
        hi = x.half().float()
        x = hi + (x - hi).half().float()
    return x


def _check(out, ref, rel, row_rel):
    """Relative error of the whole output (Frobenius) and of its worst row: one wrong row must not hide in the norm."""
    out, ref = out.double(), ref.double()
    assert torch.isfinite(out).all(), "non-finite output: the launch read memory it must not read"
    err = (out - ref).norm() / ref.norm()
    row = ((out - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-30)).max()
    assert err < rel and row < row_rel, (err.item(), row.item())


def _attn_ref(q, k, v):
    """q (P, n, 256), k / v (P, 512, 256) -> softmax(q k^T) v per head in fp64, (P, n, 256)."""
    P, n = q.shape[:2]
    qh = q.double().reshape(P, n, 8, 32).transpose(1, 2)
    kh = k.double().reshape(P, 512, 8, 32).transpose(1, 2)
    vh = v.double().reshape(P, 512, 8, 32).transpose(1, 2)
    return (torch.softmax(qh @ kh.transpose(-1, -2), -1) @ vh).transpose(1, 2).reshape(P, n, 256)


def _tc_key_split(tiles):
    """attention_tc.cu's launch rule: split the keys over a cluster pair while the doubled grid fits the 132 SMs."""
    return 2 if 2 * tiles * 8 <= 132 else 1


ATTN_SHAPES = list(dict.fromkeys([(512, 1, 1.0), (1024, 2, 2.0), (100, 3, 1.0), (257, 1, 3.0), (1, 4, 1.0), (33, 2, 6.0)] +
                                 [(nq, npairs, 1.0) for nq in (1, 31, 32, 33, 127, 128, 129, 512, 1024) for npairs in (1, 3, 16)]))


@pytest.mark.parametrize("operands", ["rowmajor", "images"])
@pytest.mark.parametrize("path", [TC, SIMT])
@pytest.mark.parametrize("nq,npairs,gain", ATTN_SHAPES)
def test_attention(capi, path, operands, nq, npairs, gain):
    """Both kernels on both operand layouts; the tensor-core kernel also with each key split forced.  Image operands
    are staged byte for byte like the row-major ones (attention_tc.cu static_assert), so the output is the same."""
    g = _gen(nq + npairs)
    q = _fix16(torch.randn(npairs * nq, 256, generator=g) * gain).cuda()
    k = _fix16(torch.randn(npairs * 512, 256, generator=g)).cuda()
    v = _fix16(torch.randn(npairs * 512, 256, generator=g)).cuda()
    ref = _attn_ref(q.view(npairs, nq, 256), k.view(npairs, 512, 256), v.view(npairs, 512, 256)).reshape(-1, 256)
    run = lambda p, ops, **kw: capi.test_attention(p, q, k, v, nq, npairs, operands=ops, **kw)
    outs = {0: run(path, operands)}
    if path == TC:
        for ks in (1, 2):
            outs[ks] = run(TC, operands, key_split=ks)
        # the launch rule: fewer than 32 rows per pair go to the SIMT kernel, the others to the key split it picks
        rule = run(SIMT, operands) if nq < 32 else outs[_tc_key_split(-(-nq // 128) * npairs)]
        assert torch.equal(outs[0], rule)
    for out in outs.values():
        _check(out, ref, ATTN_REL, ATTN_ROW)
    if operands == "images":
        for ks, out in outs.items():
            assert torch.equal(out, run(path, "rowmajor", key_split=ks))


def _context(g, ctx_pairs, slots, pairs, slot):
    """K and V of a context: (ctx_pairs*512, slots*256), random in slot `slot` of `pairs`, NaN everywhere else."""
    k = torch.full((ctx_pairs * 512, slots * 256), NAN, device="cuda")
    v = torch.full_like(k, NAN)
    for t in (k, v):
        for p in pairs:
            t[p * 512:(p + 1) * 512, slot * 256:(slot + 1) * 256] = _fix16(torch.randn(512, 256, generator=g, device="cuda"))
    return k, v


def _kv(k, v, pair, slot):
    return k[pair * 512:(pair + 1) * 512, slot * 256:(slot + 1) * 256], v[pair * 512:(pair + 1) * 512, slot * 256:(slot + 1) * 256]


@pytest.mark.parametrize("operands", ["rowmajor", "images"])
@pytest.mark.parametrize("path", [TC, SIMT])
@pytest.mark.parametrize("slot,ldq,q_col0", [(0, 1536, 0), (5, 512, 0), (5, 1536, 3 * 256)])
@pytest.mark.parametrize("nq", [1, 100, 300])
def test_attention_context_layout(capi, path, operands, slot, ldq, q_col0, nq):
    """The decoder's launches: K / V of 6 layers per pair of a 40-pair context, a chunk at pair0 = 32, q strided
    (ldq 1536: decoder layer 0's query-position columns; 512: the encoder's [q | k] rows)."""
    g = torch.Generator(device="cuda").manual_seed(slot * 7 + ldq + q_col0 + nq)
    ctx_pairs, slots, pair0, npairs = 40, 6, 32, 8
    k, v = _context(g, ctx_pairs, slots, range(pair0, pair0 + npairs), slot)
    rows = npairs * nq
    q = torch.full((rows + 5, ldq), NAN, device="cuda")
    q[:rows, q_col0:q_col0 + 256] = _fix16(torch.randn(rows, 256, generator=g, device="cuda"))
    out = torch.full((rows + 5, 256), SENTINEL, device="cuda")
    out = capi.test_attention(path, q, k, v, nq, npairs, operands=operands, pair0=pair0, slot=slot, q_col0=q_col0, out=out)
    kk, vv = zip(*[_kv(k, v, pair0 + p, slot) for p in range(npairs)])
    ref = _attn_ref(q[:rows, q_col0:q_col0 + 256].reshape(npairs, nq, 256), torch.stack(kk), torch.stack(vv)).reshape(rows, 256)
    _check(out[:rows], ref, ATTN_REL, ATTN_ROW)
    assert (out[rows:] == SENTINEL).all()


def _ragged_tiles(counts, min_tc):
    """decode_ragged_impl's tile rule: pairs with >= min_tc rows (32 in the model) get 128-row tensor-core tiles, the
    others 64-row SIMT tiles; rows are packed pair after pair.  -> (tc tiles, SIMT tiles, first row of each pair)"""
    tc, simt, first, row = [], [], [], 0
    for p, n in enumerate(counts):
        step = 128 if n >= min_tc else 64
        for i in range(0, n, step):
            (tc if n >= min_tc else simt).append((p, row + i, min(step, n - i)))
        first.append(row)
        row += n
    return tc, simt, first


@pytest.mark.parametrize("operands", ["rowmajor", "images"])
@pytest.mark.parametrize("key_split", [0, 1, 2])
@pytest.mark.parametrize("counts,min_tc", [((0, 1, 31, 32, 33, 127, 128, 129, 300), 32),    # 9 tensor-core tiles: rule KS = 1
                                           ((0, 40, 0, 5), 32),                              # 1 tensor-core tile: rule KS = 2
                                           ((1, 31, 0, 200), 1)])                            # tensor-core tiles of 1 and 31 rows
def test_attention_tile_table(capi, operands, key_split, counts, min_tc):
    """A ragged decode chunk: one tensor-core launch and one SIMT launch over tile tables write one output.  Each pair's
    rows must be bitwise those of a uniform launch of that pair with the same kernel and key split (the rows of a tile
    are independent: no arithmetic mixes them), and within the fp64 bound."""
    g = torch.Generator(device="cuda").manual_seed(sum(counts) + min_tc)
    slots, slot, pair0, q_col0 = 6, 2, 3, 2 * 256
    ctx_pairs = pair0 + len(counts) + 1
    k, v = _context(g, ctx_pairs, slots, range(pair0, pair0 + len(counts)), slot)
    tc, simt, first = _ragged_tiles(counts, min_tc)
    R = sum(counts)
    q = torch.full((R + 3, 1536), NAN, device="cuda")
    q[:R, q_col0:q_col0 + 256] = _fix16(torch.randn(R, 256, generator=g, device="cuda"))
    out = torch.full((R + 3, 256), SENTINEL, device="cuda")
    kw = dict(operands=operands, pair0=pair0, slot=slot, q_col0=q_col0)
    ks = key_split or _tc_key_split(len(tc))
    if tc:
        out = capi.test_attention(TC, q, k, v, 0, 0, tiles=tc, key_split=key_split, out=out, **kw)
    if simt:
        out = capi.test_attention(SIMT, q, k, v, 0, 0, tiles=simt, out=out, **kw)
    assert (out[R:] == SENTINEL).all()
    for p, n in enumerate(counts):
        if n == 0:
            continue
        rows = slice(first[p], first[p] + n)
        kk, vv = _kv(k, v, pair0 + p, slot)
        _check(out[rows], _attn_ref(q[None, rows, q_col0:q_col0 + 256], kk[None], vv[None])[0], ATTN_REL, ATTN_ROW)
        path = TC if n >= min_tc else SIMT
        uniform = capi.test_attention(path, q[rows].contiguous(), k, v, n, 1, key_split=ks if path == TC else 0,
                                      **dict(kw, pair0=pair0 + p))
        assert torch.equal(out[rows], uniform), p


def test_attention_rejects_bad_descriptors(capi):
    """Every argument is checked on the host: the call fails with a message and launches nothing (out is untouched)."""
    q = torch.zeros(64, 256, device="cuda")
    k = torch.zeros(2 * 512, 256, device="cuda")
    out = torch.full((64, 256), SENTINEL, device="cuda")
    bad = [
        (dict(path=TC, nq=32, npairs=2, pair0=1), "pairs 1 .. 2 of 2"),
        (dict(path=TC, nq=32, npairs=2, q=torch.zeros(64, 260, device="cuda")), "ldq 260"),
        (dict(path=SIMT, nq=32, npairs=2, q=torch.zeros(64, 512, device="cuda"), q_col0=264), "do not fit ldq 512"),
        (dict(path=TC, nq=64, npairs=2), "64 rows, q has 64"),
        (dict(path=TC, tiles=[(0, 0, 64), (1, 0, 129)]), "tile 1 has 129 rows"),
        (dict(path=SIMT, tiles=[(0, 0, 65)]), "tile 0 has 65 rows"),
        (dict(path=TC, tiles=[(0, 40, 30)]), "rows 40 .. 69 of tile 0 fall outside q"),
        (dict(path=SIMT, tiles=[(1, 0, 8)], pair0=1), "tile 0 reads pair 1 \\+ 1 of 2"),
        (dict(path=SIMT, nq=32, npairs=2, key_split=2), "key split 2"),
        (dict(path=TC, nq=32, npairs=2, slot=1), "slot 1 of 1"),
    ]
    for kw, msg in bad:
        kw = dict(kw)
        path, qq = kw.pop("path"), kw.pop("q", q)
        nq, npairs = kw.pop("nq", 0), kw.pop("npairs", 0)
        out = torch.full((qq.shape[0], 256), SENTINEL, device="cuda")
        with pytest.raises(RuntimeError, match=msg):
            capi.test_attention(path, qq, k, k, nq, npairs, out=out, **kw)
        assert (out == SENTINEL).all()


def _ffn_weights(g, wide=False):
    """linear1 / linear2 / LayerNorm parameters at the scale of the model's (xavier-uniform weights, small biases).
    wide: linear1's rows scaled so that the hidden activations span 1e-3 .. 1e2."""
    xav = lambda n, k: (torch.rand(n, k, generator=g) * 2 - 1) * (6 / (n + k)) ** 0.5
    w1, b1 = xav(1024, 256), torch.randn(1024, generator=g) * 0.02
    if wide:
        f = 10 ** (torch.rand(1024, 1, generator=g) * 5 - 2.5)
        w1, b1 = w1 * f, b1 * f[:, 0]
    w2, b2 = xav(256, 1024), torch.randn(256, generator=g) * 0.02
    ln = [(1 + 0.1 * torch.randn(256, generator=g), 0.1 * torch.randn(256, generator=g)) for _ in range(2)]
    return [_fix16(t) for t in (w1, b1, w2, b2, *ln[0], *ln[1])]


def _ffn_ref(x, w1, b1, w2, b2, g, be, g2=None, be2=None):
    x = x.double()
    h = (x @ w1.double().t() + b1.double()).relu()
    y = F.layer_norm(x + h @ w2.double().t() + b2.double(), (256,), g.double(), be.double(), 1e-5)
    return y if g2 is None else F.layer_norm(y, (256,), g2.double(), be2.double(), 1e-5)


@pytest.mark.parametrize("split", [4, 8])
@pytest.mark.parametrize("M", [1, 8, 63, 64, 65, 100, 512, 1000, 1024, 1536, 2047, 4160])
def test_fused_feed_forward(capi, M, split):
    """mlp_tc.cu with each hidden split forced: M = 1 at S = 8 leaves 7 CTAs of the cluster without a valid row, 4160
    rows are 65 row tiles (more than fit as clusters of 8).  Out of place and in place (the decoder's form), with and
    without the second LayerNorm (the last decoder layer's decoder.norm)."""
    g = _gen(M + split)
    w1, b1, w2, b2, g1, be1, g2, be2 = (t.cuda() for t in _ffn_weights(g))
    x = torch.full((M + 3, 256), NAN)
    x[:M] = _fix16(torch.randn(M, 256, generator=g))
    x = x.cuda()
    for ln2 in ((), (g2, be2)):
        ref = _ffn_ref(x[:M], w1, b1, w2, b2, g1, be1, *ln2)
        run = lambda **kw: capi.test_mlp(x, M, w1.cpu().numpy(), b1, w2.cpu().numpy(), b2, g1, be1, *ln2, split=split, **kw)
        out = run(out=torch.full_like(x, SENTINEL))
        _check(out[:M], ref, MLP_REL, MLP_ROW)
        assert (out[M:] == SENTINEL).all()
        assert torch.equal(out, run(out=torch.full_like(x, SENTINEL)))
        in_place = run(in_place=True)
        assert torch.equal(in_place[:M], out[:M]) and in_place[M:].isnan().all()


@pytest.mark.parametrize("M,rule", [(1, 8), (1024, None), (4160, 4)])
def test_fused_feed_forward_launch_rule(capi, M, rule):
    """Without a forced split the launch runs clusters of 8 while every row tile fits one wave of them (at most 16 on
    132 SMs: a single tile always does, 65 never), else clusters of 4; its output is that split's, bit for bit."""
    g = _gen(M + 3)
    w1, b1, w2, b2, g1, be1, _, _ = _ffn_weights(g)
    b1, b2, g1, be1 = (t.cuda() for t in (b1, b2, g1, be1))
    x = _fix16(torch.randn(M, 256, generator=g)).cuda()
    run = lambda split: capi.test_mlp(x, M, w1.numpy(), b1, w2.numpy(), b2, g1, be1, split=split)
    outs = {s: run(s) for s in (0, 4, 8)}
    if rule is None:
        assert torch.equal(outs[0], outs[4]) or torch.equal(outs[0], outs[8])
    else:
        assert torch.equal(outs[0], outs[rule])


@pytest.mark.parametrize("split", [4, 8])
def test_fused_feed_forward_wide_hidden_range(capi, split):
    """Hidden activations spanning 1e-3 .. 1e2: h is re-split to fp16 hi / lo in shared memory, and the lo plane of
    the large ones carries most of the output's precision."""
    g = _gen(11)
    M = 700
    w1, b1, w2, b2, g1, be1, _, _ = _ffn_weights(g, wide=True)
    b1, b2, g1, be1 = (t.cuda() for t in (b1, b2, g1, be1))
    x = _fix16(torch.randn(M, 256, generator=g)).cuda()
    h = (x.double() @ w1.cuda().double().t() + b1.double()).relu()
    pos = h[h > 0]
    assert pos.min() < 1e-3 and pos.max() > 1e2
    out = capi.test_mlp(x, M, w1.numpy(), b1, w2.numpy(), b2, g1, be1, split=split)
    _check(out, _ffn_ref(x, w1.cuda(), b1, w2.cuda(), b2, g1, be1), MLP_REL, MLP_ROW)


def _ln_rows(rows, g):
    """Rows scaled from 1e-3 to 1e3 with means up to 50 sigma, and one constant row (when there are 8 or more)."""
    scale = 10 ** torch.linspace(-3, 3, rows).reshape(-1, 1)
    mean = torch.linspace(-50, 50, rows).reshape(-1, 1) * scale
    x = torch.randn(rows, 256, generator=g) * scale + mean
    if rows >= 8:
        x[rows // 2] = 3.25
    return _fix16(x)


@pytest.mark.parametrize("op", ["layernorm", "layernorm_f32", "layernorm_twice"])
@pytest.mark.parametrize("rows", [1, 7, 8, 9, 1000])
def test_layernorm_kernels(capi, op, rows):
    g = _gen(rows)
    x = _ln_rows(rows, g).cuda()
    g1, b1, g2, b2 = (_fix16(t).cuda() for t in (1 + 0.2 * torch.randn(256, generator=g), 0.2 * torch.randn(256, generator=g),
                                                  1 + 0.2 * torch.randn(256, generator=g), 0.2 * torch.randn(256, generator=g)))
    ln = lambda t, gg, bb: F.layer_norm(t, (256,), gg.double(), bb.double(), 1e-5)
    ref = ln(x.double(), g1, b1)
    if op == "layernorm_twice":
        ref = ln(ref, g2, b2)
        out = capi.test_rowwise(op, x, g1, b1, g2, b2)
    else:
        out = capi.test_rowwise(op, x, g1, b1)
    _check(out, ref, LN_REL, LN_ROW)
    if rows >= 8 and op != "layernorm_twice":        # a constant row normalises to exactly beta
        assert torch.equal(out[rows // 2], b1)


def test_query_encode(capi):
    """lin_sine encoding of 4097 points of [0, 1] (both ends included): channel 2(k-1)+a = sin(fp32(k pi) p_a), 128 +
    2(k-1)+a = cos(...), against fp64 sin / cos of the same fp32 angle (the product rounded to nearest)."""
    n = 4097
    p = torch.linspace(0, 1, n, dtype=torch.float64).float()
    pts = torch.stack([p, p.flip(0)], 1)
    out = capi.test_rowwise("query_encode", pts.cuda()).cpu().double()
    kpi = (torch.arange(1, 65, dtype=torch.float64) * np.pi).float()
    angle = (kpi[None, :, None] * pts[:, None, :]).double().reshape(n, 128)       # fp32 product, rounded to nearest
    ref = torch.cat([angle.sin(), angle.cos()], 1)
    assert (out - ref).abs().max().item() < QENC_ABS
