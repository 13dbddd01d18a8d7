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


@pytest.mark.parametrize("path", [TC, SIMT])
@pytest.mark.parametrize("nq,npairs,gain", [(512, 1, 1.0), (1024, 2, 2.0), (100, 3, 1.0), (257, 1, 3.0), (1, 4, 1.0), (33, 2, 6.0)])
def test_attention(capi, path, nq, npairs, gain):
    g = _gen(nq + npairs)
    q = (torch.randn(npairs * nq, 256, generator=g) * gain).cuda()
    k = torch.randn(npairs * 512, 256, generator=g).cuda()
    v = torch.randn(npairs * 512, 256, generator=g).cuda()
    qh = q.double().view(npairs, nq, 8, 32).transpose(1, 2)
    kh = k.double().view(npairs, 512, 8, 32).transpose(1, 2)
    vh = v.double().view(npairs, 512, 8, 32).transpose(1, 2)
    ref = (torch.softmax(qh @ kh.transpose(-1, -2), -1) @ vh).transpose(1, 2).reshape(npairs * nq, 256)
    out = capi.test_attention(path, q, k, v, nq, npairs)
    assert _rel(out, ref) < 5e-6
