"""GPU: the head-averaged attention maps (csrc/attention_weights.cu) against fp64, in the configurations the model
launches them.  Kernel level: both maps kernels through cotr_test_attention's maps output, with the operand layouts of
every section, every tile edge, five logit classes, and the rows and memory a launch must not touch.  Model level:
decodes that span several chunks, so that later chunks launch the maps kernels at pair0 > 0."""
import pytest
import torch

from oracle import attention_oracle, fixtures

pytestmark = pytest.mark.gpu

TC, SIMT = 0, 1
OPERANDS = {TC: "images", SIMT: "rowmajor"}        # the pairing the model runs: tensor-core maps read operand images
# Inputs are split16 fixed points (_fix16), so both kernels stage exactly the values the fp64 reference sees.  q columns,
# other slots, other context pairs and q rows past npairs * nq that a launch must not read hold NaN (the hook leaves the
# other slots' operand images 0xFF, fp16 NaN): a read of any of them makes a map non-finite.  Map rows a launch does not
# own hold SENTINEL and must come back bitwise.
SENTINEL = 1000.5
NAN = float("nan")

# Bounds per logit class on (Frobenius error of the maps / their norm, worst row's error / its norm, largest error of
# an entry).  The products q_h . k_h are split16 (the tensor-core kernel drops Q_lo K_lo) and summed in fp32, so a logit
# errs in proportion to |q| |k|, and an error d in a logit moves p by about p d.  For the class whose logits reach 1e4
# the bounds are therefore proportional to the row's largest |logit|: its errors are divided by that before they are
# compared.  Largest measured on an H100 SXM (80 GB HBM3, 700 W power limit) over both kernels and every case of the
# class, in the same order:
#   n1 1.3e-7 2.7e-7 1.6e-8, n9 6.9e-7 1.5e-6 1.8e-7 (fp32 SIMT, 16 pairs x 1024 rows), n900 1.5e-6 5.7e-6 1.1e-6,
#   ties 3.0e-8 6.0e-8 2.0e-8, big 9.7e-8 2.3e-7 1.7e-8 per unit of the largest |logit| (about 1e-3 relative at 1e4).
# n9 stays within the bounds the maps kernels were first checked to (1e-6 relative, 5e-7 absolute).
BOUNDS = {
    "n1": (3e-7, 6e-7, 4e-8),           # logits ~N(0, 1)
    "n9": (1e-6, 3e-6, 4e-7),           # logits ~N(0, 9)
    "n900": (3e-6, 1.2e-5, 2.5e-6),     # logits ~N(0, 900)
    "ties": (6e-8, 1.2e-7, 4e-8),       # 2 or 3 keys tied exactly at the maximum, p = 1/2, 1/3
    "big": (2e-7, 5e-7, 4e-8),          # largest logit ~1e4 (encoder layer 0 of the qk-gain fixture reaches 7.9e3)
}
# |sum of a map row - 1|: every head's P is normalised by its own fp32 sum, whatever the error of its logits
# (measured 1.9e-7)
SUM_ABS = 4e-7
# Maps of a model call against the fp64 oracle, per layer (as in test_attention_weights_gpu.py): the maps carry the
# upstream drift of the whole network.  Maps of one pair decoded within a batch against the same pair decoded alone:
# GEMM plans depend on M, so they are not bitwise (test_batch_items_and_queries_are_independent).
MAP_REL, MAP_ABS = 5e-4, 1e-3
PAIR_ABS = 2e-4
CHUNK_ROWS = 32768          # model.cu kDecodeChunkRows


@pytest.fixture(scope="module")
def capi(built_lib):
    from cotr_b200 import capi
    capi.lib()
    return capi


def _fix16(x):
    """x rounded to a split16 fixed point: hi = fp16(x), lo = fp16(x - hi), x = hi + lo, twice (at fp16 ties the
    split of hi + lo is not the split of x)."""
    for _ in range(2):
        hi = x.half().float()
        x = hi + (x - hi).half().float()
    return x


def _ref(q, k):
    """q (P, n, 256), k (P, 512, 256) -> (mean_h softmax(q_h k_h^T) in fp64 (P, n, 512), largest |logit| of each row (P, n))."""
    P, n = q.shape[:2]
    s = q.double().reshape(P, n, 8, 32).transpose(1, 2) @ k.double().reshape(P, 512, 8, 32).permute(0, 2, 3, 1)
    return torch.softmax(s, -1).mean(1), s.abs().amax(dim=(1, 3))


def _check(out, ref, kind, scale=None):
    """Frobenius error of the maps and the worst row's error, relative to the reference's norms (in units of the row's
    largest |logit| for the 'big' class); entries >= 0 and rows summing to 1."""
    out, ref = out.double(), ref.double()
    assert torch.isfinite(out).all(), "non-finite map: the launch read memory it must not read"
    assert (out >= 0).all()
    e = out - ref
    if kind == "big":
        e = e / scale.double().unsqueeze(-1)
    frob = (e.norm() / ref.norm()).item()
    row = (e.norm(dim=-1) / ref.norm(dim=-1)).max().item()
    err = e.abs().max().item()
    sums = (out.sum(-1) - 1).abs().max().item()
    assert all(x < b for x, b in zip((frob, row, err), BOUNDS[kind])) and sums < SUM_ABS, (kind, frob, row, err, sums)


GAINS = {"n1": 1.0, "n9": 3.0, "n900": 30.0}
TIES = [(7, 300), (64, 200, 511)]        # in different 64-key chunks and at different lanes of them


def _operands(g, kind, npairs, nq):
    """q (npairs, nq, 256), k (npairs, 512, 256), split16 fixed points, whose logits q_h . k_h are of class `kind`."""
    k = torch.randn(npairs, 512, 8, 32, generator=g, device="cuda")
    q = torch.randn(npairs, nq, 8, 32, generator=g, device="cuda")
    if kind in GAINS:
        q = q * GAINS[kind] * 32 ** -0.5
    elif kind == "big":
        # every key of a head shares a large component: logits = 100 (100 + 0.01 z) + 0.5 sum_{d>0} z_d z'_d
        # ~ 1e4 + N(0, ~9), so the softmax is as spread as at N(0, 9) while |q| |k| ~ 1e4
        k[..., 0] = 100 + 0.01 * k[..., 0]
        q = 0.5 * q
        q[..., 0] = 100
    elif kind == "ties":
        # pair p: the keys of TIES[p % 2] are identical in every head, three times as long as the others, and q
        # points along them with logit 40 while the other keys' logits are ~N(0, 40^2 / (9 * 32)): the tied keys
        # share the row's maximum, p = 1/2 or 1/3 each up to e^-30
        for p in range(npairs):
            tie = TIES[p % 2]
            k[p, list(tie)] = 3 * k[p, tie[0]]
            kt = _fix16(k[p, tie[0]])                                   # (8, 32)
            q[p] = 40 * kt / (kt * kt).sum(-1, keepdim=True) + 0.01 * q[p]
    else:
        raise ValueError(kind)
    return _fix16(q.reshape(npairs, nq, 256)), _fix16(k.reshape(npairs, 512, 256))


def _layout(g, q, k, *, ctx_pairs, slots, slot, pair0, ldq, q_col0):
    """Embed the launch's q / k into the buffers of a launch as the model makes it: q (rows + 5, ldq) with the launch's
    columns at q_col0, k / v (ctx_pairs * 512, slots * 256) of a context with the launch's pairs at pair0 .. in slot
    `slot`; NaN everywhere else."""
    npairs, nq = q.shape[:2]
    rows = npairs * nq
    qb = torch.full((rows + 5, ldq), NAN, device="cuda")
    qb[:rows, q_col0:q_col0 + 256] = q.reshape(rows, 256)
    kb = torch.full((ctx_pairs * 512, slots * 256), NAN, device="cuda")
    vb = torch.full_like(kb, NAN)
    keys, cols = slice(pair0 * 512, (pair0 + npairs) * 512), slice(slot * 256, (slot + 1) * 256)
    kb[keys, cols] = k.reshape(-1, 256)
    vb[keys, cols] = _fix16(torch.randn(npairs * 512, 256, generator=g, device="cuda"))
    return qb, kb, vb


def _maps(capi, path, qb, kb, vb, nq, npairs, lay, row0=3, extra=64):
    """One hook launch with maps into a SENTINEL buffer at row0 -> the launch's rows (npairs, nq, 512); the rows around
    them must come back bitwise.  The rows after the launch's span a whole tensor-core tile, so that a store of a last
    tile's padding rows lands in them."""
    rows = npairs * nq
    maps = torch.full((row0 + rows + extra, 512), SENTINEL, device="cuda")
    capi.test_attention(path, qb, kb, vb, nq, npairs, operands=OPERANDS[path], pair0=lay["pair0"], slot=lay["slot"],
                        q_col0=lay["q_col0"], maps=maps, maps_row0=row0)
    assert (maps[:row0] == SENTINEL).all() and (maps[row0 + rows:] == SENTINEL).all()
    return maps[row0:row0 + rows].view(npairs, nq, 512)


def _run_and_check(capi, path, kind, nq, npairs, lay, seed, pairs_alone=()):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k = _operands(g, kind, npairs, nq)
    qb, kb, vb = _layout(g, q, k, **{n: lay[n] for n in ("ctx_pairs", "slots", "slot", "pair0", "ldq", "q_col0")})
    out = _maps(capi, path, qb, kb, vb, nq, npairs, lay)
    ref, scale = _ref(q, k)
    _check(out, ref, kind, scale)
    if path == TC:      # a fixed-order head sum, no atomics
        assert torch.equal(out, _maps(capi, path, qb, kb, vb, nq, npairs, lay, row0=0))
    # pair independence: pair p's rows equal a one-pair launch at pair0 + p bitwise (a pair's rows keep their place in
    # its tiles, so no arithmetic differs); a launch that ignored pair0, or indexed q or the maps by the wrong pair,
    # cannot pass this
    nan_rows = qb[npairs * nq:]
    for p in pairs_alone:
        q1 = torch.cat([qb[p * nq:(p + 1) * nq], nan_rows]).contiguous()
        one = _maps(capi, path, q1, kb, vb, nq, 1, dict(lay, pair0=lay["pair0"] + p), row0=1)
        assert torch.equal(one[0], out[p]), p
    return out


# ---- the three sections' launches --------------------------------------------------------------------------------
def _section(name, path):
    """The operand layout of a section's attention launches (model.cu encode_tail / decode_chunk)."""
    if name == "encoder":
        # q: the [q | k] rows (ldq 512); keys: the k half of the same rows (SIMT, ldk 512) or images of one slot (TC)
        return dict(ctx_pairs=2, npairs=2, pair0=0, slots=2 if path == SIMT else 1, slot=1 if path == SIMT else 0,
                    ldq=512, q_col0=0)
    # the decoder: a chunk at pair0 = 32 of a 40-pair context of 6 layers; layer 0 reads its q from the qpos projection
    # of all 6 layers (ldq 1536), layers 1-5 from their own q projection (ldq 256)
    layer = int(name[len("decoder"):])
    return dict(ctx_pairs=40, npairs=8, pair0=32, slots=6, slot=layer, ldq=1536 if layer == 0 else 256, q_col0=0)


@pytest.mark.parametrize("path", [TC, SIMT], ids=["tc", "simt"])
@pytest.mark.parametrize("section,nq", [("encoder", 512), ("decoder0", 1), ("decoder0", 100), ("decoder1", 100),
                                        ("decoder5", 1), ("decoder5", 300)])
def test_section_layouts(capi, path, section, nq):
    lay = _section(section, path)
    npairs = lay["npairs"]
    _run_and_check(capi, path, "n9", nq, npairs, lay, seed=nq + lay["slot"] + 7 * path, pairs_alone=(0, npairs - 1))


# ---- every tile edge of both kernels: 64-row tensor-core CTAs, 32-row SIMT CTAs ----------------------------------------
# a context of npairs + 2 pairs, 2 slots; the launch reads slot 1 of pairs 1 .. npairs and q columns 256 .. 511
EDGE_LAYOUT = dict(slots=2, slot=1, pair0=1, ldq=512, q_col0=256)
ROW_COUNTS = list(dict.fromkeys([(nq, npairs) for nq in (1, 31, 32, 33, 63, 64, 65, 100, 127, 128, 129, 512, 1024)
                                 for npairs in (1, 3, 16)] + [(512, 2), (1, 300)]))


@pytest.mark.parametrize("path", [TC, SIMT], ids=["tc", "simt"])
@pytest.mark.parametrize("nq,npairs", ROW_COUNTS)
def test_row_counts(capi, path, nq, npairs):
    lay = dict(EDGE_LAYOUT, ctx_pairs=npairs + 2)
    _run_and_check(capi, path, "n9", nq, npairs, lay, seed=nq * 1000 + npairs,
                   pairs_alone=(0, npairs - 1) if 1 < npairs <= 16 else ())


@pytest.mark.parametrize("path", [TC, SIMT], ids=["tc", "simt"])
@pytest.mark.parametrize("kind", ["n1", "n9", "n900", "big", "ties"])
@pytest.mark.parametrize("nq", [33, 100])
def test_logit_scales(capi, path, kind, nq):
    lay = dict(EDGE_LAYOUT, ctx_pairs=5)
    out = _run_and_check(capi, path, kind, nq, 3, lay, seed=nq + len(kind), pairs_alone=(2,))
    if kind == "ties":
        for p in range(3):
            tie = list(TIES[p % 2])
            assert ((out[p][:, tie] - 1 / len(tie)).abs() < 1e-5).all(), p


def test_rejections(capi):
    """Every argument is checked on the host: the call fails with a message and launches nothing (out and maps are
    untouched)."""
    q = torch.zeros(64, 256, device="cuda")
    k = torch.zeros(2 * 512, 256, device="cuda")
    bad = [
        # the maps arguments
        (dict(path=TC, tiles=[(0, 0, 64)]), "maps of a tile-table launch"),
        (dict(path=SIMT, tiles=[(0, 0, 64)], operands="rowmajor"), "maps of a tile-table launch"),
        (dict(path=TC, nq=32, npairs=2, operands="rowmajor"), "tensor-core maps read the keys as operand images"),
        (dict(path=SIMT, nq=32, npairs=2, operands="images"), "fp32 SIMT maps read row-major keys"),
        (dict(path=TC, nq=32, npairs=2, maps_rows=63), "map rows 0 .. 63 do not fit the 63 rows"),
        (dict(path=SIMT, nq=32, npairs=2, operands="rowmajor", maps_rows=66, maps_row0=3), "map rows 3 .. 66 do not fit the 66 rows"),
        (dict(path=TC, nq=1, npairs=1, maps_row0=-1), "map rows -1 .. -1"),
        # the attention arguments, with maps requested
        (dict(path=TC, nq=32, npairs=2, pair0=1), "pairs 1 .. 2 of 2"),
        (dict(path=TC, nq=32, npairs=2, q=torch.zeros(64, 260, device="cuda")), "ldq 260"),
        (dict(path=SIMT, nq=32, npairs=2, operands="rowmajor", q=torch.zeros(64, 512, device="cuda"), q_col0=264), "do not fit ldq 512"),
        (dict(path=TC, nq=64, npairs=2), "64 rows, q has 64"),
        (dict(path=SIMT, nq=32, npairs=2, operands="rowmajor", key_split=2), "key split 2"),
        (dict(path=TC, nq=32, npairs=2, slot=1), "slot 1 of 1"),
    ]
    for kw, msg in bad:
        kw = dict(kw)
        path, qq = kw.pop("path"), kw.pop("q", q)
        nq, npairs = kw.pop("nq", 0), kw.pop("npairs", 0)
        kw.setdefault("operands", "images")
        maps = torch.full((kw.pop("maps_rows", 64), 512), SENTINEL, device="cuda")
        out = torch.full((qq.shape[0], 256), SENTINEL, device="cuda")
        with pytest.raises(RuntimeError, match=msg):
            capi.test_attention(path, qq, k, k, nq, npairs, out=out, maps=maps, **kw)
        assert (out == SENTINEL).all() and (maps == SENTINEL).all(), msg


# ---- model level: decodes over several chunks ----------------------------------------------------------------------
def _chunks(B, Q):
    """decode_impl's chunk rule -> (pair0, npairs, query rows per pair) of each chunk, in launch order: with
    Q <= CHUNK_ROWS, CHUNK_ROWS // Q pairs per chunk; otherwise each pair's queries in slices of CHUNK_ROWS."""
    if Q <= CHUNK_ROWS:
        per = CHUNK_ROWS // Q
        return [(b0, min(per, B - b0), Q) for b0 in range(0, B, per)]
    return [(b, 1, min(CHUNK_ROWS, Q - q0)) for b in range(B) for q0 in range(0, Q, CHUNK_ROWS)]


@pytest.fixture(scope="module")
def native(built_lib):
    from cotr_b200 import capi
    sd = fixtures.make_state_dict(0)
    nat = capi.NativeModel(sd, 0)
    contexts = []

    def context(path, img):
        ctx = capi.NativeContext(nat, img.shape[0])
        contexts.append(ctx)
        nat.set_gemm_path(path)
        nat.encode_context(img, ctx)
        return ctx

    yield sd, nat, context
    nat.set_gemm_path(TC)
    torch.cuda.synchronize()
    for ctx in contexts:
        ctx.close()
    nat.close()


def _inputs(seed, B, Q):
    img, queries = fixtures.make_inputs(seed, B, Q)
    return torch.from_numpy(img).cuda(), torch.from_numpy(queries).cuda()


@pytest.mark.parametrize("path", [TC, SIMT], ids=["tc", "simt"])
def test_two_chunk_decode_matches_oracle(native, path):
    """B = 3, Q = 12 000: chunk 0 decodes pairs 0-1, chunk 1 pair 2 at pair0 = 2, whose maps go at pair 2's rows."""
    sd, nat, context = native
    B, Q = 3, 12000
    assert [c[:2] for c in _chunks(B, Q)] == [(0, 2), (2, 1)]
    img, q = _inputs(31, B, Q)
    ctx = context(path, img)
    plain = nat.decode(ctx, q)
    enc = nat.encode_context_attention(img, ctx, 0b111111)
    pred, dec = nat.decode_attention(ctx, q, 0b111111)
    assert torch.equal(pred, plain)
    with torch.device("cuda"):              # the fp64 oracle on the GPU: it is the same arithmetic on either device
        _, ref = attention_oracle.forward({n: torch.from_numpy(v).cuda() for n, v in sd.items()}, img, q, torch.float64)
    for i, w in enumerate(list(enc) + list(dec)):
        assert tuple(w.shape) == ((B, 512, 512) if i < 6 else (B, Q, 512))
        assert (w >= 0).all() and (w.double().sum(-1) - 1).abs().max().item() < 1e-5, i
        err = (w.double() - ref[i]).abs().max().item()
        rel = ((w.double() - ref[i]).norm() / ref[i].norm()).item()
        assert err < MAP_ABS and rel < MAP_REL, (i, err, rel)
    del ref
    torch.cuda.empty_cache()


@pytest.mark.parametrize("path", [TC, SIMT], ids=["tc", "simt"])
def test_chunk_boundary_pairs_match_single_pair_decodes(native, path):
    """B = 40, Q = 1000: chunk 1 decodes pairs 32-39 at pair0 = 32 (on the tensor-core path it reads the key images at
    32 * img_pair_stride).  The maps of pairs on both sides of the boundary must be those of the pair decoded alone:
    a pair or base-offset error is O(1)."""
    _, nat, context = native
    B, Q = 40, 1000
    assert [c[:2] for c in _chunks(B, Q)] == [(0, 32), (32, 8)]
    img, q = _inputs(37, B, Q)
    ctx = context(path, img)
    nat.set_gemm_path(path)
    _, maps = nat.decode_attention(ctx, q, 0b111111)
    for p in (0, 30, 31, 32, 33, 39):
        one = context(path, img[p:p + 1].contiguous())
        _, alone = nat.decode_attention(one, q[p:p + 1].contiguous(), 0b111111)
        err = (maps[:, p] - alone[:, 0]).abs().max().item()
        assert err < PAIR_ABS, (p, err)


@pytest.mark.parametrize("path", [TC, SIMT], ids=["tc", "simt"])
@pytest.mark.parametrize("B,Q,mask", [(3, 12000, 0b100001), (40, 1000, 0b010110), (1, 40000, 0b000011)])
def test_decode_map_launches_follow_the_chunk_rule(native, path, B, Q, mask):
    """The profiler's maps launches of a decode_attention call are those of the chunk rule restated in _chunks: one
    per chunk and selected layer, M = the chunk's rows.  This keeps the kernel-level configurations above honest if
    the chunking changes."""
    _, nat, context = native
    img, q = _inputs(41, B, Q)
    ctx = context(path, img)
    nat.set_gemm_path(path)
    nat.profile_begin(8192)
    nat.decode_attention(ctx, q, mask)
    recs = [r[:4] for r in nat.profile_end() if r[0].startswith("attention_weights")]
    name = "attention_weights_tc" if path == TC else "attention_weights_simt"
    layers = [l for l in range(6) if (mask >> l) & 1]
    assert recs == [(name, npairs * nq, 512, 256) for _, npairs, nq in _chunks(B, Q) for _ in layers]
