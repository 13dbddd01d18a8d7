"""The COTR network as an nn.Module shell around the native sm_90a implementation.

Reference contract (COTR/models/cotr_model.py:17-51):
  * `build(args)` -> module with attributes transformer (.d_model), corr_embed, query_proj, input_proj, backbone;
  * `state_dict()` has the reference's 381 keys / shapes (SURVEY.md appendix C) so `utils.safe_load_weights`
    (COTR/utils/utils.py:164-193) loads a reference checkpoint with strict=True; FrozenBN statistics are buffers
    (backbone.py:31-34) and `num_batches_tracked` is dropped on load (backbone.py:38-40);
  * `forward(samples, queries) -> {'pred_corrs': (B,Q,2)}` on the module's device; samples is a (B,3,256,512) tensor,
    a list of (3,256,512) tensors or a NestedTensor; the canvas size is asserted like backbone.py:80.

The arithmetic is NOT done by torch: forward hands device pointers to libcotr_b200.so (include/cotr_b200.h).
There is no CPU path; calling forward without a CUDA device or without the built library raises.
Unlike the reference constructor (backbone.py:106 `pretrained=True`) nothing is downloaded.

Attention maps: the reference calls every transformer.encoder.layers[l].self_attn and
transformer.decoder.layers[l].multihead_attn with need_weights=True (transformer.py:149-153, :192-195), so a forward
hook on one of them sees the head-averaged attention weights as output[1].  Here those modules are parameter
containers that are never called, so `forward` looks for forward hooks (plain and with_kwargs) on them itself: when
there are any, it runs the native entry points that also compute the maps of exactly the hooked layers
(cotr_encode_context_attention / cotr_decode_attention) and then calls each hook as torch would, in the reference's
firing order (encoder layers 0..5, then decoder layers 0..5), with args = () (the reference passes only keywords),
kwargs = {} for with_kwargs hooks, and output = (None, weights): weights is (B, 512, 512) for an encoder layer and
(B, Q, 512) for a decoder layer, fp32 on the module's device; output[0], the attention output, is None because it is
never materialised.  A hook's return value is ignored.  `encode_context` fires the encoder hooks and `decode` the
decoder hooks, so a caller that encodes once and decodes twice (cotr_corr_base's cycle pass) sees the encoder hooks
fire once where the reference fires them twice.  Without hooks nothing of this runs.  Forward pre-hooks and the
sharded model are not covered, and a ragged `decode` (a list of per-pair query sets) refuses decoder hooks: it
produces no attention maps.
"""
import itertools
import math

import numpy as np
import torch
from torch import nn

from .. import capi
from .misc import NestedTensor, nested_tensor_from_tensor_list

MAX_SIZE = 256     # COTR/utils/constants.py:2
_BN_FIELDS = ("weight", "bias", "running_mean", "running_var")


class _Namespace(nn.Module):
    """A stateless container node of the module tree (children are added by name)."""

    def forward(self, *a, **k):   # pragma: no cover
        raise RuntimeError("this sub-module is a parameter container; call the COTR module itself")


class FrozenBatchNorm2d(_Namespace):
    """Parameter holder for backbone.py:21-56: statistics and affine terms are buffers, folded into the conv at pack time."""

    def __init__(self, n):
        super().__init__()
        self.register_buffer("weight", torch.ones(n))
        self.register_buffer("bias", torch.zeros(n))
        self.register_buffer("running_mean", torch.zeros(n))
        self.register_buffer("running_var", torch.ones(n))

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        state_dict.pop(prefix + 'num_batches_tracked', None)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)


class _Weight(_Namespace):
    def __init__(self, shape, bias=False, init="xavier"):
        super().__init__()
        w = torch.empty(*shape)
        if init == "kaiming":
            nn.init.kaiming_normal_(w, mode="fan_out", nonlinearity="relu")
        elif len(shape) >= 2:
            nn.init.xavier_uniform_(w.view(shape[0], -1))
        else:
            nn.init.ones_(w)
        self.weight = nn.Parameter(w, requires_grad=False)
        if bias:
            self.bias = nn.Parameter(torch.zeros(shape[0]), requires_grad=False)


class _MHA(_Namespace):
    def __init__(self, d):
        super().__init__()
        w = torch.empty(3 * d, d)
        nn.init.xavier_uniform_(w)
        self.in_proj_weight = nn.Parameter(w, requires_grad=False)
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * d), requires_grad=False)
        self.out_proj = _Weight((d, d), bias=True)


def _norm(d):
    m = _Namespace()
    m.weight = nn.Parameter(torch.ones(d), requires_grad=False)
    m.bias = nn.Parameter(torch.zeros(d), requires_grad=False)
    return m


def _bottleneck(inplanes, planes, downsample):
    b = _Namespace()
    b.conv1 = _Weight((planes, inplanes, 1, 1), init="kaiming"); b.bn1 = FrozenBatchNorm2d(planes)
    b.conv2 = _Weight((planes, planes, 3, 3), init="kaiming"); b.bn2 = FrozenBatchNorm2d(planes)
    b.conv3 = _Weight((planes * 4, planes, 1, 1), init="kaiming"); b.bn3 = FrozenBatchNorm2d(planes * 4)
    if downsample:
        ds = _Namespace()
        ds.add_module("0", _Weight((planes * 4, inplanes, 1, 1), init="kaiming"))
        ds.add_module("1", FrozenBatchNorm2d(planes * 4))
        b.downsample = ds
    return b


def _resnet50_layer3_body():
    """torchvision resnet50 up to layer3 (what IntermediateLayerGetter keeps, backbone.py:70-71), as a parameter tree."""
    body = _Namespace()
    body.conv1 = _Weight((64, 3, 7, 7), init="kaiming")
    body.bn1 = FrozenBatchNorm2d(64)
    inplanes = 64
    for name, n_blocks, planes in (("layer1", 3, 64), ("layer2", 4, 128), ("layer3", 6, 256)):
        layer = _Namespace()
        for i in range(n_blocks):
            layer.add_module(str(i), _bottleneck(inplanes, planes, downsample=(i == 0)))
            inplanes = planes * 4
        body.add_module(name, layer)
    return body


def _transformer(d, ff, n_enc, n_dec):
    t = _Namespace()
    t.d_model = d
    t.nhead = 8
    enc = _Namespace(); enc_layers = _Namespace()
    for l in range(n_enc):
        e = _Namespace()
        e.self_attn = _MHA(d)
        e.linear1 = _Weight((ff, d), bias=True); e.linear2 = _Weight((d, ff), bias=True)
        e.norm1 = _norm(d); e.norm2 = _norm(d)
        enc_layers.add_module(str(l), e)
    enc.layers = enc_layers
    dec = _Namespace(); dec_layers = _Namespace()
    for l in range(n_dec):
        e = _Namespace()
        e.multihead_attn = _MHA(d)
        e.linear1 = _Weight((ff, d), bias=True); e.linear2 = _Weight((d, ff), bias=True)
        e.norm1 = _norm(d)      # present in the checkpoint, never used (transformer.py:173 vs :185-201)
        e.norm2 = _norm(d); e.norm3 = _norm(d)
        dec_layers.add_module(str(l), e)
    dec.layers = dec_layers
    dec.norm = _norm(d)
    t.encoder = enc
    t.decoder = dec
    return t


class Context:
    """Encoded image pairs: the 6-layer decoder K/V cache living on the device (see cotr_encode_context)."""

    def __init__(self, native_ctx, batch):
        self.native = native_ctx
        self.batch = batch


class ImageFeatures:
    """Backbone features of N 256x256 images (see cotr_encode_images): `tensor` is (2, N, 256, 1024) float16 on the
    device, the layer3 output in the library's split16 storage (hi and lo planes; the value is hi + lo).  They belong to
    the weights of the model that made them: `generation` changes whenever that model's weights are repacked."""

    def __init__(self, tensor, n, generation):
        self.tensor = tensor
        self.n = n
        self.generation = generation


class KeypointMatches:
    """Per-pair results of COTR.match_keypoints, lists of B device tensors (views of the call's packed outputs):
    matches[p] (M_p,2) int64 (index into the keypoints of pairs[p][0], index into those of pairs[p][1]), in ascending
    first index; corrs_ab[p] (K_a,2) / corrs_ba[p] (K_b,2) fp64, where each keypoint of a lands in b / of b in a, in
    pixels; nearest_ab[p] (K_a,) / nearest_ba[p] (K_b,) int32, the nearest keypoint of the other image (-1 if it has
    none)."""

    def __init__(self, matches, corrs_ab, corrs_ba, nearest_ab, nearest_ba):
        self.matches = matches
        self.corrs_ab = corrs_ab
        self.corrs_ba = corrs_ba
        self.nearest_ab = nearest_ab
        self.nearest_ba = nearest_ba


_generations = itertools.count(1)      # process-wide, so that features never match another model's weights


class COTR(nn.Module):
    def __init__(self, args=None):
        super().__init__()
        cfg = dict(backbone="resnet50", hidden_dim=256, dilation=False, nheads=8, layer="layer3", enc_layers=6,
                   dec_layers=6, position_embedding="lin_sine", dim_feedforward=1024)
        if args is not None:
            for k, v in cfg.items():
                got = getattr(args, k, v)
                if got != v:
                    raise NotImplementedError(
                        f"cotr_b200 implements the configuration every reference demo uses ({k}={v!r}); got {k}={got!r}")
        d = cfg["hidden_dim"]
        self.transformer = _transformer(d, cfg["dim_feedforward"], 6, 6)
        head = _Namespace(); head.num_layers = 3
        layers = _Namespace()
        for i, shp in enumerate(((d, d), (d, d), (2, d))):
            layers.add_module(str(i), _Weight(shp, bias=True))
        head.layers = layers
        self.corr_embed = head
        self.query_proj = _Namespace()            # NerfPositionalEncoding(64): stateless
        self.input_proj = _Weight((d, 1024, 1, 1), bias=True)
        backbone = _Namespace()
        b0 = _Namespace(); b0.body = _resnet50_layer3_body(); b0.num_channels = 1024
        backbone.add_module("0", b0)
        backbone.add_module("1", _Namespace())    # PositionEmbeddingSine: stateless
        backbone.num_channels = 1024
        self.backbone = backbone
        self._native = None
        self._ctx_cache = {}
        self._hook_ctx = None                     # context of hooked forwards (grown to the largest batch seen)
        self._match_ctx = None                    # context of match_keypoints (grown to the largest 2B seen)
        self._generation = next(_generations)     # the weights ImageFeatures were made with

    # ---- native handle management ---------------------------------------------------------------------
    def _invalidate(self):
        self._generation = next(_generations)
        for ctx in self._ctx_cache.values():
            ctx.close()
        self._ctx_cache = {}
        for c in (self._hook_ctx, self._match_ctx):
            if c is not None:
                c.close()
        self._hook_ctx = self._match_ctx = None
        if self._native is not None:
            self._native.close()
        self._native = None

    def _apply(self, fn, *a, **k):                # .cuda() / .to() / .float(): weights move -> repack lazily
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, *a, **k):
        self._invalidate()
        return super().load_state_dict(state_dict, *a, **k)

    def refresh_native(self):
        """Call after editing parameters in place: the packed device copy is rebuilt on the next forward."""
        self._invalidate()

    def native(self):
        if self._native is None:
            dev = next(self.parameters()).device
            if dev.type != "cuda":
                raise RuntimeError("cotr_b200.COTR runs only on a CUDA device (sm_90a): call model.cuda() first; "
                                   "there is no CPU fallback")
            idx = dev.index if dev.index is not None else torch.cuda.current_device()
            self._native = capi.NativeModel(self.state_dict(), idx)
        return self._native

    # ---- reference API --------------------------------------------------------------------------------
    def _canvas(self, samples):
        if isinstance(samples, NestedTensor):
            x = samples.tensors
        elif isinstance(samples, (list, tuple, torch.Tensor)):
            x = nested_tensor_from_tensor_list(samples).tensors
        elif hasattr(samples, "tensors"):
            x = samples.tensors
        else:
            raise TypeError(f"unsupported samples type {type(samples)}")
        assert tuple(x.shape[-2:]) == (MAX_SIZE, MAX_SIZE * 2), f"canvas must be 256x512, got {tuple(x.shape[-2:])}"  # backbone.py:80
        assert x.ndim == 4 and x.shape[1] == 3
        dev = next(self.parameters()).device
        return x.to(device=dev, dtype=torch.float32).contiguous()

    def _queries(self, queries, batch):
        dev = next(self.parameters()).device
        q = queries.to(device=dev, dtype=torch.float32).contiguous()
        assert q.ndim == 3 and q.shape[-1] == 2 and q.shape[0] == batch, f"queries must be (B,Q,2), got {tuple(q.shape)}"
        return q

    # ---- forward hooks on the attention containers (see the module docstring) ---------------------------------
    def _attention_modules(self):
        t = self.transformer
        return ([getattr(t.encoder.layers, str(l)).self_attn for l in range(6)],
                [getattr(t.decoder.layers, str(l)).multihead_attn for l in range(6)])

    @staticmethod
    def _hooked(mods):
        """bit l set: module l has at least one forward hook"""
        return sum(1 << l for l, m in enumerate(mods) if m._forward_hooks)

    @staticmethod
    def _fire(mods, mask, maps):
        n = 0
        for l, m in enumerate(mods):
            if not (mask >> l) & 1:
                continue
            output = (None, maps[n])
            n += 1
            for hook_id, hook in list(m._forward_hooks.items()):
                if m._forward_hooks_with_kwargs.get(hook_id, False):
                    hook(m, (), {}, output)
                else:
                    hook(m, (), output)

    def _encode(self, x, native_ctx):
        nat = self.native()
        enc, _ = self._attention_modules()
        mask = self._hooked(enc)
        if not mask:
            nat.encode_context(x, native_ctx)
            return
        self._fire(enc, mask, nat.encode_context_attention(x, native_ctx, mask))

    def _decode(self, native_ctx, q):
        nat = self.native()
        _, dec = self._attention_modules()
        mask = self._hooked(dec)
        if not mask:
            return nat.decode(native_ctx, q)
        pred, maps = nat.decode_attention(native_ctx, q, mask)
        self._fire(dec, mask, maps)
        return pred

    @torch.no_grad()
    def forward(self, samples, queries):
        x = self._canvas(samples)
        q = self._queries(queries, x.shape[0])
        enc, dec = self._attention_modules()
        if not (self._hooked(enc) or self._hooked(dec)):
            return {'pred_corrs': self.native().forward(x, q)}
        if self._hook_ctx is None or self._hook_ctx.max_pairs < x.shape[0]:
            if self._hook_ctx is not None:
                self._hook_ctx.close()
            self._hook_ctx = capi.NativeContext(self.native(), x.shape[0])
        self._encode(x, self._hook_ctx)
        return {'pred_corrs': self._decode(self._hook_ctx, q)}

    # ---- extensions used by cotr_b200.inference ---------------------------------------------------------
    supports_device_preprocess = True

    @torch.no_grad()
    def preprocess_canvases(self, img_from_u8, img_to_u8, rects):
        """Device-side `RefinementTask.get_task` pixels: uint8 HWC CUDA images + (n,6) int32 rectangles
        [x_from, y_from, size_from, x_to, y_to, size_to] -> (n,3,256,512) normalised fp32 canvases, bit-identical to
        the PIL resize + to_tensor + normalize of the reference (cotr_preprocess in include/cotr_b200.h)."""
        assert img_from_u8.dtype == torch.uint8 and img_to_u8.dtype == torch.uint8
        assert img_from_u8.ndim == 3 and img_from_u8.shape[2] == 3 and img_to_u8.ndim == 3 and img_to_u8.shape[2] == 3
        return self.native().preprocess(img_from_u8.contiguous(), img_to_u8.contiguous(), rects)

    @torch.no_grad()
    def refine_walk(self, images, groups, zooms, batch, max_good, rel_threshold, loc_from, loc_to, wave=8):
        """The single-query zoom-in walk of SparseEngine (converge_iters = 1) on the device (cotr_refine).  images: uint8
        HWC CUDA tensors; groups: (image_from, image_to, first, count, s_from, s_to) per group, consecutive in task order;
        loc_from / loc_to: (n,2) source points and first guesses (converted to fp64).  Returns (history (n,L+1,2) fp64,
        rects (n,L,6) int32, good (n,) int32) as numpy arrays, the number of tasks walked and the (code, chunk, level)
        status (code 1: NaN prediction, 2: non-finite position)."""
        enc, dec = self._attention_modules()
        if self._hooked(enc) or self._hooked(dec):
            raise RuntimeError("refine_walk does not fire attention hooks: remove them or use the host loop")
        dev = next(self.parameters()).device
        images = [t.contiguous() for t in images]
        assert all(t.dtype == torch.uint8 and t.ndim == 3 and t.shape[2] == 3 and t.device == dev for t in images)
        lf = torch.as_tensor(np.asarray(loc_from, dtype=np.float64).reshape(-1, 2)).to(dev)
        lt = torch.as_tensor(np.asarray(loc_to, dtype=np.float64).reshape(-1, 2)).to(dev)
        history, rects, good, walked, status = self.native().refine(images, groups, zooms, batch, wave, max_good,
                                                                    rel_threshold, lf, lt)
        return history.cpu().numpy(), rects.cpu().numpy(), good.cpu().numpy(), walked, status

    def attention_hooked(self):
        """True when a forward hook sits on an attention module: the forward then fires it, the device walks cannot."""
        enc, dec = self._attention_modules()
        return bool(self._hooked(enc) or self._hooked(dec))

    @torch.no_grad()
    def refine_grouped_batch(self, img_from, img_to, s_from, s_to, zooms, level, ids, batch_size, max_load, max_good,
                             rel_threshold, walk):
        """One grouped batch of FasterSparseEngine's zoom-in on the device (cotr_refine_grouped).  img_*: uint8 HWC CUDA
        tensors; ids: the open tasks of `level` in shuffled order; walk: the device tensors the batches of one engine call
        share, {'loc_from': (n,2) fp64, 'history': (n,L+1,2) fp64 with row 0 the first guesses, 'rects': (n,L,6) int32,
        'good': (n+1,) int32 zeroed}.  Returns (squad (n_ids,) int32: the squad of each candidate or -1,
        (n_squads, longest, num_steps, stepped, status)); status 1 / 2: a pilot's crop raises (NaN / infinite position)."""
        if self.attention_hooked():
            raise RuntimeError("refine_grouped_batch does not fire attention hooks: remove them or use the host loop")
        return self.native().refine_grouped(img_from, img_to, s_from, s_to, zooms, level, ids, batch_size, max_load, max_good,
                                            rel_threshold, walk['loc_from'], walk['history'], walk['rects'], walk['good'])

    @torch.no_grad()
    def dense_postprocess(self, pred):
        """Device-side tail of the dense pass (inference_helper.py:131-145): (n,131072,2) predictions of the canvas grid
        queries -> (n,256,512,3) [x in the other image, y, cycle confidence] (cotr_dense_postprocess)."""
        assert pred.dtype == torch.float32 and pred.ndim == 3 and pred.shape[1] == 256 * 512 and pred.shape[2] == 2
        return self.native().dense_postprocess(pred)

    @torch.no_grad()
    def flow_tile_merge(self, tile, affine, patch, flow, conf, first):
        """Device-side `c @ A + t` -> `float_image_resize` -> `merge_flow_patches` step for one 256x256x3 tile answer
        (inference_helper.py:155-160, :61-75): see cotr_flow_tile_merge in include/cotr_b200.h."""
        self.native().flow_tile_merge(tile, affine, patch, flow, conf, first)

    @torch.no_grad()
    def resize_image(self, img_u8, size):
        """Device-side `PIL.Image.fromarray(img).resize((W', H'), BILINEAR)`: (H,W,3) uint8 CUDA image -> (H',W',3) uint8,
        bit for bit (cotr_resize_image in include/cotr_b200.h).  size = (H', W')."""
        return self.native().resize_image(img_u8, size)

    @torch.no_grad()
    def resize_maps(self, maps, size):
        """Device-side `utils.float_image_resize`: (H,W) or (H,W,C) fp32 CUDA maps, C = 1 .. 3 -> size = (H', W'), bit for
        bit (cotr_resize_maps in include/cotr_b200.h)."""
        return self.native().resize_maps(maps, size)

    def _context(self, batch, reuse):
        nat = self.native()
        if reuse:
            # one cached device K/V buffer per batch size: no cudaMalloc / device-synchronising cudaFree per call.
            # The returned Context is only valid until the next encode_context(reuse=True) of the same batch size.
            native_ctx = self._ctx_cache.get(batch)
            if native_ctx is None:
                if len(self._ctx_cache) >= 4:
                    for old in self._ctx_cache.values():
                        old.close()
                    self._ctx_cache = {}
                native_ctx = self._ctx_cache[batch] = capi.NativeContext(nat, batch)
        else:
            native_ctx = capi.NativeContext(nat, batch)
        return Context(native_ctx, batch)

    @torch.no_grad()
    def encode_context(self, samples, reuse=False):
        x = self._canvas(samples)
        ctx = self._context(x.shape[0], reuse)
        self._encode(x, ctx.native)
        return ctx

    @torch.no_grad()
    def encode_images(self, images):
        """Backbone features of (N,3,256,256) images, each normalised like one half of a canvas (cotr_encode_images).
        Encode a whole image set in one call: the library runs the backbone 64 images at a time."""
        assert isinstance(images, torch.Tensor) and images.ndim == 4 and tuple(images.shape[1:]) == (3, MAX_SIZE, MAX_SIZE), \
            f"images must be (N,3,256,256), got {tuple(getattr(images, 'shape', ()))}"
        dev = next(self.parameters()).device
        x = images.to(device=dev, dtype=torch.float32).contiguous()
        return ImageFeatures(self.native().encode_images(x), x.shape[0], self._generation)

    @torch.no_grad()
    def encode_context_pairs(self, features, pairs, reuse=False):
        """The Context of the canvases [image pairs[p][0] | image pairs[p][1]] from cached ImageFeatures; `pairs` is a
        (B,2) integer tensor, array or list.  `reuse` and the encoder attention hooks work as in encode_context."""
        p32 = self._pair_table("encode_context_pairs", features, pairs)
        ctx = self._context(p32.shape[0], reuse)
        nat = self.native()
        enc, _ = self._attention_modules()
        mask = self._hooked(enc)
        if not mask:
            nat.encode_context_pairs(features.tensor, p32, ctx.native)
        else:
            self._fire(enc, mask, nat.encode_context_pairs_attention(features.tensor, p32, ctx.native, mask))
        return ctx

    def _pair_table(self, fn, features, pairs):
        """Checks that `features` are current and `pairs` is a (B,2) integer table -> int32 numpy (B,2)."""
        if features.generation != self._generation:
            raise RuntimeError(f"{fn}: these ImageFeatures were made with other weights "
                               "(load_state_dict / .to() / refresh_native since): encode the images again")
        t = features.tensor
        dev = next(self.parameters()).device
        assert t.device == dev and t.dtype == torch.float16 and t.is_contiguous() and tuple(t.shape) == (2, features.n, 256, 1024), \
            f"features.tensor must be a contiguous (2,{features.n},256,1024) float16 tensor on {dev}"
        p = pairs.detach().cpu().numpy() if isinstance(pairs, torch.Tensor) else np.asarray(pairs)
        assert p.ndim == 2 and p.shape[1] == 2 and p.shape[0] >= 1 and p.dtype.kind in "iu", \
            f"pairs must be a non-empty (B,2) integer table, got shape {p.shape} dtype {p.dtype}"
        p32 = p.astype(np.int32)
        if not np.array_equal(p32, p):
            raise RuntimeError(f"{fn}: image index outside [0, {features.n})")
        return p32

    @torch.no_grad()
    def match_keypoints(self, features, pairs, keypoints, sizes):
        """Mutual nearest-neighbour matches of keypoints across image pairs, the rule of demo_guided_matching.py:48-62,
        on the device from cached ImageFeatures (cotr_match_keypoints).  Pair p decodes the keypoints of a = pairs[p][0]
        in the context [a | b] and those of b = pairs[p][1] in [b | a], with the whole image as the patch (no zoom-in),
        and keeps (i, j) when b's keypoint j is the nearest to where a's keypoint i lands and a's keypoint i the nearest
        to where j lands.  keypoints: N (K_i,2) tensors or arrays of (x, y) pixels of the original images (as DISK
        writes them); sizes: (N,2) original (W, H), each image having been resized whole to 256x256 for encode_images.
        -> KeypointMatches.  The call makes one device-to-host copy (the B match counts, to split the lists), so it
        waits for the device.  The decode is ragged, so registered attention hooks are refused (no maps are made)."""
        p32 = self._pair_table("match_keypoints", features, pairs)
        enc, dec = self._attention_modules()
        if self._hooked(enc) or self._hooked(dec):
            raise RuntimeError("match_keypoints: attention maps are not produced for matching (ragged decode); remove the "
                               "attention hooks")
        assert len(keypoints) == features.n, f"keypoints: {len(keypoints)} sets for {features.n} images"
        dev = next(self.parameters()).device
        kp = [torch.as_tensor(k, dtype=torch.float64, device=dev) for k in keypoints]    # nested lists too, without fp32
        for i, k in enumerate(kp):
            assert k.ndim == 2 and k.shape[1] == 2, f"keypoints: set {i} must be (K,2), got {tuple(k.shape)}"
        sz = sizes.detach().cpu().numpy() if isinstance(sizes, torch.Tensor) else np.asarray(sizes)
        assert sz.shape == (features.n, 2), f"sizes must be ({features.n},2) (W, H), got {sz.shape}"
        sz32 = sz.astype(np.int32)
        if not np.array_equal(sz32, sz):
            raise RuntimeError("match_keypoints: image sizes must be integers in [1, 65536]")
        counts = np.array([k.shape[0] for k in kp], dtype=np.int64)
        offsets = np.concatenate([[0], np.cumsum(counts)])
        B = p32.shape[0]
        if self._match_ctx is None or self._match_ctx.max_pairs < 2 * B:
            if self._match_ctx is not None:
                self._match_ctx.close()
            self._match_ctx = None
            self._match_ctx = capi.NativeContext(self.native(), 2 * B)
        packed = torch.cat(kp).contiguous()
        corr, nearest, match, count = self.native().match_keypoints(features.tensor, sz32, packed, offsets, p32, self._match_ctx)
        n_match = count.cpu().numpy()
        rows = counts[p32].reshape(-1)          # rows of contexts 0, 1, ..., 2B-1
        ctx_off = np.concatenate([[0], np.cumsum(rows)])
        match = match.long()
        res = KeypointMatches([], [], [], [], [])
        for p in range(B):
            ab, ba, end = int(ctx_off[2 * p]), int(ctx_off[2 * p + 1]), int(ctx_off[2 * p + 2])
            res.matches.append(match[ab:ab + int(n_match[p])])
            res.corrs_ab.append(corr[ab:ba]); res.corrs_ba.append(corr[ba:end])
            res.nearest_ab.append(nearest[ab:ba]); res.nearest_ba.append(nearest[ba:end])
        return res

    @torch.no_grad()
    def decode(self, ctx, queries):
        """queries: a (B,Q,2) tensor, or a list / tuple of B tensors (Q_p,2) with a count Q_p >= 0 per pair (ragged
        decode, cotr_decode_ragged); then pred_corrs is a list of B (Q_p,2) views of one packed output tensor."""
        if isinstance(queries, (list, tuple)):
            return {'pred_corrs': self._decode_ragged(ctx, queries)}
        q = self._queries(queries, ctx.batch)
        return {'pred_corrs': self._decode(ctx.native, q)}

    def _decode_ragged(self, ctx, queries):
        assert len(queries) == ctx.batch, f"ragged queries: {len(queries)} query sets for a context of {ctx.batch} pairs"
        for i, q in enumerate(queries):
            assert isinstance(q, torch.Tensor) and q.ndim == 2 and q.shape[1] == 2, \
                f"ragged queries: set {i} must be a (Q,2) tensor, got {tuple(getattr(q, 'shape', ()))}"
        _, dec = self._attention_modules()
        if self._hooked(dec):
            raise RuntimeError("decode: attention maps are not produced for ragged decodes (list of query sets); remove the "
                               "decoder attention hooks or decode a (B,Q,2) tensor")
        dev = next(self.parameters()).device
        counts = [int(q.shape[0]) for q in queries]
        packed = torch.cat([q.to(device=dev, dtype=torch.float32) for q in queries]).contiguous()
        offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        pred = self.native().decode_ragged(ctx.native, packed, offsets)
        return list(pred.split(counts))


def build(args):
    return COTR(args)
